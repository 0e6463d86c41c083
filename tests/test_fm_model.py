"""The F64 FM models of tests/fm_model.py against the reference and oracle/port.py's F32 restatement (no GPU).

The GPU scan tests (tests/test_gpu_fm_scans.py) charge the kernels against these models, calibrated by the
reference's own error. This checks that rule with the port in the GPU's place: on streams with NaN runs, exact and
signed zeros and split calls, two independent F32 evaluations must sit within F32 noise of the model. A model that
dropped a rule of the reference (first sample 0, NaN across a call boundary, frozen state over skipped samples, the
pilot states after the update) would be off by far more than that.
"""
import numpy as np
import pytest

from fm_model import NarrowModel, WideModel, check_rule
from oracle import port

DEEMPHASIS = {0: "none", 50: "50us", 75: "75us"}


def _stream(lanes, n, rate, wide, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(n) / rate
    out = np.empty((lanes, n), np.complex64)
    for lane in range(lanes):
        if wide:
            left, right = np.sin(2 * np.pi * 1e3 * t + lane), 0.5 * np.sin(2 * np.pi * 3e3 * t)
            pilot = 2 * np.pi * 19e3 * t
            mpx = 0.4 * (left + right) + 0.1 * np.sin(pilot) + 0.4 * (left - right) * np.sin(2 * pilot)
            phase = 2 * np.pi * 75e3 * np.cumsum(mpx) / rate
            noise = 0.002
        else:
            phase = 20.0 * np.sin(2 * np.pi * 1e3 * t + lane)
            noise = 0.01
        out[lane] = np.exp(1j * phase) + noise * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    out[0, 0] = np.nan                                     # the first sample after reset still gives 0
    out[0, 100:117] = np.nan
    out[1, 999] = np.inf                                   # last sample of a call: the next call's first d is NaN
    out[1, 1500:1504] = [0, complex(-0.0, 0.0), complex(0.0, -0.0), -1]
    out[0, 2000:2003] = complex(-0.0, -0.0)
    out[0, 2500:2500 + 300] = np.nan
    return out


def _reference(stream, rate, wide, deemphasis_us):
    from oracle import ref
    with ref.Session() as s:
        s.add_source("src", np.ascontiguousarray(stream), 1, -1, -1)
        s.add_block("fm", "fm", {"mode": "wide" if wide else "narrow", "deemphasis": DEEMPHASIS[deemphasis_us],
                                 "sampleRate": rate}, {"signal": "src.signal"})
        s.compute()
        return s.output("fm", "signal")


@pytest.mark.parametrize("deemphasis_us", [0, 75])
@pytest.mark.parametrize("rate", [250e3, 20e6])
@pytest.mark.parametrize("wide", [False, True])
def test_fm_models_match_the_port_and_the_reference(ref, wide, rate, deemphasis_us):
    lanes, n = 2, 3000
    x = _stream(lanes, n, rate, wide, 7)
    splits = [0, 1000, 1001, 2501, n]
    model = (WideModel if wide else NarrowModel)(rate, deemphasis_us, lanes)
    ported = (port.FmWide if wide else port.FmNarrow)(rate, DEEMPHASIS[deemphasis_us], lanes)
    got, want = [], []
    for a, b in zip(splits[:-1], splits[1:]):
        part = x[:, a:b][None]
        want.append(model(part))
        got.append(np.moveaxis(ported(part), 0, 1).reshape(want[-1].shape))
    got, want = np.concatenate(got, axis=1), np.concatenate(want, axis=1)
    reference = _reference(x, rate, wide, deemphasis_us)
    assert np.all(want[0, 0] == 0) and np.isnan(want[0, 1]).all() and np.isnan(want[1, 1000]).all()
    assert np.isnan(want[0, 2500:2801]).all() and not np.isnan(want[0, 2801:]).any()
    check_rule(got, reference, want, f"port {'wide' if wide else 'narrow'} {rate:g} Hz de={deemphasis_us}")
