"""F64 models of the FM demodulator, narrow and wideband (stereo), for the scan-kernel tests (test infrastructure).

Written from the reference's per-sample rules (src/domains/dsp/fm/module_impl_native_cpu.cc:43-175), not from
oracle/port.py: every filter is evaluated in F64 by scipy.signal.lfilter / sosfilt with its state carried between
calls, so millions of samples take well under a second. Only the coefficients are the plan's F32-rounded values
(FmImpl::updateCoefficients, module_impl.cc:108-155), widened to F64, so the model is the exact operation the
F32 implementations approximate.

Rules of the reference that the model keeps:
  - the first sample after reset demodulates to 0, whatever it is;
  - d[n] is NaN when x[n] or x[n-1] is non-finite, across call boundaries too;
  - a sample whose d is NaN emits NaN and leaves every filter state untouched (the wide pilot NCO still advances),
    so each lane's finite samples are compressed, filtered and scattered back;
  - wide: the difference-channel input uses the pilot states AFTER this sample's update.
The wide pilot NCO phase is the F32 sequence of b200_fm_nco_phases_host (the plan's host twin, checked against a
serial F32 walk in tests/test_index_algebra.py).

`check_rule` is the tolerance used against the GPU: the reference's own F32 error against the model calibrates it.
"""
from __future__ import annotations

import ctypes

import numpy as np
from scipy.signal import lfilter, sosfilt

F32 = np.float32
JST_PI = 3.14159265358979323846


def coefficients(rate: float, wide: bool, deemphasis_us: int) -> dict:
    """The plan's F32 coefficients (b200_fm_plan_create, restating FmImpl::updateCoefficients) as Python floats."""
    sr = float(F32(rate))
    kf = F32(F32(75e3 if wide else 100e3) / F32(rate))
    c = dict(ref=float(F32(1.0 / (2.0 * JST_PI * float(kf)))))
    c["alpha"] = float(F32(1.0 - np.exp(-1.0 / (sr * deemphasis_us * 1e-6)))) if deemphasis_us else None
    if wide:
        c["pilot_alpha"] = float(F32(1.0 - np.exp(-2.0 * JST_PI * 200.0 / sr)))
        w = 2.0 * JST_PI * 19e3 / sr
        na = np.sin(w) / (2.0 * 20.0)
        b0, b1 = float(F32(1.0 / (1.0 + na))), float(F32(-2.0 * np.cos(w) / (1.0 + na)))
        sos = [[b0, b1, b0, 1.0, b1, float(F32((1.0 - na) / (1.0 + na)))]]
        w = 2.0 * JST_PI * 15e3 / sr
        for q in (0.51763809, 0.70710678, 1.93185165):
            al = np.sin(w) / (2.0 * q)
            lb0 = float(F32((1.0 - np.cos(w)) * 0.5 / (1.0 + al)))
            sos.append([lb0, float(F32((1.0 - np.cos(w)) / (1.0 + al))), lb0, 1.0,
                        float(F32(-2.0 * np.cos(w) / (1.0 + al))), float(F32((1.0 - al) / (1.0 + al)))])
        c["sos"] = np.array(sos)          # notch, LP0, LP1, LP2: [b0 b1 b2 1 a1 a2] (transposed DF-II in sosfilt)
    return c


def nco_phases(rate: float, n0: int, count: int) -> np.ndarray:
    """Pilot NCO phase of samples n0 .. n0 + count - 1 after reset (F32), from the plan's host twin."""
    from cyberether_b200 import _native
    lib = _native.load()
    out = np.empty(count, np.float32)
    _native.check(lib.b200_fm_nco_phases_host(float(rate), int(n0), int(count), out.ctypes.data_as(ctypes.c_void_p),
                                              None, None))
    return out


def nco_orbit(rate: float):
    """(pre, cycle) of the pilot NCO orbit: sample n >= pre has the phase of sample pre + (n - pre) mod cycle."""
    from cyberether_b200 import _native
    lib = _native.load()
    pre, cycle = ctypes.c_uint64(), ctypes.c_uint64()
    _native.check(lib.b200_fm_nco_phases_host(float(rate), 0, 0, None, ctypes.byref(pre), ctypes.byref(cycle)))
    return pre.value, cycle.value


def _one_pole(alpha, x, y_prev):
    """y += alpha (x - y) in F64 from the state y_prev; returns (y, last y)."""
    if x.size == 0:
        return x, y_prev
    y, zf = lfilter([alpha], [1.0, alpha - 1.0], x, zi=[(1.0 - alpha) * y_prev])
    return y, y[-1]


class _Discriminator:
    """d[n] = atan2(pr ci - pi cr, pr cr + pi ci) * ref over the F32 inputs, products and sums in F64 in that order
    (so a zero keeps the sign the F32 evaluation gives it); 0 for the first sample after reset; NaN when x[n] or
    x[n-1] is non-finite."""

    def __init__(self, ref, lanes):
        self.ref = ref
        self.prev = np.zeros(lanes, np.complex64)
        self.has_prev = np.zeros(lanes, bool)

    def __call__(self, streams):
        """streams: [lanes, n] complex64 (time order per lane) -> [lanes, n] F64."""
        prev = np.concatenate([self.prev[:, None], streams[:, :-1]], axis=1)
        pr, pi = prev.real.astype(np.float64), prev.imag.astype(np.float64)
        cr, ci = streams.real.astype(np.float64), streams.imag.astype(np.float64)
        with np.errstate(invalid="ignore", over="ignore"):
            re = pr * cr + pi * ci
            im = pr * ci - pi * cr
            d = np.arctan2(im, re) * self.ref
        d[~(np.isfinite(prev) & np.isfinite(streams))] = np.nan
        d[~self.has_prev, 0] = 0.0
        self.prev = streams[:, -1].copy()
        self.has_prev[:] = True
        return d


def _lanes_of(x):
    """[frames, lanes, frame_len] -> [lanes, frames * frame_len] (time order per lane)."""
    frames, lanes, n = x.shape
    return np.ascontiguousarray(np.asarray(x, np.complex64).transpose(1, 0, 2).reshape(lanes, frames * n))


class NarrowModel:
    """Narrow mode: discriminator, optional one-pole de-emphasis y += alpha (d - y). Call with [frames, lanes,
    frame_len] complex64; returns [lanes, frames * frame_len] F64."""

    def __init__(self, rate, deemphasis_us, lanes):
        c = coefficients(rate, False, deemphasis_us)
        self.alpha = c["alpha"]
        self.disc = _Discriminator(c["ref"], lanes)
        self.y = np.zeros(lanes)

    def __call__(self, x):
        d = self.disc(_lanes_of(x))
        if self.alpha is not None:
            for lane in range(d.shape[0]):
                keep = np.isfinite(d[lane])
                d[lane, keep], self.y[lane] = _one_pole(self.alpha, d[lane, keep], self.y[lane])
        return d


class WideModel:
    """Wideband (stereo) mode. Call with [frames, lanes, frame_len] complex64; returns [lanes, frames * frame_len, 2]
    F64 (left, right)."""

    def __init__(self, rate, deemphasis_us, lanes):
        c = coefficients(rate, True, deemphasis_us)
        self.rate, self.c = rate, c
        self.disc = _Discriminator(c["ref"], lanes)
        self.n = 0                                       # samples since reset: the NCO position
        self.pilot = np.zeros((lanes, 4))                # cos stage, sin stage, pilotCos, pilotSin
        self.zsum = np.zeros((lanes, 4, 2))
        self.zdiff = np.zeros((lanes, 4, 2))
        self.lr = np.zeros((lanes, 2))

    def __call__(self, x):
        c = self.c
        d = self.disc(_lanes_of(x))
        lanes, n = d.shape
        phase = nco_phases(self.rate, self.n, n).astype(np.float64)
        self.n += n
        out = np.full((lanes, n, 2), np.nan)
        a = c["pilot_alpha"]
        for lane in range(lanes):
            keep = np.isfinite(d[lane])
            v, ph = d[lane, keep], phase[keep]
            if v.size == 0:
                continue
            st = self.pilot[lane]
            cs, st[0] = _one_pole(a, v * np.cos(ph), st[0])
            ss, st[1] = _one_pole(a, v * np.sin(ph), st[1])
            pc, st[2] = _one_pole(a, cs, st[2])
            ps, st[3] = _one_pole(a, ss, st[3])
            diff_in = 2.0 * v * np.sin(2.0 * (ph + np.arctan2(pc, ps)))
            total, self.zsum[lane] = sosfilt(c["sos"], v, zi=self.zsum[lane])
            diff, self.zdiff[lane] = sosfilt(c["sos"], diff_in, zi=self.zdiff[lane])
            left, right = total + diff, total - diff
            if c["alpha"] is not None:
                left, self.lr[lane, 0] = _one_pole(c["alpha"], left, self.lr[lane, 0])
                right, self.lr[lane, 1] = _one_pole(c["alpha"], right, self.lr[lane, 1])
            out[lane, keep, 0], out[lane, keep, 1] = left, right
        return out


def check_rule(got, ref, model, label=""):
    """The tolerance of the FM scan tests, per output channel over the finite samples:
        e_ref = max|ref - model|,  e_got = max|got - model|,  e_got <= 2 e_ref + 4 2^-24 max|model|
    i.e. `got` may deviate from the F64 model by twice what the reference's own serial F32 evaluation does, plus a few
    ulps of the output scale. The NaN masks of all three must agree. Arrays: [..., n] or [..., n, 2] (channel last
    for wide). Returns [(e_got, e_ref, bound)] per channel."""
    got, ref, model = (np.asarray(a, np.float64) for a in (got, ref, model))
    assert got.shape == ref.shape == model.shape, (label, got.shape, ref.shape, model.shape)
    nan = np.isnan(model)
    assert np.array_equal(np.isnan(ref), nan), f"{label}: reference and model NaN masks differ"
    bad = np.flatnonzero(np.isnan(got).ravel() != nan.ravel())
    assert bad.size == 0, f"{label}: NaN mask differs at {bad.size} elements, first flat index {bad[:5]}"
    channels = [(got, ref, model)] if model.ndim < 3 else [(got[..., k], ref[..., k], model[..., k])
                                                           for k in range(model.shape[-1])]
    out = []
    for k, (g, r, m) in enumerate(channels):
        fin = ~np.isnan(m)
        if not fin.any():
            continue
        e_ref = float(np.abs(r[fin] - m[fin]).max())
        err = np.where(fin, np.abs(g - m), 0.0)
        e_got = float(err.max())
        bound = 2.0 * e_ref + 4.0 * 2.0 ** -24 * float(np.abs(m[fin]).max())
        where = np.unravel_index(int(err.argmax()), err.shape)
        assert e_got <= bound, (f"{label} channel {k}: e_gpu {e_got:.3e} > 2 e_ref + 4 ulp = {bound:.3e} "
                                f"(e_ref {e_ref:.3e}, max|model| {np.abs(m[fin]).max():.3e}); worst at {where}")
        out.append((e_got, e_ref, bound))
    return out
