"""The FM demodulator's scan kernels (fm.cu) at every carry boundary, against the F64 models of tests/fm_model.py.

Both modes carry state across tiles, lanes and calls:
  - narrow: fm_narrow_fused_kernel, one pass with a decoupled look-back over 2048-sample tiles; a tile of non-finite
    samples has gain 1, so the look-back must pass through it;
  - wide (stereo): three blocked scans (pilot S = 4, audio S = 8 over 2 lanes per lane, stereo S = 2), each a
    scan_tile / scan_tiles / scan_replay triple over 4096-sample tiles, carries composed with tables of A^(2^k); the
    pilot NCO phase comes from the plan's orbit table, folded at pre + (n - pre) mod cycle.

The plans are driven through the C ABI so one plan sees calls of different sizes. Every case feeds the GPU a stream
in calls and compares the concatenated output with ONE reference run (the serial F32 reference) over the whole stream
and with the F64 model, by fm_model.check_rule:
    e_gpu = max|gpu - model| <= 2 max|ref - model| + 4 2^-24 max|model|,   NaN masks identical,
per case and output channel. The reference's own F32 error calibrates the bound, so the same rule holds at 200 kHz and
at 20 MHz. Wide inputs carry a 19 kHz pilot (without one atan2(pilotCos, pilotSin) is ill-conditioned and no two F32
evaluations of the difference channel agree).
"""
import ctypes
import time

import numpy as np
import pytest

from fm_model import NarrowModel, WideModel, check_rule, coefficients, nco_orbit, nco_phases

pytestmark = pytest.mark.gpu

DEEMPHASIS = {0: "none", 50: "50us", 75: "75us"}
TILE_WIDE = 4096          # kScanTile
TILE_NARROW = 2048        # kFmTile


class _Plan:
    def __init__(self, lanes, rate, wide, deemphasis_us):
        import torch
        from cyberether_b200 import _native
        from cyberether_b200.jetstream import Context
        self.torch, self.native, self.lib = torch, _native, _native.load()
        self.dev = torch.device("cuda", torch.cuda.current_device())
        self.ctx = Context.get(self.dev)
        self.lanes, self.wide = lanes, wide
        self.handle = ctypes.c_void_p()
        self.native.check(self.lib.b200_fm_plan_create(self.ctx.handle, lanes, rate, int(wide), deemphasis_us,
                                                       ctypes.byref(self.handle)))
        self.stream = ctypes.c_void_p(torch.cuda.current_stream(self.dev).cuda_stream)

    def exec(self, x):
        """x: [frames, lanes, frame_len] complex64 (numpy) -> output on the GPU, [frames, lanes, frame_len(, 2)]."""
        torch = self.torch
        frames, lanes, n = x.shape
        xt = torch.from_numpy(np.ascontiguousarray(x)).to(self.dev)
        y = torch.empty((frames, lanes, n) + ((2,) if self.wide else ()), dtype=torch.float32, device=self.dev)
        self.native.check(self.lib.b200_fm_exec(self.handle, xt.data_ptr(), y.data_ptr(), frames, n, self.stream))
        return y

    def reset(self):
        self.native.check(self.lib.b200_fm_reset(self.handle, self.stream))

    def nco_phases(self, n0, count):
        y = self.torch.empty(count, dtype=self.torch.float32, device=self.dev)
        self.native.check(self.lib.b200_fm_nco_phases(self.handle, n0, count, y.data_ptr(), self.stream))
        return y.cpu().numpy()

    def close(self):
        self.native.check(self.lib.b200_fm_plan_destroy(self.handle))

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


def _feed(plan, stream, calls):
    """Feed stream [lanes, N] in calls [(frames, frame_len)] that cover it in order; returns [lanes, N(, 2)] F32."""
    lanes, total = stream.shape
    assert sum(f * n for f, n in calls) == total, (calls, total)
    outs, pos = [], 0
    for frames, n in calls:
        seg = stream[:, pos:pos + frames * n]
        pos += frames * n
        y = plan.exec(seg.reshape(lanes, frames, n).transpose(1, 0, 2)).cpu().numpy()
        outs.append(np.moveaxis(y, 0, 1).reshape((lanes, frames * n) + y.shape[3:]))
    return np.concatenate(outs, axis=1)


def _reference(stream, rate, wide, deemphasis_us):
    """One run of the reference over the whole stream [lanes, N] (lanes as a plain axis, no batch)."""
    from oracle import ref
    with ref.Session() as s:
        s.add_source("src", np.ascontiguousarray(stream), 1, -1, -1)
        s.add_block("fm", "fm", {"mode": "wide" if wide else "narrow", "deemphasis": DEEMPHASIS[deemphasis_us],
                                 "sampleRate": rate}, {"signal": "src.signal"})
        s.compute()
        return s.output("fm", "signal")


def _model(stream, rate, wide, deemphasis_us):
    m = (WideModel if wide else NarrowModel)(rate, deemphasis_us, stream.shape[0])
    return m(stream[None])


def _case(label, stream, rate, wide, deemphasis_us, calls, reset_at=None):
    """GPU (in `calls`, with b200_fm_reset before call index `reset_at`) vs one reference run and the model per
    segment between resets. Prints e_gpu / e_ref per channel and the wall time."""
    t0 = time.perf_counter()
    bounds = [0, len(calls)] if reset_at is None else [0, reset_at, len(calls)]
    lanes = stream.shape[0]
    got, want, model = [], [], []
    with _Plan(lanes, rate, wide, deemphasis_us) as plan:
        pos = 0
        for a, b in zip(bounds[:-1], bounds[1:]):
            if a > 0:
                plan.reset()
            part = calls[a:b]
            seg = stream[:, pos:pos + sum(f * n for f, n in part)]
            pos += seg.shape[1]
            got.append(_feed(plan, seg, part))
            want.append(_reference(seg, rate, wide, deemphasis_us))
            model.append(_model(seg, rate, wide, deemphasis_us))
    got, want, model = (np.concatenate(v, axis=1) for v in (got, want, model))
    res = check_rule(got, want, model, label)
    print(f"\n[fm-scan] {label}: " + ", ".join(f"ch{k} e_gpu/e_ref = {g:.3e}/{r:.3e} = {g / r if r else 0:.2f}"
                                             for k, (g, r, _) in enumerate(res))
          + f"; {lanes} x {stream.shape[1]} samples, {time.perf_counter() - t0:.2f} s")
    return got, want, model


def _mpx(lanes, n, rate, seed, quadrature=0.0):
    """[lanes, n] wideband FM of a stereo multiplex: (L+R), a 19 kHz pilot, (L-R) on a 38 kHz DSB-SC subcarrier locked to
    the pilot (plus `quadrature` times a 38 kHz component in quadrature to it), +-75 kHz deviation, small noise. Every
    lane has its own tones."""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / rate
    out = np.empty((lanes, n), np.complex64)
    for lane in range(lanes):
        f = 1e3 * (1 + 0.37 * lane)
        left, right = np.sin(2 * np.pi * f * t + lane), 0.5 * np.sin(2 * np.pi * 2.3 * f * t)
        pilot = 2 * np.pi * 19e3 * t + 0.1 * lane
        mpx = (0.4 * (left + right) + 0.1 * np.sin(pilot) + 0.4 * (left - right) * np.sin(2 * pilot)
               + quadrature * np.cos(2 * pilot))
        phase = 2 * np.pi * 75e3 * np.cumsum(mpx) / rate
        out[lane] = np.exp(1j * phase) + 0.002 * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    return out


def _narrow_fm(lanes, n, rate, seed):
    """[lanes, n] unit-magnitude FM (20 kHz deviation) plus small noise; a few exact zeros per lane."""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / rate
    out = np.empty((lanes, n), np.complex64)
    for lane in range(lanes):
        phase = 20.0 * (1 + 0.3 * lane) * np.sin(2 * np.pi * 1e3 * t + lane)
        out[lane] = np.exp(1j * phase) + 0.01 * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
        out[lane, rng.integers(1, n, 8)] = 0
    return out


# ---------------------------------------------------------------------------------------------------------------------
# wideband
# ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("deemphasis_us", [0, 50, 75])
@pytest.mark.parametrize("lanes,calls", [(3, [(4, 4100), (2, 8193), (5, 3001)]),
                                         (5, [(3, 5461), (1, 16383), (7, 2339)])])
def test_wide_lanes_and_frames_across_tiles(ref, lanes, calls, deemphasis_us):
    """Several lanes (LaneIndex, the audio scan's two virtual lanes per lane), frames of lengths that are no multiple of
    the 4096-sample tile, so frames and tiles cross, and carries over three calls of about 16 k samples per lane."""
    n = sum(f * m for f, m in calls)
    _case(f"wide lanes={lanes} de={deemphasis_us}", _mpx(lanes, n, 250e3, 10 + lanes), 250e3, True, deemphasis_us,
          calls)


@pytest.mark.parametrize("deemphasis_us", [0, 50, 75])
def test_wide_tile_batches_of_32(ref, deemphasis_us):
    """scan_tiles_kernel composes a lane's tiles 32 at a time: 70 * 4096 + 1234 samples are batches of 32, 32 and 7
    tiles; then 33 * 4096 are a batch of 32 and a batch of 1."""
    calls = [(1, 70 * TILE_WIDE + 1234), (33, TILE_WIDE)]
    n = sum(f * m for f, m in calls)
    _case(f"wide 32-tile batches de={deemphasis_us}", _mpx(1, n, 250e3, 20), 250e3, True, deemphasis_us, calls)


def test_wide_more_tiles_and_lanes_than_the_grid(ref):
    """600 lanes x 8292 samples: every scan has more tiles than its grid (sms * 8 CTAs), and the audio scan's 1200
    virtual lanes exceed the grid of scan_tiles_kernel, so all three kernels loop; a second call checks the carried
    lane states of lanes the loop reached on its later turns."""
    import torch
    sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    lanes, calls = 600, [(2, 4146), (1, 1000)]
    assert 2 * lanes > sms * 8 and lanes * 3 > sms * 8
    n = sum(f * m for f, m in calls)
    _case("wide 600 lanes", _mpx(lanes, n, 250e3, 30), 250e3, True, 75, calls)


def _nan_runs(stream, starts_lengths, value=np.nan):
    for start, length in starts_lengths:
        stream[:, start:start + length] = value


@pytest.mark.parametrize("deemphasis_us", [0, 50, 75])
def test_wide_nan_runs_at_thread_tile_and_call_boundaries(ref, deemphasis_us):
    """Runs of non-finite input (a run of k samples skips k + 1 discriminator outputs) of 1, 16, 17, 4095, 4097 and
    3 * 4096 + 5 samples placed on 16-sample thread chunks, on whole 4096-sample tiles (m = 0) and across calls; NaN as
    the last sample of one call and the first of the next; a stream that starts with a non-finite sample."""
    lanes, calls = 2, [(1, 20000), (2, 15000), (7, 10000)]
    n = sum(f * m for f, m in calls)
    x = _mpx(lanes, n, 250e3, 40)
    _nan_runs(x, [(1599, 1), (3200, 16), (4096 + 80 + 3, 17), (2 * TILE_WIDE, 4095), (19999, 2),
                  (7 * TILE_WIDE - 1, 4097), (10 * TILE_WIDE + 1000, 3 * TILE_WIDE + 5), (48000, 4097)])
    _nan_runs(x[1:], [(0, 1), (60001, 33), (81920, 4095)], np.inf)
    x[0, 100000] = complex(np.nan, 0.0)
    x[1, 100001] = complex(0.0, -np.inf)
    _case(f"wide NaN runs de={deemphasis_us}", x, 250e3, True, deemphasis_us, calls)


@pytest.mark.parametrize("rate,total,deemphasis_us", [(2.4e6, 4_000_000, 75), (1.024e6, 6_450_000, 50)])
def test_wide_pilot_nco_fold_on_the_device(ref, rate, total, deemphasis_us):
    """The pilot NCO phase of sample n >= pre is the orbit table's entry pre + (n - pre) mod cycle
    (fm_wide_phase_table_kernel, positioned by the plan's count of samples since reset). Irregular calls, one of them
    straddling the first folded sample pre + cycle: 3 294 318 at 2.4 MHz (short transient), 6 404 691 at 1.024 MHz
    (long transient). A 38 kHz component in quadrature to the stereo subcarrier makes the difference channel sensitive
    to the pilot phase itself."""
    pre, cycle = nco_orbit(rate)
    fold = pre + cycle
    assert fold < total
    rng = np.random.default_rng(int(rate))
    calls, pos = [], 0
    while pos < total:
        frames = int(rng.choice([1, 2, 3]))
        n = int(rng.integers(150_000, 450_000)) // frames
        if pos < fold < pos + frames * n:
            assert pos + 1000 < fold < pos + frames * n - 1000
        n = min(n, (total - pos) // frames) if pos + frames * n > total else n
        if n == 0:
            frames, n = 1, total - pos
        calls.append((frames, n))
        pos += frames * n
    starts = np.cumsum([0] + [f * m for f, m in calls])
    assert any(a < fold < b for a, b in zip(starts[:-1], starts[1:])), "no call straddles the fold"
    _case(f"wide NCO fold {rate / 1e6:g} MHz (pre {pre}, cycle {cycle})", _mpx(1, total, rate, 50, quadrature=0.3),
          rate, True, deemphasis_us, calls)


@pytest.mark.parametrize("rate", [240e3, 1.024e6, 2.4e6, 20e6])
def test_wide_device_nco_phases_fold_bit_exact(rate):
    """fm_wide_phase_table_kernel (the kernel b200_fm_exec takes its phases from) against the host twin of the orbit
    bookkeeping, bit for bit, in the transient, across the first folded sample pre + cycle, several periods later and
    far out. A wrong fold moves the phase by only a few ulps (the transient and the period differ that little), far
    below what the demodulated output can show, so the phases are checked directly."""
    pre, cycle = nco_orbit(rate)
    count = 20000
    with _Plan(1, rate, True, 0) as plan:
        for n0 in (0, max(pre, 5000) - 5000, cycle - 7000, pre + cycle - 9999, pre + 3 * cycle + 12345, 10 ** 12 + 3):
            got, want = plan.nco_phases(n0, count), nco_phases(rate, n0, count)
            bad = np.flatnonzero(got != want)
            assert bad.size == 0, f"{rate:g} Hz: {bad.size} phases differ from sample {n0 + bad[0]} on (pre {pre}, cycle {cycle})"


def test_wide_reset_mid_stream(ref):
    """b200_fm_reset between calls: every filter state, the previous sample and the NCO position start over, as in a
    fresh reference run."""
    calls = [(1, 30000), (3, 7001), (2, 9000), (1, 50000)]
    n = sum(f * m for f, m in calls)
    _case("wide reset mid-stream", _mpx(2, n, 250e3, 60), 250e3, True, 50, calls, reset_at=2)


def test_wide_scratch_regrowth_and_split_calls(ref):
    """Call sizes grow, shrink and grow on one plan (the scratch is reallocated only when a call needs more); the same
    stream in one call meets the rule too."""
    calls = [(1, 5000), (3, 50000), (1, 3000), (2, 20000), (4, 75000)]
    n = sum(f * m for f, m in calls)
    x = _mpx(2, n, 250e3, 70)
    _case("wide regrowth, split", x, 250e3, True, 0, calls)
    _case("wide regrowth, one call", x, 250e3, True, 0, [(1, n)])


@pytest.mark.parametrize("deemphasis_us", [0, 75])
@pytest.mark.parametrize("rate", [200e3, 250e3, 2.4e6, 20e6])
def test_wide_sample_rates_module_edges(ref, rate, deemphasis_us):
    """The module's edges: 200 kHz (the lowest wide rate) to 20 MHz (the highest), where the pilot and notch poles sit
    within ~1e-4 of the unit circle and the F32 power tables are least accurate."""
    calls = [(2, 30011), (1, 77777), (5, 20000)]
    n = sum(f * m for f, m in calls)
    _case(f"wide {rate / 1e6:g} MHz de={deemphasis_us}", _mpx(2, n, rate, 80), rate, True, deemphasis_us, calls)


# ---------------------------------------------------------------------------------------------------------------------
# narrow
# ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("deemphasis_us", [0, 75])
@pytest.mark.parametrize("rate", [250e3, 20e6])
def test_narrow_dropouts_longer_than_the_look_back(ref, rate, deemphasis_us):
    """Dropouts of 1.5 tiles and of 40 tiles (2048-sample tiles): the tiles inside have gain 1, so the look-back crosses
    them in its first round and in later rounds. At 250 kHz the first round looks at 1 tile, at 20 MHz at 16. Lane 2's
    40-tile dropout lies wholly inside the second call (one 60-tile frame), so within one launch the tile after it may
    have to look back past 40 gain-1 tiles (more than one 32-tile round); lane 1's spans the boundary of the first two
    calls."""
    lanes, calls = 3, [(2, 61440), (1, 122880), (3, 40000)]
    n = sum(f * m for f, m in calls)
    x = _narrow_fm(lanes, n, rate, 90)
    x[0, 5 * TILE_NARROW + 1000:5 * TILE_NARROW + 1000 + 3 * TILE_NARROW // 2] = np.nan
    x[1, 30 * TILE_NARROW + 7:70 * TILE_NARROW + 7] = np.nan
    x[2, 127880:127880 + 40 * TILE_NARROW] = np.nan                   # inside call 2: [122880, 245760)
    x[2, 250000:250000 + 3 * TILE_NARROW // 2] = np.nan
    _case(f"narrow dropouts {rate / 1e6:g} MHz de={deemphasis_us}", x, rate, False, deemphasis_us, calls)


@pytest.mark.parametrize("rate,deemphasis_us", [(500.0, 50), (500.0, 75), (700.0, 75), (1000.0, 50)])
def test_narrow_deemphasis_where_alpha_rounds_to_one(ref, rate, deemphasis_us):
    """Narrow mode has no minimum rate. Below ~0.77 kHz (75 us) or ~1.15 kHz (50 us) the de-emphasis alpha rounds to
    1.0f, so the gain (1 - alpha)^c is 1 for c = 0 and 0 for every c >= 1: the scan's identity maps and look-back must
    still compose to the reference's output (y = d per finite sample) across tiles, dropouts and calls."""
    if coefficients(rate, False, deemphasis_us)["alpha"] != 1.0:
        pytest.fail(f"alpha at {rate:g} Hz, {deemphasis_us} us no longer rounds to 1: pick a lower rate")
    lanes, calls = 2, [(3, 5000), (1, 20000), (2, 3001)]
    n = sum(f * m for f, m in calls)
    x = _narrow_fm(lanes, n, rate, 130)
    x[0, 4000:4000 + 3 * TILE_NARROW] = np.nan
    x[1, 14999] = np.nan
    _case(f"narrow {rate:g} Hz alpha = 1 de={deemphasis_us}", x, rate, False, deemphasis_us, calls)


@pytest.mark.parametrize("deemphasis_us", [0, 75])
@pytest.mark.parametrize("lanes", [1, 5])
@pytest.mark.parametrize("frame_len", [1, 3, 7])
def test_narrow_tiny_frames(ref, frame_len, lanes, deemphasis_us):
    """Frames of 1, 3 and 7 samples: one tiny tile per frame and lane, so the look-back's first round spans 32 tiles and
    predecessors are id - k * lanes."""
    calls = [(4000, frame_len), (1, frame_len), (2501, frame_len)]
    n = sum(f * m for f, m in calls)
    x = _narrow_fm(lanes, n, 250e3, 100 + frame_len)
    x[:, n // 3:n // 3 + 40] = np.nan
    _case(f"narrow frame_len={frame_len} lanes={lanes} de={deemphasis_us}", x, 250e3, False, deemphasis_us, calls)


@pytest.mark.parametrize("deemphasis_us", [0, 75])
def test_narrow_exact_zeros_and_signed_zeros(ref, deemphasis_us):
    """Exact 0, -0 and negative-real products: atan2 of (+-0, +-0), (+-0, x < 0) and (+-0, x > 0) gives 0, +-0 or +-pi
    exactly as IEEE defines; without de-emphasis those outputs equal the reference's bit for bit (sign included)."""
    special = np.array([1, 0, 0, complex(-0.0, 0.0), complex(0.0, -0.0), complex(-0.0, -0.0), 1, -1, -1, 1,
                        complex(-1, -0.0), 1, complex(1, -0.0), complex(-1, 0.0), -2, 1j, -1j, 0, 1j, complex(-0.0, 1),
                        complex(0.5, -0.0), complex(-0.5, -0.0), 0.25, 0], np.complex64)
    lanes, n = 2, 3 * TILE_NARROW + 100
    x = _narrow_fm(lanes, n, 250e3, 110)
    x[0, 10:10 + special.size] = special
    x[0, TILE_NARROW - 5:TILE_NARROW - 5 + special.size] = special              # across a tile boundary
    x[1, 1:1 + special.size] = special[::-1]
    calls = [(1, TILE_NARROW - 2), (1, 4), (1, n - TILE_NARROW - 2)]              # and across calls
    got, want, _ = _case(f"narrow zeros de={deemphasis_us}", x, 250e3, False, deemphasis_us, calls)
    if deemphasis_us == 0:
        pi_ref = np.float32(np.float32(np.pi) * np.float32(coefficients(250e3, False, 0)["ref"]))
        for lane, start in ((0, 10), (0, TILE_NARROW - 5), (1, 1)):
            g, w = got[lane, start:start + special.size + 1], want[lane, start:start + special.size + 1]
            zero, pi = w == 0, np.abs(w) == pi_ref
            assert zero.sum() >= 3 and pi.sum() >= 3, (lane, start, w)
            assert np.array_equal(g[zero | pi], w[zero | pi]), (lane, start, g, w)
            assert np.array_equal(np.signbit(g[zero | pi]), np.signbit(w[zero | pi])), (lane, start, g, w)


@pytest.mark.parametrize("deemphasis_us", [0, 75])
def test_narrow_slot_regrowth_and_split_calls(ref, deemphasis_us):
    """Calls with more look-back items than any before (the slot array grows, the epoch restarts), then with fewer (stale
    slots of older epochs must be ignored), on one plan; without de-emphasis the split stream equals one call bit for
    bit."""
    lanes = 3
    calls = [(1, 5000), (40, 8192), (3, 1000), (100, 2048), (2, 777), (9, 30000)]
    n = sum(f * m for f, m in calls)
    x = _narrow_fm(lanes, n, 250e3, 120)
    x[:, 400000:400000 + 5 * TILE_NARROW] = np.nan
    split, _, _ = _case(f"narrow regrowth de={deemphasis_us}", x, 250e3, False, deemphasis_us, calls)
    whole, _, _ = _case(f"narrow one call de={deemphasis_us}", x, 250e3, False, deemphasis_us, [(1, n)])
    if deemphasis_us == 0:
        assert np.array_equal(split, whole, equal_nan=True)
