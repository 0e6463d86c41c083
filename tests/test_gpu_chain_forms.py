"""Every fft4096_kernel form the spectral-chain entry points reach (tests/chain_forms.py) in steady state against F64,
the forms against each other bit for bit, the fallbacks those entry points take at n = 4096, the column-sum order
bit for bit, b200_chain_exec_host_typed, and the amplitude domain of the dB output.

The fused grid is G = min(rows, 2 SMs) persistent CTAs; CTA b runs rows b, b + G, b + 2G, ... The steady-state batch
7 G + G / 2 + 1 gives every CTA at least 7 rows: the 3-deep TMA rings wrap at least twice, the row parity that selects
the exchange buffer and the AGC partials flips many times, and the last round is ragged. Each failure names the worst
row, its CTA (row % G), its round (row // G) and its bin."""
import ctypes

import numpy as np
import pytest

import chain_forms as cf
from parity import approx_log10_f64, assert_db_close, db_allowance

pytestmark = pytest.mark.gpu

N = 4096
RANGE_LO, RANGE_HI = -100.0, -10.0
AGC = dict(reference=1.0, epsilon=1e-12, min_gain=0.05, max_gain=100.0)
CASES = [pytest.param(f, id=cf.form_id(f)) for f in cf.FORMS]


def _env():
    import torch
    from cyberether_b200 import _native
    from cyberether_b200.jetstream import Context
    dev = torch.device("cuda", torch.cuda.current_device())
    lib = _native.load()
    return torch, _native, lib, Context.get(dev), dev


def _stream(torch):
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _sms():
    torch, _native, lib, ctx, _ = _env()
    sms = ctypes.c_int()
    _native.check(lib.b200_ctx_sm_count(ctx.handle, ctypes.byref(sms)))
    return sms.value


def _grid():
    return 2 * _sms()


def _steady_rows():
    g = _grid()
    return 7 * g + g // 2 + 1


def _window(win):
    """The plan's window: the inverted Blackman taps (real), the same times exp(2 pi j 5.5 k / n), or None."""
    from oracle import port
    w = port.invert(port.window(N))
    if win == "WIN_REAL":
        return w
    if win == "WIN_COMPLEX":
        phasor = np.exp(2j * np.pi * 5.5 * np.arange(N) / N)
        return (w.astype(np.complex128) * phasor).astype(np.complex64)
    return None


def _special_rows(rows, g):
    """Rows on CTA and round boundaries: first and last CTA of the first rounds, a middle round, the ragged last round."""
    picks = [0, 1, g - 1, g, g + 1, 2 * g - 1, 3 * g + 7, rows - g // 2, rows - 2, rows - 1]
    return sorted({r for r in picks if 0 <= r < rows})


def _int_rows(itype, rows, seed, g, zero_rows=True):
    """[rows, n, 2] integer samples over the full range, with full-scale extreme rows (every component min or max),
    all-zero rows and DC-heavy rows (components just below max, still distinct after the F32 conversion) on CTA and
    round boundaries."""
    ty = cf.DTYPES[itype][1]
    info = np.iinfo(ty)
    rng = np.random.default_rng(seed)
    x = rng.integers(info.min, info.max, size=(rows, N, 2), dtype=ty, endpoint=True)
    span = max(16, (int(info.max) + 1) >> 12)
    for k, r in enumerate(_special_rows(rows, g)):
        kind = k % 3
        if kind == 0:
            x[r] = rng.choice(np.array([info.min, info.max], ty), size=(N, 2))
        elif kind == 1:
            x[r] = 0 if zero_rows else x[r]
        else:
            x[r] = rng.integers(int(info.max) - span, info.max, size=(N, 2), dtype=ty, endpoint=True)
    return x


def _cf32_rows(rows, seed, g, zero_rows=True):
    """Gaussian rows plus a tone, with all-zero rows on CTA and round boundaries."""
    rng = np.random.default_rng(seed)
    x = np.empty((rows, N), np.complex64)
    x.real = rng.standard_normal((rows, N), np.float32)
    x.imag = rng.standard_normal((rows, N), np.float32)
    x += (4.0 * np.exp(2j * np.pi * 300.25 * np.arange(N) / N)).astype(np.complex64)
    if zero_rows:
        x[_special_rows(rows, g)[1::3]] = 0
    return x


def _agc_level(rows, g):
    """0, 1, 2 for loud, middle and quiet rows; consecutive rows of one CTA (r, r + G) take different levels."""
    r = np.arange(rows)
    return (r // g + r % g) % 3


def _agc_rows(itype, rows, seed, g):
    rng = np.random.default_rng(seed)
    level = _agc_level(rows, g)
    if itype == "IN_CF32":
        sigma = np.array([30.0, 0.01, 1e-5], np.float32)[level][:, None]
        x = np.empty((rows, N), np.complex64)
        x.real = rng.standard_normal((rows, N), np.float32) * sigma
        x.imag = rng.standard_normal((rows, N), np.float32) * sigma
    else:
        info = np.iinfo(cf.DTYPES[itype][1])
        x = _int_rows(itype, rows, seed, g)
        signed = info.min < 0
        mid = rng.integers(-(info.max // 8) if signed else 0, info.max // 8, size=x.shape, endpoint=True)
        quiet = rng.integers(-1 if signed else 0, 1, size=x.shape, endpoint=True)
        x = np.where((level == 1)[:, None, None], mid, np.where((level == 2)[:, None, None], quiet, x)).astype(x.dtype)
    x[_special_rows(rows, g)[1::3]] = 0
    return x


def _device(torch, x, dev, misalign=0):
    """x's bytes on the device, starting `misalign` bytes past a 16-byte boundary."""
    raw = torch.from_numpy(np.ascontiguousarray(x).reshape(-1).view(np.uint8))
    buf = torch.empty(raw.numel() + 16, dtype=torch.uint8, device=dev)
    view = buf[misalign:misalign + raw.numel()]
    view.copy_(raw)
    assert view.data_ptr() % 16 == misalign
    return view


class _Plan:
    """A chain plan for [rows, n] with a window (or none) and the entry points on it."""

    def __init__(self, window, rows, n=N):
        import cyberether_b200 as cb
        self.torch, self.native, self.lib, self.ctx, self.dev = _env()
        self.n, self.coeff = n, cb.amplitude_scaling_coeff(n)
        self.scale, self.offset = cb.range_coefficients(RANGE_LO, RANGE_HI)
        self.wd = None if window is None else self.torch.from_numpy(window).to(self.dev)
        self.plan = ctypes.c_void_p()
        self.native.check(self.lib.b200_chain_plan_create(self.ctx.handle, n, max(rows, 1),
                                                          None if self.wd is None else self.wd.data_ptr(),
                                                          ctypes.byref(self.plan)))

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.torch.cuda.synchronize()
        self.native.check(self.lib.b200_chain_plan_destroy(self.plan))

    def call(self, entry, xd, dtype, rows, enable_range, colsum=None, agc=AGC):
        """Run one entry point; returns (rc, out) with out on the device."""
        out = self.torch.empty(max(rows, 1), self.n, dtype=self.torch.float32, device=self.dev)
        common = (rows, self.coeff, int(enable_range), self.scale, self.offset)
        s = _stream(self.torch)
        ptr = xd.data_ptr() if xd is not None else None
        if entry == "chain_exec":
            assert dtype == 1
            rc = self.lib.b200_chain_exec(self.plan, ptr, out.data_ptr(), *common, s)
        elif entry == "chain_exec_typed":
            rc = self.lib.b200_chain_exec_typed(self.plan, ptr, dtype, out.data_ptr(), *common, s)
        elif entry == "chain_exec_agc":
            rc = self.lib.b200_chain_exec_agc(self.plan, ptr, dtype, out.data_ptr(), *common, agc["reference"],
                                              agc["epsilon"], agc["min_gain"], agc["max_gain"], s)
        else:
            rc = self.lib.b200_chain_exec_colsum(self.plan, ptr, dtype, out.data_ptr(), *common, colsum.data_ptr(), s)
        self.torch.cuda.synchronize()
        return rc, out

    def run(self, entry, xd, dtype, rows, enable_range, colsum=None, agc=AGC):
        rc, out = self.call(entry, xd, dtype, rows, enable_range, colsum, agc)
        self.native.check(rc)
        return out[:rows].cpu().numpy()

    def cast(self, xd, dtype, count):
        y = self.torch.empty(count, dtype=self.torch.complex64, device=self.dev)
        self.native.check(self.lib.b200_cast_int(self.ctx.handle, xd.data_ptr(), dtype, y.data_ptr(), count,
                                                 _stream(self.torch)))
        self.torch.cuda.synchronize()
        return y

    def model(self, spec, enable_range):
        want = cf.db(spec, self.coeff)
        return cf.to_range(want, self.scale, self.offset) if enable_range else want


def _assert_model(got, want, spec, enable_range, what, g):
    """assert_db_close with the allowances of test_chain_exec_steady_state; names the worst row, CTA, round and bin."""
    slope, floor = (2.0 / abs(RANGE_HI - RANGE_LO), 3e-7) if enable_range else (1.0, 0.0)
    try:
        with np.errstate(invalid="ignore"):      # -inf - -inf in the masked-out elements
            assert_db_close(got, want, spec, scale=slope, floor=floor)
    except AssertionError as e:
        mask = np.isfinite(got) != np.isfinite(want)
        if mask.any():
            excess = mask.astype(np.float64)
        else:
            excess = np.abs(np.where(np.isfinite(want), got - want, 0.0)) - (db_allowance(spec) * slope + floor)
        row, col = np.unravel_index(int(np.argmax(excess)), excess.shape)
        raise AssertionError(f"{what}: {e}; worst row {row} (CTA {row % g}, round {row // g}) bin {col}: got "
                             f"{got[row, col]!r} want {want[row, col]!r}") from None


def _assert_same(got, want, what, g):
    same = (got == want) | (np.isnan(got) & np.isnan(want))
    if not same.all():
        row, col = np.argwhere(~same)[0]
        raise AssertionError(f"{what}: {int((~same).sum())} elements differ; first row {row} (CTA {row % g}, round "
                             f"{row // g}) bin {col}: {got[row, col]!r} vs {want[row, col]!r}")


def _assert_colsum(got, want, what):
    same = (got == want) | (np.isnan(got) & np.isnan(want))
    if not same.all():
        col = int(np.argwhere(~same)[0][0])
        raise AssertionError(f"{what}: {int((~same).sum())} of {got.size} column sums differ (odd columns "
                             f"{int((~same[1::2]).sum())}); first column {col}: {got[col]!r} vs {want[col]!r}")


@pytest.mark.parametrize("form", CASES)
def test_chain_form_steady_state(form):
    """One form: against F64, against its partner form bit for bit, and (COLSUM) the column sums bit for bit against
    the fused summation order applied to the spectra the same call wrote."""
    entry, mode, win, itype = form
    enable_range = mode == "MODE_AMP_RANGE"
    torch, _native, lib, ctx, dev = _env()
    g, rows = _grid(), _steady_rows()
    dtype = cf.DTYPES[itype][0]
    seed = cf.FORMS.index(form)
    window = _window(win)
    zero_rows = entry != "chain_exec_colsum" or enable_range   # in dB mode one -inf row makes every sum -inf
    if entry == "chain_exec_agc":
        x = _agc_rows(itype, rows, seed, g)
    elif itype == "IN_CF32":
        x = _cf32_rows(rows, seed, g, zero_rows)
    else:
        x = _int_rows(itype, rows, seed, g, zero_rows)
    samples = cf.exact_samples(x, itype)
    with _Plan(window, rows) as plan:
        xd = _device(torch, x, dev)
        colsum = torch.full((N,), float("nan"), dtype=torch.float32, device=dev)
        got = plan.run(entry, xd, dtype, rows, enable_range, colsum=colsum)
        # the partner form on the same samples
        if itype != "IN_CF32" and entry in ("chain_exec_typed", "chain_exec_agc"):
            cast = plan.cast(xd, dtype, rows * N)
            partner = plan.run("chain_exec" if entry == "chain_exec_typed" else "chain_exec_agc", cast, 1, rows,
                               enable_range)
            _assert_same(got, partner, f"{cf.form_id(form)} vs cast -> CF32 form", g)
        if entry == "chain_exec_colsum":
            partner = plan.run("chain_exec_typed", xd, dtype, rows, enable_range)
            _assert_same(got, partner, f"{cf.form_id(form)} spectra vs b200_chain_exec_typed", g)
            _assert_colsum(colsum.cpu().numpy(), cf.colsum_fused(got, _sms()), f"{cf.form_id(form)} column sums")
    spec = cf.spectrum(samples, window)
    if entry == "chain_exec_agc":
        raw = cf.agc_gain(samples, window, clamp=False, **AGC)
        assert (raw < AGC["min_gain"]).any() and (raw > AGC["max_gain"]).any()
        assert ((raw > 1.5 * AGC["min_gain"]) & (raw < AGC["max_gain"] / 1.5)).any()
        spec = spec * np.clip(raw, AGC["min_gain"], AGC["max_gain"])
    _assert_model(got, plan.model(spec, enable_range), spec, enable_range, cf.form_id(form), g)


# ---- fallbacks at n = 4096 -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("enable_range", [False, True])
@pytest.mark.parametrize("itype", ["IN_CI32", "IN_CU32"])
def test_chain_exec_typed_32_bit_casts_through_the_plan_scratch(itype, enable_range):
    """CI32 / CU32 have no fused form: b200_cast_int into the plan's cast scratch, then the CF32 kernel. Against F64,
    and bit for bit against b200_cast_int -> b200_chain_exec."""
    torch, _native, lib, ctx, dev = _env()
    g, rows = _grid(), _steady_rows()
    dtype = cf.DTYPES[itype][0]
    x = _int_rows(itype, rows, 40 + enable_range, g)
    window = _window("WIN_REAL")
    with _Plan(window, rows) as plan:
        xd = _device(torch, x, dev)
        got = plan.run("chain_exec_typed", xd, dtype, rows, enable_range)
        want_bits = plan.run("chain_exec", plan.cast(xd, dtype, rows * N), 1, rows, enable_range)
    _assert_same(got, want_bits, f"{itype} vs cast -> chain", g)
    spec = cf.spectrum(cf.exact_samples(x, itype), window)
    _assert_model(got, plan.model(spec, enable_range), spec, enable_range, itype, g)


@pytest.mark.parametrize("itype", cf.INT_TYPES)
def test_chain_exec_typed_misaligned_integer_input_equals_fused_form(itype):
    """Integer rows that do not start on a 16-byte boundary cannot be landed by TMA: cast, then the CF32 kernel. The
    result is bit-identical to the fused integer form on the same samples."""
    torch, _native, lib, ctx, dev = _env()
    g, rows = _grid(), _steady_rows()
    dtype = cf.DTYPES[itype][0]
    x = _int_rows(itype, rows, 50, g)
    with _Plan(_window("WIN_REAL"), rows) as plan:
        fused = plan.run("chain_exec_typed", _device(torch, x, dev), dtype, rows, True)
        shifted = plan.run("chain_exec_typed", _device(torch, x, dev, misalign=x.itemsize * 2), dtype, rows, True)
    _assert_same(shifted, fused, f"misaligned {itype} vs fused", g)


@pytest.mark.parametrize("enable_range", [False, True])
@pytest.mark.parametrize("itype,misalign", [("IN_CF32", 8), ("IN_CI32", 0)])
def test_chain_exec_colsum_unfused_sums_in_row_split_order(itype, misalign, enable_range):
    """b200_chain_exec_colsum without a fused form (misaligned CF32, CI32): the chain, then colsum_partials +
    colsum_reduce. The spectra against F64, the sums bit for bit against the row-split order."""
    torch, _native, lib, ctx, dev = _env()
    g, rows = _grid(), _steady_rows()
    dtype = cf.DTYPES[itype][0]
    x = _cf32_rows(rows, 60, g, enable_range) if itype == "IN_CF32" else _int_rows(itype, rows, 60, g, enable_range)
    window = _window("WIN_REAL")
    with _Plan(window, rows) as plan:
        colsum = torch.full((N,), float("nan"), dtype=torch.float32, device=dev)
        got = plan.run("chain_exec_colsum", _device(torch, x, dev, misalign), dtype, rows, enable_range, colsum=colsum)
    _assert_colsum(colsum.cpu().numpy(), cf.colsum_row_split(got, _sms()), f"{itype} misalign {misalign}")
    spec = cf.spectrum(cf.exact_samples(x, itype), window)
    _assert_model(got, plan.model(spec, enable_range), spec, enable_range, f"{itype} colsum", g)


@pytest.mark.parametrize("itype,misalign,message", [
    ("IN_CF32", 8, "b200_chain_exec_agc: input must be 16-byte aligned"),
    ("IN_CI8", 2, "b200_chain_exec_agc: input must be 16-byte aligned"),
    ("IN_CI32", 0, "b200_chain_exec_agc: input dtype code 12 is not CF32 / CI8 / CU8 / CI16 / CU16")])
def test_chain_exec_agc_refuses_inputs_without_a_fused_form(itype, misalign, message):
    torch, _native, lib, ctx, dev = _env()
    x = _int_rows(itype, 3, 0, 2) if itype != "IN_CF32" else _cf32_rows(3, 0, 2)
    with _Plan(_window("WIN_REAL"), 3) as plan:
        rc, _ = plan.call("chain_exec_agc", _device(torch, x, dev, misalign), cf.DTYPES[itype][0], 3, True)
    assert rc == 1
    assert lib.b200_last_error().decode() == message


# ---- column sums: the summation order, bit for bit -----------------------------------------------------------------
def _colsum_call(plan, x, itype, rows, enable_range, misalign=0):
    torch = plan.torch
    colsum = torch.full((plan.n,), float("nan"), dtype=torch.float32, device=plan.dev)
    xd = _device(torch, x, plan.dev, misalign) if rows else None
    out = plan.run("chain_exec_colsum", xd, cf.DTYPES[itype][0], rows, enable_range, colsum=colsum)
    return out, colsum.cpu().numpy()


@pytest.mark.parametrize("enable_range", [False, True])
@pytest.mark.parametrize("itype,case", [("IN_CF32", "below-grid"), ("IN_CU8", "below-grid"), ("IN_CF32", "steady"),
                                        ("IN_CI16", "steady"), ("IN_CF32", "neg-inf-rows"), ("IN_CI8", "neg-inf-rows"),
                                        ("IN_CF32", "nan-rows")])
def test_chain_exec_colsum_fused_order(itype, case, enable_range):
    """The fused sums equal chain_forms.colsum_fused applied to the spectra of the same call, in every column: a batch
    smaller than the grid, the steady-state batch, all-zero rows (-inf in dB mode, 0 in range mode), and NaN samples
    (compared by NaN mask; a NaN row reads the finite value include/b200dsp.h documents)."""
    torch, _native, lib, ctx, dev = _env()
    g = _grid()
    rows = g // 2 + 3 if case == "below-grid" else _steady_rows()
    x = _cf32_rows(rows, 70, g, False) if itype == "IN_CF32" else _int_rows(itype, rows, 70, g, False)
    if case == "neg-inf-rows":
        x[::5] = 0
    if case == "nan-rows":
        x[3::7, 100] = np.nan
    with _Plan(_window("WIN_REAL"), rows) as plan:
        out, colsum = _colsum_call(plan, x, itype, rows, enable_range)
    if case == "neg-inf-rows" and not enable_range:
        assert np.isneginf(out[::5]).all() and np.isneginf(colsum).all()
    if case == "nan-rows":       # the documented reading of a NaN spectrum (include/b200dsp.h)
        nan_db = 20.0 * approx_log10_f64(np.ldexp(1.0 - 2.0 ** -24, 129)) + plan.coeff
        assert np.abs(out[3::7] - (1.0 if enable_range else nan_db)).max() <= 1e-3
    _assert_colsum(colsum, cf.colsum_fused(out, _sms()), f"{itype} {case}")


def test_chain_exec_colsum_zero_batch_zeroes_the_sums():
    torch, _native, lib, ctx, dev = _env()
    with _Plan(_window("WIN_REAL"), 4) as plan:
        _, colsum = _colsum_call(plan, None, "IN_CF32", 0, True)
    assert np.array_equal(colsum.view(np.uint32), np.zeros(N, np.uint32))


@pytest.mark.parametrize("n,rows", [(1024, 1000), (16384, 300)])
def test_chain_exec_colsum_other_lengths_row_split_order(n, rows):
    """n != 4096: the chain, then the row-split column sums (more than one split at these batches)."""
    torch, _native, lib, ctx, dev = _env()
    from oracle import port
    x = np.random.default_rng(n).standard_normal((rows, n, 2)).astype(np.float32).view(np.complex64)[..., 0]
    assert cf.colsum_splits(rows, n, _sms()) > 1
    with _Plan(port.invert(port.window(n)), rows, n=n) as plan:
        out, colsum = _colsum_call(plan, x, "IN_CF32", rows, True)
    _assert_colsum(colsum, cf.colsum_row_split(out, _sms()), f"n={n}")


def test_chain_exec_colsum_alternating_fused_and_unfused_calls_on_one_plan():
    """One plan, batch 64 G + 1: the unfused call needs more partials than the fused one, so the plan's partial buffer
    regrows between them; every call sums in its own order."""
    torch, _native, lib, ctx, dev = _env()
    g, sms = _grid(), _sms()
    rows = 64 * g + 1
    x = _cf32_rows(rows, 80, g, False)
    assert -(-rows // 64) > g          # the unfused call's partials outgrow the fused call's
    with _Plan(_window("WIN_REAL"), rows) as plan:
        for k, misalign in enumerate([0, 8, 0, 8]):
            out, colsum = _colsum_call(plan, x, "IN_CF32", rows, True, misalign)
            order = cf.colsum_row_split if misalign else cf.colsum_fused
            _assert_colsum(colsum, order(out, sms), f"call {k} misalign {misalign}")


@pytest.mark.parametrize("decimation", [1, 2, 3, 4])
def test_lineplot_update_from_fused_colsum(decimation):
    """b200_lineplot_update_from_colsum on the fused sums of a steady-state batch, three updates: signalPoints bit for bit
    against chain_forms.lineplot_from_colsum (lineplot_finalize_kernel restated in F32)."""
    torch, _native, lib, ctx, dev = _env()
    g, rows = _grid(), _steady_rows()
    elements, averaging = N // decimation, 3
    normalization = np.float32(1.0) / (np.float32(0.5) * np.float32(rows))
    points = torch.empty(elements, 2, dtype=torch.float32, device=dev)
    average = torch.empty(elements, dtype=torch.float32, device=dev)
    s = _stream(torch)
    _native.check(lib.b200_lineplot_init(ctx.handle, points.data_ptr(), average.data_ptr(), elements, s))
    avg = np.zeros(elements, np.float32)
    with _Plan(_window("WIN_REAL"), rows) as plan:
        for k in range(3):
            x = _int_rows("IN_CI16", rows, 90 + k, g)
            colsum = torch.empty(N, dtype=torch.float32, device=dev)
            plan.run("chain_exec_colsum", _device(torch, x, dev), cf.DTYPES["IN_CI16"][0], rows, True, colsum=colsum)
            _native.check(lib.b200_lineplot_update_from_colsum(ctx.handle, colsum.data_ptr(), elements, decimation,
                                                               float(normalization), averaging, average.data_ptr(),
                                                               points.data_ptr(), s))
            torch.cuda.synchronize()
            avg = cf.lineplot_from_colsum(colsum.cpu().numpy(), decimation, normalization, averaging, avg)
            got = points.cpu().numpy()
            assert np.array_equal(got[:, 0], cf.lineplot_x(elements))
            assert np.array_equal(got[:, 1], avg), f"update {k}"
            assert np.array_equal(average.cpu().numpy(), avg)


# ---- b200_chain_exec_host_typed ------------------------------------------------------------------------------------
@pytest.mark.parametrize("chunk", [0, 7, 200, 256, 1000])
@pytest.mark.parametrize("itype", list(cf.INT_TYPES) + ["IN_CI32", "IN_CU32"])
def test_chain_exec_host_typed_equals_device_typed(itype, chunk):
    """Pinned host samples through the three-slot H2D / kernel / D2H pipeline, twice on one plan: bit-identical to
    b200_chain_exec_typed on the device, for chunks of the default size, 7 rows, a divisor of the batch, a ragged last
    chunk and more than the batch."""
    torch, _native, lib, ctx, dev = _env()
    rows, g = 600, _grid()
    dtype = cf.DTYPES[itype][0]
    x = _int_rows(itype, rows, 100 + chunk, min(rows, g))
    x_host = torch.empty(x.nbytes, dtype=torch.uint8, pin_memory=True)
    x_host.copy_(torch.from_numpy(x.reshape(-1).view(np.uint8)))
    out_host = torch.empty(rows, N, dtype=torch.float32, pin_memory=True)
    with _Plan(_window("WIN_REAL"), rows) as plan:
        want = plan.run("chain_exec_typed", _device(torch, x, dev), dtype, rows, True)
        for call in range(2):
            out_host.fill_(float("nan"))
            _native.check(lib.b200_chain_exec_host_typed(plan.plan, x_host.data_ptr(), dtype, out_host.data_ptr(), rows,
                                                         plan.coeff, 1, plan.scale, plan.offset, chunk))
            _assert_same(out_host.numpy(), want, f"{itype} chunk {chunk} call {call}", min(rows, g))


# ---- amplitude domain of the dB output -----------------------------------------------------------------------------
F32_MAX = float(np.finfo(np.float32).max)
OVERFLOW_DB_LOG = approx_log10_f64(2.0 ** 128)    # |X|^2 overflows to inf: sqrt(inf) reads as 2^128


@pytest.mark.parametrize("form", [c for c in CASES if c.values[0][3] == "IN_CF32"])
def test_chain_amplitude_overflow_threshold(form):
    """Coherent CF32 tones whose peak |X| sits at 0.5, 0.9 and 0.999 of sqrt(F32 max) follow the model; at 1.01, 2 and
    1e3 of it |X|^2 overflows in F32 and the peak bins read 20 approx_log10(2^128) + coeff (range: 1.0), as
    include/b200dsp.h states. Bins whose F64 |X|^2 lies within 1e-3 of the threshold, widened by four times the
    normwise spectrum error of parity.DELTA, are not asserted."""
    entry, mode, win, itype = form
    enable_range = mode == "MODE_AMP_RANGE"
    torch, _native, lib, ctx, dev = _env()
    window = _window(win)
    fractions = [0.5, 0.9, 0.999, 1.01, 2.0, 1e3]
    rows = len(fractions) * 3
    k = np.arange(N)
    w = np.ones(N) if window is None else window.astype(np.complex128)
    tone = np.exp(2j * np.pi * 700 * k / N)
    peak = np.abs(np.fft.fft(tone * w)).max()
    rng = np.random.default_rng(7)
    amp = np.repeat(np.array(fractions) * np.sqrt(F32_MAX) / peak, 3)[:, None]
    noise = (rng.standard_normal((rows, N)) + 1j * rng.standard_normal((rows, N))) * 1e-3
    x = (amp * (tone + noise)).astype(np.complex64)
    with _Plan(window, rows) as plan:
        colsum = torch.empty(N, dtype=torch.float32, device=dev)
        got = plan.run(entry, _device(torch, x, dev), 1, rows, enable_range, colsum=colsum, agc=AGC)
    spec = cf.spectrum(x.astype(np.complex128), window)
    if entry == "chain_exec_agc":
        spec = spec * cf.agc_gain(x.astype(np.complex128), window, **AGC)
    power = np.abs(cf.spectrum(x.astype(np.complex128), window)) ** 2
    want = plan.model(spec, enable_range)
    over = power > F32_MAX * 1.001
    mag = np.sqrt(power)
    near = np.abs(power / F32_MAX - 1.0) <= 1e-3 + 4e-6 * mag.max(axis=1, keepdims=True) / mag
    assert over[len(fractions) // 2 * 3:].any() and not over[:len(fractions) // 2 * 3].any()
    want = np.where(over, 1.0 if enable_range else 20.0 * OVERFLOW_DB_LOG + plan.coeff, want)
    keep = ~near
    slope, floor = (2.0 / abs(RANGE_HI - RANGE_LO), 3e-7) if enable_range else (1.0, 0.0)
    allow = np.where(over, 1e-3 * slope, db_allowance(spec) * slope + floor)
    err = np.abs(got - want)
    bad = keep & ~(err <= allow)
    if bad.any():
        row, col = np.argwhere(bad)[0]
        raise AssertionError(f"{cf.form_id(form)}: {int(bad.sum())} bins off; row {row} (peak "
                             f"{fractions[row // 3]} of the threshold) bin {col}: got {got[row, col]!r} want "
                             f"{want[row, col]!r}")
