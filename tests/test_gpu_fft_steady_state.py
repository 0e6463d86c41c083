"""fft_radix_kernel, and the plans built on it, in steady state against numpy F64.

fft_radix_kernel is persistent: launch_radix caps its grid at SMs x CTAs per SM (2 up to 256 threads, else 1) and each CTA
loops over blocks first, first + gridDim.x, ... of G = max(1, 4096 / n) rows each. Every shape below is derived from the
device so that each CTA runs at least three blocks (its two-stage TMA ring wraps and its exchange buffers are reused from
block to block) and, where G > 1, the last block is ragged. Default plans only. Each failure names the worst row, its
block and its bin."""
import ctypes

import numpy as np
import pytest

from parity import approx_log10_f64, assert_db_close, db_allowance

pytestmark = pytest.mark.gpu

RADIX_LENGTHS = [1 << k for k in range(4, 14)]       # 16 ... 8192: every fft_radix_kernel length


def _env():
    import torch
    from cyberether_b200 import _native
    from cyberether_b200.jetstream import Context
    dev = torch.device("cuda", torch.cuda.current_device())
    lib = _native.load()
    return torch, _native, lib, Context.get(dev), dev


def _stream(torch):
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _rows_per_block(n):
    return max(1, 4096 // n)


def _grid_cap(n):
    """launch_radix's grid cap for the n-point kernel."""
    torch, _native, lib, ctx, _ = _env()
    sms = ctypes.c_int()
    _native.check(lib.b200_ctx_sm_count(ctx.handle, ctypes.byref(sms)))
    return sms.value * (2 if max(256, n // 16) <= 256 else 1)


def _steady_rows(n):
    """At least three blocks per CTA, and a last block of G / 2 + 1 rows."""
    g = _rows_per_block(n)
    return 3 * _grid_cap(n) * g + g // 2 + 1


def _gaussian(shape, seed):
    rng = np.random.default_rng(seed)
    x = np.empty(shape, np.complex64)
    x.real = rng.standard_normal(shape, np.float32)
    x.imag = rng.standard_normal(shape, np.float32)
    return x


def _assert_rows_close(got, want, bound, what, rows_per_block=1, scale=None):
    """max|got - want| <= bound * max|X| in every row (X = want unless `scale` gives the row's spectrum)."""
    err = np.abs(got - want)
    rel = err.max(axis=1) / np.abs(want if scale is None else scale).max(axis=1)
    row = int(rel.argmax())
    assert rel[row] <= bound, (f"{what}: row {row} (block {row // rows_per_block}) bin {int(err[row].argmax())}: "
                               f"max |got - X| = {rel[row]:.3e} max |X| (bound {bound:.0e})")


def _fft_exec(x, forward=True, misalign=False):
    """b200_fft_plan_c2c(n, batch) + b200_fft_exec on a [batch, n] CF32 array."""
    torch, _native, lib, ctx, dev = _env()
    batch, n = x.shape
    src = torch.from_numpy(x).to(dev).reshape(-1)
    if misalign:                  # a view that starts on an odd sample: 8-byte but not 16-byte aligned
        base = torch.empty(batch * n + 1, dtype=torch.complex64, device=dev)
        base[1:] = src
        src = base[1:]
        assert src.data_ptr() % 16 == 8
    out = torch.empty(batch * n, dtype=torch.complex64, device=dev)
    plan = ctypes.c_void_p()
    _native.check(lib.b200_fft_plan_c2c(ctx.handle, n, batch, ctypes.byref(plan)))
    try:
        _native.check(lib.b200_fft_exec(plan, src.data_ptr(), out.data_ptr(), 1 if forward else 0, _stream(torch)))
        torch.cuda.synchronize()
    finally:
        _native.check(lib.b200_fft_plan_destroy(plan))
    return out.cpu().numpy().reshape(batch, n)


def _f64_fft(x, forward=True):
    x = x.astype(np.complex128)
    return np.fft.fft(x, axis=1) if forward else np.fft.ifft(x, axis=1) * x.shape[1]


@pytest.mark.parametrize("forward", [True, False])
@pytest.mark.parametrize("n", RADIX_LENGTHS)
def test_fft_exec_steady_state(n, forward):
    """fft_radix_kernel<MODE_C2C>; bound 2e-6 max|X| per transform as the other C2C tests."""
    rows = _steady_rows(n)
    x = _gaussian((rows, n), n + forward)
    _assert_rows_close(_fft_exec(x, forward), _f64_fft(x, forward), 2e-6, f"n={n} forward={forward}", _rows_per_block(n))


@pytest.mark.parametrize("forward", [True, False])
@pytest.mark.parametrize("n", [16, 256, 2048, 8192])
def test_fft_exec_misaligned_input_steady_state(n, forward):
    """An input that is not 16-byte aligned cannot be landed by TMA and runs the persistent fft_generic_kernel."""
    rows = _steady_rows(n)
    x = _gaussian((rows, n), 3 * n + forward)
    _assert_rows_close(_fft_exec(x, forward, misalign=True), _f64_fft(x, forward), 2e-6,
                       f"misaligned n={n} forward={forward}")


@pytest.mark.parametrize("enable_range", [False, True])
@pytest.mark.parametrize("n", RADIX_LENGTHS)
def test_chain_exec_steady_state(n, enable_range):
    """b200_chain_exec with a real window: fft_radix_kernel<MODE_AMP / MODE_AMP_RANGE, WIN_REAL> (fft4096_kernel at 4096).
    Want in F64 from the windowed rows: dB = 20 ApproxLog10|X| + coeff, range = 0.5 + 0.5 tanh(4 ((dB scale + offset) -
    0.5)) (include/b200dsp.h), compared with the allowances of test_chain_other_sizes."""
    import cyberether_b200 as cb
    from oracle import port
    torch, _native, lib, ctx, dev = _env()
    rows = _steady_rows(n)
    x = _gaussian((rows, n), 5 * n + enable_range)
    w = port.invert(port.window(n))
    assert not np.any(w.imag)
    lo, hi = -100.0, -10.0
    coeff = cb.amplitude_scaling_coeff(n)
    scale, offset = cb.range_coefficients(lo, hi)
    xd = torch.from_numpy(x).to(dev)
    wd = torch.from_numpy(w).to(dev)
    out = torch.empty(rows, n, dtype=torch.float32, device=dev)
    plan = ctypes.c_void_p()
    _native.check(lib.b200_chain_plan_create(ctx.handle, n, rows, wd.data_ptr(), ctypes.byref(plan)))
    try:
        _native.check(lib.b200_chain_exec(plan, xd.data_ptr(), out.data_ptr(), rows, coeff, int(enable_range), scale,
                                          offset, _stream(torch)))
        torch.cuda.synchronize()
    finally:
        _native.check(lib.b200_chain_plan_destroy(plan))
    got = out.cpu().numpy()
    spec = np.fft.fft(x.astype(np.complex128) * w.astype(np.complex128), axis=1)
    want = 20.0 * approx_log10_f64(np.abs(spec)) + coeff
    slope, floor = (2.0 / abs(hi - lo), 3e-7) if enable_range else (1.0, 0.0)
    if enable_range:
        want = 0.5 + 0.5 * np.tanh(4.0 * ((want * scale + offset) - 0.5))
    try:
        assert_db_close(got, want, spec, scale=slope, floor=floor)
    except AssertionError as e:
        excess = np.abs(got - want) - (db_allowance(spec) * slope + floor)
        row, col = np.unravel_index(int(np.argmax(excess)), excess.shape)
        raise AssertionError(f"n={n} range={enable_range}: {e}; worst row {row} (block {row // _rows_per_block(n)}) "
                             f"bin {col}") from None


@pytest.mark.parametrize("layout", [0, 1])
@pytest.mark.parametrize("h", RADIX_LENGTHS[1:])
def test_fft_exec_real_steady_state(h, layout):
    """b200_fft_exec_real, real rows of 2h through fft_radix_kernel<MODE_R2C> (unpack in the epilogue); bound 2e-6 max|X|
    as test_fft_exec_real_half_length_path, per row."""
    torch, _native, lib, ctx, dev = _env()
    rows, n = _steady_rows(h), 2 * h
    x = np.random.default_rng(h + layout).standard_normal((rows, n), np.float32)
    xd = torch.from_numpy(x).to(dev)
    out = torch.empty((rows, h + 1), dtype=torch.complex64, device=dev) if layout == 0 else \
        torch.empty((rows, n), dtype=torch.float32, device=dev)
    plan = ctypes.c_void_p()
    _native.check(lib.b200_fft_plan_c2c(ctx.handle, h, rows, ctypes.byref(plan)))
    try:
        _native.check(lib.b200_fft_exec_real(plan, xd.data_ptr(), out.data_ptr(), layout, _stream(torch)))
        torch.cuda.synchronize()
    finally:
        _native.check(lib.b200_fft_plan_destroy(plan))
    got = out.cpu().numpy()
    spec = np.fft.rfft(x.astype(np.float64), axis=1)
    if layout == 0:
        want = spec
    else:
        want = np.empty((rows, n))
        want[:, 0] = spec[:, 0].real
        want[:, 1:n - 1:2] = spec[:, 1:h].real
        want[:, 2:n - 1:2] = spec[:, 1:h].imag
        want[:, n - 1] = spec[:, h].real
    _assert_rows_close(got, want, 2e-6, f"h={h} layout={layout}", _rows_per_block(h), scale=spec)


def test_two_pass_plan_steady_state():
    """n = 131072, batch 30: the default 24 MB chunk holds 24 transforms, so the row pass
    fft_radix_kernel<13, MODE_C2C_T> runs 384 and then 96 rows of 8192."""
    x = _gaussian((30, 131072), 131072)
    _assert_rows_close(_fft_exec(x), _f64_fft(x), 2e-6, "two-pass n=131072")


@pytest.mark.parametrize("n", [3000, 4095])
def test_bluestein_plan_steady_state(n):
    """Bluestein through a circular convolution of m = 8192 over the whole batch (batch > 3 x SMs rows of 8192)."""
    x = _gaussian((max(400, 3 * _grid_cap(8192) + 1), n), n)
    _assert_rows_close(_fft_exec(x), _f64_fft(x), 2e-6, f"bluestein n={n}")


def test_four_step_plan_steady_state():
    """n = 2^25, batch 1: 8192-point sub-transforms over 4096 rows (and 4096-point ones over 8192); bound 1e-5 max|X| (the
    north-star tolerance). Holds about 1 GB of host memory with the F64 reference."""
    x = _gaussian((1, 1 << 25), 25)
    got = _fft_exec(x)
    _assert_rows_close(got, _f64_fft(x), 1e-5, "four-step n=2^25")
