"""pad, unpad, fold, overlap_add and phase_correction on provider b200.

1. The C ABI entry points (b200_fold, b200_overlap_add, b200_phase_correction) against F64 / numpy restatements of the
   reference loops (src/domains/dsp/{fold,overlap_add,phase_correction}/module_impl_native_cpu.cc), over three calls
   where the module carries state.
2. Each module as a single block, and the wirings that use them (the `filter` block on layouts the fused FIR does not
   take, `filter_engine`, a hand-wired overlap-add-fold graph), in the reference's own Flowgraph on the CPU provider
   and on provider b200 in one process, three cycles of fresh input each.
"""
import ctypes
import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

TWO_PI = 2.0 * math.pi


# ---- C ABI against restatements of the reference loops ------------------------------------------------------------

@pytest.fixture(scope="module")
def abi():
    import torch
    from cyberether_b200 import _native
    lib = _native.load()
    ctx = ctypes.c_void_p()
    _native.check(lib.b200_ctx_create(torch.cuda.current_device(), ctypes.byref(ctx)))
    yield lib, ctx, _native.check
    lib.b200_ctx_destroy(ctx)


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _host(t):
    import torch
    torch.cuda.synchronize()
    return t.cpu().numpy()


def _stream():
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _data(rng, shape, complex_):
    x = rng.standard_normal(shape).astype(np.float32)
    if complex_:
        x = (x + 1j * rng.standard_normal(shape).astype(np.float32)).astype(np.complex64)
    return x


def fold_model(x, axis, size, offset, channel_offsets=None, channel_axis=None):
    """FoldImplNativeCpu::foldKernel: F64 sum in ascending group order, one F64 division, one rounding."""
    n = x.shape[axis]
    groups = n // size
    xm = np.moveaxis(x, axis, -1).astype(np.complex128 if np.iscomplexobj(x) else np.float64)
    o = np.arange(size)
    if channel_offsets is None:
        offs = np.full(xm.shape[:-1] + (1,), offset % n, dtype=np.int64)
    else:
        ca = channel_axis if channel_axis < axis else channel_axis - 1      # channel axis after moving `axis` last
        shape = [1] * (xm.ndim - 1) + [1]
        shape[ca] = len(channel_offsets)
        offs = np.broadcast_to((np.asarray(channel_offsets, np.int64) % n).reshape(shape), xm.shape[:-1] + (1,))
    total = np.zeros(xm.shape[:-1] + (size,), xm.dtype)
    for g in range(groups):
        idx = (o + g * size - offs) % n
        total = total + np.take_along_axis(xm, np.broadcast_to(idx, total.shape), axis=-1)
    if np.iscomplexobj(x):
        out = np.empty(total.shape, np.complex64)
        out.real = total.real / float(groups)
        out.imag = total.imag / float(groups)
    else:
        out = (total / float(groups)).astype(np.float32)
    return np.moveaxis(out, -1, axis)


@pytest.mark.parametrize("complex_", [False, True])
@pytest.mark.parametrize("groups", [1, 2, 10])
@pytest.mark.parametrize("layout", ["scalar", "channels_before", "channels_after", "channels_3d"])
def test_fold_abi_bit_exact(abi, complex_, groups, layout):
    lib, ctx, check = abi
    rng = np.random.default_rng(groups * 7 + len(layout))
    size = 90
    n = size * groups
    if layout == "scalar":
        shape, axis, caxis, offsets, offset = (6, n), 1, None, None, 37
    elif layout == "channels_before":
        shape, axis, caxis, offsets, offset = (3, n), 1, 0, [0, 5, n - 3], 0
    elif layout == "channels_after":
        shape, axis, caxis, offsets, offset = (n, 3), 0, 1, [n, 11, 2], 0
    else:
        shape, axis, caxis, offsets, offset = (4, 2, n), 2, 1, [n // 2, n - 1], 0
    x = _data(rng, shape, complex_)
    want = fold_model(x, axis, size, offset, offsets, caxis)
    outer = int(np.prod(shape[:axis]))
    inner = int(np.prod(shape[axis + 1:]))
    out_shape = list(shape)
    out_shape[axis] = size
    xd = _dev(x)
    yd = _dev(np.zeros(out_shape, x.dtype))
    if offsets is None:
        od, channels, channel_inner = None, 0, 0
    else:
        od = _dev(np.asarray(offsets, np.uint64).view(np.int64))
        channels, channel_inner = len(offsets), int(np.prod(out_shape[caxis + 1:]))
    check(lib.b200_fold(ctx, ctypes.c_void_p(xd.data_ptr()), ctypes.c_void_p(yd.data_ptr()), int(complex_), outer, n,
                        inner, size, offset, ctypes.c_void_p(od.data_ptr()) if od is not None else None, channels,
                        channel_inner, _stream()))
    got = _host(yd)
    assert got.shape == want.shape
    assert np.array_equal(got, want)


def overlap_add_model(buf, ovl, prev, sample_axis, batch_axis):
    """OverlapAddImplNativeCpu: out = buf, + previous batch's overlap (batch 0: the carried tail); new tail = last batch."""
    out = buf.copy()
    k = ovl.shape[sample_axis]
    region = [slice(None)] * buf.ndim
    region[sample_axis] = slice(0, k)
    region = tuple(region)
    if batch_axis is None:
        add = prev
    else:
        shifted = np.roll(ovl, 1, axis=batch_axis)
        first = [slice(None)] * buf.ndim
        first[batch_axis] = slice(0, 1)
        shifted[tuple(first)] = prev
        add = shifted
    out[region] = out[region] + add
    new_prev = ovl.copy() if batch_axis is None else np.take(ovl, [ovl.shape[batch_axis] - 1], axis=batch_axis)
    return out, new_prev


@pytest.mark.parametrize("complex_", [False, True])
@pytest.mark.parametrize("shape,sample_axis,batch_axis,k", [((2, 50), 1, None, 7), ((4, 3, 50), 2, 0, 7),
                                                           ((50, 4), 0, 1, 9), ((3, 5, 2, 40), 1, 2, 5)])
def test_overlap_add_abi_bit_exact_with_state(abi, complex_, shape, sample_axis, batch_axis, k):
    lib, ctx, check = abi
    rng = np.random.default_rng(len(shape) * 10 + k)
    ovl_shape = list(shape)
    ovl_shape[sample_axis] = k
    prev_shape = list(ovl_shape)
    if batch_axis is not None:
        prev_shape[batch_axis] = 1
    dtype = np.complex64 if complex_ else np.float32
    prev = np.zeros(prev_shape, dtype)
    prev_d = _dev(prev)
    outer = int(np.prod(shape[:sample_axis]))
    inner = int(np.prod(shape[sample_axis + 1:]))
    batches = 1 if batch_axis is None else ovl_shape[batch_axis]
    stride = int(np.prod(ovl_shape)) if batch_axis is None else int(np.prod(ovl_shape[batch_axis + 1:]))
    for call in range(3):
        buf, ovl = _data(rng, shape, complex_), _data(rng, ovl_shape, complex_)
        want, prev = overlap_add_model(buf, ovl, prev, sample_axis, batch_axis)
        bd, od, yd = _dev(buf), _dev(ovl), _dev(np.zeros(shape, dtype))
        check(lib.b200_overlap_add(ctx, ctypes.c_void_p(bd.data_ptr()), ctypes.c_void_p(od.data_ptr()),
                                   ctypes.c_void_p(yd.data_ptr()), ctypes.c_void_p(prev_d.data_ptr()), int(complex_),
                                   outer, shape[sample_axis], k, inner, batches, stride, _stream()))
        assert np.array_equal(_host(yd), want), f"call {call}"
        assert np.array_equal(_host(prev_d), prev), f"state after call {call}"


def phase_model(x, phases, wrapped, batches, batch_inner, channels, channel_inner):
    """PhaseCorrectionImplNativeCpu::computeSubmit: F64 phase, F32 (cos, sin), std::complex<float> product."""
    k = np.arange(x.size)
    b = (k // batch_inner) % batches if batches > 1 else np.zeros_like(k)
    c = (k // channel_inner) % channels if channels > 1 else np.zeros_like(k)
    phi = np.asarray(phases)[c] + np.asarray(wrapped)[c] * b.astype(np.float64)
    cr, ci = np.cos(phi).astype(np.float32), np.sin(phi).astype(np.float32)
    xr, xi = x.reshape(-1).real.copy(), x.reshape(-1).imag.copy()
    out = np.empty(x.size, np.complex64)
    out.real = xr * cr - xi * ci
    out.imag = xr * ci + xi * cr
    return out.reshape(x.shape)


@pytest.mark.parametrize("shape,batch_axis,channel_axis", [((4, 64), 0, None), ((256,), None, None),
                                                           ((5, 3, 64), 0, 1), ((3, 128), None, 0),
                                                           ((3, 6, 32), 1, 0)])
def test_phase_correction_abi_with_carried_phase(abi, shape, batch_axis, channel_axis):
    lib, ctx, check = abi
    rng = np.random.default_rng(len(shape) + (batch_axis or 0) * 3)
    channels = shape[channel_axis] if channel_axis is not None else 1
    batches = shape[batch_axis] if batch_axis is not None else 1
    batch_inner = int(np.prod(shape[batch_axis + 1:])) if batch_axis is not None else 1
    channel_inner = int(np.prod(shape[channel_axis + 1:])) if channel_axis is not None else 1
    increments = [2.9 * (c + 1) - 7.5 for c in range(channels)]
    wrapped = [math.remainder(v, TWO_PI) for v in increments]
    phases = [0.0] * channels
    differing = 0
    for call in range(3):
        x = _data(rng, shape, True)
        want = phase_model(x, phases, wrapped, batches, batch_inner, channels, channel_inner)
        xd, yd = _dev(x), _dev(np.zeros(shape, np.complex64))
        ph = (ctypes.c_double * channels)(*phases)
        wr = (ctypes.c_double * channels)(*wrapped)
        check(lib.b200_phase_correction(ctx, ctypes.c_void_p(xd.data_ptr()), ctypes.c_void_p(yd.data_ptr()), x.size,
                                        batches, batch_inner, channels, channel_inner, ph, wr, _stream()))
        got = _host(yd)
        tol = 2 * np.spacing(np.abs(x).astype(np.float32))
        assert np.all(np.abs(got.real - want.real) <= tol) and np.all(np.abs(got.imag - want.imag) <= tol), f"call {call}"
        differing += int((got != want).sum())
        phases = [math.remainder(p + w * batches, TWO_PI) for p, w in zip(phases, wrapped)]
    print(f"phase_correction {shape}: {differing} of {3 * int(np.prod(shape))} elements not identical to the model")


def test_phase_correction_abi_rejects_too_many_channels(abi):
    lib, ctx, _ = abi
    n = 129
    xd = _dev(np.zeros(n, np.complex64))
    zeros = (ctypes.c_double * n)()
    assert lib.b200_phase_correction(ctx, ctypes.c_void_p(xd.data_ptr()), ctypes.c_void_p(xd.data_ptr()), n, 1, 1, n,
                                     1, zeros, zeros, _stream()) == 1
    assert b"channels" in lib.b200_last_error()


# ---- blocks in the reference Flowgraph, CPU provider vs provider b200 ----------------------------------------------

@pytest.fixture(scope="module")
def sb():
    from shim import binding
    if not binding.available():
        pytest.skip("oracle/_ref/shim/libjst_b200.so not built (needs the reference sources at build time)")
    return binding


def _cycles(shape, seed, complex_=True):
    rng = np.random.default_rng(seed)
    return [_data(rng, shape, complex_) for _ in range(3)]


def _run_graph(sb, build, feeds, reads):
    """build(session, target) wires the graph; feeds: {source: [3 arrays]}; reads: [(block, port)]. Returns
    {provider: [ {(block, port): array} per cycle ]}, {provider: session module table}."""
    outs, mods = {}, {}
    for target in (sb.CPU, sb.B200):
        with sb.Session() as s:
            blocks = build(s, target)
            per_cycle = []
            for k in range(3):
                for name, arrays in feeds.items():
                    s.write_source(name, arrays[k])
                s.compute()
                per_cycle.append({key: s.read(*key) for key in reads})
            outs[target[1]] = per_cycle
            table = {}
            for block in blocks:
                table.update(s.modules(block))
            mods[target[1]] = table
    return outs, mods


def _single(sb, block_type, config, port_in, reads, shape, axes, dtype="CF32", seed=0):
    cycles = _cycles(shape, seed, dtype == "CF32")

    def build(s, target):
        s.add_source("src", shape, dtype, target=target, **axes)
        s.add_block("dut", block_type, config, {port_in: "src.signal"}, target=target)
        return ["dut"]

    return _run_graph(sb, build, {"src": cycles}, [("dut", port) for port in reads])


@pytest.mark.parametrize("dtype", ["F32", "CF32"])
@pytest.mark.parametrize("shape,axis,size", [((6, 100), 1, 28), ((100,), 0, 1), ((3, 40, 5), 1, 12)])
def test_pad_block_bit_exact(sb, dtype, shape, axis, size):
    outs, mods = _single(sb, "pad", {"size": size, "axis": axis}, "unpadded", ["padded"], shape,
                         {"sampleAxis": len(shape) - 1}, dtype, seed=size)
    assert "runtime:pad" in mods["b200"], mods["b200"]
    for want, got in zip(outs["generic"], outs["b200"]):
        assert np.array_equal(got[("dut", "padded")], want[("dut", "padded")])


@pytest.mark.parametrize("dtype", ["F32", "CF32"])
@pytest.mark.parametrize("shape,axis,size", [((6, 100), 1, 28), ((3, 40, 5), 1, 12), ((2, 3, 50), 2, 10)])
def test_unpad_block_bit_exact(sb, dtype, shape, axis, size):
    outs, mods = _single(sb, "unpad", {"size": size, "axis": axis}, "padded", ["unpadded", "pad"], shape,
                         {"sampleAxis": len(shape) - 1}, dtype, seed=size + 1)
    assert "runtime:unpad" in mods["b200"], mods["b200"]
    for want, got in zip(outs["generic"], outs["b200"]):
        for port in ("unpadded", "pad"):
            assert np.array_equal(got[("dut", port)], want[("dut", port)]), port


@pytest.mark.parametrize("dtype", ["F32", "CF32"])
@pytest.mark.parametrize("shape,sample_axis,size,offset", [((4, 8100), 1, 810, 0), ((4, 8100), 1, 810, 4321),
                                                           ((360, 3), 0, 36, 7), ((2, 5, 64), 2, 64, 3)])
def test_fold_block_bit_exact(sb, dtype, shape, sample_axis, size, offset):
    outs, mods = _single(sb, "fold", {"size": size, "offset": offset}, "buffer", ["buffer"], shape,
                         {"sampleAxis": sample_axis}, dtype, seed=size + offset)
    assert "runtime:fold" in mods["b200"], mods["b200"]
    for want, got in zip(outs["generic"], outs["b200"]):
        assert np.array_equal(got[("dut", "buffer")], want[("dut", "buffer")])


@pytest.mark.parametrize("dtype", ["F32", "CF32"])
@pytest.mark.parametrize("shape,k,axes", [((8, 2, 800), 10, {"sampleAxis": 2, "batchAxis": 0}),
                                          ((3, 200), 17, {"sampleAxis": 1}),
                                          ((200, 4), 9, {"sampleAxis": 0, "batchAxis": 1})])
def test_overlap_add_block_bit_exact_with_state(sb, dtype, shape, k, axes):
    ovl_shape = list(shape)
    ovl_shape[axes["sampleAxis"]] = k
    bufs = _cycles(shape, 3, dtype == "CF32")
    ovls = _cycles(tuple(ovl_shape), 4, dtype == "CF32")

    def build(s, target):
        s.add_source("buf", shape, dtype, target=target, **axes)
        s.add_source("ovl", tuple(ovl_shape), dtype, target=target, **axes)
        s.add_block("dut", "overlap_add", None, {"buffer": "buf.signal", "overlap": "ovl.signal"}, target=target)
        return ["dut"]

    outs, mods = _run_graph(sb, build, {"buf": bufs, "ovl": ovls}, [("dut", "buffer")])
    assert mods["b200"]["runtime:overlap_add"][0] == 3, mods["b200"]
    for cycle, (want, got) in enumerate(zip(outs["generic"], outs["b200"])):
        assert np.array_equal(got[("dut", "buffer")], want[("dut", "buffer")]), f"cycle {cycle}"


@pytest.mark.parametrize("shape,axes,increment", [((6, 256), {"sampleAxis": 1, "batchAxis": 0}, 1.234),
                                                  ((512,), {"sampleAxis": 0}, -2.5),
                                                  ((4, 3, 64), {"sampleAxis": 2, "batchAxis": 1}, 10.0)])
def test_phase_correction_block_with_carried_phase(sb, shape, axes, increment):
    outs, mods = _single(sb, "phase_correction", {"phaseIncrement": increment}, "signal", ["signal"], shape, axes,
                         seed=int(abs(increment) * 10))
    assert mods["b200"]["runtime:phase_correction"][0] == 3, mods["b200"]
    differing = 0
    for cycle, (want, got) in enumerate(zip(outs["generic"], outs["b200"])):
        w, g = want[("dut", "signal")], got[("dut", "signal")]
        # |x| = |w| up to rounding: the correction is a unit phasor
        tol = 2 * np.spacing(np.abs(w).astype(np.float32))
        assert np.all(np.abs(g.real - w.real) <= tol) and np.all(np.abs(g.imag - w.imag) <= tol), f"cycle {cycle}"
        differing += int((g != w).sum())
    print(f"phase_correction block {shape}: {differing} of {3 * int(np.prod(shape))} elements not identical")


def _rel(got, want):
    return float(np.abs(got - want).max() / np.abs(want).max())


@pytest.mark.parametrize("heads,center", [(1, [0.0]), (3, [0.0, 1e6, -2e6])])
@pytest.mark.parametrize("shape,axes", [((4096, 3), {"sampleAxis": 0, "batchAxis": 1}),
                                        ((3, 2, 2048), {"sampleAxis": 2, "batchAxis": 0})])
def test_filter_block_unfused_layouts(sb, heads, center, shape, axes):
    """Layouts the fused FIR does not take (sample axis not innermost; rank 3) run the reference wiring on this
    provider's modules: fold with per-head offsets, phase_correction, unpad and overlap_add on the GPU."""
    cfg = {"sampleRate": 8e6, "bandwidth": 1e6, "taps": 129, "heads": heads, "center": center}
    outs, mods = _single(sb, "filter", cfg, "signal", ["buffer"], shape, axes, seed=heads)
    assert "runtime:fold" in mods["b200"] and "runtime:overlap" in mods["b200"], mods["b200"]
    assert "runtime:fir" not in mods["b200"]
    assert (heads > 1) == ("runtime:phase_correction" in mods["b200"])
    for cycle, (want, got) in enumerate(zip(outs["generic"], outs["b200"])):
        w, g = want[("dut", "buffer")], got[("dut", "buffer")]
        assert g.shape == w.shape
        err = _rel(g, w)
        print(f"filter {shape} heads={heads} cycle {cycle}: max|d|/max|want| = {err:.2e}")
        assert err <= 1e-5, f"cycle {cycle}: {err:.3e}"


@pytest.mark.parametrize("taps_cfg", [
    {"taps": 101, "heads": 2, "center": [400e3, -400e3], "bandwidth": 200e3, "sampleRate": 2e6},
    {"taps": 101, "heads": 2, "center": [0.0, 0.0], "bandwidth": 200e3, "sampleRate": 2e6},
    {"taps": 101, "heads": 1, "center": [0.0], "bandwidth": 300e3, "sampleRate": 2e6},
], ids=["resample_offset_heads", "resample_centred", "full_rate"])
def test_filter_engine_block(sb, taps_cfg):
    """filter_engine as in the Overlap-Add-Fold example: source [8, 8000] CF32 -> filter_taps -> filter_engine. The
    first case resamples by 10 with fold offsets of +-1620 bins and phase correction; the last bypasses resampling
    (2 MS/s over 300 kHz is not an integer ratio)."""
    shape = (8, 8000)
    cycles = _cycles(shape, 42)

    def build(s, target):
        s.add_source("src", shape, "CF32", target=target, sampleAxis=1, batchAxis=0)
        s.add_block("taps", "filter_taps", taps_cfg, {}, target=target)
        s.add_block("fe", "filter_engine", None, {"signal": "src.signal", "filter": "taps.coeffs"}, target=target)
        return ["taps", "fe"]

    outs, mods = _run_graph(sb, build, {"src": cycles}, [("fe", "buffer")])
    if taps_cfg["bandwidth"] == 200e3:
        assert "runtime:fold" in mods["b200"], mods["b200"]
    for cycle, (want, got) in enumerate(zip(outs["generic"], outs["b200"])):
        w, g = want[("fe", "buffer")], got[("fe", "buffer")]
        assert g.shape == w.shape
        err = _rel(g, w)
        print(f"filter_engine {taps_cfg['center']} bw={taps_cfg['bandwidth']} cycle {cycle}: max|d|/max|want| = {err:.2e}")
        assert err <= 1e-5, f"cycle {cycle}: {err:.3e}"


def test_overlap_add_fold_flowgraph(sb):
    """examples/flowgraphs/overlap-add-fold.yml in small, wired by hand: pad -> fft -> expand_dims -> multiply (with
    filter_taps -> pad -> fft) -> fold(810) -> fft(inverse) -> unpad -> overlap_add."""
    shape = (8, 8000)
    cycles = _cycles(shape, 7)

    def build(s, target):
        s.add_source("src", shape, "CF32", target=target, sampleAxis=1, batchAxis=0)
        s.add_block("pad_src", "pad", {"axis": 1, "size": 100}, {"unpadded": "src.signal"}, target=target)
        s.add_block("fft_src", "fft", {"forward": True}, {"signal": "pad_src.padded"}, target=target)
        s.add_block("exp", "expand_dims", {"axis": 1}, {"buffer": "fft_src.signal"}, target=target)
        s.add_block("flt", "filter_taps", {"taps": 101, "heads": 2, "center": [400e3, -400e3], "bandwidth": 200e3,
                                           "sampleRate": 2e6}, {}, target=target)
        s.add_block("pad_flt", "pad", {"axis": 1, "size": 7999}, {"unpadded": "flt.coeffs"}, target=target)
        s.add_block("fft_flt", "fft", {"forward": True}, {"signal": "pad_flt.padded"}, target=target)
        s.add_block("mul", "multiply", None, {"a": "exp.buffer", "b": "fft_flt.signal"}, target=target)
        s.add_block("fold", "fold", {"size": 810, "offset": 0}, {"buffer": "mul.product"}, target=target)
        s.add_block("ifft", "fft", {"forward": False}, {"signal": "fold.buffer"}, target=target)
        s.add_block("unpad", "unpad", {"axis": 2, "size": 10}, {"padded": "ifft.signal"}, target=target)
        s.add_block("ola", "overlap_add", None, {"buffer": "unpad.unpadded", "overlap": "unpad.pad"}, target=target)
        return ["pad_src", "fold", "unpad", "ola"]

    outs, mods = _run_graph(sb, build, {"src": cycles}, [("ola", "buffer")])
    assert mods["b200"]["runtime:overlap_add"][0] == 3 and mods["b200"]["runtime:fold"][0] == 3, mods["b200"]
    for cycle, (want, got) in enumerate(zip(outs["generic"], outs["b200"])):
        w, g = want[("ola", "buffer")], got[("ola", "buffer")]
        assert g.shape == w.shape == (8, 2, 800)
        err = _rel(g, w)
        print(f"overlap-add-fold cycle {cycle}: max|d|/max|want| = {err:.2e}")
        assert err <= 1e-5, f"cycle {cycle}: {err:.3e}"
