"""The index algebra of the two FFT kernels, emulated in numpy (F64) against np.fft: the 16x16x16 three-pass
scheme of fft4096_kernel (including both shared-memory exchange layouts) and the generic Stockham passes."""
import os
import re
from collections import defaultdict

import numpy as np

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "cyberether_b200", "csrc")


def W(n, e):
    return np.exp(-2j * np.pi * (e % n) / n)


def dft16(v):
    v = v.copy()

    def b4(a, b, c, d):
        s0, s1, s2, s3 = a + c, a - c, b + d, b - d
        return s0 + s2, s1 - 1j * s3, s0 - s2, s1 + 1j * s3
    for a0 in range(4):
        v[a0], v[a0 + 4], v[a0 + 8], v[a0 + 12] = b4(v[a0], v[a0 + 4], v[a0 + 8], v[a0 + 12])
    for a0 in range(4):
        for q in range(4):
            v[a0 + 4 * q] *= W(16, a0 * q)
    for q in range(4):
        v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3] = b4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3])
    return np.array([v[4 * (k & 3) + (k >> 2)] for k in range(16)])      # dft16_pos


def test_dft16_4x4_decomposition():
    rng = np.random.default_rng(0)
    x = rng.standard_normal(16) + 1j * rng.standard_normal(16)
    assert np.abs(dft16(x) - np.fft.fft(x)).max() < 1e-12


def test_fft4096_three_pass_scheme_with_padded_exchange():
    rng = np.random.default_rng(1)
    x = rng.standard_normal(4096) + 1j * rng.standard_normal(4096)
    stage = np.zeros(16 * 288, complex)                 # kFft4096X2Plane = 288, row pitch 18
    for t in range(256):                                # pass 1: thread t, registers a
        y = dft16(np.array([x[t + 256 * a] for a in range(16)]))
        for k0 in range(16):
            stage[256 * k0 + t] = y[k0] * W(4096, t * k0)
    regs = {}
    for t in range(256):                                # pass 2: t = 16 k0 + c, reads 256 k0 + 16 b + c
        k0, c = t >> 4, t & 15
        y = dft16(np.array([stage[256 * k0 + 16 * b + c] for b in range(16)]))
        regs[t] = [y[k1] * W(256, c * k1) for k1 in range(16)]
    for t in range(256):                                # exchange-2 stores (after the split barrier)
        k0, c = t >> 4, t & 15
        for k1 in range(16):
            stage[288 * k1 + 18 * k0 + c] = regs[t][k1]
    out = np.zeros(4096, complex)
    for t in range(256):                                # pass 3: t = k0 + 16 k1
        k0, k1 = t & 15, t >> 4
        y = dft16(np.array([stage[288 * k1 + 18 * k0 + c] for c in range(16)]))
        for k2 in range(16):
            out[t + 256 * k2] = y[k2]
    assert np.abs(out - np.fft.fft(x)).max() < 1e-9


def test_exchange_layouts_are_bank_conflict_free():
    """8-byte elements: a half-warp (16 lanes) must touch 16 distinct (address / 8) mod 16 classes."""
    for w in range(8):
        for half in range(2):
            lanes = [32 * w + 16 * half + i for i in range(16)]
            for k in range(16):
                assert len({(256 * k + t) % 16 for t in lanes}) == 16                        # pass-1 load/store
                assert len({(256 * (t >> 4) + 16 * k + (t & 15)) % 16 for t in lanes}) == 16     # exchange-1 load
                assert len({(288 * k + 18 * (t >> 4) + (t & 15)) % 16 for t in lanes}) == 16     # exchange-2 store
    # exchange-2 load is LDS.128 (2 elements): a quarter-warp (8 lanes) must cover all 32 banks
    for w in range(8):
        for quarter in range(4):
            lanes = [32 * w + 8 * quarter + i for i in range(8)]
            for c in range(0, 16, 2):
                banks = set()
                for t in lanes:
                    base = (288 * (t >> 4) + 18 * (t & 15) + c) * 2          # 4-byte words
                    banks.update((base + j) % 32 for j in range(4))
                assert len(banks) == 32


def stockham(x):
    n = len(x)
    log2n = int(np.log2(n))
    buf = x.astype(complex).copy()
    ns = 1
    if log2n % 2 == 1:
        new = np.zeros(n, complex)
        for j in range(n // 2):
            new[2 * j], new[2 * j + 1] = buf[j] + buf[j + n // 2], buf[j] - buf[j + n // 2]
        buf, ns = new, 2
    while ns < n:
        new = np.zeros(n, complex)
        shift = n // (4 * ns)
        for j in range(n // 4):
            k = j % ns
            u = [buf[j + t * (n // 4)] * W(n, k * t * shift) for t in range(4)]
            s0, s1, s2, s3 = u[0] + u[2], u[0] - u[2], u[1] + u[3], u[1] - u[3]
            y = [s0 + s2, s1 - 1j * s3, s0 - s2, s1 + 1j * s3]
            j0 = ((j - k) << 2) + k
            for t in range(4):
                new[j0 + t * ns] = y[t]
        buf, ns = new, ns * 4
    return buf


def test_generic_stockham_passes():
    rng = np.random.default_rng(2)
    for n in (2, 4, 8, 16, 32, 64, 512, 2048):
        x = rng.standard_normal(n) + 1j * rng.standard_normal(n)
        assert np.abs(stockham(x) - np.fft.fft(x)).max() < 1e-10 * n


def test_inverse_by_swapping_parts():
    rng = np.random.default_rng(3)
    x = rng.standard_normal(64) + 1j * rng.standard_normal(64)
    sw = lambda z: z.imag + 1j * z.real
    assert np.abs(sw(np.fft.fft(sw(x))) - np.fft.ifft(x) * 64).max() < 1e-12


def test_fir_polyphase_plane_indexing():
    """fir_decim_kernel: sample i of the staged span -> plane i mod R, row i div R; tap k of output o reads plane
    (-k) mod R at row o + hpad - m - (plane != 0), k = kp0 + m R."""
    rng = np.random.default_rng(4)
    for (L, R, qt, ob) in [(129, 8, 21, 7), (33, 4, 10, 5), (17, 1, 9, 3), (41, 40, 6, 1), (7, 3, 14, 7)]:
        lp = -(-L // R)
        lp_pad = -(-lp // ob) * ob
        hpad = lp_pad + 1
        h = rng.standard_normal(L)
        xs = rng.standard_normal(qt * R + hpad * R)          # stream; tile starts at q0 R = hpad R
        span = (qt - 1) * R + hpad * R + 1
        planes = np.zeros((R, qt + hpad + 1))
        for i in range(span):
            planes[i % R, i // R] = xs[i]
        for o in range(qt):
            acc = 0.0
            for plane in range(R):
                kp0 = (R - plane) % R
                d = hpad if plane == 0 else hpad - 1
                for m in range(lp_pad):
                    k = kp0 + m * R
                    tap = h[k] if k < L else 0.0
                    acc += tap * planes[plane, o + d - m]
            want = sum(h[k] * xs[(o + hpad) * R - k] for k in range(L))
            assert abs(acc - want) < 1e-9


def test_fir_chunk_pair_form():
    """fir_decim_kernel<.., PAIR>: the same plane algebra on 16-byte chunks (x[2n], x[2n+1]) with decimation R / 2 and
    chunk-taps g[c] = (h[2c], h[2c-1]): y[q] = sum_c h[2c] x[qR - 2c] + h[2c-1] x[qR - 2c + 1]."""
    rng = np.random.default_rng(6)
    for (L, R, qt, ob) in [(127, 8, 21, 7), (129, 8, 14, 7), (33, 4, 10, 5), (41, 40, 6, 1), (7, 2, 9, 3), (161, 40, 7, 7)]:
        C, R2 = (L + 1) // 2, R // 2
        lp = -(-C // R2)
        lp_pad = -(-lp // ob) * ob
        hpad = lp_pad + 1
        h = rng.standard_normal(L) + 1j * rng.standard_normal(L)      # complex taps: a frequency-translating head
        g = np.zeros((C, 2), complex)
        for c in range(C):
            g[c, 0] = h[2 * c]
            g[c, 1] = h[2 * c - 1] if c > 0 else 0.0
        xs = rng.standard_normal((qt + hpad) * R) + 1j * rng.standard_normal((qt + hpad) * R)   # tile starts at q0 R = hpad R
        chunks = xs.reshape(-1, 2)                           # chunk n = (x[2n], x[2n+1])
        span = (qt - 1) * R2 + hpad * R2 + 1
        planes = np.zeros((R2, qt + hpad + 1, 2), complex)
        for i in range(span):
            planes[i % R2, i // R2] = chunks[i]
        for o in range(qt):
            acc = 0.0
            for plane in range(R2):
                kp0 = (R2 - plane) % R2
                d = hpad if plane == 0 else hpad - 1
                for m in range(lp_pad):
                    c = kp0 + m * R2
                    if c < C:
                        v = planes[plane, o + d - m]
                        acc += g[c, 0] * v[0] + g[c, 1] * v[1]
            want = sum(h[k] * xs[(o + hpad) * R - k] for k in range(L))
            assert abs(acc - want) < 1e-9, (L, R, o)


def _fir_thread_loop(planes, taps, R, C, ob, o0, hpad, lp_pad, mul):
    """One thread of fir_decim_kernel as written: outputs o0 .. o0 + OB - 1 of a tile from `planes` (rows of staged
    elements per plane, None where nothing is staged) and the host's re-ordered tap table taps[plane][slot] (padded
    slots hold a poison value). Window element i lives in w[(i - s) mod OB]; after tap step s, w[(OB - 1 - s) mod OB]
    takes xq[-s - 1]; the OB-wide blocks run `full` taps, the tail loop `rem`; plane p holds lp_plane taps, from lp_thr
    without a division. C = taps in element units (L, or (L + 1) / 2 chunk-taps)."""
    lp = -(-C // R)
    lp_thr = C - (lp - 1) * R
    acc = [0] * ob
    for plane in range(R):
        d = hpad if plane == 0 else hpad - 1
        row = o0 + d                                        # xp = planes[plane] + o0 + d
        w = [planes[plane][row + i] for i in range(ob)]
        kp0 = 0 if plane == 0 else R - plane
        lp_plane = lp - (1 if kp0 >= lp_thr else 0)
        full = lp_plane // ob * ob
        slot = 0

        def tap_step(s):
            h = taps[plane][slot + s]
            for i in range(ob):
                v = w[(i - s) % ob]
                assert v is not None, "the loop read an element the tile did not stage"
                acc[i] += mul(h, v)
            assert row - s - 1 >= 0, "the slide reads below the tile"
            w[(ob - 1 - s) % ob] = planes[plane][row - s - 1]
        for _ in range(0, full, ob):
            for s in range(ob):
                tap_step(s)
            row -= ob
            slot += ob
        for s in range(ob - 1):
            if s < lp_plane - full:
                tap_step(s)
        assert slot + lp_plane - full <= lp_pad
    return acc


def _fir_tile(elements, R, qt, hpad):
    """Stage a tile starting at output q0 = hpad (stream index j0 = 0) the way the kernel does: element i -> plane
    i mod R, row i div R, for the span of (qt - 1) R + hpad R + 1 elements."""
    span = (qt - 1) * R + hpad * R + 1
    planes = [[None] * (qt + hpad + 1) for _ in range(R)]
    for i in range(span):
        planes[i % R][i // R] = elements[i]
    return planes


def _fir_table(g, R, C, lp_pad, poison):
    """Host re-ordering: plane p, slot m <- g[kp0 + m R], kp0 = (R - p) mod R; poison beyond C."""
    return [[g[(R - p) % R + m * R] if (R - p) % R + m * R < C else poison for m in range(lp_pad)] for p in range(R)]


def test_fir_thread_tap_loop_equals_direct_convolution():
    """The thread loop of fir_decim_kernel (window rotation, slide, full / rem split, lp_plane from lp_thr) replayed
    with integers for OB = 1, 3, 5, 7, every L <= 70 and R <= 20 (L < R, L = k R, L = k R + 1 among them), for the
    first and the last thread of a tile: equal to y[q] = sum_k h[k] x[q R - k]. Padded tap slots hold a poison value,
    so a loop that multiplies one instead of skipping it fails; reads of unstaged rows fail too."""
    rng = np.random.default_rng(11)
    poison = 10 ** 9
    for ob in (1, 3, 5, 7):
        threads = 2
        qt = threads * ob
        for R in range(1, 21):
            for L in range(1, 71):
                lp = -(-L // R)
                lp_pad = -(-lp // ob) * ob
                hpad = lp_pad + 1
                h = [int(v) for v in rng.integers(1, 9, L) * rng.choice([-1, 1], L)]
                x = [int(v) for v in rng.integers(1, 9, (qt + hpad) * R) * rng.choice([-1, 1], (qt + hpad) * R)]
                planes = _fir_tile(x, R, qt, hpad)
                table = _fir_table(h, R, L, lp_pad, poison)
                for t in range(threads):
                    got = _fir_thread_loop(planes, table, R, L, ob, t * ob, hpad, lp_pad, lambda a, b: a * b)
                    for i in range(ob):
                        q = hpad + t * ob + i
                        want = sum(h[k] * x[q * R - k] for k in range(L))
                        assert got[i] == want, (ob, L, R, t, i)


def test_fir_pair_thread_tap_loop_equals_direct_convolution():
    """The same loop in the chunk-pair form: elements are chunks (x[2n], x[2n+1]), decimation R / 2, chunk-taps
    g[c] = (h[2c], h[2c-1]) with h[-1] = 0, for odd L <= 69 and even R <= 20 (complex integer taps and samples)."""
    rng = np.random.default_rng(12)
    poison = (10 ** 9, 10 ** 9)

    def rnd(n):
        return [complex(a, b) for a, b in rng.integers(1, 9, (n, 2)) * rng.choice([-1, 1], (n, 2))]
    for ob in (1, 3, 5, 7):
        threads = 2
        qt = threads * ob
        for R in range(2, 21, 2):
            R2 = R // 2
            for L in range(1, 70, 2):
                C = (L + 1) // 2
                lp = -(-C // R2)
                lp_pad = -(-lp // ob) * ob
                hpad = lp_pad + 1
                h = rnd(L)
                x = rnd((qt + hpad) * R)
                g = [(h[2 * c], h[2 * c - 1] if c > 0 else 0) for c in range(C)]
                chunks = [(x[2 * n], x[2 * n + 1]) for n in range(len(x) // 2)]
                planes = _fir_tile(chunks, R2, qt, hpad)
                table = _fir_table(g, R2, C, lp_pad, poison)
                for t in range(threads):
                    got = _fir_thread_loop(planes, table, R2, C, ob, t * ob, hpad, lp_pad,
                                           lambda gc, v: gc[0] * v[0] + gc[1] * v[1])
                    for i in range(ob):
                        q = hpad + t * ob + i
                        want = sum(h[k] * x[q * R - k] for k in range(L))
                        assert got[i] == want, (ob, L, R, t, i)


def _radices(log2n):
    rem, out = 1 << log2n, []
    while rem > 1:
        r = min(16, rem)
        out.append(r)
        rem //= r
    return out


def test_fft_radix_kernel_padded_stockham_scheme():
    """fft_radix_kernel (16 <= N <= 8192): block of THREADS*16 samples, passes ping-pong between the exchange
    buffer and the stage buffer through pad(a) = a + a/16; checks the result and that every exchange store of a
    half-warp hits 16 distinct 8-byte bank pairs."""
    pad = lambda a: a + (a >> 4)
    for log2n in range(4, 14):
        n, rad = 1 << log2n, _radices(log2n)
        threads = max(256, n // 16)
        block, t_per_row = threads * 16, n // 16
        rows = block // n
        rng = np.random.default_rng(log2n)
        x = rng.standard_normal(block) + 1j * rng.standard_normal(block)
        bufs = [np.zeros(block + block // 16 + 16, complex) for _ in range(2)]
        bufs[0][:block] = x                                   # the TMA lands the block linearly
        out = np.zeros(block, complex)
        ns = 1
        for p, r in enumerate(rad):
            last = p == len(rad) - 1
            src, dst = bufs[p % 2], bufs[(p + 1) % 2]
            writes = []
            for tid in range(threads):
                g, lt = tid // t_per_row, tid % t_per_row
                for b in range(16 // r):
                    j = lt + b * t_per_row
                    k = j & (ns - 1)
                    u = [src[(g * n + j + t * (n // r)) if p == 0 else pad(g * n + j + t * (n // r))] for t in range(r)]
                    w = np.exp(-2j * np.pi * k / (r * ns))
                    y = np.fft.fft(np.array([u[t] * w ** t for t in range(r)]))
                    j0 = (j - k) * r + k
                    for t in range(r):
                        a = g * n + j0 + t * ns
                        if last:
                            out[a] = y[t]
                        else:
                            writes.append((pad(a), y[t], tid, b, t))
            banks = defaultdict(list)
            for a, val, tid, b, t in writes:
                dst[a] = val
                banks[(tid // 16, b, t)].append(a % 16)
            assert all(len(set(v)) == len(v) for v in banks.values()), (log2n, p)
            ns *= r
        want = np.fft.fft(x.reshape(rows, n), axis=1).reshape(-1)
        assert np.abs(out - want).max() < 1e-9 * n, log2n


_KERNEL_MODES = {"MODE_C2C": 0, "MODE_AMP": 1, "MODE_AMP_RANGE": 2, "MODE_C2C_T": 3, "MODE_R2C": 4}   # fft_common.cuh


def _radix_kernel_code():
    """fft_radix_kernel's source from its signature on, comments removed, and the part from its epilogue on."""
    with open(os.path.join(CSRC, "fft_radix.cuh")) as f:
        text = f.read()
    kernel = text[text.index("fft_radix_kernel(const FftParams p)"):]
    strip = lambda s: re.sub(r"//[^\n]*", "", s)
    return strip(kernel), strip(kernel[kernel.index("// ---- epilogue"):])


def _radix_block_end(epilogue):
    """The kernel code between a block's epilogue (an if / else chain) and the ring-index update that ends the block."""
    i = epilogue.index("{")
    while True:
        depth = 0
        for j in range(i, len(epilogue)):
            depth += {"{": 1, "}": -1}.get(epilogue[j], 0)
            if depth == 0:
                break
        rest = epilogue[j + 1:]
        if not rest.lstrip().startswith("else"):
            return rest[:rest.index("refill_stage = stage;")]
        i = j + 1 + rest.index("{")


def _radix_block_end_fences(tail, mode, log2n):
    """The __syncthreads / __syncwarp statements of the block end, with their `if constexpr` guards evaluated for
    (mode, log2n)."""
    names = dict(_KERNEL_MODES, MODE=_KERNEL_MODES[mode], LOG2N=log2n, N=1 << log2n, T=(1 << log2n) // 16,
                 PASSES=(log2n + 3) // 4)
    fences = []
    for m in re.finditer(r"if constexpr \(([^{}]*)\)\s*\{([^{}]*)\}|(__syncthreads|__syncwarp)\(\)", tail):
        if m.group(3):
            fences.append(m.group(3))
        elif eval(m.group(1).replace("&&", " and ").replace("||", " or "), {"__builtins__": {}}, names):
            fences += re.findall(r"__syncthreads|__syncwarp", m.group(2))
    return fences


_RADIX_SYNCTHREADS_IN_BODY = 7      # the __syncthreads statements of the kernel outside the block-end fences


def _radix_kernel_schedule(log2n, mode, block_end_fences, blocks=3, my_blocks=5):
    """Program order of every thread of one fft_radix_kernel<log2n, mode> CTA over its first `blocks` blocks (of
    `my_blocks`): ("r" | "w", buffer, element) shared-memory accesses with buffer "stage0", "stage1" or "x1", ("sync",)
    for __syncthreads, ("syncwarp",), ("wait", block) for mbar_wait on the block's stage and ("tma", stage, block) for a
    bulk copy of `block` into `stage` issued by thread 0."""
    n, rad = 1 << log2n, _radices(log2n)
    threads, t_per_row, passes = max(256, n // 16), n // 16, len(rad)
    pad = lambda a: a + (a >> 4)
    program = []
    for tid in range(threads):
        ev, (g, lt) = [], divmod(tid, t_per_row)
        row = g * n
        issued = 0

        def refill(stage):
            nonlocal issued
            if issued < my_blocks:
                if tid == 0:
                    ev.append(("tma", stage, issued))
                issued += 1

        ev.append(("sync",))                                  # after the mbarrier init
        for s in range(2):
            refill(s)
        stage, refill_stage = 0, 0
        for i in range(blocks):
            sb = f"stage{stage}"
            ev.append(("wait", i))
            ev += [("r", sb, row + lt + t * t_per_row) for t in range(16)]          # pass 0 reads the linear TMA block
            if passes == 1:
                ev.append(("sync",))
                refill(stage)
            else:
                ev += [("w", "x1", pad(row + lt * 16 + t)) for t in range(16)]
                ev.append(("sync",))
                if i >= 1:
                    refill(refill_stage)
                r1 = rad[1]
                for b in range(16 // r1):                     # pass 1 reads X1, writes the stage buffer unless last
                    j = lt + b * t_per_row
                    k = j & 15
                    ev += [("r", "x1", pad(row + j + t * (n // r1))) for t in range(r1)]
                    if passes > 2:
                        ev += [("w", sb, pad(row + (j - k) * r1 + k + t * 16)) for t in range(r1)]
            if passes > 2:
                ev.append(("sync",))
                r2 = rad[2]
                for b in range(16 // r2):                     # pass 2 reads the stage buffer, writes X1 unless last
                    j = lt + b * t_per_row
                    k = j & 255
                    ev += [("r", sb, pad(row + j + t * (n // r2))) for t in range(r2)]
                    if passes > 3:
                        ev += [("w", "x1", pad(row + (j - k) * r2 + k + t * 256)) for t in range(r2)]
            if passes > 3:
                ev.append(("sync",))
                for b in range(8):                            # pass 3 (radix 2) reads X1
                    j = lt + b * t_per_row
                    ev += [("r", "x1", pad(row + j)), ("r", "x1", pad(row + j + n // 2))]
            if mode == "MODE_R2C":                            # Z through the buffer the last pass did not read
                rl = rad[-1]
                zbuf = "x1" if passes % 2 == 1 else sb
                ev += [("w", zbuf, row + lt + b * t_per_row + t * (n // rl)) for b in range(16 // rl) for t in range(rl)]
                ev.append(("sync",))
                for j in range(9):
                    k = lt + j * t_per_row
                    if j == 8 and lt != 0:
                        break
                    ev += [("r", zbuf, row)] if k == 0 else [("r", zbuf, row + k), ("r", zbuf, row + n - k)]
                if passes % 2 == 1:
                    ev.append(("sync",))
            # the C2C, C2C_T and spectral epilogues go from registers to global memory
            ev += [("sync",) if f == "__syncthreads" else ("syncwarp",) for f in block_end_fences]
            refill_stage, stage = stage, stage ^ 1
        program.append(ev)
    return program


def _schedule_races(program):
    """Unordered pairs in a schedule. Generic accesses: different threads, the same element, at least one write, no
    __syncthreads between them, and (same warp) no __syncwarp between them. A bulk copy into a stage is in flight from
    its issue by thread 0 until each thread's wait for that block; any generic access to the stage meanwhile races."""
    by_element = defaultdict(list)
    stage_access, tma, waits = [], [], {}
    for tid, ev in enumerate(program):
        interval = epoch = 0
        for pos, e in enumerate(ev):
            if e[0] == "sync":
                interval += 1
                epoch += 1
            elif e[0] == "syncwarp":
                epoch += 1
            elif e[0] == "wait":
                waits[tid, e[1]] = pos
            elif e[0] == "tma":
                tma.append((e[1], e[2], interval, pos))
            else:
                by_element[interval, e[1], e[2]].append((tid, e[0] == "w", epoch))
                if e[1].startswith("stage"):
                    stage_access.append((tid, interval, pos, int(e[1][-1])))
    races = []
    for (interval, buf, elem), acc in by_element.items():
        if len(acc) < 2 or not any(w for _, w, _ in acc):
            continue
        for a, (ta, wa, ea) in enumerate(acc):
            for tb, wb, eb in acc[a + 1:]:
                if ta != tb and (wa or wb) and not (ta // 32 == tb // 32 and ea != eb):
                    races.append(f"{buf}[{elem}]: threads {ta} and {tb} after barrier {interval}")
    tid, interval, pos, stage = np.array(stage_access).T
    for s, block, issue_interval, issue_pos in tma:
        wait_pos = np.array([waits.get((t, block), 1 << 62) for t in range(len(program))])
        after_issue = (interval > issue_interval) | ((interval == issue_interval) & ((tid != 0) | (pos > issue_pos)))
        hit = (stage == s) & after_issue & (pos < wait_pos[tid])
        if hit.any():
            races.append(f"stage{s} refill with block {block}: thread {tid[hit][0]} touches it while in flight")
    return races


def test_fft_radix_kernel_schedule_is_race_free_across_consecutive_blocks():
    """fft_radix_kernel is persistent: a CTA runs blocks first, first + gridDim.x, ... whenever the batch exceeds the grid,
    so one block's last exchange reads meet the next block's first exchange stores, and the two-stage TMA ring wraps. For
    every length and mode family (C2C / C2C_T, amplitude / range, R2C) the model below replays three consecutive blocks of
    one CTA and checks that every pair of shared-memory accesses that could race is ordered.

    The model is a hand restatement of fft_radix.cuh: a change to the kernel's shared-memory schedule must change the
    model too. Two parts are read from the kernel source instead: the fences between a block's epilogue and the next
    block (so the test checks the kernel as it is), and the number of __syncthreads statements, which must match the
    restatement."""
    code, epilogue = _radix_kernel_code()
    tail = _radix_block_end(epilogue)
    failures = []
    for mode in ("MODE_C2C", "MODE_AMP_RANGE", "MODE_R2C"):
        for log2n in range(5 if mode == "MODE_R2C" else 4, 14):
            fences = _radix_block_end_fences(tail, mode, log2n)
            races = _schedule_races(_radix_kernel_schedule(log2n, mode, fences))
            if races:
                failures.append(f"LOG2N={log2n} {mode}: {len(races)} races, e.g. {races[0]}")
    assert not failures, "\n".join(failures)
    assert code.count("__syncthreads()") == _RADIX_SYNCTHREADS_IN_BODY + tail.count("__syncthreads()")


def test_fm_nco_wrap_identity_exhaustive():
    """fm.cu:nco_step replaces the reference's F64 wrap `(float)((double)a - 2 pi)` (taken when (double)a >= 2 pi,
    src/domains/dsp/fm/module_impl_native_cpu.cc NCO update) by fadd(fsub(a, T), C) and the test by a >= T, T = the F32
    just above 2 pi. Both are checked for EVERY F32 a in [T, T + 1) and around the threshold."""
    import numpy as np
    two_pi = 2.0 * 3.14159265358979323846
    t = np.float32(6.2831854820251465)
    c = np.float32(1.7484555314695172e-07)
    assert float(t) >= two_pi > float(np.nextafter(t, np.float32(0)))          # (double)a >= 2 pi  <=>  a >= T
    assert c == np.float32(float(t) - two_pi)
    lo = np.array([t], np.float32).view(np.uint32)[0]
    hi = np.array([t + np.float32(1.0)], np.float32).view(np.uint32)[0]
    a = np.arange(lo, hi, dtype=np.uint32).view(np.float32)
    reference = (a.astype(np.float64) - two_pi).astype(np.float32)
    ours = ((a - t).astype(np.float32) + c).astype(np.float32)
    assert len(a) == 1 << 21 and np.array_equal(reference, ours)


def test_fm_wide_nco_orbit_table_reproduces_the_serial_walk():
    """The wideband pilot NCO is an F32 running sum with wrap (fm/module_impl_native_cpu.cc:172-175). Its state is
    one float and the update is input independent, so the sequence is eventually periodic; the plan walks the orbit
    once and regenerates any slice in parallel (fm_wide_phase_table_kernel). Host twin of that bookkeeping
    (b200_fm_nco_phases_host) against a plain serial F32 walk, for sample rates from 200 kHz to 20 MHz (1.024 MHz has a
    transient of 5 M samples before its period), at the stream start, across the transient / period boundary and many
    periods later."""
    import ctypes
    from cyberether_b200 import _native
    lib = _native.load()
    lib.b200_fm_nco_phases_host.argtypes = [ctypes.c_float, ctypes.c_uint64, ctypes.c_uint64, ctypes.c_void_p,
                                            ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(ctypes.c_uint64)]
    two_pi = np.float64(2.0) * np.float64(3.14159265358979323846)

    def serial(inc, count):
        out = np.empty(count, np.float32)
        ph = np.float32(0.0)
        for i in range(count):
            out[i] = ph
            ph = np.float32(ph + inc)
            if np.float64(ph) >= two_pi:                                   # the reference's F64 compare and subtract
                ph = np.float32(np.float64(ph) - two_pi)
        return out

    for rate in (250e3, 200e3, 1.2e6, 240e3, 1.024e6, 2.4e6, 20e6):
        inc = np.float32(np.float32(2.0) * np.float64(3.14159265358979323846) * np.float32(19e3) / np.float32(rate))
        pre, cycle = ctypes.c_uint64(), ctypes.c_uint64()
        head = np.empty(60000, np.float32)
        _native.check(lib.b200_fm_nco_phases_host(rate, 0, head.size, head.ctypes.data_as(ctypes.c_void_p),
                                                  ctypes.byref(pre), ctypes.byref(cycle)))
        assert 0 < cycle.value <= 1 << 24 and pre.value < 1 << 24
        want = serial(inc, head.size)
        assert np.array_equal(head, want), rate
        # any later slice continues the same recurrence: step the serial rule from its first element
        for n0 in (pre.value + cycle.value - 7, pre.value + 3 * cycle.value + 12345, 10 ** 12 + 1):
            part = np.empty(5000, np.float32)
            _native.check(lib.b200_fm_nco_phases_host(rate, n0, part.size, part.ctypes.data_as(ctypes.c_void_p), None, None))
            ph = part[0]
            for i in range(1, part.size):
                ph = np.float32(ph + inc)
                if np.float64(ph) >= two_pi:
                    ph = np.float32(np.float64(ph) - two_pi)
                assert part[i] == ph, (rate, n0, i)
        # periodicity claim itself: P(n) == P(n + cycle) for n >= pre
        a = np.empty(4096, np.float32)
        b = np.empty(4096, np.float32)
        _native.check(lib.b200_fm_nco_phases_host(rate, pre.value, a.size, a.ctypes.data_as(ctypes.c_void_p), None, None))
        _native.check(lib.b200_fm_nco_phases_host(rate, pre.value + cycle.value, b.size, b.ctypes.data_as(ctypes.c_void_p),
                                                  None, None))
        assert np.array_equal(a, b)


def test_two_pass_plan_radix16_columns_then_strided_rows():
    """fft_twopass.cuh: n = 16 M; pass 1 = radix-16 over the 16 slabs of a row + W_n^(n2 k1), scratch [k1][n2];
    pass 2 = M-point transforms of the 16 scratch rows stored at k1 + 16 k2; inverse = swap on the way in (pass 1) and
    on the way out (pass 2)."""
    rng = np.random.default_rng(5)
    for m in (64, 1024):
        n = 16 * m
        x = rng.standard_normal(n) + 1j * rng.standard_normal(n)
        for inverse in (False, True):
            xin = x.imag + 1j * x.real if inverse else x
            slabs = xin.reshape(16, m)
            z = np.empty((16, m), complex)
            n2 = np.arange(m)
            for col in range(m):
                z[:, col] = dft16(slabs[:, col])
            z *= np.exp(-2j * np.pi * np.outer(np.arange(16), n2) / n)
            out = np.empty(n, complex)
            for k1 in range(16):
                out[k1 + 16 * np.arange(m)] = np.fft.fft(z[k1])
            if inverse:
                out = out.imag + 1j * out.real
            want = np.fft.ifft(x) * n if inverse else np.fft.fft(x)
            assert np.abs(out - want).max() < 1e-9 * np.abs(want).max()


def test_tiled_two_pass_plan_columns_then_rows():
    """fft_tile.cuh: n = M1 x 256. Pass 1 (fft_cols_kernel): per column, radix 16 (butterfly ja reads ja + t T, writes
    16 ja + t) then radix R = M1 / 16 with Ns = 16 (butterfly jj reads jj + 16 t with W_M1^(jj t), writes k1 = jj + 16 t),
    times W_n^(k1 n2); pass 2 (fft_rows256_kernel): 256-point rows, radix 16 twice, X[k1 + M1 k2]. Both exchange layouts
    (column / row pitch M + M/16 + 1) must be conflict-free for lanes that run over the columns / rows."""
    rng = np.random.default_rng(9)

    def dft_r(v):
        return np.fft.fft(np.asarray(v))

    for m1 in (64, 128, 256):
        n, t_a, radix = m1 * 256, m1 // 16, m1 // 16
        x = rng.standard_normal(n) + 1j * rng.standard_normal(n)
        z = np.zeros((m1, 256), complex)
        for col in range(0, 256, 37):                     # a few columns are enough for the algebra
            colv = x[col::256]                            # x[n1 * 256 + col]
            x1 = np.zeros(m1, complex)
            for ja in range(t_a):
                y = dft16(np.array([colv[ja + t * t_a] for t in range(16)]))
                for t in range(16):
                    x1[16 * ja + t] = y[t]
            for jj in range(16):
                u = [x1[jj + 16 * t] * W(m1, jj * t) for t in range(radix)]
                y = dft_r(u)
                for t in range(radix):
                    k1 = jj + 16 * t
                    z[k1, col] = y[t] * W(n, k1 * col)
            want = np.fft.fft(colv) * np.exp(-2j * np.pi * np.arange(m1) * col / n)
            assert np.abs(z[:, col] - want).max() < 1e-9
        pitch = m1 + m1 // 16 + 1
        columns = 4096 // m1
        for ja in range(t_a):                             # x1 stores / loads: lanes over the column g
            for t in range(16):
                for half in range(0, min(columns, 32), 16):
                    lanes = range(half, half + 16)
                    store = [8 * (g * pitch + (16 * ja + t) + (16 * ja + t) // 16) for g in lanes]
                    assert len({(a // 8) % 16 for a in store}) == 16
        for jj in range(16):
            for t in range(radix):
                e = jj + 16 * t
                load = [8 * (g * pitch + e + e // 16) for g in range(16)]
                assert len({(a // 8) % 16 for a in load}) == 16
    # pass 2 on full rows: z rows of 256 -> X[k1 + M1 k2]
    m1, n = 64, 64 * 256
    x = rng.standard_normal(n) + 1j * rng.standard_normal(n)
    z = np.fft.fft(x.reshape(m1, 256), axis=0) * np.exp(-2j * np.pi * np.outer(np.arange(m1), np.arange(256)) / n)
    out = np.zeros(n, complex)
    for k1 in range(m1):
        x1 = np.zeros(256, complex)
        for lt in range(16):
            y = dft16(np.array([z[k1, lt + 16 * t] for t in range(16)]))
            for t in range(16):
                x1[16 * lt + t] = y[t]
        for jj in range(16):
            y = dft16(np.array([x1[jj + 16 * t] * W(256, jj * t) for t in range(16)]))
            for t in range(16):
                out[k1 + m1 * (jj + 16 * t)] = y[t]
    assert np.abs(out - np.fft.fft(x)).max() < 1e-8
    pitch = 256 + 16 + 1
    for ga in range(16):                                  # pass A stores: lanes over lt; pass B loads: lanes over the row
        for t in range(16):
            assert len({((ga * pitch + 17 * lt + t)) % 16 for lt in range(16)}) == 16
    for jj in range(16):
        for t in range(16):
            e = jj + 16 * t
            assert len({(gb * pitch + e + e // 16) % 16 for gb in range(16)}) == 16


def test_real_fft_through_half_length_complex_transform():
    """b200_fft_exec_real / rfft_unpack_kernel: z[m] = x[2m] + i x[2m+1] is the real row itself viewed as complex; with
    Z = FFT_h(z), one thread per mirror pair: e = (Z[k] + conj Z[h-k]) / 2, o = (Z[k] - conj Z[h-k]) / (2i), w = W_2h^k,
    X[k] = e + w o, X[h-k] = conj(e - w o); k = 0 gives X[0] and X[h] from Z[0]; FFTPACK layout [Re X0, Re X1, Im X1, ..., Re Xh]."""
    rng = np.random.default_rng(12)
    for h in (2, 3, 8, 9, 50, 4096):
        x = rng.standard_normal(2 * h)
        z = np.fft.fft(x[0::2] + 1j * x[1::2])
        spec = np.zeros(h + 1, complex)
        for k in range(h // 2 + 1):
            if k == 0:
                spec[0] = z[0].real + z[0].imag
                spec[h] = z[0].real - z[0].imag
                continue
            a, m = z[k], z[h - k]
            e = complex(0.5 * (a.real + m.real), 0.5 * (a.imag - m.imag))
            o = complex(0.5 * (a.imag + m.imag), -0.5 * (a.real - m.real))
            t = np.exp(-1j * np.pi * k / h) * o
            spec[k] = e + t
            if 2 * k != h:
                spec[h - k] = np.conj(e - t)
        want = np.fft.rfft(x)
        assert np.abs(spec - want).max() < 1e-9 * max(1.0, np.abs(want).max())
        packed = np.empty(2 * h)
        packed[0] = spec[0].real
        packed[1:2 * h - 1:2] = spec[1:h].real
        packed[2:2 * h - 1:2] = spec[1:h].imag
        packed[2 * h - 1] = spec[h].real
        # pocketfft r2r_fftpack layout == scipy.fft.rfft's "halfcomplex" ordering (r0, r1, i1, ..., r_h)
        import scipy.fft
        assert np.abs(packed - scipy.fft.rfft(x).view(float)[[0] + list(range(2, 2 * h + 1))]).max() < 1e-9 * max(1.0, np.abs(want).max())


def test_fused_real_unpack_thread_assignment():
    """fft_radix_kernel<MODE_R2C>: the T = N / 16 threads of a row unpack the mirror pairs k = lt + j T (j < 8; k = N / 2 by
    lt = 0 alone): every k in [0, N / 2] exactly once, hence every output bin X[0 .. N] exactly once; Z goes through the
    exchange buffer the last register pass did NOT read (X1 for an odd number of passes, the stage buffer otherwise)."""
    for log2n in range(5, 14):
        n = 1 << log2n
        t = n // 16
        seen, outputs = [], []
        for lt in range(t):
            for j in range(9):
                if j == 8 and lt != 0:
                    break
                k = lt + j * t
                seen.append(k)
                outputs += [0, n] if k == 0 else ([k] if 2 * k == n else [k, n - k])
        assert sorted(seen) == list(range(n // 2 + 1))
        assert sorted(outputs) == list(range(n + 1))
        passes = (log2n + 3) // 4
        last_pass_reads = "stage" if passes % 2 == 1 else "x1"          # pass q reads the stage buffer for even q
        zbuf = "x1" if passes % 2 == 1 else "stage"
        assert zbuf != last_pass_reads


# ---- fft4096_kernel: shared-memory schedule across consecutive rows, and the forms the dispatch reaches ------------
def _fft4096_kernel_code():
    """fft4096_kernel's source from its signature on, comments removed."""
    with open(os.path.join(CSRC, "fft4096.cuh")) as f:
        text = f.read()
    return re.sub(r"//[^\n]*", "", text[text.index("fft4096_kernel(const FftParams p)"):])


def _c_eval(expr, names):
    """Value of a C integer expression of the kernel (?:, &&, ||, comparisons, bit operators, unsigned literals)."""
    expr = re.sub(r"\b(\d+)u\b", r"\1", expr.strip())
    while expr.startswith("("):
        depth = 0
        for j, ch in enumerate(expr):
            depth += {"(": 1, ")": -1}.get(ch, 0)
            if depth == 0:
                break
        if j != len(expr) - 1:
            break
        expr = expr[1:-1].strip()
    depth, question = 0, None
    for j, ch in enumerate(expr):
        depth += {"(": 1, ")": -1}.get(ch, 0)
        if depth == 0 and ch == "?" and question is None:
            question, nested = j, 0
        elif depth == 0 and question is not None and ch == "?":
            nested += 1
        elif depth == 0 and question is not None and ch == ":":
            if nested == 0:
                branch = expr[question + 1:j] if _c_eval(expr[:question], names) else expr[j + 1:]
                return _c_eval(branch, names)
            nested -= 1
    python = expr.replace("&&", " and ").replace("||", " or ")
    return eval(re.sub(r"!(?!=)", " not ", python), {"__builtins__": {}}, dict(names))


def _fft4096_schedule_expressions(code):
    """The index expressions of the kernel's cross-row reuse, read from its source."""
    find = lambda pattern: re.search(pattern, code).group(1)
    return {"buf": find(r"buf = smem_raw \+ \(([^;]*)\) \* kFft4096StageBytes;"),
            "land": find(r"land = smem_raw \+ kLandBase \+ ([^;]*) \* kLandPitch;"),
            "refill_if": find(r"if \(t == 0 && ([^{]*)\) \{\s*const uint32_t slot"),
            "slot": find(r"const uint32_t slot = ([^;]*);"),
            "agc_write": find(r"agc_partial\[([^\]]*)\]\[t >> 5\] = power;"),
            "agc_read": find(r"mean_power \+= agc_partial\[([^\]]*)\]\[w\];")}


_FFT4096_SYNCTHREADS = 3        # after the mbarrier init, (A) and (C)


def _fft4096_kernel_schedule(exprs, integer, stages, agc, rows):
    """Program order of every thread of one fft4096_kernel CTA over its first `rows` rows, in the event format of
    _radix_kernel_schedule. CF32: the row lands in stage{s}, which is also its exchange buffer. Integer input: the row lands
    in stage{s} of the landing ring and the exchanges use xchg{0|1}. agc{0|1}[warp] are the AGC partials. Elements are
    float2 slots (landing slots of integer rows: samples). Split barrier (B) is a barrier at its arrive point."""
    my_rows = rows + stages
    program = []
    for t in range(256):
        lo4, hi4 = t & 15, t >> 4
        ev, issued = [("sync",)], 0

        def issue(slot):
            nonlocal issued
            if issued < my_rows:
                if t == 0:
                    ev.append(("tma", slot, issued))
                issued += 1

        for s in range(stages):
            issue(s)
        stage = refill_stage = 0
        for i in range(rows):
            names = {"kInt": integer, "i": i, "stage": stage, "refill_stage": refill_stage, "issued": issued,
                     "my_rows": my_rows}
            buf = f"{'xchg' if integer else 'stage'}{_c_eval(exprs['buf'], names)}"
            land = f"stage{_c_eval(exprs['land'], names)}"
            ev.append(("wait", i))
            ev += [("r", land if integer else buf, t + 256 * a) for a in range(16)]       # pass 1 loads
            if agc and t % 32 == 0:
                ev.append(("w", f"agc{_c_eval(exprs['agc_write'], names)}", t >> 5))
            ev += [("w", buf, t + 256 * k) for k in range(16)]                            # pass 1 stores
            ev.append(("sync",))                                                           # (A)
            if _c_eval(exprs["refill_if"], names):
                issue(_c_eval(exprs["slot"], names))
            ev += [("r", buf, 256 * hi4 + lo4 + 16 * b) for b in range(16)]               # exchange-1 reads
            ev.append(("sync",))                                                           # (B)
            ev += [("w", buf, 18 * hi4 + lo4 + 288 * k) for k in range(16)]               # exchange-2 stores
            ev.append(("sync",))                                                           # (C)
            ev += [("r", buf, 18 * lo4 + 288 * hi4 + c) for c in range(16)]               # pass 3 (LDS.128 pairs)
            if agc:
                ev += [("r", f"agc{_c_eval(exprs['agc_read'], names)}", w) for w in range(8)]
            refill_stage = stage
            stage = (stage + 1) % stages
        program.append(ev)
    return program


def test_fft4096_kernel_schedule_is_race_free_across_consecutive_rows():
    """fft4096_kernel is persistent and reuses shared memory from row to row: the CF32 ring (refilled after barrier (A)
    with the row kStages ahead, into the previous row's stage), the integer landing ring (refilled with the current row's
    slot), the two exchange buffers of integer input (alternating by row parity), and the AGC partials (by row parity).
    The replay covers stages + 3 consecutive rows of one CTA for CF32 with 3 stages (2 CTAs/SM, with AGC), CF32 with 2
    stages (3 CTAs/SM) and integer input with 3 x 8 KiB and 2 x 16 KiB landing rings (with AGC), and checks with
    _schedule_races that every pair of accesses that could race is ordered.

    The schedule is a hand restatement of fft4096.cuh; the index expressions of the reuse (exchange buffer, landing slot,
    refill condition and slot, AGC partial rows) are read from the kernel source, and the source's __syncthreads count
    must match the restatement. Split barrier (B) is modelled as a barrier at its arrive point, which is exact because
    the code between mbar_arrive(reads_done) and mbar_wait(reads_done, ...) only calls register-only helpers."""
    code = _fft4096_kernel_code()
    exprs = _fft4096_schedule_expressions(code)
    between = code[code.index("mbar_arrive(reads_done);") + len("mbar_arrive(reads_done);"):code.index("mbar_wait(reads_done")]
    assert set(re.findall(r"(\w+)\s*\(", between)) <= {"dft16_rest", "apply_twiddles"}, between
    assert not re.search(r"\b(buf|land|smem_raw|agc_partial|full|reads_done)\b|\[", between), between
    assert code.count("__syncthreads()") == _FFT4096_SYNCTHREADS
    failures = []
    for name, integer, stages, agc in (("CF32, 3 stages", False, 3, True), ("CF32, 2 stages", False, 2, False),
                                       ("8-bit, 3 x 8 KiB", True, 3, True), ("16-bit, 2 x 16 KiB", True, 2, True)):
        races = _schedule_races(_fft4096_kernel_schedule(exprs, integer, stages, agc, stages + 3))
        if races:
            failures.append(f"{name}: {len(races)} races, e.g. {races[0]}")
    assert not failures, "\n".join(failures)


def test_fft4096_c_expressions_evaluate_as_in_c():
    names = {"kInt": False, "i": 3, "stage": 2, "refill_stage": 1, "issued": 4, "my_rows": 9}
    assert _c_eval("kInt ? (i & 1u) : stage", names) == 2
    assert _c_eval("kInt ? stage : refill_stage", names) == 1
    assert _c_eval("(kInt || i >= 1) && issued < my_rows", names)
    assert _c_eval("i & 1", dict(names, i=4)) == 0
    assert _c_eval("kInt ? (i & 1u) : stage", dict(names, kInt=True)) == 1


def _fft_cu_dispatch_forms():
    """(entry point, MODE, WIN, ITYPE) of every fft4096_kernel form fft.cu's default dispatch reaches at n = 4096."""
    with open(os.path.join(CSRC, "fft.cu")) as f:
        src = f.read()
    # launch_4096_int always runs the real-window kernel, launch_fft runs fft4096_kernel for every window at n = 4096
    assert "auto kernel = fft4096_kernel<MODE, WIN_REAL, 2, ITYPE, AGC, COLSUM>;" in src
    launch_fft = src[src.index("static int launch_fft("):]
    assert re.search(r"if \(p\.n == kFft4096N && MODE != MODE_C2C[^{]*\{\s*return launch_4096<MODE, WIN>",
                     launch_fft[:launch_fft.index("try_launch_radix")])
    entries = {"B200_CHAIN_DISPATCH": "chain_exec", "B200_INT_DISPATCH": "chain_exec_typed",
               "B200_AGC_DISPATCH": "chain_exec_agc", "B200_COLSUM_DISPATCH": "chain_exec_colsum"}
    flags = {"chain_exec_typed": "", "chain_exec_agc": ", true", "chain_exec_colsum": ", false, true"}
    forms = set()
    for macro, entry in entries.items():
        region = src[src.index(f"#define {macro}(MODE)"):src.index(f"#undef {macro}")]
        body, uses = region[:region.index("if (enable_range)")], region[region.index("if (enable_range)"):]
        modes = re.findall(rf"{macro}\((MODE_\w+)\)", uses)
        if entry == "chain_exec":
            kinds = [(w, "IN_CF32") for w in re.findall(r"launch_fft<MODE, (WIN_\w+)>", body)]
        else:
            launches = re.findall(r"launch_4096_int<MODE, (IN_\w+)((?:, (?:true|false))*)>", body)
            assert all(f == flags[entry] for _, f in launches), (macro, launches)
            kinds = [("WIN_REAL", t) for t, _ in launches]
        forms |= {(entry, m, w, t) for m in modes for w, t in kinds}
    return forms


def test_chain_forms_table_is_the_fft4096_dispatch_and_every_form_has_a_gpu_case():
    import chain_forms
    import test_gpu_chain_forms as gpu
    assert len(chain_forms.FORMS) == len(set(chain_forms.FORMS)) == 34
    assert _fft_cu_dispatch_forms() == set(chain_forms.FORMS)
    marks = [m for m in gpu.test_chain_form_steady_state.pytestmark if m.name == "parametrize"]
    assert len(marks) == 1 and marks[0].args[1] is gpu.CASES
    assert [c.values[0] for c in gpu.CASES] == chain_forms.FORMS
