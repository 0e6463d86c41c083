"""fir_decim_kernel, every form the FIR plan can pick, against an exact integer model of the streaming FIR.

Inputs and taps are integers in [-8, 8], so every product and every partial sum the kernel forms is an integer below
2^24: its F32 result is exact whatever the summation order or FMA contraction. The check is therefore bit-exact against
    y[q] = sum_k h[k] * xs[q R - k]      (xs = every sample the plan has been given since its last reset)
evaluated by an F64 FFT convolution and rounded to integers. The taps' first and last entries are non-zero and differ
from their neighbours, so a kernel that drops or misplaces an end tap fails.

Each plan reports the forms its exec can launch (b200_fir_plan_variant); every case asserts that report, so a geometry
change that moves a case to another form fails here instead of silently testing something else.
"""
import ctypes
import math
import re

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _env():
    import torch
    from cyberether_b200 import _native
    from cyberether_b200.jetstream import Context
    dev = torch.device("cuda", torch.cuda.current_device())
    return torch, _native, _native.load(), Context.get(dev), dev


def _taps(seed, L, heads, complex_taps):
    """[heads, L] integer taps in [-8, 8]; h[0] and h[L-1] non-zero and distinct from their neighbours. Real taps have
    every imaginary part exactly 0."""
    rng = np.random.default_rng(seed)
    h = rng.integers(-8, 9, (heads, L)).astype(np.complex128)
    if complex_taps:
        h += 1j * rng.integers(-8, 9, (heads, L))
    first, last = (8 - 3j, -7 + 5j) if complex_taps else (8, -7)
    h[:, -1] = last
    h[:, 0] = first
    if L > 2:
        h[h[:, 1] == first, 1] = 1
        h[h[:, -2] == last, -2] = -1
    return h.astype(np.complex64)


class _Plan:
    def __init__(self, taps, R):
        torch, self.native, self.lib, self.ctx, self.dev = _env()
        self.taps, self.R = taps, R
        self.heads, self.L = taps.shape
        self.handle = ctypes.c_void_p()
        self.native.check(self.lib.b200_fir_plan_create(self.ctx.handle, taps.ctypes.data_as(ctypes.c_void_p), self.L,
                                                        self.heads, R, ctypes.byref(self.handle)))
        self.variant = self.lib.b200_fir_plan_variant(self.handle).decode()
        self.stream = ctypes.c_void_p(torch.cuda.current_stream(self.dev).cuda_stream)

    def forms(self):
        """{form: {'OB', 'threads', 'taps', 'kind', 'qt', 'ctas'}} parsed from the plan's report."""
        out = {}
        for part in self.variant.split("; "):
            m = re.fullmatch(r"(sample|pair) OB=(\d+) threads=(\d+) taps=(const|shared) (real|complex) qt=(\d+) ctas=(\d+)",
                             part)
            assert m, self.variant
            out[m[1]] = dict(OB=int(m[2]), threads=int(m[3]), taps=m[4], kind=m[5], qt=int(m[6]), ctas=int(m[7]))
        return out

    def exec(self, x, frames, frame_len):
        import torch
        y = torch.empty(frames, self.heads, frame_len // self.R, dtype=torch.complex64, device=self.dev)
        self.native.check(self.lib.b200_fir_exec(self.handle, x.data_ptr(), y.data_ptr(), frames, frame_len, self.stream))
        return y

    def reset(self):
        self.native.check(self.lib.b200_fir_reset(self.handle, self.stream))

    def set_history(self, tail, frames_before=0):
        self.native.check(self.lib.b200_fir_set_history(self.handle, tail.data_ptr() if tail.numel() else None,
                                                        tail.numel(), frames_before, self.stream))

    def set_translation(self, frame_len, center_bins):
        bins = (ctypes.c_int64 * self.heads)(*center_bins)
        self.native.check(self.lib.b200_fir_plan_set_translation(self.handle, frame_len, bins))

    def close(self):
        self.native.check(self.lib.b200_fir_plan_destroy(self.handle))

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


def _ints(n, seed, misalign=False):
    """n CF32 samples with integer re, im in [-8, 8] on the GPU; misalign: a view 8 bytes past a 16-byte boundary."""
    import torch
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    base = torch.randint(-8, 9, (n + 1, 2), generator=g, device="cuda", dtype=torch.float32)
    x = torch.view_as_complex(base).view(-1)
    x = x[1:] if misalign else x[:n]
    assert x.data_ptr() % 16 == (8 if misalign else 0)
    return x


def _model(taps, R, segment, prefix=0):
    """Integer model of a plan fed `segment` (1-D complex GPU tensor) after a reset: outputs at stream positions
    prefix + q R (the first `prefix` samples are history handed to set_history). F64 FFT convolution per head, checked to
    lie within 1e-3 of an integer before it is rounded. Returns [n_out, heads] complex64 on the GPU."""
    import torch
    s = segment.to(torch.complex128)
    n, L = s.numel(), taps.shape[1]
    nfft = 1 << (n + L - 1 - 1).bit_length()
    sf = torch.fft.fft(s, nfft)
    cols = []
    for h in taps:
        full = torch.fft.ifft(sf * torch.fft.fft(torch.from_numpy(h.astype(np.complex128)).to(s.device), nfft))
        cols.append(full[prefix:n:R])
    y = torch.stack(cols, dim=1)
    r = torch.view_as_real(y)
    rounded = torch.round(r)
    assert (r - rounded).abs().max().item() <= 1e-3, "the F64 model is not integral: it cannot be trusted"
    assert rounded.abs().max().item() < 2 ** 24
    return torch.view_as_complex(rounded.to(torch.float32).contiguous())


def _assert_exact(got, want, what):
    """got [frames, heads, frame_out] against the model [frames * frame_out, heads]: equal in every element."""
    import torch
    frames, heads, fo = got.shape
    want = want.reshape(frames, fo, heads).transpose(1, 2)
    bad = (torch.view_as_real(got) != torch.view_as_real(want)).any(dim=-1)
    if bad.any():
        idx = bad.nonzero()
        f, h, m = idx[0].tolist()
        raise AssertionError(f"{what}: {idx.shape[0]} of {bad.numel()} outputs differ; first at frame {f} head {h} "
                             f"m {m} (q = {f * fo + m}): got {got[f, h, m].item()} want {want[f, h, m].item()}")


def _run_stream(plan, calls, misalign=False, seed=0):
    """Feed plan the calls [(frames, frame_len), ...] as one stream and check every output bit-exactly. misalign: one
    flag for every call, or one per call."""
    import torch
    flags = list(misalign) if isinstance(misalign, (list, tuple)) else [misalign] * len(calls)
    xs = [_ints(f * t, seed + 101 * i, flags[i]) for i, (f, t) in enumerate(calls)]
    want = _model(plan.taps, plan.R, torch.cat(xs))
    q = 0
    for i, ((frames, t), x) in enumerate(zip(calls, xs)):
        y = plan.exec(x, frames, t)
        n_out = frames * (t // plan.R)
        _assert_exact(y, want[q:q + n_out], f"{plan.variant}: call {i} ({frames} x {t}{', misaligned' if flags[i] else ''})")
        q += n_out


# ---- one case per compiled form: (form, L, R, heads, complex taps, expected report without qt / ctas) ------------------
# L even or R odd leaves a plan without the pair form; a sample-form case of a pair-eligible plan runs on an input that
# is not 16-byte aligned.
VARIANTS = [
    # sample form, taps in the kernel parameters
    ("sample", 127, 1, 1, False, "sample OB=7 threads=128 taps=const real"),
    ("sample", 65, 3, 1, True, "sample OB=7 threads=128 taps=const complex"),
    ("sample", 130, 8, 1, False, "sample OB=7 threads=64 taps=const real"),
    ("sample", 126, 6, 1, True, "sample OB=7 threads=64 taps=const complex"),
    ("sample", 101, 53, 1, False, "sample OB=7 threads=32 taps=const real"),
    ("sample", 254, 32, 1, True, "sample OB=7 threads=32 taps=const complex"),
    ("sample", 401, 53, 1, False, "sample OB=5 threads=32 taps=const real"),
    ("sample", 107, 53, 1, True, "sample OB=5 threads=32 taps=const complex"),
    ("sample", 160, 80, 1, False, "sample OB=3 threads=32 taps=const real"),
    ("sample", 161, 80, 1, True, "sample OB=3 threads=32 taps=const complex; pair OB=3 threads=32 taps=const complex"),
    ("sample", 256, 128, 1, False, "sample OB=1 threads=64 taps=const real"),
    ("sample", 257, 128, 1, True, "sample OB=1 threads=64 taps=const complex; pair OB=1 threads=64 taps=const complex"),
    ("sample", 401, 200, 1, False, "sample OB=1 threads=32 taps=const real; pair OB=1 threads=32 taps=const real"),
    ("sample", 199, 200, 1, True, "sample OB=1 threads=32 taps=const complex; pair OB=1 threads=32 taps=const complex"),
    # sample form, taps in shared memory
    ("sample", 2047, 1, 1, False, "sample OB=7 threads=128 taps=shared real"),
    ("sample", 1023, 1, 1, True, "sample OB=7 threads=128 taps=shared complex"),
    ("sample", 4095, 1, 1, False, "sample OB=7 threads=64 taps=shared real"),
    ("sample", 129, 8, 16, True, "sample OB=7 threads=64 taps=shared complex"),
    ("sample", 8191, 1, 1, False, "sample OB=7 threads=32 taps=shared real"),
    ("sample", 4095, 1, 2, True, "sample OB=7 threads=32 taps=shared complex"),
    ("sample", 129, 39, 32, False, "sample OB=5 threads=32 taps=shared real"),
    ("sample", 129, 8, 64, True, "sample OB=5 threads=32 taps=shared complex"),
    ("sample", 201, 14, 64, False, "sample OB=5 threads=64 taps=shared real"),
    ("sample", 201, 14, 32, True, "sample OB=5 threads=64 taps=shared complex"),
    ("sample", 8191, 4, 1, False, "sample OB=3 threads=32 taps=shared real"),
    ("sample", 161, 96, 2, True, "sample OB=3 threads=32 taps=shared complex"),
    ("sample", 511, 19, 32, False, "sample OB=3 threads=64 taps=shared real"),
    ("sample", 511, 19, 16, True, "sample OB=3 threads=64 taps=shared complex"),
    ("sample", 201, 200, 8, False, "sample OB=1 threads=32 taps=shared real"),
    ("sample", 401, 200, 1, True, "sample OB=1 threads=32 taps=shared complex"),
    ("sample", 161, 160, 8, False, "sample OB=1 threads=64 taps=shared real"),
    ("sample", 161, 19, 64, True, "sample OB=1 threads=64 taps=shared complex"),
    # chunk-pair form (16-byte aligned input of even length)
    ("pair", 127, 2, 1, False, "sample OB=7 threads=128 taps=const real; pair OB=5 threads=128 taps=const real"),
    ("pair", 129, 6, 1, True, "sample OB=7 threads=64 taps=const complex; pair OB=5 threads=128 taps=const complex"),
    ("pair", 129, 24, 3, False, "sample OB=7 threads=64 taps=const real; pair OB=5 threads=64 taps=const real"),
    ("pair", 129, 16, 1, True, "sample OB=7 threads=64 taps=const complex; pair OB=5 threads=64 taps=const complex"),
    ("pair", 257, 64, 1, False, "sample OB=5 threads=32 taps=const real; pair OB=5 threads=32 taps=const real"),
    ("pair", 201, 38, 1, True, "sample OB=7 threads=32 taps=const complex; pair OB=5 threads=32 taps=const complex"),
    ("pair", 161, 80, 1, False, "sample OB=3 threads=32 taps=const real; pair OB=3 threads=32 taps=const real"),
    ("pair", 161, 80, 1, True, "sample OB=3 threads=32 taps=const complex; pair OB=3 threads=32 taps=const complex"),
    ("pair", 257, 128, 1, False, "sample OB=1 threads=64 taps=const real; pair OB=1 threads=64 taps=const real"),
    ("pair", 257, 128, 1, True, "sample OB=1 threads=64 taps=const complex; pair OB=1 threads=64 taps=const complex"),
    ("pair", 401, 200, 1, False, "sample OB=1 threads=32 taps=const real; pair OB=1 threads=32 taps=const real"),
    ("pair", 199, 200, 1, True, "sample OB=1 threads=32 taps=const complex; pair OB=1 threads=32 taps=const complex"),
]


def _form_key(form, report):
    """('sample' | 'pair', OB, threads, taps, kind) of one form in a report (qt / ctas stripped or not)."""
    part = [p for p in report.split("; ") if p.startswith(form)][0]
    m = re.match(r"(\w+) OB=(\d+) threads=(\d+) taps=(\w+) (\w+)", part)
    return m[1], int(m[2]), int(m[3]), m[4], m[5]


def _case_id(case):
    form, L, R, heads, cplx, report = case
    _, ob, threads, taps, kind = _form_key(form, report)
    return f"{form}-OB{ob}-t{threads}-{taps}-{kind}-L{L}-R{R}-H{heads}"


def test_variant_table_has_one_case_per_form_and_both_staging_paths():
    """One case per compiled form; per form and thread count the table holds an R (in the form's own sample units) that
    divides the CTA size, which stages through the interior fast path, and one that does not."""
    keys = [_form_key(c[0], c[5]) for c in VARIANTS]
    assert len(keys) == len(set(keys)), "two cases test the same form"
    divides = {}
    for (form, L, R, heads, cplx, report), key in zip(VARIANTS, keys):
        r = R // 2 if form == "pair" else R
        divides.setdefault((form, key[2]), set()).add(key[2] % r == 0)
    assert all(v == {True, False} for v in divides.values()), divides


@pytest.mark.parametrize("case", VARIANTS, ids=_case_id)
def test_every_form_is_bit_exact_in_steady_state(case):
    """Four calls with carried history: a small first call (edge tiles only); one sized from the reported qt and CTA cap
    so every CTA runs at least three tiles and the last tile is ragged; one shorter than the L-1 samples of history
    (when L > R + 1); and a small one that starts from the history the short call left."""
    form, L, R, heads, cplx, report = case
    with _Plan(_taps(L * 131 + R, L, heads, cplx), R) as plan:
        assert re.sub(r" qt=\d+ ctas=\d+", "", plan.variant) == report
        forms = plan.forms()
        f = forms[form]
        assert f["qt"] == f["OB"] * f["threads"]
        assert f["ctas"] % plan.ctx.sm_count == 0 and 1 <= f["ctas"] // plan.ctx.sm_count <= 8, (f, plan.ctx.sm_count)
        misalign = form == "sample" and "pair" in forms
        qt = f["qt"]
        fo = 37                                   # outputs per frame: frames straddle tiles, tiles straddle frames
        frames = -(-(3 * f["ctas"] * qt + 1) // fo)
        if frames * fo % qt == 0:
            frames += 1
        short = max(1, (L - 2) // R)              # outputs of the call shorter than the history
        calls = [(2, 3 * R), (frames, fo * R), (1, short * R), (3, 2 * R)]
        assert -(-frames * fo // qt) > 3 * f["ctas"] and frames * fo % qt != 0
        if L > R + 1:
            assert short * R < L - 1
        _run_stream(plan, calls, misalign=misalign, seed=L + R)


def test_every_form_the_plans_can_pick_is_in_the_variant_table():
    """Sweep plan creation over taps, decimation, heads and tap kind; every form a plan reports must have its own case
    in VARIANTS, so a newly reachable kernel form brings its own test."""
    torch, native, lib, ctx, dev = _env()
    table = {_form_key(c[0], c[5]) for c in VARIANTS}
    ones = {False: np.ones(64 * 8191, np.complex64), True: np.full(64 * 8191, 1 + 1j, np.complex64)}
    found = {}
    for cplx in (False, True):
        ptr = ones[cplx].ctypes.data_as(ctypes.c_void_p)
        for heads in (1, 2, 3, 8, 16, 32, 64):
            for R in (1, 2, 3, 4, 5, 6, 8, 12, 14, 16, 19, 24, 32, 38, 39, 53, 64, 80, 96, 128, 160, 200, 256):
                for L in (1, 2, 3, 16, 33, 65, 127, 129, 161, 201, 257, 401, 511, 1023, 2047, 4095, 8191):
                    plan = ctypes.c_void_p()
                    if lib.b200_fir_plan_create(ctx.handle, ptr, L, heads, R, ctypes.byref(plan)) != 0:
                        assert b"does not fit" in lib.b200_last_error() and plan.value is None
                        continue
                    report = lib.b200_fir_plan_variant(plan).decode()
                    native.check(lib.b200_fir_plan_destroy(plan))
                    for form in ("sample", "pair"):
                        if form in report:
                            found.setdefault(_form_key(form, report), (L, R, heads, cplx, report))
    missing = {k: v for k, v in found.items() if k not in table}
    assert not missing, missing
    print(f"{len(found)} forms reached, all in the variant table")


@pytest.mark.parametrize("L,R,heads,cplx", [(129, 8, 1, False), (129, 6, 3, True)])
def test_pair_eligible_plan_takes_the_sample_form_on_a_misaligned_input(L, R, heads, cplx):
    """The same pair-eligible plan fed 16-byte-aligned calls (pair form) and calls offset by one sample (sample form),
    alternating over one stream: both bit-exact, and the history one form leaves is what the other continues from."""
    with _Plan(_taps(L + 7, L, heads, cplx), R) as plan:
        forms = plan.forms()
        assert "pair" in forms and "sample" in forms, plan.variant
        qt = max(forms["pair"]["qt"], forms["sample"]["qt"])
        calls = [(3, 5 * R), (-(-3 * qt // 11), 11 * R), (1, R), (2, 7 * R), (-(-2 * qt // 5), 5 * R), (4, 3 * R)]
        _run_stream(plan, calls, misalign=[i % 2 == 1 for i in range(len(calls))], seed=L)


@pytest.mark.parametrize("L,R,heads,cplx", [(32, 4, 2, False), (33, 4, 3, True), (16, 3, 16, False)])
def test_multi_head_output_layout(L, R, heads, cplx):
    """Output [frames, heads, frame_out] for frame_out in {1, 3, qt - 1, qt + 1, 3 qt + 5}: the store loop's frame walk
    crosses several frames per CTA stride when frames are short, and frames straddle tiles when they are long."""
    with _Plan(_taps(heads * L, L, heads, cplx), R) as plan:
        forms = plan.forms()
        qt = forms["pair" if "pair" in forms else "sample"]["qt"]
        calls = [(max(2, -(-3 * qt // fo) + 1), fo * R) for fo in (1, 3, qt - 1, qt + 1, 3 * qt + 5)]
        _run_stream(plan, calls, seed=heads)


def _translated_model(taps, R, stream, frame_len, center_bins):
    """F64 model of the translating heads: the integer convolution times exp(j 2 pi offset (m R mod M) / M) per output
    m of a frame and exp(j 2 pi (offset T F mod M) / M) per absolute frame F, offset = -centre bin mod M, M = T + L - 1.
    Returns (want [n_out, heads] complex128, |integer convolution|)."""
    import torch
    L = taps.shape[1]
    M, fo = frame_len + L - 1, frame_len // R
    conv = _model(taps, R, stream).to(torch.complex128)
    q = torch.arange(conv.shape[0], device=conv.device, dtype=torch.int64)
    frame, m = q // fo, q % fo
    cols = []
    for h, c in enumerate(center_bins):
        offset = (-c) % M
        k = (offset * ((m * R) % M) + offset * ((frame_len * frame) % M)) % M
        cols.append(conv[:, h] * torch.exp(2j * math.pi * k.to(torch.float64) / M))
    return torch.stack(cols, dim=1), conv.abs()


@pytest.mark.parametrize("L,R,heads,cplx", [(33, 4, 3, False), (32, 5, 2, True)])
def test_translating_heads_over_growing_calls_and_a_continued_stream(L, R, heads, cplx):
    """set_translation: the output is the integer convolution times the rotation and the per-frame phase, both F64 ->
    F32 phasors (each off by at most u = 2^-24 in modulus), applied by two F32 complex products (four products, one add
    or sub: at most 2 sqrt(2) u |a| |b| each). So |got - want| <= (1 + 1 + 4 sqrt(2)) u |conv| + O(u^2) < 8 u |conv| per
    element. The frame count grows from call to call, which re-allocates the phase table. A second plan continues the
    stream from the first one's last L - 1 samples and frame count through set_history."""
    import torch
    T = 50 * R
    bins = [3, -17, 250][:heads]
    taps = _taps(L * 3 + R, L, heads, cplx)
    frames = [2, 5, 40, 3, 61]
    xs = [_ints(f * T, 900 + i) for i, f in enumerate(frames)]
    want, mag = _translated_model(taps, R, torch.cat(xs), T, bins)
    fo = T // R
    got = []
    with _Plan(taps, R) as a:
        a.set_translation(T, bins)
        if L % 2 == 1 and R % 2 == 0:
            assert "pair" in a.forms(), a.variant
        for f, x in zip(frames[:3], xs[:3]):
            got.append(a.exec(x, f, T))
    done = sum(frames[:3])
    with _Plan(taps, R) as b:
        b.set_translation(T, bins)
        b.set_history(torch.cat(xs[:3])[-(L - 1):], frames_before=done)
        for f, x in zip(frames[3:], xs[3:]):
            got.append(b.exec(x, f, T))
    got = torch.cat([g.transpose(1, 2).reshape(-1, heads) for g in got]).to(torch.complex128)
    assert got.shape == want.shape
    err = (got - want).abs()
    tol = 8 * 2.0 ** -24 * mag
    bad = err > tol
    assert not bad.any(), (f"{bad.sum().item()} outputs beyond 8 u |conv|; first at q, head = {bad.nonzero()[0].tolist()} "
                           f"(frame_out {fo}); worst err / |conv| = {(err / mag.clamp(min=1)).max().item():.3e}")


@pytest.mark.parametrize("L,R,heads,cplx", [(16383, 1, 1, False), (8191, 1, 1, True), (33, 1024, 1, False)])
def test_plans_that_do_not_fit_the_shared_memory_tile_are_refused(L, R, heads, cplx):
    torch, native, lib, ctx, dev = _env()
    taps = _taps(L, L, heads, cplx)
    plan = ctypes.c_void_p()
    for _ in range(3):
        assert lib.b200_fir_plan_create(ctx.handle, taps.ctypes.data_as(ctypes.c_void_p), L, heads, R,
                                        ctypes.byref(plan)) == 1
        msg = lib.b200_last_error().decode()
        assert f"taps={L} heads={heads} decimation={R}" in msg and "does not fit" in msg, msg
        assert plan.value is None


def test_largest_plan_that_fits_runs_bit_exact():
    """8191 real taps at R = 1, the neighbour of the refused 16383, over calls longer and shorter than its history."""
    with _Plan(_taps(8191, 8191, 1, False), 1) as plan:
        assert plan.variant.startswith("sample OB=7 threads=32 taps=shared real"), plan.variant
        _run_stream(plan, [(1, 100), (3, 10000), (1, 8189), (2, 5000)], seed=8191)


@pytest.mark.parametrize("L,R,heads,cplx", [(65, 4, 2, True), (64, 3, 1, False)])
def test_reset_and_short_history_mid_stream(L, R, heads, cplx):
    """reset forgets the history; set_history with count < L - 1 zero-fills the front of it. Both bit-exact."""
    import torch
    with _Plan(_taps(L + R, L, heads, cplx), R) as plan:
        calls = [(3, 40 * R), (5, 70 * R)]
        _run_stream(plan, calls, seed=1)
        plan.reset()
        _run_stream(plan, calls, seed=2)
        for count in (0, 1, L // 2, L - 2):
            tail = _ints(count, 50 + count)
            xs = [_ints(f * t, 60 + count + i) for i, (f, t) in enumerate(calls)]
            plan.set_history(tail)
            want = _model(plan.taps, R, torch.cat([tail] + xs), prefix=count)
            q = 0
            for i, ((f, t), x) in enumerate(zip(calls, xs)):
                n_out = f * (t // R)
                _assert_exact(plan.exec(x, f, t), want[q:q + n_out], f"set_history({count}): call {i}")
                q += n_out
