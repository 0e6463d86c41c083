"""The forms of fft4096_kernel that the spectral-chain entry points reach at n = 4096, their F64 models and the exact
F32 summation orders of the column sums (test infrastructure).

FORMS lists (entry point, MODE, WIN, ITYPE) for every instantiation the default dispatch of fft.cu launches:
  b200_chain_exec         {AMP, AMP_RANGE} x {WIN_REAL, WIN_COMPLEX, WIN_NONE}       IN_CF32
  b200_chain_exec_typed   {AMP, AMP_RANGE} x {CI8, CU8, CI16, CU16}                  WIN_REAL (launch_4096_int)
  b200_chain_exec_agc     {AMP, AMP_RANGE} x {CF32, CI8, CU8, CI16, CU16}            WIN_REAL, AGC
  b200_chain_exec_colsum  {AMP, AMP_RANGE} x {CF32, CI8, CU8, CI16, CU16}            WIN_REAL, COLSUM

The models work in F64 from the exact input values: integer samples are (F32)v / 128 or / 32768 (unsigned samples are
not re-centred), the window is applied, np.fft.fft transforms, dB = 20 approx_log10_f64(|X|) + coeff (-inf at |X| == 0) and
range = 0.5 + 0.5 tanh(4 ((dB scale + offset) - 0.5)). AGC scales a row's spectrum by
clamp(reference / sqrt(mean |X|^2 + epsilon), min, max), with mean |X|^2 = sum |x w|^2 over the windowed row (Parseval).
"""
import numpy as np

from parity import approx_log10_f64

MODES = ("MODE_AMP", "MODE_AMP_RANGE")
INT_TYPES = ("IN_CI8", "IN_CU8", "IN_CI16", "IN_CU16")

FORMS = ([("chain_exec", m, w, "IN_CF32") for m in MODES for w in ("WIN_REAL", "WIN_COMPLEX", "WIN_NONE")] +
         [("chain_exec_typed", m, "WIN_REAL", t) for m in MODES for t in INT_TYPES] +
         [("chain_exec_agc", m, "WIN_REAL", t) for m in MODES for t in ("IN_CF32",) + INT_TYPES] +
         [("chain_exec_colsum", m, "WIN_REAL", t) for m in MODES for t in ("IN_CF32",) + INT_TYPES])

# ITYPE -> (B200_DTYPE code, numpy component type, scaler); CI32 / CU32 never reach fft4096_kernel directly
DTYPES = {"IN_CF32": (1, np.float32, None), "IN_CI8": (8, np.int8, 128.0), "IN_CU8": (9, np.uint8, 128.0),
          "IN_CI16": (10, np.int16, 32768.0), "IN_CU16": (11, np.uint16, 32768.0),
          "IN_CI32": (12, np.int32, 2147483648.0), "IN_CU32": (13, np.uint32, 2147483648.0)}


def form_id(form):
    entry, mode, win, itype = form
    return f"{entry}-{mode[5:]}-{win[4:]}-{itype[3:]}"


def exact_samples(x, itype):
    """[rows, n] complex128 of what the kernel reads: CF32 as is, integer pairs [rows, n, 2] converted to F32 (exact up to
    16 bits, rounded to nearest for 32-bit samples) and divided by the scaler."""
    if itype == "IN_CF32":
        return x.astype(np.complex128)
    scaler = DTYPES[itype][2]
    f = x.astype(np.float32).astype(np.float64)
    return (f[..., 0] + 1j * f[..., 1]) / scaler


def spectrum(samples, window):
    """F64 spectrum of the windowed rows (window None: WIN_NONE)."""
    return np.fft.fft(samples if window is None else samples * window.astype(np.complex128), axis=1)


def agc_gain(samples, window, reference, epsilon, min_gain, max_gain, clamp=True):
    """Per-row AGC gain [rows, 1] from the windowed row's power."""
    xw = samples if window is None else samples * window.astype(np.complex128)
    g = reference / np.sqrt((np.abs(xw) ** 2).sum(axis=1, keepdims=True) + epsilon)
    return np.clip(g, min_gain, max_gain) if clamp else g


def db(spec, coeff):
    mag = np.abs(spec)
    with np.errstate(divide="ignore"):
        return np.where(mag > 0, 20.0 * approx_log10_f64(mag) + coeff, -np.inf)


def to_range(db_values, scale, offset):
    return 0.5 + 0.5 * np.tanh(4.0 * ((db_values * scale + offset) - 0.5))


# ---- column sums -------------------------------------------------------------------------------------------------
def colsum_fused(out, sms):
    """The COLSUM form of fft4096_kernel: CTA b of G = min(batch, 2 SMs) adds rows b, b + G, b + 2G, ... in F32 from +0,
    then colsum_reduce adds the G partials in CTA order 0 ... G-1 from +0."""
    batch, n = out.shape
    g = min(batch, 2 * sms)
    partial = np.zeros((g, n), np.float32)
    for r0 in range(0, batch, g):
        rows = out[r0:r0 + g]
        partial[:len(rows)] += rows
    total = np.zeros(n, np.float32)
    for b in range(g):
        total += partial[b]
    return total


def colsum_splits(batch, n, sms):
    """colsum_partials' row splits for dense, 16-byte aligned [batch, n] F32 rows (n % 4 == 0: 1024 columns per CTA)."""
    column_blocks = -(-n // 1024)
    return max(1, min(-(-4 * sms // column_blocks), -(-batch // 64)))


def colsum_row_split(out, sms):
    """colsum_partials + colsum_reduce: `splits` contiguous runs of ceil(batch / splits) rows, each summed in row order
    in F32 from +0, then the runs added in order from +0."""
    batch, n = out.shape
    splits = colsum_splits(batch, n, sms)
    per = -(-batch // splits)
    total = np.zeros(n, np.float32)
    for s in range(splits):
        acc = np.zeros(n, np.float32)
        for r in range(s * per, min(batch, (s + 1) * per)):
            acc += out[r]
        total += acc
    return total


def lineplot_from_colsum(colsum, decimation, normalization, averaging, average):
    """lineplot_finalize_kernel over one partial (b200_lineplot_update_from_colsum), every step rounded to F32: the new
    average, which is also the y column of signalPoints."""
    elements = average.size
    s = np.float32(0.0) + colsum[:elements * decimation:decimation]
    amp = np.fmin(np.fmax(s * np.float32(normalization) - np.float32(1.0), np.float32(-1.0)), np.float32(1.0))
    avg = average - average / np.float32(averaging)
    return avg + amp / np.float32(averaging)


def lineplot_x(elements):
    """lineplot_init_kernel's x coordinates: e * 2.0f / (elements - 1) - 1.0f."""
    e = np.arange(elements, dtype=np.float32)
    return e * np.float32(2.0) / np.float32(elements - 1) - np.float32(1.0)
