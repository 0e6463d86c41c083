"""Throughput of the filter-stage kernels (b200_fold, b200_overlap_add, b200_phase_correction, and pad / unpad as
b200_copy_strided) at the Overlap-Add-Fold example's per-head shapes scaled to 1024 frames, plus one filter_engine cycle
in the reference Flowgraph on provider b200 against the reference CPU provider. CUDA events around device-resident
calls; GB/s over the bytes each stage must read and write. Card name and power limit are read in the same run.
Usage: python tools/bench_filter_stages.py [out.json]"""
import ctypes
import json
import math
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from cyberether_b200 import _native  # noqa: E402

assert torch.cuda.is_available(), "bench_filter_stages needs cuda:0"
lib = _native.load()
check = _native.check
dev = torch.device("cuda:0")
ctx = ctypes.c_void_p()
check(lib.b200_ctx_create(0, ctypes.byref(ctx)))
stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def timeit(fn, iters=50, warm=5):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


results = []


def report(name, ms, nbytes):
    gbs = nbytes / ms * 1e-6
    results.append({"stage": name, "ms": ms, "algorithmic_bytes": nbytes, "gbs": gbs})
    print(f"{name:58s} {ms:8.4f} ms {gbs:8.0f} GB/s")


def cf32(*shape):
    g = torch.Generator(device=dev)
    g.manual_seed(len(shape) + shape[-1])
    return torch.view_as_complex(torch.randn(*shape, 2, device=dev, generator=g))


def u64(*values):
    return (ctypes.c_uint64 * len(values))(*values)


frames, heads, m, size, taps_pad = 1024, 2, 8100, 810, 10
# fold [1024, 2, 8100] -> [1024, 2, 810], per-head offsets
x = cf32(frames, heads, m)
y = torch.empty(frames, heads, size, dtype=torch.complex64, device=dev)
offsets = torch.tensor([1620, 8100 - 1620], dtype=torch.int64, device=dev)
report(f"fold CF32 [{frames}, {heads}, {m}] -> {size} (per-head offsets)",
       timeit(lambda: check(lib.b200_fold(ctx, x.data_ptr(), y.data_ptr(), 1, frames * heads, m, 1, size, 0,
                                          offsets.data_ptr(), heads, size, stream))),
       8 * (x.numel() + y.numel()))
# phase_correction on the folded, inverse-transformed frames [1024, 2, 810]: batch axis 0, channel axis 1
wrapped = (ctypes.c_double * heads)(*[math.remainder(2 * math.pi * o * 8000 / 8100, 2 * math.pi) for o in (1620, 6480)])
phases = (ctypes.c_double * heads)(0.0, 0.0)
z = torch.empty_like(y)
report(f"phase_correction CF32 [{frames}, {heads}, {size}]",
       timeit(lambda: check(lib.b200_phase_correction(ctx, y.data_ptr(), z.data_ptr(), y.numel(), frames, heads * size,
                                                      heads, size, phases, wrapped, stream))),
       16 * y.numel())
# unpad [1024, 2, 810] -> [1024, 2, 800] + [1024, 2, 10]: two strided copies
body = torch.empty(frames, heads, size - taps_pad, dtype=torch.complex64, device=dev)
tail = torch.empty(frames, heads, taps_pad, dtype=torch.complex64, device=dev)


def unpad():
    check(lib.b200_copy_strided(ctx, z.data_ptr(), body.data_ptr(), 8, 2, u64(frames * heads, size - taps_pad),
                                u64(size, 1), u64(size - taps_pad, 1), stream))
    check(lib.b200_copy_strided(ctx, z.data_ptr() + 8 * (size - taps_pad), tail.data_ptr(), 8, 2,
                                u64(frames * heads, taps_pad), u64(size, 1), u64(taps_pad, 1), stream))


report(f"unpad CF32 [{frames}, {heads}, {size}] -> {size - taps_pad} + {taps_pad}", timeit(unpad), 16 * z.numel())
# overlap_add [1024, 2, 800] + [1024, 2, 10], batch axis 0
out = torch.empty_like(body)
previous = torch.zeros(1, heads, taps_pad, dtype=torch.complex64, device=dev)
report(f"overlap_add CF32 [{frames}, {heads}, {size - taps_pad}] + [.., {taps_pad}]",
       timeit(lambda: check(lib.b200_overlap_add(ctx, body.data_ptr(), tail.data_ptr(), out.data_ptr(),
                                                 previous.data_ptr(), 1, frames * heads, size - taps_pad, taps_pad, 1,
                                                 frames, heads * taps_pad, stream))),
       8 * (2 * body.numel() + tail.numel() + 2 * previous.numel()))
# pad [1024, 8000] -> [1024, 8100]: body copy + stride-0 copy of a zero element
s = cf32(frames, 8000)
padded = torch.empty(frames, m, dtype=torch.complex64, device=dev)
zero = torch.zeros(1, dtype=torch.complex64, device=dev)


def pad():
    check(lib.b200_copy_strided(ctx, s.data_ptr(), padded.data_ptr(), 8, 2, u64(frames, 8000), u64(8000, 1),
                                u64(m, 1), stream))
    check(lib.b200_copy_strided(ctx, zero.data_ptr(), padded.data_ptr() + 8 * 8000, 8, 2, u64(frames, m - 8000),
                                u64(0, 0), u64(m, 1), stream))


report(f"pad CF32 [{frames}, 8000] -> {m}", timeit(pad), 8 * (s.numel() + padded.numel()))

# one filter_engine cycle (source -> filter_taps -> filter_engine), Overlap-Add-Fold example configuration
engine = []
from shim import binding  # noqa: E402
if binding.available():
    taps = {"taps": 101, "heads": 2, "center": [400e3, -400e3], "bandwidth": 200e3, "sampleRate": 2e6}
    for rows in (8, 256):
        sig = (np.random.default_rng(rows).standard_normal((rows, 8000, 2)).astype(np.float32)
               .view(np.complex64)[..., 0])
        row = {"shape": [rows, 8000]}
        for target in (binding.CPU, binding.B200):
            with binding.Session() as sess:
                sess.add_source("src", sig.shape, "CF32", target=target, sampleAxis=1, batchAxis=0)
                sess.add_block("taps", "filter_taps", taps, {}, target=target)
                sess.add_block("fe", "filter_engine", None, {"signal": "src.signal", "filter": "taps.coeffs"},
                               target=target)
                sess.write_source("src", sig)
                for _ in range(3):
                    sess.compute()
                reps = 20 if target is binding.B200 else 3
                t0 = time.perf_counter()
                for _ in range(reps):
                    sess.compute()          # synchronous: returns after the cycle's device work
                row[target[1] + "_ms"] = (time.perf_counter() - t0) / reps * 1e3
        row["speedup"] = row["generic_ms"] / row["b200_ms"]
        engine.append(row)
        print(f"filter_engine cycle [{rows}, 8000]: CPU provider {row['generic_ms']:.2f} ms, b200 {row['b200_ms']:.3f} ms "
              f"({row['speedup']:.1f}x)")

smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                     capture_output=True, text=True).stdout.strip()
card = {"name": torch.cuda.get_device_name(0), "nvidia_smi": smi}
print(f"card: {card['name']} ({smi})")
lib.b200_ctx_destroy(ctx)
if len(sys.argv) > 1:
    with open(sys.argv[1], "w") as f:
        json.dump({"card": card, "stages": results, "filter_engine": engine}, f, indent=1)
