"""In-tree build of libb200dsp.so for sm_90a (nvcc cross-compiles without a GPU): every .cu is compiled to an object
in parallel (objects cached under csrc/_obj by source mtime), then linked into one shared library."""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(CSRC, "_obj")
SOURCES = ["context.cu", "elementwise.cu", "fft.cu", "fir.cu", "fm.cu", "agc.cu", "viz.cu", "filter_stages.cu"]
OUT = os.path.join(HERE, "libb200dsp.so")
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC"]


def _newest_header() -> float:
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    headers.append(os.path.join(os.path.dirname(HERE), "include", "b200dsp.h"))
    return max(os.path.getmtime(h) for h in headers)


def needs_build() -> bool:
    if not os.path.exists(OUT):
        return True
    newest = max([os.path.getmtime(os.path.join(CSRC, f)) for f in SOURCES] + [_newest_header()])
    return newest > os.path.getmtime(OUT)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return OUT
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    os.makedirs(OBJ, exist_ok=True)
    header_time = _newest_header()

    def compile_one(src: str) -> str:
        obj = os.path.join(OBJ, src.replace(".cu", ".o"))
        stale = force or not os.path.exists(obj) or \
            max(os.path.getmtime(os.path.join(CSRC, src)), header_time) > os.path.getmtime(obj)
        if stale:
            cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj]
            subprocess.run(cmd, cwd=CSRC, check=True)
        return obj

    with ThreadPoolExecutor(max_workers=min(len(SOURCES), os.cpu_count() or 1)) as pool:
        objects = list(pool.map(compile_one, SOURCES))
    subprocess.run([nvcc] + NVCC_FLAGS[:2] + ["-shared", "-o", OUT] + objects, cwd=CSRC, check=True)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
