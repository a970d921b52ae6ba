"""In-tree build of ``usearch_b200/libusearch_b200.so`` with nvcc for sm_90a (H100).

The shared library is git-ignored; ``__graft_entry__.build()`` calls :func:`build`, which rebuilds
it whenever a source, a header or this recipe is newer than the library.
"""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libusearch_b200.so")
SOURCES = ["c_abi.cu", "frozen_index.cu", "search_kernel.cu", "exact_kernel.cu", "exact_imma.cu", "exact_wgmma.cu", "builder.cu", "shards.cu", "join.cu", "indexes.cu", "surface.cu", "device_keys.cu", "grouped_filter.cu"]
HEADERS = ["device_index.h", "frozen_index.h", "metrics.cuh", "warp_primitives.cuh", "exact_args.h", "exact_i8.h", "key_map.h", "device_keys.h", "prefilter_bound.h", "search_order.h",
           "join_resolve.h", "cuda_check.h", "cuda_buffers.h", "f64_casts.h", "scalar_casts.h", os.path.join("..", "..", "include", "usearch_b200.h")]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = [
    *ARCH, "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "--shared", "-cudart", "static",
]
LINK_LIBS = ["-ldl"]


def _stale() -> bool:
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS] + [os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not _stale():
        return OUT
    def compile_one(src: str) -> str:
        obj = os.path.join(CSRC, src.replace(".cu", ".o"))
        cmd = [NVCC, *[f for f in FLAGS if f not in ("--shared",)], "-c", os.path.join(CSRC, src), "-o", obj]
        if verbose and src == "search_kernel.cu":
            cmd += ["-Xptxas", "-v"]
        proc = subprocess.run(cmd, capture_output=True, text=True)
        if proc.returncode != 0:
            sys.stderr.write(" ".join(cmd) + "\n" + proc.stdout + proc.stderr)
            raise RuntimeError(f"nvcc failed on {src}")
        if verbose:
            sys.stderr.write(proc.stderr)
        return obj

    from concurrent.futures import ThreadPoolExecutor
    with ThreadPoolExecutor(max_workers=len(SOURCES)) as pool:  # one nvcc per translation unit, side by side
        objs = list(pool.map(compile_one, SOURCES))
    cmd = [NVCC, "--shared", "-cudart", "static", *ARCH, "-o", OUT, *objs, *LINK_LIBS]
    proc = subprocess.run(cmd, capture_output=True, text=True)
    if proc.returncode != 0:
        sys.stderr.write(" ".join(cmd) + "\n" + proc.stdout + proc.stderr)
        raise RuntimeError("link failed")
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
