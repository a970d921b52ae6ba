"""Every CUDA allocation, free, stream and event the host code makes goes through the owners in cuda_buffers.h, which free
on destruction. A raw call anywhere else is memory some hand-written list has to remember to free."""
import glob
import os
import re

import common

CSRC = os.path.join(common.ROOT, "usearch_b200", "csrc")
OWNER = "cuda_buffers.h"
RAW = re.compile(r"\b(cudaMalloc|cudaFree|cudaHostAlloc|cudaFreeHost|cudaStreamDestroy|cudaEventDestroy)\s*\(")


def sources():
    paths = []
    for pattern in ("*.cu", "*.h", "*.cuh"):
        paths += glob.glob(os.path.join(CSRC, pattern))
    assert any(p.endswith(OWNER) for p in paths)
    return sorted(paths)


def test_raw_allocations_only_in_the_owners():
    offending = []
    for path in sources():
        if os.path.basename(path) == OWNER:
            continue
        with open(path, encoding="utf-8") as f:
            for number, line in enumerate(f, 1):
                if RAW.search(line):
                    offending.append(f"{os.path.basename(path)}:{number}: {line.strip()}")
    assert not offending, "raw CUDA allocation or release outside cuda_buffers.h:\n" + "\n".join(offending)


def test_no_buffer_on_the_heap():
    offending = []
    for path in sources():
        with open(path, encoding="utf-8") as f:
            for number, line in enumerate(f, 1):
                if re.search(r"\bnew\s+device_buffer_t\b", line):
                    offending.append(f"{os.path.basename(path)}:{number}: {line.strip()}")
    assert not offending, "\n".join(offending)
