"""The owners of device buffers, pinned buffers, streams and events (usearch_b200/csrc/cuda_buffers.h), natively and
without a GPU: tests/native/test_cuda_buffers.cpp links the header against counting stand-ins for the CUDA runtime."""
import os
import subprocess

import common
from usearch_b200 import build

CUDA_INCLUDE = os.path.join(os.path.dirname(os.path.dirname(build.NVCC)), "include")  # the toolkit the library builds with


def test_cuda_owners_free_exactly_once(tmp_path):
    """Scope exit frees, reserve only grows, a failed reserve leaves the owner empty, moves hand the resource over and
    free the target's own, and a vector of owners survives hundreds of reallocations with nothing leaked or freed twice."""
    exe = str(tmp_path / "test_cuda_buffers")
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-I", CUDA_INCLUDE,
                    "-I", os.path.join(common.ROOT, "usearch_b200", "csrc"),
                    os.path.join(common.ROOT, "tests", "native", "test_cuda_buffers.cpp"), "-o", exe], check=True)
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "CUDA_BUFFERS_OK" in out.stdout
