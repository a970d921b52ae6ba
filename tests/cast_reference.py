"""Both sides of the scalar-cast tests, compiled at test time into temporary directories.

* :func:`ref_cast` — the reference's own cast_gt (tests/native/ref_casts_driver.cpp against the unmodified reference
  sources, with the defines of the oracle's parity build). Needs the reference sources: :func:`reference_available`.
* :func:`host_cast` — usearch_b200/csrc/scalar_casts.h's `cast_row_host` (tests/native/scalar_casts_shim.cpp), the casts
  of `get` and the element conversions the device casts share. Needs only g++; the CPU tests pin it to the reference
  over every f32 pattern, and the GPU tests hold the device to it where the reference sources are absent."""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

import common
from oracle import bindings

NATIVE = os.path.join(common.ROOT, "tests", "native")
CSRC = os.path.join(common.ROOT, "usearch_b200", "csrc")
PARITY = ["-O2", "-ffp-contract=off", "-march=x86-64-v3"]

_libs: dict = {}


def reference_available() -> bool:
    from oracle import build as oracle_build
    return oracle_build.reference_available()


def ref_lib_path() -> str:
    """the reference's casts as a shared library (built once per process)"""
    if "ref" in _libs:
        return _libs["ref"]
    from oracle import build as oracle_build
    ref = oracle_build.REF
    defines = ["-DUSEARCH_USE_SIMSIMD=1", "-DUSEARCH_USE_FP16LIB=0", "-DUSEARCH_USE_OPENMP=0", "-DSIMSIMD_NATIVE_F16=0",
               "-DSIMSIMD_NATIVE_BF16=0", "-DSIMSIMD_DYNAMIC_DISPATCH=1", f"-I{ref}/include", f"-I{ref}/simsimd/include",
               f"-I{ref}/fp16/include", "-w", "-fPIC"]
    out = tempfile.mkdtemp(prefix="ref_casts_")
    simsimd = os.path.join(out, "simsimd.o")
    lib = os.path.join(out, "libref_casts.so")
    subprocess.run(["gcc", "-std=c11", "-O3", *defines, "-c", f"{ref}/simsimd/c/lib.c", "-o", simsimd], check=True,
                   capture_output=True)
    subprocess.run(["g++", "-std=c++17", *PARITY, *defines, "-shared", os.path.join(NATIVE, "ref_casts_driver.cpp"), simsimd,
                    "-o", lib, "-lpthread", "-lm"], check=True, capture_output=True)
    _libs["ref"] = lib
    return lib


def _ref() -> C.CDLL:
    if "ref_dll" not in _libs:
        lib = C.CDLL(ref_lib_path())
        lib.ref_cast.restype = C.c_int
        lib.ref_cast.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p]
        _libs["ref_dll"] = lib
    return _libs["ref_dll"]


def host() -> C.CDLL:
    """the shim over scalar_casts.h (built once per process)"""
    if "host" not in _libs:
        out = os.path.join(tempfile.mkdtemp(prefix="scalar_casts_"), "libscalar_casts.so")
        subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-Wextra", "-Werror", "-shared", "-fPIC", "-I", CSRC,
                        os.path.join(NATIVE, "scalar_casts_shim.cpp"), "-o", out], check=True, capture_output=True)
        lib = C.CDLL(out)
        lib.shim_cast_row.restype = C.c_int
        lib.shim_cast_row.argtypes = [C.c_uint32, C.c_uint32, C.c_size_t, C.c_void_p, C.c_void_p]
        for name in ("shim_f32_to_f16", "shim_f32_to_bf16"):
            getattr(lib, name).restype = C.c_uint16
            getattr(lib, name).argtypes = [C.c_uint32]
        lib.shim_f16_to_f32.restype = C.c_uint32
        lib.shim_f16_to_f32.argtypes = [C.c_uint16]
        _libs["host"] = lib
    return _libs["host"]


def _rows(src: np.ndarray, kind: str, dims: int) -> np.ndarray:
    return np.ascontiguousarray(src).view(np.uint8).reshape(-1, bindings.bytes_per_vector(dims, kind))


def ref_cast(src: np.ndarray, from_kind: str, to_kind: str, dims: int) -> np.ndarray:
    """cast_gt<from, to> of the reference over dense rows of raw bytes: (rows, bytes of `from`) -> (rows, bytes of `to`).
    The output starts zeroed, so a b1 row's padding bits are zero."""
    src = _rows(src, from_kind, dims)
    out = np.zeros((src.shape[0], bindings.bytes_per_vector(dims, to_kind)), dtype=np.uint8)
    rc = _ref().ref_cast(bindings.SCALAR[from_kind], bindings.SCALAR[to_kind], src.ctypes.data, src.shape[0], dims,
                         out.ctypes.data)
    if rc:
        raise RuntimeError(f"ref_cast {from_kind} -> {to_kind} failed: {rc}")
    return out


def host_cast(src: np.ndarray, from_kind: str, to_kind: str, dims: int) -> np.ndarray:
    """scalar_casts.h's cast_row_host over the same rows (its b1 rows are written whole, padding zero)"""
    src = _rows(src, from_kind, dims)
    out = np.full((src.shape[0], bindings.bytes_per_vector(dims, to_kind)), 0xA5, dtype=np.uint8)
    lib = host()
    for r in range(src.shape[0]):
        rc = lib.shim_cast_row(bindings.SCALAR[from_kind], bindings.SCALAR[to_kind], dims, src[r].ctypes.data,
                               out[r].ctypes.data)
        if rc:
            raise RuntimeError(f"cast_row_host {from_kind} -> {to_kind} failed")
    return out


def _element_bytes(kind: str) -> int:
    return {"f64": 8, "f32": 4, "f16": 2, "bf16": 2, "i8": 1, "b1": 0}[kind]


def assert_same_casts(want: np.ndarray, got: np.ndarray, src: np.ndarray, from_kind: str, to_kind: str, dims: int,
                      what: str) -> None:
    """rows of `to_kind` bytes equal, else an AssertionError naming the first differing element: its input bytes, the
    expected output (`want`) and ours (`got`)"""
    assert want.shape == got.shape, (what, want.shape, got.shape)
    bad = np.nonzero((want != got).any(axis=1))[0]
    if not bad.size:
        return
    r = int(bad[0])
    raw = _rows(src, from_kind, dims)[r]
    col = int(np.nonzero(want[r] != got[r])[0][0])
    eb, fb = _element_bytes(to_kind), _element_bytes(from_kind)
    j = col // eb if eb else col * 8  # the first differing element (b1: its byte's first element)
    span = raw[j * fb:(j + 1) * fb] if fb else raw[j // 8:j // 8 + 1]
    lo = (j * eb, (j + 1) * eb) if eb else (col, col + 1)
    raise AssertionError(f"{what}: {from_kind} -> {to_kind}, dims {dims}: {bad.size} rows differ; row {r} element {j}: "
                         f"input bytes {span[::-1].tobytes().hex()}, expected {want[r, lo[0]:lo[1]][::-1].tobytes().hex()}, "
                         f"ours {got[r, lo[0]:lo[1]][::-1].tobytes().hex()}")
