"""Host-side mirror of the reference's Python search API over the C ABI.

Mirrors, for the search path only, ``usearch.index.Index`` (/root/reference/python/usearch/index.py):
``Index.search`` (index.py:700-748) → ``_search_in_compiled`` (:191-231) → ``search_many``
(python/lib.cpp:415-461), and the result containers ``Matches`` / ``BatchMatches`` (:300-396).
Same argument names and meaning, same shapes and dtypes of the results, same padding of short
rows. Everything below goes through ``libusearch_b200.so`` with plain pointers (ctypes); there is
no CPU fallback: without the CUDA library or without a GPU the calls raise.
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass
from typing import Dict, Optional, Union

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libusearch_b200.so")

# usearch.h:40-62 ordinals
METRIC_KIND = {"cos": 1, "ip": 2, "l2sq": 3, "haversine": 4, "divergence": 5, "pearson": 6, "jaccard": 7,
               "hamming": 8, "tanimoto": 9, "sorensen": 10}
SCALAR_KIND = {"f32": 1, "f64": 2, "f16": 3, "i8": 4, "b1": 5, "bf16": 6}
_NP_TO_SCALAR = {np.dtype(np.float32): "f32", np.dtype(np.float64): "f64", np.dtype(np.float16): "f16",
                 np.dtype(np.int8): "i8", np.dtype(np.uint8): "b1"}
_BITS = {"f32": 32, "f64": 64, "f16": 16, "bf16": 16, "i8": 8, "b1": 1}


class _InitOptions(C.Structure):  # usearch.h:64-110
    _fields_ = [("metric_kind", C.c_int), ("metric", C.c_void_p), ("quantization", C.c_int),
                ("dimensions", C.c_size_t), ("connectivity", C.c_size_t), ("expansion_add", C.c_size_t),
                ("expansion_search", C.c_size_t), ("multi", C.c_bool)]


_lib: Optional[C.CDLL] = None

EXPORTED_SYMBOLS = [
    "usearch_version", "usearch_init", "usearch_free", "usearch_memory_usage", "usearch_hardware_acceleration",
    "usearch_serialized_length", "usearch_save", "usearch_load", "usearch_view", "usearch_metadata",
    "usearch_save_buffer", "usearch_load_buffer", "usearch_view_buffer", "usearch_metadata_buffer", "usearch_size",
    "usearch_capacity", "usearch_dimensions", "usearch_connectivity", "usearch_reserve", "usearch_expansion_add",
    "usearch_expansion_search", "usearch_change_expansion_add", "usearch_change_expansion_search",
    "usearch_change_threads_add", "usearch_change_threads_search", "usearch_change_metric_kind",
    "usearch_change_metric", "usearch_add", "usearch_contains", "usearch_count", "usearch_search",
    "usearch_filtered_search", "usearch_get", "usearch_remove", "usearch_rename", "usearch_distance",
    "usearch_exact_search", "usearch_clear",
    # additive
    "usearch_search_many", "usearch_b200_search_many_device", "usearch_b200_search_many_stats",
    "usearch_b200_filtered_search_many", "usearch_b200_exact_search_many", "usearch_b200_cluster_many",
    "usearch_b200_profile_phases", "usearch_b200_profile_phases_n", "usearch_b200_device", "usearch_b200_kernel_launches", "usearch_b200_last_kernel_ms",
    "usearch_b200_bytes_per_vector", "usearch_b200_max_level", "usearch_b200_add_many", "usearch_b200_add_many_device",
    "usearch_b200_shards_unique_id", "usearch_b200_shards_join", "usearch_b200_sharded_search_many",
    "usearch_b200_sharded_search_many_device", "usearch_b200_shards_payload_bytes", "usearch_b200_merge_topk",
    "usearch_b200_search_many_enqueue", "usearch_b200_search_many_finish", "usearch_b200_tune",
    "usearch_b200_launch_plan", "usearch_b200_remove_many", "usearch_b200_count_many", "usearch_b200_change_reuse_removed",
    "usearch_b200_reuse_removed", "usearch_b200_join", "usearch_b200_pairwise_distances",
    "usearch_b200_last_join_ms", "usearch_b200_indexes_init", "usearch_b200_indexes_free", "usearch_b200_indexes_merge",
    "usearch_b200_indexes_size", "usearch_b200_indexes_search_many", "usearch_b200_indexes_last_ms", "usearch_b200_merge_into",
    "usearch_b200_get_many", "usearch_b200_export_keys", "usearch_b200_export_keys_at", "usearch_b200_copy",
    "usearch_b200_levels_stats", "usearch_b200_multi", "usearch_b200_count_many_device", "usearch_b200_get_many_device",
    "usearch_b200_filtered_search_many_device", "usearch_b200_grouped_filtered_search_many",
    "usearch_b200_grouped_filtered_search_many_device", "usearch_b200_grouped_filtered_exact_search_many",
    "usearch_b200_grouped_filtered_exact_search_many_device", "usearch_b200_exact_search_device",
    "usearch_b200_grouped_excluded_search_many", "usearch_b200_grouped_excluded_search_many_device",
    "usearch_b200_grouped_excluded_exact_search_many", "usearch_b200_grouped_excluded_exact_search_many_device",
]

# the fields of usearch_b200_launch_plan, in order
LAUNCH_PLAN_FIELDS = ["stage_sets", "warps_per_sm_target", "blocks", "smem_per_warp", "heap_smem_cap", "heap_spill_cap",
                      "visits", "visited_cap", "code_pass", "code_smem_stride", "qsplit_len", "prefilter", "stage_bytes"]
_VISITS = ["hash", "bitmap", "bitmap_log"]


def load_library() -> C.CDLL:
    """Load the CUDA library. Fails loudly: there is no pure-Python or CPU implementation behind it."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                          "(nvcc, sm_90a). The GPU backend has no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    err = C.POINTER(C.c_char_p)
    lib.usearch_version.restype = C.c_char_p
    lib.usearch_init.restype = C.c_void_p
    lib.usearch_init.argtypes = [C.POINTER(_InitOptions), err]
    lib.usearch_free.argtypes = [C.c_void_p, err]
    lib.usearch_hardware_acceleration.restype = C.c_char_p
    lib.usearch_hardware_acceleration.argtypes = [C.c_void_p, err]
    for name in ("usearch_memory_usage", "usearch_serialized_length", "usearch_size", "usearch_capacity",
                 "usearch_dimensions", "usearch_connectivity", "usearch_expansion_add", "usearch_expansion_search"):
        getattr(lib, name).restype = C.c_size_t
        getattr(lib, name).argtypes = [C.c_void_p, err]
    for name in ("usearch_change_expansion_add", "usearch_change_expansion_search"):
        getattr(lib, name).argtypes = [C.c_void_p, C.c_size_t, err]
    for name in ("usearch_save", "usearch_load", "usearch_view"):
        getattr(lib, name).argtypes = [C.c_void_p, C.c_char_p, err]
    for name in ("usearch_save_buffer", "usearch_load_buffer", "usearch_view_buffer"):
        getattr(lib, name).argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, err]
    lib.usearch_metadata_buffer.argtypes = [C.c_void_p, C.c_size_t, C.POINTER(_InitOptions), err]
    lib.usearch_metadata.argtypes = [C.c_char_p, C.POINTER(_InitOptions), err]
    lib.usearch_clear.argtypes = [C.c_void_p, err]
    lib.usearch_add.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_int, err]
    lib.usearch_search.restype = C.c_size_t
    lib.usearch_search.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_size_t, C.c_void_p, C.c_void_p, err]
    lib.usearch_search_many.restype = C.c_size_t
    lib.usearch_search_many.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int, C.c_size_t,
                                        C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, err]
    lib.usearch_b200_search_many_stats.restype = C.c_size_t
    lib.usearch_b200_search_many_stats.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int,
                                                   C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                   C.c_void_p, err]
    lib.usearch_b200_search_many_device.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t,
                                                    C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                    C.c_void_p, err]
    lib.usearch_b200_search_many_enqueue.argtypes = lib.usearch_b200_search_many_device.argtypes
    lib.usearch_b200_count_many_device.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, err]
    lib.usearch_b200_get_many_device.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p, C.c_size_t,
                                                 C.c_int, C.c_void_p, C.c_void_p, err]
    lib.usearch_b200_filtered_search_many_device.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t,
                                                             C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p,
                                                             C.c_void_p, C.c_void_p, C.c_void_p, err]
    lib.usearch_b200_search_many_finish.argtypes = [C.c_void_p, err]
    lib.usearch_b200_grouped_filtered_search_many.restype = C.c_size_t
    lib.usearch_b200_grouped_filtered_search_many.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int, C.c_size_t,
                                                              C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p,
                                                              C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, err]
    lib.usearch_b200_grouped_filtered_search_many_device.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t,
                                                                     C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p,
                                                                     C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                                     err]
    lib.usearch_b200_grouped_filtered_exact_search_many.restype = C.c_size_t
    lib.usearch_b200_grouped_filtered_exact_search_many.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int,
                                                                    C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p,
                                                                    C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, err]
    lib.usearch_b200_grouped_filtered_exact_search_many_device.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t,
                                                                           C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t,
                                                                           C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                                           C.c_void_p, C.c_void_p, err]
    # the excluded entries take the grouped filtered entries' arguments
    lib.usearch_b200_grouped_excluded_search_many.restype = C.c_size_t
    lib.usearch_b200_grouped_excluded_search_many.argtypes = lib.usearch_b200_grouped_filtered_search_many.argtypes
    lib.usearch_b200_grouped_excluded_search_many_device.argtypes = lib.usearch_b200_grouped_filtered_search_many_device.argtypes
    lib.usearch_b200_grouped_excluded_exact_search_many.restype = C.c_size_t
    lib.usearch_b200_grouped_excluded_exact_search_many.argtypes = lib.usearch_b200_grouped_filtered_exact_search_many.argtypes
    lib.usearch_b200_grouped_excluded_exact_search_many_device.argtypes = \
        lib.usearch_b200_grouped_filtered_exact_search_many_device.argtypes
    lib.usearch_b200_tune.restype = C.c_int
    lib.usearch_b200_tune.argtypes = [C.c_void_p, C.c_char_p, C.c_int]
    lib.usearch_b200_launch_plan.restype = C.c_int
    lib.usearch_b200_launch_plan.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, err]
    lib.usearch_b200_filtered_search_many.restype = C.c_size_t
    lib.usearch_b200_filtered_search_many.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int,
                                                      C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p,
                                                      C.c_void_p, C.c_void_p, C.c_void_p, err]
    lib.usearch_b200_cluster_many.restype = None
    lib.usearch_b200_cluster_many.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int, C.c_size_t, C.c_void_p,
                                              C.c_void_p, C.c_void_p, C.c_void_p, err]
    lib.usearch_b200_exact_search_many.restype = C.c_size_t
    lib.usearch_b200_exact_search_many.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int, C.c_size_t,
                                                   C.c_void_p, C.c_void_p, C.c_void_p, err]
    lib.usearch_exact_search.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int,
                                         C.c_size_t, C.c_int, C.c_size_t, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p,
                                         C.c_size_t, err]
    lib.usearch_b200_exact_search_device.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int,
                                                     C.c_size_t, C.c_int, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t,
                                                     C.c_void_p, err]
    lib.usearch_b200_profile_phases.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    lib.usearch_b200_profile_phases_n.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t]
    lib.usearch_b200_profile_phases_n.restype = C.c_size_t
    lib.usearch_b200_device.argtypes = [C.c_void_p]
    lib.usearch_b200_kernel_launches.restype = C.c_uint64
    lib.usearch_b200_kernel_launches.argtypes = [C.c_void_p]
    lib.usearch_b200_last_kernel_ms.restype = C.c_float
    lib.usearch_b200_last_kernel_ms.argtypes = [C.c_void_p]
    lib.usearch_b200_bytes_per_vector.restype = C.c_size_t
    lib.usearch_b200_bytes_per_vector.argtypes = [C.c_void_p]
    lib.usearch_b200_max_level.restype = C.c_size_t
    lib.usearch_b200_max_level.argtypes = [C.c_void_p]
    lib.usearch_reserve.argtypes = [C.c_void_p, C.c_size_t, err]
    for name in ("usearch_b200_add_many", "usearch_b200_add_many_device"):
        getattr(lib, name).restype = None
        getattr(lib, name).argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int, err]
    lib.usearch_contains.restype = C.c_bool
    lib.usearch_contains.argtypes = [C.c_void_p, C.c_uint64, err]
    lib.usearch_count.restype = C.c_size_t
    lib.usearch_count.argtypes = [C.c_void_p, C.c_uint64, err]
    lib.usearch_get.restype = C.c_size_t
    lib.usearch_get.argtypes = [C.c_void_p, C.c_uint64, C.c_size_t, C.c_void_p, C.c_int, err]
    lib.usearch_remove.restype = C.c_size_t
    lib.usearch_remove.argtypes = [C.c_void_p, C.c_uint64, err]
    lib.usearch_b200_remove_many.restype = C.c_size_t
    lib.usearch_b200_remove_many.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_bool, C.POINTER(C.c_size_t), err]
    lib.usearch_b200_count_many.restype = C.c_size_t
    lib.usearch_b200_count_many.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, err]
    lib.usearch_b200_change_reuse_removed.argtypes = [C.c_void_p, C.c_bool, err]
    lib.usearch_b200_reuse_removed.restype = C.c_bool
    lib.usearch_b200_reuse_removed.argtypes = [C.c_void_p]
    lib.usearch_b200_join.restype = C.c_size_t
    lib.usearch_b200_join.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_bool, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p,
                                      err]
    lib.usearch_b200_last_join_ms.argtypes = [C.c_void_p, C.c_void_p]
    lib.usearch_b200_pairwise_distances.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, err]
    lib.usearch_rename.restype = C.c_size_t
    lib.usearch_rename.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, err]
    lib.usearch_b200_shards_unique_id.argtypes = [C.c_void_p, err]
    lib.usearch_b200_shards_join.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, err]
    lib.usearch_b200_sharded_search_many.restype = C.c_size_t
    lib.usearch_b200_sharded_search_many.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int, C.c_size_t,
                                                     C.c_void_p, C.c_void_p, C.c_void_p, err]
    lib.usearch_b200_sharded_search_many_device.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t,
                                                            C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                            C.c_void_p, err]
    lib.usearch_b200_shards_payload_bytes.restype = C.c_size_t
    lib.usearch_b200_shards_payload_bytes.argtypes = [C.c_size_t, C.c_size_t]
    lib.usearch_b200_merge_topk.argtypes = [C.c_void_p, C.c_int, C.c_size_t, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, err]
    lib.usearch_b200_indexes_init.restype = C.c_void_p
    lib.usearch_b200_indexes_init.argtypes = [err]
    lib.usearch_b200_indexes_free.argtypes = [C.c_void_p]
    lib.usearch_b200_indexes_merge.argtypes = [C.c_void_p, C.c_void_p, err]
    lib.usearch_b200_indexes_size.restype = C.c_size_t
    lib.usearch_b200_indexes_size.argtypes = [C.c_void_p, err]
    lib.usearch_b200_indexes_search_many.restype = C.c_size_t
    lib.usearch_b200_indexes_search_many.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int, C.c_size_t, C.c_bool,
                                                     C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, err]
    lib.usearch_b200_indexes_last_ms.argtypes = [C.c_void_p, C.c_void_p]
    lib.usearch_b200_merge_into.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p,
                                            C.c_void_p, C.c_void_p, err]
    lib.usearch_b200_get_many.restype = C.c_size_t
    lib.usearch_b200_get_many.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p,
                                          err]
    lib.usearch_b200_export_keys.restype = C.c_size_t
    lib.usearch_b200_export_keys.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p, err]
    lib.usearch_b200_export_keys_at.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, err]
    lib.usearch_b200_copy.restype = C.c_void_p
    lib.usearch_b200_copy.argtypes = [C.c_void_p, err]
    lib.usearch_b200_levels_stats.restype = C.c_size_t
    lib.usearch_b200_levels_stats.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, err]
    lib.usearch_b200_multi.restype = C.c_bool
    lib.usearch_b200_multi.argtypes = [C.c_void_p]
    lib.usearch_distance.restype = C.c_float
    lib.usearch_distance.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_size_t, C.c_int, err]
    _lib = lib
    return lib


def _raise(err: C.c_char_p) -> None:
    if err.value:
        raise RuntimeError(err.value.decode())


# the C entries of the key-set searches, by (excluded, exact); the device form of each is the same name + "_device"
_KEY_SET_ENTRIES = {(False, False): "usearch_b200_grouped_filtered_search_many",
                    (False, True): "usearch_b200_grouped_filtered_exact_search_many",
                    (True, False): "usearch_b200_grouped_excluded_search_many",
                    (True, True): "usearch_b200_grouped_excluded_exact_search_many"}


_KIND_TO_NP = {"f32": np.float32, "f64": np.float64, "f16": np.float16, "bf16": np.uint16, "i8": np.int8, "b1": np.uint8}
_NODE_HEAD_BYTES = 10  # a node's key and level in the reference's tape (index.hpp:2116-2195)


def _normalize_kind(dtype) -> str:
    """A kind name, or a NumPy dtype as the reference's `_normalize_dtype` maps it (uint8 -> b1); bf16 by name only."""
    if isinstance(dtype, str) and dtype in SCALAR_KIND:
        return dtype
    try:
        kind = _NP_TO_SCALAR.get(np.dtype(dtype))
    except TypeError:
        kind = None
    if kind is None:
        raise ValueError(f"Unsupported dtype {dtype!r}")
    return kind


def _as_keys(keys) -> np.ndarray:
    """Any iterable or integer array of keys, any stride -> a dense uint64 array."""
    if not isinstance(keys, np.ndarray):
        keys = np.fromiter((int(k) for k in keys), dtype=np.uint64)
    if keys.ndim != 1:
        raise ValueError("Keys must be placed in a single-dimensional array")
    return np.ascontiguousarray(keys, dtype=np.uint64)


@dataclass(frozen=True)
class IndexStats:
    """`index_gt::stats_t` (index.hpp:3133-3138)."""
    nodes: int
    edges: int
    max_edges: int
    allocated_bytes: int


class IndexedKeys:
    """The live keys of an index in slot order (index.py:453-488): `len`, `[i]` (negative too), slices, integer arrays of
    offsets, `__array__` and iteration. Each call reads the keys once on the host."""

    def __init__(self, index: "Index") -> None:
        self.index = index

    def __len__(self) -> int:
        return len(self.index)

    def _slice(self, offset: int, limit: int) -> np.ndarray:
        out = np.zeros(max(limit, 0), dtype=np.uint64)
        err = C.c_char_p()
        n = self.index._lib.usearch_b200_export_keys(self.index._h, offset, out.size, out.ctypes.data_as(C.c_void_p), C.byref(err))
        _raise(err)
        return out[:n]

    def _at(self, offsets) -> np.ndarray:
        offsets = np.asarray(offsets, dtype=np.int64).ravel()
        size = len(self)
        offsets = np.where(offsets < 0, offsets + size, offsets)
        if offsets.size and (offsets.min() < 0 or offsets.max() >= size):
            raise IndexError("Index out of range")
        offsets = np.ascontiguousarray(offsets, dtype=np.uintp)
        out = np.zeros(offsets.size, dtype=np.uint64)
        err = C.c_char_p()
        self.index._lib.usearch_b200_export_keys_at(self.index._h, offsets.ctypes.data_as(C.c_void_p), offsets.size,
                                                    out.ctypes.data_as(C.c_void_p), C.byref(err))
        _raise(err)
        return out

    def __getitem__(self, at):
        if isinstance(at, slice):
            start, stop, step = at.indices(len(self))
            if step == 1:
                return self._slice(start, stop - start)
            return self._at(np.arange(start, stop, step))
        if np.isscalar(at) or isinstance(at, int):
            return int(self._at([int(at)])[0])
        return self._at(at)

    def __array__(self, dtype=None, copy=None):
        keys = self._slice(0, len(self))
        return keys if dtype is None else keys.astype(dtype)

    def __iter__(self):
        return iter(self._slice(0, len(self)).tolist())


@dataclass
class Matches:
    """Single-query result (index.py:300-330): ``keys`` and ``distances`` trimmed to the found count."""
    keys: np.ndarray
    distances: np.ndarray
    visited_members: int = 0
    computed_distances: int = 0

    def __len__(self) -> int:
        return len(self.keys)

    def to_list(self):
        return [(int(k), float(d)) for k, d in zip(self.keys, self.distances)]


@dataclass
class BatchMatches:
    """Batch result (index.py:333-396): dense ``[nq, count]`` matrices + per-row ``counts``."""
    keys: np.ndarray
    distances: np.ndarray
    counts: np.ndarray
    visited_members: int = 0
    computed_distances: int = 0

    def __len__(self) -> int:
        return len(self.counts)

    def __getitem__(self, i: int) -> Matches:
        n = int(self.counts[i])
        return Matches(self.keys[i, :n], self.distances[i, :n])

    def to_list(self):
        return [self[i].to_list() for i in range(len(self))]

    def mean_recall(self, expected: np.ndarray, count: Optional[int] = None) -> float:
        return float(self.count_matches(expected, count)) / len(expected)

    def count_matches(self, expected: np.ndarray, count: Optional[int] = None) -> int:
        """index.py:379-393: is ``expected[i]`` anywhere among the first ``count`` results of row i."""
        hits = 0
        for i in range(len(expected)):
            n = int(self.counts[i]) if count is None else min(count, int(self.counts[i]))
            hits += int(expected[i] in self.keys[i, :n])
        return hits


def _matches(keys: np.ndarray, distances: np.ndarray, counts: np.ndarray, single: bool, visited: int, computed: int):
    """The rows of a search: :class:`Matches` trimmed to its count for one query, else :class:`BatchMatches`."""
    if single:
        n = int(counts[0])
        return Matches(keys[0, :n], distances[0, :n], visited, computed)
    return BatchMatches(keys, distances, counts, visited, computed)


class Index:
    """Drop-in for ``usearch.index.Index`` whose graph lives in B200 HBM.

    ``add`` links batches of new members into the graph on the GPU; ``load``/``view``/``restore`` take a ``.usearch``
    file built anywhere; ``search`` runs the whole batch as one persistent-kernel launch.
    """

    def __init__(self, *, ndim: int = 0, metric: str = "cos", dtype: str = "f32", connectivity: int = 16,
                 expansion_add: int = 128, expansion_search: int = 64, multi: bool = False,
                 path: Optional[str] = None, view: bool = False):
        self._lib = load_library()
        err = C.c_char_p()
        if ndim:
            opts = _InitOptions(METRIC_KIND[metric], None, SCALAR_KIND[dtype], ndim, connectivity, expansion_add,
                                expansion_search, multi)
            self._h = C.c_void_p(self._lib.usearch_init(C.byref(opts), C.byref(err)))
        else:
            self._h = C.c_void_p(self._lib.usearch_init(None, C.byref(err)))
        _raise(err)
        self._dtype = dtype
        self._expansion_search = expansion_search
        self._keepalive = None
        self.last_pruned_edges = 0  # links erased by the last remove(..., compact=True)
        self.last_join_stats = {}  # intersection_size, engagements, visited_members, computed_distances of the last join
        self.last_join_ms = {}  # its wall clock per phase: search, pair_distances, replay
        if path is not None:
            (self.view if view else self.load)(path)

    def __del__(self):
        if getattr(self, "_h", None):
            self._lib.usearch_free(self._h, None)
            self._h = None

    # ---- loading (index.py:1100-1200 `load`/`view`/`restore`) ------------------------------------
    @staticmethod
    def restore(path_or_buffer, view: bool = False) -> "Index":
        index = Index()
        (index.view if view else index.load)(path_or_buffer)
        return index

    def load(self, path_or_buffer: Union[str, os.PathLike, bytes, bytearray, np.ndarray]) -> "Index":
        err = C.c_char_p()
        if isinstance(path_or_buffer, (str, os.PathLike)):
            self._lib.usearch_load(self._h, os.fspath(path_or_buffer).encode(), C.byref(err))
            meta = self.metadata(path_or_buffer)
        else:
            buf = np.frombuffer(path_or_buffer, dtype=np.uint8) if not isinstance(path_or_buffer, np.ndarray) \
                else np.ascontiguousarray(path_or_buffer, dtype=np.uint8)
            self._lib.usearch_load_buffer(self._h, buf.ctypes.data_as(C.c_void_p), buf.size, C.byref(err))
            meta = self.metadata(buf) if not err.value else None
        _raise(err)
        self._dtype = meta["dtype"]
        self._lib.usearch_change_expansion_search(self._h, self._expansion_search, None)
        return self

    view = load  # the device copy never aliases the file: `view` == `load`

    @staticmethod
    def metadata(path_or_buffer) -> dict:
        lib = load_library()
        opts = _InitOptions()
        err = C.c_char_p()
        if isinstance(path_or_buffer, (str, os.PathLike)):
            lib.usearch_metadata(os.fspath(path_or_buffer).encode(), C.byref(opts), C.byref(err))
        else:
            buf = np.ascontiguousarray(path_or_buffer, dtype=np.uint8)
            lib.usearch_metadata_buffer(buf.ctypes.data_as(C.c_void_p), buf.size, C.byref(opts), C.byref(err))
        _raise(err)
        inv_m = {v: k for k, v in METRIC_KIND.items()}
        inv_s = {v: k for k, v in SCALAR_KIND.items()}
        return {"metric": inv_m.get(opts.metric_kind), "dtype": inv_s.get(opts.quantization),
                "ndim": opts.dimensions, "multi": bool(opts.multi)}

    def save(self, path: Optional[str] = None) -> Optional[np.ndarray]:
        err = C.c_char_p()
        if path is not None:
            self._lib.usearch_save(self._h, os.fspath(path).encode(), C.byref(err))
            _raise(err)
            return None
        n = self._lib.usearch_serialized_length(self._h, None)
        buf = np.empty(n, dtype=np.uint8)
        self._lib.usearch_save_buffer(self._h, buf.ctypes.data_as(C.c_void_p), n, C.byref(err))
        _raise(err)
        return buf

    # ---- properties (index.py:1377-1470) -----------------------------------------------------------
    size = property(lambda s: s._lib.usearch_size(s._h, None))
    ndim = property(lambda s: s._lib.usearch_dimensions(s._h, None))
    connectivity = property(lambda s: s._lib.usearch_connectivity(s._h, None))
    capacity = property(lambda s: s._lib.usearch_capacity(s._h, None))
    memory_usage = property(lambda s: s._lib.usearch_memory_usage(s._h, None))
    serialized_length = property(lambda s: s._lib.usearch_serialized_length(s._h, None))
    hardware_acceleration = property(lambda s: s._lib.usearch_hardware_acceleration(s._h, None).decode())
    dtype = property(lambda s: s._dtype)
    max_level = property(lambda s: s._lib.usearch_b200_max_level(s._h))
    kernel_launches = property(lambda s: s._lib.usearch_b200_kernel_launches(s._h))
    last_kernel_ms = property(lambda s: s._lib.usearch_b200_last_kernel_ms(s._h))
    bytes_per_vector = property(lambda s: s._lib.usearch_b200_bytes_per_vector(s._h))

    def __len__(self) -> int:
        return self.size

    @property
    def expansion_search(self) -> int:
        return self._lib.usearch_expansion_search(self._h, None)

    @expansion_search.setter
    def expansion_search(self, v: int) -> None:
        self._expansion_search = v
        self._lib.usearch_change_expansion_search(self._h, v, None)

    @property
    def expansion_add(self) -> int:
        return self._lib.usearch_expansion_add(self._h, None)

    @expansion_add.setter
    def expansion_add(self, v: int) -> None:
        self._lib.usearch_change_expansion_add(self._h, v, None)

    # ---- mutation (index.py:560-700 `add`, :800-900 `remove`/`rename`/`get`/`contains`/`count`) -------------
    def reserve(self, capacity: int) -> None:
        err = C.c_char_p()
        self._lib.usearch_reserve(self._h, int(capacity), C.byref(err))
        _raise(err)

    def add(self, keys, vectors: np.ndarray, *, copy: bool = True, threads: int = 0, log=False, progress=None):
        """`Index.add` (index.py:560-640): one key + vector, or a batch. The batch is linked into the graph on the
        GPU (builder.cu); `keys=None` numbers the rows from the current size, as the reference does. Returns the keys."""
        vectors = np.asarray(vectors)
        if vectors.ndim == 1:
            vectors = vectors[None, :]
        if not vectors.flags.c_contiguous and vectors.strides[1] != vectors.itemsize:
            vectors = np.ascontiguousarray(vectors)
        n = vectors.shape[0]
        if keys is None:
            start = len(self)
            keys = np.arange(start, start + n, dtype=np.uint64)
        keys = np.ascontiguousarray(np.atleast_1d(np.asarray(keys)), dtype=np.uint64)
        if keys.shape[0] != n:
            raise ValueError("The number of keys must match the number of vectors")
        kind = self._kind_of(vectors)
        err = C.c_char_p()
        self._lib.usearch_b200_add_many(self._h, keys.ctypes.data_as(C.c_void_p), vectors.ctypes.data_as(C.c_void_p), n,
                                        vectors.strides[0], SCALAR_KIND[kind], C.byref(err))
        _raise(err)
        return keys

    def add_device(self, keys_ptr: int, vectors_ptr: int, n: int, stride: int, kind: Optional[str] = None) -> None:
        """Batch add from DEVICE memory (raw pointers): no host round trip for the vectors."""
        err = C.c_char_p()
        self._lib.usearch_b200_add_many_device(self._h, keys_ptr, vectors_ptr, n, stride,
                                               SCALAR_KIND[kind or self._dtype], C.byref(err))
        _raise(err)

    def _count_many(self, keys) -> np.ndarray:
        keys = np.ascontiguousarray(np.fromiter(keys, dtype=np.uint64) if not isinstance(keys, np.ndarray) else keys,
                                    dtype=np.uint64)
        counts = np.zeros(keys.shape[0], dtype=np.uintp)
        self._lib.usearch_b200_count_many(self._h, keys.ctypes.data_as(C.c_void_p), keys.shape[0],
                                          counts.ctypes.data_as(C.c_void_p), None)
        return counts

    def contains(self, keys) -> Union[bool, np.ndarray]:
        """One key -> bool; an iterable of keys -> a bool array."""
        if np.isscalar(keys) or isinstance(keys, int):
            return bool(self._lib.usearch_contains(self._h, int(keys), None))
        return self._count_many(keys) > 0

    __contains__ = contains

    def count(self, keys) -> Union[int, np.ndarray]:
        """One key -> the entries stored under it; an iterable of keys -> an array of counts."""
        if np.isscalar(keys) or isinstance(keys, int):
            return int(self._lib.usearch_count(self._h, int(keys), None))
        return self._count_many(keys).astype(np.uint64)

    def get(self, keys, dtype=None, count: int = 1):
        """`Index.get` (index.py:765-809). One key: the vector stored under it (`count` > 1: up to that many rows), or
        None. An iterable or array of keys: on a plain index an ``[n, ndim]`` array, a missing key's row zero; on a multi
        index a tuple holding, per key, the matrix of all its vectors in insertion order, or None. `dtype` is one of the
        kind names, or a NumPy dtype as the reference maps it (uint8 means b1); bf16 comes back as uint16 words."""
        kind = _normalize_kind(dtype) if dtype is not None else self._dtype
        np_t = _KIND_TO_NP[kind]
        cols = (self.ndim + 7) // 8 if kind == "b1" else self.ndim
        if np.isscalar(keys) or isinstance(keys, int) or (isinstance(keys, np.ndarray) and keys.ndim == 0):
            out = np.zeros((count, cols), dtype=np_t)
            err = C.c_char_p()
            found = self._lib.usearch_get(self._h, int(keys), count, out.ctypes.data_as(C.c_void_p), SCALAR_KIND[kind],
                                          C.byref(err))
            _raise(err)
            if not found:
                return None
            return out[0] if count == 1 else out[:found]
        keys = _as_keys(keys)
        n = keys.shape[0]
        multi = self.multi
        if multi:
            rows = int(self._count_many(keys).sum())
            per_key = np.iinfo(np.uint64).max
        else:
            rows, per_key = n, 1
        out = np.zeros((rows, cols), dtype=np_t)
        counts = np.zeros(n, dtype=np.uintp)
        err = C.c_char_p()
        got = self._lib.usearch_b200_get_many(self._h, keys.ctypes.data_as(C.c_void_p), n, C.c_size_t(per_key),
                                              out.ctypes.data_as(C.c_void_p), out.strides[0] if rows else 0, SCALAR_KIND[kind],
                                              counts.ctypes.data_as(C.c_void_p), C.byref(err))
        _raise(err)
        if multi:
            ends = np.cumsum(counts.astype(np.int64))
            return tuple(out[e - int(c):e] if c else None for c, e in zip(counts, ends))
        if got == n:
            return out
        full = np.zeros((n, cols), dtype=np_t)
        full[counts.astype(bool)] = out[:got]
        return full

    def __getitem__(self, keys):
        return self.get(keys)

    def __delitem__(self, keys) -> None:
        self.remove(keys)

    @property
    def keys(self) -> "IndexedKeys":
        """Every live key, in slot order (the reference lists them in its hash table's order)."""
        return IndexedKeys(self)

    @property
    def vectors(self):
        """`get(keys)` for every live key, in the order of `keys`."""
        return self.get(np.asarray(self.keys))

    @property
    def multi(self) -> bool:
        return bool(self._lib.usearch_b200_multi(self._h))

    @property
    def nlevels(self) -> int:
        return self.max_level + 1

    def copy(self) -> "Index":
        """`Index.copy` (index.py:1152-1168): an independent index on the same GPU with the same contents, configuration,
        removed-slot queue and knobs. It stays valid when this one is deleted."""
        err = C.c_char_p()
        handle = self._lib.usearch_b200_copy(self._h, C.byref(err))
        _raise(err)
        result = Index.__new__(Index)
        result.__dict__.update(self.__dict__)
        result._h = C.c_void_p(handle)
        result._keepalive = None
        result.last_join_stats, result.last_join_ms = {}, {}
        return result

    def reset(self) -> None:
        """Release the index's device memory and keep its configuration: a later `add` starts a new graph."""
        self._lib.usearch_clear(self._h, None)

    def _levels_stats(self):
        err = C.c_char_p()
        total = np.zeros(4, dtype=np.uintp)
        levels = self._lib.usearch_b200_levels_stats(self._h, None, 0, total.ctypes.data_as(C.c_void_p), C.byref(err))
        _raise(err)
        per = np.zeros((max(levels, 1), 4), dtype=np.uintp)
        levels = self._lib.usearch_b200_levels_stats(self._h, per.ctypes.data_as(C.c_void_p), levels, None, C.byref(err))
        _raise(err)
        return [IndexStats(*(int(v) for v in row)) for row in per[:levels]], IndexStats(*(int(v) for v in total))

    @property
    def stats(self) -> "IndexStats":
        """`index_gt::stats()` over every node: nodes, edges, max_edges and allocated_bytes (the reference's node layout,
        not HBM use: see `memory_usage`)."""
        return self._levels_stats()[1]

    @property
    def levels_stats(self) -> list:
        """`index_gt::stats(stats_per_level, max_level)`: one entry per level, the node head counted on level 0 only."""
        return self._levels_stats()[0]

    def level_stats(self, level: int) -> "IndexStats":
        """`index_gt::stats(level)`: the nodes on `level` and above, the node head counted on every level."""
        per = self._levels_stats()[0]
        if level >= len(per):
            return IndexStats(0, 0, 0, 0)
        s = per[level]
        return s if level == 0 else IndexStats(s.nodes, s.edges, s.max_edges, s.allocated_bytes + _NODE_HEAD_BYTES * s.nodes)

    def remove(self, keys, *, compact: bool = False, threads: int = 0) -> int:
        """`Index.remove` (python/lib.cpp:1192-1227): one key or an iterable of keys; returns the number of entries
        removed. Their slots wait for reuse (see `reuse_removed`). With `compact`, every link that leads to a removed
        entry is erased on the GPU; `last_pruned_edges` then holds how many. `threads` is accepted for compatibility."""
        del threads
        if np.isscalar(keys) or isinstance(keys, int):
            keys = np.array([int(keys)], dtype=np.uint64)
        else:
            keys = np.ascontiguousarray(np.fromiter(keys, dtype=np.uint64) if not isinstance(keys, np.ndarray) else keys,
                                        dtype=np.uint64)
        err = C.c_char_p()
        pruned = C.c_size_t(0)
        n = self._lib.usearch_b200_remove_many(self._h, keys.ctypes.data_as(C.c_void_p), keys.shape[0], bool(compact),
                                               C.byref(pruned), C.byref(err))
        _raise(err)
        self.last_pruned_edges = int(pruned.value)
        return int(n)

    @property
    def reuse_removed(self) -> bool:
        """Whether `add` puts new entries into the slots of removed ones (oldest first) before appending. Off by default."""
        return bool(self._lib.usearch_b200_reuse_removed(self._h))

    @reuse_removed.setter
    def reuse_removed(self, on: bool) -> None:
        self._lib.usearch_b200_change_reuse_removed(self._h, bool(on), None)

    def rename(self, key_from: int, key_to: int) -> int:
        err = C.c_char_p()
        n = self._lib.usearch_rename(self._h, int(key_from), int(key_to), C.byref(err))
        _raise(err)
        return int(n)

    def clear(self) -> None:
        self._lib.usearch_clear(self._h, None)

    # ---- join and pairwise distances (index.py:1170-1200, :1263-1283) -------------------------------------------
    def join(self, other: "Index", max_proposals: int = 0, exact: bool = False, progress=None) -> Dict[int, int]:
        """`Index.join`: a one-to-one "semantic join" of `self` with `other` by stable marriages. Returns a mapping from
        keys of `self` to keys of `other`. The smaller index proposes, each proposal a search of the other one (`exact`:
        brute force); the searches run as batched GPU launches and the proposals are then replayed as the reference's
        single-threaded run makes them, so the result is deterministic.

        `max_proposals=0` means log(n) + 1 for the proposing side's size n. The reference's Python `join` adds its thread
        count instead of 1, so pass `max_proposals` explicitly to reproduce a multi-threaded reference run's budget.
        `progress` is accepted for compatibility and ignored. The four counters of the run go to `last_join_stats`, the
        wall-clock milliseconds of its three phases (proposal searches, pair distances, host replay) to `last_join_ms`."""
        del progress
        n = min(self.capacity, other.capacity)  # >= the slots of either side, removed entries included
        a_keys = np.zeros(max(n, 1), dtype=np.uint64)
        b_keys = np.zeros(max(n, 1), dtype=np.uint64)
        stats = np.zeros(4, dtype=np.uintp)
        err = C.c_char_p()
        found = self._lib.usearch_b200_join(self._h, other._h, int(max_proposals), bool(exact), a_keys.ctypes.data_as(C.c_void_p),
                                            b_keys.ctypes.data_as(C.c_void_p), a_keys.shape[0], stats.ctypes.data_as(C.c_void_p),
                                            C.byref(err))
        _raise(err)
        self.last_join_stats = dict(zip(("intersection_size", "engagements", "visited_members", "computed_distances"),
                                        (int(x) for x in stats)))
        ms = np.zeros(3, dtype=np.float32)
        self._lib.usearch_b200_last_join_ms(self._h, ms.ctypes.data_as(C.c_void_p))
        self.last_join_ms = dict(zip(("search", "pair_distances", "replay"), (float(x) for x in ms)))
        # in export order: on a repeated key (a multi index) the last pair wins, as in the reference
        return dict(zip(a_keys[:found].tolist(), b_keys[:found].tolist()))

    def pairwise_distance(self, left, right) -> Union[np.ndarray, float]:
        """`Index.pairwise_distance`: the distance between the vectors stored under two keys, or between the keys of
        two equally long arrays element by element; where a key is missing, the largest finite float. With one vector per
        key this is the reference's `distance_between(left, right).min`. Where keys hold several vectors (multi index) it
        is the minimum over every pair, a documented difference: the reference pairs only the first vector under `left`
        with each vector under `right`."""
        single = np.isscalar(left) or isinstance(left, int)
        if single != (np.isscalar(right) or isinstance(right, int)):
            raise ValueError("Pass two keys or two arrays of keys")
        left = np.ascontiguousarray(np.atleast_1d(np.asarray(left)), dtype=np.uint64)
        right = np.ascontiguousarray(np.atleast_1d(np.asarray(right)), dtype=np.uint64)
        if left.shape != right.shape:
            raise ValueError("The two key arrays must have the same length")
        out = np.zeros(left.shape[0], dtype=np.float32)
        err = C.c_char_p()
        self._lib.usearch_b200_pairwise_distances(self._h, left.ctypes.data_as(C.c_void_p), right.ctypes.data_as(C.c_void_p),
                                                  left.shape[0], out.ctypes.data_as(C.c_void_p), C.byref(err))
        _raise(err)
        return float(out[0]) if single else out

    # ---- search (index.py:700-748) ---------------------------------------------------------------
    def _query_rows(self, vectors, *, columns: bool = False):
        """(rows: `vectors` as a matrix of contiguous rows, single: whether it was one vector, its scalar kind); with
        `columns`, the row length is held to the index's dimensions."""
        vectors = np.asarray(vectors)
        single = vectors.ndim == 1
        if single:
            vectors = vectors[None, :]
        if vectors.ndim != 2:
            raise ValueError("Expects a matrix or a vector")
        if not vectors.flags.c_contiguous and vectors.strides[1] != vectors.itemsize:
            vectors = np.ascontiguousarray(vectors)  # rows must be contiguous (python/lib.cpp:426-428)
        kind = self._kind_of(vectors)
        if columns:
            expect_cols = (self.ndim * _BITS[kind] + 7) // 8 // vectors.itemsize if kind != "b1" else (self.ndim + 7) // 8
            if vectors.shape[1] != expect_cols:
                raise ValueError("The number of columns must match the dimensionality of the index")
        return vectors, single, kind

    def _kind_of(self, vectors: np.ndarray) -> str:
        if vectors.dtype == np.uint16:
            return "bf16"
        kind = _NP_TO_SCALAR.get(vectors.dtype)
        if kind is None:
            raise TypeError(f"Unsupported query dtype {vectors.dtype}")
        if kind == "b1" and self._dtype == "i8":
            return "i8"
        return kind

    def filtered_search(self, vectors: np.ndarray, count: int, allowed_keys, *, exact: bool = False) -> Union[Matches, BatchMatches]:
        """`filtered_search` (index_dense.hpp:774-779) for the predicate "key in allowed_keys". `exact=True` scans exactly
        the live entries whose key is allowed (search_exact_ with the predicate), on the GPU."""
        if exact and np.ndim(allowed_keys) != 1:  # a scalar is a key, not a set; a nested list is several sets
            raise ValueError("allowed_keys must be a flat sequence of keys")
        allowed = np.ascontiguousarray(allowed_keys, dtype=np.uint64)
        if exact:
            return self._key_set_search(vectors, count, np.array([0, allowed.size], dtype=np.uint64), allowed, None,
                                        excluded=False, exact=True)
        vectors, single, kind = self._query_rows(vectors, columns=True)
        nq = vectors.shape[0]
        keys = np.zeros((nq, count), dtype=np.uint64)
        distances = np.zeros((nq, count), dtype=np.float32)
        counts, computed, visited = (np.zeros(nq, dtype=np.uint64) for _ in range(3))
        err = C.c_char_p()
        self._lib.usearch_b200_filtered_search_many(
            self._h, vectors.ctypes.data_as(C.c_void_p), nq, vectors.strides[0], SCALAR_KIND[kind], count,
            allowed.ctypes.data_as(C.c_void_p), allowed.size, keys.ctypes.data_as(C.c_void_p),
            distances.ctypes.data_as(C.c_void_p), counts.ctypes.data_as(C.c_void_p),
            computed.ctypes.data_as(C.c_void_p), visited.ctypes.data_as(C.c_void_p), C.byref(err))
        _raise(err)
        self.last_computed, self.last_visited = computed, visited
        return _matches(keys, distances, counts, single, int(visited.sum()), int(computed.sum()))

    def grouped_filtered_search(self, vectors: np.ndarray, count: int, key_sets, groups=None, *,
                                exact: bool = False) -> Union[Matches, BatchMatches]:
        """`filtered_search` with a key set per query, as one launch: row i equals
        ``filtered_search(vectors[i], count, key_sets[groups[i]], exact=exact)``, counters included (`last_computed` /
        `last_visited`). `key_sets` is a sequence of key iterables or arrays; ``groups=None`` gives query i the set i.
        `exact=True` scans exactly the live entries of each query's set."""
        vectors, offsets, flat, groups = self._pack_key_sets(vectors, key_sets, groups)
        return self._key_set_search(vectors, count, offsets, flat, groups, excluded=False, exact=exact)

    def excluded_search(self, vectors: np.ndarray, count: int, excluded_keys, *, exact: bool = False) -> Union[Matches, BatchMatches]:
        """`filtered_search` (index_dense.hpp:774-779) for the predicate "key not in excluded_keys": every live entry but
        those stored under the given keys. `exact=True` scans exactly those entries (search_exact_ with the predicate)."""
        if np.ndim(excluded_keys) != 1:  # a scalar is a key, not a set; a nested list is several sets
            raise ValueError("excluded_keys must be a flat sequence of keys")
        excluded = np.ascontiguousarray(excluded_keys, dtype=np.uint64)
        return self._key_set_search(vectors, count, np.array([0, excluded.size], dtype=np.uint64), excluded, None,
                                    excluded=True, exact=exact)

    def grouped_excluded_search(self, vectors: np.ndarray, count: int, key_sets, groups=None, *,
                                exact: bool = False) -> Union[Matches, BatchMatches]:
        """`excluded_search` with a key set per query, as one call: row i equals
        ``excluded_search(vectors[i], count, key_sets[groups[i]], exact=exact)``, counters included (`last_computed` /
        `last_visited`). `key_sets` and `groups` as in `grouped_filtered_search`."""
        vectors, offsets, flat, groups = self._pack_key_sets(vectors, key_sets, groups)
        return self._key_set_search(vectors, count, offsets, flat, groups, excluded=True, exact=exact)

    @staticmethod
    def _pack_key_sets(vectors, key_sets, groups):
        """The CSR form of a batch's key sets: (vectors, offsets u64 [G + 1], flat keys u64, groups u32 [nq]), checked
        before any library call. ``groups=None`` gives query i the set i."""
        vectors = np.asarray(vectors)
        if vectors.ndim not in (1, 2):
            raise ValueError("Expects a matrix or a vector")
        nq = vectors.shape[0] if vectors.ndim == 2 else 1
        sets = []
        for keys in key_sets:
            if np.isscalar(keys):
                raise ValueError("key_sets must be a sequence of key sets, not of keys")
            keys = keys if isinstance(keys, np.ndarray) else np.asarray(list(keys))
            sets.append(np.ascontiguousarray(keys.reshape(-1), dtype=np.uint64))
        if groups is None:
            if len(sets) != nq:
                raise ValueError("Without groups, key_sets needs one set per query")
            groups = np.arange(nq, dtype=np.uint32)
        else:
            groups = np.asarray(groups)
            if groups.shape != (nq,):
                raise ValueError("groups needs one set index per query")
            if nq and (groups.min() < 0 or groups.max() >= len(sets)):
                raise ValueError("A query's key set index is out of range")
            groups = np.ascontiguousarray(groups, dtype=np.uint32)
        offsets = np.zeros(len(sets) + 1, dtype=np.uint64)
        offsets[1:] = np.cumsum([len(keys) for keys in sets]) if sets else []
        flat = np.concatenate(sets) if sets else np.zeros(0, dtype=np.uint64)
        return vectors, offsets, flat, groups

    def _key_set_search(self, vectors: np.ndarray, count: int, offsets: np.ndarray, flat: np.ndarray, groups, *, excluded: bool,
                        exact: bool):
        """The grouped host entry of the mode over CSR sets; ``groups=None`` with one set means set 0 for all (every mode
        but the allowed graph form). The exact forms visit no graph members: `last_visited` is zeros."""
        vectors, single, kind = self._query_rows(vectors)
        nq = vectors.shape[0]
        keys = np.zeros((nq, count), dtype=np.uint64)
        distances = np.zeros((nq, count), dtype=np.float32)
        counts, computed, visited = (np.zeros(nq, dtype=np.uint64) for _ in range(3))
        counters = (computed,) if exact else (computed, visited)
        err = C.c_char_p()
        getattr(self._lib, _KEY_SET_ENTRIES[excluded, exact])(
            self._h, vectors.ctypes.data_as(C.c_void_p), nq, vectors.strides[0], SCALAR_KIND[kind], count,
            None if groups is None else groups.ctypes.data_as(C.c_void_p), offsets.ctypes.data_as(C.c_void_p), offsets.size - 1,
            flat.ctypes.data_as(C.c_void_p), keys.ctypes.data_as(C.c_void_p), distances.ctypes.data_as(C.c_void_p),
            counts.ctypes.data_as(C.c_void_p), *(c.ctypes.data_as(C.c_void_p) for c in counters), C.byref(err))
        _raise(err)
        self.last_computed, self.last_visited = computed, visited
        return _matches(keys, distances, counts, single, int(visited.sum()), int(computed.sum()))

    def cluster(self, vectors: np.ndarray, level: int = 1, *, stats: bool = False):
        """`index_dense_gt::cluster(vector, level)` (index_dense.hpp:788-793; index.hpp:3092-3125) for every row: the
        closest member on graph level `level` (levels above the top return the entry point; 0 behaves like 1).
        Returns `(keys [nq] u64, distances [nq] f32)`; with `stats=True` the counters land in `last_computed` /
        `last_visited`."""
        vectors = np.asarray(vectors)
        if vectors.ndim == 1:
            vectors = vectors[None, :]
        if not vectors.flags.c_contiguous and vectors.strides[1] != vectors.itemsize:
            vectors = np.ascontiguousarray(vectors)
        kind = self._kind_of(vectors)
        nq = vectors.shape[0]
        keys = np.zeros(nq, dtype=np.uint64)
        distances = np.zeros(nq, dtype=np.float32)
        computed = np.zeros(nq, dtype=np.uint64)
        visited = np.zeros(nq, dtype=np.uint64)
        err = C.c_char_p()
        self._lib.usearch_b200_cluster_many(
            self._h, vectors.ctypes.data_as(C.c_void_p), nq, vectors.strides[0], SCALAR_KIND[kind], int(level),
            keys.ctypes.data_as(C.c_void_p), distances.ctypes.data_as(C.c_void_p),
            computed.ctypes.data_as(C.c_void_p) if stats else None, visited.ctypes.data_as(C.c_void_p) if stats else None,
            C.byref(err))
        _raise(err)
        if stats:
            self.last_computed, self.last_visited = computed, visited
        return keys, distances

    def search(self, vectors: np.ndarray, count: int = 10, *, stats: bool = False, threads: int = 0, exact: bool = False,
               log=False, progress=None) -> Union[Matches, BatchMatches]:
        """1-D input → :class:`Matches`; 2-D input → :class:`BatchMatches` (index.py:191-231).

        `threads`, `log` and `progress` are accepted for signature compatibility with index.py:700-748 and
        ignored (one kernel launch serves the whole batch); `exact=True` brute-forces every member on the GPU."""
        vectors, single, kind = self._query_rows(vectors, columns=True)
        nq = vectors.shape[0]
        keys = np.zeros((nq, count), dtype=np.uint64)
        distances = np.zeros((nq, count), dtype=np.float32)
        counts = np.zeros(nq, dtype=np.uint64)
        err = C.c_char_p()
        vm = cd = 0
        if exact:
            self._lib.usearch_b200_exact_search_many(
                self._h, vectors.ctypes.data_as(C.c_void_p), nq, vectors.strides[0], SCALAR_KIND[kind], count,
                keys.ctypes.data_as(C.c_void_p), distances.ctypes.data_as(C.c_void_p),
                counts.ctypes.data_as(C.c_void_p), C.byref(err))
            _raise(err)
        elif stats:
            computed = np.zeros(nq, dtype=np.uint64)
            visited = np.zeros(nq, dtype=np.uint64)
            self._lib.usearch_b200_search_many_stats(
                self._h, vectors.ctypes.data_as(C.c_void_p), nq, vectors.strides[0], SCALAR_KIND[kind], count,
                keys.ctypes.data_as(C.c_void_p), distances.ctypes.data_as(C.c_void_p),
                counts.ctypes.data_as(C.c_void_p), computed.ctypes.data_as(C.c_void_p),
                visited.ctypes.data_as(C.c_void_p), C.byref(err))
            _raise(err)
            self.last_computed, self.last_visited = computed, visited
            vm, cd = int(visited.sum()), int(computed.sum())
        else:
            self._lib.usearch_search_many(
                self._h, vectors.ctypes.data_as(C.c_void_p), nq, vectors.strides[0], SCALAR_KIND[kind], count,
                keys.ctypes.data_as(C.c_void_p), keys.strides[0], distances.ctypes.data_as(C.c_void_p),
                distances.strides[0], counts.ctypes.data_as(C.c_void_p), C.byref(err))
            _raise(err)
        return _matches(keys, distances, counts, single, vm, cd)

    def tune(self, **knobs: int) -> None:
        """Launch tuning knobs of this handle (stage_sets, warps_per_sm, prefilter, heap_head, get_chunk_rows,
        group_bitmap_mb); results never change."""
        for name, value in knobs.items():
            if self._lib.usearch_b200_tune(self._h, name.encode(), int(value)) != 0:
                raise ValueError(f"unknown knob {name}")

    def launch_plan(self, count: int = 10) -> dict:
        """The launch plan a search of `count` neighbours gets under the current knobs (see include/usearch_b200.h).
        Raises the planner's error when no plan fits, as `search` would."""
        out = np.zeros(16, dtype=np.uint64)
        err = C.c_char_p()
        self._lib.usearch_b200_launch_plan(self._h, int(count), out.ctypes.data_as(C.c_void_p), C.byref(err))
        _raise(err)
        plan = dict(zip(LAUNCH_PLAN_FIELDS, (int(v) for v in out)))
        plan["visits"] = _VISITS[plan["visits"]]
        plan["prefilter"] = bool(plan["prefilter"])
        return plan

    def profile_phases(self, enable: bool = True) -> dict:
        """Read (then reset) the kernel's per-phase cycle counters; see include/usearch_b200.h."""
        out = np.zeros(21, dtype=np.uint64)
        self._lib.usearch_b200_profile_phases_n(self._h, int(enable), out.ctypes.data_as(C.c_void_p), out.size)
        names = ["setup_descent", "heap_pop", "row_visited", "vector_wait", "distance_math", "accept", "output"]
        q = max(int(out[7]), 1)
        return {"queries": int(out[7]), **{n: float(out[i]) / q for i, n in enumerate(names)},
                "pushes": float(out[8]) / q, "avg_max_heap": float(out[9]) / q, "max_heap": int(out[10]),
                "prefiltered": float(out[11]) / q, "survivors": float(out[12]) / q, "code_wait": float(out[13]) / q,
                "prefilter_dot": float(out[14]) / q, "prefilter_bound": float(out[15]) / q,
                # what distance_math holds besides the prefilter: the survivors' FFMA pass and `finalize`, and whole
                # lists measured without it (hops before `top` is full)
                "survivor_math": float(out[4] - out[14] - out[15]) / q,
                # the part of prefilter_dot after the tensor cores: the conversion to `dot` and its stores
                "prefilter_convert": float(out[16]) / q,
                "code_passes_per_prefiltered_hop": float(out[17]) / max(int(out[18]), 1),
                "prefiltered_hops": float(out[18]) / q,
                # distance_math split: hops that start with `top` full, and the rest (whole lists: the layer-0 hops before
                # `top` fills). distance_math also subtracts the descent's vector waits, which belong to setup_descent.
                "distance_math_full": float(out[19]) / q,
                "distance_math_rest": (float(out[4]) + float(out[20]) - float(out[19])) / q,
                "descent_vector_wait": float(out[20]) / q}

    # ---- sharded search: this index is one shard of a group of processes (shards.cu) ------------------------
    def join_shards(self, rank: int, world: int, unique_id: bytes) -> None:
        """Collective. `unique_id` = the 128 bytes rank 0 got from :func:`shards_unique_id`, handed to every rank."""
        err = C.c_char_p()
        buf = (C.c_char * 128).from_buffer_copy(unique_id)
        self._lib.usearch_b200_shards_join(self._h, rank, world, buf, C.byref(err))
        _raise(err)

    def sharded_search(self, vectors: np.ndarray, count: int = 10) -> BatchMatches:
        """Collective: every rank passes the same queries and receives the merged top-`count` of all shards."""
        vectors = np.ascontiguousarray(vectors)
        if vectors.ndim == 1:
            vectors = vectors[None, :]
        kind = self._kind_of(vectors)
        nq = vectors.shape[0]
        keys = np.zeros((nq, count), dtype=np.uint64)
        distances = np.zeros((nq, count), dtype=np.float32)
        counts = np.zeros(nq, dtype=np.uint64)
        err = C.c_char_p()
        self._lib.usearch_b200_sharded_search_many(self._h, vectors.ctypes.data_as(C.c_void_p), nq, vectors.strides[0],
                                                   SCALAR_KIND[kind], count, keys.ctypes.data_as(C.c_void_p),
                                                   distances.ctypes.data_as(C.c_void_p), counts.ctypes.data_as(C.c_void_p),
                                                   C.byref(err))
        _raise(err)
        return BatchMatches(keys, distances, counts)

    def sharded_search_device(self, queries_ptr: int, nq: int, stride: int, count: int, keys_ptr: int, distances_ptr: int,
                              counts_ptr: int, computed_ptr: int = 0, visited_ptr: int = 0, stream: int = 0) -> None:
        err = C.c_char_p()
        self._lib.usearch_b200_sharded_search_many_device(self._h, queries_ptr, nq, stride, count, keys_ptr, distances_ptr,
                                                          counts_ptr, computed_ptr or None, visited_ptr or None,
                                                          stream or None, C.byref(err))
        _raise(err)

    def search_enqueue(self, queries_ptr: int, nq: int, stride: int, count: int, keys_ptr: int, distances_ptr: int,
                       counts_ptr: int, computed_ptr: int = 0, visited_ptr: int = 0, stream: int = 0) -> None:
        """Like :meth:`search_device` but returns as soon as the kernel is enqueued; call :meth:`search_finish` once."""
        err = C.c_char_p()
        self._lib.usearch_b200_search_many_enqueue(self._h, queries_ptr, nq, stride, count, keys_ptr, distances_ptr,
                                                   counts_ptr, computed_ptr or None, visited_ptr or None,
                                                   stream or None, C.byref(err))
        _raise(err)

    def search_finish(self) -> None:
        err = C.c_char_p()
        self._lib.usearch_b200_search_many_finish(self._h, C.byref(err))
        _raise(err)

    def search_device(self, queries_ptr: int, nq: int, stride: int, count: int, keys_ptr: int, distances_ptr: int,
                      counts_ptr: int, computed_ptr: int = 0, visited_ptr: int = 0, stream: int = 0) -> None:
        """Device-resident batch: raw device pointers (e.g. ``tensor.data_ptr()``) and a CUDA stream handle."""
        err = C.c_char_p()
        self._lib.usearch_b200_search_many_device(self._h, queries_ptr, nq, stride, count, keys_ptr, distances_ptr,
                                                  counts_ptr, computed_ptr or None, visited_ptr or None,
                                                  stream or None, C.byref(err))
        _raise(err)

    def count_device(self, keys_ptr: int, n: int, counts_ptr: int, stream: int = 0) -> None:
        """`count` for `n` keys in DEVICE memory: counts (uint32 [n], device) = the entries stored under each key.
        `contains` is ``counts > 0``."""
        err = C.c_char_p()
        self._lib.usearch_b200_count_many_device(self._h, keys_ptr, n, counts_ptr, stream or None, C.byref(err))
        _raise(err)

    def get_device(self, keys_ptr: int, n: int, vectors_ptr: int, counts_ptr: int, count: int = 1, stride: int = 0,
                   dtype: Optional[str] = None, stream: int = 0) -> None:
        """`get` for `n` keys in DEVICE memory into DEVICE rows: key i owns rows ``i * count`` .. ``i * count + count - 1``
        of `vectors` (`stride` bytes apart, 0 = packed) in `dtype` (default: the index's kind); counts (uint32 [n]) get
        the rows written per key, and the rows past them are zero. A key's rows are its `count` oldest entries."""
        kind = _normalize_kind(dtype) if dtype is not None else self._dtype
        err = C.c_char_p()
        self._lib.usearch_b200_get_many_device(self._h, keys_ptr, n, C.c_size_t(count), vectors_ptr, stride, SCALAR_KIND[kind],
                                               counts_ptr, stream or None, C.byref(err))
        _raise(err)

    def filtered_search_device(self, queries_ptr: int, nq: int, stride: int, count: int, allowed_ptr: int, allowed_count: int,
                               keys_ptr: int, distances_ptr: int, counts_ptr: int, computed_ptr: int = 0, visited_ptr: int = 0,
                               stream: int = 0, *, exact: bool = False) -> None:
        """`search_device` restricted to `allowed_count` keys held in DEVICE memory (uint64): the result of
        `filtered_search` with the same keys (and the same `exact`). An exact search visits no graph members: it takes no
        `visited_ptr`."""
        if exact:
            if visited_ptr:  # refused before the offsets below are made on the device
                raise ValueError("exact search has no visited_members counter")
            import torch  # the one-set CSR offsets {0, allowed_count} live in device memory as well
            offsets = torch.tensor([0, allowed_count], dtype=torch.int64, device=torch.device("cuda", self._lib.usearch_b200_device(self._h)))
            self._key_set_search_device(queries_ptr, nq, stride, count, 0, offsets.data_ptr(), 1, allowed_ptr, keys_ptr, distances_ptr,
                                        counts_ptr, computed_ptr, visited_ptr, stream, excluded=False, exact=True)
            return
        err = C.c_char_p()
        self._lib.usearch_b200_filtered_search_many_device(self._h, queries_ptr, nq, stride, count, allowed_ptr or None,
                                                           allowed_count, keys_ptr, distances_ptr, counts_ptr,
                                                           computed_ptr or None, visited_ptr or None, stream or None,
                                                           C.byref(err))
        _raise(err)

    def grouped_filtered_search_device(self, queries_ptr: int, nq: int, stride: int, count: int, groups_ptr: int, offsets_ptr: int,
                                       sets_count: int, set_keys_ptr: int, keys_ptr: int, distances_ptr: int, counts_ptr: int,
                                       computed_ptr: int = 0, visited_ptr: int = 0, stream: int = 0, *, exact: bool = False) -> None:
        """`grouped_filtered_search` on DEVICE memory: queries in the index's kind, `groups` (uint32 [nq]), `offsets`
        (uint64 [sets_count + 1]) and `set_keys` (uint64), outputs laid out as in `search_device`. With `exact=True`,
        `groups_ptr` may be 0 when `sets_count` is 1, and there is no `visited_ptr`."""
        self._key_set_search_device(queries_ptr, nq, stride, count, groups_ptr, offsets_ptr, sets_count, set_keys_ptr, keys_ptr,
                                    distances_ptr, counts_ptr, computed_ptr, visited_ptr, stream, excluded=False, exact=exact)

    def grouped_excluded_search_device(self, queries_ptr: int, nq: int, stride: int, count: int, groups_ptr: int, offsets_ptr: int,
                                       sets_count: int, set_keys_ptr: int, keys_ptr: int, distances_ptr: int, counts_ptr: int,
                                       computed_ptr: int = 0, visited_ptr: int = 0, stream: int = 0, *, exact: bool = False) -> None:
        """`grouped_excluded_search` on DEVICE memory, laid out as in `grouped_filtered_search_device`. `groups_ptr` may be
        0 when `sets_count` is 1; with `exact=True` there is no `visited_ptr`."""
        self._key_set_search_device(queries_ptr, nq, stride, count, groups_ptr, offsets_ptr, sets_count, set_keys_ptr, keys_ptr,
                                    distances_ptr, counts_ptr, computed_ptr, visited_ptr, stream, excluded=True, exact=exact)

    def _key_set_search_device(self, queries_ptr: int, nq: int, stride: int, count: int, groups_ptr: int, offsets_ptr: int,
                               sets_count: int, set_keys_ptr: int, keys_ptr: int, distances_ptr: int, counts_ptr: int,
                               computed_ptr: int, visited_ptr: int, stream: int, *, excluded: bool, exact: bool) -> None:
        """The grouped device entry of the mode; the exact forms take no `visited_ptr`."""
        if exact and visited_ptr:
            raise ValueError("exact search has no visited_members counter")
        counters = (computed_ptr or None,) if exact else (computed_ptr or None, visited_ptr or None)
        err = C.c_char_p()
        getattr(self._lib, _KEY_SET_ENTRIES[excluded, exact] + "_device")(
            self._h, queries_ptr, nq, stride, count, groups_ptr or None, offsets_ptr or None, sets_count, set_keys_ptr or None, keys_ptr,
            distances_ptr, counts_ptr, *counters, stream or None, C.byref(err))
        _raise(err)


class Indexes:
    """Drop-in for ``usearch.index.Indexes`` (index.py:1473-1514): several indexes on one GPU searched as one.

    ``search`` searches every member for every query, in merge order, and folds each member's result into the query's
    row as the reference's ``search_result_t::merge_into`` does when ``Indexes.search`` runs on one thread: keys,
    distance bits and counts equal that run's. On data without NaN the order is (distance ascending, later insertion
    first), so a later member wins a tie. The members are borrowed: this object keeps the ``Index`` objects alive."""

    def __init__(self, indexes=(), paths=(), view: bool = False, threads: int = 0):
        del threads
        self._lib = load_library()
        err = C.c_char_p()
        self._h = C.c_void_p(self._lib.usearch_b200_indexes_init(C.byref(err)))
        _raise(err)
        self._members = []
        self._view = view
        for index in indexes:
            self.merge(index)
        for path in paths:
            self.merge_path(path)

    def __del__(self):
        if getattr(self, "_h", None):
            self._lib.usearch_b200_indexes_free(self._h)
            self._h = None

    def merge(self, index: Index) -> None:
        err = C.c_char_p()
        self._lib.usearch_b200_indexes_merge(self._h, index._h, C.byref(err))
        _raise(err)
        self._members.append(index)

    def merge_path(self, path) -> None:
        """Restore the file at `path` onto the GPU and add it as the last member."""
        self.merge(Index.restore(os.fspath(path), view=self._view))

    def __len__(self) -> int:
        return int(self._lib.usearch_b200_indexes_size(self._h, None))

    @property
    def last_ms(self) -> dict:
        """Milliseconds of the last search from CUDA events: member searches (with the queries' upload), merge kernel."""
        ms = np.zeros(2, dtype=np.float32)
        self._lib.usearch_b200_indexes_last_ms(self._h, ms.ctypes.data_as(C.c_void_p))
        return {"search": float(ms[0]), "merge": float(ms[1])}

    def search(self, vectors, count: int = 10, *, threads: int = 0, exact: bool = False,
               progress=None) -> Union[Matches, BatchMatches]:
        """1-D input -> :class:`Matches`; 2-D input -> :class:`BatchMatches`. `visited_members` / `computed_distances`
        are summed over members and queries; the per-query sums over members land in `last_computed` / `last_visited`.
        `threads` and `progress` are accepted and ignored, as in `Index.search`."""
        del threads, progress
        vectors = np.asarray(vectors)
        single = vectors.ndim == 1
        if single:
            vectors = vectors[None, :]
        if vectors.ndim != 2:
            raise ValueError("Expects a matrix or a vector")
        if not vectors.flags.c_contiguous and vectors.strides[1] != vectors.itemsize:
            vectors = np.ascontiguousarray(vectors)
        if self._members:
            first = self._members[0]
            kind = first._kind_of(vectors)
            expect_cols = (first.ndim * _BITS[kind] + 7) // 8 // vectors.itemsize if kind != "b1" else (first.ndim + 7) // 8
            if vectors.shape[1] != expect_cols:
                raise ValueError("The number of columns must match the dimensionality of the index")
        else:
            kind = "bf16" if vectors.dtype == np.uint16 else _NP_TO_SCALAR.get(vectors.dtype)
            if kind is None:
                raise TypeError(f"Unsupported query dtype {vectors.dtype}")
        nq = vectors.shape[0]
        keys = np.zeros((nq, count), dtype=np.uint64)
        distances = np.zeros((nq, count), dtype=np.float32)
        counts = np.zeros(nq, dtype=np.uint64)
        computed = np.zeros(nq, dtype=np.uint64)
        visited = np.zeros(nq, dtype=np.uint64)
        err = C.c_char_p()
        self._lib.usearch_b200_indexes_search_many(
            self._h, vectors.ctypes.data_as(C.c_void_p), nq, vectors.strides[0], SCALAR_KIND[kind], count, bool(exact),
            keys.ctypes.data_as(C.c_void_p), distances.ctypes.data_as(C.c_void_p), counts.ctypes.data_as(C.c_void_p),
            computed.ctypes.data_as(C.c_void_p), visited.ctypes.data_as(C.c_void_p), C.byref(err))
        _raise(err)
        self.last_computed, self.last_visited = computed, visited
        vm, cd = int(visited.sum()), int(computed.sum())
        if single:
            n = int(counts[0])
            return Matches(keys[0, :n], distances[0, :n], vm, cd)
        return BatchMatches(keys, distances, counts, vm, cd)


def merge_into(keys: np.ndarray, distances: np.ndarray, counts: np.ndarray) -> BatchMatches:
    """The merge kernel of :class:`Indexes` on host rows: `keys` [S, nq, count] u64, `distances` [S, nq, count] f32 and
    `counts` [S, nq], folded member by member as the reference's `merge_into` folds them on one thread."""
    lib = load_library()
    keys = np.ascontiguousarray(keys, dtype=np.uint64)
    distances = np.ascontiguousarray(distances, dtype=np.float32)
    counts = np.ascontiguousarray(counts, dtype=np.uint32)
    shards, nq, count = keys.shape
    if distances.shape != keys.shape or counts.shape != (shards, nq):
        raise ValueError("keys, distances and counts must be [S, nq, count], [S, nq, count] and [S, nq]")
    out_keys = np.zeros((nq, count), dtype=np.uint64)
    out_distances = np.zeros((nq, count), dtype=np.float32)
    out_counts = np.zeros(nq, dtype=np.uint32)
    err = C.c_char_p()
    lib.usearch_b200_merge_into(keys.ctypes.data_as(C.c_void_p), distances.ctypes.data_as(C.c_void_p),
                                counts.ctypes.data_as(C.c_void_p), shards, nq, count, out_keys.ctypes.data_as(C.c_void_p),
                                out_distances.ctypes.data_as(C.c_void_p), out_counts.ctypes.data_as(C.c_void_p), C.byref(err))
    _raise(err)
    return BatchMatches(out_keys, out_distances, out_counts.astype(np.uint64))


def _rows(matrix: np.ndarray) -> np.ndarray:
    """`matrix` as it can be passed by row stride: copied only when a row's own elements are not contiguous."""
    if matrix.strides[1] != matrix.itemsize or matrix.strides[0] < 0:
        return np.ascontiguousarray(matrix)
    return matrix


def exact_search(dataset: np.ndarray, queries: np.ndarray, count: int = 10, *, metric: str = "cos",
                 dtype: Optional[str] = None, threads: int = 0) -> BatchMatches:
    """Brute-force many-to-many search over raw matrices: `usearch.index.search(dataset, query, count, metric,
    exact=True)` (python/usearch/index.py) -> `usearch_exact_search` (c/lib.cpp:468-501). Keys are dataset rows.

    The dataset may be larger than GPU memory and may be a strided view: its rows are read by stride, copied by
    `threads` host threads (0 = up to 8) into pinned staging buffers, and scanned chunk by chunk on the GPU while the
    next chunk uploads."""
    dataset = np.asarray(dataset)
    queries = np.asarray(queries)
    if dataset.ndim != 2:
        raise ValueError("Dataset must be a matrix, with a vector in each row")
    if queries.ndim == 1:
        queries = queries[None, :]
    if queries.ndim != 2 or queries.shape[1] != dataset.shape[1]:
        raise ValueError("Number of dimensions differs")
    if count < 0 or threads < 0:
        raise ValueError("count and threads must not be negative")
    kind = dtype or ("bf16" if dataset.dtype == np.uint16 else _NP_TO_SCALAR[dataset.dtype])
    scalar, metric_kind = SCALAR_KIND[kind], METRIC_KIND[metric]
    dataset, queries = _rows(dataset), _rows(queries)
    lib = load_library()
    dims = dataset.shape[1] * 8 if kind == "b1" else dataset.shape[1]
    nq = queries.shape[0]
    keys = np.zeros((nq, count), dtype=np.uint64)
    distances = np.zeros((nq, count), dtype=np.float32)
    err = C.c_char_p()
    lib.usearch_exact_search(dataset.ctypes.data_as(C.c_void_p), dataset.shape[0], dataset.strides[0],
                             queries.ctypes.data_as(C.c_void_p), nq, queries.strides[0], scalar, dims,
                             metric_kind, count, threads, keys.ctypes.data_as(C.c_void_p), keys.strides[0],
                             distances.ctypes.data_as(C.c_void_p), distances.strides[0], C.byref(err))
    _raise(err)
    return BatchMatches(keys, distances, np.full(nq, count, dtype=np.uint64))


def exact_search_device(dataset_ptr: int, n: int, dataset_stride: int, queries_ptr: int, nq: int, queries_stride: int,
                        ndim: int, count: int, keys_ptr: int, distances_ptr: int, *, metric: str = "cos", dtype: str = "f32",
                        keys_stride: int = 0, distances_stride: int = 0, stream: int = 0) -> None:
    """`exact_search` over DEVICE arrays (raw pointers, e.g. ``tensor.data_ptr()``; strides in bytes, 0 = dense outputs),
    enqueued on `stream` (0 = the default stream) without waiting for it: keys (u64 [nq, count]) and distances
    (f32 [nq, count]) are ready in stream order. `ndim` counts scalars (bits for b1). Rows already dense, 16-byte
    aligned and whole 16-byte chunks long are scanned in place; others are repacked chunk by chunk."""
    if dtype not in SCALAR_KIND:
        raise ValueError(f"Unknown dtype {dtype!r}")
    if metric not in METRIC_KIND:
        raise ValueError(f"Unknown metric {metric!r}")
    sizes = dict(n=n, dataset_stride=dataset_stride, nq=nq, queries_stride=queries_stride, ndim=ndim, count=count,
                 keys_stride=keys_stride, distances_stride=distances_stride)
    for name, value in sizes.items():
        if int(value) < 0:
            raise ValueError(f"{name} must not be negative")
    lib = load_library()
    err = C.c_char_p()
    lib.usearch_b200_exact_search_device(dataset_ptr or None, n, dataset_stride, queries_ptr or None, nq, queries_stride,
                                         SCALAR_KIND[dtype], ndim, METRIC_KIND[metric], count, keys_ptr or None, keys_stride,
                                         distances_ptr or None, distances_stride, stream or None, C.byref(err))
    _raise(err)


def search(dataset: np.ndarray, query: np.ndarray, count: int = 10, metric: str = "cos", *, exact: bool = False,
           threads: int = 0, log=False, progress=None) -> Union[Matches, BatchMatches]:
    """`usearch.index.search` (python/usearch/index.py): search a raw matrix without keeping an index. With `exact`,
    brute force (`exact_search`); without it, a temporary GPU `Index` over the rows, keyed by row number, searched once.
    A 1-D query gives :class:`Matches`, a matrix :class:`BatchMatches`. `log` and `progress` are accepted for signature
    compatibility and ignored."""
    dataset = np.asarray(dataset)
    query = np.asarray(query)
    if dataset.ndim != 2:
        raise ValueError("Dataset must be a matrix, with a vector in each row")
    if query.ndim not in (1, 2) or query.shape[-1] != dataset.shape[1]:
        raise ValueError("Number of dimensions differs")
    kind = "bf16" if dataset.dtype == np.uint16 else _NP_TO_SCALAR.get(dataset.dtype)
    if kind is None:
        raise TypeError(f"Unsupported dataset dtype {dataset.dtype}")
    if metric not in METRIC_KIND:
        raise ValueError(f"Unknown metric {metric!r}")
    if query.dtype != dataset.dtype:
        query = query.astype(dataset.dtype)
    if not exact:
        index = Index(ndim=dataset.shape[1] * 8 if kind == "b1" else dataset.shape[1], metric=metric, dtype=kind)
        index.add(None, dataset, threads=threads, log=log, progress=progress)
        return index.search(query, count, threads=threads, log=log, progress=progress)
    found = exact_search(dataset, query, count, metric=metric, dtype=kind, threads=threads)
    return found[0] if query.ndim == 1 else found


def shards_unique_id() -> bytes:
    """The 128-byte group id (an ncclUniqueId) rank 0 creates; every rank passes it to `Index.join_shards`."""
    lib = load_library()
    buf = (C.c_char * 128)()
    err = C.c_char_p()
    lib.usearch_b200_shards_unique_id(buf, C.byref(err))
    _raise(err)
    return bytes(buf)


def merge_topk(shard_results, count: int) -> BatchMatches:
    """The merge kernel on its own: `shard_results` = per-shard (keys [nq,count] u64, distances [nq,count] f32, counts [nq]),
    as `Indexes` would merge them (python/lib.cpp:350-391) but ordered by (distance, shard, position)."""
    lib = load_library()
    world = len(shard_results)
    nq = shard_results[0][0].shape[0]
    size = lib.usearch_b200_shards_payload_bytes(nq, count)
    blob = np.zeros(world * size, dtype=np.uint8)
    for r, (k, d, c) in enumerate(shard_results):
        base = r * size
        blob[base:base + nq * count * 8] = np.ascontiguousarray(k, dtype=np.uint64).view(np.uint8).ravel()
        blob[base + nq * count * 8:base + nq * count * 12] = np.ascontiguousarray(d, dtype=np.float32).view(np.uint8).ravel()
        blob[base + nq * count * 12:base + nq * count * 12 + nq * 4] = np.ascontiguousarray(c).astype(np.uint32).view(np.uint8)
    keys = np.zeros((nq, count), dtype=np.uint64)
    distances = np.zeros((nq, count), dtype=np.float32)
    counts = np.zeros(nq, dtype=np.uint32)
    err = C.c_char_p()
    lib.usearch_b200_merge_topk(blob.ctypes.data_as(C.c_void_p), world, nq, count, keys.ctypes.data_as(C.c_void_p),
                                distances.ctypes.data_as(C.c_void_p), counts.ctypes.data_as(C.c_void_p), C.byref(err))
    _raise(err)
    return BatchMatches(keys, distances, counts.astype(np.uint64))
