"""ctypes binding of the C ABI declared in include/kgpu.h (stands in for the cgo
binding shown in INTEGRATION.md -- there is no Go toolchain in this image)."""
from __future__ import annotations

import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libkgpu.so")

# every symbol include/kgpu.h declares; tests/test_abi.py checks header <-> this list <-> the .so
SYMBOLS = [
    "kgpu_version", "kgpu_create", "kgpu_destroy", "kgpu_last_error", "kgpu_set_weights",
    "kgpu_get_weights", "kgpu_set_variant", "kgpu_upload_nodes", "kgpu_update_node",
    "kgpu_set_free_mask", "kgpu_set_free_masks", "kgpu_remove_node", "kgpu_build_fit_table", "kgpu_fit_lookup", "kgpu_last_upload_ms", "kgpu_upload_gpu_memory", "kgpu_update_gpu_memory", "kgpu_num_nodes", "kgpu_score_batch",
    "kgpu_score_batch_device", "kgpu_score_batch_device_ex", "kgpu_score_pairs", "kgpu_place_batch", "kgpu_place_batch_ex", "kgpu_place_batch_gang", "kgpu_upload_domains", "kgpu_place_batch_gang_domain", "kgpu_upload_domain_levels", "kgpu_place_batch_gang_levels", "kgpu_upload_holders", "kgpu_set_holders", "kgpu_preempt_batch", "kgpu_preempt_plan", "kgpu_preempt_plan_gang", "kgpu_preempt_plan_gang_domain", "kgpu_get_free_masks", "kgpu_reduce_shards_device", "kgpu_exchange_init", "kgpu_exchange_connect", "kgpu_score_batch_exchange", "kgpu_exchange_barrier", "kgpu_kernel_launches",
    "kgpu_last_kernel_ms",
]

OK, ERR_INVALID, ERR_CUDA, ERR_NOMEM, ERR_COMM, ERR_STATE = 0, -1, -2, -3, -4, -5
NO_FIT = 0xFFFFFFFFFFFFFFFF
IPC_HANDLE_BYTES = 64
VARIANT_AUTO, VARIANT_WARP_PER_PAIR, VARIANT_LANE_PER_NODE, VARIANT_MEMO_BY_K, VARIANT_TILE_MEMO = 0, 1, 2, 3, 4
VARIANT_SPARSE = 5
BATCH_NO_MIN_MEM = 1
PLACE_DRY_RUN = 1
GANG_DOMAIN_REQUIRED, GANG_DOMAIN_PREFERRED = 1, 2
MAX_DOMAIN_LEVELS = 4

_lib = None


def load() -> ctypes.CDLL:
    """Load libkgpu.so.  Raises (never falls back) if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            "libkgpu.so not found at %s -- build it with `make` (or __graft_entry__.build()); "
            "kubegpu_b200 has no CPU fallback" % LIB_PATH)
    L = ctypes.CDLL(LIB_PATH)
    vp, i32p, u64p = ctypes.c_void_p, ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_uint64)
    i64, ci = ctypes.c_int64, ctypes.c_int
    L.kgpu_version.restype = ctypes.c_char_p
    L.kgpu_version.argtypes = []
    L.kgpu_create.restype = ci
    L.kgpu_create.argtypes = [ctypes.POINTER(ci), ci, ctypes.POINTER(vp)]
    L.kgpu_destroy.restype = ci
    L.kgpu_destroy.argtypes = [vp]
    L.kgpu_last_error.restype = ctypes.c_char_p
    L.kgpu_last_error.argtypes = [vp]
    L.kgpu_set_weights.restype = ci
    L.kgpu_set_weights.argtypes = [vp, i32p]
    L.kgpu_get_weights.restype = ci
    L.kgpu_get_weights.argtypes = [vp, i32p]
    L.kgpu_set_variant.restype = ci
    L.kgpu_set_variant.argtypes = [vp, ci]
    L.kgpu_upload_nodes.restype = ci
    L.kgpu_upload_nodes.argtypes = [vp, i32p, i32p, i64, i64]
    L.kgpu_upload_gpu_memory.restype = ci
    L.kgpu_upload_gpu_memory.argtypes = [vp, i32p, i64]
    L.kgpu_update_gpu_memory.restype = ci
    L.kgpu_update_gpu_memory.argtypes = [vp, i64, i32p]
    L.kgpu_update_node.restype = ci
    L.kgpu_update_node.argtypes = [vp, i64, i32p, ctypes.c_int32]
    L.kgpu_set_free_mask.restype = ci
    L.kgpu_set_free_mask.argtypes = [vp, i64, ctypes.c_int32]
    L.kgpu_set_free_masks.restype = ci
    L.kgpu_set_free_masks.argtypes = [vp, ctypes.POINTER(i64), i32p, i64]
    L.kgpu_build_fit_table.restype = ci
    L.kgpu_build_fit_table.argtypes = [vp]
    L.kgpu_fit_lookup.restype = ci
    L.kgpu_fit_lookup.argtypes = [vp, i64, ctypes.c_int32, ctypes.POINTER(ctypes.c_uint32)]
    L.kgpu_last_upload_ms.restype = ctypes.c_double
    L.kgpu_last_upload_ms.argtypes = [vp]
    L.kgpu_remove_node.restype = ci
    L.kgpu_remove_node.argtypes = [vp, i64]
    L.kgpu_num_nodes.restype = i64
    L.kgpu_num_nodes.argtypes = [vp]
    L.kgpu_score_batch.restype = ci
    L.kgpu_score_batch.argtypes = [vp, vp, i64, vp]          # raw addresses: numpy or pinned torch memory
    L.kgpu_score_batch_device.restype = ci
    L.kgpu_score_batch_device.argtypes = [vp, vp, i64, vp, vp]
    L.kgpu_score_batch_device_ex.restype = ci
    L.kgpu_score_batch_device_ex.argtypes = [vp, vp, i64, vp, vp, ci]
    L.kgpu_score_pairs.restype = ci
    L.kgpu_score_pairs.argtypes = [vp, ctypes.POINTER(i64), i32p, i32p, i64, ctypes.POINTER(ctypes.c_uint32)]
    L.kgpu_place_batch.restype = ci
    L.kgpu_place_batch.argtypes = [vp, vp, i64, vp]
    L.kgpu_place_batch_ex.restype = ci
    L.kgpu_place_batch_ex.argtypes = [vp, vp, i64, vp, ci]
    L.kgpu_place_batch_gang.restype = ci
    L.kgpu_place_batch_gang.argtypes = [vp, vp, vp, i64, vp, ci]
    L.kgpu_upload_domains.restype = ci
    L.kgpu_upload_domains.argtypes = [vp, i32p, i64]
    L.kgpu_place_batch_gang_domain.restype = ci
    L.kgpu_place_batch_gang_domain.argtypes = [vp, vp, vp, vp, i64, vp, ci]
    L.kgpu_upload_domain_levels.restype = ci
    L.kgpu_upload_domain_levels.argtypes = [vp, i32p, ci, i64]
    L.kgpu_place_batch_gang_levels.restype = ci
    L.kgpu_place_batch_gang_levels.argtypes = [vp, vp, vp, vp, vp, i64, vp, ci]
    L.kgpu_upload_holders.restype = ci
    L.kgpu_upload_holders.argtypes = [vp, i32p, i64]
    L.kgpu_set_holders.restype = ci
    L.kgpu_set_holders.argtypes = [vp, ctypes.POINTER(i64), i32p, i64]
    L.kgpu_preempt_batch.restype = ci
    L.kgpu_preempt_batch.argtypes = [vp, vp, vp, i64, vp, vp]
    L.kgpu_preempt_plan.restype = ci
    L.kgpu_preempt_plan.argtypes = [vp, vp, vp, i64, vp, vp]
    L.kgpu_preempt_plan_gang.restype = ci
    L.kgpu_preempt_plan_gang.argtypes = [vp, vp, vp, vp, i64, vp, vp]
    L.kgpu_preempt_plan_gang_domain.restype = ci
    L.kgpu_preempt_plan_gang_domain.argtypes = [vp, vp, vp, vp, vp, i64, vp, vp]
    L.kgpu_get_free_masks.restype = ci
    L.kgpu_get_free_masks.argtypes = [vp, i32p, i64]
    L.kgpu_reduce_shards_device.restype = ci
    L.kgpu_reduce_shards_device.argtypes = [vp, vp, ci, i64, vp, vp]
    L.kgpu_exchange_init.restype = ci
    L.kgpu_exchange_init.argtypes = [vp, ci, ci, i64, vp]
    L.kgpu_exchange_connect.restype = ci
    L.kgpu_exchange_connect.argtypes = [vp, vp]
    L.kgpu_score_batch_exchange.restype = ci
    L.kgpu_score_batch_exchange.argtypes = [vp, vp, i64, ctypes.POINTER(vp), vp, ci]
    L.kgpu_exchange_barrier.restype = ci
    L.kgpu_exchange_barrier.argtypes = [vp, vp]
    L.kgpu_kernel_launches.restype = i64
    L.kgpu_kernel_launches.argtypes = [vp]
    L.kgpu_last_kernel_ms.restype = ctypes.c_double
    L.kgpu_last_kernel_ms.argtypes = [vp]
    _lib = L
    return L
