"""The CPU libraries the tests load with ctypes, each built once per session:
    emu()       tests/emu's kernel emulation (the product kernels compiled for the CPU), built by its Makefile;
    twin(name)  oracle/oracle_b.c with the CPU twin tests/<name>_twin/, built into a temporary directory.
Every exported function's signature is declared here, once."""
import atexit
import ctypes
import functools
import glob
import os
import shutil
import subprocess
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

_i32p, _u8p, _u32p = ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_uint8), ctypes.POINTER(ctypes.c_uint32)
_u64p, _i64p = ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(ctypes.c_longlong)
_i64, _int = ctypes.c_int64, ctypes.c_int
_SCORE = [_i32p, _i32p, _i32p, _i64, _i64, _i32p, _i64, _i32p, _int, _u64p]     # topo, free, mem, n, base, pods, P, W, splits, keys
_HOLD = [_i32p, _i32p, _i32p, _i32p, _i64, _i64, _i32p, _i32p]                 # topo, free, mem, hold, n, base, pods, lvl

EMU_SIGNATURES = {
    "emu_score_sparse": (_int, _SCORE),
    "emu_score_dense": (None, _SCORE),
    "emu_score_variant": (None, [_int] + _SCORE),
    "emu_score_sparse_after_updates": (None, [_i32p, _i32p, _i64, _i32p, _i32p, _i64, _i32p, _i64, _i32p, _int, _u64p, _i32p]),
    # topo0, free0, mem, n, base, upd_idx, upd_mask, upd_topo, has_topo, m, W, W2, w2_at, pods, P, splits, keys, free_out
    "emu_score_sparse_sequence": (_int, [_i32p, _i32p, _i32p, _i64, _i64, _i32p, _i32p, _i32p, _i32p, _i64, _i32p, _i32p, _i64,
                                         _i32p, _i64, _int, _u64p, _i32p]),
    "emu_order": (_i64, [_i32p, _i64, _i32p, _i64, _i32p, _i64p]),
    "emu_tile_classes": (_i64, [_i32p, _i64, _int, _u8p, _u8p, _i64]),
    "emu_fit_nodes": (None, [_i32p, _i32p, _i64, _i32p, _i64, _i32p, _u32p]),
    "emu_validate_topo": (ctypes.c_longlong, [_i32p, _i64]),
    "emu_gather_and_min": (None, [_u64p, _i64, _i64, _u64p, _u32p, ctypes.c_uint32, _u32p, _u64p, _i32p]),
    "emu_sparse_work": (_i64, [_u8p, _i64, _i64, _i64, _i32p, _i64, _i64p, ctypes.POINTER(_int)]),
    "emu_reduce_shards": (None, [_u64p, _int, _i64, _u64p]),
    "emu_score_pair_list": (None, [_i32p, _i32p, _i32p, _i64, _i64p, _i32p, _i32p, _i64, _i32p, _u32p]),
    "emu_place_batch": (_int, [_i32p, _i32p, _i32p, _i64, _i64, _i32p, _i64, _i32p, _u64p]),
    "emu_place_batch_gang": (_int, [_i32p, _i32p, _i32p, _i64, _i64, _i32p, _i32p, _i64, _i32p, _u64p]),
    "emu_preempt_batch": (_int, _HOLD + [_i64, _i32p, _int, _u64p, _u32p]),
    "emu_preempt_plan": (_int, _HOLD + [_i64, _i32p, _u64p, _u32p]),
    "emu_preempt_plan_gang": (_int, _HOLD + [_i32p, _i64, _i32p, _u64p, _u32p]),
    "emu_chunk_int4": (_int, []),
    "emu_chunk_pos": (_int, []),
    "emu_chunk_tables": (_i64, [_i32p, _i64, _int, _i32p, _i32p]),
    "emu_score_chunks": (_int, [_i32p, _i32p, _i32p, _i64, _i64, _i32p, _i64, _i32p, _i64, _int, _u64p]),
}

TWIN_SIGNATURES = {
    "preempt_twin_batch": (None, _HOLD + [_i64, _i32p, _int, _u64p, _u32p]),
    "preempt_plan_twin": (None, _HOLD + [_i64, _i32p, _int, _u64p, _u32p]),
    "preempt_plan_gang_twin": (None, _HOLD + [_i32p, _i64, _i32p, _int, _u64p, _u32p]),
    "gang_twin_place_batch": (None, [_i32p, _i32p, _i32p, _i64, _i64, _i32p, _i32p, _i64, _i32p, _u64p]),
}


def _declare(lib, signatures):
    for name, (restype, argtypes) in signatures.items():
        fn = getattr(lib, name, None)
        if fn is not None:
            fn.restype, fn.argtypes = restype, argtypes
    return lib


@functools.cache
def emu():
    subprocess.check_call(["make", "-s", "-C", os.path.join(HERE, "emu")])
    return _declare(ctypes.CDLL(os.path.join(HERE, "emu", "_build", "libkgpu_emu.so")), EMU_SIGNATURES)


@functools.cache
def _tmpdir():
    d = tempfile.mkdtemp(prefix="kgpu_twins_")
    atexit.register(shutil.rmtree, d, True)
    return d


@functools.cache
def twin(name):
    """The twin of tests/<name>_twin/ (its one .c file) with the oracle; the preemption twin rides along, as the plan twins
    are checked against it."""
    srcs = [os.path.join(ROOT, "oracle", "oracle_b.c"), os.path.join(HERE, "preempt_twin", "preempt_twin.c")]
    srcs += [s for s in glob.glob(os.path.join(HERE, name + "_twin", "*.c")) if s not in srcs]
    so = os.path.join(_tmpdir(), "lib%s_twin.so" % name)
    subprocess.check_call(["gcc", "-O2", "-fPIC", "-Wall", "-Wextra", "-std=c11", "-pthread", "-shared", "-o", so] + srcs)
    return _declare(ctypes.CDLL(so), TWIN_SIGNATURES)
