"""The CPU libraries of the gang-domain tests, each built once per session into cpu_libs' temporary directory:
    twin()  tests/gang_domain_twin/gang_domain_twin.c with the oracle (cpu_libs.twin);
    emu()   tests/gang_domain_emu/emu_gang_domain.cc: the kernel sources and launch plan under tests/emu/cuda_emu.h.
Their exported functions' signatures are declared here."""
import ctypes
import functools
import os
import subprocess

import cpu_libs

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

_i32p, _u64p = ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_uint64)
_i64 = ctypes.c_int64
# topo, free, mem, n, base, domain, pods, gang, gang_domain, P, W, keys
_PLACE = [_i32p, _i32p, _i32p, _i64, _i64, _i32p, _i32p, _i32p, _i32p, _i64, _i32p, _u64p]


@functools.cache
def twin():
    L = cpu_libs.twin("gang_domain")
    L.gang_domain_twin_place_batch.restype, L.gang_domain_twin_place_batch.argtypes = None, _PLACE
    return L


@functools.cache
def emu():
    src = os.path.join(HERE, "gang_domain_emu", "emu_gang_domain.cc")
    so = os.path.join(cpu_libs._tmpdir(), "libgang_domain_emu.so")
    subprocess.check_call(["g++", "-std=c++20", "-O1", "-fPIC", "-shared", "-pthread", "-I" + os.path.join(HERE, "emu", "stub"),
                           "-I" + os.path.join(HERE, "emu"), "-I" + os.path.join(ROOT, "kubegpu_b200", "csrc"), "-o", so, src])
    L = ctypes.CDLL(so)
    L.emu_place_batch_gang_domain.restype, L.emu_place_batch_gang_domain.argtypes = ctypes.c_int, _PLACE
    return L
