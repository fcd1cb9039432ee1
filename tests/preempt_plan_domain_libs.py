"""The CPU libraries of the preemption-plan domain tests, each built once per session into cpu_libs' temporary directory:
    twin()  tests/preempt_plan_domain_twin/plan_domain_twin.c with the oracle (cpu_libs.twin); it also exports
            preempt_twin_batch, preempt_plan_twin and preempt_plan_gang_twin;
    emu()   tests/preempt_plan_domain_emu/emu_plan_domain.cc: the kernel sources and launch plan under tests/emu/cuda_emu.h.
Their exported functions' signatures are declared here."""
import ctypes
import functools
import os
import subprocess

import cpu_libs

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

_i32p, _u32p, _u64p = ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_uint32), ctypes.POINTER(ctypes.c_uint64)
_i64, _int = ctypes.c_int64, ctypes.c_int
# topo, free (in/out), mem, hold (in/out), n, base, domain, pods, lvl, gang, gang_domain, P, W
_PLAN = [_i32p, _i32p, _i32p, _i32p, _i64, _i64, _i32p, _i32p, _i32p, _i32p, _i32p, _i64, _i32p]


@functools.cache
def twin():
    L = cpu_libs.twin("preempt_plan_domain")
    L.preempt_plan_domain_twin.restype = None
    L.preempt_plan_domain_twin.argtypes = _PLAN + [_int, _u64p, _u32p]          # + nthreads, keys, victims
    return L


@functools.cache
def emu():
    src = os.path.join(HERE, "preempt_plan_domain_emu", "emu_plan_domain.cc")
    so = os.path.join(cpu_libs._tmpdir(), "libpreempt_plan_domain_emu.so")
    subprocess.check_call(["g++", "-std=c++20", "-O1", "-fPIC", "-shared", "-pthread", "-I" + os.path.join(HERE, "emu", "stub"),
                           "-I" + os.path.join(HERE, "emu"), "-I" + os.path.join(ROOT, "kubegpu_b200", "csrc"), "-o", so, src])
    L = ctypes.CDLL(so)
    L.emu_preempt_plan_gang_domain.restype = ctypes.c_int
    L.emu_preempt_plan_gang_domain.argtypes = _PLAN + [_u64p, _u32p]
    return L
