#!/usr/bin/env python3
"""Randomised CPU check of the kernel sources under the emulation harness (tests/emu) against the oracle:
    python scripts/emu_fuzz.py [--seconds 300] [--seed 1]
Random node counts, pod counts, free-mask densities, weights (byte-key and general layouts), memory
requirements, pod splits / work list, sequential placement with views.  Prints the failing case and exits 1."""
import argparse
import ctypes
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from kubegpu_b200 import synth  # noqa: E402
from oracle import oracle_b  # noqa: E402


def ptr(a, t=ctypes.c_int32):
    return a.ctypes.data_as(ctypes.POINTER(t))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=300)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--define", action="append", default=[], help="build knob for a private emulation build, e.g. KGPU_SP_UNROLL=2")
    a = ap.parse_args()
    emu_dir = os.path.join(ROOT, "tests", "emu")
    if a.define:
        lib = "/tmp/libkgpu_emu_%s.so" % "_".join(d.replace("=", "") for d in a.define)
        subprocess.check_call(["g++", "-std=c++20", "-O1", "-fPIC", "-shared", "-pthread"] + ["-D" + d for d in a.define] +
                              ["-I" + os.path.join(emu_dir, "stub"), "-I" + os.path.join(ROOT, "kubegpu_b200", "csrc"), "-o", lib,
                               os.path.join(emu_dir, "emu_kernels.cc")])
    else:
        subprocess.check_call(["make", "-s", "-C", emu_dir])
        lib = os.path.join(emu_dir, "_build", "libkgpu_emu.so")
    L = ctypes.CDLL(lib)
    L.emu_score_sparse.restype = None
    L.emu_score_dense.restype = None
    L.emu_place_batch.restype = ctypes.c_int
    rng = np.random.default_rng(a.seed)
    t0, n_cases = time.time(), 0
    while time.time() - t0 < a.seconds:
        n_cases += 1
        N = int(rng.choice([1, 2, 31, 33, 127, 129, int(rng.integers(1, 600))]))
        P = int(rng.choice([1, 2, 31, 513, int(rng.integers(1, 900))]))
        gen = rng.integers(0, 3)
        seed = int(rng.integers(1, 2**31))
        if gen == 0:
            topo, free, pods = synth.gen_c2(N=N, P=P, seed=seed)
            pods[:, 0] = rng.integers(-1, 10, size=P)
        elif gen == 1:
            topo, free, pods = synth.gen_c4(N=N, P=P, seed=seed)
        else:
            topo, free, pods = synth.gen_c3(N=N, P=P, seed=seed)
        dens = rng.choice(["rand", "full", "empty", "sparse", "dense"])
        if dens == "full":
            free[:] = 0xFF
        elif dens == "empty":
            free[:] = 0
        elif dens == "sparse":
            free &= rng.integers(0, 256, size=N).astype(np.int32)
        elif dens == "dense":
            free |= rng.integers(0, 256, size=N).astype(np.int32)
        wkind = rng.integers(0, 4)
        if wkind == 0:
            W = np.asarray(oracle_b.DEFAULT_WEIGHTS, dtype=np.int32).copy()
        elif wkind == 1:
            W = rng.integers(0, 2341, size=16).astype(np.int32)
        elif wkind == 2:
            W = rng.integers(0, 4096, size=16).astype(np.int32)
        else:
            W = np.full(16, int(rng.choice([0, 1, 2340, 2341, 4095])), dtype=np.int32)
        use_mem = bool(rng.integers(0, 2))
        mem = synth.gen_gpu_memory(N, seed=seed) if use_mem else None
        if use_mem:
            pods[:, 3] = rng.choice(np.array(synth.POD_MIN_MEM_CHOICES_MIB, dtype=np.int32), size=P)
        base = int(rng.choice([0, 5, 2**31 - 1000]))
        splits = int(rng.choice([1, 2, 3, 7, -1, -16, -1184]))
        want = oracle_b.score_batch(topo, free, pods, W, node_id_base=base, mem=mem)
        case = dict(N=N, P=P, gen=int(gen), seed=seed, dens=str(dens), wkind=int(wkind), use_mem=use_mem, base=base, splits=splits)
        for name, fn in (("sparse", L.emu_score_sparse), ("dense", L.emu_score_dense)):
            keys = np.empty(P, dtype=np.uint64)
            fn(ptr(topo), ptr(free), None if mem is None else ptr(mem), ctypes.c_int64(N), ctypes.c_int64(base), ptr(pods),
               ctypes.c_int64(P), ptr(W), splits if name == "sparse" else max(1, abs(splits) % 5), ptr(keys, ctypes.c_uint64))
            if not (keys == want).all():
                bad = np.nonzero(keys != want)[0]
                print("MISMATCH", name, case, "pods", bad[:8], [hex(int(x)) for x in keys[bad[:4]]], [hex(int(x)) for x in want[bad[:4]]])
                np.savez("/tmp/emu_fuzz_fail.npz", topo=topo, free=free, pods=pods, W=W, mem=mem if mem is not None else np.zeros(0))
                sys.exit(1)
        if n_cases % 3 == 0 and P <= 400:            # sequential placement (slower under emulation)
            f = free.copy()
            keys = np.empty(P, dtype=np.uint64)
            rc = L.emu_place_batch(ptr(topo), ptr(f), None if mem is None else ptr(mem), ctypes.c_int64(N), ctypes.c_int64(base),
                                   ptr(pods), ctypes.c_int64(P), ptr(W), ptr(keys, ctypes.c_uint64))
            wk, wf = oracle_b.place_batch(topo, free.copy(), pods, W, node_id_base=base, mem=mem, plain=True) if mem is None else \
                oracle_b.place_batch(topo, free.copy(), pods, W, node_id_base=base, mem=mem)
            if rc != 0 or not (keys == wk).all() or not (f == wf).all():
                print("MISMATCH place", case, rc)
                sys.exit(1)
        if n_cases % 20 == 0:
            print("%d cases, %.0f s" % (n_cases, time.time() - t0), flush=True)
    print("ok: %d random cases in %.0f s" % (n_cases, time.time() - t0))


if __name__ == "__main__":
    main()
