#!/usr/bin/env python3
"""Times kgpu_preempt_plan on synth.gen_preempt (C2's node shapes, 100k almost full nodes, 10k pods at levels 0..4)
against what a caller can do without it, and checks every result against the CPU twin
(tests/preempt_plan_twin/plan_twin.c, built here with the oracle into a temporary directory).  Prints the device name
and power limit, then
  (a) kgpu_preempt_plan: kernel time (CUDA events, median and spread of `--reps` calls) and host time per call;
  (b) the fallback: a host loop of single-pod kgpu_preempt_batch calls, each followed by kgpu_set_free_masks and
      kgpu_set_holders for the pod's node (the handle is restored afterwards);
  (c) the snapshot kgpu_preempt_batch on the whole batch, for scale;
  (d) the twin on all host cores.
(a), (b) and (d) must agree bit for bit (exit code 1 otherwise).  `--out FILE` also writes the figures as JSON."""
import ctypes
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

from kubegpu_b200 import _lib, synth  # noqa: E402
from kubegpu_b200.scorer import Scorer  # noqa: E402
from oracle import oracle_b  # noqa: E402

NO_FIT = np.uint64(_lib.NO_FIT)


def device_facts():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "unknown (nvidia-smi failed)"


def run_twin(topo, free, hold, pods, lvl):
    W = np.ascontiguousarray(oracle_b.DEFAULT_WEIGHTS, dtype=np.int32)
    nthreads = os.cpu_count() or 1
    with tempfile.TemporaryDirectory() as tmp:
        so = os.path.join(tmp, "libplan_twin.so")
        subprocess.check_call(["gcc", "-O2", "-fPIC", "-std=c11", "-pthread", "-shared", "-o", so,
                               os.path.join(ROOT, "oracle", "oracle_b.c"), os.path.join(ROOT, "tests", "preempt_plan_twin", "plan_twin.c")])
        L = ctypes.CDLL(so)
        tk = np.empty(len(pods), np.uint64)
        tv = np.empty(len(pods), np.uint32)
        p = lambda a, t=ctypes.c_int32: np.ascontiguousarray(a).ctypes.data_as(ctypes.POINTER(t))  # noqa: E731
        t0 = time.perf_counter()
        L.preempt_plan_twin(p(topo), p(free), None, p(hold), ctypes.c_int64(len(free)), ctypes.c_int64(0), p(pods), p(lvl),
                            ctypes.c_int64(len(pods)), p(W), ctypes.c_int(nthreads), p(tk, ctypes.c_uint64), p(tv, ctypes.c_uint32))
        return tk, tv, time.perf_counter() - t0, nthreads


def host_loop(s, free, hold, pods, lvl):
    """The fallback: per pod a snapshot call on the current state, then the definition's update pushed to the handle."""
    F = free.copy()
    H = hold.copy()
    keys = np.empty(len(pods), np.uint64)
    vic = np.empty(len(pods), np.uint32)
    touched = set()
    t0 = time.perf_counter()
    for p in range(len(pods)):
        k, v = s.preempt_batch(pods[p:p + 1], lvl[p:p + 1])
        keys[p], vic[p] = k[0], v[0]
        if k[0] == NO_FIT or pods[p, 0] == 0:
            continue
        n, S = (int(k[0]) >> 8) & 0xFFFFFFFF, int(k[0]) & 0xFF
        R = sum(1 << g for g in range(8) if not (F[n] >> g) & 1 and H[n, g] >= 0 and (int(v[0]) >> (H[n, g] & 7)) & 1)
        F[n] = (int(F[n]) | R) & ~S & 0xFF
        H[n, [g for g in range(8) if ((S | R) >> g) & 1]] = -1
        s.set_free_masks(np.array([n]), F[n:n + 1])
        s.set_holders(np.array([n]), H[n:n + 1])
        touched.add(n)
    elapsed = time.perf_counter() - t0
    idx = np.array(sorted(touched), np.int64)
    if len(idx):
        s.set_free_masks(idx, free[idx])
        s.set_holders(idx, hold[idx])
    return keys, vic, elapsed


def main():
    out_path = sys.argv[sys.argv.index("--out") + 1] if "--out" in sys.argv else None
    reps = int(sys.argv[sys.argv.index("--reps") + 1]) if "--reps" in sys.argv else 10
    topo, free, hold, pods, lvl = synth.gen_preempt()
    res = {"device": device_facts(), "nodes": len(free), "pods": len(pods), "reps": reps}
    print("device: %s" % res["device"], flush=True)
    calls, kerns, snap_calls, snap_kerns = [], [], [], []
    with Scorer((0,)) as s:
        s.upload_nodes(topo, free)
        s.upload_holders(hold)
        for i in range(reps + 1):                     # rep 0 warms up
            t0 = time.perf_counter()
            keys, vic = s.preempt_plan(pods, lvl)
            t1 = time.perf_counter()
            if i:
                calls.append((t1 - t0) * 1e3)
                kerns.append(s.last_kernel_ms)
            t0 = time.perf_counter()
            s.preempt_batch(pods, lvl)
            t1 = time.perf_counter()
            if i:
                snap_calls.append((t1 - t0) * 1e3)
                snap_kerns.append(s.last_kernel_ms)
        loop_k, loop_v, loop_s = host_loop(s, free, hold, pods, lvl)
        restored = bool((s.get_free_masks() == free).all())
        again = s.preempt_plan(pods, lvl)
        restored = restored and bool((again[0] == keys).all() and (again[1] == vic).all())
    tk, tv, twin_s, nthreads = run_twin(topo, free, hold, pods, lvl)
    exact_loop = bool((loop_k == keys).all() and (loop_v == vic).all())
    exact_twin = bool((tk == keys).all() and (tv == vic).all())
    med = lambda v: float(np.median(v))  # noqa: E731
    res.update({"placed_by_eviction": int((vic != 0).sum()), "placed": int((keys != NO_FIT).sum()),
                "plan_kernels_ms": med(kerns), "spread_plan_kernels_ms": [min(kerns), max(kerns)], "plan_call_ms": med(calls),
                "host_loop_s": loop_s, "snapshot_kernels_ms": med(snap_kerns), "snapshot_call_ms": med(snap_calls),
                "twin_s": twin_s, "twin_threads": nthreads, "exact_vs_host_loop": exact_loop, "exact_vs_twin": exact_twin,
                "handle_restored": restored})
    print("gen_preempt: %d nodes, %d pods; the plan places %d, %d of them by eviction"
          % (res["nodes"], res["pods"], res["placed"], res["placed_by_eviction"]))
    print("(a) kgpu_preempt_plan: kernels %.3f ms (spread %.3f - %.3f), call %.3f ms"
          % (res["plan_kernels_ms"], min(kerns), max(kerns), res["plan_call_ms"]))
    print("(b) host loop of per-pod preempt_batch + set_free_masks + set_holders: %.3f s (%.1fx the plan's call); handle restored: %s"
          % (loop_s, loop_s * 1e3 / res["plan_call_ms"], restored))
    print("(c) snapshot kgpu_preempt_batch: kernels %.3f ms, call %.3f ms" % (res["snapshot_kernels_ms"], res["snapshot_call_ms"]))
    print("(d) CPU twin on %d threads: %.2f s" % (nthreads, twin_s))
    print("bit-exact: plan vs host loop %s, plan vs twin %s" % (exact_loop, exact_twin))
    if out_path:
        with open(out_path, "w") as f:
            json.dump(res, f, indent=1)
    if not (exact_loop and exact_twin and restored):
        sys.exit(1)


if __name__ == "__main__":
    main()
