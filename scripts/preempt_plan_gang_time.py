#!/usr/bin/env python3
"""Times kgpu_preempt_plan_gang on synth.gen_preempt_gangs (gen_preempt's almost full cluster at 20k nodes, 10k pods,
about a third of them in gangs of 2..8) and checks every result against the CPU twin
(tests/preempt_plan_gang_twin/plan_gang_twin.c, built here with the oracle into a temporary directory).  Prints the
device name and power limit, then
  (a) kgpu_preempt_plan_gang: kernel time (CUDA events, median and spread of `--reps` calls) and host time per call;
  (b) kgpu_preempt_plan on the same pods without gang ids;
  (c) the fallback without gang plans: kgpu_preempt_plan, drop the first gang with a miss, plan again, until no gang
      misses (the dropped gangs get NO_FIT);
  (d) the twin on all host cores;
and the cost of gangs when nothing is undone: (a) against (b) on gen_preempt_gangs at 100k nodes, where no gang fails.
(a), (c) and (d) must agree bit for bit (exit code 1 otherwise).  `--out FILE` also writes the figures as JSON."""
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


def run_twin(topo, free, hold, pods, lvl, gang):
    W = np.ascontiguousarray(oracle_b.DEFAULT_WEIGHTS, dtype=np.int32)
    nthreads = os.cpu_count() or 1
    with tempfile.TemporaryDirectory() as tmp:
        so = os.path.join(tmp, "libplan_gang_twin.so")
        subprocess.check_call(["gcc", "-O2", "-fPIC", "-std=c11", "-pthread", "-shared", "-o", so,
                               os.path.join(ROOT, "oracle", "oracle_b.c"),
                               os.path.join(ROOT, "tests", "preempt_plan_gang_twin", "plan_gang_twin.c")])
        L = ctypes.CDLL(so)
        tk = np.empty(len(pods), np.uint64)
        tv = np.empty(len(pods), np.uint32)
        p = lambda a, t=ctypes.c_int32: np.ascontiguousarray(a).ctypes.data_as(ctypes.POINTER(t))  # noqa: E731
        t0 = time.perf_counter()
        L.preempt_plan_gang_twin(p(topo), p(free), None, p(hold), ctypes.c_int64(len(free)), ctypes.c_int64(0), p(pods), p(lvl),
                                 p(gang), ctypes.c_int64(len(pods)), p(W), ctypes.c_int(nthreads), p(tk, ctypes.c_uint64),
                                 p(tv, ctypes.c_uint32))
        return tk, tv, time.perf_counter() - t0, nthreads


def replan(s, pods, lvl, gang):
    """The fallback: plan, delete the first gang with a miss, plan again, until no gang misses."""
    keep = np.ones(len(pods), bool)
    runs = 0
    t0 = time.perf_counter()
    while True:
        idx = np.flatnonzero(keep)
        k, v = s.preempt_plan(pods[idx], lvl[idx])
        runs += 1
        g = gang[idx]
        miss = np.flatnonzero((g != 0) & (k == NO_FIT))
        if len(miss) == 0:
            break
        keep[gang == g[miss[0]]] = False
    elapsed = time.perf_counter() - t0
    keys = np.full(len(pods), NO_FIT, np.uint64)
    vic = np.zeros(len(pods), np.uint32)
    keys[idx], vic[idx] = k, v
    return keys, vic, elapsed, runs


def timed(s, reps, call):
    calls, kerns = [], []
    for i in range(reps + 1):                         # rep 0 warms up
        t0 = time.perf_counter()
        out = call()
        t1 = time.perf_counter()
        if i:
            calls.append((t1 - t0) * 1e3)
            kerns.append(s.last_kernel_ms)
    return out, calls, kerns


def main():
    out_path = sys.argv[sys.argv.index("--out") + 1] if "--out" in sys.argv else None
    reps = int(sys.argv[sys.argv.index("--reps") + 1]) if "--reps" in sys.argv else 10
    med = lambda v: float(np.median(v))  # noqa: E731
    topo, free, hold, pods, lvl, gang = synth.gen_preempt_gangs()
    res = {"device": device_facts(), "nodes": len(free), "pods": len(pods), "gangs": int(gang.max()), "reps": reps}
    print("device: %s" % res["device"], flush=True)
    with Scorer((0,)) as s:
        s.upload_nodes(topo, free)
        s.upload_holders(hold)
        (keys, vic), g_calls, g_kerns = timed(s, reps, lambda: s.preempt_plan(pods, lvl, gang=gang))
        _, p_calls, p_kerns = timed(s, reps, lambda: s.preempt_plan(pods, lvl))
        rk, rv, replan_s, runs = replan(s, pods, lvl, gang)
    tk, tv, twin_s, nthreads = run_twin(topo, free, hold, pods, lvl, gang)
    failed = sum(1 for g in range(1, gang.max() + 1) if (keys[gang == g] == NO_FIT).all())
    exact_replan = bool((rk == keys).all() and (rv == vic).all())
    exact_twin = bool((tk == keys).all() and (tv == vic).all())
    res.update({"failed_gangs": failed, "placed": int((keys != NO_FIT).sum()), "placed_by_eviction": int((vic != 0).sum()),
                "gang_plan_kernels_ms": med(g_kerns), "spread_gang_plan_kernels_ms": [min(g_kerns), max(g_kerns)],
                "gang_plan_call_ms": med(g_calls), "plan_kernels_ms": med(p_kerns),
                "spread_plan_kernels_ms": [min(p_kerns), max(p_kerns)], "plan_call_ms": med(p_calls),
                "replan_s": replan_s, "replan_runs": runs, "twin_s": twin_s, "twin_threads": nthreads,
                "exact_vs_replan": exact_replan, "exact_vs_twin": exact_twin})
    # 100k nodes: no gang fails, so (a) - (b) is what the gang bookkeeping costs
    topo, free, hold, pods, lvl, gang = synth.gen_preempt_gangs(N=100_000)
    with Scorer((0,)) as s:
        s.upload_nodes(topo, free)
        s.upload_holders(hold)
        (k100, _), g100_calls, g100_kerns = timed(s, reps, lambda: s.preempt_plan(pods, lvl, gang=gang))
        (p100, _), p100_calls, p100_kerns = timed(s, reps, lambda: s.preempt_plan(pods, lvl))
    failed100 = sum(1 for g in range(1, gang.max() + 1) if (k100[gang == g] == NO_FIT).all())
    res.update({"n100k_failed_gangs": failed100, "n100k_same_keys": bool((k100 == p100).all()),
                "n100k_gang_plan_kernels_ms": med(g100_kerns), "n100k_spread_gang_plan_kernels_ms": [min(g100_kerns), max(g100_kerns)],
                "n100k_plan_kernels_ms": med(p100_kerns), "n100k_spread_plan_kernels_ms": [min(p100_kerns), max(p100_kerns)]})
    print("gen_preempt_gangs: %d nodes, %d pods, %d gangs; %d gangs fail; %d pods placed, %d by eviction"
          % (res["nodes"], res["pods"], res["gangs"], failed, res["placed"], res["placed_by_eviction"]))
    print("(a) kgpu_preempt_plan_gang: kernels %.3f ms (spread %.3f - %.3f), call %.3f ms"
          % (res["gang_plan_kernels_ms"], min(g_kerns), max(g_kerns), res["gang_plan_call_ms"]))
    print("(b) kgpu_preempt_plan without gang ids: kernels %.3f ms (spread %.3f - %.3f), call %.3f ms"
          % (res["plan_kernels_ms"], min(p_kerns), max(p_kerns), res["plan_call_ms"]))
    print("(c) re-plan fallback: %d plan runs, %.3f s (%.1fx the gang plan's call)"
          % (runs, replan_s, replan_s * 1e3 / res["gang_plan_call_ms"]))
    print("(d) CPU twin on %d threads: %.2f s" % (nthreads, twin_s))
    print("100k nodes (%d gangs fail, keys equal to (b): %s): (a) kernels %.3f ms (spread %.3f - %.3f), (b) kernels %.3f ms "
          "(spread %.3f - %.3f)" % (failed100, res["n100k_same_keys"], res["n100k_gang_plan_kernels_ms"], min(g100_kerns),
                                    max(g100_kerns), res["n100k_plan_kernels_ms"], min(p100_kerns), max(p100_kerns)))
    print("bit-exact: gang plan vs re-plan %s, gang plan vs twin %s" % (exact_replan, exact_twin))
    if out_path:
        with open(out_path, "w") as f:
            json.dump(res, f, indent=1)
    if not (exact_replan and exact_twin):
        sys.exit(1)


if __name__ == "__main__":
    main()
