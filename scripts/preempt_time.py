#!/usr/bin/env python3
"""Times kgpu_preempt_batch on synth.gen_preempt (C2's node shapes, 100k almost full nodes, 10k pods at levels 0..4)
and checks it against the CPU twin (tests/preempt_twin/preempt_twin.c, built here with the oracle into a temporary
directory).  Prints the device name and power limit, how many pods reach the preemption kernel, the call's kernel time
(CUDA events) split into the scoring kernels and the preemption kernels (torch.profiler), and the twin's time on all
host cores.  `--out FILE` also writes the figures as JSON."""
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


def load_twin(tmp):
    so = os.path.join(tmp, "libpreempt_twin.so")
    subprocess.check_call(["gcc", "-O2", "-fPIC", "-std=c11", "-pthread", "-shared", "-o", so,
                           os.path.join(ROOT, "oracle", "oracle_b.c"), os.path.join(ROOT, "tests", "preempt_twin", "preempt_twin.c")])
    return ctypes.CDLL(so)


def kernel_split(s, pods, lvl):
    """Device time (ms) of one kgpu_preempt_batch, summed per kernel group, from torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        s.preempt_batch(pods, lvl)
        torch.cuda.synchronize()
    split = {"preemption": 0.0, "scoring": 0.0}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = getattr(e, "cuda_time_total", 0.0)
        if not t or "memcpy" in e.key.lower() or "memset" in e.key.lower():
            continue
        group = "preemption" if ("preempt_" in e.key) else "scoring"
        split[group] += t / 1e3
    return split


def main():
    out_path = sys.argv[sys.argv.index("--out") + 1] if "--out" in sys.argv else None
    reps = 10
    topo, free, hold, pods, lvl = synth.gen_preempt()
    res = {"device": device_facts(), "nodes": len(free), "pods": len(pods)}
    calls, kerns, score_kerns = [], [], []
    with Scorer((0,)) as s:
        s.upload_nodes(topo, free)
        s.upload_holders(hold)
        plain = s.score_batch(pods)
        for i in range(reps + 1):                     # rep 0 warms up
            t0 = time.perf_counter()
            keys, vic = s.preempt_batch(pods, lvl)
            t1 = time.perf_counter()
            if i:
                calls.append((t1 - t0) * 1e3)
                kerns.append(s.last_kernel_ms)
            s.score_batch(pods)
            if i:
                score_kerns.append(s.last_kernel_ms)
        try:
            split = kernel_split(s, pods, lvl)
        except Exception as e:                       # the profiler is an extra; the events above are the figure
            split = {"error": repr(e)}
    reached = (plain == NO_FIT) & (pods[:, 0] >= 1) & (pods[:, 0] <= 8) & (lvl > 0)
    W = np.ascontiguousarray(oracle_b.DEFAULT_WEIGHTS, dtype=np.int32)
    nthreads = os.cpu_count() or 1
    with tempfile.TemporaryDirectory() as tmp:
        L = load_twin(tmp)
        tk = np.empty(len(pods), np.uint64)
        tv = np.empty(len(pods), np.uint32)
        p = lambda a, t=ctypes.c_int32: np.ascontiguousarray(a).ctypes.data_as(ctypes.POINTER(t))  # noqa: E731
        t0 = time.perf_counter()
        L.preempt_twin_batch(p(topo), p(free), None, p(hold), ctypes.c_int64(len(free)), ctypes.c_int64(0), p(pods), p(lvl),
                             ctypes.c_int64(len(pods)), p(W), ctypes.c_int(nthreads), p(tk, ctypes.c_uint64), p(tv, ctypes.c_uint32))
        twin_s = time.perf_counter() - t0
    exact = bool((tk == keys).all() and (tv == vic).all())
    med = lambda v: float(np.median(v))  # noqa: E731
    res.update({"no_fit_without_eviction": int((plain == NO_FIT).sum()), "reach_preemption_kernel": int(reached.sum()),
                "placed_by_eviction": int(((plain == NO_FIT) & (keys != NO_FIT)).sum()),
                "preempt_call_ms": med(calls), "preempt_kernels_ms": med(kerns),
                "spread_preempt_kernels_ms": [min(kerns), max(kerns)], "score_batch_kernels_ms": med(score_kerns),
                "profiler_split_ms": split, "twin_s": twin_s, "twin_threads": nthreads, "reps": reps, "exact": exact})
    print("device: %s" % res["device"])
    print("gen_preempt: %d nodes, %d pods; %d fit nowhere without eviction, %d reach the preemption kernel, %d placed by eviction"
          % (res["nodes"], res["pods"], res["no_fit_without_eviction"], res["reach_preemption_kernel"], res["placed_by_eviction"]))
    print("kgpu_preempt_batch: kernels %.3f ms (spread %.3f - %.3f), call %.3f ms; score_batch alone: kernels %.3f ms"
          % (res["preempt_kernels_ms"], min(kerns), max(kerns), res["preempt_call_ms"], res["score_batch_kernels_ms"]))
    print("profiler split (one call): %s" % json.dumps(split))
    print("CPU twin on %d threads: %.2f s; keys and victims equal: %s" % (nthreads, twin_s, exact))
    if out_path:
        with open(out_path, "w") as f:
            json.dump(res, f, indent=1)
    if not exact:
        sys.exit(1)


if __name__ == "__main__":
    main()
