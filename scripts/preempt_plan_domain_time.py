#!/usr/bin/env python3
"""Times kgpu_preempt_plan_gang_domain on synth.gen_preempt_gangs (20k nodes, 10k pods, 717 gangs of 2..8) with
synth.gen_domains at domain sizes 8, 32 and 128, and checks every result against the CPU twin
(tests/preempt_plan_domain_twin/plan_domain_twin.c, built here with the oracle into a temporary directory).  Prints the
device name and power limit, then per domain size
  (a) every gang REQUIRED, (b) every gang PREFERRED, (c) gang_domain = 0, which must equal kgpu_preempt_plan_gang:
      kernel time (CUDA events, median and spread of `--reps` calls), host time per call, gangs placed in one domain /
      across domains / failed, and pods placed by eviction;
  (d) the twin on 16 host threads, for (a).
(a)-(c) must agree with the twin bit for bit and (c) with kgpu_preempt_plan_gang (exit code 1 otherwise).
`--out FILE` also writes the figures as JSON."""
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
TWIN_THREADS = 16


def device_facts():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "unknown (nvidia-smi failed)"


def twin_lib(tmp):
    so = os.path.join(tmp, "libplan_domain_twin.so")
    subprocess.check_call(["gcc", "-O2", "-fPIC", "-std=c11", "-pthread", "-shared", "-o", so,
                           os.path.join(ROOT, "oracle", "oracle_b.c"), os.path.join(ROOT, "tests", "preempt_twin", "preempt_twin.c"),
                           os.path.join(ROOT, "tests", "preempt_plan_domain_twin", "plan_domain_twin.c")])
    return ctypes.CDLL(so)


def run_twin(L, topo, free, hold, domain, pods, lvl, gang, gd):
    W = np.ascontiguousarray(oracle_b.DEFAULT_WEIGHTS, dtype=np.int32)
    p = lambda a, t=ctypes.c_int32: np.ascontiguousarray(a).ctypes.data_as(ctypes.POINTER(t))  # noqa: E731
    F, H = np.array(free, np.int32, copy=True), np.array(hold, np.int32, copy=True)
    tk, tv = np.empty(len(pods), np.uint64), np.empty(len(pods), np.uint32)
    t0 = time.perf_counter()
    L.preempt_plan_domain_twin(p(topo), p(F), None, p(H), ctypes.c_int64(len(free)), ctypes.c_int64(0), p(domain), p(pods), p(lvl),
                               p(gang), p(gd), ctypes.c_int64(len(pods)), p(W), ctypes.c_int(TWIN_THREADS), p(tk, ctypes.c_uint64),
                               p(tv, ctypes.c_uint32))
    return tk, tv, time.perf_counter() - t0


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


def outcome(keys, vic, gang, domain):
    """(gangs placed in one domain, across domains, failed; pods placed by eviction)"""
    one = across = failed = 0
    for g in range(1, int(gang.max()) + 1):
        k = keys[gang == g]
        if (k == NO_FIT).all():
            failed += 1
            continue
        doms = {int(domain[(int(x) >> 8) & 0xFFFFFFFF]) for x in k if int(x) & 0xFF}
        if len(doms) == 1 and -1 not in doms:
            one += 1
        else:
            across += 1
    return one, across, failed, int((vic != 0).sum())


def main():
    out_path = sys.argv[sys.argv.index("--out") + 1] if "--out" in sys.argv else None
    reps = int(sys.argv[sys.argv.index("--reps") + 1]) if "--reps" in sys.argv else 10
    med = lambda v: float(np.median(v))  # noqa: E731
    topo, free, hold, pods, lvl, gang = synth.gen_preempt_gangs()
    res = {"device": device_facts(), "nodes": len(free), "pods": len(pods), "gangs": int(gang.max()), "reps": reps, "sizes": {}}
    print("device: %s" % res["device"], flush=True)
    print("gen_preempt_gangs: %d nodes, %d pods, %d gangs" % (res["nodes"], res["pods"], res["gangs"]))
    ok = True
    with tempfile.TemporaryDirectory() as tmp:
        L = twin_lib(tmp)
        with Scorer((0,)) as s:
            s.upload_nodes(topo, free)
            s.upload_holders(hold)
            (gk, gv), gcalls, gkerns = timed(s, reps, lambda: s.preempt_plan(pods, lvl, gang=gang))
            print("kgpu_preempt_plan_gang: kernels %.3f ms (spread %.3f - %.3f), call %.3f ms"
                  % (med(gkerns), min(gkerns), max(gkerns), med(gcalls)))
            res["plan_gang_kernels_ms"], res["spread_plan_gang_kernels_ms"] = med(gkerns), [min(gkerns), max(gkerns)]
            for size in (8, 32, 128):
                domain = synth.gen_domains(len(free), size)
                s.upload_domains(domain)
                row = {"domains": int(domain.max()) + 1}
                for name, mode in (("a_required", 1), ("b_preferred", 2), ("c_zero", 0)):
                    gd = np.where(gang != 0, mode, 0).astype(np.int32)
                    (k, v), calls, kerns = timed(s, reps, lambda: s.preempt_plan(pods, lvl, gang=gang, gang_domain=gd))
                    tk, tv, twin_s = run_twin(L, topo, free, hold, domain, pods, lvl, gang, gd)
                    exact = bool((tk == k).all() and (tv == v).all())
                    if mode == 0:
                        exact = exact and bool((gk == k).all() and (gv == v).all())
                    ok = ok and exact
                    one, across, failed, evict = outcome(k, v, gang, domain)
                    row[name] = {"kernels_ms": med(kerns), "spread_kernels_ms": [min(kerns), max(kerns)], "call_ms": med(calls),
                                 "gangs_one_domain": one, "gangs_across": across, "gangs_failed": failed, "placed_by_eviction": evict,
                                 "twin_s": twin_s, "exact": exact}
                    print("size %3d (%4d domains) %-11s: kernels %8.3f ms (spread %.3f - %.3f), call %8.3f ms; gangs in one domain "
                          "%3d, across %3d, failed %3d; %d pods by eviction; twin (%d threads) %.2f s; bit-exact %s"
                          % (size, row["domains"], name, med(kerns), min(kerns), max(kerns), med(calls), one, across, failed, evict,
                             TWIN_THREADS, twin_s, exact), flush=True)
                res["sizes"][str(size)] = row
    if out_path:
        with open(out_path, "w") as f:
            json.dump(res, f, indent=1)
    if not ok:
        sys.exit(1)


if __name__ == "__main__":
    main()
