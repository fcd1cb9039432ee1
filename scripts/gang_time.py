#!/usr/bin/env python3
"""Times gang placement on config C2 (synth.gen_gangs: 100k nodes, 10k pods, about a third in gangs) and checks it.
Three ways to the same result:
  (a) kgpu_place_batch_gang: one call, failed gangs undone on the device;
  (b) the same pods with gang=None: plain K3, so (a) - (b) is what the gang bookkeeping and the undos cost;
  (c) the host-side fallback without the feature: dry run, drop the FIRST gang with a miss, repeat until no gang
      misses, then commit -- one full K3 run (place_init over every node included) per failed gang.
Check: (a) and (c) give the same keys and masks (c decides which gangs fail with plain K3 alone), and they equal the
oracle's plain sequential placement of the batch without the failed gangs.  Prints the device name and power limit
with the figures; `--out FILE` also writes them as JSON."""
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from kubegpu_b200 import _lib, synth  # noqa: E402
from kubegpu_b200.scorer import Scorer  # noqa: E402
from oracle import oracle_b  # noqa: E402

NO_FIT = np.uint64(_lib.NO_FIT)


def device_facts():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "unknown (nvidia-smi failed)"


def first_failed_gang(keys, gang):
    miss = np.flatnonzero((keys == NO_FIT) & (gang != 0))
    return None if len(miss) == 0 else int(gang[miss[0]])


def host_fallback(s, topo, free, pods, gang):
    """(c): returns the keys in the original pod order and the number of K3 runs."""
    keep = np.ones(len(pods), dtype=bool)
    runs = 0
    s.upload_nodes(topo, free)
    while True:
        keys = s.place_batch(pods[keep], dry_run=True)
        runs += 1
        g = first_failed_gang(keys, gang[keep])
        if g is None:
            break
        keep &= gang != g
    out = np.full(len(pods), NO_FIT, dtype=np.uint64)
    out[keep] = s.place_batch(pods[keep])
    return out, runs + 1


def main():
    out_path = sys.argv[sys.argv.index("--out") + 1] if "--out" in sys.argv else None
    reps = 5
    topo, free, pods, gang = synth.gen_gangs()
    a_call, a_kern, b_call, b_kern, c_call = [], [], [], [], []
    want = wf = None
    exact = True
    with Scorer((0,)) as s:
        for i in range(reps + 1):                     # rep 0 warms up
            s.upload_nodes(topo, free)
            t0 = time.perf_counter()
            got = s.place_batch(pods, gang=gang)
            t1 = time.perf_counter()
            if i:
                a_call.append((t1 - t0) * 1e3)
                a_kern.append(s.last_kernel_ms)
            if want is None:
                want, wf = got, s.get_free_masks()
            exact = exact and bool((got == want).all() and (s.get_free_masks() == wf).all())
            s.upload_nodes(topo, free)
            t0 = time.perf_counter()
            s.place_batch(pods)
            t1 = time.perf_counter()
            if i:
                b_call.append((t1 - t0) * 1e3)
                b_kern.append(s.last_kernel_ms)
        for i in range(3):
            t0 = time.perf_counter()
            got_c, k3_runs = host_fallback(s, topo, free, pods, gang)
            t1 = time.perf_counter()
            c_call.append((t1 - t0) * 1e3)
            exact = exact and bool((got_c == want).all() and (s.get_free_masks() == wf).all())
    failed_ids = [g for g in np.unique(gang[gang != 0]) if (want[gang == g] == NO_FIT).any()]
    keep = ~np.isin(gang, failed_ids)
    ok_keys, ok_free = oracle_b.place_batch(topo, free, pods[keep])
    exact = exact and bool((want[keep] == ok_keys).all() and (want[~keep] == NO_FIT).all() and (wf == ok_free).all())
    failed = len(failed_ids)
    res = {"device": device_facts(), "nodes": len(free), "pods": len(pods), "gang_pods": int((gang != 0).sum()),
           "gangs": int(len(np.unique(gang[gang != 0]))), "failed_gangs": failed}
    med = lambda v: float(np.median(v))  # noqa: E731
    res.update({"a_gang_call_ms": med(a_call), "a_gang_kernel_ms": med(a_kern),
                "b_plain_call_ms": med(b_call), "b_plain_kernel_ms": med(b_kern),
                "c_host_fallback_ms": med(c_call), "c_k3_runs": k3_runs, "reps": reps, "exact": exact,
                "spread_a_kernel_ms": [min(a_kern), max(a_kern)], "spread_b_kernel_ms": [min(b_kern), max(b_kern)]})
    print("device: %s" % res["device"])
    print("C2 gangs: %d nodes, %d pods, %d gangs (%d pods), %d gangs fail" %
          (res["nodes"], res["pods"], res["gangs"], res["gang_pods"], failed))
    print("(a) kgpu_place_batch_gang : kernels %.3f ms, call %.3f ms" % (res["a_gang_kernel_ms"], res["a_gang_call_ms"]))
    print("(b) gang=None             : kernels %.3f ms, call %.3f ms" % (res["b_plain_kernel_ms"], res["b_plain_call_ms"]))
    print("(c) host fallback         : %.1f ms (%d K3 runs)" % (res["c_host_fallback_ms"], k3_runs))
    print("(a) == (c) == oracle without the failed gangs: %s" % exact)
    if out_path:
        with open(out_path, "w") as f:
            json.dump(res, f, indent=1)
    if not exact:
        sys.exit(1)


if __name__ == "__main__":
    main()
