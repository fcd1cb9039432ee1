#!/usr/bin/env python3
"""Times gangs constrained to one network domain (kgpu_place_batch_gang_domain) on config C2 (synth.gen_gangs: 100k
nodes, 10k pods, about a third of them in gangs of 2..8 members), with the nodes dealt into domains of 8, 32 and 128
nodes (synth.gen_domains) and into one domain holding every node.  Per domain size:
  (a) every gang REQUIRED;
  (b) every gang PREFERRED;
  (c) the same pods with gang_domain = 0 (plain kgpu_place_batch_gang; the same for every domain size);
  (d) the CPU twin (tests/gang_domain_twin) of (a) on one host thread, which (a) must equal key for key.
Device figures are dry runs on the uploaded state: the CUDA-event time of the whole device path (place_init to the last
launch) and the wall time of the call, median of 10 with min..max (3 for the single domain, the slowest line: one warp
walks all 100k nodes per member, by chunk minima).  For each run: gangs placed
inside one domain, gangs placed across domains (PREFERRED fallbacks) and gangs that failed.  Prints the device name and
power limit with the figures; `--out FILE` also writes them as JSON."""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402

import gang_domain_libs  # noqa: E402
from kubegpu_b200 import _lib, synth  # noqa: E402
from kubegpu_b200.scorer import Scorer  # noqa: E402
from oracle import oracle_b  # noqa: E402

NO_FIT = np.uint64(_lib.NO_FIT)


def device_facts():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "unknown (nvidia-smi failed)"


def gang_runs(gang):
    out, p = [], 0
    while p < len(gang):
        e = p + 1
        while e < len(gang) and gang[e] == gang[p]:
            e += 1
        if gang[p] != 0:
            out.append((p, e))
        p = e
    return out


def outcome(keys, gang, domain):
    inside = across = failed = 0
    for a, e in gang_runs(gang):
        if (keys[a:e] == NO_FIT).any():
            failed += 1
            continue
        doms = {int(domain[(int(k) >> 8) & 0xFFFFFFFF]) for k in keys[a:e]}
        if len(doms) == 1 and -1 not in doms:
            inside += 1
        else:
            across += 1
    return {"inside_one_domain": inside, "across_domains": across, "failed": failed}


def timed(s, pods, gang, gd, reps):
    kern, call, keys = [], [], None
    for i in range(reps + 1):                       # call 0 warms up
        t0 = time.perf_counter()
        got = s.place_batch(pods, gang=gang, gang_domain=gd, dry_run=True)
        t1 = time.perf_counter()
        if i:
            kern.append(s.last_kernel_ms)
            call.append((t1 - t0) * 1e3)
        assert keys is None or (got == keys).all()
        keys = got
    stat = lambda v: {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))}
    return keys, {"kernel_ms": stat(kern), "call_ms": stat(call), "reps": reps}


def twin_place(topo, free, pods, gang, gd, domain):
    L = gang_domain_libs.twin()
    p32 = lambda a: np.ascontiguousarray(a, dtype=np.int32).ctypes.data_as(gang_domain_libs._i32p)
    W = np.ascontiguousarray(oracle_b.DEFAULT_WEIGHTS, dtype=np.int32)
    f = np.array(free, dtype=np.int32, copy=True)
    keys = np.empty(len(pods), dtype=np.uint64)
    args = [np.ascontiguousarray(a, dtype=np.int32) for a in (topo, domain, pods, gang, gd)]
    t0 = time.perf_counter()
    L.gang_domain_twin_place_batch(p32(args[0]), f.ctypes.data_as(gang_domain_libs._i32p), None, len(f), 0, p32(args[1]), p32(args[2]),
                                   p32(args[3]), p32(args[4]), len(pods), p32(W), keys.ctypes.data_as(gang_domain_libs._u64p))
    return keys, (time.perf_counter() - t0) * 1e3


def main():
    out_path = sys.argv[sys.argv.index("--out") + 1] if "--out" in sys.argv else None
    topo, free, pods, gang = synth.gen_gangs()
    N = len(free)
    member = (gang != 0).astype(np.int32)
    res = {"device": device_facts(), "nodes": N, "pods": len(pods), "gangs": len(gang_runs(gang)), "runs": []}
    print("device: %s" % res["device"])
    with Scorer((0,)) as s:
        s.upload_nodes(topo, free)
        keys, t = timed(s, pods, gang, np.zeros(len(pods), np.int32), 10)
        line = dict(t, run="(c) gang_domain = 0", **outcome(keys, gang, np.zeros(N, np.int32) - 1))
        res["runs"].append(line)
        print(json.dumps(line))
        for size in (8, 32, 128, N):
            domain = synth.gen_domains(N, size)
            s.upload_domains(domain)
            reps = 3 if size == N else 10
            req_keys = None
            for name, mode in (("(a) REQUIRED", 1), ("(b) PREFERRED", 2)):
                keys, t = timed(s, pods, gang, member * mode, reps)
                if mode == 1:
                    req_keys = keys
                line = dict(t, run=name, domain_size=size, **outcome(keys, gang, domain))
                res["runs"].append(line)
                print(json.dumps(line))
            twin_keys, twin_ms = twin_place(topo, free, pods, gang, member, domain)
            line = {"run": "(d) twin of (a), one host thread", "domain_size": size, "ms": twin_ms,
                    "equals_a": bool((twin_keys == req_keys).all())}
            res["runs"].append(line)
            print(json.dumps(line))
    if out_path:
        with open(out_path, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
