#!/usr/bin/env python3
"""Times gangs in nested network domains (kgpu_place_batch_gang_levels) on config C2 (synth.gen_gangs: 100k nodes, 10k
pods, about a third of them in gangs of 2..8 members), with racks of 32 nodes inside spines of 1024 and, separately,
of about 3 125 nodes (synth.gen_domain_levels).  Per spine size:
  (a) every gang REQUIRED, bound r = 0 (racks only: kgpu_place_batch_gang_domain on level 0);
  (b) every gang REQUIRED, r = 1 (a gang that no rack holds climbs to the spines);
  (c) every gang PREFERRED, r = 1;
  (d) the same pods as plain gangs (gang_domain = 0).
Device figures are dry runs on the uploaded state: the CUDA-event time of the whole device path (place_init to the last
launch) and the wall time of the call, median of 10 with min..max.  For each run: gangs placed inside a rack, inside a
spine, across spines (PREFERRED fallbacks) and failed, and whether the keys equal the CPU twin
(tests/gang_domain_levels_twin) key for key.  Prints the device name and power limit with the figures; `--out FILE`
also writes them as JSON."""
import ctypes
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402

import cpu_libs  # noqa: E402
from kubegpu_b200 import _lib, synth  # noqa: E402
from kubegpu_b200.scorer import Scorer  # noqa: E402
from oracle import oracle_b  # noqa: E402

NO_FIT = np.uint64(_lib.NO_FIT)
_i32p, _u64p = ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_uint64)


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


def outcome(keys, gang, dom):
    """Gangs by the lowest level whose one domain holds every member: in a rack / a spine / across, and failed."""
    res = {"in_rack": 0, "in_spine": 0, "across": 0, "failed": 0}
    for a, e in gang_runs(gang):
        if (keys[a:e] == NO_FIT).any():
            res["failed"] += 1
            continue
        nodes = [(int(k) >> 8) & 0xFFFFFFFF for k in keys[a:e]]
        for name, lv in (("in_rack", 0), ("in_spine", 1)):
            ids = {int(dom[lv][n]) for n in nodes}
            if len(ids) == 1 and -1 not in ids:
                res[name] += 1
                break
        else:
            res["across"] += 1
    return res


def timed(s, pods, gang, gd, gl, reps=10):
    kern, call, keys = [], [], None
    for i in range(reps + 1):                       # call 0 warms up
        t0 = time.perf_counter()
        got = s.place_batch(pods, gang=gang, gang_domain=gd, gang_level=gl, dry_run=True)
        t1 = time.perf_counter()
        if i:
            kern.append(s.last_kernel_ms)
            call.append((t1 - t0) * 1e3)
        assert keys is None or (got == keys).all()
        keys = got
    stat = lambda v: {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))}
    return keys, {"kernel_ms": stat(kern), "call_ms": stat(call), "reps": reps}


def twin_place(topo, free, pods, gang, gd, gl, dom):
    L = cpu_libs.twin("gang_domain_levels")
    c = lambda a: np.ascontiguousarray(a, dtype=np.int32)
    args = [c(a) for a in (topo, dom, pods, gang, gd, gl, oracle_b.DEFAULT_WEIGHTS)]
    p32 = [a.ctypes.data_as(_i32p) for a in args]
    f = np.array(free, dtype=np.int32, copy=True)
    keys = np.empty(len(pods), dtype=np.uint64)
    L.levels_twin_place_batch(p32[0], f.ctypes.data_as(_i32p), None, ctypes.c_int64(len(f)), ctypes.c_int64(0), p32[1],
                              ctypes.c_int(dom.shape[0]), p32[2], p32[3], p32[4], p32[5], ctypes.c_int64(len(pods)), p32[6],
                              keys.ctypes.data_as(_u64p))
    return keys


def main():
    out_path = sys.argv[sys.argv.index("--out") + 1] if "--out" in sys.argv else None
    topo, free, pods, gang = synth.gen_gangs()
    N, P = len(free), len(pods)
    member = (gang != 0).astype(np.int32)
    zero = np.zeros(P, np.int32)
    res = {"device": device_facts(), "nodes": N, "pods": P, "gangs": len(gang_runs(gang)), "runs": []}
    print("device: %s" % res["device"])
    with Scorer((0,)) as s:
        s.upload_nodes(topo, free)
        for spine in (1024, 3125):
            dom = synth.gen_domain_levels(N, (32, spine))
            s.upload_domains(dom)
            runs = (("(a) REQUIRED r=0", member * 1, zero), ("(b) REQUIRED r=1", member * 1, member),
                    ("(c) PREFERRED r=1", member * 2, member), ("(d) plain gangs", zero, zero))
            for name, gd, gl in runs:
                keys, t = timed(s, pods, gang, gd, gl)
                line = dict(t, run=name, rack_nodes=32, spine_nodes=spine, **outcome(keys, gang, dom))
                if gd.any():
                    line["equals_twin"] = bool((twin_place(topo, free, pods, gang, gd, gl, dom) == keys).all())
                res["runs"].append(line)
                print(json.dumps(line), flush=True)
    if out_path:
        with open(out_path, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
