#!/usr/bin/env python3
"""K1s alone on C2's cluster (100k nodes) for five batches of 10k pods -- C2's mix of k in {1,2,4,8}, then all
k = 1, 2, 4, 8 -- with one or more libkgpu builds timed alternately in the same process:
    python scripts/k1s_breakdown.py [LABEL=SPEC ...] [--launches 30] [--rounds 3] [--keep DIR] [--build-only]
SPEC is a built libkgpu.so, or git:REV[+DNAME=VALUE...] to build REV's library (git archive + make, with the
given -D flags) into a temporary directory, or into --keep DIR.  Without a SPEC: the tree's own library.
Each (build, batch) is one score_batch_device call (as bench.py's kernel_ms) per launch, L2 flushed before
each, CUDA events around it; the median and the spread over all its launches are printed next to the bucket
loops' instruction count from the build's SASS (k1s_issue_model.py), so the issue rate can be read off.  The
all-k = 1 batch has loops of nothing but per-pod overhead: it shows the per-pod and per-chunk fixed costs.
Keys must be bit-identical across builds for every batch; the script exits 1 otherwise."""
import argparse
import hashlib
import os
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
if shutil.which("cuobjdump") is None and os.path.exists("/usr/local/cuda/bin/cuobjdump"):
    os.environ["PATH"] += os.pathsep + "/usr/local/cuda/bin"

N_NODES, N_PODS = 100_000, 10_000
BATCHES = [("c2_mix", (1, 2, 4, 8)), ("k1", (1,)), ("k2", (2,)), ("k4", (4,)), ("k8", (8,))]


def build(label, spec, out_dir):
    """git:REV[+DNAME=VALUE...] -> path of the libkgpu.so built from REV with those defines."""
    rev, *defs = spec[4:].split("+")
    src = tempfile.mkdtemp(prefix="k1s_src_")
    try:
        tar = subprocess.run(["git", "-C", ROOT, "archive", rev], check=True, capture_output=True).stdout
        subprocess.run(["tar", "-x", "-C", src], input=tar, check=True)
        extra = " ".join("-D" + d for d in defs)
        subprocess.run(["make", "-C", src, "-s", "kubegpu_b200/lib/libkgpu.so", "EXTRA=" + extra], check=True,
                       stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
        dst = os.path.join(out_dir, "libkgpu_%s.so" % label)
        shutil.copy(os.path.join(src, "kubegpu_b200", "lib", "libkgpu.so"), dst)
        return dst
    finally:
        shutil.rmtree(src, ignore_errors=True)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "nvidia-smi unavailable"


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("builds", nargs="*", metavar="LABEL=SPEC")
    ap.add_argument("--launches", type=int, default=30, help="timed launches per (build, batch) and round")
    ap.add_argument("--rounds", type=int, default=3, help="the builds alternate once per round and batch")
    ap.add_argument("--keep", metavar="DIR", help="build git: specs into DIR instead of a temporary directory")
    ap.add_argument("--build-only", action="store_true")
    a = ap.parse_args()
    out_dir = a.keep or tempfile.mkdtemp(prefix="k1s_libs_")
    os.makedirs(out_dir, exist_ok=True)
    libs = []
    for b in a.builds or ["tree=" + os.path.join(ROOT, "kubegpu_b200", "lib", "libkgpu.so")]:
        label, spec = b.split("=", 1)
        libs.append((label, os.path.abspath(build(label, spec, out_dir) if spec.startswith("git:") else spec)))
    if a.build_only:
        for label, path in libs:
            print(label, path)
        return

    import numpy as np
    import torch
    import k1s_issue_model
    from kubegpu_b200 import _lib, synth
    from kubegpu_b200.scorer import Scorer

    print("# GPU:", gpu_info(), flush=True)
    topo, free, c2_pods = synth.gen_c2(N_NODES, N_PODS)
    pods = {"c2_mix": c2_pods}
    for name, ks in BATCHES[1:]:
        pods[name] = synth.make_pods(np.full(N_PODS, ks[0], dtype=np.int32))
    d_pods = {n: torch.from_numpy(p).cuda() for n, p in pods.items()}
    d_keys = torch.empty(N_PODS, dtype=torch.int64, device="cuda")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")    # > the H100's 50 MB L2
    stream = torch.cuda.Stream()
    scorers = []
    for label, path in libs:
        _lib._lib, _lib.LIB_PATH = None, path        # each Scorer keeps the library it was created with
        s = Scorer((0,))
        s.upload_nodes(topo, free)
        s.set_variant(_lib.VARIANT_SPARSE)
        scorers.append(s)
    _lib._lib = None

    def launch(s, name):
        s.score_batch_device(d_pods[name].data_ptr(), N_PODS, d_keys.data_ptr(), stream.cuda_stream, _lib.BATCH_NO_MIN_MEM)

    times = {(li, n): [] for li in range(len(libs)) for n, _ in BATCHES}
    digest = {}
    with torch.cuda.stream(stream):
        for li, s in enumerate(scorers):
            for n, _ in BATCHES:
                for _ in range(3):
                    launch(s, n)
                stream.synchronize()
                digest[(li, n)] = hashlib.sha256(d_keys.cpu().numpy().tobytes()).hexdigest()[:12]
        for _ in range(a.rounds):
            for n, _ in BATCHES:
                for li, s in enumerate(scorers):
                    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(a.launches)]
                    for e0, e1 in ev:
                        flush.zero_()
                        e0.record(stream)
                        launch(s, n)
                        e1.record(stream)
                    stream.synchronize()
                    times[(li, n)] += [e0.elapsed_time(e1) for e0, e1 in ev]

    warps = (N_NODES + 31) // 32
    print("%-10s %-7s %9s %17s %9s %12s %8s  %s" % ("build", "batch", "median_ms", "spread(min-max)", "inst/pod",
                                                   "loop_inst", "Ginst/s", "keys"))
    ok = True
    for n, ks in BATCHES:
        for li, (label, path) in enumerate(libs):
            t = np.array(times[(li, n)])
            med = float(np.median(t))
            try:
                per_pod = k1s_issue_model.per_pod(path, ks=ks)[1]
            except (SystemExit, IndexError, OSError):
                per_pod = float("nan")
            inst = per_pod * warps * N_PODS
            same = digest[(li, n)] == digest[(0, n)]
            ok &= same
            print("%-10s %-7s %9.4f %8.4f-%-8.4f %9.2f %12.4g %8.1f  %s%s" % (
                label, n, med, t.min(), t.max(), per_pod, inst, inst / (med * 1e-3) / 1e9, digest[(li, n)],
                "" if same else "  MISMATCH vs " + libs[0][0]))
    print("# Ginst/s: the bucket loops' warp instructions (model) over the median time; the H100 SXM issues at most "
          "132 SMs x 4 x clock (1.98 GHz: 1045 G/s).  launches per (build, batch): %d" % (a.launches * a.rounds))
    for s in scorers:
        s.close()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
