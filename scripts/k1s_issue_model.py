#!/usr/bin/env python3
"""Instruction count per K1s launch predicted from the SASS (no GPU needed):
    python scripts/k1s_issue_model.py <lib.so> [kernel-substr] [--ks 1,2,4,8] [--nodes 100000] [--pods 10000]
Takes the (K,F) bucket loops from sass_loops (the loops with a REDUX, in source order K = 0..8; inside one K
the loop with more instructions serves the larger F), weights them with how often a config with
f ~ Binomial(8, 1/2) per node and k uniform over --ks runs them, and prints instructions per (warp, pod),
per launch, and the time at a given issue utilisation."""
import argparse
import math
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import sass_loops  # noqa: E402


def bucket_loops(lib, sub):
    """(kernel name, [(instructions, ALU-pipe instructions, REDUX, local-memory instructions) per bucket loop])"""
    fns = sass_loops.functions(lib)
    name = [n for n in fns if sub in n][0]
    rows = fns[name]
    import re
    addr_index = {a: i for i, (a, _) in enumerate(rows)}
    loops = []
    for i, (a, ins) in enumerate(rows):
        m = re.search(r"BRA(?:\.\w+)*\s+(?:U?P\d+,\s*)?0x([0-9a-f]+)", ins)
        if m and int(m.group(1), 16) <= a and int(m.group(1), 16) in addr_index:
            loops.append((addr_index[int(m.group(1), 16)], i))
    inner = [l for l in loops if not any(o != l and l[0] <= o[0] and o[1] <= l[1] for o in loops)]
    out = []
    for lo, hi in inner:
        body = rows[lo:hi + 1]
        redux = sum(1 for _, ins in body if "REDUX" in ins)
        if redux:
            alu = sum(1 for _, ins in body if sass_loops.klass(sass_loops.opcode(ins)) == "alu")
            local = sum(1 for _, ins in body if sass_loops.opcode(ins).split(".")[0] in ("LDL", "STL"))
            out.append((len(body), alu, redux, local))
    return name, out


HEADLINE = "score_pairs_sparseILb1ELb0ELb1ELb0ELi0E"     # <PER_PAIR, !MEM, BYTE_KEYS, !STREAM, 0>: C2's kernel


def per_pod(lib, kernel=HEADLINE, ks=(1, 2, 4, 8)):
    """(kernel name, instructions per (warp, pod), of which ALU pipe) for k uniform over ks.  A loop handles
    as many pods per trip as it has REDUX (one warp min per pod); the k = 0 loop, whose pods all get the
    same key and share one REDUX, is taken at the k = 1 loop's width."""
    name, loops = bucket_loops(lib, kernel)
    sizes = [1, 1, 7, 6, 5, 4, 3, 2, 1]                 # loops per K: F = max(K,2)..8 (K <= 1: one loop)
    if len(loops) != sum(sizes):
        sys.exit("expected %d bucket loops, found %d" % (sum(sizes), len(loops)))
    table, at = {}, 0
    for K, cnt in enumerate(sizes):
        grp = [(n, al, loops[1][2] if K == 0 else redux) for n, al, redux, _ in loops[at:at + cnt]]
        at += cnt
        grp.sort(key=lambda l: l[0] / l[2])             # more instructions per pod: larger F
        for j, (n, alu, width) in enumerate(grp):
            table[(K, max(K, 2) + j if K >= 2 else 8)] = (n / width, alu / width)
    pf = [math.comb(8, f) / 256.0 for f in range(9)]
    inst = alu = 0.0
    for k in ks:
        for f in range(9):
            if f < k:
                continue
            n, al = table[(k, 8)] if k <= 1 else table[(k, f)]
            inst += pf[f] * n / len(ks)
            alu += pf[f] * al / len(ks)
    return name, inst, alu


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("lib")
    ap.add_argument("kernel", nargs="?", default=HEADLINE)
    ap.add_argument("--ks", default="1,2,4,8")
    ap.add_argument("--nodes", type=int, default=100_000)
    ap.add_argument("--pods", type=int, default=10_000)
    ap.add_argument("--issue", type=float, default=0.82, help="issue utilisation (assumed; not measured on the H100)")
    ap.add_argument("--ghz", type=float, default=1.98, help="SM clock (H100 SXM maximum: 1.98)")
    ap.add_argument("--sms", type=int, default=132, help="SM count (H100 SXM: 132)")
    ap.add_argument("--extra", type=float, default=0.15, help="pod sort + flush share on top of the loops")
    a = ap.parse_args()
    name, inst, alu = per_pod(a.lib, a.kernel, [int(x) for x in a.ks.split(",")])
    warps = (a.nodes + 31) // 32
    total = inst * warps * a.pods * (1 + a.extra)
    cycles = total / (a.sms * 4 * a.issue)
    print("#", name)
    print("instructions per (warp, pod): %.2f   of which ALU pipe: %.2f" % (inst, alu))
    print("per launch (%d nodes x %d pods, +%.0f%% sort/flush): %.3g warp instructions" % (a.nodes, a.pods, a.extra * 100, total))
    print("at %.0f%% issue utilisation, %.2f GHz: %.3f ms" % (a.issue * 100, a.ghz, cycles / (a.ghz * 1e6)))


if __name__ == "__main__":
    main()
