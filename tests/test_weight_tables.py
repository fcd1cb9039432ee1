"""Every kernel under link-weight tables other than the default one.

A key packs the subset cost into a fixed field, and a cost can reach 28 * 4095 = 114 660 (17 bits) under the tables
kgpu_set_weights accepts; the default table keeps it at 11 bits.  The tables below fill that field (flat_max,
one_level), sit on both sides of the boundary where K1s switches from byte-aligned warp keys to the general layout
(byte_edge: every weight 2340, general_edge: one level at 2341), make every answer a tie-break (zero), or mix all of it.

CPU: a plain Python-int reference with the table as a parameter (snapshot scoring, sequential placement with gang undo,
preemption's order) against Oracle B, the gang twin and the preemption twin; then the kernel sources, run on the CPU
through tests/emu, against the twins.  GPU: the device paths through Scorer, bit-exact, and weight changes on a live
handle."""
import ctypes
import itertools
import os

import numpy as np
import pytest

import cpu_libs
from kubegpu_b200 import _lib, synth
from test_gang_placement import chunk_batch, edge_batch, random_gangs, runs
from test_preemption import extreme_levels_case, min_mem_case, multi_block_case, random_holders, ties_case

NO_FIT = np.uint64(0xFFFFFFFFFFFFFFFF)
NODE_NO_FIT = 0xFFFFFFFF

L_EDGE = 9                                  # an NVLink level of gen_c4 (7..12): the level general_edge and one_level raise
_rng = np.random.default_rng(0x5EED)
TABLES = {
    "default": [64, 32, 16, 8, 4, 2, 1] + [0] * 9,
    "zero": [0] * 16,
    "flat_max": [4095] * 16,
    "byte_edge": [2340] * 16,                                           # the last table served by byte-aligned warp keys
    "general_edge": [2341 if i == L_EDGE else 2340 for i in range(16)],  # the first one that is not
    "one_level": [4095 if i == L_EDGE else 0 for i in range(16)],
    "mixed": [4095, 1, 4094, 2, 4000, 3, 2341, 2340, 0, 17, 4095, 1000, 5, 4095, 0, 77],
    "random1": _rng.integers(0, 4096, size=16).tolist(),
    "random2": _rng.integers(0, 4096, size=16).tolist(),
}
NAMES = list(TABLES)


def W_of(name):
    return np.array(TABLES[name], dtype=np.int32)


def _p(a, t=ctypes.c_int32):
    return a.ctypes.data_as(ctypes.POINTER(t))


def _opt(a):
    return None if a is None else _p(np.ascontiguousarray(a, dtype=np.int32))


def cost_of(key):
    return int(key) >> 40


# ---- batches --------------------------------------------------------------------------------------------------------
def edge_matrix(level=L_EDGE):
    """Every pair of the 8 GPUs at one link level: a k = 8 pod costs 28 * W[level] here."""
    m = np.full((8, 8), level, dtype=np.int32)
    np.fill_diagonal(m, 0)
    return m.reshape(64)


def with_edge(topo, free, pods, mem=None, at=1):
    """The batch with the edge node (all 8 GPUs free, the largest memory class) inserted at node `at`, and pods 0 and 1
    asking for 8 and 7 GPUs without a memory requirement; with mem, pods 2 and 3 ask for 8 and 7 with one."""
    topo = np.insert(np.asarray(topo, np.int32), at, edge_matrix(), axis=0)
    free = np.insert(np.asarray(free, np.int32), at, 0xFF)
    pods = np.array(pods, dtype=np.int32, copy=True)
    pods[0, 0], pods[0, 3] = 8, 0
    pods[1, 0], pods[1, 3] = 7, 0
    if mem is not None:
        mem = np.insert(np.asarray(mem, np.int32), at, max(synth.GPU_MEM_CLASSES_MIB), axis=0)
        pods[2, 0], pods[2, 3] = 8, 100_000
        pods[3, 0], pods[3, 3] = 7, 40_000
    return topo, free, pods, mem


def check_reached(name, keys, topo=None, free=None):
    """The batch does what its table is there for: under flat_max some key's cost needs 17 bits, under zero every
    fitting key costs 0, under general_edge the edge node's k = 8 cost is 28 * 2341 >= 2^16."""
    keys = np.asarray(keys, dtype=np.uint64)
    fit = keys[keys != NO_FIT]
    assert len(fit)
    if name == "flat_max":
        assert max(cost_of(k) for k in fit) >= 1 << 16
    if name == "zero":
        assert all(cost_of(k) == 0 for k in fit)
    if name == "general_edge" and topo is not None:
        e = [n for n in range(len(free)) if (topo[n] == edge_matrix()).all() and int(free[n]) & 0xFF == 0xFF]
        assert e and ref_node_key(topo[e[0]], 0xFF, 8, TABLES[name]) >> 8 == 28 * 2341 >= 1 << 16


def _node_keys_as_keys(nk):
    """Node keys (cost << 8 | S) as batch keys on node 0, for check_reached."""
    return [NO_FIT if w == NODE_NO_FIT else np.uint64((int(w) >> 8) << 40 | (int(w) & 0xFF)) for w in nk]


# ---- the plain Python reference ---------------------------------------------------------------------------------------
def ref_node_key(M, fm, k, W):
    """(cost << 8 | S) of the cheapest k-subset S of the free GPUs in fm, lowest S on ties; NODE_NO_FIT if none."""
    if not 0 <= k <= 8:
        return NODE_NO_FIT
    gpus = [i for i in range(8) if (int(fm) >> i) & 1]
    best = NODE_NO_FIT
    for S in itertools.combinations(gpus, k):
        cost = sum(int(W[int(M[i * 8 + j])]) for i, j in itertools.combinations(S, 2))
        best = min(best, cost << 8 | sum(1 << i for i in S))
    return best


def _eligible(mem, n, need):
    if mem is None or need <= 0:
        return 0xFF
    return sum(1 << i for i in range(8) if int(mem[n][i]) >= need)


class _NodeKeys:
    """ref_node_key memoised by (node, usable mask, k) for one table."""

    def __init__(self, topo, W):
        self.topo, self.W, self.memo = topo, [int(w) for w in W], {}

    def __call__(self, n, fm, k):
        key = (n, fm, k)
        if key not in self.memo:
            self.memo[key] = ref_node_key(self.topo[n], fm, k, self.W)
        return self.memo[key]


def ref_score(topo, free, pods, W, mem=None, base=0):
    """Snapshot scoring: per pod the smallest (cost, node id, S) over every node."""
    nk, out = _NodeKeys(topo, W), []
    for k, _, _, need in np.asarray(pods).tolist():
        best = None
        for n in range(len(free)):
            v = nk(n, int(free[n]) & _eligible(mem, n, need), k)
            if v != NODE_NO_FIT and (best is None or (v >> 8, n) < (best[0] >> 8, best[1])):
                best = (v, n)
        out.append(NO_FIT if best is None else np.uint64((best[0] >> 8) << 40 | (base + best[1]) << 8 | (best[0] & 0xFF)))
    return np.array(out, dtype=np.uint64)


def ref_place(topo, free, pods, W, gang=None, mem=None, base=0):
    """Sequential placement: pods in order, each takes its GPUs.  A run of pods with one nonzero gang id is placed all
    or nothing: when a member does not fit, the members before it give their GPUs back and every member gets NO_FIT.
    Returns (keys, free masks after)."""
    nk = _NodeKeys(topo, W)
    fm = [int(f) for f in free]
    pods = np.asarray(pods).tolist()
    gang = [0] * len(pods) if gang is None else [int(g) for g in gang]
    keys = [NO_FIT] * len(pods)
    p = 0
    while p < len(pods):
        e = p + 1
        while gang[p] and e < len(pods) and gang[e] == gang[p]:
            e += 1
        saved, ok = list(fm), True
        for q in range(p, e):
            k, _, _, need = pods[q]
            best = None
            for n in range(len(fm)):
                v = nk(n, fm[n] & 0xFF & _eligible(mem, n, need), k)
                if v != NODE_NO_FIT and (best is None or (v >> 8, n) < (best[0] >> 8, best[1])):
                    best = (v, n)
            if best is None:
                ok = False
                break
            keys[q] = np.uint64((best[0] >> 8) << 40 | (base + best[1]) << 8 | (best[0] & 0xFF))
            fm[best[1]] &= ~(best[0] & 0xFF)
        if not ok:
            fm = saved
            keys[p:e] = [NO_FIT] * (e - p)
        p = e
    return np.array(keys, dtype=np.uint64), np.array(fm, dtype=np.int32)


def ref_preempt(topo, free, pods, lvl, hold, W, mem=None, base=0):
    """Preemption: every node and k-subset S whose GPUs are free or held by owners of a level below the pod's; the
    smallest (max victim level, |V|, cost, node id, S).  Returns (keys, victim owner masks)."""
    W = [int(w) for w in W]
    cost = {}
    keys, vic = [], []
    for (k, _, _, need), L in zip(np.asarray(pods).tolist(), np.asarray(lvl).tolist()):
        best = None
        for n in range(len(free) if 0 <= k <= 8 else 0):
            elig = _eligible(mem, n, need)
            for S in itertools.combinations(range(8), k):
                V, ok = {}, True
                for i in S:
                    if not (elig >> i) & 1:
                        ok = False
                    elif not (int(free[n]) >> i) & 1:
                        e = int(hold[n][i])
                        if e < 0 or e >> 3 >= L:
                            ok = False
                        else:
                            V[e & 7] = e >> 3
                if not ok:
                    continue
                if (n, S) not in cost:
                    cost[n, S] = sum(W[int(topo[n][i * 8 + j])] for i, j in itertools.combinations(S, 2))
                t = (max(V.values(), default=0), len(V), cost[n, S], base + n, sum(1 << i for i in S), sum(1 << o for o in V))
                if best is None or t[:5] < best[:5]:
                    best = t
        keys.append(NO_FIT if best is None else np.uint64(best[2] << 40 | best[3] << 8 | best[4]))
        vic.append(0 if best is None else best[5])
    return np.array(keys, dtype=np.uint64), np.array(vic, dtype=np.uint32)


# ---- the twins, with the table as a parameter ---------------------------------------------------------------------------
@pytest.fixture(scope="session")
def twins():
    """(gang(topo, free, pods, gang, W, mem=None, base=0) -> (keys, free_after),
        preempt(topo, free, pods, lvl, hold, W, mem=None, base=0) -> (keys, victims)):
    tests/gang_twin/gang_twin.c and tests/preempt_twin/preempt_twin.c built with the oracle."""
    G, Pr = cpu_libs.twin("gang"), cpu_libs.twin("preempt")

    def gang(topo, free, pods, gang, W, mem=None, base=0):
        topo, pods, gang, W = (np.ascontiguousarray(a, dtype=np.int32) for a in (topo, pods, gang, W))
        f = np.array(free, dtype=np.int32, copy=True)
        keys = np.empty(len(pods), dtype=np.uint64)
        G.gang_twin_place_batch(_p(topo), _p(f), _opt(mem), len(f), base, _p(pods), _p(gang), len(pods), _p(W), _p(keys, ctypes.c_uint64))
        return keys, f

    def preempt(topo, free, pods, lvl, hold, W, mem=None, base=0):
        topo, free, pods, lvl, W = (np.ascontiguousarray(a, dtype=np.int32) for a in (topo, free, pods, lvl, W))
        keys = np.empty(len(pods), dtype=np.uint64)
        vic = np.empty(len(pods), dtype=np.uint32)
        Pr.preempt_twin_batch(_p(topo), _p(free), _opt(mem), _opt(hold), len(free), base, _p(pods), _p(lvl), len(pods), _p(W),
                              os.cpu_count() or 1, _p(keys, ctypes.c_uint64), _p(vic, ctypes.c_uint32))
        return keys, vic
    return gang, preempt


def big_k_preempt_case(seed=0, N=12, P=60, mem=False):
    """A held cluster (C2's shapes, at most a few free GPUs per node) plus the edge node, fully held, and pods of 5..8 GPUs
    at levels 1..8: most of them can only run by evicting, and the k = 7 and 8 winners carry the table's largest costs
    through the preemption key."""
    rng = np.random.default_rng(seed)
    topo, _, _ = synth.gen_c2(N=N, P=0, seed=seed + 1)
    free = (rng.integers(0, 256, size=N) & rng.integers(0, 256, size=N) & rng.integers(0, 256, size=N)).astype(np.int32)
    topo = np.insert(topo, 1, edge_matrix(), axis=0)
    free = np.insert(free, 1, 0)
    hold = random_holders(rng, free, levels=6, untracked=0.05)
    hold[1] = [(1 << 3) | 0] * 4 + [(2 << 3) | 1] * 4                  # the edge node: two owners at levels 1 and 2
    pods = synth.make_pods(rng.integers(5, 9, size=P).astype(np.int32))
    pods[:4, 0] = [8, 7, 8, 7]
    lvl = rng.integers(1, 9, size=P).astype(np.int32)
    lvl[:4] = [3, 3, 15, 2]
    gm = None
    if mem:
        gm = synth.gen_gpu_memory(N + 1, seed=seed + 2)
        gm[1] = max(synth.GPU_MEM_CLASSES_MIB)
        pods[:, 3] = np.array(synth.POD_MIN_MEM_CHOICES_MIB, np.int32)[rng.integers(0, 7, size=P)]
        pods[:4, 3] = 0
    return topo, free, pods, lvl, hold, gm


# ---- CPU: the reference against Oracle B and the twins --------------------------------------------------------------------
@pytest.mark.parametrize("name", NAMES)
def test_reference_scoring_matches_oracle(oracle_b, name):
    W = W_of(name)
    topo, free, pods = synth.gen_c4(N=30, P=40, seed=71)
    pods[5, 0], pods[6, 0], pods[7, 0] = 0, 9, -1
    topo, free, pods, _ = with_edge(topo, free, pods)
    want = ref_score(topo, free, pods, W, base=2**32 - 40)
    assert (oracle_b.score_batch(topo, free, pods, W, node_id_base=2**32 - 40) == want).all()
    assert (oracle_b.score_batch(topo, free, pods, W, node_id_base=2**32 - 40, fast=True, nthreads=3) == want).all()
    assert (oracle_b.score_batch_memo(topo, free, pods, W, node_id_base=2**32 - 40, nthreads=2) == want).all()
    check_reached(name, want, topo, free)
    for n in range(len(free)):
        for k in range(-1, 10):
            assert oracle_b.node_key(topo[n], int(free[n]), k, W) == ref_node_key(topo[n], int(free[n]), k, W), (n, k)
    topo, free, mem, pods = synth.gen_c6(N=30, P=40, seed=72)
    topo, free, pods, mem = with_edge(topo, free, pods, mem)
    want = ref_score(topo, free, pods, W, mem=mem, base=3)
    assert (oracle_b.score_batch(topo, free, pods, W, node_id_base=3, mem=mem) == want).all()
    assert (oracle_b.score_batch(topo, free, pods, W, node_id_base=3, mem=mem, fast=True, nthreads=3) == want).all()
    check_reached(name, want)


@pytest.mark.parametrize("name", NAMES)
def test_reference_placement_matches_oracle_and_gang_twin(oracle_b, twins, name):
    W = W_of(name)
    topo, free, pods = synth.gen_c4(N=20, P=60, seed=73)
    pods[9, 0], pods[10, 0] = 0, 12
    topo, free, pods, _ = with_edge(topo, free, pods)
    want, wf = ref_place(topo, free, pods, W, base=7)
    for kw in (dict(plain=True), dict(tiled=True), {}):
        k, f = oracle_b.place_batch(topo, free, pods, W, node_id_base=7, **kw)
        assert (k == want).all() and (f == wf).all(), kw
    check_reached(name, want, topo, free)
    gang = random_gangs(len(pods), seed=11)
    want, wf = ref_place(topo, free, pods, W, gang=gang, base=7)
    k, f = twins[0](topo, free, pods, gang, W, base=7)
    assert (k == want).all() and (f == wf).all()
    assert any((want[a:e] == NO_FIT).all() for _, a, e in runs(gang)) and any((want[a:e] != NO_FIT).all() for _, a, e in runs(gang))
    topo, free, mem, pods = synth.gen_c6(N=20, P=60, seed=74)
    topo, free, pods, mem = with_edge(topo, free, pods, mem)
    want, wf = ref_place(topo, free, pods, W, mem=mem, base=2)
    k, f = oracle_b.place_batch(topo, free, pods, W, node_id_base=2, mem=mem)
    assert (k == want).all() and (f == wf).all()
    want, wf = ref_place(topo, free, pods, W, gang=gang, mem=mem, base=2)
    k, f = twins[0](topo, free, pods, gang, W, mem=mem, base=2)
    assert (k == want).all() and (f == wf).all()


@pytest.mark.parametrize("name", NAMES)
def test_reference_preemption_matches_twin(twins, name):
    W = W_of(name)
    for mem in (False, True):
        topo, free, pods, lvl, hold, gm = big_k_preempt_case(seed=3 + mem, N=8, P=30, mem=mem)
        pods[10, 0], pods[11, 0], lvl[12] = 0, 9, 0
        want = ref_preempt(topo, free, pods, lvl, hold, W, mem=gm, base=5)
        got = twins[1](topo, free, pods, lvl, hold, W, mem=gm, base=5)
        assert (got[0] == want[0]).all() and (got[1] == want[1]).all(), mem
        assert (want[1] != 0).any()
        check_reached(name, want[0])
    for case in (ties_case, min_mem_case, extreme_levels_case):
        topo, free, pods, lvl, hold, gm = case()
        want = ref_preempt(topo, free, pods, lvl, hold, W, mem=gm)
        got = twins[1](topo, free, pods, lvl, hold, W, mem=gm)
        assert (got[0] == want[0]).all() and (got[1] == want[1]).all(), case.__name__


def test_zero_table_is_the_tie_break(oracle_b):
    """Under the all-zero table every answer is the lowest node, then the lowest mask; for preemption the level and
    then |V| decide before those."""
    W = TABLES["zero"]
    topo, free, pods = synth.gen_c4(N=30, P=40, seed=75)
    keys = ref_score(topo, free, pods, W, base=4)
    assert (keys != NO_FIT).sum() > 20
    for key, k in zip(keys, pods[:, 0]):
        n = next((n for n in range(len(free)) if bin(int(free[n]) & 0xFF).count("1") >= k), None)
        if n is None:
            assert key == NO_FIT
            continue
        low = sorted(i for i in range(8) if (int(free[n]) >> i) & 1)[:k]
        assert int(key) == (4 + n) << 8 | sum(1 << i for i in low)
    topo, free, pods, lvl, hold, _ = ties_case()
    keys, vic = ref_preempt(topo, free, pods, lvl, hold, W)
    assert oracle_b.unpack_key(keys[0]) == (0, 0, 0x03) and vic[0] == 0b1


# ---- CPU: the kernel sources (tests/emu) against the twins ---------------------------------------------------------------
@pytest.fixture(scope="module")
def emu():
    """The kernels compiled for the CPU (tests/emu)."""
    return cpu_libs.emu()


def emu_score(fn, topo, free, pods, W, mem=None, base=0, splits=1):
    topo, free, pods, W = (np.ascontiguousarray(a, dtype=np.int32) for a in (topo, free, pods, W))
    keys = np.empty(len(pods), dtype=np.uint64)
    fn(_p(topo), _p(free), _opt(mem), len(free), base, _p(pods), len(pods), _p(W), splits, _p(keys, ctypes.c_uint64))
    return keys


@pytest.mark.parametrize("name", NAMES)
def test_emulated_sparse_and_dense(emu, oracle_b, name):
    """K1s (+ K1m) and the dense K1 (+ K1m): with and without memory, plain grids of 1 and 3 pod splits, node ids near
    the top of the 32-bit field, three chunks of pods."""
    W = W_of(name)
    topo, free, pods = synth.gen_c4(N=300, P=70, seed=76)
    pods[5, 0], pods[6, 0], pods[7, 0] = 0, 9, -3
    topo, free, pods, _ = with_edge(topo, free, pods, at=150)
    base = 2**32 - len(free) - 1
    want = oracle_b.score_batch(topo, free, pods, W, node_id_base=base)
    check_reached(name, want, topo, free)
    for fn in (emu.emu_score_sparse, emu.emu_score_dense):
        for splits in (1, 3):
            assert (emu_score(fn, topo, free, pods, W, base=base, splits=splits) == want).all(), (fn, splits)
    topo, free, mem, pods = synth.gen_c6(N=260, P=60, seed=77)
    topo, free, pods, mem = with_edge(topo, free, pods, mem, at=200)
    want = oracle_b.score_batch(topo, free, pods, W, node_id_base=9, mem=mem)
    check_reached(name, want[:4])
    for fn in (emu.emu_score_sparse, emu.emu_score_dense):
        for splits in (1, 3):
            assert (emu_score(fn, topo, free, pods, W, mem=mem, base=9, splits=splits) == want).all(), (fn, splits)
    topo, free, pods = synth.gen_c4(N=33, P=1100, seed=78)
    topo, free, pods, _ = with_edge(topo, free, pods)
    want = oracle_b.score_batch(topo, free, pods, W, node_id_base=2**31 - 40)
    assert (emu_score(emu.emu_score_sparse, topo, free, pods, W, base=2**31 - 40, splits=3) == want).all()


@pytest.mark.parametrize("name", NAMES)
def test_emulated_sparse_work_list(emu, oracle_b, name):
    """K1s on the work list, at the pod counts where the host switches instantiation (at most 64 pods: TMA, at most
    512: the prefetching one, above: the plain one), with work lists for 1, 16 and 1184 resident blocks (runs of
    several tiles per item when few blocks are resident); K1m alongside when pods carry min_mem."""
    W = W_of(name)
    topo, free, mem, pods = synth.gen_c6(N=500, P=513, seed=79)
    pods[5, 0], pods[6, 0] = 0, 9
    topo, free, pods, mem = with_edge(topo, free, pods, mem, at=300)
    for P, use_mem, residents in ((4, False, (1, 16)), (64, True, (1, 1184)), (512, False, (16, 1184)), (513, True, (1, 16, 1184))):
        pp = pods[:P].copy()
        if not use_mem:
            pp[:, 3] = 0
        want = oracle_b.score_batch(topo, free, pp, W, node_id_base=4, mem=mem)
        check_reached(name, want, topo, free)
        for resident in residents:
            got = emu_score(emu.emu_score_sparse, topo, free, pp, W, mem=mem, base=4, splits=-resident)
            assert (got == want).all(), (P, resident)


@pytest.mark.parametrize("name", NAMES)
def test_emulated_other_variants(emu, oracle_b, name):
    """Warp per pair (1), memo by k (3) and tile memo (4), with and without min_mem."""
    W = W_of(name)
    topo, free, mem, pods = synth.gen_c6(N=200, P=40, seed=80)
    pods[5, 0], pods[6, 0] = 0, 11
    topo, free, pods, mem = with_edge(topo, free, pods, mem, at=100)
    for use_mem in (False, True):
        pp = pods.copy()
        if not use_mem:
            pp[:, 3] = 0
        want = oracle_b.score_batch(topo, free, pp, W, node_id_base=77, mem=mem)
        check_reached(name, want, topo, free)
        for variant in (1, 3, 4):
            keys = np.empty(len(pp), dtype=np.uint64)
            emu.emu_score_variant(variant, _p(topo), _p(free), _p(mem), ctypes.c_int64(len(free)), ctypes.c_int64(77), _p(pp),
                                  ctypes.c_int64(len(pp)), _p(W), 2, _p(keys, ctypes.c_uint64))
            assert (keys == want).all(), (variant, use_mem)


@pytest.mark.parametrize("name", NAMES)
def test_emulated_pair_list_and_fit_nodes(emu, oracle_b, name):
    W = W_of(name)
    topo, free, mem, pods = synth.gen_c6(N=150, P=150, seed=81)
    topo, free, pods, mem = with_edge(topo, free, pods, mem, at=20)
    N = len(free)
    rng = np.random.default_rng(6)
    idx = rng.integers(0, N, size=300).astype(np.int64)
    idx[:4] = 20
    ks = np.concatenate([pods[:, 0], rng.integers(-1, 10, size=300 - len(pods))]).astype(np.int32)
    mm = np.concatenate([pods[:, 3], np.zeros(300 - len(pods), np.int32)]).astype(np.int32)
    out = np.empty(300, dtype=np.uint32)
    emu.emu_score_pair_list(_p(topo), _p(free), _p(mem), ctypes.c_int64(N), _p(idx, ctypes.c_longlong), _p(ks), _p(mm),
                            ctypes.c_int64(300), _p(W), _p(out, ctypes.c_uint32))
    want = [oracle_b.node_key(topo[i], int(free[i]) & _eligible(mem, i, int(m)), int(k), W) for i, k, m in zip(idx, ks, mm)]
    assert out.tolist() == want
    check_reached(name, _node_keys_as_keys(want), topo, free)
    out = np.empty(9 * N, dtype=np.uint32)
    emu.emu_fit_nodes(_p(topo), _p(free), ctypes.c_int64(N), None, ctypes.c_int64(N), _p(W), _p(out, ctypes.c_uint32))
    want = [oracle_b.node_key(topo[i], int(free[i]), k, W) for k in range(9) for i in range(N)]
    assert out.tolist() == want
    lst = np.array([N - 1, 20, 3], dtype=np.int32)
    out = np.empty(27, dtype=np.uint32)
    emu.emu_fit_nodes(_p(topo), _p(free), ctypes.c_int64(N), _p(lst), ctypes.c_int64(3), _p(W), _p(out, ctypes.c_uint32))
    assert out.tolist() == [oracle_b.node_key(topo[i], int(free[i]), k, W) for k in range(9) for i in lst]


def emu_place(emu, topo, free, pods, W, mem=None, base=0):
    f = np.array(free, dtype=np.int32, copy=True)
    topo, pods, W = (np.ascontiguousarray(a, dtype=np.int32) for a in (topo, pods, W))
    keys = np.empty(len(pods), dtype=np.uint64)
    rc = emu.emu_place_batch(_p(topo), _p(f), _opt(mem), ctypes.c_int64(len(f)), ctypes.c_int64(base), _p(pods),
                             ctypes.c_int64(len(pods)), _p(W), _p(keys, ctypes.c_uint64))
    assert rc == 0
    return keys, f


@pytest.mark.parametrize("name", NAMES)
def test_emulated_sequential_placement(emu, oracle_b, name):
    """K3 with five min_mem views, and on more than 32 tiles (several supertiles) on a cluster that fills up."""
    W = W_of(name)
    topo, free, mem, pods = synth.gen_c6(N=300, P=150, seed=82)
    topo, free, pods, mem = with_edge(topo, free, pods, mem, at=130)
    assert len(set(pods[:, 3].tolist())) == 5
    keys, f = emu_place(emu, topo, free, pods, W, mem=mem, base=9)
    want, wf = oracle_b.place_batch(topo, free, pods, W, node_id_base=9, mem=mem)
    assert (keys == want).all() and (f == wf).all()
    check_reached(name, want, topo, free)
    topo, free, _ = synth.gen_c2(N=128 * 34 + 17, P=0)
    free[:] = 0
    topo[4300] = edge_matrix()
    free[[5, 4300, 4368]] = [0x0F, 0xFF, 0xFF]           # three nodes with room, in different supertiles
    pods = synth.make_pods(np.array([8, 4, 4, 2, 7, 4, 2, 1, 1, 1, 1, 1], dtype=np.int32))
    keys, f = emu_place(emu, topo, free, pods, W)
    want, wf = oracle_b.place_batch(topo, free, pods, W)
    assert (keys == want).all() and (f == wf).all()
    assert (keys == NO_FIT).any()
    check_reached(name, want, topo, free)


def emu_gang(emu, topo, free, pods, gang, W, mem=None, base=0):
    f = np.array(free, dtype=np.int32, copy=True)
    topo, pods, gang, W = (np.ascontiguousarray(a, dtype=np.int32) for a in (topo, pods, gang, W))
    keys = np.empty(len(pods), dtype=np.uint64)
    assert emu.emu_place_batch_gang(_p(topo), _p(f), _opt(mem), len(f), base, _p(pods), _p(gang), len(pods), _p(W),
                                         _p(keys, ctypes.c_uint64)) == 0
    return keys, f


@pytest.mark.parametrize("name", NAMES)
def test_emulated_gang_placement(emu, twins, name):
    W = W_of(name)
    topo, free, mem, pods = synth.gen_c6(N=300, P=150)
    topo, free, pods, mem = with_edge(topo, free, pods, mem, at=40)
    gang = random_gangs(len(pods), seed=3)
    gang[:2] = 0                                          # the k = 8 and k = 7 pods on their own
    cases = [edge_batch(), chunk_batch(), (topo, free, pods, gang, mem)]
    for topo, free, pods, gang, mem in cases:
        keys, f = emu_gang(emu, topo, free, pods, gang, W, mem=mem, base=21)
        want, wf = twins[0](topo, free, pods, gang, W, mem=mem, base=21)
        assert (keys == want).all() and (f == wf).all()
        assert any((want[a:e] == NO_FIT).all() for _, a, e in runs(gang))
    check_reached(name, want, topo, free)


def emu_preempt(emu, oracle_b, topo, free, pods, lvl, hold, W, mem=None, base=0, splits=1):
    """The scoring path's keys from the oracle, then the emulated compaction, preemption kernel and finalisation."""
    topo, free, pods, lvl, W = (np.ascontiguousarray(a, dtype=np.int32) for a in (topo, free, pods, lvl, W))
    keys = oracle_b.score_batch(topo, free, pods, W, mem=mem, node_id_base=base)
    vic = np.empty(len(pods), dtype=np.uint32)
    reached = emu.emu_preempt_batch(_p(topo), _p(free), _opt(mem), _opt(hold), len(free), base, _p(pods), _p(lvl), len(pods),
                                            _p(W), splits, _p(keys, ctypes.c_uint64), _p(vic, ctypes.c_uint32))
    return keys, vic, reached


@pytest.mark.parametrize("name", NAMES)
def test_emulated_preemption(emu, oracle_b, twins, name):
    """K4 against the twin: evictions of 7 and 8 GPUs (the cost field's top bit), with and without min_mem, ties,
    level-0 pods, and several node tiles and pod chunks."""
    W = W_of(name)
    for mem in (False, True):
        topo, free, pods, lvl, hold, gm = big_k_preempt_case(seed=7 + mem, N=40, P=120, mem=mem)
        pods[10, 0], lvl[11] = 0, 0
        keys, vic, reached = emu_preempt(emu, oracle_b, topo, free, pods, lvl, hold, W, mem=gm, base=6)
        want = twins[1](topo, free, pods, lvl, hold, W, mem=gm, base=6)
        assert (keys == want[0]).all() and (vic == want[1]).all(), mem
        assert reached > 50 and (want[1] != 0).any()
        evicting = want[1] != 0
        check_reached(name, want[0][evicting])
    for case in (ties_case, min_mem_case, extreme_levels_case):
        topo, free, pods, lvl, hold, gm = case()
        keys, vic, _ = emu_preempt(emu, oracle_b, topo, free, pods, lvl, hold, W, mem=gm, base=3)
        want = twins[1](topo, free, pods, lvl, hold, W, mem=gm, base=3)
        assert (keys == want[0]).all() and (vic == want[1]).all(), case.__name__
    topo, free, pods, lvl, hold, _ = multi_block_case()
    want = twins[1](topo, free, pods, lvl, hold, W)
    for splits in (1, 2):
        keys, vic, reached = emu_preempt(emu, oracle_b, topo, free, pods, lvl, hold, W, splits=splits)
        assert reached > 2 * 256 and (keys == want[0]).all() and (vic == want[1]).all()


# ---- the device paths ----------------------------------------------------------------------------------------------
VARIANTS = [_lib.VARIANT_AUTO, _lib.VARIANT_LANE_PER_NODE, _lib.VARIANT_WARP_PER_PAIR, _lib.VARIANT_MEMO_BY_K, _lib.VARIANT_TILE_MEMO,
            _lib.VARIANT_SPARSE]
POD_COUNTS = (1, 64, 65, 512, 513, 3000)                  # K1s: TMA up to 64 pods, the prefetching build up to 512, plain above


@pytest.fixture(scope="module")
def scorer():
    from kubegpu_b200.scorer import Scorer
    s = Scorer((0,))
    yield s
    s.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_gpu_scoring(scorer, oracle_b, name):
    """Every variant at pod counts that reach each K1s instantiation, on C4's heterogeneous nodes and on C6 with its
    GPU memory uploaded (K1m, which K1s runs with the table's key layout)."""
    W = W_of(name)
    scorer.set_weights(W)
    assert (scorer.get_weights() == W).all()
    topo, free, pods = synth.gen_c4(N=3000, P=3000, seed=90)
    pods[5, 0], pods[6, 0] = 0, 9
    c4 = with_edge(topo, free, pods, at=2000)
    topo, free, mem, pods = synth.gen_c6(N=3000, P=3000, seed=91)
    c6 = with_edge(topo, free, pods, mem, at=1000)
    for topo, free, pods, mem in (c4, c6):
        scorer.upload_nodes(topo, free, node_id_base=13)
        if mem is not None:
            scorer.upload_gpu_memory(mem)
        want = oracle_b.score_batch(topo, free, pods, W, node_id_base=13, mem=mem, fast=True, nthreads=8)
        check_reached(name, want[:1], topo, free)
        for variant in VARIANTS:
            scorer.set_variant(variant)
            for P in POD_COUNTS:
                assert (scorer.score_batch(pods[:P]) == want[:P]).all(), (variant, P, mem is not None)
    scorer.set_variant(_lib.VARIANT_AUTO)


@pytest.mark.gpu
def test_gpu_c2_size_flat_max(scorer, oracle_b):
    """C2 (100k nodes, 10k pods) with every weight at 4095: the variants agree, an oracle-checked sample, k = 8 keys at
    the top of the cost field."""
    W = W_of("flat_max")
    topo, free, pods = synth.gen_c2()
    scorer.set_weights(W)
    scorer.upload_nodes(topo, free)
    outs = []
    for variant in (_lib.VARIANT_SPARSE, _lib.VARIANT_AUTO, _lib.VARIANT_LANE_PER_NODE):
        scorer.set_variant(variant)
        outs.append(scorer.score_batch(pods))
    assert all((o == outs[0]).all() for o in outs[1:])
    sample = np.arange(0, len(pods), 625)
    assert (outs[0][sample] == oracle_b.score_batch(topo, free, pods[sample], W, fast=True, nthreads=8)).all()
    assert all(cost_of(k) == 28 * 4095 for k in outs[0][pods[:, 0] == 8])
    scorer.set_variant(_lib.VARIANT_AUTO)
    scorer.upload_nodes(topo[:1], free[:1])


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_gpu_fit_table_and_pair_queries(scorer, oracle_b, name):
    W = W_of(name)
    topo, free, mem, pods = synth.gen_c6(N=3000, P=4, seed=92)
    topo, free, pods, mem = with_edge(topo, free, pods, mem, at=1500)
    N = len(free)
    scorer.set_weights(W)
    scorer.upload_nodes(topo, free)
    scorer.upload_gpu_memory(mem)
    scorer.build_fit_table()
    rng = np.random.default_rng(7)
    nodes = np.concatenate([[0, 1500, N - 1], rng.choice(N, size=120, replace=False)])
    for i in nodes:
        for k in range(-1, 10):
            assert scorer.fit_lookup(int(i), k) == oracle_b.node_key(topo[i], int(free[i]), k, W), (i, k)
    idx = rng.integers(0, N, size=2000).astype(np.int64)
    ks = rng.integers(-1, 10, size=2000).astype(np.int32)
    mm = np.array(synth.POD_MIN_MEM_CHOICES_MIB, np.int32)[rng.integers(0, 7, size=2000)]
    idx[:4], ks[:4], mm[:4] = 1500, [8, 7, 8, 7], [0, 0, 100_000, 40_000]
    got = scorer.score_pairs(idx, ks)
    want = [oracle_b.node_key(topo[i], int(free[i]), int(k), W) for i, k in zip(idx, ks)]
    assert got.tolist() == want
    check_reached(name, _node_keys_as_keys(want), topo, free)
    got = scorer.score_pairs(idx, ks, mm)
    want = [oracle_b.node_key(topo[i], int(free[i]) & _eligible(mem, i, int(m)), int(k), W) for i, k, m in zip(idx, ks, mm)]
    assert got.tolist() == want


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_gpu_placement(scorer, oracle_b, twins, name):
    """K3 with min_mem views, dry run and committed; gangs against the gang twin, free masks included."""
    W = W_of(name)
    scorer.set_weights(W)
    topo, free, mem, pods = synth.gen_c6(N=2000, P=800, seed=93)
    topo, free, pods, mem = with_edge(topo, free, pods, mem, at=1000)
    want, wf = oracle_b.place_batch(topo, free, pods, W, node_id_base=11, mem=mem)
    check_reached(name, want, topo, free)
    scorer.upload_nodes(topo, free, node_id_base=11)
    scorer.upload_gpu_memory(mem)
    assert (scorer.place_batch(pods, dry_run=True) == want).all() and (scorer.get_free_masks() == free).all()
    assert (scorer.place_batch(pods) == want).all() and (scorer.get_free_masks() == wf).all()
    topo, free, pods, gang = synth.gen_gangs(N=3000, P=1000)
    topo, free, pods, _ = with_edge(topo, free, pods, at=5)
    gang[:2] = 0
    want, wf = twins[0](topo, free, pods, gang, W)
    assert any((want[a:e] == NO_FIT).all() for _, a, e in runs(gang))
    scorer.upload_nodes(topo, free)
    assert (scorer.place_batch(pods, dry_run=True, gang=gang) == want).all() and (scorer.get_free_masks() == free).all()
    assert (scorer.place_batch(pods, gang=gang) == want).all() and (scorer.get_free_masks() == wf).all()


def preempt_cluster(N=3000, P=1000, mem=False):
    """gen_preempt plus the edge node, held by two owners at levels 1 and 2, and pods 0 and 1 asking for 8 and 7 GPUs at
    level 3 (they must evict)."""
    topo, free, hold, pods, lvl = synth.gen_preempt(N=N, P=P)
    topo = np.insert(topo, 7, edge_matrix(), axis=0)
    free = np.insert(free, 7, 0)
    hold = np.insert(hold, 7, [(1 << 3) | 0] * 4 + [(2 << 3) | 1] * 4, axis=0)
    pods[:2, 0], lvl[:2] = [8, 7], 3
    gm = None
    if mem:
        gm = synth.gen_gpu_memory(N + 1)
        gm[7] = max(synth.GPU_MEM_CLASSES_MIB)
        pods[:, 3] = np.array(synth.POD_MIN_MEM_CHOICES_MIB, np.int32)[synth.rand_below(synth.SEED_C6, 14, len(pods), 7)]
    return topo, free, hold, pods, lvl, gm


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_gpu_preemption(scorer, oracle_b, twins, name):
    """K4 against the twin with and without GPU memory; a level-0 batch equals score_batch."""
    W = W_of(name)
    scorer.set_weights(W)
    for use_mem in (False, True):
        topo, free, hold, pods, lvl, mem = preempt_cluster(mem=use_mem)
        want = twins[1](topo, free, pods, lvl, hold, W, mem=mem)
        scorer.upload_nodes(topo, free)
        if use_mem:
            scorer.upload_gpu_memory(mem)
        scorer.upload_holders(hold)
        keys, vic = scorer.preempt_batch(pods, lvl)
        assert (keys == want[0]).all() and (vic == want[1]).all(), use_mem
        check_reached(name, want[0][want[1] != 0])
        keys, vic = scorer.preempt_batch(pods, np.zeros(len(pods), np.int32))
        plain = oracle_b.score_batch(topo, free, pods, W, mem=mem, fast=True, nthreads=8)
        assert (keys == plain).all() and (keys == scorer.score_batch(pods)).all() and (vic == 0).all()


LIVE_ORDER = ["default", "general_edge", "byte_edge", "flat_max", "zero", "mixed", "byte_edge", "one_level", "random1",
              "general_edge", "random2", "byte_edge", "default"]


@pytest.mark.gpu
def test_gpu_weight_changes_on_a_live_handle(oracle_b, twins):
    """One upload, then table after table (across the byte-key boundary in both directions), with free-mask updates
    while the K1s cache is live and while it is dirty, fit-table builds, holder uploads and committed placements in
    between.  After every change: snapshot scoring (K1s and AUTO), the fit table, per-pair queries, a dry-run placement
    and preemption.  A rejected table leaves the previous one in effect.  The mask updates stay below the count that
    makes the next K1s launch re-sort the nodes (n / 200 since the last sort), and a re-sort rebuilds every record: so
    it is the table change itself that must invalidate the cached records."""
    from kubegpu_b200.scorer import KgpuError, Scorer
    assert any(max(TABLES[a]) <= 2340 < max(TABLES[b]) for a, b in zip(LIVE_ORDER, LIVE_ORDER[1:]))
    assert any(max(TABLES[a]) > 2340 >= max(TABLES[b]) for a, b in zip(LIVE_ORDER, LIVE_ORDER[1:]))
    EDGE = 1700
    topo, free, mem, pods = synth.gen_c6(N=12_000, P=300, seed=94)
    topo, free, pods, mem = with_edge(topo, free, pods, mem, at=EDGE)
    N = len(free)
    rng = np.random.default_rng(8)
    hold = random_holders(rng, free, levels=6)
    lvl = rng.integers(0, 8, size=len(pods)).astype(np.int32)
    others = np.delete(np.arange(N), EDGE)
    fm = free.copy()
    with Scorer((0,)) as s:
        s.upload_nodes(topo, fm, node_id_base=3)
        s.upload_gpu_memory(mem)
        s.upload_holders(hold)
        s.set_variant(_lib.VARIANT_SPARSE)
        for step, name in enumerate(LIVE_ORDER):
            W = W_of(name)
            s.score_batch(pods)                                      # the cache is live, built under the previous table
            upd = rng.choice(others, size=8, replace=False)
            fm[upd] = rng.integers(0, 256, size=8)
            s.set_free_masks(upd, fm[upd])                           # records refreshed in place
            s.set_weights(W)
            assert (s.get_weights() == W).all()
            upd = rng.choice(others, size=8, replace=False)
            fm[upd] = rng.integers(0, 256, size=8)
            s.set_free_masks(upd, fm[upd])                           # the cache is dirty now
            if step % 3 == 0:
                s.build_fit_table()
            elif step % 3 == 1:
                hold = random_holders(rng, fm, levels=6)
                s.upload_holders(hold)
            else:
                few = pods[200:230].copy()
                few[:, 0] = np.minimum(few[:, 0], 4)
                want, fm = oracle_b.place_batch(topo, fm, few, W, node_id_base=3, mem=mem)
                assert (s.place_batch(few) == want).all() and (s.get_free_masks() == fm).all()
            want = oracle_b.score_batch(topo, fm, pods, W, node_id_base=3, mem=mem, fast=True, nthreads=8)
            keys = s.score_batch(pods)
            assert (keys == want).all(), name
            check_reached(name, keys, topo, fm)
            s.set_variant(_lib.VARIANT_AUTO)
            assert (s.score_batch(pods) == want).all(), name
            s.set_variant(_lib.VARIANT_SPARSE)
            for i in np.concatenate([[EDGE], rng.choice(N, size=30, replace=False)]):
                for k in range(9):
                    assert s.fit_lookup(int(i), k) == oracle_b.node_key(topo[i], int(fm[i]), k, W), (name, i, k)
            idx = rng.integers(0, N, size=300).astype(np.int64)
            idx[:4] = EDGE
            ks, mm = pods[:300, 0], pods[:300, 3]
            assert s.score_pairs(idx, ks).tolist() == [oracle_b.node_key(topo[i], int(fm[i]), int(k), W) for i, k in zip(idx, ks)]
            assert s.score_pairs(idx, ks, mm).tolist() == [oracle_b.node_key(topo[i], int(fm[i]) & _eligible(mem, i, int(m)), int(k), W)
                                                           for i, k, m in zip(idx, ks, mm)]
            dry, _ = oracle_b.place_batch(topo, fm, pods[:200], W, node_id_base=3, mem=mem)
            assert (s.place_batch(pods[:200], dry_run=True) == dry).all() and (s.get_free_masks() == fm).all()
            pk, pv = s.preempt_batch(pods, lvl)
            tk, tv = twins[1](topo, fm, pods, lvl, hold, W, mem=mem, base=3)
            assert (pk == tk).all() and (pv == tv).all(), name
            for bad in ([4096] + [0] * 15, [0] * 15 + [-1]):
                with pytest.raises(KgpuError) as e:
                    s.set_weights(bad)
                assert e.value.code == _lib.ERR_INVALID
                assert (s.get_weights() == W).all()
            assert (s.score_batch(pods) == keys).all()
