"""Preemption plans with gangs (kgpu_preempt_plan_gang): a gang's members evict and take all together, or not at all.
CPU: the fast twin (tests/preempt_plan_gang_twin/plan_gang_twin.c) against a literal reference (single-pod
preempt_twin_batch calls, the update of the definition and an explicit save/restore undo), its properties (the deletion
property, failed gangs really miss, the equalities with preempt_plan_twin and with K3's gang twin), the emulated kernel
(tests/emu) against the twin on named cases, and the build products.  GPU: the device
path bit-exact against the twin on gen_preempt_gangs and C3's cluster, the deletion property and equalities on the
device, rejected batches, and a CLI transcript."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import cpu_libs
from kubegpu_b200 import _lib, synth
from test_preempt_plan import (NO_FIT, _W, _opt, _p, apply_update, big_k_case, check_properties, random_case, tiles_case,
                               views_32_case)
from test_preemption import _row, random_holders
from test_weight_tables import W_of

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


@pytest.fixture(scope="session")
def twins():
    """(snapshot, plan, gang_plan, k3_gang): the single-pod snapshot twin, preempt_plan_twin, preempt_plan_gang_twin and
    K3's gang twin (keys of dry-run gang placement)."""
    L, K3 = cpu_libs.twin("preempt_plan_gang"), cpu_libs.twin("gang")

    def prep(topo, free, pods, lvl):
        return (np.ascontiguousarray(a, dtype=np.int32) for a in (topo, free, pods, lvl))

    def plain(fn):
        def call(topo, free, pods, lvl, hold=None, mem=None, base=0, W=None):
            topo, free, pods, lvl = prep(topo, free, pods, lvl)
            keys, vic = np.empty(len(pods), np.uint64), np.empty(len(pods), np.uint32)
            fn(_p(topo), _p(free), _opt(mem), _opt(hold), len(free), base, _p(pods), _p(lvl), len(pods), _p(_W(W)),
               os.cpu_count() or 1, _p(keys, ctypes.c_uint64), _p(vic, ctypes.c_uint32))
            return keys, vic
        return call

    def gang_plan(topo, free, pods, lvl, gang, hold=None, mem=None, base=0, W=None):
        topo, free, pods, lvl = prep(topo, free, pods, lvl)
        keys, vic = np.empty(len(pods), np.uint64), np.empty(len(pods), np.uint32)
        L.preempt_plan_gang_twin(_p(topo), _p(free), _opt(mem), _opt(hold), len(free), base, _p(pods), _p(lvl), _opt(gang),
                                 len(pods), _p(_W(W)), os.cpu_count() or 1, _p(keys, ctypes.c_uint64), _p(vic, ctypes.c_uint32))
        return keys, vic

    def k3_gang(topo, free, pods, gang, mem=None, base=0):
        topo, free, pods, _ = prep(topo, free, pods, free)
        F = free.copy()
        keys = np.empty(len(pods), np.uint64)
        K3.gang_twin_place_batch(_p(topo), _p(F), _opt(mem), len(free), base, _p(pods), _opt(gang), len(pods), _p(_W(None)),
                                 _p(keys, ctypes.c_uint64))
        return keys

    return plain(L.preempt_twin_batch), plain(L.preempt_plan_twin), gang_plan, k3_gang


def gang_runs(gang):
    """[(first, end)] of every gang (nonzero id) in the batch."""
    runs, p = [], 0
    while p < len(gang):
        e = p + 1
        while e < len(gang) and gang[e] == gang[p]:
            e += 1
        if gang[p] != 0:
            runs.append((p, e))
        p = e
    return runs


def literal_gang_plan(snapshot, topo, free, pods, lvl, gang, hold=None, mem=None, base=0, W=None):
    """The definition, literally: per pod preempt_batch alone on (F, H) and the update; a gang's state is saved before its
    first member and restored when a member misses."""
    F = np.array(free, dtype=np.int32, copy=True)
    H = np.full((len(free), 8), -1, np.int32) if hold is None else np.array(hold, dtype=np.int32, copy=True)
    keys = np.full(len(pods), NO_FIT, np.uint64)
    vic = np.zeros(len(pods), np.uint32)
    p = 0
    while p < len(pods):
        e = p + 1
        while gang[p] != 0 and e < len(pods) and gang[e] == gang[p]:
            e += 1
        saved = (F.copy(), H.copy())
        for m in range(p, e):
            k, v = snapshot(topo, F, pods[m:m + 1], lvl[m:m + 1], hold=H, mem=mem, base=base, W=W)
            keys[m], vic[m] = k[0], v[0]
            if k[0] != NO_FIT:
                if pods[m, 0] > 0:
                    apply_update(F, H, k[0], v[0], base)
            elif gang[p] != 0:
                F, H = saved
                keys[p:e], vic[p:e] = NO_FIT, 0
                break
        p = e
    return keys, vic


def random_gangs(rng, P, start=0.3):
    """Random layouts: runs of 1..6 pods, about a third with a gang id."""
    gang = np.zeros(P, np.int32)
    p, gid = 0, 0
    while p < P:
        n = int(rng.integers(1, 7))
        if rng.random() < start:
            gid += 1
            gang[p:p + n] = gid
        p += n
    return gang


def failed_gangs(keys, gang, pods):
    """The gang runs whose members all got NO_FIT although some member was valid (a k = 0 member of a gang that stands
    would not be NO_FIT)."""
    return [(a, e) for a, e in gang_runs(gang) if (keys[a:e] == NO_FIT).all()]


def without(pods, lvl, gang, runs):
    keep = np.ones(len(pods), bool)
    for a, e in runs:
        keep[a:e] = False
    return pods[keep], lvl[keep], gang[keep], keep


# ---- the twin ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(8))
def test_twin_matches_literal_definition(twins, seed):
    snapshot, plan, gang_plan, _ = twins
    N = [7, 12, 25, 40][seed % 4]
    topo, free, pods, lvl, hold, mem = random_case(200 + seed, N=N, P=60, mem=seed % 2 == 1)
    gang = random_gangs(np.random.default_rng(seed), len(pods))
    want = literal_gang_plan(snapshot, topo, free, pods, lvl, gang, hold, mem=mem, base=5)
    got = gang_plan(topo, free, pods, lvl, gang, hold=hold, mem=mem, base=5)
    assert (got[0] == want[0]).all() and (got[1] == want[1]).all()
    check_properties(pods, *got)
    assert failed_gangs(got[0], gang, pods) and (got[1] != 0).sum() >= 2
    # invalid k inside gangs occurs in these cases
    assert any(((pods[a:e, 0] < 0) | (pods[a:e, 0] > 8)).any() for a, e in gang_runs(gang))


@pytest.mark.parametrize("seed", range(6))
def test_twin_properties(twins, seed):
    """Deletion property; each failed gang misses on the state its predecessors leave; all-zero ids and singleton gangs
    are preempt_plan_twin."""
    snapshot, plan, gang_plan, _ = twins
    topo, free, pods, lvl, hold, mem = random_case(300 + seed, N=25, P=80, mem=seed % 2 == 0)
    gang = random_gangs(np.random.default_rng(50 + seed), len(pods))
    keys, vic = gang_plan(topo, free, pods, lvl, gang, hold=hold, mem=mem)
    bad = failed_gangs(keys, gang, pods)
    assert bad
    dp, dl, _, keep = without(pods, lvl, gang, bad)
    k2, v2 = plan(topo, free, dp, dl, hold=hold, mem=mem)
    assert (k2 == keys[keep]).all() and (v2 == vic[keep]).all()
    for i, (a, e) in enumerate(bad):
        before = [r for r in bad[:i]]
        pp, pl, _, kp = without(pods[:e], lvl[:e], gang[:e], before)
        k3, _ = plan(topo, free, pp, pl, hold=hold, mem=mem)
        tail = k3[-(e - a):]
        assert (tail == NO_FIT).any() or ((pods[a:e, 0] < 0) | (pods[a:e, 0] > 8)).any()
    base = plan(topo, free, pods, lvl, hold=hold, mem=mem)
    for g in (np.zeros(len(pods), np.int32), np.arange(1, len(pods) + 1, dtype=np.int32), None):
        got = gang_plan(topo, free, pods, lvl, g, hold=hold, mem=mem)
        assert (got[0] == base[0]).all() and (got[1] == base[1]).all()


@pytest.mark.parametrize("mem", [False, True])
def test_twin_level_zero_is_k3_gangs(twins, mem):
    """No holder table, or every level 0: the keys of K3's gang twin and no victims."""
    _, _, gang_plan, k3_gang = twins
    topo, free, pods, gang = synth.gen_gangs(N=400, P=600)
    gm = synth.gen_gpu_memory(len(free), seed=3) if mem else None
    if mem:
        pods[:, 3] = np.array(synth.POD_MIN_MEM_CHOICES_MIB, np.int32)[np.random.default_rng(1).integers(0, 7, len(pods))]
    want = k3_gang(topo, free, pods, gang, mem=gm, base=3)
    assert failed_gangs(want, gang, pods)
    hold = random_holders(np.random.default_rng(1), free)
    keys, vic = gang_plan(topo, free, pods, np.zeros(len(pods), np.int32), gang, hold=hold, mem=gm, base=3)
    assert (keys == want).all() and (vic == 0).all()
    keys, vic = gang_plan(topo, free, pods, np.full(len(pods), 9, np.int32), gang, mem=gm, base=3)
    assert (keys == want).all() and (vic == 0).all()


# ---- named cases -------------------------------------------------------------------------------------------------------
def victim_reuse_case():
    """Two full nodes.  A level-3 gang {k=4, k=8}: the first member evicts a1 on A, the second fits nowhere, so the gang
    fails; a later level-3 pod then names a1 itself."""
    topo = np.stack([synth.shape_matrix([[4], [4]])] * 2)
    free = np.zeros(2, np.int32)
    hold = np.array([_row(*[(1, 0)] * 4, *[(2, 1)] * 4), _row(*[(2, 0)] * 4, *[(5, 1)] * 4)], np.int32)
    pods = synth.make_pods(np.array([4, 8, 4], np.int32))
    lvl = np.array([3, 3, 3], np.int32)
    gang = np.array([1, 1, 0], np.int32)
    return topo, free, pods, lvl, hold, None, gang


def same_node_case():
    """One node with four 2-GPU owners: a gang of three k = 2 members all lands on node 0 (the others are held at level
    15), the fourth member asks for 8 and misses; undoing in the right order restores node 0 exactly, so the next pods
    see the original owners."""
    topo = np.stack([synth.shape_matrix([[2, 2], [2, 2]])] * 2)
    free = np.zeros(2, np.int32)
    hold = np.array([_row((1, 0), (1, 0), (1, 1), (1, 1), (1, 2), (1, 2), (1, 3), (1, 3)), _row(*[(15, 0)] * 8)], np.int32)
    pods = synth.make_pods(np.array([2, 2, 2, 8, 2, 2, 2, 2], np.int32))
    lvl = np.array([2, 2, 2, 2, 2, 2, 2, 2], np.int32)
    gang = np.array([5, 5, 5, 5, 0, 0, 0, 0], np.int32)
    return topo, free, pods, lvl, hold, None, gang


def rescan_case():
    """130 nodes, two tiles.  Node 1 has GPUs 0, 1 free; node 0 none, with a level-1 owner of 6 GPUs.  A level-2 gang
    member with k = 4 evicts that owner and leaves GPUs 4, 5 free, so node 0 becomes the tile minimum of the level-0
    k = 2 column (same cost as node 1, lower node).  The next member (k = 8) misses; the undo raises node 0's key in that
    column again, so the tile must be rescanned: the next level-0 pod goes to node 1, not node 0."""
    N = 130
    topo = np.stack([synth.shape_matrix([[4], [4]])] * N)
    free = np.zeros(N, np.int32)
    free[1] = 0x03
    hold = np.array([_row(*[(1, 0)] * 6, *[(3, 1)] * 2)] + [_row(None, None, *[(3, 1)] * 6)] +
                    [_row(*[(3, 0)] * 8)] * (N - 2), np.int32)
    pods = synth.make_pods(np.array([4, 8, 2, 2], np.int32))
    lvl = np.array([2, 2, 0, 0], np.int32)
    gang = np.array([1, 1, 0, 0], np.int32)
    return topo, free, pods, lvl, hold, None, gang


def chunk_case():
    """tiles_case (1100 pods, three node tiles) with a gang across pod 1024 whose last member cannot fit."""
    topo, free, pods, lvl, hold, mem = tiles_case()
    gang = random_gangs(np.random.default_rng(8), len(pods))
    gang[gang > 0] += 1000
    gang[1018:1030] = 7
    pods[1018:1029, 0] = 2
    lvl[1018:1030] = 6
    pods[1029, 0] = 9                                      # k outside 0..8: the gang fails after 11 members
    return topo, free, pods, lvl, hold, mem, gang


CASES = {"victim_reuse": victim_reuse_case, "same_node": same_node_case, "rescan": rescan_case, "chunk": chunk_case}


def test_case_claims(twins):
    _, plan, gang_plan, _ = twins
    topo, free, pods, lvl, hold, _, gang = victim_reuse_case()
    blind = plan(topo, free, pods, lvl, hold=hold)
    assert blind[1][0] == 1 and blind[0][1] == NO_FIT and blind[0][2] != NO_FIT and blind[1][2] != 1
    keys, vic = gang_plan(topo, free, pods, lvl, gang, hold=hold)
    assert (keys[:2] == NO_FIT).all() and (vic[:2] == 0).all()
    assert (int(keys[2]) >> 8) & 0xFFFFFFFF == 0 and vic[2] == 1
    topo, free, pods, lvl, hold, _, gang = same_node_case()
    blind = plan(topo, free, pods, lvl, hold=hold)
    assert {(int(k) >> 8) & 0xFFFFFFFF for k in blind[0][:3]} == {0} and blind[0][3] == NO_FIT
    keys, vic = gang_plan(topo, free, pods, lvl, gang, hold=hold)
    assert (keys[:4] == NO_FIT).all() and list(vic[4:]) == [1, 2, 4, 8]
    topo, free, pods, lvl, hold, _, gang = rescan_case()
    blind = plan(topo, free, pods, lvl, hold=hold)
    assert (int(blind[0][0]) >> 8) & 0xFFFFFFFF == 0 and blind[1][0] == 1 and blind[0][1] == NO_FIT
    assert (int(blind[0][2]) >> 8) & 0xFFFFFFFF == 0 and blind[1][2] == 0              # the freed GPUs of node 0
    keys, vic = gang_plan(topo, free, pods, lvl, gang, hold=hold)
    assert (keys[:2] == NO_FIT).all() and (int(keys[2]) >> 8) & 0xFFFFFFFF == 1 and keys[3] == NO_FIT
    topo, free, pods, lvl, hold, _, gang = chunk_case()
    keys, vic = gang_plan(topo, free, pods, lvl, gang, hold=hold)
    blind = plan(topo, free, pods, lvl, hold=hold)
    assert (keys[1018:1030] == NO_FIT).all() and (blind[1][1018:1029] != 0).any() and (blind[0][1018:1024] != NO_FIT).all()


# ---- the kernel on the CPU (tests/emu) -------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu():
    return cpu_libs.emu()


def emu_gang_plan(emu, topo, free, pods, lvl, gang, hold, mem=None, base=0, W=None):
    topo, free, pods, lvl, gang = (np.ascontiguousarray(a, dtype=np.int32) for a in (topo, free, pods, lvl, gang))
    keys = np.empty(len(pods), dtype=np.uint64)
    vic = np.empty(len(pods), dtype=np.uint32)
    ncol = emu.emu_preempt_plan_gang(_p(topo), _p(free), _opt(mem), _opt(hold), len(free), base, _p(pods), _p(lvl), _p(gang),
                                     len(pods), _p(_W(W)), _p(keys, ctypes.c_uint64), _p(vic, ctypes.c_uint32))
    return keys, vic, ncol


@pytest.mark.parametrize("name", sorted(CASES))
def test_emulated_gang_plan_cases(emu, twins, name):
    topo, free, pods, lvl, hold, mem, gang = CASES[name]()
    keys, vic, _ = emu_gang_plan(emu, topo, free, pods, lvl, gang, hold, mem=mem, base=3)
    want = twins[2](topo, free, pods, lvl, gang, hold=hold, mem=mem, base=3)
    assert (keys == want[0]).all() and (vic == want[1]).all(), (keys, want[0], vic, want[1])
    assert failed_gangs(keys, gang, pods)


def test_emulated_gang_plan_32_views(emu, twins):
    topo, free, pods, lvl, hold, mem = views_32_case()
    gang = random_gangs(np.random.default_rng(4), len(pods), start=0.5)
    keys, vic, ncol = emu_gang_plan(emu, topo, free, pods, lvl, gang, hold, mem=mem)
    want = twins[2](topo, free, pods, lvl, gang, hold=hold, mem=mem)
    assert ncol > 32 and (keys == want[0]).all() and (vic == want[1]).all()


@pytest.mark.parametrize("table", ["flat_max", "general_edge"])
def test_emulated_gang_plan_weight_tables(emu, twins, table):
    W = W_of(table)
    topo, free, pods, lvl, hold, mem = big_k_case()
    gang = random_gangs(np.random.default_rng(6), len(pods), start=0.6)
    keys, vic, _ = emu_gang_plan(emu, topo, free, pods, lvl, gang, hold, W=W)
    want = twins[2](topo, free, pods, lvl, gang, hold=hold, W=W)
    lit = literal_gang_plan(twins[0], topo, free, pods, lvl, gang, hold, W=W)
    assert (keys == want[0]).all() and (vic == want[1]).all()
    assert (lit[0] == want[0]).all() and (lit[1] == want[1]).all()


@pytest.mark.parametrize("seed", range(4))
def test_emulated_gang_plan_random(emu, twins, seed):
    topo, free, pods, lvl, hold, mem = random_case(400 + seed, N=40, P=120, mem=seed % 2 == 0)
    gang = random_gangs(np.random.default_rng(seed), len(pods))
    keys, vic, _ = emu_gang_plan(emu, topo, free, pods, lvl, gang, hold, mem=mem, base=seed)
    want = twins[2](topo, free, pods, lvl, gang, hold=hold, mem=mem, base=seed)
    assert (keys == want[0]).all() and (vic == want[1]).all()


# ---- build products ----------------------------------------------------------------------------------------------------
def test_gang_plan_kernel_has_no_local_memory():
    if shutil.which("cuobjdump") is None or not os.path.exists(_lib.LIB_PATH):
        pytest.skip("cuobjdump or libkgpu.so missing")
    out = subprocess.run(["cuobjdump", "-res-usage", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    lines = out.splitlines()
    found = 0
    for i, line in enumerate(lines):
        if re.search(r"Function _ZN4kgpu\d+gang_plan_sequential\w*:", line):
            found += 1
            assert re.search(r"STACK:0\b", lines[i + 1]) and re.search(r"LOCAL:0\b", lines[i + 1]), lines[i + 1]
    assert found == 1


def test_gang_plan_entry_point_allocates_only_through_buffers():
    src = open(os.path.join(ROOT, "kubegpu_b200", "csrc", "kgpu.cu")).read()
    body = src.split("int kgpu_preempt_plan_gang(", 1)[1].split("\nint kgpu_", 1)[0]
    assert "d_plan_pre.reserve(" in body and not re.search(r"cuda(Malloc|Free)\w*\s*\(", body)


# ---- the device path ---------------------------------------------------------------------------------------------------
def _evicted_before_miss(plan, topo, free, hold, pods, lvl, gang, bad, mem, enough):
    """How many failed gangs had a member given victims before the miss, on the state the kept pods before them leave."""
    found = 0
    for i, (a, e) in enumerate(bad):
        pp, pl, _, _ = without(pods[:e], lvl[:e], gang[:e], bad[:i])
        k, v = plan(topo, free, pp, pl, hold=hold, mem=mem)
        k, v = k[-(e - a):], v[-(e - a):]
        miss = int(np.flatnonzero(k == NO_FIT)[0]) if (k == NO_FIT).any() else e - a
        found += bool((v[:miss] != 0).any())
        if found >= enough:
            break
    return found


@pytest.mark.gpu
@pytest.mark.parametrize("use_mem", [False, True])
def test_gang_plan_gen_preempt_gangs(twins, use_mem):
    """gen_preempt_gangs (20k nodes, 10k pods), with and without C6's per-GPU memory: bit-exact against the twin, the
    handle's state untouched, the deletion property on the device."""
    from kubegpu_b200.scorer import Scorer
    _, plan, gang_plan, _ = twins
    topo, free, hold, pods, lvl, gang = synth.gen_preempt_gangs()
    mem = None
    if use_mem:
        mem = synth.gen_gpu_memory(len(free))
        pods[:, 3] = np.array(synth.POD_MIN_MEM_CHOICES_MIB, np.int32)[synth.rand_below(synth.SEED_C6, 14, len(pods), 7)]
    want_k, want_v = gang_plan(topo, free, pods, lvl, gang, hold=hold, mem=mem)
    bad = failed_gangs(want_k, gang, pods)
    dp, dl, _, keep = without(pods, lvl, gang, bad)
    with Scorer((0,)) as s:
        s.upload_nodes(topo, free)
        if use_mem:
            s.upload_gpu_memory(mem)
        s.upload_holders(hold)
        snap_before = s.preempt_batch(pods, lvl)
        keys, vic = s.preempt_plan(pods, lvl, gang=gang)
        assert (keys == want_k).all() and (vic == want_v).all()
        assert (s.get_free_masks() == free).all()
        snap_after = s.preempt_batch(pods, lvl)
        assert (snap_after[0] == snap_before[0]).all() and (snap_after[1] == snap_before[1]).all()
        k2, v2 = s.preempt_plan(dp, dl)                                            # the deletion property
        assert (k2 == keys[keep]).all() and (v2 == vic[keep]).all()
    check_properties(pods, keys, vic)
    assert (vic != 0).sum() >= 1000
    assert _evicted_before_miss(plan, topo, free, hold, pods, lvl, gang, bad, mem, 10) >= 10


@pytest.mark.gpu
def test_gang_plan_equalities():
    """gang=None, all-zero ids and singleton gangs are preempt_plan; with no holder table or every level 0 the keys are
    place_batch(dry_run=True, gang=gang) with victims 0, on gen_gangs and on C6 with gangs."""
    from kubegpu_b200.scorer import Scorer
    topo, free, hold, pods, lvl, gang = synth.gen_preempt_gangs(N=5000, P=2000)
    with Scorer((0,)) as s:
        s.upload_nodes(topo, free, node_id_base=7)
        s.upload_holders(hold)
        want = s.preempt_plan(pods, lvl)
        for g in (None, np.zeros(len(pods), np.int32), np.arange(1, len(pods) + 1, dtype=np.int32)):
            got = s.preempt_plan(pods, lvl, gang=g)
            assert (got[0] == want[0]).all() and (got[1] == want[1]).all()
    for name in ("gangs", "c6"):
        topo, free, pods, gang = synth.gen_gangs()
        mem = None
        if name == "c6":
            topo, free, mem, pods = synth.gen_c6()
            gang = random_gangs(np.random.default_rng(9), len(pods))
        with Scorer((0,)) as s:
            s.upload_nodes(topo, free)
            if mem is not None:
                s.upload_gpu_memory(mem)
            want = s.place_batch(pods, dry_run=True, gang=gang)
            assert failed_gangs(want, gang, pods) or name == "c6"
            keys, vic = s.preempt_plan(pods, np.full(len(pods), 5, np.int32), gang=gang)          # no holder table
            assert (keys == want).all() and (vic == 0).all()
            s.upload_holders(random_holders(np.random.default_rng(2), free))
            keys, vic = s.preempt_plan(pods, np.zeros(len(pods), np.int32), gang=gang)            # every level 0
            assert (keys == want).all() and (vic == 0).all()


@pytest.mark.gpu
def test_gang_plan_c3_cluster(twins):
    """C3's 1M-node cluster with a small gang batch, against the twin."""
    from kubegpu_b200.scorer import Scorer
    topo, free, pods = synth.gen_c3(P=96)
    rng = np.random.default_rng(4)
    hold = random_holders(rng, free, levels=4)
    lvl = rng.choice(np.array([0, 2, 5], np.int32), size=len(pods))
    gang = random_gangs(rng, len(pods), start=0.5)
    want = twins[2](topo, free, pods, lvl, gang, hold=hold, base=11)
    with Scorer((0,)) as s:
        s.upload_nodes(topo, free, node_id_base=11)
        s.upload_holders(hold)
        keys, vic = s.preempt_plan(pods, lvl, gang=gang)
    assert (keys == want[0]).all() and (vic == want[1]).all()


@pytest.mark.gpu
def test_gang_plan_rejected_batches():
    """A split gang id, lvl out of range, 8 min_mem values and 33 (level, min_mem) pairs are KGPU_ERR_INVALID; the state
    and the next answer stay."""
    from kubegpu_b200.scorer import KgpuError, Scorer
    topo, free, hold, pods, lvl, gang = synth.gen_preempt_gangs(N=5000, P=200)
    split = gang.copy()
    split[-1] = split[np.flatnonzero(split)[0]]
    split[-2] = 0
    many_mem = pods.copy()
    many_mem[:8, 3] = np.arange(1, 9) * 1000
    many_views = pods.copy()
    many_views[:, 3] = 0
    views_lvl = lvl.copy()
    views_lvl[:33] = np.tile(np.arange(1, 12), 3)
    many_views[:33, 3] = np.repeat(np.array([0, 1000, 2000]), 11)
    with Scorer((0,)) as s:
        s.upload_nodes(topo, free)
        s.upload_holders(hold)
        want = s.preempt_plan(pods, lvl, gang=gang)
        for bad_pods, bad_lvl, bad_gang in ((pods, lvl, split), (pods, np.where(np.arange(len(lvl)) == 5, 16, lvl), gang),
                                            (many_mem, lvl, gang), (many_views, views_lvl, gang)):
            with pytest.raises(KgpuError) as e:
                s.preempt_plan(bad_pods, bad_lvl, gang=bad_gang)
            assert e.value.code == _lib.ERR_INVALID
        assert (s.get_free_masks() == free).all()
        got = s.preempt_plan(pods, lvl, gang=gang)
        assert (got[0] == want[0]).all() and (got[1] == want[1]).all()


@pytest.mark.gpu
def test_gang_plan_two_devices_is_a_state_error():
    import torch
    from kubegpu_b200.scorer import KgpuError, Scorer
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    topo, free, hold, pods, lvl, gang = synth.gen_preempt_gangs(N=1000, P=10)
    with Scorer((0, 1)) as s:
        s.upload_nodes(topo, free)
        with pytest.raises(KgpuError) as e:
            s.preempt_plan(pods, lvl, gang=gang)
        assert e.value.code == _lib.ERR_STATE


@pytest.mark.gpu
def test_host_mirror_gang_plan():
    """sched_cli on a full two-node cluster: a two-member high-priority gang whose second member cannot fit.
    preemptplan (gang-blind) gives the first member a victim; preemptgangplan gives both members fits=0 and no victims,
    and a later pod of the same command gets that victim instead."""
    from test_preemption import CLI, _node_line
    if not os.path.exists(CLI):
        subprocess.check_call(["make", "-s", "-C", ROOT, "kubegpu_b200/lib/kgpu_sched_cli"])
    ids = ["GPU-%02d" % i for i in range(8)]
    lines = [_node_line("A", [[4], [4]], ids), _node_line("B", [[4], [4]], ids),
             "pod a1 priority=1 run c req=4", "pod a2 priority=5 run c req=4",
             "pod b1 priority=5 run c req=4", "pod b2 priority=5 run c req=4",
             "pod g1 priority=3 gang=7 run c req=4", "pod g2 priority=3 gang=7 run c req=8",
             "pod h1 priority=3 run c req=4",
             "placebatch a1 a2 b1 b2",
             "preemptplan g1 g2 h1",
             "preemptgangplan g1 g2 h1"]
    got = subprocess.run([CLI], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True).stdout
    blind = got.split("> preemptplan g1 g2 h1\n")[1].splitlines()
    gang = got.split("> preemptgangplan g1 g2 h1\n")[1].splitlines()
    assert blind[0] == "  err=" and gang[0] == "  err="
    assert " fits=1 " in blind[1] and blind[1].endswith("victims=a1") and " fits=0 " in blind[2] and " fits=0 " in blind[3]
    assert " fits=0 " in gang[1] and gang[1].endswith("victims=") and " fits=0 " in gang[2] and gang[2].endswith("victims=")
    assert gang[3].startswith("  h1 fits=1 ") and " node=A " in gang[3] and gang[3].endswith("victims=a1")
