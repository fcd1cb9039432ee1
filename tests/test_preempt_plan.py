"""Preemption plans (kgpu_preempt_plan): pods in order, each evicting only victims no earlier pod has claimed.
CPU: a literal reference (a loop of single-pod preempt_twin_batch calls plus the update of the definition) against the
fast sequential twin (tests/preempt_plan_twin/plan_twin.c), the properties of the definition, the emulated kernels
(tests/emu) against the twin, and the kernels' resource usage.  GPU: the device path bit-exact
against the twin on gen_preempt at C2's size and on C3's cluster, the equalities with preempt_batch and dry-run
placement, rejected batches, and the handle's state left alone."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import cpu_libs
from kubegpu_b200 import _lib, synth
from test_preemption import _row, random_holders
from test_weight_tables import TABLES, W_of, edge_matrix

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
NO_FIT = np.uint64(0xFFFFFFFFFFFFFFFF)


def _p(a, t=ctypes.c_int32):
    return a.ctypes.data_as(ctypes.POINTER(t))


def _opt(a):
    return None if a is None else _p(np.ascontiguousarray(a, dtype=np.int32))


def _W(W):
    from oracle import oracle_b
    return np.ascontiguousarray(oracle_b.DEFAULT_WEIGHTS if W is None else W, dtype=np.int32)


@pytest.fixture(scope="session")
def twins():
    """(snapshot, plan): both (topo, free, pods, lvl, hold=None, mem=None, base=0, W=None) -> (keys, victims)."""
    L = cpu_libs.twin("preempt_plan")

    def wrap(fn):
        def call(topo, free, pods, lvl, hold=None, mem=None, base=0, W=None):
            topo, free, pods, lvl = (np.ascontiguousarray(a, dtype=np.int32) for a in (topo, free, pods, lvl))
            keys = np.empty(len(pods), dtype=np.uint64)
            vic = np.empty(len(pods), dtype=np.uint32)
            fn(_p(topo), _p(free), _opt(mem), _opt(hold), len(free), base, _p(pods), _p(lvl), len(pods), _p(_W(W)),
               os.cpu_count() or 1, _p(keys, ctypes.c_uint64), _p(vic, ctypes.c_uint32))
            return keys, vic
        return call
    return wrap(L.preempt_twin_batch), wrap(L.preempt_plan_twin)


def apply_update(F, H, key, vic, base):
    """The definition's update after a pod that fits on node n with mask S and victims vic."""
    n, S = ((int(key) >> 8) & 0xFFFFFFFF) - base, int(key) & 0xFF
    R = sum(1 << g for g in range(8) if not (F[n] >> g) & 1 and H[n, g] >= 0 and (int(vic) >> (H[n, g] & 7)) & 1)
    F[n] = (int(F[n]) | R) & ~S & 0xFF
    for g in range(8):
        if ((S | R) >> g) & 1:
            H[n, g] = -1
    return n, S


def literal_plan(snapshot, topo, free, pods, lvl, hold=None, mem=None, base=0, W=None):
    """The definition, literally: per pod, preempt_batch alone on (F, H), then the update."""
    F = np.array(free, dtype=np.int32, copy=True)
    H = np.full((len(free), 8), -1, np.int32) if hold is None else np.array(hold, dtype=np.int32, copy=True)
    keys = np.empty(len(pods), np.uint64)
    vic = np.empty(len(pods), np.uint32)
    for p in range(len(pods)):
        k, v = snapshot(topo, F, pods[p:p + 1], lvl[p:p + 1], hold=H, mem=mem, base=base, W=W)
        keys[p], vic[p] = k[0], v[0]
        if k[0] != NO_FIT:
            apply_update(F, H, k[0], v[0], base)
    return keys, vic


def check_properties(pods, keys, vic, base=0):
    """Victim sets of pods on one node are disjoint, and so are their GPU sets."""
    seen_v, seen_g = {}, {}
    for p in range(len(pods)):
        if keys[p] == NO_FIT or pods[p, 0] == 0:
            continue
        n = (int(keys[p]) >> 8) & 0xFFFFFFFF
        S = int(keys[p]) & 0xFF
        assert not seen_v.get(n, 0) & int(vic[p]), ("shared victim", p)
        assert not seen_g.get(n, 0) & S, ("shared GPU", p)
        seen_v[n] = seen_v.get(n, 0) | int(vic[p])
        seen_g[n] = seen_g.get(n, 0) | S


def random_case(seed, N=7, P=40, mem=False):
    """7..40 nodes, levels 0..15, k from -1 to 9, owners spanning several GPUs, entries on free GPUs, level-15 holders."""
    rng = np.random.default_rng(seed)
    topo, _, _ = synth.gen_c4(N=N, P=0, seed=seed + 1)
    free = (rng.integers(0, 256, size=N) & rng.integers(0, 256, size=N) & rng.integers(0, 256, size=N)).astype(np.int32)
    hold = random_holders(rng, free, owners=4)
    hold[0] = [15 << 3 | 1] * 8
    pods = synth.make_pods(rng.integers(-1, 10, size=P).astype(np.int32))
    lvl = rng.integers(0, 16, size=P).astype(np.int32)
    gm = None
    if mem:
        gm = synth.gen_gpu_memory(N, seed=seed + 2)
        pods[:, 3] = np.array(synth.POD_MIN_MEM_CHOICES_MIB, np.int32)[rng.integers(0, 7, size=P)]
    return topo, free, pods, lvl, hold, gm


# ---- the twin against the literal definition ---------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(8))
def test_twin_matches_literal_definition(twins, seed):
    snapshot, plan = twins
    N = [7, 12, 25, 40][seed % 4]
    topo, free, pods, lvl, hold, mem = random_case(seed, N=N, P=60, mem=seed % 2 == 1)
    want = literal_plan(snapshot, topo, free, pods, lvl, hold, mem=mem, base=5)
    got = plan(topo, free, pods, lvl, hold=hold, mem=mem, base=5)
    assert (got[0] == want[0]).all() and (got[1] == want[1]).all()
    check_properties(pods, *got)
    assert (got[1] != 0).sum() >= 2 and (got[0] == NO_FIT).any()
    # P = 1 is the snapshot
    for p in range(0, len(pods), 7):
        one = plan(topo, free, pods[p:p + 1], lvl[p:p + 1], hold=hold, mem=mem, base=5)
        snap = snapshot(topo, free, pods[p:p + 1], lvl[p:p + 1], hold=hold, mem=mem, base=5)
        assert one[0][0] == snap[0][0] and one[1][0] == snap[1][0]


@pytest.mark.parametrize("mem", [False, True])
def test_twin_level_zero_is_sequential_placement(twins, oracle_b, mem):
    """Every lvl 0, or no holder table: Oracle B's sequential placement and no victims."""
    _, plan = twins
    topo, free, gm, pods = synth.gen_c6(N=300, P=400)
    gm = gm if mem else None
    if not mem:
        pods[:, 3] = 0
    want, _ = oracle_b.place_batch(topo, free, pods, mem=gm, node_id_base=3, plain=True)
    hold = random_holders(np.random.default_rng(1), free)
    keys, vic = plan(topo, free, pods, np.zeros(len(pods), np.int32), hold=hold, mem=gm, base=3)
    assert (keys == want).all() and (vic == 0).all()
    keys, vic = plan(topo, free, pods, np.full(len(pods), 9, np.int32), mem=gm, base=3)
    assert (keys == want).all() and (vic == 0).all()


# ---- hand-made cases ----------------------------------------------------------------------------------------------------
def ties_case():
    """Identical nodes and owners: ties on class, cost and node go to the lower node, then the lower mask."""
    m = synth.shape_matrix([[2, 2], [2, 2]])
    topo = np.stack([m] * 4)
    free = np.zeros(4, np.int32)
    row = _row((1, 0), (1, 0), (1, 1), (1, 1), (1, 2), (1, 2), (1, 3), (1, 3))
    hold = np.array([row] * 4, np.int32)
    pods = synth.make_pods(np.array([2, 2, 2, 2, 2, 4, 4, 1], np.int32))
    lvl = np.array([2, 2, 2, 2, 2, 3, 3, 2], np.int32)
    return topo, free, pods, lvl, hold, None


def freed_gpus_case():
    """A level-3 pod evicts a 4-GPU owner for 2 GPUs; the next level-0 pods use the other 2 without evicting."""
    topo = np.stack([synth.shape_matrix([[4], [4]])] * 2)
    free = np.zeros(2, np.int32)
    hold = np.array([_row(*[(1, 0)] * 4, *[(2, 1)] * 4), _row(*[(2, 0)] * 8)], np.int32)
    pods = synth.make_pods(np.array([2, 1, 1, 1], np.int32))
    lvl = np.array([3, 0, 0, 0], np.int32)
    return topo, free, pods, lvl, hold, None


def no_batch_victims_case():
    """A later level-15 pod must not evict the GPUs an earlier level-1 pod of the batch took."""
    topo = np.stack([synth.shape_matrix([[8]])] * 2)
    free = np.array([0xFF, 0x00], np.int32)
    hold = np.array([_row(*[None] * 8), _row(*[(14, 0)] * 8)], np.int32)
    pods = synth.make_pods(np.array([8, 8, 8], np.int32))
    lvl = np.array([1, 15, 15], np.int32)
    return topo, free, pods, lvl, hold, None


def tiles_case(N=300, P=1100):
    """Three node tiles and more pods than one staging chunk (1024)."""
    rng = np.random.default_rng(11)
    topo, _, _ = synth.gen_c4(N=N, P=0, seed=77)
    free = (rng.integers(0, 256, size=N) & rng.integers(0, 256, size=N) & rng.integers(0, 256, size=N)).astype(np.int32)
    hold = random_holders(rng, free, levels=6)
    pods = synth.make_pods(np.array([1, 2, 3, 5, 8], np.int32)[rng.integers(0, 5, size=P)])
    lvl = rng.integers(0, 8, size=P).astype(np.int32)
    return topo, free, pods, lvl, hold, None


def views_32_case():
    """Exactly 32 (level > 0, min_mem) views: levels 1..8 x 4 memory needs, plus level-0 pods."""
    rng = np.random.default_rng(3)
    N, P = 40, 120
    topo, _, _ = synth.gen_c4(N=N, P=0, seed=5)
    free = (rng.integers(0, 256, size=N) & rng.integers(0, 256, size=N)).astype(np.int32)
    hold = random_holders(rng, free, levels=8)
    mem = synth.gen_gpu_memory(N, seed=9)
    pods = synth.make_pods(rng.integers(1, 9, size=P).astype(np.int32))
    lvl = np.concatenate([np.repeat(np.arange(1, 9), 4), rng.integers(0, 9, size=P - 32)]).astype(np.int32)
    needs = np.array([0, 8_000, 20_000, 40_000], np.int32)
    pods[:, 3] = np.concatenate([np.tile(needs, 8), needs[rng.integers(0, 4, size=P - 32)]])
    return topo, free, pods, lvl, hold, mem


def big_k_case(seed=0, N=12, P=60):
    """C2's shapes, mostly held, plus an 'edge' node with every pair at one link level, fully held: k = 7 and 8 winners
    carry the table's largest costs through the key."""
    rng = np.random.default_rng(seed)
    topo, _, _ = synth.gen_c2(N=N, P=0, seed=seed + 1)
    free = (rng.integers(0, 256, size=N) & rng.integers(0, 256, size=N) & rng.integers(0, 256, size=N)).astype(np.int32)
    topo = np.insert(topo, 1, edge_matrix(), axis=0)
    free = np.insert(free, 1, 0)
    hold = random_holders(rng, free, levels=6, untracked=0.05)
    hold[1] = [(1 << 3) | 0] * 4 + [(2 << 3) | 1] * 4
    pods = synth.make_pods(rng.integers(5, 9, size=P).astype(np.int32))
    pods[:4, 0] = [8, 7, 8, 7]
    lvl = rng.integers(1, 9, size=P).astype(np.int32)
    lvl[:4] = [3, 3, 15, 2]
    return topo, free, pods, lvl, hold, None


CASES = {"ties": ties_case, "freed_gpus": freed_gpus_case, "no_batch_victims": no_batch_victims_case}


def test_case_claims(twins):
    _, plan = twins
    topo, free, pods, lvl, hold, _ = ties_case()
    keys, vic = plan(topo, free, pods, lvl, hold=hold)
    nodes = [(int(k) >> 8) & 0xFFFFFFFF for k in keys[:5]]
    assert nodes == [0, 0, 0, 0, 1] and [int(k) & 0xFF for k in keys[:4]] == [0x03, 0x0C, 0x30, 0xC0]
    assert list(vic[:5]) == [1, 2, 4, 8, 1]
    topo, free, pods, lvl, hold, _ = freed_gpus_case()
    keys, vic = plan(topo, free, pods, lvl, hold=hold)
    assert vic[0] == 1 and int(keys[0]) & 0xFF == 0x03 and (vic[1:] == 0).all()
    assert [int(k) & 0xFFFFFFFFFF for k in keys[1:3]] == [0x04, 0x08] and keys[3] == NO_FIT
    topo, free, pods, lvl, hold, _ = no_batch_victims_case()
    keys, vic = plan(topo, free, pods, lvl, hold=hold)
    assert (int(keys[0]) >> 8) & 0xFFFFFFFF == 0 and vic[0] == 0
    assert (int(keys[1]) >> 8) & 0xFFFFFFFF == 1 and vic[1] == 1 and keys[2] == NO_FIT


# ---- the kernels on the CPU (tests/emu) -------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu():
    return cpu_libs.emu()


def emu_plan(emu, topo, free, pods, lvl, hold, mem=None, base=0, W=None):
    topo, free, pods, lvl = (np.ascontiguousarray(a, dtype=np.int32) for a in (topo, free, pods, lvl))
    keys = np.empty(len(pods), dtype=np.uint64)
    vic = np.empty(len(pods), dtype=np.uint32)
    ncol = emu.emu_preempt_plan(_p(topo), _p(free), _opt(mem), _opt(hold), len(free), base, _p(pods), _p(lvl), len(pods),
                                _p(_W(W)), _p(keys, ctypes.c_uint64), _p(vic, ctypes.c_uint32))
    return keys, vic, ncol


@pytest.mark.parametrize("name", sorted(CASES))
def test_emulated_plan_cases(emu, twins, name):
    topo, free, pods, lvl, hold, mem = CASES[name]()
    keys, vic, _ = emu_plan(emu, topo, free, pods, lvl, hold, mem=mem, base=3)
    want = twins[1](topo, free, pods, lvl, hold=hold, mem=mem, base=3)
    assert (keys == want[0]).all() and (vic == want[1]).all(), (keys, want[0], vic, want[1])


def test_emulated_plan_several_tiles_and_chunks(emu, twins):
    topo, free, pods, lvl, hold, mem = tiles_case()
    keys, vic, _ = emu_plan(emu, topo, free, pods, lvl, hold, base=2)
    want = twins[1](topo, free, pods, lvl, hold=hold, base=2)
    assert (keys == want[0]).all() and (vic == want[1]).all()
    assert (vic != 0).sum() > 50 and len(pods) > 1024


def test_emulated_plan_32_views(emu, twins):
    topo, free, pods, lvl, hold, mem = views_32_case()
    views = {(int(l), int(m)) for l, m in zip(lvl, pods[:, 3]) if l > 0}
    assert len(views) == 32
    keys, vic, ncol = emu_plan(emu, topo, free, pods, lvl, hold, mem=mem)
    want = twins[1](topo, free, pods, lvl, hold=hold, mem=mem)
    assert ncol > 32 and (keys == want[0]).all() and (vic == want[1]).all()


@pytest.mark.parametrize("seed", range(4))
def test_emulated_plan_random(emu, twins, seed):
    topo, free, pods, lvl, hold, mem = random_case(100 + seed, N=40, P=120, mem=seed % 2 == 0)
    keys, vic, _ = emu_plan(emu, topo, free, pods, lvl, hold, mem=mem, base=seed)
    want = twins[1](topo, free, pods, lvl, hold=hold, mem=mem, base=seed)
    assert (keys == want[0]).all() and (vic == want[1]).all()


@pytest.mark.parametrize("table", ["flat_max", "general_edge"])
def test_emulated_plan_weight_tables(emu, twins, table):
    """The full 17-bit cost field and the byte-key boundary: the edge node's k = 8 cost is 28 * W[level]."""
    W = W_of(table)
    topo, free, pods, lvl, hold, mem = big_k_case()
    keys, vic, _ = emu_plan(emu, topo, free, pods, lvl, hold, W=W)
    want = twins[1](topo, free, pods, lvl, hold=hold, W=W)
    lit = literal_plan(twins[0], topo, free, pods, lvl, hold, W=W)
    assert (keys == want[0]).all() and (vic == want[1]).all()
    assert (lit[0] == want[0]).all() and (lit[1] == want[1]).all()
    assert max(int(k) >> 40 for k in keys if k != NO_FIT) >= 1 << 16, TABLES[table][:2]


# ---- build products ----------------------------------------------------------------------------------------------------
def test_plan_kernels_have_no_local_memory():
    if shutil.which("cuobjdump") is None or not os.path.exists(_lib.LIB_PATH):
        pytest.skip("cuobjdump or libkgpu.so missing")
    out = subprocess.run(["cuobjdump", "-res-usage", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    lines = out.splitlines()
    found = set()
    for i, line in enumerate(lines):
        m = re.search(r"Function (_ZN4kgpu\d+(plan_\w+?)E\S*):", line)
        if m:
            found.add(m.group(2))
            assert re.search(r"STACK:0\b", lines[i + 1]) and re.search(r"LOCAL:0\b", lines[i + 1]), lines[i + 1]
    assert found == {"plan_init", "plan_sequential"}, found


def test_plan_entry_point_allocates_only_through_buffers():
    src = open(os.path.join(ROOT, "kubegpu_b200", "csrc", "kgpu.cu")).read()
    body = src.split("int kgpu_preempt_plan(", 1)[1].split("\nint kgpu_", 1)[0]
    assert "reserve(" in body and not re.search(r"cuda(Malloc|Free)\w*\s*\(", body)


# ---- the device path -----------------------------------------------------------------------------------------------
def _nodes_of(keys):
    return (keys.astype(np.uint64) >> np.uint64(8)) & np.uint64(0xFFFFFFFF)


@pytest.mark.gpu
@pytest.mark.parametrize("use_mem", [False, True])
def test_plan_gen_preempt(twins, use_mem):
    """gen_preempt at C2's size (100k nodes, 10k pods), with and without C6's per-GPU memory: every key and victim set
    against the twin; victims and GPUs never shared; the handle's state untouched."""
    from kubegpu_b200.scorer import Scorer
    topo, free, hold, pods, lvl = synth.gen_preempt()
    mem = None
    if use_mem:
        mem = synth.gen_gpu_memory(len(free))
        pods[:, 3] = np.array(synth.POD_MIN_MEM_CHOICES_MIB, np.int32)[synth.rand_below(synth.SEED_C6, 14, len(pods), 7)]
    want_k, want_v = twins[1](topo, free, pods, lvl, hold=hold, mem=mem)
    with Scorer((0,)) as s:
        s.upload_nodes(topo, free)
        if use_mem:
            s.upload_gpu_memory(mem)
        s.upload_holders(hold)
        snap_before = s.preempt_batch(pods, lvl)
        keys, vic = s.preempt_plan(pods, lvl)
        assert (keys == want_k).all() and (vic == want_v).all()
        assert (s.get_free_masks() == free).all()
        snap_after = s.preempt_batch(pods, lvl)
        assert (snap_after[0] == snap_before[0]).all() and (snap_after[1] == snap_before[1]).all()
    assert (vic != 0).sum() >= 2000
    check_properties(pods, keys, vic)


@pytest.mark.gpu
def test_plan_equalities():
    """P = 1 is preempt_batch; no holder table, or every level 0, is place_batch(dry_run=True) -- on C2 and on C6 with
    GPU memory."""
    from kubegpu_b200.scorer import Scorer
    topo, free, hold, pods, lvl = synth.gen_preempt(N=20_000, P=2000)
    with Scorer((0,)) as s:
        s.upload_nodes(topo, free, node_id_base=7)
        s.upload_holders(hold)
        for p in range(0, 2000, 97):
            one = s.preempt_plan(pods[p:p + 1], lvl[p:p + 1])
            snap = s.preempt_batch(pods[p:p + 1], lvl[p:p + 1])
            assert one[0][0] == snap[0][0] and one[1][0] == snap[1][0]
    for name in ("c2", "c6"):
        if name == "c2":
            topo, free, pods = synth.gen_c2()
            mem = None
        else:
            topo, free, mem, pods = synth.gen_c6()
        with Scorer((0,)) as s:
            s.upload_nodes(topo, free)
            if mem is not None:
                s.upload_gpu_memory(mem)
            want = s.place_batch(pods, dry_run=True)
            keys, vic = s.preempt_plan(pods, np.full(len(pods), 5, np.int32))          # no holder table
            assert (keys == want).all() and (vic == 0).all()
            s.upload_holders(random_holders(np.random.default_rng(2), free))
            keys, vic = s.preempt_plan(pods, np.zeros(len(pods), np.int32))            # every level 0
            assert (keys == want).all() and (vic == 0).all()


@pytest.mark.gpu
def test_plan_c3_cluster(twins):
    """C3's 1M-node cluster (7813 node tiles) with a small batch, against the twin."""
    from kubegpu_b200.scorer import Scorer
    topo, free, pods = synth.gen_c3(P=96)
    rng = np.random.default_rng(4)
    hold = random_holders(rng, free, levels=4)
    lvl = rng.choice(np.array([0, 2, 5], np.int32), size=len(pods))
    want = twins[1](topo, free, pods, lvl, hold=hold, base=11)
    with Scorer((0,)) as s:
        s.upload_nodes(topo, free, node_id_base=11)
        s.upload_holders(hold)
        keys, vic = s.preempt_plan(pods, lvl)
    assert (keys == want[0]).all() and (vic == want[1]).all() and (keys != NO_FIT).all()


@pytest.mark.gpu
def test_plan_rejected_batches():
    """lvl outside 0..15, 8 distinct min_mem values and 33 (level, min_mem) pairs are KGPU_ERR_INVALID; the state stays."""
    from kubegpu_b200.scorer import KgpuError, Scorer
    topo, free, hold, pods, lvl = synth.gen_preempt(N=5000, P=200)
    many_mem = pods.copy()
    many_mem[:8, 3] = np.arange(1, 9) * 1000
    many_views = pods.copy()
    many_views[:, 3] = 0
    views_lvl = lvl.copy()
    views_lvl[:33] = np.tile(np.arange(1, 12), 3)
    many_views[:33, 3] = np.repeat(np.array([0, 1000, 2000]), 11)
    ok_views, views_ok_lvl = many_views.copy(), views_lvl.copy()
    ok_views[32, 3], views_ok_lvl[32] = 0, 1                                   # (11, 2000) becomes (1, 0): 32 pairs
    with Scorer((0,)) as s:
        s.upload_nodes(topo, free)
        s.upload_holders(hold)
        want = s.preempt_plan(pods, lvl)
        s.preempt_plan(ok_views, views_ok_lvl)                                     # 32 pairs are fine
        for bad_pods, bad_lvl in ((pods, np.where(np.arange(len(lvl)) == 5, 16, lvl)),
                                  (pods, np.where(np.arange(len(lvl)) == 5, -1, lvl)),
                                  (many_mem, lvl), (many_views, views_lvl)):
            with pytest.raises(KgpuError) as e:
                s.preempt_plan(bad_pods, bad_lvl)
            assert e.value.code == _lib.ERR_INVALID
        assert (s.get_free_masks() == free).all()
        got = s.preempt_plan(pods, lvl)
        assert (got[0] == want[0]).all() and (got[1] == want[1]).all()


@pytest.mark.gpu
def test_plan_two_devices_is_a_state_error():
    import torch
    from kubegpu_b200.scorer import KgpuError, Scorer
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    topo, free, hold, pods, lvl = synth.gen_preempt(N=1000, P=10)
    with Scorer((0, 1)) as s:
        s.upload_nodes(topo, free)
        with pytest.raises(KgpuError) as e:
            s.preempt_plan(pods, lvl)
        assert e.value.code == _lib.ERR_STATE


@pytest.mark.gpu
def test_host_mirror_plan_names_different_victims():
    """sched_cli on a full two-node cluster: two identical high-priority pods get the same victim from preemptbatch and
    different victims from preemptplan; a preemptbatch afterwards shows the mirror's state unchanged."""
    from test_preemption import CLI, _node_line
    if not os.path.exists(CLI):
        subprocess.check_call(["make", "-s", "-C", ROOT, "kubegpu_b200/lib/kgpu_sched_cli"])
    ids = ["GPU-%02d" % i for i in range(8)]
    lines = [_node_line("A", [[4], [4]], ids), _node_line("B", [[4], [4]], ids),
             "pod a1 priority=1 run c req=4", "pod a2 priority=2 run c req=4",
             "pod b1 priority=1 run c req=4", "pod b2 priority=2 run c req=4",
             "pod h1 priority=3 run c req=4", "pod h2 priority=3 run c req=4",
             "placebatch a1 a2 b1 b2",
             "preemptbatch h1 h2",
             "preemptplan h1 h2",
             "preemptbatch h1 h2"]
    got = subprocess.run([CLI], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True).stdout
    snap = got.split("> preemptbatch h1 h2\n")[1].splitlines()
    plan = got.split("> preemptplan h1 h2\n")[1].splitlines()
    again = got.split("> preemptbatch h1 h2\n")[2].splitlines()
    assert snap[0] == "  err=" and plan[0] == "  err="
    assert " node=A " in snap[1] and snap[1].endswith("victims=a1") and " node=A " in snap[2] and snap[2].endswith("victims=a1")
    assert " node=A " in plan[1] and plan[1].endswith("victims=a1") and " node=B " in plan[2] and plan[2].endswith("victims=b1")
    assert again[:3] == snap[:3]
