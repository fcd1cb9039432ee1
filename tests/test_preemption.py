"""Preemption (kgpu_preempt_batch): for pods that fit nowhere, the node, GPUs and lowest-priority running pods to evict.
CPU: the twin (tests/preempt_twin/preempt_twin.c, built with the oracle) against an independent Python brute force,
the emulated kernels (tests/emu) against the twin, and the kernel's resource usage.  GPU: the
device path bit-exact against the twin on gen_preempt at C2's size, the equalities with score_batch, table updates and
resets, rejected tables, and the host mirror's victims by name."""
import ctypes
import itertools
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import cpu_libs
from kubegpu_b200 import _lib, synth

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CLI = os.path.join(ROOT, "kubegpu_b200", "lib", "kgpu_sched_cli")
NO_FIT = np.uint64(0xFFFFFFFFFFFFFFFF)


def _p(a, t=ctypes.c_int32):
    return a.ctypes.data_as(ctypes.POINTER(t))


def _opt(a):
    return None if a is None else _p(np.ascontiguousarray(a, dtype=np.int32))


@pytest.fixture(scope="session")
def twin():
    """preempt(topo, free, pods, lvl, hold=None, mem=None, base=0) -> (keys, victims)."""
    from oracle import oracle_b
    L = cpu_libs.twin("preempt")
    W = np.ascontiguousarray(oracle_b.DEFAULT_WEIGHTS, dtype=np.int32)

    def preempt(topo, free, pods, lvl, hold=None, mem=None, base=0):
        topo, free, pods, lvl = (np.ascontiguousarray(a, dtype=np.int32) for a in (topo, free, pods, lvl))
        keys = np.empty(len(pods), dtype=np.uint64)
        vic = np.empty(len(pods), dtype=np.uint32)
        L.preempt_twin_batch(_p(topo), _p(free), _opt(mem), _opt(hold), len(free), base, _p(pods), _p(lvl), len(pods), _p(W),
                             os.cpu_count() or 1, _p(keys, ctypes.c_uint64), _p(vic, ctypes.c_uint32))
        return keys, vic
    return preempt


def brute_force(topo, free, pods, lvl, hold, mem=None, base=0):
    """The definition in plain Python: every node, every k-subset, the tuple (max victim level, |V|, cost, node, S)."""
    from oracle import oracle_b
    W = [int(w) for w in oracle_b.DEFAULT_WEIGHTS]
    keys, vic = [], []
    for (k, _, _, need), L in zip(pods.tolist(), lvl.tolist()):
        best = None
        if 0 <= k <= 8:
            for n in range(len(free)):
                M = topo[n]
                for S in itertools.combinations(range(8), k):
                    V, ok = {}, True
                    for i in S:
                        if mem is not None and need > 0 and mem[n][i] < need:
                            ok = False
                        elif not (free[n] >> i) & 1:
                            e = int(hold[n][i])
                            if e < 0 or e >> 3 >= L:
                                ok = False
                            else:
                                V[e & 7] = e >> 3
                    if not ok:
                        continue
                    cost = sum(W[M[i * 8 + j]] for i, j in itertools.combinations(S, 2))
                    mask = sum(1 << i for i in S)
                    t = (max(V.values(), default=0), len(V), cost, base + n, mask, sum(1 << o for o in V))
                    best = t if best is None or t[:5] < best[:5] else best
        keys.append(NO_FIT if best is None else np.uint64((best[2] << 40) | (best[3] << 8) | best[4]))
        vic.append(0 if best is None else best[5])
    return np.array(keys, dtype=np.uint64), np.array(vic, dtype=np.uint32)


def random_holders(rng, free, levels=16, owners=8, untracked=0.1):
    """A valid table: each node's GPUs go to random owners (one level per owner), some entries -1; free GPUs keep
    entries too (they must be ignored)."""
    N = len(free)
    own = rng.integers(0, owners, size=(N, 8))
    olvl = rng.integers(0, levels, size=(N, 8))
    hold = (np.take_along_axis(olvl, own, axis=1) << 3 | own).astype(np.int32)
    hold[rng.random((N, 8)) < untracked] = -1
    return hold


def random_case(seed, N=7, P=40, mem=False):
    rng = np.random.default_rng(seed)
    topo, _, _ = synth.gen_c4(N=N, P=0, seed=seed + 1)
    free = rng.integers(0, 256, size=N).astype(np.int32) & rng.integers(0, 256, size=N).astype(np.int32)
    hold = random_holders(rng, free)
    pods = synth.make_pods(rng.integers(-1, 10, size=P).astype(np.int32))
    lvl = rng.integers(0, 16, size=P).astype(np.int32)
    gm = None
    if mem:
        gm = synth.gen_gpu_memory(N, seed=seed + 2)
        pods[:, 3] = np.array(synth.POD_MIN_MEM_CHOICES_MIB, np.int32)[rng.integers(0, 7, size=P)]
    return topo, free, pods, lvl, hold, gm


# ---- the twin --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(6))
def test_twin_matches_brute_force(twin, seed):
    topo, free, pods, lvl, hold, mem = random_case(seed, mem=seed % 2 == 1)
    want = brute_force(topo, free, pods, lvl, hold, mem=mem, base=5)
    got = twin(topo, free, pods, lvl, hold=hold, mem=mem, base=5)
    assert (got[0] == want[0]).all() and (got[1] == want[1]).all()
    assert (got[1] != 0).any() and (got[0] == NO_FIT).any() and set(pods[:, 0].tolist()) >= {-1, 0, 8, 9}


def test_twin_without_holders_is_score_batch(twin, oracle_b):
    topo, free, mem, pods = synth.gen_c6(N=300, P=200)
    lvl = np.full(len(pods), 15, np.int32)
    keys, vic = twin(topo, free, pods, lvl, mem=mem, base=9)
    assert (keys == oracle_b.score_batch(topo, free, pods, mem=mem, node_id_base=9)).all() and (vic == 0).all()


# ---- the kernels on the CPU (tests/emu) -------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu():
    return cpu_libs.emu()


def emu_preempt(emu, topo, free, pods, lvl, hold, mem=None, base=0, splits=1):
    """The scoring path's keys from the oracle, then the emulated compaction, preemption kernel and finalisation."""
    from oracle import oracle_b
    topo, free, pods, lvl = (np.ascontiguousarray(a, dtype=np.int32) for a in (topo, free, pods, lvl))
    keys = oracle_b.score_batch(topo, free, pods, mem=mem, node_id_base=base)
    vic = np.empty(len(pods), dtype=np.uint32)
    W = np.ascontiguousarray(oracle_b.DEFAULT_WEIGHTS, dtype=np.int32)
    reached = emu.emu_preempt_batch(_p(topo), _p(free), _opt(mem), _opt(hold), len(free), base, _p(pods), _p(lvl), len(pods),
                                    _p(W), splits, _p(keys, ctypes.c_uint64), _p(vic, ctypes.c_uint32))
    return keys, vic, reached


def _row(*owners):
    """A holder row from (level, owner) per slot, None = -1."""
    return [-1 if o is None else o[0] << 3 | o[1] for o in owners]


def ties_case():
    """Identical nodes and owners: ties on level, |V| and cost go to the lower node, then the lower mask."""
    m = synth.shape_matrix([[2, 2], [2, 2]])
    topo = np.stack([m] * 4)
    free = np.array([0x00, 0x00, 0x01, 0x00], np.int32)
    row = _row((1, 0), (1, 0), (1, 1), (1, 1), (2, 2), (2, 2), (1, 3), (1, 3))
    hold = np.array([row, row, row, _row((1, 0), (1, 0), (1, 1), (1, 1), (1, 2), (1, 2), (1, 3), (1, 3))], np.int32)
    pods = synth.make_pods(np.array([2, 2, 4, 4, 3, 8, 1], np.int32))
    lvl = np.array([2, 3, 2, 3, 2, 3, 2], np.int32)
    return topo, free, pods, lvl, hold, None


def big_owner_case():
    """An owner whose eviction frees more GPUs than S uses, next to a smaller owner of the same level."""
    topo = np.stack([synth.shape_matrix([[4], [4]]), synth.shape_matrix([[2, 2], [2, 2]])])
    free = np.array([0x00, 0x80], np.int32)
    hold = np.array([_row(*[(1, 0)] * 4, *[(2, 1)] * 4), _row(*[(1, 0)] * 6, (1, 1), None)], np.int32)
    pods = synth.make_pods(np.array([2, 2, 3, 6, 8], np.int32))
    lvl = np.array([2, 3, 2, 2, 3], np.int32)
    return topo, free, pods, lvl, hold, None


def min_mem_case():
    """min_mem makes an evictable GPU unusable, so a costlier or higher-level set must go."""
    topo = np.stack([synth.shape_matrix([[4], [4]])] * 2)
    free = np.array([0x01, 0x00], np.int32)
    hold = np.array([_row(None, (0, 0), (0, 1), (0, 1), (1, 2), (1, 2), (1, 3), (1, 3)),
                     _row(*[(0, 0)] * 2, *[(1, 1)] * 2, *[(2, 2)] * 4)], np.int32)
    mem = np.full((2, 8), 81_920, np.int32)
    mem[0, 1] = mem[0, 2] = 16_384
    pods = synth.make_pods(np.array([2, 2, 4, 4], np.int32))
    pods[:, 3] = [0, 40_000, 40_000, 0]
    lvl = np.array([3, 3, 3, 3], np.int32)
    return topo, free, pods, lvl, hold, mem


def free_entries_case():
    """Entries on free GPUs are ignored: a free GPU's stale entry names neither a victim nor a level."""
    topo = np.stack([synth.shape_matrix([[8]])] * 2)
    free = np.array([0x0F, 0x03], np.int32)
    hold = np.array([_row((9, 5), (9, 5), (9, 6), (9, 6), (1, 0), (1, 0), (2, 1), (2, 1)),
                     _row((0, 7), (0, 7), (1, 0), (1, 0), (1, 0), (1, 1), (1, 1), (1, 1))], np.int32)
    pods = synth.make_pods(np.array([6, 6, 5, 8, 4], np.int32))
    lvl = np.array([2, 3, 2, 2, 1], np.int32)
    return topo, free, pods, lvl, hold, None


def extreme_levels_case():
    """Level-15 holders are never evicted; level-0 pods evict nothing; level-15 pods evict everything below."""
    topo = np.stack([synth.shape_matrix([[2, 2], [2, 2]])] * 3)
    free = np.array([0x00, 0x00, 0x00], np.int32)
    hold = np.array([_row(*[(15, 0)] * 8), _row(*[(14, 0)] * 4, *[(0, 1)] * 4), _row(*[(15, 0)] * 4, *[(3, 1)] * 4)], np.int32)
    pods = synth.make_pods(np.array([4, 4, 4, 8, 8, 2, 1], np.int32))
    lvl = np.array([0, 15, 1, 15, 14, 4, 0], np.int32)
    return topo, free, pods, lvl, hold, None


def k_edge_case():
    """k = 0 fits on the first node, k outside 0..8 never, with or without evictable GPUs."""
    topo = np.stack([synth.shape_matrix([[4], [4]])] * 2)
    free = np.array([0x00, 0x00], np.int32)
    hold = np.array([_row(*[(0, 0)] * 8), _row(*[(0, 1)] * 8)], np.int32)
    pods = synth.make_pods(np.array([0, -1, 9, 0, 8, 100], np.int32))
    lvl = np.array([5, 5, 5, 0, 5, 15], np.int32)
    return topo, free, pods, lvl, hold, None


def whole_node_case():
    """One owner holds a whole node: any k on that node evicts exactly it."""
    topo = np.stack([synth.shape_matrix([[8]]), synth.shape_matrix([[4, 4]])])
    free = np.array([0x00, 0x00], np.int32)
    hold = np.array([_row(*[(2, 3)] * 8), _row(*[(1, 0)] * 8)], np.int32)
    pods = synth.make_pods(np.array([1, 2, 4, 8, 8], np.int32))
    lvl = np.array([3, 3, 2, 3, 2], np.int32)
    return topo, free, pods, lvl, hold, None


def multi_block_case():
    """300 nodes (three node tiles) and 700 pods, most of them reaching the kernel (more than two 256-pod chunks)."""
    rng = np.random.default_rng(11)
    topo, _, _ = synth.gen_c4(N=300, P=0, seed=77)
    free = (rng.integers(0, 256, size=300) & rng.integers(0, 256, size=300) & rng.integers(0, 256, size=300)).astype(np.int32)
    hold = random_holders(rng, free, levels=6)
    pods = synth.make_pods(np.array([5, 6, 7, 8], np.int32)[rng.integers(0, 4, size=700)])
    lvl = rng.integers(1, 8, size=700).astype(np.int32)
    return topo, free, pods, lvl, hold, None


CASES = {"ties": ties_case, "big_owner": big_owner_case, "min_mem": min_mem_case, "free_entries": free_entries_case,
         "extreme_levels": extreme_levels_case, "k_edge": k_edge_case, "whole_node": whole_node_case}


@pytest.mark.parametrize("name", sorted(CASES))
def test_emulated_preemption_matches_twin(emu, twin, name):
    topo, free, pods, lvl, hold, mem = CASES[name]()
    keys, vic, _ = emu_preempt(emu, topo, free, pods, lvl, hold, mem=mem, base=3)
    want = twin(topo, free, pods, lvl, hold=hold, mem=mem, base=3)
    assert (keys == want[0]).all() and (vic == want[1]).all(), (keys, want[0], vic, want[1])
    assert (want[1] != 0).any()
    bf = brute_force(topo, free, pods, lvl, hold, mem=mem, base=3)
    assert (bf[0] == want[0]).all() and (bf[1] == want[1]).all()


def test_emulated_preemption_several_blocks_and_chunks(emu, twin):
    topo, free, pods, lvl, hold, mem = multi_block_case()
    for splits in (1, 2):
        keys, vic, reached = emu_preempt(emu, topo, free, pods, lvl, hold, splits=splits)
        want = twin(topo, free, pods, lvl, hold=hold)
        assert reached > 2 * 256 and (keys == want[0]).all() and (vic == want[1]).all()


@pytest.mark.parametrize("seed", range(4))
def test_emulated_preemption_random(emu, twin, seed):
    topo, free, pods, lvl, hold, mem = random_case(100 + seed, N=40, P=120, mem=seed % 2 == 0)
    keys, vic, _ = emu_preempt(emu, topo, free, pods, lvl, hold, mem=mem, base=seed)
    want = twin(topo, free, pods, lvl, hold=hold, mem=mem, base=seed)
    assert (keys == want[0]).all() and (vic == want[1]).all()


def test_case_claims(twin):
    """The hand-made cases do what their names say."""
    from oracle import oracle_b
    topo, free, pods, lvl, hold, _ = ties_case()
    keys, vic = twin(topo, free, pods, lvl, hold=hold)
    assert oracle_b.unpack_key(keys[0]) == (2, 0, 0x03) and vic[0] == 0b1      # first node, first pair
    topo, free, pods, lvl, hold, _ = big_owner_case()
    keys, vic = twin(topo, free, pods, lvl, hold=hold)
    assert vic[0] == 0b1 and bin(int(keys[0]) & 0xFF).count("1") == 2          # evicts a 4-GPU owner for 2 GPUs
    topo, free, pods, lvl, hold, mem = min_mem_case()
    k_nomem, _ = twin(topo, free, pods[:1], lvl[:1], hold=hold, mem=mem)
    k_mem, _ = twin(topo, free, pods[1:2], lvl[1:2], hold=hold, mem=mem)
    assert int(k_nomem[0]) & 0x06 and not int(k_mem[0]) & 0x06
    topo, free, pods, lvl, hold, _ = extreme_levels_case()
    keys, vic = twin(topo, free, pods, lvl, hold=hold)
    assert keys[0] == NO_FIT and keys[6] == NO_FIT and vic[1] == 0b10 and (int(keys[1]) >> 8) & 0xFFFFFFFF == 1
    topo, free, pods, lvl, hold, _ = k_edge_case()
    keys, vic = twin(topo, free, pods, lvl, hold=hold)
    assert keys[0] == 0 and keys[3] == 0 and (keys[[1, 2, 5]] == NO_FIT).all() and vic[4] == 0b1


# ---- build products ----------------------------------------------------------------------------------------------------
def test_preempt_kernels_have_no_local_memory():
    if shutil.which("cuobjdump") is None or not os.path.exists(_lib.LIB_PATH):
        pytest.skip("cuobjdump or libkgpu.so missing")
    out = subprocess.run(["cuobjdump", "-res-usage", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    lines = out.splitlines()
    found = set()
    for i, line in enumerate(lines):
        m = re.search(r"Function (_ZN4kgpu\d+(preempt_\w+?|scatter_holders)E\S*):", line)
        if m:
            found.add(m.group(2))
            assert re.search(r"STACK:0\b", lines[i + 1]) and re.search(r"LOCAL:0\b", lines[i + 1]), lines[i + 1]
    assert found == {"preempt_compact", "preempt_lane_per_node", "preempt_finalize", "scatter_holders"}, found


# ---- the device path -----------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("use_mem", [False, True])
def test_preempt_batch_gen_preempt(twin, oracle_b, use_mem):
    """gen_preempt at C2's size (100k nodes, 10k pods), with and without C6's per-GPU memory: every key and victim set."""
    from kubegpu_b200.scorer import Scorer
    topo, free, hold, pods, lvl = synth.gen_preempt()
    mem = None
    if use_mem:
        mem = synth.gen_gpu_memory(len(free))
        pods[:, 3] = np.array(synth.POD_MIN_MEM_CHOICES_MIB, np.int32)[synth.rand_below(synth.SEED_C6, 14, len(pods), 7)]
    want_k, want_v = twin(topo, free, pods, lvl, hold=hold, mem=mem)
    with Scorer((0,)) as s:
        s.upload_nodes(topo, free)
        if use_mem:
            s.upload_gpu_memory(mem)
        s.upload_holders(hold)
        keys, vic = s.preempt_batch(pods, lvl)
        assert (keys == want_k).all() and (vic == want_v).all()
        plain = s.score_batch(pods)
    evicting = (plain == NO_FIT) & (keys != NO_FIT)
    assert evicting.sum() > 2000 and (vic[evicting] != 0).all() and (vic[plain != NO_FIT] == 0).all()


@pytest.mark.gpu
def test_preempt_batch_equals_score_batch_without_eviction(oracle_b):
    from kubegpu_b200.scorer import Scorer
    topo, free, hold, pods, lvl = synth.gen_preempt(N=20_000, P=3000)
    with Scorer((0,)) as s:
        s.upload_nodes(topo, free, node_id_base=7)
        plain_before = s.score_batch(pods)
        keys, vic = s.preempt_batch(pods, lvl)                 # no table yet
        assert (keys == plain_before).all() and (vic == 0).all()
        s.upload_holders(hold)
        keys, vic = s.preempt_batch(pods, np.zeros(len(pods), np.int32))
        assert (keys == s.score_batch(pods)).all() and (vic == 0).all()
        small = pods[pods[:, 0] <= 2]                          # every k <= 2 pod fits without eviction
        keys, vic = s.preempt_batch(small, np.full(len(small), 4, np.int32))
        assert (keys != NO_FIT).all() and (keys == s.score_batch(small)).all() and (vic == 0).all()


@pytest.mark.gpu
def test_set_holders_and_reset(twin, oracle_b):
    """Rows replaced with set_holders (a node listed twice gets its last row) answer as the twin on the new table;
    upload_nodes resets the table to all -1."""
    from kubegpu_b200.scorer import Scorer
    topo, free, hold, pods, lvl = synth.gen_preempt(N=20_000, P=3000)
    rng = np.random.default_rng(5)
    idx = rng.choice(len(free), size=4000, replace=False)
    rows = random_holders(rng, free[idx], levels=5)
    idx = np.concatenate([idx, idx[:10]])
    rows = np.concatenate([rows, np.full((10, 8), -1, np.int32)])
    new = hold.copy()
    new[idx] = rows                                            # numpy: the last assignment wins as well
    want_k, want_v = twin(topo, free, pods, lvl, hold=new)
    with Scorer((0,)) as s:
        s.upload_nodes(topo, free)
        s.upload_holders(hold)
        s.set_holders(idx, rows)
        keys, vic = s.preempt_batch(pods, lvl)
        assert (keys == want_k).all() and (vic == want_v).all()
        s.upload_nodes(topo, free)
        keys, vic = s.preempt_batch(pods, lvl)
        assert (keys == s.score_batch(pods)).all() and (vic == 0).all()
        s.set_holders(idx[:10], hold[idx[:10]])                # first use after the reset: every other row is -1
        only = np.full_like(hold, -1)
        only[idx[:10]] = hold[idx[:10]]
        want_k, want_v = twin(topo, free, pods, lvl, hold=only)
        keys, vic = s.preempt_batch(pods, lvl)
        assert (keys == want_k).all() and (vic == want_v).all()


@pytest.mark.gpu
def test_invalid_tables_are_rejected(twin):
    from kubegpu_b200.scorer import KgpuError, Scorer
    topo, free, hold, pods, lvl = synth.gen_preempt(N=5000, P=1000)
    want = twin(topo, free, pods, lvl, hold=hold)
    bad_rows = [_row(*[(1, 0)] * 7, (2, 0)),                   # an owner with two levels
                [128] + [-1] * 7,                               # level 16
                [-2] + [-1] * 7]                                # neither -1 nor an entry
    with Scorer((0,)) as s:
        s.upload_nodes(topo, free)
        s.upload_holders(hold)
        for row in bad_rows:
            bad = hold.copy()
            bad[17] = row
            for call in (lambda: s.upload_holders(bad), lambda: s.set_holders([3, 17], bad[[3, 17]])):
                with pytest.raises(KgpuError) as e:
                    call()
                assert e.value.code == _lib.ERR_INVALID
        with pytest.raises(KgpuError) as e:
            s.preempt_batch(pods, np.full(len(pods), 16, np.int32))
        assert e.value.code == _lib.ERR_INVALID
        keys, vic = s.preempt_batch(pods, lvl)
        assert (keys == want[0]).all() and (vic == want[1]).all()


def _node_line(name, shape, ids):
    from oracle import oracle_a as oa
    res = oa.shape_to_resources(shape)
    res = {k.replace("/gpu/%d/" % i, "/gpu/%s/" % ids[i]): v for i, k in enumerate(sorted(res, key=lambda s: int(s.split("/gpu/")[1].split("/")[0])))
           for v in [res[k]]}
    return "addnode %s %d %s" % (name, sum(sum(g) for g in shape), " ".join("%s=%d" % kv for kv in sorted(res.items())))


@pytest.mark.gpu
def test_host_mirror_names_victims():
    """sched_cli: placebatch fills two nodes; preemptbatch names the lowest-level running pods on the best node; after
    ReturnPodResources of a victim the freed GPUs serve without eviction and it is no longer named."""
    if not os.path.exists(CLI):
        subprocess.check_call(["make", "-s", "-C", ROOT, "kubegpu_b200/lib/kgpu_sched_cli"])
    ids = ["GPU-%02d" % i for i in range(8)]
    lines = [_node_line("A", [[4], [4]], ids), _node_line("B", [[4], [4]], ids),
             "pod a1 priority=1 run c req=4", "pod a2 priority=3 run c req=4",
             "pod b1 priority=2 run c req=4", "pod b2 priority=2 run c req=4",
             "pod hi priority=3 run c req=4", "pod top priority=9 run c req=8", "pod low run c req=4",
             "placebatch a1 a2 b1 b2",
             "preemptbatch hi top low",
             "return a1",
             "preemptbatch hi top low"]
    got = subprocess.run([CLI], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True).stdout
    first = got.split("> preemptbatch hi top low\n")[1].splitlines()
    assert first[0] == "  err="
    assert first[1].startswith("  hi fits=1 ") and " node=A " in first[1] and first[1].endswith("victims=a1")
    assert first[2].startswith("  top fits=1 ") and " node=B mask=0xff" in first[2] and first[2].endswith("victims=b1,b2")
    assert first[3] == "  low fits=0 cost=0 node= mask=0x00 victims="
    second = got.split("> preemptbatch hi top low\n")[2].splitlines()
    assert second[1].startswith("  hi fits=1 ") and " node=A " in second[1] and second[1].endswith("victims=")
    assert second[2].endswith("victims=b1,b2") and "a1" not in "".join(second)
