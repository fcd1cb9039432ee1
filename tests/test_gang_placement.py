"""Gangs in sequential placement (kgpu_place_batch_gang): a run of consecutive pods with the same nonzero gang id is
placed all or nothing.  CPU: the gang twin (tests/gang_twin/gang_twin.c, built with the oracle) against the deletion
property and against a gang-by-gang construction on top of the oracle's plain sequential placement, and the emulated
kernel (place_sequential<true>, tests/emu) against the twin.  GPU: the device path bit-exact against
the twin, dry runs, bad ids, and the host mirror's reordering."""
import ctypes
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


@pytest.fixture(scope="session")
def twin():
    """place(topo, free, pods, gang, mem=None, base=0) -> (keys, free_after): gang_twin.c built with the oracle."""
    from oracle import oracle_b
    L = cpu_libs.twin("gang")
    W = np.ascontiguousarray(oracle_b.DEFAULT_WEIGHTS, dtype=np.int32)

    def place(topo, free, pods, gang, mem=None, base=0):
        topo, pods, gang = (np.ascontiguousarray(a, dtype=np.int32) for a in (topo, pods, gang))
        assert gang.size == len(pods)
        starts = [g for g, _, _ in runs(gang)]
        if len(set(starts)) != len(starts):
            raise ValueError("a gang id appears in two separate runs")
        f = np.array(free, dtype=np.int32, copy=True)
        keys = np.empty(len(pods), dtype=np.uint64)
        memp = None if mem is None else _p(np.ascontiguousarray(mem, dtype=np.int32))
        L.gang_twin_place_batch(_p(topo), _p(f), memp, len(f), base, _p(pods), _p(gang), len(pods), _p(W), _p(keys, ctypes.c_uint64))
        return keys, f
    return place


def random_gangs(P, seed, share=0.5):
    """Gang ids for P pods: runs of 1..6 consecutive pods, about `share` of the pods in a gang, ids 1, 2, ..."""
    rng = np.random.default_rng(seed)
    gang = np.zeros(P, dtype=np.int32)
    p, gid = 0, 0
    while p < P:
        n = int(rng.integers(1, 7))
        if rng.random() < share:
            gid += 1
            gang[p:p + n] = gid
        p += n
    return gang


def runs(gang):
    """[(id, first, end)] of the nonzero runs."""
    out, p = [], 0
    while p < len(gang):
        e = p + 1
        while e < len(gang) and gang[e] == gang[p]:
            e += 1
        if gang[p] != 0:
            out.append((int(gang[p]), p, e))
        p = e
    return out


def by_deletion(ob, topo, free, pods, gang, keys, mem=None, base=0):
    """The plain twin on the batch without the gangs that failed in `keys`, NO_FIT for their pods."""
    failed = np.isin(gang, [g for g, a, e in runs(gang) if (keys[a:e] == NO_FIT).any()])
    kk, ff = ob.place_batch(topo, free, pods[~failed], mem=mem, node_id_base=base)
    want = np.full(len(pods), NO_FIT, dtype=np.uint64)
    want[~failed] = kk
    return want, ff


def by_segments(ob, topo, free, pods, gang, mem=None, base=0):
    """Gang semantics built from the plain twin alone: each gang placed on the current state, kept only if every
    member fits."""
    state = np.array(free, dtype=np.int32, copy=True)
    want = np.full(len(pods), NO_FIT, dtype=np.uint64)
    p = 0
    while p < len(pods):
        e = p + 1
        while e < len(pods) and gang[e] == gang[p]:
            e += 1
        if gang[p] == 0:
            e = p + 1
        kk, ff = ob.place_batch(topo, state, pods[p:e], mem=mem, node_id_base=base)
        if gang[p] == 0 or (kk != NO_FIT).all():
            want[p:e], state = kk, ff
        p = e
    return want, state


def miss_at(ob, topo, free, pods, gang):
    """{gang id: index of its first member that misses on the state before the gang, or None}, from the plain twin."""
    state, p, out = np.array(free, dtype=np.int32, copy=True), 0, {}
    for g, a, e in runs(gang):
        _, state = ob.place_batch(topo, state, pods[p:a])
        kk, ff = ob.place_batch(topo, state, pods[a:e])
        miss = np.flatnonzero(kk == NO_FIT)
        out[g] = int(miss[0]) if len(miss) else None
        if not len(miss):
            state = ff
        p = e
    return out


def check_consistent(ob, free, pods, gang, keys, free_after, base=0):
    """No GPU is used twice, every gang is placed whole or not at all, and the masks add up."""
    fm = np.array(free, dtype=np.int64) & 0xFF
    for key, k in zip(keys, pods[:, 0]):
        u = ob.unpack_key(key)
        if u is None:
            continue
        _, node, mask = u
        assert bin(mask).count("1") == k and mask & ~fm[node - base] == 0
        fm[node - base] &= ~mask
    assert (fm == (np.asarray(free_after) & 0xFF)).all()
    for _, a, e in runs(gang):
        assert (keys[a:e] == NO_FIT).all() or (keys[a:e] != NO_FIT).all()


def edge_batch():
    """10 full nodes (80 GPUs) and a batch whose gangs fail at the last member, in the middle, at the first member (k
    outside 0..8, and no fit), a gang of one that fits and one that fails, adjacent gangs, and a k = 0 member undone."""
    topo, _, _ = synth.gen_c2(N=10, P=0)
    free = np.full(10, 0xFF, dtype=np.int32)
    spec = ([(2, 0)] + [(8, 1)] * 3 +                # 6 full nodes left
            [(8, 2)] * 7 +                           # g2 misses at its last member
            [(8, 3)] * 8 +                           # g3 misses in the middle
            [(9, 4), (2, 4)] +                       # g4: k = 9 first
            [(8, 5)] * 6 +                           # fits only if g2 and g3 gave everything back
            [(8, 6), (1, 6)] +                       # g6 misses at its first member
            [(4, 7), (4, 8)] +                       # gangs of one: g7 fits, g8 does not
            [(1, 9), (1, 9), (0, 10), (1, 10)] +     # g9 fits, g10 (adjacent) misses after a k = 0 member
            [(1, 0), (-1, 0)])
    pods = synth.make_pods(np.array([k for k, _ in spec], dtype=np.int32))
    gang = np.array([g for _, g in spec], dtype=np.int32)
    return topo, free, pods, gang, None


def chunk_batch():
    """A failing gang across pod index 1024 (the kernel stages 1024 pods at a time) and one that fits after it."""
    topo, _, _ = synth.gen_c2(N=4, P=0)
    free = np.full(4, 0xFF, dtype=np.int32)
    ks = np.full(1040, -1, dtype=np.int32)
    ks[::7] = 0
    ks[3], ks[500] = 8, 8                         # two nodes taken, 16 GPUs left
    gang = np.zeros(1040, dtype=np.int32)
    ks[1018:1027], gang[1018:1027] = 2, 5         # 9 x 2 GPUs > 16: the 9th member (pod 1026) misses
    ks[1027:1031], gang[1027:1031] = 4, 6         # fits in what the failed gang gave back
    ks[1031:1033] = 8
    return topo, free, synth.make_pods(ks), gang, None


def views_batch(N=300, P=150, seed=3):
    """Memory-aware pods (five min_mem views) in gangs."""
    topo, free, mem, pods = synth.gen_c6(N=N, P=P)
    return topo, free, pods, random_gangs(P, seed), mem


def wide_batch():
    """More than 32 tiles per supertile (the kernel's uncached supertile path): 8 views need > 2048 tiles."""
    N = 128 * 2049 + 5
    topo, free, _ = synth.gen_c2(N=N, P=0)
    free[:] = 0
    hot = [3, 140_000, N - 1, 200_000]
    free[hot] = [0xFF, 0x0F, 0xFF, 0xF0]
    mem = np.full((N, 8), 81_920, dtype=np.int32)
    mem[140_000] = 16_384
    ks = np.array([4, 4, 8, 2, 2, 4, 8, 4, 4, 2, 1, 1, 4], dtype=np.int32)
    pods = synth.make_pods(ks)
    pods[:, 3] = [0, 1000, 2000, 3000, 4000, 5000, 6000, 7000, 0, 1000, 0, 0, 0]
    gang = np.array([1, 1, 1, 0, 2, 2, 3, 3, 3, 0, 4, 4, 0], dtype=np.int32)
    return topo, free, pods, gang, mem


def one_node_batch():
    topo, _, _ = synth.gen_c4(N=1, P=0)
    free = np.array([0xFF], dtype=np.int32)
    pods = synth.make_pods(np.array([2, 2, 8, 1, 4, 4, 2, 2], dtype=np.int32))
    gang = np.array([0, 1, 1, 0, 2, 2, 2, 3], dtype=np.int32)
    return topo, free, pods, gang, None


SMALL_CASES = {"edges": edge_batch, "chunk": chunk_batch, "views": views_batch, "one_node": one_node_batch}


# ---- the twin ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["c1", "c2", "c4", "c6"])
def test_twin_equals_deletion_property(twin, oracle_b, name):
    mem = None
    if name == "c1":
        topo, free, _ = synth.gen_c1()
        pods = synth.make_pods(np.array([3, 4, 1, 2, 8, 4, 4, 2, 0, 9, 1, 1] * 3, dtype=np.int32))
    elif name == "c2":
        topo, free, pods = synth.gen_c2(N=300, P=400)
    elif name == "c4":
        topo, free, pods = synth.gen_c4(N=257, P=300)
    else:
        topo, free, mem, pods = synth.gen_c6(N=300, P=300)
    gang = random_gangs(len(pods), seed=len(name) + len(pods))
    keys, fa = twin(topo, free, pods, gang, mem=mem, base=13)
    want, wf = by_deletion(oracle_b, topo, free, pods, gang, keys, mem=mem, base=13)
    assert (keys == want).all() and (fa == wf).all()
    seg_keys, seg_free = by_segments(oracle_b, topo, free, pods, gang, mem=mem, base=13)
    assert (keys == seg_keys).all() and (fa == seg_free).all()
    check_consistent(oracle_b, free, pods, gang, keys, fa, base=13)
    g = runs(gang)
    assert any((keys[a:e] == NO_FIT).all() for _, a, e in g) and any((keys[a:e] != NO_FIT).all() for _, a, e in g)


@pytest.mark.parametrize("use_mem", [False, True])
def test_twin_without_gangs_is_place_batch(twin, oracle_b, use_mem):
    topo, free, mem, pods = synth.gen_c6(N=300, P=200)
    mem = mem if use_mem else None
    k1, f1 = twin(topo, free, pods, np.zeros(len(pods), np.int32), mem=mem, base=4)
    k2, f2 = oracle_b.place_batch(topo, free, pods, mem=mem, node_id_base=4)
    assert (k1 == k2).all() and (f1 == f2).all()


def test_twin_rejects_split_gang(twin):
    topo, free, pods = synth.gen_c2(N=10, P=4)
    with pytest.raises(ValueError):
        twin(topo, free, pods, np.array([1, 0, 1, 1], np.int32))


def test_gen_gangs_has_failing_and_placed_gangs(twin, oracle_b):
    topo, free, pods, gang = synth.gen_gangs(N=20_000, P=2000)
    assert set(pods[gang != 0, 0].tolist()) == {4, 8} and 0.2 < (gang != 0).mean() < 0.5
    for _, a, e in runs(gang):
        assert 2 <= e - a <= 8 and len(set(pods[a:e, 0].tolist())) == 1
    keys, _ = twin(topo, free, pods, gang)
    fails = [(keys[a:e] == NO_FIT).all() for _, a, e in runs(gang)]
    assert any(fails) and not all(fails)


# ---- the kernel on the CPU (tests/emu) -------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu():
    return cpu_libs.emu()


def emu_place(emu, topo, free, pods, gang, mem=None, base=0):
    from oracle import oracle_b
    f = np.array(free, dtype=np.int32, copy=True)
    topo, pods, gang = (np.ascontiguousarray(a, dtype=np.int32) for a in (topo, pods, gang))
    W = np.ascontiguousarray(oracle_b.DEFAULT_WEIGHTS, dtype=np.int32)
    keys = np.empty(len(pods), dtype=np.uint64)
    memp = None if mem is None else _p(np.ascontiguousarray(mem, dtype=np.int32))
    rc = emu.emu_place_batch_gang(_p(topo), _p(f), memp, len(f), base, _p(pods), _p(gang), len(pods), _p(W), _p(keys, ctypes.c_uint64))
    assert rc == 0
    return keys, f


@pytest.mark.parametrize("name", ["edges", "chunk", "views", "one_node"])
def test_emulated_gang_placement_matches_twin(emu, twin, name):
    topo, free, pods, gang, mem = SMALL_CASES[name]()
    keys, f = emu_place(emu, topo, free, pods, gang, mem=mem, base=21)
    want, wf = twin(topo, free, pods, gang, mem=mem, base=21)
    assert (keys == want).all() and (f == wf).all()
    assert any((want[a:e] == NO_FIT).all() for _, a, e in runs(gang))


def test_gang_edge_cases_are_what_they_claim(oracle_b):
    """Where each gang of the hand-made batches misses, from the oracle's plain sequential placement."""
    topo, free, pods, gang, _ = edge_batch()
    assert miss_at(oracle_b, topo, free, pods, gang) == {1: None, 2: 6, 3: 6, 4: 0, 5: None, 6: 0, 7: None, 8: 0, 9: None, 10: 1}
    topo, free, pods, gang, _ = chunk_batch()
    assert miss_at(oracle_b, topo, free, pods, gang) == {5: 8, 6: None}


def test_emulated_gang_placement_uncached_supertiles(emu, twin, oracle_b):
    topo, free, pods, gang, mem = wide_batch()
    assert len(set(pods[:, 3].tolist())) == 8
    keys, f = emu_place(emu, topo, free, pods, gang, mem=mem)
    want, wf = twin(topo, free, pods, gang, mem=mem)
    assert (keys == want).all() and (f == wf).all()
    placed = [bool((want[a:e] != NO_FIT).all()) for _, a, e in runs(gang)]
    assert any(placed) and not all(placed)


# ---- build products ----------------------------------------------------------------------------------------------------
def test_gang_kernel_has_no_spills():
    """Both instantiations of place_sequential: no local memory, and the static shared memory plus the dynamic
    supertile minima (2 x 36 KB) fit in one block's 227 KB."""
    if shutil.which("cuobjdump") is None or not os.path.exists(_lib.LIB_PATH):
        pytest.skip("cuobjdump or libkgpu.so missing")
    out = subprocess.run(["cuobjdump", "-res-usage", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    found = {}
    lines = out.splitlines()
    for i, line in enumerate(lines):
        m = re.search(r"Function (_ZN4kgpu16place_sequentialILb([01])EE\S*):", line)
        if m:
            usage = lines[i + 1]
            found[m.group(2)] = usage
            assert re.search(r"STACK:0\b", usage) and re.search(r"LOCAL:0\b", usage), usage
            shared = int(re.search(r"SHARED:(\d+)", usage).group(1))
            assert shared + 2 * 4608 * 8 <= 227 * 1024, usage
    assert set(found) == {"0", "1"}, sorted(found)


# ---- the device path -----------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_place_batch_gang_c2_size(twin, oracle_b):
    """gen_gangs at C2's size (100k nodes, 10k pods, a third of them in gangs): every key and mask, then a second
    cycle on the state the first one left."""
    from kubegpu_b200.scorer import Scorer
    topo, free, pods, gang = synth.gen_gangs()
    want, wf = twin(topo, free, pods, gang)
    assert any((want[a:e] == NO_FIT).all() for _, a, e in runs(gang))
    with Scorer((0,)) as s:
        s.upload_nodes(topo, free)
        got = s.place_batch(pods, gang=gang)
        assert (got == want).all() and (s.get_free_masks() == wf).all()
        more, mf = twin(topo, wf, pods[:3000], gang[:3000])
        assert (s.place_batch(pods[:3000], gang=gang[:3000]) == more).all() and (s.get_free_masks() == mf).all()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["edges", "chunk", "views", "one_node", "wide"])
def test_place_batch_gang_small_cases(twin, oracle_b, name):
    from kubegpu_b200.scorer import Scorer
    topo, free, pods, gang, mem = dict(SMALL_CASES, wide=wide_batch)[name]()
    want, wf = twin(topo, free, pods, gang, mem=mem, base=21)
    with Scorer((0,)) as s:
        s.upload_nodes(topo, free, node_id_base=21)
        if mem is not None:
            s.upload_gpu_memory(mem)
        assert (s.place_batch(pods, gang=gang) == want).all() and (s.get_free_masks() == wf).all()


@pytest.mark.gpu
def test_place_batch_gang_dry_run(twin, oracle_b):
    """The dry run proposes what the committing run places and leaves the masks alone."""
    from kubegpu_b200.scorer import Scorer
    topo, free, pods, gang = synth.gen_gangs(N=20_000, P=3000)
    with Scorer((0,)) as s:
        s.upload_nodes(topo, free)
        before = s.get_free_masks()
        dry = s.place_batch(pods, dry_run=True, gang=gang)
        assert (s.get_free_masks() == before).all()
        assert (s.place_batch(pods, gang=gang) == dry).all()
        want, wf = twin(topo, free, pods, gang)
        assert (dry == want).all() and (s.get_free_masks() == wf).all()


@pytest.mark.gpu
def test_place_batch_gang_rejects_split_ids(oracle_b):
    from kubegpu_b200.scorer import KgpuError, Scorer
    topo, free, pods = synth.gen_c2(N=1000, P=6)
    with Scorer((0,)) as s:
        s.upload_nodes(topo, free)
        with pytest.raises(KgpuError) as e:
            s.place_batch(pods, gang=np.array([3, 3, 0, 4, 3, 3], np.int32))
        assert e.value.code == _lib.ERR_INVALID and "two separate runs" in str(e.value)
        assert (s.get_free_masks() == free).all()
        with pytest.raises(ValueError):
            s.place_batch(pods, gang=np.zeros(5, np.int32))


def _node_line(name, shape, ids):
    from oracle import oracle_a as oa
    res = oa.shape_to_resources(shape)
    res = {k.replace("/gpu/%d/" % i, "/gpu/%s/" % ids[i]): v for i, k in enumerate(sorted(res, key=lambda s: int(s.split("/gpu/")[1].split("/")[0])))
           for v in [res[k]]}
    return "addnode %s %d %s" % (name, sum(sum(g) for g in shape), " ".join("%s=%d" % kv for kv in sorted(res.items())))


@pytest.mark.gpu
def test_host_mirror_places_gangs_in_caller_order(twin, oracle_b):
    """sched_cli: gang ids that collide in 32 bits stay apart, members move up to their gang's first member, and the
    placements come back in the caller's order; ProposeBatch proposes exactly what PlaceBatch then places."""
    if not os.path.exists(CLI):
        subprocess.check_call(["make", "-s", "-C", ROOT, "kubegpu_b200/lib/kgpu_sched_cli"])
    ids = ["GPU-%02d" % i for i in range(8)]
    # caller order, with (k, gang id); 7 and 7 + 2**32 are different gangs
    spec = [("s1", 2, 0), ("a1", 4, 7), ("s2", 2, 0), ("b1", 4, 7 + 2 ** 32), ("a2", 4, 7), ("b2", 8, 7 + 2 ** 32), ("s3", 4, 0)]
    names = " ".join(n for n, _, _ in spec)
    script = "\n".join([_node_line("A", [[2, 2], [2, 2]], ids), _node_line("B", [[4], [2, 2]], ids)] +
                       ["pod %s gang=%d run c req=%d" % (n, g, k) for n, k, g in spec] +
                       ["proposebatch " + names, "placebatch " + names]) + "\n"
    got = subprocess.run([CLI], input=script, capture_output=True, text=True, check=True).stdout
    # what the device sees: s1, a1, a2, s2, b1, b2, s3 with gangs 0, 1, 1, 0, 2, 2, 0
    dev = [0, 1, 4, 2, 3, 5, 6]
    pods = synth.make_pods(np.array([spec[i][1] for i in dev], np.int32))
    tA, tB = synth.shape_matrix([[2, 2], [2, 2]]), synth.shape_matrix([[4], [2, 2]])
    want, _ = twin(np.stack([tA, tB]), np.array([0xFF, 0xFF], np.int32), pods, np.array([0, 1, 1, 0, 2, 2, 0], np.int32))
    by_name = {spec[i][0]: want[j] for j, i in enumerate(dev)}
    assert by_name["b1"] == NO_FIT and by_name["b2"] == NO_FIT and by_name["s3"] != NO_FIT
    lines = []
    for n, _, _ in spec:
        u = oracle_b.unpack_key(by_name[n])
        lines.append("  %s fits=0 cost=0 node= mask=0x00" % n if u is None else
                     "  %s fits=1 cost=%d node=%s mask=0x%02x" % (n, u[0], "AB"[u[1]], u[2]))
    for cmd in ("proposebatch", "placebatch"):
        out = got.split("> %s %s\n" % (cmd, names))[1].splitlines()
        assert out[0] == "  err=" and out[1:8] == lines, (cmd, out)
