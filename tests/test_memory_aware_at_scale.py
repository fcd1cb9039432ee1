"""Memory-aware scoring (K1m: the MEM instantiation of score_pairs_sparse and its dense counterparts in score_pairs.cuh)
checked on EVERY pod of full-size batches, and at the requirement values where an eligibility test goes wrong.

Under snapshot scoring a pod's key depends on the pod only through k and the set of GPUs its requirement leaves
eligible.  Every uploaded memory value lies in V, the cluster's distinct values, so `mem >= need` holds exactly when
`mem >= ceil_V(need)` (the smallest value of V at or above need).  A batch therefore falls into at most 9 x (|V| + 2)
classes; class_keys runs Oracle B once per class and scatters the answer back to every pod.  That is exact, not a
sample, so C6's 10k pods x 100k nodes are checked in seconds.  The reduction itself is checked against the plain oracle
on the CPU.

The adversarial cluster plants, per GPU memory class, a node with eight free GPUs on weight-0 links whose GPUs all carry
exactly that class, plus nodes with 0-MiB and INT32_MAX-MiB GPUs.  The adversarial batch asks for every class value v,
v - 1 and v + 1, 0, negative values, 1, INT32_MAX, and for runs of values that share K1m's min_mem hash sub-bucket but
not their eligibility class (the kernel rebuilds its penalised costs whenever the requirement changes)."""
import ctypes
import os
import time

import numpy as np
import pytest

import cpu_libs
from kubegpu_b200 import _lib, synth

INT32_MAX = 2**31 - 1
CLASSES = synth.GPU_MEM_CLASSES_MIB
FLAT_MAX = np.full(16, 4095, np.int32)              # every cost field bit in use: the general (non-byte) key format
NVLINK = 12                                          # an NVLink level: weight 0 in the default table
NTHREADS = os.cpu_count() or 1
VARIANTS = [_lib.VARIANT_AUTO, _lib.VARIANT_LANE_PER_NODE, _lib.VARIANT_WARP_PER_PAIR, _lib.VARIANT_MEMO_BY_K,
            _lib.VARIANT_TILE_MEMO, _lib.VARIANT_SPARSE]
# a SPARSE kgpu_score_batch with memory-constrained pods: any_mem_pod, then (sp_prepare_chunks +) K1s for the pods
# without a requirement and again for those with one
SPARSE_LAUNCHES = {True: 5, False: 3}
# values of one K1m min_mem sub-bucket ((w * 0x9E3779B1 mod 2^32) >> 30 == 1) in five different eligibility classes
SUB_SAME = (16_383, 16_385, 32_769, 81_920, 184_319, 2_147_483_646)


def _p(a, t=ctypes.c_int32):
    return a.ctypes.data_as(ctypes.POINTER(t))


def sub_bucket(w):
    return int((int(w) * 0x9E3779B1) & 0xFFFFFFFF) >> 30


def _timed(label, fn):
    t0 = time.perf_counter()
    out = fn()
    print("%s: %.2f s" % (label, time.perf_counter() - t0))
    return out


# ---- the class-collapsed reference ---------------------------------------------------------------------------------
def pod_classes(pods, mem):
    """(representative pod index per class, class of every pod).  A class is (canonical k, canonical need): k outside
    0..8 is one invalid value; need <= 0, or no memory uploaded, is 0; otherwise ceil_V(need), or max(V) + 1 when no
    value of V is that large."""
    pods = np.asarray(pods, np.int32).reshape(-1, 4)
    k = pods[:, 0].astype(np.int64)
    k = np.where((k >= 0) & (k <= 8), k, 9)
    need = pods[:, 3].astype(np.int64)
    if mem is None:
        canon = np.zeros(len(pods), np.int64)
    else:
        V = np.unique(np.asarray(mem, np.int64))
        pos = np.searchsorted(V, need, side="left")
        ceil = np.where(pos < len(V), V[np.minimum(pos, len(V) - 1)], V[-1] + 1)
        canon = np.where(need <= 0, 0, ceil)
    _, first, inverse = np.unique(k * (1 << 33) + canon, return_index=True, return_inverse=True)
    return first, inverse.reshape(-1)


def class_keys(oracle_b, topo, free, pods, W, base, mem):
    """Oracle B's keys for every pod, from one oracle call on one representative pod per class."""
    pods = np.asarray(pods, np.int32).reshape(-1, 4)
    first, inverse = pod_classes(pods, mem)
    rep = oracle_b.score_batch(topo, free, pods[first], W, node_id_base=base, fast=True, nthreads=NTHREADS, mem=mem)
    return rep[inverse]


# ---- the adversarial cluster and batch -----------------------------------------------------------------------------
def planted_nodes(N):
    """One node per memory class, in increasing class order: near node 0, a third in, the middle, the last node."""
    return [3, N // 3 + 5, N // 2 + 1, N - 1]


def adversarial_cluster(N, zero=True, top=True, seed=0):
    """gen_c6's nodes with a node of eight free GPUs on weight-0 links planted per memory class (all its GPUs carry
    exactly that class), and a few nodes with 0-MiB GPUs (zero) and INT32_MAX-MiB GPUs (top), whole or every other
    GPU.  Returns (topo, free, mem)."""
    topo, free, mem, _ = synth.gen_c6(N=N, P=0)
    topo, free, mem = topo.copy(), free.copy(), mem.copy()
    nv = np.full((8, 8), NVLINK, np.int32)
    np.fill_diagonal(nv, 0)
    planted = planted_nodes(N)
    for v, i in zip(CLASSES, planted):
        topo[i], free[i], mem[i] = nv.reshape(64), 0xFF, v
    rng = np.random.default_rng(seed)
    special = rng.choice(np.setdiff1d(np.arange(N), planted), size=16, replace=False)
    if zero:
        mem[special[:4]] = 0
        mem[special[4:8], ::2] = 0
    if top:
        mem[special[8:12]] = INT32_MAX
        mem[special[12:], 1::2] = INT32_MAX
        free[special[8:12]] = 0xFF
    return np.ascontiguousarray(topo), np.ascontiguousarray(free), np.ascontiguousarray(mem)


def boundary_requirements():
    vals = {0, -1, -(2**31), 1, 16_384, 81_920, CLASSES[-1] + 1, 1_000_000, INT32_MAX - 1, INT32_MAX}
    for v in CLASSES:
        vals |= {v - 1, v, v + 1}
    return np.array(sorted(vals), np.int64)


def adversarial_pods(P, seed=0):
    """k mostly 1..8, some 0 and some outside 0..8; a quarter of the pods keep no requirement, the others draw one of
    boundary_requirements().  Inside the second chunk of 512 pods (the first for P < 1024), runs of one k whose
    requirements alternate through SUB_SAME."""
    rng = np.random.default_rng(seed)
    k = rng.integers(1, 9, size=P)
    u = rng.random(P)
    k[u < 0.04] = 0
    odd = (u >= 0.04) & (u < 0.07)
    k[odd] = rng.choice([-7, -1, 9, 100], size=int(odd.sum()))
    pods = synth.make_pods(k.astype(np.int32))
    has = rng.random(P) < 0.75
    pods[has, 3] = rng.choice(boundary_requirements(), size=int(has.sum())).astype(np.int32)
    start = 552 if P >= 1024 else 0
    for j, kk in enumerate((2, 4, 8, 1, 6, 3)):
        b, e = min(P, start + 36 * j), min(P, start + 36 * (j + 1))
        pods[b:e, 0] = kk
        pods[b:e, 3] = np.resize(np.array(SUB_SAME, np.int32), e - b)
    return pods


def distinct_pods(pods):
    """bench.py's noncollapsible batch: C6's pods, every one with its own min_mem."""
    p7 = pods.copy()
    p7[:, 3] = 1_000 + (synth.rand_below(synth.SEED_C6, 21, len(p7), 180_000) // 10_000) * 10_000 + np.arange(len(p7)) % 10_000
    return p7


def assert_keys(got, want, pods, what):
    bad = np.flatnonzero(got != want)
    if len(bad):
        i = int(bad[0])
        raise AssertionError("%s: %d of %d keys differ; first at pod %d (k %d, min_mem %d): got %x, want %x"
                             % (what, len(bad), len(want), i, pods[i, 0], pods[i, 3], int(got[i]), int(want[i])))


# ---- CPU: the reduction and the batch ------------------------------------------------------------------------------
def test_sub_same_shares_a_bucket_not_a_class():
    assert {sub_bucket(w) for w in SUB_SAME} == {1}
    V = sorted(set(CLASSES) | {INT32_MAX})
    assert len({next(v for v in V if v >= w) for w in SUB_SAME}) == 5
    assert (16_384 & 0xFFFF) == (81_920 & 0xFFFF)


@pytest.mark.parametrize("memkind", ["none", "with_zero", "with_int32_max", "both"])
def test_class_keys_equal_the_plain_oracle(oracle_b, memkind):
    """The reduction equals Oracle B's plain (all-subsets, one pod at a time) definition on every pod."""
    topo, free, mem = adversarial_cluster(2000, zero=memkind in ("with_zero", "both"), top=memkind in ("with_int32_max", "both"))
    if memkind == "none":
        mem = None
    else:
        assert (0 in mem) == (memkind != "with_int32_max") and (INT32_MAX in mem) == (memkind != "with_zero")
    pods = adversarial_pods(3000, seed=len(memkind))
    for W, base in ((oracle_b.DEFAULT_WEIGHTS, 0), (FLAT_MAX, 11)):
        want = oracle_b.score_batch(topo, free, pods, W, node_id_base=base, mem=mem)
        assert_keys(class_keys(oracle_b, topo, free, pods, W, base, mem), want, pods, memkind)
    first, _ = pod_classes(pods, mem)
    assert len(first) <= 10 * ((len(np.unique(mem)) if mem is not None else 0) + 2)     # k = 0..8 or invalid


def test_adversarial_batch_is_not_vacuous(oracle_b):
    """Every v / v + 1 pair of a class value leads to different keys for some k, and most constrained pods get keys
    that differ from their unconstrained ones."""
    topo, free, mem = adversarial_cluster(2000)
    W = oracle_b.DEFAULT_WEIGHTS
    probe = synth.make_pods(np.repeat(np.arange(1, 9, dtype=np.int32), 2 * len(CLASSES)))
    probe[:, 3] = np.tile(np.array([[v, v + 1] for v in CLASSES], np.int32).reshape(-1), 8)
    keys = class_keys(oracle_b, topo, free, probe, W, 0, mem).reshape(8, len(CLASSES), 2)
    assert (keys[:, :, 0] != keys[:, :, 1]).any(axis=0).all()
    pods = adversarial_pods(3000)
    want = class_keys(oracle_b, topo, free, pods, W, 0, mem)
    plain = class_keys(oracle_b, topo, free, pods, W, 0, None)
    constrained = (pods[:, 3] > 0) & (pods[:, 0] >= 1) & (pods[:, 0] <= 8)
    assert (want[constrained] != plain[constrained]).mean() > 0.5
    assert (want[pods[:, 3] <= 0] == plain[pods[:, 3] <= 0]).all()


# ---- CPU: the kernels through the emulator ------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu():
    return cpu_libs.emu()


@pytest.fixture(scope="module")
def small_cluster():
    return adversarial_cluster(600)


def _emu_sparse(emu, topo, free, mem, pods, W, splits, base):
    keys = np.zeros(len(pods), np.uint64)
    route = emu.emu_score_sparse(_p(topo), _p(free), None if mem is None else _p(mem), ctypes.c_int64(len(free)), ctypes.c_int64(base),
                                 _p(pods), ctypes.c_int64(len(pods)), _p(np.asarray(W, np.int32)), splits, _p(keys, ctypes.c_uint64))
    return keys, route


@pytest.mark.parametrize("wname", ["default", "flat_max"])
@pytest.mark.parametrize("with_mem", [True, False])
def test_emulated_sparse_routes(oracle_b, emu, small_cluster, wname, with_mem):
    """K1s + its MEM instantiation on every route: the plain grid, the work list with the blocks' own sort, prepared
    chunk tables, and (few pods) runs of tiles on the streaming and TMA instantiations.  Without an upload every GPU's
    memory is unlimited: INT32_MAX requirements exclude nothing."""
    topo, free, mem = small_cluster
    mem = mem if with_mem else None
    W = oracle_b.DEFAULT_WEIGHTS if wname == "default" else FLAT_MAX
    byte = 8 if wname == "default" else 0
    pods = adversarial_pods(1100, seed=5)
    want = class_keys(oracle_b, topo, free, pods, W, 7, mem)
    # (pods, splits, route): 0 = every block sorts its pods, 1 = prepared chunk tables, 2 = STREAM, 3 = TMA
    for P, splits, route in ((1100, 3, 0), (1100, -64, 0), (1100, -2, 1), (400, -8, 2), (60, -8, 3)):
        got, r = _emu_sparse(emu, topo, free, mem, pods[:P], W, splits, 7)
        assert r == route | 4 | byte, (P, splits, r)
        assert_keys(got, want[:P], pods, "P %d splits %d" % (P, splits))


@pytest.mark.parametrize("wname, resident", [("default", 1), ("flat_max", 4)])
def test_emulated_prepared_chunks(oracle_b, emu, small_cluster, wname, resident):
    """emu_score_chunks on a chunk-aligned list: sp_prepare_chunks<true> builds the MEM tables, the blocks copy them."""
    topo, free, mem = small_cluster
    W = oracle_b.DEFAULT_WEIGHTS if wname == "default" else FLAT_MAX
    pods = adversarial_pods(1100, seed=resident)
    want = class_keys(oracle_b, topo, free, pods, W, 3, mem)
    for prepare in (1, 0):
        keys = np.zeros(len(pods), np.uint64)
        aligned = emu.emu_score_chunks(_p(topo), _p(free), _p(mem), ctypes.c_int64(len(free)), ctypes.c_int64(3), _p(pods),
                                       ctypes.c_int64(len(pods)), _p(np.asarray(W, np.int32)), ctypes.c_int64(resident), prepare,
                                       _p(keys, ctypes.c_uint64))
        assert aligned == 1
        assert_keys(keys, want, pods, "prepare %d" % prepare)


@pytest.mark.parametrize("variant", [0, 3, 4])
def test_emulated_dense_k1m(oracle_b, emu, small_cluster, variant):
    """The dense kernels: K1 + K1m as LANE_PER_NODE launches them (0), memo by k (3), tile memo (4).  (Warp per pair is
    too slow to emulate at this size; the GPU tests run it.)"""
    topo, free, mem = small_cluster
    W = np.asarray(oracle_b.DEFAULT_WEIGHTS, np.int32)
    pods = adversarial_pods(1100, seed=9)
    keys = np.zeros(len(pods), np.uint64)
    args = [_p(topo), _p(free), _p(mem), ctypes.c_int64(len(free)), ctypes.c_int64(5), _p(pods), ctypes.c_int64(len(pods)), _p(W), 3,
            _p(keys, ctypes.c_uint64)]
    if variant == 0:
        emu.emu_score_dense(*args)
    else:
        emu.emu_score_variant(variant, *args)
    assert_keys(keys, class_keys(oracle_b, topo, free, pods, W, 5, mem), pods, "variant %d" % variant)


# ---- GPU -----------------------------------------------------------------------------------------------------------
def score_twice(s, pods):
    """Keys of a repeated score_batch call and the launches it made (the first call built the work list and caches)."""
    s.score_batch(pods)
    l0 = s.kernel_launches
    keys = s.score_batch(pods)
    return keys, s.kernel_launches - l0


@pytest.fixture(scope="module")
def c6_full(oracle_b):
    """gen_c6 at full size with 10 037 pods (its first 10 000 are C6's batch), bench.py's all-distinct batch, and the
    reference keys of both."""
    topo, free, mem, pods = _timed("gen_c6 100k", lambda: synth.gen_c6(P=10_037))
    batches = {"c6": pods, "distinct": distinct_pods(pods)}
    want = {name: _timed("oracle %s (%d classes)" % (name, len(pod_classes(pp, mem)[0])),
                         lambda pp=pp: class_keys(oracle_b, topo, free, pp, oracle_b.DEFAULT_WEIGHTS, 0, mem))
            for name, pp in batches.items()}
    return topo, free, mem, batches, want


@pytest.fixture(scope="module")
def adv100k(oracle_b):
    """The adversarial cluster at 100k nodes and a 4 000-pod adversarial batch (8 chunks: chunk-aligned on 132 SMs)."""
    topo, free, mem = _timed("adversarial cluster 100k", lambda: adversarial_cluster(100_000))
    pods = adversarial_pods(4000, seed=1)
    want = {name: _timed("oracle adversarial %s" % name, lambda W=W: class_keys(oracle_b, topo, free, pods, W, 0, mem))
            for name, W in (("default", oracle_b.DEFAULT_WEIGHTS), ("flat_max", FLAT_MAX))}
    return topo, free, mem, pods, want


@pytest.mark.gpu
@pytest.mark.parametrize("variant", VARIANTS)
def test_gpu_c6_full_size(c6_full, variant):
    """C6 (100k nodes) with its 10 000 pods and the all-distinct batch, and both at a ragged 10 037: every key.  SPARSE
    runs the prepared MEM route (5 launches); a 513-pod batch is below the alignment threshold (3 launches)."""
    from kubegpu_b200.scorer import Scorer
    topo, free, mem, batches, want = c6_full
    with Scorer((0,)) as s:
        s.set_variant(variant)
        s.upload_nodes(topo, free)
        s.upload_gpu_memory(mem)
        for name, pods in batches.items():
            for P in (10_000, 10_037, 513):
                got, launches = score_twice(s, pods[:P])
                print("variant %d %s P %d: %.3f ms, %d launches" % (variant, name, P, s.last_kernel_ms, launches))
                assert_keys(got, want[name][:P], pods, "variant %d %s P %d" % (variant, name, P))
                if variant == _lib.VARIANT_SPARSE:
                    assert launches == SPARSE_LAUNCHES[P > 513]


@pytest.mark.gpu
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("wname", ["default", "flat_max"])
def test_gpu_adversarial_100k(adv100k, variant, wname):
    """The adversarial batch on the adversarial cluster at 100k nodes, with byte keys (default weights) and the general
    key format (flat_max)."""
    from kubegpu_b200.scorer import Scorer
    topo, free, mem, pods, want = adv100k
    with Scorer((0,)) as s:
        s.set_variant(variant)
        if wname == "flat_max":
            s.set_weights(FLAT_MAX)
        s.upload_nodes(topo, free)
        s.upload_gpu_memory(mem)
        got, launches = score_twice(s, pods)
        print("variant %d %s: %.3f ms, %d launches" % (variant, wname, s.last_kernel_ms, launches))
        assert_keys(got, want[wname], pods, "variant %d %s" % (variant, wname))
        if variant == _lib.VARIANT_SPARSE:
            assert launches == SPARSE_LAUNCHES[True]


@pytest.mark.gpu
@pytest.mark.parametrize("variant", [_lib.VARIANT_SPARSE, _lib.VARIANT_AUTO])
def test_gpu_device_entry(oracle_b, adv100k, variant):
    """score_batch_device on a non-default stream (the device flag decides which pods K1m takes): the adversarial batch,
    then the same batch with every min_mem zeroed, where the MEM launches run and must leave every key alone.  Before
    the memory is uploaded no requirement excludes a GPU, INT32_MAX included."""
    import torch
    from kubegpu_b200.scorer import Scorer
    topo, free, mem, pods, want = adv100k
    nomem = pods.copy()
    nomem[:, 3] = 0
    plain = class_keys(oracle_b, topo, free, nomem, oracle_b.DEFAULT_WEIGHTS, 0, None)
    stream = torch.cuda.Stream()
    d_keys = torch.empty(len(pods), dtype=torch.int64, device="cuda")

    def run(s, batch):
        d_pods = torch.from_numpy(batch).cuda()
        torch.cuda.synchronize()
        l0 = s.kernel_launches
        s.score_batch_device(d_pods.data_ptr(), len(batch), d_keys.data_ptr(), stream.cuda_stream)
        stream.synchronize()
        return d_keys.cpu().numpy().view(np.uint64).copy(), s.kernel_launches - l0

    with Scorer((0,)) as s:
        s.set_variant(variant)
        s.upload_nodes(topo, free)
        got, _ = run(s, pods)
        assert_keys(got, plain, pods, "before the memory upload")
        s.upload_gpu_memory(mem)
        run(s, pods)
        got, launches = run(s, pods)
        assert_keys(got, want["default"], pods, "adversarial")
        assert launches == 5
        got, launches = run(s, nomem)
        assert_keys(got, plain, nomem, "min_mem zeroed")
        assert launches == 5


@pytest.mark.gpu
def test_gpu_stale_order(oracle_b, adv100k):
    """After a scored call, fewer than n / 200 nodes of the lowest classes become all-free (some with class-boundary
    memory, some with all-NVLink links): every key is right on the stale order, and the next call re-sorts nothing.
    Crossing n / 200 changed nodes, the call re-sorts (build_order: 3 launches, compact_nodes over every slot: 1)."""
    from kubegpu_b200.scorer import Scorer
    topo, free, mem, pods, _ = adv100k
    topo, free, mem = topo.copy(), free.copy(), mem.copy()
    N = len(free)
    W = oracle_b.DEFAULT_WEIGHTS
    pop = np.array([bin(int(f) & 0xFF).count("1") for f in free])
    low = np.flatnonzero(pop <= 1)
    rng = np.random.default_rng(3)
    rng.shuffle(low)
    first, second = low[:400], low[400:600]
    nv = np.full((8, 8), NVLINK, np.int32)
    np.fill_diagonal(nv, 0)
    boundary = [np.full(8, v, np.int32) for v in CLASSES] + [np.array([0, INT32_MAX] * 4, np.int32),
                                                               np.array([CLASSES[0], CLASSES[0] - 1] * 4, np.int32)]
    with Scorer((0,)) as s:
        s.set_variant(_lib.VARIANT_SPARSE)
        s.upload_nodes(topo, free)
        s.upload_gpu_memory(mem)
        s.score_batch(pods)
        free[first] = 0xFF
        s.set_free_masks(first, free[first])
        for j, i in enumerate(first[:60]):
            mem[i] = boundary[j % len(boundary)]
            s.update_gpu_memory(int(i), mem[i])
        for i in first[60:100]:
            topo[i] = nv.reshape(64)
            s.update_node(int(i), topo[i], int(free[i]))
        assert (400 + 40) * 200 <= N
        l0 = s.kernel_launches
        got = s.score_batch(pods)
        assert s.kernel_launches - l0 == SPARSE_LAUNCHES[True]           # no re-sort
        want = class_keys(oracle_b, topo, free, pods, W, 0, mem)
        assert_keys(got, want, pods, "stale order")
        free[second] = 0xFF
        s.set_free_masks(second, free[second])
        l0 = s.kernel_launches
        got = s.score_batch(pods)
        assert s.kernel_launches - l0 == SPARSE_LAUNCHES[True] + 3 + 1   # re-sorted
        assert_keys(got, class_keys(oracle_b, topo, free, pods, W, 0, mem), pods, "after the re-sort")


@pytest.mark.gpu
def test_gpu_one_million_nodes(oracle_b):
    """C6 at 1M nodes (the adversarial cluster) with 2 048 adversarial pods and node ids at the top of the 32-bit field:
    the prepared MEM route on about 7 800 tiles."""
    from kubegpu_b200.scorer import Scorer
    N = 1_000_000
    base = 2**32 - 1 - N
    topo, free, mem = _timed("adversarial cluster 1M", lambda: adversarial_cluster(N))
    pods = adversarial_pods(2048, seed=2)
    want = _timed("oracle 1M", lambda: class_keys(oracle_b, topo, free, pods, oracle_b.DEFAULT_WEIGHTS, base, mem))
    with Scorer((0,)) as s:
        s.set_variant(_lib.VARIANT_SPARSE)
        s.upload_nodes(topo, free, node_id_base=base)
        s.upload_gpu_memory(mem)
        got, launches = score_twice(s, pods)
        print("1M nodes: %.3f ms, %d launches" % (s.last_kernel_ms, launches))
    assert launches == SPARSE_LAUNCHES[True]
    assert_keys(got, want, pods, "1M nodes")
    assert (got[got != _lib.NO_FIT] >> np.uint64(8) & np.uint64(0xFFFFFFFF)).max() >= base + N // 2


def seven_requirements():
    return np.array([CLASSES[0], CLASSES[0] + 1, CLASSES[1], CLASSES[2] + 1, CLASSES[3], CLASSES[3] + 1, INT32_MAX], np.int32)


@pytest.mark.gpu
def test_gpu_pairs_place_preempt(oracle_b):
    """Per-pair queries with the adversarial requirements against node_key on the eligible mask; K3 (place_batch) and
    preempt_batch with seven boundary requirements against Oracle B's sequential placement and the preemption twin."""
    from kubegpu_b200.scorer import Scorer
    topo, free, mem = adversarial_cluster(20_000)
    rng = np.random.default_rng(4)
    W = oracle_b.DEFAULT_WEIGHTS
    n = 20_000
    idx = np.concatenate([rng.integers(0, n, size=n - 40), np.repeat(planted_nodes(n), 10)]).astype(np.int64)
    ks = rng.integers(0, 9, size=len(idx)).astype(np.int32)
    mm = rng.choice(boundary_requirements(), size=len(idx)).astype(np.int32)
    mm[-40:] = np.resize(np.array(SUB_SAME, np.int32), 40)
    elig = np.array([int(free[i]) & (sum(1 << g for g in range(8) if mem[i][g] >= m) if m > 0 else 0xFF)
                     for i, m in zip(idx, mm)])
    want_pairs = np.array([oracle_b.node_key(topo[i], f, int(k)) for i, f, k in zip(idx, elig, ks)], np.uint32)
    pods = adversarial_pods(600, seed=6)
    pods[:, 3] = np.where(pods[:, 3] > 0, rng.choice(seven_requirements(), size=len(pods)), pods[:, 3])
    pods[:, 0] = np.clip(pods[:, 0], 0, 8)
    want_place, free_after = _timed("oracle place_batch", lambda: oracle_b.place_batch(topo, free, pods, W, mem=mem))
    topo_p, free_p, hold, ppods, lvl = synth.gen_preempt(N=n, P=1000)
    ppods[:, 3] = np.where(rng.random(len(ppods)) < 0.7, rng.choice(seven_requirements(), size=len(ppods)), 0)
    L = cpu_libs.twin("preempt")
    want_pk = np.empty(len(ppods), np.uint64)
    want_pv = np.empty(len(ppods), np.uint32)
    L.preempt_twin_batch(_p(topo_p), _p(free_p), _p(mem), _p(hold), n, 0, _p(ppods), _p(lvl), len(ppods), _p(np.asarray(W, np.int32)),
                         NTHREADS, _p(want_pk, ctypes.c_uint64), _p(want_pv, ctypes.c_uint32))
    with Scorer((0,)) as s:
        s.upload_nodes(topo, free)
        unlimited = s.score_pairs(idx[:50], ks[:50], np.full(50, INT32_MAX, np.int32))
        assert (unlimited == s.score_pairs(idx[:50], ks[:50])).all()     # nothing uploaded: INT32_MAX excludes nothing
        s.upload_gpu_memory(mem)
        got = s.score_pairs(idx, ks, mm)
        assert (got == want_pairs).all(), np.flatnonzero(got != want_pairs)[:10]
        keys = s.place_batch(pods)
        assert_keys(keys, want_place, pods, "place_batch")
        assert (s.get_free_masks() == free_after).all()
        s.upload_nodes(topo_p, free_p)
        s.upload_gpu_memory(mem)
        s.upload_holders(hold)
        pk, pv = s.preempt_batch(ppods, lvl)
    assert_keys(pk, want_pk, ppods, "preempt_batch")
    assert (pv == want_pv).all()
    assert (pv != 0).any() and (want_place != np.uint64(_lib.NO_FIT)).mean() > 0.5


@pytest.mark.gpu
def test_gpu_two_devices(c6_full, adv100k):
    """A two-device handle: each 50k-node shard is chunk-aligned, so both run the prepared MEM route (2 x 5 launches and
    the shard reduction)."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from kubegpu_b200.scorer import Scorer
    for topo, free, mem, pods, want in ((c6_full[0], c6_full[1], c6_full[2], c6_full[3]["c6"][:10_000], c6_full[4]["c6"][:10_000]),
                                        adv100k[:4] + (adv100k[4]["default"],)):
        with Scorer((0, 1)) as s:
            s.set_variant(_lib.VARIANT_SPARSE)
            s.upload_nodes(topo, free)
            s.upload_gpu_memory(mem)
            got, launches = score_twice(s, pods)
        assert launches == 2 * SPARSE_LAUNCHES[True] + 1
        assert_keys(got, want, pods, "two devices")
