"""The kernel SOURCES (kubegpu_b200/csrc/score_pairs*.cuh + generated enumeration) compiled with g++ against a
small CUDA shim (tests/emu/cuda_emu.h: one OS thread per CUDA thread, real barriers, emulated warp
collectives) and run on the CPU against the oracle.  Small sizes only -- this is a logic check that works
without a GPU (e.g. for kernel edits between GPU runs); bit-exactness on the H100 is tests/test_gpu_*.py."""
import ctypes

import numpy as np
import pytest

import cpu_libs
from kubegpu_b200 import synth


@pytest.fixture(scope="module")
def emu():
    return cpu_libs.emu()


def _run(fn, topo, free, pods, W, mem=None, base=0, splits=1):
    topo, free, pods, W = (np.ascontiguousarray(a, dtype=np.int32) for a in (topo, free, pods, W))
    P = pods.shape[0]
    keys = np.empty(P, dtype=np.uint64)
    p32 = ctypes.POINTER(ctypes.c_int32)
    memp = None if mem is None else np.ascontiguousarray(mem, dtype=np.int32).ctypes.data_as(p32)
    fn(topo.ctypes.data_as(p32), free.ctypes.data_as(p32), memp, free.shape[0], base, pods.ctypes.data_as(p32), P,
       W.ctypes.data_as(p32), splits, keys.ctypes.data_as(ctypes.POINTER(ctypes.c_uint64)))
    return keys


@pytest.mark.parametrize("kernel", ["sparse", "dense"])
def test_emulated_kernels_match_oracle(emu, oracle_b, kernel):
    fn = emu.emu_score_sparse if kernel == "sparse" else emu.emu_score_dense
    W = oracle_b.DEFAULT_WEIGHTS
    # C1 fixture, a C4 sample with k in 1..8 plus invalid k, two pod splits, a node-id base
    topo, free, pods = synth.gen_c1()
    assert (_run(fn, topo, free, pods, W) == oracle_b.score_batch(topo, free, pods, W)).all()
    topo, free, pods = synth.gen_c4(N=300, P=70)
    pods[5, 0], pods[6, 0], pods[7, 0] = 0, 9, -3
    want = oracle_b.score_batch(topo, free, pods, W, node_id_base=1000)
    assert (_run(fn, topo, free, pods, W, base=1000, splits=2) == want).all()
    # maximum weights (cost field at its largest) and everything free (K1s degenerates to the dense work)
    wmax = np.full(16, 4095, dtype=np.int32)
    full = np.full(130, 0xFF, dtype=np.int32)
    p9 = synth.make_pods(np.arange(0, 9, dtype=np.int32))
    assert (_run(fn, topo[:130], full, p9, wmax) == oracle_b.score_batch(topo[:130], full, p9, wmax)).all()


@pytest.mark.parametrize("kernel", ["sparse", "dense"])
def test_emulated_memory_aware_path(emu, oracle_b, kernel):
    fn = emu.emu_score_sparse if kernel == "sparse" else emu.emu_score_dense
    topo, free, mem, pods = synth.gen_c6(N=260, P=60)
    want = oracle_b.score_batch(topo, free, pods, mem=mem)
    assert (_run(fn, topo, free, pods, oracle_b.DEFAULT_WEIGHTS, mem=mem) == want).all()
    assert (want != oracle_b.score_batch(topo, free, pods)).any()


def _p(a, t=ctypes.c_int32):
    return a.ctypes.data_as(ctypes.POINTER(t))


@pytest.mark.parametrize("variant", [1, 3, 4])
def test_emulated_other_variants_match_oracle(emu, oracle_b, variant):
    """warp-per-pair (the north_star mapping), memo-by-k and tile-memo, incl. their memory-aware routes."""
    W = np.ascontiguousarray(oracle_b.DEFAULT_WEIGHTS, dtype=np.int32)
    topo, free, mem, pods = synth.gen_c6(N=200, P=40)
    pods[3, 0], pods[4, 0] = 0, 11
    for use_mem in (False, True):
        pp = pods.copy()
        if not use_mem:
            pp[:, 3] = 0
        keys = np.empty(len(pp), dtype=np.uint64)
        emu.emu_score_variant(variant, _p(topo), _p(free), _p(mem), ctypes.c_int64(len(free)), ctypes.c_int64(77), _p(pp),
                              ctypes.c_int64(len(pp)), _p(W), 2, _p(keys, ctypes.c_uint64))
        want = oracle_b.score_batch(topo, free, pp, W, node_id_base=77, mem=mem)
        assert (keys == want).all(), (variant, use_mem)


def test_emulated_reduce_shards(emu, oracle_b):
    rng = np.random.default_rng(5)
    g = rng.integers(0, 2**63, size=(4, 300), dtype=np.uint64)
    g[:, 7] = np.uint64(0xFFFFFFFFFFFFFFFF)
    out = np.empty(300, dtype=np.uint64)
    emu.emu_reduce_shards(_p(g, ctypes.c_uint64), 4, ctypes.c_int64(300), _p(out, ctypes.c_uint64))
    assert (out == g.min(axis=0)).all()


def test_emulated_pair_list(emu, oracle_b):
    W = np.ascontiguousarray(oracle_b.DEFAULT_WEIGHTS, dtype=np.int32)
    topo, free, mem, pods = synth.gen_c6(N=150, P=150)
    rng = np.random.default_rng(6)
    idx = rng.integers(0, 150, size=150).astype(np.int64)
    ks = np.ascontiguousarray(pods[:, 0]); mm = np.ascontiguousarray(pods[:, 3])
    out = np.empty(150, dtype=np.uint32)
    emu.emu_score_pair_list(_p(topo), _p(free), _p(mem), ctypes.c_int64(150), _p(idx, ctypes.c_longlong), _p(ks), _p(mm),
                            ctypes.c_int64(150), _p(W), _p(out, ctypes.c_uint32))
    for i in range(150):
        one = np.array([[ks[i], 0, 0, mm[i]]], dtype=np.int32)
        want = oracle_b.score_batch(topo[idx[i]:idx[i] + 1], free[idx[i]:idx[i] + 1], one, W, mem=mem[idx[i]:idx[i] + 1])[0]
        got = 0xFFFFFFFF if want == 0xFFFFFFFFFFFFFFFF else ((int(want) >> 40) << 8) | (int(want) & 0xFF)
        assert int(out[i]) == got, i


def _place(emu, topo, free, pods, W, mem=None, base=0):
    f = np.ascontiguousarray(free, dtype=np.int32).copy()
    pods = np.ascontiguousarray(pods, dtype=np.int32)
    keys = np.empty(len(pods), dtype=np.uint64)
    memp = None if mem is None else _p(np.ascontiguousarray(mem, dtype=np.int32))
    rc = emu.emu_place_batch(_p(np.ascontiguousarray(topo, dtype=np.int32)), _p(f), memp, ctypes.c_int64(len(f)),
                             ctypes.c_int64(base), _p(pods), ctypes.c_int64(len(pods)), _p(W), _p(keys, ctypes.c_uint64))
    return rc, keys, f


def test_emulated_sequential_placement(emu, oracle_b):
    """K3 (place_init + the persistent place_sequential block) against the stateful oracle."""
    W = np.ascontiguousarray(oracle_b.DEFAULT_WEIGHTS, dtype=np.int32)
    topo, free, pods = synth.gen_c4(N=300, P=120)
    pods[9, 0] = 0
    pods[10, 0] = 12
    rc, keys, f_emu = _place(emu, topo, free, pods, W, base=5)
    want_keys, want_free = oracle_b.place_batch(topo, free.copy(), pods, W, node_id_base=5)
    assert rc == 0 and (keys == want_keys).all() and (f_emu == want_free).all()


def test_emulated_sequential_placement_many_tiles(emu, oracle_b):
    """More than one supertile (33+ tiles) and a cluster that fills up: later pods find nothing."""
    W = np.ascontiguousarray(oracle_b.DEFAULT_WEIGHTS, dtype=np.int32)
    topo, free, _ = synth.gen_c2(N=128 * 34 + 17, P=0)
    free[:] = 0
    free[[5, 4300, 4368]] = [0x0F, 0xF0, 0xFF]           # three nodes with room, in different supertiles
    pods = synth.make_pods(np.array([4, 4, 2, 8, 4, 2, 1, 1, 1, 1, 1], dtype=np.int32))
    rc, keys, f_emu = _place(emu, topo, free, pods, W)
    want_keys, want_free = oracle_b.place_batch(topo, free.copy(), pods, W)
    assert rc == 0 and (keys == want_keys).all() and (f_emu == want_free).all()
    assert (keys == np.uint64(0xFFFFFFFFFFFFFFFF)).any() and f_emu.sum() == 0


def test_emulated_sequential_placement_memory_aware(emu, oracle_b):
    """Pods with min_mem: one table set ("view") per distinct requirement; 4 requirements + the plain view."""
    W = np.ascontiguousarray(oracle_b.DEFAULT_WEIGHTS, dtype=np.int32)
    topo, free, mem, pods = synth.gen_c6(N=300, P=150)
    assert len(set(pods[:, 3].tolist())) == 5
    rc, keys, f_emu = _place(emu, topo, free, pods, W, mem=mem, base=9)
    want_keys, want_free = oracle_b.place_batch(topo, free.copy(), pods, W, node_id_base=9, mem=mem)
    assert rc == 0 and (keys == want_keys).all() and (f_emu == want_free).all()
    plain_keys, _ = oracle_b.place_batch(topo, free.copy(), np.hstack([pods[:, :3], np.zeros((150, 1), np.int32)]), W, node_id_base=9)
    assert (plain_keys != want_keys).any()
    # without uploaded GPU memory the requirement excludes nothing (kgpu.h): same as the plain batch
    rc, keys, _ = _place(emu, topo, free, pods, W, mem=None, base=9)
    assert rc == 0 and (keys == plain_keys).all()
    # eight distinct requirements are one too many
    pods[:8, 3] = np.arange(1, 9) * 1000
    assert _place(emu, topo, free, pods, W, mem=mem)[0] == -1


@pytest.mark.parametrize("wmax", [2340, 2341])
def test_emulated_sparse_warp_key_layouts(emu, oracle_b, wmax):
    """2340 is the largest weight served by the byte-aligned warp key (cost < 2^16), 2341 the first that
    takes the general layout; both with ragged free masks so warps mix lanes that can and cannot serve k."""
    topo, free, pods = synth.gen_c4(N=400, P=90, seed=77)
    W = np.array([wmax - i for i in range(16)], dtype=np.int32)
    want = oracle_b.score_batch(topo, free, pods, W, node_id_base=3)
    assert (_run(emu.emu_score_sparse, topo, free, pods, W, base=3, splits=3) == want).all()


def test_emulated_sparse_work_list(emu, oracle_b):
    """K1s driven by the work list (per-tile pod ranges of about equal work, heaviest first) instead of the
    plain (tiles x splits) grid: same keys; every (tile, pod) covered exactly once."""
    W = oracle_b.DEFAULT_WEIGHTS
    topo, free, mem, pods = synth.gen_c6(N=900, P=700)
    pods[5, 0], pods[6, 0] = 0, 9
    want = oracle_b.score_batch(topo, free, pods, W, node_id_base=4, mem=mem)
    for resident in (1, 16, 1184):
        assert (_run(emu.emu_score_sparse, topo, free, pods, W, mem=mem, base=4, splits=-resident) == want).all(), resident


@pytest.mark.parametrize("P", [1, 31, 32, 512, 513, 1000, 10_000])
@pytest.mark.parametrize("resident", [1, 16, 1184])
def test_sparse_work_list_partitions_the_tile_pod_plane(emu, P, resident):
    """Every (tile, pod) cell is covered exactly once; items come heaviest first; pod ranges start on multiples of
    32; runs of several tiles only when the whole batch fits one chunk of the block's pod sort."""
    rng = np.random.default_rng(P + resident)
    ntile = 57 if P > 512 else 700
    tile_class = np.sort(rng.integers(0, 9, size=ntile).astype(np.uint8))[::-1].copy()      # the order puts class 8 first
    out = np.zeros((200_000, 4), dtype=np.int32)
    weight = np.zeros(200_000, dtype=np.int64)
    n = emu.emu_sparse_work(_p(tile_class, ctypes.c_uint8), ctypes.c_int64(ntile), ctypes.c_int64(P), ctypes.c_int64(resident),
                            _p(out), ctypes.c_int64(len(out)), _p(weight, ctypes.c_longlong), None)
    items, weight = out[:n], weight[:n]
    assert 1 <= n <= len(out)
    assert (np.diff(weight) <= 0).all() and (weight > 0).all()                     # heaviest first
    assert (items[:, 3] >= 1).all()
    if P > 512:
        assert (items[:, 3] == 1).all()
    else:
        assert ((items[:, 1] == 0) & (items[:, 2] == P)).all()                     # runs carry the whole (one-chunk) batch
        assert items[:, 3].max() <= 16
        if resident == 1:
            assert items[:, 3].max() > 1                                           # few resident blocks: tiles are grouped
    cover = np.zeros((ntile, P), dtype=np.int32)
    for t, b, e, nt in items:
        assert b % 32 == 0 and e > b and 0 <= t and t + nt <= ntile
        cover[t:t + nt, b:e] += 1
    assert (cover == 1).all()


def test_emulated_sparse_single_class_tiles(emu, oracle_b):
    """Tiles whose slots are one class in increasing node id take the flush's direct 32-bit min over the
    warp keys (warp index in the key); C2's few shapes make cost ties across warps and nodes the rule."""
    W = oracle_b.DEFAULT_WEIGHTS
    topo, free, pods = synth.gen_c2(N=300, P=64)
    free[:] = 0xFF
    free[[7, 100, 299]] = [0x0F, 0x00, 0x3C]              # stragglers form small mixed tail tiles
    pods = synth.make_pods(np.array([1, 2, 3, 4, 5, 6, 7, 8, 0] * 7, dtype=np.int32))
    want = oracle_b.score_batch(topo, free, pods, W, node_id_base=40)
    assert (_run(emu.emu_score_sparse, topo, free, pods, W, base=40, splits=2) == want).all()
    # the same with every pod's cheapest nodes taken away one by one: winners move across warps and tiles
    for taken in (0, 1, 2, 31, 32, 127, 128, 129):
        free[taken] = 0
        want = oracle_b.score_batch(topo, free, pods, W, node_id_base=40)
        assert (_run(emu.emu_score_sparse, topo, free, pods, W, base=40) == want).all(), taken


@pytest.mark.parametrize("kernel", ["sparse", "dense"])
def test_emulated_ragged_sizes(emu, oracle_b, kernel):
    """More pods than one shared-memory chunk (three chunks, the last one ragged), pod splits that do not
    divide the batch, a node count that fills neither a warp nor a tile, and a single node."""
    fn = emu.emu_score_sparse if kernel == "sparse" else emu.emu_score_dense
    W = oracle_b.DEFAULT_WEIGHTS
    topo, free, pods = synth.gen_c4(N=33, P=1100)
    want = oracle_b.score_batch(topo, free, pods, W, node_id_base=2**31 - 40)     # ids near the top of the 32-bit field
    assert (_run(fn, topo, free, pods, W, base=2**31 - 40, splits=3) == want).all()
    assert (_run(fn, topo[:1], free[:1], pods[:40], W) == oracle_b.score_batch(topo[:1], free[:1], pods[:40], W)).all()
    none_free = np.zeros(5, dtype=np.int32)
    got = _run(fn, topo[:5], none_free, pods[:16], W)
    assert (got == oracle_b.score_batch(topo[:5], none_free, pods[:16], W)).all()


def test_emulated_gather_and_min_single_rank(emu):
    """peer_exchange.cuh with world = 1: the keys land in the rank's slot and come back as the final keys (NO_FIT included),
    the local key array is left at NO_FIT for the next step's K1, the last block resets the ticket and publishes the epoch;
    P = 0 is a pure barrier.  (One block only: the emulation runs blocks one after the other, and every block of
    this kernel waits for the flag its rank's LAST block publishes -- on the GPU all blocks are resident.)"""
    P, MP = 250, 1000
    rng = np.random.default_rng(3)
    local = rng.integers(1, 2**60, size=P, dtype=np.uint64)
    local[::7] = np.uint64(0xFFFFFFFFFFFFFFFF)
    sent = local.copy()
    slots = rng.integers(1, 2**60, size=MP, dtype=np.uint64)           # stale content of an earlier epoch: must be overwritten
    final = np.zeros(MP, dtype=np.uint64)
    flags = np.zeros(16, dtype=np.uint32)
    ticket = np.zeros(1, dtype=np.uint32)
    err = np.zeros(1, dtype=np.int32)
    u64, u32 = ctypes.c_uint64, ctypes.c_uint32
    emu.emu_gather_and_min(_p(local, u64), ctypes.c_int64(P), ctypes.c_int64(MP), _p(slots, u64), _p(flags, u32), 1, _p(ticket, u32),
                           _p(final, u64), _p(err))
    assert (final[:P] == sent).all() and (slots[:P] == sent).all() and flags[0] == 1 and ticket[0] == 0 and err[0] == 0
    assert (local == np.uint64(0xFFFFFFFFFFFFFFFF)).all()
    emu.emu_gather_and_min(_p(local, u64), ctypes.c_int64(0), ctypes.c_int64(MP), _p(slots, u64), _p(flags, u32), 2, _p(ticket, u32),
                           _p(final, u64), _p(err))
    assert flags[0] == 2 and ticket[0] == 0 and (final[:P] == sent).all()


# ---- node_state.cuh: device-side order, incremental record refresh, fit table, value-domain check ---------
def _host_order(free, tile=128):
    order = []
    for f in range(8, -1, -1):
        order += [i for i in range(len(free)) if bin(int(free[i]) & 0xFF).count("1") == f]
        while len(order) % 32:
            order.append(-1)
    while len(order) % tile:
        order.append(-1)
    return np.array(order, dtype=np.int32)


@pytest.mark.parametrize("n", [1, 31, 1000, 1024, 1025, 3333])
def test_emulated_device_order_is_the_stable_class_sort(emu, n):
    """order_count / order_scan / order_scatter == the host's nine-pass stable sort by free count (classes 8..0,
    padded to warps, total padded to tiles), slot_of is its inverse, class counts are right."""
    free = synth.rand_below(0xABC0 + n, 1, n, 256).astype(np.int32)
    if n == 1000:
        free[:] = 0xFF                                  # one class only
    want = _host_order(free)
    cap = (n + 11 * 128) // 128 * 128
    order = np.empty(cap, dtype=np.int32)
    slot_of = np.empty(n, dtype=np.int32)
    cc = np.zeros(9, dtype=np.int64)
    n_slots = emu.emu_order(_p(free), ctypes.c_int64(n), _p(order), ctypes.c_int64(cap), _p(slot_of), _p(cc, ctypes.c_longlong))
    assert n_slots == len(want)
    assert (order[:n_slots] == want).all() and (order[n_slots:] == -1).all()
    assert (order[slot_of] == np.arange(n)).all()
    assert cc.tolist() == [int((np.array([bin(int(x) & 0xFF).count("1") for x in free]) == c).sum()) for c in range(9)]


def test_emulated_incremental_mask_updates_equal_fresh_upload(emu, oracle_b):
    """kgpu_set_free_masks: records of the listed nodes are refreshed in place (stale order), K1s then gives the
    keys of a fresh upload with the final masks -- including nodes whose free count crossed class boundaries
    and a node that went from 0 to 8 free GPUs."""
    W = oracle_b.DEFAULT_WEIGHTS
    topo, free, pods = synth.gen_c4(N=520, P=90)
    free0 = free.copy()
    free0[7] = 0
    upd_idx = np.array([7, 0, 100, 101, 102, 300, 519, 260], dtype=np.int32)
    upd_mask = np.array([0xFF, 0x00, 0x0F, 0xF0, 0x81, 0xFF, 0x01, 0x3C], dtype=np.int32)
    final = free0.copy()
    final[upd_idx] = upd_mask
    for splits in (1, 2):
        keys = np.empty(len(pods), dtype=np.uint64)
        out_free = np.empty_like(free0)
        emu.emu_score_sparse_after_updates(_p(np.ascontiguousarray(topo, dtype=np.int32)), _p(free0), ctypes.c_int64(len(free0)),
                                           _p(upd_idx), _p(upd_mask), ctypes.c_int64(len(upd_idx)), _p(pods), ctypes.c_int64(len(pods)),
                                           _p(np.ascontiguousarray(W, dtype=np.int32)), splits, _p(keys, ctypes.c_uint64), _p(out_free))
        assert (out_free == final).all()
        assert (keys == oracle_b.score_batch(topo, final, pods, W)).all()


def test_emulated_fit_table_rows(emu, oracle_b):
    W = np.ascontiguousarray(oracle_b.DEFAULT_WEIGHTS, dtype=np.int32)
    topo, free, _ = synth.gen_c4(N=200, P=1)
    topo = np.ascontiguousarray(topo, dtype=np.int32)
    out = np.empty(9 * 200, dtype=np.uint32)
    emu.emu_fit_nodes(_p(topo), _p(free), ctypes.c_int64(200), None, ctypes.c_int64(200), _p(W), _p(out, ctypes.c_uint32))
    for i in range(0, 200, 7):
        for k in range(9):
            assert int(out[k * 200 + i]) == oracle_b.node_key(topo[i], int(free[i]), k)
    lst = np.array([199, 3, 50], dtype=np.int32)
    out = np.empty(27, dtype=np.uint32)
    emu.emu_fit_nodes(_p(topo), _p(free), ctypes.c_int64(200), _p(lst), ctypes.c_int64(3), _p(W), _p(out, ctypes.c_uint32))
    for j, i in enumerate(lst):
        for k in range(9):
            assert int(out[k * 3 + j]) == oracle_b.node_key(topo[i], int(free[i]), k)


def test_emulated_validate_topo(emu):
    topo, _, _ = synth.gen_c4(N=100, P=1)
    topo = np.ascontiguousarray(topo, dtype=np.int32)
    assert emu.emu_validate_topo(_p(topo), ctypes.c_int64(100)) == -1
    topo[40, 9] = 16
    topo[77, 3] = -1
    assert emu.emu_validate_topo(_p(topo), ctypes.c_int64(100)) == 40 * 64 + 9


@pytest.mark.parametrize("resident", [1, 3])
def test_emulated_multi_tile_items_few_pods(emu, oracle_b, resident):
    """Few pods (one chunk): a block walks a RUN of tiles, sorts the pods once, carries the per-pod minimum in
    shared memory and flushes once.  Cost ties across tiles must still go to the lower node id, winners move
    between tiles, invalid k and memory-constrained pods ride along."""
    W = oracle_b.DEFAULT_WEIGHTS
    topo, free, pods = synth.gen_c2(N=1500, P=40)            # few shapes: ties across tiles are the rule
    pods[3, 0], pods[4, 0] = 0, 9
    for trial in range(3):
        want = oracle_b.score_batch(topo, free, pods, W, node_id_base=7)
        assert (_run(emu.emu_score_sparse, topo, free, pods, W, base=7, splits=-resident) == want).all(), trial
        for key in want:                                      # take the winners away: the next trial finds others
            if key != np.uint64(0xFFFFFFFFFFFFFFFF):
                free[(int(key >> np.uint64(8)) & 0xFFFFFFFF) - 7] = 0
    topo, free, mem, pods = synth.gen_c6(N=900, P=33)
    want = oracle_b.score_batch(topo, free, pods, mem=mem)
    assert (_run(emu.emu_score_sparse, topo, free, pods, W, mem=mem, splits=-resident) == want).all()
    p1 = synth.make_pods(np.array([3], dtype=np.int32))       # a single pod
    assert (_run(emu.emu_score_sparse, topo, free, p1, W, splits=-resident) == oracle_b.score_batch(topo, free, p1, W)).all()


@pytest.mark.parametrize("P", [2, 4, 5, 63, 64, 65, 130])
@pytest.mark.parametrize("wmax", [6, 2341])
def test_emulated_few_pod_instantiations_at_their_boundaries(emu, oracle_b, P, wmax):
    """The three few-pod instantiations and the pod counts where the host switches between them: at most 4 pods
    (TMA, 7 blocks per SM), at most 64 (TMA, 8 blocks), at most 512 (next tile's record prefetched into registers);
    byte-aligned and general warp keys; heterogeneous nodes so that tiles mix classes (the flush then compares node ids
    explicitly) and S' has to be expanded through ragged permutations; an invalid k and a k = 0 pod ride along."""
    topo, free, pods = synth.gen_c4(N=700, P=P, seed=1000 + P)
    pods[0, 0] = 0
    if P > 4:
        pods[4, 0] = 9
    W = np.array([max(1, wmax - 3 * i) for i in range(16)], dtype=np.int32)
    want = oracle_b.score_batch(topo, free, pods, W, node_id_base=11)
    for resident in (1, 2):                                   # runs of many tiles / of a few tiles per item
        assert (_run(emu.emu_score_sparse, topo, free, pods, W, base=11, splits=-resident) == want).all(), resident


@pytest.mark.parametrize("pad", [32, 128])
def test_tile_classes_from_class_counts_equal_slot_maxima(emu, pad):
    """The hosts derive each tile's class from the order's class counts alone (launch_plan.h: tile_classes); that must be
    the largest free count among the tile's nodes, with classes padded to warps (32) or to whole tiles (128)."""
    rng = np.random.default_rng(pad)
    for n in (1, 127, 1000, 3333):
        free = (rng.integers(0, 256, size=n) & rng.integers(0, 256, size=n)).astype(np.int32)
        if n == 1000:
            free[rng.random(n) < 0.5] = 0xFF
        cap = (n + 11 * 128) // 128
        got, want = np.zeros(cap, np.uint8), np.zeros(cap, np.uint8)
        tiles = emu.emu_tile_classes(_p(free), n, pad, _p(got, ctypes.c_uint8), _p(want, ctypes.c_uint8), cap)
        assert 1 <= tiles <= cap
        assert (got[:tiles] == want[:tiles]).all(), n


K1S_ROUTES = {"in_block_sort": 0, "prepared": 1, "stream": 2, "tma": 3}


@pytest.mark.parametrize("route", sorted(K1S_ROUTES))
@pytest.mark.parametrize("mem", [False, True])
@pytest.mark.parametrize("byte_keys", [True, False])
def test_emulated_k1s_routes(emu, oracle_b, route, mem, byte_keys):
    """Each K1s route the host plan can pick (TMA, STREAM, prepared chunk tables, the blocks' own pod sort), with and without
    the MEM launch and byte keys, is reached (emu_score_sparse reports the route it took) and gives Oracle B's keys."""
    P, splits = {"tma": (40, -1), "stream": (300, -1), "prepared": (600, -1), "in_block_sort": (600, -1184)}[route]
    topo, free, gmem, pods = synth.gen_c6(N=300, P=P, seed=P)
    pods[2, 0], pods[3, 0] = 0, 9
    if not mem:
        pods[:, 3] = 0
    W = np.array([(2340 if byte_keys else 2341) - 5 * i for i in range(16)], dtype=np.int32)
    want = oracle_b.score_batch(topo, free, pods, W, node_id_base=5, mem=gmem, fast=True, nthreads=4)
    keys = np.empty(P, dtype=np.uint64)
    got = emu.emu_score_sparse(_p(topo), _p(free), _p(gmem), len(free), 5, _p(pods), P, _p(W), splits, _p(keys, ctypes.c_uint64))
    assert got == K1S_ROUTES[route] | (4 if mem else 0) | (8 if byte_keys else 0)
    assert (keys == want).all()


# ---- a handle's K1s cache over a sequence of state changes, on every route -----------------------------------------
ALL_FIFTEEN = np.full(64, 15, dtype=np.int32)          # every link on level 15: the cheapest level of the tables below


def _order_layout(emu, free):
    """The order kgpu_upload_nodes builds for these masks: order[n_slots] (-1 = padding) and its 128-slot tiles."""
    n = len(free)
    cap = (n + 11 * 128) // 128 * 128
    order, slot_of, cc = np.empty(cap, np.int32), np.empty(n, np.int32), np.empty(9, np.int64)
    n_slots = emu.emu_order(_p(free), n, _p(order), cap, _p(slot_of), _p(cc, ctypes.c_longlong))
    return order[:n_slots], slot_of


def _sequence_updates(emu, topo, free):
    """(updates, named nodes): a list of (node, new mask, new topology row or None) that covers a node going from 0 to 8
    free GPUs and one from 8 to 0, a node changing class in an ordered tile (one class, ids increasing) and one in a
    mixed-class tile, the last node, the node just before a run of padding slots, a node updated twice, node A made the
    unique cheapest node by its topology and node B, with a lower id in another tile, tied with A for k <= 4."""
    order, slot_of = _order_layout(emu, free)
    pop = np.array([bin(int(f) & 0xFF).count("1") for f in free])
    tiles = order.reshape(-1, 128)
    ordered = [t for t in range(len(tiles))
               if all(tiles[t][i] < 0 or (tiles[t][i - 1] >= 0 and tiles[t][i - 1] < tiles[t][i]) for i in range(1, 128))]
    mixed = [t for t in range(len(tiles)) if len({int(pop[x]) for x in tiles[t] if x >= 0}) > 1]
    assert ordered and mixed
    in_ordered = int(tiles[ordered[0]][5])
    in_mixed = next(int(x) for x in tiles[mixed[0]] if x >= 0 and pop[x] not in (0, 8))
    before_pad = next(int(order[s]) for s in range(len(order) - 1) if order[s] >= 0 and order[s + 1] < 0)
    empty = next(i for i in range(len(free)) if pop[i] == 0 and i not in (in_ordered, in_mixed, before_pad))
    full = next(i for i in range(len(free)) if pop[i] == 8 and i not in (in_ordered, in_mixed, before_pad))
    a = len(free) - 40
    b = next(i for i in range(len(free) // 3) if slot_of[i] // 128 != slot_of[a] // 128 and
             i not in (in_ordered, in_mixed, before_pad, empty, full))
    named = dict(a=a, b=b, in_ordered=in_ordered, in_mixed=in_mixed, before_pad=before_pad, empty=empty, full=full,
                 last=len(free) - 1)
    upd =[(empty, 0xFF, None), (full, 0x00, None),
           (in_ordered, 0xFF if pop[in_ordered] < 8 else 0x01, None), (in_mixed, 0x80 if pop[in_mixed] > 1 else 0xFE, None),
           (a, 0xFF, ALL_FIFTEEN), (len(free) - 1, 0xF7, None), (before_pad, 0x3C, None),
           (in_mixed, 0xFF, None), (b, 0x0F, ALL_FIFTEEN), (len(free) - 1, 0xFF, topo[0].copy()),
           (before_pad, 0xFF, topo[1].copy())]
    return upd, named


@pytest.mark.parametrize("route", sorted(K1S_ROUTES))
@pytest.mark.parametrize("mem", [False, True])
@pytest.mark.parametrize("byte_keys", [True, False])
def test_emulated_k1s_after_a_sequence_of_state_changes(emu, oracle_b, route, mem, byte_keys):
    """K1s on records refreshed in place while the order stays stale (kgpu_set_free_masks, kgpu_update_node with a new
    topology) and recompacted over the stale order by a weight change half way through, on each route, with and without
    the MEM launch, byte and general keys, a node-id base and GPU memory: Oracle B's keys on the final state."""
    P, splits = {"tma": (40, -1), "stream": (300, -1), "prepared": (600, -1), "in_block_sort": (600, -1184)}[route]
    N, base = 700, 1000
    topo, free, _ = synth.gen_c2(N=N, P=0, seed=77)            # four shapes: cost ties across nodes and tiles are the rule
    topo, free = topo.copy(), free.copy()
    gmem = synth.gen_gpu_memory(N, seed=78)
    _, _, _, pods = synth.gen_c6(N=1, P=P, seed=P)
    pods[2, 0], pods[3, 0] = 0, 9
    if not mem:
        pods[:, 3] = 0
    top = 2340 if byte_keys else 2341
    W = np.array([top - 5 * i for i in range(16)], dtype=np.int32)
    W2 = W.copy()
    W2[1], W2[5] = W[5], W[1]                                   # C2's levels 1 and 5 swap costs; level 15 stays cheapest
    upd, named = _sequence_updates(emu, topo, free)
    gmem[[named["a"], named["b"]]] = synth.GPU_MEM_CLASSES_MIB[-1]
    m = len(upd)
    idx = np.array([u[0] for u in upd], np.int32)
    masks = np.array([u[1] for u in upd], np.int32)
    rows = np.stack([u[2] if u[2] is not None else np.zeros(64, np.int32) for u in upd]).astype(np.int32)
    has = np.array([u[2] is not None for u in upd], np.int32)
    final_topo, final_free = topo.copy(), free.copy()
    for i, mk, row in upd:
        final_free[i] = mk
        if row is not None:
            final_topo[i] = row
    want = oracle_b.score_batch(final_topo, final_free, pods, W2, node_id_base=base, mem=gmem, fast=True, nthreads=4)
    winners = {int(k >> np.uint64(8)) & 0xFFFFFFFF for k in want if k != np.uint64(0xFFFFFFFFFFFFFFFF)}
    assert {named["a"] + base, named["b"] + base} <= winners          # A wins k > 4, B (lower id, another tile) k <= 4
    keys = np.empty(P, np.uint64)
    out_free = np.empty(N, np.int32)
    got = emu.emu_score_sparse_sequence(_p(topo), _p(free), _p(gmem), N, base, _p(idx), _p(masks), _p(rows), _p(has), m,
                                        _p(W), _p(W2), m // 2, _p(pods), P, splits, _p(keys, ctypes.c_uint64), _p(out_free))
    assert got == K1S_ROUTES[route] | (4 if mem else 0) | (8 if byte_keys else 0)
    assert (out_free == final_free).all()
    bad = np.flatnonzero(keys != want)
    assert len(bad) == 0, "%d keys differ, first pod %d (k %d): got %x want %x" % (
        len(bad), bad[0], pods[bad[0], 0], int(keys[bad[0]]), int(want[bad[0]]))
