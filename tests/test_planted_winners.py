"""Planted winners: every scorer must find the best node wherever it sits in the node order.

A batch's key is a minimum over all nodes, so a kernel that never looks at some tile, warp, lane or work item still
gives the right keys unless the true winner sits exactly there.  Generated clusters put their winners in very few
places (the first few hundred nodes of a class), so this file builds clusters whose winners are known in closed form
and moves them through every place the kernels divide the work by:

  * background: every GPU pair at a background link level, free masks uniform over 0..255 (every class 0..8 exists);
  * plant t_k (k = 2..8): a node with EXACTLY k free GPUs at random positions whose pairs all sit at level L_k, with
    W[L_2] < W[L_3] < ... < W[L_8] < every background weight.  Then t_k is the unique cheapest home of a k-GPU pod:
    key = (C(k,2) * W[L_k]) << 40 | (base + t_k) << 8 | free_mask[t_k].  A larger plant costs more for k, a smaller one
    cannot hold k GPUs, and with exactly k free GPUs no subset of t_k mixes in a background pair;
  * k = 1 costs 0 everywhere (lowest node id with a free GPU, its lowest free GPU), k = 0 is node 0 with mask 0,
    k outside 0..8 is NO_FIT.

A round plants t_2..t_8 (kgpu_update_node), scores a batch that covers every k, checks every key and restores the
hosts.  Hosts are picked by their SLOT in K1s's order (node_state.cuh: stable sort by free count, classes 8..0 padded
to 32 slots, 128-slot tiles): "fresh" hosts already have k free GPUs, and over the rounds every tile of classes 2..8
holds one; "stale" hosts have another free count, keep their slot (compact_nodes with a list) and cover the class 0/1
tiles.  "Index" rounds cover every 128-node index tile of the dense kernels.  The CPU half runs the sweep through the
kernel emulation and checks, on the GPU sweep's own schedule, that it reaches every tile, warp, lane, multi-tile run
and work item it is meant to."""
import ctypes
import math
import os
import re

import numpy as np
import pytest

import cpu_libs
from kubegpu_b200 import _lib, synth

NO_FIT = np.uint64(_lib.NO_FIT)
TILE, WARP, CHUNK = 128, 32, 512              # SP_THREADS (slots per K1s tile, nodes per dense tile), warp, SP_CHUNK
KS = range(2, 9)
INVALID_K = (9, -1, 100, -7)
H100_SMS = 132
RESORT_DIV = 200      # a handle re-sorts its order once more than n / 200 nodes changed since it was built (kgpu.cu)
BIG_N = 1_100_000     # above 2^20 nodes order_scan carries class offsets across its 1024-block chunks
# cluster seeds of the GPU tests; the coverage tests check the schedules of these very clusters
SEED_ROUTES, SEED_NO_MIN_MEM, SEED_VARIANTS, SEED_PAIRS, SEED_BIG, SEED_SHARDS = 7, 8, 9, 10, 11, 12
SPARSE_SRC = os.path.join(cpu_libs.ROOT, "kubegpu_b200", "csrc", "score_pairs_sparse.cuh")


def minblocks(name):
    """Resident blocks per SM of a K1s instantiation, as score_pairs_sparse.cuh defines them."""
    with open(SPARSE_SRC) as f:
        return int(re.search(r"#define %s (\d+)" % name, f.read()).group(1))


def _p(a, t=ctypes.c_int32):
    return None if a is None else a.ctypes.data_as(ctypes.POINTER(t))


def popcount(free):
    return np.unpackbits(np.asarray(free, np.int64).astype(np.uint8)[:, None], axis=1).sum(axis=1)


# ---- the cluster ---------------------------------------------------------------------------------------------------
class Cluster:
    """Background nodes and a weight table whose plants win in closed form.  table: "default" (the default weights,
    L_k = 9 - k, background level 0), "byte" (background levels 8..15 drawn per pair, largest weight 2340: the
    byte-aligned warp key) or "general" (largest weight 4095: the general key layout)."""

    def __init__(self, N, table, base=0, seed=0):
        rng = np.random.default_rng([seed, N])
        self.N, self.base, self.table = N, base, table
        self.free = rng.integers(0, 256, size=N).astype(np.int32)
        if table == "default":
            self.W = np.array([64, 32, 16, 8, 4, 2, 1] + [0] * 9, np.int32)
            self.L = {k: 9 - k for k in KS}
            self.topo = np.zeros((N, 64), np.int32)
        else:
            top = {"byte": 2340, "general": 4095}[table]
            self.W = np.zeros(16, np.int32)
            levels = rng.permutation(8)                       # plant levels in no particular weight order
            plant_w = np.sort(rng.choice(top // 2, size=7, replace=False))
            self.L = {k: int(levels[k - 2]) for k in KS}
            self.W[levels[:7]] = plant_w
            self.W[levels[7]] = rng.integers(0, top + 1)       # a level no pair uses
            bg = rng.integers(top // 2 + 1, top + 1, size=8)
            bg[rng.integers(8)] = top
            self.W[8:] = bg
            iu = np.triu_indices(8, 1)
            m = np.zeros((N, 8, 8), np.int32)
            m[:, iu[0], iu[1]] = 8 + rng.integers(0, 8, size=(N, 28))
            self.topo = (m + m.transpose(0, 2, 1)).reshape(N, 64)
        assert all(self.W[self.L[k]] < self.W[self.L[k + 1]] for k in range(2, 8))
        assert self.W[self.L[8]] < min(self.W[lv] for lv in self.background_levels())
        self.seed = seed

    def background_levels(self):
        return [0] if self.table == "default" else list(range(8, 16))

    def cost(self, k):
        return math.comb(k, 2) * int(self.W[self.L[k]])

    def plant(self, node, k, tag):
        """(topology row, free mask) of node as plant t_k: exactly k free GPUs, their pairs at level L_k."""
        rng = np.random.default_rng([self.seed, tag, k, node])
        gpus = rng.choice(8, size=k, replace=False)
        row = self.topo[node].reshape(8, 8).copy()
        for a in gpus:
            for b in gpus:
                if a != b:
                    row[a, b] = self.L[k]
        return row.reshape(64), int(sum(1 << int(g) for g in gpus))

    def expected(self, plants, pods, free=None):
        """Closed-form keys of pods on the background with plants {k: (node, mask)} (and masks `free`, if given)."""
        assert sorted(plants) == list(KS) and len({node for node, _ in plants.values()}) == 7
        if free is None:
            free = self.free.copy()
            for node, mask in plants.values():
                free[node] = mask
        lowest = int(np.flatnonzero(free & 0xFF)[0])
        best = {0: np.uint64(self.base << 8), 1: np.uint64((self.base + lowest) << 8 | (int(free[lowest]) & -int(free[lowest])) & 0xFF)}
        for k, (node, mask) in plants.items():
            best[k] = np.uint64(self.cost(k) << 40 | (self.base + node) << 8 | mask)
        return np.array([best.get(int(k), NO_FIT) for k in np.asarray(pods)[:, 0]], np.uint64)


def make_batch(blocks, seed, mem_copies=True):
    """blocks x 32 pods (16 without copies): each block holds every k in 0..8, an invalid k and six more k in 1..8,
    each pod twice, once without and once with min_mem_mib = 1 (which excludes nothing while no GPU memory is
    uploaded, so the MEM instantiation must give the same keys); shuffled inside the block, so that every 32-pod range
    holds every k of both launches."""
    rng = np.random.default_rng(seed)
    out = []
    for b in range(blocks):
        ks = list(range(9)) + [INVALID_K[b % len(INVALID_K)]] + list(rng.integers(1, 9, size=6))
        p = synth.make_pods(np.array(ks, np.int32))
        if mem_copies:
            q = p.copy()
            q[:, 3] = 1
            p = np.vstack([p, q])
        out.append(p[rng.permutation(len(p))])
    pods = np.vstack(out)
    pods[:, 1] = np.arange(len(pods))
    return np.ascontiguousarray(pods)


# ---- K1s's order and the schedule -----------------------------------------------------------------------------------
class Layout:
    """The order kgpu_upload_nodes builds for masks `free`: slot_of[node], order[slot] (-1: padding), class c's slots
    [start[c], start[c] + count[c]), tile classes (the largest class of every tile)."""

    def __init__(self, free):
        self.free = np.array(free, np.int32)
        pop = popcount(free)
        self.pop = pop
        self.count = np.bincount(pop, minlength=9)
        self.start = np.zeros(9, np.int64)
        s = 0
        parts = []
        for c in range(8, -1, -1):
            self.start[c] = s
            nodes = np.flatnonzero(pop == c)
            pad = -len(nodes) % WARP
            parts += [nodes, np.full(pad, -1)]
            s += len(nodes) + pad
        parts.append(np.full(-s % TILE, -1))
        self.order = np.concatenate(parts).astype(np.int64)
        self.n_slots = len(self.order)
        self.slot_of = np.empty(len(free), np.int64)
        real = self.order >= 0
        self.slot_of[self.order[real]] = np.flatnonzero(real)
        self.tiles = self.n_slots // TILE
        self.tile_class = np.zeros(self.tiles, np.uint8)
        for c in range(9):
            if self.count[c]:
                t = self.class_tiles(c)
                self.tile_class[t] = np.maximum(self.tile_class[t], c)

    def class_tiles(self, c):
        if not self.count[c]:
            return np.zeros(0, np.int64)
        return np.arange(self.start[c] // TILE, (self.start[c] + self.count[c] - 1) // TILE + 1)

    def class_slots_in_tile(self, c, t):
        lo = max(self.start[c], t * TILE)
        hi = min(self.start[c] + self.count[c], (t + 1) * TILE)
        return np.arange(lo, hi)


def fresh_rounds(lay, tiles_of=None):
    """Rounds of fresh plants (host already has k free GPUs): round r puts t_k in tile r mod (class k's tile count) of
    class k, or in tiles_of(k, r) if given; the first round takes every class's first slot, the last visit of its last
    tile its last slot, the others a slot that moves through the tile.  No two plants of a round share a tile unless
    the classes leave no other choice (a class of one tile that it shares with a neighbour)."""
    tiles = {k: lay.class_tiles(k) for k in KS}
    R = max(len(t) for t in tiles.values()) if tiles_of is None else tiles_of(None, None)
    rounds, ends = [], set()
    for r in range(R):
        used, plants = set(), {}
        for k in sorted(KS, key=lambda k: -len(tiles[k])):            # the class with most tiles first: visited once
            tl = tiles[k]
            if not len(tl):
                continue
            cands = [tiles_of(k, r)] if tiles_of else [tl[(r + d) % len(tl)] for d in range(len(tl))]
            t = next((int(t) for t in cands if int(t) not in used), int(cands[0]))    # shared only on tiny clusters
            used.add(t)
            slots = lay.class_slots_in_tile(k, t)
            if t == tl[0] and (k, 0) not in ends:
                slot = slots[0]
                ends.add((k, 0))
            elif t == tl[-1] and (k, -1) not in ends:
                slot = slots[-1]
                ends.add((k, -1))
            else:
                slot = slots[(r * 37 + k * 11) % len(slots)]
            plants[k] = int(lay.order[slot])
        rounds.append(("fresh", plants))
    return rounds


def stale_rounds(lay, tiles=None, every=16):
    """Rounds of stale plants (host has another free count, its slot stays where the order put it): every tile
    holding class 0 or 1 slots, the class 8 tiles and every `every`-th other tile (or `tiles`), seven per round."""
    if tiles is None:
        low = set(lay.class_tiles(0).tolist()) | set(lay.class_tiles(1).tolist()) | set(lay.class_tiles(8).tolist())
        tiles = sorted(low | set(range(0, lay.tiles, every)))
    rounds = []
    for i in range(0, len(tiles), 7):
        plants, left = {}, list(KS)
        for m, t in enumerate(tiles[i:i + 7]):
            sl = np.arange(t * TILE, (t + 1) * TILE)
            nodes = lay.order[sl]
            for k in sorted(left, key=lambda k: (k - 2 - m - i // 7) % 7):
                ok = np.flatnonzero((nodes >= 0) & (lay.pop[np.maximum(nodes, 0)] != k))
                if len(ok):
                    plants[k] = int(nodes[ok[(i * 53 + m * 29) % len(ok)]])
                    left.remove(k)
                    break
        used = set(tiles[i:i + 7])
        for j, k in enumerate(left):                  # the last group is short: its other plants go to earlier tiles
            for t in tiles[j::7] + list(range(lay.tiles)):
                if t in used:
                    continue
                used.add(t)
                nodes = lay.order[t * TILE:(t + 1) * TILE]
                ok = [int(x) for x in nodes if x >= 0 and lay.pop[x] != k and int(x) not in plants.values()]
                if ok:
                    plants[k] = ok[(i * 53 + j * 29) % len(ok)]
                    break
        rounds.append(("stale", plants))
    return rounds


def index_rounds(N):
    """Rounds over the node index: every 128-node tile of the dense kernels holds a plant, at a lane that moves."""
    tiles = (N + TILE - 1) // TILE
    rounds = []
    for i in range(0, tiles, 7):
        plants = {}
        for m in range(7):                            # the last round wraps around to the first tiles
            t = (i + m) % tiles
            plants[2 + (m + i // 7) % 7] = min(N - 1, t * TILE + (i * 37 + m * 29) % TILE)
        rounds.append(("index", plants))
    return rounds


def k1s_schedule(lay):
    return fresh_rounds(lay) + stale_rounds(lay)


def big_schedule(lay):
    """The short sweep at BIG_N nodes: the first and last tiles of every class (its last nodes lie above 2^20), fresh,
    then stale plants in the last tiles of classes 0, 1 and 8 and a few others."""
    picks = [0, -1, -2, -3, 1, -5, -9, -17, -33, -65, 2, -129, -257, -513, -1025, 3]

    def tiles_of(k, r):
        if k is None:
            return len(picks)
        tl = lay.class_tiles(k)
        return tl[picks[r] % len(tl)]
    last = [int(lay.class_tiles(c)[-1]) for c in range(9) if lay.count[c]]
    extra = [int(lay.class_tiles(c)[-2]) for c in (8, 4, 1, 0) if len(lay.class_tiles(c)) > 1]
    return fresh_rounds(lay, tiles_of) + stale_rounds(lay, tiles=sorted(set(last + extra)))


# ---- the closed form against Oracle B -------------------------------------------------------------------------------
TABLES = ["default", "byte", "general"]


@pytest.mark.parametrize("table", TABLES)
def test_closed_form_is_oracle_b(oracle_b, table):
    """The closed-form keys equal Oracle B's on fresh, stale and index rounds; every plant is strictly cheaper than the
    cheapest background node for its k, and a plant of exactly k free GPUs is what makes that so."""
    N = 1500
    for base in (0, 2**32 - 1 - N):
        cl = Cluster(N, table, base)
        pods = make_batch(2, seed=1)
        bg = oracle_b.score_batch(cl.topo, cl.free, pods, cl.W, node_id_base=base)
        for k in KS:
            assert min(int(x) >> 40 for x in bg[pods[:, 0] == k]) > cl.cost(k), k
        lay = Layout(cl.free)
        for kind, plants in k1s_schedule(lay)[::3] + index_rounds(N)[:2]:
            topo, free = cl.topo.copy(), cl.free.copy()
            pl = {}
            for k, node in plants.items():
                topo[node], free[node] = cl.plant(node, k, 0)
                pl[k] = (node, int(free[node]))
            want = oracle_b.score_batch(topo, free, pods, cl.W, node_id_base=base)
            assert (cl.expected(pl, pods) == want).all(), (kind, plants)
    # a spare free GPU breaks it: t_8 costs 28 * W[L_8] = 896, an 8-subset of seven L_7 GPUs and one more 784
    cl = Cluster(300, "default")
    topo, free = cl.topo.copy(), cl.free.copy()
    topo[10], free[10] = cl.plant(10, 8, 0)
    row = np.zeros((8, 8), np.int32)
    row[:7, :7] = cl.L[7]
    np.fill_diagonal(row, 0)
    topo[20], free[20] = row.reshape(64), 0xFF
    got = oracle_b.score_batch(topo, free, synth.make_pods(np.array([8], np.int32)), cl.W)
    assert int(got[0]) >> 40 == 21 * 16 + 7 * 64 == 784 < cl.cost(8) == 896


# ---- the emulated sweep (CPU) -----------------------------------------------------------------------------------------
EMU_N = 2000
K1S_ROUTES = {"in_block_sort": 0, "prepared": 1, "stream": 2, "tma": 3}
# (32-pod blocks, resident blocks the work list is cut for): runs of up to 16 tiles for the few-pod routes
EMU_ROUTES = {"tma": (2, -1), "stream": (10, -2), "prepared": (32, -8), "in_block_sort": (20, -64)}
EMU_CASES = [("tma", "default"), ("tma", "general"), ("stream", "byte"), ("stream", "general"), ("prepared", "general"),
             ("in_block_sort", "byte")]


@pytest.fixture(scope="module")
def emu():
    return cpu_libs.emu()


def emu_k1s_round(emu, cl, plants, pods, splits):
    """K1s on the background's order with the plants applied through the incremental path (stale order), as a
    handle runs it after kgpu_update_node.  Returns (route code, keys, {k: (node, mask)})."""
    idx = np.array(list(plants.values()), np.int32)
    rows, masks, pl = [], [], {}
    for k, node in plants.items():
        row, mask = cl.plant(node, k, 0)
        rows.append(row)
        masks.append(mask)
        pl[k] = (node, mask)
    rows = np.ascontiguousarray(np.array(rows, np.int32).reshape(-1, 64))
    masks = np.array(masks, np.int32)
    has = np.ones(len(idx), np.int32)
    P = len(pods)
    keys = np.empty(P, np.uint64)
    out_free = np.empty(cl.N, np.int32)
    code = emu.emu_score_sparse_sequence(_p(cl.topo), _p(cl.free), None, cl.N, cl.base, _p(idx), _p(masks), _p(rows), _p(has),
                                         len(idx), _p(cl.W), None, len(idx), _p(pods), P, splits, _p(keys, ctypes.c_uint64),
                                         _p(out_free))
    return code, keys, pl


def _diff(keys, want, pods, kind, plants, lay=None):
    bad = np.flatnonzero(keys != want)
    if not len(bad):
        return ""
    p = bad[0]
    k = int(pods[p, 0])
    where = ""
    if lay is not None and k in plants:
        s = int(lay.slot_of[plants[k]])
        where = " (slot %d: tile %d, warp %d, lane %d)" % (s, s // TILE, s % TILE // WARP, s % WARP)
    return "%s round %s: %d keys differ; pod %d (k %d, min_mem %d) got %x want %x%s" % (
        kind, plants, len(bad), p, k, pods[p, 3], int(keys[p]), int(want[p]), where)


@pytest.mark.parametrize("route,table", EMU_CASES)
def test_emulated_planted_sweep(emu, oracle_b, route, table):
    """Every fresh and stale round through K1s and K1m on the route's work list: every key equals the closed form,
    and the first round's keys Oracle B's."""
    base = 0 if table == "byte" else 2**32 - 1 - EMU_N
    cl = Cluster(EMU_N, table, base, seed=3)
    lay = Layout(cl.free)
    blocks, splits = EMU_ROUTES[route]
    pods = make_batch(blocks, seed=blocks)
    rounds = k1s_schedule(lay)
    assert len(rounds) >= 5
    for i, (kind, plants) in enumerate(rounds):
        code, keys, pl = emu_k1s_round(emu, cl, plants, pods, splits)
        assert code == K1S_ROUTES[route] | 4 | (0 if table == "general" else 8)
        want = cl.expected(pl, pods)
        if i == 0:
            topo, free = cl.topo.copy(), cl.free.copy()
            for k, (node, mask) in pl.items():
                topo[node], free[node] = cl.plant(node, k, 0)
            assert (oracle_b.score_batch(topo, free, pods, cl.W, node_id_base=base, fast=True, nthreads=4) == want).all()
        assert not _diff(keys, want, pods, kind, plants, lay), _diff(keys, want, pods, kind, plants, lay)


@pytest.mark.parametrize("variant", [_lib.VARIANT_WARP_PER_PAIR, _lib.VARIANT_LANE_PER_NODE, _lib.VARIANT_MEMO_BY_K,
                                     _lib.VARIANT_TILE_MEMO])
def test_emulated_planted_sweep_dense_variants(emu, variant, oracle_b):
    """The kernels that tile by node index, on index rounds (a plant in every 128-node tile) and a fresh and a stale
    round, every k with and without a memory requirement (K1m, or inline for warp-per-pair); the first round's keys
    are also Oracle B's."""
    N = 900
    cl = Cluster(N, "byte", 2**32 - 1 - N, seed=4)
    lay = Layout(cl.free)
    pods = make_batch(1, seed=5)
    rounds = index_rounds(N) + fresh_rounds(lay)[:1] + stale_rounds(lay)[:1]
    assert len(rounds) == 4
    for i, (kind, plants) in enumerate(rounds):
        topo, free = cl.topo.copy(), cl.free.copy()
        pl = {}
        for k, node in plants.items():
            topo[node], free[node] = cl.plant(node, k, 0)
            pl[k] = (node, int(free[node]))
        keys = np.empty(len(pods), np.uint64)
        if variant == _lib.VARIANT_LANE_PER_NODE:
            emu.emu_score_dense(_p(topo), _p(free), None, N, cl.base, _p(pods), len(pods), _p(cl.W), 2, _p(keys, ctypes.c_uint64))
        else:
            emu.emu_score_variant(variant, _p(topo), _p(free), None, N, cl.base, _p(pods), len(pods), _p(cl.W), 2,
                                  _p(keys, ctypes.c_uint64))
        want = cl.expected(pl, pods)
        if i == 0:
            assert (oracle_b.score_batch(topo, free, pods, cl.W, node_id_base=cl.base) == want).all()
        assert not _diff(keys, want, pods, kind, plants), _diff(keys, want, pods, kind, plants)


# ---- the GPU sweep's schedule reaches what it is meant to (CPU) ------------------------------------------------------
GPU_N, SHARD_N = 100_000, 10_000
# route -> (cluster size, 32-pod blocks, resident blocks of the instantiation on an H100's 132 SMs, chunk-aligned list)
GPU_ROUTES = {
    "tma": (GPU_N, 2, lambda: H100_SMS * minblocks("KGPU_SP_TMA_MINBLOCKS"), False),
    "stream": (GPU_N, 10, lambda: H100_SMS * minblocks("KGPU_SP_STREAM_MINBLOCKS"), False),
    "prepared": (GPU_N, 80, lambda: H100_SMS * minblocks("KGPU_SP_MINBLOCKS"), True),
    "in_block_sort": (SHARD_N, 80, lambda: H100_SMS * minblocks("KGPU_SP_MINBLOCKS"), False),
}


def work_list(emu, tile_class, P, resident):
    cap = 400_000
    out = np.zeros((cap, 4), np.int32)
    aligned = ctypes.c_int(0)
    n = emu.emu_sparse_work(_p(tile_class, ctypes.c_uint8), len(tile_class), P, resident, _p(out), cap, None,
                            ctypes.byref(aligned))
    assert 0 < n <= cap
    return out[:n], bool(aligned.value)


def handle_layouts(cl, rounds):
    """The order K1s walks at every round's score when gpu_sweep drives a single-device handle, as kgpu.cu keeps it:
    an upload marks the order dirty; a K1s launch rebuilds a dirty order from the masks of that moment, or one that more
    than n / RESORT_DIV node updates have gone stale; an update counts toward that only while the order is live."""
    free, dirty, stale, lay, out = None, True, 0, None, {}
    for step, arg in sweep_steps(cl, rounds):
        if step == "upload":
            free, dirty = cl.free.copy(), True
        elif step == "update":
            free[arg[0]] = arg[2]
            stale += 0 if dirty else 1
        else:
            if dirty or stale * RESORT_DIV > cl.N:
                lay = lay if lay is not None and (free == lay.free).all() else Layout(free)
                dirty, stale = False, 0
            if step == "score":
                out[arg[0]] = lay
    return out


# (route, cluster seed, mem copies in the batch) of the GPU sweeps on the K1s routes
COVERAGE_CASES = [(r, SEED_ROUTES, True) for r in sorted(GPU_ROUTES)] + [("stream", SEED_NO_MIN_MEM, False)]


@pytest.mark.parametrize("route,seed,mem_copies", COVERAGE_CASES)
def test_gpu_schedule_covers_every_tile_warp_lane_and_item(emu, route, seed, mem_copies):
    """On the GPU sweep's own cluster, batch and schedule, with the work list cut as on an H100: the handle walks the
    background's order at every round (re-uploads included); every tile of classes 2..8 holds a fresh plant, every
    class 0/1 tile a stale one; warps 0..3 and lanes 0 and 31 hold plants; so do the first and last slot of every class;
    the first, a middle and the last tile of every multi-tile run (few-pod routes) and every work item with a pod of
    the plant's k in its range (many-pod routes)."""
    N, blocks, resident, aligned_want = GPU_ROUTES[route]
    cl = Cluster(N, "default", seed=seed)             # the masks (and so the order) do not depend on the table
    lay = Layout(cl.free)
    pods = make_batch(blocks, seed=blocks) if mem_copies else make_batch(2 * blocks, seed=2 * blocks, mem_copies=False)
    P = len(pods)
    rounds = k1s_schedule(lay)
    walked = handle_layouts(cl, rounds)
    assert sorted(walked) == list(range(len(rounds)))
    assert all((w.order == lay.order).all() for w in walked.values())
    where = {"fresh": set(), "stale": set()}          # (tile, k)
    slots = set()
    for kind, plants in rounds:
        tiles = {int(lay.slot_of[n]) // TILE for n in plants.values()}
        assert len(tiles) == 7 or (N < GPU_N and len(tiles) == 6)      # 10k nodes: class 8 has one tile, shared with 7
        for k, node in plants.items():
            s = int(lay.slot_of[node])
            assert (lay.pop[node] == k) == (kind == "fresh")
            where[kind].add((s // TILE, k))
            slots.add(s)
    fresh_tiles = {t for t, _ in where["fresh"]}
    stale_tiles = {t for t, _ in where["stale"]}
    assert {t for t in range(lay.tiles) if lay.tile_class[t] >= 2} <= fresh_tiles
    assert {t for t in range(lay.tiles) if lay.tile_class[t] <= 1} <= stale_tiles
    for c in KS:
        assert {int(lay.start[c]), int(lay.start[c] + lay.count[c] - 1)} <= slots, c
    assert {s % TILE // WARP for s in slots} == {0, 1, 2, 3}
    assert {0, WARP - 1} <= {s % WARP for s in slots}
    planted = where["fresh"] | where["stale"]
    items, aligned = work_list(emu, lay.tile_class, P, resident())
    assert aligned == aligned_want
    if P <= CHUNK:
        runs = items[items[:, 3] > 1]
        assert len(runs) and (items[:, 3] >= 1).all()
        for t, _, _, nt in items:
            assert {t, t + nt // 2, t + nt - 1} <= {tt for tt, _ in planted}, (t, nt)
    else:
        assert (items[:, 3] == 1).all()
        ks_of_tile = {}
        for t, k in planted:
            ks_of_tile.setdefault(t, set()).add(k)
        for t, b, e, _ in items:
            assert ks_of_tile.get(int(t), set()) & set(pods[b:e, 0].tolist()), (t, b, e)


def test_big_schedule_reaches_the_nodes_above_two_to_the_twenty():
    """The short sweep at 1.1M nodes plants fresh and stale hosts above node 2^20 in every class, and in the first tile
    of every class, on the order the handle walks."""
    cl = Cluster(BIG_N, "default", seed=SEED_BIG)
    lay = Layout(cl.free)
    rounds = big_schedule(lay)
    assert len(rounds) <= 24
    assert all((w.order == lay.order).all() for w in handle_layouts(cl, rounds).values())
    high = {kind: set() for kind in ("fresh", "stale")}
    first = set()
    for kind, plants in rounds:
        assert len({int(lay.slot_of[n]) // TILE for n in plants.values()}) == len(plants)
        for k, node in plants.items():
            if node >= 1 << 20:
                high[kind].add(int(lay.pop[node]))
            first.add(int(lay.slot_of[node]) // TILE)
    assert high["fresh"] == set(KS)
    assert {0, 1, 8} <= high["stale"]
    assert {int(lay.class_tiles(k)[0]) for k in KS} <= first


# ---- the GPU sweep -----------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def scorer():
    from kubegpu_b200.scorer import Scorer
    s = Scorer((0,))
    yield s
    s.close()


def sweep_steps(cl, rounds):
    """The calls of a sweep, in order: ("upload", None) uploads the background, ("prime", None) scores the batch once
    on it, ("update", (node, row, mask)) is kgpu_update_node, ("score", (round, kind, plants, {k: (node, mask)})) scores
    a planted round.  The upload and the score that follows it build the order from the background; the background is
    uploaded again before the updates since then would make the handle re-sort, so that the order K1s walks is the
    background's at every round (handle_layouts checks this)."""
    changed = None
    for i, (kind, plants) in enumerate(rounds):
        if changed is None or (changed + len(plants)) * RESORT_DIV > cl.N:
            yield "upload", None
            yield "prime", None
            changed = 0
        pl = {}
        for k, node in plants.items():
            row, mask = cl.plant(node, k, 0)
            yield "update", (node, row, mask)
            pl[k] = (node, mask)
        yield "score", (i, kind, plants, pl)
        for node in plants.values():
            yield "update", (node, cl.topo[node], int(cl.free[node]))
        changed += 2 * len(plants)


def gpu_sweep(s, cl, rounds, pods, score, check_oracle=None):
    """Run sweep_steps on handle s; every planted round's keys must equal the closed form (and, for the first and last
    round, check_oracle's)."""
    lay = Layout(cl.free) if cl.N <= 2 * GPU_N else None
    for step, arg in sweep_steps(cl, rounds):
        if step == "upload":
            s.upload_nodes(cl.topo, cl.free, node_id_base=cl.base)
        elif step == "prime":
            score(pods)
        elif step == "update":
            s.update_node(*arg)
        else:
            i, kind, plants, pl = arg
            keys = score(pods)
            want = cl.expected(pl, pods)
            assert not _diff(keys, want, pods, kind, plants, lay), _diff(keys, want, pods, kind, plants, lay)
            if check_oracle is not None and i in (0, len(rounds) - 1):
                check_oracle(pl, keys)


def _oracle_check(oracle_b, cl, pods):
    """Oracle B on one pod per distinct (k, min_mem) of the batch, on the planted cluster."""
    def check(pl, keys):
        topo, free = cl.topo.copy(), cl.free.copy()
        for k, (node, mask) in pl.items():
            topo[node], free[node] = cl.plant(node, k, 0)
        _, first = np.unique(pods[:, 0].astype(np.int64) * 2 + (pods[:, 3] > 0), return_index=True)
        want = oracle_b.score_batch(topo, free, pods[first], cl.W, node_id_base=cl.base, fast=True, nthreads=os.cpu_count() or 1)
        assert (keys[first] == want).all()
    return check


@pytest.mark.gpu
@pytest.mark.parametrize("route", sorted(GPU_ROUTES))
@pytest.mark.parametrize("table", TABLES)
def test_gpu_planted_sweep_k1s_routes(scorer, oracle_b, route, table):
    """K1s and K1m (VARIANT_SPARSE) on each route at full size: every fresh and stale round's keys equal the closed
    form, the first and last round's also Oracle B's."""
    N, blocks, _, _ = GPU_ROUTES[route]
    cl = Cluster(N, table, 0 if table == "default" else 2**32 - 1 - N, seed=SEED_ROUTES)
    pods = make_batch(blocks, seed=blocks)
    scorer.set_variant(_lib.VARIANT_SPARSE)
    scorer.set_weights(cl.W)
    try:
        gpu_sweep(scorer, cl, k1s_schedule(Layout(cl.free)), pods, scorer.score_batch, _oracle_check(oracle_b, cl, pods))
    finally:
        scorer.set_weights(oracle_b.DEFAULT_WEIGHTS)


@pytest.mark.gpu
def test_gpu_planted_sweep_device_entry_without_min_mem(scorer):
    """kgpu_score_batch_device_ex with KGPU_BATCH_NO_MIN_MEM (no flag kernel, no K1m) on the register-prefetch route."""
    import torch
    cl = Cluster(GPU_N, "byte", 2**32 - 1 - GPU_N, seed=SEED_NO_MIN_MEM)
    pods = make_batch(2 * GPU_ROUTES["stream"][1], seed=2 * GPU_ROUTES["stream"][1], mem_copies=False)
    assert CHUNK >= len(pods) > 64 and (pods[:, 3] == 0).all()
    d_pods = torch.from_numpy(pods).cuda()
    d_keys = torch.empty(len(pods), dtype=torch.int64, device="cuda")
    st = torch.cuda.current_stream().cuda_stream

    def score(p):
        scorer.score_batch_device(d_pods.data_ptr(), len(p), d_keys.data_ptr(), st, _lib.BATCH_NO_MIN_MEM)
        torch.cuda.synchronize()
        return d_keys.cpu().numpy().view(np.uint64)
    scorer.set_variant(_lib.VARIANT_SPARSE)
    scorer.set_weights(cl.W)
    try:
        gpu_sweep(scorer, cl, k1s_schedule(Layout(cl.free)), pods, score)
    finally:
        scorer.set_weights([64, 32, 16, 8, 4, 2, 1] + [0] * 9)


@pytest.mark.gpu
@pytest.mark.parametrize("variant", [_lib.VARIANT_AUTO, _lib.VARIANT_MEMO_BY_K, _lib.VARIANT_LANE_PER_NODE,
                                     _lib.VARIANT_WARP_PER_PAIR, _lib.VARIANT_TILE_MEMO])
def test_gpu_planted_sweep_other_variants(scorer, oracle_b, variant):
    """The variants that tile by node index: the K1s schedule plus a plant in every 128-node index tile."""
    cl = Cluster(GPU_N, "general", 2**32 - 1 - GPU_N, seed=SEED_VARIANTS)
    pods = make_batch(2, seed=2)
    scorer.set_variant(variant)
    scorer.set_weights(cl.W)
    try:
        rounds = k1s_schedule(Layout(cl.free)) + index_rounds(GPU_N)
        gpu_sweep(scorer, cl, rounds, pods, scorer.score_batch, _oracle_check(oracle_b, cl, pods))
    finally:
        scorer.set_weights(oracle_b.DEFAULT_WEIGHTS)


@pytest.mark.gpu
def test_gpu_planted_pairs_preemption_and_dry_run_placement(scorer, oracle_b):
    """On the planted rounds: kgpu_score_pairs on every plant (k fits, k + 1 does not), kgpu_preempt_batch without a
    holder table at level 0 (the scoring keys, no victims), and a dry-run placement of one pod per k = 8..2, then
    k = 1, 0 and an invalid k, in which every pod takes its own plant (checked against Oracle B's placement too)."""
    cl = Cluster(GPU_N, "byte", 0, seed=SEED_PAIRS)
    lay = Layout(cl.free)
    pods = make_batch(2, seed=3)
    seq = synth.make_pods(np.array([8, 7, 6, 5, 4, 3, 2, 1, 0, 9], np.int32))
    scorer.set_variant(_lib.VARIANT_AUTO)
    scorer.set_weights(cl.W)
    rounds = k1s_schedule(lay)
    pick = rounds[::8] + rounds[-2:]

    def score(p):
        keys, victims = scorer.preempt_batch(p, np.zeros(len(p), np.int32))
        assert (victims == 0).all()
        return keys
    try:
        gpu_sweep(scorer, cl, pick, pods, score)
        # kgpu_score_pairs and the placement read the masks and the topology, not K1s's order: no re-uploads needed
        for n, (kind, plants) in enumerate(pick):
            pl = {}
            for k, node in plants.items():
                row, mask = cl.plant(node, k, 0)
                scorer.update_node(node, row, mask)
                pl[k] = (node, mask)
            idx = np.array([pl[k][0] for k in KS] * 2, np.int64)
            ks = np.array(list(KS) + [k + 1 for k in KS], np.int32)
            got = scorer.score_pairs(idx, ks)
            want = [cl.cost(k) << 8 | pl[k][1] for k in KS] + [0xFFFFFFFF] * 7
            assert got.tolist() == want, (kind, plants)
            free = cl.free.copy()
            for node, mask in pl.values():
                free[node] = mask
            got = scorer.place_batch(seq, dry_run=True)
            want = [cl.expected(pl, seq[i:i + 1], free)[0] for i in range(7)]
            for node, _ in pl.values():
                free[node] = 0
            want += list(cl.expected(pl, seq[7:], free))
            assert got.tolist() == [int(w) for w in want], (kind, plants)
            if n in (0, len(pick) - 1):
                topo, f = cl.topo.copy(), cl.free.copy()
                for k, (node, mask) in pl.items():
                    topo[node], f[node] = cl.plant(node, k, 0)
                assert (oracle_b.place_batch(topo, f, seq, cl.W, node_id_base=cl.base)[0] == got).all()
            assert (scorer.get_free_masks()[[v[0] for v in pl.values()]] == [v[1] for v in pl.values()]).all()
            for node in plants.values():
                scorer.update_node(node, cl.topo[node], int(cl.free[node]))
    finally:
        scorer.set_weights(oracle_b.DEFAULT_WEIGHTS)


@pytest.mark.gpu
@pytest.mark.parametrize("route", ["tma", "prepared"])
def test_gpu_planted_sweep_past_two_to_the_twenty_nodes(scorer, oracle_b, route):
    """1.1M nodes (the order's class offsets carried across order_scan's 1024-block chunks): fresh and stale plants
    in the first and last tiles of every class."""
    cl = Cluster(BIG_N, "default", 0, seed=SEED_BIG)
    pods = make_batch(GPU_ROUTES[route][1], seed=6)
    scorer.set_variant(_lib.VARIANT_SPARSE)
    scorer.set_weights(cl.W)
    try:
        gpu_sweep(scorer, cl, big_schedule(Layout(cl.free)), pods, scorer.score_batch, _oracle_check(oracle_b, cl, pods))
    finally:
        scorer.upload_nodes(cl.topo[:1], cl.free[:1])


@pytest.mark.gpu
def test_gpu_planted_shard_edges_on_a_multi_device_handle(oracle_b):
    """With two or more GPUs: plants on the first and last node of every shard of one handle."""
    import torch
    G = torch.cuda.device_count()
    if G < 2:
        pytest.skip("needs two or more CUDA devices")
    from kubegpu_b200.scorer import Scorer
    N = 40_000
    cl = Cluster(N, "general", 2**32 - 1 - N, seed=SEED_SHARDS)
    per = (N + G - 1) // G
    edges = sorted({g * per for g in range(G)} | {min(N, (g + 1) * per) - 1 for g in range(G)})
    rounds = []
    for i in range(0, len(edges), 7):
        rounds.append(("shard edges", {2 + m: node for m, node in enumerate(edges[i:i + 7])}))
    pods = make_batch(4, seed=4)
    with Scorer(tuple(range(G))) as s:
        s.set_variant(_lib.VARIANT_SPARSE)
        s.set_weights(cl.W)
        gpu_sweep(s, cl, rounds, pods, s.score_batch, _oracle_check(oracle_b, cl, pods))
