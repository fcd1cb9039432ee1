"""Seeded synthetic (node-topology, pod-request) inputs for the BASELINE configs.

Layouts (SURVEY.md 8(d)):
  topo       int32[N][64]  row-major 8x8 link-level matrix, symmetric, diag 0.
                           Value domain 0..15: 0 unknown, 1..6 the NVML P2P levels
                           the reference uses (cross-CPU .. same-board, see
                           nvidiagpuplugin/gpu/nvidia/nvidia_gpu_manager.go:159-174),
                           7..12 NVLink 1..6 links (extension, config C4).
  free_mask  int32[N]      bit i set = GPU i present and free (low 8 bits used).
  pods       int32[P][4]   {k, pod_id, flags, reserved}.

The generator is counter based (one splitmix64 finaliser per value) so any
language can restate it in five lines and produce identical arrays:
  u64(seed, stream, i) = mix(seed + stream*0xD1342543DE82EF95 + i*0x9E3779B97F4A7C15)
"""
from __future__ import annotations

import numpy as np

SEED_C2 = 0xB2000001
SEED_C3 = 0xB2000002
SEED_C4 = 0xB2000003
SEED_C5 = 0xB2000005
SEED_GANGS = 0xB2000007

_M64 = np.uint64(0xFFFFFFFFFFFFFFFF)


def _mix(z: np.ndarray) -> np.ndarray:
    with np.errstate(over="ignore"):
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def rand_u64(seed: int, stream: int, n: int, start: int = 0) -> np.ndarray:
    """n counter-based 64-bit values for indices start..start+n-1."""
    with np.errstate(over="ignore"):
        base = np.uint64(seed & 0xFFFFFFFFFFFFFFFF) + np.uint64(stream) * np.uint64(0xD1342543DE82EF95)
        idx = np.arange(start, start + n, dtype=np.uint64)
        return _mix(base + idx * np.uint64(0x9E3779B97F4A7C15))


def rand_below(seed: int, stream: int, n: int, bound: int, start: int = 0) -> np.ndarray:
    """Uniform ints in [0,bound) (top 32 bits, multiply-shift; bound < 2**31)."""
    hi = rand_u64(seed, stream, n, start) >> np.uint64(32)
    return ((hi * np.uint64(bound)) >> np.uint64(32)).astype(np.int64)


# ---- group shapes -> link-level matrices ---------------------------------------
LEVEL_SAME_GRP0, LEVEL_SAME_GRP1, LEVEL_CROSS = 5, 3, 1   # nvidia_gpu_manager_test.go:16

C2_SHAPES = ([[8]], [[4], [4]], [[2, 2], [2, 2]], [[4, 4]])


def shape_matrix(shape, same_grp0=LEVEL_SAME_GRP0, same_grp1=LEVEL_SAME_GRP1, cross=LEVEL_CROSS) -> np.ndarray:
    """int32[64] matrix for a 2-level shape such as [[4],[2,2]]; GPU index = position
    in the shape as written (callers pass shapes already in sorted-tree order)."""
    owner = []
    g0 = 0
    for a, grp1 in enumerate(shape):
        for cnt in grp1:
            owner += [(a, g0)] * cnt
            g0 += 1
    assert len(owner) <= 8
    m = np.zeros((8, 8), dtype=np.int32)
    for i, (a1, b1) in enumerate(owner):
        for j, (a2, b2) in enumerate(owner):
            if i != j:
                m[i, j] = same_grp0 if b1 == b2 else (same_grp1 if a1 == a2 else cross)
    return m.reshape(64)


def make_pods(ks: np.ndarray) -> np.ndarray:
    pods = np.zeros((len(ks), 4), dtype=np.int32)
    pods[:, 0] = ks
    pods[:, 1] = np.arange(len(ks), dtype=np.int32)
    return pods


def gen_c2(N: int = 100_000, P: int = 10_000, seed: int = SEED_C2, node_start: int = 0):
    """Config C2 / C5: shape uniform over C2_SHAPES, free_mask uniform 0..255,
    k uniform over {1,2,4,8}.  ``node_start`` lets a rank generate only its shard."""
    mats = np.stack([shape_matrix(s) for s in C2_SHAPES])
    # gather the 256-byte rows as 32 int64 words: the same array, 15x faster than fancy-indexing 64 int32
    topo = np.take(np.ascontiguousarray(mats, dtype=np.int32).view(np.int64), rand_below(seed, 1, N, len(C2_SHAPES), node_start), axis=0).view(np.int32)
    free = rand_below(seed, 2, N, 256, node_start).astype(np.int32)
    ks = np.array([1, 2, 4, 8], dtype=np.int32)[rand_below(seed, 3, P, 4)]
    return np.ascontiguousarray(topo, dtype=np.int32), free, make_pods(ks)


def gen_c3(N: int = 1_000_000, P: int = 100_000, seed: int = SEED_C3, node_start: int = 0):
    """Config C3: as C2 but k uniform over 1..8."""
    topo, free, _ = gen_c2(N, 0, seed, node_start)
    ks = (1 + rand_below(seed, 3, P, 8)).astype(np.int32)
    return topo, free, make_pods(ks)


def gen_c4(N: int = 262_144, P: int = 1024, seed: int = SEED_C4, node_start: int = 0):
    """Config C4: heterogeneous, non-ultrametric.  Each unordered pair i<j draws a
    PCIe level 1..6 w.p. 0.7 or an NVLink level 7..12 w.p. 0.3; n_gpus in {4,8};
    GPUs >= n_gpus are absent (matrix 0, never free); k uniform over 1..8."""
    pair_i, pair_j = np.triu_indices(8, 1)
    r = rand_u64(seed, 1, N * 28, node_start * 28).reshape(N, 28)
    is_nvl = (r & np.uint64(0xFFFF)) < np.uint64(int(0.3 * 65536))
    lvl = (1 + ((r >> np.uint64(16)) % np.uint64(6))).astype(np.int32) + np.where(is_nvl, 6, 0).astype(np.int32)
    n_gpus = np.where(rand_below(seed, 4, N, 2, node_start) == 0, 4, 8)
    present = (pair_j[None, :] < n_gpus[:, None])
    lvl = np.where(present, lvl, 0).astype(np.int32)
    topo = np.zeros((N, 8, 8), dtype=np.int32)
    topo[:, pair_i, pair_j] = lvl
    topo[:, pair_j, pair_i] = lvl
    free = (rand_below(seed, 2, N, 256, node_start) & ((1 << n_gpus) - 1)).astype(np.int32)
    ks = (1 + rand_below(seed, 3, P, 8)).astype(np.int32)
    return topo.reshape(N, 64), free, make_pods(ks)


def gen_c1():
    """Config C1: 16 nodes x 4 pods from the reference's fixtures: [[2,2],[2,2]]
    (gpu_test.go:14-23), [[4],[2,2]] (gpu_test.go:24-33), 4 x K80 singletons
    (nvidia_gpu_manager_test.go:17; own groups, no topology -> level 0), empty."""
    t1 = shape_matrix([[2, 2], [2, 2]])
    t2 = shape_matrix([[4], [2, 2]])
    k80 = np.zeros(64, dtype=np.int32)
    empty = np.zeros(64, dtype=np.int32)
    topo = np.stack([t1, t2, k80, empty] * 4).astype(np.int32)
    free = np.array([0xFF, 0xFF, 0x0F, 0x00] * 4, dtype=np.int32)
    return topo, free, make_pods(np.array([1, 2, 3, 4], dtype=np.int32))


SEED_C6 = 0xB2000006
GPU_MEM_CLASSES_MIB = (16_384, 32_768, 81_920, 184_320)      # 16 / 32 / 80 / 180 GiB parts
POD_MIN_MEM_CHOICES_MIB = (0, 0, 0, 8_000, 20_000, 40_000, 100_000)


def gen_gpu_memory(N: int, seed: int = SEED_C6, node_start: int = 0) -> np.ndarray:
    """int32[N][8] MiB per GPU: 80 % of the nodes carry one memory class on all GPUs, 20 % mix classes
    per GPU (SURVEY.md 8(f) rank 3: the node agent advertises `<gpu>/memory` per GPU)."""
    classes = np.array(GPU_MEM_CLASSES_MIB, dtype=np.int32)
    node_class = rand_below(seed, 11, N, len(classes), node_start)
    mixed = rand_below(seed, 12, N, 5, node_start) == 0
    per_gpu = rand_below(seed, 13, N * 8, len(classes), node_start * 8).reshape(N, 8)
    idx = np.where(mixed[:, None], per_gpu, node_class[:, None])
    return np.ascontiguousarray(classes[idx], dtype=np.int32)


def gen_c6(N: int = 100_000, P: int = 10_000, seed: int = SEED_C6, node_start: int = 0):
    """Memory-aware config (not in BASELINE.json; exercises the per-pod min_mem path): C4's heterogeneous
    topologies, per-GPU memory classes, pods with k in 1..8 and a min_mem drawn from
    POD_MIN_MEM_CHOICES_MIB.  Returns (topo, free, mem, pods)."""
    topo, free, pods = gen_c4(N, P, seed, node_start)
    mem = gen_gpu_memory(N, seed, node_start)
    pods[:, 3] = np.array(POD_MIN_MEM_CHOICES_MIB, dtype=np.int32)[rand_below(seed, 14, P, len(POD_MIN_MEM_CHOICES_MIB))]
    return topo, free, mem, pods


SEED_PREEMPT = 0xB2000008


def gen_preempt(N: int = 100_000, P: int = 10_000, seed: int = SEED_PREEMPT):
    """An almost full cluster for preemption: C2's node shapes, each node packed from slot 0 with running pods of 1, 2,
    4 or 8 GPUs (aligned blocks, the size uniform over those that fit at the position) at priority levels 0..3.  At most
    one block of 1 or 2 GPUs per node is left free (a quarter of the small blocks are, until one is), so no node has
    more than 2 free GPUs.  The pending pods are C2's (k uniform over {1, 2, 4, 8}) with levels uniform over 0..4: every
    k = 4 or 8 pod fits nowhere without eviction.
    Returns (topo, free, holders[N][8], pods, lvl[P]); holders as kgpu_upload_holders takes them."""
    topo, _, pods = gen_c2(N, P, seed)
    hold = np.full((N, 8), -1, dtype=np.int32)
    free = np.zeros(N, dtype=np.int32)
    pos = np.zeros(N, dtype=np.int64)
    owner = np.zeros(N, dtype=np.int64)
    has_free = np.zeros(N, dtype=bool)
    for step in range(8):
        live = pos < 8
        align = np.where(pos == 0, 8, pos & -pos)
        size = np.minimum(1 << rand_below(seed, 30 + step, N, 4), align)
        empty = live & (size <= 2) & ~has_free & (rand_below(seed, 40 + step, N, 4) == 0)
        held = live & ~empty
        entry = (rand_below(seed, 50 + step, N, 4) << 3) | owner
        for g in range(8):
            blk = (g >= pos) & (g < pos + size)
            hold[blk & held, g] = entry[blk & held]
            free |= np.where(blk & empty, 1 << g, 0).astype(np.int32)
        has_free |= empty
        owner += held
        pos = np.where(live, pos + size, pos)
    lvl = rand_below(seed, 24, P, 5).astype(np.int32)
    return topo, free, hold, pods, lvl


SEED_PREEMPT_GANGS = 0xB2000009


def gen_preempt_gangs(N: int = 20_000, P: int = 10_000, seed: int = SEED_PREEMPT_GANGS, gang_start: float = 0.1):
    """gen_preempt's almost full cluster and pods, with high-priority training jobs mixed in: at each pod that is not yet
    in a gang, a gang starts with probability ``gang_start`` (about a third of the pods end up in gangs).  A gang has
    2..8 consecutive members, one level in 1..4, and each member's k is drawn from {4, 8} on its own.  Mixed k within a
    gang is what makes a member miss after earlier members were given victims; the default 20k nodes keep the cluster
    small enough that such gangs occur (at 100k nodes none fails).  Ids are 1, 2, ... in order.
    Returns (topo, free, holders[N][8], pods, lvl[P], gang[P])."""
    topo, free, hold, pods, lvl = gen_preempt(N, P, seed)
    start = rand_below(seed, 61, P, 1 << 20) < int(gang_start * (1 << 20))
    size = 2 + rand_below(seed, 62, P, 7)
    glvl = (1 + rand_below(seed, 63, P, 4)).astype(np.int32)
    kg = np.array([4, 8], dtype=np.int32)[rand_below(seed, 64, P, 2)]
    gang = np.zeros(P, dtype=np.int32)
    p, gid = 0, 0
    while p < P:
        if start[p]:
            gid += 1
            end = min(P, p + int(size[p]))
            gang[p:end] = gid
            lvl[p:end] = glvl[p]
            pods[p:end, 0] = kg[p:end]
            p = end
        else:
            p += 1
    return topo, free, hold, pods, lvl, gang


def gen_gangs(N: int = 100_000, P: int = 10_000, seed: int = SEED_GANGS, gang_start: float = 0.1):
    """C2's cluster and pod stream, with distributed training jobs mixed in: at each pod that is not yet in a gang,
    a gang starts with probability ``gang_start`` (default: about a third of the pods end up in gangs).  A gang has
    2..8 members that all want the same k in {4, 8} and sit next to each other; ids are 1, 2, ... in order.  At C2's
    size the nodes with 8 free GPUs run out early, so many k = 8 gangs fail part way.
    Returns (topo, free, pods, gang[P])."""
    topo, free, pods = gen_c2(N, P, seed)
    start = rand_below(seed, 21, P, 1 << 20) < int(gang_start * (1 << 20))
    size = 2 + rand_below(seed, 22, P, 7)
    kg = np.array([4, 8], dtype=np.int32)[rand_below(seed, 23, P, 2)]
    gang = np.zeros(P, dtype=np.int32)
    p, gid = 0, 0
    while p < P:
        if start[p]:
            gid += 1
            end = min(P, p + int(size[p]))
            gang[p:end] = gid
            pods[p:end, 0] = kg[p]
            p = end
        else:
            p += 1
    return topo, free, pods, gang


SEED_DOMAINS = 0xB200000A


def gen_domains(N: int, size: int, seed: int = SEED_DOMAINS) -> np.ndarray:
    """Network domains for N nodes: the nodes dealt into domains of ``size`` (the last one may be smaller) by a seeded
    permutation, so a domain is not a contiguous index range.  Returns int32[N], ids 0 .. ceil(N / size) - 1."""
    order = np.argsort(rand_u64(seed, 31, N), kind="stable")
    dom = np.empty(N, dtype=np.int32)
    dom[order] = (np.arange(N) // size).astype(np.int32)
    return dom


def gen_domain_levels(N: int, sizes, seed: int = SEED_DOMAINS) -> np.ndarray:
    """Nested network domains for N nodes, for example racks of 32 inside spines of 1024: int32[len(sizes), N].  The
    nodes are laid out in a seeded permutation (so no domain is a contiguous index range) and level 0 cuts it into
    domains of sizes[0] slots, as gen_domains(N, sizes[0], seed) does.  Level l + 1 groups whole level-l domains: each
    goes to the one whose range of sizes[l + 1] slots holds its first slot, so its domains hold about sizes[l + 1]
    nodes (exactly that many, but the last, when sizes[l + 1] is a multiple of sizes[l]).  Sizes must increase."""
    sizes = [int(s) for s in sizes]
    if not sizes or sizes[0] < 1 or any(b <= a for a, b in zip(sizes, sizes[1:])):
        raise ValueError("sizes must be positive and increasing")
    order = np.argsort(rand_u64(seed, 31, N), kind="stable")
    out = np.empty((len(sizes), N), dtype=np.int32)
    out[0, order] = (np.arange(N) // sizes[0]).astype(np.int32)
    lead = out[0].astype(np.int64) * sizes[0]                  # each node's level-l domain's first slot
    for lv in range(1, len(sizes)):
        out[lv] = (lead // sizes[lv]).astype(np.int32)
        first = np.full(int(out[lv].max()) + 1 if N else 0, np.iinfo(np.int64).max, np.int64)
        np.minimum.at(first, out[lv], lead)
        lead = first[out[lv]]
    return out
