// place_sequential.cuh -- K3: stateful sequential placement (SURVEY.md 8(f) rank 2), memory-aware.
//
// Semantics (bit-exact against the CPU twin used by the tests):
//   for p = 0 .. P-1, in order:
//       key_p = min over nodes of (cost<<40 | node_id<<8 | S)   given the CURRENT free masks, where
//               only GPUs with at least the pod's min_mem MiB count as free for that pod
//       if key_p != NO_FIT:  free_mask[node] &= ~S              (the pod takes those GPUs)
// This is what TakePodResources would make of a scheduling cycle if the reference's plugin
// tracked usage (it is a no-op there: gpuschedulerplugin/gpu_scheduler.go:57-63), and it has no
// snapshot-scoring collapse: every placement changes the state the next pod sees.
//
// Views.  The distinct min_mem values of a batch (at most PLACE_MAX_VIEWS - 1, the host checks) define
// VIEWS of the cluster: view 0 sees every free GPU, view v only the free GPUs with >= min_mem[v] MiB.
// GPU memory never changes, so a view is the same computation with (free & ok_v) as the free mask,
// and every table below exists once per view.
//
// Device data (v = view, k = 0..8 GPUs wanted):
//   nodebest[v][k][Npad] uint32  (cost<<8 | S) of every node, INF32 = no fit                      (global)
//   tilebest[v][k][T]    uint64  min over each 128-node tile of (cost<<40 | node_id<<8 | S)      (global)
//   super[v][k][ST]      uint64  min over each supertile (super_tiles tiles)                     (SHARED)
// place_init       : grid (tiles, views): full enumeration for all 9 k (lane per node) -> nodebest, tilebest
// place_sequential : ONE persistent block walks the pods.  Per pod: argmin over super[v][k] in shared
//                    memory (the winning key already names node and subset), one barrier; commit; then
//                    each warp takes (view, k) tasks on its own: re-enumerate the winner node (lane per
//                    subset), refresh the minimum of its tile and of its supertile -- the global loads of
//                    a task (topology row, node-key row of the tile, tile minima of the supertile) do not
//                    depend on each other, so a pod costs one round trip to L2; one barrier.
#pragma once
#include "score_pairs.cuh"

namespace kgpu {

constexpr int PLACE_TILE = 128;
#ifndef KGPU_PLACE_THREADS
#define KGPU_PLACE_THREADS 320      // 10 warps: one per k (9 busy with one view), cheap block barrier
#endif
constexpr int PLACE_THREADS = KGPU_PLACE_THREADS;
constexpr int PLACE_WARPS = PLACE_THREADS / 32;
constexpr int PLACE_MAX_VIEWS = 8;
constexpr int PLACE_SUPER_CAP = 4608;       // uint64 entries of static shared memory (36 KB) for super[][][]

struct PlaceViews {
    int32_t n;                              // 1 .. PLACE_MAX_VIEWS
    int32_t min_mem[PLACE_MAX_VIEWS];       // min_mem[0] = 0
};

// host + device: tiles per supertile (a multiple of 32) such that views * 9 * ceil(T / super_tiles) fits
__host__ __device__ inline int64_t place_super_tiles(int64_t T, int views) {
    int64_t st = 32;
    while ((int64_t)views * 9 * ((T + st - 1) / st) > PLACE_SUPER_CAP) st *= 2;
    return st;
}

__device__ __forceinline__ unsigned long long warp_min_u64(unsigned long long v) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) v = min(v, __shfl_xor_sync(0xFFFFFFFFu, v, off));
    return v;
}

__device__ __forceinline__ unsigned long long wide_key(uint32_t nk, unsigned long long node_id) {
    return nk == INF32 ? ~0ull : (((unsigned long long)(nk >> 8) << 40) | (node_id << 8) | (nk & 0xFFu));
}

// GPUs of `node` that view `need` may use (gpu_mem == nullptr: unlimited memory)
__device__ __forceinline__ uint32_t view_ok_mask(const int32_t *__restrict__ gpu_mem, int64_t node, int32_t need) {
    if (gpu_mem == nullptr || need <= 0) return 0xFFu;
    uint32_t ok = 0;
#pragma unroll
    for (int g = 0; g < 8; g++)
        if (__ldg(gpu_mem + node * 8 + g) >= need) ok |= 1u << g;
    return ok;
}

__global__ void __launch_bounds__(PLACE_TILE)
place_init(const int4 *__restrict__ topo4, const int32_t *__restrict__ free_mask, const int32_t *__restrict__ gpu_mem,
           int64_t N, int64_t Npad, int64_t node_id_base, Weights W, PipeConsts pc, PlaceViews views,
           uint32_t *__restrict__ nodebest, unsigned long long *__restrict__ tilebest, int64_t T) {
    __shared__ int32_t sW[16];
    __shared__ unsigned long long sRed[9][PLACE_TILE / 32];
    const int tid = threadIdx.x;
    if (tid == 0) {
#pragma unroll
        for (int i = 0; i < 16; i++) sW[i] = W.w[i];
    }
    __syncthreads();
    const int64_t tile = blockIdx.x;
    const int v = blockIdx.y;
    int32_t need = 0;
#pragma unroll
    for (int i = 0; i < PLACE_MAX_VIEWS; i++)
        if (i == v) need = views.min_mem[i];
    const int64_t node = tile * PLACE_TILE + tid;
    const bool valid = node < N;
    PairCosts C;
    uint32_t free;
    stage_node(topo4, free_mask, node, valid, sW, C, free, valid ? view_ok_mask(gpu_mem, node, need) : 0xFFu);
#pragma unroll 1
    for (int k = 0; k <= 8; k++) {
        uint32_t key = node_key(k, C, pc, free, valid);
        if (key >= PEN) key = INF32;
        nodebest[((int64_t)v * 9 + k) * Npad + node] = key;
        const unsigned long long w = warp_min_u64(wide_key(key, (unsigned long long)(node_id_base + node)));
        if ((tid & 31) == 0) sRed[k][tid >> 5] = w;
    }
    __syncthreads();
    if (tid < 9) {
        unsigned long long b = ~0ull;
#pragma unroll
        for (int w = 0; w < PLACE_TILE / 32; w++) b = min(b, sRed[tid][w]);
        tilebest[((int64_t)v * 9 + tid) * T + tile] = b;
    }
}

// Subset costs of one node from half tables.  With the 8 GPUs split into halves lo = GPUs 0..3, hi = GPUs 4..7,
//   cost(S) = A[S_lo] + B[S_hi] + sum over i in S_lo of R[i][S_hi]
// A, B: link cost inside a half (16 entries each); R[i][h]: links from GPU i of the low half to the GPUs of
// h (4 x 16 entries).  The warp builds the 96 entries once per placement (three per lane, a handful of adds
// each); a subset then costs two loads and at most four predicated load-adds instead of 28 tests.
constexpr int PLACE_HALF = 96;
__device__ __forceinline__ void build_half_tables(const int32_t *sCost, int32_t *half, int lane) {
    {
        const int m = lane & 15, base = lane < 16 ? 0 : 4;
        int32_t a = 0;
#pragma unroll
        for (int i = 0; i < 4; i++)
#pragma unroll
            for (int j = i + 1; j < 4; j++)
                if (((m >> i) & 1) && ((m >> j) & 1)) a += sCost[(base + i) * 8 + base + j];
        half[lane] = a;                                   // A at [0,16), B at [16,32)
    }
#pragma unroll
    for (int e = lane; e < 64; e += 32) {                 // R[i][h] at [32 + 16 i + h]
        const int i = e >> 4, h = e & 15;
        int32_t r = 0;
#pragma unroll
        for (int j = 0; j < 4; j++)
            if ((h >> j) & 1) r += sCost[i * 8 + 4 + j];
        half[32 + e] = r;
    }
}

// The half tables of EVERY node, once per batch (they depend on topology and weights only): half_all[node][96].
// place_sequential then fetches a winner's tables with three coalesced loads instead of rebuilding them on its
// per-pod chain.  Warp per node.
__global__ void __launch_bounds__(128)
place_half_tables(const int32_t *__restrict__ topo, int64_t N, Weights W, int32_t *__restrict__ half_all) {
    __shared__ int32_t sW[16];
    __shared__ int32_t sCost[4][64];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) {
#pragma unroll
        for (int i = 0; i < 16; i++) sW[i] = W.w[i];
    }
    __syncthreads();
    for (int64_t node = (int64_t)blockIdx.x * 4 + warp; node < N; node += (int64_t)gridDim.x * 4) {
        __syncwarp();
        sCost[warp][lane] = sW[__ldg(topo + node * 64 + lane) & 15];
        sCost[warp][lane + 32] = sW[__ldg(topo + node * 64 + lane + 32) & 15];
        __syncwarp();
        build_half_tables(sCost[warp], half_all + node * PLACE_HALF, lane);
    }
}

__device__ __forceinline__ void prefetch_l1(const void *p) {
#ifdef __CUDACC__
    asm volatile("prefetch.global.L1 [%0];" ::"l"(p));
#else
    (void)p;
#endif
}

// (cost<<8 | S) of one node for k GPUs, computed by a whole warp: lane per candidate subset.
// `subsets` = the k-subsets of 8 in increasing order in SHARED memory (the constant-memory table indexed by lane would
// serialise: one address per cycle).
__device__ __forceinline__ uint32_t node_key_warp(int k, const int32_t *half, uint32_t fm, int lane, const uint8_t *subsets, int nsub) {
    if (k == 0) return 0u;
    uint32_t key = INF32;
    for (int s = lane; s < nsub; s += 32) {
        const uint32_t S = subsets[s];
        if (S & ~fm) continue;
        const uint32_t lo = S & 15u, hi = S >> 4;
        uint32_t cost = (uint32_t)half[lo] + (uint32_t)half[16 + hi];
#pragma unroll
        for (int i = 0; i < 4; i++)
            if ((lo >> i) & 1u) cost += (uint32_t)half[32 + 16 * i + hi];
        key = min(key, (cost << 8) | S);
    }
    return __reduce_min_sync(0xFFFFFFFFu, key);
}

// Warp minimum of 64-bit keys with two REDUX.MIN (high word, then the low words of the lanes that hold it)
// instead of five rounds of two 32-bit shuffles + compare-select.
__device__ __forceinline__ unsigned long long warp_min_u64_redux(unsigned long long v) {
    const uint32_t hi = (uint32_t)(v >> 32), lo = (uint32_t)v;
    const uint32_t mhi = __reduce_min_sync(0xFFFFFFFFu, hi);
    const uint32_t mlo = __reduce_min_sync(0xFFFFFFFFu, hi == mhi ? lo : 0xFFFFFFFFu);
    return ((unsigned long long)mhi << 32) | mlo;
}

// Tile minimum of one (view, k) row, as the refresh computes it: every lane folds the node keys of its nodes of the tile
// (offset `off` in the tile) into a 32-bit composite cost << 15 | node offset << 8 | S (cost <= 28 * 4095 < 2^17), and
// tile_min_key takes the warp's minimum with one REDUX and widens it to the 64-bit key.
__device__ __forceinline__ uint32_t tile_fold(uint32_t m, uint32_t key, int off) {
    if (key != INF32) m = min(m, ((key >> 8) << 15) | ((uint32_t)off << 8) | (key & 0xFFu));
    return m;
}
__device__ __forceinline__ unsigned long long tile_min_key(uint32_t m, int64_t node_id_base, int tile) {
    m = __reduce_min_sync(0xFFFFFFFFu, m);
    return m == INF32 ? ~0ull
                      : (((unsigned long long)(m >> 15) << 40) |
                         ((unsigned long long)(node_id_base + (int64_t)tile * PLACE_TILE + ((m >> 8) & 127u)) << 8) | (m & 0xFFu));
}

constexpr int PLACE_POD_CHUNK = 1024;       // pod requests staged in shared memory (16 KB)
constexpr size_t PLACE_DYN_SMEM = 2 * (size_t)PLACE_SUPER_CAP * sizeof(unsigned long long);

// One persistent block.  Per pod (the serial chain; v4):
//   1. every warp finds the winner by itself: the supertile minima of (view, k) sit in shared memory (<= a few
//      entries per lane), the minimum IS the winning (cost, node, subset); two REDUX.  No barrier: the minima are
//      double buffered by UPDATE EPOCH (an epoch = one pod that placed something): winners are read from copy
//      e & 1, refreshed values are written to copy (e + 1) & 1 at once and to copy e & 1 one epoch later (by the
//      same lane, before its new writes), i.e. after the barrier that ends epoch e -- so no warp can see a
//      refreshed minimum while another still looks for the winner.
//   2. commit + refresh, warp per (view, k) task.  Sequential placement keeps hitting the same few nodes (the
//      cheapest node takes pods until it is full), so every warp CACHES, in registers / its shared-memory rows,
//      what it loaded for the previous winner: the node's half tables and free mask (same node), the node keys of
//      its tile (same tile), the tile minima of its supertile (same supertile).  A pod whose winner stays in the
//      cached supertile touches no global memory on the chain (stores are fire and forget); otherwise all loads
//      of the task are issued together.  Re-enumeration: lane per subset from the half tables; tile minimum: one
//      REDUX over a 32-bit composite (cost << 15 | node offset << 8 | S; cost < 2^17); supertile minimum: two.
//   3. ONE barrier.
// Pod requests are staged PLACE_POD_CHUNK at a time; indices are 32-bit shifts (supertiles are 32 << j tiles).
//
// Gangs (GANG = true, gang[P] != nullptr): a maximal run of consecutive pods with the same nonzero gang id is placed
// all or nothing.  When a member misses (NO_FIT or k outside 0..8), the members placed before it give their GPUs back,
// last first: each undo is step 2 with free mask c_fm | S instead of c_fm & ~S, i.e. one more epoch, so the double-
// buffered supertile minima and the per-warp caches need no special case.  The members' keys are read back from
// keys[] (tid 0 wrote them; the barrier before the walk makes them visible), so a gang may cross a staging chunk.
// Members after the miss are not tried; every member's key becomes NO_FIT.  The host guarantees that no id appears
// in two separate runs.  GANG = false is the plain kernel, with no gang bookkeeping on its chain.
template <bool GANG = false>
__global__ void __launch_bounds__(PLACE_THREADS, 1)
place_sequential(const int32_t *__restrict__ topo, int32_t *__restrict__ free_mask, const int32_t *__restrict__ gpu_mem,
                 int64_t N, int64_t Npad, int64_t node_id_base, const int4 *__restrict__ pods4, int64_t P, Weights W,
                 PlaceViews views, uint32_t *__restrict__ nodebest, unsigned long long *__restrict__ tilebest, int64_t T,
                 const int32_t *__restrict__ half_all /*[N][96], place_half_tables*/, unsigned long long *__restrict__ keys,
                 const int32_t *__restrict__ gang = nullptr /*[P], GANG only*/) {
    __shared__ int32_t sViewMin[PLACE_MAX_VIEWS];                 // static indexing of the kernel parameter only
    __shared__ int32_t sHalf[PLACE_WARPS][PLACE_HALF];            // per warp: the cached node's half tables (node_key_warp)
    __shared__ uint8_t sSub[9][72];                               // the k-subsets of 8 GPUs, increasing
    __shared__ int32_t sNsub[9];
#ifdef __CUDACC__
    extern __shared__ unsigned long long sSuperDyn[];             // super[copy][v][k][ST]: 2 x 36 KB of DYNAMIC shared memory
    unsigned long long (*sSuper)[PLACE_SUPER_CAP] = reinterpret_cast<unsigned long long (*)[PLACE_SUPER_CAP]>(sSuperDyn);
#else
    __shared__ unsigned long long sSuper[2][PLACE_SUPER_CAP];     // (CPU emulation build)
#endif
    __shared__ int32_t sPendIdx[PLACE_MAX_VIEWS * 9];             // per task: entry still to be written to the other copy
    __shared__ unsigned long long sPendVal[PLACE_MAX_VIEWS * 9];
    __shared__ int4 sPods[PLACE_POD_CHUNK];
    __shared__ int32_t sGang[GANG ? PLACE_POD_CHUNK : 1];         // gang id of each staged pod (4 KB, GANG only)
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int V = views.n;
    const int super_tiles = (int)place_super_tiles(T, V);         // 32 << j
    const int st_shift = 31 - __clz(super_tiles);
    const int ST = (int)((T + super_tiles - 1) >> st_shift);
    const int Ti = (int)T;
    (void)W;
    if (tid == 0) {
#pragma unroll
        for (int i = 0; i < PLACE_MAX_VIEWS; i++) sViewMin[i] = views.min_mem[i];
    }
    if (tid < 9) {
        const int n = c_nsub[tid];
        sNsub[tid] = n;
        for (int i = 0; i < n; i++) sSub[tid][i] = c_subsets[tid][i];
    }
    if (tid < PLACE_MAX_VIEWS * 9) sPendIdx[tid] = -1;
    // supertile minima from the tile minima place_init left in memory (both copies)
    for (int idx = tid; idx < V * 9 * ST; idx += PLACE_THREADS) {
        const int vk = idx / ST, st = idx - vk * ST;
        const int t1 = min(Ti, (st + 1) << st_shift);
        unsigned long long b = ~0ull;
        for (int t = st << st_shift; t < t1; t++) b = min(b, tilebest[(int64_t)vk * T + t]);
        sSuper[0][idx] = b;
        sSuper[1][idx] = b;
    }
    uint32_t epoch = 0;                                           // block-uniform: pods that placed something so far
    const int ntask = V * 9;
    // what this warp has cached for its FIRST task (task == warp)
    int c_node = -1, c_tile = -1, c_st = -1;                      // warp-uniform
    uint32_t c_fm = 0;
    int32_t c_mem = 0x7FFFFFFF;                                   // lanes 0..7: memory of the cached node's GPUs
    uint32_t nbr[PLACE_TILE / 32];                                // per lane: node keys of the cached tile
    unsigned long long tsr = ~0ull;                               // per lane: minimum of tile c_st * 32 + lane (super_tiles == 32 only)
#pragma unroll
    for (int j = 0; j < PLACE_TILE / 32; j++) nbr[j] = INF32;

    int64_t g_first = 0;                                          // GANG, block-uniform: first pod of the current gang,
    int32_t g_id = 0;                                             // its id (0: the pod is on its own)
    bool g_failed = false;                                        // and whether one of its members has missed

    for (int64_t p0 = 0; p0 < P; p0 += PLACE_POD_CHUNK) {
        const int pn = (int)min((int64_t)PLACE_POD_CHUNK, P - p0);
        __syncthreads();
        for (int i = tid; i < pn; i += PLACE_THREADS) {
            sPods[i] = __ldg(pods4 + p0 + i);
            if constexpr (GANG) sGang[i] = __ldg(gang + p0 + i);
        }
        __syncthreads();
#pragma unroll 1
        for (int pi = 0; pi < pn; pi++) {
            const int4 req = sPods[pi];                       // block-uniform
            const int k = req.x;
            if constexpr (GANG) {
                const int32_t id = sGang[pi];
                if (id == 0 || id != g_id) {                  // a pod on its own, or the first member of a gang
                    g_first = p0 + pi;
                    g_id = id;
                    g_failed = false;
                } else if (g_failed) {                        // a later member of a gang that has failed: not tried
                    if (tid == 0) keys[p0 + pi] = ~0ull;
                    continue;
                }
            }
            unsigned long long win = ~0ull;
            if (k < 0 || k > 8) {
                if (tid == 0) keys[p0 + pi] = ~0ull;
                if (!GANG || g_id == 0) continue;
            } else {
                int v = 0;                                    // the pod's view: the one with its min_mem
                for (int j = 1; j < V; j++)
                    if (req.w == sViewMin[j]) v = j;
                // 1. the winner, by every warp for itself
                const unsigned long long *sp = sSuper[epoch & 1] + (v * 9 + k) * ST;
                unsigned long long best = ~0ull;
                for (int s = lane; s < ST; s += 32) best = min(best, sp[s]);
                win = warp_min_u64_redux(best);
                if (tid == 0) keys[p0 + pi] = win;
                if (win == ~0ull || k == 0)                   // nothing fits / nothing to take (block-uniform)
                    if (!GANG || win != ~0ull || g_id == 0) continue;
            }
            // The placement step 2 commits: this pod's (take), or -- GANG, a member has missed -- those of the members
            // placed before it, last first, each given back (one epoch each).
            bool take = true;
            int64_t back = p0 + pi;                           // GANG: the member being given back
            if constexpr (GANG) {
                if (win == ~0ull) {
                    __syncthreads();                          // the members' keys (tid 0 wrote them) are visible
                    take = false;
                    while (--back >= g_first && ((win = keys[back]) & 0xFFull) == 0) {}     // k == 0 took nothing
                }
            }
#pragma unroll 1
            while (take || back >= g_first) {
                // 2. commit and refresh, warp by warp: the winner node loses S (take) or, undoing a gang member, gets S back
                const uint32_t nid = (uint32_t)(win >> 8);
                const int node = (int)((int64_t)nid - node_id_base);
                const uint32_t S = (uint32_t)(win & 0xFFull);
                const int tile = node >> 7, st = tile >> st_shift;
                static_assert(PLACE_TILE == 128, "tile index is node >> 7");
                if (warp < min(PLACE_WARPS, ntask)) {
                    const int64_t vk0 = warp;                     // this warp's first (cached) task
                    const bool new_node = node != c_node, new_tile = tile != c_tile;
                    const bool cache_super = super_tiles == 32;
                    const bool new_st = !cache_super || st != c_st;
                    // every global load this pod needs from this warp, issued before anything waits
                    int32_t h0 = 0, h1 = 0, h2 = 0;
                    uint32_t fm_mem = 0;
                    if (new_node) {                               // the winner's half tables: three coalesced loads (L1 if prefetched)
                        const int32_t *src = half_all + (int64_t)node * PLACE_HALF;
                        h0 = __ldg(src + lane);
                        h1 = __ldg(src + lane + 32);
                        h2 = __ldg(src + lane + 64);
                        fm_mem = (uint32_t)free_mask[node] & 0xFFu;       // before or after warp 0's write-back: & ~S (| S) below either way
                        c_mem = (gpu_mem != nullptr && lane < 8) ? __ldg(gpu_mem + (int64_t)node * 8 + lane) : 0x7FFFFFFF;
                    }
                    if (new_tile) {
#pragma unroll
                        for (int j = 0; j < PLACE_TILE / 32; j++) nbr[j] = nodebest[vk0 * Npad + tile * PLACE_TILE + lane + 32 * j];
                    }
                    unsigned long long sb0 = ~0ull;               // !cache_super: minimum over the supertile's OTHER tiles
                    if (cache_super) {
                        if (new_st) {
                            const int t = (st << 5) + lane;
                            tsr = t < Ti ? tilebest[vk0 * T + t] : ~0ull;
                        }
                    } else {
                        for (int t = (st << st_shift) + lane; t < min(Ti, (st + 1) << st_shift); t += 32)
                            if (t != tile) sb0 = min(sb0, tilebest[vk0 * T + t]);
                    }
                    int32_t *half = sHalf[warp];
                    if (new_node) {
                        __syncwarp();
                        half[lane] = h0;
                        half[lane + 32] = h1;
                        half[lane + 64] = h2;
                        __syncwarp();
                        c_fm = fm_mem;
                        c_node = node;
                    }
                    c_tile = tile;
                    c_st = st;
                    const uint32_t fm = take ? (c_fm & ~S) : (c_fm | S);
                    c_fm = fm;
                    if (warp == 0 && lane == 0) free_mask[node] = (int32_t)fm;
                    for (int task = warp; task < ntask; task += PLACE_WARPS) {
                        const int tv = task / 9, tk = task - tv * 9;
                        const int64_t vk = task;
                        const bool cached = task == warp;
                        uint32_t nb[PLACE_TILE / 32];
                        unsigned long long sb = sb0;
                        if (!cached) {                            // more tasks than warps (several views): load now
#pragma unroll
                            for (int j = 0; j < PLACE_TILE / 32; j++) nb[j] = nodebest[vk * Npad + tile * PLACE_TILE + lane + 32 * j];
                            sb = ~0ull;
                            for (int t = (st << st_shift) + lane; t < min(Ti, (st + 1) << st_shift); t += 32)
                                if (t != tile) sb = min(sb, tilebest[vk * T + t]);
                        }
                        const uint32_t ok = tv == 0 ? 0xFFu : (__ballot_sync(0xFFFFFFFFu, c_mem >= sViewMin[tv]) & 0xFFu);
                        const uint32_t nk = node_key_warp(tk, half, fm & ok, lane, sSub[tk], sNsub[tk]);
                        uint32_t m = INF32;
#pragma unroll
                        for (int j = 0; j < PLACE_TILE / 32; j++) {
                            const int off = lane + 32 * j;
                            uint32_t key = cached ? nbr[j] : nb[j];
                            if (tile * PLACE_TILE + off == node) {
                                key = nk;
                                if (cached) nbr[j] = nk;
                            }
                            m = tile_fold(m, key, off);
                        }
                        const unsigned long long tb = tile_min_key(m, node_id_base, tile);
                        if (cached && cache_super) {
                            if (lane == (tile & 31)) tsr = tb;
                            sb = warp_min_u64_redux(tsr);
                        } else {
                            sb = warp_min_u64_redux(min(sb, tb));
                        }
                        if (lane == 0) {
                            nodebest[vk * Npad + node] = nk;
                            tilebest[vk * T + tile] = tb;
                            // last epoch's refreshed minimum reaches the copy the winners are read from NEXT epoch ...
                            const int pe = sPendIdx[task];
                            if (pe >= 0) sSuper[(epoch + 1) & 1][pe] = sPendVal[task];
                            // ... and this epoch's goes to that copy now, to the other one an epoch later
                            sSuper[(epoch + 1) & 1][vk * ST + st] = sb;
                            sPendIdx[task] = (int)(vk * ST + st);
                            sPendVal[task] = sb;
                        }
#ifndef KGPU_PLACE_PREFETCH
#define KGPU_PLACE_PREFETCH 0      // 0: off (default), 1: half tables + mask, 2: + the node-key row of the candidate's tile.  Off because on C2 the candidate search and the prefetch instructions on the chain cost more than the L1 hits save (not re-measured on the H100)
#endif
                        if (cached && KGPU_PLACE_PREFETCH) {
                            // The next winner for THIS warp's (view, k), unless another pod changes that first: the minimum of
                            // the row this warp has just brought up to date (copy (epoch + 1) & 1 is written by this warp
                            // only).  Every second pod opens a node nobody has touched yet (a node holds at most 8 GPUs'
                            // worth of pods), so its half tables and mask are brought into this SM's L1 now, off the chain.
                            __syncwarp();
                            const unsigned long long *row = sSuper[(epoch + 1) & 1] + vk * ST;
                            unsigned long long cb = ~0ull;
                            for (int s2 = lane; s2 < ST; s2 += 32) cb = min(cb, row[s2]);
                            cb = warp_min_u64_redux(cb);
                            if (cb != ~0ull) {
                                const int64_t cand = (int64_t)((cb >> 8) & 0xFFFFFFFFull) - node_id_base;
                                if (cand != c_node) {
                                    if (lane < 4) prefetch_l1(lane < 3 ? (const void *)(half_all + cand * PLACE_HALF + 32 * lane) : (const void *)(free_mask + cand));
                                    if (KGPU_PLACE_PREFETCH >= 2 && lane >= 4 && lane < 8)
                                        prefetch_l1(nodebest + vk * Npad + (cand & ~(int64_t)127) + 32 * (lane - 4));
                                }
                            }
                        }
                    }
                }
#ifndef KGPU_PLACE_HELPER
#define KGPU_PLACE_HELPER 1        // a warp without a task (warp 9 with one view) prefetches the NEXT pod's candidate into L1
#endif
                else if (KGPU_PLACE_HELPER && take && pi + 1 < pn) {
                    // Off the chain: the next pod's winner under the state BEFORE this pod's update is its winner afterwards
                    // too unless it is this pod's node (a placement only RAISES the keys of one node).  While the other warps
                    // refresh, bring what they will load for that node into this SM's L1: its half tables and mask, and for
                    // every task the node-key row of its tile and the tile minima of its supertile.
                    const int4 rq = sPods[pi + 1];
                    const int k2 = rq.x;
                    if (k2 >= 1 && k2 <= 8) {
                        int v2 = 0;
                        for (int j = 1; j < V; j++)
                            if (rq.w == sViewMin[j]) v2 = j;
                        const unsigned long long *sp2 = sSuper[epoch & 1] + (v2 * 9 + k2) * ST;
                        unsigned long long b2 = ~0ull;
                        for (int s2 = lane; s2 < ST; s2 += 32) b2 = min(b2, sp2[s2]);
                        b2 = warp_min_u64_redux(b2);
                        const int64_t cand = (int64_t)((b2 >> 8) & 0xFFFFFFFFull) - node_id_base;
                        if (b2 != ~0ull && cand != node) {
                            const int64_t ctile = cand >> 7, cst = ctile >> st_shift;
                            const int rows = ntask * 4, mins = ntask * 2;       // 128-byte lines: 4 per node-key row, 2 per 32 tile minima
                            for (int e = lane; e < 4 + rows + mins; e += 32) {
                                const void *q;
                                if (e < 3) q = half_all + cand * PLACE_HALF + 32 * e;
                                else if (e == 3) q = free_mask + cand;
                                else if (e < 4 + rows) { const int t = (e - 4) >> 2, j = (e - 4) & 3; q = nodebest + (int64_t)t * Npad + ctile * PLACE_TILE + 32 * j; }
                                else { const int t = (e - 4 - rows) >> 1, j = (e - 4 - rows) & 1; q = tilebest + (int64_t)t * T + min((int64_t)Ti - 1, (cst << st_shift) + 16 * j); }
                                prefetch_l1(q);
                            }
                        }
                    }
                }
                epoch++;
                __syncthreads();
                if (take) break;
                while (--back >= g_first && ((win = keys[back]) & 0xFFull) == 0) {}
            }
            if constexpr (GANG) {
                if (!take) {                                  // every member gets NO_FIT
                    __syncthreads();                          // once every thread has read the keys
                    for (int64_t m = g_first + tid; m <= p0 + pi; m += PLACE_THREADS) keys[m] = ~0ull;
                    g_failed = true;
                }
            }
        }
    }
}

}  // namespace kgpu
