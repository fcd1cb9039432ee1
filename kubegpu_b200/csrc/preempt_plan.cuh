// preempt_plan.cuh -- K5: preemption plans for a whole batch (kgpu_preempt_plan[_gang]), sm_90a.
//
// Definition (include/kgpu.h).  Pods are taken in order on a working copy (F, H) of the free masks and the holder
// table.  Pod p gets what kgpu_preempt_batch would give it alone on (F, H); if it fits on node n with GPUs S and
// victims V, then with R = the non-free GPUs of n held by an owner in V:  F[n] = (F[n] | R) & ~S  and H[n][g] = -1 for
// g in S | R.  GPUs the batch takes are therefore never evictable by a later pod of the batch, and owners are never
// renumbered, so victim bits name the holder table as it was at the call.
//
// Columns.  A pod's answer on one node depends on the node's state and on (k, level, min_mem) only.  The host lists
// the distinct triples of the batch with k in 1..8 as COLUMNS (at most PLAN_MAX_COLS, sorted by k so that warps stay
// on one k) and gives every pod its column.  Level-0 columns are plain sequential placement (nothing is evictable).
//
// Device data (c = column):
//   nodekey[c][Npad]  uint64  K4's lane key of the node: (level 4 | |V| 4) << 56 | cost << 39 | local node << 8 | S,
//                             ~0 = no candidate on the node                                                   (global)
//   tilekey[c][T]     uint64  minimum of nodekey over each 128-node tile                                       (global)
// plan_init       : grid (tiles, column groups), lane per node: K4's class search for each column -> both tables.
// plan_sequential : ONE persistent block walks the pods.  Per pod: the minimum of tilekey[c] over the tiles is the
//                   winner (its key names node and S); one thread applies the update to (F, H) and writes the key and
//                   the victims; then one thread per column re-runs the class search on the winner's node, and a tile
//                   minimum is rescanned (warp per column) only where the node held it and its key went up.
// gang_plan_sequential: plan_sequential with gangs (kgpu_preempt_plan_gang): a failed gang's placed members are undone
//                   from per-member pre-images of (F[n], H[n]); both kernels share plan_sequential_body<GANG>.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "place_sequential.cuh"
#include "preempt.cuh"

namespace kgpu {

constexpr int PLAN_TILE = 128;
constexpr int PLAN_MAX_COLS = 320;              // 8 k x (8 level-0 views + 32 (level > 0, min_mem) views)
constexpr int PLAN_THREADS = PLAN_MAX_COLS;     // plan_sequential: one thread per column in the refresh
constexpr int PLAN_WARPS = PLAN_THREADS / 32;
constexpr int PLAN_INIT_COLS = 8;               // columns per plan_init block
constexpr int PLAN_POD_CHUNK = 1024;            // pods staged in shared memory by plan_sequential

// The node state K4 reads, from one holder row: byte o of gm = owner o's non-free GPUs, nibble o of lvp = its level.
__device__ __forceinline__ void plan_owners(const int32_t (&h)[8], uint32_t F, uint64_t &gm, uint32_t &lvp) {
    gm = 0;
    lvp = 0;
#pragma unroll
    for (int g = 0; g < 8; g++) {
        if (h[g] < 0 || ((F >> g) & 1u)) continue;
        const uint32_t o = (uint32_t)h[g] & 7u;
        gm |= 1ull << (8 * o + g);
        lvp = (lvp & ~(15u << (4 * o))) | (((uint32_t)h[g] >> 3) << (4 * o));
    }
}

// Pair costs without any free-mask penalty (availability is per column), from the node's topology row.
__device__ __forceinline__ void plan_pair_costs(const int4 *__restrict__ topo4, int64_t node, bool valid, const int32_t *sW,
                                                PairCosts &C) {
    int4 q[16];
#pragma unroll
    for (int t = 0; t < 16; t++) q[t] = valid ? __ldg(topo4 + node * 16 + t) : make_int4(0, 0, 0, 0);
    for_each_pair(C, [&](int i, int j) -> uint32_t {
        const int4 v = q[i * 2 + (j >> 2)];
        const int l = (j & 3) == 0 ? v.x : (j & 3) == 1 ? v.y : (j & 3) == 2 ? v.z : v.w;
        return (uint32_t)sW[l & 15] << 8;
    });
}

// One node, one column: the best (class, cost, S) as (class << 56 | cost << 39 | S), ~0 if nothing fits.  The steps of
// preempt_bucket (preempt.cuh) for a single lane: class 0 if the available free GPUs suffice, else the lowest level m*
// whose owners free enough, the smallest fitting victim count s* among those owners, and the best dense key over
// every victim set of that size.
template <int K>
__device__ __forceinline__ unsigned long long plan_class_key(const PairCosts &C, const PipeConsts pc, uint32_t F, uint64_t gm,
                                                             uint32_t lvp, uint32_t elig, int32_t L) {
    const uint32_t A0 = F & elig;
    if (__popc(A0) >= K) {
        const uint32_t b = preempt_dense<K>(C, pc, A0);
        return ((unsigned long long)(b >> 8) << 39) | (b & 0xFFu);
    }
    uint32_t E = 0, lvmask = 0;
#pragma unroll
    for (int o = 0; o < 8; o++) {
        const uint32_t lo = (lvp >> (4 * o)) & 15u;
        if (((uint32_t)(gm >> (8 * o)) & elig & 0xFFu) && (int32_t)lo < L) { E |= 1u << o; lvmask |= 1u << lo; }
    }
    uint32_t X = 0, acc = A0, m = 16;
#pragma unroll 1
    for (uint32_t lm = lvmask; lm; lm &= lm - 1) {          // levels in ascending order
        const uint32_t lv = (uint32_t)__ffs(lm) - 1;
#pragma unroll
        for (int o = 0; o < 8; o++)
            if (((E >> o) & 1u) && ((lvp >> (4 * o)) & 15u) == lv) { X |= 1u << o; acc |= (uint32_t)(gm >> (8 * o)) & 0xFFu; }
        if (__popc(acc & elig) >= K) { m = lv; break; }
    }
    if (m == 16) return ~0ull;
    uint32_t smin = 9;
#pragma unroll 1
    for (uint32_t V = X; V; V = (V - 1) & X) {
        const uint32_t s = (uint32_t)__popc(V);
        if (s < smin && __popc((A0 | gpus_of(gm, V)) & elig) >= K) smin = s;
    }
    uint32_t best = INF32;
#pragma unroll 1
    for (uint32_t V = X; V; V = (V - 1) & X) {
        if ((uint32_t)__popc(V) != smin) continue;
        const uint32_t A = (A0 | gpus_of(gm, V)) & elig;
        if (__popc(A) >= K) best = min(best, preempt_dense<K>(C, pc, A));
    }
    return ((unsigned long long)(m << 4 | smin) << 56) | ((unsigned long long)(best >> 8) << 39) | (best & 0xFFu);
}

// The node's key for column col = {k, level, min_mem, -}, with the local node field; ~0 if nothing fits.
__device__ __forceinline__ unsigned long long plan_node_key(const PairCosts &C, const PipeConsts pc, uint32_t F, uint64_t gm,
                                                            uint32_t lvp, const int32_t (&mem)[8], int4 col, int64_t node) {
    uint32_t elig = 0xFFu;
    if (col.z > 0) {
        elig = 0;
#pragma unroll
        for (int g = 0; g < 8; g++) elig |= mem[g] >= col.z ? 1u << g : 0u;
    }
    unsigned long long v;
    switch (col.x) {
        case 1: v = plan_class_key<1>(C, pc, F, gm, lvp, elig, col.y); break;
        case 2: v = plan_class_key<2>(C, pc, F, gm, lvp, elig, col.y); break;
        case 3: v = plan_class_key<3>(C, pc, F, gm, lvp, elig, col.y); break;
        case 4: v = plan_class_key<4>(C, pc, F, gm, lvp, elig, col.y); break;
        case 5: v = plan_class_key<5>(C, pc, F, gm, lvp, elig, col.y); break;
        case 6: v = plan_class_key<6>(C, pc, F, gm, lvp, elig, col.y); break;
        case 7: v = plan_class_key<7>(C, pc, F, gm, lvp, elig, col.y); break;
        default: v = plan_class_key<8>(C, pc, F, gm, lvp, elig, col.y); break;
    }
    return v == ~0ull ? v : v | ((unsigned long long)node << 8);
}

// grid = (T node tiles, ceil(ncol / PLAN_INIT_COLS)); lane per node.  free_mask / hold: the working copies at the start.
__global__ void __launch_bounds__(PLAN_TILE)
plan_init(const int4 *__restrict__ topo4, const int32_t *__restrict__ free_mask, const int4 *__restrict__ mem4,
          const int4 *__restrict__ hold4, int64_t N, int64_t Npad, int64_t T, const int4 *__restrict__ cols, int ncol,
          Weights W, PipeConsts pc, unsigned long long *__restrict__ nodekey, unsigned long long *__restrict__ tilekey) {
    __shared__ int32_t sW[16];
    __shared__ unsigned long long sRed[PLAN_INIT_COLS][PLAN_TILE / 32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) {
#pragma unroll
        for (int i = 0; i < 16; i++) sW[i] = W.w[i];
    }
    __syncthreads();
    const int64_t tile = blockIdx.x;
    const int64_t node = tile * PLAN_TILE + tid;
    const bool valid = node < N;
    PairCosts C;
    plan_pair_costs(topo4, node, valid, sW, C);
    const uint32_t F = valid ? (uint32_t)__ldg(free_mask + node) & 0xFFu : 0u;
    int32_t mem[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    int32_t h[8] = {-1, -1, -1, -1, -1, -1, -1, -1};
    if (valid) {
        const int4 m0 = __ldg(mem4 + node * 2), m1 = __ldg(mem4 + node * 2 + 1);
        mem[0] = m0.x; mem[1] = m0.y; mem[2] = m0.z; mem[3] = m0.w;
        mem[4] = m1.x; mem[5] = m1.y; mem[6] = m1.z; mem[7] = m1.w;
        const int4 h0 = __ldg(hold4 + node * 2), h1 = __ldg(hold4 + node * 2 + 1);
        h[0] = h0.x; h[1] = h0.y; h[2] = h0.z; h[3] = h0.w;
        h[4] = h1.x; h[5] = h1.y; h[6] = h1.z; h[7] = h1.w;
    }
    uint64_t gm;
    uint32_t lvp;
    plan_owners(h, F, gm, lvp);
    const int c0 = (int)blockIdx.y * PLAN_INIT_COLS, cn = min(PLAN_INIT_COLS, ncol - c0);
#pragma unroll 1
    for (int i = 0; i < cn; i++) {
        const int c = c0 + i;
        const unsigned long long key = valid ? plan_node_key(C, pc, F, gm, lvp, mem, __ldg(cols + c), node) : ~0ull;
        nodekey[(int64_t)c * Npad + node] = key;
        const unsigned long long w = warp_min_u64_redux(key);
        if (lane == 0) sRed[i][warp] = w;
    }
    __syncthreads();
    if (tid < cn) {
        unsigned long long b = ~0ull;
#pragma unroll
        for (int w = 0; w < PLAN_TILE / 32; w++) b = min(b, sRed[tid][w]);
        tilekey[(int64_t)(c0 + tid) * T + tile] = b;
    }
}

// Steps 3 and 4 of plan_sequential for node n, whose new state the block has staged in sF / sH: every column's key of the
// node; the tile minimum follows at once where it can (the key went down, or the node did not hold the minimum),
// otherwise it is rescanned, warp per column, from the 128 node keys of the tile.  Ends with a barrier.
__device__ __forceinline__ void plan_refresh(int64_t n, const int4 *__restrict__ topo4, const int4 *__restrict__ mem4, int64_t Npad,
                                             int64_t T, int ncol, PipeConsts pc, unsigned long long *nodekey,
                                             unsigned long long *tilekey, const int32_t *sW, const int4 *sCol, const int32_t &sF,
                                             const int32_t *sH, int32_t *sResc, int &sNresc) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t tile = n / PLAN_TILE;
    // 3. every column's key of the node under the new state
    if (tid < ncol) {
        PairCosts C;
        plan_pair_costs(topo4, n, true, sW, C);
        const uint32_t F = (uint32_t)sF & 0xFFu;
        int32_t mem[8], h[8];
        const int4 m0 = __ldg(mem4 + n * 2), m1 = __ldg(mem4 + n * 2 + 1);
        mem[0] = m0.x; mem[1] = m0.y; mem[2] = m0.z; mem[3] = m0.w;
        mem[4] = m1.x; mem[5] = m1.y; mem[6] = m1.z; mem[7] = m1.w;
#pragma unroll
        for (int g = 0; g < 8; g++) h[g] = sH[g];
        uint64_t gm;
        uint32_t lvp;
        plan_owners(h, F, gm, lvp);
        const unsigned long long old = tilekey[(int64_t)tid * T + tile];
        const unsigned long long key = plan_node_key(C, pc, F, gm, lvp, mem, sCol[tid], n);
        nodekey[(int64_t)tid * Npad + n] = key;
        if (key < old) tilekey[(int64_t)tid * T + tile] = key;
        else if (key != old && old != ~0ull && (int64_t)((old >> 8) & 0x7FFFFFFFull) == n) sResc[atomicAdd(&sNresc, 1)] = tid;
    }
    __syncthreads();
    // 4. rescans: warp per column, the 128 node keys of the tile
    const int nr = sNresc;
    for (int j = warp; j < nr; j += PLAN_WARPS) {
        const int cc = sResc[j];
        const unsigned long long *row = nodekey + (int64_t)cc * Npad + tile * PLAN_TILE;
        unsigned long long m = ~0ull;
#pragma unroll
        for (int q = 0; q < PLAN_TILE / 32; q++) m = min(m, row[lane + 32 * q]);
        m = warp_min_u64_redux(m);
        if (lane == 0) tilekey[(int64_t)cc * T + tile] = m;
    }
    __syncthreads();
}

// One block of PLAN_THREADS.  pcol[p] = pod p's column, -1 for k outside 1..8 (k == 0 fits on the first node and takes
// nothing).  free_mask and hold are the working copies (F, H) and are updated in place; keys[p] and victims[p] are
// written for every pod.
//
// Gangs (GANG = true): a maximal run of consecutive pods with the same nonzero id gang[p] evicts and takes all or
// nothing.  The thread that applies a member's update first stores the node's state before it, (F[n], H[n]), in pre[p]
// ({F, holder bytes 0..3, holder bytes 4..7, 0}).  When a member misses (no candidate, or k outside 0..8), the members
// placed before it are undone, last first: their keys are read back from keys[] (k == 0 members took nothing), (F[n],
// H[n]) is restored from pre[], and steps 3 and 4 refresh the node as after a placement.  An undo can raise a key on the
// node that holds its tile's minimum (a placement frees a victim's other GPUs), so the rescan is needed here too.  Keys
// and pre-images are in global memory, so a gang may cross a staging chunk.  Members after the miss are not tried, and
// every member gets NO_FIT and victims 0.  The host guarantees that no id appears in two separate runs.  GANG = false
// is the plain kernel, with no gang bookkeeping on its chain.
// W by reference: a by-value copy changes the plain kernel's code.
template <bool GANG>
__device__ __forceinline__ void plan_sequential_body(const int4 *__restrict__ topo4, int32_t *free_mask, const int4 *__restrict__ mem4,
                                                     int32_t *hold, int64_t N, int64_t Npad, int64_t T, int64_t node_id_base,
                                                     const int4 *__restrict__ pods4, const int32_t *__restrict__ pcol, int64_t P,
                                                     const int4 *__restrict__ cols, int ncol, const Weights &W, PipeConsts pc,
                                                     unsigned long long *nodekey, unsigned long long *tilekey,
                                                     unsigned long long *__restrict__ keys, uint32_t *__restrict__ victims,
                                                     const int32_t *__restrict__ gang, int4 *__restrict__ pre) {
    __shared__ int32_t sW[16];
    __shared__ int4 sCol[PLAN_MAX_COLS];
    __shared__ int32_t sK[PLAN_POD_CHUNK], sPcol[PLAN_POD_CHUNK];
    __shared__ int32_t sGang[GANG ? PLAN_POD_CHUNK : 1];             // gang id of each staged pod (GANG only)
    __shared__ unsigned long long sRed[PLAN_WARPS];
    __shared__ unsigned long long sWin;
    __shared__ int32_t sF, sH[8];
    __shared__ int32_t sResc[PLAN_MAX_COLS];
    __shared__ int sNresc;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid < 16) sW[tid] = W.w[tid];
    if (tid < ncol) sCol[tid] = __ldg(cols + tid);
    const int Ti = (int)T;
    int64_t g_first = 0;                                              // GANG, block-uniform: first pod of the current gang,
    int32_t g_id = 0;                                                 // its id (0: the pod is on its own)
    bool g_failed = false;                                            // and whether one of its members has missed
    for (int64_t p0 = 0; p0 < P; p0 += PLAN_POD_CHUNK) {
        const int pn = (int)min((int64_t)PLAN_POD_CHUNK, P - p0);
        __syncthreads();
        for (int i = tid; i < pn; i += PLAN_THREADS) {
            sK[i] = __ldg(pods4 + p0 + i).x;
            sPcol[i] = __ldg(pcol + p0 + i);
            if constexpr (GANG) sGang[i] = __ldg(gang + p0 + i);
        }
        __syncthreads();
#pragma unroll 1
        for (int pi = 0; pi < pn; pi++) {
            const int64_t p = p0 + pi;
            const int c = sPcol[pi];                          // block-uniform
            if constexpr (GANG) {
                const int32_t id = sGang[pi];
                if (id == 0 || id != g_id) {                  // a pod on its own, or the first member of a gang
                    g_first = p;
                    g_id = id;
                    g_failed = false;
                } else if (g_failed) {                        // a later member of a gang that has failed: not tried
                    if (tid == 0) {
                        keys[p] = ~0ull;
                        victims[p] = 0;
                    }
                    continue;
                }
            }
            if (c < 0) {
                if (tid == 0) {
                    keys[p] = (sK[pi] == 0 && N > 0) ? (unsigned long long)node_id_base << 8 : ~0ull;
                    victims[p] = 0;
                }
                if (!GANG || g_id == 0 || sK[pi] == 0) continue;
            } else {
                // 1. the winner: the minimum over the tile minima of the pod's column
                unsigned long long b = ~0ull;
                for (int t = tid; t < Ti; t += PLAN_THREADS) b = min(b, tilekey[(int64_t)c * T + t]);
                b = warp_min_u64_redux(b);
                if (lane == 0) sRed[warp] = b;
                __syncthreads();
                if (warp == 0) {
                    b = warp_min_u64_redux(lane < PLAN_WARPS ? sRed[lane] : ~0ull);
                    if (lane == 0) {
                        sWin = b;
                        sNresc = 0;
                        if (b == ~0ull) {
                            keys[p] = ~0ull;
                            victims[p] = 0;
                        } else {
                            // 2. the update of (F, H): victims from the working table, their GPUs freed, S taken
                            const int64_t n = (int64_t)((b >> 8) & 0x7FFFFFFFull);
                            const uint32_t S = (uint32_t)b & 0xFFu, cost = (uint32_t)(b >> 39) & 0x1FFFFu;
                            const uint32_t f = (uint32_t)free_mask[n] & 0xFFu;
                            int32_t h[8];
                            uint32_t vic = 0;
#pragma unroll
                            for (int g = 0; g < 8; g++) {
                                h[g] = hold[n * 8 + g];
                                if (((S & ~f) >> g) & 1u) vic |= 1u << (h[g] & 7);
                            }
                            if constexpr (GANG) {
                                if (g_id != 0) {              // the pre-image of (F[n], H[n]) an undo restores
                                    uint32_t lo = 0, hi = 0;
#pragma unroll
                                    for (int g = 0; g < 4; g++) {
                                        lo |= ((uint32_t)h[g] & 0xFFu) << (8 * g);
                                        hi |= ((uint32_t)h[g + 4] & 0xFFu) << (8 * g);
                                    }
                                    pre[p] = make_int4((int32_t)f, (int32_t)lo, (int32_t)hi, 0);
                                }
                            }
                            uint32_t R = 0;
#pragma unroll
                            for (int g = 0; g < 8; g++)
                                if (!((f >> g) & 1u) && h[g] >= 0 && ((vic >> (h[g] & 7)) & 1u)) R |= 1u << g;
                            const uint32_t nf = (f | R) & ~S;
#pragma unroll
                            for (int g = 0; g < 8; g++) {
                                if (((S | R) >> g) & 1u) h[g] = -1;
                                hold[n * 8 + g] = h[g];
                                sH[g] = h[g];
                            }
                            free_mask[n] = (int32_t)nf;
                            sF = (int32_t)nf;
                            keys[p] = ((unsigned long long)cost << 40) | ((unsigned long long)(node_id_base + n) << 8) | S;
                            victims[p] = vic;
                        }
                    }
                }
                __syncthreads();
                const unsigned long long win = sWin;
                if (win == ~0ull) {                           // nothing changes
                    if (!GANG || g_id == 0) continue;
                } else {
                    plan_refresh((int64_t)((win >> 8) & 0x7FFFFFFFull), topo4, mem4, Npad, T, ncol, pc, nodekey, tilekey, sW, sCol,
                                 sF, sH, sResc, sNresc);
                    continue;
                }
            }
            if constexpr (GANG) {
                // A member has missed: the members placed before it are undone, last first (k == 0 members took nothing).
                __syncthreads();                              // once every thread is past this pod's reads of sF, sH
                int64_t back = p;
                unsigned long long key;
#pragma unroll 1
                while (--back >= g_first) {
                    if (((key = keys[back]) & 0xFFull) == 0) continue;
                    const int64_t n = (int64_t)((key >> 8) & 0xFFFFFFFFull) - node_id_base;
                    if (tid == 0) {
                        const int4 q = pre[back];
                        free_mask[n] = q.x;
                        sF = q.x;
#pragma unroll
                        for (int g = 0; g < 8; g++) {
                            const int32_t v = (int32_t)(int8_t)(((uint32_t)(g < 4 ? q.y : q.z) >> (8 * (g & 3))) & 0xFFu);
                            hold[n * 8 + g] = v;
                            sH[g] = v;
                        }
                        sNresc = 0;
                    }
                    __syncthreads();
                    plan_refresh(n, topo4, mem4, Npad, T, ncol, pc, nodekey, tilekey, sW, sCol, sF, sH, sResc, sNresc);
                }
                __syncthreads();                              // once every thread has read the keys
                for (int64_t m = g_first + tid; m <= p; m += PLAN_THREADS) {     // every member gets NO_FIT and victims 0
                    keys[m] = ~0ull;
                    victims[m] = 0;
                }
                g_failed = true;
            }
        }
    }
}

__global__ void __launch_bounds__(PLAN_THREADS, 1)
plan_sequential(const int4 *__restrict__ topo4, int32_t *free_mask, const int4 *__restrict__ mem4, int32_t *hold, int64_t N,
                int64_t Npad, int64_t T, int64_t node_id_base, const int4 *__restrict__ pods4, const int32_t *__restrict__ pcol,
                int64_t P, const int4 *__restrict__ cols, int ncol, Weights W, PipeConsts pc, unsigned long long *nodekey,
                unsigned long long *tilekey, unsigned long long *__restrict__ keys, uint32_t *__restrict__ victims) {
    plan_sequential_body<false>(topo4, free_mask, mem4, hold, N, Npad, T, node_id_base, pods4, pcol, P, cols, ncol, W, pc, nodekey,
                                tilekey, keys, victims, nullptr, nullptr);
}

// plan_sequential with gangs: gang[P] ids, pre[P] the members' pre-images (scratch).
__global__ void __launch_bounds__(PLAN_THREADS, 1)
gang_plan_sequential(const int4 *__restrict__ topo4, int32_t *free_mask, const int4 *__restrict__ mem4, int32_t *hold, int64_t N,
                     int64_t Npad, int64_t T, int64_t node_id_base, const int4 *__restrict__ pods4, const int32_t *__restrict__ pcol,
                     int64_t P, const int4 *__restrict__ cols, int ncol, Weights W, PipeConsts pc, unsigned long long *nodekey,
                     unsigned long long *tilekey, unsigned long long *__restrict__ keys, uint32_t *__restrict__ victims,
                     const int32_t *__restrict__ gang, int4 *__restrict__ pre) {
    plan_sequential_body<true>(topo4, free_mask, mem4, hold, N, Npad, T, node_id_base, pods4, pcol, P, cols, ncol, W, pc, nodekey,
                               tilekey, keys, victims, gang, pre);
}

}  // namespace kgpu
