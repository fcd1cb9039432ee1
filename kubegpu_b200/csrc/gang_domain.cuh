// gang_domain.cuh -- the domain step of kgpu_place_batch_gang_domain: one CONSTRAINED gang (consecutive pods with the
// same nonzero gang id and the same nonzero gang_domain) placed inside one network domain (include/kgpu.h has the
// definition).  It runs between the place_sequential launches of the batch, on the tables K3 keeps current:
//   nodebest[v][k][Npad]  (cost << 8 | S) of every node under the free masks F
//   tilebest[v][k][T]     the minimum of every 128-node tile
// and leaves them current for the launches after it (place_sequential rebuilds its supertile minima from tilebest).
//
// domain_trial  : warp per domain, grid-strided over the D domains.  The warp places the members in order inside its
//                 domain on a working copy F_d of F and, if every member fits, atomicMin's (C_d << 32 | d) into *best.
//                 F_d lives in per-node scratch: node n's working mask is dmask[n] when dstamp[n] == the trial's stamp,
//                 F[n] otherwise.  Domains are disjoint, so no two warps touch one node, and the scratch bounds neither
//                 the domain size nor the member count.  Per member, lanes walk the domain's node list 32 at a time; a
//                 lane's candidate is nodebest[v][k][n], or, for a node the trial has already changed, the node
//                 re-scored by the whole warp under F_d from its half tables (node_key_warp, as in K3's refresh).
//                 One REDUX pair per member gives the winner.
// Levels (kgpu_place_batch_gang_levels): a gang with level bound r gets one domain_trial launch per level 0..r, each on
//                 that level's domains and writing its own best[l]; a launch whose lower levels already have a winner
//                 exits at once, and domain_commit takes the lowest level with one.  Domain ids are the table's (level
//                 bases added), so the commit needs no level.  kgpu_place_batch_gang_domain is r = 0.
// domain_commit : one block.  If a domain won, warp 0 reruns its trial (same function, new stamp: the same keys),
//                 storing the members' keys, and the block applies F_d to F node by node.  If none did: REQUIRED gives
//                 every member NO_FIT; PREFERRED places the members over all nodes as K3's GANG path would (winner =
//                 minimum of tilebest[v][k] over the T tiles), giving the GPUs back on a miss.  Every node whose mask
//                 changes gets all V x 9 nodebest rows re-scored and its tile's tilebest entries refreshed.
// C_d: a member costs at most 28 * 4095 = 114 660, so a gang of up to DOM_MAX_MEMBERS members keeps C_d within 32 bits
// (the host refuses larger constrained gangs).
#pragma once
#include "place_sequential.cuh"

namespace kgpu {

constexpr int DOM_THREADS = 256;                 // domain_trial: 8 warps, one domain each at a time
constexpr int DOM_WARPS = DOM_THREADS / 32;
constexpr int DOM_COMMIT_THREADS = 288;          // domain_commit: 9 warps, one per k of a view
constexpr int DOM_COMMIT_WARPS = DOM_COMMIT_THREADS / 32;
constexpr int64_t DOM_MAX_MEMBERS = 37000;       // 37 000 * 114 660 < 2^32
constexpr int GANG_DOMAIN_REQUIRED = 1, GANG_DOMAIN_PREFERRED = 2;
constexpr int DOM_CHUNK = 32;                    // nodes per chunk of the chunked walk

// What both kernels read and write, besides the gang's pods.
struct DomainArgs {
    int32_t *free_mask;                          // F [N]: read by the trial, written by the commit
    const int32_t *gpu_mem;                      // [N][8]
    int64_t Npad, T, node_id_base;
    PlaceViews views;
    uint32_t *nodebest;                          // [views][9][Npad]
    unsigned long long *tilebest;                // [views][9][T]
    const int32_t *half_all;                     // [N][96]  place_half_tables
    const int32_t *dom_off, *dom_nodes;          // domain d's nodes: dom_nodes[dom_off[d] .. dom_off[d + 1])
    int32_t *dmask;                              // [N] working masks of the trials
    uint32_t *dstamp;                            // [N] the stamp of the trial that wrote dmask[n]
    // The chunked walk (levels with large domains; all null / 0 = the plain walk only).  Each domain's node list is cut
    // into chunks of DOM_CHUNK consecutive entries; chunks are numbered over the whole table, in list order, so chunk c
    // is dom_nodes[chunk_begin[c] .. chunk_begin[c + 1]).
    const int32_t *dom_chunk;                    // domain g's chunks: dom_chunk[g] .. dom_chunk[g + 1] (laid out as dom_off)
    const int32_t *chunk_begin;                  // [chunks + 1]
    unsigned long long *cmin;                    // [views * 9][chunks] each chunk's minimum wide key under F
    uint32_t *cstamp;                            // [chunks] the stamp of the trial that changed a node of the chunk
    int64_t chunks;
};

struct DomainShared {
    int32_t view_min[PLACE_MAX_VIEWS];
    uint8_t sub[9][72];                          // the k-subsets of 8 GPUs, increasing (node_key_warp)
    int32_t nsub[9];
};

__device__ __forceinline__ void domain_shared_init(DomainShared &sh, const PlaceViews &views, int tid) {
    if (tid == 0) {
#pragma unroll
        for (int i = 0; i < PLACE_MAX_VIEWS; i++) sh.view_min[i] = views.min_mem[i];
    }
    if (tid < 9) {
        const int n = c_nsub[tid];
        sh.nsub[tid] = n;
        for (int i = 0; i < n; i++) sh.sub[tid][i] = c_subsets[tid][i];
    }
}

// the view of a pod with memory requirement `need`: the one with its min_mem (0 without one)
__device__ __forceinline__ int domain_pod_view(const DomainShared &sh, int V, int32_t need) {
    int v = 0;
    for (int j = 1; j < V; j++)
        if (need == sh.view_min[j]) v = j;
    return v;
}

// One trial, by one warp: the j members pods4[0..j) placed in order inside domain d on F_d (see the top).  Returns C_d,
// or -1 when a member asks for k outside 0..8 or does not fit.  keys != nullptr: lane 0 stores every member's key.
// The minimum wide key over the list entries [b, b1) (at most 32), by the whole warp, under F_d: a node this trial has
// changed is re-scored by the whole warp from its half tables, the others read nodebest.
__device__ __forceinline__ unsigned long long domain_scan32(const DomainArgs &a, const DomainShared &sh, const uint32_t *nb, int k,
                                                            int32_t need, uint32_t stamp, int64_t b, int64_t b1, int lane) {
    const int64_t e = b + lane;
    int32_t n = -1;
    uint32_t nk = INF32;
    bool changed = false;
    if (e < b1) {
        n = __ldg(a.dom_nodes + e);
        changed = a.dstamp[n] == stamp;
        if (!changed) nk = nb[n];
    }
    uint32_t todo = __ballot_sync(0xFFFFFFFFu, changed);
    while (todo) {
        const int src = __ffs(todo) - 1;
        todo &= todo - 1;
        const int32_t m = __shfl_sync(0xFFFFFFFFu, n, src);
        const uint32_t fm = (uint32_t)a.dmask[m] & view_ok_mask(a.gpu_mem, m, need);
        const uint32_t key = node_key_warp(k, a.half_all + (int64_t)m * PLACE_HALF, fm, lane, sh.sub[k], sh.nsub[k]);
        if (lane == src) nk = key;
    }
    return n >= 0 ? wide_key(nk, (unsigned long long)(a.node_id_base + n)) : ~0ull;
}

template <bool CHUNKED>
__device__ __forceinline__ int64_t domain_try(const DomainArgs &a, const DomainShared &sh, int d, uint32_t stamp,
                                              const int4 *__restrict__ pods4, int64_t j, unsigned long long *keys, int lane) {
    const int64_t b0 = __ldg(a.dom_off + d), b1 = __ldg(a.dom_off + d + 1);
    int64_t cost = 0;
#pragma unroll 1
    for (int64_t i = 0; i < j; i++) {
        const int4 req = __ldg(pods4 + i);
        const int k = req.x;
        if (k < 0 || k > 8) return -1;
        const int v = domain_pod_view(sh, a.views.n, req.w);
        const int32_t need = sh.view_min[v];
        const uint32_t *nb = a.nodebest + ((int64_t)v * 9 + k) * a.Npad;
        unsigned long long best = ~0ull;
        int32_t chunk = -1;                             // chunked walk: the chunk the winner sits in
        if (CHUNKED) {                                  // lane per chunk: its minimum, or a rescan if this trial changed it
            const int64_t h0 = __ldg(a.dom_chunk + d), h1 = __ldg(a.dom_chunk + d + 1);
            const unsigned long long *cm = a.cmin + ((int64_t)v * 9 + k) * a.chunks;
            int32_t mine = -1;
#pragma unroll 1
            for (int64_t hb = h0; hb < h1; hb += 32) {
                const int64_t c = hb + lane;
                unsigned long long cand = ~0ull;
                bool stamped = false;
                if (c < h1) {
                    stamped = a.cstamp[c] == stamp;
                    if (!stamped) cand = cm[c];
                }
                uint32_t todo = __ballot_sync(0xFFFFFFFFu, stamped);
                while (todo) {
                    const int src = __ffs(todo) - 1;
                    todo &= todo - 1;
                    const int64_t cc = __shfl_sync(0xFFFFFFFFu, c, src);
                    const unsigned long long m =
                        warp_min_u64_redux(domain_scan32(a, sh, nb, k, need, stamp, __ldg(a.chunk_begin + cc), __ldg(a.chunk_begin + cc + 1), lane));
                    if (lane == src) cand = m;
                }
                if (cand < best) best = cand, mine = (int32_t)c;
            }
            const unsigned long long w = warp_min_u64_redux(best);
            const uint32_t own = __ballot_sync(0xFFFFFFFFu, best == w && w != ~0ull);
            chunk = __shfl_sync(0xFFFFFFFFu, mine, own ? __ffs(own) - 1 : 0);
            best = w;
        } else {                                        // lane per node, 32 at a time
#pragma unroll 1
            for (int64_t b = b0; b < b1; b += 32) best = min(best, domain_scan32(a, sh, nb, k, need, stamp, b, b1, lane));
            best = warp_min_u64_redux(best);
        }
        if (keys != nullptr && lane == 0) keys[i] = best;
        if (best == ~0ull) return -1;
        cost += (int64_t)(best >> 40);
        const uint32_t S = (uint32_t)(best & 0xFFull);
        if (lane == 0 && S != 0) {
            const int64_t n = (int64_t)((best >> 8) & 0xFFFFFFFFull) - a.node_id_base;
            const uint32_t fm = a.dstamp[n] == stamp ? (uint32_t)a.dmask[n] : ((uint32_t)a.free_mask[n] & 0xFFu);
            a.dmask[n] = (int32_t)(fm & ~S);
            a.dstamp[n] = stamp;
            if (CHUNKED) a.cstamp[chunk] = stamp;
        }
        __syncwarp();                                   // lane 0's scratch writes are seen by the next member's walk
    }
    return cost;
}

// Node n of F gets `mask`: all V x 9 node keys re-scored (warp per (view, k), node_key_warp), then the minima of its
// tile.  Called by every thread of the block with the same arguments; the mask is stored after the first barrier, so
// callers may compute it from F[n].
__device__ __forceinline__ void domain_apply(const DomainArgs &a, const DomainShared &sh, int64_t n, uint32_t mask, int tid) {
    const int lane = tid & 31, warp = tid >> 5;
    const int ntask = a.views.n * 9;
    const int tile = (int)(n >> 7);
    for (int task = warp; task < ntask; task += DOM_COMMIT_WARPS) {
        const int tv = task / 9, tk = task - tv * 9;
        const uint32_t ok = view_ok_mask(a.gpu_mem, n, sh.view_min[tv]);
        const uint32_t nk = node_key_warp(tk, a.half_all + n * PLACE_HALF, mask & ok, lane, sh.sub[tk], sh.nsub[tk]);
        if (lane == 0) a.nodebest[(int64_t)task * a.Npad + n] = nk;
    }
    __syncthreads();
    if (tid == 0) a.free_mask[n] = (int32_t)mask;
    for (int task = warp; task < ntask; task += DOM_COMMIT_WARPS) {
        const uint32_t *row = a.nodebest + (int64_t)task * a.Npad + (int64_t)tile * PLACE_TILE;
        uint32_t m = INF32;
#pragma unroll
        for (int q = 0; q < PLACE_TILE / 32; q++) m = tile_fold(m, row[lane + 32 * q], lane + 32 * q);
        const unsigned long long tb = tile_min_key(m, a.node_id_base, tile);
        if (lane == 0) a.tilebest[(int64_t)task * a.T + tile] = tb;
    }
    __syncthreads();
}

// The chunk minima of one level for the chunked walk: chunks c0 .. c0 + C - 1, one warp per chunk (grid-strided), one
// grid row per (view, k) pair of the gang, pairs[y] = v * 9 + k.  cmin[pair][c] = the minimum of wide_key(nodebest) over
// the chunk's nodes under F.  Exits at once when a lower level of the step has a winner, as domain_trial does.
__global__ void __launch_bounds__(DOM_THREADS)
domain_chunk_min(DomainArgs a, int64_t c0, int64_t C, const int32_t *__restrict__ pairs, const unsigned long long *best, int32_t level) {
    for (int l = 0; l < level; l++)
        if (best[l] != ~0ull) return;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int32_t pair = __ldg(pairs + blockIdx.y);
    const uint32_t *nb = a.nodebest + (int64_t)pair * a.Npad;
    for (int64_t c = c0 + (int64_t)blockIdx.x * DOM_WARPS + warp; c < c0 + C; c += (int64_t)gridDim.x * DOM_WARPS) {
        const int64_t e = __ldg(a.chunk_begin + c) + lane;
        unsigned long long key = ~0ull;
        if (e < __ldg(a.chunk_begin + c + 1)) {
            const int32_t n = __ldg(a.dom_nodes + e);
            key = wide_key(nb[n], (unsigned long long)(a.node_id_base + n));
        }
        key = warp_min_u64_redux(key);
        if (lane == 0) a.cmin[(int64_t)pair * a.chunks + c] = key;
    }
}

// The trials of one level: the D domains base .. base + D - 1 of the table (kgpu_upload_domain_levels lays the levels out
// one after another; level 0 has base 0).  best[0 .. level] are the step's per-level results: the kernel exits at once
// when a lower level has a winner, else atomicMin's (C_d << 32 | base + d) into best[level].
__global__ void __launch_bounds__(DOM_THREADS)
domain_trial(DomainArgs a, const int4 *__restrict__ pods4, int64_t j, int32_t D, uint32_t stamp, unsigned long long *best,
             int32_t level = 0, int32_t base = 0, int32_t chunked = 0) {
    __shared__ DomainShared sh;
    for (int l = 0; l < level; l++)
        if (best[l] != ~0ull) return;                   // the gang takes the lowest level that fits
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    domain_shared_init(sh, a.views, tid);
    __syncthreads();
    for (int d = base + (int)blockIdx.x * DOM_WARPS + warp; d < base + D; d += (int)gridDim.x * DOM_WARPS) {
        if (__ldg(a.dom_off + d) == __ldg(a.dom_off + d + 1)) continue;
        const int64_t c = chunked ? domain_try<true>(a, sh, d, stamp, pods4, j, nullptr, lane)
                                  : domain_try<false>(a, sh, d, stamp, pods4, j, nullptr, lane);
        if (c >= 0 && lane == 0) atomicMin(best + level, ((unsigned long long)c << 32) | (uint32_t)d);
    }
}

// One block per launch, so the register budget is the block's alone (min blocks 1): at the default bound the two walks'
// reruns spill.
__global__ void __launch_bounds__(DOM_COMMIT_THREADS, 1)
domain_commit(DomainArgs a, const int4 *__restrict__ pods4, int64_t j, int mode, uint32_t stamp,
              const unsigned long long *best, unsigned long long *keys, int32_t levels = 1, int32_t chunked_levels = 0) {
    __shared__ DomainShared sh;
    __shared__ unsigned long long sRed[DOM_COMMIT_WARPS];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    domain_shared_init(sh, a.views, tid);
    __syncthreads();
    unsigned long long won = ~0ull;                     // the lowest level with a winner: best[0 .. levels)
    int wl = 0;
    for (; wl < levels; wl++)
        if ((won = best[wl]) != ~0ull) break;
    if (won != ~0ull) {                                 // domain won: its trial again, then F_d into F
        if (warp == 0) {
            if ((chunked_levels >> wl) & 1) domain_try<true>(a, sh, (int)(uint32_t)won, stamp, pods4, j, keys, lane);
            else domain_try<false>(a, sh, (int)(uint32_t)won, stamp, pods4, j, keys, lane);
        }
        __syncthreads();
        for (int64_t i = 0; i < j; i++) {
            const unsigned long long key = keys[i];
            if ((key & 0xFFull) == 0) continue;         // k = 0 took nothing
            const int64_t n = (int64_t)((key >> 8) & 0xFFFFFFFFull) - a.node_id_base;
            domain_apply(a, sh, n, (uint32_t)a.dmask[n], tid);
        }
        return;
    }
    if (mode == GANG_DOMAIN_REQUIRED) {
        for (int64_t i = tid; i < j; i += DOM_COMMIT_THREADS) keys[i] = ~0ull;
        return;
    }
    // PREFERRED and no domain fits: all or nothing over every node
    int64_t i = 0;
    for (; i < j; i++) {
        const int4 req = __ldg(pods4 + i);
        const int k = req.x;
        if (k < 0 || k > 8) break;
        const int v = domain_pod_view(sh, a.views.n, req.w);
        const unsigned long long *tb = a.tilebest + ((int64_t)v * 9 + k) * a.T;
        unsigned long long b = ~0ull;
        for (int64_t t = tid; t < a.T; t += DOM_COMMIT_THREADS) b = min(b, tb[t]);
        b = warp_min_u64_redux(b);
        if (lane == 0) sRed[warp] = b;
        __syncthreads();
        unsigned long long win = ~0ull;
#pragma unroll
        for (int w = 0; w < DOM_COMMIT_WARPS; w++) win = min(win, sRed[w]);
        if (tid == 0) keys[i] = win;
        __syncthreads();                                // sRed is free again
        if (win == ~0ull) break;
        const uint32_t S = (uint32_t)(win & 0xFFull);
        if (S == 0) continue;
        const int64_t n = (int64_t)((win >> 8) & 0xFFFFFFFFull) - a.node_id_base;
        domain_apply(a, sh, n, ((uint32_t)a.free_mask[n] & 0xFFu) & ~S, tid);
    }
    if (i == j) return;
    // a member missed: the members before it give their GPUs back, last first, and every member gets NO_FIT
    for (int64_t q = i - 1; q >= 0; q--) {
        const unsigned long long key = keys[q];         // tid 0 wrote it before a barrier
        const uint32_t S = (uint32_t)(key & 0xFFull);
        if (S == 0) continue;
        const int64_t n = (int64_t)((key >> 8) & 0xFFFFFFFFull) - a.node_id_base;
        domain_apply(a, sh, n, ((uint32_t)a.free_mask[n] & 0xFFu) | S, tid);
    }
    __syncthreads();                                    // every thread has read the keys
    for (int64_t q = tid; q < j; q += DOM_COMMIT_THREADS) keys[q] = ~0ull;
}

}  // namespace kgpu
