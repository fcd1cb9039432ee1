// preempt_plan_domain.cuh -- the domain step of kgpu_preempt_plan_gang_domain: one CONSTRAINED gang (consecutive pods with
// the same nonzero gang id and the same nonzero gang_domain) planned inside one network domain (include/kgpu.h has the
// definition).  It runs between the gang_plan_sequential launches of the batch, on the tables K5 keeps current for the
// working state (F, H):
//   nodekey[c][Npad]  K5's key of every node for column c: (level 4 | |V| 4) << 56 | cost << 39 | local node << 8 | S
//   tilekey[c][T]     the minimum of every 128-node tile
// and leaves them current for the launches after it.
//
// domain_plan_trial  : warp per domain, grid-strided over the D domains.  The warp plans the members in order inside its
//                      domain on a working copy (F_d, H_d) and writes the trial's score (L_d << 51 | V_d << 32 | C_d), or
//                      ~0 when a member misses, to score[d].  (F_d, H_d) lives in per-node scratch: node n's working
//                      mask and packed holder row are dmask[n] / dhold[n] when dstamp[n] == the trial's stamp, F[n] /
//                      H[n] otherwise.  Domains are disjoint, so no two warps touch one node.  Per member, lanes walk the
//                      domain's node list 32 at a time; a lane's candidate is nodekey[c][n], or, for a node the trial has
//                      already changed, plan_node_key on the scratch state (a per-lane function, so no warp-wide
//                      re-score).  One 64-bit REDUX min per member gives the winner; lane 0 applies the update rule.
// domain_plan_commit : one block of PLAN_THREADS.  The winner is the smallest (score[d], d).  If a domain won, warp 0
//                      reruns its trial (same function, new stamp: the same keys), storing keys and victims, and the
//                      block copies each changed node's final scratch state into (F, H) and refreshes its keys and tile
//                      minima with plan_refresh.  If none did: REQUIRED gives every member NO_FIT and victims 0;
//                      PREFERRED runs plan_sequential_body<true> on the gang, the all-or-nothing gang plan over every node.
// Score fields: L < 16 (4 bits); V_d <= 8 victims x DOM_MAX_MEMBERS < 2^19; C_d <= 114 660 x DOM_MAX_MEMBERS < 2^32.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "gang_domain.cuh"
#include "preempt_plan.cuh"

namespace kgpu {

// What both kernels read and write, besides the gang's pods.
struct PlanDomainArgs {
    const int4 *topo4;                           // [N][16]
    int32_t *free_mask;                          // F [N]: read by the trial, written by the commit
    const int4 *mem4;                            // [N][2]
    int32_t *hold;                               // H [N][8]
    int64_t N, Npad, T, node_id_base;
    const int4 *cols;                            // the batch's columns {k, level, min_mem, 0}
    int ncol;
    unsigned long long *nodekey;                 // [ncol][Npad]
    unsigned long long *tilekey;                 // [ncol][T]
    const int32_t *dom_off, *dom_nodes;          // domain d's nodes: dom_nodes[dom_off[d] .. dom_off[d + 1])
    int32_t *dmask;                              // [N] working masks of the trials
    uint2 *dhold;                                // [N] working holder rows, one byte per GPU (as gang_plan_sequential's pre[])
    uint32_t *dstamp;                            // [N] the stamp of the trial that wrote dmask[n] / dhold[n]
};

__device__ __forceinline__ void plan_unpack_row(uint2 q, int32_t (&h)[8]) {
#pragma unroll
    for (int g = 0; g < 8; g++) h[g] = (int32_t)(int8_t)(((g < 4 ? q.x : q.y) >> (8 * (g & 3))) & 0xFFu);
}

__device__ __forceinline__ uint2 plan_pack_row(const int32_t (&h)[8]) {
    uint32_t lo = 0, hi = 0;
#pragma unroll
    for (int g = 0; g < 4; g++) {
        lo |= ((uint32_t)h[g] & 0xFFu) << (8 * g);
        hi |= ((uint32_t)h[g + 4] & 0xFFu) << (8 * g);
    }
    return make_uint2(lo, hi);
}

// One trial, by one warp: the j members pods4[0..j) (columns pcol[0..j)) planned in order inside domain d on (F_d, H_d)
// (see the top).  Returns the score L << 51 | V << 32 | C, or ~0 when a member asks for k outside 0..8 or has no
// candidate.  keys != nullptr: lane 0 stores every member's key and victims.
__device__ __forceinline__ unsigned long long domain_plan_try(const PlanDomainArgs &a, const int32_t *sW, PipeConsts pc, int d,
                                                              uint32_t stamp, const int4 *__restrict__ pods4,
                                                              const int32_t *__restrict__ pcol, int64_t j, unsigned long long *keys,
                                                              uint32_t *victims, int lane) {
    const int64_t b0 = __ldg(a.dom_off + d), b1 = __ldg(a.dom_off + d + 1);
    uint32_t L = 0, V = 0, C = 0;
#pragma unroll 1
    for (int64_t i = 0; i < j; i++) {
        const int c = __ldg(pcol + i);
        unsigned long long best;
        if (c < 0) {                                    // k outside 1..8: k = 0 takes the domain's lowest node, else a miss
            if (__ldg(pods4 + i).x != 0) return ~0ull;
            best = (unsigned long long)__ldg(a.dom_nodes + b0) << 8;
        } else {
            const int4 col = __ldg(a.cols + c);
            const unsigned long long *nk = a.nodekey + (int64_t)c * a.Npad;
            best = ~0ull;
#pragma unroll 1
            for (int64_t b = b0; b < b1; b += 32) {
                const int64_t e = b + lane;
                if (e >= b1) continue;
                const int64_t n = __ldg(a.dom_nodes + e);
                unsigned long long key;
                if (a.dstamp[n] == stamp) {             // changed by this trial: re-scored on (F_d, H_d)
                    PairCosts pcs;
                    plan_pair_costs(a.topo4, n, true, sW, pcs);
                    int32_t mem[8], h[8];
                    const int4 m0 = __ldg(a.mem4 + n * 2), m1 = __ldg(a.mem4 + n * 2 + 1);
                    mem[0] = m0.x; mem[1] = m0.y; mem[2] = m0.z; mem[3] = m0.w;
                    mem[4] = m1.x; mem[5] = m1.y; mem[6] = m1.z; mem[7] = m1.w;
                    plan_unpack_row(a.dhold[n], h);
                    const uint32_t F = (uint32_t)a.dmask[n] & 0xFFu;
                    uint64_t gm;
                    uint32_t lvp;
                    plan_owners(h, F, gm, lvp);
                    key = plan_node_key(pcs, pc, F, gm, lvp, mem, col, n);
                } else {
                    key = nk[n];
                }
                best = min(best, key);
            }
            best = warp_min_u64_redux(best);
            if (best == ~0ull) return ~0ull;
        }
        const int64_t n = (int64_t)((best >> 8) & 0x7FFFFFFFull);
        const uint32_t S = (uint32_t)best & 0xFFu, cost = (uint32_t)(best >> 39) & 0x1FFFFu;
        if (lane == 0) {
            uint32_t vic = 0;
            if (S != 0) {                               // the update rule of kgpu_preempt_plan on (F_d, H_d)
                const bool mine = a.dstamp[n] == stamp;
                const uint32_t f = mine ? (uint32_t)a.dmask[n] & 0xFFu : (uint32_t)a.free_mask[n] & 0xFFu;
                int32_t h[8];
                if (mine) {
                    plan_unpack_row(a.dhold[n], h);
                } else {
#pragma unroll
                    for (int g = 0; g < 8; g++) h[g] = a.hold[n * 8 + g];
                }
#pragma unroll
                for (int g = 0; g < 8; g++)
                    if (((S & ~f) >> g) & 1u) vic |= 1u << (h[g] & 7);
                uint32_t R = 0;
#pragma unroll
                for (int g = 0; g < 8; g++)
                    if (!((f >> g) & 1u) && h[g] >= 0 && ((vic >> (h[g] & 7)) & 1u)) R |= 1u << g;
#pragma unroll
                for (int g = 0; g < 8; g++)
                    if (((S | R) >> g) & 1u) h[g] = -1;
                a.dmask[n] = (int32_t)((f | R) & ~S);
                a.dhold[n] = plan_pack_row(h);
                a.dstamp[n] = stamp;
            }
            if (keys != nullptr) {
                keys[i] = ((unsigned long long)cost << 40) | ((unsigned long long)(a.node_id_base + n) << 8) | S;
                victims[i] = vic;
            }
        }
        L = max(L, (uint32_t)(best >> 60));
        V += (uint32_t)(best >> 56) & 15u;
        C += cost;
        __syncwarp();                                   // lane 0's scratch writes are seen by the next member's walk
    }
    return ((unsigned long long)L << 51) | ((unsigned long long)V << 32) | C;
}

__global__ void __launch_bounds__(DOM_THREADS)
domain_plan_trial(PlanDomainArgs a, Weights W, PipeConsts pc, const int4 *__restrict__ pods4, const int32_t *__restrict__ pcol,
                  int64_t j, int32_t D, uint32_t stamp, unsigned long long *score) {
    __shared__ int32_t sW[16];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid < 16) sW[tid] = W.w[tid];
    __syncthreads();
    for (int d = (int)blockIdx.x * DOM_WARPS + warp; d < D; d += (int)gridDim.x * DOM_WARPS) {
        const unsigned long long s =
            __ldg(a.dom_off + d) == __ldg(a.dom_off + d + 1) ? ~0ull : domain_plan_try(a, sW, pc, d, stamp, pods4, pcol, j, nullptr, nullptr, lane);
        if (lane == 0) score[d] = s;
    }
}

// gang[0..j) and pre[0..j): the gang's ids and pre-image scratch, for the PREFERRED fallback.
__global__ void __launch_bounds__(PLAN_THREADS, 1)
domain_plan_commit(PlanDomainArgs a, Weights W, PipeConsts pc, const int4 *__restrict__ pods4, const int32_t *__restrict__ pcol,
                   const int32_t *__restrict__ gang, int64_t j, int mode, int32_t D, uint32_t stamp,
                   const unsigned long long *__restrict__ score, unsigned long long *__restrict__ keys, uint32_t *__restrict__ victims,
                   int4 *__restrict__ pre) {
    __shared__ int32_t sW[16];
    __shared__ int4 sCol[PLAN_MAX_COLS];
    __shared__ unsigned long long sRed[PLAN_WARPS];
    __shared__ uint32_t sRedD[PLAN_WARPS];
    __shared__ int32_t sF, sH[8];
    __shared__ int32_t sResc[PLAN_MAX_COLS];
    __shared__ int sNresc;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid < 16) sW[tid] = W.w[tid];
    if (tid < a.ncol) sCol[tid] = __ldg(a.cols + tid);
    // the winner: the smallest (score[d], d); each thread keeps its first d of the smallest score it sees
    unsigned long long b = ~0ull;
    uint32_t bd = 0xFFFFFFFFu;
    for (int d = tid; d < D; d += PLAN_THREADS) {
        const unsigned long long s = __ldg(score + d);
        if (s < b) { b = s; bd = (uint32_t)d; }
    }
    const unsigned long long wb = warp_min_u64_redux(b);
    const uint32_t wd = __reduce_min_sync(0xFFFFFFFFu, b == wb ? bd : 0xFFFFFFFFu);
    if (lane == 0) { sRed[warp] = wb; sRedD[warp] = wd; }
    __syncthreads();
    unsigned long long won = ~0ull;
    uint32_t wdom = 0xFFFFFFFFu;
#pragma unroll
    for (int w = 0; w < PLAN_WARPS; w++)
        if (sRed[w] < won || (sRed[w] == won && sRedD[w] < wdom)) { won = sRed[w]; wdom = sRedD[w]; }
    if (won != ~0ull) {                                 // a domain won: its trial again, then (F_d, H_d) into (F, H)
        if (warp == 0) domain_plan_try(a, sW, pc, (int)wdom, stamp, pods4, pcol, j, keys, victims, lane);
        __syncthreads();
#pragma unroll 1
        for (int64_t i = 0; i < j; i++) {
            const unsigned long long key = keys[i];
            if ((key & 0xFFull) == 0) continue;         // k = 0 took nothing
            const int64_t n = (int64_t)((key >> 8) & 0xFFFFFFFFull) - a.node_id_base;
            if (a.dstamp[n] != stamp) continue;         // an earlier member's node, already applied
            __syncthreads();                            // every thread has read dstamp[n]
            if (tid == 0) {
                const int32_t f = a.dmask[n];
                int32_t h[8];
                plan_unpack_row(a.dhold[n], h);
                a.free_mask[n] = f;
                sF = f;
#pragma unroll
                for (int g = 0; g < 8; g++) {
                    a.hold[n * 8 + g] = h[g];
                    sH[g] = h[g];
                }
                a.dstamp[n] = 0;
                sNresc = 0;
            }
            __syncthreads();
            plan_refresh(n, a.topo4, a.mem4, a.Npad, a.T, a.ncol, pc, a.nodekey, a.tilekey, sW, sCol, sF, sH, sResc, sNresc);
        }
        return;
    }
    if (mode == GANG_DOMAIN_REQUIRED) {
        for (int64_t i = tid; i < j; i += PLAN_THREADS) {
            keys[i] = ~0ull;
            victims[i] = 0;
        }
        return;
    }
    // PREFERRED and no domain fits: the gang plan over every node, all or nothing
    plan_sequential_body<true>(a.topo4, a.free_mask, a.mem4, a.hold, a.N, a.Npad, a.T, a.node_id_base, pods4, pcol, j, a.cols, a.ncol, W,
                               pc, a.nodekey, a.tilekey, keys, victims, gang, pre);
}

}  // namespace kgpu
