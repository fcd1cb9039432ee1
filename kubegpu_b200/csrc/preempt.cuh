// preempt.cuh -- K4: preemption for the pods that fit nowhere (kgpu_preempt_batch), sm_90a.
//
// Definition (include/kgpu.h).  Node n has a holder table row hold[n][8]: -1, or level << 3 | owner, for each GPU
// slot; entries of free GPUs are ignored.  Pod p (k GPUs, min_mem, level L) may use GPU i of node n if it is free, or
// if it is held by an owner of level < L; either way it must pass min_mem.  A candidate is (n, S) with S a k-subset of
// usable GPUs; its victims V(S) are the owners of S's GPUs that are not free.  The winner is the smallest
// (max level in V, |V|, cost(S), node id, S), with an empty V first.
//
// The kernel enumerates victim SETS, not subsets S.  Per (pod, node) lane:
//   1. E = the owners with level < L that hold at least one GPU the pod may use (an owner that frees nothing usable
//      only makes V bigger).  V = {} is the class (0, 0).
//   2. m* = the lowest level m such that evicting every owner of E with level <= m frees enough GPUs.  Any V that
//      fits inside those owners has max level m* (a V of lower max level would have made a lower m fit).
//   3. s* = the smallest |V| of a fitting V among those owners, by enumerating their subsets (popcount checks only).
//   4. For every V of size s* that fits, the dense node_key_k<K> over free | GPUs(V) with the min_mem penalties
//      applied as K1m does; the best (cost << 8 | S) over them.  In the first fitting class (m*, s*) every usable S has
//      V(S) = V: an S that left one of V's owners unused would fit a strictly smaller set, which is in an earlier class.
// Steps 3 and 4 run only on the lanes whose class equals the warp's minimum (a warp REDUX after each step): the
// others cannot win.  The lane key is (level 4 | |V| 4 | cost 17 | local node 31 | S 8) = 64 bits, reduced over the
// warp (two 32-bit REDUX.MIN), the block (shared rows) and the grid (REDG.MIN.64 into a per-pod scratch key);
// preempt_finalize turns it into the standard key and the victims' owner mask.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "score_pairs.cuh"

namespace kgpu {

constexpr int PRE_THREADS = 128;
constexpr int PRE_WARPS = PRE_THREADS / 32;
constexpr int PRE_CHUNK = 256;                  // pods per shared-memory chunk
constexpr uint32_t PRE_NO_CLASS = 0xFFFu;

// The pods that reach K4: no key from scoring, k in 1..8 (k = 0 fits wherever there is a node) and a level above 0
// (a level-0 pod evicts nothing).  idx[] gets their positions in any order; *count must be 0 before the launch.
__global__ void preempt_compact(const int4 *__restrict__ pods4, const int32_t *__restrict__ lvl,
                                const unsigned long long *__restrict__ keys, int64_t P, int32_t *__restrict__ idx,
                                int *__restrict__ count) {
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= P) return;
    const int k = __ldg(pods4 + p).x;
    if (keys[p] == ~0ull && k >= 1 && k <= 8 && __ldg(lvl + p) > 0) idx[atomicAdd(count, 1)] = (int32_t)p;
}

// GPU mask freed by evicting the owners in V (bit o = owner o): byte o of gm is owner o's non-free GPUs.
__device__ __forceinline__ uint32_t gpus_of(uint64_t gm, uint32_t V) {
    uint32_t g = 0;
    for (uint32_t u = V; u; u &= u - 1) g |= (uint32_t)(gm >> (8 * (__ffs(u) - 1))) & 0xFFu;
    return g;
}

// This lane's best (cost << 8 | S) over k-subsets of `avail` (>= K GPUs): min_mem-style penalties on the rest.
template <int K>
__device__ __forceinline__ uint32_t preempt_dense(const PairCosts &C, const PipeConsts pc, uint32_t avail) {
    if constexpr (K == 1) {
        return best_k1(avail, pc);
    } else {
        uint32_t pen[8];
#pragma unroll
        for (int g = 0; g < 8; g++) pen[g] = (avail >> g) & 1u ? 0u : PEN;
        PairCosts C2;
        apply_pens(C, C2, pen);
        return node_key_k<K>(C2, pc, avail, true);
    }
}

template <int K>
__device__ __forceinline__ void preempt_bucket(const PairCosts &C, const PipeConsts pc, uint32_t F, uint64_t gm,
                                               uint32_t lvp, const int32_t (&mem)[8], uint64_t node_field, int lane,
                                               const uint16_t *sIdx, const int32_t *sLvl, const int32_t *sMin,
                                               int begin, int end, unsigned long long *sBestW) {
#pragma unroll 1
    for (int i = begin; i < end; i++) {
        const int p = sIdx[i];
        const int32_t L = sLvl[p], need = sMin[p];
        uint32_t elig = 0xFFu;
        if (need > 0) {
            elig = 0;
#pragma unroll
            for (int g = 0; g < 8; g++) elig |= mem[g] >= need ? 1u << g : 0u;
        }
        const uint32_t A0 = F & elig;
        // evictable owners that free something usable, and the levels they carry
        uint32_t E = 0, lvmask = 0;
#pragma unroll
        for (int o = 0; o < 8; o++) {
            const uint32_t lo = (lvp >> (4 * o)) & 15u;
            if (((uint32_t)(gm >> (8 * o)) & elig & 0xFFu) && (int32_t)lo < L) { E |= 1u << o; lvmask |= 1u << lo; }
        }
        uint32_t cls = PRE_NO_CLASS, X = 0;      // class = level << 4 | |V|; 15 = size not known yet
        bool sized = true;
        if (__popc(A0) >= K) {
            cls = 0;
        } else {
            uint32_t acc = A0;
#pragma unroll 1
            for (uint32_t lm = lvmask; lm; lm &= lm - 1) {          // levels in ascending order
                const uint32_t m = (uint32_t)__ffs(lm) - 1;
#pragma unroll
                for (int o = 0; o < 8; o++)
                    if (((E >> o) & 1u) && ((lvp >> (4 * o)) & 15u) == m) { X |= 1u << o; acc |= (uint32_t)(gm >> (8 * o)); }
                if (__popc(acc & elig & 0xFFu) >= K) { cls = m << 4 | 15u; sized = false; break; }
            }
        }
        // step 3 only where the level can still win
        const uint32_t wlevel = __reduce_min_sync(0xFFFFFFFFu, cls) >> 4;
        if (!sized) {
            if ((cls >> 4) == wlevel) {
                uint32_t smin = 9;
#pragma unroll 1
                for (uint32_t V = X; V; V = (V - 1) & X) {
                    const uint32_t s = (uint32_t)__popc(V);
                    if (s < smin && __popc((A0 | gpus_of(gm, V)) & elig) >= K) smin = s;
                }
                cls = (cls & ~15u) | smin;
            } else {
                cls = PRE_NO_CLASS;
            }
        }
        const uint32_t wcls = __reduce_min_sync(0xFFFFFFFFu, cls);
        unsigned long long v = ~0ull;
        if (cls != PRE_NO_CLASS && cls == wcls) {
            uint32_t best = INF32;
            if (cls == 0) {
                best = preempt_dense<K>(C, pc, A0);
            } else {
                const uint32_t s = cls & 15u;
#pragma unroll 1
                for (uint32_t V = X; V; V = (V - 1) & X) {
                    if ((uint32_t)__popc(V) != s) continue;
                    const uint32_t A = (A0 | gpus_of(gm, V)) & elig;
                    if (__popc(A) >= K) best = min(best, preempt_dense<K>(C, pc, A));
                }
            }
            v = ((unsigned long long)cls << 56) | ((unsigned long long)(best >> 8) << 39) | node_field | (best & 0xFFu);
        }
        const uint32_t hi = __reduce_min_sync(0xFFFFFFFFu, (uint32_t)(v >> 32));
        const uint32_t lo = __reduce_min_sync(0xFFFFFFFFu, (uint32_t)(v >> 32) == hi ? (uint32_t)v : INF32);
        if (lane == 0) sBestW[p] = ((unsigned long long)hi << 32) | lo;
    }
}

// grid = (node tiles of 128, pod splits); the compacted pods idx[0 .. *count) are walked in chunks, grid-strided over
// blockIdx.y, so the host sizes the grid from P alone.  pkey[j] (one per compacted pod, ~0 before the launch) gets the
// REDG.MIN of the block results.
__global__ void __launch_bounds__(PRE_THREADS, 3)
preempt_lane_per_node(const int4 *__restrict__ topo4, const int32_t *__restrict__ free_mask,
                      const int4 *__restrict__ mem4, const int4 *__restrict__ hold4, int64_t N,
                      const int4 *__restrict__ pods4, const int32_t *__restrict__ lvl, const int32_t *__restrict__ idx,
                      const int *__restrict__ count, Weights W, PipeConsts pc, unsigned long long *__restrict__ pkey) {
    __shared__ int32_t sW[16];
    __shared__ int32_t sCnt[10], sOff[11];
    __shared__ uint8_t sK[PRE_CHUNK];
    __shared__ uint16_t sIdx[PRE_CHUNK];
    __shared__ int32_t sLvl[PRE_CHUNK], sMin[PRE_CHUNK];
    __shared__ unsigned long long sBest[PRE_WARPS][PRE_CHUNK];

    const int tid = threadIdx.x, lane = tid & 31;
    unsigned long long *const sBestW = sBest[tid >> 5];
    const int cnt_all = *count;
    if (tid == 0) {
#pragma unroll
        for (int i = 0; i < 16; i++) sW[i] = W.w[i];
    }
    __syncthreads();

    const int64_t node = (int64_t)blockIdx.x * PRE_THREADS + tid;
    const bool valid = node < N;
    // pair costs WITHOUT the free-mask penalty: availability is per pod here
    PairCosts C;
    {
        int4 q[16];
#pragma unroll
        for (int t = 0; t < 16; t++) q[t] = valid ? __ldg(topo4 + node * 16 + t) : make_int4(0, 0, 0, 0);
        for_each_pair(C, [&](int i, int j) -> uint32_t {
            const int4 v = q[i * 2 + (j >> 2)];
            const int l = (j & 3) == 0 ? v.x : (j & 3) == 1 ? v.y : (j & 3) == 2 ? v.z : v.w;
            return (uint32_t)sW[l & 15] << 8;
        });
    }
    const uint32_t F = valid ? (uint32_t)__ldg(free_mask + node) & 0xFFu : 0u;
    int32_t mem[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    uint64_t gm = 0;          // byte o: the non-free GPUs owner o holds
    uint32_t lvp = 0;         // nibble o: owner o's level
    if (valid) {
        const int4 lo = __ldg(mem4 + node * 2), hi = __ldg(mem4 + node * 2 + 1);
        mem[0] = lo.x; mem[1] = lo.y; mem[2] = lo.z; mem[3] = lo.w;
        mem[4] = hi.x; mem[5] = hi.y; mem[6] = hi.z; mem[7] = hi.w;
        const int4 h0 = __ldg(hold4 + node * 2), h1 = __ldg(hold4 + node * 2 + 1);
        const int32_t h[8] = {h0.x, h0.y, h0.z, h0.w, h1.x, h1.y, h1.z, h1.w};
#pragma unroll
        for (int g = 0; g < 8; g++) {
            if (h[g] < 0 || ((F >> g) & 1u)) continue;
            const uint32_t o = (uint32_t)h[g] & 7u;
            gm |= 1ull << (8 * o + g);
            lvp = (lvp & ~(15u << (4 * o))) | (((uint32_t)h[g] >> 3) << (4 * o));
        }
    }
    const uint64_t node_field = (uint64_t)(valid ? node : 0) << 8;

    for (int64_t c0 = (int64_t)blockIdx.y * PRE_CHUNK; c0 < cnt_all; c0 += (int64_t)gridDim.y * PRE_CHUNK) {
        const int cn = (int)min((int64_t)PRE_CHUNK, (int64_t)cnt_all - c0);
        __syncthreads();
        if (tid < 10) sCnt[tid] = 0;
        __syncthreads();
        for (int i = tid; i < cn; i += PRE_THREADS) {
            const int32_t p = __ldg(idx + c0 + i);
            const int4 req = __ldg(pods4 + p);
            const int b = (req.x < 1 || req.x > 8) ? 9 : req.x;
            sK[i] = (uint8_t)b;
            sLvl[i] = __ldg(lvl + p);
            sMin[i] = req.w;
            atomicAdd(&sCnt[b], 1);
        }
        __syncthreads();
        if (tid == 0) {
            int acc = 0;
#pragma unroll
            for (int b = 0; b < 10; b++) { sOff[b] = acc; acc += sCnt[b]; sCnt[b] = sOff[b]; }
            sOff[10] = acc;
        }
        __syncthreads();
        for (int i = tid; i < cn; i += PRE_THREADS) sIdx[atomicAdd(&sCnt[sK[i]], 1)] = (uint16_t)i;
        __syncthreads();
        preempt_bucket<1>(C, pc, F, gm, lvp, mem, node_field, lane, sIdx, sLvl, sMin, sOff[1], sOff[2], sBestW);
        preempt_bucket<2>(C, pc, F, gm, lvp, mem, node_field, lane, sIdx, sLvl, sMin, sOff[2], sOff[3], sBestW);
        preempt_bucket<3>(C, pc, F, gm, lvp, mem, node_field, lane, sIdx, sLvl, sMin, sOff[3], sOff[4], sBestW);
        preempt_bucket<4>(C, pc, F, gm, lvp, mem, node_field, lane, sIdx, sLvl, sMin, sOff[4], sOff[5], sBestW);
        preempt_bucket<5>(C, pc, F, gm, lvp, mem, node_field, lane, sIdx, sLvl, sMin, sOff[5], sOff[6], sBestW);
        preempt_bucket<6>(C, pc, F, gm, lvp, mem, node_field, lane, sIdx, sLvl, sMin, sOff[6], sOff[7], sBestW);
        preempt_bucket<7>(C, pc, F, gm, lvp, mem, node_field, lane, sIdx, sLvl, sMin, sOff[7], sOff[8], sBestW);
        preempt_bucket<8>(C, pc, F, gm, lvp, mem, node_field, lane, sIdx, sLvl, sMin, sOff[8], sOff[9], sBestW);
        __syncthreads();
        for (int i = tid; i < cn; i += PRE_THREADS) {
            if (sK[i] == 9) continue;
            unsigned long long b = ~0ull;
#pragma unroll
            for (int w = 0; w < PRE_WARPS; w++) b = min(b, sBest[w][i]);
            if (b != ~0ull) atomicMin(&pkey[c0 + i], b);
        }
    }
}

// pkey[j] -> keys[idx[j]] (cost << 40 | node_id << 8 | S) and victims[idx[j]] (the owners of S's non-free GPUs).
__global__ void preempt_finalize(const unsigned long long *__restrict__ pkey, const int32_t *__restrict__ idx,
                                 const int *__restrict__ count, const int32_t *__restrict__ free_mask,
                                 const int32_t *__restrict__ hold, int64_t node_id_base,
                                 unsigned long long *__restrict__ keys, uint32_t *__restrict__ victims) {
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= *count) return;
    const unsigned long long v = pkey[j];
    if (v == ~0ull) return;
    const int64_t n = (int64_t)((v >> 8) & 0x7FFFFFFFull);
    const uint32_t S = (uint32_t)v & 0xFFu, cost = (uint32_t)(v >> 39) & 0x1FFFFu;
    const int32_t p = idx[j];
    keys[p] = ((unsigned long long)cost << 40) | ((unsigned long long)(node_id_base + n) << 8) | S;
    const uint32_t used = S & ~(uint32_t)free_mask[n];
    uint32_t own = 0;
#pragma unroll
    for (int g = 0; g < 8; g++)
        if ((used >> g) & 1u) own |= 1u << (hold[n * 8 + g] & 7);
    victims[p] = own;
}

// kgpu_set_holders: rows[i] (8 entries) -> hold[idx[i]]; idx holds distinct local indices.
__global__ void scatter_holders(const int32_t *__restrict__ idx, const int4 *__restrict__ rows, int64_t m,
                                int4 *__restrict__ hold4) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const int64_t n = idx[i];
    hold4[n * 2] = rows[i * 2];
    hold4[n * 2 + 1] = rows[i * 2 + 1];
}

}  // namespace kgpu
