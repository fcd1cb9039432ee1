// node_state.cuh -- device-side upkeep of the node array: everything that used to be an O(N) host pass in
// kgpu_upload_nodes (value-domain check, the K1s order) and everything a state change needs (batched free-mask
// scatter with an incremental refresh of the compacted pair-cost cache, the per-cycle (node, k) fit table that
// serves PodFitsDevice without a launch per call).
//
//   validate_topo_dev   every topo value in 0..15?  first offending element through an atomic min
//   order_count / order_scan / order_scatter
//                       the K1s order = stable counting sort of the node indices by popcount(free_mask),
//                       classes 8 .. 0, every class padded to whole warps with -1 (`pad`), the total to whole tiles.
//                       Stable = increasing node index inside a class, which the in-warp tie-break of K1s
//                       relies on (score_pairs_sparse.cuh).
//   fit_nodes           (cost<<8 | S) of every listed node for k = 0..8 -> fit[k][i]   (AddNode / Take / Return
//                       keep the host copy current; kgpu_fit_lookup reads it: gpu_scheduler.go:34-44)
// compact_nodes (score_pairs_sparse.cuh) takes the same optional node list + new masks.
#pragma once
#include "score_pairs.cuh"

namespace kgpu {

constexpr int ORD_BLOCK = 1024;             // nodes per block of the counting sort
constexpr int ORD_META = 16;                // int64 meta[]: class counts [0..8], n_slots [9]

__global__ void __launch_bounds__(256)
validate_topo_dev(const int4 *__restrict__ topo4, int64_t n_int4, unsigned long long *__restrict__ first_bad) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_int4) return;
    const int4 v = __ldg(topo4 + i);
    const uint32_t worst = max(max((uint32_t)v.x, (uint32_t)v.y), max((uint32_t)v.z, (uint32_t)v.w));
    if (worst > 15u) {
        const int c = (uint32_t)v.x > 15u ? 0 : (uint32_t)v.y > 15u ? 1 : (uint32_t)v.z > 15u ? 2 : 3;
        atomicMin(first_bad, (unsigned long long)(i * 4 + c));
    }
}

// pass 1: cnt[c * nb + b] = nodes of class c in block b
__global__ void __launch_bounds__(ORD_BLOCK)
order_count(const int32_t *__restrict__ free_mask, int64_t N, int32_t *__restrict__ cnt, int nb) {
    __shared__ int32_t s[9];
    const int tid = threadIdx.x;
    if (tid < 9) s[tid] = 0;
    __syncthreads();
    const int64_t node = (int64_t)blockIdx.x * ORD_BLOCK + tid;
    const int f = node < N ? __popc((uint32_t)__ldg(free_mask + node) & 0xFFu) : -1;
#pragma unroll
    for (int c = 0; c < 9; c++) {
        const uint32_t b = __ballot_sync(0xFFFFFFFFu, f == c);
        if ((tid & 31) == 0 && b) atomicAdd(&s[c], __popc(b));
    }
    __syncthreads();
    if (tid < 9) cnt[tid * nb + blockIdx.x] = s[tid];
}

// pass 2 (one block): off[c * nb + b] = first slot of block b's class-c nodes; meta = class counts, n_slots
__global__ void __launch_bounds__(ORD_BLOCK)
order_scan(const int32_t *__restrict__ cnt, int nb, int32_t *__restrict__ off, long long *__restrict__ meta, int tile,
           int pad /*every class is padded to a multiple of this many slots: 32 (warps) or `tile` (class-pure tiles)*/) {
    __shared__ int32_t sWarp[32];
    __shared__ int32_t sTotal;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    int32_t running = 0;                        // the same value in every thread
    for (int c = 8; c >= 0; c--) {
        int32_t carry = 0;
        for (int chunk = 0; chunk < nb; chunk += ORD_BLOCK) {
            const int i = chunk + tid;
            const int32_t v = i < nb ? cnt[c * nb + i] : 0;
            int32_t incl = v;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const int32_t up = __shfl_up_sync(0xFFFFFFFFu, incl, d);
                if (lane >= d) incl += up;
            }
            if (lane == 31) sWarp[warp] = incl;
            __syncthreads();
            if (warp == 0) {
                const int32_t w = sWarp[lane];
                int32_t wi = w;
#pragma unroll
                for (int d = 1; d < 32; d <<= 1) {
                    const int32_t up = __shfl_up_sync(0xFFFFFFFFu, wi, d);
                    if (lane >= d) wi += up;
                }
                sWarp[lane] = wi - w;           // exclusive prefix of the warp totals
                if (lane == 31) sTotal = wi;
            }
            __syncthreads();
            if (i < nb) off[c * nb + i] = running + carry + sWarp[warp] + incl - v;
            carry += sTotal;
            __syncthreads();
        }
        if (tid == 0) meta[c] = carry;
        running += (carry + pad - 1) / pad * pad;
    }
    if (tid == 0) meta[9] = ((long long)running + tile - 1) / tile * tile;
}

// pass 3: order[slot] = node and slot_of[node] = slot, stable inside a class (order must be pre-set to -1)
__global__ void __launch_bounds__(ORD_BLOCK)
order_scatter(const int32_t *__restrict__ free_mask, int64_t N, const int32_t *__restrict__ off, int nb,
              int32_t *__restrict__ order, int32_t *__restrict__ slot_of) {
    __shared__ int32_t sCnt[9][32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t node = (int64_t)blockIdx.x * ORD_BLOCK + tid;
    const int f = node < N ? __popc((uint32_t)__ldg(free_mask + node) & 0xFFu) : -1;
    int rank = 0;
#pragma unroll
    for (int c = 0; c < 9; c++) {
        const uint32_t b = __ballot_sync(0xFFFFFFFFu, f == c);
        if (lane == 0) sCnt[c][warp] = __popc(b);
        if (f == c) rank = __popc(b & ((1u << lane) - 1u));
    }
    __syncthreads();
    if (f < 0) return;
    int before = 0;
    for (int w = 0; w < warp; w++) before += sCnt[f][w];
    const int32_t slot = off[f * nb + blockIdx.x] + before + rank;
    order[slot] = (int32_t)node;
    slot_of[node] = slot;
}

// p[0..n) = v.  kgpu_upload_nodes: every GPU's memory is INT32_MAX MiB until kgpu_upload_gpu_memory, so that no positive
// min_mem excludes it (a byte-wise memset reaches only 0x7F7F7F7F, which a requirement above it would fail).
__global__ void fill_i32(int32_t *__restrict__ p, int64_t n, int32_t v) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}

__global__ void scatter_masks(const int32_t *__restrict__ idx, const int32_t *__restrict__ mask, int64_t n, int32_t *free_mask) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) free_mask[idx[i]] = mask[i];
}

// fit[k * n + i] = (cost<<8 | S) of node list[i] (or node i) for k GPUs, INF32 = does not fit.
__global__ void __launch_bounds__(128)
fit_nodes(const int4 *__restrict__ topo4, const int32_t *__restrict__ free_mask, const int32_t *__restrict__ list /*nullable*/,
          int64_t n, Weights W, PipeConsts pc, uint32_t *__restrict__ fit) {
    __shared__ int32_t sW[16];
    if (threadIdx.x == 0) {
#pragma unroll
        for (int i = 0; i < 16; i++) sW[i] = W.w[i];
    }
    __syncthreads();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t node = list ? (int64_t)__ldg(list + i) : i;
    PairCosts C;
    uint32_t free;
    stage_node(topo4, free_mask, node, true, sW, C, free);
#pragma unroll 1
    for (int k = 0; k <= 8; k++) {
        const uint32_t key = node_key(k, C, pc, free, true);
        fit[(int64_t)k * n + i] = key >= PEN ? INF32 : key;
    }
}

}  // namespace kgpu
