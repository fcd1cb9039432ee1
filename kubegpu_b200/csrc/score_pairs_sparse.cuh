// score_pairs_sparse.cuh -- K1s: the lane-per-node scorer made aware of free-mask sparsity.
//
// Only subsets of a node's FREE GPUs can be placements (the CPU twin skips the others with
// `if (S & ~free) continue`).  K1 (score_pairs.cuh) enumerates all C(8,k) subsets for every pair
// because the 32 lanes of a warp (32 nodes) run in lockstep whatever their free masks are.  K1s
// removes that waste without leaving the lane-per-node mapping:
//   * the handle keeps an ORDER of the nodes grouped by f = popcount(free_mask) (a stable counting sort
//     on the device, node_state.cuh: each class in increasing node id, padded to whole warps), so
//     all lanes of a warp have the same f;
//   * compact_nodes (below) permutes every node's GPUs so that the free ones sit at positions 0..f-1
//     (increasing GPU index, so subset order is preserved) and stores its 28 pair costs in that order
//     as a RECORD in slot order, tile-transposed: a block stages its 128 slots with seven fully
//     coalesced 16-byte loads (120 B per node streamed: what bounds the kernel when pods are few);
//   * F = max f over the warp (REDUX.MAX on the CURRENT records, so a stale order only costs speed,
//     never correctness) selects generated code that enumerates the C(F,k) subsets of positions
//     0..F-1 only (subset_dp_sparse_gen.cuh); F < k: the warp has nothing to do for those pods;
//   * the (tile, pod) plane is cut into work items of about equal work (sparse_work.h); with few pods
//     an item is a run of tiles and the STREAM instantiation prefetches the next tile's record.
// Per pair the enumeration is still done in full for the candidate subsets, with the same
// per-pod multiplier device as K1 (see score_pairs.cuh); results are bit-identical.
#pragma once
#include "score_pairs.cuh"
#include "subset_dp_sparse_gen.cuh"

namespace kgpu {

#ifndef KGPU_SP_THREADS
#define KGPU_SP_THREADS 128          // threads per block; 256 halves the per-pod block flushes (set KGPU_SP_MINBLOCKS 4 with it)
#endif
constexpr int SP_THREADS = KGPU_SP_THREADS;
constexpr int SP_WARPS = SP_THREADS / 32;
constexpr int SP_CHUNK = 512;       // pods per shared-memory chunk; sIdx packs (position | k << 9) in 16 bits
static_assert(SP_CHUNK == 512, "sparse_work.h: kSparseChunk must equal SP_CHUNK");
constexpr int SP_ROW = 29;          // padded row of 28 pair costs per lane in shared memory
#ifndef KGPU_SP_MINBLOCKS
#define KGPU_SP_MINBLOCKS 8          // 64 registers, 32 warps/SM.  H100 SXM (400 W limit): 7 blocks (72 registers) take 0.512
                                     // against 0.514 ms on C2 but 49.3 against 48.5 ms on C3; 6 blocks lose on both
#endif
#ifndef KGPU_SP_UNROLL
#define KGPU_SP_UNROLL 1          // pods per trip of a (K,F) bucket loop
#endif
#ifndef KGPU_SP_UNROLL_SMALL
#define KGPU_SP_UNROLL_SMALL KGPU_SP_UNROLL   // the same for the loops that enumerate <= KGPU_SP_SMALL subsets
#endif
#ifndef KGPU_SP_SMALL
#define KGPU_SP_SMALL 6
#endif
#define KGPU_PRAGMA(x) _Pragma(#x)
#define KGPU_UNROLL(n) KGPU_PRAGMA(unroll n)

__host__ __device__ constexpr int sp_choose(int n, int k) { return k == 0 ? 1 : sp_choose(n - 1, k - 1) * n / k; }
__host__ __device__ constexpr int sp_unroll(int K, int F) {
    return (K <= 1 || sp_choose(F, K) <= KGPU_SP_SMALL) ? KGPU_SP_UNROLL_SMALL : KGPU_SP_UNROLL;
}
__host__ __device__ constexpr int sp_pidx(int i, int j) { return 7 * i - i * (i - 1) / 2 + (j - i - 1); }  // i<j

template <int K, int F>
__device__ __forceinline__ uint32_t node_key_kf(const PairCosts &C, const PipeConsts pc, uint32_t nfree, bool valid) {
    if (K == 0) return valid ? 0u : INF32;
    if (K == 1) return nfree ? pc.one : INF32;          // free GPUs are compacted: the lowest one is position 0
    return best_kf<(K < 2 ? 2 : K), (F < 2 ? 2 : F)>(C, pc);
}

// Pod table of a chunk, in BUCKET order (pods grouped by k): the per-pod multiplier the enumeration runs
// on (see score_pairs.cuh: it makes every instruction of the enumeration depend on per-pod data), one
// array read by every warp, and one row per warp for the warp's result per pod.  Each bucket starts at a
// multiple of 4 positions and is padded to one with dummy pods (multiplier 1, result never read: sIdx
// marks them).  A bucket loop handles sp_width(K, F) pods per trip: one LDS of their multipliers, the
// enumerations, one STS of the results, loop control once.
constexpr int SP_PAD = 4;            // bucket alignment in positions: the widest trip
constexpr uint16_t SP_DUMMY = 0xFFFFu;
constexpr int SP_MEM_SUB = 4;        // MEM launch: pods of one k are sub-bucketed by a hash of min_mem, so equal requirements sit together
// positions of a chunk of CH pods (nine padded buckets, then the pods not for this launch), rounded to whole
// trips, plus one trip: the prefetch build reads one past a bucket's end
__host__ __device__ constexpr int sp_tab_len(int CH) { return (CH + 9 * (SP_PAD - 1) + SP_PAD - 1) / SP_PAD * SP_PAD + SP_PAD; }
// What the pod sort makes of a chunk.  It depends on the chunk's pods only, never on the tile, so for a launch over
// many pods sp_prepare_chunks builds it once per chunk into global memory in exactly this layout, and a block copies
// it in with 16-byte loads instead of sorting.
template <int N>
struct alignas(16) SpChunkTab {
    uint32_t one[N];                 // MEM: the pods' min_mem instead (the MEM loops derive `one` from K)
    uint16_t idx[N];                 // bucket-order position -> chunk position (SP_DUMMY: padding)
    int32_t off[12];                 // off[k]: where bucket k starts; off[9]: end of the served pods; off[11]: bit k = bucket k has pods
};
template <int N>
struct alignas(16) SpTab {
    SpChunkTab<N> c;
    uint32_t best[SP_WARPS][N];      // warp key of the best (node, subset) of this warp for the pod, INF32 = none
};
static_assert(sp_tab_len(SP_CHUNK) % 4 == 0, "rows of the pod table must stay 16-byte aligned");
constexpr int SP_POS = sp_tab_len(SP_CHUNK);
constexpr int SP_CHUNK_INT4 = (int)(sizeof(SpChunkTab<SP_POS>) / 16);      // 16-byte words of a prepared chunk table: 207
static_assert(sizeof(SpChunkTab<SP_POS>) % 16 == 0, "prepared chunk tables are copied in 16-byte words");

// The chunk's pod sort: pods4[0..cn), cn <= CH, into `tab` in bucket order -- the pods that want k GPUs for k = 0..8
// (MEM: sub-bucketed by a hash of min_mem), each k padded with dummy pods to a multiple of SP_PAD, then the pods not for
// this launch (k outside 0..8, or on the other side of min_mem).  cnt: NB shared counters.  acc != nullptr: the
// positions' running minima of a multi-tile item are reset as well.  All NT threads of the block call it, between two
// barriers of the caller's (the table is only read after the second).
template <bool MEM, int CH, int NT, int N>
__device__ __forceinline__ void sp_sort_chunk(const int4 *__restrict__ pods4, int cn, int32_t *cnt, SpChunkTab<N> &tab,
                                              unsigned long long *acc, int tid) {
    constexpr int SUB = MEM ? SP_MEM_SUB : 1, NB = 9 * SUB + 1;
    constexpr int PPT = (CH + NT - 1) / NT;            // pods per thread
    if (tid < NB) cnt[tid] = 0;
    __syncthreads();
    // each thread keeps its pods' buckets and multipliers in registers from the count to the scatter
    int bkt[PPT];
    uint32_t mult[PPT];
#pragma unroll
    for (int u = 0; u < PPT; u++) {
        const int i = tid + u * NT;
        bkt[u] = 9 * SUB;
        mult[u] = 0;
        if (i < cn) {
            const int4 req = __ldg(pods4 + i);
            const bool wants_mem = req.w > 0;
            if (req.x >= 0 && req.x <= 8 && wants_mem == MEM)
                bkt[u] = req.x * SUB + (MEM ? (int)(((uint32_t)req.w * 0x9E3779B1u) >> 30) : 0);
            // the per-pod multiplier: the pod's own k less what its bucket adds back (= 1 at run time)
            mult[u] = MEM ? (uint32_t)req.w : (uint32_t)(req.x - (bkt[u] < 9 ? bkt[u] - 1 : 0));
            atomicAdd(&cnt[bkt[u]], 1);
        }
    }
    __syncthreads();
    if (tid < 32) {                                    // warp 0, lane k: bucket k.  off[k]: where k's pods start; cnt: running positions
        const int k = tid;
        int c_sub[SUB], c = 0;
#pragma unroll
        for (int u = 0; u < SUB; u++) { c_sub[u] = k < 9 ? cnt[k * SUB + u] : 0; c += c_sub[u]; }
        const int padded = (c + SP_PAD - 1) / SP_PAD * SP_PAD;
        int end = padded;                              // inclusive prefix sum over lanes 0..8
#pragma unroll
        for (int d = 1; d < 16; d <<= 1) {
            const int t = __shfl_up_sync(0xFFFFFFFFu, end, d);
            if (k >= d) end += t;
        }
        const int served = __shfl_sync(0xFFFFFFFFu, end, 8);
        const uint32_t nonempty = __ballot_sync(0xFFFFFFFFu, c > 0);
        if (k < 9) {
            int a = end - padded;
            tab.off[k] = a;
#pragma unroll
            for (int u = 0; u < SUB; u++) { cnt[k * SUB + u] = a; a += c_sub[u]; }
            for (; a < end; a++) {                     // dummy pods up to the next multiple of SP_PAD
                tab.idx[a] = SP_DUMMY;
                tab.one[a] = MEM ? 0u : 1u;
            }
        } else if (k == 9) {
            cnt[9 * SUB] = served;                     // the pods not for this launch follow bucket 8
            tab.off[9] = served;
            tab.off[10] = 0;
            tab.off[11] = (int)nonempty;
        }
    }
    __syncthreads();
#pragma unroll
    for (int u = 0; u < PPT; u++) {
        const int i = tid + u * NT;
        if (i < cn) {
            const int at = atomicAdd(&cnt[bkt[u]], 1);
            tab.idx[at] = (uint16_t)i;
            if (acc) acc[at] = ~0ull;
            tab.one[at] = mult[u];
        }
    }
}

// One block per SP_CHUNK pods of the batch: the chunk's sorted pod table (sp_sort_chunk, as a K1s block would make it)
// into chunks[chunk][SP_CHUNK_INT4].  Launched before a K1s launch over more than one chunk of pods, on its stream;
// the K1s blocks whose pod range covers a whole chunk (or ends at P) copy the table instead of sorting.
template <bool MEM>
__global__ void __launch_bounds__(SP_THREADS)
sp_prepare_chunks(const int4 *__restrict__ pods4, int64_t P, const int *__restrict__ mem_flag, int4 *__restrict__ chunks) {
    if (MEM && *mem_flag == 0) return;                 // (the MEM K1s launch exits at once as well)
    constexpr int NB = 9 * (MEM ? SP_MEM_SUB : 1) + 1;
    __shared__ int32_t sCnt[NB];
    __shared__ SpChunkTab<SP_POS> sChunk;
    const int tid = threadIdx.x;
    const int64_t c0 = (int64_t)blockIdx.x * SP_CHUNK;
    sp_sort_chunk<MEM, SP_CHUNK, SP_THREADS>(pods4 + c0, (int)min((int64_t)SP_CHUNK, P - c0), sCnt, sChunk, nullptr, tid);
    __syncthreads();
    int4 *const dst = chunks + (int64_t)blockIdx.x * SP_CHUNK_INT4;
    for (int q = tid; q < SP_CHUNK_INT4; q += SP_THREADS) dst[q] = reinterpret_cast<const int4 *>(&sChunk)[q];
}

// Pods per trip of the (K, F) bucket loop.  Four share the multiplier load, the result store and the loop
// control; two where four pods' enumerations in flight push values into local memory (cuobjdump -sass).  The
// MEM loops also hold the penalised copy of the pair costs, which (4, 8) does not fit beside four pods.
__host__ __device__ constexpr int sp_width(int K, int F, bool MEM) {
    return (K == 3 && F >= 7) || ((K == 5 || K == 6) && F == 8) || (MEM && K == 4 && F == 8) ? 2 : 4;
}

// Warp key.  BYTE_KEYS (every cost < 2^16, i.e. every weight <= 2340): cost<<16 | lane<<8 | S, built
// from the lane key (cost<<8 | S) with ONE PRMT whose selector also encodes "this lane cannot serve
// k = K" (nfree < K, loop invariant): it then picks four 0xFF bytes = INF32.  Otherwise:
// cost<<13 | lane<<8 | S with an IMAD for the shift and two LOP3.
struct SpFmt {
    uint32_t lane_hi;   // BYTE_KEYS: lane<<8 | 0xFFFF0000          else: feasible ? lane<<8 : 0xFFFFFFFF
    uint32_t sel;       // BYTE_KEYS: feasible ? 0x2150 : 0x7777     else: unused
};
template <bool BYTE_KEYS>
__device__ __forceinline__ SpFmt sp_fmt(uint32_t lane_field, bool feasible) {
    SpFmt f;
    if (BYTE_KEYS) { f.lane_hi = lane_field | 0xFFFF0000u; f.sel = feasible ? 0x2150u : 0x7777u; }
    else           { f.lane_hi = feasible ? lane_field : 0xFFFFFFFFu; f.sel = 0u; }
    return f;
}
template <bool BYTE_KEYS>
__device__ __forceinline__ uint32_t sp_warp_key(uint32_t key, const SpFmt f, uint32_t thirty_two) {
    if (BYTE_KEYS) return __byte_perm(key, f.lane_hi, f.sel);
    return ((key * thirty_two) & 0xFFFFE000u) | ((key & 0xFFu) | f.lane_hi);
}

#ifndef KGPU_SP_PREFETCH
#define KGPU_SP_PREFETCH 0       // 1: load the next trip's multipliers one trip ahead (reads one trip past a bucket's end)
#endif
template <int W>
__device__ __forceinline__ void sp_load_ones(const uint32_t *p, uint32_t (&ones)[W]) {
    static_assert(W == 2 || W == 4, "a trip is 2 or 4 pods");
    if (W == 4) {
        const uint4 o = *reinterpret_cast<const uint4 *>(p);                 // one LDS.128
        ones[0] = o.x; ones[1] = o.y; ones[2 % W] = o.z; ones[3 % W] = o.w;
    } else {
        const uint2 o = *reinterpret_cast<const uint2 *>(p);                 // one LDS.64
        ones[0] = o.x; ones[1] = o.y;
    }
}

// One (K, F) loop: all pods of the chunk that want K GPUs, enumerating positions 0..F-1.  one: the chunk's
// multipliers, best: this warp's result row, both indexed by bucket-order position.
template <int K, int F, bool PER_PAIR, bool MEM, bool BYTE_KEYS>
__device__ __forceinline__ void sp_bucket(const PairCosts &C, const PipeConsts pc, uint32_t nfree, bool valid,
                                          const int32_t (&mem)[8], uint32_t lane_field, const uint32_t *one,
                                          uint32_t *best, int begin, int end) {
    constexpr int W = sp_width(K, F, MEM);
    // (begin >> 30) is 0; tying the test to this chunk's bucket offset keeps the compiler from hoisting the
    // nine per-K selectors to the top of the kernel, where they cost nine registers for the whole run.
    const uint32_t need_free = (uint32_t)K + ((uint32_t)begin >> 30);
    const SpFmt fmt = sp_fmt<BYTE_KEYS>(lane_field, MEM ? true : (valid && nfree >= need_free));
    const uint32_t thirty_two = pc.one << 5;       // a register, so that the shift is an IMAD (kernel parameter: opaque)
    int32_t last_need = -1;                        // MEM: the requirement C2 / elig were last built for
    uint32_t elig = 0;
    PairCosts C2 = C;
#if KGPU_SP_PREFETCH
    uint32_t nxt[W];
    sp_load_ones<W>(one + begin, nxt);
#endif
    KGPU_UNROLL((sp_unroll(K, F)))
    // byte offsets (4 bytes per position, begin and end are multiples of SP_PAD): uniform, because begin and end
    // come from shared memory, so the loop runs on the uniform datapath and both addresses are base + offset
    for (uint32_t off = (uint32_t)begin * 4u; off != (uint32_t)end * 4u; off += 4u * W) {
        const uint32_t *const op = reinterpret_cast<const uint32_t *>(reinterpret_cast<const char *>(one) + off);
        uint32_t ones[W], v[W];
#if KGPU_SP_PREFETCH
#pragma unroll
        for (int g = 0; g < W; g++) ones[g] = nxt[g];
        sp_load_ones<W>(op + W, nxt);              // next trip's multipliers: their LDS latency overlaps this trip
#else
        sp_load_ones<W>(op, ones);
#endif
#pragma unroll
        for (int g = 0; g < W; g++) {
            PipeConsts pcl = pc;
            if (MEM) {
                const int32_t need = (int32_t)ones[g];
                if (need != last_need) {               // warp-uniform; rare: the sort puts equal requirements together
                    last_need = need;
                    uint32_t pen[8];
                    elig = 0;
#pragma unroll
                    for (int q = 0; q < 8; q++) {
                        const bool lt = mem[q] < need;
                        pen[q] = lt ? PEN : 0u;
                        if (!lt && (uint32_t)q < nfree) elig |= 1u << q;      // position q: free and big enough
                    }
                    if (K >= 2) apply_pens(C, C2, pen);
                }
                uint32_t key;
                if (K == 0) key = valid ? 0u : INF32;
                else if (K == 1) key = elig ? (elig & (0u - elig)) : INF32;
                else key = best_kf<(K < 2 ? 2 : K), (F < 2 ? 2 : F)>(C2, pcl);
                v[g] = key >= PEN ? INF32 : sp_warp_key<BYTE_KEYS>(key, fmt, thirty_two);
            } else {
                if (PER_PAIR) {                        // un-hoistable per-pair work: see score_pairs.cuh
                    pcl.one = ones[g];
                    if (K >= 5) pcl.minus_one = 0u - pcl.one;
                }
                // lanes that cannot serve K (fmt says so) compute a key like the others and drop it
                const uint32_t key = K == 0 ? 0u : K == 1 ? pcl.one : best_kf<(K < 2 ? 2 : K), (F < 2 ? 2 : F)>(C, pcl);
                v[g] = sp_warp_key<BYTE_KEYS>(key, fmt, thirty_two);
            }
        }
        uint32_t m[W];
#pragma unroll
        for (int g = 0; g < W; g++) m[g] = __reduce_min_sync(0xFFFFFFFFu, v[g]);
        if (lane_field == 0) {
            void *const bp = reinterpret_cast<char *>(best) + off;
            if (W == 4) *reinterpret_cast<uint4 *>(bp) = make_uint4(m[0], m[1], m[2 % W], m[3 % W]);   // one STS.128
            else *reinterpret_cast<uint2 *>(bp) = make_uint2(m[0], m[1]);                              // one STS.64
        }
    }
}

template <int K, bool PER_PAIR, bool MEM, bool BYTE_KEYS>
__device__ __forceinline__ void sp_run_k(int F, const PairCosts &C, const PipeConsts pc, uint32_t nfree, bool valid,
                                         const int32_t (&mem)[8], uint32_t lane_field, const uint32_t *one,
                                         uint32_t *best, int begin, int end) {
    if (begin >= end) return;
    if (F < K) {                                   // no lane of this warp has K free GPUs: no result for these pods
        for (int q = begin / 4 + (int)(lane_field >> 8); q < end / 4; q += 32)
            reinterpret_cast<uint4 *>(best)[q] = make_uint4(INF32, INF32, INF32, INF32);
        return;
    }
#define KGPU_SP_CASE(FF)                                                                                         \
    case FF:                                                                                                     \
        if (FF >= K) sp_bucket<K, (FF >= K ? FF : K), PER_PAIR, MEM, BYTE_KEYS>(C, pc, nfree, valid, mem, lane_field, one, best, begin, end); \
        break;
    if (K <= 1) {                                  // F does not matter for k = 0, 1
        sp_bucket<K, 8, PER_PAIR, MEM, BYTE_KEYS>(C, pc, nfree, valid, mem, lane_field, one, best, begin, end);
        return;
    }
    switch (F) {
        KGPU_SP_CASE(2) KGPU_SP_CASE(3) KGPU_SP_CASE(4) KGPU_SP_CASE(5) KGPU_SP_CASE(6) KGPU_SP_CASE(7) KGPU_SP_CASE(8)
        default: break;
    }
#undef KGPU_SP_CASE
}

// Compacted pair-cost cache, in SLOT order and tile-transposed, so that a K1s block stages its 128 nodes with
// fully coalesced loads (what matters when few pods amortise the staging: the HBM-bound regime):
//   rec  [tile][7][SP_THREADS] int4   word 4t+q of slot s = compacted scaled pair cost number 4t+q of the slot's
//                                     node (free GPUs first, ascending; pairs touching a non-free position carry PEN)
//   meta [slot] uint32                position -> GPU index as eight 3-bit fields | free count << 24 | tile ordered << 31
// Padding slots (order[slot] < 0) hold PEN costs, the identity permutation and free count 0.
// Built for every slot after an upload, a re-sort or a weight change (list == nullptr: item = slot), and for the
// listed NODES only after a state change (kgpu_set_free_masks / kgpu_update_node: item -> node list[item] ->
// slot_of[node]; `new_mask`, if given, is scattered into free_mask by the same threads).  A node keeps its slot
// when its free count changes: the order is then stale, which costs speed (the warp's F is the max over its
// lanes), never correctness; the host re-sorts when enough nodes have changed.
__host__ __device__ constexpr int64_t sp_rec_index(int64_t slot, int t) {
    return ((slot / SP_THREADS) * 7 + t) * SP_THREADS + slot % SP_THREADS;
}
__global__ void __launch_bounds__(SP_THREADS)
compact_nodes(const int4 *__restrict__ topo4, int32_t *free_mask, int64_t n_items, Weights W,
              const int32_t *__restrict__ order /*[n_slots]*/, const int32_t *__restrict__ slot_of /*[N]*/,
              int4 *__restrict__ rec, uint32_t *__restrict__ meta,
              const int32_t *__restrict__ list = nullptr /*[n_items] node indices, or every slot*/,
              const int32_t *__restrict__ new_mask = nullptr /*[n_items] with list: masks to store first*/) {
    __shared__ int32_t sW[16];
    __shared__ uint32_t sRow[SP_THREADS * SP_ROW];
    const int tid = threadIdx.x;
    if (tid == 0) {
#pragma unroll
        for (int i = 0; i < 16; i++) sW[i] = W.w[i];
    }
    __syncthreads();
    const int64_t item = (int64_t)blockIdx.x * SP_THREADS + tid;
    // Bit 31 of meta: "the tile's slots are in increasing node id, padding only at its end" -- then (cost, warp, lane)
    // order IS (cost, node) order and K1s's flush can min the four warp keys directly.  A property of the ORDER, so it
    // is decided here once per full build (a block is a tile then) and preserved by the per-node refreshes.
    uint32_t ordered_bit = 0;
    if (!list) {                                      // n_items = n_slots: whole tiles, every thread takes part
        const int32_t nd = __ldg(order + item);
        const int32_t prev = tid > 0 ? __ldg(order + item - 1) : -1;
        ordered_bit = __syncthreads_and(tid == 0 || nd < 0 || (prev >= 0 && prev < nd)) ? 0x80000000u : 0u;
    }
    if (item >= n_items) return;
    int64_t node, slot;
    if (list) { node = __ldg(list + item); slot = __ldg(slot_of + node); }
    else      { slot = item; node = __ldg(order + slot); }
    if (node < 0) {                                   // padding slot
#pragma unroll
        for (int t = 0; t < 7; t++) rec[sp_rec_index(slot, t)] = make_int4((int)PEN, (int)PEN, (int)PEN, (int)PEN);
        meta[slot] = 0xFAC688u | ordered_bit;         // identity permutation (7<<21 | 6<<18 | ... | 0), free count 0
        return;
    }
    if (new_mask) free_mask[node] = __ldg(new_mask + item);
    const uint32_t free = (uint32_t)(new_mask ? __ldg(new_mask + item) : free_mask[node]) & 0xFFu;
    uint32_t *row = sRow + tid * SP_ROW;
    {
        const int4 *src = topo4 + node * 16;
        int4 q[16];
#pragma unroll
        for (int t = 0; t < 16; t++) q[t] = make_int4(0, 0, 0, 0);
        q[0] = __ldg(src + 0);  q[1] = __ldg(src + 1);
        q[2] = __ldg(src + 2);  q[3] = __ldg(src + 3);
        q[4] = __ldg(src + 4);  q[5] = __ldg(src + 5);
        q[7] = __ldg(src + 7);  q[9] = __ldg(src + 9);
        q[11] = __ldg(src + 11); q[13] = __ldg(src + 13);
#pragma unroll
        for (int i = 0; i < 8; i++)
#pragma unroll
            for (int j = i + 1; j < 8; j++) {
                const int4 v = q[i * 2 + (j >> 2)];
                const int lvl = (j & 3) == 0 ? v.x : (j & 3) == 1 ? v.y : (j & 3) == 2 ? v.z : v.w;
                row[sp_pidx(i, j)] = (uint32_t)sW[lvl & 15] << 8;
            }
    }
    const uint32_t nfree = (uint32_t)__popc(free);
    uint32_t perm = 0;                                // nibbles here, 3-bit fields in meta
    {
        int pos = 0;
#pragma unroll
        for (int g = 0; g < 8; g++)
            if ((free >> g) & 1u) { perm |= (uint32_t)g << (4 * pos); pos++; }
#pragma unroll
        for (int g = 0; g < 8; g++)
            if (!((free >> g) & 1u)) { perm |= (uint32_t)g << (4 * pos); pos++; }
    }
    {
        uint32_t p3 = 0;
#pragma unroll
        for (int g = 0; g < 8; g++) p3 |= ((perm >> (4 * g)) & 7u) << (3 * g);
        if (list) ordered_bit = meta[slot] & 0x80000000u;
        meta[slot] = p3 | (nfree << 24) | ordered_bit;
    }
    uint32_t wds[28];
#pragma unroll
    for (int i = 0; i < 8; i++)
#pragma unroll
        for (int j = i + 1; j < 8; j++) {          // i < j are POSITIONS
            const int a = (int)((perm >> (4 * i)) & 7u), b = (int)((perm >> (4 * j)) & 7u);
            const int lo = min(a, b), hi = max(a, b);
            uint32_t cst = row[7 * lo - ((lo * (lo - 1)) >> 1) + (hi - lo - 1)];
            if ((uint32_t)j >= nfree) cst += PEN;
            wds[sp_pidx(i, j)] = cst;
        }
#pragma unroll
    for (int t = 0; t < 7; t++)
        rec[sp_rec_index(slot, t)] = make_int4((int)wds[4 * t], (int)wds[4 * t + 1], (int)wds[4 * t + 2], (int)wds[4 * t + 3]);
}

// ---- TMA (cp.async.bulk) + mbarrier helpers of the TMA instantiation ------------------------------------------
// One-dimensional bulk copies need no tensor map: [dst in shared], [src in global], bytes (multiples of 16, 16-byte
// aligned), completion counted in bytes on an mbarrier.  The CPU emulation build copies synchronously.
constexpr int SP_SLAB_REC = 7 * SP_THREADS * 16;                    // a tile's records
constexpr int SP_SLAB = SP_SLAB_REC + SP_THREADS * 4 + SP_THREADS * 4;   // + meta + order: 15360 bytes at 128 threads
#ifndef KGPU_SP_TMA_STAGES
#define KGPU_SP_TMA_STAGES 1      // slabs per block: more slabs cost blocks per SM (see KGPU_SP_TMA_MINBLOCKS)
#endif
constexpr int SP_TMA_STAGES = KGPU_SP_TMA_STAGES;
constexpr size_t SP_TMA_DYN_SMEM = (size_t)SP_TMA_STAGES * SP_SLAB + 128;     // + alignment slack
#ifdef __CUDACC__
__device__ __forceinline__ uint32_t sp_smem_addr(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void sp_mbar_init(unsigned long long *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(sp_smem_addr(bar)), "r"(count));
}
__device__ __forceinline__ void sp_mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void sp_mbar_expect_tx(unsigned long long *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(sp_smem_addr(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void sp_bulk_g2s(void *dst, const void *src, uint32_t bytes, unsigned long long *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(sp_smem_addr(dst)), "l"(src), "r"(bytes), "r"(sp_smem_addr(bar)) : "memory");
}
__device__ __forceinline__ bool sp_mbar_wait(unsigned long long *bar, uint32_t parity) {     // false: gave up after ~2 s
    const long long t0 = clock64();
    uint32_t done = 0;
    while (!done) {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(done) : "r"(sp_smem_addr(bar)), "r"(parity) : "memory");
        if (!done && clock64() - t0 > 4000000000LL) return false;
    }
    return true;
}
#else
inline void sp_mbar_init(unsigned long long *, uint32_t) {}
inline void sp_mbar_fence_init() {}
inline void sp_mbar_expect_tx(unsigned long long *, uint32_t) {}
inline void sp_bulk_g2s(void *dst, const void *src, uint32_t bytes, unsigned long long *) { std::memcpy(dst, src, bytes); }
inline bool sp_mbar_wait(unsigned long long *, uint32_t) { return true; }
#endif

// grid = (work items) or (slot tiles, pod splits); block = SP_THREADS.  order[slot] = node index or -1 (padding).
// STREAM (few pods, runs of tiles: the HBM-bound regime): the NEXT tile's record is loaded into a second register
// set before the current tile's bucket loops, so every block always has a tile in flight from DRAM while it
// computes (96 registers, 5 blocks per SM: 75 KB in flight per SM against the ~25 KB that 3.35 TB/s x ~1 us of
// DRAM latency need on an H100's 132 SMs).  Without it a block slot alternates between waiting for its tile and
// computing on it.
#ifndef KGPU_SP_STREAM_MINBLOCKS
#define KGPU_SP_STREAM_MINBLOCKS 5
#endif
// TMA (at most 64 pods, runs of tiles): the streaming path with the tiles staged by the TMA engine instead -- a
// slab (records + meta + order of a tile, 15 KB) per stage in shared memory, filled by cp.async.bulk and signalled on an
// mbarrier; the threads copy their part out to registers and the slab is refilled at once, so the next tile is in
// flight while this one is scored.  The pod tables shrink to 64 pods and there are no prefetch registers, so 7 or 8
// blocks fit an SM: TMA = blocks per SM of the instantiation (0: not a TMA one).  Measured on an H100 SXM (400 W
// limit), 10.5M nodes: 7 blocks (72 registers, no spill) take 0.426 / 0.504 ms at 32 / 64 pods against 0.444 / 0.515
// with 8 (64 registers, spills) and 0.428 / 0.512 with 6; at 1 and 4 pods all three take 0.421 - 0.423 ms.
#ifndef KGPU_SP_TMA_MINBLOCKS
#define KGPU_SP_TMA_MINBLOCKS 7
#endif
constexpr int SP_TMA_PODS = 64;
template <bool PER_PAIR, bool MEM, bool BYTE_KEYS, bool STREAM = false, int TMA = 0>
__global__ void __launch_bounds__(SP_THREADS, TMA ? TMA : STREAM ? KGPU_SP_STREAM_MINBLOCKS : MEM ? 4 : KGPU_SP_MINBLOCKS)
score_pairs_sparse(const int4 *__restrict__ rec, const uint32_t *__restrict__ meta,
                   const int32_t *__restrict__ gpu_mem, const int32_t *__restrict__ order,
                   const int *__restrict__ mem_flag, int64_t node_id_base, const int4 *__restrict__ pods4, int64_t P,
                   int pods_per_split, const int4 *__restrict__ work, PipeConsts pc, unsigned long long *__restrict__ keys,
                   const int4 *__restrict__ chunks = nullptr /*sp_prepare_chunks' tables of this batch, or none*/) {
    if (MEM && *mem_flag == 0) return;
    static_assert(!TMA || (STREAM && !MEM), "the TMA instantiation is a streaming one");
    constexpr int SUB = MEM ? SP_MEM_SUB : 1, NB = 9 * SUB + 1;     // sort buckets: (k, sub) for k = 0..8, then "not for this launch"
    constexpr int CH = TMA ? SP_TMA_PODS : SP_CHUNK;                // pods per chunk of the block's pod sort
    constexpr int POS = sp_tab_len(CH);                // bucket-order positions
    __shared__ int32_t sCnt[NB];
    __shared__ SpTab<POS> sTab;                        // bucket order: multipliers, positions, offsets | per-warp results
    __shared__ int32_t sF[SP_WARPS];                   // !STREAM: every warp's F, so that a block skips the k no slot can serve
    uint16_t (&sIdx)[POS] = sTab.c.idx;
    int32_t (&sOff)[12] = sTab.c.off;                  // sOff[11]: bit k set = bucket k has pods (STREAM builds test it per tile)
    // position g -> byte (1 << GPU index), g = 0..3 | 4..7.  STREAM builds (few pods per tile) keep the slot's
    // permutation word in sHotLo instead and expand the winner's S' in the flush: per pod, not per node.
    __shared__ uint32_t sHotLo[SP_THREADS], sHotHi[STREAM ? 1 : SP_THREADS];
    __shared__ int32_t sNode[SP_THREADS];              // slot -> node index (-1 = padding)
    // multi-tile items: running minimum per pod position across the tiles as cost << 32 | node index (a node has ONE best
    // subset, so this orders like the final key) and where it came from: tile of the run << 16 | slot << 8 | S'.  The final
    // key -- S' expanded through the slot's permutation word, the node id -- is built once per item, not per tile.
    constexpr bool CAN_MULTI = STREAM || MEM;          // the hosts hand runs of tiles to these instantiations only
    __shared__ unsigned long long sAcc[CAN_MULTI ? POS : 1];
    __shared__ uint32_t sWin[CAN_MULTI ? POS : 1];
    __shared__ unsigned long long sBar[SP_TMA_STAGES]; // TMA: "slab of this stage has landed"
#ifdef __CUDACC__
    extern __shared__ __align__(128) unsigned char sDynRing[];      // TMA: SP_TMA_STAGES slabs
    unsigned char *const ring = sDynRing;
#else
    __shared__ __attribute__((aligned(128))) unsigned char sRingEmu[SP_TMA_STAGES * SP_SLAB];
    unsigned char *const ring = sRingEmu;
#endif

    const int tid = threadIdx.x;
    uint32_t *const best_row = sTab.best[tid >> 5];
    const uint32_t lane_field = (uint32_t)(tid & 31) << 8;

    // ---- staging: the node's compacted pair costs (7 x 16 B), permutation and free count ----------
    // which tile, which pods: a work item {tile, pod_begin, pod_end} of the host's list (sparse_work.h), or the
    // plain grid (tile = blockIdx.x, equal pod ranges along blockIdx.y) when there is no list
    int64_t tile_first = blockIdx.x, p_begin = (int64_t)blockIdx.y * pods_per_split, p_end = min(P, p_begin + pods_per_split);
    int ntiles = 1;
    if (work != nullptr) {
        const int4 item = __ldg(work + blockIdx.x);
        tile_first = item.x; p_begin = item.y; p_end = item.z; ntiles = item.w;
    }
    // ntiles > 1 (few pods: p_end - p_begin <= SP_CHUNK, the host guarantees it): the block walks a run of tiles;
    // the pods are sorted once (first tile), the per-pod minimum is carried in sAcc and flushed once at the end.
    const bool multi = CAN_MULTI && ntiles > 1;        // (otherwise every tile of a run is flushed on its own: slower, still exact)
    // a slot's record: seven coalesced 16-byte loads + node index + permutation / free count
    auto load_tile = [&](int64_t t, int4 (&r)[7], int32_t &nd, uint32_t &m) {
        const int4 *src = rec + t * (7 * SP_THREADS) + tid;
#pragma unroll
        for (int q = 0; q < 7; q++) r[q] = __ldg(src + q * SP_THREADS);
        nd = __ldg(order + t * SP_THREADS + tid);
        m = __ldg(meta + t * SP_THREADS + tid);
    };
    int4 nx[7];
    int32_t nx_node = -1;
    uint32_t nx_pm = 0;
    // TMA: thread 0 asks the TMA engine for a tile's slab (three bulk copies counted on the stage's mbarrier)
    auto tma_fetch = [&](int64_t t, int stage) {
        unsigned char *slab = ring + (size_t)stage * SP_SLAB;
        sp_mbar_expect_tx(&sBar[stage], (uint32_t)SP_SLAB);
        sp_bulk_g2s(slab, rec + t * (7 * SP_THREADS), (uint32_t)SP_SLAB_REC, &sBar[stage]);
        sp_bulk_g2s(slab + SP_SLAB_REC, meta + t * SP_THREADS, (uint32_t)(SP_THREADS * 4), &sBar[stage]);
        sp_bulk_g2s(slab + SP_SLAB_REC + SP_THREADS * 4, order + t * SP_THREADS, (uint32_t)(SP_THREADS * 4), &sBar[stage]);
    };
    if (TMA) {
        if (tid == 0) {
#pragma unroll
            for (int st = 0; st < SP_TMA_STAGES; st++) sp_mbar_init(&sBar[st], 1);
            sp_mbar_fence_init();
        }
        __syncthreads();
        if (tid == 0) {
#pragma unroll
            for (int st = 0; st < SP_TMA_STAGES; st++)
                if (st < ntiles) tma_fetch(tile_first + st, st);
        }
#ifndef __CUDACC__
        __syncthreads();                               // (emulation: the "TMA" is a memcpy by thread 0)
#endif
    } else if (STREAM) {
        load_tile(tile_first, nx, nx_node, nx_pm);
    }
#pragma unroll 1
    for (int tt = 0; tt < ntiles; tt++) {
    const int64_t tile_index = tile_first + tt;
    if (!TMA && tt > 0) __syncthreads();               // the previous tile's flush has read sNode / sHot* (TMA: the barrier below)
    int4 rw[7];
    int32_t node;
    uint32_t pm;                                       // eight 3-bit GPU indices | free count << 24 | tile ordered << 31
    if (TMA) {
        const int stage = tt % SP_TMA_STAGES;
        const bool landed = sp_mbar_wait(&sBar[stage], (uint32_t)((tt / SP_TMA_STAGES) & 1));
        const unsigned char *slab = ring + (size_t)stage * SP_SLAB;
        const int4 *srec = reinterpret_cast<const int4 *>(slab);
#pragma unroll
        for (int q = 0; q < 7; q++) rw[q] = srec[q * SP_THREADS + tid];
        pm = reinterpret_cast<const uint32_t *>(slab + SP_SLAB_REC)[tid];
        node = landed ? reinterpret_cast<const int32_t *>(slab + SP_SLAB_REC + SP_THREADS * 4)[tid] : -1;   // a slab that never came scores nothing
        // ONE barrier per tile before the loops: every thread has copied its part of the slab out (it can be refilled)
        // and has finished the previous tile's flush (sNode / sHotLo / the pod table can be rewritten)
        __syncthreads();
        if (tid == 0 && tt + SP_TMA_STAGES < ntiles) tma_fetch(tile_index + SP_TMA_STAGES, tt % SP_TMA_STAGES);
    } else if (STREAM) {
#pragma unroll
        for (int q = 0; q < 7; q++) rw[q] = nx[q];
        node = nx_node;
        pm = nx_pm;
        if (tt + 1 < ntiles) load_tile(tile_index + 1, nx, nx_node, nx_pm);     // in flight during this tile's loops
    } else {
        load_tile(tile_index, rw, node, pm);           // issued before anything waits on them
    }
    const bool valid = node >= 0;
    sNode[tid] = node;
    const uint32_t nfree = (pm >> 24) & 0xFu;            // 0 for padding slots
    if (STREAM) {
        if (!multi) sHotLo[tid] = pm;
    } else {
        uint32_t lo = 0, hi = 0;
#pragma unroll
        for (int g = 0; g < 4; g++) {
            lo |= (1u << ((pm >> (3 * g)) & 7u)) << (8 * g);
            hi |= (1u << ((pm >> (3 * g + 12)) & 7u)) << (8 * g);
        }
        sHotLo[tid] = lo;
        sHotHi[tid] = hi;
    }
    // Are the tile's slots in increasing node id (one class, padding only at the end)?  Then (cost, warp, lane)
    // order IS (cost, node) order and the flush can min the four warp keys directly.  Decided when the records were
    // built (bit 31 of every meta word of the tile): no barrier, no neighbour load here.
    bool ordered = BYTE_KEYS && (pm >> 31) != 0;
    if (STREAM && !TMA) {
        // The register-prefetch instantiation keeps the two block barriers the in-kernel check used to have: they hold
        // the block's four warps in step, so the next tile's 14 KB are requested together, which streamed faster than
        // letting the warps drift apart (not re-measured on the H100).  (The TMA instantiation has
        // one thread request the slab: it runs on two barriers per tile, the one above and the one before the flush.)
        __syncthreads();
        ordered = __syncthreads_and(ordered) != 0;
    }
    PairCosts C;
    for_each_pair(C, [&](int i, int j) -> uint32_t {
        const int w = sp_pidx(i, j);
        const int4 v = rw[w >> 2];
        return (uint32_t)((w & 3) == 0 ? v.x : (w & 3) == 1 ? v.y : (w & 3) == 2 ? v.z : v.w);
    });
    int32_t mem[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (MEM && valid) {
#pragma unroll
        for (int g = 0; g < 8; g++) mem[g] = __ldg(gpu_mem + (int64_t)node * 8 + ((pm >> (3 * g)) & 7u));
    }
    const int F = (int)__reduce_max_sync(0xFFFFFFFFu, nfree);    // warp-uniform bound on usable positions
    if (!STREAM && lane_field == 0) sF[tid >> 5] = F;             // read after the first chunk's prologue barrier

    for (int64_t c0 = p_begin; c0 < p_end; c0 += CH) {
        const int cn = (int)min((int64_t)CH, p_end - c0);
        if (!multi || tt == 0) {                   // the chunk's pod table (once per item when it walks several tiles)
        __syncthreads();
        // a whole chunk of the batch (or its last, up to P): its table was prepared for the launch -- one coalesced copy
        if (!STREAM && !multi && chunks != nullptr && c0 % CH == 0 && (c0 + CH <= p_end || p_end == P)) {
            const int4 *const src = chunks + (c0 / CH) * SP_CHUNK_INT4;
            for (int q = tid; q < SP_CHUNK_INT4; q += SP_THREADS) reinterpret_cast<int4 *>(&sTab.c)[q] = __ldg(src + q);
        } else {
            sp_sort_chunk<MEM, CH, SP_THREADS>(pods4 + c0, cn, sCnt, sTab.c, CAN_MULTI && multi ? sAcc : nullptr, tid);
        }
        __syncthreads();
        }   // pod table

        // few pods per tile: most buckets are empty and nine (two loads, compare, branch) prologues per tile show; one
        // word says which buckets to enter
        const uint32_t kmask = STREAM ? (uint32_t)sOff[11] : 0x1FFu;
        // k above every warp's F: no slot of the tile can serve those pods, so their buckets are neither entered (no
        // rows of INF32) nor flushed.  (A multi-tile item reads its chunk's table once, before the barrier sF needs.)
        int fb = 8;
        if (!STREAM && !multi) {
            fb = sF[0];
#pragma unroll
            for (int w = 1; w < SP_WARPS; w++) fb = max(fb, (int)sF[w]);
        }
#define KGPU_SP_RUN(K) \
        if ((!STREAM || ((kmask >> K) & 1u)) && K <= fb) sp_run_k<K, PER_PAIR, MEM, BYTE_KEYS>(F, C, pc, nfree, valid, mem, lane_field, sTab.c.one, best_row, sOff[K], sOff[K + 1]);
        KGPU_SP_RUN(0) KGPU_SP_RUN(1) KGPU_SP_RUN(2) KGPU_SP_RUN(3) KGPU_SP_RUN(4) KGPU_SP_RUN(5) KGPU_SP_RUN(6) KGPU_SP_RUN(7) KGPU_SP_RUN(8)
#undef KGPU_SP_RUN
        __syncthreads();

        // block result per pod: min over the warps of (cost, node id), S' -> real GPU mask through the
        // winner's one-hot bytes, REDG.MIN.64 into keys[pod].  Ordered tile + byte keys: the warp index goes
        // into bits 13.. of the warp key (its lane byte has 3 spare bits) and plain 32-bit mins decide;
        // otherwise (a tile of two classes) node ids are compared explicitly.
        const int served = sOff[min(fb, 8) + 1];   // the buckets above fb, then bucket 9 (not for this launch), sit at the end
        for (int i = tid; i < served; i += SP_THREADS) {
            if (sIdx[i] == SP_DUMMY) continue;
            uint32_t best_m = INF32, cost = 0;
            int best_slot = -1;
            if (BYTE_KEYS && ordered) {
#pragma unroll
                for (int w = 0; w < SP_WARPS; w++) best_m = min(best_m, sTab.best[w][i] | ((uint32_t)w << 13));   // INF32 stays INF32
                if (best_m != INF32) { best_slot = (int)((best_m >> 8) & (uint32_t)(SP_THREADS - 1)); cost = best_m >> 16; }
            } else {
                unsigned long long best = ~0ull;   // cost<<32 | node index
#pragma unroll
                for (int w = 0; w < SP_WARPS; w++) {
                    const uint32_t m = sTab.best[w][i];
                    if (m == INF32) continue;
                    const int s = w * 32 + (int)((m >> 8) & 31u);
                    const unsigned long long cand = ((unsigned long long)(m >> (BYTE_KEYS ? 16 : 13)) << 32) | (uint32_t)sNode[s];
                    if (cand < best) { best = cand; best_slot = s; best_m = m; cost = (uint32_t)(best >> 32); }
                }
            }
            if (best_slot >= 0 && multi) {
                const unsigned long long cand = ((unsigned long long)cost << 32) | (uint32_t)sNode[best_slot];
                if (cand < sAcc[i]) {                        // position i belongs to this thread for the whole item
                    sAcc[i] = cand;
                    sWin[i] = ((uint32_t)tt << 16) | ((uint32_t)best_slot << 8) | (best_m & 0xFFu);
                }
            } else if (best_slot >= 0) {
                // S' bit g set -> byte g of the one-hot words; OR the selected bytes together
                uint32_t S;
                if (STREAM) {                          // bit g of S' -> GPU index in the g-th 3-bit field of the permutation word
                    const uint32_t perm = sHotLo[best_slot];
                    S = 0;
#pragma unroll
                    for (int g = 0; g < 8; g++) S |= ((best_m >> g) & 1u) << ((perm >> (3 * g)) & 7u);
                } else {
                    const uint32_t sel_lo = (((best_m & 0xFu) * 0x00204081u) & 0x01010101u) * 0xFFu;
                    const uint32_t sel_hi = ((((best_m >> 4) & 0xFu) * 0x00204081u) & 0x01010101u) * 0xFFu;
                    uint32_t t = (sHotLo[best_slot] & sel_lo) | (sHotHi[best_slot] & sel_hi);
                    t |= t >> 16;
                    S = (t | (t >> 8)) & 0xFFu;
                }
                const unsigned long long nid = (unsigned long long)(node_id_base + (long long)sNode[best_slot]);
                const unsigned long long key = ((unsigned long long)cost << 40) | (nid << 8) | S;
                atomicMin(&keys[c0 + sIdx[i]], key);
            }
        }
    }
    }   // tiles of the item
    if (multi) {
        const int served = sOff[9];
        for (int i = tid; i < served; i += SP_THREADS) {
            const unsigned long long a = sAcc[i];
            if (sIdx[i] == SP_DUMMY || a == ~0ull) continue;
            const uint32_t w = sWin[i];
            const uint32_t perm = __ldg(meta + (tile_first + (int64_t)(w >> 16)) * SP_THREADS + ((w >> 8) & 0xFFu));
            uint32_t S = 0;
#pragma unroll
            for (int g = 0; g < 8; g++) S |= ((w >> g) & 1u) << ((perm >> (3 * g)) & 7u);
            const unsigned long long nid = (unsigned long long)(node_id_base + (long long)(int32_t)(uint32_t)a);
            atomicMin(&keys[p_begin + sIdx[i]], ((a >> 32) << 40) | (nid << 8) | S);
        }
    }
}

// The host's choice of K1s instantiation for a batch (launch_plan.h: sparse_route), and the one kernel it names; mem: the
// launch for the memory-constrained pods.  Every instantiation takes the same arguments (the streaming ones ignore
// `chunks`), so libkgpu and the CPU emulation launch whatever this returns.
struct SparseRoute {
    bool stream, tma, prepared, byte_keys;
};
using SparseKernel = void (*)(const int4 *, const uint32_t *, const int32_t *, const int32_t *, const int *, int64_t,
                              const int4 *, int64_t, int, const int4 *, PipeConsts, unsigned long long *, const int4 *);
inline SparseKernel sparse_kernel(const SparseRoute &r, bool mem) {
    if (mem) return r.byte_keys ? score_pairs_sparse<true, true, true> : score_pairs_sparse<true, true, false>;
    if (r.tma)
        return r.byte_keys ? score_pairs_sparse<true, false, true, true, KGPU_SP_TMA_MINBLOCKS>
                           : score_pairs_sparse<true, false, false, true, KGPU_SP_TMA_MINBLOCKS>;
    if (r.stream) return r.byte_keys ? score_pairs_sparse<true, false, true, true> : score_pairs_sparse<true, false, false, true>;
    return r.byte_keys ? score_pairs_sparse<true, false, true> : score_pairs_sparse<true, false, false>;
}

}  // namespace kgpu
