// kgpu.cu -- C ABI of libkgpu (include/kgpu.h) over the sm_90a kernels in
// score_pairs.cuh.  No CPU fallback: every entry point needs a CUDA device.
#include "../../include/kgpu.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <array>
#include <chrono>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <unordered_set>
#include <vector>

#include "buffer.h"
#include "multi_device.h"
#include "gang_domain.cuh"
#include "place_sequential.cuh"
#include "preempt.cuh"
#include "preempt_plan.cuh"
#include "preempt_plan_domain.cuh"
#include "sparse_work.h"
#include "peer_exchange.cuh"
#include "score_pairs.cuh"
#include "score_pairs_sparse.cuh"
#include "node_state.cuh"
#include "launch_plan.h"

namespace {

thread_local std::string t_last_error;

// F2/F2N multipliers handed to the kernels as arguments so that ptxas cannot fold them
// (subset_dp_gen.cuh: pins those adds to the FMA pipe).
const kgpu::PipeConsts PC = {1u, 0xFFFFFFFFu};

const int32_t kDefaultWeights[16] = {64, 32, 16, 8, 4, 2, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0};

}  // namespace

// One device's shard of the node array plus its scratch buffers.
struct kgpu_shard {
    int dev = -1;
    int sm_count = 0;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    kgpu::DeviceBuffer<int32_t> d_topo;   // [n][64]
    kgpu::DeviceBuffer<int32_t> d_free;   // [n]
    kgpu::DeviceBuffer<int32_t> d_mem;    // [n][8] MiB per GPU (INT32_MAX = unconstrained until uploaded)
    kgpu::DeviceBuffer<int> d_flag;       // "batch has memory-constrained pods"
    kgpu::DeviceBuffer<int4> d_rec;       // K1s: [tiles][7][SP_THREADS] compacted scaled pair costs, slot order (compact_nodes)
    kgpu::DeviceBuffer<uint32_t> d_meta;  // K1s: [n_slots] position -> GPU index (3-bit fields) | free count << 24
    bool compact_dirty = true;       // topology / weights changed for every node since the cache was built
    bool order_dirty = true;         // the order (slots by free count) must be rebuilt before the next K1s launch
    int64_t stale_nodes = 0;         // nodes whose free count changed since the order was built (re-sort when many)
    kgpu::DeviceBuffer<int32_t> d_order;     // K1s: slot -> node index, grouped by popcount(free), -1 = padding
    kgpu::DeviceBuffer<int32_t> d_slot_of;   // K1s: node index -> slot
    kgpu::DeviceBuffer<int32_t> d_ord_cnt, d_ord_off;   // counting sort scratch [9][blocks]
    kgpu::DeviceBuffer<long long> d_ord_meta;           // class counts [9], n_slots
    kgpu::DeviceBuffer<unsigned long long> d_bad;       // validate_topo_dev: first out-of-domain element
    kgpu::DeviceBuffer<int32_t> d_upd;        // state-change scratch: [m] node indices | [m] masks
    kgpu::DeviceBuffer<uint32_t> d_fit_patch; // [9][m] fit-table rows of the nodes a state change touched
    kgpu::DeviceBuffer<uint32_t> d_fit;       // (node, k) fit table on the device [9][n]
    kgpu::PinnedBuffer<uint32_t> h_fit;       // pinned host copy [9][n]: kgpu_fit_lookup / kgpu_score_pairs read it
    bool fit_valid = false;
    kgpu::DeviceBuffer<int4> d_query;         // kgpu_score_pairs with min_mem: {node lo, node hi, k, min_mem}
    kgpu::DeviceBuffer<uint32_t> d_qout;
    kgpu::DeviceBuffer<int32_t> d_free_scratch;   // kgpu_place_batch_ex(KGPU_PLACE_DRY_RUN): the masks the dry run consumes
    kgpu::DeviceBuffer<int32_t> d_hold;       // [n][8] holder table (kgpu_upload_holders / kgpu_set_holders), allocated on first upload
    bool has_hold = false;           // false = every entry is -1 (no upload since the last kgpu_upload_nodes)
    kgpu::DeviceBuffer<int32_t> d_lvl;        // kgpu_preempt_batch scratch [P]: pod levels, compacted pod positions,
    kgpu::DeviceBuffer<int32_t> d_pidx;       //   their preemption keys, victims, and the compacted count
    kgpu::DeviceBuffer<unsigned long long> d_pkey;
    kgpu::DeviceBuffer<uint32_t> d_victims;
    kgpu::DeviceBuffer<int> d_pcnt;
    kgpu::DeviceBuffer<int32_t> d_plan_free;   // kgpu_preempt_plan: working copies of the free masks [n]
    kgpu::DeviceBuffer<int32_t> d_plan_hold;   //   and of the holder table [n][8],
    kgpu::DeviceBuffer<int4> d_plan_cols;      //   the batch's columns {k, level, min_mem, 0}, each pod's column [P],
    kgpu::DeviceBuffer<int32_t> d_plan_pcol;
    kgpu::DeviceBuffer<unsigned long long> d_plan_nodekey;   //   per-column node keys [cols][Npad]
    kgpu::DeviceBuffer<unsigned long long> d_plan_tilekey;   //   and their tile minima [cols][T]
    kgpu::DeviceBuffer<int4> d_plan_pre;       // kgpu_preempt_plan_gang: each placed member's pre-image {F, H row} [P]
    kgpu::DeviceBuffer<int32_t> d_dom_off;     // kgpu_upload_domain_levels (launch_plan.h: domain_table): each level's
    kgpu::DeviceBuffer<int32_t> d_dom_nodes;   //   [D_l + 1] domain ranges of d_dom_nodes, level 0 first
    int32_t n_dom = 0;               // D_0; 0 = no node in a level-0 domain (so after kgpu_upload_nodes)
    std::vector<kgpu::DomainLevel> dom_levels = {{0, 0}};   // each level's D_l and base in d_dom_off, its chunks
    kgpu::DeviceBuffer<int32_t> d_dom_chunk;   // the chunked walk: each domain's chunk range (laid out as d_dom_off),
    kgpu::DeviceBuffer<int32_t> d_chunk_begin; //   each chunk's first entry of d_dom_nodes [chunks + 1],
    int64_t n_chunks = 0;
    kgpu::DeviceBuffer<unsigned long long> d_dom_cmin;   //   per call: the chunk minima [views * 9][chunks],
    kgpu::DeviceBuffer<uint32_t> d_dom_cstamp;           //   each chunk's trial stamp [chunks]
    kgpu::DeviceBuffer<int32_t> d_dom_pairs;             //   and each chunked trial's (view, k) pairs
    kgpu::DeviceBuffer<int32_t> d_dom_mask;    // domain steps: per-node working mask of the trials [n]
    kgpu::DeviceBuffer<uint32_t> d_dom_stamp;  //   and the stamp of the trial that wrote it [n]
    kgpu::DeviceBuffer<unsigned long long> d_dom_best;   //   per (step, level): (C_d << 32 | d) of the best trial
    kgpu::DeviceBuffer<uint2> d_dom_hold;      // plan domain steps: per-node working holder row of the trials [n]
    kgpu::DeviceBuffer<unsigned long long> d_dom_score;  //   and each domain's trial score [D]
    int64_t class_count[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    int64_t n_slots = 0;
    int64_t n = 0;
    int64_t node_id_base = 0;
    kgpu::DeviceBuffer<int32_t> d_pods;       // [P][4]
    kgpu::DeviceBuffer<int32_t> d_gang;       // [P] kgpu_place_batch_gang / kgpu_preempt_plan_gang: gang id per pod
    kgpu::DeviceBuffer<unsigned long long> d_keys;     // [P]
    kgpu::DeviceBuffer<unsigned long long> d_gather;   // [ndev][P] (multi-device only)
    kgpu::DeviceBuffer<unsigned long long> d_bestk;    // [9] memo variant
    std::vector<uint8_t> tile_class;         // K1s: max free-GPU count per 128-slot tile of the order (host copy)
    std::vector<kgpu::SparseWorkItem> h_work;   // K1s work list for work_P pods (sparse_work.h)
    kgpu::DeviceBuffer<int4> d_work;
    int64_t work_P = -1;
    bool work_aligned = false;                  // its pod ranges are whole chunks: K1s launches take prepared chunk tables
    kgpu::DeviceBuffer<int4> d_chunks;          // [chunks][SP_CHUNK_INT4] sp_prepare_chunks: the batch's sorted pod tables
    bool tma_attr_done = false;                 // cudaFuncSetAttribute of the TMA instantiations done on this device
    bool place_attr_done = false;               // the same for place_sequential<false / true> (PLACE_DYN_SMEM)
    kgpu::DeviceBuffer<uint32_t> d_nodebest;    // [views][9][Npad]  K3 tables
    kgpu::DeviceBuffer<int32_t> d_half;         // [Npad][96]  K3: half tables of every node (place_half_tables)
    kgpu::DeviceBuffer<unsigned long long> d_tilebest;   // [views][9][T]
};

struct kgpu_ctx {
    std::mutex mu;
    std::string err;
    std::vector<kgpu_shard> shards;
    int32_t W[16];
    int variant = KGPU_VARIANT_AUTO;
    int64_t n_total = 0;
    int64_t launches = 0;
    double last_kernel_ms = 0.0;
    bool subsets_uploaded = false;
    double last_upload_ms = 0.0;
    kgpu::MultiDevice *multi = nullptr;   // NCCL communicator set, ndev > 1 only
    // peer-memory key exchange (kgpu_exchange_*): one allocation per rank, mapped by every peer:
    //   slots[2][world][max_pods] uint64 | flags[PEER_MAX_WORLD] uint32 | ticket | error ;  local[] and final_keys[] are private
    struct {
        int world = 0, rank = 0;
        int64_t max_pods = 0;
        kgpu::DeviceBuffer<unsigned char> base;
        void *peer_base[kgpu::PEER_MAX_WORLD] = {};
        kgpu::DeviceBuffer<unsigned long long> local;
        kgpu::DeviceBuffer<unsigned long long> final_keys;   // [2][max_pods]: the global keys of the last two epochs
        uint32_t epoch = 0;
        bool connected = false;
    } xch;
};

namespace {

int fail(kgpu_ctx *h, int code, const char *fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    t_last_error = buf;
    if (h) h->err = buf;
    return code;
}

#define KGPU_CUDA(h, expr)                                                                          \
    do {                                                                                            \
        cudaError_t e__ = (expr);                                                                   \
        if (e__ != cudaSuccess)                                                                     \
            return fail((h), e__ == cudaErrorMemoryAllocation ? KGPU_ERR_NOMEM : KGPU_ERR_CUDA,      \
                        "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__); \
    } while (0)

int upload_subset_tables(kgpu_ctx *h) {
    uint8_t subs[9][70];
    uint8_t nsub[9];
    kgpu::subset_tables(subs, nsub);
    for (auto &s : h->shards) {
        KGPU_CUDA(h, cudaSetDevice(s.dev));
        KGPU_CUDA(h, cudaMemcpyToSymbol(kgpu::c_subsets, subs, sizeof subs));
        KGPU_CUDA(h, cudaMemcpyToSymbol(kgpu::c_nsub, nsub, sizeof nsub));
    }
    h->subsets_uploaded = true;
    return KGPU_OK;
}

// Scratch sized by a call's batch grows with headroom, so that a slowly growing batch reallocates rarely: pod-indexed
// buffers to P + P / 4 pods (at least 1024), the update and query lists to m + m / 2 entries (at least 256).
int64_t pod_headroom(int64_t P) { return std::max<int64_t>(1024, P + P / 4); }
int64_t list_headroom(int64_t m) { return std::max<int64_t>(256, m + m / 2); }

// The pods and keys of a P-pod batch on shard s, and with several devices the all-gather's receive buffer.
int reserve_pods(kgpu_ctx *h, kgpu_shard &s, int64_t P) {
    const int64_t cap = pod_headroom(P), G = (int64_t)h->shards.size();
    KGPU_CUDA(h, cudaSetDevice(s.dev));
    KGPU_CUDA(h, s.d_pods.reserve(4 * P, 4 * cap));
    KGPU_CUDA(h, s.d_keys.reserve(P, cap));
    if (G > 1) KGPU_CUDA(h, s.d_gather.reserve(G * P, G * cap));
    return KGPU_OK;
}

// Classes of the K1s order are padded to whole warps (32).  Padding them to whole tiles (KGPU_ORDER_PAD=128: no block ever
// mixes classes) loses on an H100 SXM (400 W limit): K1s on C2 takes 0.086 against 0.085 ms on a 12.5k-node shard and
// 0.524 - 0.527 against 0.514 - 0.518 ms at 100k nodes, so the smaller order stays.
const int kOrderPad = [] { const char *e = getenv("KGPU_ORDER_PAD"); const int v = e ? atoi(e) : 0; return v == 128 ? (int)kgpu::SP_THREADS : 32; }();

// (Re)build the K1s order of shard s on the device: stable counting sort of the node indices by free-GPU
// count (node_state.cuh).  One 80-byte read-back tells the host the class sizes (grid size, work list).
int build_order(kgpu_ctx *h, kgpu_shard &s) {
    KGPU_CUDA(h, cudaSetDevice(s.dev));
    const int64_t need_slots = s.n + 10 * kgpu::SP_THREADS;
    const int64_t slots = (need_slots + kgpu::SP_THREADS - 1) / kgpu::SP_THREADS * kgpu::SP_THREADS;
    KGPU_CUDA(h, s.d_order.reserve(need_slots, slots));
    KGPU_CUDA(h, s.d_meta.reserve(need_slots, slots));
    KGPU_CUDA(h, s.d_rec.reserve(7 * need_slots, 7 * slots));
    const int nb = (int)((s.n + kgpu::ORD_BLOCK - 1) / kgpu::ORD_BLOCK);
    KGPU_CUDA(h, s.d_ord_cnt.reserve(9 * nb));
    KGPU_CUDA(h, s.d_ord_off.reserve(9 * nb));
    long long meta[kgpu::ORD_META] = {0};
    if (s.n > 0) {
        KGPU_CUDA(h, cudaMemsetAsync(s.d_order, 0xFF, (size_t)s.d_order.capacity() * 4, s.stream));
        kgpu::order_count<<<nb, kgpu::ORD_BLOCK, 0, s.stream>>>(s.d_free, s.n, s.d_ord_cnt, nb);
        kgpu::order_scan<<<1, kgpu::ORD_BLOCK, 0, s.stream>>>(s.d_ord_cnt, nb, s.d_ord_off, s.d_ord_meta, kgpu::SP_THREADS, kOrderPad);
        kgpu::order_scatter<<<nb, kgpu::ORD_BLOCK, 0, s.stream>>>(s.d_free, s.n, s.d_ord_off, nb, s.d_order, s.d_slot_of);
        h->launches += 3;
        KGPU_CUDA(h, cudaGetLastError());
        KGPU_CUDA(h, cudaMemcpyAsync(meta, s.d_ord_meta, sizeof meta, cudaMemcpyDeviceToHost, s.stream));
        KGPU_CUDA(h, cudaStreamSynchronize(s.stream));
    }
    for (int c = 0; c < 9; c++) s.class_count[c] = meta[c];
    s.n_slots = meta[9];
    s.tile_class = kgpu::tile_classes(s.class_count, kOrderPad, s.n_slots);
    s.work_P = -1;
    s.order_dirty = false;
    s.stale_nodes = 0;
    s.compact_dirty = true;            // records are stored in slot order
    return KGPU_OK;
}

// Bring the K1s node cache of shard s up to date (order, compacted records); everything runs on s.stream and
// has completed when this returns, so a following launch on any stream sees it.
int ensure_node_cache(kgpu_ctx *h, kgpu_shard &s) {
    static const int64_t resort_div = [] { const char *e = getenv("KGPU_RESORT_DIV"); int v = e ? atoi(e) : 0; return (int64_t)(v > 0 ? v : 200); }();
    // Nodes whose free count changed keep their slot, so their warp enumerates for the LARGEST count among its 32
    // lanes, and a stale order makes every later step slower.  So re-sort as soon as more than n / 200 nodes have changed
    // (KGPU_RESORT_DIV).  Measured on an H100 SXM (400 W limit), C2 with 1 % of the nodes changing before every step
    // (scripts/churn_time.py, median of 30 steps, wall clock): n / 50: 0.97 ms, n / 200: 0.91, n / 800: 0.88 (within
    // the noise of this measurement), never re-sorting: 1.50 ms and growing.
    if (!s.order_dirty && s.stale_nodes * resort_div > s.n) s.order_dirty = true;
    if (!s.order_dirty && !s.compact_dirty) return KGPU_OK;
    if (s.order_dirty) {
        const int rc = build_order(h, s);
        if (rc != KGPU_OK) return rc;
    }
    KGPU_CUDA(h, cudaSetDevice(s.dev));
    if (s.compact_dirty && s.n_slots > 0) {
        kgpu::Weights W;
        memcpy(W.w, h->W, sizeof W.w);
        kgpu::compact_nodes<<<(unsigned)(s.n_slots / kgpu::SP_THREADS), kgpu::SP_THREADS, 0, s.stream>>>(
            reinterpret_cast<const int4 *>(s.d_topo.get()), s.d_free, s.n_slots, W, s.d_order, s.d_slot_of, s.d_rec, s.d_meta);
        h->launches++;
        KGPU_CUDA(h, cudaGetLastError());
    }
    s.compact_dirty = false;
    KGPU_CUDA(h, cudaStreamSynchronize(s.stream));
    return KGPU_OK;
}

// (node, k) fit table of shard s: fit_nodes over every node, one copy to the pinned host array.
int build_fit_table(kgpu_ctx *h, kgpu_shard &s) {
    KGPU_CUDA(h, cudaSetDevice(s.dev));
    KGPU_CUDA(h, s.d_fit.reserve(9 * s.n));
    KGPU_CUDA(h, s.h_fit.reserve(9 * s.n));
    if (s.n > 0) {
        kgpu::Weights W;
        memcpy(W.w, h->W, sizeof W.w);
        kgpu::fit_nodes<<<(unsigned)((s.n + 127) / 128), 128, 0, s.stream>>>(reinterpret_cast<const int4 *>(s.d_topo.get()), s.d_free,
                                                                          nullptr, s.n, W, PC, s.d_fit);
        h->launches++;
        KGPU_CUDA(h, cudaGetLastError());
        KGPU_CUDA(h, cudaMemcpyAsync(s.h_fit, s.d_fit, (size_t)s.n * 36, cudaMemcpyDeviceToHost, s.stream));
        KGPU_CUDA(h, cudaStreamSynchronize(s.stream));
    }
    s.fit_valid = true;
    return KGPU_OK;
}

// State change of m nodes of shard s (local indices idx, already distinct): masks != nullptr scatters the new
// free masks; either way the compacted records of exactly those nodes are refreshed, and the fit table's rows
// if it is valid.  One H2D copy, one or two kernels, one small D2H copy (fit rows), synchronous.
int apply_node_updates(kgpu_ctx *h, kgpu_shard &s, const int32_t *idx, const int32_t *masks, int64_t m) {
    if (m <= 0) return KGPU_OK;
    KGPU_CUDA(h, cudaSetDevice(s.dev));
    KGPU_CUDA(h, s.d_upd.reserve(2 * m, 2 * list_headroom(m)));
    if (s.fit_valid) KGPU_CUDA(h, s.d_fit_patch.reserve(9 * m, 9 * list_headroom(m)));
    int32_t *d_masks = masks ? s.d_upd + m : nullptr;
    KGPU_CUDA(h, cudaMemcpyAsync(s.d_upd, idx, (size_t)m * 4, cudaMemcpyHostToDevice, s.stream));
    if (masks) KGPU_CUDA(h, cudaMemcpyAsync(d_masks, masks, (size_t)m * 4, cudaMemcpyHostToDevice, s.stream));
    kgpu::Weights W;
    memcpy(W.w, h->W, sizeof W.w);
    const int4 *topo4 = reinterpret_cast<const int4 *>(s.d_topo.get());
    const bool cache_live = !s.order_dirty && !s.compact_dirty;
    if (cache_live) {
        kgpu::compact_nodes<<<(unsigned)((m + kgpu::SP_THREADS - 1) / kgpu::SP_THREADS), kgpu::SP_THREADS, 0, s.stream>>>(
            topo4, s.d_free, m, W, s.d_order, s.d_slot_of, s.d_rec, s.d_meta, s.d_upd, d_masks);
        h->launches++;
        s.stale_nodes += m;
    } else if (masks) {
        kgpu::scatter_masks<<<(unsigned)((m + 255) / 256), 256, 0, s.stream>>>(s.d_upd, d_masks, m, s.d_free);
        h->launches++;
    }
    KGPU_CUDA(h, cudaGetLastError());
    if (s.fit_valid) {
        // rows of the changed nodes -> the persistent patch buffer -> the host table
        kgpu::fit_nodes<<<(unsigned)((m + 127) / 128), 128, 0, s.stream>>>(topo4, s.d_free, s.d_upd, m, W, PC, s.d_fit_patch);
        h->launches++;
        KGPU_CUDA(h, cudaGetLastError());
        std::vector<uint32_t> rows((size_t)m * 9);
        KGPU_CUDA(h, cudaMemcpyAsync(rows.data(), s.d_fit_patch, (size_t)m * 36, cudaMemcpyDeviceToHost, s.stream));
        KGPU_CUDA(h, cudaStreamSynchronize(s.stream));
        for (int k = 0; k < 9; k++)
            for (int64_t i = 0; i < m; i++) s.h_fit[(int64_t)k * s.n + idx[i]] = rows[(size_t)((int64_t)k * m + i)];
    } else {
        KGPU_CUDA(h, cudaStreamSynchronize(s.stream));
    }
    return KGPU_OK;
}

// Enqueue K1 for P pods on shard s: d_keys[p] = best placement over this shard's nodes.
// has_mem: 1 / 0 = the host knows whether some pod carries min_mem > 0; -1 = unknown (device buffers).
int launch_score(kgpu_ctx *h, kgpu_shard &s, const int32_t *d_pods, int64_t P, unsigned long long *d_keys,
                 cudaStream_t st, int has_mem, bool keys_are_clean = false) {
    if (P <= 0) return KGPU_OK;
    if ((reinterpret_cast<uintptr_t>(d_pods) & 15u) != 0)
        return fail(h, KGPU_ERR_INVALID, "pods pointer must be 16-byte aligned");
    KGPU_CUDA(h, cudaSetDevice(s.dev));
    kgpu::Weights W;
    memcpy(W.w, h->W, sizeof W.w);
    const int4 *topo4 = reinterpret_cast<const int4 *>(s.d_topo.get());
    const int4 *pods4 = reinterpret_cast<const int4 *>(d_pods);

    const int4 *mem4 = reinterpret_cast<const int4 *>(s.d_mem.get());
    if (!keys_are_clean) KGPU_CUDA(h, cudaMemsetAsync(d_keys, 0xFF, (size_t)P * 8, st));
    if (s.n == 0) return KGPU_OK;

    // AUTO (the default): whatever is cheapest for THIS batch with identical keys -- pods without a memory requirement
    // are memoisable by k under snapshot scoring (best[k] over all nodes once, then a gather: memo_best_by_k /
    // memo_gather), pods with one go to K1m (the sparse MEM instantiation).  The per-pair kernels are the explicitly
    // named variants (KGPU_VARIANT_SPARSE = what bench.py's headline times, per north_star).
    const bool automode = h->variant == KGPU_VARIANT_AUTO;
    const bool memo = automode || h->variant == KGPU_VARIANT_MEMO_BY_K;
    const bool wpp = h->variant == KGPU_VARIANT_WARP_PER_PAIR;
    const bool sparse_main = h->variant == KGPU_VARIANT_SPARSE;
    const bool sparse = sparse_main || (automode && has_mem != 0);
    if (sparse) {                      // order + compacted records current?  (no-op unless nodes / masks / weights changed)
        const int rc = ensure_node_cache(h, s);
        if (rc != KGPU_OK) return rc;
    }
    if (!wpp && has_mem != 0) {   // which pods go to K1m?  (flag read by its blocks; skipped when the host knows there are none)
        KGPU_CUDA(h, cudaMemsetAsync(s.d_flag, 0, sizeof(int), st));
        kgpu::any_mem_pod<<<(unsigned)((P + 255) / 256), 256, 0, st>>>(pods4, P, s.d_flag);
        h->launches++;
    }
    if (memo) {
        KGPU_CUDA(h, cudaMemsetAsync(s.d_bestk, 0xFF, 9 * 8, st));
        int blocks = (int)std::min<int64_t>((s.n + kgpu::LPN_THREADS - 1) / kgpu::LPN_THREADS, (int64_t)s.sm_count * 4);
        kgpu::memo_best_by_k<<<blocks, kgpu::LPN_THREADS, 0, st>>>(topo4, s.d_free, s.n, s.node_id_base, W, PC, s.d_bestk);
        kgpu::memo_gather<<<(unsigned)((P + 255) / 256), 256, 0, st>>>(pods4, P, s.d_bestk, d_keys);
        h->launches += 2;
    }
    const int tile = wpp ? kgpu::WPP_TILE : kgpu::LPN_THREADS;
    const int64_t tiles = sparse ? s.n_slots / kgpu::SP_THREADS : (s.n + tile - 1) / tile;
    // Pod splits: enough blocks for ~8 waves of resident CTAs, but each block keeps
    // >= 128 pods so staging its node tile stays amortised.
    const int64_t resident = (int64_t)s.sm_count * (wpp ? 8 : sparse ? KGPU_SP_MINBLOCKS : KGPU_LPN_MINBLOCKS);
    static const int64_t waves = [] { const char *e = getenv("KGPU_WAVES"); int v = e ? atoi(e) : 0; return (int64_t)(v > 0 ? v : 8); }();
    int64_t splits = std::max<int64_t>(1, (waves * resident + tiles - 1) / tiles);
    splits = std::min<int64_t>(splits, std::max<int64_t>(1, P / 128));
    splits = std::min<int64_t>(splits, 65535);
    const int64_t per = kgpu::pods_per_split(P, splits);
    splits = (P + per - 1) / per;
    if (tiles > 0x7FFFFFFFLL || per > 0x7FFFFFFFLL) return fail(h, KGPU_ERR_INVALID, "batch too large for one launch");
    dim3 grid((unsigned)tiles, (unsigned)splits);
    if (wpp) {
        kgpu::score_pairs_warp_per_pair<<<grid, kgpu::WPP_THREADS, 0, st>>>(topo4, s.d_free, s.d_mem, s.n, s.node_id_base, pods4, P,
                                                                            (int)per, W, PC, d_keys);
        h->launches++;
    } else {
        if (h->variant == KGPU_VARIANT_TILE_MEMO) {
            kgpu::score_pairs_lane_per_node<false, false><<<grid, kgpu::LPN_THREADS, 0, st>>>(
                topo4, s.d_free, mem4, s.d_flag, s.n, s.node_id_base, pods4, P, (int)per, W, PC, d_keys);
            h->launches++;
        } else if (h->variant == KGPU_VARIANT_LANE_PER_NODE) {
            kgpu::score_pairs_lane_per_node<true, false><<<grid, kgpu::LPN_THREADS, 0, st>>>(
                topo4, s.d_free, mem4, s.d_flag, s.n, s.node_id_base, pods4, P, (int)per, W, PC, d_keys);
            h->launches++;
        }
        if (sparse) {
            // The work list (sparse_work.h: items of about equal work, heaviest first; runs of tiles when the batch is
            // one chunk) instead of the plain grid, whose equal pod ranges leave a tail.  Measured on an H100 SXM (400 W
            // limit), C2: 0.514 - 0.518 ms against 0.573 - 0.581 with the plain grid; KGPU_SP_WORKLIST=0 forces it.
            static const int worklist_mode = [] { const char *e = getenv("KGPU_SP_WORKLIST"); return e ? atoi(e) : -1; }();
            const bool use_work = worklist_mode != 0;
            static const int tma_mode = [] { const char *e = getenv("KGPU_SP_TMA"); return e ? atoi(e) : 1; }();
            const int4 *d_work = nullptr;
            if (use_work) {
                if (s.work_P != P) {
                    kgpu::SparseWorkParams prm;
                    static const int max_run = [] { const char *e = getenv("KGPU_SP_MAXRUN"); return e ? atoi(e) : 0; }();
                    if (max_run > 0) prm.max_run = max_run;
                    static const int env_tail = [] { const char *e = getenv("KGPU_SP_TAIL"); return e ? atoi(e) : -1; }();
                    static const int env_waves = [] { const char *e = getenv("KGPU_SP_WAVES"); return e ? atoi(e) : -1; }();
                    static const int env_floor = [] { const char *e = getenv("KGPU_SP_FLOOR"); return e ? atoi(e) : -1; }();
                    if (env_tail >= 0) prm.tail_percent = env_tail;
                    if (env_waves > 0) prm.waves = env_waves;
                    if (env_floor > 0) prm.floor = env_floor;
                    const int64_t res_list = kgpu::sparse_list_resident(P, tma_mode, s.sm_count, resident);
                    kgpu::build_sparse_work(s.tile_class, P, res_list, s.h_work, prm);
                    s.work_aligned = kgpu::sparse_work_chunk_aligned((int64_t)s.tile_class.size(), P, res_list, prm);
                    KGPU_CUDA(h, s.d_work.reserve((int64_t)s.h_work.size()));
                    static_assert(sizeof(kgpu::SparseWorkItem) == sizeof(int4), "work item layout");
                    KGPU_CUDA(h, cudaMemcpyAsync(s.d_work, s.h_work.data(), s.h_work.size() * sizeof(int4), cudaMemcpyHostToDevice, st));
                    s.work_P = P;
                }
                d_work = s.d_work;
                grid = dim3((unsigned)s.h_work.size(), 1);
            }
            // Whole-chunk pod ranges: every chunk's pod table is built once for the launch (sp_prepare_chunks, on the
            // same stream just before each K1s launch) rather than by each of the ~900 blocks that score it (C2).
            const kgpu::SparseRoute route = kgpu::sparse_route(P, use_work, s.work_aligned, tma_mode, h->W);
            const int64_t n_chunks = (P + kgpu::SP_CHUNK - 1) / kgpu::SP_CHUNK;
            if (route.prepared) {
                if (n_chunks > 0x7FFFFFFFLL) return fail(h, KGPU_ERR_INVALID, "batch too large for one launch");
                const int64_t cap_chunks = (pod_headroom(P) + kgpu::SP_CHUNK - 1) / kgpu::SP_CHUNK;
                KGPU_CUDA(h, s.d_chunks.reserve(n_chunks * kgpu::SP_CHUNK_INT4, cap_chunks * kgpu::SP_CHUNK_INT4));
            }
            const int4 *d_chunks = route.prepared ? s.d_chunks.get() : nullptr;
            if (route.tma && !s.tma_attr_done) {   // static + dynamic shared memory may pass 48 KB with more stages: opt in, once per device
                kgpu::SparseRoute r = route;
                r.byte_keys = true;
                cudaError_t e = cudaFuncSetAttribute(kgpu::sparse_kernel(r, false), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kgpu::SP_TMA_DYN_SMEM);
                r.byte_keys = false;
                if (e == cudaSuccess) e = cudaFuncSetAttribute(kgpu::sparse_kernel(r, false), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kgpu::SP_TMA_DYN_SMEM);
                if (e != cudaSuccess) return fail(h, KGPU_ERR_CUDA, "cudaFuncSetAttribute(TMA K1s): %s", cudaGetErrorString(e));
                s.tma_attr_done = true;
            }
            auto launch = [&](bool mem) {
                if (route.prepared) {
                    if (mem) kgpu::sp_prepare_chunks<true><<<(unsigned)n_chunks, kgpu::SP_THREADS, 0, st>>>(pods4, P, s.d_flag, s.d_chunks);
                    else kgpu::sp_prepare_chunks<false><<<(unsigned)n_chunks, kgpu::SP_THREADS, 0, st>>>(pods4, P, s.d_flag, s.d_chunks);
                    h->launches++;
                }
                const kgpu::SparseKernel k1s = kgpu::sparse_kernel(route, mem);
                k1s<<<grid, kgpu::SP_THREADS, route.tma && !mem ? kgpu::SP_TMA_DYN_SMEM : 0, st>>>(
                    s.d_rec, s.d_meta, s.d_mem, s.d_order, s.d_flag, s.node_id_base, pods4, P, (int)per, d_work, PC, d_keys, d_chunks);
                h->launches++;
            };
            if (sparse_main) launch(false);
            if (has_mem != 0) launch(true);
        } else if (has_mem != 0) {   // K1m: the memory-constrained pods (its blocks exit at once if the flag is 0)
            kgpu::score_pairs_lane_per_node<true, true><<<grid, kgpu::LPN_THREADS, 0, st>>>(
                topo4, s.d_free, mem4, s.d_flag, s.n, s.node_id_base, pods4, P, (int)per, W, PC, d_keys);
            h->launches++;
        }
    }
    KGPU_CUDA(h, cudaGetLastError());
    return KGPU_OK;
}

int validate_topo(kgpu_ctx *h, const int32_t *topo, int64_t n) {
    for (int64_t i = 0; i < n * 64; i++)
        if ((uint32_t)topo[i] > 15u)
            return fail(h, KGPU_ERR_INVALID, "topo[%lld][%d] = %d outside the link-level domain 0..15",
                        (long long)(i / 64), (int)(i % 64), topo[i]);
    return KGPU_OK;
}

// Which shard holds local node index idx (contiguous split)?
kgpu_shard *shard_of(kgpu_ctx *h, int64_t idx, int64_t *local) {
    int64_t off = 0;
    for (auto &s : h->shards) {
        if (idx < off + s.n) { *local = idx - off; return &s; }
        off += s.n;
    }
    return nullptr;
}

void free_shard(kgpu_shard &s) {
    if (s.dev < 0) return;
    cudaSetDevice(s.dev);
    if (s.ev0) cudaEventDestroy(s.ev0);
    if (s.ev1) cudaEventDestroy(s.ev1);
    if (s.stream) cudaStreamDestroy(s.stream);
    s = kgpu_shard();                  // frees the buffers
}

}  // namespace

extern "C" {

const char *kgpu_version(void) { return "0.2.0"; }

const char *kgpu_last_error(kgpu_t *h) {
    if (h) {
        std::lock_guard<std::mutex> g(h->mu);
        t_last_error = h->err;   // return storage that outlives the lock
    }
    return t_last_error.c_str();
}

int kgpu_create(const int *dev_ids, int ndev, kgpu_t **out) {
    if (!out) return fail(nullptr, KGPU_ERR_INVALID, "kgpu_create: out is NULL");
    *out = nullptr;
    if (!dev_ids || ndev < 1 || ndev > 64) return fail(nullptr, KGPU_ERR_INVALID, "kgpu_create: need 1..64 device ids");
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0)
        return fail(nullptr, KGPU_ERR_CUDA, "kgpu_create: no usable CUDA device (%s); libkgpu has no CPU path",
                    e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0");
    kgpu_ctx *h = new (std::nothrow) kgpu_ctx();
    if (!h) return fail(nullptr, KGPU_ERR_NOMEM, "kgpu_create: out of host memory");
    memcpy(h->W, kDefaultWeights, sizeof h->W);
    h->shards.resize((size_t)ndev);
    int rc = KGPU_OK;
    for (int i = 0; i < ndev && rc == KGPU_OK; i++) {
        kgpu_shard &s = h->shards[(size_t)i];
        if (dev_ids[i] < 0 || dev_ids[i] >= count) {
            rc = fail(nullptr, KGPU_ERR_INVALID, "kgpu_create: device id %d out of range (have %d)", dev_ids[i], count);
            break;
        }
        s.dev = dev_ids[i];
        auto step = [&](cudaError_t ce, const char *what) {
            if (ce != cudaSuccess && rc == KGPU_OK)
                rc = fail(nullptr, KGPU_ERR_CUDA, "kgpu_create: %s on device %d: %s", what, s.dev, cudaGetErrorString(ce));
        };
        step(cudaSetDevice(s.dev), "cudaSetDevice");
        step(cudaDeviceGetAttribute(&s.sm_count, cudaDevAttrMultiProcessorCount, s.dev), "query SM count");
        step(cudaStreamCreateWithFlags(&s.stream, cudaStreamNonBlocking), "cudaStreamCreate");
        step(cudaEventCreate(&s.ev0), "cudaEventCreate");
        step(cudaEventCreate(&s.ev1), "cudaEventCreate");
        step(s.d_bestk.reserve(9), "cudaMalloc");
        step(s.d_flag.reserve(1), "cudaMalloc");
        step(s.d_ord_meta.reserve(kgpu::ORD_META), "cudaMalloc");
        step(s.d_bad.reserve(1), "cudaMalloc");
    }
    if (rc == KGPU_OK && ndev > 1) {
        std::vector<int> devs(dev_ids, dev_ids + ndev);
        std::string why;
        h->multi = kgpu::MultiDevice::create(devs, &why);
        if (!h->multi) rc = fail(nullptr, KGPU_ERR_COMM, "kgpu_create: %s", why.c_str());
    }
    if (rc == KGPU_OK) rc = upload_subset_tables(h);
    if (rc != KGPU_OK) {
        std::string keep = t_last_error;
        for (auto &s : h->shards) free_shard(s);
        delete h->multi;
        delete h;
        t_last_error = keep;
        return rc;
    }
    *out = h;
    return KGPU_OK;
}

int kgpu_destroy(kgpu_t *h) {
    if (!h) return KGPU_OK;
    for (auto &s : h->shards) {
        if (s.dev >= 0) { cudaSetDevice(s.dev); cudaStreamSynchronize(s.stream); }
    }
    delete h->multi;
    if (h->xch.connected)              // unmap the peers' exchange memory before this rank's is freed (delete h)
        for (int r = 0; r < h->xch.world; r++)
            if (r != h->xch.rank && h->xch.peer_base[r]) cudaIpcCloseMemHandle(h->xch.peer_base[r]);
    for (auto &s : h->shards) free_shard(s);
    delete h;
    return KGPU_OK;
}

int kgpu_set_weights(kgpu_t *h, const int32_t w[KGPU_NUM_LEVELS]) {
    if (!h || !w) return fail(h, KGPU_ERR_INVALID, "kgpu_set_weights: NULL argument");
    std::lock_guard<std::mutex> g(h->mu);
    for (int i = 0; i < 16; i++)
        if (w[i] < 0 || w[i] > KGPU_MAX_WEIGHT)
            return fail(h, KGPU_ERR_INVALID, "kgpu_set_weights: w[%d] = %d outside 0..%d", i, w[i], KGPU_MAX_WEIGHT);
    memcpy(h->W, w, sizeof h->W);
    for (auto &s : h->shards) { s.compact_dirty = true; s.fit_valid = false; }
    return KGPU_OK;
}

int kgpu_get_weights(kgpu_t *h, int32_t w[KGPU_NUM_LEVELS]) {
    if (!h || !w) return fail(h, KGPU_ERR_INVALID, "kgpu_get_weights: NULL argument");
    std::lock_guard<std::mutex> g(h->mu);
    memcpy(w, h->W, sizeof h->W);
    return KGPU_OK;
}

int kgpu_set_variant(kgpu_t *h, int variant) {
    if (!h) return fail(h, KGPU_ERR_INVALID, "kgpu_set_variant: NULL handle");
    std::lock_guard<std::mutex> g(h->mu);
    if (variant < KGPU_VARIANT_AUTO || variant > KGPU_VARIANT_SPARSE)
        return fail(h, KGPU_ERR_INVALID, "kgpu_set_variant: unknown variant %d", variant);
    h->variant = variant;
    return KGPU_OK;
}

namespace {
// kgpu_upload_nodes after its argument checks: shard g gets the contiguous range [g * per, ...).  The caller empties
// the handle when this fails.
int upload_nodes(kgpu_ctx *h, const int32_t *topo, const int32_t *free_mask, int64_t n, int64_t node_id_base, int64_t per) {
    int64_t off = 0;
    for (auto &s : h->shards) {
        const int64_t cnt = std::max<int64_t>(0, std::min<int64_t>(per, n - off));
        KGPU_CUDA(h, cudaSetDevice(s.dev));
        KGPU_CUDA(h, s.d_topo.reserve(64 * cnt));
        KGPU_CUDA(h, s.d_free.reserve(cnt));
        KGPU_CUDA(h, s.d_mem.reserve(8 * cnt));
        KGPU_CUDA(h, s.d_slot_of.reserve(cnt));
        if (cnt > 0) {
            // per-GPU memory is unconstrained (INT32_MAX MiB) until kgpu_upload_gpu_memory says otherwise
            kgpu::fill_i32<<<(unsigned)((cnt * 8 + 255) / 256), 256, 0, s.stream>>>(s.d_mem, cnt * 8, INT32_MAX);
            h->launches++;
            KGPU_CUDA(h, cudaMemcpyAsync(s.d_topo, topo + off * 64, (size_t)cnt * 256, cudaMemcpyHostToDevice, s.stream));
            KGPU_CUDA(h, cudaMemcpyAsync(s.d_free, free_mask + off, (size_t)cnt * 4, cudaMemcpyHostToDevice, s.stream));
            // value-domain check on the device (levels 0..15): one 8-byte read-back instead of an O(64 N) host pass
            KGPU_CUDA(h, cudaMemsetAsync(s.d_bad, 0xFF, sizeof(unsigned long long), s.stream));
            kgpu::validate_topo_dev<<<(unsigned)((cnt * 16 + 255) / 256), 256, 0, s.stream>>>(
                reinterpret_cast<const int4 *>(s.d_topo.get()), cnt * 16, s.d_bad);
            h->launches++;
            KGPU_CUDA(h, cudaGetLastError());
        }
        s.n = cnt;
        s.has_hold = false;            // a new node array has no holders
        s.n_dom = 0;                   // and no domains
        s.dom_levels = {{0, 0}};
        s.n_chunks = 0;
        s.node_id_base = node_id_base + off;
        s.order_dirty = true;
        s.compact_dirty = true;
        s.fit_valid = false;
        off += cnt;
    }
    h->n_total = n;
    // all devices copy concurrently; then the verdicts, then the K1s order + compacted records (device side)
    off = 0;
    for (auto &s : h->shards) {
        if (s.n > 0) {
            unsigned long long bad = ~0ull;
            KGPU_CUDA(h, cudaSetDevice(s.dev));
            KGPU_CUDA(h, cudaMemcpyAsync(&bad, s.d_bad, sizeof bad, cudaMemcpyDeviceToHost, s.stream));
            KGPU_CUDA(h, cudaStreamSynchronize(s.stream));
            if (bad != ~0ull) {
                const long long el = (long long)bad;
                return fail(h, KGPU_ERR_INVALID, "topo[%lld][%d] = %d outside the link-level domain 0..15",
                            (long long)(off + el / 64), (int)(el % 64), topo[(off + el / 64) * 64 + el % 64]);
            }
        }
        off += s.n;
    }
    for (auto &s : h->shards) {
        const int rc = ensure_node_cache(h, s);
        if (rc != KGPU_OK) return rc;
    }
    return KGPU_OK;
}
}  // namespace

int kgpu_upload_nodes(kgpu_t *h, const int32_t *topo, const int32_t *free_mask, int64_t n, int64_t node_id_base) {
    if (!h) return fail(h, KGPU_ERR_INVALID, "kgpu_upload_nodes: NULL handle");
    std::lock_guard<std::mutex> g(h->mu);
    if (n < 0 || (n > 0 && (!topo || !free_mask))) return fail(h, KGPU_ERR_INVALID, "kgpu_upload_nodes: bad arguments");
    if (node_id_base < 0 || node_id_base + n > 0xFFFFFFFFLL)
        return fail(h, KGPU_ERR_INVALID, "kgpu_upload_nodes: node ids must fit in 32 bits");
    const auto t_begin = std::chrono::steady_clock::now();
    const int64_t G = (int64_t)h->shards.size();
    const int64_t per = (n + G - 1) / G;     // contiguous ranges: shard g holds [g*per, ...)
    if (per > 0x7FFFFFFFLL - 4096) return fail(h, KGPU_ERR_INVALID, "kgpu_upload_nodes: more than 2^31 nodes per device");
    const int rc = upload_nodes(h, topo, free_mask, n, node_id_base, per);
    if (rc != KGPU_OK) {               // a failed upload leaves the handle EMPTY (n = 0 everywhere), never half old / half new
        for (auto &s : h->shards) { s.n = 0; s.n_slots = 0; s.n_dom = 0; s.order_dirty = true; s.compact_dirty = true; s.fit_valid = false; s.work_P = -1; }
        h->n_total = 0;
        return rc;
    }
    h->last_upload_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_begin).count();
    return KGPU_OK;
}

int kgpu_upload_gpu_memory(kgpu_t *h, const int32_t *mem_mib, int64_t n) {
    if (!h) return fail(h, KGPU_ERR_INVALID, "kgpu_upload_gpu_memory: NULL handle");
    std::lock_guard<std::mutex> g(h->mu);
    if (n != h->n_total || (n > 0 && !mem_mib)) return fail(h, KGPU_ERR_INVALID, "kgpu_upload_gpu_memory: n must equal kgpu_num_nodes");
    for (int64_t i = 0; i < n * 8; i++)
        if (mem_mib[i] < 0) return fail(h, KGPU_ERR_INVALID, "kgpu_upload_gpu_memory: negative memory at node %lld", (long long)(i / 8));
    int64_t off = 0;
    for (auto &s : h->shards) {
        if (s.n > 0) {
            KGPU_CUDA(h, cudaSetDevice(s.dev));
            KGPU_CUDA(h, cudaMemcpyAsync(s.d_mem, mem_mib + off * 8, (size_t)s.n * 32, cudaMemcpyHostToDevice, s.stream));
            KGPU_CUDA(h, cudaStreamSynchronize(s.stream));
        }
        off += s.n;
    }
    return KGPU_OK;
}

int kgpu_update_gpu_memory(kgpu_t *h, int64_t idx, const int32_t mem_mib[8]) {
    if (!h || !mem_mib) return fail(h, KGPU_ERR_INVALID, "kgpu_update_gpu_memory: NULL argument");
    std::lock_guard<std::mutex> g(h->mu);
    if (idx < 0 || idx >= h->n_total) return fail(h, KGPU_ERR_INVALID, "kgpu_update_gpu_memory: index %lld out of range", (long long)idx);
    for (int i = 0; i < 8; i++)
        if (mem_mib[i] < 0) return fail(h, KGPU_ERR_INVALID, "kgpu_update_gpu_memory: negative memory");
    int64_t local = 0;
    kgpu_shard *s = shard_of(h, idx, &local);
    KGPU_CUDA(h, cudaSetDevice(s->dev));
    KGPU_CUDA(h, cudaMemcpyAsync(s->d_mem + local * 8, mem_mib, 32, cudaMemcpyHostToDevice, s->stream));
    KGPU_CUDA(h, cudaStreamSynchronize(s->stream));
    return KGPU_OK;
}

int kgpu_update_node(kgpu_t *h, int64_t idx, const int32_t topo[64], int32_t free_mask) {
    if (!h || !topo) return fail(h, KGPU_ERR_INVALID, "kgpu_update_node: NULL argument");
    std::lock_guard<std::mutex> g(h->mu);
    if (idx < 0 || idx >= h->n_total) return fail(h, KGPU_ERR_INVALID, "kgpu_update_node: index %lld out of range", (long long)idx);
    int rc = validate_topo(h, topo, 1);
    if (rc != KGPU_OK) return rc;
    int64_t local = 0;
    kgpu_shard *s = shard_of(h, idx, &local);
    KGPU_CUDA(h, cudaSetDevice(s->dev));
    KGPU_CUDA(h, cudaMemcpyAsync(s->d_topo + local * 64, topo, 256, cudaMemcpyHostToDevice, s->stream));
    const int32_t li = (int32_t)local;
    return apply_node_updates(h, *s, &li, &free_mask, 1);      // new mask + this node's record (and fit row) only
}

int kgpu_set_free_masks(kgpu_t *h, const int64_t *idx, const int32_t *free_mask, int64_t n) {
    if (!h) return fail(h, KGPU_ERR_INVALID, "kgpu_set_free_masks: NULL handle");
    std::lock_guard<std::mutex> g(h->mu);
    if (n < 0 || (n > 0 && (!idx || !free_mask))) return fail(h, KGPU_ERR_INVALID, "kgpu_set_free_masks: bad arguments");
    for (int64_t i = 0; i < n; i++)
        if (idx[i] < 0 || idx[i] >= h->n_total)
            return fail(h, KGPU_ERR_INVALID, "kgpu_set_free_masks: index %lld out of range", (long long)idx[i]);
    // per shard: local indices, the LAST entry wins when a node is listed more than once
    int64_t off = 0;
    for (auto &s : h->shards) {
        std::vector<int32_t> li, lm;
        if (n == 1) {
            if (idx[0] >= off && idx[0] < off + s.n) { li.push_back((int32_t)(idx[0] - off)); lm.push_back(free_mask[0]); }
        } else {
            std::vector<std::pair<int32_t, int64_t>> ent;     // (local index, position in the call)
            for (int64_t i = 0; i < n; i++)
                if (idx[i] >= off && idx[i] < off + s.n) ent.emplace_back((int32_t)(idx[i] - off), i);
            std::sort(ent.begin(), ent.end());
            for (size_t e = 0; e < ent.size(); e++)
                if (e + 1 == ent.size() || ent[e + 1].first != ent[e].first) { li.push_back(ent[e].first); lm.push_back(free_mask[ent[e].second]); }
        }
        off += s.n;
        if (li.empty()) continue;
        const int rc = apply_node_updates(h, s, li.data(), lm.data(), (int64_t)li.size());
        if (rc != KGPU_OK) return rc;
    }
    return KGPU_OK;
}

int kgpu_set_free_mask(kgpu_t *h, int64_t idx, int32_t free_mask) {
    if (!h) return fail(h, KGPU_ERR_INVALID, "kgpu_set_free_mask: NULL handle");
    {
        std::lock_guard<std::mutex> g(h->mu);
        if (idx < 0 || idx >= h->n_total) return fail(h, KGPU_ERR_INVALID, "kgpu_set_free_mask: index %lld out of range", (long long)idx);
    }
    return kgpu_set_free_masks(h, &idx, &free_mask, 1);
}

int kgpu_remove_node(kgpu_t *h, int64_t idx) { return kgpu_set_free_mask(h, idx, 0); }

int64_t kgpu_num_nodes(kgpu_t *h) {
    if (!h) return 0;
    std::lock_guard<std::mutex> g(h->mu);
    return h->n_total;
}

int kgpu_score_batch(kgpu_t *h, const int32_t *pods, int64_t P, uint64_t *out_keys) {
    if (!h) return fail(h, KGPU_ERR_INVALID, "kgpu_score_batch: NULL handle");
    std::lock_guard<std::mutex> g(h->mu);
    if (P < 0 || (P > 0 && (!pods || !out_keys))) return fail(h, KGPU_ERR_INVALID, "kgpu_score_batch: bad arguments");
    if (P == 0) return KGPU_OK;
    const size_t G = h->shards.size();
    for (auto &s : h->shards) {
        int rc = reserve_pods(h, s, P);
        if (rc != KGPU_OK) return rc;
    }
    int has_mem = 0;
    for (int64_t p = 0; p < P && !has_mem; p++) has_mem = pods[4 * p + 3] > 0;
    // every device: pods H2D, K1 over its node shard (devices run concurrently)
    for (auto &s : h->shards) {
        KGPU_CUDA(h, cudaSetDevice(s.dev));
        KGPU_CUDA(h, cudaMemcpyAsync(s.d_pods, pods, (size_t)P * 16, cudaMemcpyHostToDevice, s.stream));
        KGPU_CUDA(h, cudaEventRecord(s.ev0, s.stream));
        int rc = launch_score(h, s, s.d_pods, P, s.d_keys, s.stream, has_mem);
        if (rc != KGPU_OK) return rc;
        KGPU_CUDA(h, cudaEventRecord(s.ev1, s.stream));
    }
    kgpu_shard &s0 = h->shards[0];
    if (G > 1) {
        // one all-gather of every shard's per-pod best over NVLink, then K2 on device 0
        std::vector<const void *> send(G);
        std::vector<void *> recv(G);
        std::vector<cudaStream_t> streams(G);
        for (size_t i = 0; i < G; i++) { send[i] = h->shards[i].d_keys; recv[i] = h->shards[i].d_gather; streams[i] = h->shards[i].stream; }
        std::string why;
        if (!h->multi->all_gather_u64(send, recv, (size_t)P, streams, &why))
            return fail(h, KGPU_ERR_COMM, "kgpu_score_batch: %s", why.c_str());
        KGPU_CUDA(h, cudaSetDevice(s0.dev));
        kgpu::reduce_shards<<<(unsigned)((P + 255) / 256), 256, 0, s0.stream>>>(s0.d_gather, (int)G, P, s0.d_keys);
        h->launches++;
        KGPU_CUDA(h, cudaGetLastError());
    }
    KGPU_CUDA(h, cudaSetDevice(s0.dev));
    KGPU_CUDA(h, cudaMemcpyAsync(out_keys, s0.d_keys, (size_t)P * 8, cudaMemcpyDeviceToHost, s0.stream));
    double worst = 0.0;
    for (auto &s : h->shards) {
        KGPU_CUDA(h, cudaSetDevice(s.dev));
        KGPU_CUDA(h, cudaStreamSynchronize(s.stream));
        float ms = 0.f;
        KGPU_CUDA(h, cudaEventElapsedTime(&ms, s.ev0, s.ev1));
        worst = std::max(worst, (double)ms);
    }
    h->last_kernel_ms = worst;
    return KGPU_OK;
}

namespace {
// A gang is ONE run of consecutive pods: the kernels only look at neighbours, so an id in two separate runs is refused.
int check_gang_runs(kgpu_ctx *h, const char *fn, const int32_t *gang, int64_t P) {
    std::unordered_set<int32_t> seen;
    for (int64_t p = 0; p < P; p++) {
        if (gang[p] == 0 || (p > 0 && gang[p - 1] == gang[p])) continue;
        if (!seen.insert(gang[p]).second)
            return fail(h, KGPU_ERR_INVALID, "%s: gang id %d appears in two separate runs (again at pod %lld)", fn, gang[p], (long long)p);
    }
    return KGPU_OK;
}
}  // namespace

int kgpu_place_batch(kgpu_t *h, const int32_t *pods, int64_t P, uint64_t *out_keys) {
    return kgpu_place_batch_ex(h, pods, P, out_keys, 0);
}

int kgpu_place_batch_ex(kgpu_t *h, const int32_t *pods, int64_t P, uint64_t *out_keys, int flags) {
    return kgpu_place_batch_gang(h, pods, nullptr, P, out_keys, flags);
}

int kgpu_place_batch_gang(kgpu_t *h, const int32_t *pods, const int32_t *gang, int64_t P, uint64_t *out_keys, int flags) {
    return kgpu_place_batch_gang_domain(h, pods, gang, nullptr, P, out_keys, flags);
}

namespace {
// gang_domain: every value 0, REQUIRED or PREFERRED, nonzero only on gang members, the same for all members of a gang,
// and a constrained gang small enough for the 32-bit cost sum of its trials.  fn names the entry point in the messages.
int check_gang_domain(kgpu_ctx *h, const char *fn, const int32_t *gang, const int32_t *gang_domain, int64_t P) {
    for (int64_t p = 0; p < P; p++) {
        const int32_t v = gang_domain[p];
        if (v != 0 && v != KGPU_GANG_DOMAIN_REQUIRED && v != KGPU_GANG_DOMAIN_PREFERRED)
            return fail(h, KGPU_ERR_INVALID, "%s: gang_domain[%lld] = %d is not 0, REQUIRED (1) or PREFERRED (2)", fn, (long long)p, v);
        if (v != 0 && (!gang || gang[p] == 0))
            return fail(h, KGPU_ERR_INVALID, "%s: gang_domain[%lld] = %d on a pod without a gang", fn, (long long)p, v);
        if (gang && p > 0 && gang[p] != 0 && gang[p] == gang[p - 1] && v != gang_domain[p - 1])
            return fail(h, KGPU_ERR_INVALID, "%s: the members of gang %d disagree on gang_domain (%d at pod %lld, %d at pod %lld)", fn,
                        gang[p], gang_domain[p - 1], (long long)(p - 1), v, (long long)p);
    }
    for (const kgpu::PlaceSegment &sg : kgpu::place_segments(gang, gang_domain, P))
        if (sg.mode != 0 && sg.end - sg.begin > kgpu::DOM_MAX_MEMBERS)
            return fail(h, KGPU_ERR_INVALID, "%s: gang %d has %lld members with a domain constraint, more than %lld", fn, gang[sg.begin],
                        (long long)(sg.end - sg.begin), (long long)kgpu::DOM_MAX_MEMBERS);
    return KGPU_OK;
}
}  // namespace

namespace {
// kgpu_upload_domains is the one-level case, with its own name and messages (flat: domain[i] rather than domain[l][i]).
int upload_domain_levels(kgpu_ctx *h, const char *fn, bool flat, const int32_t *domain, int levels, int64_t n) {
    if (!h) return fail(h, KGPU_ERR_INVALID, "%s: NULL handle", fn);
    std::lock_guard<std::mutex> g(h->mu);
    if (h->shards.size() != 1) return fail(h, KGPU_ERR_STATE, "%s: needs a single-device handle", fn);
    if (levels < 1 || levels > KGPU_MAX_DOMAIN_LEVELS)
        return fail(h, KGPU_ERR_INVALID, "%s: levels = %d is outside 1..%d", fn, levels, KGPU_MAX_DOMAIN_LEVELS);
    if (n != h->n_total || (n > 0 && !domain)) return fail(h, KGPU_ERR_INVALID, "%s: n must equal kgpu_num_nodes", fn);
    kgpu::DomainTable t;
    const kgpu::DomainTableError e = kgpu::domain_table(domain, levels, n, t);
    switch (e.kind) {
    case kgpu::DomainTableError::none: break;
    case kgpu::DomainTableError::out_of_range:
        if (flat)
            return fail(h, KGPU_ERR_INVALID, "%s: domain[%lld] = %d is neither -1 nor 0..%lld", fn, (long long)e.node, e.id,
                        (long long)(n - 1));
        return fail(h, KGPU_ERR_INVALID, "%s: domain[%d][%lld] = %d is neither -1 nor 0..%lld", fn, e.level, (long long)e.node, e.id,
                    (long long)(n - 1));
    case kgpu::DomainTableError::no_parent:
        return fail(h, KGPU_ERR_INVALID, "%s: level %d: node %lld is in domain %d but in no level-%d domain (-1)", fn, e.level,
                    (long long)e.node, e.id, e.level + 1);
    case kgpu::DomainTableError::split:
        return fail(h, KGPU_ERR_INVALID, "%s: level %d: domain %d is not nested: node %lld is in level-%d domain %d, node %lld in %d",
                    fn, e.level, e.id, (long long)e.other_node, e.level + 1, e.other, (long long)e.node, e.other2);
    }
    kgpu_shard &s = h->shards[0];
    KGPU_CUDA(h, cudaSetDevice(s.dev));
    KGPU_CUDA(h, s.d_dom_off.reserve((int64_t)t.off.size()));
    KGPU_CUDA(h, s.d_dom_chunk.reserve((int64_t)t.chunk.size()));
    KGPU_CUDA(h, s.d_chunk_begin.reserve((int64_t)t.chunk_begin.size()));
    KGPU_CUDA(h, cudaMemcpyAsync(s.d_dom_chunk, t.chunk.data(), t.chunk.size() * 4, cudaMemcpyHostToDevice, s.stream));
    KGPU_CUDA(h, cudaMemcpyAsync(s.d_chunk_begin, t.chunk_begin.data(), t.chunk_begin.size() * 4, cudaMemcpyHostToDevice, s.stream));
    KGPU_CUDA(h, s.d_dom_nodes.reserve(std::max<int64_t>(1, (int64_t)t.nodes.size())));
    KGPU_CUDA(h, cudaMemcpyAsync(s.d_dom_off, t.off.data(), t.off.size() * 4, cudaMemcpyHostToDevice, s.stream));
    if (!t.nodes.empty()) KGPU_CUDA(h, cudaMemcpyAsync(s.d_dom_nodes, t.nodes.data(), t.nodes.size() * 4, cudaMemcpyHostToDevice, s.stream));
    KGPU_CUDA(h, cudaStreamSynchronize(s.stream));
    s.n_dom = t.level[0].D;
    s.dom_levels = t.level;
    s.n_chunks = (int64_t)t.chunk_begin.size() - 1;
    return KGPU_OK;
}
}  // namespace

int kgpu_upload_domains(kgpu_t *h, const int32_t *domain, int64_t n) {
    return upload_domain_levels(h, "kgpu_upload_domains", true, domain, 1, n);
}

int kgpu_upload_domain_levels(kgpu_t *h, const int32_t *domain, int levels, int64_t n) {
    return upload_domain_levels(h, "kgpu_upload_domain_levels", false, domain, levels, n);
}

namespace {
// gang_level: within 0..levels-1 on constrained pods, 0 on the others, the same for all members of a gang.
int check_gang_level(kgpu_ctx *h, const char *fn, const int32_t *gang, const int32_t *gang_domain, const int32_t *gang_level,
                     int64_t P, int levels) {
    for (int64_t p = 0; p < P; p++) {
        const int32_t r = gang_level[p];
        if ((gang_domain == nullptr || gang_domain[p] == 0) && r != 0)
            return fail(h, KGPU_ERR_INVALID, "%s: gang_level[%lld] = %d on a pod without a domain constraint", fn, (long long)p, r);
        if (r < 0 || r >= levels)
            return fail(h, KGPU_ERR_INVALID, "%s: gang_level[%lld] = %d is outside 0..%d (the domain table has %d level%s)", fn,
                        (long long)p, r, levels - 1, levels, levels == 1 ? "" : "s");
        if (gang && p > 0 && gang[p] != 0 && gang[p] == gang[p - 1] && r != gang_level[p - 1])
            return fail(h, KGPU_ERR_INVALID, "%s: the members of gang %d disagree on gang_level (%d at pod %lld, %d at pod %lld)", fn,
                        gang[p], gang_level[p - 1], (long long)(p - 1), r, (long long)p);
    }
    return KGPU_OK;
}

// kgpu_place_batch_gang_levels under the name fn: kgpu_place_batch_gang_domain is gang_level == NULL, and its messages
// keep the names they have always had.
int place_batch_levels(kgpu_t *h, const char *fn, const int32_t *pods, const int32_t *gang, const int32_t *gang_domain,
                       const int32_t *gang_level, int64_t P, uint64_t *out_keys, int flags) {
    if (!h) return fail(h, KGPU_ERR_INVALID, "kgpu_place_batch: NULL handle");
    std::lock_guard<std::mutex> g(h->mu);
    if (h->shards.size() != 1) return fail(h, KGPU_ERR_STATE, "kgpu_place_batch: needs a single-device handle");
    if (P < 0 || (P > 0 && (!pods || !out_keys))) return fail(h, KGPU_ERR_INVALID, "kgpu_place_batch: bad arguments");
    if (P == 0) return KGPU_OK;
    if (gang) {
        const int rc = check_gang_runs(h, "kgpu_place_batch_gang", gang, P);
        if (rc != KGPU_OK) return rc;
    }
    if (gang_domain) {
        const int rc = check_gang_domain(h, fn, gang, gang_domain, P);
        if (rc != KGPU_OK) return rc;
    }
    if (gang_level) {
        const int rc = check_gang_level(h, fn, gang, gang_domain, gang_level, P, (int)h->shards[0].dom_levels.size());
        if (rc != KGPU_OK) return rc;
    }
    kgpu::PlaceViews views;
    if (!kgpu::place_views(pods, P, views))
        return fail(h, KGPU_ERR_INVALID, "kgpu_place_batch: more than %d distinct min_mem values in one batch", kgpu::PLACE_MAX_VIEWS - 1);
    kgpu_shard &s = h->shards[0];
    const int rc = reserve_pods(h, s, P);
    if (rc != KGPU_OK) return rc;
    if (gang) KGPU_CUDA(h, s.d_gang.reserve(P, pod_headroom(P)));
    KGPU_CUDA(h, cudaMemcpyAsync(s.d_pods, pods, (size_t)P * 16, cudaMemcpyHostToDevice, s.stream));
    if (gang) KGPU_CUDA(h, cudaMemcpyAsync(s.d_gang, gang, (size_t)P * 4, cudaMemcpyHostToDevice, s.stream));
    const bool dry = (flags & KGPU_PLACE_DRY_RUN) != 0;
    int32_t *d_free = s.d_free;
    if (dry && s.n > 0) {                  // place on a scratch copy of the masks: conflict-free proposals, nothing taken
        KGPU_CUDA(h, s.d_free_scratch.reserve(s.n));
        KGPU_CUDA(h, cudaMemcpyAsync(s.d_free_scratch, s.d_free, (size_t)s.n * 4, cudaMemcpyDeviceToDevice, s.stream));
        d_free = s.d_free_scratch;
    }
    if (s.n == 0) {
        KGPU_CUDA(h, cudaMemsetAsync(s.d_keys, 0xFF, (size_t)P * 8, s.stream));
    } else {
        const int64_t T = (s.n + kgpu::PLACE_TILE - 1) / kgpu::PLACE_TILE, Npad = T * kgpu::PLACE_TILE;
        KGPU_CUDA(h, s.d_nodebest.reserve(Npad * views.n * 9));
        KGPU_CUDA(h, s.d_tilebest.reserve(T * views.n * 9));
        KGPU_CUDA(h, s.d_half.reserve(Npad * kgpu::PLACE_HALF));
        kgpu::Weights W;
        memcpy(W.w, h->W, sizeof W.w);
        KGPU_CUDA(h, cudaEventRecord(s.ev0, s.stream));
        kgpu::place_init<<<dim3((unsigned)T, (unsigned)views.n), kgpu::PLACE_TILE, 0, s.stream>>>(
            reinterpret_cast<const int4 *>(s.d_topo.get()), d_free, s.d_mem, s.n, Npad, s.node_id_base, W, PC, views, s.d_nodebest,
            s.d_tilebest, T);
        kgpu::place_half_tables<<<(unsigned)std::min<int64_t>((s.n + 3) / 4, (int64_t)s.sm_count * 16), 128, 0, s.stream>>>(
            s.d_topo, s.n, W, s.d_half);
        h->launches += 2;
        if (!s.place_attr_done) {          // 72 KB of dynamic shared memory: opt in, once per device
            KGPU_CUDA(h, cudaFuncSetAttribute(kgpu::place_sequential<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kgpu::PLACE_DYN_SMEM));
            KGPU_CUDA(h, cudaFuncSetAttribute(kgpu::place_sequential<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kgpu::PLACE_DYN_SMEM));
            s.place_attr_done = true;
        }
        const std::vector<kgpu::PlaceSegment> segs = kgpu::place_segments(gang, gang_domain, P, gang_level);
        int64_t trials = 0;            // one best[] entry and one stamp per (step, level), one stamp per commit
        std::vector<int32_t> pairs;    // the (view, k) pairs of every step that climbs to a chunked level, step after step
        std::vector<int64_t> pair_at;
        for (const kgpu::PlaceSegment &sg : segs) {
            if (sg.mode == 0) continue;
            trials += sg.level + 1;
            pair_at.push_back((int64_t)pairs.size());
            bool chunked = false;
            for (int32_t l = 0; l <= sg.level; l++) chunked = chunked || kgpu::domain_level_chunked(s.dom_levels[(size_t)l]);
            if (chunked) kgpu::domain_pairs(pods, sg.begin, sg.end, views, pairs);
        }
        pair_at.push_back((int64_t)pairs.size());
        kgpu::DomainArgs da = {};
        if (trials > 0) {
            KGPU_CUDA(h, s.d_dom_mask.reserve(s.n));
            KGPU_CUDA(h, s.d_dom_stamp.reserve(s.n));
            KGPU_CUDA(h, s.d_dom_best.reserve(trials, pod_headroom(trials)));
            KGPU_CUDA(h, s.d_dom_off.reserve(1));
            KGPU_CUDA(h, cudaMemsetAsync(s.d_dom_stamp, 0, (size_t)s.n * 4, s.stream));
            KGPU_CUDA(h, cudaMemsetAsync(s.d_dom_best, 0xFF, (size_t)trials * 8, s.stream));
            da = kgpu::DomainArgs{d_free, s.d_mem, Npad, T, s.node_id_base, views, s.d_nodebest, s.d_tilebest, s.d_half,
                                  s.d_dom_off, s.d_dom_nodes, s.d_dom_mask, s.d_dom_stamp};
            if (!pairs.empty()) {
                KGPU_CUDA(h, s.d_dom_cmin.reserve(views.n * 9 * s.n_chunks));
                KGPU_CUDA(h, s.d_dom_cstamp.reserve(s.n_chunks));
                KGPU_CUDA(h, s.d_dom_pairs.reserve((int64_t)pairs.size(), pod_headroom((int64_t)pairs.size())));
                KGPU_CUDA(h, cudaMemsetAsync(s.d_dom_cstamp, 0, (size_t)s.n_chunks * 4, s.stream));
                KGPU_CUDA(h, cudaMemcpyAsync(s.d_dom_pairs, pairs.data(), pairs.size() * 4, cudaMemcpyHostToDevice, s.stream));
                da.dom_chunk = s.d_dom_chunk, da.chunk_begin = s.d_chunk_begin, da.cmin = s.d_dom_cmin, da.cstamp = s.d_dom_cstamp;
                da.chunks = s.n_chunks;
            }
        }
        const int4 *pods4 = reinterpret_cast<const int4 *>(s.d_pods.get());
        int64_t slot = 0, step = 0;
        uint32_t stamp = 0;
        for (const kgpu::PlaceSegment &sg : segs) {
            const int64_t p0 = sg.begin, np = sg.end - sg.begin;
            if (sg.mode != 0) {
                int32_t chunked_levels = 0;
                const int64_t npair = pair_at[(size_t)step + 1] - pair_at[(size_t)step];
                for (int32_t l = 0; l <= sg.level; l++) {
                    const kgpu::DomainLevel lv = s.dom_levels[(size_t)l];
                    const bool chunked = kgpu::domain_level_chunked(lv) && npair > 0;
                    if (chunked) {
                        kgpu::domain_chunk_min<<<dim3(kgpu::domain_trial_blocks(lv.C, (int64_t)s.sm_count * 8), (unsigned)npair),
                                                 kgpu::DOM_THREADS, 0, s.stream>>>(da, lv.chunk0, lv.C, s.d_dom_pairs + pair_at[(size_t)step],
                                                                                   s.d_dom_best + slot, l);
                        h->launches++;
                    }
                    chunked_levels |= chunked ? 1 << l : 0;
                    kgpu::domain_trial<<<kgpu::domain_trial_blocks(lv.D, (int64_t)s.sm_count * 8), kgpu::DOM_THREADS, 0, s.stream>>>(
                        da, pods4 + p0, np, lv.D, ++stamp, s.d_dom_best + slot, l, lv.base, chunked ? 1 : 0);
                }
                kgpu::domain_commit<<<1, kgpu::DOM_COMMIT_THREADS, 0, s.stream>>>(da, pods4 + p0, np, sg.mode, ++stamp,
                                                                                 s.d_dom_best + slot, s.d_keys + p0, sg.level + 1,
                                                                                 chunked_levels);
                slot += sg.level + 1;
                step++;
                h->launches += sg.level + 1;
            } else if (gang) {
                kgpu::place_sequential<true><<<1, kgpu::PLACE_THREADS, kgpu::PLACE_DYN_SMEM, s.stream>>>(
                    s.d_topo, d_free, s.d_mem, s.n, Npad, s.node_id_base, pods4 + p0, np, W, views, s.d_nodebest, s.d_tilebest, T,
                    s.d_half, s.d_keys + p0, s.d_gang + p0);
            } else {
                kgpu::place_sequential<false><<<1, kgpu::PLACE_THREADS, kgpu::PLACE_DYN_SMEM, s.stream>>>(
                    s.d_topo, d_free, s.d_mem, s.n, Npad, s.node_id_base, pods4 + p0, np, W, views, s.d_nodebest, s.d_tilebest, T,
                    s.d_half, s.d_keys + p0);
            }
            h->launches++;
        }
        if (!dry) {
            s.order_dirty = true;        // the free masks have changed on the device: re-sort + recompact lazily
            s.fit_valid = false;
        }
        KGPU_CUDA(h, cudaGetLastError());
        KGPU_CUDA(h, cudaEventRecord(s.ev1, s.stream));
    }
    KGPU_CUDA(h, cudaMemcpyAsync(out_keys, s.d_keys, (size_t)P * 8, cudaMemcpyDeviceToHost, s.stream));
    KGPU_CUDA(h, cudaStreamSynchronize(s.stream));
    if (s.n > 0) {
        float ms = 0.f;
        KGPU_CUDA(h, cudaEventElapsedTime(&ms, s.ev0, s.ev1));
        h->last_kernel_ms = ms;
    }
    return KGPU_OK;
}
}  // namespace

int kgpu_place_batch_gang_domain(kgpu_t *h, const int32_t *pods, const int32_t *gang, const int32_t *gang_domain, int64_t P,
                                 uint64_t *out_keys, int flags) {
    return place_batch_levels(h, "kgpu_place_batch_gang_domain", pods, gang, gang_domain, nullptr, P, out_keys, flags);
}

int kgpu_place_batch_gang_levels(kgpu_t *h, const int32_t *pods, const int32_t *gang, const int32_t *gang_domain,
                                 const int32_t *gang_level, int64_t P, uint64_t *out_keys, int flags) {
    return place_batch_levels(h, "kgpu_place_batch_gang_levels", pods, gang, gang_domain, gang_level, P, out_keys, flags);
}

namespace {
// Holder rows: every entry -1 or level << 3 | owner (level 0..15, owner 0..7), one level per owner within a row.
int validate_holders(kgpu_ctx *h, const char *fn, const int32_t *rows, int64_t n) {
    for (int64_t r = 0; r < n; r++) {
        int32_t level_of[8] = {-1, -1, -1, -1, -1, -1, -1, -1};
        for (int g = 0; g < 8; g++) {
            const int32_t e = rows[r * 8 + g];
            if (e == -1) continue;
            if (e < 0 || e > 127)
                return fail(h, KGPU_ERR_INVALID, "%s: row %lld GPU %d: entry %d is neither -1 nor level << 3 | owner with level 0..15",
                            fn, (long long)r, g, e);
            const int32_t o = e & 7, lv = e >> 3;
            if (level_of[o] >= 0 && level_of[o] != lv)
                return fail(h, KGPU_ERR_INVALID, "%s: row %lld: owner %d has levels %d and %d", fn, (long long)r, o, level_of[o], lv);
            level_of[o] = lv;
        }
    }
    return KGPU_OK;
}

// The holder table of shard s exists on the device (first use: allocated and set to all -1).
int ensure_holders(kgpu_ctx *h, kgpu_shard &s) {
    KGPU_CUDA(h, cudaSetDevice(s.dev));
    KGPU_CUDA(h, s.d_hold.reserve(8 * s.n));    // grows only with n, that is after kgpu_upload_nodes cleared has_hold
    if (!s.has_hold && s.n > 0) KGPU_CUDA(h, cudaMemsetAsync(s.d_hold, 0xFF, (size_t)s.n * 32, s.stream));
    s.has_hold = true;
    return KGPU_OK;
}

}  // namespace

int kgpu_upload_holders(kgpu_t *h, const int32_t *holders, int64_t n) {
    if (!h) return fail(h, KGPU_ERR_INVALID, "kgpu_upload_holders: NULL handle");
    std::lock_guard<std::mutex> g(h->mu);
    if (h->shards.size() != 1) return fail(h, KGPU_ERR_STATE, "kgpu_upload_holders: needs a single-device handle");
    if (n != h->n_total || (n > 0 && !holders)) return fail(h, KGPU_ERR_INVALID, "kgpu_upload_holders: n must equal kgpu_num_nodes");
    int rc = validate_holders(h, "kgpu_upload_holders", holders, n);
    if (rc != KGPU_OK) return rc;
    kgpu_shard &s = h->shards[0];
    rc = ensure_holders(h, s);
    if (rc != KGPU_OK) return rc;
    if (n > 0) KGPU_CUDA(h, cudaMemcpyAsync(s.d_hold, holders, (size_t)n * 32, cudaMemcpyHostToDevice, s.stream));
    KGPU_CUDA(h, cudaStreamSynchronize(s.stream));
    return KGPU_OK;
}

int kgpu_set_holders(kgpu_t *h, const int64_t *idx, const int32_t *holders, int64_t n) {
    if (!h) return fail(h, KGPU_ERR_INVALID, "kgpu_set_holders: NULL handle");
    std::lock_guard<std::mutex> g(h->mu);
    if (h->shards.size() != 1) return fail(h, KGPU_ERR_STATE, "kgpu_set_holders: needs a single-device handle");
    if (n < 0 || (n > 0 && (!idx || !holders))) return fail(h, KGPU_ERR_INVALID, "kgpu_set_holders: bad arguments");
    for (int64_t i = 0; i < n; i++)
        if (idx[i] < 0 || idx[i] >= h->n_total)
            return fail(h, KGPU_ERR_INVALID, "kgpu_set_holders: index %lld out of range", (long long)idx[i]);
    int rc = validate_holders(h, "kgpu_set_holders", holders, n);
    if (rc != KGPU_OK || n == 0) return rc;
    // the LAST row wins when a node is listed more than once; one staging buffer: [m] local indices | [m][8] rows
    std::vector<std::pair<int64_t, int64_t>> ent((size_t)n);
    for (int64_t i = 0; i < n; i++) ent[(size_t)i] = {idx[i], i};
    std::sort(ent.begin(), ent.end());
    std::vector<int64_t> pick;
    for (size_t e = 0; e < ent.size(); e++)
        if (e + 1 == ent.size() || ent[e + 1].first != ent[e].first) pick.push_back(ent[e].second);
    const int64_t m = (int64_t)pick.size();
    const int64_t rows_off = (m + 3) / 4 * 4;        // rows start 16-byte aligned
    std::vector<int32_t> stage((size_t)(rows_off + m * 8));
    for (int64_t j = 0; j < m; j++) {
        stage[(size_t)j] = (int32_t)idx[pick[(size_t)j]];
        memcpy(&stage[(size_t)(rows_off + j * 8)], holders + pick[(size_t)j] * 8, 32);
    }
    kgpu_shard &s = h->shards[0];
    rc = ensure_holders(h, s);
    if (rc != KGPU_OK) return rc;
    const int64_t half = (int64_t)stage.size() / 2 + 1;               // d_upd is sized as two lists of this length
    KGPU_CUDA(h, s.d_upd.reserve(2 * half, 2 * list_headroom(half)));
    KGPU_CUDA(h, cudaMemcpyAsync(s.d_upd, stage.data(), stage.size() * 4, cudaMemcpyHostToDevice, s.stream));
    kgpu::scatter_holders<<<(unsigned)((m + 255) / 256), 256, 0, s.stream>>>(
        s.d_upd, reinterpret_cast<const int4 *>(s.d_upd + rows_off), m, reinterpret_cast<int4 *>(s.d_hold.get()));
    h->launches++;
    KGPU_CUDA(h, cudaGetLastError());
    KGPU_CUDA(h, cudaStreamSynchronize(s.stream));
    return KGPU_OK;
}

int kgpu_preempt_batch(kgpu_t *h, const int32_t *pods, const int32_t *lvl, int64_t P, uint64_t *out_keys,
                       uint32_t *out_victims) {
    if (!h) return fail(h, KGPU_ERR_INVALID, "kgpu_preempt_batch: NULL handle");
    std::lock_guard<std::mutex> g(h->mu);
    if (h->shards.size() != 1) return fail(h, KGPU_ERR_STATE, "kgpu_preempt_batch: needs a single-device handle");
    if (P < 0 || (P > 0 && (!pods || !lvl || !out_keys || !out_victims)))
        return fail(h, KGPU_ERR_INVALID, "kgpu_preempt_batch: bad arguments");
    for (int64_t p = 0; p < P; p++)
        if (lvl[p] < 0 || lvl[p] > 15) return fail(h, KGPU_ERR_INVALID, "kgpu_preempt_batch: lvl[%lld] = %d outside 0..15", (long long)p, lvl[p]);
    if (P == 0) return KGPU_OK;
    if (P > 0x7FFFFFFFLL) return fail(h, KGPU_ERR_INVALID, "kgpu_preempt_batch: more than 2^31 pods");
    kgpu_shard &s = h->shards[0];
    int rc = reserve_pods(h, s, P);
    if (rc != KGPU_OK) return rc;
    const int64_t cap = pod_headroom(P);
    KGPU_CUDA(h, s.d_lvl.reserve(P, cap));
    KGPU_CUDA(h, s.d_pidx.reserve(P, cap));
    KGPU_CUDA(h, s.d_pkey.reserve(P, cap));
    KGPU_CUDA(h, s.d_victims.reserve(P, cap));
    KGPU_CUDA(h, s.d_pcnt.reserve(1));
    int has_mem = 0;
    for (int64_t p = 0; p < P && !has_mem; p++) has_mem = pods[4 * p + 3] > 0;
    KGPU_CUDA(h, cudaMemcpyAsync(s.d_pods, pods, (size_t)P * 16, cudaMemcpyHostToDevice, s.stream));
    KGPU_CUDA(h, cudaMemsetAsync(s.d_victims, 0, (size_t)P * 4, s.stream));
    KGPU_CUDA(h, cudaEventRecord(s.ev0, s.stream));
    // 1. the scoring path, unchanged: every pod that fits without eviction keeps its key (victims 0)
    rc = launch_score(h, s, s.d_pods, P, s.d_keys, s.stream, has_mem);
    if (rc != KGPU_OK) return rc;
    if (s.has_hold && s.n > 0) {
        // 2. the NO_FIT pods that may evict, compacted on the device; 3. K4 over them only
        const int4 *pods4 = reinterpret_cast<const int4 *>(s.d_pods.get());
        KGPU_CUDA(h, cudaMemcpyAsync(s.d_lvl, lvl, (size_t)P * 4, cudaMemcpyHostToDevice, s.stream));
        KGPU_CUDA(h, cudaMemsetAsync(s.d_pcnt, 0, sizeof(int), s.stream));
        KGPU_CUDA(h, cudaMemsetAsync(s.d_pkey, 0xFF, (size_t)P * 8, s.stream));
        const unsigned pb = (unsigned)((P + 255) / 256);
        kgpu::preempt_compact<<<pb, 256, 0, s.stream>>>(pods4, s.d_lvl, s.d_keys, P, s.d_pidx, s.d_pcnt);
        kgpu::Weights W;
        memcpy(W.w, h->W, sizeof W.w);
        // the compacted count stays on the device: size the grid from P (blocks beyond the count exit at once) for
        // about 8 waves of resident blocks
        const int64_t tiles = (s.n + kgpu::PRE_THREADS - 1) / kgpu::PRE_THREADS;
        if (tiles > 0x7FFFFFFFLL) return fail(h, KGPU_ERR_INVALID, "kgpu_preempt_batch: too many nodes for one launch");
        int64_t splits = std::max<int64_t>(1, (8 * (int64_t)s.sm_count * 4 + tiles - 1) / tiles);
        splits = std::min<int64_t>({splits, (P + kgpu::PRE_CHUNK - 1) / kgpu::PRE_CHUNK, 65535});
        kgpu::preempt_lane_per_node<<<dim3((unsigned)tiles, (unsigned)splits), kgpu::PRE_THREADS, 0, s.stream>>>(
            reinterpret_cast<const int4 *>(s.d_topo.get()), s.d_free, reinterpret_cast<const int4 *>(s.d_mem.get()),
            reinterpret_cast<const int4 *>(s.d_hold.get()), s.n, pods4, s.d_lvl, s.d_pidx, s.d_pcnt, W, PC, s.d_pkey);
        kgpu::preempt_finalize<<<pb, 256, 0, s.stream>>>(s.d_pkey, s.d_pidx, s.d_pcnt, s.d_free, s.d_hold, s.node_id_base,
                                                         s.d_keys, s.d_victims);
        h->launches += 3;
        KGPU_CUDA(h, cudaGetLastError());
    }
    KGPU_CUDA(h, cudaEventRecord(s.ev1, s.stream));
    KGPU_CUDA(h, cudaMemcpyAsync(out_keys, s.d_keys, (size_t)P * 8, cudaMemcpyDeviceToHost, s.stream));
    KGPU_CUDA(h, cudaMemcpyAsync(out_victims, s.d_victims, (size_t)P * 4, cudaMemcpyDeviceToHost, s.stream));
    KGPU_CUDA(h, cudaStreamSynchronize(s.stream));
    float ms = 0.f;
    KGPU_CUDA(h, cudaEventElapsedTime(&ms, s.ev0, s.ev1));
    h->last_kernel_ms = ms;
    return KGPU_OK;
}

namespace {
// kgpu_preempt_plan[_gang]: the batch's checks and its columns (launch_plan.h)
int plan_columns(kgpu_ctx *h, const char *fn, const int32_t *pods, const int32_t *lvl, int64_t P, std::vector<int4> &cols,
                 std::vector<int32_t> &pcol) {
    for (int64_t p = 0; p < P; p++)
        if (lvl[p] < 0 || lvl[p] > 15) return fail(h, KGPU_ERR_INVALID, "%s: lvl[%lld] = %d outside 0..15", fn, (long long)p, lvl[p]);
    if (P > 0x7FFFFFFFLL) return fail(h, KGPU_ERR_INVALID, "%s: more than 2^31 pods", fn);
    switch (kgpu::plan_columns(pods, lvl, P, cols, pcol)) {
        case kgpu::PlanColumns::too_many_min_mem:
            return fail(h, KGPU_ERR_INVALID, "%s: more than %d distinct min_mem values in one batch", fn, kgpu::PLACE_MAX_VIEWS - 1);
        case kgpu::PlanColumns::too_many_views:
            return fail(h, KGPU_ERR_INVALID, "%s: more than 32 distinct (level > 0, min_mem) pairs in one batch", fn);
        case kgpu::PlanColumns::ok:
            break;
    }
    if (h->shards[0].n > 0x7FFFFFFFLL) return fail(h, KGPU_ERR_INVALID, "%s: too many nodes for the key's node field", fn);
    return KGPU_OK;
}

// The plan's kernels on the working state (F, H), once the batch is on the device (d_pods, d_plan_pcol and, with gangs,
// d_gang and d_plan_pre), then the results back to the host.  segs (launch_plan.h: place_segments) cut the batch: each
// range without a constrained gang is one plan_sequential (gang_plan_sequential with gangs) launch on its pods, each
// constrained gang one domain step, domain_plan_trial + domain_plan_commit.  The handle's masks and holder table are
// never written.
int plan_launch(kgpu_ctx *h, kgpu_shard &s, int64_t P, const std::vector<int4> &cols, bool gang,
                const std::vector<kgpu::PlaceSegment> &segs, uint64_t *out_keys, uint32_t *out_victims) {
    const int ncol = (int)cols.size();
    KGPU_CUDA(h, cudaEventRecord(s.ev0, s.stream));
    if (s.n == 0) {
        KGPU_CUDA(h, cudaMemsetAsync(s.d_keys, 0xFF, (size_t)P * 8, s.stream));
        KGPU_CUDA(h, cudaMemsetAsync(s.d_victims, 0, (size_t)P * 4, s.stream));
    } else {
        const int64_t T = (s.n + kgpu::PLAN_TILE - 1) / kgpu::PLAN_TILE, Npad = T * kgpu::PLAN_TILE;
        KGPU_CUDA(h, s.d_plan_free.reserve(s.n));
        KGPU_CUDA(h, s.d_plan_hold.reserve(8 * s.n));
        KGPU_CUDA(h, cudaMemcpyAsync(s.d_plan_free, s.d_free, (size_t)s.n * 4, cudaMemcpyDeviceToDevice, s.stream));
        if (s.has_hold) KGPU_CUDA(h, cudaMemcpyAsync(s.d_plan_hold, s.d_hold, (size_t)s.n * 32, cudaMemcpyDeviceToDevice, s.stream));
        else KGPU_CUDA(h, cudaMemsetAsync(s.d_plan_hold, 0xFF, (size_t)s.n * 32, s.stream));
        kgpu::Weights W;
        memcpy(W.w, h->W, sizeof W.w);
        if (ncol > 0) {
            KGPU_CUDA(h, s.d_plan_cols.reserve(ncol));
            KGPU_CUDA(h, s.d_plan_nodekey.reserve(ncol * Npad));
            KGPU_CUDA(h, s.d_plan_tilekey.reserve(ncol * T));
            KGPU_CUDA(h, cudaMemcpyAsync(s.d_plan_cols, cols.data(), (size_t)ncol * 16, cudaMemcpyHostToDevice, s.stream));
            const unsigned groups = (unsigned)((ncol + kgpu::PLAN_INIT_COLS - 1) / kgpu::PLAN_INIT_COLS);
            kgpu::plan_init<<<dim3((unsigned)T, groups), kgpu::PLAN_TILE, 0, s.stream>>>(
                reinterpret_cast<const int4 *>(s.d_topo.get()), s.d_plan_free, reinterpret_cast<const int4 *>(s.d_mem.get()),
                reinterpret_cast<const int4 *>(s.d_plan_hold.get()), s.n, Npad, T, s.d_plan_cols, ncol, W, PC, s.d_plan_nodekey,
                s.d_plan_tilekey);
            h->launches++;
        }
        const int64_t steps = std::count_if(segs.begin(), segs.end(), [](const kgpu::PlaceSegment &sg) { return sg.mode != 0; });
        kgpu::PlanDomainArgs da = {};
        if (steps > 0) {               // the trials' scratch: stamps 2 i + 1 (trials of step i) and 2 i + 2 (its commit)
            KGPU_CUDA(h, s.d_dom_mask.reserve(s.n));
            KGPU_CUDA(h, s.d_dom_hold.reserve(s.n));
            KGPU_CUDA(h, s.d_dom_stamp.reserve(s.n));
            KGPU_CUDA(h, s.d_dom_score.reserve(std::max<int64_t>(1, s.n_dom)));
            if (s.n_dom == 0) KGPU_CUDA(h, s.d_dom_off.reserve(1));
            KGPU_CUDA(h, cudaMemsetAsync(s.d_dom_stamp, 0, (size_t)s.n * 4, s.stream));
            da = kgpu::PlanDomainArgs{reinterpret_cast<const int4 *>(s.d_topo.get()), s.d_plan_free,
                                      reinterpret_cast<const int4 *>(s.d_mem.get()), s.d_plan_hold, s.n, Npad, T, s.node_id_base,
                                      s.d_plan_cols, ncol, s.d_plan_nodekey, s.d_plan_tilekey, s.d_dom_off, s.d_dom_nodes,
                                      s.d_dom_mask, s.d_dom_hold, s.d_dom_stamp};
        }
        const int4 *pods4 = reinterpret_cast<const int4 *>(s.d_pods.get());
        int64_t step = 0;
        for (const kgpu::PlaceSegment &sg : segs) {
            const int64_t p0 = sg.begin, np = sg.end - sg.begin;
            if (sg.mode != 0) {
                const uint32_t stamp = (uint32_t)(2 * step + 1);
                kgpu::domain_plan_trial<<<kgpu::domain_trial_blocks(s.n_dom, (int64_t)s.sm_count * 8), kgpu::DOM_THREADS, 0, s.stream>>>(
                    da, W, PC, pods4 + p0, s.d_plan_pcol + p0, np, s.n_dom, stamp, s.d_dom_score);
                kgpu::domain_plan_commit<<<1, kgpu::PLAN_THREADS, 0, s.stream>>>(
                    da, W, PC, pods4 + p0, s.d_plan_pcol + p0, s.d_gang + p0, np, sg.mode, s.n_dom, stamp + 1, s.d_dom_score,
                    s.d_keys + p0, s.d_victims + p0, s.d_plan_pre + p0);
                step++;
            } else if (gang) {
                kgpu::gang_plan_sequential<<<1, kgpu::PLAN_THREADS, 0, s.stream>>>(
                    reinterpret_cast<const int4 *>(s.d_topo.get()), s.d_plan_free, reinterpret_cast<const int4 *>(s.d_mem.get()),
                    s.d_plan_hold, s.n, Npad, T, s.node_id_base, pods4 + p0, s.d_plan_pcol + p0, np, s.d_plan_cols, ncol, W, PC,
                    s.d_plan_nodekey, s.d_plan_tilekey, s.d_keys + p0, s.d_victims + p0, s.d_gang + p0, s.d_plan_pre + p0);
            } else {
                kgpu::plan_sequential<<<1, kgpu::PLAN_THREADS, 0, s.stream>>>(
                    reinterpret_cast<const int4 *>(s.d_topo.get()), s.d_plan_free, reinterpret_cast<const int4 *>(s.d_mem.get()),
                    s.d_plan_hold, s.n, Npad, T, s.node_id_base, pods4 + p0, s.d_plan_pcol + p0, np, s.d_plan_cols, ncol, W, PC,
                    s.d_plan_nodekey, s.d_plan_tilekey, s.d_keys + p0, s.d_victims + p0);
            }
            h->launches += sg.mode != 0 ? 2 : 1;
        }
        KGPU_CUDA(h, cudaGetLastError());
    }
    KGPU_CUDA(h, cudaEventRecord(s.ev1, s.stream));
    KGPU_CUDA(h, cudaMemcpyAsync(out_keys, s.d_keys, (size_t)P * 8, cudaMemcpyDeviceToHost, s.stream));
    KGPU_CUDA(h, cudaMemcpyAsync(out_victims, s.d_victims, (size_t)P * 4, cudaMemcpyDeviceToHost, s.stream));
    KGPU_CUDA(h, cudaStreamSynchronize(s.stream));
    float ms = 0.f;
    KGPU_CUDA(h, cudaEventElapsedTime(&ms, s.ev0, s.ev1));
    h->last_kernel_ms = ms;
    return KGPU_OK;
}
}  // namespace

int kgpu_preempt_plan(kgpu_t *h, const int32_t *pods, const int32_t *lvl, int64_t P, uint64_t *out_keys,
                      uint32_t *out_victims) {
    if (!h) return fail(h, KGPU_ERR_INVALID, "kgpu_preempt_plan: NULL handle");
    std::lock_guard<std::mutex> g(h->mu);
    if (h->shards.size() != 1) return fail(h, KGPU_ERR_STATE, "kgpu_preempt_plan: needs a single-device handle");
    if (P < 0 || (P > 0 && (!pods || !lvl || !out_keys || !out_victims)))
        return fail(h, KGPU_ERR_INVALID, "kgpu_preempt_plan: bad arguments");
    if (P == 0) return KGPU_OK;
    std::vector<int4> cols;
    std::vector<int32_t> pcol;
    int rc = plan_columns(h, "kgpu_preempt_plan", pods, lvl, P, cols, pcol);
    if (rc != KGPU_OK) return rc;
    kgpu_shard &s = h->shards[0];
    rc = reserve_pods(h, s, P);
    if (rc != KGPU_OK) return rc;
    const int64_t cap = pod_headroom(P);
    KGPU_CUDA(h, s.d_victims.reserve(P, cap));
    KGPU_CUDA(h, s.d_plan_pcol.reserve(P, cap));
    KGPU_CUDA(h, cudaMemcpyAsync(s.d_pods, pods, (size_t)P * 16, cudaMemcpyHostToDevice, s.stream));
    KGPU_CUDA(h, cudaMemcpyAsync(s.d_plan_pcol, pcol.data(), (size_t)P * 4, cudaMemcpyHostToDevice, s.stream));
    return plan_launch(h, s, P, cols, false, kgpu::place_segments(nullptr, nullptr, P), out_keys, out_victims);
}

int kgpu_preempt_plan_gang(kgpu_t *h, const int32_t *pods, const int32_t *lvl, const int32_t *gang, int64_t P,
                           uint64_t *out_keys, uint32_t *out_victims) {
    if (!gang) return kgpu_preempt_plan(h, pods, lvl, P, out_keys, out_victims);
    if (!h) return fail(h, KGPU_ERR_INVALID, "kgpu_preempt_plan_gang: NULL handle");
    std::lock_guard<std::mutex> g(h->mu);
    if (h->shards.size() != 1) return fail(h, KGPU_ERR_STATE, "kgpu_preempt_plan_gang: needs a single-device handle");
    if (P < 0 || (P > 0 && (!pods || !lvl || !out_keys || !out_victims)))
        return fail(h, KGPU_ERR_INVALID, "kgpu_preempt_plan_gang: bad arguments");
    if (P == 0) return KGPU_OK;
    int rc = check_gang_runs(h, "kgpu_preempt_plan_gang", gang, P);
    if (rc != KGPU_OK) return rc;
    std::vector<int4> cols;
    std::vector<int32_t> pcol;
    rc = plan_columns(h, "kgpu_preempt_plan_gang", pods, lvl, P, cols, pcol);
    if (rc != KGPU_OK) return rc;
    kgpu_shard &s = h->shards[0];
    rc = reserve_pods(h, s, P);
    if (rc != KGPU_OK) return rc;
    const int64_t cap = pod_headroom(P);
    KGPU_CUDA(h, s.d_victims.reserve(P, cap));
    KGPU_CUDA(h, s.d_plan_pcol.reserve(P, cap));
    KGPU_CUDA(h, s.d_gang.reserve(P, cap));
    KGPU_CUDA(h, s.d_plan_pre.reserve(P, cap));
    KGPU_CUDA(h, cudaMemcpyAsync(s.d_pods, pods, (size_t)P * 16, cudaMemcpyHostToDevice, s.stream));
    KGPU_CUDA(h, cudaMemcpyAsync(s.d_plan_pcol, pcol.data(), (size_t)P * 4, cudaMemcpyHostToDevice, s.stream));
    KGPU_CUDA(h, cudaMemcpyAsync(s.d_gang, gang, (size_t)P * 4, cudaMemcpyHostToDevice, s.stream));
    return plan_launch(h, s, P, cols, true, kgpu::place_segments(gang, nullptr, P), out_keys, out_victims);
}

int kgpu_preempt_plan_gang_domain(kgpu_t *h, const int32_t *pods, const int32_t *lvl, const int32_t *gang,
                                  const int32_t *gang_domain, int64_t P, uint64_t *out_keys, uint32_t *out_victims) {
    const char *fn = "kgpu_preempt_plan_gang_domain";
    if (!h) return fail(h, KGPU_ERR_INVALID, "%s: NULL handle", fn);
    std::lock_guard<std::mutex> g(h->mu);
    if (h->shards.size() != 1) return fail(h, KGPU_ERR_STATE, "%s: needs a single-device handle", fn);
    if (P < 0 || (P > 0 && (!pods || !lvl || !out_keys || !out_victims))) return fail(h, KGPU_ERR_INVALID, "%s: bad arguments", fn);
    if (P == 0) return KGPU_OK;
    int rc = gang ? check_gang_runs(h, fn, gang, P) : KGPU_OK;
    if (rc != KGPU_OK) return rc;
    if (gang_domain) {
        rc = check_gang_domain(h, fn, gang, gang_domain, P);
        if (rc != KGPU_OK) return rc;
    }
    std::vector<int4> cols;
    std::vector<int32_t> pcol;
    rc = plan_columns(h, fn, pods, lvl, P, cols, pcol);
    if (rc != KGPU_OK) return rc;
    kgpu_shard &s = h->shards[0];
    rc = reserve_pods(h, s, P);
    if (rc != KGPU_OK) return rc;
    const int64_t cap = pod_headroom(P);
    KGPU_CUDA(h, s.d_victims.reserve(P, cap));
    KGPU_CUDA(h, s.d_plan_pcol.reserve(P, cap));
    KGPU_CUDA(h, cudaMemcpyAsync(s.d_pods, pods, (size_t)P * 16, cudaMemcpyHostToDevice, s.stream));
    KGPU_CUDA(h, cudaMemcpyAsync(s.d_plan_pcol, pcol.data(), (size_t)P * 4, cudaMemcpyHostToDevice, s.stream));
    if (gang) {
        KGPU_CUDA(h, s.d_gang.reserve(P, cap));
        KGPU_CUDA(h, s.d_plan_pre.reserve(P, cap));
        KGPU_CUDA(h, cudaMemcpyAsync(s.d_gang, gang, (size_t)P * 4, cudaMemcpyHostToDevice, s.stream));
    }
    return plan_launch(h, s, P, cols, gang != nullptr, kgpu::place_segments(gang, gang_domain, P), out_keys, out_victims);
}

int kgpu_get_free_masks(kgpu_t *h, int32_t *out_free_mask, int64_t n) {
    if (!h) return fail(h, KGPU_ERR_INVALID, "kgpu_get_free_masks: NULL handle");
    std::lock_guard<std::mutex> g(h->mu);
    if (n != h->n_total || (n > 0 && !out_free_mask)) return fail(h, KGPU_ERR_INVALID, "kgpu_get_free_masks: n must equal kgpu_num_nodes");
    int64_t off = 0;
    for (auto &s : h->shards) {
        if (s.n > 0) {
            KGPU_CUDA(h, cudaSetDevice(s.dev));
            KGPU_CUDA(h, cudaMemcpyAsync(out_free_mask + off, s.d_free, (size_t)s.n * 4, cudaMemcpyDeviceToHost, s.stream));
            KGPU_CUDA(h, cudaStreamSynchronize(s.stream));
        }
        off += s.n;
    }
    return KGPU_OK;
}

int kgpu_build_fit_table(kgpu_t *h) {
    if (!h) return fail(h, KGPU_ERR_INVALID, "kgpu_build_fit_table: NULL handle");
    std::lock_guard<std::mutex> g(h->mu);
    for (auto &s : h->shards) {
        const int rc = build_fit_table(h, s);
        if (rc != KGPU_OK) return rc;
    }
    return KGPU_OK;
}

int kgpu_fit_lookup(kgpu_t *h, int64_t node_idx, int32_t k, uint32_t *out_node_key) {
    if (!h || !out_node_key) return fail(h, KGPU_ERR_INVALID, "kgpu_fit_lookup: NULL argument");
    std::lock_guard<std::mutex> g(h->mu);
    if (node_idx < 0 || node_idx >= h->n_total) return fail(h, KGPU_ERR_INVALID, "kgpu_fit_lookup: node index %lld out of range", (long long)node_idx);
    int64_t local = 0;
    kgpu_shard *s = shard_of(h, node_idx, &local);
    if (!s->fit_valid) {                          // built lazily, kept current by the state-change calls
        const int rc = build_fit_table(h, *s);
        if (rc != KGPU_OK) return rc;
    }
    *out_node_key = (k < 0 || k > 8) ? UINT32_MAX : s->h_fit[(int64_t)k * s->n + local];
    return KGPU_OK;
}

int kgpu_score_pairs(kgpu_t *h, const int64_t *node_idx, const int32_t *k, const int32_t *min_mem_mib, int64_t n,
                     uint32_t *out_node_keys) {
    if (!h) return fail(h, KGPU_ERR_INVALID, "kgpu_score_pairs: NULL handle");
    std::lock_guard<std::mutex> g(h->mu);
    if (n < 0 || (n > 0 && (!node_idx || !k || !out_node_keys))) return fail(h, KGPU_ERR_INVALID, "kgpu_score_pairs: bad arguments");
    for (int64_t i = 0; i < n; i++)
        if (node_idx[i] < 0 || node_idx[i] >= h->n_total)
            return fail(h, KGPU_ERR_INVALID, "kgpu_score_pairs: node index %lld out of range", (long long)node_idx[i]);
    // Pairs without a memory requirement are answered from the (node, k) fit table's host copy: no launch,
    // no copy per call (PodFitsDevice is called once per (node, pod) by the core: gpu_scheduler.go:34-44).
    // The others go to the device in one packed copy, routed to the shard that holds their node.
    kgpu::Weights W;
    memcpy(W.w, h->W, sizeof W.w);
    int64_t off = 0;
    for (auto &s : h->shards) {
        std::vector<int4> q;
        std::vector<int64_t> pos;
        for (int64_t i = 0; i < n; i++) {
            if (node_idx[i] < off || node_idx[i] >= off + s.n) continue;
            const int64_t local = node_idx[i] - off;
            if (!min_mem_mib || min_mem_mib[i] <= 0) {
                if (!s.fit_valid) {
                    const int rc = build_fit_table(h, s);
                    if (rc != KGPU_OK) return rc;
                }
                out_node_keys[i] = (k[i] < 0 || k[i] > 8) ? UINT32_MAX : s.h_fit[(int64_t)k[i] * s.n + local];
            } else {
                q.push_back(make_int4((int)(local & 0xFFFFFFFFLL), (int)(local >> 32), k[i], min_mem_mib[i]));
                pos.push_back(i);
            }
        }
        off += s.n;
        if (q.empty()) continue;
        const int64_t m = (int64_t)q.size();
        KGPU_CUDA(h, cudaSetDevice(s.dev));
        KGPU_CUDA(h, s.d_query.reserve(m, list_headroom(m)));
        KGPU_CUDA(h, s.d_qout.reserve(m, list_headroom(m)));
        KGPU_CUDA(h, cudaMemcpyAsync(s.d_query, q.data(), (size_t)m * 16, cudaMemcpyHostToDevice, s.stream));
        kgpu::score_pair_list<<<(unsigned)((m + 127) / 128), 128, 0, s.stream>>>(
            reinterpret_cast<const int4 *>(s.d_topo.get()), s.d_free, s.d_mem, s.n, s.d_query, m, W, PC, s.d_qout);
        h->launches++;
        KGPU_CUDA(h, cudaGetLastError());
        std::vector<uint32_t> res((size_t)m);
        KGPU_CUDA(h, cudaMemcpyAsync(res.data(), s.d_qout, (size_t)m * 4, cudaMemcpyDeviceToHost, s.stream));
        KGPU_CUDA(h, cudaStreamSynchronize(s.stream));
        for (int64_t j = 0; j < m; j++) out_node_keys[pos[(size_t)j]] = res[(size_t)j];
    }
    return KGPU_OK;
}

int kgpu_score_batch_device(kgpu_t *h, const int32_t *d_pods, int64_t P, uint64_t *d_keys, void *stream) {
    if (!h) return fail(h, KGPU_ERR_INVALID, "kgpu_score_batch_device: NULL handle");
    std::lock_guard<std::mutex> g(h->mu);
    if (h->shards.size() != 1) return fail(h, KGPU_ERR_STATE, "kgpu_score_batch_device: needs a single-device handle");
    if (P < 0 || (P > 0 && (!d_pods || !d_keys))) return fail(h, KGPU_ERR_INVALID, "kgpu_score_batch_device: bad arguments");
    kgpu_shard &s = h->shards[0];
    return launch_score(h, s, d_pods, P, reinterpret_cast<unsigned long long *>(d_keys), (cudaStream_t)stream, -1);
}

int kgpu_score_batch_device_ex(kgpu_t *h, const int32_t *d_pods, int64_t P, uint64_t *d_keys, void *stream, int batch_flags) {
    if (!h) return fail(h, KGPU_ERR_INVALID, "kgpu_score_batch_device_ex: NULL handle");
    std::lock_guard<std::mutex> g(h->mu);
    if (h->shards.size() != 1) return fail(h, KGPU_ERR_STATE, "kgpu_score_batch_device_ex: needs a single-device handle");
    if (P < 0 || (P > 0 && (!d_pods || !d_keys))) return fail(h, KGPU_ERR_INVALID, "kgpu_score_batch_device_ex: bad arguments");
    kgpu_shard &s = h->shards[0];
    return launch_score(h, s, d_pods, P, reinterpret_cast<unsigned long long *>(d_keys), (cudaStream_t)stream,
                        (batch_flags & KGPU_BATCH_NO_MIN_MEM) ? 0 : -1);
}

namespace {
// one allocation per rank, mapped by every peer: slots[2][world][max_pods] uint64 | flags[PEER_MAX_WORLD] uint32 | ticket | error
size_t xch_slot_bytes(int world, int64_t max_pods) { return (size_t)2 * world * max_pods * 8; }
size_t xch_bytes(int world, int64_t max_pods) { return xch_slot_bytes(world, max_pods) + kgpu::PEER_MAX_WORLD * 4 + 16; }
unsigned long long *xch_slots(void *base, int world, int64_t max_pods, int buf) {
    return reinterpret_cast<unsigned long long *>(base) + (int64_t)buf * world * max_pods;
}
uint32_t *xch_flags(void *base, int world, int64_t max_pods) {
    return reinterpret_cast<uint32_t *>(reinterpret_cast<char *>(base) + xch_slot_bytes(world, max_pods));
}
}  // namespace

int kgpu_exchange_init(kgpu_t *h, int world, int rank, int64_t max_pods, unsigned char *out_handle) {
    if (!h) return fail(h, KGPU_ERR_INVALID, "kgpu_exchange_init: NULL handle");
    std::lock_guard<std::mutex> g(h->mu);
    static_assert(sizeof(cudaIpcMemHandle_t) == KGPU_IPC_HANDLE_BYTES, "IPC handle size");
    if (h->shards.size() != 1) return fail(h, KGPU_ERR_STATE, "kgpu_exchange_init: needs a single-device handle");
    if (world < 1 || world > kgpu::PEER_MAX_WORLD || rank < 0 || rank >= world || max_pods < 1 || !out_handle)
        return fail(h, KGPU_ERR_INVALID, "kgpu_exchange_init: bad arguments (world <= %d)", kgpu::PEER_MAX_WORLD);
    if (h->xch.base) return fail(h, KGPU_ERR_STATE, "kgpu_exchange_init: already initialised");
    kgpu_shard &s = h->shards[0];
    KGPU_CUDA(h, cudaSetDevice(s.dev));
    KGPU_CUDA(h, h->xch.base.reserve((int64_t)xch_bytes(world, max_pods)));
    KGPU_CUDA(h, h->xch.local.reserve(max_pods));
    KGPU_CUDA(h, h->xch.final_keys.reserve(2 * max_pods));
    KGPU_CUDA(h, cudaMemset(h->xch.base, 0xFF, xch_slot_bytes(world, max_pods)));
    KGPU_CUDA(h, cudaMemset(h->xch.local, 0xFF, (size_t)max_pods * 8));                                   // the exchange kernel keeps it that way
    KGPU_CUDA(h, cudaMemset(xch_flags(h->xch.base, world, max_pods), 0, kgpu::PEER_MAX_WORLD * 4 + 16));  // flags, ticket, error
    KGPU_CUDA(h, cudaDeviceSynchronize());
    cudaIpcMemHandle_t ipc;
    KGPU_CUDA(h, cudaIpcGetMemHandle(&ipc, h->xch.base));
    memcpy(out_handle, &ipc, sizeof ipc);
    h->xch.world = world; h->xch.rank = rank; h->xch.max_pods = max_pods; h->xch.epoch = 0; h->xch.connected = false;
    return KGPU_OK;
}

int kgpu_exchange_connect(kgpu_t *h, const unsigned char *handles) {
    if (!h) return fail(h, KGPU_ERR_INVALID, "kgpu_exchange_connect: NULL handle");
    std::lock_guard<std::mutex> g(h->mu);
    if (!h->xch.base) return fail(h, KGPU_ERR_STATE, "kgpu_exchange_connect: call kgpu_exchange_init first");
    if (!handles) return fail(h, KGPU_ERR_INVALID, "kgpu_exchange_connect: NULL handles");
    if (h->xch.connected) return fail(h, KGPU_ERR_STATE, "kgpu_exchange_connect: already connected");
    KGPU_CUDA(h, cudaSetDevice(h->shards[0].dev));
    for (int r = 0; r < h->xch.world; r++) {
        if (r == h->xch.rank) { h->xch.peer_base[r] = h->xch.base; continue; }
        cudaIpcMemHandle_t ipc;
        memcpy(&ipc, handles + (size_t)r * KGPU_IPC_HANDLE_BYTES, sizeof ipc);
        KGPU_CUDA(h, cudaIpcOpenMemHandle(&h->xch.peer_base[r], ipc, cudaIpcMemLazyEnablePeerAccess));
    }
    h->xch.connected = true;
    return KGPU_OK;
}

namespace {
// K1 (P > 0) + the exchange kernel on `st`; *d_final (may be NULL) receives where the global keys will be
int exchange_step(kgpu_ctx *h, const int32_t *d_pods, int64_t P, const uint64_t **d_final_keys, cudaStream_t st, int batch_flags) {
    kgpu_shard &s = h->shards[0];
    KGPU_CUDA(h, cudaSetDevice(s.dev));
    const int world = h->xch.world;
    const int64_t mp = h->xch.max_pods;
    int *d_err = reinterpret_cast<int *>(xch_flags(h->xch.base, world, mp) + kgpu::PEER_MAX_WORLD + 1);
    if (h->xch.epoch > 0 && (h->xch.epoch & 1023u) == 0) {     // now and then: did a wait time out?  (costs a sync, so rarely)
        int err = 0;
        KGPU_CUDA(h, cudaMemcpyAsync(&err, d_err, sizeof err, cudaMemcpyDeviceToHost, st));
        KGPU_CUDA(h, cudaStreamSynchronize(st));
        if (err) return fail(h, KGPU_ERR_COMM, "key exchange: a rank waited more than ~10 s for its peers (ranks out of step or a peer died)");
    }
    const uint32_t epoch = ++h->xch.epoch;
    const int buf = (int)(epoch & 1u);
    unsigned long long *fin = h->xch.final_keys + (int64_t)buf * mp;
    if (d_final_keys) *d_final_keys = reinterpret_cast<const uint64_t *>(fin);
    if (P > 0) {
        // K1 accumulates into xch.local (kept at NO_FIT between steps by the exchange kernel)
        const int rc = launch_score(h, s, d_pods, P, h->xch.local, st, (batch_flags & KGPU_BATCH_NO_MIN_MEM) ? 0 : -1, true);
        if (rc != KGPU_OK) return rc;
    }
    kgpu::PeerTable tab;
    memset(&tab, 0, sizeof tab);
    for (int r = 0; r < world; r++) {
        tab.slots[r] = xch_slots(h->xch.peer_base[r], world, mp, buf);
        tab.flags[r] = xch_flags(h->xch.peer_base[r], world, mp);
    }
    unsigned int *ticket = reinterpret_cast<unsigned int *>(xch_flags(h->xch.base, world, mp) + kgpu::PEER_MAX_WORLD);
    kgpu::gather_and_min<<<(unsigned)std::max<int64_t>(1, (P + 255) / 256), 256, 0, st>>>(h->xch.local, P, mp, tab, h->xch.rank, world, epoch, ticket,
                                                                                        fin, d_err);
    h->launches++;
    KGPU_CUDA(h, cudaGetLastError());
    return KGPU_OK;
}
}  // namespace

int kgpu_score_batch_exchange(kgpu_t *h, const int32_t *d_pods, int64_t P, const uint64_t **d_final_keys, void *stream,
                              int batch_flags) {
    if (!h) return fail(h, KGPU_ERR_INVALID, "kgpu_score_batch_exchange: NULL handle");
    std::lock_guard<std::mutex> g(h->mu);
    if (!h->xch.connected) return fail(h, KGPU_ERR_STATE, "kgpu_score_batch_exchange: exchange not connected");
    if (P < 0 || P > h->xch.max_pods || (P > 0 && !d_pods) || !d_final_keys)
        return fail(h, KGPU_ERR_INVALID, "kgpu_score_batch_exchange: bad arguments (P <= max_pods of kgpu_exchange_init)");
    return exchange_step(h, d_pods, P, d_final_keys, (cudaStream_t)stream, batch_flags);
}

int kgpu_exchange_barrier(kgpu_t *h, void *stream) {
    if (!h) return fail(h, KGPU_ERR_INVALID, "kgpu_exchange_barrier: NULL handle");
    std::lock_guard<std::mutex> g(h->mu);
    if (!h->xch.connected) return fail(h, KGPU_ERR_STATE, "kgpu_exchange_barrier: exchange not connected");
    return exchange_step(h, nullptr, 0, nullptr, (cudaStream_t)stream, 0);
}

int kgpu_reduce_shards_device(kgpu_t *h, const uint64_t *d_gathered, int G, int64_t P, uint64_t *d_out, void *stream) {
    if (!h) return fail(h, KGPU_ERR_INVALID, "kgpu_reduce_shards_device: NULL handle");
    std::lock_guard<std::mutex> g(h->mu);
    if (G < 1 || P < 0 || (P > 0 && (!d_gathered || !d_out))) return fail(h, KGPU_ERR_INVALID, "kgpu_reduce_shards_device: bad arguments");
    if (P == 0) return KGPU_OK;
    kgpu_shard &s = h->shards[0];
    KGPU_CUDA(h, cudaSetDevice(s.dev));
    kgpu::reduce_shards<<<(unsigned)((P + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<const unsigned long long *>(d_gathered), G, P, reinterpret_cast<unsigned long long *>(d_out));
    h->launches++;
    KGPU_CUDA(h, cudaGetLastError());
    return KGPU_OK;
}

int64_t kgpu_kernel_launches(kgpu_t *h) {
    if (!h) return 0;
    std::lock_guard<std::mutex> g(h->mu);
    return h->launches;
}

double kgpu_last_upload_ms(kgpu_t *h) {
    if (!h) return 0.0;
    std::lock_guard<std::mutex> g(h->mu);
    return h->last_upload_ms;
}

double kgpu_last_kernel_ms(kgpu_t *h) {
    if (!h) return 0.0;
    std::lock_guard<std::mutex> g(h->mu);
    return h->last_kernel_ms;
}

}  // extern "C"
