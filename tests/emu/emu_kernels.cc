// emu_kernels.cc -- runs the real kernel sources (kubegpu_b200/csrc/*.cuh) on the CPU through cuda_emu.h.
// TEST INFRASTRUCTURE ONLY.  Every host plan around the launches (subset tables, views, plan columns, tile classes, the
// K1s instantiation and its work list) comes from launch_plan.h, as in kgpu.cu; this file only stages the inputs and
// launches.  One translation unit: the kernel headers define globals (c_subsets, ...).
#include "cuda_emu.h"

#include <algorithm>
#include <cstdlib>
#include <vector>

#include "score_pairs.cuh"
#include "score_pairs_sparse.cuh"
#include "place_sequential.cuh"
#include "preempt.cuh"
#include "preempt_plan.cuh"
#include "sparse_work.h"
#include "peer_exchange.cuh"
#include "node_state.cuh"
#include "launch_plan.h"

namespace {

const kgpu::PipeConsts kPC = {1u, 0xFFFFFFFFu};

kgpu::Weights weights_of(const int32_t *W) {
    kgpu::Weights w;
    std::memcpy(w.w, W, sizeof w.w);
    return w;
}

// The device arrays of one call: 64-byte aligned (the kernels load int4), zero-filled, freed when the call returns.
struct Staging {
    std::vector<void *> owned;
    Staging() = default;
    Staging(const Staging &) = delete;
    ~Staging() {
        for (void *p : owned) free(p);
    }
    template <class T>
    T *aligned_array(size_t n) {
        void *p = nullptr;
        if (posix_memalign(&p, 64, std::max<size_t>(64, n * sizeof(T))) != 0) abort();
        std::memset(p, 0, std::max<size_t>(64, n * sizeof(T)));
        owned.push_back(p);
        return (T *)p;
    }
    // n Ts copied from src, or every byte = fill when src is null
    template <class T>
    T *copy(const void *src, size_t n, int fill = 0) {
        T *p = aligned_array<T>(n);
        if (src && n) std::memcpy(p, src, n * sizeof(T));
        else if (fill) std::memset(p, fill, n * sizeof(T));
        return p;
    }
    int4 *topo(const int32_t *topo, int64_t n) { return copy<int4>(topo, (size_t)n * 16); }
    int4 *pods(const int32_t *pods, int64_t P) { return copy<int4>(pods, (size_t)P); }
    // GPU memory per node: unconstrained (INT32_MAX MiB) without an upload, as in kgpu.cu
    int32_t *mem(const int32_t *gpu_mem, int64_t n) {
        int32_t *p = copy<int32_t>(gpu_mem, (size_t)n * 8);
        if (!gpu_mem) std::fill(p, p + n * 8, INT32_MAX);
        return p;
    }
};

void upload_subset_tables() { kgpu::subset_tables(kgpu::c_subsets, kgpu::c_nsub); }

// The K1s node cache as build_order + ensure_node_cache make it: the device-side counting sort of the nodes by free
// count (classes padded to `pad` slots), then, given the topology, the compacted slot-ordered records.
struct Cache {
    std::vector<int32_t> order, slot_of;
    int64_t class_count[9] = {0};
    int64_t n_slots = 0, pad;
    Staging st;
    int4 *rec = nullptr;
    uint32_t *meta = nullptr;
    Cache(int32_t *free_mask, int64_t n, int64_t pad_ = 32, const int4 *topo4 = nullptr, const kgpu::Weights *Ws = nullptr)
        : pad(pad_) {
        const int nb = (int)((n + kgpu::ORD_BLOCK - 1) / kgpu::ORD_BLOCK);
        const int64_t cap = (n + 11 * kgpu::SP_THREADS) / kgpu::SP_THREADS * kgpu::SP_THREADS;
        order.assign((size_t)cap, -1);
        slot_of.assign((size_t)std::max<int64_t>(1, n), -1);
        std::vector<int32_t> cnt((size_t)nb * 9), off((size_t)nb * 9);
        long long m[kgpu::ORD_META] = {0};
        emu::launch(dim3((unsigned)nb), dim3(kgpu::ORD_BLOCK), [&] { kgpu::order_count(free_mask, n, cnt.data(), nb); });
        emu::launch(dim3(1), dim3(kgpu::ORD_BLOCK), [&] { kgpu::order_scan(cnt.data(), nb, off.data(), m, kgpu::SP_THREADS, (int)pad); });
        emu::launch(dim3((unsigned)nb), dim3(kgpu::ORD_BLOCK),
                    [&] { kgpu::order_scatter(free_mask, n, off.data(), nb, order.data(), slot_of.data()); });
        for (int k = 0; k < 9; k++) class_count[k] = m[k];
        n_slots = m[9];
        if (!topo4) return;
        rec = st.aligned_array<int4>(order.size() * 7);
        meta = st.aligned_array<uint32_t>(order.size());
        emu::launch(dim3((unsigned)(n_slots / kgpu::SP_THREADS)), dim3(kgpu::SP_THREADS),
                    [&] { kgpu::compact_nodes(topo4, free_mask, n_slots, *Ws, order.data(), slot_of.data(), rec, meta); });
    }
};

// K1s and its MEM instantiation as launch_score runs them.  splits >= 1: the plain (tiles x splits) grid; splits < 0: the
// work list cut for -splits resident blocks, on the route launch_plan.h picks.  allow_prepared = false keeps every
// block's own pod sort on a chunk-aligned list.
struct K1sRun {
    kgpu::SparseRoute route;
    bool aligned, mem;
};
K1sRun launch_k1s(const Cache &c, const int32_t *mem, int64_t node_id_base, const int4 *pods4, int64_t P, const int32_t *W,
                  int splits, bool allow_prepared, unsigned long long *keys) {
    int flag = 0;
    for (int64_t p = 0; p < P; p++) flag |= pods4[p].w > 0;
    dim3 grid((unsigned)(c.n_slots / kgpu::SP_THREADS), (unsigned)std::max(1, splits));
    std::vector<kgpu::SparseWorkItem> items;
    bool aligned = false;
    if (splits < 0) {
        const std::vector<uint8_t> tc = kgpu::tile_classes(c.class_count, c.pad, c.n_slots);
        kgpu::build_sparse_work(tc, P, -splits, items);
        aligned = kgpu::sparse_work_chunk_aligned((int64_t)tc.size(), P, -splits);
        grid = dim3((unsigned)items.size(), 1);
    }
    static_assert(sizeof(kgpu::SparseWorkItem) == sizeof(int4), "work item layout");
    const int4 *work = splits < 0 ? reinterpret_cast<const int4 *>(items.data()) : nullptr;
    const kgpu::SparseRoute r = kgpu::sparse_route(P, splits < 0, aligned && allow_prepared, 1, W);
    const int per = (int)kgpu::pods_per_split(P, std::max(1, splits));
    const int64_t chunks = (P + kgpu::SP_CHUNK - 1) / kgpu::SP_CHUNK;
    Staging st;
    int4 *tabs = r.prepared ? st.aligned_array<int4>((size_t)chunks * kgpu::SP_CHUNK_INT4) : nullptr;
    auto run = [&](bool m) {
        if (r.prepared)
            emu::launch(dim3((unsigned)chunks), dim3(kgpu::SP_THREADS), [&] {
                if (m) kgpu::sp_prepare_chunks<true>(pods4, P, &flag, tabs); else kgpu::sp_prepare_chunks<false>(pods4, P, &flag, tabs);
            });
        const kgpu::SparseKernel k1s = kgpu::sparse_kernel(r, m);
        emu::launch(grid, dim3(kgpu::SP_THREADS),
                    [&] { k1s(c.rec, c.meta, mem, c.order.data(), &flag, node_id_base, pods4, P, per, work, kPC, keys, tabs); });
    };
    run(false);
    if (flag) run(true);
    return K1sRun{r, aligned, flag != 0};
}

// The pod sort as a K1s block runs it in its chunk prologue, one block per chunk: its shared-memory table, dumped.
template <bool MEM>
void block_sort(const int4 *pods4, int64_t P, int4 *out) {
    constexpr int NB = 9 * (MEM ? kgpu::SP_MEM_SUB : 1) + 1;
    __shared__ int32_t sCnt[NB];
    __shared__ kgpu::SpTab<kgpu::SP_POS> sTab;
    const int tid = threadIdx.x;
    const int64_t c0 = (int64_t)blockIdx.x * kgpu::SP_CHUNK;
    __syncthreads();
    kgpu::sp_sort_chunk<MEM, kgpu::SP_CHUNK, kgpu::SP_THREADS>(pods4 + c0, (int)min((int64_t)kgpu::SP_CHUNK, P - c0), sCnt,
                                                               sTab.c, nullptr, tid);
    __syncthreads();
    if (tid == 0) std::memcpy(out + (int64_t)blockIdx.x * kgpu::SP_CHUNK_INT4, &sTab.c, sizeof sTab.c);
    __syncthreads();
}

}  // namespace

extern "C" {

// K1s (+ its MEM instantiation) exactly as kgpu.cu launches them: device-built order, compact cache, grid or work list.
// Returns the route: 0 = every block sorts its pods, 1 = prepared chunk tables, 2 = STREAM, 3 = TMA; | 4 when the MEM
// launch ran, | 8 with byte keys.
int emu_score_sparse(const int32_t *topo, const int32_t *free_mask_in, const int32_t *gpu_mem /*nullable*/, int64_t n,
                     int64_t node_id_base, const int32_t *pods, int64_t P, const int32_t *W, int splits, unsigned long long *keys) {
    std::memset(keys, 0xFF, (size_t)P * 8);
    if (n == 0 || P == 0) return -1;
    std::vector<int32_t> free_mask(free_mask_in, free_mask_in + n);
    Staging st;
    const kgpu::Weights Ws = weights_of(W);
    Cache c(free_mask.data(), n, 32, st.topo(topo, n), &Ws);
    const K1sRun run = launch_k1s(c, st.mem(gpu_mem, n), node_id_base, st.pods(pods, P), P, W, splits, true, keys);
    const kgpu::SparseRoute &r = run.route;
    return (r.tma ? 3 : r.stream ? 2 : r.prepared ? 1 : 0) | (run.mem ? 4 : 0) | (r.byte_keys ? 8 : 0);
}

// kgpu_upload_nodes + kgpu_set_free_masks + kgpu_score_batch: the cache is built for free_mask0, then the m listed
// nodes get new masks through the incremental path (compact_nodes with a list; the order stays as it was, i.e.
// stale), then K1s runs.  Must equal a fresh upload with the final masks.
void emu_score_sparse_after_updates(const int32_t *topo, const int32_t *free_mask0, int64_t n, const int32_t *upd_idx,
                                    const int32_t *upd_mask, int64_t m, const int32_t *pods, int64_t P, const int32_t *W,
                                    int splits, unsigned long long *keys, int32_t *free_mask_out) {
    std::memset(keys, 0xFF, (size_t)P * 8);
    std::vector<int32_t> free_mask(free_mask0, free_mask0 + n);
    Staging st;
    const int4 *topo4 = st.topo(topo, n);
    const kgpu::Weights Ws = weights_of(W);
    Cache c(free_mask.data(), n, 32, topo4, &Ws);
    if (m > 0)
        emu::launch(dim3((unsigned)((m + kgpu::SP_THREADS - 1) / kgpu::SP_THREADS)), dim3(kgpu::SP_THREADS), [&] {
            kgpu::compact_nodes(topo4, free_mask.data(), m, Ws, c.order.data(), c.slot_of.data(), c.rec, c.meta, upd_idx, upd_mask);
        });
    launch_k1s(c, st.mem(nullptr, n), 0, st.pods(pods, P), P, W, splits, true, keys);
    std::memcpy(free_mask_out, free_mask.data(), (size_t)n * 4);
}

// A handle's K1s cache over a sequence of state changes, then K1s.  The cache is built for (topo0, free0) as by
// kgpu_upload_nodes; update j then goes through the incremental path on the order that stays as it was (stale):
//   has_topo[j] == 0  kgpu_set_free_masks: consecutive such updates are one batched compact_nodes(list, new_mask), a batch
//                     being cut where a node repeats;
//   has_topo[j] != 0  kgpu_update_node: row j of upd_topo is written over the node's topology, then compact_nodes over
//                     that one node with its new mask.
// With W2, before update w2_at (after the last one if w2_at >= m) the weights become W2 the way kgpu_set_weights +
// ensure_node_cache apply them: one compact_nodes over every slot of the stale order, no re-sort; later updates use W2.
// K1s then runs with the final weights (route and splits as for emu_score_sparse, which it returns the route code of);
// free_out receives the final masks.
int emu_score_sparse_sequence(const int32_t *topo0, const int32_t *free0, const int32_t *gpu_mem /*nullable*/, int64_t n,
                              int64_t node_id_base, const int32_t *upd_idx, const int32_t *upd_mask, const int32_t *upd_topo,
                              const int32_t *has_topo, int64_t m, const int32_t *W, const int32_t *W2 /*nullable*/, int64_t w2_at,
                              const int32_t *pods, int64_t P, int splits, unsigned long long *keys, int32_t *free_out) {
    std::memset(keys, 0xFF, (size_t)P * 8);
    if (n == 0 || P == 0) return -1;
    std::vector<int32_t> free_mask(free0, free0 + n);
    Staging st;
    int4 *topo4 = st.topo(topo0, n);
    kgpu::Weights Ws = weights_of(W);
    const int32_t *Wcur = W;
    Cache c(free_mask.data(), n, 32, topo4, &Ws);
    std::vector<int32_t> bidx, bmask;
    auto refresh = [&](const int32_t *idx, const int32_t *mask, int64_t cnt) {
        emu::launch(dim3((unsigned)((cnt + kgpu::SP_THREADS - 1) / kgpu::SP_THREADS)), dim3(kgpu::SP_THREADS), [&] {
            kgpu::compact_nodes(topo4, free_mask.data(), cnt, Ws, c.order.data(), c.slot_of.data(), c.rec, c.meta, idx, mask);
        });
    };
    auto flush = [&] {
        if (!bidx.empty()) refresh(bidx.data(), bmask.data(), (int64_t)bidx.size());
        bidx.clear();
        bmask.clear();
    };
    auto set_weights = [&] {
        flush();
        Ws = weights_of(W2);
        Wcur = W2;
        emu::launch(dim3((unsigned)(c.n_slots / kgpu::SP_THREADS)), dim3(kgpu::SP_THREADS), [&] {
            kgpu::compact_nodes(topo4, free_mask.data(), c.n_slots, Ws, c.order.data(), c.slot_of.data(), c.rec, c.meta);
        });
    };
    for (int64_t j = 0; j < m; j++) {
        if (W2 && j == w2_at) set_weights();
        if (has_topo[j]) {
            flush();
            std::memcpy(reinterpret_cast<int32_t *>(topo4) + (int64_t)upd_idx[j] * 64, upd_topo + j * 64, 256);
            refresh(upd_idx + j, upd_mask + j, 1);
        } else {
            if (std::find(bidx.begin(), bidx.end(), upd_idx[j]) != bidx.end()) flush();
            bidx.push_back(upd_idx[j]);
            bmask.push_back(upd_mask[j]);
        }
    }
    if (W2 && w2_at >= m) set_weights();
    flush();
    const K1sRun run = launch_k1s(c, st.mem(gpu_mem, n), node_id_base, st.pods(pods, P), P, Wcur, splits, true, keys);
    std::memcpy(free_out, free_mask.data(), (size_t)n * 4);
    const kgpu::SparseRoute &r = run.route;
    return (r.tma ? 3 : r.stream ? 2 : r.prepared ? 1 : 0) | (run.mem ? 4 : 0) | (r.byte_keys ? 8 : 0);
}

// The device-built order alone: order[cap] (cap = n + 9*32 + 2*tile rounded down to tiles), slot_of[n], class counts.
int64_t emu_order(const int32_t *free_mask, int64_t n, int32_t *order_out, int64_t cap, int32_t *slot_of_out, long long *class_count) {
    std::vector<int32_t> f(free_mask, free_mask + n);
    Cache c(f.data(), n);
    for (int64_t i = 0; i < cap; i++) order_out[i] = i < (int64_t)c.order.size() ? c.order[(size_t)i] : -1;
    std::memcpy(slot_of_out, c.slot_of.data(), (size_t)n * 4);
    for (int k = 0; k < 9; k++) class_count[k] = c.class_count[k];
    return c.n_slots;
}

// The tile classes of the order built with classes padded to `pad` slots, twice: from_counts as the hosts derive them
// (launch_plan.h: tile_classes), from_slots as the largest free count among each tile's nodes.  Returns the tile count.
int64_t emu_tile_classes(const int32_t *free_mask, int64_t n, int pad, uint8_t *from_counts, uint8_t *from_slots, int64_t cap) {
    std::vector<int32_t> f(free_mask, free_mask + n);
    Cache c(f.data(), n, pad);
    const std::vector<uint8_t> tc = kgpu::tile_classes(c.class_count, c.pad, c.n_slots);
    std::vector<uint8_t> slots(tc.size(), 0);
    for (int64_t sl = 0; sl < c.n_slots; sl++)
        if (c.order[(size_t)sl] >= 0) {
            uint8_t &m = slots[(size_t)(sl / kgpu::SP_THREADS)];
            m = std::max<uint8_t>(m, (uint8_t)__builtin_popcount((unsigned)f[(size_t)c.order[(size_t)sl]] & 0xFFu));
        }
    for (size_t t = 0; t < tc.size() && (int64_t)t < cap; t++) {
        from_counts[t] = tc[t];
        from_slots[t] = slots[t];
    }
    return (int64_t)tc.size();
}

// fit_nodes (the (node, k) fit table), optionally over a list; out[k * m + i]
void emu_fit_nodes(const int32_t *topo, const int32_t *free_mask, int64_t n, const int32_t *list /*nullable*/, int64_t m,
                   const int32_t *W, uint32_t *out) {
    Staging st;
    const int4 *topo4 = st.topo(topo, n);
    const kgpu::Weights Ws = weights_of(W);
    emu::launch(dim3((unsigned)((m + 127) / 128)), dim3(128), [&] { kgpu::fit_nodes(topo4, free_mask, list, m, Ws, kPC, out); });
}

// validate_topo_dev: index of the first value outside 0..15, or -1
long long emu_validate_topo(const int32_t *topo, int64_t n) {
    Staging st;
    const int4 *topo4 = st.topo(topo, n);
    unsigned long long bad = ~0ull;
    emu::launch(dim3((unsigned)((n * 16 + 255) / 256)), dim3(256), [&] { kgpu::validate_topo_dev(topo4, n * 16, &bad); });
    return bad == ~0ull ? -1 : (long long)bad;
}

// The peer-exchange kernel with world = 1 (the rank stores into its own slot array and passes its own barrier):
// exercises the stores, the ticket, the flag protocol and the final minimum, not the cross-GPU part.
void emu_gather_and_min(unsigned long long *local, int64_t P, int64_t max_pods, unsigned long long *slots, uint32_t *flags,
                        uint32_t epoch, unsigned int *ticket, unsigned long long *final_keys, int *error) {
    kgpu::PeerTable tab;
    std::memset(&tab, 0, sizeof tab);
    tab.slots[0] = slots;
    tab.flags[0] = flags;
    emu::launch(dim3((unsigned)std::max<int64_t>(1, (P + 255) / 256)), dim3(256),
                [&] { kgpu::gather_and_min(local, P, max_pods, tab, 0, 1, epoch, ticket, final_keys, error); });
}

// The host-side work-list builder alone (sparse_work.h) with default parameters: items as int32[.][4] {tile, pod_begin,
// pod_end, ntiles}, their model weights if weight_out is given, *aligned (if given) = whether sparse_work_chunk_aligned
// chose whole chunks.  Returns the count.
int64_t emu_sparse_work(const uint8_t *tile_class, int64_t tiles, int64_t P, int64_t resident, int32_t *out, int64_t cap,
                        long long *weight_out /*nullable*/, int *aligned /*nullable*/) {
    std::vector<kgpu::SparseWorkItem> items;
    std::vector<int64_t> weight;
    kgpu::build_sparse_work(std::vector<uint8_t>(tile_class, tile_class + tiles), P, resident, items, kgpu::SparseWorkParams(), &weight);
    if (aligned) *aligned = kgpu::sparse_work_chunk_aligned(tiles, P, resident) ? 1 : 0;
    for (size_t i = 0; i < items.size() && (int64_t)i < cap; i++) {
        std::memcpy(out + 4 * i, &items[i], 16);
        if (weight_out) weight_out[i] = weight[i];
    }
    return (int64_t)items.size();
}

// Dense K1 (+ K1m) as kgpu.cu launches them.
void emu_score_dense(const int32_t *topo, const int32_t *free_mask, const int32_t *gpu_mem /*nullable*/, int64_t n,
                     int64_t node_id_base, const int32_t *pods, int64_t P, const int32_t *W, int splits,
                     unsigned long long *keys) {
    std::memset(keys, 0xFF, (size_t)P * 8);
    if (n == 0 || P == 0) return;
    Staging st;
    const int4 *topo4 = st.topo(topo, n), *pods4 = st.pods(pods, P);
    const int4 *mem4 = reinterpret_cast<const int4 *>(st.mem(gpu_mem, n));
    const kgpu::Weights Ws = weights_of(W);
    int flag = 0;
    for (int64_t p = 0; p < P; p++) flag |= pods[4 * p + 3] > 0;
    const dim3 grid((unsigned)((n + kgpu::LPN_THREADS - 1) / kgpu::LPN_THREADS), (unsigned)std::max(1, splits));
    const int per = (int)kgpu::pods_per_split(P, std::max(1, splits));
    emu::launch(grid, dim3(kgpu::LPN_THREADS), [&] {
        kgpu::score_pairs_lane_per_node<true, false>(topo4, free_mask, mem4, &flag, n, node_id_base, pods4, P, per, Ws, kPC, keys);
    });
    if (flag)
        emu::launch(grid, dim3(kgpu::LPN_THREADS), [&] {
            kgpu::score_pairs_lane_per_node<true, true>(topo4, free_mask, mem4, &flag, n, node_id_base, pods4, P, per, Ws, kPC, keys);
        });
}

// The other K1 variants as kgpu.cu launches them: 1 = warp per pair (north_star mapping), 3 = memo by k,
// 4 = tile memo.  Memory-constrained pods go to K1m for variants 3 and 4, inline for variant 1.
void emu_score_variant(int variant, const int32_t *topo, const int32_t *free_mask, const int32_t *gpu_mem, int64_t n,
                       int64_t node_id_base, const int32_t *pods, int64_t P, const int32_t *W, int splits,
                       unsigned long long *keys) {
    std::memset(keys, 0xFF, (size_t)P * 8);
    if (n == 0 || P == 0) return;
    upload_subset_tables();
    Staging st;
    const int4 *topo4 = st.topo(topo, n), *pods4 = st.pods(pods, P);
    const int32_t *mem = st.mem(gpu_mem, n);
    const int4 *mem4 = reinterpret_cast<const int4 *>(mem);
    const kgpu::Weights Ws = weights_of(W);
    int flag = 0;
    emu::launch(dim3((unsigned)((P + 255) / 256)), dim3(256), [&] { kgpu::any_mem_pod(pods4, P, &flag); });
    const int per = (int)kgpu::pods_per_split(P, std::max(1, splits));
    if (variant == 1) {
        const dim3 grid((unsigned)((n + kgpu::WPP_TILE - 1) / kgpu::WPP_TILE), (unsigned)std::max(1, splits));
        emu::launch(grid, dim3(kgpu::WPP_THREADS), [&] {
            kgpu::score_pairs_warp_per_pair(topo4, free_mask, mem, n, node_id_base, pods4, P, per, Ws, kPC, keys);
        });
    } else {
        const dim3 grid((unsigned)((n + kgpu::LPN_THREADS - 1) / kgpu::LPN_THREADS), (unsigned)std::max(1, splits));
        if (variant == 3) {
            unsigned long long bestk[9];
            std::memset(bestk, 0xFF, sizeof bestk);
            emu::launch(dim3(std::min<unsigned>(grid.x, 3)), dim3(kgpu::LPN_THREADS),
                        [&] { kgpu::memo_best_by_k(topo4, free_mask, n, node_id_base, Ws, kPC, bestk); });
            emu::launch(dim3((unsigned)((P + 255) / 256)), dim3(256), [&] { kgpu::memo_gather(pods4, P, bestk, keys); });
        } else {
            emu::launch(grid, dim3(kgpu::LPN_THREADS), [&] {
                kgpu::score_pairs_lane_per_node<false, false>(topo4, free_mask, mem4, &flag, n, node_id_base, pods4, P, per, Ws, kPC, keys);
            });
        }
        if (flag)
            emu::launch(grid, dim3(kgpu::LPN_THREADS), [&] {
                kgpu::score_pairs_lane_per_node<true, true>(topo4, free_mask, mem4, &flag, n, node_id_base, pods4, P, per, Ws, kPC, keys);
            });
    }
}

// K2
void emu_reduce_shards(const unsigned long long *gathered, int G, int64_t P, unsigned long long *out) {
    emu::launch(dim3((unsigned)((P + 255) / 256)), dim3(256), [&] { kgpu::reduce_shards(gathered, G, P, out); });
}

// kgpu_score_pairs (the min_mem path: packed queries)
void emu_score_pair_list(const int32_t *topo, const int32_t *free_mask, const int32_t *gpu_mem, int64_t n,
                         const long long *node_idx, const int32_t *ks, const int32_t *min_mem, int64_t m, const int32_t *W,
                         uint32_t *out) {
    Staging st;
    const int4 *topo4 = st.topo(topo, n);
    const int32_t *mem = st.mem(gpu_mem, n);
    int4 *q = st.aligned_array<int4>((size_t)m);
    for (int64_t i = 0; i < m; i++)
        q[i] = make_int4((int)(node_idx[i] & 0xFFFFFFFFLL), (int)(node_idx[i] >> 32), ks[i], min_mem ? min_mem[i] : 0);
    const kgpu::Weights Ws = weights_of(W);
    emu::launch(dim3((unsigned)((m + 127) / 128)), dim3(128),
                [&] { kgpu::score_pair_list(topo4, free_mask, mem, n, q, m, Ws, kPC, out); });
}

// K3: place_init + place_half_tables + place_sequential as kgpu_place_batch_gang launches them (views from the batch's
// distinct min_mem values; with gang[P], the caller has checked that every gang id forms one run); free_mask is
// updated in place like the device copy.  Returns 0, or -1 for too many views.
int emu_place_batch_gang(const int32_t *topo, int32_t *free_mask, const int32_t *gpu_mem /*nullable*/, int64_t n,
                         int64_t node_id_base, const int32_t *pods, const int32_t *gang /*nullable*/, int64_t P, const int32_t *W,
                         unsigned long long *keys) {
    std::memset(keys, 0xFF, (size_t)P * 8);
    if (n == 0 || P == 0) return 0;
    kgpu::PlaceViews views;
    if (!kgpu::place_views(pods, P, views)) return -1;
    upload_subset_tables();
    Staging st;
    const int4 *topo4 = st.topo(topo, n), *pods4 = st.pods(pods, P);
    const int32_t *topo32 = reinterpret_cast<const int32_t *>(topo4), *mem = st.mem(gpu_mem, n);
    const int64_t T = (n + kgpu::PLACE_TILE - 1) / kgpu::PLACE_TILE, Npad = T * kgpu::PLACE_TILE;
    uint32_t *nodebest = st.aligned_array<uint32_t>((size_t)Npad * 9 * views.n);
    unsigned long long *tilebest = st.aligned_array<unsigned long long>((size_t)T * 9 * views.n);
    int32_t *half_all = st.aligned_array<int32_t>((size_t)Npad * kgpu::PLACE_HALF);
    const kgpu::Weights Ws = weights_of(W);
    emu::launch(dim3((unsigned)T, (unsigned)views.n), dim3(kgpu::PLACE_TILE),
                [&] { kgpu::place_init(topo4, free_mask, mem, n, Npad, node_id_base, Ws, kPC, views, nodebest, tilebest, T); });
    emu::launch(dim3((unsigned)std::min<int64_t>((n + 3) / 4, 8)), dim3(128), [&] { kgpu::place_half_tables(topo32, n, Ws, half_all); });
    emu::launch(dim3(1), dim3(kgpu::PLACE_THREADS), [&] {
        if (gang)
            kgpu::place_sequential<true>(topo32, free_mask, mem, n, Npad, node_id_base, pods4, P, Ws, views, nodebest, tilebest, T,
                                         half_all, keys, gang);
        else
            kgpu::place_sequential(topo32, free_mask, mem, n, Npad, node_id_base, pods4, P, Ws, views, nodebest, tilebest, T, half_all,
                                   keys);
    });
    return 0;
}

int emu_place_batch(const int32_t *topo, int32_t *free_mask, const int32_t *gpu_mem /*nullable*/, int64_t n,
                    int64_t node_id_base, const int32_t *pods, int64_t P, const int32_t *W, unsigned long long *keys) {
    return emu_place_batch_gang(topo, free_mask, gpu_mem, n, node_id_base, pods, nullptr, P, W, keys);
}

// Steps 2-3 of kgpu_preempt_batch as it launches them: keys[P] holds the scoring path's keys on entry (the caller
// computes them with the oracle) and the preemption keys on return; victims[P] is zeroed first.  splits = the grid's
// pod dimension.  Returns how many pods reached the preemption kernel.
int emu_preempt_batch(const int32_t *topo, const int32_t *free_mask, const int32_t *gpu_mem /*nullable*/,
                      const int32_t *hold /*nullable*/, int64_t n, int64_t node_id_base, const int32_t *pods,
                      const int32_t *lvl, int64_t P, const int32_t *W, int splits, unsigned long long *keys,
                      uint32_t *victims) {
    std::memset(victims, 0, (size_t)P * 4);
    if (n == 0 || P == 0 || !hold) return 0;
    Staging st;
    const int4 *topo4 = st.topo(topo, n), *pods4 = st.pods(pods, P);
    const int4 *mem4 = reinterpret_cast<const int4 *>(st.mem(gpu_mem, n));
    const int4 *hold4 = st.copy<int4>(hold, (size_t)n * 2);
    int32_t *idx = st.aligned_array<int32_t>((size_t)P);
    unsigned long long *pkey = st.copy<unsigned long long>(nullptr, (size_t)P, 0xFF);
    int count = 0;
    const kgpu::Weights Ws = weights_of(W);
    const unsigned pb = (unsigned)((P + 127) / 128);
    emu::launch(dim3(pb), dim3(128), [&] { kgpu::preempt_compact(pods4, lvl, keys, P, idx, &count); });
    const unsigned tiles = (unsigned)((n + kgpu::PRE_THREADS - 1) / kgpu::PRE_THREADS);
    emu::launch(dim3(tiles, (unsigned)splits), dim3(kgpu::PRE_THREADS), [&] {
        kgpu::preempt_lane_per_node(topo4, free_mask, mem4, hold4, n, pods4, lvl, idx, &count, Ws, kPC, pkey);
    });
    emu::launch(dim3(pb), dim3(128), [&] {
        kgpu::preempt_finalize(pkey, idx, &count, free_mask, reinterpret_cast<const int32_t *>(hold4), node_id_base, keys, victims);
    });
    return count;
}

// kgpu_preempt_plan_gang as it launches the kernels (gang == nullptr: kgpu_preempt_plan), with the same columns; any
// batch whose columns fit the kernels runs, also one beyond libkgpu's limits.  Returns the number of columns, or -1.
int emu_preempt_plan_gang(const int32_t *topo, const int32_t *free_mask, const int32_t *gpu_mem /*nullable*/,
                          const int32_t *hold /*nullable*/, int64_t n, int64_t node_id_base, const int32_t *pods, const int32_t *lvl,
                          const int32_t *gang /*nullable*/, int64_t P, const int32_t *W, unsigned long long *keys, uint32_t *victims) {
    std::vector<int4> colv;
    std::vector<int32_t> pcolv;
    kgpu::plan_columns(pods, lvl, P, colv, pcolv);
    const int ncol = (int)colv.size();
    if (ncol > kgpu::PLAN_MAX_COLS) return -1;
    if (n == 0) {
        for (int64_t p = 0; p < P; p++) { keys[p] = ~0ull; victims[p] = 0; }
        return ncol;
    }
    Staging st;
    const int4 *cols = st.copy<int4>(colv.data(), (size_t)ncol), *topo4 = st.topo(topo, n), *pods4 = st.pods(pods, P);
    const int32_t *pcol = st.copy<int32_t>(pcolv.data(), (size_t)P);
    const int4 *mem4 = reinterpret_cast<const int4 *>(st.mem(gpu_mem, n));
    int32_t *F = st.copy<int32_t>(free_mask, (size_t)n), *H = st.copy<int32_t>(hold, (size_t)n * 8, 0xFF);
    const int64_t T = (n + kgpu::PLAN_TILE - 1) / kgpu::PLAN_TILE, Npad = T * kgpu::PLAN_TILE;
    unsigned long long *nodekey = st.aligned_array<unsigned long long>((size_t)(ncol * Npad));
    unsigned long long *tilekey = st.aligned_array<unsigned long long>((size_t)(ncol * T));
    const kgpu::Weights Ws = weights_of(W);
    if (ncol > 0) {
        const unsigned groups = (unsigned)((ncol + kgpu::PLAN_INIT_COLS - 1) / kgpu::PLAN_INIT_COLS);
        emu::launch(dim3((unsigned)T, groups), dim3(kgpu::PLAN_TILE), [&] {
            kgpu::plan_init(topo4, F, mem4, reinterpret_cast<const int4 *>(H), n, Npad, T, cols, ncol, Ws, kPC, nodekey, tilekey);
        });
    }
    const int32_t *gang_ids = gang ? st.copy<int32_t>(gang, (size_t)P) : nullptr;
    int4 *pre = gang ? st.aligned_array<int4>((size_t)P) : nullptr;
    emu::launch(dim3(1), dim3(kgpu::PLAN_THREADS), [&] {
        if (gang)
            kgpu::gang_plan_sequential(topo4, F, mem4, H, n, Npad, T, node_id_base, pods4, pcol, P, cols, ncol, Ws, kPC, nodekey, tilekey,
                                       keys, victims, gang_ids, pre);
        else
            kgpu::plan_sequential(topo4, F, mem4, H, n, Npad, T, node_id_base, pods4, pcol, P, cols, ncol, Ws, kPC, nodekey, tilekey, keys,
                                  victims);
    });
    return ncol;
}

int emu_preempt_plan(const int32_t *topo, const int32_t *free_mask, const int32_t *gpu_mem /*nullable*/,
                     const int32_t *hold /*nullable*/, int64_t n, int64_t node_id_base, const int32_t *pods, const int32_t *lvl,
                     int64_t P, const int32_t *W, unsigned long long *keys, uint32_t *victims) {
    return emu_preempt_plan_gang(topo, free_mask, gpu_mem, hold, n, node_id_base, pods, lvl, nullptr, P, W, keys, victims);
}

int emu_chunk_int4() { return kgpu::SP_CHUNK_INT4; }
int emu_chunk_pos() { return kgpu::SP_POS; }

// Both tables of every chunk of the batch, [chunks][SP_CHUNK_INT4] int4 each: sp_prepare_chunks<mem> into `prepared`,
// the block's own sort into `sorted`.  Returns the chunk count.
int64_t emu_chunk_tables(const int32_t *pods, int64_t P, int mem, int32_t *prepared, int32_t *sorted) {
    const int64_t chunks = (P + kgpu::SP_CHUNK - 1) / kgpu::SP_CHUNK;
    Staging st;
    const int4 *pods4 = st.pods(pods, P);
    int4 *prep = st.aligned_array<int4>((size_t)chunks * kgpu::SP_CHUNK_INT4);
    int4 *sort = st.aligned_array<int4>((size_t)chunks * kgpu::SP_CHUNK_INT4);
    int flag = 1;
    emu::launch(dim3((unsigned)chunks), dim3(kgpu::SP_THREADS), [&] {
        if (mem) kgpu::sp_prepare_chunks<true>(pods4, P, &flag, prep); else kgpu::sp_prepare_chunks<false>(pods4, P, &flag, prep);
    });
    emu::launch(dim3((unsigned)chunks), dim3(kgpu::SP_THREADS), [&] {
        if (mem) block_sort<true>(pods4, P, sort); else block_sort<false>(pods4, P, sort);
    });
    std::memcpy(prepared, prep, (size_t)chunks * kgpu::SP_CHUNK_INT4 * 16);
    std::memcpy(sorted, sort, (size_t)chunks * kgpu::SP_CHUNK_INT4 * 16);
    return chunks;
}

// K1s on the work list for `resident` blocks as kgpu.cu launches it; prepare = 0 keeps every block's own pod sort even
// on a chunk-aligned list.  Returns 1 if the list was chunk-aligned.
int emu_score_chunks(const int32_t *topo, const int32_t *free_mask_in, const int32_t *gpu_mem /*nullable*/, int64_t n,
                     int64_t node_id_base, const int32_t *pods, int64_t P, const int32_t *W, int64_t resident, int prepare,
                     unsigned long long *keys) {
    std::memset(keys, 0xFF, (size_t)P * 8);
    std::vector<int32_t> free_mask(free_mask_in, free_mask_in + n);
    Staging st;
    const kgpu::Weights Ws = weights_of(W);
    Cache c(free_mask.data(), n, 32, st.topo(topo, n), &Ws);
    return launch_k1s(c, st.mem(gpu_mem, n), node_id_base, st.pods(pods, P), P, W, -(int)resident, prepare != 0, keys).aligned ? 1 : 0;
}

}  // extern "C"
