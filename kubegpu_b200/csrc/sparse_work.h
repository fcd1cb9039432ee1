// sparse_work.h -- host side of K1s: the work list.  Plain C++ (no CUDA), shared by kgpu.cu and the
// CPU emulation driver of the tests.
//
// A K1s block stages a 128-slot tile of the node order and scores a RANGE of the batch's pods against it.
// What a pod costs depends on the tile's class F (the largest number of free GPUs among its nodes): the
// bucket loops enumerate C(F,k) subsets, about 1 warp instruction per pod for F = 1 and about 110 for F = 8
// (scripts/k1s_issue_model.py).  Equal pod ranges for every tile therefore give blocks whose run times differ
// by two orders of magnitude (a long tail at the end of the launch), and with few tiles (a
// shard of a multi-GPU run) either too few blocks or ranges so short that staging and the per-chunk pod sort
// dominate.  The work list cuts the (tile, pod) plane into items of about equal WORK instead, heaviest first:
//   * many pods:  an item is one tile x a pod range (several chunks of the block's pod sort); on planes with enough
//     (tile, chunk) cells the ranges are whole chunks, whose sorted pod tables are built once per launch;
//   * few pods (the whole batch fits one chunk -- the HBM-bound regime, where the node records are streamed
//     once and hardly reused): an item is a RUN of consecutive tiles x all pods; the block sorts the pods once,
//     keeps the per-pod running minimum in shared memory across its tiles and flushes it once.
#pragma once
#include <algorithm>
#include <cstdint>
#include <numeric>
#include <vector>

namespace kgpu {

struct SparseWorkItem {
    int32_t tile, pod_begin, pod_end, ntiles;     // 16 bytes: one LDG.128 per block; ntiles > 1 only with pod ranges <= one chunk
};

// warp instructions per pod for a tile of class F (k uniform over 1..8, byte-key build) + ~2 for the
// per-chunk pod sort and the block flush; per-block fixed cost (block launch, staging, first sort): ~600;
// per further tile of a multi-tile item (staging, table reset, flush into shared memory): ~150
constexpr int32_t kSparsePodCost[9] = {2, 3, 4, 6, 9, 16, 31, 58, 114};
constexpr int64_t kSparseFixedCost = 600;
constexpr int64_t kSparseTileCost = 150;
constexpr int64_t kSparseChunk = 512;           // == SP_CHUNK (score_pairs_sparse.cuh static_asserts it)

struct SparseWorkParams {
    int64_t waves = 3;          // big items per resident block
    int64_t floor = 8;          // an item carries at least floor * kSparseFixedCost of work (<= 1/floor overhead)
    int64_t tail_percent = -1;  // the last part of every tile's pods (-1: 15 % on big shards, 0 on small ones, see below) ...
    int64_t tail_div = 4;       // ... goes into ranges a quarter as long: they fill the end of the launch
    int64_t max_run = 16;       // tiles per multi-tile item at most (H100 SXM, 400 W limit, 10.5M nodes x 32 / 256 pods:
                                // 0.624 / 2.382 ms for 1, 0.425 / 1.636 for 4, 0.427 / 1.587 for 16, 0.478 / 1.637 for 64)
};

// Many pods: do the pod ranges start and end on whole chunks (or end at P)?  Then every block takes its chunks' pod
// tables from the ones sp_prepare_chunks builds once per launch instead of sorting each chunk itself.  Only when the
// plane has at least `waves` such (tile, chunk) cells per resident block: on a small shard (C5's 10k nodes: ~80 tiles
// x 20 chunks) whole chunks leave too few items, and 32-pod ranges with the block's own sort are faster.
inline bool sparse_work_chunk_aligned(int64_t tiles, int64_t P, int64_t resident_blocks,
                                      const SparseWorkParams prm = SparseWorkParams()) {
    if (P <= kSparseChunk) return false;
    return tiles * ((P + kSparseChunk - 1) / kSparseChunk) >= std::max<int64_t>(1, prm.waves * resident_blocks);
}

// `out` = the items in launch order (heaviest first; the grid runs them in index order); `weight_out`, if
// given, receives their model cost.  Pod ranges are multiples of 32 pods, and of kSparseChunk pods (or end at P)
// when sparse_work_chunk_aligned says so.
inline void build_sparse_work(const std::vector<uint8_t> &tile_class, int64_t P, int64_t resident_blocks,
                              std::vector<SparseWorkItem> &out, const SparseWorkParams prm = SparseWorkParams(),
                              std::vector<int64_t> *weight_out = nullptr) {
    out.clear();
    if (weight_out) weight_out->clear();
    if (P <= 0 || tile_class.empty()) return;
    std::vector<SparseWorkItem> items;
    std::vector<int64_t> weight;
    int64_t total = 0;
    for (uint8_t f : tile_class) total += kSparseTileCost + P * kSparsePodCost[std::min<int>(f, 8)];
    const int64_t slots = std::max<int64_t>(1, prm.waves * resident_blocks);
    const int64_t gran = sparse_work_chunk_aligned((int64_t)tile_class.size(), P, resident_blocks, prm) ? kSparseChunk : 32;
    if (P <= kSparseChunk) {
        // few pods: runs of consecutive tiles, cut when the run's work reaches the target
        const int64_t target = std::max<int64_t>(total / slots, 2 * kSparseFixedCost);
        size_t t = 0;
        while (t < tile_class.size()) {
            int64_t w = kSparseFixedCost;
            size_t e = t;
            while (e < tile_class.size() && (int64_t)(e - t) < prm.max_run) {
                w += kSparseTileCost + P * kSparsePodCost[std::min<int>(tile_class[e], 8)];
                e++;
                if (w >= target) break;
            }
            items.push_back(SparseWorkItem{(int32_t)t, 0, (int32_t)P, (int32_t)(e - t)});
            weight.push_back(w);
            t = e;
        }
    } else {
        const int64_t target = std::max<int64_t>(total / slots, prm.floor * kSparseFixedCost);
        // short tail ranges help a little when every resident block gets several items anyway, and only add fixed cost
        // on small shards.  Measured on an H100 SXM (400 W limit), C2's pods: 100k nodes 0.514 - 0.518 ms with 15 %,
        // 0.517 - 0.520 with 25 %, 0.520 without; 12.5k nodes 0.085 ms without, 0.087 with 15 %
        const int64_t tail_percent = prm.tail_percent >= 0 ? prm.tail_percent : ((int64_t)tile_class.size() * 4 >= resident_blocks ? 15 : 0);
        for (size_t t = 0; t < tile_class.size(); t++) {
            const int64_t c = kSparsePodCost[std::min<int>(tile_class[t], 8)];
            const int64_t per = std::max<int64_t>(gran, (target - kSparseFixedCost) / c / gran * gran);
            const int64_t small = std::max<int64_t>(gran, per / std::max<int64_t>(1, prm.tail_div) / gran * gran);
            const int64_t big_end = P * (100 - tail_percent) / 100 / per * per;
            int64_t b = 0;
            while (b < P) {
                const int64_t e = std::min(P, b + (b < big_end ? per : small));
                items.push_back(SparseWorkItem{(int32_t)t, (int32_t)b, (int32_t)e, 1});
                weight.push_back(kSparseFixedCost + (e - b) * c);
                b = e;
            }
        }
    }
    std::vector<size_t> idx(items.size());
    std::iota(idx.begin(), idx.end(), (size_t)0);
    std::stable_sort(idx.begin(), idx.end(), [&](size_t a, size_t b) { return weight[a] > weight[b]; });
    out.reserve(items.size());
    for (size_t i : idx) {
        out.push_back(items[i]);
        if (weight_out) weight_out->push_back(weight[i]);
    }
}

}  // namespace kgpu
