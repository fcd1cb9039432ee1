// launch_plan.h -- the host-side plans around libkgpu's launches, written once: kgpu.cu launches what they say on the
// device and the CPU emulation of the tests (tests/emu) launches the same on the CPU.  Host code only, no CUDA runtime
// calls; it names the kernels' constants, so it comes after their headers.
#pragma once
#include <algorithm>
#include <array>
#include <cstdint>
#include <cstring>
#include <utility>
#include <vector>

#include "gang_domain.cuh"
#include "place_sequential.cuh"
#include "score_pairs_sparse.cuh"
#include "sparse_work.h"

namespace kgpu {

// c_subsets / c_nsub: the k-subsets of the eight GPUs in increasing mask order, for k = 0..8
inline void subset_tables(uint8_t subs[9][70], uint8_t nsub[9]) {
    std::memset(subs, 0, 9 * 70);
    for (int k = 0; k <= 8; k++) {
        int c = 0;
        for (unsigned S = 0; S < 256; S++)
            if (__builtin_popcount(S) == k) subs[k][c++] = (uint8_t)S;
        nsub[k] = (uint8_t)c;
    }
}

// K3: the batch's distinct memory requirements are the views the sequential kernels keep tables for (view 0: none).
// False when there are more than PLACE_MAX_VIEWS - 1 of them.
inline bool place_views(const int32_t *pods, int64_t P, PlaceViews &views) {
    std::memset(&views, 0, sizeof views);
    views.n = 1;
    for (int64_t p = 0; p < P; p++) {
        const int32_t need = pods[4 * p + 3];
        if (need <= 0 || pods[4 * p] < 0 || pods[4 * p] > 8) continue;
        bool seen = false;
        for (int j = 1; j < views.n; j++) seen = seen || views.min_mem[j] == need;
        if (seen) continue;
        if (views.n == PLACE_MAX_VIEWS) return false;
        views.min_mem[views.n++] = need;
    }
    return true;
}

// kgpu_place_batch_gang_levels: the batch cut into segments, in order.  A constrained gang (a run of consecutive pods with
// the same nonzero gang id and a nonzero gang_domain, which the host has checked its members agree on) is one domain
// step, mode = its gang_domain, level = its gang_level (0 without gang_level): one domain_trial per level 0..level, then
// domain_commit.  Every maximal pod range without one is one place_sequential launch on pods + begin, mode = 0.
// gang_domain == nullptr (or all 0): one segment, the whole batch.  Preemption plans (kgpu_preempt_plan_gang_domain) are
// cut the same way, without levels: plan_sequential / gang_plan_sequential per plain range, domain_plan_trial +
// domain_plan_commit per constrained gang.
struct PlaceSegment {
    int64_t begin, end;
    int32_t mode, level;
};
inline std::vector<PlaceSegment> place_segments(const int32_t *gang, const int32_t *gang_domain, int64_t P,
                                                const int32_t *gang_level = nullptr) {
    std::vector<PlaceSegment> seg;
    int64_t p = 0, plain = 0;
    while (p < P) {
        if (gang_domain == nullptr || gang_domain[p] == 0) {
            p++;
            continue;
        }
        int64_t e = p + 1;
        while (e < P && gang[e] == gang[p]) e++;
        if (plain < p) seg.push_back({plain, p, 0, 0});
        seg.push_back({p, e, gang_domain[p], gang_level ? gang_level[p] : 0});
        p = plain = e;
    }
    if (plain < P) seg.push_back({plain, P, 0, 0});
    return seg;
}

// kgpu_upload_domains: the node lists of the domains in one counting pass.  domain[n] is -1 (no domain) or 0..n-1;
// D = 1 + the largest id.  off[D + 1]; nodes[] holds each domain's nodes in increasing index, -1 nodes left out.
// Returns the index of the first value outside -1..n-1 (nothing built), or -1.
inline int64_t domain_lists(const int32_t *domain, int64_t n, std::vector<int32_t> &off, std::vector<int32_t> &nodes) {
    int32_t D = 0;
    for (int64_t i = 0; i < n; i++) {
        if (domain[i] < -1 || domain[i] >= n) return i;
        D = std::max(D, domain[i] + 1);
    }
    off.assign((size_t)D + 1, 0);
    for (int64_t i = 0; i < n; i++)
        if (domain[i] >= 0) off[(size_t)domain[i] + 1]++;
    for (int32_t d = 0; d < D; d++) off[(size_t)d + 1] += off[(size_t)d];
    nodes.assign((size_t)off[(size_t)D], 0);
    std::vector<int32_t> at(off.begin(), off.end() - 1);
    for (int64_t i = 0; i < n; i++)
        if (domain[i] >= 0) nodes[(size_t)at[(size_t)domain[i]]++] = (int32_t)i;
    return -1;
}

// kgpu_upload_domain_levels: every level's domain_lists, one level after another in one off[] and one nodes[].  Level
// l's D_l domains have their ranges at off[base_l .. base_l + D_l], and those ranges index the shared nodes[]; level 0
// comes first with base 0, so off[0 .. D_0] and nodes[] read alone are level 0's domain_lists (what the level-0-only
// callers read).  Domain d of level l is the table's domain base_l + d.  For the chunked walk every domain's list is cut
// into chunks of DOM_CHUNK entries, numbered over the whole table in list order: chunk c is nodes[chunk_begin[c] ..
// chunk_begin[c + 1]), domain g's chunks are chunk[g] .. chunk[g + 1] (chunk[] laid out as off[]), level l's are
// chunk0 .. chunk0 + C - 1.  largest: the level's largest domain, which picks its walk (domain_level_chunked).
struct DomainLevel {
    int32_t D, base;
    int64_t largest, chunk0, C;
};
struct DomainTable {
    std::vector<int32_t> off, nodes, chunk, chunk_begin = {0};
    std::vector<DomainLevel> level;
};
// Why domain_table refused an upload: kind out_of_range: domain[level][node] = id is outside -1..n-1; no_parent: node
// is in level-`level` domain id but in no level + 1 domain (other = -1); split: level-`level` domain id has node
// other_node in level + 1 domain other and node `node` in level + 1 domain other2.
struct DomainTableError {
    enum Kind { none, out_of_range, no_parent, split } kind = none;
    int level = 0;
    int64_t node = -1, other_node = -1;
    int32_t id = 0, other = 0, other2 = 0;
};
// domain[levels][n]: builds t, or leaves it untouched and says why not.  Nesting: a node with a level-l domain has a
// level-(l + 1) domain, the same one for every node of its level-l domain (one pass per level).
inline DomainTableError domain_table(const int32_t *domain, int levels, int64_t n, DomainTable &t) {
    DomainTableError err;
    DomainTable out;
    for (int l = 0; l < levels; l++) {
        std::vector<int32_t> off, nodes;
        const int32_t *dl = domain + (int64_t)l * n;
        const int64_t bad = domain_lists(dl, n, off, nodes);
        if (bad >= 0) {
            err.kind = DomainTableError::out_of_range, err.level = l, err.node = bad, err.id = dl[bad];
            return err;
        }
        const int32_t shift = (int32_t)out.nodes.size();
        DomainLevel lv = {(int32_t)off.size() - 1, (int32_t)out.off.size(), 0, (int64_t)out.chunk_begin.size() - 1, 0};
        for (size_t d = 0; d < off.size(); d++) {
            out.off.push_back(off[d] + shift);
            out.chunk.push_back((int32_t)out.chunk_begin.size() - 1);
            if (d + 1 == off.size()) break;
            lv.largest = std::max<int64_t>(lv.largest, off[d + 1] - off[d]);
            for (int32_t e = off[d] + DOM_CHUNK; e < off[d + 1]; e += DOM_CHUNK) out.chunk_begin.push_back(e + shift);
            if (off[d + 1] > off[d]) out.chunk_begin.push_back(off[d + 1] + shift);
        }
        lv.C = (int64_t)out.chunk_begin.size() - 1 - lv.chunk0;
        out.level.push_back(lv);
        out.nodes.insert(out.nodes.end(), nodes.begin(), nodes.end());
    }
    for (int l = 0; l + 1 < levels; l++) {
        const int32_t *dl = domain + (int64_t)l * n, *up = domain + (int64_t)(l + 1) * n;
        std::vector<int64_t> first((size_t)out.level[(size_t)l].D, -1);   // the first node seen of each level-l domain
        for (int64_t i = 0; i < n; i++) {
            const int32_t d = dl[i];
            if (d < 0) continue;
            if (up[i] < 0) {
                err.kind = DomainTableError::no_parent, err.level = l, err.node = i, err.id = d, err.other = -1;
                return err;
            }
            int64_t &f = first[(size_t)d];
            if (f < 0) f = i;
            else if (up[f] != up[i]) {
                err.kind = DomainTableError::split, err.level = l, err.node = i, err.other_node = f, err.id = d;
                err.other = up[f], err.other2 = up[i];
                return err;
            }
        }
    }
    t = std::move(out);
    return err;
}

// A level whose largest domain has more than DOM_CHUNKED_MIN nodes is walked by chunk minima (a domain_chunk_min launch
// before each of its trials); smaller ones by the plain walk, whose trial is a single launch.  At racks of 8..128 nodes
// the plain walk measures as fast as before the chunked walk existed; at spines of 1024 and more the chunked walk is
// faster (DESIGN.md §6).  force: the chunked walk everywhere (the emulator's test seam, not a user option).
constexpr int64_t DOM_CHUNKED_MIN = 256;
inline bool domain_level_chunked(const DomainLevel &lv, bool force = false) {
    return lv.C > 0 && (force || lv.largest > DOM_CHUNKED_MIN);
}

// The distinct (view, k) pairs v * 9 + k of the members pods[begin .. end) with k in 0..8, view as domain_pod_view
// picks it: the rows domain_chunk_min builds for the step.
inline void domain_pairs(const int32_t *pods, int64_t begin, int64_t end, const PlaceViews &views, std::vector<int32_t> &pairs) {
    const size_t first = pairs.size();
    for (int64_t p = begin; p < end; p++) {
        const int32_t k = pods[4 * p];
        if (k < 0 || k > 8) continue;
        int v = 0;
        for (int j = 1; j < views.n; j++)
            if (pods[4 * p + 3] == views.min_mem[j]) v = j;
        const int32_t pr = v * 9 + k;
        if (std::find(pairs.begin() + (std::ptrdiff_t)first, pairs.end(), pr) == pairs.end()) pairs.push_back(pr);
    }
}

// domain_trial's grid: warp per domain, at most max_blocks blocks (grid-strided beyond), at least one
inline unsigned domain_trial_blocks(int64_t D, int64_t max_blocks) {
    return (unsigned)std::max<int64_t>(1, std::min<int64_t>((D + DOM_WARPS - 1) / DOM_WARPS, max_blocks));
}

// Preemption plans: the batch's columns, the distinct (k, level, min_mem) with k in 1..8, sorted (k first, so warps stay
// on one k); pcol[p] = pod p's column, -1 for k outside 1..8.  lvl must already lie in 0..15.  Both are filled in whatever
// the status: it says which of libkgpu's limits the batch passes, which keep the columns within PLAN_MAX_COLS.
enum class PlanColumns { ok, too_many_min_mem, too_many_views };
inline PlanColumns plan_columns(const int32_t *pods, const int32_t *lvl, int64_t P, std::vector<int4> &cols,
                                std::vector<int32_t> &pcol) {
    std::vector<std::array<int32_t, 3>> trip;
    std::vector<int32_t> mems;
    std::vector<std::pair<int32_t, int32_t>> views;      // (level, min_mem) with level > 0
    for (int64_t p = 0; p < P; p++) {
        const int32_t k = pods[4 * p], need = std::max<int32_t>(0, pods[4 * p + 3]);
        if (k < 0 || k > 8) continue;
        if (need > 0) mems.push_back(need);
        if (lvl[p] > 0) views.push_back({lvl[p], need});
        if (k > 0) trip.push_back({k, lvl[p], need});
    }
    std::sort(trip.begin(), trip.end());
    trip.erase(std::unique(trip.begin(), trip.end()), trip.end());
    std::sort(mems.begin(), mems.end());
    mems.erase(std::unique(mems.begin(), mems.end()), mems.end());
    std::sort(views.begin(), views.end());
    views.erase(std::unique(views.begin(), views.end()), views.end());
    const int ncol = (int)trip.size();           // <= 8 k x (8 level-0 + 32 other views) = PLAN_MAX_COLS
    cols.resize((size_t)ncol);
    for (int c = 0; c < ncol; c++) cols[(size_t)c] = make_int4(trip[(size_t)c][0], trip[(size_t)c][1], trip[(size_t)c][2], 0);
    pcol.assign((size_t)P, -1);
    for (int64_t p = 0; p < P; p++) {
        const int32_t k = pods[4 * p];
        if (k < 1 || k > 8) continue;
        const std::array<int32_t, 3> t = {k, lvl[p], std::max<int32_t>(0, pods[4 * p + 3])};
        pcol[(size_t)p] = (int32_t)(std::lower_bound(trip.begin(), trip.end(), t) - trip.begin());
    }
    if (mems.size() > (size_t)PLACE_MAX_VIEWS - 1) return PlanColumns::too_many_min_mem;
    if (views.size() > 32) return PlanColumns::too_many_views;
    return PlanColumns::ok;
}

// K1s: the largest free count of every SP_THREADS-slot tile of the order, from the class layout alone: class c's nodes
// sit in [start, start + count), every class padded to a multiple of `pad` slots, classes 8 first.
inline std::vector<uint8_t> tile_classes(const int64_t class_count[9], int64_t pad, int64_t n_slots) {
    std::vector<uint8_t> tc((size_t)(n_slots / SP_THREADS), 0);
    int64_t start = 0;
    for (int c = 8; c >= 0; c--) {
        const int64_t cnt = class_count[c];
        if (cnt > 0)
            for (int64_t t = start / SP_THREADS; t <= (start + cnt - 1) / SP_THREADS; t++)
                tc[(size_t)t] = std::max<uint8_t>(tc[(size_t)t], (uint8_t)c);
        start += (cnt + pad - 1) / pad * pad;
    }
    return tc;
}

// The byte-aligned warp key of K1s: every cost < 2^16 <=> 28 * max weight < 65536
inline bool byte_keys(const int32_t *W) {
    for (int i = 0; i < 16; i++)
        if (W[i] > 2340) return false;
    return true;
}

// Which K1s instantiation runs a batch of P pods.  On the work list (use_work), a batch of one chunk is cut into runs of
// tiles and goes to the STREAM instantiation (next tile's record prefetched into registers), at most SP_TMA_PODS pods to
// the TMA one (tiles staged by cp.async.bulk; tma_mode 0 turns it off); a chunk-aligned list takes the chunk tables
// sp_prepare_chunks builds once per launch, otherwise every block sorts its pods itself.  The MEM launch is never a
// streaming one.  sparse_kernel (score_pairs_sparse.cuh) names the instantiation.
inline SparseRoute sparse_route(int64_t P, bool use_work, bool aligned, int tma_mode, const int32_t *W) {
    SparseRoute r;
    r.stream = use_work && P <= kSparseChunk;
    r.tma = r.stream && tma_mode != 0 && P <= SP_TMA_PODS;
    r.prepared = use_work && aligned;
    r.byte_keys = byte_keys(W);
    return r;
}

// The resident blocks the work list is cut for: those of the instantiation that will run it.
inline int64_t sparse_list_resident(int64_t P, int tma_mode, int64_t sm_count, int64_t resident) {
    if (tma_mode != 0 && P <= SP_TMA_PODS) return sm_count * KGPU_SP_TMA_MINBLOCKS;
    if (P <= kSparseChunk) return sm_count * KGPU_SP_STREAM_MINBLOCKS;
    return resident;
}

// Pods per split of a plain (tiles x splits) grid: equal ranges rounded up to whole warps of pods
inline int64_t pods_per_split(int64_t P, int64_t splits) {
    const int64_t per = (P + splits - 1) / splits;
    return (per + 31) / 32 * 32;
}

}  // namespace kgpu
