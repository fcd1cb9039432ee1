// emu_levels.cc -- kgpu_place_batch_gang_levels' launches run on the CPU through tests/emu/cuda_emu.h: the real kernel
// sources (place_sequential.cuh, gang_domain.cuh) and the real host plans (launch_plan.h: domain_table, place_views,
// place_segments, domain_trial_blocks), launched as kgpu.cu launches them.  TEST INFRASTRUCTURE ONLY;
// tests/test_gang_domain_levels.py builds it into a temporary directory.  One translation unit: the kernel headers define
// globals (c_subsets, ...).
#include "cuda_emu.h"

#include <algorithm>
#include <cstdlib>
#include <vector>

#include "score_pairs.cuh"
#include "place_sequential.cuh"
#include "gang_domain.cuh"
#include "launch_plan.h"

namespace {

const kgpu::PipeConsts kPC = {1u, 0xFFFFFFFFu};

// The device arrays of one call: 64-byte aligned (the kernels load int4), zero-filled, freed when the call returns.
struct Staging {
    std::vector<void *> owned;
    Staging() = default;
    Staging(const Staging &) = delete;
    ~Staging() {
        for (void *p : owned) free(p);
    }
    template <class T>
    T *array(size_t n, const void *src = nullptr) {
        void *p = nullptr;
        const size_t bytes = std::max<size_t>(64, n * sizeof(T));
        if (posix_memalign(&p, 64, bytes) != 0) abort();
        std::memset(p, 0, bytes);
        if (src && n) std::memcpy(p, src, n * sizeof(T));
        owned.push_back(p);
        return (T *)p;
    }
};

}  // namespace

extern "C" {

// domain_table on domain[levels][n]: 0 and the table's sizes (D per level in D_out[levels], total off and node entries
// in sizes[2]), or the error kind (launch_plan.h: DomainTableError) with info[6] = {level, node, other_node, id, other,
// other2}.
int emu_domain_table(const int32_t *domain, int levels, int64_t n, int32_t *D_out, int64_t *sizes, int64_t *info) {
    kgpu::DomainTable t;
    const kgpu::DomainTableError e = kgpu::domain_table(domain, levels, n, t);
    if (e.kind != kgpu::DomainTableError::none) {
        const int64_t v[6] = {e.level, e.node, e.other_node, e.id, e.other, e.other2};
        std::memcpy(info, v, sizeof v);
        return (int)e.kind;
    }
    for (int l = 0; l < levels; l++) D_out[l] = t.level[(size_t)l].D;
    sizes[0] = (int64_t)t.off.size(), sizes[1] = (int64_t)t.nodes.size();
    return 0;
}

// place_init + place_half_tables, then the segments of place_segments as kgpu_place_batch_gang_levels launches them:
// place_sequential (GANG when gang != nullptr) on each pod range without a constrained gang; for each constrained gang
// one domain_trial per level 0..gang_level, then domain_commit.  domain[levels][n] (nullable: one level, every node
// -1); gang_level nullable (all 0); gpu_mem nullable (INT32_MAX MiB, as in kgpu.cu).  The caller has checked the inputs
// as libkgpu does.  free_mask is updated in place like the device copy.  force_chunked: every level with a domain is
// walked by chunk minima, whatever its size (domain_level_chunked's test seam).  Returns the number of launches, or -1
// for too many views or a table domain_table refuses.
int emu_place_batch_gang_levels(const int32_t *topo, int32_t *free_mask, const int32_t *gpu_mem, int64_t n, int64_t node_id_base,
                                const int32_t *domain, int levels, const int32_t *pods, const int32_t *gang,
                                const int32_t *gang_domain, const int32_t *gang_level, int64_t P, const int32_t *W,
                                unsigned long long *keys, int force_chunked) {
    std::memset(keys, 0xFF, (size_t)P * 8);
    kgpu::DomainTable tab;
    tab.off = {0}, tab.level = {{0, 0}};
    if (domain && kgpu::domain_table(domain, levels, n, tab).kind != kgpu::DomainTableError::none) return -1;
    if (n == 0 || P == 0) return 0;
    kgpu::PlaceViews views;
    if (!kgpu::place_views(pods, P, views)) return -1;
    kgpu::subset_tables(kgpu::c_subsets, kgpu::c_nsub);
    Staging st;
    const int4 *topo4 = st.array<int4>((size_t)n * 16, topo), *pods4 = st.array<int4>((size_t)P, pods);
    const int32_t *topo32 = reinterpret_cast<const int32_t *>(topo4);
    int32_t *mem = st.array<int32_t>((size_t)n * 8, gpu_mem);
    if (!gpu_mem) std::fill(mem, mem + n * 8, INT32_MAX);
    const int64_t T = (n + kgpu::PLACE_TILE - 1) / kgpu::PLACE_TILE, Npad = T * kgpu::PLACE_TILE;
    uint32_t *nodebest = st.array<uint32_t>((size_t)Npad * 9 * views.n);
    unsigned long long *tilebest = st.array<unsigned long long>((size_t)T * 9 * views.n);
    int32_t *half_all = st.array<int32_t>((size_t)Npad * kgpu::PLACE_HALF);
    kgpu::Weights Ws;
    std::memcpy(Ws.w, W, sizeof Ws.w);
    emu::launch(dim3((unsigned)T, (unsigned)views.n), dim3(kgpu::PLACE_TILE),
                [&] { kgpu::place_init(topo4, free_mask, mem, n, Npad, node_id_base, Ws, kPC, views, nodebest, tilebest, T); });
    emu::launch(dim3((unsigned)std::min<int64_t>((n + 3) / 4, 8)), dim3(128), [&] { kgpu::place_half_tables(topo32, n, Ws, half_all); });
    int launches = 2;
    kgpu::DomainArgs da{free_mask, mem, Npad, T, node_id_base, views, nodebest, tilebest, half_all,
                        st.array<int32_t>(tab.off.size(), tab.off.data()), st.array<int32_t>(tab.nodes.size(), tab.nodes.data()),
                        st.array<int32_t>((size_t)n), st.array<uint32_t>((size_t)n)};
    const std::vector<kgpu::PlaceSegment> segs = kgpu::place_segments(gang, gang_domain, P, gang_level);
    int64_t trials = 0;
    std::vector<int32_t> pairs;
    std::vector<int64_t> pair_at;
    for (const kgpu::PlaceSegment &sg : segs) {
        if (sg.mode == 0) continue;
        trials += sg.level + 1;
        pair_at.push_back((int64_t)pairs.size());
        bool chunked = false;
        for (int32_t l = 0; l <= sg.level; l++) chunked = chunked || kgpu::domain_level_chunked(tab.level[(size_t)l], force_chunked != 0);
        if (chunked) kgpu::domain_pairs(pods, sg.begin, sg.end, views, pairs);
    }
    pair_at.push_back((int64_t)pairs.size());
    const int64_t chunks = (int64_t)tab.chunk_begin.size() - 1;
    if (!pairs.empty()) {
        da.dom_chunk = st.array<int32_t>(tab.chunk.size(), tab.chunk.data());
        da.chunk_begin = st.array<int32_t>(tab.chunk_begin.size(), tab.chunk_begin.data());
        da.cmin = st.array<unsigned long long>((size_t)(views.n * 9 * chunks));
        da.cstamp = st.array<uint32_t>((size_t)chunks);
        da.chunks = chunks;
    }
    const int32_t *pairs_dev = st.array<int32_t>(pairs.size(), pairs.data());
    std::vector<unsigned long long> best((size_t)std::max<int64_t>(1, trials), ~0ull);
    int64_t slot = 0, step = 0;
    uint32_t stamp = 0;
    for (const kgpu::PlaceSegment &sg : segs) {
        const int64_t p0 = sg.begin, np = sg.end - sg.begin;
        if (sg.mode != 0) {
            int32_t chunked_levels = 0;
            const int64_t npair = pair_at[(size_t)step + 1] - pair_at[(size_t)step];
            for (int32_t l = 0; l <= sg.level; l++) {
                const kgpu::DomainLevel lv = tab.level[(size_t)l];
                const bool chunked = kgpu::domain_level_chunked(lv, force_chunked != 0) && npair > 0;
                if (chunked) {
                    emu::launch(dim3(kgpu::domain_trial_blocks(lv.C, 4), (unsigned)npair), dim3(kgpu::DOM_THREADS), [&] {
                        kgpu::domain_chunk_min(da, lv.chunk0, lv.C, pairs_dev + pair_at[(size_t)step], best.data() + slot, l);
                    });
                    launches++;
                }
                chunked_levels |= chunked ? 1 << l : 0;
                const uint32_t s = ++stamp;
                emu::launch(dim3(kgpu::domain_trial_blocks(lv.D, 4)), dim3(kgpu::DOM_THREADS),
                            [&] { kgpu::domain_trial(da, pods4 + p0, np, lv.D, s, best.data() + slot, l, lv.base, chunked ? 1 : 0); });
            }
            const uint32_t s = ++stamp;
            emu::launch(dim3(1), dim3(kgpu::DOM_COMMIT_THREADS), [&] {
                kgpu::domain_commit(da, pods4 + p0, np, sg.mode, s, best.data() + slot, keys + p0, sg.level + 1, chunked_levels);
            });
            slot += sg.level + 1;
            step++;
            launches += sg.level + 2;
            continue;
        }
        emu::launch(dim3(1), dim3(kgpu::PLACE_THREADS), [&] {
            if (gang)
                kgpu::place_sequential<true>(topo32, free_mask, mem, n, Npad, node_id_base, pods4 + p0, np, Ws, views, nodebest, tilebest,
                                             T, half_all, keys + p0, gang + p0);
            else
                kgpu::place_sequential(topo32, free_mask, mem, n, Npad, node_id_base, pods4 + p0, np, Ws, views, nodebest, tilebest, T,
                                       half_all, keys + p0);
        });
        launches++;
    }
    return launches;
}

}  // extern "C"
