// emu_gang_domain.cc -- kgpu_place_batch_gang_domain's launches run on the CPU through tests/emu/cuda_emu.h: the real
// kernel sources (place_sequential.cuh, gang_domain.cuh) and the real launch plan (launch_plan.h: place_views,
// place_segments, domain_lists, domain_trial_blocks).  TEST INFRASTRUCTURE ONLY; tests/gang_domain_libs.py builds it
// into a temporary directory.  One translation unit: the kernel headers define globals (c_subsets, ...).
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

// place_init + place_half_tables, then the segments of place_segments as kgpu_place_batch_gang_domain launches them:
// place_sequential (GANG when gang != nullptr) on each pod range without a constrained gang, domain_trial +
// domain_commit for each constrained gang.  The caller has checked the gang ids and gang_domain values as libkgpu does.
// domain[n] is the node's domain (nullable: every node -1); gpu_mem nullable (unconstrained, INT32_MAX MiB, as in
// kgpu.cu).  free_mask is updated in place like the device copy.  Returns the number of domain steps, or -1 for too many
// views or a bad domain value.
int emu_place_batch_gang_domain(const int32_t *topo, int32_t *free_mask, const int32_t *gpu_mem, int64_t n, int64_t node_id_base,
                                const int32_t *domain, const int32_t *pods, const int32_t *gang, const int32_t *gang_domain, int64_t P,
                                const int32_t *W, unsigned long long *keys) {
    std::memset(keys, 0xFF, (size_t)P * 8);
    std::vector<int32_t> doff(1, 0), dnodes;
    if (domain && kgpu::domain_lists(domain, n, doff, dnodes) >= 0) return -1;
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
    const int32_t D = (int32_t)doff.size() - 1;
    kgpu::DomainArgs da{free_mask, mem, Npad, T, node_id_base, views, nodebest, tilebest, half_all,
                        st.array<int32_t>(doff.size(), doff.data()), st.array<int32_t>(dnodes.size(), dnodes.data()),
                        st.array<int32_t>((size_t)n), st.array<uint32_t>((size_t)n)};
    int steps = 0;
    for (const kgpu::PlaceSegment &sg : kgpu::place_segments(gang, gang_domain, P)) {
        const int64_t p0 = sg.begin, np = sg.end - sg.begin;
        if (sg.mode != 0) {
            const uint32_t stamp = (uint32_t)(2 * steps + 1);
            unsigned long long best = ~0ull;
            emu::launch(dim3(kgpu::domain_trial_blocks(D, 4)), dim3(kgpu::DOM_THREADS),
                        [&] { kgpu::domain_trial(da, pods4 + p0, np, D, stamp, &best); });
            emu::launch(dim3(1), dim3(kgpu::DOM_COMMIT_THREADS),
                        [&] { kgpu::domain_commit(da, pods4 + p0, np, sg.mode, stamp + 1, &best, keys + p0); });
            steps++;
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
    }
    return steps;
}

}  // extern "C"
