// emu_plan_domain.cc -- kgpu_preempt_plan_gang_domain's launches run on the CPU through tests/emu/cuda_emu.h: the real
// kernel sources (preempt_plan.cuh, preempt_plan_domain.cuh) and the real launch plan (launch_plan.h: plan_columns,
// place_segments, domain_lists, domain_trial_blocks).  TEST INFRASTRUCTURE ONLY; tests/preempt_plan_domain_libs.py
// builds it into a temporary directory.  One translation unit: the kernel headers define globals (c_subsets, ...).
#include "cuda_emu.h"

#include <algorithm>
#include <cstdlib>
#include <vector>

#include "score_pairs.cuh"
#include "place_sequential.cuh"
#include "preempt_plan.cuh"
#include "preempt_plan_domain.cuh"
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

// plan_init, then the segments of place_segments as kgpu_preempt_plan_gang_domain launches them: plan_sequential
// (gang_plan_sequential when gang != nullptr) on each pod range without a constrained gang, domain_plan_trial +
// domain_plan_commit for each constrained gang.  The caller has checked gang ids and gang_domain values as libkgpu does.
// domain[n] is the node's domain (nullable: every node -1); gpu_mem and hold nullable as in kgpu.cu.  free_mask and
// hold (when given) are the working state (F, H) and are updated in place, so the caller sees the final state.
// Returns the number of domain steps, or -1 for too many columns or a bad domain value.
int emu_preempt_plan_gang_domain(const int32_t *topo, int32_t *free_mask, const int32_t *gpu_mem, int32_t *hold, int64_t n,
                                 int64_t node_id_base, const int32_t *domain, const int32_t *pods, const int32_t *lvl,
                                 const int32_t *gang, const int32_t *gang_domain, int64_t P, const int32_t *W,
                                 unsigned long long *keys, uint32_t *victims) {
    std::vector<int32_t> doff(1, 0), dnodes;
    if (domain && kgpu::domain_lists(domain, n, doff, dnodes) >= 0) return -1;
    std::vector<int4> colv;
    std::vector<int32_t> pcolv;
    kgpu::plan_columns(pods, lvl, P, colv, pcolv);
    const int ncol = (int)colv.size();
    if (ncol > kgpu::PLAN_MAX_COLS) return -1;
    if (n == 0 || P == 0) {
        for (int64_t p = 0; p < P; p++) { keys[p] = ~0ull; victims[p] = 0; }
        return 0;
    }
    kgpu::subset_tables(kgpu::c_subsets, kgpu::c_nsub);
    Staging st;
    const int4 *cols = st.array<int4>((size_t)ncol, colv.data()), *topo4 = st.array<int4>((size_t)n * 16, topo);
    const int4 *pods4 = st.array<int4>((size_t)P, pods);
    const int32_t *pcol = st.array<int32_t>((size_t)P, pcolv.data());
    int32_t *mem = st.array<int32_t>((size_t)n * 8, gpu_mem);
    if (!gpu_mem) std::fill(mem, mem + n * 8, INT32_MAX);
    const int4 *mem4 = reinterpret_cast<const int4 *>(mem);
    int32_t *H = st.array<int32_t>((size_t)n * 8, hold);
    if (!hold) std::fill(H, H + n * 8, -1);
    const int64_t T = (n + kgpu::PLAN_TILE - 1) / kgpu::PLAN_TILE, Npad = T * kgpu::PLAN_TILE;
    unsigned long long *nodekey = st.array<unsigned long long>((size_t)(ncol * Npad));
    unsigned long long *tilekey = st.array<unsigned long long>((size_t)(ncol * T));
    kgpu::Weights Ws;
    std::memcpy(Ws.w, W, sizeof Ws.w);
    if (ncol > 0) {
        const unsigned groups = (unsigned)((ncol + kgpu::PLAN_INIT_COLS - 1) / kgpu::PLAN_INIT_COLS);
        emu::launch(dim3((unsigned)T, groups), dim3(kgpu::PLAN_TILE), [&] {
            kgpu::plan_init(topo4, free_mask, mem4, reinterpret_cast<const int4 *>(H), n, Npad, T, cols, ncol, Ws, kPC, nodekey, tilekey);
        });
    }
    const int32_t D = (int32_t)doff.size() - 1;
    const int32_t *gang_ids = gang ? st.array<int32_t>((size_t)P, gang) : nullptr;
    int4 *pre = st.array<int4>((size_t)P);
    unsigned long long *score = st.array<unsigned long long>((size_t)std::max<int32_t>(1, D));
    kgpu::PlanDomainArgs da{topo4, free_mask, mem4, H, n, Npad, T, node_id_base, cols, ncol, nodekey, tilekey,
                            st.array<int32_t>(doff.size(), doff.data()), st.array<int32_t>(dnodes.size(), dnodes.data()),
                            st.array<int32_t>((size_t)n), st.array<uint2>((size_t)n), st.array<uint32_t>((size_t)n)};
    int steps = 0;
    for (const kgpu::PlaceSegment &sg : kgpu::place_segments(gang, gang_domain, P)) {
        const int64_t p0 = sg.begin, np = sg.end - sg.begin;
        if (sg.mode != 0) {
            const uint32_t stamp = (uint32_t)(2 * steps + 1);
            emu::launch(dim3(kgpu::domain_trial_blocks(D, 4)), dim3(kgpu::DOM_THREADS),
                        [&] { kgpu::domain_plan_trial(da, Ws, kPC, pods4 + p0, pcol + p0, np, D, stamp, score); });
            emu::launch(dim3(1), dim3(kgpu::PLAN_THREADS), [&] {
                kgpu::domain_plan_commit(da, Ws, kPC, pods4 + p0, pcol + p0, gang_ids + p0, np, sg.mode, D, stamp + 1, score, keys + p0,
                                         victims + p0, pre + p0);
            });
            steps++;
            continue;
        }
        emu::launch(dim3(1), dim3(kgpu::PLAN_THREADS), [&] {
            if (gang)
                kgpu::gang_plan_sequential(topo4, free_mask, mem4, H, n, Npad, T, node_id_base, pods4 + p0, pcol + p0, np, cols, ncol, Ws,
                                           kPC, nodekey, tilekey, keys + p0, victims + p0, gang_ids + p0, pre + p0);
            else
                kgpu::plan_sequential(topo4, free_mask, mem4, H, n, Npad, T, node_id_base, pods4 + p0, pcol + p0, np, cols, ncol, Ws, kPC,
                                      nodekey, tilekey, keys + p0, victims + p0);
        });
    }
    if (hold) std::memcpy(hold, H, (size_t)n * 32);
    return steps;
}

}  // extern "C"
