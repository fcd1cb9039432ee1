// emu_preempt.cc -- the preemption kernels (preempt.cuh) compiled from the product source with g++ against
// tests/emu/cuda_emu.h and run on the CPU.  TEST INFRASTRUCTURE ONLY: tests/test_preemption.py builds it and checks it
// against the CPU twin (preempt_twin.c).
#include "cuda_emu.h"

#include <algorithm>
#include <cstdlib>

#include "preempt.cuh"

namespace {

const kgpu::PipeConsts kPC = {1u, 0xFFFFFFFFu};

template <class T>
T *aligned_array(size_t n) {
    void *p = nullptr;
    if (posix_memalign(&p, 64, std::max<size_t>(64, n * sizeof(T))) != 0) abort();
    std::memset(p, 0, std::max<size_t>(64, n * sizeof(T)));
    return (T *)p;
}

}  // namespace

extern "C" {

// Steps 2-3 of kgpu_preempt_batch as it launches them: keys[P] holds the scoring path's keys on entry (the caller
// computes them with the oracle) and the preemption keys on return; victims[P] is zeroed first.  splits = the grid's
// pod dimension.  Returns how many pods reached the preemption kernel.
int emu_preempt_batch(const int32_t *topo, const int32_t *free_mask, const int32_t *gpu_mem /*nullable*/,
                      const int32_t *hold /*nullable*/, int64_t n, int64_t node_id_base, const int32_t *pods,
                      const int32_t *lvl, int64_t P, const int32_t *W, int splits, unsigned long long *keys,
                      uint32_t *victims) {
    std::memset(victims, 0, (size_t)P * 4);
    if (n == 0 || P == 0 || !hold) return 0;
    int4 *topo4 = aligned_array<int4>((size_t)n * 16);
    std::memcpy(topo4, topo, (size_t)n * 256);
    int4 *pods4 = aligned_array<int4>((size_t)P);
    std::memcpy(pods4, pods, (size_t)P * 16);
    int4 *mem4 = aligned_array<int4>((size_t)n * 2);
    if (gpu_mem) std::memcpy(mem4, gpu_mem, (size_t)n * 32); else std::memset(mem4, 0x7F, (size_t)n * 32);
    int4 *hold4 = aligned_array<int4>((size_t)n * 2);
    std::memcpy(hold4, hold, (size_t)n * 32);
    int32_t *idx = aligned_array<int32_t>((size_t)P);
    unsigned long long *pkey = aligned_array<unsigned long long>((size_t)P);
    std::memset(pkey, 0xFF, (size_t)P * 8);
    int count = 0;
    kgpu::Weights Ws;
    std::memcpy(Ws.w, W, sizeof Ws.w);
    const unsigned pb = (unsigned)((P + 127) / 128);
    emu::launch(dim3(pb), dim3(128), [&] { kgpu::preempt_compact(pods4, lvl, keys, P, idx, &count); });
    const unsigned tiles = (unsigned)((n + kgpu::PRE_THREADS - 1) / kgpu::PRE_THREADS);
    emu::launch(dim3(tiles, (unsigned)splits), dim3(kgpu::PRE_THREADS), [&] {
        kgpu::preempt_lane_per_node(topo4, free_mask, mem4, hold4, n, pods4, lvl, idx, &count, Ws, kPC, pkey);
    });
    emu::launch(dim3(pb), dim3(128), [&] {
        kgpu::preempt_finalize(pkey, idx, &count, free_mask, reinterpret_cast<const int32_t *>(hold4), node_id_base, keys, victims);
    });
    free(topo4); free(pods4); free(mem4); free(hold4); free(idx); free(pkey);
    return count;
}

}  // extern "C"
