// emu_gang.cc -- the gang instantiation of K3 (place_sequential<true>) compiled from the product source with g++
// against tests/emu/cuda_emu.h and run on the CPU.  TEST INFRASTRUCTURE ONLY: tests/test_gang_placement.py builds it
// and checks it against the CPU twin (gang_twin.c).
#include "cuda_emu.h"

#include <algorithm>
#include <cstdlib>

#include "place_sequential.cuh"

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

// K3 with gangs: place_init + place_half_tables + place_sequential<true> with gang[P], as kgpu_place_batch_gang launches
// them (views from the batch's distinct min_mem values; the caller has checked that every gang id forms one run);
// free_mask is updated in place like the device copy.  Returns 0, or -1 for too many views.
int emu_place_batch_gang(const int32_t *topo, int32_t *free_mask, const int32_t *gpu_mem /*nullable*/, int64_t n,
                         int64_t node_id_base, const int32_t *pods, const int32_t *gang, int64_t P, const int32_t *W,
                         unsigned long long *keys) {
    std::memset(keys, 0xFF, (size_t)P * 8);
    if (n == 0 || P == 0) return 0;
    kgpu::PlaceViews views;
    std::memset(&views, 0, sizeof views);
    views.n = 1;
    for (int64_t p = 0; p < P; p++) {
        const int32_t need = pods[4 * p + 3];
        if (need <= 0 || pods[4 * p] < 0 || pods[4 * p] > 8) continue;
        bool seen = false;
        for (int j = 1; j < views.n; j++) seen = seen || views.min_mem[j] == need;
        if (seen) continue;
        if (views.n == kgpu::PLACE_MAX_VIEWS) return -1;
        views.min_mem[views.n++] = need;
    }
    for (int k = 0; k <= 8; k++) {
        int c = 0;
        for (unsigned S = 0; S < 256; S++)
            if (__builtin_popcount(S) == k) kgpu::c_subsets[k][c++] = (uint8_t)S;
        kgpu::c_nsub[k] = (uint8_t)c;
    }
    int4 *topo4 = aligned_array<int4>((size_t)n * 16);
    std::memcpy(topo4, topo, (size_t)n * 256);
    int4 *pods4 = aligned_array<int4>((size_t)P);
    std::memcpy(pods4, pods, (size_t)P * 16);
    int32_t *mem = aligned_array<int32_t>((size_t)n * 8);
    if (gpu_mem) std::memcpy(mem, gpu_mem, (size_t)n * 32); else std::memset(mem, 0x7F, (size_t)n * 32);
    const int64_t T = (n + kgpu::PLACE_TILE - 1) / kgpu::PLACE_TILE, Npad = T * kgpu::PLACE_TILE;
    uint32_t *nodebest = aligned_array<uint32_t>((size_t)Npad * 9 * views.n);
    unsigned long long *tilebest = aligned_array<unsigned long long>((size_t)T * 9 * views.n);
    kgpu::Weights Ws;
    std::memcpy(Ws.w, W, sizeof Ws.w);
    emu::launch(dim3((unsigned)T, (unsigned)views.n), dim3(kgpu::PLACE_TILE),
                [&] { kgpu::place_init(topo4, free_mask, mem, n, Npad, node_id_base, Ws, kPC, views, nodebest, tilebest, T); });
    int32_t *half_all = aligned_array<int32_t>((size_t)Npad * kgpu::PLACE_HALF);
    emu::launch(dim3((unsigned)std::min<int64_t>((n + 3) / 4, 8)), dim3(128),
                [&] { kgpu::place_half_tables(reinterpret_cast<const int32_t *>(topo4), n, Ws, half_all); });
    emu::launch(dim3(1), dim3(kgpu::PLACE_THREADS), [&] {
        kgpu::place_sequential<true>(reinterpret_cast<const int32_t *>(topo4), free_mask, mem, n, Npad, node_id_base, pods4, P, Ws,
                                     views, nodebest, tilebest, T, half_all, keys, gang);
    });
    free(topo4); free(pods4); free(mem); free(nodebest); free(tilebest); free(half_all);
    return 0;
}

}  // extern "C"
