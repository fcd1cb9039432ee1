// emu_plan_gang.cc -- gang_plan_sequential (preempt_plan.cuh) compiled from the product source with g++ against
// tests/emu/cuda_emu.h and run on the CPU.  TEST INFRASTRUCTURE ONLY: tests/test_preempt_plan_gang.py builds it and
// checks it against the CPU twin (plan_gang_twin.c).  It includes emu_plan.cc, so the library also exports
// emu_preempt_plan.
#include "../preempt_plan_twin/emu_plan.cc"

extern "C" {

// kgpu_preempt_plan_gang as it launches the kernels, with the same column list.  Returns the number of columns.
int emu_preempt_plan_gang(const int32_t *topo, const int32_t *free_mask, const int32_t *gpu_mem /*nullable*/,
                          const int32_t *hold /*nullable*/, int64_t n, int64_t node_id_base, const int32_t *pods, const int32_t *lvl,
                          const int32_t *gang, int64_t P, const int32_t *W, unsigned long long *keys, uint32_t *victims) {
    std::vector<std::array<int32_t, 3>> trip;
    for (int64_t p = 0; p < P; p++)
        if (pods[4 * p] >= 1 && pods[4 * p] <= 8) trip.push_back({pods[4 * p], lvl[p], std::max<int32_t>(0, pods[4 * p + 3])});
    std::sort(trip.begin(), trip.end());
    trip.erase(std::unique(trip.begin(), trip.end()), trip.end());
    const int ncol = (int)trip.size();
    if (ncol > kgpu::PLAN_MAX_COLS) return -1;
    int4 *cols = aligned_array<int4>((size_t)ncol);
    for (int c = 0; c < ncol; c++) cols[c] = make_int4(trip[(size_t)c][0], trip[(size_t)c][1], trip[(size_t)c][2], 0);
    int32_t *pcol = aligned_array<int32_t>((size_t)P);
    for (int64_t p = 0; p < P; p++) {
        pcol[p] = -1;
        if (pods[4 * p] < 1 || pods[4 * p] > 8) continue;
        const std::array<int32_t, 3> t = {pods[4 * p], lvl[p], std::max<int32_t>(0, pods[4 * p + 3])};
        pcol[p] = (int32_t)(std::lower_bound(trip.begin(), trip.end(), t) - trip.begin());
    }
    const int64_t T = (n + kgpu::PLAN_TILE - 1) / kgpu::PLAN_TILE, Npad = T * kgpu::PLAN_TILE;
    int4 *topo4 = aligned_array<int4>((size_t)n * 16);
    std::memcpy(topo4, topo, (size_t)n * 256);
    int4 *pods4 = aligned_array<int4>((size_t)P);
    std::memcpy(pods4, pods, (size_t)P * 16);
    int32_t *gang_ids = aligned_array<int32_t>((size_t)P);
    std::memcpy(gang_ids, gang, (size_t)P * 4);
    int4 *pre = aligned_array<int4>((size_t)P);
    int4 *mem4 = aligned_array<int4>((size_t)n * 2);
    if (gpu_mem) std::memcpy(mem4, gpu_mem, (size_t)n * 32); else std::memset(mem4, 0x7F, (size_t)n * 32);
    int32_t *F = aligned_array<int32_t>((size_t)n);
    std::memcpy(F, free_mask, (size_t)n * 4);
    int32_t *H = aligned_array<int32_t>((size_t)n * 8);
    if (hold) std::memcpy(H, hold, (size_t)n * 32); else std::memset(H, 0xFF, (size_t)n * 32);
    unsigned long long *nodekey = aligned_array<unsigned long long>((size_t)(ncol * Npad));
    unsigned long long *tilekey = aligned_array<unsigned long long>((size_t)(ncol * T));
    kgpu::Weights Ws;
    std::memcpy(Ws.w, W, sizeof Ws.w);
    if (n > 0 && ncol > 0) {
        const unsigned groups = (unsigned)((ncol + kgpu::PLAN_INIT_COLS - 1) / kgpu::PLAN_INIT_COLS);
        emu::launch(dim3((unsigned)T, groups), dim3(kgpu::PLAN_TILE), [&] {
            kgpu::plan_init(topo4, F, mem4, reinterpret_cast<const int4 *>(H), n, Npad, T, cols, ncol, Ws, kPC, nodekey, tilekey);
        });
    }
    if (n > 0) {
        emu::launch(dim3(1), dim3(kgpu::PLAN_THREADS), [&] {
            kgpu::gang_plan_sequential(topo4, F, mem4, H, n, Npad, T, node_id_base, pods4, pcol, P, cols, ncol, Ws, kPC, nodekey,
                                       tilekey, keys, victims, gang_ids, pre);
        });
    } else {
        for (int64_t p = 0; p < P; p++) { keys[p] = ~0ull; victims[p] = 0; }
    }
    free(cols); free(pcol); free(topo4); free(pods4); free(gang_ids); free(pre); free(mem4); free(F); free(H); free(nodekey);
    free(tilekey);
    return ncol;
}

}  // extern "C"
