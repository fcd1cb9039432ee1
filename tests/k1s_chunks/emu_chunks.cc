// emu_chunks.cc -- K1s's per-launch chunk tables (sp_prepare_chunks, score_pairs_sparse.cuh) compiled from the product
// source with g++ against tests/emu/cuda_emu.h and run on the CPU.  TEST INFRASTRUCTURE ONLY:
// tests/test_k1s_chunk_tables.py builds it and checks the prepared tables against the block's own pod sort and the
// prepared-path keys against the oracle and the in-kernel path.
#include "cuda_emu.h"

#include <algorithm>
#include <cstdlib>
#include <vector>

#include "score_pairs.cuh"
#include "score_pairs_sparse.cuh"
#include "sparse_work.h"
#include "node_state.cuh"

namespace {

const kgpu::PipeConsts kPC = {1u, 0xFFFFFFFFu};

template <class T>
T *aligned_array(size_t n) {
    void *p = nullptr;
    if (posix_memalign(&p, 64, std::max<size_t>(64, n * sizeof(T))) != 0) abort();
    std::memset(p, 0, std::max<size_t>(64, n * sizeof(T)));
    return (T *)p;
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

struct Cache {
    std::vector<int32_t> order, slot_of;
    int4 *rec = nullptr;
    uint32_t *meta = nullptr;
    int64_t n_slots = 0;
    ~Cache() { free(rec); free(meta); }
};

// build_order + ensure_node_cache of kgpu.cu: the device-side counting sort of the nodes, then the compacted records
void build_cache(const int4 *topo4, int32_t *free_mask, int64_t n, const kgpu::Weights &Ws, Cache &c) {
    const int nb = (int)((n + kgpu::ORD_BLOCK - 1) / kgpu::ORD_BLOCK);
    const int64_t cap = (n + 11 * kgpu::SP_THREADS) / kgpu::SP_THREADS * kgpu::SP_THREADS;
    c.order.assign((size_t)cap, -1);
    c.slot_of.assign((size_t)std::max<int64_t>(1, n), -1);
    std::vector<int32_t> cnt((size_t)nb * 9), off((size_t)nb * 9);
    long long meta[kgpu::ORD_META] = {0};
    emu::launch(dim3((unsigned)nb), dim3(kgpu::ORD_BLOCK), [&] { kgpu::order_count(free_mask, n, cnt.data(), nb); });
    emu::launch(dim3(1), dim3(kgpu::ORD_BLOCK), [&] { kgpu::order_scan(cnt.data(), nb, off.data(), meta, kgpu::SP_THREADS, 32); });
    emu::launch(dim3((unsigned)nb), dim3(kgpu::ORD_BLOCK),
                [&] { kgpu::order_scatter(free_mask, n, off.data(), nb, c.order.data(), c.slot_of.data()); });
    c.n_slots = meta[9];
    c.rec = aligned_array<int4>(c.order.size() * 7);
    c.meta = aligned_array<uint32_t>(c.order.size());
    emu::launch(dim3((unsigned)(c.n_slots / kgpu::SP_THREADS)), dim3(kgpu::SP_THREADS),
                [&] { kgpu::compact_nodes(topo4, free_mask, c.n_slots, Ws, c.order.data(), c.slot_of.data(), c.rec, c.meta); });
}

}  // namespace

extern "C" {

int emu_chunk_int4() { return kgpu::SP_CHUNK_INT4; }
int emu_chunk_pos() { return kgpu::SP_POS; }

// Both tables of every chunk of the batch, [chunks][SP_CHUNK_INT4] int4 each: sp_prepare_chunks<mem> into `prepared`,
// the block's own sort into `sorted`.  Returns the chunk count.
int64_t emu_chunk_tables(const int32_t *pods, int64_t P, int mem, int32_t *prepared, int32_t *sorted) {
    const int64_t chunks = (P + kgpu::SP_CHUNK - 1) / kgpu::SP_CHUNK;
    int4 *pods4 = aligned_array<int4>((size_t)P);
    std::memcpy(pods4, pods, (size_t)P * 16);
    int4 *prep = aligned_array<int4>((size_t)chunks * kgpu::SP_CHUNK_INT4);
    int4 *sort = aligned_array<int4>((size_t)chunks * kgpu::SP_CHUNK_INT4);
    int flag = 1;
    emu::launch(dim3((unsigned)chunks), dim3(kgpu::SP_THREADS), [&] {
        if (mem) kgpu::sp_prepare_chunks<true>(pods4, P, &flag, prep); else kgpu::sp_prepare_chunks<false>(pods4, P, &flag, prep);
    });
    emu::launch(dim3((unsigned)chunks), dim3(kgpu::SP_THREADS), [&] {
        if (mem) block_sort<true>(pods4, P, sort); else block_sort<false>(pods4, P, sort);
    });
    std::memcpy(prepared, prep, (size_t)chunks * kgpu::SP_CHUNK_INT4 * 16);
    std::memcpy(sorted, sort, (size_t)chunks * kgpu::SP_CHUNK_INT4 * 16);
    free(pods4); free(prep); free(sort);
    return chunks;
}

// K1s (and its MEM instantiation when some pod carries min_mem) on the work list of sparse_work.h for `resident` blocks,
// as kgpu.cu launches them: with prepare != 0 each launch is preceded by sp_prepare_chunks and takes its tables (when
// the list is chunk-aligned), otherwise every block sorts its chunks.  Returns 1 if the list was chunk-aligned.
int emu_score_chunks(const int32_t *topo, const int32_t *free_mask_in, const int32_t *gpu_mem /*nullable*/, int64_t n,
                     int64_t node_id_base, const int32_t *pods, int64_t P, const int32_t *W, int64_t resident, int prepare,
                     unsigned long long *keys) {
    std::memset(keys, 0xFF, (size_t)P * 8);
    std::vector<int32_t> free_mask(free_mask_in, free_mask_in + n);
    int4 *topo4 = aligned_array<int4>((size_t)n * 16);
    std::memcpy(topo4, topo, (size_t)n * 256);
    int4 *pods4 = aligned_array<int4>((size_t)P);
    std::memcpy(pods4, pods, (size_t)P * 16);
    int32_t *mem = aligned_array<int32_t>((size_t)n * 8);
    if (gpu_mem) std::memcpy(mem, gpu_mem, (size_t)n * 32); else std::memset(mem, 0x7F, (size_t)n * 32);
    kgpu::Weights Ws;
    std::memcpy(Ws.w, W, sizeof Ws.w);
    Cache c;
    build_cache(topo4, free_mask.data(), n, Ws, c);
    std::vector<uint8_t> tile_class((size_t)(c.n_slots / kgpu::SP_THREADS), 0);
    for (int64_t sl = 0; sl < c.n_slots; sl++)
        if (c.order[(size_t)sl] >= 0) {
            uint8_t &tc = tile_class[(size_t)(sl / kgpu::SP_THREADS)];
            tc = std::max<uint8_t>(tc, (uint8_t)__builtin_popcount((unsigned)free_mask[(size_t)c.order[(size_t)sl]] & 0xFFu));
        }
    std::vector<kgpu::SparseWorkItem> items;
    kgpu::build_sparse_work(tile_class, P, resident, items);
    const bool aligned = kgpu::sparse_work_chunk_aligned((int64_t)tile_class.size(), P, resident);
    const int4 *work = reinterpret_cast<const int4 *>(items.data());
    const int64_t chunks = (P + kgpu::SP_CHUNK - 1) / kgpu::SP_CHUNK;
    int4 *tabs = aligned_array<int4>((size_t)chunks * kgpu::SP_CHUNK_INT4);
    const int4 *ch = prepare && aligned ? tabs : nullptr;
    int flag = 0;
    for (int64_t p = 0; p < P; p++) flag |= pods[4 * p + 3] > 0;
    bool byte_keys = true;
    for (int i = 0; i < 16; i++) byte_keys = byte_keys && W[i] <= 2340;
    const dim3 grid((unsigned)items.size());
#define EMU_PREPARE(MEMF) \
    if (ch) emu::launch(dim3((unsigned)chunks), dim3(kgpu::SP_THREADS), [&] { kgpu::sp_prepare_chunks<MEMF>(pods4, P, &flag, tabs); })
#define EMU_SPARSE(MEMF, BK)                                                                                                  \
    emu::launch(grid, dim3(kgpu::SP_THREADS), [&] {                                                                           \
        kgpu::score_pairs_sparse<true, MEMF, BK, false>(c.rec, c.meta, mem, c.order.data(), &flag, node_id_base, pods4, P, 0, work, \
                                                      kPC, keys, ch);                                                         \
    })
    EMU_PREPARE(false);
    if (byte_keys) EMU_SPARSE(false, true); else EMU_SPARSE(false, false);
    if (flag) {
        EMU_PREPARE(true);
        if (byte_keys) EMU_SPARSE(true, true); else EMU_SPARSE(true, false);
    }
#undef EMU_SPARSE
#undef EMU_PREPARE
    free(topo4); free(pods4); free(mem); free(tabs);
    return aligned ? 1 : 0;
}

// build_sparse_work with default parameters: items as int32[.][4] {tile, pod_begin, pod_end, ntiles}; *aligned = whether
// sparse_work_chunk_aligned chose whole chunks.  Returns the count.
int64_t emu_work_list(const uint8_t *tile_class, int64_t tiles, int64_t P, int64_t resident, int32_t *out, int64_t cap,
                      int *aligned) {
    std::vector<kgpu::SparseWorkItem> items;
    kgpu::build_sparse_work(std::vector<uint8_t>(tile_class, tile_class + tiles), P, resident, items);
    *aligned = kgpu::sparse_work_chunk_aligned(tiles, P, resident) ? 1 : 0;
    for (size_t i = 0; i < items.size() && (int64_t)i < cap; i++) std::memcpy(out + 4 * i, &items[i], 16);
    return (int64_t)items.size();
}

}  // extern "C"
