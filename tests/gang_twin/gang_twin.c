/*
 * gang_twin.c -- CPU twin of sequential placement with gangs (kgpu_place_batch_gang).  TEST INFRASTRUCTURE ONLY:
 * compiled together with oracle/oracle_b.c (it scores nodes with kgpu_oracle_node_key, the oracle's definition) by
 * tests/test_gang_placement.py.
 *
 * Pods are placed in order as by the oracle's sequential placement: key_p = min over nodes of
 * (cost << 40 | node_id << 8 | S) under the CURRENT free masks, where a pod with min_mem > 0 (pods[4p+3]) only sees
 * the GPUs with at least that many MiB (mem may be NULL: no constraint); a pod that fits takes S.  A gang is a maximal
 * run of consecutive pods with the same nonzero gang[p] (the caller has checked that no id appears in two separate
 * runs).  When a gang member does not fit, or asks for k outside 0..8, the members of its gang placed before it give
 * their GPUs back, the members after it are not tried, and every member gets NO_FIT: the free masks are as they were
 * before the gang's first member.  Masks keep their low 8 bits.
 */
#include <stdint.h>
#include <stdlib.h>

#define NO_FIT UINT64_MAX
#define NODE_NO_FIT UINT32_MAX

uint32_t kgpu_oracle_node_key(const int32_t *M, int32_t free_mask, int k, const int32_t *W);

static int32_t eligible(int32_t free_mask, const int32_t *mem8, int32_t min_mem)
{
    if (!mem8 || min_mem <= 0) return free_mask;
    unsigned ok = 0;
    for (int i = 0; i < 8; i++)
        if (mem8[i] >= min_mem) ok |= 1u << i;
    return (int32_t)((unsigned)free_mask & ok);
}

/* the 9 node keys of node n without a memory requirement (only the nodes a take or an undo touches change) */
static void refresh(const int32_t *topo, const int32_t *free_mask, const int32_t *W, int64_t n, uint32_t *nb)
{
    for (int k = 0; k <= 8; k++) nb[9 * n + k] = kgpu_oracle_node_key(topo + 64 * n, free_mask[n], k, W);
}

void gang_twin_place_batch(const int32_t *topo, int32_t *free_mask, const int32_t *mem, int64_t N, int64_t node_id_base,
                           const int32_t *pods, const int32_t *gang, int64_t P, const int32_t *W, uint64_t *out_keys)
{
    uint32_t *nb = (uint32_t *)malloc(sizeof(uint32_t) * 9 * (size_t)(N > 0 ? N : 1));
    for (int64_t n = 0; n < N; n++) refresh(topo, free_mask, W, n, nb);
    int64_t first = 0;                  /* first pod of the current gang */
    int failed = 0;                     /* a member of the current gang has missed */
    for (int64_t p = 0; p < P; p++) {
        out_keys[p] = NO_FIT;
        if (gang[p] == 0 || p == 0 || gang[p] != gang[p - 1]) {
            first = p;
            failed = 0;
        } else if (failed) {
            continue;
        }
        const int k = pods[4 * p];
        const int32_t need = pods[4 * p + 3];
        uint64_t best = NO_FIT;
        if (k >= 0 && k <= 8) {
            for (int64_t n = 0; n < N; n++) {
                uint32_t nk = (mem && need > 0)
                                  ? kgpu_oracle_node_key(topo + 64 * n, eligible(free_mask[n], mem + 8 * n, need), k, W)
                                  : nb[9 * n + k];
                if (nk == NODE_NO_FIT) continue;
                uint64_t key = ((uint64_t)(nk >> 8) << 40) | ((uint64_t)(node_id_base + n) << 8) | (nk & 0xFFu);
                if (key < best) best = key;
            }
        }
        out_keys[p] = best;
        if (best != NO_FIT) {
            int64_t n = (int64_t)((best >> 8) & 0xFFFFFFFFu) - node_id_base;
            free_mask[n] = (int32_t)(((uint32_t)free_mask[n] & 0xFFu) & ~(uint32_t)(best & 0xFFu));
            refresh(topo, free_mask, W, n, nb);
        } else if (gang[p] != 0) {
            for (int64_t q = p - 1; q >= first; q--) {          /* undo, last member first */
                int64_t n = (int64_t)((out_keys[q] >> 8) & 0xFFFFFFFFu) - node_id_base;
                free_mask[n] = (int32_t)(((uint32_t)free_mask[n] & 0xFFu) | (uint32_t)(out_keys[q] & 0xFFu));
                refresh(topo, free_mask, W, n, nb);
                out_keys[q] = NO_FIT;
            }
            failed = 1;
        }
    }
    free(nb);
}
