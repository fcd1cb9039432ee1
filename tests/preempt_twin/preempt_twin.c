/*
 * preempt_twin.c -- CPU twin of preemption (kgpu_preempt_batch).  TEST INFRASTRUCTURE ONLY: compiled together with
 * oracle/oracle_b.c (subset costs are the oracle's kgpu_oracle_subset_cost) by tests/test_preemption.py and
 * scripts/preempt_time.py.
 *
 * The definition, enumerated literally: for pod p (k = pods[4p], min_mem = pods[4p+3], level lvl[p]) every node n and
 * every k-subset S of its 8 slots is looked at.  GPU i is available if it is free, or if hold[n][i] != -1 and its level
 * (hold >> 3) is < lvl[p]; with min_mem > 0 and mem != NULL it must also have mem[n][i] >= min_mem.  S is a candidate if
 * all its GPUs are available; its victims V(S) are the owners (hold & 7) of its GPUs that are not free.  The winner is
 * the smallest (max level in V, |V|, cost(S), node id, S), an empty V counting as level 0, size 0.  hold == NULL means
 * every entry is -1.  k outside 0..8 or no candidate: NO_FIT and victims 0.  No victim-set shortcut: every S is scored.
 * Nodes are split over nthreads threads, each keeping its own best per pod; the per-thread bests are merged at the end.
 */
#include <pthread.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define NO_FIT UINT64_MAX

uint32_t kgpu_oracle_subset_cost(const int32_t *M, unsigned S, const int32_t *W);

typedef struct {
    uint32_t hi;    /* max level << 24 | |V| << 20 | cost */
    uint64_t lo;    /* node id << 8 | S */
    uint32_t victims;
} best_t;

typedef struct {
    const int32_t *topo, *free_mask, *mem, *hold, *pods, *lvl, *W;
    int64_t n0, n1, node_id_base, P;
    best_t *best;
} job_t;

static void *run(void *arg)
{
    const job_t *j = (const job_t *)arg;
    uint32_t cost[256];
    uint8_t own[256], maxlvl[256], usable[256];
    uint8_t subsets[9][70];             /* the k-subsets of 8 slots, each list in increasing order */
    int nsub[9] = {0};
    for (unsigned S = 0; S < 256; S++) {
        const int k = __builtin_popcount(S);
        subsets[k][nsub[k]++] = (uint8_t)S;
    }
    for (int64_t p = 0; p < j->P; p++) j->best[p].hi = UINT32_MAX;
    for (int64_t n = j->n0; n < j->n1; n++) {
        const int32_t *M = j->topo + 64 * n;
        const unsigned F = (unsigned)j->free_mask[n] & 0xFFu;
        unsigned below[17] = {0};            /* below[L]: the non-free GPUs held at a level < L */
        for (int i = 0; i < 8; i++) {
            const int32_t e = j->hold ? j->hold[8 * n + i] : -1;
            if (e >= 0 && !((F >> i) & 1u))
                for (int L = (e >> 3) + 1; L <= 16; L++) below[L] |= 1u << i;
        }
        for (unsigned S = 0; S < 256; S++) {
            cost[S] = kgpu_oracle_subset_cost(M, S, j->W);
            own[S] = 0; maxlvl[S] = 0; usable[S] = 1;          /* usable: no non-free GPU of S is marked -1 */
            for (int i = 0; i < 8; i++) {
                if (!((S >> i) & 1u) || ((F >> i) & 1u)) continue;
                const int32_t e = j->hold ? j->hold[8 * n + i] : -1;
                if (e < 0) { usable[S] = 0; continue; }
                own[S] |= (uint8_t)(1u << (e & 7));
                if ((e >> 3) > maxlvl[S]) maxlvl[S] = (uint8_t)(e >> 3);
            }
        }
        for (int64_t p = 0; p < j->P; p++) {
            const int k = j->pods[4 * p];
            const int32_t need = j->pods[4 * p + 3], L = j->lvl[p];
            if (k < 0 || k > 8) continue;
            unsigned elig = 0xFFu;
            if (j->mem && need > 0) {
                elig = 0;
                for (int i = 0; i < 8; i++)
                    if (j->mem[8 * n + i] >= need) elig |= 1u << i;
            }
            const unsigned avail = (F | below[L < 0 ? 0 : L > 16 ? 16 : L]) & elig;    /* the available GPUs */
            if (__builtin_popcount(avail) < k) continue;
            best_t *b = &j->best[p];
            for (int s = 0; s < nsub[k]; s++) {
                const unsigned S = subsets[k][s];
                if ((S & ~avail) || !usable[S]) continue;
                const unsigned used = S & ~F;
                if (used && maxlvl[S] >= L) continue;
                const uint32_t hi = ((uint32_t)maxlvl[S] << 24) | ((uint32_t)__builtin_popcount(own[S]) << 20) | cost[S];
                const uint64_t lo = ((uint64_t)(j->node_id_base + n) << 8) | S;
                if (hi < b->hi || (hi == b->hi && lo < b->lo)) { b->hi = hi; b->lo = lo; b->victims = own[S]; }
            }
        }
    }
    return NULL;
}

void preempt_twin_batch(const int32_t *topo, const int32_t *free_mask, const int32_t *mem, const int32_t *hold, int64_t N,
                        int64_t node_id_base, const int32_t *pods, const int32_t *lvl, int64_t P, const int32_t *W,
                        int nthreads, uint64_t *out_keys, uint32_t *out_victims)
{
    if (nthreads < 1) nthreads = 1;
    if (nthreads > N) nthreads = N > 0 ? (int)N : 1;
    job_t *jobs = (job_t *)calloc((size_t)nthreads, sizeof(job_t));
    pthread_t *th = (pthread_t *)calloc((size_t)nthreads, sizeof(pthread_t));
    for (int t = 0; t < nthreads; t++) {
        job_t *j = &jobs[t];
        j->topo = topo; j->free_mask = free_mask; j->mem = mem; j->hold = hold; j->pods = pods; j->lvl = lvl; j->W = W;
        j->n0 = N * t / nthreads; j->n1 = N * (t + 1) / nthreads;
        j->node_id_base = node_id_base; j->P = P;
        j->best = (best_t *)malloc(sizeof(best_t) * (size_t)(P > 0 ? P : 1));
        pthread_create(&th[t], NULL, run, j);
    }
    for (int t = 0; t < nthreads; t++) pthread_join(th[t], NULL);
    for (int64_t p = 0; p < P; p++) {
        best_t b = {UINT32_MAX, 0, 0};
        for (int t = 0; t < nthreads; t++) {
            const best_t *c = &jobs[t].best[p];
            if (c->hi < b.hi || (c->hi == b.hi && c->lo < b.lo)) b = *c;
        }
        if (b.hi == UINT32_MAX) {
            out_keys[p] = NO_FIT;
            out_victims[p] = 0;
        } else {
            out_keys[p] = ((uint64_t)(b.hi & 0xFFFFFu) << 40) | b.lo;
            out_victims[p] = b.victims;
        }
    }
    for (int t = 0; t < nthreads; t++) free(jobs[t].best);
    free(jobs);
    free(th);
}
