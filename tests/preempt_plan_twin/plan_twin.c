/*
 * plan_twin.c -- fast sequential CPU twin of kgpu_preempt_plan.  TEST INFRASTRUCTURE ONLY: compiled together with
 * oracle/oracle_b.c (subset costs are the oracle's kgpu_oracle_subset_cost) by tests/test_preempt_plan.py and
 * scripts/preempt_plan_time.py.
 *
 * A pod's answer on one node depends on the node's state and on the pod's (k, level, min_mem) only, so the twin keeps,
 * for every such COLUMN of the batch, every node's best candidate and the minimum of each 128-node tile.  A node's best
 * candidate is found literally, as preempt_twin.c does: every k-subset S of available GPUs, ordered by (max victim
 * level, |V|, cost, node, S), packed into one 64-bit key (level 4 | |V| 4 | cost 17 | node 31 | S 8).  Per pod: the
 * winner is the minimum over the tile minima of its column; the update of the definition (include/kgpu.h) is applied;
 * only the winner's node is re-evaluated, for every column, and its tile minimum rescanned.  The initial evaluation is
 * split over nthreads threads.
 */
#include <pthread.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define NO_FIT UINT64_MAX
#define TILE 128

uint32_t kgpu_oracle_subset_cost(const int32_t *M, unsigned S, const int32_t *W);

typedef struct {
    int k, level, need;
} col_t;

typedef struct {
    const int32_t *topo, *mem, *W;
    const int32_t *F, *H;
    const col_t *cols;
    int ncol;
    int64_t N, Npad, n0, n1;
    uint64_t *nodekey;
} job_t;

/* every column's key of node n under masks F / holder rows H (8 per node) */
static void eval_node(const job_t *j, int64_t n)
{
    uint32_t cost[256];
    const int32_t *M = j->topo + 64 * n, *h = j->H + 8 * n;
    const unsigned F = (unsigned)j->F[n] & 0xFFu;
    for (unsigned S = 0; S < 256; S++) cost[S] = kgpu_oracle_subset_cost(M, S, j->W);
    for (int c = 0; c < j->ncol; c++) {
        const col_t *col = &j->cols[c];
        unsigned elig = 0xFFu;
        if (j->mem && col->need > 0) {
            elig = 0;
            for (int i = 0; i < 8; i++)
                if (j->mem[8 * n + i] >= col->need) elig |= 1u << i;
        }
        unsigned avail = F;
        for (int i = 0; i < 8; i++)
            if (!((F >> i) & 1u) && h[i] >= 0 && (h[i] >> 3) < col->level) avail |= 1u << i;
        avail &= elig;
        uint64_t best = NO_FIT;
        if (__builtin_popcount(avail) >= col->k) {
            for (unsigned S = 0; S < 256; S++) {
                if ((S & ~avail) || __builtin_popcount(S) != col->k) continue;
                unsigned own = 0, maxl = 0;
                for (int i = 0; i < 8; i++) {
                    if (!((S >> i) & 1u) || ((F >> i) & 1u)) continue;
                    own |= 1u << (h[i] & 7);
                    if ((unsigned)(h[i] >> 3) > maxl) maxl = (unsigned)(h[i] >> 3);
                }
                const uint64_t key = ((uint64_t)(maxl << 4 | (unsigned)__builtin_popcount(own)) << 56) | ((uint64_t)cost[S] << 39) |
                                     ((uint64_t)n << 8) | S;
                if (key < best) best = key;
            }
        }
        j->nodekey[(int64_t)c * j->Npad + n] = best;
    }
}

static void *run(void *arg)
{
    const job_t *j = (const job_t *)arg;
    for (int64_t n = j->n0; n < j->n1; n++) eval_node(j, n);
    return NULL;
}

static uint64_t tile_min(const job_t *j, int c, int64_t t)
{
    uint64_t b = NO_FIT;
    for (int64_t n = t * TILE; n < (t + 1) * TILE && n < j->N; n++) {
        const uint64_t v = j->nodekey[(int64_t)c * j->Npad + n];
        if (v < b) b = v;
    }
    return b;
}

void preempt_plan_twin(const int32_t *topo, const int32_t *free_mask, const int32_t *mem, const int32_t *hold, int64_t N,
                       int64_t node_id_base, const int32_t *pods, const int32_t *lvl, int64_t P, const int32_t *W,
                       int nthreads, uint64_t *out_keys, uint32_t *out_victims)
{
    /* columns: the distinct (k, level, min_mem) with k in 1..8 */
    col_t *cols = (col_t *)malloc(sizeof(col_t) * (size_t)(P > 0 ? P : 1));
    int *pcol = (int *)malloc(sizeof(int) * (size_t)(P > 0 ? P : 1));
    int ncol = 0;
    for (int64_t p = 0; p < P; p++) {
        const int k = pods[4 * p], need = pods[4 * p + 3] > 0 ? pods[4 * p + 3] : 0;
        pcol[p] = -1;
        if (k < 1 || k > 8) continue;
        int c = 0;
        while (c < ncol && !(cols[c].k == k && cols[c].level == lvl[p] && cols[c].need == need)) c++;
        if (c == ncol) { cols[c].k = k; cols[c].level = lvl[p]; cols[c].need = need; ncol++; }
        pcol[p] = c;
    }
    const int64_t T = (N + TILE - 1) / TILE, Npad = T * TILE;
    int32_t *F = (int32_t *)malloc(sizeof(int32_t) * (size_t)(N > 0 ? N : 1));
    int32_t *H = (int32_t *)malloc(sizeof(int32_t) * 8 * (size_t)(N > 0 ? N : 1));
    uint64_t *nodekey = (uint64_t *)malloc(sizeof(uint64_t) * (size_t)(ncol * Npad > 0 ? ncol * Npad : 1));
    uint64_t *tilekey = (uint64_t *)malloc(sizeof(uint64_t) * (size_t)(ncol * T > 0 ? ncol * T : 1));
    if (N > 0) memcpy(F, free_mask, sizeof(int32_t) * (size_t)N);
    for (int64_t i = 0; i < 8 * N; i++) H[i] = hold ? hold[i] : -1;
    job_t base = {topo, mem, W, F, H, cols, ncol, N, Npad, 0, N, nodekey};

    if (nthreads < 1) nthreads = 1;
    if (nthreads > N) nthreads = N > 0 ? (int)N : 1;
    job_t *jobs = (job_t *)calloc((size_t)nthreads, sizeof(job_t));
    pthread_t *th = (pthread_t *)calloc((size_t)nthreads, sizeof(pthread_t));
    for (int t = 0; t < nthreads; t++) {
        jobs[t] = base;
        jobs[t].n0 = N * t / nthreads;
        jobs[t].n1 = N * (t + 1) / nthreads;
        pthread_create(&th[t], NULL, run, &jobs[t]);
    }
    for (int t = 0; t < nthreads; t++) pthread_join(th[t], NULL);
    for (int c = 0; c < ncol; c++)
        for (int64_t t = 0; t < T; t++) tilekey[(int64_t)c * T + t] = tile_min(&base, c, t);

    for (int64_t p = 0; p < P; p++) {
        out_keys[p] = NO_FIT;
        out_victims[p] = 0;
        const int c = pcol[p];
        if (c < 0) {
            if (pods[4 * p] == 0 && N > 0) out_keys[p] = (uint64_t)node_id_base << 8;
            continue;
        }
        uint64_t b = NO_FIT;
        for (int64_t t = 0; t < T; t++)
            if (tilekey[(int64_t)c * T + t] < b) b = tilekey[(int64_t)c * T + t];
        if (b == NO_FIT) continue;
        const int64_t n = (int64_t)((b >> 8) & 0x7FFFFFFFu);
        const unsigned S = (unsigned)(b & 0xFFu), f = (unsigned)F[n] & 0xFFu;
        int32_t *h = H + 8 * n;
        unsigned vic = 0, R = 0;
        for (int i = 0; i < 8; i++)
            if (((S & ~f) >> i) & 1u) vic |= 1u << (h[i] & 7);
        for (int i = 0; i < 8; i++)
            if (!((f >> i) & 1u) && h[i] >= 0 && ((vic >> (h[i] & 7)) & 1u)) R |= 1u << i;
        F[n] = (int32_t)((f | R) & ~S);
        for (int i = 0; i < 8; i++)
            if (((S | R) >> i) & 1u) h[i] = -1;
        out_keys[p] = (((b >> 39) & 0x1FFFFu) << 40) | ((uint64_t)(node_id_base + n) << 8) | S;
        out_victims[p] = vic;
        eval_node(&base, n);
        for (int cc = 0; cc < ncol; cc++) tilekey[(int64_t)cc * T + n / TILE] = tile_min(&base, cc, n / TILE);
    }
    free(jobs); free(th); free(cols); free(pcol); free(F); free(H); free(nodekey); free(tilekey);
}
