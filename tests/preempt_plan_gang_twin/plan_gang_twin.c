/*
 * plan_gang_twin.c -- fast sequential CPU twin of kgpu_preempt_plan_gang.  TEST INFRASTRUCTURE ONLY: compiled together
 * with oracle/oracle_b.c by tests/test_preempt_plan_gang.py and scripts/preempt_plan_gang_time.py.  It includes
 * plan_twin.c for the node evaluation and tile minima (eval_node, tile_min), so the library also exports
 * preempt_plan_twin.
 *
 * Pods are taken as by preempt_plan_twin.  Before a gang member's update its node's (F[n], H[n]) is saved; when a member
 * misses (no candidate, or k outside 0..8), the members placed before it are undone last first -- (F[n], H[n]) restored,
 * the node re-evaluated and its tile minima rescanned -- the members after it are skipped, and every member gets NO_FIT
 * and victims 0.  gang == NULL is preempt_plan_twin.
 */
#include "../preempt_plan_twin/plan_twin.c"

typedef struct {
    int32_t F, H[8];
} pre_t;

static void refresh(const job_t *j, uint64_t *tilekey, int64_t T, int64_t n)
{
    eval_node(j, n);
    for (int c = 0; c < j->ncol; c++) tilekey[(int64_t)c * T + n / TILE] = tile_min(j, c, n / TILE);
}

void preempt_plan_gang_twin(const int32_t *topo, const int32_t *free_mask, const int32_t *mem, const int32_t *hold, int64_t N,
                            int64_t node_id_base, const int32_t *pods, const int32_t *lvl, const int32_t *gang, int64_t P,
                            const int32_t *W, int nthreads, uint64_t *out_keys, uint32_t *out_victims)
{
    /* columns: the distinct (k, level, min_mem) with k in 1..8 */
    col_t *cols = (col_t *)malloc(sizeof(col_t) * (size_t)(P > 0 ? P : 1));
    int *pcol = (int *)malloc(sizeof(int) * (size_t)(P > 0 ? P : 1));
    pre_t *pre = (pre_t *)malloc(sizeof(pre_t) * (size_t)(P > 0 ? P : 1));
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

    int64_t g_first = 0;
    int32_t g_id = 0;
    int g_failed = 0;
    for (int64_t p = 0; p < P; p++) {
        const int32_t id = gang ? gang[p] : 0;
        out_keys[p] = NO_FIT;
        out_victims[p] = 0;
        if (id == 0 || id != g_id) {
            g_first = p;
            g_id = id;
            g_failed = 0;
        } else if (g_failed) {
            continue;
        }
        const int c = pcol[p];
        uint64_t b = NO_FIT;
        if (c < 0) {
            if (pods[4 * p] == 0 && N > 0) out_keys[p] = (uint64_t)node_id_base << 8;
        } else {
            for (int64_t t = 0; t < T; t++)
                if (tilekey[(int64_t)c * T + t] < b) b = tilekey[(int64_t)c * T + t];
        }
        if (b != NO_FIT) {
            const int64_t n = (int64_t)((b >> 8) & 0x7FFFFFFFu);
            const unsigned S = (unsigned)(b & 0xFFu), f = (unsigned)F[n] & 0xFFu;
            int32_t *h = H + 8 * n;
            pre[p].F = F[n];
            memcpy(pre[p].H, h, sizeof pre[p].H);
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
            refresh(&base, tilekey, T, n);
            continue;
        }
        if (g_id == 0 || (c < 0 && pods[4 * p] == 0)) continue;
        /* a member has missed: undo the members before it, last first */
        for (int64_t m = p - 1; m >= g_first; m--) {
            const uint64_t key = out_keys[m];
            if ((key & 0xFFu) == 0) continue;                  /* k == 0 took nothing */
            const int64_t n = (int64_t)((key >> 8) & 0xFFFFFFFFu) - node_id_base;
            F[n] = pre[m].F;
            memcpy(H + 8 * n, pre[m].H, sizeof pre[m].H);
            refresh(&base, tilekey, T, n);
        }
        for (int64_t m = g_first; m <= p; m++) {
            out_keys[m] = NO_FIT;
            out_victims[m] = 0;
        }
        g_failed = 1;
    }
    free(jobs); free(th); free(cols); free(pcol); free(pre); free(F); free(H); free(nodekey); free(tilekey);
}
