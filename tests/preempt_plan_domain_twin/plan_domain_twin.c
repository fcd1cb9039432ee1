/*
 * plan_domain_twin.c -- CPU twin of kgpu_preempt_plan_gang_domain.  TEST INFRASTRUCTURE ONLY: compiled together with
 * oracle/oracle_b.c by tests/test_preempt_plan_domain.py and scripts/preempt_plan_domain_time.py.  It includes
 * plan_gang_twin.c (and through it plan_twin.c) for the node evaluation, tile minima and refresh, so the library also
 * exports preempt_plan_twin and preempt_plan_gang_twin.
 *
 * Pods and gangs with gang_domain 0 are taken as by preempt_plan_gang_twin.  A constrained gang runs one trial per domain
 * with at least one node, on scratch copies (F_d, H_d) of the touched nodes (valid where stamp[n] == the trial's stamp).
 * A member's candidate on an untouched node is the node's key under (F, H); on a touched node it is evaluated literally
 * under (F_d, H_d) (every k-subset of available GPUs, as plan_twin.c's eval_node) and cached until the node changes
 * again.  The trial with the smallest (L_d, V_d, C_d, d) is run again and its touched nodes copied into (F, H); with no
 * winner a REQUIRED gang gets NO_FIT and a PREFERRED gang is taken as a plain gang.  domain may be NULL (every node -1).
 * free_mask and hold (when given) receive the final (F, H).  The caller has checked gang and gang_domain as libkgpu does.
 */
#include "../preempt_plan_gang_twin/plan_gang_twin.c"

typedef struct {
    job_t base;                 /* F, H and the node keys of the working state */
    uint64_t *tilekey;
    int64_t T, id_base;
    const int32_t *pods;
    const int *pcol;
    pre_t *pre;
    int32_t *fd, *hd;           /* the trials' working masks and holder rows [N], [N][8] */
    uint32_t *stamp, *ver;      /* the trial that wrote fd[n] / hd[n], and a change counter per node */
    uint64_t *ckey;             /* [ncol][N] cached key of a touched node under (fd, hd), valid where cver == ver[n] */
    uint32_t *cver;
    uint32_t next_ver;
} pd_t;

/* the update rule on one node's (f, h); returns the victims */
static unsigned update(int32_t *f, int32_t *h, unsigned S)
{
    const unsigned F = (unsigned)*f & 0xFFu;
    unsigned vic = 0, R = 0;
    for (int i = 0; i < 8; i++)
        if (((S & ~F) >> i) & 1u) vic |= 1u << (h[i] & 7);
    for (int i = 0; i < 8; i++)
        if (!((F >> i) & 1u) && h[i] >= 0 && ((vic >> (h[i] & 7)) & 1u)) R |= 1u << i;
    *f = (int32_t)((F | R) & ~S);
    for (int i = 0; i < 8; i++)
        if (((S | R) >> i) & 1u) h[i] = -1;
    return vic;
}

/* column c's key of node n under mask F and holder row h (plan_twin.c's eval_node for one column) */
static uint64_t col_key(const job_t *j, int64_t n, int c, unsigned F, const int32_t *h)
{
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
    if (__builtin_popcount(avail) < col->k) return best;
    for (unsigned S = 0; S < 256; S++) {
        if ((S & ~avail) || __builtin_popcount(S) != col->k) continue;
        unsigned own = 0, maxl = 0;
        for (int i = 0; i < 8; i++) {
            if (!((S >> i) & 1u) || ((F >> i) & 1u)) continue;
            own |= 1u << (h[i] & 7);
            if ((unsigned)(h[i] >> 3) > maxl) maxl = (unsigned)(h[i] >> 3);
        }
        const uint64_t key = ((uint64_t)(maxl << 4 | (unsigned)__builtin_popcount(own)) << 56) |
                             ((uint64_t)kgpu_oracle_subset_cost(j->topo + 64 * n, S, j->W) << 39) | ((uint64_t)n << 8) | S;
        if (key < best) best = key;
    }
    return best;
}

/* pods [p, e) over all nodes, as preempt_plan_gang_twin's loop */
static void take_run(pd_t *t, int64_t p, int64_t e, const int32_t *gang, uint64_t *keys, uint32_t *vics)
{
    job_t *b = &t->base;
    int64_t g_first = p;
    int32_t g_id = 0;
    int g_failed = 0;
    for (int64_t q = p; q < e; q++) {
        const int32_t id = gang ? gang[q] : 0;
        keys[q] = NO_FIT;
        vics[q] = 0;
        if (id == 0 || id != g_id) {
            g_first = q;
            g_id = id;
            g_failed = 0;
        } else if (g_failed) {
            continue;
        }
        const int c = t->pcol[q];
        uint64_t best = NO_FIT;
        if (c < 0) {
            if (t->pods[4 * q] == 0 && b->N > 0) keys[q] = (uint64_t)t->id_base << 8;
        } else {
            for (int64_t i = 0; i < t->T; i++)
                if (t->tilekey[(int64_t)c * t->T + i] < best) best = t->tilekey[(int64_t)c * t->T + i];
        }
        if (best != NO_FIT) {
            const int64_t n = (int64_t)((best >> 8) & 0x7FFFFFFFu);
            int32_t *F = (int32_t *)b->F, *H = (int32_t *)b->H + 8 * n;
            t->pre[q].F = F[n];
            memcpy(t->pre[q].H, H, sizeof t->pre[q].H);
            vics[q] = update(F + n, H, (unsigned)(best & 0xFFu));
            keys[q] = (((best >> 39) & 0x1FFFFu) << 40) | ((uint64_t)(t->id_base + n) << 8) | (best & 0xFFu);
            refresh(b, t->tilekey, t->T, n);
            continue;
        }
        if (g_id == 0 || (c < 0 && t->pods[4 * q] == 0)) continue;
        for (int64_t m = q - 1; m >= g_first; m--) {        /* a member has missed: undo, last first */
            if ((keys[m] & 0xFFu) == 0) continue;
            const int64_t n = (int64_t)((keys[m] >> 8) & 0xFFFFFFFFu) - t->id_base;
            ((int32_t *)b->F)[n] = t->pre[m].F;
            memcpy((int32_t *)b->H + 8 * n, t->pre[m].H, sizeof t->pre[m].H);
            refresh(b, t->tilekey, t->T, n);
        }
        for (int64_t m = g_first; m <= q; m++) {
            keys[m] = NO_FIT;
            vics[m] = 0;
        }
        g_failed = 1;
    }
}

/* one trial of the members [p, e) inside the domain whose nodes are list[0..len), stamp st.  Returns the score
 * L << 51 | V << 32 | C, or NO_FIT if a member misses.  keys / vics (nullable) get the members' results. */
static uint64_t trial(pd_t *t, const int32_t *list, int64_t len, uint32_t st, int64_t p, int64_t e, uint64_t *keys, uint32_t *vics)
{
    const job_t *b = &t->base;
    uint64_t L = 0, V = 0, C = 0;
    for (int64_t q = p; q < e; q++) {
        const int c = t->pcol[q];
        uint64_t best = NO_FIT;
        if (c < 0) {
            if (t->pods[4 * q] != 0) return NO_FIT;
            best = (uint64_t)list[0] << 8;
        } else {
            for (int64_t i = 0; i < len; i++) {
                const int64_t n = list[i];
                uint64_t key;
                if (t->stamp[n] == st) {
                    const size_t at = (size_t)c * (size_t)b->N + (size_t)n;
                    if (t->cver[at] != t->ver[n]) {
                        t->ckey[at] = col_key(b, n, c, (unsigned)t->fd[n] & 0xFFu, t->hd + 8 * n);
                        t->cver[at] = t->ver[n];
                    }
                    key = t->ckey[at];
                } else {
                    key = b->nodekey[(int64_t)c * b->Npad + n];
                }
                if (key < best) best = key;
            }
            if (best == NO_FIT) return NO_FIT;
        }
        const int64_t n = (int64_t)((best >> 8) & 0x7FFFFFFFu);
        const unsigned S = (unsigned)(best & 0xFFu);
        unsigned vic = 0;
        if (S != 0) {
            if (t->stamp[n] != st) {
                t->fd[n] = b->F[n];
                memcpy(t->hd + 8 * n, b->H + 8 * n, 8 * sizeof(int32_t));
                t->stamp[n] = st;
            }
            vic = update(t->fd + n, t->hd + 8 * n, S);
            t->ver[n] = ++t->next_ver;
        }
        if (keys) {
            keys[q] = (((best >> 39) & 0x1FFFFu) << 40) | ((uint64_t)(t->id_base + n) << 8) | S;
            vics[q] = vic;
        }
        if ((best >> 60) > L) L = best >> 60;
        V += (best >> 56) & 15u;
        C += (best >> 39) & 0x1FFFFu;
    }
    return L << 51 | V << 32 | C;
}

void preempt_plan_domain_twin(const int32_t *topo, int32_t *free_mask, const int32_t *mem, int32_t *hold, int64_t N,
                              int64_t node_id_base, const int32_t *domain, const int32_t *pods, const int32_t *lvl,
                              const int32_t *gang, const int32_t *gang_domain, int64_t P, const int32_t *W, int nthreads,
                              uint64_t *out_keys, uint32_t *out_victims)
{
    const size_t PP = (size_t)(P > 0 ? P : 1), NN = (size_t)(N > 0 ? N : 1);
    col_t *cols = (col_t *)malloc(sizeof(col_t) * PP);
    int *pcol = (int *)malloc(sizeof(int) * PP);
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
    int32_t *F = (int32_t *)malloc(sizeof(int32_t) * NN);
    int32_t *H = (int32_t *)malloc(sizeof(int32_t) * 8 * NN);
    const size_t nk = (size_t)ncol * (size_t)Npad > 0 ? (size_t)ncol * (size_t)Npad : 1;
    uint64_t *nodekey = (uint64_t *)malloc(sizeof(uint64_t) * nk);
    uint64_t *tilekey = (uint64_t *)malloc(sizeof(uint64_t) * (size_t)(ncol * T > 0 ? ncol * T : 1));
    if (N > 0) memcpy(F, free_mask, sizeof(int32_t) * (size_t)N);
    for (int64_t i = 0; i < 8 * N; i++) H[i] = hold ? hold[i] : -1;
    pd_t t;
    memset(&t, 0, sizeof t);
    t.base = (job_t){topo, mem, W, F, H, cols, ncol, N, Npad, 0, N, nodekey};
    t.tilekey = tilekey, t.T = T, t.id_base = node_id_base, t.pods = pods, t.pcol = pcol;
    t.pre = (pre_t *)malloc(sizeof(pre_t) * PP);
    t.fd = (int32_t *)calloc(NN, sizeof(int32_t));
    t.hd = (int32_t *)calloc(8 * NN, sizeof(int32_t));
    t.stamp = (uint32_t *)calloc(NN, sizeof(uint32_t));
    t.ver = (uint32_t *)calloc(NN, sizeof(uint32_t));
    t.ckey = (uint64_t *)malloc(sizeof(uint64_t) * (size_t)(ncol > 0 ? ncol : 1) * NN);
    t.cver = (uint32_t *)calloc((size_t)(ncol > 0 ? ncol : 1) * NN, sizeof(uint32_t));

    if (nthreads < 1) nthreads = 1;
    if (nthreads > N) nthreads = N > 0 ? (int)N : 1;
    job_t *jobs = (job_t *)calloc((size_t)nthreads, sizeof(job_t));
    pthread_t *th = (pthread_t *)calloc((size_t)nthreads, sizeof(pthread_t));
    for (int i = 0; i < nthreads; i++) {
        jobs[i] = t.base;
        jobs[i].n0 = N * i / nthreads;
        jobs[i].n1 = N * (i + 1) / nthreads;
        pthread_create(&th[i], NULL, run, &jobs[i]);
    }
    for (int i = 0; i < nthreads; i++) pthread_join(th[i], NULL);
    for (int c = 0; c < ncol; c++)
        for (int64_t i = 0; i < T; i++) tilekey[(int64_t)c * T + i] = tile_min(&t.base, c, i);

    /* the domains' node lists, in increasing node index */
    int64_t D = 0;
    for (int64_t n = 0; domain && n < N; n++)
        if (domain[n] + 1 > D) D = domain[n] + 1;
    int64_t *off = (int64_t *)calloc((size_t)D + 2, sizeof(int64_t));
    int64_t *at = (int64_t *)calloc((size_t)D + 1, sizeof(int64_t));
    int32_t *list = (int32_t *)malloc(sizeof(int32_t) * NN);
    for (int64_t n = 0; domain && n < N; n++)
        if (domain[n] >= 0) off[domain[n] + 1]++;
    for (int64_t d = 0; d < D; d++) off[d + 1] += off[d];
    memcpy(at, off, sizeof(int64_t) * (size_t)D);
    for (int64_t n = 0; domain && n < N; n++)
        if (domain[n] >= 0) list[at[domain[n]]++] = (int32_t)n;

    uint32_t st = 0;
    int64_t p = 0;
    while (p < P) {
        const int mode = gang_domain ? gang_domain[p] : 0;
        int64_t e = p + 1;
        if (mode == 0) {                                  /* the maximal range without a constrained gang */
            while (e < P && !(gang_domain && gang_domain[e] != 0)) e++;
            take_run(&t, p, e, gang, out_keys, out_victims);
            p = e;
            continue;
        }
        while (e < P && gang[e] == gang[p]) e++;
        uint64_t best_s = NO_FIT;
        int64_t best_d = -1;
        for (int64_t d = 0; d < D; d++) {
            if (off[d] == off[d + 1]) continue;
            const uint64_t s = trial(&t, list + off[d], off[d + 1] - off[d], ++st, p, e, NULL, NULL);
            if (s < best_s) best_s = s, best_d = d;
        }
        if (best_d >= 0) {
            ++st;
            trial(&t, list + off[best_d], off[best_d + 1] - off[best_d], st, p, e, out_keys, out_victims);
            for (int64_t q = p; q < e; q++) {
                const int64_t n = (int64_t)((out_keys[q] >> 8) & 0xFFFFFFFFu) - node_id_base;
                if ((out_keys[q] & 0xFFu) == 0 || t.stamp[n] != st) continue;
                F[n] = t.fd[n];
                memcpy(H + 8 * n, t.hd + 8 * n, 8 * sizeof(int32_t));
                t.stamp[n] = 0;
                refresh(&t.base, tilekey, T, n);
            }
        } else if (mode == 1) {
            for (int64_t q = p; q < e; q++) out_keys[q] = NO_FIT, out_victims[q] = 0;
        } else {
            take_run(&t, p, e, gang, out_keys, out_victims);
        }
        p = e;
    }
    if (N > 0) memcpy(free_mask, F, sizeof(int32_t) * (size_t)N);
    if (hold) memcpy(hold, H, sizeof(int32_t) * 8 * (size_t)N);
    free(jobs); free(th); free(cols); free(pcol); free(F); free(H); free(nodekey); free(tilekey);
    free(t.pre); free(t.fd); free(t.hd); free(t.stamp); free(t.ver); free(t.ckey); free(t.cver);
    free(off); free(at); free(list);
}
