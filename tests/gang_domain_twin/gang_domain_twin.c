/*
 * gang_domain_twin.c -- CPU twin of sequential placement with gangs constrained to one network domain
 * (kgpu_place_batch_gang_domain).  TEST INFRASTRUCTURE ONLY: compiled together with oracle/oracle_b.c (it scores nodes
 * with kgpu_oracle_node_key, the oracle's definition) by tests/test_gang_domain.py.
 *
 * Literally the definition in include/kgpu.h.  Pods are taken in order on the masks F.  A pod on its own, and a gang
 * with gang_domain 0, are placed as by gang_twin.c: each member gets the minimum over all nodes of
 * (cost << 40 | node_id << 8 | S) under F (a pod with min_mem > 0 only sees the GPUs with at least that many MiB; mem may
 * be NULL) and takes S; when a gang member misses (or asks for k outside 0..8) the members before it give their GPUs
 * back and every member gets NO_FIT.  A constrained gang (gang_domain 1 = REQUIRED, 2 = PREFERRED) runs one trial per
 * domain with at least one node, on a copy of F; the domain with the smallest (sum of costs, id) wins and its trial is
 * committed; with no winner a REQUIRED gang gets NO_FIT and a PREFERRED one is placed as a gang with gang_domain 0.
 * domain may be NULL (every node -1).  The caller has checked gang and gang_domain as libkgpu does.  Masks keep their
 * low 8 bits.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define NO_FIT UINT64_MAX
#define NODE_NO_FIT UINT32_MAX
#define MAX_VIEWS 64

uint32_t kgpu_oracle_node_key(const int32_t *M, int32_t free_mask, int k, const int32_t *W);

typedef struct {
    const int32_t *topo, *mem, *W;
    int32_t *F;                 /* the masks */
    int64_t N, base;
    int nviews;
    int32_t view_min[MAX_VIEWS];
    uint32_t *cache;            /* [view][N][9] node keys under F, valid where valid[view][n] */
    uint8_t *valid;
    int32_t *fd;                /* a trial's working masks, where stamp[n] == the trial's stamp */
    uint32_t *stamp;
} twin_t;

static int32_t eligible(const twin_t *t, int64_t n, int32_t mask, int32_t need)
{
    if (!t->mem || need <= 0) return mask;
    unsigned ok = 0;
    for (int i = 0; i < 8; i++)
        if (t->mem[8 * n + i] >= need) ok |= 1u << i;
    return (int32_t)((unsigned)mask & ok);
}

static int view_of(const twin_t *t, int32_t need)
{
    for (int v = 1; v < t->nviews; v++)
        if (t->view_min[v] == need) return v;
    return 0;
}

/* node key of node n for k GPUs under mask (k in 0..8) */
static uint32_t key_under(const twin_t *t, int64_t n, int32_t mask, int k, int32_t need)
{
    return kgpu_oracle_node_key(t->topo + 64 * n, eligible(t, n, mask, need), k, t->W);
}

/* node key of node n for k GPUs under F */
static uint32_t key_f(twin_t *t, int64_t n, int k, int32_t need)
{
    const int v = view_of(t, need);
    const size_t at = (size_t)v * (size_t)t->N + (size_t)n;
    if (!t->valid[at]) {
        for (int kk = 0; kk <= 8; kk++) t->cache[at * 9 + kk] = key_under(t, n, t->F[n], kk, t->view_min[v]);
        t->valid[at] = 1;
    }
    return t->cache[at * 9 + k];
}

static void set_f(twin_t *t, int64_t n, int32_t mask)
{
    t->F[n] = mask;
    for (int v = 0; v < t->nviews; v++) t->valid[(size_t)v * (size_t)t->N + (size_t)n] = 0;
}

static uint64_t wide(uint32_t nk, int64_t node_id)
{
    return nk == NODE_NO_FIT ? NO_FIT : ((uint64_t)(nk >> 8) << 40) | ((uint64_t)node_id << 8) | (nk & 0xFFu);
}

static int64_t node_of(const twin_t *t, uint64_t key) { return (int64_t)((key >> 8) & 0xFFFFFFFFu) - t->base; }

/* pods [p, e) over all nodes; all or nothing when gang (gang_twin.c's loop) */
static void place_run(twin_t *t, const int32_t *pods, int64_t p, int64_t e, int gang, uint64_t *keys)
{
    for (int64_t q = p; q < e; q++) {
        const int k = pods[4 * q];
        const int32_t need = pods[4 * q + 3];
        uint64_t best = NO_FIT;
        if (k >= 0 && k <= 8)
            for (int64_t n = 0; n < t->N; n++) {
                const uint64_t key = wide(key_f(t, n, k, need), t->base + n);
                if (key < best) best = key;
            }
        keys[q] = best;
        if (best != NO_FIT) {
            const int64_t n = node_of(t, best);
            set_f(t, n, (int32_t)(((uint32_t)t->F[n] & 0xFFu) & ~(uint32_t)(best & 0xFFu)));
        } else if (gang) {
            for (int64_t r = q - 1; r >= p; r--) {           /* undo, last member first */
                const int64_t n = node_of(t, keys[r]);
                set_f(t, n, (int32_t)(((uint32_t)t->F[n] & 0xFFu) | (uint32_t)(keys[r] & 0xFFu)));
            }
            for (int64_t r = p; r < e; r++) keys[r] = NO_FIT;
            return;
        }
    }
}

/* one trial: the members [p, e) inside the domain whose nodes are list[0..len), on a copy of F.  Returns the cost sum,
 * or -1 if a member does not fit.  keys (nullable) get the members' keys. */
static int64_t trial(twin_t *t, const int32_t *list, int64_t len, uint32_t st, const int32_t *pods, int64_t p, int64_t e,
                     uint64_t *keys)
{
    int64_t cost = 0;
    for (int64_t q = p; q < e; q++) {
        const int k = pods[4 * q];
        const int32_t need = pods[4 * q + 3];
        if (k < 0 || k > 8) return -1;
        uint64_t best = NO_FIT;
        for (int64_t i = 0; i < len; i++) {
            const int64_t n = list[i];
            const uint32_t nk = t->stamp[n] == st ? key_under(t, n, t->fd[n], k, need) : key_f(t, n, k, need);
            const uint64_t key = wide(nk, t->base + n);
            if (key < best) best = key;
        }
        if (keys) keys[q] = best;
        if (best == NO_FIT) return -1;
        cost += (int64_t)(best >> 40);
        const int64_t n = node_of(t, best);
        if (t->stamp[n] != st) {
            t->fd[n] = t->F[n] & 0xFF;
            t->stamp[n] = st;
        }
        t->fd[n] &= ~(int32_t)(best & 0xFFu);
    }
    return cost;
}

void gang_domain_twin_place_batch(const int32_t *topo, int32_t *free_mask, const int32_t *mem, int64_t N, int64_t node_id_base,
                                  const int32_t *domain, const int32_t *pods, const int32_t *gang, const int32_t *gang_domain,
                                  int64_t P, const int32_t *W, uint64_t *out_keys)
{
    twin_t t;
    memset(&t, 0, sizeof t);
    t.topo = topo, t.mem = mem, t.W = W, t.F = free_mask, t.N = N, t.base = node_id_base;
    t.nviews = 1;
    for (int64_t p = 0; p < P; p++) {
        const int32_t need = pods[4 * p + 3];
        if (!mem || need <= 0 || view_of(&t, need) != 0 || t.nviews == MAX_VIEWS) continue;
        t.view_min[t.nviews++] = need;
    }
    const size_t NN = (size_t)(N > 0 ? N : 1);
    t.cache = (uint32_t *)malloc(sizeof(uint32_t) * 9 * NN * (size_t)t.nviews);
    t.valid = (uint8_t *)calloc(NN * (size_t)t.nviews, 1);
    t.fd = (int32_t *)calloc(NN, sizeof(int32_t));
    t.stamp = (uint32_t *)calloc(NN, sizeof(uint32_t));
    /* the domains' node lists, in increasing node index */
    int64_t D = 0;
    for (int64_t n = 0; domain && n < N; n++)
        if (domain[n] + 1 > D) D = domain[n] + 1;
    int64_t *off = (int64_t *)calloc((size_t)D + 2, sizeof(int64_t));
    int32_t *list = (int32_t *)malloc(sizeof(int32_t) * NN);
    for (int64_t n = 0; domain && n < N; n++)
        if (domain[n] >= 0) off[domain[n] + 1]++;
    for (int64_t d = 0; d < D; d++) off[d + 1] += off[d];
    int64_t *at = (int64_t *)malloc(sizeof(int64_t) * ((size_t)D + 1));
    memcpy(at, off, sizeof(int64_t) * ((size_t)D + 1));
    for (int64_t n = 0; domain && n < N; n++)
        if (domain[n] >= 0) list[at[domain[n]]++] = (int32_t)n;
    uint32_t st = 0;
    int64_t p = 0;
    while (p < P) {
        int64_t e = p + 1;
        while (gang[p] != 0 && e < P && gang[e] == gang[p]) e++;
        const int mode = gang_domain ? gang_domain[p] : 0;
        if (mode == 0) {
            place_run(&t, pods, p, e, gang[p] != 0, out_keys);
            p = e;
            continue;
        }
        int64_t best_c = -1, best_d = -1;
        for (int64_t d = 0; d < D; d++) {
            if (off[d] == off[d + 1]) continue;
            const int64_t c = trial(&t, list + off[d], off[d + 1] - off[d], ++st, pods, p, e, NULL);
            if (c >= 0 && (best_d < 0 || c < best_c)) best_c = c, best_d = d;
        }
        if (best_d >= 0) {
            ++st;
            trial(&t, list + off[best_d], off[best_d + 1] - off[best_d], st, pods, p, e, out_keys);
            for (int64_t q = p; q < e; q++) {
                const int64_t n = node_of(&t, out_keys[q]);
                if (t.stamp[n] == st) set_f(&t, n, t.fd[n]);
            }
        } else if (mode == 1) {
            for (int64_t q = p; q < e; q++) out_keys[q] = NO_FIT;
        } else {
            place_run(&t, pods, p, e, 1, out_keys);
        }
        p = e;
    }
    free(t.cache);
    free(t.valid);
    free(t.fd);
    free(t.stamp);
    free(off);
    free(at);
    free(list);
}
