/*
 * levels_twin.c -- CPU twin of placement with nested network domains (kgpu_place_batch_gang_levels).  TEST
 * INFRASTRUCTURE ONLY: built with oracle/oracle_b.c by tests/test_gang_domain_levels.py.  It includes the one-level twin
 * (gang_domain_twin.c) for its trial, plain-gang placement and key cache, and adds the level climb of include/kgpu.h
 * literally: a constrained gang with bound r tries every non-empty domain of level 0, then of level 1, ... up to r, on
 * the masks F; the first level with a fitting trial wins and the gang takes its domain with the smallest (sum of costs,
 * id).  With none, REQUIRED gives NO_FIT and PREFERRED places the gang as a plain gang.  domain is [levels][N];
 * gang_level may be NULL (all 0).  The caller has checked the inputs as libkgpu does.
 */
#include "../gang_domain_twin/gang_domain_twin.c"

typedef struct {
    int64_t D;
    int64_t *off;               /* [D + 1] ranges of list */
    int32_t *list;              /* the level's domains' nodes, each in increasing node index */
} level_t;

static void level_lists(level_t *lv, const int32_t *domain, int64_t N)
{
    lv->D = 0;
    for (int64_t n = 0; n < N; n++)
        if (domain[n] + 1 > lv->D) lv->D = domain[n] + 1;
    lv->off = (int64_t *)calloc((size_t)lv->D + 2, sizeof(int64_t));
    lv->list = (int32_t *)malloc(sizeof(int32_t) * (size_t)(N > 0 ? N : 1));
    for (int64_t n = 0; n < N; n++)
        if (domain[n] >= 0) lv->off[domain[n] + 1]++;
    for (int64_t d = 0; d < lv->D; d++) lv->off[d + 1] += lv->off[d];
    int64_t *at = (int64_t *)malloc(sizeof(int64_t) * ((size_t)lv->D + 1));
    memcpy(at, lv->off, sizeof(int64_t) * ((size_t)lv->D + 1));
    for (int64_t n = 0; n < N; n++)
        if (domain[n] >= 0) lv->list[at[domain[n]]++] = (int32_t)n;
    free(at);
}

void levels_twin_place_batch(const int32_t *topo, int32_t *free_mask, const int32_t *mem, int64_t N, int64_t node_id_base,
                             const int32_t *domain, int levels, const int32_t *pods, const int32_t *gang,
                             const int32_t *gang_domain, const int32_t *gang_level, int64_t P, const int32_t *W,
                             uint64_t *out_keys)
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
    level_t lv[4];
    for (int l = 0; l < levels; l++) level_lists(&lv[l], domain + (int64_t)l * N, N);
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
        const int r = gang_level ? gang_level[p] : 0;
        int64_t best_c = -1, best_d = -1;
        int wl = -1;
        for (int l = 0; l <= r && best_d < 0; l++) {            /* the climb: stop at the first level that fits */
            for (int64_t d = 0; d < lv[l].D; d++) {
                const int64_t *off = lv[l].off;
                if (off[d] == off[d + 1]) continue;
                const int64_t c = trial(&t, lv[l].list + off[d], off[d + 1] - off[d], ++st, pods, p, e, NULL);
                if (c >= 0 && (best_d < 0 || c < best_c)) best_c = c, best_d = d, wl = l;
            }
        }
        if (best_d >= 0) {
            const int64_t *off = lv[wl].off;
            ++st;
            trial(&t, lv[wl].list + off[best_d], off[best_d + 1] - off[best_d], st, pods, p, e, out_keys);
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
    for (int l = 0; l < levels; l++) {
        free(lv[l].off);
        free(lv[l].list);
    }
    free(t.cache);
    free(t.valid);
    free(t.fd);
    free(t.stamp);
}
