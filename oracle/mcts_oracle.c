/*
 * mcts_oracle.c — TEST INFRASTRUCTURE ONLY.  See mcts_oracle.h.  Citations are file:line in /root/reference.
 * Arithmetic notes that bind bit-exactness (verified against the compiled reference, tests/test_oracle_pins.py):
 *   - core.h:93-95: `sqrt(float)` resolves to the float overload; q is evaluated entirely in float.
 *   - core.h:233-258: _value/_variance/delta are double, array stores narrow to float.
 *   - built with -ffp-contract=off: the reference (g++ -O3, baseline x86-64) emits no FMA.
 */
#include "mcts_oracle.h"
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <stdio.h>

/* ------------------------------------------------------------------ special.h:26-33 */
double mo_norm_quantile(double t) {
    double l2 = log(2), l22 = log(22), l41 = log(41);
    double alpha = 1 - 1 / t;
    return 10 * log(1 - log(-log(alpha) / l2) / l22) / l41;
}

/* core.h:93's bound coefficient for many n at once: mo_norm_quantile narrowed to float, as the engine's host table holds it */
void mo_norm_quantile_f32(const int32_t *n, int count, float *out) {
    for (int i = 0; i < count; ++i) out[i] = (float)mo_norm_quantile((double)n[i]);
}

/* ------------------------------------------------------------------ core.h:111-144 */
int mo_unique_child_obs(int index, const int32_t *child, const float *score, const int32_t *n2o,
                        int32_t *c_nodes, int32_t *c_obs) {
    int k = 0;
    for (int i = 0; i < MO_NA; ++i) {
        int c = child[(size_t)index * MO_NA + i];
        if (c == 0) continue;                       /* core.h:128 */
        int o = n2o[c];
        int j = 0;
        while (j < k && c_obs[j] != o) ++j;         /* std::find, core.h:132 */
        if (j == k) { c_nodes[k] = c; c_obs[k] = o; ++k; }
        else if (score[c] > score[c_nodes[j]]) c_nodes[j] = c;   /* strict >, core.h:139 */
    }
    return k;
}

/* ------------------------------------------------------------------ core.h:83-105 */
int mo_policy_clt(const int32_t *nodes, const int32_t *visit, const float *value, const float *variance, int k) {
    int n = 0;
    for (int i = 0; i < k; ++i) n += visit[i];
    int max_idx = 0;
    float max_q = 0;
    float bound_coeff = (float)mo_norm_quantile((double)n);     /* core.h:93: double -> float */
    for (int i = 0; i < k; ++i) {
        float ratio = variance[i] / (float)visit[i];
        float root = sqrtf(ratio);
        float prod = bound_coeff * root;
        float q = value[i] + prod;
        if (i == 0) max_q = q;
        else if (q > max_q) { max_q = q; max_idx = i; }
    }
    return nodes[max_idx];
}

static uint32_t libc_rand(void *ctx) { (void)ctx; return (uint32_t)rand(); }

/* xorshift32 on a caller-owned state: the injectable stand-in for rand() that the device twins also use */
uint32_t mo_xorshift32(void *ctx) {
    uint32_t *st = (uint32_t *)ctx, s = *st;
    s ^= s << 13; s ^= s >> 17; s ^= s << 5;
    *st = s;
    return s;
}

/* ------------------------------------------------------------------ core.h:167-224 (check_low core.h:65-77) */
int mo_select_trace_obs(int index, const int32_t *child, const int32_t *visit, const float *value,
                        const float *variance, const float *score, const int32_t *n2o, int low,
                        int32_t *trace, int max_trace, mo_rand_fn rnd, void *ctx) {
    if (!rnd) rnd = libc_rand;
    int D = 0;
    int32_t c_nodes[MO_NA], c_obs[MO_NA], _visit[MO_NA];
    float _value[MO_NA], _variance[MO_NA];
    for (;;) {
        if (D >= max_trace) return -1;
        trace[D++] = index;
        int k = mo_unique_child_obs(index, child, score, n2o, c_nodes, c_obs);
        if (k == 0) break;
        int lowlist[MO_NA], nl = 0;
        for (int i = 0; i < k; ++i) if (visit[c_obs[i]] < low) lowlist[nl++] = c_obs[i];
        int o = nl ? lowlist[rnd(ctx) % (uint32_t)nl] : 0;
        if (o == 0) {
            for (int i = 0; i < k; ++i) {
                int _o = c_obs[i], _c = c_nodes[i];
                _visit[i] = visit[_o];
                float t = value[_o] + score[_c];            /* core.h:213, left to right in float */
                _value[i] = t - score[index];
                _variance[i] = variance[_o];
            }
            index = mo_policy_clt(c_nodes, _visit, _value, _variance, k);
        } else {
            int j = 0;
            while (c_obs[j] != o) ++j;
            index = c_nodes[j];
        }
    }
    return D;
}

/* ------------------------------------------------------------------ core.h:226-260 */
void mo_backup_trace_obs(const int32_t *trace, int D, int32_t *visit, float *value, float *variance,
                         const int32_t *n2o, const float *score, double _value, double _variance, double gamma) {
    for (int i = D - 1; i >= 0; --i) {
        int idx = trace[i];
        _value -= score[idx];
        int o = n2o[idx];
        if (visit[o] == 0) {
            value[o] = (float)_value;
            variance[o] = (float)_variance;
        } else {
            double delta = _value - value[o];
            value[o] = (float)(value[o] + delta / (visit[o] + 1));
            double delta2 = _value - value[o];
            variance[o] = (float)(variance[o] + (delta * delta2 - variance[o]) / (visit[o] + 1));
        }
        visit[o] += 1;
        _value = gamma * _value + score[idx];
    }
}

/* ------------------------------------------------------------------ core.h:262-301 */
void mo_backup_trace_mixture_obs(const int32_t *trace, int D, int32_t *visit, float *value, float *variance,
                                 const int32_t *n2o, const float *score, double _value, double _variance, double gamma) {
    for (int i = D - 1; i >= 0; --i) {
        int idx = trace[i];
        _value -= score[idx];
        int o = n2o[idx];
        visit[o] += 1;
        double v_sq_diff = _value * _value - (double)(value[o] * value[o]);   /* float*float product, core.h:285 */
        double v_tmp = value[o];
        double delta = (_value - value[o]) / visit[o];
        value[o] = (float)(value[o] + delta);
        double var_diff = _variance - variance[o];
        variance[o] = (float)(variance[o] + ((var_diff + v_sq_diff) / visit[o] - delta * (v_tmp + value[o])));
        _value = gamma * _value + score[idx];
        _variance *= (gamma * gamma);
    }
}

/* ------------------------------------------------------------------ core.h:303-381 */
void mo_backup_trace_obs_LP(const int32_t *trace, int D, int32_t *visit, float *value, float *variance,
                            const int32_t *n2o, const float *score, const uint8_t *end, const int32_t *c_nodes,
                            const int32_t *c_obs, int k, const float *v, const float *var, double gamma,
                            int mixture, int averaged) {
    void (*backup)(const int32_t *, int, int32_t *, float *, float *, const int32_t *, const float *, double, double, double) =
        mixture ? mo_backup_trace_mixture_obs : mo_backup_trace_obs;
    if (k > 0) {
        double v_tmp = 0, var_tmp = 0;
        for (int i = 0; i < k; ++i) {
            int c = c_nodes[i], o = c_obs[i];
            if (visit[o] == 0) {
                visit[o] += 1;
                if (end[c]) { value[o] = 0; variance[o] = 0; }
                else { value[o] = v[i]; variance[o] = var[i]; }
            }
            if (averaged) {
                v_tmp += score[c] + gamma * value[o];
                var_tmp += variance[o];
            } else {
                backup(trace, D, visit, value, variance, n2o, score, value[o] + gamma * score[c],
                       gamma * gamma * variance[o], gamma);       /* core.h:358-360 (value + gamma*score, as written) */
            }
        }
        if (averaged) {
            v_tmp /= (double)k;
            var_tmp *= (gamma * gamma / (double)k);
            backup(trace, D, visit, value, variance, n2o, score, v_tmp, var_tmp, gamma);
        }
    } else {
        backup(trace, D, visit, value, variance, n2o, score, score[trace[D - 1]], 0, gamma);
    }
}

/* ------------------------------------------------------------------ core.h:32-50 */
int mo_get_all_childs(int index, const int32_t *child, int M, uint8_t *mark) {
    int32_t *queue = (int32_t *)malloc(sizeof(int32_t) * (size_t)M);
    memset(mark, 0, (size_t)M);
    int head = 0, tail = 0, count = 0;
    queue[tail++] = index; mark[index] = 1; count = 1;
    while (head < tail) {
        int n = queue[head++];
        for (int c = 0; c < MO_NA; ++c) {
            int ch = child[(size_t)n * MO_NA + c];
            if (!mark[ch]) { mark[ch] = 1; queue[tail++] = ch; ++count; }
        }
    }
    free(queue);
    return count;
}

/* test evaluator: exact in integer + exactly representable floats, so device and host agree bit for bit */
void mo_synthetic_eval(const uint32_t *k, float *v, float *var) {
    uint32_t h = 2166136261u;
    for (int i = 0; i < 11; ++i) { h ^= k[i]; h *= 16777619u; }
    h ^= h >> 15; h *= 2246822519u; h ^= h >> 13;
    *v = (float)((h >> 7) & 0x3fffu) * 0.00390625f;
    *var = 0.5f + (float)((h >> 21) & 0x3ffu) * 0.0625f;
}

/* test evaluator for the distributional mode: integer hash per bin -> weights 1..256, normalised with one float division */
void mo_synthetic_dist(const uint32_t *k, int bins, float *dist) {
    uint32_t raw[256], sum = 0;
    for (int b = 0; b < bins; ++b) {
        uint32_t h = 2166136261u;
        for (int i = 0; i < 11; ++i) { h ^= k[i]; h *= 16777619u; }
        h ^= (uint32_t)b * 0x9E3779B9u; h *= 16777619u;
        h ^= h >> 15; h *= 2246822519u; h ^= h >> 13;
        raw[b] = ((h >> 9) & 0xffu) + 1u;
        sum += raw[b];
    }
    for (int b = 0; b < bins; ++b) dist[b] = (float)raw[b] / (float)sum;
}

/* dist_oracle.c */
int do_select_trace_distributional(int index, const int32_t *child, const float *node_stats, int low, int32_t *trace,
                                   int max_trace, mo_rand_fn rnd, void *ctx);
void do_backup_trace_distributional(const int32_t *trace, int D, float *node_stats, float *node_dist, int bins, double r,
                                    const float *dist, double vmin, double vmax);
void dn_forward(const float *weights, const int8_t *states, int k, int bins, float *dist);   /* distnet_oracle.c */

/* ================================================================== tree agent (agents/agent.py) */
void vo_forward(const float *weights, const int8_t *states, int k, float *v, float *var); /* valuenet_oracle.c */

typedef struct { int32_t *slot; int cap; int words; } mo_table; /* open addressing; slot = idx, 0 empty, -1 tombstone */

struct mo_agent {
    mo_config cfg;
    int app, scoring, randomizer;
    int M, root, episode;
    int32_t *child; int32_t *visit_n; float *value_n, *variance_n; int32_t *episode_n; float *score; uint8_t *end_n;
    uint32_t *game;                 /* game_arr, agent.py:70 — 20 words per slot */
    int32_t *available; int n_avail;             /* deque, popped from the right (agent.py:99) */
    int32_t *n2o; uint32_t *ostate; int32_t *ovisit; float *ovalue, *ovariance; uint8_t *oend;
    int32_t *oavailable; int n_oavail;
    mo_table ntab, otab;
    uint32_t rng;
    long counters[6];
    int32_t last_trace[512]; int last_D;
    int overflow;
    uint8_t *end_scratch;
    float *nstat, *ndist;          /* MO_MODE_DIST: node_stats f32[M][5], node_dist f32[M][bins] */
    uint8_t *replay_rows; int replay_n;   /* ValueSim.memory rows (212 B), filled by remove_nodes */
    /* overflow_reset (the engine's policy beyond the reference, include/b200_tetris_mcts.h; used by bench.py): see drop_tree() */
    int reroot_pending, reset_hit, in_expand; long resets;
    uint32_t live[TO_RECORD_WORDS];       /* the game last handed to update_root (the object play.py owns) */
    /* CPU model of the engine's PATH CACHE (search_dev.cuh, B200_PATH_CACHE): per level of the last trace the node, its de-duplicated
     * children and THEIR statistics as the engine keeps them next to the trace.  The model applies the engine's coherence rules (natural-slot
     * update at backup, invalidation on a transposition inside the path, on collection, re-rooting and tree drop) and CHECKS at every
     * selection that every cached value still equals the arena's: pc_errors must stay 0.  Diagnostic only (mo_agent_pc_*). */
    int pc_on, pc_len; long pc_errors, pc_irregular, pc_shared, pc_levels, pc_sims, pc_full_walks;
    int32_t pc_node[512]; int pc_k[512]; int32_t pc_cn[512][MO_NA], pc_co[512][MO_NA];
    int32_t pc_visit[512][MO_NA]; float pc_value[512][MO_NA], pc_variance[512][MO_NA];
    /* layout of the engine: the entry of level L keeps the children's statistics as of the walk that FILLED it; the statistics of the child
     * the walk picked there (pc_pick) are read from the own-statistics record of level L+1, which the backup rewrites every simulation */
    int pc_pick[512]; int32_t pc_own_visit[512]; float pc_own_value[512], pc_own_variance[512];
    /* the last selection's phase 1: levels served, and {served levels whose pick changed, stopped at a cached level by check_low, ended on a
     * cached terminal leaf} */
    int pc_last_served, pc_last_ev[3];
};

static uint64_t hash_words(const uint32_t *w, int n) {
    uint64_t h = 1469598103934665603ull;
    for (int i = 0; i < n; ++i) { h ^= w[i]; h *= 1099511628211ull; }
    h ^= h >> 29;
    return h;
}
static void tab_init(mo_table *t, int M, int words) {
    int cap = 16; while (cap < 4 * M) cap <<= 1;
    t->cap = cap; t->words = words; t->slot = (int32_t *)calloc((size_t)cap, sizeof(int32_t));
}
static int tab_find(const mo_table *t, const uint32_t *store, const uint32_t *key) {
    uint32_t p = (uint32_t)hash_words(key, t->words) & (uint32_t)(t->cap - 1);
    for (;;) {
        int s = t->slot[p];
        if (s == 0) return 0;
        if (s > 0 && memcmp(store + (size_t)s * t->words, key, sizeof(uint32_t) * (size_t)t->words) == 0) return s;
        p = (p + 1) & (uint32_t)(t->cap - 1);
    }
}
static void tab_insert(mo_table *t, const uint32_t *key, int idx) {
    uint32_t p = (uint32_t)hash_words(key, t->words) & (uint32_t)(t->cap - 1);
    while (t->slot[p] > 0) p = (p + 1) & (uint32_t)(t->cap - 1);
    t->slot[p] = idx;
}
static void tab_erase(mo_table *t, const uint32_t *store, const uint32_t *key) {
    uint32_t p = (uint32_t)hash_words(key, t->words) & (uint32_t)(t->cap - 1);
    for (;;) {
        int s = t->slot[p];
        if (s == 0) return;
        if (s > 0 && memcmp(store + (size_t)s * t->words, key, sizeof(uint32_t) * (size_t)t->words) == 0) { t->slot[p] = -1; return; }
        p = (p + 1) & (uint32_t)(t->cap - 1);
    }
}

static uint32_t agent_rand(void *ctx) { /* per-agent xorshift32 (replaces libc rand / random.randint, SURVEY H4) */
    mo_agent *a = (mo_agent *)ctx;
    uint32_t s = a->rng;
    s ^= s << 13; s ^= s >> 17; s ^= s << 5;
    a->rng = s;
    return s;
}

mo_agent *mo_agent_create(const mo_config *cfg, int app, int scoring, int randomizer) {
    mo_agent *a = (mo_agent *)calloc(1, sizeof(mo_agent));
    a->cfg = *cfg; a->app = app; a->scoring = scoring; a->randomizer = randomizer;
    int M = a->M = cfg->max_nodes;
    a->child = (int32_t *)calloc((size_t)M * MO_NA, 4);
    a->visit_n = (int32_t *)calloc((size_t)M, 4); a->value_n = (float *)calloc((size_t)M, 4);
    a->variance_n = (float *)calloc((size_t)M, 4); a->episode_n = (int32_t *)calloc((size_t)M, 4);
    a->score = (float *)calloc((size_t)M, 4); a->end_n = (uint8_t *)calloc((size_t)M, 1);
    a->game = (uint32_t *)calloc((size_t)M * TO_RECORD_WORDS, 4);
    /* agent.py:70: every slot starts as a fresh env(*env_args) object (default-seeded in the oracle env) */
    to_game g0; uint32_t rec0[TO_RECORD_WORDS];
    to_init(&g0, app, scoring, randomizer); to_pack(&g0, rec0);
    for (int i = 0; i < M; ++i) memcpy(a->game + (size_t)i * TO_RECORD_WORDS, rec0, sizeof(rec0));
    a->available = (int32_t *)malloc(sizeof(int32_t) * (size_t)M);
    for (int i = 1; i < M; ++i) a->available[i - 1] = i;   /* agent.py:72 deque(range(1, M)) */
    a->n_avail = M - 1;
    a->n2o = (int32_t *)calloc((size_t)M, 4);
    a->ostate = (uint32_t *)calloc((size_t)M * TO_OBSKEY_WORDS, 4);
    a->ovisit = (int32_t *)calloc((size_t)M, 4); a->ovalue = (float *)calloc((size_t)M, 4);
    a->ovariance = (float *)calloc((size_t)M, 4); a->oend = (uint8_t *)calloc((size_t)M, 1);
    if (cfg->mode == MO_MODE_DIST) {
        a->nstat = (float *)calloc((size_t)M * 5, 4);
        a->ndist = (float *)calloc((size_t)M * (size_t)cfg->dist_bins, 4);
    }
    a->oavailable = (int32_t *)malloc(sizeof(int32_t) * (size_t)M);
    for (int i = 1; i < M; ++i) a->oavailable[i - 1] = i;
    a->n_oavail = M - 1;
    tab_init(&a->ntab, M, TO_RECORD_WORDS); tab_init(&a->otab, M, TO_OBSKEY_WORDS);
    a->rng = cfg->search_seed ? cfg->search_seed : 0x2545F491u;
    return a;
}

void mo_agent_destroy(mo_agent *a) {
    if (!a) return;
    free(a->child); free(a->visit_n); free(a->value_n); free(a->variance_n); free(a->episode_n); free(a->score);
    free(a->end_n); free(a->game); free(a->available); free(a->n2o); free(a->ostate); free(a->ovisit);
    free(a->ovalue); free(a->ovariance); free(a->oend); free(a->oavailable); free(a->ntab.slot); free(a->otab.slot); free(a->end_scratch); free(a->nstat); free(a->ndist);
    free(a);
}

/* The engine's overflow_reset policy (NOT in the reference, which dies at this point: IndexError agent.py:99 / UB agent.cpp:227-231):
 * a collection that leaves fewer than max_nodes/8 free node slots means the reachable set itself fills the arena; the whole tree is
 * dropped (every array zeroed except the game slots, free lists as at construction, both tables emptied) and the agent re-roots at
 * the live game before its next simulation / inside the running update_root.  Mirrors k_gc + reset_tree (kernels.cuh, search_dev.cuh). */
static void drop_tree(mo_agent *a) {
    int M = a->M;
    memset(a->child, 0, (size_t)M * MO_NA * 4);
    memset(a->visit_n, 0, (size_t)M * 4); memset(a->value_n, 0, (size_t)M * 4); memset(a->variance_n, 0, (size_t)M * 4);
    memset(a->episode_n, 0, (size_t)M * 4); memset(a->score, 0, (size_t)M * 4); memset(a->end_n, 0, (size_t)M);
    memset(a->n2o, 0, (size_t)M * 4);
    memset(a->ostate, 0, (size_t)M * TO_OBSKEY_WORDS * 4);
    memset(a->ovisit, 0, (size_t)M * 4); memset(a->ovalue, 0, (size_t)M * 4); memset(a->ovariance, 0, (size_t)M * 4); memset(a->oend, 0, (size_t)M);
    if (a->nstat) { memset(a->nstat, 0, (size_t)M * 5 * 4); memset(a->ndist, 0, (size_t)M * (size_t)a->cfg.dist_bins * 4); }
    for (int i = 1; i < M; ++i) { a->available[i - 1] = i; a->oavailable[i - 1] = i; }
    a->n_avail = M - 1; a->n_oavail = M - 1;
    memset(a->ntab.slot, 0, sizeof(int32_t) * (size_t)a->ntab.cap);
    memset(a->otab.slot, 0, sizeof(int32_t) * (size_t)a->otab.cap);
    a->reroot_pending = 1; a->reset_hit = 1; a->resets += 1;
    a->pc_len = 0;
}

static void remove_nodes_ref(mo_agent *a);
static void remove_nodes(mo_agent *a) {
    a->pc_len = 0;                  /* path cache: a collection invalidates it (k_gc) */
    remove_nodes_ref(a);
    if (a->cfg.overflow_reset && a->n_avail < a->M / 8) drop_tree(a);
}

/* agent.py:206-257 remove_nodes -> get_all_childs + update_available + reset_arrays */
static void remove_nodes_ref(mo_agent *a) {
    int M = a->M;
    a->counters[3] += 1;
    uint8_t *occ = (uint8_t *)malloc((size_t)M), *oocc = (uint8_t *)calloc((size_t)M, 1);
    mo_get_all_childs(a->root, a->child, M, occ);                     /* agent.py:210 */
    a->n_avail = 0;
    for (int i = 0; i < M; ++i) if (!occ[i]) a->available[a->n_avail++] = i;   /* agent.py:192, ascending */
    for (int i = 0; i < M; ++i) if (occ[i]) oocc[a->n2o[i]] = 1;      /* agent.py:198 */
    a->n_oavail = 0;
    for (int i = 0; i < M; ++i) if (!oocc[i]) a->oavailable[a->n_oavail++] = i;
    /* reset_arrays agent.py:227-244 */
    if (a->cfg.stale_pop) {
        for (int j = 0; j < a->n_avail; ++j)   /* pop(arr[idx]) by the slot's CURRENT (possibly stale) game */
            tab_erase(&a->ntab, a->game, a->game + (size_t)a->available[j] * TO_RECORD_WORDS);
    } else {
        memset(a->ntab.slot, 0, sizeof(int32_t) * (size_t)a->ntab.cap);
        for (int i = 1; i < M; ++i) if (occ[i]) tab_insert(&a->ntab, a->game + (size_t)i * TO_RECORD_WORDS, i);
    }
    for (int j = 0; j < a->n_avail; ++j) {
        int i = a->available[j];
        memset(a->child + (size_t)i * MO_NA, 0, sizeof(int32_t) * MO_NA);
        a->visit_n[i] = 0; a->value_n[i] = 0; a->variance_n[i] = 0; a->episode_n[i] = 0; a->score[i] = 0; a->end_n[i] = 0;
        if (a->nstat) { memset(a->nstat + (size_t)i * 5, 0, 20); memset(a->ndist + (size_t)i * a->cfg.dist_bins, 0, 4 * (size_t)a->cfg.dist_bins); }
    }
    /* ValueSim.remove_nodes -> store_nodes(self.obs_available) (ValueSim.py:101-159): freed observations with
     * visit >= min_visits_to_store and not end, in ascending index order, until the memory is full */
    if (a->cfg.replay_cap > 0) {
        if (!a->replay_rows) { a->replay_rows = (uint8_t *)malloc((size_t)a->cfg.replay_cap * 212); a->replay_n = 0; }
        for (int j = 0; j < a->n_oavail && a->replay_n < a->cfg.replay_cap; ++j) {
            int i = a->oavailable[j];
            if (a->ovisit[i] < a->cfg.replay_min_visits || a->ovisit[i] == 0 || a->oend[i]) continue;
            uint8_t *dst = a->replay_rows + (size_t)a->replay_n * 212;
            const uint32_t *key = a->ostate + (size_t)i * TO_OBSKEY_WORDS;
            for (int r = 0; r < 20; ++r)
                for (int c = 0; c < 10; ++c) dst[r * 10 + c] = (uint8_t)((key[r >> 1] >> ((r & 1) * 16 + c)) & 1);
            for (int q = 0; q < 4; ++q) dst[(key[10] >> (8 * q)) & 0xff] = 0xff;
            float f[3] = {a->ovalue[i], a->ovariance[i], (float)a->ovisit[i]};
            memcpy(dst + 200, f, 12);
            a->replay_n += 1;
        }
    }
    for (int j = 0; j < a->n_oavail; ++j)
        tab_erase(&a->otab, a->ostate, a->ostate + (size_t)a->oavailable[j] * TO_OBSKEY_WORDS);
    for (int j = 0; j < a->n_oavail; ++j) {
        int i = a->oavailable[j];
        memset(a->ostate + (size_t)i * TO_OBSKEY_WORDS, 0, sizeof(uint32_t) * TO_OBSKEY_WORDS);
        a->ovisit[i] = 0; a->ovalue[i] = 0; a->ovariance[i] = 0; a->oend[i] = 0;
    }
    /* tombstones accumulate only between rebuilds; compact both tables so probe chains stay short */
    {
        mo_table *tabs[2] = {&a->ntab, &a->otab};
        for (int t = 0; t < 2; ++t) {
            mo_table *tb = tabs[t];
            const uint32_t *store = t == 0 ? a->game : a->ostate;
            int32_t *old = tb->slot;
            tb->slot = (int32_t *)calloc((size_t)tb->cap, sizeof(int32_t));
            for (int p = 0; p < tb->cap; ++p) if (old[p] > 0) tab_insert(tb, store + (size_t)old[p] * tb->words, old[p]);
            free(old);
        }
    }
    free(occ); free(oocc);
}

/* agent.py:90-130 new_node */
static int new_node(mo_agent *a, const to_game *g) {
    uint32_t rec[TO_RECORD_WORDS];
    to_pack(g, rec);
    int idx = tab_find(&a->ntab, a->game, rec);
    if (idx) return idx;
    if (a->n_avail == 0) {
        remove_nodes(a);                                  /* agent.py:96-97 */
        if (a->reset_hit && a->in_expand) return -1;      /* overflow_reset: the tree was dropped under a running expansion */
    }
    if (a->n_avail == 0) { a->overflow = 1; return 0; }   /* reference: IndexError / UB (agent.cpp:227-231) */
    idx = a->available[--a->n_avail];                     /* agent.py:99 pop() from the right */
    memcpy(a->game + (size_t)idx * TO_RECORD_WORDS, rec, sizeof(rec));
    a->episode_n[idx] = a->episode;
    a->score[idx] = (float)g->score;
    if (a->nstat) a->nstat[(size_t)idx * 5 + 2] = (float)g->score;   /* node_stats[idx][2] = reward (core_distributional.py:86,112) */
    tab_insert(&a->ntab, rec, idx);
    uint32_t key[TO_OBSKEY_WORDS];
    to_obskey(g, key);
    int o = tab_find(&a->otab, a->ostate, key);
    if (!o) {
        o = a->oavailable[--a->n_oavail];
        memcpy(a->ostate + (size_t)o * TO_OBSKEY_WORDS, key, sizeof(key));
        a->oend[o] = (uint8_t)g->end;
        tab_insert(&a->otab, key, o);
    }
    a->n2o[idx] = o;
    return idx;
}

/* agent.py:136-145 expand */
static int expand(mo_agent *a, int leaf) {                /* returns -1 when overflow_reset dropped the tree under it */
    to_game g, t;
    to_unpack(&g, a->game + (size_t)leaf * TO_RECORD_WORDS);
    a->counters[1] += 1;
    a->in_expand = 1; a->reset_hit = 0;
    for (int i = 0; i < MO_NA; ++i) {
        t = g;
        to_play(&t, i);
        int c = new_node(a, &t);
        if (c < 0) { a->in_expand = 0; a->counters[1] -= 1; return -1; }   /* the engine counts an expansion when it completes */
        a->child[(size_t)leaf * MO_NA + i] = c;
    }
    a->in_expand = 0;
    return 0;
}

void mo_agent_update_root(mo_agent *a, const uint32_t *rec20) {
    to_game g;
    to_unpack(&g, rec20);
    memcpy(a->live, rec20, sizeof(a->live));
    a->pc_len = 0;                  /* path cache: a new root invalidates it (k_update_root) */
    a->reset_hit = 0;
    a->root = new_node(a, &g);      /* a tree dropped earlier (or inside this call) is simply re-rooted here */
    a->reroot_pending = 0;
    if (g.end) a->episode += 1;
}

static void evaluate(mo_agent *a, const int32_t *obs, int k, float *v, float *var) {
    a->counters[2] += k;
    if (a->cfg.eval_mode == MO_EVAL_SYNTHETIC) {
        for (int i = 0; i < k; ++i) mo_synthetic_eval(a->ostate + (size_t)obs[i] * TO_OBSKEY_WORDS, v + i, var + i);
        return;
    }
    int8_t states[MO_NA * 200];
    for (int i = 0; i < k; ++i) { /* obs key -> int8[20,10] (agent.py:122 stores getState()) */
        const uint32_t *key = a->ostate + (size_t)obs[i] * TO_OBSKEY_WORDS;
        for (int r = 0; r < 20; ++r)
            for (int c = 0; c < 10; ++c) states[i * 200 + r * 10 + c] = (int8_t)((key[r >> 1] >> ((r & 1) * 16 + c)) & 1);
        for (int j = 0; j < 4; ++j) states[i * 200 + ((key[10] >> (8 * j)) & 0xff)] = -1;
    }
    if (a->cfg.eval_mode == MO_EVAL_NET) vo_forward(a->cfg.weights, states, k, v, var);
    else a->cfg.eval_cb(a->cfg.eval_ctx, states, k, v, var);
}

/* ---- path-cache model (see struct mo_agent) */
static int pc_pick_of(const mo_agent *a, int L, int next_node) {
    for (int j = 0; j < a->pc_k[L]; ++j) if (a->pc_cn[L][j] == next_node) return j;
    return -1;
}
static void pc_fill(mo_agent *a, int L, const int32_t *trace, int D) {
    int node = trace[L];
    a->pc_node[L] = node;
    int k = mo_unique_child_obs(node, a->child, a->score, a->n2o, a->pc_cn[L], a->pc_co[L]);
    a->pc_k[L] = k;
    for (int j = 0; j < k; ++j) {
        int o = a->pc_co[L][j];
        a->pc_visit[L][j] = a->ovisit[o]; a->pc_value[L][j] = a->ovalue[o]; a->pc_variance[L][j] = a->ovariance[o];
    }
    a->pc_pick[L] = L + 1 < D ? pc_pick_of(a, L, trace[L + 1]) : -1;
}
/* The engine's phase 1 (select_trace, search_dev.cuh) restated lane for lane: eight lanes evaluate eight consecutive cached levels, the walk
 * follows the cached path up to the first lane that stops.  Returns the number of levels served; *idx_out = the node the walk stands on
 * afterwards (the leaf if *ended), picks[] = the pick (index into the level's child list) of every served level.  Checked against the true
 * walk in pc_on_select: a wrong stop rule shows up as pc_errors. */
static int pc_emulate_phase1(const mo_agent *a, int root, int *idx_out, int *ended_out, int *picks, int *ev) {
    int D = 0, idx = root, fast = a->pc_len > 0, ended = 0;
    const int pcl = a->pc_len;
    while (fast) {
        int have[8], e_node[8], pick[8], next[8], leaf[8], bail[8], changed[8], lowb[8];
        for (int lane = 0; lane < 8; ++lane) {
            int L = D + lane;
            have[lane] = L < pcl; e_node[lane] = 0; pick[lane] = 7; next[lane] = 0; leaf[lane] = 0; bail[lane] = 0; changed[lane] = 0; lowb[lane] = 0;
            if (!have[lane]) continue;
            e_node[lane] = a->pc_node[L];
            int k = a->pc_k[L];
            if (k == 0) { leaf[lane] = 1; continue; }
            int32_t vis[MO_NA]; float val[MO_NA], var[MO_NA];
            int lowhit = 0;
            for (int j = 0; j < k; ++j) {
                int32_t v = a->pc_visit[L][j]; float vl = a->pc_value[L][j], vr = a->pc_variance[L][j];
                if (j == a->pc_pick[L]) { v = a->pc_own_visit[L + 1]; vl = a->pc_own_value[L + 1]; vr = a->pc_own_variance[L + 1]; }
                if (v < a->cfg.low) lowhit = 1;
                int c = a->pc_cn[L][j];
                float t = vl + a->score[c];
                vis[j] = v; val[j] = t - a->score[a->pc_node[L]]; var[j] = vr;
            }
            if (lowhit) { bail[lane] = 1; lowb[lane] = 1; continue; }
            int nx = mo_policy_clt(a->pc_cn[L], vis, val, var, k);
            for (int j = 0; j < k; ++j) if (a->pc_cn[L][j] == nx) pick[lane] = j;
            next[lane] = nx;
        }
        for (int lane = 0; lane < 8; ++lane) {
            int expect = lane == 0 ? idx : next[lane - 1];
            if (have[lane] && e_node[lane] != expect) bail[lane] = 1;
            changed[lane] = have[lane] && !leaf[lane] && !bail[lane] && pick[lane] != a->pc_pick[D + lane];
        }
        int first = 8;
        for (int lane = 7; lane >= 0; --lane) if (!have[lane] || bail[lane] || leaf[lane] || changed[lane]) first = lane;
        int first_served = first < 8 && have[first] && !bail[first];
        int served = first + (first_served ? 1 : 0);
        for (int lane = 0; lane < served; ++lane) { picks[D + lane] = leaf[lane] ? -1 : pick[lane]; ev[0] += changed[lane]; }
        if (first < 8 && lowb[first] && e_node[first] == (first == 0 ? idx : next[first - 1])) ev[1] += 1;
        int last_next = next[served > 0 ? served - 1 : 0];
        ended = first_served && leaf[first];
        ev[2] |= ended;
        D += served;
        if (ended) idx = e_node[first];
        else if (served > 0) idx = last_next;
        if (ended) fast = 0;
        else if (first < 8 || D >= pcl) fast = 0;
    }
    *idx_out = idx; *ended_out = ended;
    return D;
}

static void pc_on_select(mo_agent *a, const int32_t *trace, int D) {
    if (!a->pc_on) return;
    {   /* the engine's phase 1 must serve a prefix of the TRUE trace, stand on the true next node (or the true leaf), with the true picks */
        int idx = 0, ended = 0, picks[512];
        a->pc_last_ev[0] = a->pc_last_ev[1] = a->pc_last_ev[2] = 0;
        int P = pc_emulate_phase1(a, trace[0], &idx, &ended, picks, a->pc_last_ev);
        a->pc_last_served = P;
        int bad = P > D || (ended ? (P != D || idx != trace[D - 1]) : (P < D ? idx != trace[P] : 1));
        if (P == D && !ended) bad = 1;                       /* a walk that serves every level must have ended on a cached leaf */
        for (int L = 0; L < P && L + 1 < D && !bad; ++L) bad = picks[L] < 0 || a->pc_cn[L][picks[L]] != trace[L + 1];
        if (P > 0 && P <= D && !bad && picks[P - 1] < 0 && !ended) bad = 1;
        if (bad) {
            if (a->pc_errors < 5) fprintf(stderr, "path-cache model: phase-1 emulation disagrees with the walk (served %d of %d, ended %d, idx %d)\n", P, D, ended, idx);
            a->pc_errors += 1;
        }
    }
    int L = 0;
    while (L < a->pc_len && L < D && a->pc_node[L] == trace[L]) {
        int32_t cn[MO_NA], co[MO_NA];
        int k = mo_unique_child_obs(trace[L], a->child, a->score, a->n2o, cn, co);
        int bad = k != a->pc_k[L];
        for (int j = 0; j < k && !bad; ++j) {
            int o = co[j];
            /* what the engine's walk reads for child j: the entry, except for the child picked last time (own record of the next level) */
            int32_t vis = a->pc_visit[L][j]; float val = a->pc_value[L][j], var = a->pc_variance[L][j];
            if (j == a->pc_pick[L]) { vis = a->pc_own_visit[L + 1]; val = a->pc_own_value[L + 1]; var = a->pc_own_variance[L + 1]; }
            bad = cn[j] != a->pc_cn[L][j] || o != a->pc_co[L][j] || vis != a->ovisit[o] ||
                  memcmp(&val, &a->ovalue[o], 4) != 0 || memcmp(&var, &a->ovariance[o], 4) != 0;
        }
        if (bad) {
            if (a->pc_errors < 5) fprintf(stderr, "path-cache model: stale entry at level %d of %d (node %d)\n", L, D, trace[L]);
            a->pc_errors += 1;
        }
        /* the walk picks another child than last time: the old pick's latest statistics go back into the entry, the new pick is recorded */
        int np = L + 1 < D ? pc_pick_of(a, L, trace[L + 1]) : -1;
        if (np != a->pc_pick[L]) {
            int op = a->pc_pick[L];
            if (op >= 0) { a->pc_visit[L][op] = a->pc_own_visit[L + 1]; a->pc_value[L][op] = a->pc_own_value[L + 1]; a->pc_variance[L][op] = a->pc_own_variance[L + 1]; }
            a->pc_pick[L] = np;
        }
        ++L;
    }
    a->pc_shared += L; a->pc_levels += D; a->pc_sims += 1;
    if (L == 0) a->pc_full_walks += 1;
    for (; L < D; ++L) pc_fill(a, L, trace, D);
    a->pc_len = D;
}
static void pc_on_backup(mo_agent *a, const int32_t *trace, int D, int expanded) {
    if (!a->pc_on || a->pc_len == 0) return;             /* invalidated since the selection (collection / tree drop inside the expansion) */
    int newlen = expanded ? D - 1 : D;                   /* the expanded leaf's entry says "no children": stale */
    /* Stale copies after this backup, by level, as k_backup (backup_game) finds them: (a) an observation twice on the trace (i < j): the
     * backup runs leaf -> root in windows of 32 levels, so the own record of the deeper occurrence (read by level j-1) holds an
     * intermediate value.  k_backup truncates at the shallower occurrence i when the two lie in different windows, and below the window
     * (its lowest level - 1) when they share one, whose levels it then folds one by one without writing own records; (b) a cached child
     * observation that is some trace node's own without being that level's picked child.  Everything above the shallowest stale level stays
     * valid: the cache is truncated there. */
    int stale = newlen;
    for (int i = 0; i < D; ++i)
        for (int j = i + 1; j < D; ++j) {
            if (a->n2o[trace[i]] != a->n2o[trace[j]]) continue;
            int wi = (D - 1 - i) / 32, wj = (D - 1 - j) / 32;  /* window index counted from the leaf */
            int bottom = D - 1 - 32 * wi - 31;                 /* the window's lowest level */
            int s_ij = wi == wj ? (bottom - 1 > 0 ? bottom - 1 : 0) : i;
            if (s_ij < stale) stale = s_ij;
        }
    for (int L = 0; L < stale; ++L)
        for (int j = 0; j < a->pc_k[L]; ++j) {
            if (j == a->pc_pick[L]) continue;
            for (int i = 0; i < D; ++i) if (a->pc_co[L][j] == a->n2o[trace[i]] && L < stale) stale = L;
        }
    if (stale < newlen) { a->pc_irregular += 1; newlen = stale; }
    for (int i = 0; i < D; ++i) {                        /* the backup rewrites the own record of every trace level */
        int o = a->n2o[trace[i]];
        a->pc_own_visit[i] = a->ovisit[o]; a->pc_own_value[i] = a->ovalue[o]; a->pc_own_variance[i] = a->ovariance[o];
    }
    a->pc_len = newlen;
}
void mo_agent_pc_enable(mo_agent *a, int on) { a->pc_on = on; a->pc_len = 0; }

/* The path-cache model over a given sequence of simulations on a fixed tree in the reference's layout (child[M][7], score, n2o): every walk
 * ends at a terminal leaf, nothing is expanded, the cache starts empty.  Simulation s walks traces[trace_off[s] .. trace_off[s+1]) on the
 * statistics visit / value / variance[s][M] and its backup leaves [s+1][M].  Per simulation: served[s] = the levels the engine's phase 1
 * serves, pc_len[s] = the valid length after the backup, ev[s][3] = {served levels whose pick changed, stops at a cached level because of
 * check_low, the walk ended on a cached terminal leaf}.  Returns the number of stale reads the model found (0 when the rules hold). */
long mo_pc_replay(int M, const int32_t *child, const float *score, const int32_t *n2o, int low, int S, const int32_t *traces,
                  const int32_t *trace_off, const int32_t *visit, const float *value, const float *variance, int32_t *served,
                  int32_t *pc_len, int32_t *ev) {
    mo_config cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.max_nodes = M; cfg.low = low;
    mo_agent *a = mo_agent_create(&cfg, 1, 0, 0);
    memcpy(a->child, child, (size_t)M * MO_NA * 4); memcpy(a->score, score, (size_t)M * 4); memcpy(a->n2o, n2o, (size_t)M * 4);
    a->pc_on = 1; a->pc_len = 0;
    for (int s = 0; s < S; ++s) {
        const int32_t *tr = traces + trace_off[s];
        const int D = trace_off[s + 1] - trace_off[s];
        const size_t b = (size_t)s * M;
        memcpy(a->ovisit, visit + b, (size_t)M * 4); memcpy(a->ovalue, value + b, (size_t)M * 4); memcpy(a->ovariance, variance + b, (size_t)M * 4);
        pc_on_select(a, tr, D);
        served[s] = a->pc_last_served;
        for (int k = 0; k < 3; ++k) ev[3 * s + k] = a->pc_last_ev[k];
        memcpy(a->ovisit, visit + b + M, (size_t)M * 4); memcpy(a->ovalue, value + b + M, (size_t)M * 4); memcpy(a->ovariance, variance + b + M, (size_t)M * 4);
        pc_on_backup(a, tr, D, 0);
        pc_len[s] = a->pc_len;
    }
    long err = a->pc_errors;
    mo_agent_destroy(a);
    return err;
}
void mo_agent_pc_stats(const mo_agent *a, long *out7) {
    out7[0] = a->pc_errors; out7[1] = a->pc_irregular; out7[2] = a->pc_shared; out7[3] = a->pc_levels; out7[4] = a->pc_sims; out7[5] = a->pc_full_walks; out7[6] = a->pc_len;
}

int mo_agent_mcts(mo_agent *a, int sims) {
    const mo_config *cf = &a->cfg;
    for (int s = 0; s < sims; ++s) {
        if (a->reroot_pending) {        /* overflow_reset: the tree was dropped; re-root at the live game (reset_tree, search_dev.cuh) */
            to_game lv;
            to_unpack(&lv, a->live);
            a->reset_hit = 0;
            a->root = new_node(a, &lv);
            a->reroot_pending = 0;
        }
        if (cf->mode == MO_MODE_DIST) {
            /* The loop agents/DistValueSimOnline.py:36-75 sketches (not runnable upstream), on the numba cores:
             * select_trace_distributional -> r = leaf score; leaf not ended: dist = net(leaf state), expand;
             * ended: all mass in bin 0 (v_dummy, DistValueSimOnline.py:26-27) -> backup_trace_distributional */
            float dist[256];
            int D = do_select_trace_distributional(a->root, a->child, a->nstat, cf->low, a->last_trace, 512, agent_rand, a);
            if (D < 0) return -2;
            a->last_D = D; a->counters[0] += 1; a->counters[4] += D;
            int leaf = a->last_trace[D - 1];
            to_game lg;
            to_unpack(&lg, a->game + (size_t)leaf * TO_RECORD_WORDS);
            if (!lg.end) {
                const uint32_t *key = a->ostate + (size_t)a->n2o[leaf] * TO_OBSKEY_WORDS;
                a->counters[2] += 1;
                if (cf->eval_mode == MO_EVAL_SYNTHETIC) mo_synthetic_dist(key, cf->dist_bins, dist);
                else {
                    int8_t st[200];
                    for (int r = 0; r < 20; ++r)
                        for (int c = 0; c < 10; ++c) st[r * 10 + c] = (int8_t)((key[r >> 1] >> ((r & 1) * 16 + c)) & 1);
                    for (int j = 0; j < 4; ++j) st[(key[10] >> (8 * j)) & 0xff] = -1;
                    if (cf->eval_mode == MO_EVAL_CALLBACK) cf->eval_cb(cf->eval_ctx, st, 1, dist, NULL);   /* dist_bins probabilities into v */
                    else dn_forward(cf->weights, st, 1, cf->dist_bins, dist);
                }
                if (expand(a, leaf) < 0) continue;       /* tree dropped: this simulation is abandoned */
                if (a->overflow) return -1;
            } else {
                memset(dist, 0, sizeof(float) * (size_t)cf->dist_bins);
                dist[0] = 1.f;
            }
            do_backup_trace_distributional(a->last_trace, D, a->nstat, a->ndist, cf->dist_bins, (double)lg.score, dist, cf->dist_vmin, cf->dist_vmax);
            continue;
        }
        int D = mo_select_trace_obs(a->root, a->child, a->ovisit, a->ovalue, a->ovariance, a->score, a->n2o, cf->low,
                                    a->last_trace, 512, agent_rand, a);
        if (D < 0) return -2;
        a->last_D = D;
        a->counters[0] += 1; a->counters[4] += D;
        if (cf->mode == MO_MODE_LP) pc_on_select(a, a->last_trace, D);
        int leaf = a->last_trace[D - 1];
        to_game lg;
        to_unpack(&lg, a->game + (size_t)leaf * TO_RECORD_WORDS);
        if (cf->mode == MO_MODE_LP) {                     /* ValueSimLP.py:44-70 */
            int32_t c_nodes[MO_NA], c_obs[MO_NA]; float v[MO_NA], var[MO_NA]; int k = 0;
            if (!lg.end) {
                if (expand(a, leaf) < 0) continue;       /* tree dropped: this simulation is abandoned (no evaluation, no backup) */
                if (a->overflow) return -1;
                k = mo_unique_child_obs(leaf, a->child, a->score, a->n2o, c_nodes, c_obs);
                evaluate(a, c_obs, k, v, var);
            }
            const uint8_t *endarr = a->end_n;
            if (cf->lp_end_from_obs) { /* agent.cpp:538 tests end_obs[o]; backup_trace_obs_LP indexes end[] by child id */
                if (!a->end_scratch) a->end_scratch = (uint8_t *)calloc((size_t)a->M, 1);
                for (int i = 0; i < k; ++i) a->end_scratch[c_nodes[i]] = a->oend[c_obs[i]];
                endarr = a->end_scratch;
            }
            if (cf->lp_var_gamma2) {
                mo_backup_trace_obs_LP(a->last_trace, D, a->ovisit, a->ovalue, a->ovariance, a->n2o, a->score, endarr,
                                       c_nodes, c_obs, k, v, var, cf->gamma, 0, 1);
            } else { /* agent.cpp:517-566 variant: var_tmp /= k (no gamma^2) */
                if (k > 0) {
                    double v_tmp = 0, var_tmp = 0;
                    for (int i = 0; i < k; ++i) {
                        int c = c_nodes[i], o = c_obs[i];
                        if (a->ovisit[o] == 0) {
                            a->ovisit[o] += 1;
                            if (endarr[c]) { a->ovalue[o] = 0; a->ovariance[o] = 0; }
                            else { a->ovalue[o] = v[i]; a->ovariance[o] = var[i]; }
                        }
                        v_tmp += a->score[c] + cf->gamma * a->ovalue[o];
                        var_tmp += a->ovariance[o];
                    }
                    v_tmp /= k; var_tmp /= k;
                    /* agent.cpp:496 takes float _val/_var */
                    mo_backup_trace_obs(a->last_trace, D, a->ovisit, a->ovalue, a->ovariance, a->n2o, a->score,
                                        (double)(float)v_tmp, (double)(float)var_tmp, cf->gamma);
                } else {
                    mo_backup_trace_obs(a->last_trace, D, a->ovisit, a->ovalue, a->ovariance, a->n2o, a->score,
                                        a->score[leaf], 0, cf->gamma);
                }
            }
            if (cf->lp_end_from_obs) for (int i = 0; i < k; ++i) a->end_scratch[c_nodes[i]] = 0;
            pc_on_backup(a, a->last_trace, D, !lg.end);
        } else if (cf->mode == MO_MODE_SINGLE) {          /* ValueSim.py:76-94 */
            double _value = (double)lg.score, _variance = 0;
            if (!lg.end) {
                float v, var; int32_t o = a->n2o[leaf];
                evaluate(a, &o, 1, &v, &var);
                /* ValueSim.py:86: int + np.float32 -> float32 under numpy>=2 (NEP 50), the version in this image */
                float sum = (float)lg.score + v;
                _value = (double)sum; _variance = (double)var;
                if (expand(a, leaf) < 0) continue;
                if (a->overflow) return -1;
            }
            mo_backup_trace_obs(a->last_trace, D, a->ovisit, a->ovalue, a->ovariance, a->n2o, a->score, _value, _variance, cf->gamma);
        } else {                                          /* Vanilla.py:41-64 */
            double _value, _variance;
            if (!lg.end) {
                to_game r = lg;
                while (!r.end) { to_play(&r, (int)(agent_rand(a) % MO_NA)); a->counters[5] += 1; }
                _value = (double)r.score; _variance = cf->rollout_variance;
                if (expand(a, leaf) < 0) continue;
                if (a->overflow) return -1;
            } else { _value = (double)lg.score; _variance = 0; }
            mo_backup_trace_obs(a->last_trace, D, a->ovisit, a->ovalue, a->ovariance, a->n2o, a->score, _value, _variance, cf->gamma);
        }
    }
    return 0;
}

/* agent.py:153-185 compute_stats + get_action */
int mo_agent_get_action(mo_agent *a, float *stats) {
    int idx = a->root;
    if (a->cfg.mode == MO_MODE_DIST) {                      /* DistValueSimOnline.py:77-104: visit, mean + reward - root reward, variance */
        for (int i = 0; i < MO_NA; ++i) {
            int c = a->child[(size_t)idx * MO_NA + i];
            const float *ns = a->nstat + (size_t)c * 5;
            stats[i] = ns[0];
            stats[MO_NA + i] = (ns[1] + ns[2]) - a->nstat[(size_t)idx * 5 + 2];
            stats[2 * MO_NA + i] = ns[3];
        }
        int b = 0;
        for (int i = 1; i < MO_NA; ++i) if (stats[MO_NA + i] > stats[MO_NA + b]) b = i;
        return b;
    }
    for (int i = 0; i < MO_NA; ++i) {
        int c = a->child[(size_t)idx * MO_NA + i];
        int o = a->n2o[c];
        float diff = a->score[c] - a->score[idx];           /* agent.py:171 */
        stats[i] = (float)a->ovisit[o];
        stats[MO_NA + i] = a->ovalue[o] + diff;             /* agent.py:175 */
        stats[2 * MO_NA + i] = a->ovariance[o];
    }
    int best = 0;
    for (int i = 1; i < MO_NA; ++i) if (stats[MO_NA + i] > stats[MO_NA + best]) best = i;   /* np.argmax: first max */
    return best;
}

int mo_agent_root(const mo_agent *a) { return a->root; }
/* TreeAgent.remove_nodes() is a public method (agents/agent.py:246-257): a caller may collect between moves */
void mo_agent_remove_nodes(mo_agent *a) { remove_nodes(a); }
int mo_agent_n_free(const mo_agent *a) { return a->n_avail; }   /* len(self.available), agents/agent.py:72 */
int mo_agent_episode(const mo_agent *a) { return a->episode; }
long mo_agent_counter(const mo_agent *a, int w) { return (w >= 0 && w < 6) ? a->counters[w] : (w == 7 ? a->resets : -1); }

void mo_agent_export(const mo_agent *a, int32_t *child, float *score, int32_t *episode, int32_t *n2o, int32_t *visit,
                     float *value, float *variance, uint8_t *obs_end, uint32_t *game_recs, uint32_t *obs_keys) {
    size_t M = (size_t)a->M;
    if (child) memcpy(child, a->child, M * MO_NA * 4);
    if (score) memcpy(score, a->score, M * 4);
    if (episode) memcpy(episode, a->episode_n, M * 4);
    if (n2o) memcpy(n2o, a->n2o, M * 4);
    if (visit) memcpy(visit, a->ovisit, M * 4);
    if (value) memcpy(value, a->ovalue, M * 4);
    if (variance) memcpy(variance, a->ovariance, M * 4);
    if (obs_end) memcpy(obs_end, a->oend, M);
    if (game_recs) memcpy(game_recs, a->game, M * TO_RECORD_WORDS * 4);
    if (obs_keys) memcpy(obs_keys, a->ostate, M * TO_OBSKEY_WORDS * 4);
}

int mo_agent_replay(mo_agent *a, uint8_t *rows212, int max_rows) {   /* copy out and empty (ValueSim.py:183 memory_index = 0) */
    int n = a->replay_n < max_rows ? a->replay_n : max_rows;
    if (n > 0 && rows212) memcpy(rows212, a->replay_rows, (size_t)n * 212);
    a->replay_n = 0;
    return n;
}

void mo_agent_export_dist(const mo_agent *a, float *node_stats, float *node_dist) {
    if (!a->nstat) return;
    if (node_stats) memcpy(node_stats, a->nstat, (size_t)a->M * 5 * 4);
    if (node_dist) memcpy(node_dist, a->ndist, (size_t)a->M * (size_t)a->cfg.dist_bins * 4);
}

int mo_agent_last_trace(const mo_agent *a, int32_t *trace, int max) {
    int n = a->last_D < max ? a->last_D : max;
    memcpy(trace, a->last_trace, sizeof(int32_t) * (size_t)n);
    return a->last_D;
}
