/*
 * mcts_oracle.h — TEST INFRASTRUCTURE ONLY (CPU oracle; never shipped, never on the product path).
 *
 * Plain-C restatement of the reference's search step: the five exported kernels of
 * agents/cppmodule/core.{h,cpp} and the tree agent of agents/agent.py + ValueSim.py / ValueSimLP.py / Vanilla.py.
 * Each function cites the reference file:line it follows.  The core functions are pinned against the
 * reference's OWN core.cpp compiled into oracle/_ref/ (tests/golden/gen_golden.py, tests/test_oracle_pins.py);
 * the agent is pinned against the reference's own Python agents run on the oracle env.
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may use this.
 */
#ifndef MCTS_ORACLE_H
#define MCTS_ORACLE_H
#include <stdint.h>
#include "tetris_oracle.h"
#ifdef __cplusplus
extern "C" {
#endif

#define MO_NA 7 /* n_actions, core.h:17 */

typedef uint32_t (*mo_rand_fn)(void *ctx); /* stands in for libc rand() of core.h:62,76 */

double mo_norm_quantile(double t);                                             /* special.h:26-33 */
void mo_norm_quantile_f32(const int32_t *n, int count, float *out);            /* (float)mo_norm_quantile(n[i]) */
int mo_unique_child_obs(int index, const int32_t *child, const float *score, const int32_t *n2o,
                        int32_t *c_nodes, int32_t *c_obs);                     /* core.h:111-144 */
int mo_policy_clt(const int32_t *nodes, const int32_t *visit, const float *value, const float *variance, int k); /* core.h:83-105 */
int mo_select_trace_obs(int index, const int32_t *child, const int32_t *visit, const float *value,
                        const float *variance, const float *score, const int32_t *n2o, int low,
                        int32_t *trace, int max_trace, mo_rand_fn rnd, void *ctx); /* core.h:167-224 */
void mo_backup_trace_obs(const int32_t *trace, int D, int32_t *visit, float *value, float *variance,
                         const int32_t *n2o, const float *score, double v, double var, double gamma); /* core.h:226-260 */
void mo_backup_trace_mixture_obs(const int32_t *trace, int D, int32_t *visit, float *value, float *variance,
                                 const int32_t *n2o, const float *score, double v, double var, double gamma); /* core.h:262-301 */
void mo_backup_trace_obs_LP(const int32_t *trace, int D, int32_t *visit, float *value, float *variance,
                            const int32_t *n2o, const float *score, const uint8_t *end, const int32_t *c_nodes,
                            const int32_t *c_obs, int k, const float *v, const float *var, double gamma,
                            int mixture, int averaged);                         /* core.h:303-381 */
int mo_get_all_childs(int index, const int32_t *child, int M, uint8_t *mark);  /* core.h:32-50 */
void mo_synthetic_eval(const uint32_t *obskey12, float *v, float *var);        /* test evaluator shared with the device */

/* ---- tree agent (agents/agent.py TreeAgent + ValueSim/ValueSimLP/Vanilla mcts loops) ---- */
enum { MO_MODE_LP = 0, MO_MODE_SINGLE = 1, MO_MODE_VANILLA = 2, MO_MODE_DIST = 3 /* agents/core_distributional.py loop, see mcts_oracle.c */ };
enum { MO_EVAL_SYNTHETIC = 0, MO_EVAL_NET = 1, MO_EVAL_CALLBACK = 2 };
typedef void (*mo_eval_fn)(void *ctx, const int8_t *states, int k, float *v, float *var);

typedef struct {
    int max_nodes;      /* ValueSim.py:16 (100000) / agent.py:36 (500000) */
    int mode;           /* MO_MODE_* */
    double gamma;       /* ValueSim.py:14 0.999, Vanilla.py:9 0.99 */
    int low;            /* ValueSimLP.py:27 (1), Vanilla.py:27 (5) */
    int lp_end_from_obs;   /* SURVEY N1: 0 = Python path (node 'end' never written), 1 = agent.cpp:538 */
    int lp_var_gamma2;     /* SURVEY N1: 1 = core.h:365 (gamma^2/k), 0 = agent.cpp:558 (1/k) */
    double rollout_variance; /* Vanilla.py:54 1e3 */
    int eval_mode;      /* MO_EVAL_* */
    const float *weights;  /* MO_EVAL_NET: packed as valuenet_oracle.c expects */
    mo_eval_fn eval_cb; void *eval_ctx;   /* MO_MODE_DIST: called with k = 1 and var = NULL, writes dist_bins probabilities to v */
    uint32_t search_seed;  /* per-agent xorshift stream replacing rand()/random.randint (SURVEY H4) */
    int stale_pop;         /* agent.py:229-232 erases by the freed slot's STALE game; 1 = reproduce */
    int dist_bins;         /* MO_MODE_DIST: atoms (DistValueSimOnline.py:13: 50) */
    double dist_vmin, dist_vmax;   /* value range (DistValueSimOnline.py:13: 0, 5000) */
    int replay_min_visits, replay_cap;   /* ValueSim.py:14 min_visits_to_store / memory_size; 0 = no replay memory */
    int overflow_reset;    /* NOT the reference: the engine's bench policy (b200_config.overflow_reset) — a collection that leaves fewer than
                              max_nodes/8 free slots drops the tree and re-roots at the live game; 0 = reference behaviour (overflow is an error) */
} mo_config;

typedef struct mo_agent mo_agent;
mo_agent *mo_agent_create(const mo_config *cfg, int app, int scoring, int randomizer);
void mo_agent_destroy(mo_agent *a);
void mo_agent_update_root(mo_agent *a, const uint32_t *rec20);            /* agent.py:296-301 */
int mo_agent_mcts(mo_agent *a, int sims);                                 /* ValueSimLP.py:13-70 etc.; returns 0 or <0 on arena overflow */
int mo_agent_get_action(mo_agent *a, float *stats21);                     /* agent.py:153-185 */
int mo_agent_root(const mo_agent *a);
void mo_agent_remove_nodes(mo_agent *a);                                 /* agent.py:246-257, called explicitly */
int mo_agent_n_free(const mo_agent *a);                                   /* len(self.available) */
int mo_agent_replay(mo_agent *a, uint8_t *rows212, int max_rows);   /* ValueSim.memory rows stored by remove_nodes; empties the memory */
int mo_agent_episode(const mo_agent *a);
long mo_agent_counter(const mo_agent *a, int which); /* 0 sims, 1 expansions, 2 evals, 3 gcs, 4 trace levels, 5 rollout steps, 7 trees dropped (overflow_reset) */
/* export in the reference's array layout (agent.py:58-88); any pointer may be NULL */
void mo_agent_export(const mo_agent *a, int32_t *child, float *score, int32_t *episode, int32_t *n2o,
                     int32_t *visit, float *value, float *variance, uint8_t *obs_end, uint32_t *game_recs,
                     uint32_t *obs_keys);
int mo_agent_last_trace(const mo_agent *a, int32_t *trace, int max);
/* CPU model of the engine's path cache (diagnostic): enable, then out7 = {stale entries found (must be 0), invalidations by a transposition
 * inside the path, levels served from the cache, levels walked, simulations, simulations that found no cache, current valid length} */
void mo_agent_pc_enable(mo_agent *a, int on);
/* the path-cache model over given walks on a fixed tree of terminal leaves: levels served, valid length and events per simulation */
long mo_pc_replay(int M, const int32_t *child, const float *score, const int32_t *n2o, int low, int S, const int32_t *traces,
                  const int32_t *trace_off, const int32_t *visit, const float *value, const float *variance, int32_t *served,
                  int32_t *pc_len, int32_t *ev);
void mo_agent_pc_stats(const mo_agent *a, long *out7);
void mo_agent_export_dist(const mo_agent *a, float *node_stats, float *node_dist);   /* MO_MODE_DIST: f32[M][5], f32[M][bins] */
void mo_synthetic_dist(const uint32_t *obskey12, int bins, float *dist);             /* test evaluator shared with the device */
#ifdef __cplusplus
}
#endif
#endif
