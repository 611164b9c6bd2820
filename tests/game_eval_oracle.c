/*
 * game_eval_oracle.c — TEST INFRASTRUCTURE ONLY: the C oracle's Vanilla agent with an injected leaf-game evaluator in place of its rollout,
 * a restatement of MCTSAgent::mcts with evaluator type 1 (agents/cppmodule/agent.cpp:440-459): select (low from the config), expand the
 * leaf, evaluate a copy of its packed record with the caller's function, and back (value, variance) up as they are; a game-over leaf backs
 * its score up with variance 0.  The oracle itself (oracle/mcts_oracle.c) is compiled into this file unchanged by inclusion, so the walk,
 * the expansion, the collections and the backup are the oracle's own; an agent made by oracle_py.Agent (liboracle.so, the same source) is
 * driven here through its handle.  Compiled by tests/game_eval_twins.py with the oracle Makefile's flags.
 */
#include "mcts_oracle.c"

typedef void (*ge_eval_fn)(void *ctx, const uint32_t *rec20, float *v, float *var);

/* sims simulations of a MO_MODE_VANILLA agent; returns 0, -1 on arena overflow, -2 on a trace deeper than 512 levels */
int ge_agent_mcts(mo_agent *a, int sims, ge_eval_fn fn, void *ctx) {
    const mo_config *cf = &a->cfg;
    if (cf->mode != MO_MODE_VANILLA || !fn) return -3;
    for (int s = 0; s < sims; ++s) {
        if (a->reroot_pending) {        /* overflow_reset: the tree was dropped; re-root at the live game, as mo_agent_mcts does */
            to_game lv;
            to_unpack(&lv, a->live);
            a->reset_hit = 0;
            a->root = new_node(a, &lv);
            a->reroot_pending = 0;
        }
        int D = mo_select_trace_obs(a->root, a->child, a->ovisit, a->ovalue, a->ovariance, a->score, a->n2o, cf->low,
                                    a->last_trace, 512, agent_rand, a);
        if (D < 0) return -2;
        a->last_D = D;
        a->counters[0] += 1; a->counters[4] += D;
        int leaf = a->last_trace[D - 1];
        to_game lg;
        to_unpack(&lg, a->game + (size_t)leaf * TO_RECORD_WORDS);
        double _value = (double)lg.score, _variance = 0;
        if (!lg.end) {
            uint32_t rec[TO_RECORD_WORDS];
            memcpy(rec, a->game + (size_t)leaf * TO_RECORD_WORDS, sizeof(rec));
            if (expand(a, leaf) < 0) continue;       /* tree dropped: this simulation is abandoned (no evaluation, no backup) */
            if (a->overflow) return -1;
            float v, var;
            fn(ctx, rec, &v, &var);                  /* agent.cpp:450-454 */
            a->counters[2] += 1;
            _value = (double)v; _variance = (double)var;
        }
        mo_backup_trace_obs(a->last_trace, D, a->ovisit, a->ovalue, a->ovariance, a->n2o, a->score, _value, _variance, cf->gamma);
    }
    return 0;
}

/* the agent's check_low stream (what the engine's b200_debug_game_state reads) */
uint32_t ge_agent_rng(const mo_agent *a) { return a->rng; }
