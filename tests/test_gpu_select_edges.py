"""The engine's own walk (k_select_expand -> select_trace, cached and uncached) and action choice (k_root_stats) against the reference's
own core.cpp and agent.py on the designed trees of tests/golden/select_edges_golden.npz.  Each case is loaded into one game of an
engine (b200_debug_load_tree) and searched by the production b200_run_sims: every walk ends at a terminal leaf, so a simulation is
k_select_expand and k_backup's terminal backup on exactly the designed statistics (exact q ties, NaN / infinite q, negative variance,
visit sums at the z(n) table edges and past 2^31, duplicates, check_low draws, chains around the path cache's 8-level rounds, repicks,
transpositions).  The cases are spread over engines of 1, 7, 13 and 64 games in several orders, so that each walks with different warp
partners, with the path cache off and on, the deep lane off and on, one run_sims(1) per simulation and run_sims(k) graph replays.
After every simulation each game's trace must equal the reference's and visit / value / variance must match bit for bit (any NaN equal
to any NaN); at the end of a case its check_low stream, root statistics and action (get_stats, and play_move on the graph-replay runs)
must match.  With the path cache on, each game's valid cache length after every backup and the levels the walks served (counter 13)
must equal the CPU path-cache model's (mcts_oracle.c pc_*, oracle.pc_replay) on the same walks."""
import os

import numpy as np
import pytest

import gpu_twins as G
import select_edges as SE

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "select_edges_golden.npz")
MAX_NODES = 512
GAMES = (1, 7, 13, 64)
ORDERS = 2


@pytest.fixture(scope="module")
def cases():
    cs = SE.load(GOLD)
    assert all(c["digest_ok"] for c in cs), "design() no longer makes the golden's inputs: regenerate tests/golden/select_edges_golden.npz"
    assert max(len(c["n2o"]) for c in cs) <= MAX_NODES
    return cs


@pytest.fixture(scope="module")
def weights():
    from tetris_mcts_b200.model.model_vv import init_weights
    return init_weights(0)


@pytest.fixture(scope="module")
def models(cases, oracle):
    """The path-cache model's (served levels, valid length, events) per simulation of every LP case."""
    return {id(c): SE.pc_model(c, oracle) for c in cases if c["mode"] == "lp" and "trace_full" not in c["tags"]}


def _engine(n, c, weights):
    # net_tc: the deep lane runs only with the tensor-core network (no walk here ends at a leaf that needs it).  Live games are set so that
    # play_move can step them and re-root; the re-rooted node comes from the top of the free lists, above every designed tree.
    from tetris_mcts_b200 import pyTetris as PT
    from tetris_mcts_b200.engine import BatchedEngine
    eng = BatchedEngine(n, max_nodes=MAX_NODES, mode=c["mode"], gamma=c["gamma"], low=c["low"], eval_kind="net_tc", weights=weights,
                        trace_max=SE.TRACE_MAX, path_cache=False)
    eng.set_games(PT.new_games(n, (1, 0, 0), np.arange(7, 7 + n, dtype=np.uint32)))
    return eng


def _layouts(group, n, rng):
    """Orders of the group's cases over n games: every case in every order, the last engine of an order topped up from its start."""
    out = []
    for _ in range(1 if n == 1 else ORDERS):
        order = [group[i] for i in rng.permutation(len(group))]
        for k in range(0, len(order), n):
            part = order[k:k + n]
            out.append(part + [order[j % len(order)] for j in range(n - len(part))])
    return out


def _check_sim(eng, games, s, bad, where):
    for g, c in enumerate(games):
        if s >= c["sims"]:
            continue
        d = eng.export_game(g)
        M = len(c["n2o"])
        if not np.array_equal(d["last_trace"], c["traces"][s]):
            bad.append((where, g, c["tags"], s, "trace", d["last_trace"].tolist(), c["traces"][s].tolist()))
            continue
        for name, w in zip(("visit", "value", "variance"), c["states"][s]):
            if not SE.same_bits(d[name][:M], w):
                bad.append((where, g, c["tags"], s, name))


def _check_pc(eng, games, s, models, cache, served, bad, where):
    """After simulation s: each game's valid cache length equals the model's; `served` = counter 13's growth over the simulations just run,
    equal to the model's sum when every game of the engine is still within its case (None: not checked)."""
    for g, c in enumerate(games):
        if s >= c["sims"]:
            continue
        _, pcl = G.debug_game_state(eng, g)
        want = int(models[id(c)][1][s]) if cache else 0
        if pcl != want:
            bad.append((where, g, c["tags"], s, "pc_len", pcl, want))
    if served is not None:
        got, want = served
        if got != want:
            bad.append((where, s, "levels served from the path cache", got, want))


def _check_end(eng, games, done, bad, where, played=None):
    stats, action = eng.get_stats() if played is None else played
    for g, c in enumerate(games):
        if c["sims"] != done:
            continue
        rng, _ = G.debug_game_state(eng, g)
        if SE.xorshift32(rng) != c["rng_next"]:
            bad.append((where, g, c["tags"], "check_low stream"))
        if not SE.same_bits(stats[g], c["stats"]) or int(action[g]) != c["action"]:
            bad.append((where, g, c["tags"], "action", int(action[g]), c["action"], stats[g][1].tolist(), c["stats"][1].tolist()))


def test_walk_and_action_match_reference(cases, weights, models):
    main = [c for c in cases if "trace_full" not in c["tags"]]
    groups = {}
    for c in main:
        groups.setdefault((c["mode"], c["gamma"], c["low"]), []).append(c)
    rng = np.random.default_rng(5)
    bad, runs, total = [], 0, 0
    for key, group in sorted(groups.items(), key=lambda kv: str(kv[0])):
        for n in GAMES:
            eng = _engine(n, group[0], weights)
            try:
                for games in _layouts(group, n, rng):
                    for cache in ((False, True) if key[0] == "lp" else (False,)):
                        for deep in (0, max(1, n // 4)):
                            for each in (True, False):
                                eng.set_path_cache(cache)
                                eng.set_deep_lane(deep)
                                for g, c in enumerate(games):
                                    G.debug_load_tree(eng, g, c)
                                where = (key, n, cache, deep, "run_sims(1)" if each else "run_sims(k)")
                                stops = sorted({c["sims"] for c in games})

                                def model_served(lo, hi):       # counter 13 over simulations lo..hi-1, while every game is in its case
                                    if hi > stops[0]:
                                        return None
                                    return sum(int(models[id(c)][0][lo:hi].sum()) for c in games) if cache else 0
                                done = 0
                                for stop in stops:
                                    played = None
                                    if each:
                                        for s in range(done, stop):
                                            before = eng.counters()["cached_levels"]
                                            eng.run_sims(1)
                                            got = eng.counters()["cached_levels"] - before
                                            want = model_served(s, s + 1)
                                            _check_sim(eng, games, s, bad, where)
                                            _check_pc(eng, games, s, models, cache, None if want is None else (got, want), bad, where)
                                            total += got
                                    else:
                                        before = eng.counters()["cached_levels"]
                                        if stop == stops[-1]:           # the last stretch as a move: run_sims, get_stats, env_step, update_root
                                            played = eng.play_move(stop - done, auto_reset=False)[::-1]
                                        else:
                                            eng.run_sims(stop - done)
                                        got = eng.counters()["cached_levels"] - before
                                        want = model_served(done, stop)
                                        _check_sim(eng, games, stop - 1, bad, where)
                                        if played is None:              # update_root empties the cache
                                            _check_pc(eng, games, stop - 1, models, cache, None if want is None else (got, want), bad, where)
                                        elif want is not None and got != want:
                                            bad.append((where, stop - 1, "levels served from the path cache", got, want))
                                    done = stop
                                    _check_end(eng, games, done, bad, where, played)
                                runs += 1
            finally:
                eng.close()
    assert not bad, (len(bad), bad[:12])
    assert total > 0
    print("\nselect edges: %d cases, %d engine runs, %d levels served from the path cache in the run_sims(1) runs" % (len(main), runs, total))


def test_trace_full(cases, weights):
    """A walk longer than trace_max stops with ST_TRACE_FULL and backs nothing up; the other games of the engine go on."""
    full = [c for c in cases if "trace_full" in c["tags"]]
    other = [c for c in cases if "chain" in c["tags"] and c["mode"] == "lp" and c["gamma"] == full[0]["gamma"] and c["low"] == full[0]["low"]
             and "trace_full" not in c["tags"]]
    assert full and other and len(full[0]["traces"][0]) == SE.TRACE_MAX + 1
    for cache in (False, True):
        eng = _engine(1 + len(other), full[0], weights)
        try:
            eng.set_path_cache(cache)
            games = full[:1] + other
            for g, c in enumerate(games):
                G.debug_load_tree(eng, g, c)
            eng.run_sims(1)
            st = eng.status()
            assert st[0] == 4 and not st[1:].any(), st   # B200_ERR_TRACE_FULL
            d = eng.export_game(0)
            M = len(full[0]["n2o"])
            for name in ("visit", "value", "variance"):
                assert SE.same_bits(d[name][:M], full[0][name]), name
            for g, c in enumerate(games[1:], 1):
                d = eng.export_game(g)
                assert np.array_equal(d["last_trace"], c["traces"][0]), c["tags"]
                assert all(SE.same_bits(d[k][:len(c["n2o"])], w) for k, w in zip(("visit", "value", "variance"), c["states"][0])), c["tags"]
        finally:
            eng.close()


def test_twin_first_select(gpu_lib, cases):
    """The operator twin (b200_select_trace_obs, select_trace over the reference's layout) on each case's first walk."""
    bad = []
    for i, c in enumerate(cases):
        st = np.array([c["seed"]], np.uint32)
        tr = G.select_trace_obs(c["root"], c["child"], c["visit"].copy(), c["value"].copy(), c["variance"].copy(), c["score"], c["n2o"],
                                c["low"], rng_state=st, max_trace=SE.TRACE_MAX + 1)
        if not np.array_equal(tr, c["traces"][0]):
            bad.append((i, c["tags"], tr.tolist(), c["traces"][0].tolist()))
    assert not bad, bad


def test_twin_drawn_observation_zero(gpu_lib, oracle):
    """A child whose observation id is 0 under `low`: when check_low draws observation 0, core.h:202-205 falls through to policy_clt.
    The twin must walk as the C oracle does, for seeds that draw it and seeds that do not."""
    outcomes = set()
    for c in SE.zero_obs_case():
        want_st, got_st = np.array([c["seed"]], np.uint32), np.array([c["seed"]], np.uint32)
        want = oracle.select_trace_obs(c["root"], c["child"], c["visit"], c["value"], c["variance"], c["score"], c["n2o"], c["low"],
                                       rng_state=want_st)
        got = G.select_trace_obs(c["root"], c["child"], c["visit"].copy(), c["value"].copy(), c["variance"].copy(), c["score"], c["n2o"],
                                 c["low"], rng_state=got_st)
        assert np.array_equal(got, want) and got_st[0] == want_st[0], (c["seed"], got, want)
        outcomes.add(int(want[1]))
    assert len(outcomes) >= 2, outcomes
