"""The distributional search (mode "dist", BASELINE configs[4]) against oracle agents in mode 3, every move: action and stats[3,7], the live
games, the node_stats / node_dist arrays (export_dist) and the search arena (export_game) of the shadowed games, and the counters.  The
oracle runs the reference's loop (agents/DistValueSimOnline.py:36-75 on core_distributional.py's numba cores, oracle/dist_oracle.c); its
evaluator is the engine's synthetic histogram or, for the network runs, the same distributional network on a side engine.  Every test
asserts that the path it covers ran (collections, dropped trees, finished games), so none can pass vacuously."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ARGS = (1, 0, 0)
ARENA_KEYS = ("child", "n2o", "episode", "score", "game")


def search_seed(seed, g):
    s = (seed + 0x9E3779B9 * (g + 1)) & 0xffffffff
    return s or 0x2545F491


def shadow(oracle, n, M, sims, moves, seed, bins=50, vmin=0.0, vmax=5000.0, low=5, eval_kind="synthetic", dist_weights=None, eval_cb=None,
           headroom=0, overflow_reset=False, remove_at=(), timing=False, sample=None):
    """Run the engine (play_move) and shadow the games in `sample` (default: all) with oracle agents.  Returns (counters of the engine,
    summed oracle counters of the sample, finished games in the sample)."""
    from tetris_mcts_b200 import pyTetris as PT
    from tetris_mcts_b200.engine import BatchedEngine
    recs = PT.new_games(n, ARGS, np.arange(seed, seed + n, dtype=np.uint32))
    eng = BatchedEngine(n, max_nodes=M, mode="dist", eval_kind=eval_kind, dist_weights=dist_weights, seed=seed, low=low,
                        overflow_reset=overflow_reset, dist_bins=bins, dist_vmin=vmin, dist_vmax=vmax)
    eng.set_games(recs)
    eng.set_gc_headroom(headroom)
    eng.set_timing(timing)
    sample = list(range(n)) if sample is None else sample
    agents = {g: oracle.Agent(max_nodes=M, mode=3, low=low, eval_mode=2 if eval_cb else 0, eval_cb=eval_cb, search_seed=search_seed(seed, g),
                              dist_bins=bins, dist_vmin=vmin, dist_vmax=vmax, overflow_reset=int(overflow_reset)) for g in sample}
    games = {g: oracle.Game(record=recs[g]) for g in sample}
    for g in sample:
        agents[g].update_root(games[g].record())
    finished = 0
    for mv in range(moves):
        actions, stats = eng.play_move(sims, auto_reset=True)
        live = eng.get_games()
        for g in sample:
            ag = agents[g]
            ag.mcts(sims)
            a, st = ag.get_action()
            assert a == actions[g] and np.array_equal(st, stats[g]), "move %d game %d\n%s\n%s" % (mv, g, st, stats[g])
            games[g].play(a)
            ag.update_root(games[g].record())
            if games[g].end:
                finished += 1
                games[g].reset()
                ag.update_root(games[g].record())
            if headroom and ag.n_free < headroom:
                ag.remove_nodes()
            assert np.array_equal(live[g], games[g].record()), "live game %d differs after move %d" % (g, mv)
        if mv in remove_at:
            eng.remove_nodes()
            for g in sample:
                agents[g].remove_nodes()
    for g in sample:
        ns, nd = eng.export_dist(g)
        wns, wnd = agents[g].export_dist()
        assert np.array_equal(ns, wns), "node_stats of game %d" % g
        d = np.argwhere(nd.view(np.uint32) != wnd.view(np.uint32))
        assert not len(d), "node_dist of game %d differs first at node %d bin %d: %r vs %r" % (g, d[0][0], d[0][1], nd[tuple(d[0])], wnd[tuple(d[0])])
        ex, want = eng.export_game(g), agents[g].export()
        assert ex["root"] == agents[g].root, g
        for k in ARENA_KEYS:
            assert np.array_equal(ex[k], want[k]), (g, k)
    c = eng.counters()
    oc = {k: sum(agents[g].counter(i) for g in sample) for k, i in (("sims", 0), ("expansions", 1), ("gcs", 3), ("tree_resets", 7))}
    assert c["sims"] == n * sims * moves and (eng.status() == 0).all()
    if len(sample) == n:
        for k in oc:
            assert c[k] == oc[k], (k, c[k], oc[k])
        assert c["games_finished"] == finished, (c["games_finished"], finished)
    eng.close()
    return c, oc, finished


@pytest.mark.parametrize("bins,vmin,vmax", [(2, 0.0, 5000.0), (33, 0.0, 5000.0), (64, 0.0, 5000.0), (56, 0.0, 5000.0), (35, 0.0, 45.0),
                                            (30, 0.0, 1000.0), (50, -300.0, 700.0)])
@pytest.mark.parametrize("low", [0, 1, 5])
def test_dist_search_atoms_and_ranges(gpu_lib, oracle, bins, vmin, vmax, low):
    """Synthetic histograms, every game shadowed, played until games end (game-over leaves back up the one-hot at bin 0).  (56, 0, 5000),
    (35, 0, 45) and (30, 0, 1000) are configurations where int(b + x / delta) truncates one bin further than b + int(x / delta) for
    integer score differences x; (35, 0, 45) is small enough that most traces clamp into the top bin."""
    c, oc, finished = shadow(oracle, n=12, M=6000, sims=40, moves=80, seed=100 + bins, bins=bins, vmin=vmin, vmax=vmax, low=low)
    assert finished > 0, "no game ended: no game-over leaf was backed up"


@pytest.mark.parametrize("timing", [False, True])
def test_dist_search_collections(gpu_lib, oracle, timing):
    """Arenas small enough that expansions suspend for in-expansion collections, the head-room policy, one explicit remove_nodes() and
    overflow_reset tree drops; the CUDA-graph path of play_move and its direct launches (set_timing) alike."""
    c, oc, _ = shadow(oracle, n=32, M=700, sims=40, moves=40, seed=57, bins=33, vmin=0.0, vmax=1000.0, low=1, headroom=150,
                      overflow_reset=True, remove_at=(7,), timing=timing)
    assert c["gcs"] > 32 and c["tree_resets"] > 0, c
    c2, _, _ = shadow(oracle, n=16, M=900, sims=50, moves=30, seed=58, bins=56, low=5)                # lazy collections inside expansions only
    assert c2["gcs"] > 0, c2


@pytest.mark.parametrize("kind", ["net", "net_tc"])
def test_dist_network_batch_position_invariant(gpu_lib, oracle, kind):
    """What the network shadow relies on: a board's distnet output is the same bits alone and inside batches of 2 to 20000 boards, at
    several positions."""
    from arena_gen import boards
    from tetris_mcts_b200.engine import BatchedEngine
    from tetris_mcts_b200.agents.DistValueSimOnline import init_dist_weights
    side = BatchedEngine(1, max_nodes=64, mode="dist", eval_kind=kind, dist_weights=init_dist_weights(0, 50))
    probe = boards(5, 99)
    alone = np.stack([side.distnet(probe[i:i + 1])[0] for i in range(len(probe))])
    for n in (2, 3, 127, 129, 1000, 20000):
        batch = boards(n, n)
        for pos in sorted({0, n // 2, n - 1}):
            b = batch.copy()
            b[pos] = probe[pos % len(probe)]
            out = side.distnet(b)
            assert np.array_equal(out[pos], alone[pos % len(probe)]), (kind, n, pos)
    side.close()


@pytest.mark.parametrize("kind", ["net", "net_tc"])
def test_dist_search_with_network(gpu_lib, oracle, kind):
    """The network evaluator: the oracle agents get each leaf's distnet output from a side engine holding the same weights."""
    from tetris_mcts_b200.engine import BatchedEngine
    from tetris_mcts_b200.agents.DistValueSimOnline import init_dist_weights
    w = init_dist_weights(0, 50)
    side = BatchedEngine(1, max_nodes=64, mode="dist", eval_kind=kind, dist_weights=w)
    c, oc, _ = shadow(oracle, n=24, M=2048, sims=60, moves=12, seed=5, eval_kind=kind, dist_weights=w, eval_cb=side.distnet,
                      overflow_reset=True, headroom=2048 * 5 // 32)
    assert c["gcs"] > 0, c
    side.close()


def test_dist_bench_config_sampled_games_exact(gpu_lib, oracle):
    """configs[4] as bench.py runs it: 2048 games, 1500 simulations per move, 32768 slots, net_tc with init_dist_weights(0, 50), head-room
    32768 * 5 / 32, overflow_reset, play_move.  Games 0, n - 1 and 14 seeded others are shadowed until sampled games have collected."""
    from tetris_mcts_b200.engine import BatchedEngine
    from tetris_mcts_b200.agents.DistValueSimOnline import init_dist_weights
    n, M = 2048, 32768
    w = init_dist_weights(0, 50)
    side = BatchedEngine(1, max_nodes=64, mode="dist", eval_kind="net_tc", dist_weights=w)
    sample = sorted(set([0, n - 1] + list(np.random.default_rng(7).choice(n, 14, replace=False))))
    c, oc, _ = shadow(oracle, n=n, M=M, sims=1500, moves=5, seed=123, eval_kind="net_tc", dist_weights=w, eval_cb=side.distnet,
                      overflow_reset=True, headroom=M * 5 // 32, sample=sample)
    assert c["gcs"] > 0 and oc["gcs"] > 0, (c, oc)
    side.close()
