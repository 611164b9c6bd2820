"""eval_kind net_fp16: the value network on the tensor cores with one fp16 term per operand (valuenet_tc.cuh, NT = 1).

The network is held to the error contract tests/f16_ref.py derives (act3 per element within 2^-10 of the board's largest |term| sum
plus the split's floor; v and var within 2^-11 relative plus the `saturated` / `subnormal` allowances) against the float64 reference of
tests/f64_ref.py.  The search on its outputs is held to the C oracle exactly, as for net_tc: the LP search is deterministic given the
evaluator and the piece sequence, so oracle agents fed a net_fp16 side engine's outputs must make the same decisions, statistics and arenas."""
import io
import re

import numpy as np
import pytest

import f16_ref as H
import f64_ref as R
from arena_gen import boards as random_boards

pytestmark = pytest.mark.gpu
ARGS = (1, 0, 0)
ENV_ARGS = ((20, 10), 1, 0, 0)


def search_seed(seed, g):
    s = (seed + 0x9E3779B9 * (g + 1)) & 0xffffffff
    return s or 0x2545F491


def engine(kind, w, n=1, **kw):
    from tetris_mcts_b200.engine import BatchedEngine
    return BatchedEngine(n, max_nodes=64, eval_kind=kind, weights=w, **kw)


def act3(eng, states):
    from tetris_mcts_b200 import _lib as L
    s = np.ascontiguousarray(np.asarray(states, np.int8).reshape(-1, 200))
    out = np.zeros((len(s), 1792), np.float32)
    L.check(L.lib().b200_debug_act3(eng.h, L.ptr(s), len(s), L.ptr(out)))
    return out


def check_act3(eng, w, states, what):
    got = act3(eng, states)
    _, _, ref = R.valuenet(w, states)
    ratio = np.abs(got - ref) / H.act3_bound(w, states)
    assert np.isfinite(got).all(), what
    if ratio.max() > 1:
        b, e = np.unravel_index(int(np.argmax(ratio)), ratio.shape)
        pytest.fail("%s: act3 board %d channel %d pixel (%d, %d): got %.9g want %.9g (error / bound %.3g)" %
                    (what, b, e // 56, (e % 56) // 4, e % 4, got[b, e], ref[b, e], ratio.max()))
    return float(ratio.max())


def check_outputs(v, var, w, states, what, allowance=None):
    rv, rvar, _ = R.valuenet(w, states)
    sv, svar = H.out_sensitivity(w, states, allowance)
    assert np.isfinite(v).all() and np.isfinite(var).all(), what
    ev, evar = H.out_excess(v, rv, sv), H.out_excess(var, rvar, svar)
    assert ev <= 1 and evar <= 1, "%s: error / bound v %.3g var %.3g" % (what, ev, evar)
    return max(ev, evar)


@pytest.fixture(scope="module")
def fam(oracle):
    return R.board_families(oracle)


def test_every_weight_and_board_family_with_hot_swaps(gpu_lib, fam):
    """Every weight family x every board family on ONE engine, the weights swapped in between as the online loop swaps them."""
    wf = R.weight_families(0)
    eng = engine("net_fp16", wf["init"])
    allb = np.concatenate(list(fam.values()))
    for wname, w in list(wf.items()) + [("init again", wf["init"])]:
        eng.load_weights(w)
        worst = 0.0
        for bname, b in fam.items():
            v, var = eng.valuenet(b)
            worst = max(worst, check_outputs(v, var, w, b, "%s / %s" % (wname, bname), R.ALLOWANCE.get(wname.split()[0])))
        r3 = check_act3(eng, w, allb, wname)
        print("\n[net_fp16] %-14s act3 error/bound %.3f  outputs error/bound %.3f" % (wname, r3, worst))
    eng.close()


def test_batch_sizes_and_passes(gpu_lib, oracle):
    """Batches of 1, 7, 300 (not a multiple of 128) and more than one pass of k_tc_fc over all SMs; every board's outputs do not depend
    on the batch it is in, and a small batch after a large one (stale act3 tiles past it) is unaffected."""
    import torch
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    Fp = n_sm * 128
    w = R.weight_families(2)["trained_bounds"]
    big = Fp + n_sm * 16 + 45
    pool = np.concatenate(list(R.board_families(oracle, 1).values()) + [random_boards(big, 23)])[:big]
    eng = engine("net_fp16", w)
    vb, varb = eng.valuenet(pool)
    rng = np.random.default_rng(1)
    sub = np.union1d(np.r_[0:4, Fp - 2:Fp + 2, big - 3:big], rng.choice(big, 400, replace=False))
    check_outputs(vb[sub], varb[sub], w, pool[sub], "batch %d" % big)
    for n in (1, 7, 300):
        idx = rng.permutation(big)[:n]
        s = pool[idx]
        v, var = eng.valuenet(s)
        check_outputs(v, var, w, s, "batch %d" % n)
        check_act3(eng, w, s, "batch %d" % n)
        assert np.array_equal(v, vb[idx]) and np.array_equal(var, varb[idx]), n
    eng.close()


def test_agrees_with_net_tc_within_the_fp16_bound(gpu_lib, oracle):
    """On random and real positions, net_fp16 against net_tc (itself within 1e-5 of float64)."""
    from tetris_mcts_b200.model.model_vv import init_weights
    s = np.concatenate([random_boards(2000, 5), R.real_positions(2000, 11, oracle)])
    worst = {}
    for name, w in (("init", init_weights(0)), ("trained_bounds", R.weight_families(4)["trained_bounds"])):
        e16, etc = engine("net_fp16", w), engine("net_tc", w)
        v16, var16 = e16.valuenet(s)
        vtc, vartc = etc.valuenet(s)
        for a, b in ((v16, vtc), (var16, vartc)):
            assert np.all(np.abs(a.astype(np.float64) - b) <= (H.OUT_RTOL + 2e-5) * np.abs(b)), name
        worst[name] = max(float(np.max(np.abs(v16 - vtc.astype(np.float64)) / np.abs(vtc))),
                          float(np.max(np.abs(var16 - vartc.astype(np.float64)) / np.abs(vartc))))
        assert worst[name] > 0                                            # one product per product is not the split
        e16.close(); etc.close()
    print("\nnet_fp16 vs net_tc, largest relative difference of v / var on 4000 positions: %s" %
          ", ".join("%s %.3g" % kv for kv in worst.items()))


def test_load_refuses_weights_outside_fp16_range(gpu_lib):
    from tetris_mcts_b200 import _lib as L
    w = R.init_weights(0)
    states = random_boards(16, 1)
    eng = engine("net_fp16", w)
    fits = w.copy()
    fits[320 + 5] = 1023.0
    eng.load_weights(fits)
    loaded = eng.valuenet(states)
    for off, x in ((7, -1100.0), (320 + 5, 1024.0), (9568 + 100, -1100.0), (18816 + 123456, 1100.0), (18816 + 7, np.nan)):
        bad = w.copy()
        bad[off] = x
        with pytest.raises(L.B200Error) as ei:
            eng.load_weights(bad)
        assert ei.value.code == 1 and "65504" in str(ei.value) and "net_fp16" in str(ei.value)
        assert all(np.array_equal(a, b) for a, b in zip(loaded, eng.valuenet(states))), off
    eng.close()


def test_distributional_mode_is_refused(gpu_lib):
    from tetris_mcts_b200 import _lib as L
    from tetris_mcts_b200.engine import BatchedEngine
    with pytest.raises(L.B200Error) as ei:
        BatchedEngine(4, max_nodes=256, mode="dist", eval_kind="net_fp16")
    assert ei.value.code == 1 and "net_fp16" in str(ei.value)
    eng = engine("net_fp16", R.init_weights(0))                            # nor is there a distributional network to load
    with pytest.raises(L.B200Error) as ei:
        eng.load_dist_weights(R.dist_init_weights(0, 50), 50)
    assert ei.value.code == 1
    eng.close()


@pytest.mark.parametrize("case", ["plain", "collections_and_drops"])
def test_search_is_exact_given_the_same_evaluator(gpu_lib, oracle, case):
    """Oracle agents fed a one-game net_fp16 side engine's outputs shadow the engine move for move (tests/test_gpu_engine.py run_pair):
    actions, stats[3,7], live games and arenas; the second case has arenas small enough for collections and dropped trees."""
    from test_gpu_engine import run_pair
    from tetris_mcts_b200.engine import BatchedEngine
    w = oracle.seeded_weights(0)
    side = BatchedEngine(1, max_nodes=64, eval_kind="net_fp16", weights=w)

    def cb(states):
        return side.valuenet(states)

    if case == "plain":
        run_pair(oracle, "lp", n=3, M=2048, sims=25, moves=4, eval_kind="net_fp16", weights=w, eval_cb=cb)
    else:
        c = run_pair(oracle, "lp", n=8, M=512, sims=40, moves=20, eval_kind="net_fp16", weights=w, eval_cb=cb,
                     engine_kw=dict(overflow_reset=True), agent_kw=dict(overflow_reset=1))
        assert c["gcs"] > 0 and c["tree_resets"] > 0, c
    side.close()


@pytest.mark.parametrize("deep_lane", [0, 164])
def test_bench_config_sampled_games_exact(gpu_lib, oracle, deep_lane):
    """The benchmarked configuration (16384 games x 500 simulations, max_nodes 8192, head-room 1280, overflow_reset, one CUDA graph per
    simulation step, b200_play_move) on net_fp16, with the deep lane off and on: sampled games shadowed by oracle agents exactly, as
    tests/test_gpu_bench_config.py does for net_tc."""
    from tetris_mcts_b200 import pyTetris as PT
    from tetris_mcts_b200.engine import BatchedEngine
    from tetris_mcts_b200.model.model_vv import init_weights
    n, M, sims, moves, headroom, seed = 16384, 8192, 500, 9, 8192 * 5 // 32, 123
    recs = PT.new_games(n, ARGS, np.arange(seed, seed + n, dtype=np.uint32))
    w = init_weights(0)
    eng = BatchedEngine(n, max_nodes=M, mode="lp", eval_kind="net_fp16", weights=w, seed=seed, overflow_reset=True)
    eng.set_games(recs)
    eng.set_gc_headroom(headroom)
    eng.set_deep_lane(deep_lane)
    side = BatchedEngine(1, max_nodes=64, eval_kind="net_fp16", weights=w)

    def cb(states):
        return side.valuenet(states)

    sample = sorted(set([0, n - 1] + list(np.random.default_rng(7).choice(n, 14, replace=False))))
    agents = {g: oracle.Agent(max_nodes=M, mode=0, gamma=0.999, low=1, eval_mode=2, eval_cb=cb, search_seed=search_seed(seed, g),
                              overflow_reset=1) for g in sample}
    games = {g: oracle.Game(record=recs[g]) for g in sample}
    for g in sample:
        agents[g].update_root(games[g].record())
    for mv in range(moves):
        actions, stats = eng.play_move(sims, auto_reset=True)
        live = eng.get_games()
        for g in sample:
            agents[g].mcts(sims)
            a, st = agents[g].get_action()
            assert a == actions[g] and np.array_equal(st, stats[g]), "move %d game %d\n%s\n%s" % (mv, g, st, stats[g])
            games[g].play(a)
            agents[g].update_root(games[g].record())
            if games[g].end:
                games[g].reset()
                agents[g].update_root(games[g].record())
            if agents[g].n_free < headroom:
                agents[g].remove_nodes()
            assert np.array_equal(live[g], games[g].record()), "live game %d differs after move %d" % (g, mv)
    c = eng.counters()
    assert c["sims"] == n * sims * moves and (eng.status() == 0).all()
    assert c["gcs"] > 0
    for g in sample:
        ex, want = eng.export_game(g), agents[g].export()
        assert ex["root"] == agents[g].root, g
        for k in ("child", "n2o", "episode", "score", "visit", "value", "variance", "obs_end", "obs_key", "game"):
            assert np.array_equal(ex[k], want[k]), (g, k)
    print("net_fp16 bench-config parity (deep lane %d): %d sampled games x %d moves exact; collections %d, trees dropped %d"
          % (deep_lane, len(sample), moves, c["gcs"], c["tree_resets"]))
    side.close()
    eng.close()


def test_two_engines_with_the_same_seeds_are_identical(gpu_lib):
    from tetris_mcts_b200 import pyTetris as PT
    from tetris_mcts_b200.engine import BatchedEngine
    from tetris_mcts_b200.model.model_vv import init_weights
    n, M, sims, seed = 1024, 2048, 120, 5
    recs = PT.new_games(n, ARGS, np.arange(seed, seed + n, dtype=np.uint32))
    engs = []
    for _ in range(2):
        e = BatchedEngine(n, max_nodes=M, mode="lp", eval_kind="net_fp16", weights=init_weights(3), seed=seed, overflow_reset=True)
        e.set_games(recs)
        e.set_gc_headroom(M * 5 // 32)
        e.set_deep_lane(32)
        engs.append(e)
    for mv in range(6):
        (a0, s0), (a1, s1) = [e.play_move(sims, auto_reset=True) for e in engs]
        assert a0.tobytes() == a1.tobytes() and s0.tobytes() == s1.tobytes(), mv
        assert engs[0].get_games().tobytes() == engs[1].get_games().tobytes(), mv
    assert engs[0].counters() == engs[1].counters()
    for e in engs:
        e.close()


def test_model_and_agents_take_net_fp16(gpu_lib):
    from tetris_mcts_b200.agents.ValueSimLP import ValueSimLP
    from tetris_mcts_b200.model.model_vv import Model_VV
    from tetris_mcts_b200.pyTetris import Tetris
    from tetris_mcts_b200 import _lib as L
    s = random_boards(64, 9)
    m = Model_VV(seed=4, eval_kind="net_fp16")
    assert m._eng.eval_kind == L.EVAL_NET_FP16
    eng = engine("net_fp16", m.weights)
    v, var = m.inference(s[:, None])
    ev, evar = eng.valuenet(s)
    assert np.array_equal(v[:, 0], ev) and np.array_equal(var[:, 0], evar)
    eng.close(); m.close()
    game = Tetris(*ENV_ARGS)
    agent = ValueSimLP(sims=60, env=Tetris, env_args=ENV_ARGS, benchmark=False, online=False, min_visit=40, eval_kind="net_fp16")
    assert agent._eng.eval_kind == L.EVAL_NET_FP16
    agent.update_root(game)
    for _ in range(4):
        a = agent.play()
        assert 0 <= a < 7
        game.play(a)
        agent.update_root(game)
    assert agent.counters()["sims"] == 240
    agent.close()


def test_play_batched_with_net_fp16(gpu_lib, tmp_path, monkeypatch):
    from tetris_mcts_b200 import play_batched as PB
    monkeypatch.chdir(tmp_path)
    out = io.StringIO()
    ngames, moves, _ = PB.run(PB.parse_args(["--agent_type", "ValueSimLP", "--mcts_sims", "20", "--ngames", "4", "--n_parallel", "64",
                                             "--max_nodes", "1024", "--endless", "--max_moves", "400", "--eval_kind", "net_fp16"]), out=out)
    eps = re.findall(r"Episode:\s+\d+ Score:\s+\d+ Lines Cleared:\s+\d+", out.getvalue())
    assert ngames == 4 and len(eps) == 4, out.getvalue()[-2000:]


def test_play_batched_online_with_net_fp16(gpu_lib, tmp_path, monkeypatch):
    """--online --eval_kind net_fp16: the trainer is unchanged (fp32 / fp64), the search engine takes the trained weights and goes on
    searching with them in net_fp16."""
    from tetris_mcts_b200 import play_batched as PB
    from tetris_mcts_b200 import pyTetris as PT
    from tetris_mcts_b200.engine import BatchedEngine
    from tetris_mcts_b200.model.model_vv import Model_VV
    from tetris_mcts_b200 import _lib as L
    buf = io.StringIO()
    monkeypatch.setattr(PB, "perr", dict(file=buf, flush=True))
    monkeypatch.chdir(tmp_path)
    states = PT.states_of(PT.new_games(16, (1, 0, 0), np.arange(40, 56, dtype=np.uint32)))
    seen = {}

    class Recording(BatchedEngine):
        def close(self):
            if getattr(self, "h", None) and self.n_games == 64:
                seen["kind"] = self.eval_kind
                seen["out"] = self.valuenet(states)
                seen["sims"] = self.counters()["sims"]
            super().close()
    monkeypatch.setattr(PB, "BatchedEngine", Recording)
    timing = {}
    PB.run(PB.parse_args(["--agent_type", "ValueSimLP", "--mcts_sims", "64", "--ngames", "64", "--n_parallel", "64", "--max_nodes", "1024",
                          "--endless", "--online", "--max_moves", "160", "--train_max_iters", "200", "--train_batch_size", "256",
                          "--memory_size", "2000", "--memory_growth_rate", "150", "--eval_kind", "net_fp16"]), out=io.StringIO(), timing=timing)
    assert timing["trainings"] >= 1, buf.getvalue()[-2000:]
    assert seen["kind"] == L.EVAL_NET_FP16 and seen["sims"] == 64 * 64 * timing["moves"]
    m = Model_VV(seed=9, eval_kind="net_fp16")
    m.load("pytorch_model/model_checkpoint")
    v, var = m.inference(states[:, None])
    assert np.array_equal(seen["out"][0], v[:, 0]) and np.array_equal(seen["out"][1], var[:, 0])
    init = Model_VV(seed=0, eval_kind="net_fp16")                          # the run started from init_weights(0): the weights moved
    v0, _ = init.inference(states[:, None])
    assert not np.array_equal(v0[:, 0], v[:, 0])
    m.close(); init.close()
