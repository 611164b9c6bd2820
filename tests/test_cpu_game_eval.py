"""The caller's leaf-game evaluator (eval_kind "external_game") where no GPU is needed: the C oracle with an injected evaluator against the
reference's own agent.cpp with evaluator type 1 (agent_type1_golden.npz), the host helpers pyTetris.per_game and record_fields, and
play_batched's --game_evaluator / VanillaC checks."""
import os

import numpy as np
import pytest

from game_eval_twins import FLOAT_CHAIN_DIVERGENCE, GameEvalAgent, evaluate, evaluate_batch, golden_span

GOLD = os.path.join(os.path.dirname(__file__), "golden", "agent_type1_golden.npz")


def stream_of_game0(engine_seed):
    s = (int(engine_seed) + 0x9E3779B9) & 0xffffffff
    return s or 0x2545F491


def replay_oracle(oracle, z, case):
    """the C oracle in MODE_VANILLA with the golden's evaluator injected, driven as the golden's generator drove agent.cpp"""
    p = "c%d_" % case
    app, scoring, randomizer = (int(x) for x in z[p + "env"])
    special = bool(z[p + "special"])
    seen = []

    def f(rec):
        seen.append(rec)
        return evaluate(rec, special)
    ag = GameEvalAgent(oracle.Agent(max_nodes=int(z["max_nodes"]), mode=2, gamma=float(z[p + "gamma"]), low=1, eval_mode=0,
                                    search_seed=stream_of_game0(z[p + "engine_seed"]), app=app, scoring=scoring, randomizer=randomizer), f)
    g = oracle.Game(record=z[p + "start"])
    ag.update_root(g.record())
    acts, recs, off = [], [], [0]
    for _ in range(len(z[p + "actions"])):
        ag.mcts(int(z[p + "sims"]))
        a, _st = ag.get_action()
        acts.append(a)
        off.append(len(seen))
        g.play(a)
        ag.update_root(g.record())
        if g.end:
            g.reset()
            ag.update_root(g.record())
        recs.append(g.record())
    return ag, np.array(acts), np.stack(recs), np.array(off), np.stack(seen)


def test_oracle_game_eval_reproduces_reference(oracle):
    """Every action, every game record after a move and every record handed to the evaluator (so every simulation's walk) equal the
    reference's own MCTSAgent(..., f, 1, False) on four cases: VanillaC's settings over game overs, gamma 1 with integer outputs, other
    env_args, and NaN / +-inf / negative outputs.  Two agree to the end; in the other two (gamma 0.99) the reference's float value chain
    (agent.cpp:496-513) makes its walk differ at a pinned evaluation (game_eval_twins.FLOAT_CHAIN_DIVERGENCE), and everything before it agrees."""
    z = np.load(GOLD)
    for case in range(int(z["n_cases"])):
        p = "c%d_" % case
        ag, acts, recs, off, seen = replay_oracle(oracle, z, case)
        moves, evals = golden_span(z, case)
        assert moves >= 10 and evals >= 250, case
        assert np.array_equal(acts[:moves], z[p + "actions"][:moves]), case
        assert np.array_equal(recs[:moves], z[p + "records"][:moves]), case
        assert np.array_equal(off[:moves + 1], z[p + "eval_off"][:moves + 1]), case
        assert np.array_equal(seen[:evals], z[p + "eval_recs"][:evals]), case
        if FLOAT_CHAIN_DIVERGENCE[case] is not None:                       # the divergence is where it is pinned, not earlier or later
            assert not np.array_equal(seen[evals], z[p + "eval_recs"][evals]), case
        else:
            assert len(seen) == evals and np.array_equal(acts, z[p + "actions"]), case
        assert ag.counter(5) == 0 and ag.counter(2) == len(seen)           # no rollout; one evaluation per expanded leaf
    assert int(z["c0_resets"]) > 0 and int(z["c1_resets"]) > 0 and float(z["c1_gamma"]) == 1.0 and tuple(z["c2_env"]) == (2, 1, 1)
    v, var = evaluate_batch(z["c3_eval_recs"], special=True)
    assert np.isnan(v).any() and np.isposinf(v).any() and np.isneginf(v).any() and (v < 0).any() and np.isnan(var).any() and (var < 0).any()


def test_record_fields_on_host_records(oracle):
    from tetris_mcts_b200.pyTetris import record_fields
    z = np.load(GOLD)
    g = oracle.Game(app=1, scoring=0, randomizer=0, seed=4)
    rng = np.random.default_rng(0)
    while not g.end:                                        # a finished game, with line clears and a combo somewhere on the way
        g.play(int(rng.integers(0, 7)))
    words = rng.integers(0, 2**32, (100, 20), dtype=np.uint64).astype(np.uint32)     # every bit pattern of the decoded words
    recs = np.concatenate([z["c0_records"], z["c2_records"], z["c3_eval_recs"][:200], g.record()[None], words])
    ref = dict(end=[(int(r[10]) >> 21) & 1 for r in recs], score=[int(np.int32(r[13])) for r in recs],
               line_clears=[int(np.int32(r[14])) for r in recs], combo=[int(r[11]) >> 8 for r in recs])
    assert ref["end"][-101] == 1 and any(ref["score"]) and min(ref["score"]) < 0 < max(ref["combo"])
    fields = record_fields(recs)
    for k, want in ref.items():
        assert fields[k].dtype == np.int32 and fields[k].tolist() == want, k
    import torch
    t = record_fields(torch.from_numpy(recs.view(np.int32)))
    for k in ref:
        assert t[k].tolist() == ref[k], k


def test_per_game_wraps_a_reference_style_function():
    """pyTetris.per_game(f) calls f once per record, on a Tetris of a COPY of the record, in row order, and returns float32 (v, var)"""
    from tetris_mcts_b200 import pyTetris as PT
    z = np.load(GOLD)
    recs = z["c3_eval_recs"][:50].copy()
    before = recs.copy()
    got = []

    def f(game):
        got.append(game.get_record())
        game.set_record(np.zeros(20, np.uint32))         # f may play or change its game: the caller's record is not touched
        return evaluate(got[-1], True)
    v, var = PT.per_game(f)(recs)
    assert np.array_equal(recs, before) and np.array_equal(np.stack(got), before)
    wv, wvar = evaluate_batch(before, True)
    assert v.dtype == var.dtype == np.float32
    assert np.array_equal(v, wv, equal_nan=True) and np.array_equal(var, wvar, equal_nan=True)


@pytest.mark.parametrize("argv, msg", [
    (["--agent_type", "ValueSimLP", "--game_evaluator", "m:f"], "--game_evaluator needs --agent_type Vanilla or VanillaC"),
    (["--agent_type", "ValueSim", "--game_evaluator", "m:f"], "--game_evaluator needs --agent_type Vanilla or VanillaC"),
    (["--agent_type", "VanillaC", "--game_evaluator", "m:f", "--evaluator", "m:g"], "--game_evaluator cannot be combined with --evaluator"),
    (["--agent_type", "Vanilla", "--game_evaluator", "m:f", "--evaluator", "m:g"], "--evaluator cannot be combined with --agent_type Vanilla"),
    (["--agent_type", "Vanilla", "--game_evaluator", "m:f", "--online"], "--game_evaluator cannot be combined with --online"),
    (["--agent_type", "VanillaC", "--game_evaluator", "mf"], "--game_evaluator takes MODULE:FACTORY"),
    (["--agent_type", "Vanilla", "--game_evaluator", "m:f", "--checkpoint_dir", "ck"], "--checkpoint_dir cannot be combined with --game_evaluator"),
    (["--agent_type", "VanillaC", "--checkpoint_dir", "ck"], "--checkpoint_dir cannot be combined with --game_evaluator or --agent_type VanillaC"),
    (["--agent_type", "VanillaC", "--evaluator", "m:g"], "--evaluator cannot be combined with --agent_type VanillaC"),
    (["--agent_type", "VanillaC", "--online", "--trainer", "m:t"], "--trainer cannot be combined with --agent_type VanillaC"),
])
def test_play_batched_refusals(argv, msg, capsys):
    from tetris_mcts_b200.play_batched import parse_args
    with pytest.raises(SystemExit):
        parse_args(argv)
    assert msg in capsys.readouterr().err


def test_play_batched_accepts_game_evaluator_and_vanillac():
    from tetris_mcts_b200.play_batched import MODES, parse_args
    a = parse_args(["--agent_type", "Vanilla", "--game_evaluator", "mymod:make"])
    assert a.game_evaluator == "mymod:make" and a.agent_type == "Vanilla"
    a = parse_args(["--agent_type", "VanillaC", "--game_evaluator", "mymod:make"])
    assert a.game_evaluator == "mymod:make"
    assert parse_args(["--agent_type", "VanillaC"]).game_evaluator is None
    assert MODES["VanillaC"] == ("vanilla", 0.99, 1) and MODES["Vanilla"] == ("vanilla", 0.99, 5)


def test_vanillac_signature_is_the_references():
    import inspect
    from tetris_mcts_b200.agents.VanillaC import VanillaC
    params = list(inspect.signature(VanillaC.__init__).parameters.values())
    names = [q.name for q in params]
    assert names[1:7] == ["sims", "max_nodes", "projection", "gamma", "benchmark", "LP"]
    defaults = {q.name: q.default for q in params}
    assert (defaults["sims"], defaults["max_nodes"], defaults["projection"], defaults["gamma"], defaults["benchmark"], defaults["LP"]) == \
        (100, 500000, True, 0.99, False, False)
    from tetris_mcts_b200.agents.Vanilla import Vanilla
    with pytest.raises(ValueError):
        Vanilla(evaluator=lambda b: b)
    with pytest.raises(ValueError):
        VanillaC(evaluator=lambda b: b)


def test_product_never_imports_the_oracle_or_the_test_evaluator():
    root = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tetris_mcts_b200")
    for d, _, files in os.walk(root):
        for fn in files:
            if fn.endswith((".py", ".cu", ".cuh")):
                txt = open(os.path.join(d, fn), errors="ignore").read()
                for bad in ("oracle_py", "liboracle", "import oracle", "game_eval_twins"):
                    assert bad not in txt, (fn, bad)
