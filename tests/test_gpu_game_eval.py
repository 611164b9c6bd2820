"""The caller's leaf-game evaluator (eval_kind "external_game", B200_BOARD_RECORD) and the device game calls (b200_tetris_*_dev) on the GPU.

- The device game calls against the C oracle env and the host entry points, bit for bit, on more than 10^6 (record, action) pairs, and
  playout_dev against a CPU restatement.
- The engine against the reference's own agent.cpp (agent_type1_golden.npz) and against oracle agents fed the same evaluator, simulation by
  simulation: the records handed out, and at the end of every move the actions, statistics and live games; at the end the arenas, the
  check_low streams and the counters.  Collections, dropped trees, game overs, several games per engine and NaN / inf outputs occur.
- The step API's refusals, a save / load round trip, and repeatability."""
import os

import numpy as np
import pytest

from game_eval_twins import GameEvalAgent, evaluate, evaluate_batch, evaluate_torch, golden_span, playout_cpu

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "agent_type1_golden.npz")
ARENA_KEYS = ("child", "n2o", "episode", "score", "game", "visit", "value", "variance", "obs_end", "obs_key")
ENVS = [(1, 0, 0), (1, 1, 0), (2, 0, 1), (3, 1, 1), (1, 0, 1), (2, 1, 0), (4, 0, 0), (1, 1, 1)]


def search_seed(seed, g):
    s = (seed + 0x9E3779B9 * (g + 1)) & 0xffffffff
    return s or 0x2545F491


def lib_error():
    from tetris_mcts_b200._lib import B200Error
    return B200Error


# ---------------------------------------------------------------------------------------------------- device game calls
def test_step_and_state_dev_against_oracle(gpu_lib, oracle):
    """2^20 + (record, action) pairs over eight env settings, actions 0..7, a quarter of the games over before the first step: every step of
    step_games_dev equals the oracle's to_play_records; states_of_dev (int8 and float32) equals the host b200_tetris_state on every record
    and the oracle's getState on a sample."""
    import torch
    from tetris_mcts_b200 import pyTetris as PT
    n, steps = 8192, 130
    recs = np.concatenate([PT.new_games(n // len(ENVS), e, np.arange(1 + i * n, 1 + i * n + n // len(ENVS), dtype=np.uint32))
                           for i, e in enumerate(ENVS)])
    dev = torch.from_numpy(recs.view(np.int32)).cuda()
    PT.playout_dev(dev[: n // 4], torch.arange(1, n // 4 + 1, dtype=torch.int32, device="cuda"), 7)      # game over before any step
    rng = np.random.default_rng(5)
    pairs, ended = 0, 0
    for s in range(steps):
        host = dev.cpu().numpy().view(np.uint32).copy()
        ended += int(((host[:, 10] >> 21) & 1).sum())
        if s % 13 == 0:
            st8, st32 = PT.states_of_dev(dev, "int8"), PT.states_of_dev(dev, "float32")
            want = PT.states_of(host)
            assert np.array_equal(st8.cpu().numpy()[:, 0], want) and np.array_equal(st32.cpu().numpy()[:, 0], want.astype(np.float32))
            for i in rng.choice(n, 64, replace=False):
                assert np.array_equal(want[i], oracle.Game(record=host[i]).state()), (s, i)
        a = rng.integers(0, 8, n).astype(np.int32)
        PT.step_games_dev(dev, torch.from_numpy(a).cuda())
        want = oracle.play_records(host.copy(), a)
        assert np.array_equal(dev.cpu().numpy().view(np.uint32), want), s
        pairs += n
    assert pairs >= 2**20 and ended > n // 4 * steps


@pytest.mark.parametrize("n_actions", [7, 8])
def test_playout_dev_against_cpu(gpu_lib, oracle, n_actions):
    """final records, streams and step counts of playout_dev equal a CPU restatement, at max_steps 0, 1, a few, and unlimited, with a zero
    stream and games already over among the rows"""
    import torch
    from tetris_mcts_b200 import pyTetris as PT
    n = 384
    recs = np.concatenate([PT.new_games(n // len(ENVS), e, np.arange(7 + i * n, 7 + i * n + n // len(ENVS), dtype=np.uint32))
                           for i, e in enumerate(ENVS)])
    states = np.random.default_rng(n_actions).integers(0, 2**32, n, dtype=np.uint64).astype(np.uint32)
    states[:3] = 0
    for max_steps in (0, 1, 37, 2**31 - 1):
        dev = torch.from_numpy(recs.view(np.int32)).cuda()
        rng = torch.from_numpy(states.view(np.int32)).cuda()
        steps = PT.playout_dev(dev, rng, n_actions, max_steps)
        got_r, got_s, got_k = dev.cpu().numpy().view(np.uint32), rng.cpu().numpy().view(np.uint32), steps.cpu().numpy()
        for i in range(n):
            r, s, k = playout_cpu(oracle.Game, recs[i], states[i], n_actions, max_steps)
            assert np.array_equal(got_r[i], r) and got_s[i] == s and got_k[i] == k, (max_steps, i)
        if max_steps == 2**31 - 1:
            assert ((got_r[:, 10] >> 21) & 1).all() and got_k.max() > 100
            recs_over = got_r.copy()
    dev = torch.from_numpy(recs_over.view(np.int32)).cuda()                # games over: nothing moves, the stream stays
    rng = torch.from_numpy(states.view(np.int32)).cuda()
    assert (PT.playout_dev(dev, rng, n_actions).cpu().numpy() == 0).all()
    assert np.array_equal(dev.cpu().numpy().view(np.uint32), recs_over)
    assert np.array_equal(rng.cpu().numpy().view(np.uint32)[3:], states[3:]) and (rng.cpu().numpy().view(np.uint32)[:3] == 0x2545F491).all()


def test_device_game_call_refusals(gpu_lib):
    import torch
    from tetris_mcts_b200 import _lib as L
    from tetris_mcts_b200 import pyTetris as PT
    recs = torch.zeros((4, 20), dtype=torch.int32, device="cuda")
    for bad in (recs.cpu(), recs.float(), recs[:, :19], recs.t().contiguous()[:4], torch.zeros(81, dtype=torch.int32, device="cuda")[1:].view(4, 20)):
        with pytest.raises(ValueError):
            PT.states_of_dev(bad)
    with pytest.raises(ValueError):
        PT.step_games_dev(recs, torch.zeros(3, dtype=torch.int32, device="cuda"))
    rng = torch.zeros(4, dtype=torch.int32, device="cuda")
    for k in (0, 9):
        with pytest.raises(L.B200Error):
            PT.playout_dev(recs, rng, k)
    with pytest.raises(L.B200Error):
        PT.playout_dev(recs, rng, 7, -1)
    assert PT.states_of_dev(recs[:0]).shape == (0, 1, 20, 10)


# ---------------------------------------------------------------------------------------------------- the engine
def engine(n, M, seed, gamma=0.99, low=1, env=(1, 0, 0), headroom=0):
    from tetris_mcts_b200.engine import BatchedEngine
    eng = BatchedEngine(n, max_nodes=M, mode="vanilla", eval_kind="external_game", gamma=gamma, low=low, seed=seed, overflow_reset=True,
                        env_args=((20, 10),) + tuple(env))
    if headroom:
        eng.set_gc_headroom(headroom)
    return eng


def step(eng, f):
    """one simulation step through the step API, with ids: ({game: record handed out}, n_rows)"""
    import torch
    rows, _ = eng.ext_capacity()
    buf = torch.empty((rows, 20), dtype=torch.int32, device="cuda")
    ids = torch.empty(rows, dtype=torch.int32, device="cuda")
    n = eng.ext_step_begin(buf, "record", ids)
    recs = buf[:n].cpu().numpy().view(np.uint32).copy()
    gids = ids[:n].cpu().numpy()
    assert (np.diff(gids) > 0).all()                                      # ascending game order
    v, var = f(recs)
    out = torch.from_numpy(np.stack([v, var], 1).astype(np.float32)).cuda()
    torch.cuda.synchronize()
    eng.ext_step_end(out)
    return dict(zip(gids.tolist(), recs)), n


def shadow(oracle, n, M, sims, moves, seed, headroom, gamma=0.99, low=1, env=(1, 0, 0), special=False, form="steps", f=None, oracle_f=None):
    """The engine (form "steps": the step API with ids, compared simulation by simulation; "device" / "host": play_move(game_evaluator=))
    against one oracle agent per game fed the same evaluator.  f: the engine's evaluator (numpy uint32 [n,20] -> (v, var) for "steps" and
    "host", torch for "device"), oracle_f: the oracle's f(rec) -> (v, var).  Returns the engine's counters and the games finished."""
    import torch
    from tetris_mcts_b200 import pyTetris as PT
    f = f or ((lambda r: evaluate_torch(r, special)) if form == "device" else (lambda r: evaluate_batch(r, special)))
    oracle_f = oracle_f or (lambda r: evaluate(r, special))
    recs = PT.new_games(n, env, np.arange(seed, seed + n, dtype=np.uint32))
    eng = engine(n, M, seed, gamma, low, env, headroom)
    eng.set_games(recs)
    agents, seen = [], {}
    for g in range(n):
        def fg(rec, g=g):
            seen[g] = rec
            return oracle_f(rec)
        agents.append(GameEvalAgent(oracle.Agent(max_nodes=M, mode=2, gamma=gamma, low=low, eval_mode=0, search_seed=search_seed(seed, g),
                                                 overflow_reset=1, app=env[0], scoring=env[1], randomizer=env[2]), fg))
    games = [oracle.Game(record=recs[g]) for g in range(n)]
    for g in range(n):
        agents[g].update_root(games[g].record())
    finished, handed = 0, 0
    for mv in range(moves):
        if form == "steps":
            for s in range(sims):
                got, rows = step(eng, f)
                handed += rows
                seen.clear()
                for ag in agents:
                    ag.mcts(1)
                assert sorted(got) == sorted(seen), (mv, s, sorted(got), sorted(seen))
                for g in got:
                    assert np.array_equal(got[g], seen[g]), (mv, s, g)
            stats, actions = eng.get_stats()
            eng.env_step(None)
            eng.update_root(True)
        else:
            actions, stats = eng.play_move(sims, auto_reset=True, game_evaluator=f, host=form == "host")
            for ag in agents:
                ag.mcts(sims)
        live = eng.get_games()
        for g in range(n):
            ag = agents[g]
            a, st = ag.get_action()
            assert np.array_equal(st, stats[g], equal_nan=True), "move %d game %d\n%s\n%s" % (mv, g, st, stats[g])
            # with a NaN value at the root the engine picks the first NaN, as np.argmax in agent.py:181-185 does; the oracle skips NaN, as
            # agent.cpp's std::max_element does.  Both games then follow the engine's action.
            assert actions[g] == (int(np.argmax(st[1])) if np.isnan(st[1]).any() else a), (mv, g, actions[g], a, st[1])
            a = int(actions[g])
            games[g].play(a)
            ag.update_root(games[g].record())
            if games[g].end:
                finished += 1
                games[g].reset()
                ag.update_root(games[g].record())
            if headroom and ag.n_free < headroom:
                ag.remove_nodes()
            assert np.array_equal(live[g], games[g].record()), "live game %d differs after move %d" % (g, mv)
    import gpu_twins as G
    for g in range(n):
        ex, want = eng.export_game(g), agents[g].export()
        assert ex["root"] == agents[g].root, g
        for k in ARENA_KEYS:                                              # NaN as NaN: the device's payload is its own
            assert np.array_equal(ex[k], want[k], equal_nan=ex[k].dtype.kind == "f"), (g, k)
        assert G.debug_game_state(eng, g)[0] == agents[g].rng(), g                 # the check_low stream
    c = eng.counters()
    oc = {k: sum(ag.counter(i) for ag in agents) for k, i in (("sims", 0), ("expansions", 1), ("eval_requests", 2), ("gcs", 3),
                                                              ("tree_resets", 7))}
    for k in oc:
        assert c[k] == oc[k], (k, c[k], oc[k])
    assert c["rollout_steps"] == 0 and c["games_finished"] == finished and (eng.status() == 0).all()
    if form == "steps":
        assert c["eval_requests"] == handed
    return eng, c, finished


def test_engine_reproduces_reference_golden(gpu_lib, oracle):
    """agent_type1_golden.npz (the reference's own agent.cpp, evaluator type 1): every record handed out, every action and every record
    after a move, up to the pinned float-chain divergence (all of it for gamma 1 and the NaN / inf case)."""
    z = np.load(GOLD)
    for case in range(int(z["n_cases"])):
        p = "c%d_" % case
        moves, evals = golden_span(z, case)
        env, special = tuple(int(x) for x in z[p + "env"]), bool(z[p + "special"])
        eng = engine(1, int(z["max_nodes"]), (int(z[p + "engine_seed"])) & 0xffffffff, float(z[p + "gamma"]), 1, env)
        eng.set_games(z[p + "start"][None])
        handed = []
        for mv in range(moves):
            for _ in range(int(z[p + "sims"])):
                got, _n = step(eng, lambda r: evaluate_batch(r, special))
                handed += list(got.values())
            stats, actions = eng.get_stats()
            assert actions[0] == z[p + "actions"][mv], (case, mv)
            eng.env_step(None)
            eng.update_root(True)
            assert np.array_equal(eng.get_games()[0], z[p + "records"][mv]), (case, mv)
        done = int(z[p + "eval_off"][moves])
        assert done <= evals and len(handed) == done and np.array_equal(np.stack(handed), z[p + "eval_recs"][:done]), case
        eng.close()


@pytest.mark.parametrize("special", [False, True])
def test_engine_against_oracle_per_simulation(gpu_lib, oracle, special):
    """several games per engine, a small arena (collections between moves and inside steps, dropped trees), game overs, terminal leaves;
    special: NaN / +-inf / negative values and NaN / negative variances"""
    eng, c, finished = shadow(oracle, n=12, M=600, sims=30, moves=45, seed=21 + special, headroom=140, special=special)
    assert c["gcs"] > 0 and c["tree_resets"] > 0 and (finished > 0 or special), (c, finished)   # NaN-led games outlast the 45 moves
    eng.close()


@pytest.mark.parametrize("form", ["device", "host"])
def test_engine_against_oracle_play_move(gpu_lib, oracle, form):
    """BatchedEngine.play_move(game_evaluator=) in both forms, gamma 1 and low 5 (Vanilla's), other env_args"""
    eng, c, finished = shadow(oracle, n=10, M=600, sims=25, moves=40, seed=31, headroom=140, gamma=1.0, low=5, env=(2, 1, 1), form=form,
                              special=form == "host")
    assert c["gcs"] > 0, c
    eng.close()


def test_engine_with_device_playouts_against_oracle(gpu_lib, oracle):
    """a device evaluator built on playout_dev, seeded per (game, step) from the record and a step counter the caller keeps, against the
    oracle fed the CPU restatement of the same playouts: VanillaC's random_playout (n_actions 8, variance 1e5) with known streams"""
    import torch
    from tetris_mcts_b200 import pyTetris as PT
    step_no = [0]

    def seed_of(rec):
        return (int(rec[12]) * 2654435761 + int(np.int32(rec[13])) * 40503 + step_no[0] * 97 + 1) & 0xffffffff

    def dev_f(recs):                                                     # numpy rows (the step form) -> playout on the device
        seeds = np.array([seed_of(r) for r in recs], np.uint32)
        games = torch.from_numpy(recs.view(np.int32).copy()).cuda()
        PT.playout_dev(games, torch.from_numpy(seeds.view(np.int32)).cuda(), 8)
        v = PT.record_fields(games)["score"].to(torch.float32).cpu().numpy()
        step_no[0] += 1
        return v, np.full(len(v), 1e5, np.float32)

    def oracle_f(rec):
        r, _s, _k = playout_cpu(oracle.Game, rec, seed_of(rec), 8, 2**31 - 1)
        return float(np.int32(r[13])), 1e5

    def oracle_f_step(rec):                                              # the oracle runs its games after the engine's step: one step behind
        step_no[0] -= 1
        out = oracle_f(rec)
        step_no[0] += 1
        return out
    eng, c, _ = shadow(oracle, n=6, M=4000, sims=20, moves=12, seed=41, headroom=0, f=dev_f, oracle_f=oracle_f_step)
    eng.close()


def test_step_api_refusals(gpu_lib):
    import torch
    from tetris_mcts_b200 import _lib as L
    from tetris_mcts_b200.engine import BatchedEngine
    for mode in ("lp", "single", "dist"):
        with pytest.raises(L.B200Error) as e:
            BatchedEngine(4, max_nodes=256, mode=mode, eval_kind="external_game")
        assert e.value.code == 1 and "external" in str(e.value) and "B200_MODE_VANILLA" in str(e.value)
    with pytest.raises(L.B200Error):
        BatchedEngine(4, max_nodes=256, mode="vanilla", eval_kind="external")
    eng = engine(4, 512, 3)
    assert eng.ext_capacity() == (4, 2)
    buf = torch.empty((4, 20), dtype=torch.int32, device="cuda")
    for dtype in ("int8", "float32"):
        with pytest.raises(L.B200Error):
            eng.ext_step_begin(torch.empty((4, 1, 20, 10), dtype=getattr(torch, dtype), device="cuda"), dtype)
    with pytest.raises(L.B200Error):
        eng.ext_step_begin(torch.empty(84, dtype=torch.int32, device="cuda")[1:], "record")            # not 16-byte aligned
    for call in (lambda: eng.run_sims(1), lambda: eng.play_move(1), lambda: eng.load_weights(np.zeros(L.N_WEIGHTS, np.float32)),
                 lambda: eng.valuenet(np.zeros((1, 200), np.int8))):
        with pytest.raises(L.B200Error) as e:
            call()
        assert "external_game" in str(e.value) and "b200_ext_step_begin" in str(e.value)
    n = eng.ext_step_begin(buf, "record")
    assert n == 4
    for call in (lambda: eng.ext_step_begin(buf, "record"), lambda: eng.update_root(True), lambda: eng.env_step(None),
                 lambda: eng.remove_nodes(), lambda: eng.set_games(eng.get_games()), lambda: eng.save("/nonexistent/x")):
        with pytest.raises(L.B200Error) as e:
            call()
        assert "open" in str(e.value)
    eng.ext_step_end(torch.zeros((4, 2), dtype=torch.float32, device="cuda"))
    with pytest.raises(L.B200Error):
        eng.ext_step_end(torch.zeros((4, 2), dtype=torch.float32, device="cuda"))
    with pytest.raises(ValueError):                                       # wrong output shape: raises before anything is submitted
        eng.run_sims(1, game_evaluator=lambda r: (torch.zeros(5, device="cuda"), torch.zeros(4, device="cuda")))
    eng.ext_step_end(torch.zeros((4, 2), dtype=torch.float32, device="cuda"))
    for bad in (lambda r: (torch.zeros(len(r), device="cuda", dtype=torch.float64), torch.zeros(len(r), device="cuda")),
                lambda r: (torch.zeros(len(r)), torch.zeros(len(r))), lambda r: torch.zeros((len(r), 2), device="cuda")):
        with pytest.raises(ValueError):
            eng.run_sims(1, game_evaluator=bad)
        eng.ext_step_end(torch.zeros((4, 2), dtype=torch.float32, device="cuda"))
    with pytest.raises(ValueError):
        eng.run_sims(1, game_evaluator=lambda r: (np.zeros(len(r)), np.zeros(len(r), np.float32)), host=True)
    eng.ext_step_end(torch.zeros((4, 2), dtype=torch.float32, device="cuda"))
    with pytest.raises(ValueError):
        eng.run_sims(1, evaluator=lambda b: b, game_evaluator=lambda r: r)
    eng.close()
    ext = BatchedEngine(4, max_nodes=256, mode="lp", eval_kind="external")
    with pytest.raises(L.B200Error) as e:
        ext.ext_step_begin(buf, "record")
    assert "B200_BOARD_RECORD" in str(e.value)
    ext.close()


def run_game_engine(moves, save_at=None, path=None):
    """8 games, VanillaC-like settings with a device evaluator that depends on the record only; optionally saved, destroyed and loaded"""
    from tetris_mcts_b200 import pyTetris as PT
    from tetris_mcts_b200.engine import BatchedEngine
    eng = engine(8, 3000, 77, headroom=600)
    eng.set_games(PT.new_games(8, (1, 0, 0), np.arange(3, 11, dtype=np.uint32)))
    out = []
    for mv in range(moves):
        if mv == save_at:
            eng.save(path)
            eng.close()
            eng = BatchedEngine.load(path)
        actions, stats = eng.play_move(20, game_evaluator=lambda r: evaluate_torch(r, True))
        out.append((actions.copy(), stats.copy(), eng.get_games()))
    arenas = [eng.export_game(g) for g in range(8)]
    c = eng.counters()
    eng.close()
    return out, arenas, c


def test_save_load_continues_and_runs_repeat(gpu_lib, tmp_path):
    a = run_game_engine(30)
    b = run_game_engine(30)
    c = run_game_engine(30, save_at=14, path=str(tmp_path / "img"))
    for other in (b, c):
        for (a1, s1, g1), (a2, s2, g2) in zip(a[0], other[0]):
            assert np.array_equal(a1, a2) and np.array_equal(s1.view(np.uint32), s2.view(np.uint32)) and np.array_equal(g1, g2)   # same device: same bits
        for x, y in zip(a[1], other[1]):
            for k in ARENA_KEYS:
                assert np.array_equal(x[k].view(np.uint8), y[k].view(np.uint8)), k
        assert a[2] == other[2]
    assert a[2]["gcs"] > 0


MYGAMEEVAL = """import torch


def make(device):
    def f(recs):
        v = recs[:, 13].to(torch.float32) + (recs[:, :10] != 0).sum(1).to(torch.float32)
        return v, torch.full_like(v, 100.0)
    return f
"""


def test_vanillac_agent_and_play_batched(gpu_lib, tmp_path, monkeypatch):
    """the VanillaC shim plays with its default device playout and with a host per_game(random_playout); play_batched runs VanillaC and
    Vanilla --game_evaluator with a torch evaluator"""
    import io
    import sys
    from random import randint
    from tetris_mcts_b200 import play_batched as PB
    from tetris_mcts_b200.agents.VanillaC import VanillaC
    from tetris_mcts_b200.pyTetris import Tetris, per_game

    def random_playout(game):                                             # agents/VanillaC.py:5-8, unchanged
        while not game.end:
            game.play(randint(0, 7))
        return game.score, 1e5
    for kw in (dict(), dict(game_evaluator=per_game(random_playout), game_evaluator_on_device=False)):
        ag = VanillaC(sims=12, max_nodes=4000, **kw)
        game = Tetris((20, 10), 1, 0, 0)
        ag.update_root(game)
        for _ in range(3):
            a = ag.play()
            assert 0 <= a < 7 and ag.get_stats()[0].sum() > 0
            game.play(a)
            ag.update_root(game)
        assert ag.counters()["rollout_steps"] == 0 and ag.counters()["eval_requests"] > 0
        ag.close()
    mod = tmp_path / "mygameeval.py"
    mod.write_text(MYGAMEEVAL)
    monkeypatch.syspath_prepend(str(tmp_path))
    monkeypatch.chdir(tmp_path)
    for argv in (["--agent_type", "VanillaC"], ["--agent_type", "Vanilla", "--game_evaluator", "mygameeval:make"]):
        out = io.StringIO()
        timing = {}
        PB.run(PB.parse_args(argv + ["--n_parallel", "64", "--mcts_sims", "20", "--max_moves", "6", "--endless", "--max_nodes", "2048"]),
               out=out, timing=timing)
        assert timing["moves"] == 6, (argv, timing)
    sys.modules.pop("mygameeval", None)
