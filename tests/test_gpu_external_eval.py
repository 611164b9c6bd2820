"""The caller-supplied evaluator (eval_kind "external", b200_ext_step_begin / b200_ext_step_end) on the GPU.

- Exact against the oracle: the engine's evaluator is the integer-exact torch function of tests/ext_eval_twins.py, the oracle agents' eval_cb
  its numpy twin; every game is shadowed (actions, stats, live games every move; arenas, node_stats / node_dist and counters at the end).
  Every case asserts that collections, dropped trees (overflow_reset) and finished games occurred.
- Equivalence with the built-in networks: an external engine whose evaluator is a side engine's network is bit-identical to the built-in kind.
- The board hand-out, a real torch network, and the errors of the step API."""
import numpy as np
import pytest

from ext_eval_twins import dist_np, dist_torch, value_np, value_torch

pytestmark = pytest.mark.gpu
ARGS = (1, 0, 0)
ARENA_KEYS = ("child", "n2o", "episode", "score", "game", "visit", "value", "variance", "obs_end", "obs_key")
ORACLE_MODE = {"lp": 0, "single": 1, "dist": 3}


def search_seed(seed, g):
    s = (seed + 0x9E3779B9 * (g + 1)) & 0xffffffff
    return s or 0x2545F491


def shadow(oracle, mode, n, M, sims, moves, seed, headroom, bins=50, lp_end_from_obs=0, path_cache=False, host=False, dist_list=False,
           replay=None, bad_output_at=None):
    """play_move(evaluator=...) on an external engine against oracle agents on every game.  Returns (counters, finished games)."""
    import torch
    from tetris_mcts_b200 import pyTetris as PT
    from tetris_mcts_b200.engine import BatchedEngine
    low = 1
    recs = PT.new_games(n, ARGS, np.arange(seed, seed + n, dtype=np.uint32))
    eng = BatchedEngine(n, max_nodes=M, mode=mode, eval_kind="external", seed=seed, low=low, overflow_reset=True, dist_bins=bins,
                        lp_end_from_obs=bool(lp_end_from_obs), path_cache=path_cache)
    eng.set_games(recs)
    eng.set_gc_headroom(headroom)
    if replay:
        eng.replay_enable(min_visits=replay, capacity=200000)
    if mode == "dist":
        cb = lambda st: dist_np(st, bins)                                      # noqa: E731
        ev = (lambda st: [dist_np(st, bins)]) if dist_list else cb if host else dist_torch(bins)
    else:
        cb = value_np
        ev = (lambda st: tuple(x.reshape(-1, 1) for x in value_np(st))) if host else value_torch
    agents = [oracle.Agent(max_nodes=M, mode=ORACLE_MODE[mode], low=low, eval_mode=2, eval_cb=cb, search_seed=search_seed(seed, g),
                           dist_bins=bins, overflow_reset=1, lp_end_from_obs=lp_end_from_obs,
                           replay_min_visits=replay or 0, replay_cap=200000 if replay else 0) for g in range(n)]
    games = [oracle.Game(record=recs[g]) for g in range(n)]
    for g in range(n):
        agents[g].update_root(games[g].record())
    finished = 0
    for mv in range(moves):
        if mv == bad_output_at:                         # a wrong-shaped output: ValueError, the step stays open, a correct end completes it
            seen = {}

            def bad(b):
                seen["boards"] = b
                return torch.zeros(b.shape[0] + 1, device=b.device), torch.zeros(b.shape[0], device=b.device)
            with pytest.raises(ValueError):
                eng.run_sims(1, evaluator=bad)
            for call in (lambda: eng.run_sims(1, evaluator=ev), lambda: eng.update_root(True), lambda: eng.env_step(None)):
                with pytest.raises(gpu_lib_error()):
                    call()
            v, var = value_torch(seen["boards"])
            out = torch.stack([v, var], 1).contiguous()
            torch.cuda.synchronize()
            eng.ext_step_end(out)
            eng.run_sims(sims - 1, evaluator=ev)
            stats, actions = eng.get_stats()
            eng.env_step(None)
            eng.update_root(True)
        else:
            actions, stats = eng.play_move(sims, auto_reset=True, evaluator=ev, host=host)
        live = eng.get_games()
        for g in range(n):
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
            if ag.n_free < headroom:
                ag.remove_nodes()
            assert np.array_equal(live[g], games[g].record()), "live game %d differs after move %d" % (g, mv)
    for g in range(n):
        ex, want = eng.export_game(g), agents[g].export()
        assert ex["root"] == agents[g].root, g
        for k in (ARENA_KEYS if mode != "dist" else ("child", "n2o", "episode", "score", "game")):
            assert np.array_equal(ex[k], want[k]), (g, k)
        if mode == "dist":
            ns, nd = eng.export_dist(g)
            wns, wnd = agents[g].export_dist()
            assert np.array_equal(ns, wns) and np.array_equal(nd.view(np.uint32), wnd.view(np.uint32)), g
    c = eng.counters()
    oc = {k: sum(ag.counter(i) for ag in agents) for k, i in (("sims", 0), ("expansions", 1), ("gcs", 3), ("tree_resets", 7))}
    for k in oc:
        assert c[k] == oc[k], (k, c[k], oc[k])
    assert c["sims"] == n * sims * moves and c["games_finished"] == finished and (eng.status() == 0).all()
    assert c["gcs"] > 0 and c["tree_resets"] > 0 and finished > 0, (c, finished)
    if replay:
        buf = torch.zeros((200000, 212), dtype=torch.uint8, device="cuda")
        got = buf[:eng.replay_drain_into(buf.data_ptr(), 200000)].cpu().numpy()
        want = np.concatenate([ag.replay() for ag in agents])
        key = lambda a: a[np.lexsort(a.T[::-1])]                               # noqa: E731
        assert len(want) > 0 and np.array_equal(key(got), key(want))
    eng.close()
    return c, finished


def gpu_lib_error():
    from tetris_mcts_b200._lib import B200Error
    return B200Error


@pytest.mark.parametrize("lp_end_from_obs,path_cache", [(0, False), (0, True), (1, False), (1, True)])
def test_lp_exact_against_oracle(gpu_lib, oracle, lp_end_from_obs, path_cache):
    shadow(oracle, "lp", n=24, M=700, sims=30, moves=60, seed=31 + lp_end_from_obs, headroom=150, lp_end_from_obs=lp_end_from_obs,
           path_cache=path_cache, replay=3 if (lp_end_from_obs, path_cache) == (0, True) else None)


def test_single_exact_against_oracle(gpu_lib, oracle):
    shadow(oracle, "single", n=24, M=700, sims=30, moves=60, seed=41, headroom=150)


@pytest.mark.parametrize("bins", [2, 50, 64])
def test_dist_exact_against_oracle(gpu_lib, oracle, bins):
    shadow(oracle, "dist", n=24, M=700, sims=40, moves=60, seed=51 + bins, headroom=150, bins=bins)


def test_host_evaluator_lp(gpu_lib, oracle):
    shadow(oracle, "lp", n=16, M=700, sims=30, moves=60, seed=61, headroom=150, host=True, path_cache=True)


def test_host_evaluator_dist_list_of_one(gpu_lib, oracle):
    shadow(oracle, "dist", n=16, M=700, sims=40, moves=60, seed=62, headroom=150, bins=50, host=True, dist_list=True)


def test_wrong_output_leaves_the_step_open(gpu_lib, oracle):
    """A wrong-shaped output raises ValueError before anything is submitted; mutating calls fail while the step is open; a correct
    ext_step_end then completes it and the shadow still matches."""
    shadow(oracle, "lp", n=16, M=700, sims=30, moves=60, seed=71, headroom=150, bad_output_at=3)


# ----------------------------------------------------------------------------------------------- equivalence with the built-in networks
def _builtin_pair(mode, kind, n, M, seed, headroom, bins=50):
    from tetris_mcts_b200 import pyTetris as PT
    from tetris_mcts_b200.engine import BatchedEngine
    from tetris_mcts_b200.model.model_vv import init_weights
    from tetris_mcts_b200.agents.DistValueSimOnline import init_dist_weights
    recs = PT.new_games(n, ARGS, np.arange(seed, seed + n, dtype=np.uint32))
    kw = dict(mode=mode, seed=seed, overflow_reset=True, dist_bins=bins)
    if mode == "dist":
        w = dict(dist_weights=init_dist_weights(0, bins))
    else:
        w = dict(weights=init_weights(0))
    ref = BatchedEngine(n, max_nodes=M, eval_kind=kind, **kw, **w)
    ext = BatchedEngine(n, max_nodes=M, eval_kind="external", **kw)
    side = BatchedEngine(1, max_nodes=64, mode=mode, eval_kind=kind, dist_bins=bins, **w)
    for e in (ref, ext):
        e.set_games(recs)
        e.set_gc_headroom(headroom)
    return ref, ext, side, (side.distnet if mode == "dist" else side.valuenet)


def _equivalence(mode, kind, n, M, sims, moves, seed, headroom, sample=None):
    ref, ext, side, ev = _builtin_pair(mode, kind, n, M, seed, headroom)
    for mv in range(moves):
        a0, s0 = ref.play_move(sims, auto_reset=True)
        a1, s1 = ext.play_move(sims, auto_reset=True, evaluator=ev, host=True)
        assert a0.tobytes() == a1.tobytes() and s0.tobytes() == s1.tobytes(), (mode, kind, mv)
        assert ref.get_games().tobytes() == ext.get_games().tobytes(), (mode, kind, mv)
    for g in (range(n) if sample is None else sample):
        x0, x1 = ref.export_game(g), ext.export_game(g)
        for k in ARENA_KEYS:
            assert x0[k].tobytes() == x1[k].tobytes(), (mode, kind, g, k)
        if mode == "dist":
            assert all(p.tobytes() == q.tobytes() for p, q in zip(ref.export_dist(g), ext.export_dist(g))), (kind, g)
    c0, c1 = ref.counters(), ext.counters()
    c0.pop("max_trace_len"), c1.pop("max_trace_len")
    assert c0 == c1 and c0["gcs"] > 0, (c0, c1)
    for e in (ref, ext, side):
        e.close()


@pytest.mark.parametrize("mode,kind", [("lp", "net"), ("lp", "net_tc"), ("lp", "net_fp16"), ("single", "net"), ("single", "net_tc"),
                                       ("single", "net_fp16"), ("dist", "net"), ("dist", "net_tc"), ("dist", "dist_fp16")])
def test_equivalent_to_builtin_network(gpu_lib, mode, kind):
    _equivalence(mode, kind, n=32, M=700, sims=30, moves=12, seed=81, headroom=150)


def test_equivalent_to_builtin_network_large(gpu_lib):
    """2048 games x 200 simulations x 3 moves with collections: bit-identical to the built-in net_tc every move"""
    _equivalence("lp", "net_tc", n=2048, M=1024, sims=200, moves=3, seed=82, headroom=1024 * 5 // 32, sample=[0, 1, 777, 2047])


# ----------------------------------------------------------------------------------------------- the board hand-out
@pytest.mark.parametrize("mode", ["lp", "single", "dist"])
@pytest.mark.parametrize("dtype", ["int8", "float32"])
def test_board_hand_out(gpu_lib, oracle, mode, dtype):
    import torch
    from tetris_mcts_b200 import pyTetris as PT
    from tetris_mcts_b200.engine import BatchedEngine
    n, M, seed = 40, 1024, 91
    eng = BatchedEngine(n, max_nodes=M, mode=mode, eval_kind="external", seed=seed, overflow_reset=True)
    eng.set_games(PT.new_games(n, ARGS, np.arange(seed, seed + n, dtype=np.uint32)))
    ev = dist_torch(50) if mode == "dist" else value_torch
    eng.run_sims(20, evaluator=ev)
    rows, cols = eng.ext_capacity()
    assert (rows, cols) == ((7 * n if mode == "lp" else n), (50 if mode == "dist" else 2))
    boards = torch.full((rows, 1, 20, 10), 9, dtype=getattr(torch, dtype), device="cuda")
    ids = torch.full((rows,), -1, dtype=torch.int32, device="cuda")
    checked = 0
    for _ in range(3):
        ids.fill_(-1)
        torch.cuda.synchronize()
        before = eng.counters()["eval_requests"]
        k = eng.ext_step_begin(boards, dtype, ids)
        assert eng.counters()["eval_requests"] - before == k and 0 < k <= rows
        idv, bv = ids[:k].cpu().numpy(), boards[:k].cpu().numpy().reshape(k, 200)
        assert (np.diff(idv) > 0).all() and (ids[k:].cpu().numpy() == -1).all()
        for r in range(k):
            g, slot = divmod(int(idv[r]), 8)
            ex = eng.export_game(g)
            leaf = int(ex["last_trace"][-1])
            node = int(ex["child"][leaf][slot]) if mode == "lp" else leaf
            assert mode == "lp" or slot == 7
            want = oracle.obskey_to_state(ex["obs_key"][ex["n2o"][node]]).ravel()
            assert np.array_equal(bv[r].astype(np.int64), want.astype(np.int64)), (mode, dtype, r, g, slot)
            checked += 1
        out = torch.zeros((rows, cols), dtype=torch.float32, device="cuda")
        if mode == "dist":
            out[:k] = ev(boards[:k].float())
        else:
            v, var = ev(boards[:k].float())
            out[:k, 0], out[:k, 1] = v, var
        eng.ext_step_end(out)
    assert checked > 0 and (eng.status() == 0).all()
    eng.close()


# ----------------------------------------------------------------------------------------------- a real torch network
def test_torch_value_network_drives_a_search(gpu_lib):
    import os
    import sys
    import torch
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))
    from external_eval_bench import module_evaluator, value_net
    from tetris_mcts_b200 import pyTetris as PT
    from tetris_mcts_b200.engine import BatchedEngine
    from tetris_mcts_b200.model.model_vv import init_weights
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    n, M, seed = 256, 2048, 101
    w = init_weights(0)
    ev = module_evaluator(value_net(w, torch.device("cuda", 0)))
    eng = BatchedEngine(n, max_nodes=M, mode="lp", eval_kind="external", seed=seed, overflow_reset=True)
    eng.set_games(PT.new_games(n, ARGS, np.arange(seed, seed + n, dtype=np.uint32)))
    for _ in range(3):
        eng.play_move(40, auto_reset=True, evaluator=ev)
    assert (eng.status() == 0).all()
    rows, _ = eng.ext_capacity()
    boards = torch.zeros((rows, 1, 20, 10), dtype=torch.float32, device="cuda")
    k = eng.ext_step_begin(boards, "float32")
    assert k > 0
    v, var = ev(boards[:k])
    ref = BatchedEngine(1, max_nodes=64, eval_kind="net", weights=w)
    rv, rvar = ref.valuenet(boards[:k].to(torch.int8).cpu().numpy())
    assert np.allclose(v.cpu().numpy(), rv, rtol=1e-5, atol=1e-5) and np.allclose(var.cpu().numpy(), rvar, rtol=1e-5, atol=1e-5)
    out = torch.stack([v, var], 1).contiguous()
    eng.ext_step_end(out)
    eng.sync()
    assert (eng.status() == 0).all()
    for e in (eng, ref):
        e.close()


# ----------------------------------------------------------------------------------------------- errors
def test_step_api_errors(gpu_lib):
    import torch
    from tetris_mcts_b200 import pyTetris as PT
    from tetris_mcts_b200.engine import BatchedEngine
    from tetris_mcts_b200.model.model_vv import init_weights
    E = gpu_lib.B200Error
    with pytest.raises(E):
        BatchedEngine(4, max_nodes=256, mode="vanilla", eval_kind="external")
    eng = BatchedEngine(4, max_nodes=256, mode="lp", eval_kind="external")
    recs = PT.new_games(4, ARGS, np.arange(4, dtype=np.uint32))
    eng.set_games(recs)
    for call in (lambda: eng.run_sims(1), lambda: eng.play_move(1), lambda: eng.load_weights(init_weights(0)),
                 lambda: eng.valuenet(np.zeros((1, 200), np.int8))):
        with pytest.raises(E, match="b200_ext_step_begin"):
            call()
    rows, cols = eng.ext_capacity()
    boards = torch.zeros((rows, 1, 20, 10), dtype=torch.float32, device="cuda")
    out = torch.zeros((rows, cols), dtype=torch.float32, device="cuda")
    with pytest.raises(E):
        eng.ext_step_end(out)                                                   # no open step
    eng.ext_step_begin(boards)
    with pytest.raises(E):
        eng.ext_step_begin(boards)                                              # a second begin
    for call in (lambda: eng.update_root(True), lambda: eng.set_games(recs), lambda: eng.env_step(None), lambda: eng.remove_nodes(),
                 lambda: eng.set_stream(None), lambda: eng.replay_enable(1, 10), lambda: eng.set_path_cache(False)):
        with pytest.raises(E, match="b200_ext_step_end"):
            call()
    eng.export_game(0), eng.counters(), eng.status(), eng.get_stats()      # reading calls work while a step is open
    eng.ext_step_end(out)
    eng.run_sims(2, evaluator=value_torch)
    eng.update_root(True)
    assert (eng.status() == 0).all()
    eng.close()
