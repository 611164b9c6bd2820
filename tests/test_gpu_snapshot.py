"""Engine images (b200_engine_save / b200_engine_load, BatchedEngine.save / .load) and play_batched --checkpoint_dir / --resume.  A resume is
correct when the continued run is bit-identical to the uninterrupted one: every comparison here is exact."""
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ARGS = (1, 0, 0)


def search_seed(seed, g):                          # k_init_arena's stream of game g (test_gpu_engine.search_seed)
    s = (seed + 0x9E3779B9 * (g + 1)) & 0xffffffff
    return s or 0x2545F491


def arena_offset(data):
    """byte offset of the arena field in an image (the fields before it: {u32 id, u32 0, u64 nbytes, payload, u64 checksum})"""
    import struct
    off = 16
    while True:
        fid, _z, nbytes = struct.unpack_from("<IIQ", data, off)
        if fid == 128:
            return off
        off += 16 + nbytes + 8


def _reload(eng, path):
    from tetris_mcts_b200.engine import BatchedEngine
    eng.save(path)
    eng.close()
    return BatchedEngine.load(path)


def resume_against_oracle(oracle, tmp_path, mode, n, M, sims, k, m, engine_kw=None, agent_kw=None, seed=123, eval_kind="synthetic", weights=None,
                          eval_cb=None):
    """test_gpu_engine.run_pair's oracle comparison over k + m moves, with the engine saved, destroyed and loaded after move k"""
    from tetris_mcts_b200 import pyTetris as PT
    from tetris_mcts_b200.engine import BatchedEngine
    mode_id = {"lp": 0, "single": 1, "vanilla": 2}[mode]
    recs = PT.new_games(n, ARGS, np.arange(seed, seed + n, dtype=np.uint32))
    eng = BatchedEngine(n, max_nodes=M, mode=mode, eval_kind=eval_kind, weights=weights, seed=seed, **(engine_kw or {}))
    eng.set_games(recs)
    kw = dict(max_nodes=M, mode=mode_id, gamma=0.99 if mode == "vanilla" else 0.999, low=5 if mode == "vanilla" else 1,
              eval_mode=0 if eval_cb is None else 2, eval_cb=eval_cb)
    kw.update(agent_kw or {})
    agents = [oracle.Agent(search_seed=search_seed(seed, g), **kw) for g in range(n)]
    games = [oracle.Game(record=recs[g]) for g in range(n)]
    for g in range(n):
        agents[g].update_root(games[g].record())
    before = None
    for mv in range(k + m):
        if mv == k:
            before = eng.counters()
            eng = _reload(eng, str(tmp_path / "eng.img"))
            assert eng.counters() == before
        eng.run_sims(sims)
        stats, action = eng.get_stats()
        for g in range(n):
            agents[g].mcts(sims)
            a, st = agents[g].get_action()
            assert np.array_equal(st, stats[g]) and a == action[g], (mv, g)
            games[g].play(a)
            agents[g].update_root(games[g].record())
            if games[g].end:
                games[g].reset()
                agents[g].update_root(games[g].record())
        eng.env_step(None)
        eng.update_root(auto_reset=True)
        assert np.array_equal(eng.get_games(), np.stack([gm.record() for gm in games])), mv
        if mv >= k and (mv - k) % 10 == 0 or mv == k + m - 1:
            for g in range(min(n, 4)):
                ex, want = eng.export_game(g), agents[g].export()
                assert ex["root"] == agents[g].root
                for key in ("child", "n2o", "episode", "score", "visit", "value", "variance", "obs_end", "obs_key", "game"):
                    assert np.array_equal(ex[key], want[key]), (mv, g, key)
    c = eng.counters()
    assert c["gcs"] == sum(a.counter(3) for a in agents) and c["expansions"] == sum(a.counter(1) for a in agents)
    eng.close()
    return before, c


@pytest.mark.parametrize("case", [
    dict(mode="lp", n=12, M=1500, sims=12, k=40, m=70),
    dict(mode="lp", n=12, M=1500, sims=12, k=40, m=70, engine_kw=dict(stale_pop=False), agent_kw=dict(stale_pop=0)),
    dict(mode="lp", n=8, M=2048, sims=40, k=4, m=8, engine_kw=dict(lp_end_from_obs=True, lp_var_gamma2=False),
         agent_kw=dict(lp_end_from_obs=1, lp_var_gamma2=0)),
    dict(mode="lp", n=8, M=1500, sims=12, k=60, m=80, engine_kw=dict(path_cache=True)),
    dict(mode="single", n=12, M=1500, sims=20, k=20, m=40),
    dict(mode="vanilla", n=8, M=4096, sims=40, k=3, m=5),
], ids=["lp", "lp_no_stale_pop", "lp_agent_cpp", "lp_path_cache", "single", "vanilla"])
def test_save_destroy_load_continue_against_the_oracle(gpu_lib, oracle, tmp_path, case):
    before, after = resume_against_oracle(oracle, tmp_path, **case)
    if case["M"] == 1500:   # the moves after the resume collect and finish games
        assert after["gcs"] > before["gcs"] and after["games_finished"] > before["games_finished"]


@pytest.mark.parametrize("mode", ["lp", "single"])
def test_save_destroy_load_continue_against_the_oracle_net_tc(gpu_lib, oracle, tmp_path, mode):
    """the same with the tensor-core value network: the reloaded engine searches with the weights its image holds, the oracle agent is fed
    the outputs of the same network (test_gpu_engine.test_real_network_search_is_exact_given_the_same_evaluator)"""
    from tetris_mcts_b200.engine import BatchedEngine
    w = oracle.seeded_weights(0)
    side = BatchedEngine(1, max_nodes=64, eval_kind="net_tc", weights=w)
    resume_against_oracle(oracle, tmp_path, mode, n=3, M=2048, sims=25, k=3, m=4, eval_kind="net_tc", weights=w,
                          eval_cb=lambda states: side.valuenet(states))
    side.close()


def _compare(a, b, games, dist=False, skip=()):
    assert np.array_equal(a.get_games(), b.get_games())
    ca, cb = a.counters(), b.counters()
    assert {k: v for k, v in ca.items() if k not in skip} == {k: v for k, v in cb.items() if k not in skip}
    assert np.array_equal(a.status(), b.status())
    assert np.array_equal(a.finished_games(), b.finished_games())
    for g in games:
        ea, eb = a.export_game(g), b.export_game(g)
        for key in ea:
            assert np.array_equal(ea[key], eb[key]), (g, key)
        if dist:
            for x, y in zip(a.export_dist(g), b.export_dist(g)):
                assert np.array_equal(x.view(np.uint32), y.view(np.uint32)), g


def engine_against_engine(tmp_path, make, k, m, sims, staging=None, setup=None, dist=False):
    """engine A plays k moves and is saved; B is loaded from the image; both play m moves and must agree exactly at every move"""
    import tetris_mcts_b200._lib as L
    from tetris_mcts_b200.engine import BatchedEngine
    a = make()
    if setup:
        setup(a)
    for _ in range(k):
        a.play_move(sims, auto_reset=True)
    path = str(tmp_path / "a.img")
    if staging:
        L.check(L.lib().b200_snapshot_set_staging(int(staging)))
    try:
        size = a.save(path)
        b = BatchedEngine.load(path)
    finally:
        L.check(L.lib().b200_snapshot_set_staging(0))
    assert size == os.path.getsize(path) and not os.path.exists(path + ".tmp")
    assert (b.mode, b.eval_kind, b.n_games, b.max_nodes, b.path_cache) == (a.mode, a.eval_kind, a.n_games, a.max_nodes, a.path_cache)
    before = a.counters()
    sample = sorted(set(np.linspace(0, a.n_games - 1, 5).astype(int)))
    _compare(a, b, sample, dist)
    for _ in range(m):
        xa, sa = a.play_move(sims, auto_reset=True)
        xb, sb = b.play_move(sims, auto_reset=True)
        assert np.array_equal(xa, xb) and np.array_equal(sa.view(np.uint32), sb.view(np.uint32))
        _compare(a, b, sample[:2], dist)
    _compare(a, b, sample, dist)
    after = a.counters()
    a.close(); b.close()
    return before, after


def test_engine_against_engine_net_fp16_thousands_of_games_many_chunks(gpu_lib, tmp_path):
    """2048 games with the path cache on (restored empty), the deep lane set, overflow_reset and a between-moves collection, through a
    1 MB staging buffer (hundreds of chunks)"""
    from tetris_mcts_b200.engine import BatchedEngine
    from tetris_mcts_b200 import pyTetris as PT
    from tetris_mcts_b200.model.model_vv import init_weights
    n, M = 2048, 256

    def make():
        e = BatchedEngine(n, max_nodes=M, mode="lp", eval_kind="net_fp16", weights=init_weights(3), seed=5, overflow_reset=True, path_cache=True)
        e.set_games(PT.new_games(n, ARGS, np.arange(n, dtype=np.uint32) + 7))
        e.set_gc_headroom(M * 5 // 32)
        e.set_deep_lane(64)
        return e
    before, after = engine_against_engine(tmp_path, make, k=6, m=8, sims=24, staging=1 << 20)
    assert after["gcs"] > before["gcs"] and after["tree_resets"] > before["tree_resets"]


@pytest.mark.parametrize("kind", ["net_tc", "dist_fp16"])
def test_engine_against_engine_distributional(gpu_lib, tmp_path, kind):
    from tetris_mcts_b200.engine import BatchedEngine
    from tetris_mcts_b200 import pyTetris as PT
    rng = np.random.default_rng(4)
    atoms = 50
    need = 512 + 32 + 16384 + 32 + 128 * 2048 + 128 + atoms * 128 + atoms
    dw = (rng.standard_normal(need) * 0.02).astype(np.float32)
    n, M = 96, 1024

    def make():
        e = BatchedEngine(n, max_nodes=M, mode="dist", eval_kind=kind, dist_weights=dw, dist_bins=atoms, seed=11)
        e.set_games(PT.new_games(n, ARGS, np.arange(n, dtype=np.uint32) + 3))
        return e
    before, after = engine_against_engine(tmp_path, make, k=5, m=12, sims=30, dist=True)
    assert after["gcs"] > before["gcs"]


def test_engine_against_engine_overflow_reset_and_game_over(gpu_lib, tmp_path):
    """net_tc with arenas small enough that collections cannot shrink them (tree drops) and games that end (auto_reset) after the resume"""
    from tetris_mcts_b200.engine import BatchedEngine
    from tetris_mcts_b200 import pyTetris as PT
    from tetris_mcts_b200.model.model_vv import init_weights
    n, M = 64, 256

    def make():
        e = BatchedEngine(n, max_nodes=M, mode="lp", eval_kind="net_tc", weights=init_weights(1), seed=9, overflow_reset=True)
        e.set_games(PT.new_games(n, ARGS, np.arange(n, dtype=np.uint32)))
        return e
    before, after = engine_against_engine(tmp_path, make, k=30, m=120, sims=16)
    assert after["tree_resets"] > before["tree_resets"] and after["games_finished"] > before["games_finished"]


@pytest.mark.parametrize("policy", [0, 1, 2, 3])
def test_replay_memory_and_policies_continue_after_a_restore(gpu_lib, tmp_path, policy):
    """a small memory under each accumulation policy: the decisions, memory_index and the memory's bytes after every move agree between the
    uninterrupted engine and the one restored mid-run, over trainings and (policies 0 and 1) trimmings after the restore: the policy-0
    drops and random trimmings draw from the restored mt19937 and sampler.  The episode count the policy is given stays 0 until move 130, so
    that the memory fills and policies 0 and 1 trim it, then advances, so that policies 0-2 train.  One game per engine: the rows of one
    collection launch over several games land in the order the CTAs reach the memory's counter (k_gc), so only a one-game memory has the
    same byte order in two engines."""
    import torch
    from tetris_mcts_b200.engine import BatchedEngine
    from tetris_mcts_b200 import pyTetris as PT
    n, M, cap = 1, 512, 100
    a = BatchedEngine(n, max_nodes=M, mode="lp", eval_kind="synthetic", seed=2, overflow_reset=True)
    a.set_games(PT.new_games(n, ARGS, np.arange(n, dtype=np.uint32) + 1))
    a.set_gc_headroom(M * 5 // 32)
    a.replay_enable(min_visits=2, capacity=cap)
    a.replay_policy(policy, episodes_per_train=4, memory_growth_rate=40)
    bufs = [torch.empty((2 * cap, 212), dtype=torch.uint8, device="cuda") for _ in range(2)]
    torch.cuda.synchronize()

    def episode(mv):
        return 0 if mv < 130 else (mv - 128) // 2

    def move(e, i, mv):
        e.play_move(24, auto_reset=True)
        train, idx = e.replay_policy_step(episode(mv))
        e.replay_peek_into(bufs[i].data_ptr(), max(idx, 1))
        rows = bufs[i][:idx].cpu().numpy()
        if train:
            e.replay_policy_trained(episode(mv))
        return train, idx, rows
    for mv in range(40):
        move(a, 0, mv)
    a.save(str(tmp_path / "p.img"))
    b = BatchedEngine.load(str(tmp_path / "p.img"))
    trained = trimmed = 0
    prev = np.zeros((0, 212), np.uint8)
    gcs = a.counters()["gcs"]
    for mv in range(40, 170):
        ra, rb = move(a, 0, mv), move(b, 1, mv)
        assert ra[0] == rb[0] and ra[1] == rb[1] and np.array_equal(ra[2], rb[2]), (policy, mv)
        m = min(len(prev), len(ra[2]))
        trimmed += int(not np.array_equal(prev[:m], ra[2][:m]))   # rows leave the middle only when a trimming compacts the memory
        trained += int(ra[0])
        prev = np.zeros((0, 212), np.uint8) if ra[0] else ra[2]
    assert a.counters() == b.counters() and a.counters()["gcs"] >= gcs + 5
    assert trained > 0, policy
    if policy in (0, 1):
        assert trimmed > 0, policy
    a.close(); b.close()


def test_external_evaluator_resume_and_open_step_refused(gpu_lib, tmp_path):
    import torch
    import tetris_mcts_b200._lib as L
    from tetris_mcts_b200.engine import BatchedEngine
    from tetris_mcts_b200 import pyTetris as PT
    n, M = 64, 1024

    def evaluator(boards):                         # integer-exact outputs of the board alone
        s = boards.reshape(len(boards), -1).sum(dim=1)
        return (s * 0.25).contiguous(), (s * 0 + 2.0).contiguous()
    a = BatchedEngine(n, max_nodes=M, mode="lp", eval_kind="external", seed=4)
    a.set_games(PT.new_games(n, ARGS, np.arange(n, dtype=np.uint32) + 5))
    for _ in range(6):
        a.play_move(20, evaluator=evaluator)
    rows, cols = a.ext_capacity()
    boards = torch.empty((rows, 1, 20, 10), dtype=torch.float32, device="cuda")
    out = torch.zeros((rows, cols), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    a.ext_step_begin(boards)
    with pytest.raises(L.B200Error) as ei:
        a.save(str(tmp_path / "x.img"))
    assert ei.value.code == 1 and "step is open" in str(ei.value)
    assert not os.path.exists(tmp_path / "x.img")
    a.ext_step_end(out)                            # (a step of zeros: the same one for both engines below)
    a.sync()
    a.save(str(tmp_path / "x.img"))
    b = BatchedEngine.load(str(tmp_path / "x.img"))
    assert b.eval_kind == L.EVAL_EXTERNAL
    for _ in range(8):
        xa, sa = a.play_move(20, evaluator=evaluator)
        xb, sb = b.play_move(20, evaluator=evaluator)
        assert np.array_equal(xa, xb) and np.array_equal(sa.view(np.uint32), sb.view(np.uint32))
    _compare(a, b, [0, 31, 63], skip=("cached_levels",))   # saved mid-move: A's path cache was warm, B's restarted empty (no result changes)
    a.close(); b.close()


def test_bad_images_are_refused_with_a_message(gpu_lib, tmp_path):
    import tetris_mcts_b200._lib as L
    from tetris_mcts_b200.engine import BatchedEngine
    from tetris_mcts_b200 import pyTetris as PT
    e = BatchedEngine(16, max_nodes=512, mode="lp", eval_kind="synthetic", seed=1)
    e.set_games(PT.new_games(16, ARGS, np.arange(16, dtype=np.uint32)))
    for _ in range(3):
        e.play_move(20)
    good = str(tmp_path / "good.img")
    e.save(good)
    data = open(good, "rb").read()
    arena = arena_offset(data)
    first_game = arena + 16 + 8 + 16 * 8 + 8
    flipped = bytearray(data)
    flipped[first_game + 4 * 200] ^= 0x10                        # a word of game 0's records
    version = bytearray(data)
    version[8] = 2
    cases = {"truncated": (data[:len(data) // 2], "truncated"), "flipped": (bytes(flipped), "game 0: checksum mismatch"),
             "version": (bytes(version), "format version 2"), "magic": (b"NOTSNAP!" + data[8:], "wrong magic"),
             "unknown field": (data[:16] + b"\xff\x00\x00\x00" + data[20:], "unknown field 255")}
    for name, (blob, msg) in cases.items():
        p = str(tmp_path / (name.replace(" ", "_") + ".img"))
        open(p, "wb").write(blob)
        h = L.P()
        rc = L.lib().b200_engine_load(os.fsencode(p), -1, __import__("ctypes").byref(h))
        assert rc == 1 and not h.value, name
        assert msg in L.lib().b200_last_error().decode(), (name, L.lib().b200_last_error())
    b = BatchedEngine.load(good)                                 # a valid image still loads after the refusals
    x1, s1 = e.play_move(20)
    x2, s2 = b.play_move(20)
    assert np.array_equal(x1, x2) and np.array_equal(s1, s2)
    e.close(); b.close()


# ------------------------------------------------------------------ play_batched --online --checkpoint_dir / --resume
# one game per rank: the rows of one collection launch over several games enter the replay memory in the order the CTAs reach its counter,
# so a run of several games per rank trains on another row order, and plays on differently, each time it runs (resumed or not)
RUN = ["--agent_type", "ValueSimLP", "--mcts_sims", "64", "--ngames", "100000", "--max_nodes", "1024", "--endless",
       "--online", "--train_max_iters", "200", "--train_batch_size", "256", "--memory_size", "2000", "--memory_growth_rate", "60", "--save"]


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _play(cwd, argv, world=1):
    port = _free_port()
    procs = []
    for r in range(world):
        env = {k: v for k, v in os.environ.items() if k not in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_PORT")}
        env["PYTHONPATH"] = ROOT + os.pathsep + env.get("PYTHONPATH", "")
        if world > 1:
            env.update(RANK=str(r), WORLD_SIZE=str(world), LOCAL_RANK="0", MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        cmd = [sys.executable, "-m", "tetris_mcts_b200.play_batched"] + argv + (["--dist_backend", "gloo"] if world > 1 else [])
        procs.append(subprocess.Popen(cmd, cwd=cwd, env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True))
    out = [p.communicate(timeout=1500) for p in procs]
    for p, (so, se) in zip(procs, out):
        assert p.returncode == 0, se[-3000:]
    return out[0]


def _saved_rows(d, world):
    import glob
    parts = []
    for r in range(world):
        suffix = "" if world == 1 else ".rank%d" % r
        parts += [np.load(f) for f in sorted(glob.glob(os.path.join(d, "data", "data0%s.*.npy" % suffix)))]
    return np.concatenate(parts) if parts else None


def _resume_run(tmp_path, n, k, world, kind):
    import torch
    a, b = tmp_path / "a", tmp_path / "b"
    a.mkdir(); b.mkdir()
    base = RUN + ["--train_kind", kind, "--n_parallel", str(world)]
    so_a, se_a = _play(a, base + ["--max_moves", str(n)], world)
    so_b1, se_b1 = _play(b, base + ["--max_moves", str(k), "--checkpoint_dir", "ckpt", "--checkpoint_every", "25"], world)
    so_b2, se_b2 = _play(b, base + ["--max_moves", str(n), "--checkpoint_dir", "ckpt", "--resume"], world)
    eps = lambda s: [ln for ln in s.splitlines() if ln.startswith("Episode:")]         # noqa: E731
    mem = lambda s: [ln for ln in s.splitlines() if ln.startswith("Memory usage")]     # noqa: E731
    assert eps(so_a) == eps(so_b1) + eps(so_b2)
    assert mem(se_a) == mem(se_b1) + mem(se_b2) and mem(se_b2)
    assert "Training data size" in se_b2, "no training after the resume point"
    ca = torch.load(a / "pytorch_model" / "model_checkpoint", weights_only=False)
    cb = torch.load(b / "pytorch_model" / "model_checkpoint", weights_only=False)
    for key in ca["model_state_dict"]:
        assert torch.equal(ca["model_state_dict"][key], cb["model_state_dict"][key]), key
    for i, st in ca["optimizer_state_dict"]["state"].items():
        sb = cb["optimizer_state_dict"]["state"][i]
        assert st["step"] == sb["step"] and torch.equal(st["exp_avg"], sb["exp_avg"]) and torch.equal(st["exp_avg_sq"], sb["exp_avg_sq"])
    ra, rb = _saved_rows(a, world), _saved_rows(b, world)
    assert ra is not None and ra.tobytes() == rb.tobytes()


@pytest.mark.parametrize("kind", ["fp64", "tf32"])
def test_play_batched_online_resume_is_the_uninterrupted_run(gpu_lib, tmp_path, kind):
    _resume_run(tmp_path, n=140, k=70, world=1, kind=kind)


def test_play_batched_two_ranks_gloo_resume(gpu_lib, tmp_path):
    _resume_run(tmp_path, n=120, k=60, world=2, kind="fp64")
