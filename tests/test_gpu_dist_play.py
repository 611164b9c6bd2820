"""The distributional agent as a product: root values on the device (b200_dist_root_values_dev, BatchedEngine.dist_root_values) bit for bit
the operator twin b200_dist_mean_variance on each root row, Model_Dist on the engine's kernels with the reference's checkpoint layout, and
play_batched --agent_type DistValueSimOnline: the same moves as an engine driven move by move and as the C oracle's distributional agent,
--evaluator, --save rows, --resume and two ranks."""
import io
import os
import socket
import subprocess
import sys
from collections import OrderedDict

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENV = ((20, 10), 1, 0, 0)


def search_seed(seed, g):                          # k_init_arena's stream of game g
    s = (seed + 0x9E3779B9 * (g + 1)) & 0xffffffff
    return s or 0x2545F491


def twin_root_values(eng):
    """b200_dist_mean_variance (the operator twin) on export_dist(g)'s root row, game by game"""
    from tetris_mcts_b200.agents.core_distributional import mean_variance
    out = np.zeros((eng.n_games, 2), np.float64)
    for g in range(eng.n_games):
        _ns, nd = eng.export_dist(g)
        out[g] = mean_variance(nd[eng.export_game(g)["root"]], eng.cfg.dist_vmin, eng.cfg.dist_vmax)
    return out


def external_dist(atoms):
    """a device evaluator of mode dist: a softmax of the board cells, integer-exact inputs"""
    import torch

    def ev(boards):
        n = boards.shape[0]
        x = boards.reshape(n, 200)[:, :atoms] * 0.7 + torch.arange(atoms, device=boards.device, dtype=torch.float32) * 0.05
        return torch.softmax(x, dim=1).contiguous()
    return ev


@pytest.mark.parametrize("atoms,vmin,vmax,n", [(2, 0.0, 1000.0, 9), (33, 0.0, 45.0, 20), (50, 0.0, 5000.0, 33), (64, 0.0, 5000.0, 130)])
@pytest.mark.parametrize("kind", ["net_tc", "dist_fp16", "external"])
def test_root_values_are_the_twin_on_the_root_row(gpu_lib, atoms, vmin, vmax, n, kind):
    import torch
    from tetris_mcts_b200 import pyTetris as PT
    from tetris_mcts_b200.agents.DistValueSimOnline import init_dist_weights
    from tetris_mcts_b200.engine import BatchedEngine
    M = 600
    eng = BatchedEngine(n, max_nodes=M, mode="dist", eval_kind=kind, dist_weights=None if kind == "external" else init_dist_weights(0, atoms),
                        dist_bins=atoms, dist_vmin=vmin, dist_vmax=vmax, seed=11, overflow_reset=True)
    eng.set_games(PT.new_games(n, ENV, np.arange(40, 40 + n, dtype=np.uint32)))
    eng.set_gc_headroom(M * 5 // 32)
    ev = external_dist(atoms) if kind == "external" else None
    assert np.array_equal(eng.dist_root_values(), np.zeros((n, 2)))        # fresh roots: no backup yet, the twin's (0, 0)
    dev = torch.empty((n, 2), dtype=torch.float64, device="cuda:0")
    nonzero = 0
    for mv in range(8):
        eng.run_sims(30, evaluator=ev)
        got = eng.dist_root_values()
        want = twin_root_values(eng)
        assert np.array_equal(got.view(np.uint64), want.view(np.uint64)), (mv, np.argwhere(got != want)[:3])
        assert eng.dist_root_values(out=dev) is dev and np.array_equal(dev.cpu().numpy(), got)
        nonzero += int((got[:, 0] != 0).sum())
        eng.get_stats()
        eng.env_step(None)
        eng.update_root(True)
        if mv % 3 == 2:                                                     # the roots the re-rooting gave, before any search below them
            assert np.array_equal(eng.dist_root_values().view(np.uint64), twin_root_values(eng).view(np.uint64))
    assert nonzero > 0 and eng.counters()["gcs"] > 0, eng.counters()
    eng.close()


def test_root_values_refused_outside_mode_dist(gpu_lib):
    from tetris_mcts_b200 import _lib as L
    from tetris_mcts_b200.engine import BatchedEngine
    eng = BatchedEngine(4, max_nodes=256, mode="lp", eval_kind="synthetic")
    with pytest.raises(L.B200Error) as ei:
        eng.dist_root_values()
    assert ei.value.code == 1 and "B200_MODE_DIST" in str(ei.value)
    eng.close()


# ------------------------------------------------------------------ Model_Dist
def reference_checkpoint(path, w, atoms=50):
    """torch.save of model/model.py's layout: {'model_state_dict': Net's seq.* tensors, 'optimizer_state_dict'}, written here with torch"""
    import torch
    shapes = [("seq.conv1.weight", (32, 1, 4, 4)), ("seq.conv1.bias", (32,)), ("seq.conv2.weight", (32, 32, 4, 4)), ("seq.conv2.bias", (32,)),
              ("seq.fc1.weight", (128, 2048)), ("seq.fc1.bias", (128,)), ("seq.fc_v.weight", (atoms, 128)), ("seq.fc_v.bias", (atoms,))]
    sd, off = OrderedDict(), 0
    for name, shape in shapes:
        k = int(np.prod(shape))
        sd[name] = torch.tensor(w[off:off + k].reshape(shape))
        off += k
    assert off == w.size
    torch.save({"model_state_dict": sd, "optimizer_state_dict": {"state": {}, "param_groups": []}}, path)


@pytest.mark.parametrize("kind", ["net", "net_tc"])
def test_model_dist_loads_the_reference_checkpoint(gpu_lib, oracle, tmp_path, kind):
    import torch
    from tetris_mcts_b200.model.model_distributional import Model_Dist
    z = np.load(os.path.join(ROOT, "tests", "golden", "distnet_golden.npz"))
    w = oracle.seeded_dist_weights(int(z["seed"]))
    reference_checkpoint(str(tmp_path / "model_checkpoint"), w)
    m = Model_Dist(atoms=50, eval_kind=kind)
    m.load(str(tmp_path / "model_checkpoint"))
    assert np.array_equal(m.weights, w)
    boards = z["states"].reshape(-1, 1, 20, 10)
    out, = m.inference(boards)
    assert np.allclose(out, z["dist"], rtol=1e-5, atol=1e-7 if kind == "net" else 1e-6), np.abs(out - z["dist"]).max()
    padded = np.zeros((len(boards), 1, 22, 10), np.float32)
    padded[:, :, 2:] = boards
    assert np.array_equal(m.inference(padded)[0], out)
    padded[0, 0, 0, 0] = 1
    with pytest.raises(ValueError):
        m.inference(padded)
    m.save(str(tmp_path / "again"))
    ck = torch.load(str(tmp_path / "again"), weights_only=False)
    assert list(ck["model_state_dict"]) == list(torch.load(str(tmp_path / "model_checkpoint"), weights_only=False)["model_state_dict"])
    m2 = Model_Dist(atoms=50, eval_kind=kind)
    m2.load(str(tmp_path / "again"))
    assert np.array_equal(m2.weights.view(np.uint32), w.view(np.uint32))
    assert np.array_equal(m2.inference(boards)[0], out)
    with pytest.raises(NotImplementedError):
        m2.train(None)
    m.close(); m2.close()


def test_dist_value_sim_takes_a_state_dict_or_a_path(gpu_lib, oracle, tmp_path):
    from tetris_mcts_b200.agents.DistValueSimOnline import DistValueSim
    from tetris_mcts_b200.model.model_distributional import dist_weights_to_state_dict
    w = oracle.seeded_dist_weights(4)
    reference_checkpoint(str(tmp_path / "ck"), w)
    from arena_gen import boards
    b = boards(7, 3)
    outs = []
    for src in (w, dist_weights_to_state_dict(w), str(tmp_path / "ck")):
        a = DistValueSim(dist_weights=src, eval_kind="net")
        outs.append(a._eng.distnet(b))
        a._eng.close()
    assert np.array_equal(outs[0], outs[1]) and np.array_equal(outs[0], outs[2])


# ------------------------------------------------------------------ play_batched --agent_type DistValueSimOnline
def run_play(tmp, argv):
    """play_batched.run in directory tmp -> (stdout lines, saved rows or None)"""
    import glob
    from tetris_mcts_b200 import play_batched as PB
    cwd = os.getcwd()
    os.chdir(tmp)
    try:
        out = io.StringIO()
        PB.run(PB.parse_args(argv), out=out)
    finally:
        os.chdir(cwd)
    files = sorted(glob.glob(os.path.join(str(tmp), "data", "data0.*.npy")))
    return out.getvalue(), (np.concatenate([np.load(f) for f in files]) if files else None)


def episodes(text):
    return [ln for ln in text.splitlines() if ln.startswith("Episode:")]


N, M, SIMS, SEED = 24, 1024, 50, 123
BASE = ["--agent_type", "DistValueSimOnline", "--n_parallel", str(N), "--max_nodes", str(M), "--mcts_sims", str(SIMS), "--seed", str(SEED),
        "--endless", "--ngames", "100000"]


def test_play_batched_is_the_engine_and_the_oracle(gpu_lib, oracle, tmp_path):
    """play_batched's rows (boards, stats, policy, actions, value / variance) and Episode lines against a BatchedEngine driven move by move
    (run_sims, get_stats, the twin on export_dist's root row, env_step, update_root), and the first games' actions against the C oracle's
    distributional agent fed the engine's network outputs"""
    from tetris_mcts_b200 import pyTetris as PT
    from tetris_mcts_b200.agents.DistValueSimOnline import init_dist_weights
    from tetris_mcts_b200.data import rows_from_move
    from tetris_mcts_b200.engine import BatchedEngine
    moves = 90
    text, rows = run_play(tmp_path, BASE + ["--max_moves", str(moves), "--save"])
    assert "No distributional checkpoint" not in text                     # said on sys.stdout, not in the game log
    w = init_dist_weights(0, 50)
    eng = BatchedEngine(N, max_nodes=M, mode="dist", gamma=0.999, low=5, eval_kind="net_tc", dist_weights=w, seed=SEED, overflow_reset=True)
    eng.set_games(PT.new_games(N, ENV, np.arange(SEED, SEED + N, dtype=np.uint32)))
    eng.set_gc_headroom(M * 5 // 32)
    side = BatchedEngine(1, max_nodes=64, mode="dist", eval_kind="net_tc", dist_weights=w)
    sample = [0, 1, 2]
    agents = {g: oracle.Agent(max_nodes=M, mode=3, low=5, eval_mode=2, eval_cb=side.distnet, search_seed=search_seed(SEED, g), dist_bins=50,
                              dist_vmin=0.0, dist_vmax=5000.0, overflow_reset=1) for g in sample}
    games = {g: oracle.Game(record=eng.get_games()[g]) for g in sample}
    for g in sample:
        agents[g].update_root(games[g].record())
    episode_of, ngames, want_rows, want_eps = np.zeros(N, np.int32), 0, [], []
    for mv in range(moves):
        before = eng.get_games()
        eng.run_sims(SIMS)
        stats, actions = eng.get_stats()
        rv = twin_root_values(eng)
        eng.env_step(None)
        eng.update_root(True)
        want_rows.append(rows_from_move(before, actions, stats, 0, episode_of, rv[:, 0], rv[:, 1]))
        for g, score, lines, _ep in eng.finished_games():
            ngames += 1
            episode_of[g] = ngames
            want_eps.append("Episode: {:>5} Score: {:>10} Lines Cleared: {:>10}".format(ngames, int(score), int(lines)))
        for g in sample:
            agents[g].mcts(SIMS)
            a, st = agents[g].get_action()
            assert a == actions[g] and np.array_equal(st, stats[g]), (mv, g)
            games[g].play(a)
            agents[g].update_root(games[g].record())
            if games[g].end:
                games[g].reset()
                agents[g].update_root(games[g].record())
            if agents[g].n_free < M * 5 // 32:
                agents[g].remove_nodes()
    want = np.concatenate(want_rows)
    assert rows is not None and len(rows) == len(want) == N * moves
    for f in want.dtype.names:
        assert np.array_equal(rows[f], want[f]), f
    assert rows.tobytes() == want.tobytes()
    assert (rows["value"] != 0).all()
    assert episodes(text) == want_eps and len(want_eps) > 0, len(want_eps)
    assert eng.counters()["gcs"] > 0
    eng.close(); side.close()


def test_evaluator_plays_as_the_built_in_network(gpu_lib, tmp_path, monkeypatch):
    """--evaluator with a function returning a side engine's distnet outputs (eval_kind net) against --eval_kind net"""
    (tmp_path / "mod").mkdir()
    (tmp_path / "mod" / "side_dist.py").write_text(
        "import numpy as np, torch\n"
        "from tetris_mcts_b200.engine import BatchedEngine\n"
        "from tetris_mcts_b200.agents.DistValueSimOnline import init_dist_weights\n"
        "def make(device):\n"
        "    side = BatchedEngine(1, max_nodes=64, mode='dist', eval_kind='net', dist_weights=init_dist_weights(0, 50))\n"
        "    def ev(boards):\n"
        "        return [torch.from_numpy(side.distnet(boards.to(torch.int8).cpu().numpy())).to(boards.device)]\n"
        "    return ev\n")
    monkeypatch.syspath_prepend(str(tmp_path / "mod"))
    (tmp_path / "a").mkdir(); (tmp_path / "b").mkdir()
    args = BASE + ["--max_moves", "30", "--save"]
    ta, ra = run_play(tmp_path / "a", args + ["--eval_kind", "net"])
    tb, rb = run_play(tmp_path / "b", args + ["--evaluator", "side_dist:make"])
    assert ra.tobytes() == rb.tobytes() and episodes(ta) == episodes(tb)


def test_resume_is_the_uninterrupted_run(gpu_lib, tmp_path):
    """a run stopped at a checkpoint and resumed writes the rows, Episode lines and final games of the run that went on, with 64 games"""
    a, b = tmp_path / "a", tmp_path / "b"
    a.mkdir(); b.mkdir()
    base = ["--agent_type", "DistValueSimOnline", "--n_parallel", "64", "--max_nodes", "768", "--mcts_sims", "40", "--endless", "--ngames",
            "100000", "--save", "--eval_kind", "dist_fp16", "--atoms", "33", "--vmax", "1000"]
    import pickle
    from tetris_mcts_b200 import play_batched as PB
    ta, ra = run_play(a, base + ["--max_moves", "100"])
    tb1, _ = run_play(b, base + ["--max_moves", "51", "--checkpoint_dir", "ckpt", "--checkpoint_every", "20"])   # the last one at move 51
    tb2, rb = run_play(b, base + ["--max_moves", "100", "--checkpoint_dir", "ckpt", "--resume"])
    assert episodes(ta) == episodes(tb1) + episodes(tb2) and episodes(ta)
    assert ra is not None and ra.tobytes() == rb.tobytes()
    with open(PB.checkpoint_paths(str(b / "ckpt"), 100, 0)[1], "rb") as f:
        st = pickle.load(f)
    assert st["dist_weights"] == "init_dist_weights(0, 33)" and st["flags"]["atoms"] == 33
    with pytest.raises(ValueError, match="--atoms"):
        run_play(b, base[:-4] + ["--atoms", "50", "--vmax", "1000", "--max_moves", "110", "--checkpoint_dir", "ckpt", "--resume"])


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def test_two_ranks_gloo_finish_the_games_of_one(gpu_lib, tmp_path):
    """torchrun's layout by hand: two processes on one GPU (gloo) over 48 games finish the same games, numbered alike, as one process"""
    argv = ["--agent_type", "DistValueSimOnline", "--n_parallel", "48", "--max_nodes", "768", "--mcts_sims", "40", "--endless", "--ngames",
            "100000", "--max_moves", "80", "--dist_backend", "gloo"]

    def launch(d, world):
        d.mkdir()
        port, procs = _free_port(), []
        for r in range(world):
            env = {k: v for k, v in os.environ.items() if k not in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_PORT")}
            env["PYTHONPATH"] = ROOT + os.pathsep + env.get("PYTHONPATH", "")
            if world > 1:
                env.update(RANK=str(r), WORLD_SIZE=str(world), LOCAL_RANK="0", MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
            procs.append(subprocess.Popen([sys.executable, "-m", "tetris_mcts_b200.play_batched"] + argv, cwd=d, env=env,
                                          stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True))
        out = [p.communicate(timeout=900) for p in procs]
        for p, (so, se) in zip(procs, out):
            assert p.returncode == 0, se[-3000:]
        return out
    (so1, _), = launch(tmp_path / "w1", 1)
    (so2a, _), (so2b, _) = launch(tmp_path / "w2", 2)
    assert episodes(so1) == episodes(so2a) and len(episodes(so1)) > 0
    assert so2b.strip() == ""                                                 # rank 0 alone prints
