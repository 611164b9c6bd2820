"""The online self-play loop on the device: training from the device replay memory (b200_trainer_train_rows_dev, _loss_rows_dev,
b200_rows_stats_dev, Model_VV.train_rows) and the agents that train on their own after collections (ValueSim / ValueSimLP online=True,
play_batched --online), as the reference's remove_nodes -> train_nodes / OnlineMCTSAgent::remove_nodes do (agents/ValueSim.py:101-185,
agents/cppmodule/agent.cpp:619-708)."""
import os
import re

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "train_golden.npz")
TRAIN_RE = (r'Iteration:\s*(?P<iter>\d*)\s*training loss:\s*(?P<t_loss>\d*\.\d*)\s*validation loss:\s*(?P<v_loss>\d*\.\d*)±\s*'
            r'(?P<v_loss_err>\d*\.\d*|nan)\s*gradient norm:\s*(?P<g_norm>\d*\.\d*)')                          # web/parseLog.py:61-64
DATASIZE_RE = r'Training data size:\s*(?P<tsize>\d*)\s*Validation data size:\s*(?P<vsize>\d*)'            # web/parseLog.py:65-66
QUEUE_RE = r'Memory usage: (?P<filled>\d*) / (?P<size>\d*).*'                                               # web/parseLog.py:67
ENV_ARGS = ((20, 10), 1, 0, 0)


@pytest.fixture
def log(monkeypatch):
    """stderr of the training loop, the agents and play_batched (their lines go to the stream bound at import, as the reference's perr)"""
    import io
    from tetris_mcts_b200 import play_batched as PB
    from tetris_mcts_b200.agents import ValueSim as VS
    from tetris_mcts_b200.model import model_vv as MV
    buf = io.StringIO()
    for mod in (PB, VS, MV):
        monkeypatch.setattr(mod, "perr", dict(file=buf, flush=True))
    return buf


def take(buf):
    s = buf.getvalue()
    buf.seek(0); buf.truncate()
    return s


def golden_rows():
    from tetris_mcts_b200 import replay
    z = np.load(GOLD)
    visit = np.round(z["weight"] * 100).astype(np.float32)
    return z, replay.memory_to_rows(z["states"], z["value"], z["variance"], visit), visit


def to_device(rows):
    import torch
    d = torch.from_numpy(np.ascontiguousarray(rows)).cuda()
    torch.cuda.synchronize()
    return d


@pytest.mark.parametrize("weighted,clip", [(True, 0.0), (False, 0.0), (True, 0.5), (False, 0.05)])
def test_train_rows_dev_is_bit_identical_to_step_rows_dev(gpu_lib, weighted, clip):
    """K device-sampled steps == K step_rows_dev calls fed the numpy restatement of the sampler: per-step log, weights, Yogi state."""
    from tetris_mcts_b200.model.model_vv import init_weights
    from tetris_mcts_b200.model.trainer import Trainer, sample_indices
    z, rows, visit = golden_rows()
    dev = to_device(rows)
    n_train, batch, iters, seed, first = 86, 64, 6, 12345, 200
    scale = float(len(rows) / visit.astype(np.float64).sum())
    a, b = Trainer(init_weights(3), max_batch=128), Trainer(init_weights(3), max_batch=128)
    for t in (a, b):
        t.set_out_ubound(*z["ubound"])
    log = a.train_rows_dev(dev.data_ptr(), n_train, batch, iters, seed, first, scale, weighted=weighted, grad_clip=clip)
    ref = []
    for it in range(iters):
        idx = sample_indices(seed, first + it, batch, n_train)
        assert idx.min() >= 0 and idx.max() < n_train
        r = b.step_rows_dev(dev.data_ptr(), len(rows), idx, scale, weighted=weighted, grad_clip=clip)
        ref.append([r["loss"], r["loss_std"], r["grad_norm"]])
    ref = np.array(ref)
    assert np.array_equal(log, ref), (log, ref)
    if clip > 0:
        assert (ref[:, 2] > clip).any(), "clipping was not exercised"
    assert np.array_equal(a.weights(), b.weights())
    (ma, va, sa), (mb, vb, sb) = a.state(), b.state()
    assert sa == sb == iters and np.array_equal(ma, mb) and np.array_equal(va, vb)
    # a second call continues the same optimiser state (Yogi step counter on the host)
    log2 = a.train_rows_dev(dev.data_ptr(), n_train, batch, 2, seed, first + iters, scale, weighted=weighted, grad_clip=clip)
    for it in range(2):
        r = b.step_rows_dev(dev.data_ptr(), len(rows), sample_indices(seed, first + iters + it, batch, n_train), scale, weighted=weighted, grad_clip=clip)
        assert list(log2[it]) == [r["loss"], r["loss_std"], r["grad_norm"]]
    assert np.array_equal(a.weights(), b.weights())
    a.close(); b.close()


def test_validation_loss_on_device_rows(gpu_lib, tmp_path):
    """loss_rows_dev == Trainer.loss on the same host batch exactly; the chunked validation figure of train_rows == compute_loss on host
    arrays of the same split (up to the float32 sum numpy takes of each chunk's weights)."""
    from tetris_mcts_b200.model.model_vv import Model_VV, init_weights
    from tetris_mcts_b200.model.trainer import Trainer
    z, rows, visit = golden_rows()
    dev = to_device(rows)
    scale = float(len(rows) / visit.astype(np.float64).sum())
    w = (visit * np.float32(scale)).astype(np.float32)
    t = Trainer(init_weights(1), max_batch=128)
    t.set_out_ubound(*z["ubound"])
    for weighted in (True, False):
        first, n = 17, 50
        mean, std, wsum = t.loss_rows_dev(dev.data_ptr(), first, n, scale, weighted=weighted)
        hm, hs = t.loss([z["states"][first:first + n], z["value"][first:first + n], z["variance"][first:first + n], w[first:first + n]], weighted=weighted)
        assert (mean, std) == (hm, hs)
        assert abs(wsum - w[first:first + n].astype(np.float64).sum()) <= 1e-12 * wsum
    t.close()
    m = Model_VV(seed=1)
    m._trainer_obj().set_out_ubound(*z["ubound"])
    n_train = len(rows) - int(len(rows) * 0.1)
    got = m._loss_rows(dev.data_ptr(), n_train, len(rows), scale, chunksize=4)
    want = m.compute_loss([z["states"][n_train:], z["value"][n_train:], z["variance"][n_train:], w[n_train:]], weighted=True, chunksize=4)
    assert abs(got["loss"] - want["loss"]) <= 1e-6 * abs(want["loss"]) and abs(got["loss_std"] - want["loss_std"]) <= 1e-6 * abs(want["loss_std"])
    m.close()


def test_row_statistics(gpu_lib):
    from tetris_mcts_b200.model.model_vv import init_weights
    from tetris_mcts_b200.model.trainer import Trainer
    from tetris_mcts_b200 import replay
    rng = np.random.default_rng(5)
    n = 123457
    rows = replay.memory_to_rows(rng.integers(-1, 2, (n, 20, 10)), rng.normal(50, 30, n), rng.uniform(0, 900, n), rng.integers(25, 5000, n))
    dev = to_device(rows)
    t = Trainer(init_weights(0), max_batch=16)
    for k in (1, 1000, n):
        mv, mvar, vsum = t.rows_stats(dev.data_ptr(), k)
        f = np.ascontiguousarray(rows[:k, 200:212]).view(np.float32).reshape(k, 3)
        assert mv == f[:, 0].max() and mvar == f[:, 1].max()
        assert abs(vsum - f[:, 2].astype(np.float64).sum()) <= 1e-13 * vsum
    t.close()


def test_train_rows_loop(gpu_lib, tmp_path, monkeypatch, log):
    """Model_VV.train_rows: the reference's log lines, the checkpoint of the best model re-loaded and published, options outside what its
    callers use refused, and too few rows skipped with the reference's 'Not enough training data' line."""
    import torch
    from tetris_mcts_b200.model.model_vv import Model_VV
    monkeypatch.chdir(tmp_path)
    z, rows, visit = golden_rows()
    dev = to_device(rows)
    m = Model_VV(seed=2)
    assert m.train_rows(dev.data_ptr(), 9, batch_size=32, iters_per_val=10, max_iters=30) is False
    assert "Not enough training data" in take(log) and not os.path.exists("pytorch_model")
    with pytest.raises(ValueError):
        m.train_rows(dev.data_ptr(), len(rows), shuffle=True)
    assert m.train_rows(dev.data_ptr(), len(rows), batch_size=32, iters_per_val=10, max_iters=60, seed=4) is True
    err = take(log)
    ds = re.search(DATASIZE_RE, err)
    assert ds and (int(ds.group("tsize")), int(ds.group("vsize"))) == (87, 9)
    assert len(re.findall(TRAIN_RE, err)) >= 1
    ck = torch.load("pytorch_model/model_checkpoint", map_location="cpu", weights_only=False)
    m2 = Model_VV(seed=7)
    m2.load("pytorch_model/model_checkpoint")
    assert np.array_equal(m2.weights, m.weights) and ck["optimizer_state_dict"]["state"][0]["step"] % 10 == 0
    s = z["states"][:16]
    assert np.array_equal(np.concatenate(m.inference(s), 1), np.concatenate(m2.inference(s), 1))
    # out_ubound of the trained model = [max value, max variance] of the rows (model_vv.py:227-231)
    f = np.ascontiguousarray(rows[:, 200:212]).view(np.float32).reshape(-1, 3)
    assert m.weights[-4] == f[:, 0].max() and m.weights[-3] == f[:, 1].max()
    m.close(); m2.close()


def _small_arena(monkeypatch, max_nodes):
    from tetris_mcts_b200.agents import agent as A
    orig = A.TreeAgent.__init__

    def init(self, *a, **k):
        k["max_nodes"] = max_nodes
        orig(self, *a, **k)
    monkeypatch.setattr(A.TreeAgent, "__init__", init)


def _play(agent, moves, stop=None):
    from tetris_mcts_b200.pyTetris import Tetris
    game = Tetris(*ENV_ARGS)
    agent.update_root(game)
    for _ in range(moves):
        game.play(agent.play())
        if game.end:
            game.reset()
        agent.update_root(game)
        if stop and stop():
            break


def test_valuesimlp_online_trains_on_its_own(gpu_lib, tmp_path, monkeypatch, log):
    from tetris_mcts_b200.agents.ValueSimLP import ValueSimLP
    from tetris_mcts_b200.model.model_vv import Model_VV
    from tetris_mcts_b200.pyTetris import Tetris
    _small_arena(monkeypatch, 8192)
    kw = dict(sims=300, env=Tetris, env_args=ENV_ARGS, benchmark=False, min_visit=40, memory_size=400, memory_growth_rate=40, overflow_reset=True)
    (tmp_path / "on").mkdir(); (tmp_path / "off").mkdir()
    monkeypatch.chdir(tmp_path / "on")
    agent = ValueSimLP(online=True, **kw)
    agent._online.kw["max_iters"] = 300                         # bounds the test's training time (the agent's own default is 50000)
    _play(agent, 120, stop=lambda: agent.n_trains >= 2)
    err = take(log)
    assert agent.n_trains >= 2, err[-2000:]
    assert "Enough training data" in err and "Training complete." in err and len(re.findall(TRAIN_RE, err)) >= 2
    assert os.path.isfile("data/dump.npz") and os.path.isfile("pytorch_model/model_checkpoint")
    d = np.load("data/dump.npz")
    assert set(d.files) == {"states", "values", "variance", "weights"} and (d["weights"] >= 25).all()
    m = Model_VV(seed=9, eval_kind="net_tc")                    # the agent's evaluator (TreeAgent default)
    m.load("pytorch_model/model_checkpoint")
    states = d["states"][:32, 0]
    v, var = agent._eng.valuenet(states)
    mv, mvar = m.inference(states[:, None])
    assert np.allclose(v, mv[:, 0], rtol=1e-5, atol=1e-5) and np.allclose(var, mvar[:, 0], rtol=1e-5, atol=1e-5)
    memory = agent.train_nodes()                                # by hand: None while the memory is below the next threshold
    assert memory is None or len(memory) == 4
    agent.close(); m.close()
    # the same agent offline never trains
    monkeypatch.chdir(tmp_path / "off")
    off = ValueSimLP(online=False, **kw)
    _play(off, 40)
    assert off.model is None and off.train_nodes() is None and off.n_trains == 0
    assert not os.path.exists("pytorch_model") and not os.path.exists("data")
    off.close()


def test_play_batched_online_end_to_end(gpu_lib, tmp_path, monkeypatch, log):
    import io
    from tetris_mcts_b200 import play_batched as PB
    from tetris_mcts_b200 import pyTetris as PT
    from tetris_mcts_b200.engine import BatchedEngine
    from tetris_mcts_b200.model.model_vv import Model_VV
    monkeypatch.chdir(tmp_path)
    states = PT.states_of(PT.new_games(16, (1, 0, 0), np.arange(40, 56, dtype=np.uint32)))
    seen = {}

    class Recording(BatchedEngine):                             # the outputs of the search engine's network when the run ends
        def close(self):
            if getattr(self, "h", None) and self.n_games == 64:
                seen["out"] = self.valuenet(states)
            super().close()
    monkeypatch.setattr(PB, "BatchedEngine", Recording)
    base = ["--agent_type", "ValueSimLP", "--mcts_sims", "64", "--ngames", "64", "--n_parallel", "64", "--max_nodes", "1024", "--endless",
            "--online", "--max_moves", "160", "--train_max_iters", "200", "--train_batch_size", "256"]
    timing = {}
    PB.run(PB.parse_args(base + ["--memory_size", "2000", "--memory_growth_rate", "150"]), out=io.StringIO(), timing=timing)
    err = take(log)
    usage = [m for m in (re.search(QUEUE_RE, ln) for ln in err.splitlines() if ln.startswith("Memory usage")) if m]
    assert usage and all(int(m.group("size")) == 2000 and int(m.group("filled")) <= 2000 for m in usage)
    assert timing["trainings"] >= 2, err[-2000:]
    assert len(re.findall(DATASIZE_RE, err)) >= 2 and len(re.findall(TRAIN_RE, err)) >= 2
    assert timing["train_s"] > 0 and timing["search_s"] > 0
    m = Model_VV(seed=9, eval_kind="net_tc")                    # play_batched's evaluator
    m.load("pytorch_model/model_checkpoint")
    v, var = m.inference(states[:, None])
    assert np.allclose(seen["out"][0], v[:, 0], rtol=1e-5, atol=1e-5) and np.allclose(seen["out"][1], var[:, 0], rtol=1e-5, atol=1e-5)
    m.close()
    # accumulation policy 1 (episodes): a small memory fills and is trimmed (weighted_trimming) while too few games have finished
    os.remove("pytorch_model/model_checkpoint")
    PB.run(PB.parse_args(base + ["--memory_size", "100", "--accumulation_policy", "1", "--episodes_per_train", "100000", "--max_moves", "80"]),
           out=io.StringIO(), timing=timing)
    err = take(log)
    filled = [int(m.group("filled")) for m in (re.search(QUEUE_RE, ln) for ln in err.splitlines()) if m]
    assert filled and max(filled) <= 100 and max(filled) >= 50 and timing["trainings"] == 0
    assert not os.path.exists("pytorch_model/model_checkpoint")
