"""The caller's training function (OnlineMCTSAgent(..., train=), agents/cppmodule/agent.cpp:588-616,698-702) on the device: online.CallbackTrainer
under play_batched --trainer and ValueSim(train=).  The built-in loop rebuilt through the callback, the arrays it receives under every
accumulation policy, the caller's network trained in place (eval_kind external), returned weights loaded into the tensor-core networks,
a raising callback, and two ranks."""
import io
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

from ext_eval_twins import value_torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ARGS = ((20, 10), 1, 0, 0)
REC = {}                                       # what this module's evaluators and training functions saw (they run inside play_batched)


def _fixed_states(n=16):
    from tetris_mcts_b200 import pyTetris as PT
    return PT.states_of(PT.new_games(n, (1, 0, 0), np.arange(40, 40 + n, dtype=np.uint32)))


@pytest.fixture
def log(monkeypatch):
    """stderr of play_batched, the agents and the training loop"""
    from tetris_mcts_b200 import play_batched as PB
    from tetris_mcts_b200.agents import ValueSim as VS
    from tetris_mcts_b200.model import model_vv as MV
    buf = io.StringIO()
    for mod in (PB, VS, MV):
        monkeypatch.setattr(mod, "perr", dict(file=buf, flush=True))
    return buf


# ------------------------------------------------------------------ 1. the built-in loop, rebuilt through the callback
def rebuilt_builtin(device):
    """mode 2: the rows back into 212-byte rows (replay.memory_to_rows) and Model_VV.train_rows with play_batched's own arguments, seeded by
    this function's training count, as OnlineTrainer.train does; returns the trained weights as a state_dict"""
    import torch
    from tetris_mcts_b200 import replay
    from tetris_mcts_b200.model.model_vv import Model_VV, weights_to_state_dict
    m = Model_VV(device=device.index, seed=0, eval_kind="net", train_kind="fp64")         # play_batched's weights in a fresh directory: init_weights(0)
    REC.update(model=m, sizes=[])

    def train(state, value, variance, visit, size):
        assert all(isinstance(a, torch.Tensor) and a.device == device for a in (state, value, variance, visit))
        rows = torch.from_numpy(replay.memory_to_rows(*(a.cpu().numpy() for a in (state, value, variance, visit)))).to(device)
        torch.cuda.synchronize(device)
        assert m.train_rows(rows.data_ptr(), size, batch_size=256, iters_per_val=100, max_iters=200, seed=len(REC["sizes"]))
        REC["sizes"].append(size)
        return weights_to_state_dict(m.weights)
    return train


def _recorded_run(monkeypatch, argv, rec):
    from tetris_mcts_b200 import play_batched as PB
    from tetris_mcts_b200.engine import BatchedEngine
    states = _fixed_states()
    real_play = BatchedEngine.play_move

    class Recording(BatchedEngine):
        def play_move(self, *a, **k):
            actions, stats = real_play(self, *a, **k)
            rec.setdefault("actions", []).append(np.array(actions).copy())
            return actions, stats

        def close(self):
            if getattr(self, "h", None):
                rec["out"] = self.valuenet(states)
            super().close()
    monkeypatch.setattr(PB, "BatchedEngine", Recording)
    out, timing = io.StringIO(), {}
    PB.run(PB.parse_args(argv), out=out, timing=timing)
    rec["stdout"], rec["timing"] = out.getvalue(), timing
    return rec


def test_builtin_loop_rebuilt_through_the_callback(gpu_lib, tmp_path, monkeypatch, log):
    """mode 2 with the built-in training inside the callback reproduces play_batched --online bit for bit: every action, every Episode: line,
    the size of every training, the checkpoint and the search network's outputs at the end.  One game (the rows of one multi-game collection
    enter the memory in CTA order), policy 2 on a 60-row memory (every training has 60 rows: the built-in path never skips one)."""
    import torch
    from tetris_mcts_b200 import online as OL
    base = ["--agent_type", "ValueSimLP", "--mcts_sims", "64", "--ngames", "100000", "--n_parallel", "1", "--max_nodes", "1024", "--endless",
            "--online", "--max_moves", "220", "--memory_size", "60", "--accumulation_policy", "2", "--episodes_per_train", "100000"]
    (tmp_path / "builtin").mkdir(); (tmp_path / "callback").mkdir()
    monkeypatch.chdir(tmp_path / "builtin")
    sizes = []
    real_train = OL.OnlineTrainer.train

    def train(self, n_rows, current_episode, dump_path=None):
        ok = real_train(self, n_rows, current_episode, dump_path)
        sizes.append((n_rows, ok))
        return ok
    monkeypatch.setattr(OL.OnlineTrainer, "train", train)
    a = _recorded_run(monkeypatch, base + ["--train_max_iters", "200", "--train_batch_size", "256"], {})
    err_a = log.getvalue()
    log.seek(0); log.truncate()
    monkeypatch.chdir(tmp_path / "callback")
    b = _recorded_run(monkeypatch, base + ["--trainer", __name__ + ":rebuilt_builtin"], {})
    err_b = log.getvalue()
    REC.pop("model").close()
    assert all(ok for _n, ok in sizes) and len(sizes) >= 2, err_a[-2000:]
    assert [n for n, _ok in sizes] == REC["sizes"] and set(REC["sizes"]) == {60}
    assert a["timing"]["trainings"] == b["timing"]["trainings"] == len(sizes)
    assert len(a["actions"]) == len(b["actions"]) == 220 and all(np.array_equal(x, y) for x, y in zip(a["actions"], b["actions"]))
    eps = lambda s: [ln for ln in s.splitlines() if ln.startswith("Episode:")]     # noqa: E731
    assert eps(a["stdout"]) == eps(b["stdout"])
    mem = lambda s: [ln for ln in s.splitlines() if ln.startswith(("Memory usage", "Training data size", "Iteration:"))]   # noqa: E731
    assert mem(err_a) == mem(err_b)
    assert err_b.count("Training complete.") == len(sizes) and "Training complete." not in err_a
    ca = torch.load(tmp_path / "builtin" / "pytorch_model" / "model_checkpoint", weights_only=False)["model_state_dict"]
    cb = torch.load(tmp_path / "callback" / "pytorch_model" / "model_checkpoint", weights_only=False)["model_state_dict"]
    assert all(torch.equal(ca[k], cb[k]) for k in ca)
    for x, y in zip(a["out"], b["out"]):
        assert x.tobytes() == y.tobytes()


# ------------------------------------------------------------------ 2. contents and timing under accumulation policies 0-3
def _engine(kind="external", n=1, M=512, seed=2, weights=None):
    from tetris_mcts_b200 import pyTetris as PT
    from tetris_mcts_b200.engine import BatchedEngine
    e = BatchedEngine(n, max_nodes=M, mode="lp", eval_kind=kind, seed=seed, overflow_reset=True, weights=weights)
    e.set_games(PT.new_games(n, ARGS, np.arange(n, dtype=np.uint32) + 1))
    e.set_gc_headroom(M * 5 // 32)
    return e


@pytest.mark.parametrize("policy", [0, 1, 2, 3])
def test_arrays_and_timing_under_every_policy(gpu_lib, policy):
    """three twin engines searching with the board-exact torch evaluator: one trains through the device form, one through the host form, one
    by hand (replay_policy_trained alone).  Inside each callback its arrays equal rows_to_memory of a peek taken there, bit for bit, and
    size is the memory_index of replay_policy_step; after it the memory is empty, and the three engines take the same decisions with the same
    memory_index and memory bytes after every move (the policy counted the training as the hand-driven one did)."""
    import torch
    from tetris_mcts_b200 import replay
    from tetris_mcts_b200.online import CallbackTrainer
    cap = 100
    engines = [_engine() for _ in range(3)]
    peek = torch.empty((cap, 212), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    calls = {False: [], True: []}

    def recorder(eng, host):
        def train(state, value, variance, visit, size):
            eng.replay_peek_into(peek.data_ptr(), size)
            want = replay.rows_to_memory(peek[:size].cpu().numpy())
            for got, w in zip((state, value, variance, visit), want):
                if host:
                    assert isinstance(got, np.ndarray) and got.dtype == np.float32
                else:
                    assert isinstance(got, torch.Tensor) and got.dtype == torch.float32 and got.is_contiguous() and got.device == peek.device
                    got = got.cpu().numpy()
                assert got.shape == w.shape and got.tobytes() == w.tobytes()
            calls[host].append(size)
        return train
    trainers = [CallbackTrainer(engines[0], None, cap, recorder(engines[0], False), external=True),
                CallbackTrainer(engines[1], None, cap, recorder(engines[1], True), host=True, external=True)]
    for e in engines:
        e.replay_enable(min_visits=2, capacity=cap)
        e.replay_policy(policy, episodes_per_train=4, memory_growth_rate=40)
    sizes, hand = [], torch.empty((cap, 212), dtype=torch.uint8, device="cuda")
    for mv in range(170):
        episode = 0 if mv < 130 else (mv - 128) // 2               # the memory fills (policies 0 and 1 trim it) before episodes advance
        res = []
        for i, e in enumerate(engines):
            actions, _ = e.play_move(24, evaluator=value_torch)
            train, idx = e.replay_policy_step(episode)
            if train:
                if i < 2:
                    before = len(calls[i == 1])
                    assert trainers[i].train(idx, episode) is True
                    assert calls[i == 1][before:] == [idx]
                    assert e.replay_drain_into(hand.data_ptr(), cap) == 0              # empty (draining nothing changes nothing)
                else:
                    e.replay_policy_trained(episode)
                    sizes.append(idx)
            e.replay_peek_into(hand.data_ptr(), cap)
            res.append((actions.tolist(), train, idx, hand[:0 if train else idx].cpu().numpy().tobytes()))
        assert res[0] == res[1] == res[2], (policy, mv)
    assert calls[False] == calls[True] == sizes and len(sizes) >= 2, (policy, sizes)
    assert trainers[0].n_trains == len(sizes) and trainers[0].train_seconds > 0
    for t in trainers:
        t.close()
    for e in engines:
        e.close()


# ------------------------------------------------------------------ 3. mode 1 trains the searching network
def tiny_evaluator(device):
    import torch
    torch.manual_seed(0)
    net = torch.nn.Linear(200, 2).to(device)
    REC.update(net=net, pending=None, checked=0, trainings=0)

    def ev(boards):
        with torch.no_grad():
            out = net(boards.reshape(len(boards), 200))
            v, var = out[:, 0].contiguous(), torch.nn.functional.softplus(out[:, 1]).contiguous()
            if REC["pending"] is not None:                    # the first evaluation after a training: the trained module, not an older one
                frozen, old = REC["pending"]
                want, stale = frozen(boards.reshape(len(boards), 200)), old(boards.reshape(len(boards), 200))
                assert torch.equal(out, want) and not torch.equal(out, stale)
                REC["pending"] = None
                REC["checked"] += 1
        return v, var
    return ev


def tiny_trainer(device):
    import copy
    import torch

    def train(state, value, variance, visit, size):
        net = REC["net"]
        old = copy.deepcopy(net)
        opt = torch.optim.SGD(net.parameters(), lr=1e-4)
        x, y, w = state.reshape(size, 200), value[:, 0] / 100, visit[:, 0] / visit.mean()
        for _ in range(5):
            opt.zero_grad()
            loss = ((net(x)[:, 0] - y) ** 2 * w).mean()
            loss.backward()
            opt.step()
        REC["pending"] = (copy.deepcopy(net), old)
        REC["trainings"] += 1
    return train


def test_mode1_trains_the_searching_network(gpu_lib, tmp_path, monkeypatch, log):
    from tetris_mcts_b200 import play_batched as PB
    monkeypatch.chdir(tmp_path)
    argv = ["--agent_type", "ValueSimLP", "--mcts_sims", "64", "--ngames", "100000", "--n_parallel", "64", "--max_nodes", "512", "--endless",
            "--online", "--max_moves", "100", "--memory_size", "2000", "--memory_growth_rate", "150",
            "--evaluator", __name__ + ":tiny_evaluator", "--trainer", __name__ + ":tiny_trainer"]
    timing = {}
    PB.run(PB.parse_args(argv), out=io.StringIO(), timing=timing)
    err = log.getvalue()
    assert REC["trainings"] >= 1 and timing["trainings"] == REC["trainings"], err[-2000:]
    assert REC["checked"] >= 1 and REC["checked"] >= REC["trainings"] - 1
    assert err.count("Training complete.") == REC["trainings"] and "Iteration:" not in err
    assert not os.path.exists("pytorch_model")                   # the built-in trainer never ran


def _small_arena(monkeypatch, max_nodes):
    from tetris_mcts_b200.agents import agent as A
    orig = A.TreeAgent.__init__

    def init(self, *a, **k):
        k["max_nodes"] = max_nodes
        orig(self, *a, **k)
    monkeypatch.setattr(A.TreeAgent, "__init__", init)


def test_valuesimc_style_training_through_valuesimlp(gpu_lib, tmp_path, monkeypatch, log):
    """ValueSimC's pair: Model_VV.inference as the (host) evaluator and a training() that runs Model_VV.train_data with ValueSimC's
    arguments on the host arrays, through ValueSimLP(online=True, evaluator=, train=)"""
    from tetris_mcts_b200.agents.ValueSimLP import ValueSimLP
    from tetris_mcts_b200.model.model_vv import Model_VV
    from tetris_mcts_b200.pyTetris import Tetris
    _small_arena(monkeypatch, 8192)
    monkeypatch.chdir(tmp_path)
    model = Model_VV(seed=0)
    w0 = model.weights.copy()
    seen = []

    def training(state, value, variance, visit, d_size):
        assert all(isinstance(a, np.ndarray) and a.dtype == np.float32 and len(a) == d_size for a in (state, value, variance, visit))
        assert state.shape == (d_size, 1, 20, 10) and value.shape == variance.shape == visit.shape == (d_size, 1)
        seen.append(d_size)
        if d_size < 10:                                          # train_data's validation split needs ten rows
            return
        model.train_data([state, value, variance, visit], iters_per_val=100, batch_size=512, max_iters=300,
                         sample_replacement=True, oversampling=False)
        model.training(False)
    agent = ValueSimLP(online=True, evaluator=model.inference, train=training, sims=300, env=Tetris, env_args=ARGS, benchmark=False,
                       min_visit=40, memory_size=400, memory_growth_rate=40, overflow_reset=True)
    game = Tetris(*ARGS)
    agent.update_root(game)
    for _ in range(150):
        game.play(agent.play())
        if game.end:
            game.reset()
        agent.update_root(game)
        if any(s >= 10 for s in seen):
            break
    err = log.getvalue()
    assert any(s >= 10 for s in seen) and agent.n_trains == len(seen), err[-2000:]
    assert "Enough training data" in err and err.count("Training complete.") == len(seen) and "Training data size" in err
    assert os.path.isfile("data/dump.npz") and os.path.isfile("pytorch_model/model_checkpoint")
    assert not np.array_equal(model.weights, w0)
    states = _fixed_states()
    v, var = model.inference(states[:, None])                    # the agent's evaluator is the trained model
    assert np.isfinite(v).all() and np.isfinite(var).all()
    agent.close(); model.close()


# ------------------------------------------------------------------ 4. mode 2 weights into the tensor-core networks
def _memory_engine(kind, w0, rows):
    e = _engine(kind=kind, n=4, weights=w0)
    e.replay_enable(min_visits=1, capacity=len(rows))
    e.replay_policy(3, memory_growth_rate=1)                        # every fill of the memory trains
    return e


def _rows(n, seed):
    from tetris_mcts_b200 import replay
    rng = np.random.default_rng(seed)
    return replay.memory_to_rows(rng.integers(-1, 2, (n, 1, 20, 10)), rng.normal(50, 30, (n, 1)), rng.uniform(0, 900, (n, 1)),
                                 rng.integers(25, 5000, (n, 1)))


def _fill(e, rows):
    e.replay_append(rows)
    return e.replay_policy_step(0)


@pytest.mark.parametrize("kind", ["net_tc", "net_fp16"])
def test_mode2_weights_reach_the_search(gpu_lib, kind):
    import tetris_mcts_b200._lib as L
    from tetris_mcts_b200.engine import BatchedEngine
    from tetris_mcts_b200.model.model_vv import init_weights, weights_to_state_dict
    from tetris_mcts_b200.online import CallbackTrainer
    states = _fixed_states()
    rows = _rows(50, 1)
    w0 = init_weights(0)
    e = _memory_engine(kind, w0, rows)
    ret = []
    tr = CallbackTrainer(e, w0, len(rows), lambda *a: ret[-1])

    def fresh(w):
        f = BatchedEngine(1, max_nodes=64, eval_kind=kind, weights=w)
        out = f.valuenet(states)
        f.close()
        return out

    def same(a, b):
        return all(x.tobytes() == y.tobytes() for x, y in zip(a, b))
    for w, held in ((init_weights(5), 5), (weights_to_state_dict(init_weights(6)), 6), (None, 6)):
        assert _fill(e, rows) == (True, len(rows))
        ret.append(w)
        assert tr.train(len(rows), 0) is True
        assert _fill(e, rows[:0])[1] == 0                           # trained: the memory is empty
        assert same(e.valuenet(states), fresh(init_weights(held))), held
        assert not same(e.valuenet(states), fresh(w0))
        assert np.array_equal(tr.weights, init_weights(held))
    big = init_weights(7)
    big[0] = 2000.0                                                 # conv1: |w| * 64 > 65504
    sd = weights_to_state_dict(init_weights(8))
    del sd["out_ubound"]
    current = e.valuenet(states)
    for bad, exc in ((big, L.B200Error), (init_weights(8)[:-1], ValueError), (init_weights(8).astype(np.float64), ValueError), (sd, ValueError)):
        assert _fill(e, rows) == (True, len(rows))
        ret.append(bad)
        with pytest.raises(exc):
            tr.train(len(rows), 0)
        assert same(e.valuenet(states), current)
        assert e.replay_policy_step(0) == (True, len(rows))         # the memory was not marked trained
        e.replay_drain_into(tr.buf.data_ptr(), len(rows))
    assert tr.n_trains == 3 and np.array_equal(tr.weights, init_weights(6))
    tr.close(); e.close()


# ------------------------------------------------------------------ 5. a raising callback
def test_raising_callback_leaves_the_engine_usable(gpu_lib):
    import torch
    from tetris_mcts_b200.model.model_vv import init_weights
    from tetris_mcts_b200.online import CallbackTrainer
    w0 = init_weights(0)
    e = _engine(kind="net_tc", n=16, M=1024, weights=w0)
    e.replay_enable(min_visits=2, capacity=5000)
    e.replay_policy(3, memory_growth_rate=100000)
    mode = {"raise": True, "calls": 0}

    def train(state, value, variance, visit, size):
        mode["calls"] += 1
        if mode["raise"]:
            raise RuntimeError("caller's training failed")
    tr = CallbackTrainer(e, w0, 5000, train)
    buf = torch.empty((5000, 212), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    for _ in range(60):
        e.play_move(32)
        train_now, idx = e.replay_policy_step(0)
        if train_now and idx > 0:
            break
    assert train_now and idx > 0
    e.replay_peek_into(buf.data_ptr(), idx)
    rows = buf[:idx].cpu().numpy()
    with pytest.raises(RuntimeError, match="caller's training failed"):
        tr.train(idx, 0)
    assert tr.n_trains == 0 and mode["calls"] == 1
    assert e.replay_policy_step(0) == (True, idx)                  # untouched: same rows, the policy still says train (n_trains 0)
    e.replay_peek_into(buf.data_ptr(), idx)
    assert np.array_equal(buf[:idx].cpu().numpy(), rows)
    e.play_move(32)                                                # the next move and the next training proceed
    mode["raise"] = False
    train_now, idx2 = e.replay_policy_step(0)
    assert train_now and idx2 >= idx
    assert tr.train(idx2, 0) is True and tr.n_trains == 1
    assert e.replay_policy_step(0) == (False, 0)                   # trained: empty, and the threshold is n_trains * growth now
    tr.close(); e.close()
    # mode 1: a callback that returns weights is refused, and the memory stays as it was
    x = _engine()
    x.replay_enable(min_visits=2, capacity=500)
    x.replay_policy(3, memory_growth_rate=100000)
    tx = CallbackTrainer(x, None, 500, lambda *a: w0, external=True)
    for _ in range(80):
        x.play_move(24, evaluator=value_torch)
        train_now, idx = x.replay_policy_step(0)
        if train_now and idx > 0:
            break
    assert train_now and idx > 0
    with pytest.raises(ValueError, match="returns None"):
        tx.train(idx, 0)
    assert x.replay_policy_step(0) == (True, idx) and tx.n_trains == 0
    tx.close(); x.close()


# ------------------------------------------------------------------ 6. two ranks (gloo, one GPU)
def rank_trainer(device):
    """mode 2: records a digest of every array it receives and returns weights that differ by rank"""
    import hashlib
    from tetris_mcts_b200 import distributed as D
    from tetris_mcts_b200.model.model_vv import init_weights
    rank = D.rank_world()[0]
    REC.update(digests=[], sizes=[], returned=[])

    def train(state, value, variance, visit, size):
        h = hashlib.sha256()
        for a in (state, value, variance, visit):
            h.update(a.cpu().numpy().tobytes())
        REC["digests"].append(h.hexdigest())
        REC["sizes"].append(size)
        w = init_weights(1000 + 10 * len(REC["returned"]) + rank)
        REC["returned"].append(w)
        return w
    return train


RUN2 = ["--agent_type", "ValueSimLP", "--mcts_sims", "64", "--ngames", "100000", "--n_parallel", "2", "--max_nodes", "1024", "--endless",
        "--online", "--max_moves", "80", "--memory_size", "2000", "--memory_growth_rate", "100", "--dist_backend", "gloo",
        "--trainer", "test_gpu_train_callback:rank_trainer"]


def test_two_ranks_gloo(gpu_lib, tmp_path):
    from tetris_mcts_b200.engine import BatchedEngine
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    procs = []
    for r in range(2):
        env = {k: v for k, v in os.environ.items() if k not in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_PORT")}
        env["PYTHONPATH"] = os.pathsep.join([ROOT, os.path.dirname(os.path.abspath(__file__)), env.get("PYTHONPATH", "")])
        env.update(RANK=str(r), WORLD_SIZE="2", LOCAL_RANK="0", MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        procs.append(subprocess.Popen([sys.executable, os.path.abspath(__file__), "worker", str(tmp_path)] + RUN2, cwd=tmp_path, env=env,
                                      stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True))
    out = [p.communicate(timeout=1500) for p in procs]
    for p, (so, se) in zip(procs, out):
        assert p.returncode == 0, se[-3000:]
    r0, r1 = (np.load(tmp_path / ("rank%d.npz" % r)) for r in range(2))
    assert len(r0["digests"]) >= 1 and list(r0["digests"]) == list(r1["digests"]) and list(r0["sizes"]) == list(r1["sizes"])
    assert out[0][1].count("Training complete.") == len(r0["digests"]) and "Training complete." not in out[1][1]   # rank 0 alone prints
    assert not np.array_equal(r0["last"], r1["last"])               # the ranks' callbacks returned different weights ...
    assert r0["out"].tobytes() == r1["out"].tobytes()               # ... and both searches hold rank 0's
    f = BatchedEngine(1, max_nodes=64, eval_kind="net_tc", weights=r0["last"])
    want = np.stack(f.valuenet(_fixed_states()))
    f.close()
    assert r0["out"].tobytes() == want.tobytes()


def _worker(out_dir, argv):
    sys.path.insert(0, ROOT)
    import importlib
    from tetris_mcts_b200 import distributed as D
    from tetris_mcts_b200 import play_batched as PB
    states = _fixed_states()
    seen = {}
    real_close = PB.BatchedEngine.close

    def close(self):
        if getattr(self, "h", None) and self.max_nodes == 1024:
            seen["out"] = np.stack(self.valuenet(states))
        real_close(self)
    PB.BatchedEngine.close = close
    PB.main(argv)
    rec = importlib.import_module("test_gpu_train_callback").REC
    np.savez(os.path.join(out_dir, "rank%d.npz" % D.env_world()[0]), digests=np.array(rec["digests"]), sizes=np.array(rec["sizes"]),
             last=rec["returned"][-1], out=seen["out"])


if __name__ == "__main__" and len(sys.argv) > 2 and sys.argv[1] == "worker":
    _worker(sys.argv[2], sys.argv[3:])
