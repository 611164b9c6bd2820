"""play_batched --train_lag: the start / install schedule of the pipelined online trainer, its pending state across state() / restore(),
and the refused flag combinations.  A fake engine and a fake Model_VV stand in for the device; no device needed."""
import contextlib
import io
import random
import time
import types

import numpy as np
import pytest


class FakeEngine:
    """What play_batched.run and OnlineTrainer ask of a BatchedEngine.  One collection per move; the policy says train at `points`."""
    points = ()
    cfg = types.SimpleNamespace(device=0)

    def __init__(self, *a, **k):
        self.moves, self.events, self.trained = 0, [], 0

    def set_games(self, recs):
        pass

    def set_gc_headroom(self, n):
        pass

    def set_stream(self, s):
        pass

    def replay_enable(self, **k):
        pass

    def replay_policy(self, *a, **k):
        pass

    def play_move(self, sims, **k):
        self.moves += 1
        return np.zeros(1, np.int32), None

    def counters(self):
        return {"gcs": self.moves}

    def finished_games(self):
        return []

    def replay_policy_step(self, ngames):
        return self.moves in self.points, 20 + self.moves

    def replay_peek_into(self, ptr, n):
        pass

    def replay_policy_trained(self, ep):
        self.events.append(("start", self.moves))

    def load_weights(self, w):
        self.events.append(("install", self.moves, int(w[0])))

    def close(self):
        pass


class FakeTrainer:
    def __init__(self):
        self.w, self.state_ = np.zeros(4, np.float32), (np.zeros(2, np.float32), np.zeros(2, np.float32), 0)

    def set_stream(self, s):
        pass

    def set_weights(self, w):
        self.w = np.array(w)

    def state(self):
        return self.state_

    def set_state(self, m, v, step):
        self.state_ = (m, v, step)


class FakeModel:
    """Model_VV: train_rows takes a random while and leaves weights [seed + 1, ...] and Yogi step seed + 1"""

    def __init__(self, **k):
        self.weights, self._dp, self._trainer, self._eng = None, None, FakeTrainer(), types.SimpleNamespace(load_weights=lambda w: None)

    def _trainer_obj(self):
        return self._trainer

    def train_rows(self, ptr, n, seed, **kw):
        time.sleep(random.random() * 0.02)
        self.weights = np.full(4, seed + 1, np.float32)
        self._trainer.w = self.weights
        self._trainer.state_ = (np.full(2, seed, np.float32), np.full(2, -seed, np.float32), seed + 1)
        return True

    def close(self):
        pass


@pytest.fixture
def fakes(monkeypatch):
    import torch
    from tetris_mcts_b200 import online
    from tetris_mcts_b200 import play_batched as PB
    from tetris_mcts_b200.model import model_vv as MV

    class CpuTrainer(online.OnlineTrainer):
        """OnlineTrainer with its row buffer on the host and no streams"""

        def _row_buffer(self, capacity):
            return torch.empty((capacity, 212), dtype=torch.uint8)

        def _search_on_own_stream(self):
            pass

        def _stream(self):
            return types.SimpleNamespace(cuda_stream=0)

    monkeypatch.setattr(torch.cuda, "device", lambda *a: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "stream", lambda *a: contextlib.nullcontext())
    monkeypatch.setattr(MV, "Model_VV", FakeModel)
    monkeypatch.setattr(MV, "perr", dict(file=io.StringIO()))
    monkeypatch.setattr(online, "OnlineTrainer", CpuTrainer)
    monkeypatch.setattr(PB, "BatchedEngine", FakeEngine)
    monkeypatch.setattr(PB.PT, "new_games", lambda n, env_args, seeds: np.zeros((n, 20), np.uint32))
    monkeypatch.setattr(PB, "perr", dict(file=io.StringIO()))
    return CpuTrainer


def expected(points, lag, moves):
    """the schedule of the issue: start after move s, install after move s + lag; a training point within the lag installs first"""
    ev, pending, n = [], None, 0
    for m in range(1, moves + 1):
        if m in points:
            if pending is not None:
                ev.append(("install", m, pending[1]))
            ev.append(("start", m))
            n += 1
            pending = (m + lag, n)
        if pending is not None and m >= pending[0]:
            ev.append(("install", m, pending[1]))
            pending = None
    return ev, n


@pytest.mark.parametrize("lag,points", [
    (0, (3, 4, 9)),
    (1, (3, 4, 9)),             # 4 is inside the lag of 3: its start installs 3's weights first
    (3, (2, 4, 5, 12, 19)),     # 19: the run ends with a training in flight
    (5, (1, 2, 3)),
    (2, ()),
])
def test_schedule(fakes, monkeypatch, lag, points):
    from tetris_mcts_b200 import play_batched as PB
    seen = {}
    monkeypatch.setattr(FakeEngine, "points", points)
    monkeypatch.setattr(FakeEngine, "close", lambda self: seen.setdefault("events", self.events))
    timing = {}
    args = PB.parse_args(["--online", "--max_moves", "20", "--ngames", "999", "--n_parallel", "4", "--train_lag", str(lag)])
    PB.run(args, out=io.StringIO(), timing=timing)
    ev, n = expected(points, lag, 20)
    assert seen["events"] == ev
    assert timing["trainings"] == n and timing["moves"] == 20
    assert timing["search_s"] == pytest.approx(timing["total_s"] - timing["wait_s"])


def test_pending_state_round_trip(fakes):
    eng = FakeEngine()
    t = fakes(eng, np.zeros(4, np.float32), 64, train_lag=3)
    eng.moves = 7
    assert t.start(40, 5, move=7) and not t.due(9) and t.due(10)
    st = t.state()                                      # joins the training in flight; the search keeps its weights
    assert st["n_trains"] == 1 and st["weights"][0] == 0
    assert st["pending"]["move"] == 10 and st["pending"]["weights"][0] == 1 and st["optimizer"][2] == 1
    assert ("install", 7, 1) not in eng.events
    eng2 = FakeEngine()
    r = fakes(eng2, None, 64, train_lag=3)
    r.restore(st)
    assert eng2.events == [("install", 0, 0)]           # the search's weights, as the image holds them
    assert r.model._trainer.w[0] == 1 and r.model._trainer.state_[2] == 1     # the trainer goes on from the finished training
    assert not r.due(9) and r.due(10)
    eng2.moves = 10
    assert r.install() and eng2.events[-1] == ("install", 10, 1) and r.weights[0] == 1
    assert r.state()["pending"] is None and not r.install()
    # the next training draws with seed n_trains, as the uninterrupted trainer would
    assert r.start(40, 6, move=11)
    r.install()
    assert r.weights[0] == 2 and r.n_trains == 2


def test_too_few_rows_start_nothing(fakes):
    eng = FakeEngine()
    t = fakes(eng, np.zeros(4, np.float32), 64, train_lag=2)
    assert not t.start(9, 0, move=1)
    assert t._pending is None and t.n_trains == 0 and eng.events == []
    t.after_move(4)
    assert t.train(10, 0) and eng.events == [("start", 0)] and t._pending["move"] == 6      # train_lag 2 after the last completed move
    assert not t.train(9, 0) and eng.events[-1] == ("install", 0, 1)                        # a training point installs the one in flight
    eng = FakeEngine()
    t = fakes(eng, np.zeros(4, np.float32), 64, train_lag=0)
    assert t.train(10, 0) and eng.events == [("start", 0), ("install", 0, 1)] and t._pending is None


def test_start_refuses_a_second_training_in_flight(fakes):
    t = fakes(FakeEngine(), np.zeros(4, np.float32), 64, train_lag=2)
    t.start(20, 0, move=1)
    with pytest.raises(RuntimeError, match="install"):
        t.start(20, 0, move=2)
    t.close()


def test_training_error_is_raised_at_install(fakes, monkeypatch):
    def boom(self, *a, **k):
        raise ValueError("boom")
    monkeypatch.setattr(FakeModel, "train_rows", boom)
    t = fakes(FakeEngine(), np.zeros(4, np.float32), 64, train_lag=2)
    t.start(20, 0, move=1)
    with pytest.raises(ValueError, match="boom"):
        t.install()
    assert t._pending is None


def _error(capsys, argv):
    from tetris_mcts_b200 import play_batched as PB
    with pytest.raises(SystemExit):
        PB.parse_args(argv)
    return capsys.readouterr().err


@pytest.mark.parametrize("argv,msg", [
    (["--online", "--train_lag", "-1"], "--train_lag takes a number of moves >= 0"),
    (["--train_lag", "2"], "--train_lag needs --online"),
    (["--online", "--train_lag", "1", "--trainer", "m:f"], "--train_lag > 0 cannot be combined with --trainer"),
    (["--online", "--train_lag", "1", "--trainer", "m:f", "--evaluator", "m:e"], "--train_lag > 0 cannot be combined with --evaluator"),
])
def test_refusals(capsys, argv, msg):
    assert msg in _error(capsys, argv)


def test_refused_above_one_rank(capsys, monkeypatch):
    monkeypatch.setenv("WORLD_SIZE", "2")
    assert "--train_lag > 0 cannot run with a world size above 1" in _error(capsys, ["--online", "--train_lag", "1"])
    monkeypatch.setenv("WORLD_SIZE", "1")
    from tetris_mcts_b200 import play_batched as PB
    assert PB.parse_args(["--online", "--train_lag", "1"]).train_lag == 1


def test_flag_defaults_and_resume():
    from tetris_mcts_b200 import play_batched as PB
    assert PB.parse_args([]).train_lag == 0 and "train_lag" in PB.RESUME_FLAGS
    assert PB.parse_args(["--online", "--train_lag", "0", "--trainer", "m:f"]).train_lag == 0
