"""play_batched --train_lag on the device: a pipelined run (training on its own thread while the search plays on) against a single-threaded
twin written here, which trains synchronously at the same moves, holds the weights and loads them after move s + L; and a run checkpointed
with a training in flight, then resumed, against the uninterrupted run.  Compared bit for bit: every move's actions, the final games, the
finished-games log, the counters, the memory rows of every training, the weights and Yogi state after every training and the install moves."""
import io

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
# one game: with several, the rows of one collection enter the memory in the order the k_gc CTAs reach its counter (DESIGN §4c), so no two
# runs train on the same rows.  A 256-slot arena collects every move or two; memory growth 0 makes every collection a training point, which
# starts a training once 10 rows are there (about every 15 moves) and otherwise installs the one in flight early (lag 3).
N, SIMS, NODES, MOVES = 1, 50, 256, 150
FLAGS = ["--agent_type", "ValueSimLP", "--mcts_sims", str(SIMS), "--ngames", "100000", "--n_parallel", str(N), "--max_nodes", str(NODES),
         "--endless", "--online", "--memory_size", "3000", "--memory_growth_rate", "0", "--train_max_iters", "100", "--train_batch_size", "128"]


class Rec:
    """what one run did, recorded by the engine and the trainer"""

    def __init__(self):
        self.actions, self.installs, self.rows, self.trained, self.starts, self.points, self.end = [], [], [], [], [], [], None


@pytest.fixture
def recorder(monkeypatch, gpu_lib):
    import torch
    from tetris_mcts_b200 import play_batched as PB
    from tetris_mcts_b200.engine import BatchedEngine
    from tetris_mcts_b200.model import model_vv as MV
    box = {}

    class Recording(BatchedEngine):
        def play_move(self, *a, **k):
            actions, stats = super().play_move(*a, **k)
            box["rec"].actions.append(actions.copy())
            return actions, stats

        def load_weights(self, w):
            super().load_weights(w)
            if self.n_games == N and self.max_nodes == NODES:      # the search engine, not Model_VV's validation engine
                box["rec"].installs.append((len(box["rec"].actions), np.array(w, np.float32)))

        def replay_peek_into(self, ptr, n):
            super().replay_peek_into(ptr, n)
            rows = torch.empty((max(n, 1), 212), dtype=torch.uint8, device="cuda")
            super().replay_peek_into(rows.data_ptr(), n)
            box["rec"].rows.append((len(box["rec"].actions), rows[:n].cpu().numpy()))

        def replay_policy_step(self, ep):
            train_now, n = super().replay_policy_step(ep)
            if train_now:
                box["rec"].points.append(len(box["rec"].actions))
            return train_now, n

        def replay_policy_trained(self, ep):
            super().replay_policy_trained(ep)
            box["rec"].starts.append(len(box["rec"].actions))

        def close(self):
            if getattr(self, "h", None) and self.max_nodes == NODES:
                box["rec"].end = (self.get_games(), self.counters())
            super().close()

    orig = MV.Model_VV.train_rows

    def train_rows(self, *a, **k):
        ok = orig(self, *a, **k)
        m, v, step = self._trainer.state()
        box["rec"].trained.append((self.weights.copy(), m, v, step))
        return ok
    monkeypatch.setattr(PB, "BatchedEngine", Recording)
    monkeypatch.setattr(MV.Model_VV, "train_rows", train_rows)
    monkeypatch.setattr(PB, "perr", dict(file=io.StringIO(), flush=True))
    monkeypatch.setattr(MV, "perr", dict(file=io.StringIO(), flush=True))

    def record(rec):
        box["rec"] = rec
        return rec
    return record, Recording


def pipelined(record, path, monkeypatch, kind, lag, extra=()):
    from tetris_mcts_b200 import play_batched as PB
    monkeypatch.chdir(path)
    rec, out = record(Rec()), io.StringIO()
    timing = {}
    PB.run(PB.parse_args(FLAGS + ["--train_kind", kind, "--train_lag", str(lag), "--max_moves", str(MOVES)] + list(extra)), out=out, timing=timing)
    rec.log, rec.timing = out.getvalue(), timing
    return rec


def serial_twin(record, Recording, path, monkeypatch, kind, lag):
    """play_batched's loop for one process, written out with the training on this thread: train at the policy's moves, hold the weights,
    load them after move s + lag (or at the next training point, if that comes first)"""
    import torch
    from tetris_mcts_b200 import distributed as D
    from tetris_mcts_b200 import play_batched as PB
    from tetris_mcts_b200 import pyTetris as PT
    from tetris_mcts_b200.model.model_vv import Model_VV, init_weights, rows_validation_size
    monkeypatch.chdir(path)
    rec, out = record(Rec()), io.StringIO()
    args = PB.parse_args(FLAGS + ["--train_kind", kind])
    env_args = ((20, 10), args.app, args.tetris_scoring, args.tetris_randomizer)
    w = init_weights(0)
    eng = Recording(N, max_nodes=NODES, mode="lp", gamma=0.999, low=1, eval_kind="net_tc", weights=w, env_args=env_args,
                    seed=args.seed & 0xFFFFFFFF, device=0, overflow_reset=True)
    eng.set_games(PT.new_games(N, env_args, D.shard_seeds(args.seed, N, 0, 1)))
    eng.set_gc_headroom(NODES * 5 // 32)
    eng.replay_enable(min_visits=25, capacity=args.memory_size)
    eng.replay_policy(args.accumulation_policy, episodes_per_train=args.episodes_per_train, memory_growth_rate=args.memory_growth_rate)
    buf = torch.empty((args.memory_size, 212), dtype=torch.uint8, device="cuda")
    model = Model_VV(device=0, eval_kind="net", train_kind=kind)
    model.weights = w
    model._eng.load_weights(w)
    kw = dict(batch_size=args.train_batch_size, iters_per_val=100, max_iters=args.train_max_iters, checkpoint="pytorch_model/model_checkpoint")
    ngames, gcs, n_trains, held = 0, 0, 0, None
    for move in range(1, MOVES + 1):
        eng.play_move(SIMS, auto_reset=True, want_stats=False)
        collected = eng.counters()["gcs"] != gcs
        gcs = eng.counters()["gcs"]
        for _g, score, lines, _ep in eng.finished_games():
            ngames += 1
            out.write(PB.EPISODE_FMT.format(ngames, int(score), int(lines)) + "\n")
        if collected:
            train_now, n = eng.replay_policy_step(ngames)
            if train_now:
                if held is not None:
                    eng.load_weights(held[1])
                    held = None
                eng.replay_peek_into(buf.data_ptr(), n)
                if rows_validation_size(n) > 0:
                    eng.replay_policy_trained(ngames)
                    model.train_rows(buf.data_ptr(), n, seed=n_trains, **kw)
                    n_trains += 1
                    held = (move + lag, model.weights.copy())
        if held is not None and move >= held[0]:
            eng.load_weights(held[1])
            held = None
    eng.close()
    model.close()
    rec.log = out.getvalue()
    return rec


def assert_same(a, b):
    assert len(a.actions) == len(b.actions) == MOVES
    for m, (x, y) in enumerate(zip(a.actions, b.actions)):
        assert np.array_equal(x, y), "actions differ at move %d" % (m + 1)
    assert np.array_equal(a.end[0], b.end[0]) and a.end[1] == b.end[1]
    ep = lambda s: [ln for ln in s.splitlines() if ln.startswith("Episode:")]       # noqa: E731
    assert ep(a.log) == ep(b.log)
    assert [m for m, _r in a.rows] == [m for m, _r in b.rows]
    assert all(x.tobytes() == y.tobytes() for (_m, x), (_n, y) in zip(a.rows, b.rows))
    assert len(a.trained) == len(b.trained) >= 2
    for (wa, ma, va, sa), (wb, mb, vb, sb) in zip(a.trained, b.trained):
        assert np.array_equal(wa, wb) and np.array_equal(ma, mb) and np.array_equal(va, vb) and sa == sb
    assert a.starts == b.starts and a.points == b.points and [m for m, _w in a.installs] == [m for m, _w in b.installs]
    assert all(np.array_equal(x, y) for (_m, x), (_n, y) in zip(a.installs, b.installs))


@pytest.mark.parametrize("kind", ["fp64", "tf32"])
@pytest.mark.parametrize("lag", [0, 1, 3])
def test_pipelined_run_is_the_serial_twin(recorder, tmp_path, monkeypatch, kind, lag):
    record, Recording = recorder
    (tmp_path / "p").mkdir(); (tmp_path / "s").mkdir()
    a = pipelined(record, tmp_path / "p", monkeypatch, kind, lag)
    b = serial_twin(record, Recording, tmp_path / "s", monkeypatch, kind, lag)
    print("lag %d %s: trainings start %s, installs %s, timing %s" % (lag, kind, b.starts, [m for m, _w in b.installs], a.timing))
    assert_same(a, b)
    assert a.timing["trainings"] == len(b.trained) and a.timing["wait_s"] <= a.timing["total_s"]
    installs = [m for m, _w in a.installs[1:]]                      # installs[0]: the weights the engine was created with
    forced = [s for s in a.starts if [p for p in a.points if s < p < s + lag]]
    on_time = [s for s in a.starts if s + lag in installs and not [p for p in a.points if s < p < s + lag]]
    if lag == 3:                                                    # a training point inside the lag installs the training in flight
        assert forced and all(min(p for p in a.points if p > s) in installs for s in forced)
    if lag == 1:                                                    # no training point can come inside a lag of 1: each goes in after move s + 1
        assert on_time == [s for s in a.starts if s < MOVES]


def test_resume_with_a_training_in_flight(recorder, tmp_path, monkeypatch):
    """checkpointed one move after a training started, with no training point at that move (lag 3: still in flight), resumed: the
    uninterrupted run, install moves included"""
    import pickle
    from tetris_mcts_b200 import play_batched as PB
    record, _ = recorder
    for d in ("a", "b"):
        (tmp_path / d).mkdir()
    a = pipelined(record, tmp_path / "a", monkeypatch, "tf32", 3)
    k = next(s for s in a.starts if s + 1 not in a.points and s + 3 < MOVES) + 1
    b1 = pipelined(record, tmp_path / "b", monkeypatch, "tf32", 3, ["--max_moves", str(k), "--checkpoint_dir", "ckpt"])
    with open(PB.checkpoint_paths(str(tmp_path / "b" / "ckpt"), k, 0)[1], "rb") as f:
        pending = pickle.load(f)["trainer"]["pending"]
    assert pending is not None and pending["move"] == k + 2
    b2 = pipelined(record, tmp_path / "b", monkeypatch, "tf32", 3, ["--checkpoint_dir", "ckpt", "--resume"])
    assert len(b1.actions) == k and len(b2.actions) == MOVES - k
    assert [x.tobytes() for x in a.actions] == [x.tobytes() for x in b1.actions + b2.actions]
    assert np.array_equal(a.end[0], b2.end[0]) and a.end[1] == b2.end[1]
    ep = lambda s: [ln for ln in s.splitlines() if ln.startswith("Episode:")]       # noqa: E731
    assert ep(a.log) == ep(b1.log) + ep(b2.log)
    assert [m for m, _w in a.installs[1:]] == [m for m, _w in b1.installs[1:]] + [k + m for m, _w in b2.installs[1:]]
    assert all(np.array_equal(x, y) for (_m, x), (_n, y) in zip(a.installs[1:], b1.installs[1:] + b2.installs[1:]))
    assert [r.tobytes() for _m, r in a.rows] == [r.tobytes() for _m, r in b1.rows + b2.rows]
    for (wa, ma, va, sa), (wb, mb, vb, sb) in zip(a.trained, b1.trained + b2.trained):
        assert np.array_equal(wa, wb) and np.array_equal(ma, mb) and np.array_equal(va, vb) and sa == sb
    assert len(a.trained) == len(b1.trained) + len(b2.trained)
