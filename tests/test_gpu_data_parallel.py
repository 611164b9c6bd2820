"""Data-parallel online training on the device: the slice gradient and the ordered apply of the trainer (b200_trainer_grad_rows_dev /
_apply_grads_dev), the device append to the replay memory (b200_replay_append_dev), and play_batched --online as two processes (gloo on one
GPU; NCCL when two GPUs are visible) against a single-process run.

Run as a script (`python test_gpu_data_parallel.py worker OUT ARGS...`) this file is one rank of such a run; the tests start it."""
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def golden_rows():
    from tetris_mcts_b200 import replay
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", "train_golden.npz"))
    visit = np.round(z["weight"] * 100).astype(np.float32)
    return z, replay.memory_to_rows(z["states"], z["value"], z["variance"], visit), visit


def to_device(a):
    import torch
    d = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    torch.cuda.synchronize()
    return d


def trainers(n, kind, max_batch, z):
    from tetris_mcts_b200.model.model_vv import init_weights
    from tetris_mcts_b200.model.trainer import Trainer
    out = []
    for _ in range(n):
        t = Trainer(init_weights(3), max_batch=max_batch, kind=kind)
        t.set_out_ubound(*z["ubound"])
        out.append(t)
    return out


def dp_step(ts, dev, n_train, batch, seed, it, scale, weighted, clip, parts):
    """one emulated data-parallel step: trainer r computes slice r, every trainer applies all parts"""
    import torch
    from tetris_mcts_b200 import distributed as D
    R = len(ts)
    for r, t in enumerate(ts):
        lo, hi = D.batch_slice(batch, r, R)
        t.grad_rows_dev(dev.data_ptr(), n_train, batch, lo, hi, seed, it, scale, parts[r].data_ptr(), weighted=weighted)
    for t in ts:
        t.read_log(0)                                            # every slice is written before any trainer reads the parts
    for t in ts:
        t.apply_grads_dev(parts.data_ptr(), R, clip, it)
    torch.cuda.synchronize()


def tensor_slices():
    from tetris_mcts_b200.model.model_vv import WEIGHT_KEYS
    off, out = 0, []
    for name, shape in WEIGHT_KEYS[:10]:
        n = int(np.prod(shape))
        out.append((name, slice(off, off + n)))
        off += n
    return out


# ------------------------------------------------------------------------------------------------ world 1 is the existing step
@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["fp64", "tc"])
@pytest.mark.parametrize("weighted,clip,batch", [(True, 0.0, 64), (False, 0.5, 64), (True, 0.05, 2049), (False, 0.0, 2048)])
def test_world1_slice_is_train_rows_dev(gpu_lib, kind, weighted, clip, batch):
    """grad_rows_dev(0, batch) + apply_grads_dev(n_parts=1) == train_rows_dev, step by step: weights, gradients, Yogi state and gradient norm
    bit for bit; the loss up to reassociation.  2048 / 2049 rows straddle the tc kind's 2048-k chunk of fc1's weight gradient."""
    import torch
    from tetris_mcts_b200.model.trainer import GRAD_VEC
    z, rows, visit = golden_rows()
    dev = to_device(rows)
    n_train, seed, steps = 86, 777, 30
    scale = float(len(rows) / visit.astype(np.float64).sum())
    a, b = trainers(2, kind, batch, z)
    part = torch.empty((1, GRAD_VEC), dtype=torch.float64, device="cuda")
    for it in range(steps):
        ref = a.train_rows_dev(dev.data_ptr(), n_train, batch, 1, seed, it, scale, weighted=weighted, grad_clip=clip)[0]
        b.grad_rows_dev(dev.data_ptr(), n_train, batch, 0, batch, seed, it, scale, part.data_ptr(), weighted=weighted)
        b.apply_grads_dev(part.data_ptr(), 1, clip, it)
        got = b.read_log(it + 1)[it]
        assert got[2] == ref[2], (it, got, ref)
        assert got[0] == pytest.approx(ref[0], rel=1e-12) and got[1] == pytest.approx(ref[1], rel=1e-9)
        assert np.array_equal(a.grads(), b.grads()), it
    assert np.array_equal(a.weights(), b.weights())
    (ma, va, sa), (mb, vb, sb) = a.state(), b.state()
    assert sa == sb == steps and np.array_equal(ma, mb) and np.array_equal(va, vb)
    if clip > 0:
        assert b.read_log(steps)[:, 2].max() > clip, "clipping was not exercised"
    a.close(); b.close()


# ------------------------------------------------------------------------------------------------ the ordered sum
def _ordered(parts):
    s = parts[0].copy()
    for p in parts[1:]:
        s = s + p
    return s.astype(np.float32)


@pytest.mark.gpu
def test_grad_reduce_is_the_ordered_sum(gpu_lib):
    """k_grad_reduce == numpy's left-to-right fp64 sum in ascending part order, rounded once, bit for bit, on parts of wide dynamic range with
    cancellations; every summation order other than swapping the first two parts gives other bits.  The loss moments join as Chan's formula."""
    import itertools
    import torch
    from tetris_mcts_b200.model.trainer import GRAD_VEC, N_TRAIN
    z, _rows, _v = golden_rows()
    (t,) = trainers(1, "fp64", 64, z)
    rng = np.random.default_rng(5)
    for R in (1, 2, 3, 5, 8):
        p = rng.standard_normal((R, N_TRAIN)) * 10.0 ** rng.integers(-30, 17, size=(R, N_TRAIN))
        if R == 3:                                               # (p0 + p1) + p2 = 0 in both; p0 + p2 first gives 1 in the first, p1 + p2 in the second
            p[:, 0] = [1e16, 1.0, -1e16]
            p[:, 1] = [1.0, -1e16, 1e16]
        full = np.zeros((R, GRAD_VEC))
        full[:, :N_TRAIN] = p
        cnt, mean, m2 = rng.integers(1, 400, R).astype(float), rng.standard_normal(R) * 3, rng.random(R) * 50
        full[:, N_TRAIN:] = np.stack([cnt, mean, m2], 1)
        dev = to_device(full)
        t.apply_grads_dev(dev.data_ptr(), R, 0.0, 0)
        log = t.read_log(1)[0]
        want = _ordered(p)
        got = t.grads()
        assert np.array_equal(got.view(np.int32), want.view(np.int32)), R
        n, m, q = cnt[0], mean[0], m2[0]
        for r in range(1, R):
            d, nn = mean[r] - m, n + cnt[r]
            m, q, n = m + d * cnt[r] / nn, q + m2[r] + d * d * n * cnt[r] / nn, nn
        assert log[0] == m and log[1] == np.sqrt(q / n)
        if R == 3:
            assert want[0] == 0.0 and want[1] == 0.0
            for perm in itertools.permutations(range(R)):
                if set(perm[:2]) != {0, 1}:
                    other = _ordered(p[list(perm)])
                    assert not np.array_equal(other[:2].view(np.int32), want[:2].view(np.int32)), perm
    t.close()


# ------------------------------------------------------------------------------------------------ emulated ranks in one process
@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["fp64", "tc"])
@pytest.mark.parametrize("R,batch", [(2, 64), (3, 1000), (8, 8)])
def test_emulated_ranks(gpu_lib, kind, R, batch):
    """R trainers from the same weights, each computing its slice and all applying the same R parts, stay bit-identical over 50 steps; one
    step's gradient is world 1's within 2 ulp (fp64) / 1e-5 of each tensor's norm (tc), and 50 steps' weights within 1e-5 of each norm."""
    import torch
    from tetris_mcts_b200.model.trainer import GRAD_VEC
    z, rows, visit = golden_rows()
    dev = to_device(rows)
    n_train, seed, steps = 86, 4242, 50
    scale = float(len(rows) / visit.astype(np.float64).sum())
    ts = trainers(R, kind, batch, z)
    (ref,) = trainers(1, kind, batch, z)
    parts = torch.empty((R, GRAD_VEC), dtype=torch.float64, device="cuda")
    for it in range(steps):
        dp_step(ts, dev, n_train, batch, seed, it, scale, True, 0.0, parts)
        ref.train_rows_dev(dev.data_ptr(), n_train, batch, 1, seed, it, scale, weighted=True)
        if it == 0:
            g, gr = ts[0].grads(), ref.grads()
            if kind == "fp64":
                tol = 2 * np.spacing(np.maximum(np.abs(g), np.abs(gr)))
                bad = np.flatnonzero(np.abs(g.astype(np.float64) - gr) > tol)
                assert bad.size == 0, (bad[:5], g[bad[:5]], gr[bad[:5]])
            else:
                for name, sl in tensor_slices():
                    assert np.linalg.norm(g[sl] - gr[sl]) <= 1e-5 * np.linalg.norm(gr[sl]), name
    w0, s0 = ts[0].weights(), ts[0].state()
    for t in ts[1:]:
        s = t.state()
        assert np.array_equal(t.weights(), w0) and np.array_equal(s[0], s0[0]) and np.array_equal(s[1], s0[1]) and s[2] == s0[2] == steps
    wr = ref.weights()
    for name, sl in tensor_slices():
        assert np.linalg.norm(w0[sl].astype(np.float64) - wr[sl]) <= 1e-5 * np.linalg.norm(wr[sl]), name
    for t in ts + [ref]:
        t.close()


# ------------------------------------------------------------------------------------------------ argument checks
@pytest.mark.gpu
def test_bad_arguments_leave_the_weights(gpu_lib):
    import torch
    from tetris_mcts_b200 import _lib as L
    from tetris_mcts_b200.model.trainer import GRAD_VEC
    z, rows, _v = golden_rows()
    dev = to_device(rows)
    (t,) = trainers(1, "fp64", 64, z)
    w0 = t.weights()
    part = torch.zeros((2, GRAD_VEC), dtype=torch.float64, device="cuda")
    for batch, lo, hi in [(64, -1, 10), (64, 10, 10), (64, 20, 10), (64, 0, 65), (200, 0, 65), (200, 100, 200), (0, 0, 0)]:
        with pytest.raises(L.B200Error) as e:
            t.grad_rows_dev(dev.data_ptr(), 86, batch, lo, hi, 1, 0, 1.0, part.data_ptr())
        assert e.value.code == 1, (batch, lo, hi)
    with pytest.raises(L.B200Error) as e:
        t.grad_rows_dev(dev.data_ptr(), 0, 64, 0, 64, 1, 0, 1.0, part.data_ptr())
    assert e.value.code == 1
    for n_parts, slot in [(0, 0), (-1, 0), (1, -1)]:
        with pytest.raises(L.B200Error) as e:
            t.apply_grads_dev(part.data_ptr(), n_parts, 0.0, slot)
        assert e.value.code == 1
    with pytest.raises(L.B200Error):
        t.read_log(10 ** 6)
    assert np.array_equal(t.weights(), w0) and t.state()[2] == -1
    t.close()


# ------------------------------------------------------------------------------------------------ b200_replay_append_dev
@pytest.mark.gpu
@pytest.mark.parametrize("policy", [3, 0])
def test_replay_append_dev_equals_append(gpu_lib, policy):
    """the device append stores what the host append stores: bytes and count, truncated at capacity (policy 0: at its staging area)"""
    import torch
    from tetris_mcts_b200.engine import BatchedEngine
    _z, rows, _v = golden_rows()
    rows = np.concatenate([rows, rows[::-1]])[:150]
    engs = [BatchedEngine(4, max_nodes=64, eval_kind="synthetic") for _ in range(2)]
    for e in engs:
        e.replay_enable(min_visits=25, capacity=50)
        e.replay_policy(policy)
    dev = to_device(rows)
    for lo, hi in [(0, 30), (30, 30), (30, 70), (70, 150)]:
        engs[0].replay_append(rows[lo:hi])
        engs[1].replay_append_dev(dev.data_ptr() + lo * 212, hi - lo)
    outs = []
    for e in engs:
        buf = torch.zeros((100, 212), dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        n = e.replay_drain_into(buf.data_ptr(), 100)
        outs.append((n, buf.cpu().numpy()))
        e.close()
    assert outs[0][0] == outs[1][0] == (100 if policy == 0 else 50)
    assert np.array_equal(outs[0][1], outs[1][1]) and np.array_equal(outs[0][1][:outs[0][0]], rows[:outs[0][0]])


# ------------------------------------------------------------------------------------------------ play_batched --online over ranks
RUN = ["--agent_type", "ValueSimLP", "--mcts_sims", "64", "--ngames", "100000", "--n_parallel", "64", "--max_nodes", "1024", "--endless",
       "--online", "--max_moves", "120", "--train_max_iters", "200", "--train_batch_size", "256", "--memory_size", "2000",
       "--memory_growth_rate", "150"]


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _launch(tmp, world, backend, local_ranks):
    """play_batched RUN as `world` processes (world 1: no process group) in directory tmp -> [(returncode, stdout, stderr)], one per rank"""
    port = _free_port()
    procs = []
    for r in range(world):
        env = {k: v for k, v in os.environ.items() if k not in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_PORT")}
        env["PYTHONPATH"] = ROOT + os.pathsep + env.get("PYTHONPATH", "")
        if world > 1:
            env.update(RANK=str(r), WORLD_SIZE=str(world), LOCAL_RANK=str(local_ranks[r]), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        cmd = [sys.executable, os.path.abspath(__file__), "worker", str(tmp)] + RUN + ["--dist_backend", backend]
        procs.append(subprocess.Popen(cmd, cwd=tmp, env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True))
    out = []
    for p in procs:
        so, se = p.communicate(timeout=1500)
        out.append((p.returncode, so, se))
    return out


def _load(tmp, rank):
    z = np.load(os.path.join(tmp, "rank%d.npz" % rank), allow_pickle=True)
    return {k: z[k] for k in z.files}


def _check_world2(tmp, res):
    for rc, so, se in res:
        assert rc == 0, se[-3000:]
    r0, r1 = _load(tmp, 0), _load(tmp, 1)
    assert int(r0["n_trains"]) >= 2 and int(r0["n_trains"]) == int(r1["n_trains"])
    for k in range(int(r0["n_trains"])):                                   # after every training: the same bits on both ranks
        for key in ("w", "m", "v", "step"):
            assert np.array_equal(r0["%s%d" % (key, k)], r1["%s%d" % (key, k)]), (key, k)
    assert int(r0["saves"]) >= 1 and int(r1["saves"]) == 0              # rank 0 alone writes the checkpoint
    return r0, r1


def _episodes(stdout):
    return [int(ln.split()[1]) for ln in stdout.splitlines() if ln.startswith("Episode:")]


@pytest.mark.gpu
def test_play_batched_two_ranks_gloo(gpu_lib, tmp_path):
    """two processes on one GPU (gloo) against one process over the same 64 games: the same actions and memory (as a multiset of rows) up
    to the first training, bit-identical weights and optimiser state on both ranks after every training, rank 0 alone printing, the
    episodes of both ranks numbered 1..n, and a clean exit."""
    d1, d2 = tmp_path / "w1", tmp_path / "w2"
    d1.mkdir(); d2.mkdir()
    (rc, so1, se1), = _launch(d1, 1, "gloo", [0])
    assert rc == 0, se1[-3000:]
    res = _launch(d2, 2, "gloo", [0, 0])
    r0, r1 = _check_world2(d2, res)
    w1 = _load(d1, 0)
    first = int(w1["first_train_move"])
    assert first == int(r0["first_train_move"]) == int(r1["first_train_move"]) and first > 0
    a1, a2 = w1["actions"][:first], np.concatenate([r0["actions"], r1["actions"]], axis=1)[:first]
    assert a1.shape == a2.shape and np.array_equal(a1, a2)
    assert np.array_equal(w1["rows0"], r0["rows0"])                    # rows sorted bytewise: the same multiset
    eps = _episodes(res[0][1])
    assert eps == list(range(1, len(eps) + 1)) and len(eps) == int(r0["finished"]) + int(r1["finished"]) > 0
    assert res[1][1] == "" and "Memory usage" not in res[1][2] and "Iteration:" not in res[1][2]
    assert "Iteration:" in res[0][2] and "Memory usage" in res[0][2]
    e1 = _episodes(so1)                                                 # the games finished before the first training are numbered alike
    n_same = int(w1["finished_by_first"])
    assert n_same == int(r0["finished_by_first"]) + int(r1["finished_by_first"])
    assert [ln for ln in so1.splitlines() if ln.startswith("Episode:")][:n_same] == \
        [ln for ln in res[0][1].splitlines() if ln.startswith("Episode:")][:n_same] and e1[:n_same] == eps[:n_same]
    assert os.path.isfile(d2 / "pytorch_model" / "model_checkpoint")


@pytest.mark.gpu
def test_play_batched_two_ranks_nccl(gpu_lib, tmp_path):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("NCCL needs two GPUs (one per rank)")
    res = _launch(tmp_path, 2, "nccl", [0, 1])
    _check_world2(tmp_path, res)


def _worker(out_dir, argv):
    """one rank of RUN, recording what the tests compare into out_dir/rank{r}.npz"""
    sys.path.insert(0, ROOT)
    from tetris_mcts_b200 import distributed as D
    from tetris_mcts_b200 import online as OL
    from tetris_mcts_b200 import play_batched as PB
    from tetris_mcts_b200.model import model_vv as MV
    rec = dict(actions=[], finished=0, finished_by_first=None, first_train_move=None, n_trains=0, saves=0, moves=0)
    real_play, real_fin, real_train, real_save = PB.BatchedEngine.play_move, PB.BatchedEngine.finished_games, OL.OnlineTrainer.train, MV.Model_VV.save

    def play_move(self, *a, **k):
        actions, stats = real_play(self, *a, **k)
        if self.n_games > 1:
            rec["actions"].append(np.array(actions, np.int32).copy())
            rec["moves"] += 1
        return actions, stats

    def finished_games(self):
        f = real_fin(self)
        if self.n_games > 1:
            rec["finished"] += len(f)
        return f

    def train(self, n_rows, current_episode, dump_path=None):
        ok = real_train(self, n_rows, current_episode, dump_path)
        if ok:
            k = rec["n_trains"]
            if k == 0:
                rec["first_train_move"], rec["finished_by_first"] = rec["moves"], rec["finished"]
            if k == 0 and D.rank_world()[0] == 0:
                r = self.buf[:n_rows].cpu().numpy()
                rec["rows0"] = r[np.lexsort(r.T[::-1])]
            t = self.model._trainer
            m, v, step = t.state()
            rec.update({"w%d" % k: t.weights(), "m%d" % k: m, "v%d" % k: v, "step%d" % k: np.array(step)})
            rec["n_trains"] += 1
        return ok

    def save(self, *a, **k):
        rec["saves"] += 1
        return real_save(self, *a, **k)

    PB.BatchedEngine.play_move, PB.BatchedEngine.finished_games, OL.OnlineTrainer.train, MV.Model_VV.save = play_move, finished_games, train, save
    PB.main(argv)
    rank = D.env_world()[0]
    rec["actions"] = np.stack(rec["actions"])
    np.savez(os.path.join(out_dir, "rank%d.npz" % rank), **{k: np.asarray(v) for k, v in rec.items() if v is not None})


if __name__ == "__main__" and len(sys.argv) > 2 and sys.argv[1] == "worker":
    _worker(sys.argv[2], sys.argv[3:])
