"""The tensor-core trainer kind (Trainer(kind="tc"), B200_TRAIN_TC: k_gemm_tc in tetris_mcts_b200/csrc/trainer.cu) against the reference's
goldens, against float64 autograd (tests/f64_ref.py) and against the fp64 kind, plus its exactness within the kind and the online loop
running on it.

Error analysis of the 3xTF32 split (trainer.cu header).  Each fp32 operand x is stored as big + small, two tf32 terms: |x - big - small|
<= 2^-22 |x| down to fp32's subnormal floor (tf32 has fp32's exponent range, so no family leaves the normal range that fp32 itself holds).
A product carries <= 3 * 2^-22 |a b| (two residuals and the dropped small * small).  The tensor core sums one 32-k tile (its fp32
accumulation truncates: <= 4e-6 of the tile's |terms|), tile sums are added with round-to-nearest fp32 adds over <= 2048 k (<= 4e-6
worst case, ~5e-7 typical) and chunks of 2048 k as fp64 partials, so the error does not grow with the batch.  Every GEMM output is thus
within ~1e-6 (typical) of its |term| sum, and the loss, the gradient norm and each
gradient tensor (its L2 norm, which is at least of the order of the |term| sums of its largest elements) are held to 1e-5 — the bound
the fp64 kind meets — on every weight family; no family needs an allowance on top of it."""
import os

import numpy as np
import pytest

import f64_ref as R

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "train_golden.npz")
TG_BM, TG_KCHUNK = 64, 2048                 # k_gemm_tc's output tile rows and fp32 chain cap (trainer.cu)
PIXELS = (144, 96, 56)                      # conv1 / conv2 / conv3 output pixels per board: the GEMMs' M (forward) and K (weight gradient)


def edge_batches():
    """batch sizes at which a conv GEMM's M = B * pixels first fills whole 64-row tiles (and one past it), and at which a weight
    gradient's K = B * pixels (conv) or B (fc1) crosses the 2048-term chunk edge"""
    out = set()
    for p in PIXELS:
        b = TG_BM // np.gcd(TG_BM, p)
        out.update((b, b + 1))
        b = TG_KCHUNK // p
        out.update((b, b + 1))
    out.update((TG_KCHUNK, TG_KCHUNK + 1))
    return sorted(out)


BATCHES = sorted(set([1, 2, 63, 64, 65, 127, 128, 129, 1024, 4096] + edge_batches()))


def training_set(oracle, n=4096, seed=9):
    """positions of random-play games with targets in the thousands, clamped variances at rows 0..49 and zero weights at rows 50..79"""
    s = R.real_positions(n, seed, oracle)
    rng = np.random.default_rng(seed)
    filled = (s > 0).sum(axis=(1, 2)).astype(np.float32)
    value = (80.0 * filled + rng.uniform(0, 400, n)).astype(np.float32)
    variance = (filled ** 2 * 20.0 + rng.uniform(0, 50, n)).astype(np.float32)
    variance[:50] = 0.05
    visits = rng.integers(0, 300, n).astype(np.float32)
    visits[50:80] = 0
    return s, value, variance, visits


@pytest.fixture(scope="module")
def tset(oracle):
    return training_set(oracle)


@pytest.fixture(scope="module")
def dev_rows(gpu_lib, tset):
    import torch
    from tetris_mcts_b200 import replay
    rows = replay.memory_to_rows(*tset)
    d = torch.from_numpy(rows).cuda()
    torch.cuda.synchronize()
    return d, len(rows)


def pick(B, n=4096):
    idx = np.random.default_rng(B).permutation(n)[:B].astype(np.int32)
    idx[: min(B, 3)] = [0, 60, 4000][: min(B, 3)]                   # a clamped variance and a zero weight at every B > 2
    return idx


def check_against_f64(r, g, w, batch, weighted, what, grads_ref=None):
    """loss, loss_std, grad_norm within 1e-5 relative; each gradient tensor within 1e-5 of its own L2 norm (of grads_ref when given,
    else of float64 autograd); names tensor and element"""
    ref = R.train_loss_and_grads(w, batch, weighted)
    for k in ("loss", "loss_std", "grad_norm"):                          # (loss_std is 0 at B = 1)
        assert abs(r[k] - ref[k]) <= 1e-5 * abs(ref[k]) + 1e-9 * abs(ref["loss"]), (what, k, r[k], ref[k])
    if grads_ref is not None:
        ref["grad_flat"] = np.asarray(grads_ref, np.float64)
    off, worst = 0, 0.0
    g = np.asarray(g, np.float64)
    for name, shape in R.VN_SHAPES[:10]:
        n = R.grads_size(name)
        a, b = g[off:off + n], ref["grad_flat"][off:off + n]
        nrm = np.linalg.norm(b)
        d = np.abs(a - b)
        i = int(np.argmax(d))
        if d[i] > 1e-5 * nrm:
            pytest.fail("%s: %s element %s: got %.9g want %.9g (|d| %.3g > 1e-5 * ||grad|| = %.3g)"
                        % (what, name, np.unravel_index(i, shape), a[i], b[i], d[i], 1e-5 * nrm))
        worst = max(worst, float(d[i] / nrm) if nrm > 0 else 0.0)
        off += n
    return worst


def test_unknown_kind_is_refused(gpu_lib):
    from tetris_mcts_b200 import _lib as L
    from tetris_mcts_b200.model.trainer import _lib
    import ctypes as C
    h = C.c_void_p()
    w = R.init_weights(0)
    assert _lib().b200_trainer_create_kind(0, L.ptr(w), 16, 7, C.byref(h)) == 1 and not h.value          # B200_ERR_BAD_ARG


@pytest.mark.skipif(not os.path.exists(GOLD), reason="golden vectors not generated")
@pytest.mark.parametrize("tag,weighted,clip", [("w", True, 0.0), ("u", False, 0.0), ("c", True, 0.5)])
def test_training_steps_match_the_reference(gpu_lib, tag, weighted, clip):
    """the reference's own Model_VV.train goldens at the fp64 kind's tolerances"""
    from tetris_mcts_b200.model.model_vv import init_weights
    from tetris_mcts_b200.model.trainer import Trainer
    z = np.load(GOLD)
    keep = z["keep_index"]
    batch = [z["states"], z["value"], z["variance"], z["weight"]]
    t = Trainer(init_weights(int(z["seed"])), max_batch=128, kind="tc")
    t.set_out_ubound(*z["ubound"])
    steps = z[tag + "_steps"]

    def close(a, b, what):
        a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
        assert np.allclose(a, b, rtol=1e-5, atol=1e-5 * np.abs(b).max() * 1e-2), "%s: max abs err %.3g" % (what, np.abs(a - b).max())
    for it in range(len(steps)):
        r = t.step(batch, weighted=weighted, grad_clip=clip)
        for j, k in enumerate(("loss", "loss_std", "grad_norm")):
            assert abs(r[k] - steps[it, j]) <= 1e-5 * abs(steps[it, j]) + 1e-6, (it, k, r, steps[it])
        if it == 0:
            close(t.grads()[keep], z[tag + "_grad0"], "gradients of step 1")
    close(t.weights()[:R.N_TRAIN][keep], z[tag + "_weights"], "weights")
    if tag == "w":
        m, v, step = t.state()
        assert step == len(steps)
        close(m[keep], z["w_exp_avg"], "exp_avg")
        close(v[keep], z["w_exp_avg_sq"], "exp_avg_sq")
    t.close()


@pytest.mark.parametrize("B", BATCHES)
def test_against_float64_autograd(gpu_lib, tset, dev_rows, B):
    """one step at each batch size, weighted and unweighted, against float64 autograd; step_rows_dev equals step bit for bit"""
    from tetris_mcts_b200.model.trainer import Trainer
    s, value, variance, visits = tset
    idx = pick(B)
    w = R.init_weights(3)
    ub = (float(value[idx].max()), float(variance[idx].max()))
    w[R.N_TRAIN:R.N_TRAIN + 2] = ub
    scale = np.float32(1.0 / max(float(visits[idx].mean()), 1.0))
    wts = (visits * scale).astype(np.float32)
    rows, n_rows = dev_rows
    for weighted in (True, False):
        batch = [s[idx], value[idx], variance[idx], wts[idx]]
        t1, t2 = Trainer(w, max_batch=4096, kind="tc"), Trainer(w, max_batch=4096, kind="tc")
        r = t1.step(batch, weighted=weighted)
        worst = check_against_f64(r, t1.grads(), w, batch, weighted, "B=%d weighted=%s" % (B, weighted))
        print("B=%d weighted=%s: largest gradient error / tensor norm %.3g" % (B, weighted, worst))
        r2 = t2.step_rows_dev(rows.data_ptr(), n_rows, idx, float(scale), weighted=weighted)
        assert r2 == r and np.array_equal(t1.weights(), t2.weights()), (B, weighted)
        t1.close(); t2.close()


def _families(trained):
    fam = R.weight_families(4)
    fam["trained"] = trained
    return fam


@pytest.fixture(scope="module")
def trained_weights(gpu_lib, tset):
    """300 seeded steps of the fp64 kind at a raised learning rate: weights far from init"""
    from tetris_mcts_b200.model.model_vv import init_weights
    from tetris_mcts_b200.model.trainer import Trainer, sample_indices
    s, value, variance, visits = tset
    t = Trainer(init_weights(7), max_batch=512, lr=2e-2)
    t.set_out_ubound(float(value.max()), float(variance.max()))
    wts = (visits / visits.mean()).astype(np.float32)
    for it in range(300):
        idx = sample_indices(11, it, 256, len(s))
        t.step([s[idx], value[idx], variance[idx], wts[idx]], weighted=True)
    w = t.weights()
    t.close()
    assert float(np.abs(w[:R.N_TRAIN] - init_weights(7)[:R.N_TRAIN]).max()) > 0.05
    return w


@pytest.mark.parametrize("family", ["init", "act_1e3", "subnormal", "mostly_dead", "all_live", "saturated", "trained_bounds", "trained"])
def test_weight_families_against_float64(gpu_lib, tset, trained_weights, family):
    """Every family is held to float64 autograd at 1e-5, except the gradient tensors of `saturated`.  Its variance logit is ~25, where
    the fp32 sigmoid of the shared head (k_head, as the reference's fp32 torch) is exactly 1, so s (1 - s) = 0 replaces float64's
    1.4e-11 and the conv / fc1 gradients lose that path entirely: a property of fp32 storage that both kinds share, not of the GEMMs.
    There the tc kind's gradients are held to the fp64 kind's at the same 1e-5 of each tensor's norm (the split's ~3e-6 plus the fp64
    kind's rounding once to fp32); loss, loss_std and gradient norm still go against float64."""
    from tetris_mcts_b200.model.trainer import Trainer
    s, value, variance, visits = tset
    w = _families(trained_weights)[family].copy()
    idx = pick(300)
    wts = (visits / max(float(visits[idx].mean()), 1.0)).astype(np.float32)
    batch = [s[idx], value[idx], variance[idx], wts[idx]]
    for weighted in (True, False):
        grads_ref = None
        if family == "saturated":
            t64 = Trainer(w, max_batch=512, kind="fp64")
            t64.step(batch, weighted=weighted)
            grads_ref = t64.grads()
            t64.close()
        t = Trainer(w, max_batch=512, kind="tc")
        r = t.step(batch, weighted=weighted)
        worst = check_against_f64(r, t.grads(), w, batch, weighted, "%s weighted=%s" % (family, weighted), grads_ref)
        print("%s weighted=%s: largest gradient error / tensor norm %.3g" % (family, weighted, worst))
        t.close()


def test_long_same_sign_reduction(gpu_lib, oracle):
    """The conv weight gradients at B = 4096 reduce over 590 k (conv1), 393 k and 229 k terms.  With every ReLU live (`all_live`) the net
    is linear, and with every target above its prediction the output gradients share one sign, so each weight gradient is a sum of
    terms of mostly one sign: the running fp32 sum grows to the size of the result and every addition rounds at 2^-24 of it.  Held to
    1e-5 of each tensor's norm as everywhere.  Round-to-nearest sums of the 32-k tile sums stay below 1e-5 here even without the 2048-k chunks
    (their error grows like sqrt(n)); the chunk length rests on the worst-case bound in trainer.cu's header."""
    from tetris_mcts_b200.model.trainer import Trainer
    w = R.weight_families(5)["all_live"].copy()
    s = R.real_positions(4096, 21, oracle)
    t0 = Trainer(w, max_batch=4096, kind="fp64")
    pred = t0.loss([s, np.zeros(4096, np.float32), np.ones(4096, np.float32), None], want_pred=True)[2]
    t0.close()
    value = (pred[:, 0] + np.random.default_rng(0).uniform(20, 30, 4096)).astype(np.float32)
    batch = [s, value, np.full(4096, 50.0, np.float32), None]
    t = Trainer(w, max_batch=4096, kind="tc")
    r = t.step(batch, weighted=False)
    worst = check_against_f64(r, t.grads(), w, batch, False, "same-sign B=4096")
    print("same-sign B=4096: largest gradient error / tensor norm %.3g" % worst)
    t.close()


@pytest.mark.parametrize("weighted,clip", [(True, 0.0), (False, 0.5)])
def test_train_rows_dev_is_bit_identical_to_step_rows_dev(gpu_lib, dev_rows, weighted, clip):
    """K device-sampled steps == K step_rows_dev calls fed the sampler's indices: per-step log, weights, Yogi state"""
    from tetris_mcts_b200.model.model_vv import init_weights
    from tetris_mcts_b200.model.trainer import Trainer, sample_indices
    rows, n_rows = dev_rows
    batch, iters, seed, first, scale = 300, 5, 777, 40, 1.0 / 150
    a, b = Trainer(init_weights(2), max_batch=512, kind="tc"), Trainer(init_weights(2), max_batch=512, kind="tc")
    for t in (a, b):
        t.set_out_ubound(5000.0, 1e5)
    log = a.train_rows_dev(rows.data_ptr(), n_rows, batch, iters, seed, first, scale, weighted=weighted, grad_clip=clip)
    for it in range(iters):
        r = b.step_rows_dev(rows.data_ptr(), n_rows, sample_indices(seed, first + it, batch, n_rows), scale, weighted=weighted, grad_clip=clip)
        assert (r["loss"], r["loss_std"], r["grad_norm"]) == tuple(log[it]), it
    assert np.array_equal(a.weights(), b.weights())
    ma, va, sa = a.state()
    mb, vb, sb = b.state()
    assert sa == sb == iters and np.array_equal(ma, mb) and np.array_equal(va, vb)
    a.close(); b.close()


def test_reproducible_and_no_stale_tiles(gpu_lib, tset):
    """two trainers on the same inputs end with identical weights; a small batch after a large one gives the bits of a fresh trainer"""
    from tetris_mcts_b200.model.trainer import Trainer
    s, value, variance, visits = tset
    w = R.init_weights(6)
    w[R.N_TRAIN:R.N_TRAIN + 2] = (float(value.max()), float(variance.max()))
    wts = (visits / visits.mean()).astype(np.float32)
    big = pick(4096)
    small = big[:37]
    a, b, c = (Trainer(w, max_batch=4096, kind="tc") for _ in range(3))
    for t in (a, b):
        for _ in range(3):
            t.step([s[big], value[big], variance[big], wts[big]], weighted=True)
    assert np.array_equal(a.weights(), b.weights()) and np.array_equal(a.grads(), b.grads())
    c.set_weights(a.weights())
    r_after = a.step([s[small], value[small], variance[small], wts[small]], weighted=True)
    r_fresh = c.step([s[small], value[small], variance[small], wts[small]], weighted=True)
    assert r_after == r_fresh and np.array_equal(a.grads(), c.grads())
    a.close(); b.close(); c.close()


def test_trains_like_the_fp64_kind(gpu_lib, tset, dev_rows):
    """Same init, same device-sampled batches, 300 steps of each kind: step-1 gradients agree within the float64 bound (both kinds hold
    the same weights there), and both lower the loss.  Later steps drift apart chaotically and are held only to the loss going down."""
    from tetris_mcts_b200.model.model_vv import init_weights
    from tetris_mcts_b200.model.trainer import Trainer, sample_indices
    s, value, variance, visits = tset
    rows, n_rows = dev_rows
    batch, seed, scale = 512, 3, float(1.0 / visits.mean())
    w = init_weights(4)
    w[R.N_TRAIN:R.N_TRAIN + 2] = (float(value.max()), float(variance.max()))
    ts = {k: Trainer(w, max_batch=batch, kind=k) for k in ("fp64", "tc")}
    logs = {}
    for k, t in ts.items():
        logs[k] = [t.train_rows_dev(rows.data_ptr(), n_rows, batch, 1, seed, 0, scale)]
    g64, gtc = ts["fp64"].grads().astype(np.float64), ts["tc"].grads().astype(np.float64)
    off = 0
    for name, _ in R.VN_SHAPES[:10]:
        n = R.grads_size(name)
        d = np.abs(gtc[off:off + n] - g64[off:off + n]).max()
        assert d <= 2e-5 * np.linalg.norm(g64[off:off + n]), (name, d)       # each kind within 1e-5 of float64
        off += n
    idx = sample_indices(seed, 0, batch, n_rows)
    ref = R.train_loss_and_grads(w, [s[idx], value[idx], variance[idx], (visits[idx] * np.float32(scale)).astype(np.float32)], True)
    check_against_f64(dict(zip(("loss", "loss_std", "grad_norm"), logs["tc"][0][0])), gtc, w,
                      [s[idx], value[idx], variance[idx], (visits[idx] * np.float32(scale)).astype(np.float32)], True, "tc step 1")
    assert abs(logs["fp64"][0][0, 0] - ref["loss"]) <= 1e-5 * abs(ref["loss"])
    for k, t in ts.items():
        logs[k].append(t.train_rows_dev(rows.data_ptr(), n_rows, batch, 299, seed, 1, scale))
        loss = np.concatenate(logs[k])[:, 0]
        first, last = loss[:20].mean(), loss[-20:].mean()
        print("%s: loss %.4f -> %.4f" % (k, first, last))
        assert np.isfinite(loss).all() and last < first, k
        t.close()


TRAIN_RE = (r'Iteration:\s*(?P<iter>\d*)\s*training loss:\s*(?P<t_loss>\d*\.\d*)\s*validation loss:\s*(?P<v_loss>\d*\.\d*)±\s*'
            r'(?P<v_loss_err>\d*\.\d*|nan)\s*gradient norm:\s*(?P<g_norm>\d*\.\d*)')                          # web/parseLog.py:61-64
DATASIZE_RE = r'Training data size:\s*(?P<tsize>\d*)\s*Validation data size:\s*(?P<vsize>\d*)'            # web/parseLog.py:65-66


@pytest.fixture
def log(monkeypatch):
    """stderr of the training loop, the agents and play_batched (their lines go to the stream bound at import)"""
    import io
    from tetris_mcts_b200 import play_batched as PB
    from tetris_mcts_b200.agents import ValueSim as VS
    from tetris_mcts_b200.model import model_vv as MV
    buf = io.StringIO()
    for mod in (PB, VS, MV):
        monkeypatch.setattr(mod, "perr", dict(file=buf, flush=True))
    return buf


def test_play_batched_online_trains_with_the_tc_kind(gpu_lib, tmp_path, monkeypatch, log):
    """play_batched --online --train_kind tc trains, logs in the reference's format, checkpoints, and hot-swaps the trained network: the
    search engine's outputs then equal Model_VV.inference with the checkpoint's weights"""
    import io
    import re
    from tetris_mcts_b200 import play_batched as PB
    from tetris_mcts_b200 import pyTetris as PT
    from tetris_mcts_b200 import online as ON
    from tetris_mcts_b200.engine import BatchedEngine
    from tetris_mcts_b200.model.model_vv import Model_VV
    monkeypatch.chdir(tmp_path)
    states = PT.states_of(PT.new_games(16, (1, 0, 0), np.arange(40, 56, dtype=np.uint32)))
    seen, kinds = {}, []

    class Recording(BatchedEngine):
        def close(self):
            if getattr(self, "h", None) and self.n_games == 64:
                seen["out"] = self.valuenet(states)
            super().close()
    monkeypatch.setattr(PB, "BatchedEngine", Recording)
    orig_model = ON.OnlineTrainer._model

    def model(self):
        m = orig_model(self)
        kinds.append(m._trainer_obj().kind)
        return m
    monkeypatch.setattr(ON.OnlineTrainer, "_model", model)
    args = ["--agent_type", "ValueSimLP", "--mcts_sims", "64", "--ngames", "64", "--n_parallel", "64", "--max_nodes", "1024", "--endless",
            "--online", "--max_moves", "160", "--train_max_iters", "200", "--train_batch_size", "256", "--memory_size", "2000",
            "--memory_growth_rate", "150", "--train_kind", "tc"]
    timing = {}
    PB.run(PB.parse_args(args), out=io.StringIO(), timing=timing)
    err = log.getvalue()
    assert timing["trainings"] >= 1, err[-2000:]
    assert kinds and set(kinds) == {"tc"}
    assert re.search(DATASIZE_RE, err) and re.search(TRAIN_RE, err)
    assert os.path.isfile("pytorch_model/model_checkpoint")
    print("play_batched --online --train_kind tc: %d trainings, train %.2f s of %.2f s" % (timing["trainings"], timing["train_s"], timing["total_s"]))
    m = Model_VV(seed=9, eval_kind="net_tc")
    m.load("pytorch_model/model_checkpoint")
    v, var = m.inference(states[:, None])
    assert np.allclose(seen["out"][0], v[:, 0], rtol=1e-5, atol=1e-5) and np.allclose(seen["out"][1], var[:, 0], rtol=1e-5, atol=1e-5)
    m.close()


def test_valuesimlp_online_trains_with_the_tc_kind(gpu_lib, tmp_path, monkeypatch, log):
    import re
    from tetris_mcts_b200.agents import agent as A
    from tetris_mcts_b200.agents.ValueSimLP import ValueSimLP
    from tetris_mcts_b200.model.model_vv import Model_VV
    from tetris_mcts_b200.pyTetris import Tetris
    orig = A.TreeAgent.__init__

    def init(self, *a, **k):
        k["max_nodes"] = 8192
        orig(self, *a, **k)
    monkeypatch.setattr(A.TreeAgent, "__init__", init)
    monkeypatch.chdir(tmp_path)
    env_args = ((20, 10), 1, 0, 0)
    agent = ValueSimLP(online=True, sims=300, env=Tetris, env_args=env_args, benchmark=False, min_visit=40, memory_size=400,
                       memory_growth_rate=40, overflow_reset=True, train_kind="tc")
    agent._online.kw["max_iters"] = 300
    game = Tetris(*env_args)
    agent.update_root(game)
    for _ in range(120):
        game.play(agent.play())
        if game.end:
            game.reset()
        agent.update_root(game)
        if agent.n_trains >= 1:
            break
    err = log.getvalue()
    assert agent.n_trains >= 1 and agent.model._trainer_obj().kind == "tc", err[-2000:]
    assert len(re.findall(TRAIN_RE, err)) >= 1 and os.path.isfile("pytorch_model/model_checkpoint")
    m = Model_VV(seed=9, eval_kind="net_tc")
    m.load("pytorch_model/model_checkpoint")
    states = np.load("data/dump.npz")["states"][:32, 0]
    v, var = agent._eng.valuenet(states)
    mv, mvar = m.inference(states[:, None])
    assert np.allclose(v, mv[:, 0], rtol=1e-5, atol=1e-5) and np.allclose(var, mvar[:, 0], rtol=1e-5, atol=1e-5)
    agent.close(); m.close()


def test_checkpoint_moves_between_kinds(gpu_lib, tset, tmp_path):
    """a checkpoint is weights plus Yogi state in both kinds: saved from a tc run, loaded into an fp64 Model_VV, it resumes the same state"""
    from tetris_mcts_b200.model.model_vv import Model_VV
    s, value, variance, visits = tset
    batch = [s[:256, None], value[:256, None], variance[:256, None], (visits[:256, None] / visits[:256].mean()).astype(np.float32)]
    a = Model_VV(seed=3, train_kind="tc")
    for _ in range(3):
        a.train(batch, weighted=True)
    ck = str(tmp_path / "ck")
    a.save(ck, verbose=False)
    b = Model_VV(seed=8, train_kind="fp64")
    b.load(ck)
    assert np.array_equal(b.weights, a.weights)
    ma, va, sa = a._trainer_obj().state()
    mb, vb, sb = b._trainer_obj().state()
    assert sa == sb == 3 and np.array_equal(ma, mb) and np.array_equal(va, vb)
    a.close(); b.close()
