"""The tf32 trainer kind (Trainer(kind="tf32"), B200_TRAIN_TF32: k_gemm_tf32 in tetris_mcts_b200/csrc/trainer.cu) on the device.

Per element: after each step every stage is checked from the buffers the kernels read (tests/train_tf32_ref.py): the conv1-3 / fc1
forward, fc1's weight gradient, dflat, the three conv weight gradients and the implicit input gradients da2 / da1 against their
admissible sets; layout, bias gradients, head, loss, norm, clip and Yogi bit for bit.

Whole tensors against float64 autograd, with a bound derived from the operand rounding alone.  Each operand is rna_tf32(x), |x -
rna_tf32(x)| <= u |x| with u = 2^-11, so a product of two rounded operands is within 2u + u^2 < E = 2^-10 of |a b|, and a GEMM output
is within E of its |term| sum plus the tc kind's accumulation bound (~1e-5).  To first order these errors add along a result's path.
The loss sits behind the four forward products (conv1-3, fc1): the loss and loss_std are held to LOSS_BOUND = 4 E relative, the
gradient norm to GRAD_BOUND = 8 E.  A gradient element is a sum over the batch's pixels whose terms cancel, and the forward error
reaches it through the head, whose GaussianLL gradient (mean - pred) can cancel too, so a norm-relative bound does not follow for every
element; each element is instead held to error_bound: the forward error at the logits passed through the head's own sensitivity, plus
8 E for the products on its backward path and the activations it reads, both carried to the element with absolute values.  A ReLU
whose input lies within its error of zero may switch, which a first-order bound does not see (an element that is exactly 0 in the
kind and small in float64); for it every element also gets the tensor-level GRAD_BOUND of its tensor's norm.
As for the tc kind, the `saturated` family's gradients are held to the fp64 kind's (fp32's sigmoid saturates in both)."""
import os

import numpy as np
import pytest

import f64_ref as R
import train_layer_ref as T
import train_tf32_ref as TF
from test_gpu_train_layers import (FAMILY_BATCHES, Before, _batch, _fail, _pick, _same, dev_rows, families, read_buffers,  # noqa: F401
                                   tset)
from test_gpu_trainer_tc import DATASIZE_RE, TRAIN_RE, log  # noqa: F401

pytestmark = pytest.mark.gpu
LOSS_BOUND = 4 * 2.0 ** -10 + 1e-5
GRAD_BOUND = 8 * 2.0 ** -10 + 1e-5
EDGE = [1, 2, 3, 4, 9, 14, 15, 16, 17, 21, 22, 36, 37, 300, 1024, 4096]    # conv / fc1 tile and 2048-k chunk edges, then the largest
NO_BUFFERS = ("col1", "col2", "col3", "dcol3", "dcol2")


def tf32_buffers(t, B):
    from tetris_mcts_b200.model.trainer import DEBUG_ROWS
    bf = {k: t.debug_buffer(k, B) for k in DEBUG_ROWS if k not in NO_BUFFERS}
    bf["d_sumsq"] = t.debug_buffer("d_sumsq", 0)
    return bf


def check_step(t, before, r, B, weighted, what, x0=None, clip=0.0, raw=None):
    """every stage of the step t just took from `before`"""
    bf = tf32_buffers(t, B)
    g = t.grads()
    _fail(TF.step_checks(before.w, bf, B, weighted, grad=g if raw is None else raw, x0=x0), what)
    assert (r["loss"], r["loss_std"]) == T.std_mean(bf["lossv"]), what
    gn = T.grad_norm(bf["d_sumsq"])
    assert r["grad_norm"] == gn, (what, r["grad_norm"], gn)
    coef = T.clip_coef(gn, clip)
    if raw is not None:
        assert _same(g, T.clipped(raw, coef)), what
    p, m, v = T.yogi(before.w[:T.N_TRAIN], g, before.m, before.v, T.yogi_step(before.step))
    m_after, v_after, _ = t.state()
    for name, a, b in (("weights", t.weights()[:T.N_TRAIN], p), ("exp_avg", m_after, m), ("exp_avg_sq", v_after, v)):
        assert _same(a, b), (what, "Yogi", name)


@pytest.mark.parametrize("family", ["init", "act_1e3", "subnormal", "mostly_dead", "all_live", "saturated", "trained_bounds", "trained"])
def test_every_stage_on_every_weight_family(gpu_lib, tset, families, family):
    """batches of 1, 2, 37, 300 and then 5 on one trainer, weighted and unweighted in turn"""
    from tetris_mcts_b200.model.trainer import Trainer
    t = Trainer(families[family].copy(), max_batch=512, kind="tf32")
    for i, B in enumerate(FAMILY_BATCHES):
        weighted = i % 2 == 0
        batch = _batch(tset, _pick(B, i))
        before = Before(t)
        r = t.step(batch, weighted=weighted)
        check_step(t, before, r, B, weighted, "tf32 %s B=%d weighted=%s" % (family, B, weighted), x0=T.states_to_float(batch[0]))
    t.close()


def test_every_stage_at_the_edge_batches(gpu_lib, tset):
    """init weights at tile and chunk edges, 4096 once, then a small batch after the largest; clipping on one step"""
    from tetris_mcts_b200.model.trainer import Trainer
    t = Trainer(R.init_weights(3), max_batch=4096, kind="tf32")
    t.set_out_ubound(float(tset[1].max()), float(tset[2].max()))
    for i, B in enumerate(EDGE + [3]):
        weighted = i % 2 == 1
        batch = _batch(tset, _pick(B, 7))
        before = Before(t)
        r = t.step(batch, weighted=weighted)
        check_step(t, before, r, B, weighted, "tf32 B=%d weighted=%s" % (B, weighted), x0=T.states_to_float(batch[0]))
    t.close()
    w = R.init_weights(5)
    a, b = Trainer(w, max_batch=512, kind="tf32"), Trainer(w, max_batch=512, kind="tf32")
    batch = _batch(tset, _pick(300, 3))
    before = Before(a)
    b.step(batch, weighted=True)
    r = a.step(batch, weighted=True, grad_clip=0.05)
    assert T.clip_coef(r["grad_norm"], 0.05) is not None
    check_step(a, before, r, 300, True, "tf32 clip", x0=T.states_to_float(batch[0]), clip=0.05, raw=b.grads())
    a.close(); b.close()


def head_dz(z, ub, lb, mean, var, wt, Bg):
    """k_head's dz as a float64 function of the logits z [B, 2]"""
    sg = 1.0 / (1.0 + np.exp(-z))
    mp, vp = sg[:, 0] * ub[0] + lb[0], sg[:, 1] * ub[1] + lb[1]
    diff = mean - mp
    t2 = (diff * diff + var) / vp
    gl = wt / Bg
    return np.stack([gl * (-2.0 * diff / vp) * ub[0] * sg[:, 0] * (1 - sg[:, 0]), gl * (1.0 / vp - t2 / vp) * ub[1] * sg[:, 1] * (1 - sg[:, 1])], 1)


def error_bound(w, bf, weighted, B):
    """tensor name -> a first-order bound on each gradient element's error from the operand rounding (u = 2^-11 per operand, so each
    product within E = 2^-10 of its |term| sum), float64, from the step's buffers:
    - the forward pass in absolute values (|x0| through |W|, |bias| and the step's ReLU masks) gives each activation's expanded |term|
      sum F >= |activation|; the logits carry the four forward products: |z_err| <= 4 E (F_h |Wo|^T), and the head passes that on through its own
      sensitivity, |J| dz_err with J = d dz / d z (central differences of head_dz); where the mean - pred of GaussianLL cancels, J is
      large, so this term is what the operand rounding costs a gradient through the loss;
    - every product on the backward path (dflat, da2, da1, the weight gradient) and the forward activations a weight gradient reads
      (col, flat, h: at most four products deep) add <= 8 E of the |term| sums;
    both carried to every gradient element by the backward pass with |W|, the activations' F and the step's own ReLU masks (back)."""
    E = 2.0 ** -10
    p = {k: np.abs(v.astype(np.float64)) for k, v in T.params(w).items()}
    f = {k: np.asarray(bf[k], np.float64) for k in ("x0", "a1", "a2", "flat", "h", "dz")}
    pr = T.params(w)
    z = np.asarray(bf["h"], np.float32).astype(np.float64) @ pr["fow"].astype(np.float64).T + pr["fob"].astype(np.float64)[None]
    ub, lb = pr["ub"].astype(np.float64), pr["lb"].astype(np.float64)
    mean = np.asarray(bf["value"], np.float64).reshape(-1)
    var = np.maximum(np.asarray(bf["variance"], np.float32).reshape(-1), np.float32(0.1)).astype(np.float64)
    wt = np.asarray(bf["weight"], np.float64).reshape(-1) if weighted else np.ones(B)
    J = np.zeros((B, 2, 2))
    for i in range(2):
        hz = np.zeros_like(z)
        hz[:, i] = 1e-5 * (1 + np.abs(z[:, i]))
        J[:, :, i] = (head_dz(z + hz, ub, lb, mean, var, wt, B) - head_dz(z - hz, ub, lb, mean, var, wt, B)) / (2 * hz[:, i:i + 1])
    col, F = {1: np.abs(T.im2col(bf["x0"], 20, 10, 1).astype(np.float64))}, {}
    for i, (H, W, act) in ((1, (18, 8, "a1")), (2, (16, 6, "a2")), (3, (0, 0, "a3"))):
        F[i] = (col[i] @ p["c%dw" % i].T + p["c%db" % i][None]) * (np.asarray(bf[act], np.float32).reshape(-1, 32) > 0)
        if H:
            col[i + 1] = T.im2col(F[i].astype(np.float32), H, W, 32).astype(np.float64)
    F_flat = T.nhwc_to_flat(F[3].astype(np.float32)).astype(np.float64)
    F_h = (F_flat @ p["f1w"].T + p["f1b"][None]) * (f["h"] > 0)
    z_err = 4 * E * (F_h @ p["fow"].T)
    seed = np.einsum("bji,bi->bj", np.abs(J), z_err)

    def back(sd):
        """|sd| (B x 2, at dz) carried to every gradient element with absolute values and the step's ReLU masks"""
        out = {"fc_out.weight": sd.T @ F_h, "fc_out.bias": sd.sum(0)}
        dh = (sd @ p["fow"]) * (f["h"] > 0)
        out["fc1.weight"], out["fc1.bias"] = dh.T @ F_flat, dh.sum(0)
        d = T.flat_to_nhwc_relu((dh @ p["f1w"]).astype(np.float32), bf["flat"]).astype(np.float64)          # [B*56, 32]
        for i, (H, W, act) in ((3, (16, 6, "a2")), (2, (18, 8, "a1")), (1, (20, 10, None))):
            out["conv%d.weight" % i], out["conv%d.bias" % i] = d.T @ col[i], d.sum(0)
            if act:
                A, Bm = TF.dgrad_operands(d.astype(np.float32), p["c%dw" % i].astype(np.float32), H, W)
                d = (A.astype(np.float64) @ Bm.astype(np.float64)) * (f[act].reshape(-1, 32) > 0)
        return out
    prop, mag = back(seed), back(np.abs(f["dz"]))
    return {k: prop[k] + 8 * E * mag[k] for k in prop}


def check_against_f64(r, g, w, batch, weighted, what, bf, grads_ref=None):
    """loss, loss_std within LOSS_BOUND, grad_norm within GRAD_BOUND; each gradient element within error_bound + GRAD_BOUND of its
    tensor's norm -> (largest error / tensor norm, largest error / its bound)"""
    ref = R.train_loss_and_grads(w, batch, weighted)
    for k, bound in (("loss", LOSS_BOUND), ("loss_std", LOSS_BOUND), ("grad_norm", GRAD_BOUND)):
        assert abs(r[k] - ref[k]) <= bound * abs(ref[k]) + 1e-9 * abs(ref["loss"]), (what, k, r[k], ref[k])
    if grads_ref is not None:
        ref["grad_flat"] = np.asarray(grads_ref, np.float64)
    off, worst, used = 0, 0.0, 0.0
    g = np.asarray(g, np.float64)
    eb = error_bound(w, bf, weighted, len(batch[0]))
    for name, shape in R.VN_SHAPES[:10]:
        n = R.grads_size(name)
        a, b = g[off:off + n], ref["grad_flat"][off:off + n]
        nrm = np.linalg.norm(b)
        d = np.abs(a - b)
        allow = eb[name].reshape(-1) + GRAD_BOUND * nrm
        with np.errstate(divide="ignore", invalid="ignore"):
            i = int(np.argmax(np.where(allow > 0, d / allow, np.where(d > 0, np.inf, 0.0))))
        assert d[i] <= allow[i], "%s: %s element %s: got %.9g want %.9g (|d| %.3g > bound %.3g; ||grad|| %.3g)" % (
            what, name, np.unravel_index(i, shape), a[i], b[i], d[i], allow[i], nrm)
        used = max(used, float(d[i] / allow[i]) if allow[i] > 0 else 0.0)
        i = int(np.argmax(d))
        worst = max(worst, float(d[i] / nrm) if nrm > 0 else 0.0)
        off += n
    return worst, used


@pytest.mark.parametrize("family", ["init", "act_1e3", "subnormal", "mostly_dead", "all_live", "saturated", "trained_bounds", "trained"])
def test_against_float64_autograd(gpu_lib, tset, families, family):
    from tetris_mcts_b200.model.trainer import Trainer
    w = families[family].copy()
    for B in (37, 1024):
        batch = _batch(tset, _pick(B, 2))
        for weighted in (True, False):
            grads_ref = None
            if family == "saturated":
                t64 = Trainer(w, max_batch=1024, kind="fp64")
                t64.step(batch, weighted=weighted)
                grads_ref = t64.grads()
                t64.close()
            t = Trainer(w, max_batch=1024, kind="tf32")
            r = t.step(batch, weighted=weighted)
            worst, used = check_against_f64(r, t.grads(), w, batch, weighted, "%s B=%d weighted=%s" % (family, B, weighted),
                                            tf32_buffers(t, B), grads_ref)
            print("%s B=%d weighted=%s: largest gradient error / tensor norm %.3g, largest use of the element bound %.3f" % (
                family, B, weighted, worst, used))
            t.close()


def test_reproducible_and_no_stale_tiles(gpu_lib, tset):
    """two trainers on the same inputs end with identical weights; a small batch after a large one gives the bits of a fresh trainer"""
    from tetris_mcts_b200.model.trainer import Trainer
    w = R.init_weights(6)
    w[R.N_TRAIN:R.N_TRAIN + 2] = (float(tset[1].max()), float(tset[2].max()))
    big = _batch(tset, _pick(4096))
    small = _batch(tset, _pick(37))
    a, b, c = (Trainer(w, max_batch=4096, kind="tf32") for _ in range(3))
    for t in (a, b):
        for _ in range(3):
            t.step(big, weighted=True)
    assert np.array_equal(a.weights(), b.weights()) and np.array_equal(a.grads(), b.grads())
    c.set_weights(a.weights())
    assert a.step(small, weighted=True) == c.step(small, weighted=True) and np.array_equal(a.grads(), c.grads())
    a.close(); b.close(); c.close()


@pytest.mark.parametrize("weighted,clip", [(True, 0.0), (False, 0.5)])
def test_train_rows_dev_is_bit_identical_to_step_rows_dev(gpu_lib, dev_rows, weighted, clip):
    from tetris_mcts_b200.model.trainer import Trainer, sample_indices
    d, rows = dev_rows
    n_rows, batch, iters, seed, first, scale = len(rows), 300, 5, 777, 40, 1.0 / 150
    a, b = Trainer(R.init_weights(2), max_batch=512, kind="tf32"), Trainer(R.init_weights(2), max_batch=512, kind="tf32")
    for t in (a, b):
        t.set_out_ubound(5000.0, 1e5)
    log_ = a.train_rows_dev(d.data_ptr(), n_rows, batch, iters, seed, first, scale, weighted=weighted, grad_clip=clip)
    for it in range(iters):
        r = b.step_rows_dev(d.data_ptr(), n_rows, sample_indices(seed, first + it, batch, n_rows), scale, weighted=weighted, grad_clip=clip)
        assert (r["loss"], r["loss_std"], r["grad_norm"]) == tuple(log_[it]), it
    assert np.array_equal(a.weights(), b.weights())
    ma, va, sa = a.state()
    mb, vb, sb = b.state()
    assert sa == sb == iters and np.array_equal(ma, mb) and np.array_equal(va, vb)
    a.close(); b.close()


@pytest.mark.parametrize("ranks", [1, 2, 3])
def test_grad_rows_dev_slices(gpu_lib, dev_rows, ranks):
    """each slice's unrounded fp64 gradient against its pre-rounding sets; apply_grads_dev's gradient is the ordered fp64 sum of the
    parts rounded once; one part covering the batch is bit-identical to a train_rows_dev step"""
    import torch
    from tetris_mcts_b200.model.trainer import GRAD_VEC, Trainer, sample_indices
    d, rows = dev_rows
    n_rows, batch, seed, it, scale = len(rows), 301, 5, 2, np.float32(1.0 / 150)
    t = Trainer(R.init_weights(9), max_batch=512, kind="tf32")
    t.set_out_ubound(5000.0, 1e5)
    w = t.weights()
    idx = sample_indices(seed, it, batch, n_rows)
    cuts = np.linspace(0, batch, ranks + 1).astype(int)
    parts = torch.zeros((ranks, GRAD_VEC), dtype=torch.float64, device="cuda")
    for r, (lo, hi) in enumerate(zip(cuts[:-1], cuts[1:])):
        t.grad_rows_dev(d.data_ptr(), n_rows, batch, int(lo), int(hi), seed, it, float(scale), parts[r].data_ptr(), weighted=True)
        B = int(hi - lo)
        bf = tf32_buffers(t, B)
        x0 = T.gather_rows(rows, idx[lo:hi], scale)[0]
        _fail(TF.step_checks(w, bf, B, True, grad64=parts[r].cpu().numpy()[:T.N_TRAIN], Bg=batch, x0=x0),
              "tf32 slice [%d, %d) of %d" % (lo, hi, batch))
    t.apply_grads_dev(parts.data_ptr(), ranks, 0.0, 0)
    t.read_log(1)
    p = parts.cpu().numpy()[:, :T.N_TRAIN]
    s = p[0].copy()
    for r in range(1, ranks):
        s = s + p[r]
    assert _same(t.grads(), s.astype(np.float32))
    if ranks == 1:
        u = Trainer(R.init_weights(9), max_batch=512, kind="tf32")
        u.set_out_ubound(5000.0, 1e5)
        u.train_rows_dev(d.data_ptr(), n_rows, batch, 1, seed, it, float(scale), weighted=True)
        assert np.array_equal(u.grads(), t.grads()) and np.array_equal(u.weights(), t.weights())
        u.close()
    t.close()


def test_debug_buffers_refused(gpu_lib):
    from tetris_mcts_b200 import _lib as L
    from tetris_mcts_b200.model.trainer import NO_BUFFERS as NB, Trainer
    assert set(NB["tf32"]) == set(NO_BUFFERS)
    t = Trainer(R.init_weights(0), max_batch=16, kind="tf32")
    for name in NO_BUFFERS:
        with pytest.raises(L.B200Error) as e:
            t.debug_buffer(name, 1)
        assert e.value.code == 1 and "tf32" in str(e.value)
    assert t.debug_buffer("da1", 16).shape == (16, 144 * 32) and t.debug_buffer("a2", 16).shape == (16, 96 * 32)
    t.close()


def test_checkpoint_moves_between_kinds(gpu_lib, tset, tmp_path):
    """a tf32 checkpoint (weights and Yogi state) loads into fp64 and tc models, and a tc checkpoint into a tf32 model"""
    from tetris_mcts_b200.model.model_vv import Model_VV
    s, value, variance, visits = tset
    batch = [s[:256, None], value[:256, None], variance[:256, None], (visits[:256, None] / visits[:256].mean()).astype(np.float32)]
    for src, dst in (("tf32", "fp64"), ("tf32", "tc"), ("tc", "tf32")):
        a = Model_VV(seed=3, train_kind=src)
        for _ in range(3):
            a.train(batch, weighted=True)
        ck = str(tmp_path / ("ck_" + src + dst))
        a.save(ck, verbose=False)
        b = Model_VV(seed=8, train_kind=dst)
        b.load(ck)
        assert np.array_equal(b.weights, a.weights)
        ma, va, sa = a._trainer_obj().state()
        mb, vb, sb = b._trainer_obj().state()
        assert sa == sb == 3 and np.array_equal(ma, mb) and np.array_equal(va, vb), (src, dst)
        b.train(batch, weighted=True)
        assert b._trainer_obj().state()[2] == 4
        a.close(); b.close()


def test_trains_like_the_other_kinds(gpu_lib, tset, dev_rows):
    """same init and device-sampled batches, 300 steps of each kind: every kind lowers the loss"""
    from tetris_mcts_b200.model.trainer import Trainer
    s, value, variance, visits = tset
    d, rows = dev_rows
    batch, seed, scale = 512, 3, float(1.0 / visits.mean())
    w = R.init_weights(4)
    w[R.N_TRAIN:R.N_TRAIN + 2] = (float(value.max()), float(variance.max()))
    for k in ("fp64", "tc", "tf32"):
        t = Trainer(w, max_batch=batch, kind=k)
        loss = t.train_rows_dev(d.data_ptr(), len(rows), batch, 300, seed, 0, scale)[:, 0]
        first, last = loss[:20].mean(), loss[-20:].mean()
        print("%s: loss %.4f -> %.4f" % (k, first, last))
        assert np.isfinite(loss).all() and last < first, k
        t.close()


def test_play_batched_online_trains_with_the_tf32_kind(gpu_lib, tmp_path, monkeypatch, log):  # noqa: F811
    """play_batched --online --train_kind tf32 trains, logs in the reference's format, checkpoints, and hot-swaps the trained network"""
    import io
    import re
    from tetris_mcts_b200 import online as ON
    from tetris_mcts_b200 import play_batched as PB
    from tetris_mcts_b200 import pyTetris as PT
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
            "--memory_growth_rate", "150", "--train_kind", "tf32"]
    timing = {}
    PB.run(PB.parse_args(args), out=io.StringIO(), timing=timing)
    err = log.getvalue()
    assert timing["trainings"] >= 1, err[-2000:]
    assert kinds and set(kinds) == {"tf32"}
    assert re.search(DATASIZE_RE, err) and re.search(TRAIN_RE, err)
    assert os.path.isfile("pytorch_model/model_checkpoint")
    print("play_batched --online --train_kind tf32: %d trainings, train %.2f s of %.2f s" % (timing["trainings"], timing["train_s"], timing["total_s"]))
    m = Model_VV(seed=9, eval_kind="net_tc")
    m.load("pytorch_model/model_checkpoint")
    v, var = m.inference(states[:, None])
    assert np.allclose(seen["out"][0], v[:, 0], rtol=1e-5, atol=1e-5) and np.allclose(seen["out"][1], var[:, 0], rtol=1e-5, atol=1e-5)
    m.close()
