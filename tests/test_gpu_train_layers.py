"""The device trainer held stage by stage to tests/train_layer_ref.py: after each step the batch buffers (Trainer.debug_buffer), the
gradient and the optimiser state are read back, and every stage is checked from the inputs the kernel itself read — layout bit for bit,
the 12 products per element against their admissible sets, the bias gradients, the head, loss, gradient norm, clip and Yogi bit for bit.
Both trainer kinds, every weight family plus trained weights, weighted and unweighted, batches on both sides of every tile and chunk
edge, a small batch after a large one on the same trainer, clipping, 300 Yogi steps with a resume and a reset, and data-parallel slices."""
import numpy as np
import pytest

import f64_ref as R
import train_layer_ref as T

pytestmark = pytest.mark.gpu
TG_BM, TG_KCHUNK = 64, 2048                 # k_gemm_tc's output tile rows and fp32 chain cap (trainer.cu)
PIXELS = (144, 96, 56)                      # conv1 / conv2 / conv3 output pixels per board


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


BATCHES = sorted(set([1, 2, 300, 4096] + edge_batches()))
# the edge batches each kind is restated at (run time: the tc kind at 4096 once, neither at 2048, where no k range of either kind starts)
CHECKED = {"fp64": [b for b in BATCHES if b != 2048], "tc": [b for b in BATCHES if b < 2048] + [4096]}
FAMILY_BATCHES = (1, 2, 37, 300, 5)          # per weight family; 5 right after 300 on the same trainer (stale rows)


@pytest.fixture(scope="module")
def tset(oracle):
    n, seed = 4096, 9
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
def dev_rows(gpu_lib, tset):
    import torch
    from tetris_mcts_b200 import replay
    rows = replay.memory_to_rows(*tset)
    d = torch.from_numpy(rows).cuda()
    torch.cuda.synchronize()
    return d, rows


@pytest.fixture(scope="module")
def families(gpu_lib, tset):
    """R.weight_families(4) plus `trained`: 300 seeded fp64-kind steps at lr 2e-2"""
    from tetris_mcts_b200.model.trainer import Trainer, sample_indices
    s, value, variance, visits = tset
    t = Trainer(R.init_weights(7), max_batch=512, lr=2e-2)
    t.set_out_ubound(float(value.max()), float(variance.max()))
    wts = (visits / visits.mean()).astype(np.float32)
    for it in range(300):
        idx = sample_indices(11, it, 256, len(s))
        t.step([s[idx], value[idx], variance[idx], wts[idx]], weighted=True)
    fam = R.weight_families(4)
    fam["trained"] = t.weights()
    t.close()
    return fam


def read_buffers(t, B):
    from tetris_mcts_b200.model.trainer import DEBUG_ROWS
    bf = {k: t.debug_buffer(k, B) for k in DEBUG_ROWS}
    bf["d_sumsq"] = t.debug_buffer("d_sumsq", 0)
    return bf


def _fail(checks, what):
    for c in checks:
        if c.bad():
            pytest.fail(c.describe(what))


def _same(a, b):
    a, b = np.asarray(a), np.asarray(b, np.asarray(a).dtype)
    it = np.uint64 if a.dtype == np.float64 else np.uint32
    return np.array_equal(a.reshape(-1).view(it), b.reshape(-1).view(it))


class Before:
    """weights and Yogi state read before a step"""

    def __init__(self, t):
        self.w = t.weights()
        self.m, self.v, self.step = t.state()


def check_step(t, before, r, B, weighted, what, x0=None, clip=0.0, raw=None, hyper=None, stats=None):
    """every stage of the step t just took from `before`; raw: the unclipped fp32 gradient (a twin trainer's) when clip applies"""
    bf = read_buffers(t, B)
    g = t.grads()
    cs = T.step_checks(before.w, bf, B, t.kind, weighted, grad=g if raw is None else raw, x0=x0)
    _fail(cs, what)
    if stats is not None:
        for c in cs:
            if isinstance(c, T.GemmCheck):
                s = stats.setdefault((t.kind, c.name), [1.0, 0, 0.0])
                s[0], s[1], s[2] = min(s[0], c.single()), max(s[1], c.widest), max(s[2], c.used if t.kind == "tc" else 0.0)
            elif isinstance(c, T.SetCheck):
                s = stats.setdefault(("head", c.name), [0, 0, 0])
                s[1] = max(s[1], int(c.width.max()))
    mean, std = T.std_mean(bf["lossv"])
    assert (r["loss"], r["loss_std"]) == (mean, std), (what, r, mean, std)
    gn = T.grad_norm(bf["d_sumsq"])
    assert r["grad_norm"] == gn, (what, r["grad_norm"], gn)
    coef = T.clip_coef(gn, clip)
    if raw is not None:
        assert _same(g, T.clipped(raw, coef)), (what, "clipped gradient != RN32(raw * coef)", coef)
    c = T.yogi_step(before.step, hyper)
    p, m, v = T.yogi(before.w[:T.N_TRAIN], g, before.m, before.v, c)
    w_after = t.weights()
    m_after, v_after, step_after = t.state()
    assert step_after == T.next_step(before.step)[0], (what, step_after)
    for name, a, b in (("weights", w_after[:T.N_TRAIN], p), ("exp_avg", m_after, m), ("exp_avg_sq", v_after, v)):
        if not _same(a, b):
            i = int(np.argmax(a.view(np.uint32) != b.view(np.uint32)))
            pytest.fail("%s: Yogi %s element %d: got %r, restated %r (%d differ)" % (what, name, i, a[i], b[i],
                                                                                 int((a.view(np.uint32) != b.view(np.uint32)).sum())))
    return bf


def _batch(tset, idx):
    s, value, variance, visits = tset
    wts = (visits / max(float(visits[idx].mean()), 1.0)).astype(np.float32)
    return [s[idx], value[idx], variance[idx], wts[idx]]


def _pick(B, seed=0):
    idx = np.random.default_rng(B + 1000 * seed).permutation(4096)[:B].astype(np.int32)
    idx[: min(B, 3)] = [0, 60, 4000][: min(B, 3)]                   # a clamped variance and a zero weight at every B > 2
    return idx


def test_debug_buffer_refusals(gpu_lib):
    from tetris_mcts_b200 import _lib as L
    from tetris_mcts_b200.model.trainer import Trainer
    t = Trainer(R.init_weights(0), max_batch=16)
    for name, n in (("nope", 1), ("a1", 17), ("a1", -1)):
        with pytest.raises(L.B200Error) as e:
            t.debug_buffer(name, n)
        assert e.value.code == 1
    assert t.debug_buffer("a1", 16).shape == (16, 144 * 32) and t.debug_buffer("d_sumsq", 0).shape == (10,)
    t.close()


STATS = {}


@pytest.mark.parametrize("kind", ["fp64", "tc"])
@pytest.mark.parametrize("family", ["init", "act_1e3", "subnormal", "mostly_dead", "all_live", "saturated", "trained_bounds", "trained"])
def test_every_stage_on_every_weight_family(gpu_lib, tset, families, kind, family):
    """batches of 1, 2, 37, 300 and then 5 on one trainer, weighted and unweighted in turn"""
    from tetris_mcts_b200.model.trainer import Trainer
    w = families[family].copy()
    t = Trainer(w, max_batch=512, kind=kind)
    for i, B in enumerate(FAMILY_BATCHES):
        weighted = i % 2 == 0
        batch = _batch(tset, _pick(B, i))
        before = Before(t)
        r = t.step(batch, weighted=weighted)
        check_step(t, before, r, B, weighted, "%s %s B=%d weighted=%s" % (kind, family, B, weighted), x0=T.states_to_float(batch[0]),
                   stats=STATS)
    t.close()


@pytest.mark.parametrize("kind", ["fp64", "tc"])
def test_every_stage_at_the_edge_batches(gpu_lib, tset, kind):
    """init weights at every tile and chunk edge batch; the tc kind at 4096 once; a small batch after the largest"""
    from tetris_mcts_b200.model.trainer import Trainer
    t = Trainer(R.init_weights(3), max_batch=4096, kind=kind)
    t.set_out_ubound(float(tset[1].max()), float(tset[2].max()))
    for i, B in enumerate(CHECKED[kind] + [3]):
        weighted = i % 2 == 1
        batch = _batch(tset, _pick(B, 7))
        before = Before(t)
        r = t.step(batch, weighted=weighted)
        check_step(t, before, r, B, weighted, "%s B=%d weighted=%s" % (kind, B, weighted), x0=T.states_to_float(batch[0]), stats=STATS)
    t.close()


@pytest.mark.parametrize("kind", ["fp64", "tc"])
def test_clipping_is_the_raw_gradient_times_the_coefficient(gpu_lib, tset, kind):
    """clip < the gradient norm: the clipped gradient is RN32(raw * coef) bit for bit, raw from a twin stepped without clipping; clip
    above the norm leaves the gradient alone"""
    from tetris_mcts_b200.model.trainer import Trainer
    w = R.init_weights(5)
    for B, clip in ((300, 0.05), (37, 1e6)):
        batch = _batch(tset, _pick(B, 3))
        a, b = Trainer(w, max_batch=512, kind=kind), Trainer(w, max_batch=512, kind=kind)
        before = Before(a)
        b.step(batch, weighted=True)
        raw = b.grads()
        r = a.step(batch, weighted=True, grad_clip=clip)
        assert (T.clip_coef(r["grad_norm"], clip) is not None) == (clip < 1)
        check_step(a, before, r, B, True, "%s B=%d clip=%g" % (kind, B, clip), x0=T.states_to_float(batch[0]), clip=clip, raw=raw)
        a.close(); b.close()


@pytest.mark.parametrize("kind", ["fp64", "tc"])
def test_yogi_over_300_device_row_steps(gpu_lib, dev_rows, kind):
    """step_rows_dev on sample_indices batches: every stage at steps 1-10 and every 25th (the gathered rows included); then a set_state
    resume at step 300 and a set_state(-1) reset, one step each; then non-default set_hyper values"""
    from tetris_mcts_b200.model.trainer import Trainer, sample_indices
    d, rows = dev_rows
    n_rows, scale = len(rows), np.float32(1.0 / 150)
    t = Trainer(R.init_weights(8), max_batch=512, kind=kind)
    t.set_out_ubound(5000.0, 1e5)

    def one(it, what, B=64, hyper=None, check=True):
        idx = sample_indices(21, it, B, n_rows)
        before = Before(t) if check else None
        r = t.step_rows_dev(d.data_ptr(), n_rows, idx, float(scale), weighted=True)
        if check:
            x0, value, variance, weight = T.gather_rows(rows, idx, scale)
            bf = check_step(t, before, r, B, True, "%s %s" % (kind, what), x0=x0, hyper=hyper)
            for k, v in (("value", value), ("variance", variance), ("weight", weight)):
                assert _same(bf[k][:, 0], v), (what, k)
    for it in range(300):
        one(it, "step %d" % (it + 1), check=it < 10 or (it + 1) % 25 == 0)
    m, v, step = t.state()
    assert step == 300
    t.set_state(m, v, 300)
    one(300, "resumed at 300")
    t.set_state(None, None, -1)
    one(301, "after reset")
    hyper = dict(lr=3e-3, beta1=0.8, beta2=0.99, eps=1e-4, wd=0.0)
    t2 =Trainer(t.weights(), max_batch=512, kind=kind, lr=hyper["lr"], betas=(hyper["beta1"], hyper["beta2"]), eps=hyper["eps"],
                 weight_decay=hyper["wd"])
    t.close()
    t = t2
    for it in range(3):
        one(302 + it, "set_hyper step %d" % (it + 1), hyper=hyper)
    t.close()


@pytest.mark.parametrize("kind", ["fp64", "tc"])
@pytest.mark.parametrize("ranks", [1, 2, 3])
def test_grad_rows_dev_slices(gpu_lib, dev_rows, kind, ranks):
    """each rank's unrounded fp64 slice gradient (weight and bias gradients) against the pre-rounding intervals; the slice's dz uses the
    whole batch's size"""
    import torch
    from tetris_mcts_b200.model.trainer import GRAD_VEC, Trainer, sample_indices
    d, rows = dev_rows
    n_rows, batch, seed, it, scale = len(rows), 301, 5, 2, np.float32(1.0 / 150)
    t = Trainer(R.init_weights(9), max_batch=512, kind=kind)
    t.set_out_ubound(5000.0, 1e5)
    w = t.weights()
    idx = sample_indices(seed, it, batch, n_rows)
    cuts = np.linspace(0, batch, ranks + 1).astype(int)
    out = torch.zeros(GRAD_VEC, dtype=torch.float64, device="cuda")
    for lo, hi in zip(cuts[:-1], cuts[1:]):
        t.grad_rows_dev(d.data_ptr(), n_rows, batch, int(lo), int(hi), seed, it, float(scale), out.data_ptr(), weighted=True)
        B = int(hi - lo)
        bf = read_buffers(t, B)                                   # synchronises the trainer's stream: the slice is written
        g64 = out.cpu().numpy()[:T.N_TRAIN]
        x0 = T.gather_rows(rows, idx[lo:hi], scale)[0]
        cs = T.step_checks(w, bf, B, kind, True, grad64=g64, Bg=batch, x0=x0)
        _fail(cs, "%s slice [%d, %d) of %d" % (kind, lo, hi, batch))
    t.close()


def test_print_stage_statistics():
    """the per-product statistics the tests above gathered (single-value fraction (min over steps), widest set in ulps, largest use of
    the tc bound); the head rows give the widest set of each output"""
    for (kind, name), (single, widest, used) in sorted(STATS.items()):
        print("%-5s %-16s single %.3f  widest %d  used %.4f" % (kind, name, single, widest, used))
