"""Both device paths of the value networks (`net`: fp32 CUDA cores; `net_tc`: wgmma tensor cores with the fp16 x 2 operand split) and the
device trainer, against the float64 restatement in tests/f64_ref.py, on weights and boards chosen for where the kernels can go wrong.

Error analysis of the fp16 x 2 split (valuenet_tc.cuh, distnet_tc.cuh).  Every split operand x (activations scaled by 16, conv / fc1 weights
by 64, both exact powers of two) is stored as x1 + x2 with x1 = fp16(x), x2 = fp16(x - x1):
  - normal range: |x - x1| <= 2^-11 |x| and x2 rounds that to 11 bits, so |x - x1 - x2| <= 2^-22 |x|.  A product is accumulated as
    a1*b2 + a2*b1 + a1*b1 in fp32; the dropped a2*b2 is <= 2^-22 |ab|.  Each dot product therefore carries <= ~3 * 2^-22 of the sum of
    its |terms| from the split, plus fp32 accumulation (the wgmma accumulates in fp32; the tap / k sums add a few roundings).
  - overflow: x1 is infinite once the scaled value passes 65504: |a| >= ~4094 for activations, |w| >= ~1023.5 for weights.  Weights are
    refused at load time (b200_load_weights / b200_load_dist_weights return BAD_ARG); activations depend on the boards and are not checked.
  - subnormal floor: x2 is subnormal once |x| * 2^-11 < 2^-14 (|a| < 2^-7, |w| < 2^-9); its spacing is 2^-24, so the representation
    error becomes absolute: <= 2^-25 / 16 = 2^-29 for an activation, 2^-25 / 64 = 2^-31 for a weight.
Bounds used below (f64_ref computes every |term| sum in float64 from the same weights):
  - act3 (layer check, per element, both paths): |d| <= 2^-19 T3_max + 2^-26 per board, T3 = |a2| * |W3| + |b3|.  The relative part
    covers three split layers (<= 3 * 2^-22 each) and the fp32 sums inside wgmma; its order is not documented, so this is a statistical
    allowance (random-sign roundings grow like sqrt(K) 2^-24, K = 288), measured at <= 0.25 of the bound.  2^-26 (f64_ref.ACT_FLOOR) is
    8 x the 2^-29 floor, for the element's own floor and those carried from act1 / act2 through conv2 / conv3 (whose weight rows have
    2-norms ~0.6).  The bound separates the split from a single fp16: act3 kept as its high term alone breaks it by 12-75x on every weight
    family, the split stays under 0.12 of it (test_cpu_f64_ref.py::test_act3_bound_tells_the_split_from_a_single_fp16).
  - outputs: rtol 1e-5 (north_star), except for the two families f64_ref.ALLOWANCE names, which get |d out / d z| times an allowance on
    the logit z (f64_ref.valuenet_sensitivity):
      `saturated` (v = ub * sigmoid(~-25) ~ 1e-9: d v / v = d z, so the output is only as good as its logit): 67 * 2^-24 S_out, the worst
      case of the logit's own fp32 sum (each lane sums 64 products, then two shuffle adds), plus 2^-18 S_fc1 for the fc1 sums carried
      into it (1792-term wgmma sums: statistical, as above).  Measured 1.0e-5 relative on v, against an allowance of up to 2.2e-3.
      `subnormal` (activations in 2^-18 .. 2^-7, conv1 / fc1 weights below 2^-9): 2^-24 ||w_out_k||_2 sigma_max(W_fc1), the act3 floor
      carried into z: act3 errors of at most 2^-26, independent and uniform, give z an error of standard deviation
      2^-26 / sqrt(3) ||(w_out_k o relu mask) W_fc1||_2 <= 2^-26 / sqrt(3) ||w_out_k||_2 sigma_max(W_fc1), and 2^-24 is ~7 of those.
      That adds up to 6.9e-6 of the outputs, so this family is held to ~1.7e-5.
  - distributional probabilities: |d p| <= (1e-5 + 2 e_z) p + 1e-36 (p_i = exp(z_i - z_max) / sum), e_z = 0 except for `saturated`
    (128 * 2^-24 S_v + 2^-18 S_fc1, k_tdc_fc sums 128 products per logit) and `subnormal` (2^-24 ||w_v_a||_2 sigma_max(W_fc1)):
    f64_ref.distnet_sensitivity.
The CUDA-core path `net` meets the same bounds (its fp32 sums are shorter than the wgmma's).  The trainer keeps fp32 activations and
accumulates in fp64: loss, loss_std and gradient norm within 1e-5, each gradient tensor within 1e-5 of its norm, of float64 autograd."""
import numpy as np
import pytest

import f64_ref as R
from arena_gen import boards as random_boards

pytestmark = pytest.mark.gpu
KINDS = ["net", "net_tc"]


@pytest.fixture(scope="module")
def fam(oracle):
    return R.board_families(oracle)


@pytest.fixture(scope="module")
def n_sm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def engine(kind, w=None, dist_w=None, atoms=50):
    from tetris_mcts_b200.engine import BatchedEngine
    if dist_w is not None:
        return BatchedEngine(1, max_nodes=64, mode="dist", eval_kind=kind, dist_bins=atoms, dist_weights=dist_w)
    return BatchedEngine(1, max_nodes=64, eval_kind=kind, weights=w)


def act3(eng, states):
    from tetris_mcts_b200 import _lib as L
    s = np.ascontiguousarray(np.asarray(states, np.int8).reshape(-1, 200))
    out = np.zeros((len(s), 1792), np.float32)
    L.check(L.lib().b200_debug_act3(eng.h, L.ptr(s), len(s), L.ptr(out)))
    return out


def out_excess(got, ref, sens):
    """largest |got - ref| / bound; <= 1 passes"""
    return float(np.max(np.abs(np.asarray(got, np.float64) - ref) / (1e-5 * np.abs(ref) + sens)))


def max_rel(got, ref):
    return float(np.max(np.abs(np.asarray(got, np.float64) - ref) / np.abs(ref)))


def check_outputs(eng, w, states, what, allowance=None):
    """rtol 1e-5, plus the rounding allowance of an ill-conditioned family (f64_ref.ALLOWANCE)"""
    v, var = eng.valuenet(states)
    rv, rvar, _ = R.valuenet(w, states)
    sv, svar, _ = R.valuenet_sensitivity(w, states, allowance)
    assert np.isfinite(v).all() and np.isfinite(var).all(), what
    ev, evar = out_excess(v, rv, sv), out_excess(var, rvar, svar)
    assert ev <= 1 and evar <= 1, "%s: error / bound v %.3g var %.3g (max rel %.3g / %.3g)" % (what, ev, evar, max_rel(v, rv), max_rel(var, rvar))
    return max_rel(v, rv), max_rel(var, rvar)


def check_act3(eng, w, states, what, cells=None):
    got = act3(eng, states)
    _, _, ref = R.valuenet(w, states)
    _, _, t3 = R.valuenet_sensitivity(w, states)
    bound = 2.0 ** -19 * t3.max(1, keepdims=True) + R.ACT_FLOOR          # per board, scaled by its activation magnitude
    ratio = np.abs(got - ref) / bound
    if ratio.max() > 1:
        b, e = np.unravel_index(int(np.argmax(ratio)), ratio.shape)
        c, y, x = e // 56, (e % 56) // 4, e % 4
        where = "" if cells is None else " impulse at cell (row %d, col %d)" % divmod(int(cells[b]), 10)
        pytest.fail("%s: act3 board %d%s channel %d pixel (%d, %d): got %.9g want %.9g (bound %.3g)" %
                    (what, b, where, c, y, x, got[b, e], ref[b, e], bound[b, 0]))
    return float(ratio.max())


@pytest.mark.parametrize("kind", KINDS)
def test_value_net_weight_and_board_families(gpu_lib, fam, kind):
    """Every weight family x every board family; prints the per-family error table (max relative error against float64)."""
    wf = R.weight_families(0)
    eng = engine(kind, wf["init"])
    allb = np.concatenate(list(fam.values()))
    rows = []
    for wname, w in wf.items():
        eng.load_weights(w)                                                # the hot swap the online loop uses
        for bname, b in fam.items():
            ev, evar = check_outputs(eng, w, b, "%s / %s / %s" % (kind, wname, bname), R.ALLOWANCE.get(wname))
            rows.append((wname, bname, ev, evar))
        r3 = check_act3(eng, w, allb, "%s / %s" % (kind, wname))
        st = R.valuenet_stats(w, allb)
        print("\n[%s] %-14s act3 err/bound %.3f  max|act| %.3g max|w| %.3g max|logit| %.3g  worst rel v %.3g var %.3g" %
              (kind, wname, r3, st["act"], st["weight"], st["logit"], max(r[2] for r in rows if r[0] == wname),
               max(r[3] for r in rows if r[0] == wname)))
    eng.close()


@pytest.mark.parametrize("kind", KINDS)
def test_impulse_boards_cell_by_cell(gpu_lib, kind):
    """One settled cell, then one falling-piece cell, at each of the 200 cells: a transposed tap, a misplaced column or a wrong key decode
    shows on the cells it touches; the failure names the cell and the channel."""
    imp = R.impulse_boards()
    cells = np.concatenate([np.arange(200), np.arange(200)])
    for wname in ("init", "act_1e3"):
        w = R.weight_families(1)[wname]
        eng = engine(kind, w)
        check_act3(eng, w, imp, "%s / %s" % (kind, wname), cells=cells)
        v, var = eng.valuenet(imp)
        rv, rvar, _ = R.valuenet(w, imp)
        bad = np.nonzero((np.abs(v - rv) > 1e-5 * np.abs(rv)) | (np.abs(var - rvar) > 1e-5 * np.abs(rvar)))[0]
        assert len(bad) == 0, "%s / %s: outputs wrong for the impulse at cells %s" % (
            kind, wname, [("piece " if i >= 200 else "settled ") + "(%d, %d)" % divmod(int(cells[i]), 10) for i in bad[:8]])
        eng.close()


def self_play_training_set(oracle, n=3000, seed=4):
    """positions of random-play games with targets in the thousands (value ~ 80 x filled cells, variance up to ~1e5)"""
    s = R.real_positions(n, seed, oracle)
    rng = np.random.default_rng(seed)
    filled = (s > 0).sum(axis=(1, 2)).astype(np.float32)
    value = (80.0 * filled + rng.uniform(0, 400, n)).astype(np.float32)
    variance = (filled ** 2 * 20.0 + rng.uniform(0, 50, n)).astype(np.float32)
    variance[:50] = 0.05                                               # below the 0.1 clamp
    visits = rng.integers(0, 300, n).astype(np.float32)
    visits[50:80] = 0                                                  # zero weights
    return s, value, variance, visits


@pytest.fixture(scope="module")
def trained_weights(gpu_lib, oracle):
    """A few hundred seeded Trainer steps at a raised learning rate: weights far from init, out_ubound = the targets' maxima."""
    from tetris_mcts_b200.model.model_vv import init_weights
    from tetris_mcts_b200.model.trainer import Trainer, sample_indices
    s, value, variance, visits = self_play_training_set(oracle)
    t = Trainer(init_weights(7), max_batch=512, lr=2e-2)
    t.set_out_ubound(float(value.max()), float(variance.max()))
    wts = (visits / visits.mean()).astype(np.float32)
    first = last = None
    for it in range(300):
        idx = sample_indices(11, it, 256, len(s))
        r = t.step([s[idx], value[idx], variance[idx], wts[idx]], weighted=True)
        first = first or r["loss"]
        last = r["loss"]
    w = t.weights()
    t.close()
    init = init_weights(7)
    moved = float(np.abs(w[:R.N_TRAIN] - init[:R.N_TRAIN]).max())
    print("\ntrained: loss %.4g -> %.4g, max |w - w_init| %.3g, max |w| %.3g, out_ubound %s" % (first, last, moved, R.split_max(w), w[R.N_TRAIN:R.N_TRAIN + 2]))
    assert last < first and moved > 0.05
    return w, s


@pytest.mark.parametrize("kind", KINDS)
def test_trained_weights(gpu_lib, fam, trained_weights, kind):
    w, train_boards = trained_weights
    b = np.concatenate(list(fam.values()) + [train_boards[:1000]])
    st = R.valuenet_stats(w, b)
    print("\n[%s] trained weights: max|w| %.4g max|act| %.4g (fp16 headroom x%.3g for 16a) max|fc1| %.4g max|logit| %.4g" %
          (kind, st["weight"], st["act"], 65504 / 16 / st["act"], st["fc1"], st["logit"]))
    eng = engine(kind, w)
    ev, evar = check_outputs(eng, w, b, "%s / trained" % kind)
    r3 = check_act3(eng, w, b, "%s / trained" % kind)
    print("[%s] trained weights: max rel v %.3g var %.3g, act3 err/bound %.3f" % (kind, ev, evar, r3))
    eng.close()


def _edges(n, n_sm):
    """row indices on each side of every 128-row FC tile, of every conv pass (n_sm CTAs x 4 warpgroups x runs of 4 boards) and of
    every FC pass (n_sm CTAs x 128 rows)"""
    idx = set()
    for period in (128, n_sm * 16, n_sm * 128):
        for k in range(period, n + 1, period):
            idx.update((k - 2, k - 1, k, k + 1))
    return np.array(sorted(i for i in idx | {0, n - 1} if 0 <= i < n), np.int64)


def test_batch_sizes_across_pass_and_tile_boundaries(gpu_lib, oracle, n_sm):
    P, Fp = n_sm * 16, n_sm * 128                       # boards per k_tc_conv pass, rows per k_tc_fc pass
    sizes = [1, 2, 3, 4, 5, 127, 128, 129, P - 1, P, P + 1, Fp - 1, Fp, Fp + 1, 2 * Fp + P + 45]
    w = R.weight_families(2)["trained_bounds"]
    pool = np.concatenate([random_boards(sizes[-1], 17)] + list(R.board_families(oracle, 1).values()))
    rng = np.random.default_rng(0)
    e_tc, e_net = engine("net_tc", w), engine("net", w)
    small = {}
    for n in sizes:
        s = pool[rng.permutation(len(pool))[:n]] if n < len(pool) else pool[:n]
        v, var = e_tc.valuenet(s)
        v32, var32 = e_net.valuenet(s)
        sub = np.union1d(_edges(n, n_sm), rng.choice(n, min(n, 300), replace=False))
        for kind, (a, b) in (("net_tc", (v, var)), ("net", (v32, var32))):
            rv, rvar, _ = R.valuenet(w, s[sub])
            assert max_rel(a[sub], rv) <= 1e-5 and max_rel(b[sub], rvar) <= 1e-5, (kind, n)
        assert np.allclose(v, v32, rtol=2e-5, atol=0) and np.allclose(var, var32, rtol=2e-5, atol=0), n     # the whole batch
        if n <= 129:
            small[n] = (s, v, var)
        if n >= Fp:                                     # no dependence on where a board sits in the batch
            shift = P + 57
            v2, var2 = e_tc.valuenet(np.roll(s, shift, axis=0))
            assert np.array_equal(np.roll(v, shift), v2) and np.array_equal(np.roll(var, shift), var2), n
    for n, (s, v, var) in small.items():                # a small batch after the largest: act3 tiles past n hold stale boards
        v2, var2 = e_tc.valuenet(s)
        assert np.array_equal(v, v2) and np.array_equal(var, var2), n
        a = act3(e_tc, s)
        _, _, ref = R.valuenet(w, s)
        assert np.allclose(a, ref, rtol=2e-6, atol=2e-6), n
    e_tc.close(); e_net.close()


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("atoms", [2, 3, 33, 50, 64])
def test_distributional_net_families(gpu_lib, fam, kind, atoms):
    allb = np.concatenate(list(fam.values()))
    worst = {}
    eng = None
    for wname, w in R.dist_weight_families(5, atoms).items():
        if eng is None:
            eng = engine(kind, dist_w=w, atoms=atoms)
        else:
            eng.load_dist_weights(w, atoms)
        got = eng.distnet(allb)
        ref, _ = R.distnet(w, allb, atoms)
        ez = R.distnet_sensitivity(w, allb, atoms, R.ALLOWANCE.get(wname))[:, None]
        assert np.isfinite(got).all() and (got >= 0).all(), (wname, atoms)
        assert np.abs(got.sum(1) - 1).max() < 1e-5, (wname, atoms)
        ratio = np.abs(got - ref) / ((1e-5 + 2 * ez) * ref + 1e-36)
        if ratio.max() > 1:
            b, a = np.unravel_index(int(np.argmax(ratio)), ratio.shape)
            pytest.fail("%s atoms %d %s: board %d atom %d got %.9g want %.9g" % (kind, atoms, wname, b, a, got[b, a], ref[b, a]))
        big = ref > 1e-30
        worst[wname] = float(np.max(np.abs(got[big] - ref[big]) / ref[big]))
    print("\n[%s] atoms %d max rel err: %s" % (kind, atoms, ", ".join("%s %.3g" % kv for kv in worst.items())))
    eng.close()


@pytest.mark.parametrize("B", [1, 2, 63, 64, 65, 96, 257, 1024, 4096])
def test_trainer_against_float64_autograd(gpu_lib, oracle, B):
    """One step at each batch size, weighted and unweighted: loss, loss_std, gradient norm and every gradient tensor against float64
    autograd; and step_rows_dev (batch gathered on the device from replay rows) bit for bit against step."""
    import torch
    from tetris_mcts_b200 import replay
    from tetris_mcts_b200.model.trainer import Trainer
    s, value, variance, visits = self_play_training_set(oracle, n=4096, seed=9)
    rng = np.random.default_rng(B)
    idx = rng.permutation(4096)[:B].astype(np.int32)
    idx[: min(B, 3)] = [0, 60, 4000][: min(B, 3)]                          # a clamped variance and a zero weight at every B > 2
    w = R.init_weights(3)
    ub = (float(value[idx].max()), float(variance[idx].max()))
    w[R.N_TRAIN:R.N_TRAIN + 2] = ub
    scale = np.float32(1.0 / max(float(visits[idx].mean()), 1.0))
    wts = (visits * scale).astype(np.float32)
    rows = replay.memory_to_rows(s, value, variance, visits)
    dev_rows = torch.from_numpy(rows).cuda()
    torch.cuda.synchronize()
    for weighted in (True, False):
        batch = [s[idx], value[idx], variance[idx], wts[idx]]
        t1, t2 = Trainer(w, max_batch=4096), Trainer(w, max_batch=4096)
        for t in (t1, t2):
            t.set_out_ubound(*ub)
        r = t1.step(batch, weighted=weighted)
        g = t1.grads().astype(np.float64)
        ref = R.train_loss_and_grads(w, batch, weighted)
        for k in ("loss", "loss_std", "grad_norm"):                      # (loss_std is 0 at B = 1)
            assert abs(r[k] - ref[k]) <= 1e-5 * abs(ref[k]) + 1e-9 * abs(ref["loss"]), (B, weighted, k, r[k], ref[k])
        off = 0
        for name, _ in R.VN_SHAPES[:10]:
            n = R.grads_size(name)
            d = np.abs(g[off:off + n] - ref["grad_flat"][off:off + n]).max()
            assert d <= 1e-5 * np.linalg.norm(ref["grad_flat"][off:off + n]), (B, weighted, name, d)
            off += n
        r2 = t2.step_rows_dev(dev_rows.data_ptr(), len(rows), idx, float(scale), weighted=weighted)
        assert r2 == r and np.array_equal(t1.weights(), t2.weights()), (B, weighted)
        t1.close(); t2.close()


def test_tensor_core_load_refuses_weights_outside_fp16_range(gpu_lib):
    """|64 w| > 65504 would become an fp16 infinity in the split, and NaN would poison every output: net_tc refuses such weights and keeps
    the ones it had; net takes the large ones."""
    from tetris_mcts_b200 import _lib as L
    w = R.init_weights(0)
    states = random_boards(16, 1)
    eng = engine("net_tc", w)
    before = eng.valuenet(states)
    fits = w.copy()
    fits[320 + 5] = 1023.0                                                 # conv2: 64 * 1023 = 65472 fits
    eng.load_weights(fits)
    loaded = eng.valuenet(states)
    for off, x in ((7, -1100.0), (320 + 5, 1024.0), (9568 + 100, -1100.0), (18816 + 123456, 1100.0), (18816 + 7, np.nan)):   # conv1-3, fc1
        bad = w.copy()
        bad[off] = x
        with pytest.raises(L.B200Error) as ei:
            eng.load_weights(bad)
        assert ei.value.code == 1 and "65504" in str(ei.value) and "non-finite" in str(ei.value)
        assert all(np.array_equal(a, b) for a, b in zip(loaded, eng.valuenet(states))), off      # still the `fits` weights
    bad = w.copy()
    bad[18816 + 123456] = 1100.0
    eng.load_weights(w)
    assert all(np.array_equal(a, b) for a, b in zip(before, eng.valuenet(states)))
    e32 = engine("net", bad)
    assert all(np.isfinite(x).all() for x in e32.valuenet(states))
    e32.close()
    dw = R.dist_init_weights(0, 50)
    ed = engine("net_tc", dist_w=dw)
    p0 = ed.distnet(states)
    for off, x in ((3, 2000.0), (544 + 77, -2000.0), (16960 + 5000, 2000.0), (16960 + 9, np.inf)):   # conv1, conv2, fc1
        bad = dw.copy()
        bad[off] = x
        with pytest.raises(L.B200Error) as ei:
            ed.load_dist_weights(bad, 50)
        assert ei.value.code == 1 and "non-finite" in str(ei.value)
        assert np.array_equal(p0, ed.distnet(states)), off
    bad = dw.copy()
    bad[16960 + 5000] = 2000.0
    ed.close()
    en = engine("net", dist_w=bad)
    assert np.isfinite(en.distnet(states)).all()
    en.close()
