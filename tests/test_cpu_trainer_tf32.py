"""The tf32 trainer kind's restatement (tests/train_tf32_ref.py) pinned on the CPU before the device is held to it.

- The implicit gather (k_gemm_tf32's OP_CONV index arithmetic) equals im2col for every conv shape, edge pixels included.
- The implicit input gradient, in float64, equals col2im_relu(dY . W) up to the order of the sum.
- A numpy emulation of a whole tf32 step lies inside every set on every weight family.
- Each deliberate defect (a 3xTF32 operand, RZ for RNA, a transposed tap, a dropped k tile, a missing ReLU mask) is flagged on every
  weight family where it changes a value.
- "tf32" is a trainer kind and a --train_kind choice."""
import numpy as np
import pytest

import f64_ref as R
import train_layer_ref as T
import train_tf32_ref as TF

F32, F64 = np.float32, np.float64


@pytest.mark.parametrize("layer", ["conv1", "conv2", "conv3"])
def test_implicit_gather_is_im2col(layer):
    H, W, C = TF.CONV_IN[layer]
    n = 3
    act = np.random.default_rng(1).permutation(n * H * W * C).astype(F32)           # distinct values: each element's own number
    got = TF.implicit_col(act, H, W, C, n)
    want = T.im2col(act, H, W, C)
    assert got.shape == want.shape == (n * (H - 2) * (W - 2), C * 9)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    # every input element is read: the corner pixels once, the inner ones by all nine taps
    reads = np.bincount(got.ravel().astype(np.int64), minlength=act.size)
    assert reads.min() >= 1 and reads.max() == 9


@pytest.mark.parametrize("H,W", [(16, 6), (18, 8)])
def test_implicit_input_gradient_is_col2im_of_dY_W(H, W):
    """sum_k A[m][k] B[k][ci] masked by act > 0 equals col2im_relu(dY . W) in float64 (1e-12 of the |term| sums: only the order differs)"""
    rng = np.random.default_rng(H)
    n = 3
    dY = rng.standard_normal((n * (H - 2) * (W - 2), 32)).astype(F32)
    Wt = rng.standard_normal((32, 288)).astype(F32)
    act = rng.standard_normal((n * H * W, 32)).astype(F32)
    A, Bm = TF.dgrad_operands(dY, Wt, H, W)
    got = np.where(act > 0, A.astype(F64) @ Bm.astype(F64), 0.0)
    dcol = dY.astype(F64) @ Wt.astype(F64)
    OH, OW = H - 2, W - 2
    d = dcol.reshape(n, OH, OW, 32, 9)
    s = np.zeros((n, H, W, 32))
    for ky in range(3):
        for kx in range(3):
            s[:, ky:ky + OH, kx:kx + OW, :] += d[..., ky * 3 + kx]
    want = np.where(act > 0, s.reshape(-1, 32), 0.0)
    tsum = np.abs(A.astype(F64)) @ np.abs(Bm.astype(F64))
    assert (np.abs(got - want) <= 1e-12 * tsum + 1e-300).all()
    # the fp32 path of the other kinds (col2im_relu of the rounded dcol) agrees to fp32 rounding
    c2i = T.col2im_relu(dcol.astype(F32), act, H, W, 32).astype(F64)
    assert (np.abs(c2i - want) <= 2.0 ** -20 * tsum).all()


def _batch(oracle, B, seed=0):
    s = R.real_positions(max(B, 64), 3 + seed, oracle)[:B]
    rng = np.random.default_rng(seed)
    value = rng.uniform(0, 400, B).astype(F32)
    variance = rng.uniform(0, 50, B).astype(F32)
    variance[0] = 0.05
    weight = rng.uniform(0, 2, B).astype(F32)
    weight[-1] = 0
    return T.states_to_float(s), value, variance, weight


def _run(w, b, weighted=True, mutant=None):
    x0, value, variance, weight = b
    bf, g, _ = TF.emulate_step(w, x0, value, variance, weight, weighted, mutant=mutant)
    return bf, g, TF.step_checks(w, bf, len(x0), weighted, grad=g, x0=x0)


@pytest.mark.parametrize("B", [2, 15])
def test_emulation_lies_in_every_set(oracle, B):
    b = _batch(oracle, B)
    fams = R.weight_families(0)
    if B > 2:
        fams = {k: fams[k] for k in ("init", "all_live")}
    print("\n[tf32 B=%d] product: single-value fraction / widest (ulps) / largest use of the bound" % B)
    rows = {}
    for fam, w in fams.items():
        for weighted in (True, False):
            _, _, cs = _run(w, b, weighted)
            for c in cs:
                assert c.bad() == 0, c.describe("tf32 %s B=%d weighted=%s" % (fam, B, weighted))
                if isinstance(c, T.GemmCheck) and weighted:
                    rows.setdefault(c.name, []).append("%.3f/%d/%.3f" % (c.single(), c.widest, c.used))
    for k, v in rows.items():
        print("  %-40s %s" % (k, " ".join(v)))


# where a defect changes no value: with every ReLU live, no mask applies, so dropping it changes nothing; with every ReLU dead, conv2
# gathers a1 = 0 in any tap order
NO_OPS = {("no_mask", "all_live"), ("tap", "mostly_dead")}


def test_mutants_are_flagged_on_every_weight_family(oracle):
    b = _batch(oracle, 2, 1)
    print("\nmutant     family          flagged  first stage flagged")
    for m in TF.MUTANTS:
        for fam, w in R.weight_families(0).items():
            bf, g, cs = _run(w, b, True, m)
            bf0, g0, _ = _run(w, b, True, None)
            noop = np.array_equal(g, g0) and all(np.array_equal(bf[k], bf0[k]) for k in bf)
            bad = [c for c in cs if c.bad()]
            print("  %-9s %-14s %8d  %s" % (m, fam, sum(c.bad() for c in bad), bad[0].name if bad else "no-op" if noop else "-"))
            assert bad or noop, (m, fam)
            assert not noop or (m, fam) in NO_OPS, (m, fam)


def test_tf32_is_a_trainer_kind():
    from tetris_mcts_b200 import play_batched as PB
    from tetris_mcts_b200.model import trainer as TR
    assert TR.KINDS["tf32"] == 2 and set(TR.NO_BUFFERS["tf32"]) == {"col1", "col2", "col3", "dcol3", "dcol2"}
    assert PB.parse_args(["--train_kind", "tf32"]).train_kind == "tf32"
    # the buffers a tf32 trainer does not allocate, per sample: 355 392 B, 1.46 GB at max_batch 4096
    per = 4 * sum(TR.DEBUG_ROWS[k] for k in TR.NO_BUFFERS["tf32"])
    assert per == 355392 and abs(per * 4096 / 1e9 - 1.456) < 1e-3
