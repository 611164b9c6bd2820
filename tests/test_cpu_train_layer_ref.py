"""The stage-by-stage trainer check of tests/train_layer_ref.py pinned on the CPU before the device is held to it.

- The tf32 split (cvt.rna.tf32.f32) restated on the bits: ties away from zero, negative values, subnormals, the overflow edge, and
  x - big exact in fp32.
- numpy emulations of a whole step of both kinds (fp64: float64 accumulation; tc: a truncating sequential sum per 32-k tile, a
  round-to-nearest chain, fp64 chunks) lie inside every set, on every weight family and on batches with partial tiles and several k ranges.
- Each deliberate defect (train_layer_ref.STEP_MUTANTS, YOGI_MUTANTS) is flagged on every weight family.  The printed tables show which
  of them the older checks accept: each gradient tensor within 1e-5 of its norm against float64 autograd, and rtol 1e-5 on the goldens'
  keep_index.
- The restated split rules, over the GPU test's batch list, cover one and several k ranges for every product where the shape allows it."""
import numpy as np
import pytest

import f64_ref as R
import train_layer_ref as T
from test_gpu_train_layers import CHECKED

F32 = np.float32
KEEP = np.arange(0, R.N_TRAIN, 19)[:24316]           # a strided subset like the goldens' keep_index


def test_tf32_split_matches_the_bit_level_definition():
    """ties away from zero, negative values, subnormals, (2 - 2^-11) 2^127 -> inf, and x - big exact in fp32"""
    cases = [(1 + 2.0 ** -11, 1 + 2.0 ** -10), (-(1 + 2.0 ** -11), -(1 + 2.0 ** -10)), (1 + 3 * 2.0 ** -11, 1 + 2.0 ** -9),
             (1 + 2.0 ** -11 - 2.0 ** -23, 1.0), (-(1 + 2.0 ** -11 - 2.0 ** -23), -1.0), (1 - 2.0 ** -24, 1.0),
             (2.0 ** -140, 0.0), (2.0 ** -136, 2.0 ** -136), (0x1000 * 2.0 ** -149, 0x2000 * 2.0 ** -149), (0xFFF * 2.0 ** -149, 0.0),
             (-(0x3000 * 2.0 ** -149), -(0x4000 * 2.0 ** -149)), ((2 - 2.0 ** -11) * 2.0 ** 127, np.inf),
             ((2 - 2.0 ** -11 - 2.0 ** -23) * 2.0 ** 127, (2 - 2.0 ** -10) * 2.0 ** 127), (0.0, 0.0), (np.inf, np.inf)]
    x = np.array([c[0] for c in cases], F32)
    assert np.array_equal(x.astype(np.float64), [c[0] for c in cases])
    got = T.tf32_rna(x).astype(np.float64)
    assert np.array_equal(got, [c[1] for c in cases]), list(zip(x, got))
    bits = T.tf32_rna(x[np.isfinite(got)]).view(np.uint32)
    assert (bits & 0x1FFF == 0).all()
    rng = np.random.default_rng(4)
    y = (rng.standard_normal(100000) * 10.0 ** rng.integers(-30, 30, 100000)).astype(F32)
    y[:1000] = (rng.integers(1, 1 << 23, 1000) * 2.0 ** -149).astype(F32)             # subnormals
    big, small = T.tf32_split(y)
    assert np.array_equal((y - big).astype(np.float64), y.astype(np.float64) - big.astype(np.float64))     # exact in fp32
    r = np.abs(y.astype(np.float64) - big - small.astype(np.float64))
    assert (r <= 2.0 ** -22 * np.abs(y.astype(np.float64)) + 2.0 ** -137).all()


def _batch(oracle, B, seed=0):
    s = R.real_positions(max(B, 64), 3 + seed, oracle)[:B]
    rng = np.random.default_rng(seed)
    value = rng.uniform(0, 400, B).astype(F32)
    variance = rng.uniform(0, 50, B).astype(F32)
    variance[0] = 0.05                                         # clamped at 0.1
    weight = rng.uniform(0, 2, B).astype(F32)
    weight[-1] = 0
    return T.states_to_float(s), value, variance, weight


def _run(w, b, kind, weighted=True, mutant=None, Bg=None):
    x0, value, variance, weight = b
    bf, g, _ = T.emulate_step(w, x0, value, variance, weight, weighted, kind, Bg=Bg, mutant=mutant)
    return bf, g, T.step_checks(w, bf, len(x0), kind, weighted, grad=g, Bg=Bg, x0=x0)


@pytest.mark.parametrize("kind,shapes", [("fp64", (2, 30)), ("tc", (2, 15))])
def test_emulation_lies_in_every_set(oracle, kind, shapes):
    """every stage of the emulated step, on every weight family; prints per product the fraction of single-value sets, the widest set and
    (tc) the largest use of the bound"""
    for B in shapes:
        b = _batch(oracle, B)
        fams = R.weight_families(0) if B == shapes[0] or kind == "fp64" else {k: R.weight_families(0)[k] for k in ("init", "all_live")}
        print("\n[%s B=%d] product: single-value fraction / widest (ulps) / largest use of the bound, per weight family" % (kind, B))
        rows = {}
        for fam, w in fams.items():
            for weighted in (True, False):
                _, _, cs = _run(w, b, kind, weighted)
                for c in cs:
                    assert c.bad() == 0, c.describe("%s %s B=%d weighted=%s" % (kind, fam, B, weighted))
                for c in cs:
                    if isinstance(c, T.GemmCheck) and weighted:
                        rows.setdefault(c.name, []).append("%.3f/%d/%.3f" % (c.single(), c.widest, c.used if kind == "tc" else 0))
        for k, v in rows.items():
            print("  %-14s %s" % (k, " ".join(v)))


def _old_checks(w, b, weighted, g, weights_after=None, weights_ref=None):
    """(largest gradient error / (1e-5 ||tensor||) against float64 autograd, largest keep_index error / rtol-1e-5 allowance); <= 1 accepts"""
    x0, value, variance, weight = b
    ref = R.train_loss_and_grads(w, [x0.astype(np.int8), value, variance, weight], weighted)
    worst, off = 0.0, 0
    for name, _ in R.VN_SHAPES[:10]:
        n = R.grads_size(name)
        nrm = np.linalg.norm(ref["grad_flat"][off:off + n])
        d = np.abs(g[off:off + n].astype(np.float64) - ref["grad_flat"][off:off + n]).max()
        worst = max(worst, d / (1e-5 * nrm) if nrm > 0 else (np.inf if d > 0 else 0.0))
        off += n
    a, r = (g, ref["grad_flat"]) if weights_after is None else (weights_after, weights_ref)
    a, r = np.asarray(a, np.float64)[KEEP], np.asarray(r, np.float64)[KEEP]
    gold = float((np.abs(a - r) / (1e-5 * np.abs(r) + 1e-5 * np.abs(r).max() * 1e-2)).max())
    return worst, gold


MUTANT_B = {"fp64": 30, "tc": 15, "layout": 2, "head": 30}
# the one defect that changes no value on one family: with every ReLU live, a2 > 0 and a1 > 0 mask nothing either way
NO_OPS = {("col2im_wrong_mask", "all_live")}
# the one defect that stays inside its sets on two families: the s recovered from the rounded pred lies within the values expf's 2 ulp
# already admit for s where the logits barely vary (mostly_dead: every ReLU dead, z = fc_out's bias on every row) or the sigmoid
# saturates (saturated: s = 1 exactly and s ~ 1e-11)
INSIDE_THE_SET = {("sigmoid_from_pred", "mostly_dead"), ("sigmoid_from_pred", "saturated")}


def test_step_mutants_are_flagged_on_every_weight_family(oracle):
    """fp64 kind: fp32 accumulation (conv2), bias added before the final rounding, split-k partials rounded to fp32; tc kind: the last
    32-k tile of each range dropped, the last range's partial counted twice, a_s b_b dropped, bias added before k_finish's rounding; layout: ky /
    kx swapped in col2, da2 masked by the wrong activation, flat in HWC order; head: s (1 - s) from the rounded pred, a slice's dz scaled by
    its own B (a slice of 30 rows of a batch of 90).  Each is flagged by the stage checks on every weight family where it changes any value
    (NO_OPS lists where it does not), except INSIDE_THE_SET; the table records the old checks' verdict (error / allowance; <= 1 accepts)."""
    print("\nmutant              family          flagged  first stage flagged            autograd 1e-5  keep_index rtol 1e-5")
    for group, muts in T.STEP_MUTANTS.items():
        kind = "tc" if group == "tc" else "fp64"
        B = MUTANT_B[group]
        b = _batch(oracle, B, 1)
        for m in muts:
            for fam, w in R.weight_families(0).items():
                Bg = 3 * B if m == "dz_own_B" else None
                bf, g, cs = _run(w, b, kind, True, m, Bg)
                bf0, g0, _ = _run(w, b, kind, True, None, Bg)
                noop = np.array_equal(g, g0) and all(np.array_equal(bf[k], bf0[k]) for k in bf)
                bad = [c for c in cs if c.bad()]
                ag, gold = _old_checks(w, b, True, g) if Bg is None else (np.nan, np.nan)
                print("  %-18s %-14s %8d  %-30s %8.3f %-7s %8.3f %s" % (
                    m, fam, sum(c.bad() for c in bad), bad[0].name if bad else "no-op: every value unchanged" if noop else "-", ag,
                    "accepts" if ag <= 1 else "rejects", gold, "accepts" if gold <= 1 else "rejects"))
                assert bad or noop or (m, fam) in INSIDE_THE_SET, (m, fam)
                assert not noop or (m, fam) in NO_OPS, (m, fam)


YOGI_CASES = [(-1, {}), (-1, {"wd": 0.0}), (2, {}), (149, {}), (299, {}), (9, {"lr": 3e-3, "beta1": 0.8, "beta2": 0.99, "eps": 1e-4, "wd": 0.0})]


def test_yogi_mutants_are_flagged_on_every_weight_family(oracle):
    """the step counter off by one from step 100 on, exp_avg_sq initialised from the decayed gradient, sign(0) taken as +1, eps inside
    the sqrt: each changes the weights or the state bit for bit in one of YOGI_CASES (step before the step, hyper-parameters) on every
    weight family; the table records the rtol-1e-5 keep_index verdict on the weights (<= 1 accepts)"""
    b = _batch(oracle, 2, 2)
    print("\nYogi mutant        family          elements differing (weights / exp_avg / exp_avg_sq)   keep_index rtol 1e-5 on weights")
    for fam, w in R.weight_families(0).items():
        _, g, _ = _run(w, b, "fp64")
        p0 = w[:T.N_TRAIN]
        rng = np.random.default_rng(5)
        m0 = (g * rng.uniform(0.5, 1.5, T.N_TRAIN)).astype(F32)
        v0 = (g * g * rng.uniform(0.5, 1.5, T.N_TRAIN)).astype(F32)
        for mut in T.YOGI_MUTANTS:
            diff, gold = [0, 0, 0], 0.0
            for step_before, hyper in YOGI_CASES:
                c = T.yogi_step(step_before, hyper)
                cm = T.yogi_step(step_before, hyper, mut)
                ref = T.yogi(p0, g, m0, v0, c)
                got = T.yogi(p0, g, m0, v0, cm, mut)
                for i in range(3):
                    diff[i] += int((ref[i].view(np.uint32) != got[i].view(np.uint32)).sum())
                a, r = got[0].astype(np.float64)[KEEP], ref[0].astype(np.float64)[KEEP]
                gold = max(gold, float((np.abs(a - r) / (1e-5 * np.abs(r) + 1e-5 * np.abs(r).max() * 1e-2)).max()))
            print("  %-17s %-14s %9d / %9d / %9d                      %8.3f %s" % (mut, fam, diff[0], diff[1], diff[2], gold,
                                                                                 "accepts" if gold <= 1 else "rejects"))
            assert sum(diff) > 0, (mut, fam)


def test_the_restated_loss_and_norm_match_plain_float64():
    """std_mean and sumsq restate the kernels' order; they agree with float64 to rounding, and the DFMA chain is emulated exactly"""
    rng = np.random.default_rng(3)
    for n in (1, 2, 255, 256, 257, 4096):
        x = (rng.standard_normal(n) * 100).astype(F32)
        mean, std = T.std_mean(x)
        assert abs(mean - x.astype(np.float64).mean()) <= 1e-12 * np.abs(x).max()
        assert abs(std - x.astype(np.float64).std()) <= 1e-10 * (x.astype(np.float64).std() + 1e-300) + 1e-12 * np.abs(x).max()
    a, b, c = np.array([1 + 2.0 ** -30]), np.array([1 + 2.0 ** -30]), np.array([-1.0])
    assert T.fma64(a, b, c)[0] == 2.0 ** -29 + 2.0 ** -60 != (a * b + c)[0]
    g = (rng.standard_normal(T.N_TRAIN) * 1e-3).astype(F32)
    ss = T.sumsq(g)
    for i in range(10):
        seg = g[T.T_OFF[i]:T.T_OFF[i + 1]].astype(np.float64)
        assert abs(ss[i] - (seg * seg).sum()) <= 1e-12 * ss[i]


def test_split_rules_cover_every_product():
    """Over the GPU test's batches of each kind: every product runs as one k range and as several in each kind wherever some batch up to 4096 allows
    it; the tc kind hits both the small-grid ranges (>= 256 k, < 2048) and full 2048-k chunks; partial 64-row tiles and K not a multiple
    of 32 occur."""
    for kind in ("fp64", "tc"):
        for name in T.product_shapes(1):
            possible = {T.ranges(T.product_shapes(B)[name][2], T.kps_of(name, B, kind)).__len__() > 1 for B in range(1, 4097)}
            seen = {len(T.ranges(T.product_shapes(B)[name][2], T.kps_of(name, B, kind))) > 1 for B in CHECKED[kind]}
            assert seen == possible, (kind, name, seen, possible)
            print("%-5s %-13s one range: %-5s several: %s" % (kind, name, False in seen, True in seen))
    kps = [T.kps_of(n, B, "tc") for B in CHECKED["tc"] for n in T.product_shapes(B) if n != "fc_out_wgrad"]
    assert T.TG_KCHUNK in kps and any(256 <= k < T.TG_KCHUNK and k % 32 == 0 for k in kps)
    for kind, batches in CHECKED.items():
        assert any(B * 144 % 64 for B in batches) and any(B * 56 % 64 for B in batches) and any(B % 64 for B in batches)
    assert T.product_shapes(1)["conv1"][2] % 32 != 0
