"""The layer-by-layer check of tests/f16_layer_ref.py pinned on the CPU before the device is held to it.

- numpy's float32 -> float16 cast, which the restatement uses for the loader's weights and for the epilogue, rounds like __float2half_rn on
  the subnormal and overflow edges.
- The float64 emulations of net_fp16 and dist_fp16 (tests/f16_ref.py, tests/f16_dist_ref.py) fall inside the admissible set of every
  element of every layer, on every weight family and board family.
- Each deliberate defect of those emulations (f16_ref.MUTANTS, and bfloat16 for fp16) is flagged on every weight family it applies to,
  while the whole-network contracts (f16_ref.act3_bound, f16_dist_ref.act2_bound) accept most of them: the printed table is the measure.
- The two-term form accepts a canonical split and flags a pair with the same sum that is not canonical.
- The fc stage: the exact fp32 fma the head restatement uses agrees with exact rational arithmetic; the emulations' fc1 accumulator and
  outputs lie in the fc1 and head sets; each fc defect (f16_layer_ref.FC_MUTANTS) is flagged on every weight family, while the old output
  contracts (f16_ref.out_excess, the dist_fp16 probability bound) accept most of them: the printed table is the measure."""
from fractions import Fraction

import numpy as np
import pytest
import torch

import f16_dist_ref as D
import f16_layer_ref as L
import f16_ref as H
import f64_ref as R

ATOMS = 50


@pytest.fixture(scope="module")
def fam(oracle):
    return R.board_families(oracle)


def _terms(layers):
    return [[a.numpy()] for a in layers]


def _emulated(dist, w, b, dtype=torch.float16, mutant=None):
    if dist:
        return _terms(D.emulate_layers(w, b, ATOMS, dtype, mutant))
    return _terms(H.emulate_layers(w, b, dtype, mutant))


def _weight_families(dist):
    return R.dist_weight_families(5, ATOMS) if dist else R.weight_families(0)


def test_numpy_fp16_rounding_matches_float2half_rn_on_the_edges():
    """Round to nearest even as CUDA's __float2half_rn defines it: overflow past 65504 + half an ulp, ties to even in the subnormals and
    at the subnormal / normal boundary, underflow to zero at and below 2^-25."""
    cases = [(65504.0, 65504.0), (65519.99609375, 65504.0), (65520.0, np.inf), (-65520.0, -np.inf), (1e9, np.inf),
             (2.0 ** -24, 2.0 ** -24), (2.0 ** -25, 0.0), (-(2.0 ** -25), -0.0), (2.0 ** -25 * (1 + 2.0 ** -10), 2.0 ** -24),
             (3 * 2.0 ** -25, 2.0 ** -23), (5 * 2.0 ** -25, 2.0 ** -23), (2.0 ** -14 - 2.0 ** -25, 2.0 ** -14),
             (2.0 ** -14 - 3 * 2.0 ** -25, 2.0 ** -14 - 2.0 ** -23), (1 + 2.0 ** -11, 1.0), (1 + 3 * 2.0 ** -11, 1 + 2.0 ** -9)]
    x = np.array([c[0] for c in cases], np.float32)
    assert np.array_equal(x.astype(np.float64), [c[0] for c in cases])       # every input is an fp32 value
    with np.errstate(over="ignore"):
        got = x.astype(np.float16).astype(np.float64)
    want = np.array([c[1] for c in cases])
    assert np.array_equal(got, want) and np.array_equal(np.signbit(got), np.signbit(want)), list(zip(x, got, want))
    s = np.array([2.0 ** -20, -3.0], np.float32)                             # the loader's second term of 64 w
    t = L.weight_terms(s / 64, 2)
    assert np.array_equal(t[0] + t[1], s.astype(np.float64))


@pytest.mark.parametrize("dist", [False, True], ids=["value", "dist"])
def test_fp16_emulation_lies_in_every_admissible_set(fam, dist):
    """Every element of every layer of the emulation, checked on the emulation's own previous layer; prints the fraction of elements whose
    admissible set is a single fp16 value, per weight family, layer and board family."""
    names = list(fam)
    allb = np.concatenate([fam[k] for k in names])
    cut = np.cumsum([0] + [len(fam[k]) for k in names])
    print("\n[%s] fraction of elements with exactly one admissible fp16 value (%s)" % ("dist_fp16" if dist else "net_fp16", ", ".join(names)))
    for wname, w in _weight_families(dist).items():
        checks = L.check_stack(w, allb, _emulated(dist, w, allb), dist)
        for c in checks:
            assert c.bad() == 0, c.describe(wname)
            fr = [float(c.single[cut[i]:cut[i + 1]].mean()) for i in range(len(names))]
            print("  %-14s act%d  all %.3f  |  %s" % (wname, c.layer, float(c.single.mean()), " ".join("%.3f" % f for f in fr)))


def _flagged(dist, w, b, layers):
    return sum(c.bad() for c in L.check_stack(w, b, layers, dist))


@pytest.mark.parametrize("dist", [False, True], ids=["value", "dist"])
def test_mutants_are_flagged_on_every_weight_family(fam, dist):
    """RZ activations, RZ weights, bias added after the rounding, scale x8 instead of x16 (`subnormal` family: elsewhere it is exact),
    bfloat16, and a missing conv2 block: each is flagged by the layer check on every weight family.  The table also records whether the
    whole-network contract (act3 / act2 within 2^-10 of the board's largest |term| sum) accepts the mutant's last layer."""
    b = np.concatenate(list(fam.values()))
    wf = _weight_families(dist)
    variants = [(m, torch.float16, m) for m in H.MUTANTS] + [("bf16", torch.bfloat16, None)]
    last = "act2" if dist else "act3"
    print("\n[%s] mutant        weight family   flagged elements   old %s contract (error / bound; <= 1 accepts)" %
          ("dist_fp16" if dist else "net_fp16", last))
    for name, dtype, mutant in variants:
        for wname, w in wf.items():
            if name == "scale8" and wname != "subnormal":
                continue
            layers = _emulated(dist, w, b, dtype, mutant)
            if dist:
                ref, bound = D.act2(w, b, ATOMS), D.act2_bound(w, b, ATOMS)
            else:
                ref, bound = R.valuenet(w, b)[2], H.act3_bound(w, b)
            ratio = float((np.abs(layers[-1][0].reshape(len(b), -1) - ref) / bound).max())
            n = _flagged(dist, w, b, layers)
            print("  %-15s %-14s %10d          %7.3f  %s" % (name, wname, n, ratio, "accepts" if ratio <= 1 else "rejects"))
            assert n > 0, (name, wname)


def _split_emulation(w, b, layer_in, dist, layer):
    """the two-term kernel's output of one layer, restated: z rounded to fp32, the activation, the canonical split"""
    z, _ = L.preactivation(w, layer_in, dist, layer, 2)
    o = L.epilogue32(z, dist)
    x1 = o.astype(np.float16)
    x2 = (o - x1.astype(np.float32)).astype(np.float16)
    return [x1.astype(np.float64) / 16, x2.astype(np.float64) / 16]


@pytest.mark.parametrize("dist", [False, True], ids=["value", "dist"])
def test_two_term_check_accepts_the_canonical_split_only(fam, dist):
    b = np.concatenate([fam["real"], fam["partial_piece"]])
    w = _weight_families(dist)["init"]
    layers, inp = [], b
    for layer in range(1, 3 if dist else 4):
        layers.append(_split_emulation(w, b, inp, dist, layer))
        inp = layers[-1]
    assert all(c.bad() == 0 for c in L.check_stack(w, b, layers, dist))
    x1, x2 = layers[-1]                                  # same sum, not canonical: x1 one ulp up, x2 carrying the difference
    big = x1 * 16 > 1
    up = np.nextafter((x1 * 16).astype(np.float16), np.float16(np.inf)).astype(np.float64) / 16
    bent = [np.where(big, up, x1), np.where(big, x2 - (up - x1), x2)]
    c = L.Check(w, layers[-2], bent, dist, len(layers))
    assert big.sum() > 1000 and (~c.ok)[big].mean() > 0.99 and c.ok[~big].all()


def _rn32(q):
    """a Fraction -> the fp32 value nearest to it, ties to even, with IEEE overflow (exact reference for fma32)"""
    if q == 0:
        return 0.0
    sign, q = (-1 if q < 0 else 1), abs(q)
    e = q.numerator.bit_length() - q.denominator.bit_length()
    if Fraction(2) ** e > q:
        e -= 1
    quantum = Fraction(2) ** (max(e, -126) - 23)
    v = round(q / quantum) * quantum                               # round() on a Fraction ties to even
    return sign * (np.inf if v >= Fraction(2) ** 128 else float(v))


def test_fma32_is_correctly_rounded():
    """Constructed cases: a product exactly on an fp32 midpoint with an addend far below float64's precision on either side (the TwoSum
    correction; a plain float64 fma rounded to fp32 ties to even there), exact ties to even, subnormal results and ties, overflow at and
    just below the rounding threshold; then random triples, including cancelling ones.  Each against exact rational arithmetic."""
    f = np.float32
    mx = float(np.finfo(np.float32).max)
    cases = [(1 + 2.0 ** -12, 1 + 2.0 ** -12, 2.0 ** -80), (1 + 2.0 ** -12, 1 + 2.0 ** -12, -(2.0 ** -80)), (1 + 2.0 ** -12, 1 + 2.0 ** -12, 0.0),
             (3.0, 1 + 2.0 ** -23, -(2.0 ** -80)), (3.0, 1 + 2.0 ** -23, 2.0 ** -80), (3.0, 1 + 2.0 ** -23, 0.0),
             (-3.0, 1 + 2.0 ** -23, 2.0 ** -80), (2.0 ** -100, 2.0 ** -30, 0.0), (3 * 2.0 ** -75, 2.0 ** -75, 0.0),
             (3 * 2.0 ** -75, 2.0 ** -75, 2.0 ** -149), (2.0 ** -75, 2.0 ** -75, -(2.0 ** -149)), (2.0 ** 127, 2.0, 0.0),
             (mx, 1.0, 2.0 ** 103), (mx, 1.0, 2.0 ** 103 - 2.0 ** 79), (-mx, 1.0, -(2.0 ** 103)), (mx, -1.0, mx), (2.0 ** -149, 0.5, 0.0)]
    assert L.fma32(f(cases[0][0]), f(cases[0][1]), f(cases[0][2])) != np.float32(np.float64(cases[0][0]) ** 2 + cases[0][2])
    rng = np.random.default_rng(11)
    n = 4000
    m = rng.integers(1 << 23, 1 << 24, (3, n)).astype(np.float64) * rng.choice([-1.0, 1.0], (3, n))
    ex = rng.integers(-40, 20, (3, n))
    ex[2, : n // 4] = ex[0, : n // 4] + ex[1, : n // 4] + rng.integers(-30, 10, n // 4)    # addends near the product: cancellation
    a, b, c = (np.ldexp(m[i], ex[i] - 23).astype(np.float32) for i in range(3))
    c[n // 4: n // 2] = -(a[n // 4: n // 2].astype(np.float64) * b[n // 4: n // 2]).astype(np.float32)      # nearly exact cancellation
    trip = [tuple(f(x) for x in t) for t in cases] + list(zip(a, b, c))
    A, B, C = (np.array([t[i] for t in trip], np.float32) for i in range(3))
    with np.errstate(over="ignore"):
        got = L.fma32(A, B, C)
    want = [_rn32(Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z))) for x, y, z in trip]
    bad = [(t, g, w) for t, g, w in zip(trip, got, want) if not float(g) == w]
    assert not bad, bad[:5]


def test_exp_range_brackets_the_exact_exp_by_two_ulp():
    x = np.concatenate([np.float32([0, -1e-30, 1e-30, -87.3, -103.5, -110, 88.7]),
                        np.random.default_rng(2).uniform(-100, 80, 20000).astype(np.float32)])
    lo, hi = L.exp_range(x)
    e = np.exp(x.astype(np.float64))
    assert (lo <= L.exp_rn(x)).all() and (L.exp_rn(x) <= hi).all()
    assert (lo.astype(np.float64) <= e).all() and (e <= hi.astype(np.float64)).all()
    w = L.ordinal32(hi) - L.ordinal32(lo)
    normal = e > 2.0 ** -125
    assert (w[normal] >= 3).all() and (w[normal] <= 7).all(), (w.min(), w.max())      # 4 or more fp32 values
    assert L.exp_range(np.float32([0]))[0][0] < 1 < L.exp_range(np.float32([0]))[1][0]


def _fc_inputs(dist, w, b):
    last = _emulated(dist, w, b)[-1]
    return last, L.fc1_emulated(w, last, dist)


@pytest.mark.parametrize("dist", [False, True], ids=["value", "dist"])
def test_fp16_emulation_lies_in_the_fc1_and_head_sets(fam, dist):
    """fc1 emulated as an fp32 accumulation of the exact products, the head restated with a correctly rounded exp; prints the fraction of
    the fc1 bound used and the width of the head's admissible sets in fp32 ulps."""
    b = np.concatenate(list(fam.values()))
    print("\n[%s] fc1 bound used (max)   head set width in ulps (median / max)" % ("dist_fp16" if dist else "net_fp16"))
    for wname, w in _weight_families(dist).items():
        last, d = _fc_inputs(dist, w, b)
        c = L.Fc1Check(w, last, d, dist)
        assert c.bad() == 0, c.describe(wname)
        hc = L.HeadCheck(w, d, L.head_outputs(w, d, dist), dist)
        assert hc.bad() == 0, hc.describe(wname)
        print("  %-14s %.4f              %4.1f / %d" % (wname, float(c.used.max()), float(np.median(hc.width)), int(hc.width.max())))


def _old_contract(dist, w, wname, b, out):
    """largest error / bound of the whole-network output contract; <= 1 accepts"""
    if dist:
        ref, _ = R.distnet(w, b, ATOMS)
        return D.prob_excess(out, ref, D.logit_bound(w, b, ATOMS, R.ALLOWANCE.get(wname)))
    v, var, _ = R.valuenet(w, b)
    sv, svar = H.out_sensitivity(w, b, R.ALLOWANCE.get(wname))
    return max(H.out_excess(out[:, 0], v, sv), H.out_excess(out[:, 1], var, svar))


@pytest.mark.parametrize("dist", [False, True], ids=["value", "dist"])
def test_fc_mutants_are_flagged_on_every_weight_family(fam, dist):
    """The last fc1 k block dropped, fc1's bias added twice or left out, ReLU for LeakyReLU in the distributional fc1 epilogue, fc_out /
    fc_v weights transposed within a 16-column block: each is flagged by the fc1 or head check on every weight family.  A
    reciprocal-multiply for the softmax division and the fast-math exp are measured only (f16_layer_ref.FC_MEASURED_ONLY).  The table
    records whether the whole-network output contract accepts each."""
    b = np.concatenate(list(fam.values()))
    print("\n[%s] fc mutant        weight family   flagged fc1 / head   old output contract (error / bound; <= 1 accepts)" %
          ("dist_fp16" if dist else "net_fp16"))
    for wname, w in _weight_families(dist).items():
        last, d = _fc_inputs(dist, w, b)
        for m in L.FC_MUTANTS:
            if not L.fc_mutant_applies(m, dist):
                continue
            dm = L.fc1_emulated(w, last, dist, m) if m == "drop_kblock" else d
            out = L.head_outputs(w, dm, dist, m)
            n1, n2 = L.Fc1Check(w, last, dm, dist).bad(), L.HeadCheck(w, dm, out, dist).bad()
            ratio = _old_contract(dist, w, wname, b, out)
            print("  %-16s %-14s %7d / %-7d      %9.3f  %s" % (m, wname, n1, n2, ratio, "accepts" if ratio <= 1 else "rejects"))
            assert n1 + n2 > 0 or m in L.FC_MEASURED_ONLY, (m, wname)
