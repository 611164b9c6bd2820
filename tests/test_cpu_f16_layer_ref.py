"""The layer-by-layer check of tests/f16_layer_ref.py pinned on the CPU before the device is held to it.

- numpy's float32 -> float16 cast, which the restatement uses for the loader's weights and for the epilogue, rounds like __float2half_rn on
  the subnormal and overflow edges.
- The float64 emulations of net_fp16 and dist_fp16 (tests/f16_ref.py, tests/f16_dist_ref.py) fall inside the admissible set of every
  element of every layer, on every weight family and board family.
- Each deliberate defect of those emulations (f16_ref.MUTANTS, and bfloat16 for fp16) is flagged on every weight family it applies to,
  while the whole-network contracts (f16_ref.act3_bound, f16_dist_ref.act2_bound) accept most of them: the printed table is the measure.
- The two-term form accepts a canonical split and flags a pair with the same sum that is not canonical."""
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
