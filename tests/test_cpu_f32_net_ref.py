"""The stage-by-stage restatement of the fp32 CUDA-core networks (tests/f32_net_ref.py) pinned on the CPU before the device is held to it.

- The fast exact fma agrees with f16_layer_ref.fma32 and with exact rational arithmetic, midpoints and subnormals included; both follow
  IEEE on +-inf and NaN operands.  (The device check compares NaN with NaN and zeros by value: f32_net_ref.same.)
- The key decode keeps four piece cells, as the observation key does.
- The restatement is the reference network and not only the kernels' order: on every weight family and board family it meets the old
  allowances against float64 (act3 within 2^-19 T3 + 2^-26, outputs within rtol 1e-5 plus the ill-conditioned families' allowances,
  probabilities within (1e-5 + 2 e_z) p + 1e-36), and it lies in its own sets (trivially, except for the head).
- Each deliberate defect (f32_net_ref.NET_MUTANTS) is flagged on every weight family it changes; the printed table records which of them
  the old allowances accept."""
from fractions import Fraction

import numpy as np
import pytest

import f16_layer_ref as L
import f32_net_ref as N
import f64_ref as R
from test_cpu_f16_layer_ref import _rn32

ATOMS = 50
F = np.float32


@pytest.fixture(scope="module")
def fam(oracle):
    return R.board_families(oracle)


def _families(dist, huge=False):
    f = dict(R.dist_weight_families(5, ATOMS) if dist else R.weight_families(0))
    if huge:
        f["huge"] = N.huge_dist_weights(5, ATOMS) if dist else N.huge_value_weights(0)
    return f


def _f64(x):
    return np.asarray(x, np.float32).astype(np.float64)


def test_fast_fma_is_exact():
    """Products on fp32 midpoints with tiny addends on either side (where a float64 fma rounded again to fp32 ties the wrong way),
    subnormal results and ties, the overflow threshold, cancellation and 200000 random triples: the fast fma equals fma32 everywhere and
    exact rational arithmetic on the constructed cases and 3000 random ones."""
    mx = float(np.finfo(np.float32).max)
    cases = [(1 + 2.0 ** -12, 1 + 2.0 ** -12, 2.0 ** -80), (1 + 2.0 ** -12, 1 + 2.0 ** -12, -(2.0 ** -80)), (3.0, 1 + 2.0 ** -23, -(2.0 ** -80)),
             (3.0, 1 + 2.0 ** -23, 2.0 ** -80), (3.0, 1 + 2.0 ** -23, 0.0), (3 * 2.0 ** -75, 2.0 ** -75, 0.0), (3 * 2.0 ** -75, 2.0 ** -75, 2.0 ** -149),
             (2.0 ** -75, 2.0 ** -75, -(2.0 ** -149)), (2.0 ** -149, 0.5, 0.0), (2.0 ** -126, 0.75, -(2.0 ** -149)), (mx, 1.0, 2.0 ** 103),
             (mx, 1.0, 2.0 ** 103 - 2.0 ** 79), (-mx, 1.0, -(2.0 ** 103)), (mx, 2.0, -mx), (2.0 ** 127, 2.0, 0.0), (1.0, -1.0, 1.0)]
    rng = np.random.default_rng(5)
    n = 200000
    m = rng.integers(1 << 23, 1 << 24, (3, n)).astype(np.float64) * rng.choice([-1.0, 1.0], (3, n))
    ex = rng.integers(-75, 40, (3, n))
    ex[2, : n // 3] = ex[0, : n // 3] + ex[1, : n // 3] + rng.integers(-30, 5, n // 3)
    a, b, c = (np.ldexp(m[i], ex[i] - 23).astype(np.float32) for i in range(3))
    A, B, C = (np.concatenate([np.array([t[i] for t in cases], np.float32), x]) for i, x in enumerate((a, b, c)))
    with np.errstate(over="ignore"):
        got = N.fma(_f64(A), _f64(B), _f64(C)).astype(np.float32)
        ref = L.fma32(A, B, C)
    assert np.array_equal(got.view(np.uint32), ref.view(np.uint32))
    k = len(cases) + 3000
    want = [_rn32(Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z))) for x, y, z in zip(A[:k], B[:k], C[:k])]
    bad = [(A[i], B[i], C[i], got[i], want[i]) for i in range(k) if not float(got[i]) == want[i]]
    assert not bad, bad[:5]
    assert (N.fma(_f64(A[:k]), _f64(B[:k]), _f64(C[:k])) != N.round32(_f64(A[:k]) * _f64(B[:k]) + _f64(C[:k]))).sum() >= 2   # the fallback ran


def test_fma_on_inf_and_nan():
    """IEEE fma: inf times a non-zero finite is inf, inf times 0 is NaN, inf - inf is NaN, NaN anywhere gives NaN, and a finite product
    beyond fp32's range added to an opposite addend rounds once (no intermediate overflow)."""
    inf, nan, mx = np.inf, np.nan, float(np.finfo(np.float32).max)
    cases = [(inf, 1.0, 1.0, inf), (inf, -2.0, 5.0, -inf), (-inf, -1.0, 5.0, inf), (inf, 0.0, 1.0, nan), (0.0, -inf, 1.0, nan),
             (inf, 1.0, -inf, nan), (1.0, -inf, inf, nan), (2.0, 3.0, inf, inf), (2.0, 3.0, -inf, -inf), (1.0, 1.0, nan, nan),
             (nan, 0.0, 1.0, nan), (1.0, nan, inf, nan), (mx, 2.0, -mx, mx), (mx, 2.0, 0.0, inf), (-mx, 2.0, 0.0, -inf), (mx, 1.0, mx, inf)]
    A, B, C, W = (np.array([t[i] for t in cases], np.float32) for i in range(4))
    with np.errstate(over="ignore", invalid="ignore"):
        for got in (L.fma32(A, B, C), N.fma(_f64(A), _f64(B), _f64(C)).astype(np.float32)):
            assert np.array_equal(got, W, equal_nan=True), list(zip(cases, got))
    assert N.same(np.float32([np.nan, -0.0, 0.0, 1.0]), [np.nan, 0.0, -0.0, 1.0]).all()
    assert not N.same(np.float32([np.nan, 1.0, np.inf]), [1.0, np.nextafter(F(1), F(2)), -np.inf]).any()


def test_key_decode_keeps_four_piece_cells():
    s = np.zeros((2, 200), np.int8)
    s[0, [3, 50, 77, 120, 199]] = -1                   # five negative cells: the key holds the first four
    s[0, [0, 198]] = 1
    s[1, 10] = -1
    x = N.board_input(s)
    assert x[0].ravel()[[3, 50, 77, 120]].tolist() == [-1] * 4 and x[0].ravel()[199] == 0 and x[0].ravel()[[0, 198]].tolist() == [1, 1]
    assert x[1].ravel()[10] == -1 and (np.abs(x[1]).sum() == 1)
    xd = N.board_input(s, dist=True)
    assert xd.shape == (2, 22, 10) and not xd[:, :2].any() and np.array_equal(xd[:, 2:], x)


@pytest.mark.parametrize("dist", [False, True], ids=["value", "dist"])
def test_restatement_is_the_reference_network_and_lies_in_its_own_sets(fam, dist):
    """Every weight family x every board family: the old allowances against float64 hold, and every stage of the restatement (with a
    correctly rounded exp) lies in its own set; prints the error / bound and the head set widths."""
    b = np.concatenate(list(fam.values()))
    print("\n[net %s] family          old allowance (error / bound)   head set width (median / max ulps)" % ("dist" if dist else "value"))
    for wname, w in _families(dist).items():
        st = N.forward(w, b, dist)
        c = N.StageCheck(w, b, {k: v.astype(np.float32) for k, v in st.items()}, dist)
        assert c.total() == 0, c.describe(wname)
        ratio = _old_allowance(dist, w, wname, b, st)
        print("  %-14s  %s   %.1f / %d" % (wname, " ".join("%s %.3f" % kv for kv in ratio.items()), float(np.median(c.width)), int(c.width.max())))
        assert max(v for k, v in ratio.items() if k != "rtol") <= 1, (wname, ratio)


def _old_allowance(dist, w, wname, b, st):
    """the old checks, error / bound (<= 1 accepts): value: act3 (2^-19 T3_max + 2^-26 per board), v and var (rtol 1e-5 + the family's
    allowance); distributional: probabilities ((1e-5 + 2 e_z) p + 1e-36) and the golden check's rtol 1e-5 / atol 1e-7"""
    out = np.asarray(st["out"], np.float64)
    if dist:
        ref, _ = R.distnet(w, b, ATOMS)
        ez = R.distnet_sensitivity(w, b, ATOMS, R.ALLOWANCE.get(wname))[:, None]
        with np.errstate(invalid="ignore"):
            return {"p": float(np.nanmax(np.abs(out - ref) / ((1e-5 + 2 * ez) * ref + 1e-36), initial=0) if np.isfinite(out).all() else np.inf),
                    "rtol": float(np.max(np.abs(out - ref) / (1e-5 * np.abs(ref) + 1e-7)) if np.isfinite(out).all() else np.inf)}
    v, var, a3 = R.valuenet(w, b)
    sv, svar, t3 = R.valuenet_sensitivity(w, b, R.ALLOWANCE.get(wname))
    bound = 2.0 ** -19 * t3.max(1, keepdims=True) + R.ACT_FLOOR
    got3 = np.asarray(st["act3"], np.float64).reshape(len(b), -1)
    r3 = float(np.max(np.abs(got3 - a3) / bound)) if np.isfinite(got3).all() else np.inf
    ro = max(float(np.max(np.abs(out[:, 0] - v) / (1e-5 * np.abs(v) + sv))), float(np.max(np.abs(out[:, 1] - var) / (1e-5 * np.abs(var) + svar))))
    return {"act3": r3, "out": ro if np.isfinite(out).all() else np.inf}


def _mutant_forward(w, b, dist, clean, m):
    """the mutant network from its first changed stage on (earlier stages are the clean ones) -> dict stage -> fp32"""
    stages = N.DN_STAGES if dist else N.VN_STAGES
    first = stages.index(N.MUTANT_STAGES[dist][m][0])
    st = {s: clean[s] for s in stages[:first]}
    for i in range(first, len(stages)):
        s = stages[i]
        prev = st[stages[i - 1]] if i else None
        if s == "out":
            st[s] = N.head_outputs(w, prev, dist, m)
        elif s.startswith("act"):
            st[s] = N.conv_layer(w, b if s == "act1" else prev, dist, int(s[3:]), m)
        elif s == "fc1":
            st[s] = N.fc1(w, prev, dist, m)
        else:
            st[s] = N.dist_logits(w, prev, m)
        st[s] = np.asarray(st[s], np.float32)
    return st


def _flagged(w, b, dist, st, m):
    """elements out of their restated set, over the stages from the mutant's first one on, each restated from the mutant's own previous stage"""
    stages = N.DN_STAGES if dist else N.VN_STAGES
    n = 0
    for i in range(stages.index(N.MUTANT_STAGES[dist][m][0]), len(stages)):
        s = stages[i]
        want = N.stage_from(w, b, st[stages[i - 1]] if i else None, s, dist)
        n += int((~(N.in_set(st[s], *want) if s == "out" else N.same(st[s], want))).sum())
    return n


@pytest.mark.parametrize("dist", [False, True], ids=["value", "dist"])
def test_mutants_are_flagged_on_every_weight_family_they_change(fam, dist):
    """Each mutant of f32_net_ref.NET_MUTANTS that applies to this network, on every weight family and `huge`: flagged by the stage
    check wherever it changes a value (except NET_MEASURED_ONLY, measured); the table records whether the old allowances accept it."""
    b = np.concatenate([fam["real"][:24], fam["partial_piece"][:8], fam["full_rows"][:4]])
    print("\n[net %s] mutant              family          changed   flagged   old allowances (error / bound; <= 1 accepts)" %
          ("dist" if dist else "value"))
    missed = []
    for wname, w in _families(dist, huge=True).items():
        clean = {k: np.asarray(v, np.float32) for k, v in N.forward(w, b, dist).items()}
        for m in N.MUTANT_STAGES[dist]:
            st = _mutant_forward(w, b, dist, clean, m)
            changed = int(sum((~N.same(st[s], clean[s])).sum() for s in st))
            n = _flagged(w, b, dist, st, m) if changed else 0
            old = _old_allowance(dist, w, wname, b, st) if wname != "huge" else {}
            print("  %-19s %-14s %8d %9d   %s" % (m, wname, changed, n, " ".join("%s %.3g (%s)" % (k, v, "accepts" if v <= 1 else "rejects")
                                                                                  for k, v in old.items())))
            if changed and not n and m not in N.NET_MEASURED_ONLY:
                missed.append((m, wname))
    assert not missed, missed
