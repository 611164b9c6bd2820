"""The float64 reference (tests/f64_ref.py) pinned before anything is measured against it: it must agree, to fp32 accuracy, with the
outputs recorded from the reference's own torch modules (valuenet / distnet / train goldens) and with the C oracle's restatements."""
import os

import numpy as np
import pytest
import torch

import f64_ref as R

GOLD = os.path.join(os.path.dirname(__file__), "golden")
RTOL = 1e-6          # the goldens are fp32 results: a handful of ulp away from the exact value


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.max(np.abs(a - b) / np.abs(b)))


def test_weight_generators_match_the_product():
    from tetris_mcts_b200.agents.DistValueSimOnline import init_dist_weights
    from tetris_mcts_b200.model.model_vv import init_weights
    assert np.array_equal(R.init_weights(3), init_weights(3))
    assert np.array_equal(R.dist_init_weights(3, 50), init_dist_weights(3))


def test_valuenet_matches_reference_golden():
    z = np.load(os.path.join(GOLD, "valuenet_golden.npz"))
    for seed in z["seeds"]:
        v, var, _ = R.valuenet(R.init_weights(int(seed)), z["states"])
        assert rel(v, z["v_%d" % seed]) < RTOL and rel(var, z["var_%d" % seed]) < RTOL


def test_distnet_matches_reference_golden():
    z = np.load(os.path.join(GOLD, "distnet_golden.npz"))
    p, _ = R.distnet(R.dist_init_weights(int(z["seed"]), 50), z["states"], 50)
    assert np.allclose(p, z["dist"], rtol=1e-6, atol=1e-8), np.abs(p - z["dist"]).max()
    assert np.allclose(p.sum(1), 1.0, atol=1e-12)


@pytest.mark.parametrize("tag,weighted,clip", [("w", True, 0.0), ("u", False, 0.0), ("c", True, 0.5)])
def test_train_loss_and_grads_match_reference_golden(tag, weighted, clip):
    """Step 1 of the recorded training runs: loss, loss_std, gradient norm and the gradients (after clip_grad_norm_ for "c")."""
    z = np.load(os.path.join(GOLD, "train_golden.npz"))
    w = R.init_weights(int(z["seed"]))
    w[R.N_TRAIN:R.N_TRAIN + 2] = z["ubound"]
    r = R.train_loss_and_grads(w, [z["states"], z["value"], z["variance"], z["weight"]], weighted)
    loss, loss_std, gnorm = z[tag + "_steps"][0]
    assert rel(r["loss"], loss) < RTOL and rel(r["loss_std"], loss_std) < RTOL
    assert rel(r["grad_norm"], gnorm) < 1e-5          # the recorded norm is a sum of fp32 per-tensor norms
    g = r["grad_flat"] * (min(1.0, clip / (r["grad_norm"] + 1e-6)) if clip else 1.0)
    want = z[tag + "_grad0"]
    keep = z["keep_index"]
    names = [n for n, _ in R.VN_SHAPES[:10]]
    off = 0
    for n in names:                                   # every tensor within 1e-5 of its own norm
        size = R.grads_size(n)
        sel = (keep >= off) & (keep < off + size)
        got, ref = g[keep[sel]], want[sel]
        assert np.abs(got - ref).max() <= 1e-5 * np.linalg.norm(ref), (n, np.abs(got - ref).max(), np.linalg.norm(ref))
        off += size


def test_fp32_restatement_of_the_loss_agrees():
    """The fp32 variant of the same code (used where the device trainer's fp32 activation storage dominates) is the fp64 one to 1e-5."""
    z = np.load(os.path.join(GOLD, "train_golden.npz"))
    w = R.init_weights(0)
    w[R.N_TRAIN:R.N_TRAIN + 2] = z["ubound"]
    b = [z["states"], z["value"], z["variance"], z["weight"]]
    a, c = R.train_loss_and_grads(w, b, True), R.train_loss_and_grads(w, b, True, dtype=torch.float32)
    assert rel(c["loss"], a["loss"]) < 1e-5 and rel(c["grad_norm"], a["grad_norm"]) < 1e-5


def test_valuenet_families_match_the_c_oracle(oracle):
    boards = np.concatenate(list(R.board_families(oracle).values()))
    for name, w in R.weight_families(0).items():
        v, var, _ = R.valuenet(w, boards)
        ov, ovar = oracle.valuenet_forward(w, boards)
        assert rel(ov, v) < 2e-6 and rel(ovar, var) < 2e-6, name


@pytest.mark.parametrize("atoms", [2, 50, 64])
def test_distnet_families_match_the_c_oracle(oracle, atoms):
    boards = np.concatenate(list(R.board_families(oracle).values()))
    for name, w in R.dist_weight_families(1, atoms).items():
        p, logits = R.distnet(w, boards, atoms)
        o = oracle.distnet_forward(w, boards, atoms)
        bound = 1e-5 + 8 * 2.0 ** -24 * np.abs(logits).max()
        assert np.all(np.abs(o - p) <= bound * p + 1e-30), (name, atoms)


def test_board_families_cover_the_edges(oracle):
    fam = R.board_families(oracle)
    imp = fam["impulse"]
    assert len(imp) == 400 and all((np.abs(b) == 1).sum() == 1 for b in imp)
    piece_cells = [np.argwhere(b == -1) for b in fam["bottom_and_col9"]]
    assert any((c[:, 1] == 9).any() for c in piece_cells) and all((c[:, 0] >= 13).all() for c in piece_cells)
    assert sorted({int((b == -1).sum()) for b in fam["partial_piece"]}) == [1, 2, 3]
    assert (fam["full_rows"][:, 19] == 1).all() and not fam["empty"][0].any()
    for w in R.weight_families(0).values():
        assert R.split_max(w) * 64 < 65504                          # all families load on the tensor-core path


def test_subnormal_family_sits_in_the_low_term_subnormal_regime(oracle):
    """Normal high fp16 term, subnormal low term: 2^-18 <= |a| < 2^-7 for the activations, |w| < 2^-9 for conv1 and fc1."""
    import torch.nn.functional as F
    from arena_gen import boards
    b = np.concatenate(list(R.board_families(oracle).values()) + [boards(300, 3)])
    p = R.unpack(R.weight_families(0)["subnormal"], R.VN_SHAPES)
    a = R._x(b, torch.float64)
    for l in (1, 2, 3):
        a = F.relu(F.conv2d(a, p["conv%d.weight" % l], p["conv%d.bias" % l]))
        nz = a[a > 0]
        assert ((nz >= 2.0 ** -18) & (nz < 2.0 ** -7)).double().mean() > 0.9, l
    assert float(p["conv1.weight"].abs().max()) < 2.0 ** -9 and float(p["fc1.weight"].abs().max()) < 2.0 ** -9


def test_act3_bound_tells_the_split_from_a_single_fp16(oracle):
    """The layer check's bound (2^-19 T3 per board + ACT_FLOOR) holds for act3 stored as the two fp16 terms, subnormal low terms
    included, and fails for act3 kept as the high term alone: on every weight family, the subnormal one in particular."""
    from arena_gen import boards
    b = np.concatenate(list(R.board_families(oracle).values()) + [boards(300, 3)])
    for name, w in R.weight_families(0).items():
        v, var, a3 = R.valuenet(w, b)
        _, _, t3 = R.valuenet_sensitivity(w, b)
        bound = 2.0 ** -19 * t3.max(1, keepdims=True) + R.ACT_FLOOR
        assert (np.abs(R.split_act(a3, 2) - a3) / bound).max() < 0.25, name
        assert (np.abs(R.split_act(a3, 1) - a3) / bound).max() > 4, name
        sv, svar, _ = R.valuenet_sensitivity(w, b, R.ALLOWANCE.get(name))       # and the outputs of the split act3 meet their bound
        v2, var2 = R.valuenet_head(w, R.split_act(a3, 2))
        assert np.all(np.abs(v2 - v) <= 1e-5 * np.abs(v) + sv) and np.all(np.abs(var2 - var) <= 1e-5 * np.abs(var) + svar), name
