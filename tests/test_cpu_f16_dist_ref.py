"""The dist_fp16 error contract (tests/f16_dist_ref.py) pinned on the CPU before the device is held to it: a float64 emulation of one fp16
term per operand uses at most about half of the act2 and probability bounds on every distributional weight family, board family and atom
count, and the act2 bound is tight enough that the same emulation with bfloat16 (8 significant bits instead of 11) breaks it on every
family.  Measured ratios (largest error / bound): act2 fp16 0.155, bf16 1.06 .. 1.07; probabilities fp16 <= 0.002."""
import numpy as np
import pytest
import torch

import f16_dist_ref as D
import f64_ref as R


@pytest.fixture(scope="module")
def allb(oracle):
    return np.concatenate(list(R.board_families(oracle).values()))


@pytest.mark.parametrize("atoms", [2, 33, 50, 64])
def test_act2_bound_holds_for_fp16_and_fails_for_bf16(allb, atoms):
    for name, w in R.dist_weight_families(5, atoms).items():
        ref = D.act2(w, allb, atoms)
        bound = D.act2_bound(w, allb, atoms)
        _, e16 = D.emulate(w, allb, atoms, torch.float16)
        _, ebf = D.emulate(w, allb, atoms, torch.bfloat16)
        r16, rbf = (np.abs(e16 - ref) / bound).max(), (np.abs(ebf - ref) / bound).max()
        assert r16 < 0.5, (name, atoms, r16)
        assert rbf > 1, (name, atoms, rbf)


@pytest.mark.parametrize("atoms", [2, 33, 50, 64])
def test_probabilities_of_the_fp16_emulation_meet_their_bound(allb, atoms):
    for name, w in R.dist_weight_families(5, atoms).items():
        ref, _ = R.distnet(w, allb, atoms)
        p16, _ = D.emulate(w, allb, atoms, torch.float16)
        ez = D.logit_bound(w, allb, atoms, R.ALLOWANCE.get(name))
        assert D.prob_excess(p16, ref, ez) < 0.5, (name, atoms)
        assert np.abs(p16.sum(1) - 1).max() < 1e-12, (name, atoms)


def test_fp16_emulation_is_not_the_split():
    """One fp16 term differs from the float64 network by far more than the split does: the emulation is not accidentally exact."""
    from arena_gen import boards
    w = R.dist_init_weights(0, 50)
    b = boards(64, 5)
    ref = D.act2(w, b, 50)
    _, e16 = D.emulate(w, b, 50, torch.float16)
    assert np.abs(e16 - ref).max() > 100 * np.abs(R.split_act(ref, 2) - ref).max()
    p, _ = R.distnet(w, b, 50)
    assert np.abs(D.emulate(w, b, 50)[0] - p).max() > 0


def test_engine_maps_the_kind_name():
    from tetris_mcts_b200 import _lib as L
    assert L.EVAL_DIST_FP16 == 4 and L.EVAL_NET_FP16 == 3
    from tetris_mcts_b200.agents.DistValueSimOnline import DistValueSim
    import inspect
    assert 'kwargs.pop("eval_kind", "net")' in inspect.getsource(DistValueSim.__init__)     # the agent's default stays "net"
