"""The net_fp16 error contract (tests/f16_ref.py) pinned on the CPU before the device is held to it: a float64 emulation of one fp16 term
per operand sits well inside the act3 and output bounds on every weight family, and the act3 bound is tight enough that the same
emulation with bfloat16 (8 significant bits instead of 11) breaks it on every family.  Without the second half the bound would not test
the precision at all.  Measured ratios (largest error / bound): act3 fp16 0.15 .. 0.31, bf16 1.11 .. 2.80; outputs fp16 <= 0.10."""
import numpy as np
import pytest
import torch

import f16_ref as H
import f64_ref as R


def test_act3_bound_holds_for_fp16_and_fails_for_bf16(oracle):
    from arena_gen import boards
    b = np.concatenate(list(R.board_families(oracle).values()) + [boards(300, 3)])
    for name, w in R.weight_families(0).items():
        v, var, a3 = R.valuenet(w, b)
        bound = H.act3_bound(w, b)
        _, _, e16 = H.emulate(w, b, torch.float16)
        _, _, ebf = H.emulate(w, b, torch.bfloat16)
        r16, rbf = (np.abs(e16 - a3) / bound).max(), (np.abs(ebf - a3) / bound).max()
        assert r16 < 0.4, (name, r16)
        assert rbf > 1, (name, rbf)


def test_outputs_of_the_fp16_emulation_meet_their_bound(oracle):
    from arena_gen import boards
    b = np.concatenate(list(R.board_families(oracle).values()) + [boards(300, 3)])
    for name, w in R.weight_families(0).items():
        v, var, _ = R.valuenet(w, b)
        sv, svar = H.out_sensitivity(w, b, R.ALLOWANCE.get(name))
        v16, var16, _ = H.emulate(w, b, torch.float16)
        assert H.out_excess(v16, v, sv) < 0.25 and H.out_excess(var16, var, svar) < 0.25, name


def test_fp16_emulation_is_not_the_split():
    """One fp16 term differs from the float64 network by far more than the split does: the emulation is not accidentally exact."""
    w = R.init_weights(0)
    from arena_gen import boards
    b = boards(64, 5)
    v, _, a3 = R.valuenet(w, b)
    v16, _, e16 = H.emulate(w, b, torch.float16)
    assert np.abs(e16 - a3).max() > 100 * np.abs(R.split_act(a3, 2) - a3).max()
    assert np.abs(v16 - v).max() > 0


def test_play_batched_keeps_net_tc_as_its_default():
    from tetris_mcts_b200 import play_batched as PB
    assert PB.parse_args([]).eval_kind == "net_tc"
    assert PB.parse_args(["--eval_kind", "net_fp16"]).eval_kind == "net_fp16"
    with pytest.raises(SystemExit):
        PB.parse_args(["--eval_kind", "synthetic"])
