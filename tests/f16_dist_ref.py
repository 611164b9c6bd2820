"""The error contract of eval_kind dist_fp16 (the distributional network with one fp16 term per operand and one product per product:
distnet_tc.cuh with NT = 1) and a float64 emulation of that arithmetic, for the tests that hold the device to it.  tests/f16_ref.py
does the same for the value network's net_fp16; the steps below are the same ones applied to model_distributional.py's layers.

Every operand the tensor cores read is scaled by an exact power of two (activations x16, conv / fc1 weights x64) and rounded once to fp16,
x1 = fp16(x): |x - x1| <= 2^-11 |x| in the normal range.  The input board is exact ({-1, 0, 1}), fc_v and the softmax stay fp32.
act2 (per element, per board): |d| <= 2^-10 T2_max + ACT_FLOOR, T2 = |a1| * |W2| + |b2| (the sum of |terms| of each act2 element, 512 per
    element), |a1| the absolute conv1 activations of the float64 network.
    The relative part is c 2^-11 with c = 2.  act2's own rounding to fp16 on the way to HBM is a worst case of 2^-11 |a2| <= 2^-11 T2_max
    (c = 1): LeakyReLU(0.01) keeps a relative error relative (|leaky(x) - leaky(y)| <= |x - y| and it never grows |x|).  The other three
    roundings (conv1's weights and its output act1, conv2's weights) enter act2 through sums of 512 products with independent signs, so they
    grow like sqrt(512) 2^-11 times the typical term, not like the |term| sum T2: 3 / sqrt(512) ~ 0.13 of 2^-11 T2 per standard deviation,
    and the second 2^-11 T2_max (c = 2 in all) is ~7 of those, with the fp32 sums (2^-24 per addition) negligible beside it.  This part is a
    statistical allowance, as in the value network's contract; the worst case of a sum of |terms| (c = 4) would let bfloat16 through
    (at 0.53 of it).
    ACT_FLOOR (2^-26, f64_ref.ACT_FLOOR) is the split's floor and still covers one term: below fp16's normal range (16 |a| < 2^-14,
    64 |w| < 2^-14) the rounding error is absolute, at most 2^-29 per activation and 2^-31 per weight; act2's own floor and act1's carried
    through a row of W2 (2-norm ~0.6 in the init family) stay under 2^-28, a quarter of the floor.
probabilities: |d p| <= 2 e_z p + 1e-36 (p_i = exp(z_i - z_max) / sum: d p_i / p_i = d z_i - sum_j p_j d z_j, so |d p_i| <= 2 max |d z| p_i).
    e_z bounds the logit error per board: DZ_K S_fc1, S_fc1 = (|a2| . |W_fc1|^T + |b_fc1|) . |W_v|^T (max over atoms), the fc1 terms
    carried into the logit through |W_v|, with DZ_K = 4 * 2^-11: act2's relative part (c = 2), fc1's rounded weight (1) and one more for
    act2's rounding of small elements, which the element-wise T2_max bound lets exceed 2^-10 |a2|.  On top of it, the `saturated` and
    `subnormal` families keep the fp32 allowances of f64_ref.distnet_sensitivity ("cond": fc_v's own fp32 sums against a bias of +-60;
    "floor": the split's floor carried into the logits).  1e-36 absorbs fp32 underflow of the smallest probabilities.
Measured on the float64 emulation below (tests/test_cpu_f16_dist_ref.py), as the largest error / bound over f64_ref.dist_weight_families
x f64_ref.board_families x atoms 2, 33, 50, 64:
    act2           fp16 0.155         bf16 1.06 .. 1.07 (every family breaks the bound)
    probabilities  fp16 <= 0.002      bf16 <= 0.013
The probability bound is loose by design (a sum of |terms| through |W_v|, as the value network's `saturated` allowance is): it guards
against a wrong logit, while the act2 check is the one that tells fp16 from a coarser format.
"""
import numpy as np
import torch
import torch.nn.functional as F

import f16_ref as H
import f64_ref as R

ACT2_REL = 2.0 ** -10          # c 2^-11, c = 2
DZ_K = 4 * 2.0 ** -11          # logit error per unit of S_fc1


def _pad(states, dtype=torch.float64):
    return F.pad(R._x(states, dtype), (0, 0, 2, 0))             # two empty rows on top: 22x10 (model_distributional.py:27)


def act2_bound(w, states, atoms):
    """per board: ACT2_REL * T2_max + ACT_FLOOR, shape [n, 1]"""
    p = R.unpack(w, R.dn_shapes(atoms))
    with torch.no_grad():
        a1 = F.leaky_relu(F.conv2d(_pad(states), p["conv1.weight"], p["conv1.bias"]), 0.01)
        t2 = F.conv2d(a1.abs(), p["conv2.weight"].abs(), p["conv2.bias"].abs()).flatten(1)
    return ACT2_REL * t2.numpy().max(1, keepdims=True) + R.ACT_FLOOR


def act2(w, states, atoms):
    """float64 act2 in torch flatten order c*64 + y*4 + x (the order b200_debug_dist_act2 returns)"""
    p = R.unpack(w, R.dn_shapes(atoms))
    with torch.no_grad():
        a = F.leaky_relu(F.conv2d(_pad(states), p["conv1.weight"], p["conv1.bias"]), 0.01)
        return F.leaky_relu(F.conv2d(a, p["conv2.weight"], p["conv2.bias"]), 0.01).flatten(1).numpy()


def logit_bound(w, states, atoms, allowance=None):
    """e_z per board, shape [n, 1] (see the module docstring)"""
    p = R.unpack(w, R.dn_shapes(atoms))
    with torch.no_grad():
        a = torch.from_numpy(act2(w, states, atoms))
        s_fc1 = (a.abs() @ p["fc1.weight"].abs().T + p["fc1.bias"].abs()) @ p["fc_v.weight"].abs().T
    ez = DZ_K * s_fc1.max(1).values.numpy()
    return (ez + R.distnet_sensitivity(w, states, atoms, allowance))[:, None]


def prob_excess(got, ref, ez):
    """largest |got - ref| / (2 e_z ref + 1e-36); <= 1 passes"""
    return float(np.max(np.abs(np.asarray(got, np.float64) - ref) / (2 * ez * ref + 1e-36)))


def _leaky_round(t, scale, dtype, rz=False):
    """the epilogue on t * scale: fp32 rounding (the fma), x > 0 ? x : 0.01f * x in fp32, rounding to `dtype` (toward zero with rz);
    over scale"""
    s = (t * scale).to(torch.float32)
    s = torch.where(s > 0, s, s * torch.tensor(0.01, dtype=torch.float32))
    return (H._rz16(s) if rz else s.to(dtype).to(torch.float64)) / scale


_round = H._round


def emulate_layers(w, states, atoms, dtype=torch.float16, mutant=None):
    """The conv stack of emulate: [act1, act2] as float64 tensors [n, 32, H, W] (each element an fp16 term / 16); mutant: one of
    f16_ref.MUTANTS, as there."""
    p = R.unpack(w, R.dn_shapes(atoms))
    for k in R.SPLIT_DN:
        p[k] = _round(p[k], 64.0, dtype, mutant == "rz_weight")
    if mutant == "no_conv2_block":
        p["conv2.weight"][:, :16, 0] = 0
    sa = 8.0 if mutant == "scale8" else 16.0
    a, out = _pad(states), []
    with torch.no_grad():
        for l in (1, 2):
            wl, bl = p["conv%d.weight" % l], p["conv%d.bias" % l]
            if mutant == "bias_after":
                a = F.leaky_relu(_round(F.conv2d(a, wl), sa, dtype) + bl[None, :, None, None], 0.01)
            else:
                a = _leaky_round(F.conv2d(a, wl, bl), sa, dtype, mutant == "rz_act")
            out.append(a)
    return out


def emulate(w, states, atoms, dtype=torch.float16):
    """The dist_fp16 arithmetic in float64: every conv / fc1 weight (x64) and every conv activation (x16, after the epilogue's fp32
    rounding and fp32 LeakyReLU) rounded once to `dtype` (torch.float16 as the device does; torch.bfloat16 to show that the act2 bound
    tells a coarser format apart), exact sums.  -> (probabilities, act2) like f64_ref.distnet and act2 above."""
    p = R.unpack(w, R.dn_shapes(atoms))
    for k in R.SPLIT_DN:
        p[k] = _round(p[k], 64.0, dtype)
    with torch.no_grad():
        a2 = emulate_layers(w, states, atoms, dtype)[-1].flatten(1)
        h = F.leaky_relu(a2 @ p["fc1.weight"].T + p["fc1.bias"], 0.01)
        probs = torch.softmax(h @ p["fc_v.weight"].T + p["fc_v.bias"], 1)
    return probs.numpy(), a2.numpy()
