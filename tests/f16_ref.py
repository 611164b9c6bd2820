"""The error contract of eval_kind net_fp16 (one fp16 term per operand, one product per product: valuenet_tc.cuh with NT = 1) and a
float64 emulation of that arithmetic, for the tests that hold the device to it.

Derivation (the same steps test_gpu_net_precision's docstring takes for the fp16 x 2 split, with one term).  Every operand the tensor
cores read is scaled by an exact power of two (activations x16, conv / fc1 weights x64) and rounded once to fp16, x1 = fp16(x):
  - normal range: |x - x1| <= 2^-11 |x| (11 significant bits), against 2^-22 for x1 + x2.
  - subnormal floor and overflow: unchanged from the split, because the scaling is unchanged: absolute errors of at most 2^-29 per
    activation and 2^-31 per weight below fp16's normal range, infinities past |a| ~4094 / |w| ~1023.5 (weights refused at load).
  - a product a1*b1 of two rounded operands is within (2 + 2^-11) 2^-11 |ab| of ab; the sums run in fp32 (2^-24 per addition, negligible
    against 2^-11 even over 1792 terms).
act3 (per element, per board): |d| <= 2^-10 T3_max + ACT_FLOOR, T3 = |a2| * |W3| + |b3| as f64_ref.valuenet_sensitivity returns it.
    The relative part is c 2^-11 with c = 2.  act3's own rounding to fp16 on the way to HBM is a worst case of 2^-11 |a3| <= 2^-11 T3_max
    (c = 1).  The other six roundings (conv1: weight and output; conv2: weight, input and output; conv3: weight and input) enter act3
    through sums of 288 products (conv2 / conv3 rows of 2-norm ~0.6) with independent signs, so they grow like sqrt(288) 2^-11 times the
    typical term, not like the |term| sum T3: 6 / sqrt(288) ~ 0.35 of 2^-11 T3 per standard deviation, and one more 2^-11 T3_max
    (c = 2 in all) is ~3 of those, with the fp32 sums (2^-24 per addition) negligible beside it.  This part is a statistical allowance,
    as the split's 2^-19 is; the worst case of a sum of |terms| (c = 7) would not tell fp16 from bf16.  ACT_FLOOR (2^-26) is f64_ref's:
    the floors are the split's.
outputs: |d out| <= 2^-11 |out| + |d out / d z| A, A = 0 except for the two families f64_ref.ALLOWANCE names:
    `saturated` ("cond"): v = ub * sigmoid(z), z ~ -25: d v / v = d z, so v is as good as its logit's absolute error, which the fp16
      operands of fc1 set: A = 4 * 2^-11 S_fc1 (act3's relative part, c = 2, and fc1's two rounded operands, carried into z through
      |w_out|; the fp32 terms of the split's "cond" allowance are ~2^-9 of this and left out).
    `subnormal` ("floor"): the split's floor allowance, f64_ref.valuenet_sensitivity(..., "floor"), unchanged.
    On the other families |d out / out| = (1 - sigmoid(z)) |d z| and |z| is a few units: the fc1 sums and the act3 errors enter z with
    random signs, so its absolute error stays near 2^-11 / 10 and 2^-11 of |out| is a statistical allowance with head-room ~10.
Measured on the float64 emulation below (tests/test_cpu_f16_ref.py), as the largest error / bound over the weight families of
f64_ref.weight_families(0) on f64_ref.board_families(oracle) plus 300 random boards:
    act3     fp16 0.15 .. 0.31      bf16 1.11 .. 2.80 (every family breaks the bound)
    outputs  fp16 0.002 .. 0.10     bf16 up to 0.72
"""
import numpy as np
import torch
import torch.nn.functional as F

import f64_ref as R

ACT3_REL = 2.0 ** -10          # c 2^-11, c = 2
OUT_RTOL = 2.0 ** -11          # relative part of the output bound
COND_K = 4 * 2.0 ** -11        # "saturated": allowance on the logit per unit of S_fc1


def act3_bound(w, states):
    """per board: ACT3_REL * T3_max + ACT_FLOOR, shape [n, 1]"""
    _, _, t3 = R.valuenet_sensitivity(w, states)
    return ACT3_REL * t3.max(1, keepdims=True) + R.ACT_FLOOR


def out_sensitivity(w, states, allowance=None):
    """-> (sens_v, sens_var): |d out / d z_k| times the family's allowance on the logit (see the module docstring)"""
    if allowance == "floor":
        sv, svar, _ = R.valuenet_sensitivity(w, states, "floor")
        return sv, svar
    if allowance is None:
        n = len(np.asarray(states).reshape(-1, 200))
        return np.zeros(n), np.zeros(n)
    p = R.unpack(w, R.VN_SHAPES)
    x = R._x(states, torch.float64)
    with torch.no_grad():
        a1 = F.relu(F.conv2d(x, p["conv1.weight"], p["conv1.bias"]))
        a2 = F.relu(F.conv2d(a1, p["conv2.weight"], p["conv2.bias"]))
        a3 = F.relu(F.conv2d(a2, p["conv3.weight"], p["conv3.bias"])).flatten(1)
        h = F.relu(a3 @ p["fc1.weight"].T + p["fc1.bias"])
        z = h @ p["fc_out.weight"].T + p["fc_out.bias"]
        s_fc1 = (a3 @ p["fc1.weight"].abs().T + p["fc1.bias"].abs()) @ p["fc_out.weight"].abs().T
        sg = torch.sigmoid(z)
        sens = p["out_ubound"] * sg * (1 - sg) * COND_K * s_fc1
    return sens[:, 0].numpy(), sens[:, 1].numpy()


def out_excess(got, ref, sens):
    """largest |got - ref| / bound; <= 1 passes"""
    return float(np.max(np.abs(np.asarray(got, np.float64) - ref) / (OUT_RTOL * np.abs(ref) + sens)))


def _rz16(t):
    """float32 tensor -> its float16 neighbour toward zero (as float64)"""
    x = t.numpy()
    h = x.astype(np.float16)
    over = np.abs(h.astype(np.float32)) > np.abs(x)
    h[over] = np.nextafter(h[over], np.float16(0))
    return torch.from_numpy(h.astype(np.float64))


def _round(t, scale, dtype, rz=False):
    """t * scale rounded to fp32 (the epilogue's fma; exact for the weights), then to `dtype` (toward zero with rz), over scale"""
    s = (t * scale).to(torch.float32)
    return (_rz16(s) if rz else s.to(dtype).to(torch.float64)) / scale


# deliberate defects emulate_layers can apply, for the tests that show a check catches them
MUTANTS = ("rz_act", "rz_weight", "bias_after", "scale8", "no_conv2_block")


def emulate_layers(w, states, dtype=torch.float16, mutant=None):
    """The conv stack of emulate: [act1, act2, act3] as float64 tensors [n, 32, H, W] (each element an fp16 term / 16).  mutant: one of
    MUTANTS: activations rounded toward zero, weights rounded toward zero, each bias added after the rounding, activations scaled by 8
    instead of 16, conv2 without its (dy = 0, input channels 0..15) block of products."""
    p = R.unpack(w, R.VN_SHAPES)
    for k in R.SPLIT_VN:
        p[k] = _round(p[k], 64.0, dtype, mutant == "rz_weight")
    if mutant == "no_conv2_block":
        p["conv2.weight"][:, :16, 0] = 0
    sa = 8.0 if mutant == "scale8" else 16.0
    a, out = R._x(states, torch.float64), []
    with torch.no_grad():
        for l in (1, 2, 3):
            wl, bl = p["conv%d.weight" % l], p["conv%d.bias" % l]
            if mutant == "bias_after":
                a = F.relu(_round(F.conv2d(a, wl), sa, dtype) + bl[None, :, None, None])
            else:
                a = F.relu(_round(F.conv2d(a, wl, bl), sa, dtype, mutant == "rz_act"))
            out.append(a)
    return out


def emulate(w, states, dtype=torch.float16):
    """The net_fp16 arithmetic in float64: every conv / fc1 weight (x64) and every conv activation (x16, after the epilogue's fp32
    rounding) rounded once to `dtype` (torch.float16 as the device does; torch.bfloat16 to show that the bounds tell a coarser format
    apart), exact sums.  -> (v, var, act3) like f64_ref.valuenet."""
    p = R.unpack(w, R.VN_SHAPES)
    for k in R.SPLIT_VN:
        p[k] = _round(p[k], 64.0, dtype)
    with torch.no_grad():
        act3 = emulate_layers(w, states, dtype)[-1].flatten(1)
        h = F.relu(act3 @ p["fc1.weight"].T + p["fc1.bias"])
        out = torch.sigmoid(h @ p["fc_out.weight"].T + p["fc_out.bias"]) * p["out_ubound"] + p["out_lbound"]
    o = out.numpy()
    return o[:, 0], o[:, 1], act3.numpy()
