"""Layer-by-layer float64 restatement of the tensor-core conv stacks (valuenet_tc.cuh k_tc_conv, distnet_tc.cuh k_tdc_conv) with one fp16
term per operand (net_fp16, dist_fp16) or two (net_tc): given the activations a layer reads, it names for every element of the layer's output
the fp16 values the kernel may write.  The whole-network contracts of tests/f16_ref.py and tests/f16_dist_ref.py allow 2^-10 of the board's
largest |term| sum; this check is near bit-exact, one layer at a time.

What is restated exactly:
- weights: the loader scales each float32 conv weight by 64 (exact) and rounds it to fp16, round to nearest even (host_split2: the first term
  is __float2half_rn(64 w), the second __float2half_rn(64 w - first), the difference exact in fp32).  numpy's float32 -> float16 cast is the
  same IEEE rounding, on the subnormal and overflow edges too (tests/test_cpu_f16_layer_ref.py pins both).
- products: fp16 x fp16 is exact in fp32 and in float64.  Two terms multiply a1*w1 + a1*w2 + a2*w1 (a2*w2 is not issued).
- epilogue, on the activations scaled by 16: o = fmaf(acc, K, 16 b) in fp32 (K = 16 / 64 for conv1, 2^-10 * 16 for the others; 16 b is
  exact), then ReLU (value network) or x > 0 ? x : 0.01f * x in fp32 (distributional network), then __float2half_rn (one term) or the
  split x1 = rn16(o), x2 = rn16(o - x1) (o - x1 exact in fp32).  conv2 / conv3 first add their dx accumulators in fp32.
The accumulation assumption: the kernel's fp32 value before the activation is reached from the exact products by n fp32 operations in some
order, each with some rounding (wgmma's accumulation truncates), and each loses less than 2^-23 of S, the sum of |terms| of that value
(K |products| plus 16 |b|): every partial sum is at most S, and one fp32 rounding, to nearest or toward zero, moves a value by less than one
ulp, 2^-23 of it.  No order, rounding mode or internal precision of the tensor core is assumed, and nothing is fitted to a measurement:
n = the products summed into the element (conv1: the 16 taps of its K = 16 MMA, 9 of them used, per weight term) + the fp32 adds that
combine accumulators (dx taps; conv1's two weight terms) + 1 for the fma.  So |o_pre - z| <= n 2^-23 S for the exact pre-activation z
(plus float64's own rounding of z, (n + 2) 2^-52 S).  Both ends of that interval go through the restated epilogue, which is monotone,
so the admissible set of one term is an fp16 range [lo16, hi16].  Two terms: x1 must lie in that range, the pair must be canonical
(|x2| <= half an fp16 ulp of x1), and x1 + x2 must lie in the fp32 interval of o widened by x2's own rounding (half an fp16 ulp of x2,
2^-22 of |o| or 2^-25 below fp16's normal range).
"""
import numpy as np
import torch
import torch.nn.functional as F

import f64_ref as R

GRID = {False: {1: (18, 8), 2: (16, 6), 3: (14, 4)}, True: {1: (19, 7), 2: (16, 4)}}    # [dist][layer] -> (H, W) of the output


def n_ops(dist, layer, nt):
    """fp32 operations per output element (module docstring): products + accumulator adds + the fma"""
    if layer == 1:
        return 16 * nt + (nt - 1) + 1
    taps, dx = (16, 4) if dist else (9, 3)
    return taps * 32 * (3 if nt == 2 else 1) + (dx - 1) + 1


def dist_atoms(w):
    n = np.asarray(w).size - (544 + 16416 + 128 * 2048 + 128)
    assert n % 129 == 0, n
    return n // 129


def weight_terms(w, nt):
    """float32 weights -> nt float64 arrays of fp16 terms of 64 w, as the loader splits them (host_split2)"""
    s = np.asarray(w, np.float32) * np.float32(64)
    x1 = s.astype(np.float16)
    if nt == 1:
        return [x1.astype(np.float64)]
    return [x1.astype(np.float64), (s - x1.astype(np.float32)).astype(np.float16).astype(np.float64)]


def _conv_params(w, dist, layer):
    shapes = R.dn_shapes(dist_atoms(w)) if dist else R.VN_SHAPES
    p = R.unpack(w, shapes, torch.float32)
    return p["conv%d.weight" % layer].numpy(), p["conv%d.bias" % layer].numpy().astype(np.float64)


def preactivation(w, inp, dist, layer, nt):
    """-> (z, h): the exact pre-activation of every output element, scaled by 16 ([n, 32, H, W] float64), and the half-width of the
    interval the kernel's fp32 value lies in.  inp: the boards (int8 [n, 200]) for layer 1, else the list of nt float64 arrays
    [n, 32, H, W] of the previous layer's terms divided by 16, as b200_debug_tc_acts returns them."""
    wt, b = _conv_params(w, dist, layer)
    wt = weight_terms(wt, nt)
    if layer == 1:
        x = R._x(inp, torch.float64)
        if dist:
            x = F.pad(x, (0, 0, 2, 0))
        pairs, k = [(x, wt[s]) for s in range(nt)], 0.25
    else:
        a = [torch.from_numpy(np.asarray(t, np.float64) * 16) for t in inp]
        pairs, k = [(a[0], wt[0])] + ([(a[0], wt[1]), (a[1], wt[0])] if nt == 2 else []), 2.0 ** -6
    acc = sum(F.conv2d(x, torch.from_numpy(wk)) for x, wk in pairs)
    s = sum(F.conv2d(x.abs(), torch.from_numpy(np.abs(wk))) for x, wk in pairs)
    b16 = torch.from_numpy(16 * b)[None, :, None, None]
    z = (k * acc + b16).numpy()
    sz = (k * s + b16.abs()).numpy()
    n = n_ops(dist, layer, nt)
    return z, (n * 2.0 ** -23 + (n + 2) * 2.0 ** -52) * sz


def epilogue32(v, dist):
    """float64 -> the fp32 value the epilogue hands to the fp16 conversion (fp32 rounding, then the activation in fp32)"""
    o = np.asarray(v, np.float64).astype(np.float32)
    if dist:
        return np.where(o > 0, o, o * np.float32(0.01))
    return np.maximum(o, np.float32(0))


def _spacing16(x):
    return np.spacing(np.abs(np.asarray(x, np.float64)).astype(np.float16)).astype(np.float64)


def ordinal16(x):
    """fp16 values -> integers in which neighbouring fp16 values differ by one (distances in ulps)"""
    b = np.asarray(x, np.float64).astype(np.float16).view(np.uint16).astype(np.int64)
    return np.where(b & 0x8000, -(b & 0x7fff), b)


class Check:
    """The admissible set of one layer and the kernel's (or an emulation's) output held to it.
    ok: bool [n, 32, H, W]; single: where exactly one fp16 value is admissible (one term: lo16 == hi16)."""

    def __init__(self, w, inp, got, dist, layer):
        nt = len(got)
        z, h = preactivation(w, inp, dist, layer, nt)
        lo, hi = epilogue32(z - h, dist), epilogue32(z + h, dist)
        self.lo16, self.hi16 = lo.astype(np.float16).astype(np.float64), hi.astype(np.float16).astype(np.float64)
        g = [np.asarray(t, np.float64) * 16 for t in got]
        self.got = g
        ok = (g[0] >= self.lo16) & (g[0] <= self.hi16)
        if nt == 2:
            e = _spacing16(g[1]) / 2
            ok &= np.abs(g[1]) <= _spacing16(g[0]) / 2
            ok &= (g[0] + g[1] >= lo.astype(np.float64) - e) & (g[0] + g[1] <= hi.astype(np.float64) + e)
        self.ok, self.single = ok, self.lo16 == self.hi16
        self.dist, self.layer, self.nt = dist, layer, nt

    def bad(self):
        return int((~self.ok).sum())

    def describe(self, what, index=None):
        """the first failing element (or `index`): board, channel, pixel, value and admissible range in fp16 ulps"""
        b, c, y, x = index if index is not None else np.argwhere(~self.ok)[0]
        g1 = self.got[0][b, c, y, x]
        o, lo, hi = ordinal16(g1), ordinal16(self.lo16[b, c, y, x]), ordinal16(self.hi16[b, c, y, x])
        s = "%s: act%d board %d channel %d pixel (%d, %d): x1 = %r, admissible [%r, %r] = [%+d, %+d] ulps from x1" % (
            what, self.layer, b, c, y, x, g1 / 16, self.lo16[b, c, y, x] / 16, self.hi16[b, c, y, x] / 16, lo - o, hi - o)
        if self.nt == 2:
            s += ", x2 = %r (half an ulp of x1: %r)" % (self.got[1][b, c, y, x] / 16, _spacing16(g1) / 32)
        return s + " (%d elements out of their set)" % self.bad()


def check_stack(w, states, layers, dist):
    """layers: [act1, act2(, act3)], each a list of nt arrays [n, 32, H, W] (term / 16) -> [Check per layer], each layer checked on the
    previous layer as given"""
    out, inp = [], states
    for i, got in enumerate(layers):
        out.append(Check(w, inp, got, dist, i + 1))
        inp = got
    return out
