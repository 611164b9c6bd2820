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

The fc stage (k_tc_fc, k_tdc_fc) is checked in two steps, each from what the kernel itself computed before it:
- fc1's raw fp32 accumulator d, from the last conv layer's terms (Fc1Check): exact products, the accumulation bounded as above with n =
  1792 / 2048 products per term pair.  About 2^-12 of the |term| sum for one term: a structural check that does not resolve operand
  rounding.
- the outputs, from d (HeadCheck): restated in fp32 operation for operation and in the kernel's order (bias and activation, fc_out's
  per-lane fmaf chains and shuffle adds or fc_v's fmaf chain, the sigmoid and affine or the softmax).  fmaf is emulated exactly (fma32);
  numpy's fp32 +, * and / are correctly rounded (53 >= 2 * 24 + 2, so float64's double rounding is harmless).  expf is the one operation
  without defined semantics: CUDA documents at most 2 ulp of error without --use_fast_math, which build.py does not pass, and every value
  within 2 ulp is admitted.  Each output gets a set a few fp32 values wide.  Pinning the order is deliberate: an order-free bound on the
  256- / 128-term fp32 sums is hundreds of ulps of an output, too wide to see a changed bias, activation or weight layout.  A change to
  the order of the kernels' head must change value_logits / dist_logits in the same commit.
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


# ---------------------------------------------------------------------------------------------------- the fc stage (k_tc_fc, k_tdc_fc)
FC1 = {False: (256, 1792, 56), True: (128, 2048, 64)}          # [dist] -> (fc1 outputs, fc1 inputs, pixels per channel)
UNSCALE = np.float32(2.0 ** -10)
FLT_MAX = float(np.finfo(np.float32).max)
# deliberate defects of the fc stage, for the tests that show the fc1 and head checks catch them (see fc1_emulated / head_outputs).
# Two are measured, not required to be flagged, because they move an output by about one ulp, inside the 2 ulp that expf itself may err
# by: recip (the softmax's division as a multiply by the reciprocal) and fast_exp (the softmax's expf replaced by __expf, whose error
# grows with the argument).
FC_MUTANTS = ("drop_kblock", "bias_twice", "no_bias", "relu", "recip", "wout_transposed", "fast_exp")
FC_MEASURED_ONLY = ("recip", "fast_exp")


def fc_mutant_applies(name, dist):
    """relu, recip and fast_exp change the distributional head only"""
    return dist or name not in ("relu", "recip", "fast_exp")


def _rd32(v):
    """float64 -> the largest fp32 value <= v"""
    v = np.asarray(v, np.float64)
    with np.errstate(over="ignore"):
        r = v.astype(np.float32)
    return np.where(r.astype(np.float64) > v, np.nextafter(r, np.float32(-np.inf)), r)


def _ru32(v):
    """float64 -> the smallest fp32 value >= v"""
    v = np.asarray(v, np.float64)
    with np.errstate(over="ignore"):
        r = v.astype(np.float32)
    return np.where(r.astype(np.float64) < v, np.nextafter(r, np.float32(np.inf)), r)


def fma32(a, b, c):
    """fmaf(a, b, c) on fp32 arrays, exactly: the float64 product of two fp32 values is exact, TwoSum gives p + c = s + e exactly, and s
    rounded to fp32 is the correctly rounded result unless s lies exactly on an fp32 midpoint (every fp32 midpoint is a float64 value, so
    s and p + c are on the same side of all others); on a midpoint with e != 0 the result is the neighbour on e's side."""
    a, b, c = (np.asarray(x, np.float32).astype(np.float64) for x in (a, b, c))
    p = a * b
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)
    rd, ru = _rd32(s), _ru32(s)
    rd64, ru64 = rd.astype(np.float64), np.where(np.isinf(ru), 2.0 ** 128, ru.astype(np.float64))   # overflow rounds as if at 2^128
    with np.errstate(over="ignore"):
        r = s.astype(np.float32)
    mid = (rd64 != ru64) & (s - rd64 == ru64 - s) & (e != 0)
    return np.where(mid, np.where(e > 0, ru, rd), r)


def exp_range(x):
    """fp32 arguments -> (lo, hi): the smallest and largest fp32 values within 2 ulp of exp(x), CUDA's documented maximum error of expf
    (without --use_fast_math).  ulp = that of the exact result; float64's own error of exp (< 2^-52 relative) widens the interval by 2^-50."""
    x = np.asarray(x, np.float32).astype(np.float64)
    e = np.exp(x)
    _, ex = np.frexp(e)
    ulp = np.ldexp(1.0, np.where(e > 0, np.maximum(ex - 24, -149), -149))
    lo = np.maximum(_ru32(e * (1 - 2.0 ** -50) - 2 * ulp), np.float32(0))
    top = e * (1 + 2.0 ** -50) + 2 * ulp
    hi = np.where(top > FLT_MAX, np.float32(np.inf), _rd32(top))
    return lo, hi


def exp_rn(x):
    """correctly rounded fp32 exp (the emulation's; float64 exp rounded once)"""
    return np.exp(np.asarray(x, np.float32).astype(np.float64)).astype(np.float32)


def fast_exp(x):
    """__expf as the fast-math intrinsic computes it, for the mutant: 2^(x * log2(e) rounded to fp32), flushed to zero below 2^-126"""
    t = np.asarray(x, np.float32) * np.float32(np.log2(np.e))
    e = np.exp2(t.astype(np.float64)).astype(np.float32)
    return np.where(e < np.float32(2.0 ** -126), np.float32(0), e)


def ordinal32(x):
    """fp32 values -> integers in which neighbouring fp32 values differ by one"""
    b = np.asarray(x, np.float32).view(np.int32).astype(np.int64)
    return np.where(b < 0, -(b & 0x7fffffff), b)


def _fc_params(w, dist):
    shapes = R.dn_shapes(dist_atoms(w)) if dist else R.VN_SHAPES
    return {k: v.numpy() for k, v in R.unpack(w, shapes, torch.float32).items()}


def _last_terms(last):
    """the previous layer's terms ([n, 32, H, W] each, term / 16) -> nt float64 arrays [n, K] of fp16 terms in torch flatten order"""
    return [np.asarray(t, np.float64).reshape(len(t), -1) * 16 for t in last]


def _fc1_pairs(w, last, dist):
    a = _last_terms(last)
    wt = weight_terms(_fc_params(w, dist)["fc1.weight"], len(a))
    return [(a[0], wt[0])] + ([(a[0], wt[1]), (a[1], wt[0])] if len(a) == 2 else [])


def kernel_k_order(dist):
    """torch flatten index (c * pixels + pixel) of the fc kernels' k' = pixel * 32 + c, in k' order (16 consecutive k' = one k block)"""
    _, k, npix = FC1[dist]
    kp = np.arange(k)
    return (kp & 31) * npix + (kp >> 5)


class Fc1Check:
    """fc1's fp32 accumulator d (before x 2^-10, the bias and the activation), per element, from the previous layer's terms as the kernel
    read them.  The products a1*w1 (+ a1*w2 + a2*w1) of fp16 terms (activations x16, weights x64) are exact; the accumulation is bounded as
    for the conv layers: each of n = 1792 / 2048 products per term pair (x3 for two terms) loses less than 2^-23 of the |term| sum S, so
    |d - z| <= n 2^-23 S (+ float64's own (n + 2) 2^-52 S).  That is about 2^-12 S for one term: a structural check (a missing or doubled
    k block, a wrong weight row or input column, wrong term pairs, a stale or misrouted tile), which does not resolve operand rounding.
    ok: bool [n, N]; used: |d - z| / h."""

    def __init__(self, w, last, d, dist):
        pairs = _fc1_pairs(w, last, dist)
        z = sum(a @ wk.T for a, wk in pairs)
        s = sum(np.abs(a) @ np.abs(wk).T for a, wk in pairs)
        n = FC1[dist][1] * len(pairs)
        self.z, self.h = z, (n * 2.0 ** -23 + (n + 2) * 2.0 ** -52) * s
        self.got = np.asarray(d, np.float32).astype(np.float64)
        err = np.abs(self.got - z)
        self.ok = err <= self.h
        with np.errstate(invalid="ignore", divide="ignore"):
            self.used = np.where(self.h > 0, err / self.h, np.where(err > 0, np.inf, 0.0))

    def bad(self):
        return int((~self.ok).sum())

    def describe(self, what):
        b, c = np.argwhere(~self.ok)[0] if self.bad() else np.unravel_index(np.argmax(self.used), self.used.shape)
        return "%s: fc1 board %d output %d: d = %r, z = %r, |d - z| = %.3g of the bound (%d elements out of it)" % (
            what, b, c, self.got[b, c], self.z[b, c], self.used[b, c], self.bad())


def fc1_emulated(w, last, dist, mutant=None):
    """an fp32 accumulation of fc1's exact products, in the kernel's k order, one k at a time (term pairs small first); mutant
    "drop_kblock" leaves out the last k block (16 inputs) -> d [n, N] fp32"""
    pairs = _fc1_pairs(w, last, dist)
    order = kernel_k_order(dist)
    if mutant == "drop_kblock":
        order = order[:-16]
    acc = np.zeros((len(pairs[0][0]), FC1[dist][0]), np.float32)
    for k in order:
        for a, wk in pairs:
            acc = acc + (a[:, k:k + 1] * wk[None, :, k]).astype(np.float32)
    return acc


def _fc1_out(p, d, dist, mutant):
    """fc1's epilogue in fp32: act(d * 2^-10 + b) (the product is exact, so fma and mul-then-add agree), act = ReLU (value) or
    x > 0 ? x : 0.01f * x (distributional)"""
    b = p["fc1.bias"]
    if mutant == "no_bias":
        x = np.asarray(d, np.float32) * UNSCALE
    else:
        x = fma32(d, UNSCALE, b[None, :])
        if mutant == "bias_twice":
            x = x + b[None, :]
    if dist and mutant != "relu":
        return np.where(x > 0, x, x * np.float32(0.01))
    return np.maximum(x, np.float32(0))


def _transposed16(wm):
    """the mutant's weights: columns 4i + j and 4j + i swapped within each 16-column block"""
    i = np.arange(wm.shape[-1])
    blk, r = i // 16, i % 16
    return wm[..., blk * 16 + (r % 4) * 4 + r // 4]


def value_logits(w, d, mutant=None):
    """k_tc_fc's fc_out in fp32 from fc1's accumulator d [n, 256]: lane qd chains fmaf over columns 8j + 2qd + e (j ascending, e inner)
    from 0, the xor-1 then xor-2 shuffle adds, then + bout -> [n, 2]"""
    p = _fc_params(w, False)
    h = _fc1_out(p, d, False, mutant)
    wo = _transposed16(p["fc_out.weight"]) if mutant == "wout_transposed" else p["fc_out.weight"]
    acc = np.zeros((len(h), 4, 2), np.float32)                    # [board, qd, output]
    qd = np.arange(4)
    for j in range(32):
        for e in range(2):
            c = 8 * j + 2 * qd + e
            acc = fma32(h[:, c][:, :, None], wo.T[c][None], acc)
    x = (acc[:, 0] + acc[:, 1]) + (acc[:, 2] + acc[:, 3])
    return x + p["fc_out.bias"][None, :]


def value_outputs(w, x, t):
    """1.f / (1.f + t) with t = expf(-x), then __fadd_rn(__fmul_rn(s, ub), lb), in fp32"""
    p = _fc_params(w, False)
    s = np.float32(1) / (np.float32(1) + np.asarray(t, np.float32))
    return s * p["out_ubound"][None, :] + p["out_lbound"][None, :]


def dist_logits(w, d, mutant=None):
    """k_tdc_fc's fc_v in fp32 from fc1's accumulator d [n, 128]: logits = bv, then fmaf over c ascending -> [n, atoms]"""
    p = _fc_params(w, True)
    h = _fc1_out(p, d, True, mutant)
    wv = _transposed16(p["fc_v.weight"]) if mutant == "wout_transposed" else p["fc_v.weight"]
    lg = np.broadcast_to(p["fc_v.bias"][None, :], (len(h), wv.shape[0])).astype(np.float32)
    for c in range(128):
        lg = fma32(h[:, c:c + 1], wv[None, :, c], lg)
    return lg


def _seq_sum(e):
    s = np.zeros(e.shape[:-1], np.float32)
    for a in range(e.shape[-1]):
        s = s + e[..., a]
    return s


def head_outputs(w, d, dist, mutant=None):
    """the fc stage's outputs with a correctly rounded exp (or the mutant's) -> [n, 2] (v, var) or [n, atoms] probabilities"""
    ex = fast_exp if mutant == "fast_exp" else exp_rn
    if not dist:
        x = value_logits(w, d, mutant)
        return value_outputs(w, x, ex(-x))
    lg = dist_logits(w, d, mutant)
    e = ex(lg - lg.max(1, keepdims=True))
    s = _seq_sum(e)[:, None]
    return e * (np.float32(1) / s) if mutant == "recip" else e / s


class HeadCheck:
    """The outputs, per output, from the kernel's own fc1 accumulator d, restated in fp32 operation for operation and in the kernel's order
    (value_logits / dist_logits, then the sigmoid and affine or the softmax).  The one operation without defined IEEE semantics is expf,
    taken anywhere within 2 ulp of the exact exp of its argument (exp_range).  Value network: the output is monotone in t = expf(-x), so
    the ends of t give the ends of the set.  Softmax, max, then e_a = expf(lg_a - mx), sum = e_0 + e_1 + ... in atom order from 0.f,
    p_a = e_a / sum: p_a falls as any other e_b rises (the RN sum is monotone in each addend, the RN division in its divisor), so its lowest
    value has the other e's at their high ends and its highest at their low ends; e_a itself is taken at every fp32 value of its range.
    The restated order is deliberate: an order-free bound on the 256- / 128-term fp32 sums is hundreds of ulps of an output, too wide to see
    a changed activation, bias or division.  A change to the order of the kernel's head must change value_logits / dist_logits with it.
    lo, hi: fp32 [n, outputs]; ok: bool; width: hi - lo in ulps."""

    def __init__(self, w, d, got, dist):
        if dist:
            self.lo, self.hi = self._softmax_range(dist_logits(w, d))
        else:
            x = value_logits(w, d)
            t_lo, t_hi = exp_range(-x)
            o1, o2 = value_outputs(w, x, t_lo), value_outputs(w, x, t_hi)
            self.lo, self.hi = np.minimum(o1, o2), np.maximum(o1, o2)
        self.got = np.asarray(got, np.float32)
        self.ok = (self.got >= self.lo) & (self.got <= self.hi)
        self.width = ordinal32(self.hi) - ordinal32(self.lo)

    @staticmethod
    def _softmax_range(lg):
        e_lo, e_hi = exp_range(lg - lg.max(1, keepdims=True))
        n_atoms = lg.shape[1]
        b_lo, b_hi = e_lo.view(np.int32), e_hi.view(np.int32)          # non-negative fp32: the bits count ulps
        p_lo = np.full(lg.shape, np.inf, np.float32)
        p_hi = np.full(lg.shape, -np.inf, np.float32)
        eye = np.eye(n_atoms, dtype=bool)[None]
        for k in range(int((b_hi - b_lo).max()) + 1):
            ea = np.minimum(b_lo + k, b_hi).view(np.float32)              # e_a at the k-th value of its range
            for other, pick in ((e_hi, np.minimum), (e_lo, np.maximum)):
                es = np.where(eye, ea[:, None, :], other[:, :, None])    # [board, atom b, atom a]: e_b, with e_a in the diagonal
                p = ea / _seq_sum(np.moveaxis(es, 1, 2))
                if pick is np.minimum:
                    p_lo = np.minimum(p_lo, p)
                else:
                    p_hi = np.maximum(p_hi, p)
        return p_lo, p_hi

    def bad(self):
        return int((~self.ok).sum())

    def describe(self, what):
        b, o = np.argwhere(~self.ok)[0] if self.bad() else np.unravel_index(np.argmax(self.width), self.width.shape)
        g = ordinal32(self.got[b, o])
        return "%s: output board %d index %d = %r, admissible [%r, %r] = [%+d, %+d] ulps from it (%d outputs out of their set)" % (
            what, b, o, self.got[b, o], self.lo[b, o], self.hi[b, o], ordinal32(self.lo[b, o]) - g, ordinal32(self.hi[b, o]) - g, self.bad())
