"""Stage-by-stage fp32 restatement of the CUDA-core networks of eval_kind `net` (valuenet_simt.cuh k_vn_conv / k_vn_fc, distnet_simt.cuh
k_dn_conv / k_dn_fc), in the kernels' own operation order, from the input each kernel itself read (b200_debug_net_acts exports every stage).

These kernels spell out every operation: fixed-order fmaf chains, IEEE fp32 adds and divisions (the build passes no --use_fast_math, so
-prec-div=true), a fixed shuffle tree and explicit __fmul_rn / __fadd_rn in the affine.  So every element before the head is ONE fp32
value, predictable bit for bit from the previous stage:
- key decode: the cell's bit of the bitboard (s > 0), then -1 on the first four cells with s < 0 (the key holds four piece cells; the
  distributional network gets two empty rows on top, 22x10);
- k_vn_conv: conv1 acc = b1, fmaf over dy then dx; conv2 / conv3 acc = bias, fmaf over ci, then dy, then dx (ci outermost); ReLU fmaxf(acc, 0);
- k_vn_fc: fc1 acc = 0, fmaf over k' = (y*32 + c)*4 + x (the kernel's order, not torch's) -> the exported accumulator; then
  h = fmaxf(acc + b, 0), lane tx chains fmaf(h, w_out, p) from 0 over columns tx*4 + j (j < 4), then 128 + tx*4 + (j - 4), butterfly adds
  over xor 16, 8, 4, 2, 1, x = p + b_out, s = 1 / (1 + expf(-x)), __fadd_rn(__fmul_rn(s, ub), lb);
- k_dn_conv: acc = bias, fmaf over (ci,) dy, then dx; LeakyReLU x > 0 ? x : 0.01f * x with 0.01f rounded to fp32 first;
- k_dn_fc: fc1 acc = bias, fmaf over torch k = c*64 + y*4 + x -> the exported pre-activation; LeakyReLU; fc_v acc = bias, fmaf over k
  ascending -> the exported logits; softmax: max (fmaxf), expf(l - mx), a sequential sum from 0.f in atom order, e / sum.
fmaf is emulated exactly (fma below, pinned against f16_layer_ref.fma32 and rational arithmetic); numpy's fp32 +, * and / through float64
are correctly rounded (53 >= 2 * 24 + 2).  fmaxf is np.fmax, not np.maximum: CUDA's fmaxf(NaN, 0) is 0, so a NaN sum leaves a ReLU as 0.

The one operation without defined semantics is expf (CUDA documents at most 2 ulp without --use_fast_math).  The head is therefore a set,
built as f16_layer_ref.HeadCheck builds it: the value outputs are monotone in t = expf(-x), so the ends of t's 2-ulp range give the ends
of the set; the probabilities come from HeadCheck._softmax_range on the kernel's own logits.

Comparison: `same` holds the kernel's value to the restated one bit for bit, except that NaN equals NaN (any payload) and zeros compare by
value (+0 == -0), which is what fmaxf and the LeakyReLU leave undefined or unobservable downstream.

The weights may be any finite fp32 values (net takes them all; net_tc refuses |w| * 64 > 65504), so sums can overflow to +-inf and
inf - inf gives NaN: `huge_value_weights` / `huge_dist_weights` make some act2 / act3 and fc1 sums overflow, and the restatement follows
the kernels through it.

NET_MUTANTS are deliberate defects, each a one-line change to the restatement, for the tests that show this check (and not the old
statistical allowances) catches them."""
import numpy as np

import f16_layer_ref as L
import f64_ref as R

TINY = 2.0 ** -126
_LOW29, _MID29 = np.int64((1 << 29) - 1), np.int64(1 << 28)
C001 = float(np.float32(0.01))           # the kernels' 0.01f
VN_GRID = {1: (18, 8), 2: (16, 6), 3: (14, 4)}
DN_GRID = {1: (19, 7), 2: (16, 4)}

# deliberate defects; each changes the stages named in MUTANT_STAGES.  Measured only (not required to be flagged), because with the exact
# exp the emulation uses they stay inside expf's 2-ulp slack on some families: sigmoid_recip (a reciprocal of 1 + t rounded toward zero
# and multiplied by 1: a correctly rounded reciprocal would equal the division bit for bit, so only an approximate one differs, by an
# ulp of s); affine_fma (fmaf(s, ub, lb) rounds once instead of twice: one ulp of the output at most); butterfly_up (xor 1, 2, 4, 8, 16
# reassociates the 32 lane sums: a few ulps of the logit x, which moves v by ub s (1 - s) dx); softmax_recip (e * (1 / sum): one ulp).
# np_maximum changes only NaN inputs of a ReLU (value network); in the softmax's max it would change nothing observable, since a NaN
# logit makes every probability NaN either way.
NET_MUTANTS = ("mul_add_conv2", "mul_add_conv3", "mul_add_fc1", "tap_major", "conv_bias_last", "fc1_torch_order", "fc1_bias_start",
               "butterfly_up", "affine_fma", "sigmoid_recip", "leaky_double", "dn_fc1_bias_after", "fcv_descending", "softmax_reversed",
               "softmax_pairwise", "softmax_no_max", "softmax_recip", "np_maximum")
NET_MEASURED_ONLY = ("sigmoid_recip", "affine_fma", "butterfly_up", "softmax_recip")
# [dist] -> mutant -> the stages it changes (value: act1 act2 act3 fc1 out; distributional: act1 act2 fc1 logits out)
MUTANT_STAGES = {
    False: {"mul_add_conv2": ("act2",), "mul_add_conv3": ("act3",), "mul_add_fc1": ("fc1",), "tap_major": ("act2", "act3"),
            "conv_bias_last": ("act1", "act2", "act3"), "fc1_torch_order": ("fc1",), "fc1_bias_start": ("fc1",), "butterfly_up": ("out",),
            "affine_fma": ("out",), "sigmoid_recip": ("out",), "np_maximum": ("act1", "act2", "act3", "out")},
    True: {"mul_add_conv2": ("act2",), "mul_add_fc1": ("fc1",), "tap_major": ("act2",), "conv_bias_last": ("act1", "act2"),
           "leaky_double": ("act1", "act2", "logits"), "dn_fc1_bias_after": ("fc1",), "fcv_descending": ("logits",),
           "softmax_reversed": ("out",), "softmax_pairwise": ("out",), "softmax_no_max": ("out",), "softmax_recip": ("out",)},
}


def round32(x):
    """float64 -> float64 holding the nearest fp32 value (IEEE overflow to +-inf)"""
    with np.errstate(over="ignore", invalid="ignore"):
        return np.asarray(x, np.float64).astype(np.float32).astype(np.float64)


def fma(a, b, c):
    """fmaf on float64 arrays holding fp32 values (broadcasting) -> float64 holding the fp32 result, exactly.  a * b is exact in float64
    and s = a * b + c is rounded once; rounding s to fp32 is then the correctly rounded fmaf (rounding is monotone and every fp32 midpoint
    is a float64 value, so s lies on the same side of every midpoint as a * b + c) unless s lies exactly on a midpoint (its low 29
    fraction bits 1000...0), where the second rounding may tie the wrong way, or in fp32's subnormal range, whose midpoints have another
    bit pattern.  Those elements, a small fraction, go through f16_layer_ref.fma32 (TwoSum)."""
    with np.errstate(over="ignore", invalid="ignore"):
        s = a * b + c
        r = s.astype(np.float32)
    s = np.ascontiguousarray(s)
    sus = ((s.view(np.int64) & _LOW29) == _MID29) | ((np.abs(s) < TINY) & (s != 0))
    if sus.any():
        a_, b_, c_ = np.broadcast_arrays(a, b, c)
        with np.errstate(over="ignore", invalid="ignore"):
            r[sus] = L.fma32(a_[sus], b_[sus], c_[sus])
    return r.astype(np.float64)


def mul_add(a, b, c):
    """the contraction-off mutant: __fmul_rn then __fadd_rn"""
    with np.errstate(over="ignore", invalid="ignore"):
        return round32(round32(a * b) + c)


def same(got, want):
    """bit equality, except NaN == NaN and +0 == -0 (module docstring) -> bool array"""
    g, w = np.asarray(got, np.float32), np.asarray(want, np.float64).astype(np.float32)
    return (g.view(np.uint32) == w.view(np.uint32)) | (np.isnan(g) & np.isnan(w)) | ((g == 0) & (w == 0))


def board_input(states, dist=False):
    """the kernels' key decode: int8 [n, 200] -> float64 [n, 20, 10] (dist: [n, 22, 10], two empty rows on top)"""
    s = np.asarray(states, np.int8).reshape(-1, 200)
    x = (s > 0).astype(np.float64)
    neg = s < 0
    x[neg & (np.cumsum(neg, 1) <= 4)] = -1.0
    x = x.reshape(-1, 20, 10)
    if dist:
        x = np.concatenate([np.zeros((len(x), 2, 10)), x], 1)
    return x


def _params(w, dist):
    shapes = R.dn_shapes(L.dist_atoms(w)) if dist else R.VN_SHAPES
    return {k: v.numpy().astype(np.float64) for k, v in R.unpack(w, shapes).items()}


def relu(x, mutant=None):
    return (np.maximum if mutant == "np_maximum" else np.fmax)(x, 0.0)


def leaky(x, mutant=None):
    with np.errstate(invalid="ignore", over="ignore"):
        return np.where(x > 0, x, round32(x * (0.01 if mutant == "leaky_double" else C001)))


def conv_acc(inp, wt, bias, layer, mutant=None):
    """one conv layer's fp32 accumulator from its input [n, ci, H, W] (float64 holding fp32): acc = bias, then fmaf over ci, dy, dx"""
    n, ci, H, Wd = inp.shape
    co, _, k, _ = wt.shape
    Ho, Wo = H - k + 1, Wd - k + 1
    f = mul_add if mutant == "mul_add_conv%d" % layer else fma
    last = mutant == "conv_bias_last"
    acc = np.zeros((n, co, Ho, Wo)) if last else np.broadcast_to(bias[None, :, None, None], (n, co, Ho, Wo)).copy()
    if mutant == "tap_major" and ci > 1:
        order = [(c, dy, dx) for dy in range(k) for dx in range(k) for c in range(ci)]
    else:
        order = [(c, dy, dx) for c in range(ci) for dy in range(k) for dx in range(k)]
    for c, dy, dx in order:
        acc = f(inp[:, c:c + 1, dy:dy + Ho, dx:dx + Wo], wt[None, :, c, dy, dx, None, None], acc)
    if last:
        acc = round32(acc + bias[None, :, None, None])
    return acc


def conv_layer(w, inp, dist, layer, mutant=None):
    """act<layer> [n, 32, H, W] float64 from the previous stage as the kernel read it (layer 1: the boards, int8 [n, 200])"""
    p = _params(w, dist)
    x = board_input(inp, dist)[:, None] if layer == 1 else np.asarray(inp, np.float32).astype(np.float64)
    acc = conv_acc(x, p["conv%d.weight" % layer], p["conv%d.bias" % layer], layer, mutant)
    return leaky(acc, mutant) if dist else relu(acc, mutant)


def vn_kernel_k_order():
    """torch flatten index (c*56 + y*4 + x) of k_vn_fc's k' = (y*32 + c)*4 + x, in k' order"""
    kp = np.arange(1792)
    return ((kp >> 2) & 31) * 56 + (kp >> 7) * 4 + (kp & 3)


def fc1(w, last, dist, mutant=None):
    """value: k_vn_fc's fc1 accumulator (before the bias) from act3; distributional: k_dn_fc's fc1 pre-activation (bias included) from
    act2.  last: [n, 32, H, W] or [n, K] in torch flatten order -> [n, 256] / [n, 128] float64"""
    p = _params(w, dist)
    a = np.asarray(last, np.float32).astype(np.float64).reshape(len(last), -1)
    wt, b = p["fc1.weight"], p["fc1.bias"]
    f = mul_add if mutant == "mul_add_fc1" else fma
    if dist:
        start = mutant == "dn_fc1_bias_after"
        acc = np.zeros((len(a), 128)) if start else np.broadcast_to(b[None], (len(a), 128)).copy()
        order = range(2048)
    else:
        acc = np.broadcast_to(b[None], (len(a), 256)).copy() if mutant == "fc1_bias_start" else np.zeros((len(a), 256))
        order = np.arange(1792) if mutant == "fc1_torch_order" else vn_kernel_k_order()
        start = False
    for k in order:
        acc = f(a[:, k:k + 1], wt[None, :, k], acc)
    if start:
        acc = round32(acc + b[None])
    return acc


LANE_COLS = np.array([[tx * 4 + j if j < 4 else 128 + tx * 4 + (j - 4) for j in range(8)] for tx in range(32)])   # [lane][j]


def value_logits(w, d, mutant=None):
    """k_vn_fc's logits x = p + b_out from fc1's accumulator d [n, 256] -> float64 [n, 2]"""
    p = _params(w, False)
    d = np.asarray(d, np.float32).astype(np.float64)
    h = relu(d if mutant == "fc1_bias_start" else round32(d + p["fc1.bias"][None]), mutant)
    wo = p["fc_out.weight"]                                     # [2, 256]
    acc = np.zeros((len(h), 32, 2))                            # [row, lane, output]
    for j in range(8):
        c = LANE_COLS[:, j]
        acc = fma(h[:, c][:, :, None], wo.T[c][None], acc)
    lane = np.arange(32)
    for off in ((1, 2, 4, 8, 16) if mutant == "butterfly_up" else (16, 8, 4, 2, 1)):
        acc = round32(acc + acc[:, lane ^ off])
    return round32(acc[:, 0] + p["fc_out.bias"][None])


def value_outputs(w, x, t, mutant=None):
    """s = 1.f / (1.f + t) with t = expf(-x), then __fadd_rn(__fmul_rn(s, ub), lb) (f16_layer_ref.value_outputs), or the mutants'"""
    if mutant not in ("affine_fma", "sigmoid_recip"):
        with np.errstate(over="ignore", invalid="ignore"):
            return L.value_outputs(w, x, t).astype(np.float64)
    p = _params(w, False)
    t = np.asarray(t, np.float32).astype(np.float64)
    if mutant == "sigmoid_recip":
        s = L._rd32(1.0 / round32(1.0 + t)).astype(np.float64)
        return round32(round32(s * p["out_ubound"][None]) + p["out_lbound"][None])
    s = round32(1.0 / round32(1.0 + t))
    return fma(s, p["out_ubound"][None], p["out_lbound"][None])


def dist_logits(w, pre, mutant=None):
    """k_dn_fc's fc_v from fc1's pre-activation [n, 128] -> logits float64 [n, atoms]"""
    p = _params(w, True)
    h = leaky(np.asarray(pre, np.float32).astype(np.float64), mutant)
    wv = p["fc_v.weight"]
    acc = np.broadcast_to(p["fc_v.bias"][None], (len(h), wv.shape[0])).copy()
    for k in (range(127, -1, -1) if mutant == "fcv_descending" else range(128)):
        acc = fma(h[:, k:k + 1], wv[None, :, k], acc)
    return acc


def softmax(lg, exp=L.exp_rn, mutant=None):
    """k_dn_fc's softmax on the logits [n, atoms] with the given fp32 exp -> float64 [n, atoms]"""
    lg = np.asarray(lg, np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        mx = np.zeros(len(lg), np.float32) if mutant == "softmax_no_max" else np.fmax.reduce(lg, 1)
        e = exp(lg - mx[:, None]).astype(np.float32)
        if mutant == "softmax_pairwise":
            parts = [e[:, a] for a in range(e.shape[1])]
            while len(parts) > 1:
                parts = [parts[i] + parts[i + 1] if i + 1 < len(parts) else parts[i] for i in range(0, len(parts), 2)]
            s = parts[0]
        else:
            s = np.zeros(len(e), np.float32)
            for a in (range(e.shape[1] - 1, -1, -1) if mutant == "softmax_reversed" else range(e.shape[1])):
                s = s + e[:, a]
        if mutant == "softmax_recip":
            return (e * (np.float32(1) / s[:, None])).astype(np.float64)
        return (e / s[:, None]).astype(np.float64)


def head_set(w, stage_in, dist):
    """the outputs' admissible sets from the kernel's own fc1 accumulator (value) or logits (distributional) -> (lo, hi) fp32.  NaN in
    both ends: the output is NaN whatever expf returns."""
    if not dist:
        x = value_logits(w, stage_in).astype(np.float32)
        with np.errstate(over="ignore", invalid="ignore"):
            t_lo, t_hi = L.exp_range(-x)
            o1, o2 = value_outputs(w, x, t_lo), value_outputs(w, x, t_hi)
        return np.fmin(o1, o2).astype(np.float32), np.fmax(o1, o2).astype(np.float32)
    lg = np.asarray(stage_in, np.float32)
    # NaN or +inf logits, or all of them -inf, make every probability NaN (expf(NaN) and inf - inf poison the sum); the others have a
    # finite max, so HeadCheck's set applies (an expf(-inf) is exactly 0, inside exp_range(-inf))
    nan_row = np.isnan(lg).any(1) | np.isposinf(lg).any(1) | np.isneginf(lg).all(1)
    with np.errstate(over="ignore", invalid="ignore"):
        lo, hi = L.HeadCheck._softmax_range(np.where(nan_row[:, None], np.float32(0), lg))
    lo[nan_row], hi[nan_row] = np.nan, np.nan
    return lo, hi


def in_set(got, lo, hi):
    g = np.asarray(got, np.float32)
    return ((g >= lo) & (g <= hi)) | (np.isnan(g) & np.isnan(lo) & np.isnan(hi))


def head_outputs(w, stage_in, dist, mutant=None, exp=L.exp_rn):
    """the outputs with the given exp (default: correctly rounded), or the mutant's"""
    if dist:
        return softmax(stage_in, exp, mutant)
    x = value_logits(w, stage_in, mutant).astype(np.float32)
    with np.errstate(over="ignore"):
        return value_outputs(w, x, exp(-x), mutant)


# ---------------------------------------------------------------------------------------------------- the whole network, stage by stage
VN_STAGES = ("act1", "act2", "act3", "fc1", "out")
DN_STAGES = ("act1", "act2", "fc1", "logits", "out")


def forward(w, states, dist, mutant=None, exp=L.exp_rn):
    """every stage of the network, each from the previous restated stage -> dict stage -> array (act<l> [n, 32, H, W], fc1, logits, out)"""
    st = {}
    inp = states
    for layer in ((1, 2) if dist else (1, 2, 3)):
        inp = st["act%d" % layer] = conv_layer(w, inp, dist, layer, mutant)
    st["fc1"] = fc1(w, inp, dist, mutant)
    if dist:
        st["logits"] = dist_logits(w, st["fc1"], mutant)
        st["out"] = head_outputs(w, st["logits"], True, mutant, exp)
    else:
        st["out"] = head_outputs(w, st["fc1"], False, mutant, exp)
    return st


def stage_from(w, states, prev, stage, dist, mutant=None):
    """one stage restated from the previous stage as given (prev: the kernel's or the restatement's own) -> array; "out" -> (lo, hi)"""
    if stage.startswith("act"):
        layer = int(stage[3:])
        return conv_layer(w, states if layer == 1 else prev, dist, layer, mutant)
    if stage == "fc1":
        return fc1(w, prev, dist, mutant)
    if stage == "logits":
        return dist_logits(w, prev, mutant)
    return head_set(w, prev, dist)


class StageCheck:
    """A network's stages as some source computed them (the device export, or an emulation), each held to the restatement from that
    source's own previous stage: every element before the head bit for bit (`same`), every output inside its expf set.
    bad[stage]: elements that differ; width: head set widths in fp32 ulps (NaN sets count 0)."""

    def __init__(self, w, states, got, dist):
        self.bad, self.first = {}, {}
        stages = DN_STAGES if dist else VN_STAGES
        prev = None
        for s in stages:
            want = stage_from(w, states, prev, s, dist)
            g = np.asarray(got[s])
            if s == "out":
                lo, hi = want
                ok = in_set(g, lo, hi)
                with np.errstate(invalid="ignore"):
                    wd = L.ordinal32(np.nan_to_num(hi, nan=0.0)) - L.ordinal32(np.nan_to_num(lo, nan=0.0))
                self.width, self.lo, self.hi = wd, lo, hi
            else:
                ok = same(g, want)
            self.bad[s] = int((~ok).sum())
            if self.bad[s]:
                i = tuple(np.argwhere(~ok)[0])
                self.first[s] = (i, float(g[i]), (float(want[0][i]), float(want[1][i])) if s == "out" else float(want[i]))
            prev = g

    def total(self):
        return sum(self.bad.values())

    def describe(self, what):
        s = next(k for k in self.bad if self.bad[k])
        i, g, want = self.first[s]
        return "%s: %s element %s = %r, restated %r (%d elements of %s differ; all stages: %s)" % (
            what, s, i, g, want, self.bad[s], s, self.bad)


# ---------------------------------------------------------------------------------------------------- weights that overflow fp32
def huge_value_weights(seed=0):
    """init_weights(seed) with conv1 / conv2 scaled by 2^40 / 2^88 (biases by the running product), fc1 by 2^-100 and fc_out by the
    inverse of what is left: finite weights that net accepts (net_tc refuses them) and float64 logits as before, but act2 / act3 near
    fp32's 2^128, so that some act2 / act3 sums overflow to +-inf and the fc1 sums that meet them become +-inf or NaN (inf - inf)"""
    return R._rescale(R.init_weights(seed), (2.0 ** 40, 2.0 ** 88, 1.0), 2.0 ** -100)


def huge_dist_weights(seed, atoms):
    """dist_init_weights with conv1 / conv2 scaled by 2^60 / 2^69 (biases by the running product), fc1 by 2^-109 and fc_v by 2^-20: some
    act2 sums overflow fp32, and the fc1 sums and logits that meet them become +-inf or NaN"""
    sh = R.dn_shapes(atoms)
    d = R.unpack(R.dist_init_weights(seed, atoms), sh)
    d["conv1.weight"] *= 2.0 ** 60; d["conv1.bias"] *= 2.0 ** 60                 # noqa: E702
    d["conv2.weight"] *= 2.0 ** 69; d["conv2.bias"] *= 2.0 ** 129                # noqa: E702
    d["fc1.weight"] *= 2.0 ** -109; d["fc1.bias"] *= 2.0 ** 20                    # noqa: E702
    d["fc_v.weight"] *= 2.0 ** -20
    return R.pack({k: v.numpy() for k, v in d.items()}, sh)
