"""Stage-by-stage float64 restatement of one training step of the device trainer (tetris_mcts_b200/csrc/trainer.cu): each check takes the
inputs the kernel itself read (earlier stages as Trainer.debug_buffer exports them) and names, for every output element, the values the
kernel may write.  The trainer's other tests hold whole gradient tensors to 1e-5 of their norm; these checks see single elements.

Bit for bit (the kernels' operations restated in their order):
- layout: k_states_to_float / k_gather_rows, the three k_im2col, k_nhwc_to_flat, k_flat_to_nhwc_relu, k_col2im_relu (<= 9 taps in
  ascending tap order, summed in fp64 from 0.0, rounded once, masked by act > 0) and k_dh (both products of fp32 values are exact in
  fp64, so fma(a, b, c d) is float64's c*d + a*b);
- bias gradients (k_colsum): 8 warps stride the rows with sequential fp64 sums, the 8 partials are added in ascending order, rounded once;
- the head's z (an fp64 fma chain in ascending k, each product exact);
- the loss (k_std_mean: 256 strided sequential partials, then the tree; the second pass's `a += d * d` is a DFMA in the SASS and is
  emulated exactly), the per-tensor sums of squares (k_sumsq), the gradient norm, the clip coefficient and k_scale, and Yogi (k_yogi,
  every operation an _rn intrinsic) with the YogiConst fields from the host's double arithmetic (Python's float ** is the same libm pow).

Per element, as an admissible set (GemmCheck), the 12 products of a step: conv1-3 and fc1 forward, fc_out's weight gradient (k_gemm in
both kinds), fc1's weight gradient, dflat, the three conv weight gradients, dcol3 and dcol2.  The k ranges of each product come from the
restated split rules (fp64_kps: gemm's split-k; tc_kps: tc_k_per_split).  Per range z with |term| sum T_z:
- fp64 kind: fp32 x fp32 products are exact in fp64; the kernel's fma chain and float64's own matmul each stay within K_z 2^-53 T_z.
- tc kind: operands split exactly as the kernel does (big = rna_tf32(x), small = rna_tf32(x - big)); a_s b_b + a_b b_s + a_b b_b is
  exact in float64, a_s b_s is dropped.  The accumulation is bounded without a model of the hardware: inside a 32-k tile each of at most
  96 product adds loses less than 2^-23 of the tile's |term| sum (wgmma truncates), each round-to-nearest FADD into the chunk's fp32
  accumulator at most 2^-24 of the chunk's, and the accumulator is an fp32 value.  This is a structural check: about 1.5e-5 of T, it
  finds missing, doubled or misrouted tiles, chunks and cross products, but does not resolve operand rounding.
Then k_finish's fp64 sum of the partials in ascending z (or the single range's accumulator), one fp32 rounding, the bias in fp32 and
ReLU: every step is monotone, so the rounded value lies in [RN32(lo), RN32(hi)], and the output is admissible when some fp32 value of
that range gives it after the bias and ReLU (which keeps the check sharp where the bias cancels).  grad_rows_dev's unrounded fp64 slice
gradient is held to [lo, hi] itself.

The head (k_head: pred, lossv, dz) is restated in fp32 operation for operation in the order of the SASS, not the source: diff * diff +
var is one FFMA (fma32), and the sigmoid's 1 + expf(-x) is one FFMA (expf's final scaling fused with the add), rounded once.  expf may
err by its documented 2 ulp and logf by 1 ulp; every combination of those values is enumerated and nothing else is admitted.  The
divisions are IEEE (numpy's fp32 division)."""
from fractions import Fraction

import numpy as np

import f16_layer_ref as L

N_TRAIN, N_ALL, N_TENSORS = 478338, 478342, 10
OFF = dict(c1w=0, c1b=288, c2w=320, c2b=9536, c3w=9568, c3b=18784, f1w=18816, f1b=477568, fow=477824, fob=478336, ub=478338, lb=478340)
T_OFF = (0, 288, 320, 9536, 9568, 18784, 18816, 477568, 477824, 478336, 478338)
TG_BM, TG_BK, TG_KCHUNK = 64, 32, 2048
F32, F64 = np.float32, np.float64
TENSORS = ("conv1.weight", "conv1.bias", "conv2.weight", "conv2.bias", "conv3.weight", "conv3.bias", "fc1.weight", "fc1.bias",
           "fc_out.weight", "fc_out.bias")


def params(w):
    """state_dict vector -> float32 views: conv weights [32][Kc] (k = ci*9 + ky*3 + kx), fc1 [256][1792], fc_out [2][256], biases, bounds"""
    w = np.asarray(w, F32)
    o = OFF
    return dict(c1w=w[0:288].reshape(32, 9), c1b=w[288:320], c2w=w[320:9536].reshape(32, 288), c2b=w[9536:9568],
                c3w=w[9568:18784].reshape(32, 288), c3b=w[18784:18816], f1w=w[o["f1w"]:o["f1b"]].reshape(256, 1792),
                f1b=w[o["f1b"]:o["fow"]], fow=w[o["fow"]:o["fob"]].reshape(2, 256), fob=w[o["fob"]:o["ub"]], ub=w[o["ub"]:o["lb"]],
                lb=w[o["lb"]:N_ALL])


# ---------------------------------------------------------------------------------------------------- split rules
def fp64_kps(M, N, K):
    """gemm()'s k range length: split-k only for K >= 4096 on grids of < 264 tiles"""
    splits = 1
    tiles = -(-M // 64) * -(-N // 64)
    if K >= 4096 and tiles < 132 * 2:
        splits = -(-528 // tiles)
        splits = min(splits, -(-K // 512))
    return -(-(-(-K // splits)) // 16) * 16


def tc_kps(M, N, K, BN):
    """tc_k_per_split: chunks of <= 2048 k, and on small grids more ranges of >= 256 k"""
    tiles = -(-M // TG_BM) * -(-N // BN)
    splits = -(-K // TG_KCHUNK)
    if K >= 512 and tiles * splits < 132 * 2:
        splits = max(splits, min(-(-264 // tiles), K // 256))
    return -(-(-(-K // splits)) // TG_BK) * TG_BK


def product_shapes(B):
    """name -> (M, N, K, BN, tc shape (M, N) when it differs, e.g. a transposed weight gradient), of each product at batch B"""
    return {"conv1": (B * 144, 32, 9, 32, None), "conv2": (B * 96, 32, 288, 32, None), "conv3": (B * 56, 32, 288, 32, None),
            "fc1": (B, 256, 1792, 64, None), "fc_out_wgrad": (2, 256, B, None, None), "fc1_wgrad": (256, 1792, B, 64, None),
            "dflat": (B, 1792, 256, 64, None), "conv3_wgrad": (32, 288, B * 56, 32, (288, 32)), "conv2_wgrad": (32, 288, B * 96, 32, (288, 32)),
            "conv1_wgrad": (32, 9, B * 144, 32, (9, 32)), "dcol3": (B * 56, 288, 32, 64, None), "dcol2": (B * 96, 288, 32, 64, None)}


def kps_of(name, B, kind):
    """k range length of product `name` in a trainer of `kind` (fc_out's weight gradient is k_gemm in both kinds)"""
    M, N, K, BN, tshape = product_shapes(B)[name]
    if kind == "fp64" or BN is None:
        return fp64_kps(M, N, K)
    if tshape:
        M, N = tshape
    return tc_kps(M, N, K, BN)


def ranges(K, kps):
    return [(kb, min(K, kb + kps)) for kb in range(0, K, kps)]


# ---------------------------------------------------------------------------------------------------- fp32 helpers
def tf32_rna(x):
    """cvt.rna.tf32.f32 on the bits: keep 10 mantissa bits, round to nearest with ties away from zero (add half of the dropped field to
    the magnitude, carry into the exponent), so (2 - 2^-11) 2^127 and above round to infinity; subnormals round at the same bit"""
    b = np.asarray(x, F32).view(np.uint32)
    r = ((b.astype(np.uint64) + 0x1000) & 0xFFFFE000).astype(np.uint32)
    special = (b & 0x7F800000) == 0x7F800000
    return np.where(special, b, r).view(F32)


def tf32_split(x):
    x = np.asarray(x, F32)
    big = tf32_rna(x)
    return big, tf32_rna(x - big)


def rz32(v):
    """float64 -> fp32 rounded toward zero"""
    v = np.asarray(v, F64)
    r = v.astype(F32)
    return np.where(np.abs(r.astype(F64)) > np.abs(v), np.nextafter(r, F32(0)), r)


def _down(v):
    return np.nextafter(v, -np.inf)


def _up(v):
    return np.nextafter(v, np.inf)


def fin(parts):
    """k_finish's fp64 sum in ascending z from 0.0"""
    s = np.zeros_like(parts[0], F64)
    for p in parts:
        s = s + p
    return s


def post(x, bias, relu):
    """the epilogue of either path: fp32 value x (+ bias in fp32), ReLU"""
    v = np.asarray(x, F32)
    if bias is not None:
        v = v + bias
    return np.maximum(v, F32(0)) if relu else v


def ulps(a, b):
    return L.ordinal32(b) - L.ordinal32(a)


# ---------------------------------------------------------------------------------------------------- the products
def range_interval(a, b, kind):
    """a [M, k], b [k, N] fp32 (one k range) -> (lo, hi, s, h) float64 [M, N]: the range's partial (fp64 accumulator, or the tc kind's
    fp32 accumulator) lies in [lo, hi]; s is float64's value of the exact sum and h the bound"""
    k = a.shape[1]
    if kind == "fp64":
        a64, b64 = a.astype(F64), b.astype(F64)
        s = a64 @ b64
        t = np.abs(a64) @ np.abs(b64)
        h = (2 * k + 4) * 2.0 ** -53 * t * (1 + 2.0 ** -40)
        return _down(s - h), _up(s + h), s, h
    (ab, as_), (bb, bs) = tf32_split(a), tf32_split(b)
    ab, as_, bb, bs = (x.astype(F64) for x in (ab, as_, bb, bs))
    s = as_ @ bb + ab @ bs + ab @ bb
    t = np.abs(as_) @ np.abs(bb) + np.abs(ab) @ np.abs(bs) + np.abs(ab) @ np.abs(bb)
    nt = -(-k // TG_BK)
    h = ((96 * 2.0 ** -23 + nt * 2.0 ** -24) * (1 + 2.0 ** -20) + (3 * k + 6) * 2.0 ** -53) * t + (96 + nt) * 2.0 ** -149
    return L._ru32(_down(s - h)).astype(F64), L._rd32(_up(s + h)).astype(F64), s, h


class GemmCheck:
    """One product C = A B (+ bias, ReLU) of a step in a trainer of `kind`, per element.  A: [M, K], Bm: [K, N] fp32 (views are fine),
    got: the kernel's fp32 output [M, N], or got64: grad_rows_dev's unrounded fp64 output.  Rows are checked in blocks, so only counts,
    the first failure and statistics are kept: single (fraction of one-value sets), widest (ulps of
    the set's larger end), used (largest |got - s| / h, meaningful for the tc kind, whose sets are wider than one rounding)."""

    def __init__(self, name, kind, A, Bm, kps, got=None, bias=None, relu=False, got64=None, block=1 << 21):
        M, K = A.shape
        N = Bm.shape[1]
        self.name, self.kind, self.n = name, kind, M * N
        self.nbad, self.first, self.n_single, self.widest, self.used = 0, None, 0, 0, 0.0
        rs = ranges(K, kps)
        self.n_ranges = len(rs)
        mb = max(1, block // max(N, 1))
        for m0 in range(0, M, mb):
            m1 = min(M, m0 + mb)
            lo, hi, s, h = [], [], 0.0, 0.0
            for kb, ke in rs:
                l, u, sz, hz = range_interval(np.asarray(A[m0:m1, kb:ke], F32), np.asarray(Bm[kb:ke], F32), kind)
                lo.append(l); hi.append(u); s = s + sz; h = h + hz          # noqa: E702
            flo, fhi = fin(lo), fin(hi)
            if got64 is not None:
                g = np.asarray(got64[m0:m1], F64)
                ok = (g >= flo) & (g <= fhi)
                self._note(ok, m0, g, flo, fhi, None)
                self.n_single += int((flo == fhi).sum())
                gu = g
            else:
                g = np.asarray(got[m0:m1], F32)
                xlo, xhi = flo.astype(F32), fhi.astype(F32)
                b = None if bias is None else np.asarray(bias, F32)[None, :]
                ok = self._admissible(g, xlo, xhi, b, relu)
                plo, phi = post(xlo, b, relu), post(xhi, b, relu)
                self._note(ok, m0, g, plo, phi, xhi)
                self.n_single += int((plo == phi).sum())
                sp = np.spacing(np.maximum(np.abs(plo), np.abs(phi))).astype(F64)
                self.widest = max(self.widest, int(round(float(((phi.astype(F64) - plo.astype(F64)) / sp).max()))))
                gu = g.astype(F64) - (0 if b is None else b.astype(F64))
                if relu:
                    gu = np.where(g > 0, gu, s)                             # a clamped output says nothing about the sum
            with np.errstate(invalid="ignore", divide="ignore"):
                u = np.where(h > 0, np.abs(gu - s) / h, 0.0)
            self.used = max(self.used, float(u.max()))

    @staticmethod
    def _admissible(g, xlo, xhi, b, relu):
        """some fp32 x in [xlo, xhi] with post(x) == g: post is monotone, so its preimage of g is an fp32 interval; it meets [xlo, xhi]
        iff it holds xlo, xhi, or (lying inside) the fp32 values next to g - bias"""
        ok = post(xlo, b, relu) == g
        ok |= post(xhi, b, relu) == g
        x0 = (g.astype(F64) - (0 if b is None else b.astype(F64))).astype(F32)
        for k in range(-2, 3):
            xb = _step(x0, k)
            inside = (xb >= xlo) & (xb <= xhi)
            ok |= inside & (post(xb, b, relu) == g)
        return ok

    def _note(self, ok, m0, g, lo, hi, _):
        bad = ~ok
        nb = int(bad.sum())
        if nb and self.first is None:
            i, j = np.argwhere(bad)[0]
            gv, l, u = g[i, j], lo[i, j], hi[i, j]
            if g.dtype == F64:
                self.first = "row %d column %d: got %r (fp64), admissible [%r, %r]" % (m0 + i, j, gv, l, u)
            else:
                o = L.ordinal32(gv)
                self.first = "row %d column %d: got %r, admissible [%r, %r] = [%+d, %+d] ulps from it" % (
                    m0 + i, j, gv, l, u, L.ordinal32(l) - o, L.ordinal32(u) - o)
        self.nbad += nb

    def bad(self):
        return self.nbad

    def describe(self, what=""):
        return "%s: %s (%s kind, %d k range%s): %s (%d of %d elements out of their set)" % (
            what, self.name, self.kind, self.n_ranges, "" if self.n_ranges == 1 else "s", self.first, self.nbad, self.n)

    def single(self):
        return self.n_single / max(self.n, 1)


class ExactCheck:
    """a stage restated bit for bit: got and want must hold the same fp32 (or fp64) bits"""

    def __init__(self, name, got, want):
        self.name = name
        g, w = np.asarray(got), np.asarray(want, np.asarray(got).dtype)
        self.got, self.want = g.reshape(-1), w.reshape(-1)
        it = np.uint64 if g.dtype == F64 else np.uint32
        self.ok = self.got.view(it) == self.want.view(it)

    def bad(self):
        return int((~self.ok).sum())

    def describe(self, what=""):
        i = int(np.argmax(~self.ok))
        g, w = self.got[i], self.want[i]
        d = ""
        if self.got.dtype == F32:
            d = " (%+d ulps)" % (L.ordinal32(g) - L.ordinal32(w))
        return "%s: %s element %d: got %r, restated %r%s (%d of %d elements differ)" % (what, self.name, i, g, w, d, self.bad(), self.ok.size)


class SetCheck:
    """an fp32 output against an explicit set of candidate values (the head): ok where got equals one of them; width in ulps"""

    def __init__(self, name, got, match, lo, hi):
        self.name, self.got, self.ok, self.lo, self.hi = name, np.asarray(got, F32), match, lo, hi
        self.width = ulps(lo, hi)

    def bad(self):
        return int((~self.ok).sum())

    def describe(self, what=""):
        i = np.unravel_index(int(np.argmax(~self.ok)), self.ok.shape)
        g = self.got[i]
        o = L.ordinal32(g)
        return "%s: %s element %s: got %r, admissible set within [%r, %r] = [%+d, %+d] ulps from it (%d elements out of their set)" % (
            what, self.name, i, g, self.lo[i], self.hi[i], L.ordinal32(self.lo[i]) - o, L.ordinal32(self.hi[i]) - o, self.bad())


# ---------------------------------------------------------------------------------------------------- layout stages
def states_to_float(states):
    return np.asarray(states, np.int8).reshape(-1, 200).astype(F32)


def gather_rows(rows, idx, wscale):
    """k_gather_rows: (x0 [n, 200], value, variance, weight = visit * wscale in fp32) from 212-byte rows"""
    r = np.asarray(rows, np.uint8).reshape(-1, 212)[np.asarray(idx)]
    f = np.ascontiguousarray(r[:, 200:212]).view(F32)
    return r[:, :200].view(np.int8).astype(F32), f[:, 0].copy(), f[:, 1].copy(), f[:, 2] * F32(wscale)


def im2col(act, H, W, C, swap=False):
    """act [B, H*W*C] (NHWC) -> col [B*(H-2)*(W-2), C*9], col[(b, y, x)][ci*9 + ky*3 + kx] = act[b][y+ky][x+kx][ci]; swap: ky and kx
    exchanged (a defect)"""
    a = np.asarray(act, F32).reshape(-1, H, W, C)
    OH, OW = H - 2, W - 2
    taps = [a[:, ky:ky + OH, kx:kx + OW, :] for ky in range(3) for kx in range(3)]
    if swap:
        taps = [taps[kx * 3 + ky] for ky in range(3) for kx in range(3)]
    return np.stack(taps, -1).reshape(-1, C * 9)


def nhwc_to_flat(a3, hwc=False):
    a = np.asarray(a3, F32).reshape(-1, 56, 32)
    return a.reshape(-1, 1792) if hwc else a.transpose(0, 2, 1).reshape(-1, 1792)


def flat_to_nhwc_relu(dflat, flat):
    d = np.where(np.asarray(flat, F32) > 0, np.asarray(dflat, F32), F32(0))
    return d.reshape(-1, 32, 56).transpose(0, 2, 1).reshape(-1, 32)


def col2im_relu(dcol, act, H, W, C):
    """the adjoint of im2col: per input element the <= 9 (pixel, tap) pairs that read it, ascending tap order, fp64 from 0.0, rounded
    once, masked by act > 0 -> [B*H*W, C]"""
    OH, OW = H - 2, W - 2
    d = np.asarray(dcol, F32).reshape(-1, OH, OW, C, 9).astype(F64)
    B = d.shape[0]
    s = np.zeros((B, H, W, C), F64)
    for ky in range(3):
        for kx in range(3):
            t = np.zeros((B, H, W, C), F64)
            t[:, ky:ky + OH, kx:kx + OW, :] = d[..., ky * 3 + kx]
            s = s + t
    a = np.asarray(act, F32).reshape(B, H, W, C)
    return np.where(a > 0, s.astype(F32), F32(0)).reshape(-1, C)


def dh_of(dz, wo, h):
    """k_dh: fma(dz0, Wo0k, dz1 * Wo1k) in fp64 (both products exact), rounded, masked by h > 0"""
    dz = np.asarray(dz, F32).astype(F64)
    wo = np.asarray(wo, F32).astype(F64)
    v = dz[:, 1:2] * wo[1][None] + dz[:, 0:1] * wo[0][None]
    return np.where(np.asarray(h, F32) > 0, v.astype(F32), F32(0))


def seqsum(x, axis=0):
    """a sequential float64 sum from 0.0 along `axis` (np.add.accumulate is sequential; np.sum is pairwise)"""
    x = np.asarray(x, F64)
    if x.shape[axis] == 0:
        return np.zeros(np.delete(x.shape, axis), F64)
    return np.add.accumulate(x, axis=axis).take(-1, axis=axis) + 0.0


def colsum(X, out64=False):
    """k_colsum: out[n] = sum over 8 warps (ascending) of the warp's sequential fp64 sum over rows m = w, w + 8, ..., rounded once"""
    X = np.asarray(X, F32)
    M, N = X.shape
    pad = -M % 8
    Xp = np.concatenate([X.astype(F64), np.zeros((pad, N), F64)]).reshape(-1, 8, N)
    part = seqsum(Xp, 0)
    t = seqsum(part, 0)
    return t if out64 else t.astype(F32)


# ---------------------------------------------------------------------------------------------------- the head (k_head)
def log_range(x):
    """fp32 arguments -> (lo, hi): the fp32 values within 1 ulp of log(x), logf's documented maximum error (ulp of the exact result)"""
    e = np.log(np.asarray(x, F32).astype(F64))
    _, ex = np.frexp(e)
    ulp = np.ldexp(1.0, np.where(e != 0, np.maximum(ex - 24, -149), -149))
    return L._ru32(e - np.abs(e) * 2.0 ** -50 - ulp), L._rd32(e + np.abs(e) * 2.0 ** -50 + ulp)


def head_z(h, wo):
    """z = fma(h_k, Wo_jk, z) in ascending k from 0.0, fp64 (each product exact) -> [B, 2] float64"""
    h64 = np.asarray(h, F32).astype(F64)
    wo = np.asarray(wo, F32).astype(F64)
    z = np.zeros((len(h64), 2), F64)
    for k in range(256):
        z = z + h64[:, k:k + 1] * wo[:, k][None]
    return z


def _fp32_values(lo, hi, i):
    """the i-th fp32 value of [lo, hi] (non-negative lo), clamped at hi"""
    return np.minimum(lo.view(np.int32) + i, hi.view(np.int32)).astype(np.int32).view(F32)


def head_ops(s, ub, lb, mean, var, w, Bg, l1, l2, mutant=None):
    """k_head after the sigmoid, fp32 in the SASS's order -> (mp, vp, lossv, dz0, dz1); l1, l2 = logf(vp), logf(var)"""
    mp = s[0] * ub[0] + lb[0]
    vp = s[1] * ub[1] + lb[1]
    diff = mean - mp
    t2 = L.fma32(diff, diff, var) / vp
    lv = ((l1 + t2) - l2) - F32(1)
    lossv = w * lv
    gl = w / F32(Bg)
    dvp = gl * (F32(1) / vp - t2 / vp)
    dmp = gl * ((F32(-2) * diff) / vp)
    s0, s1 = s
    if mutant == "sigmoid_from_pred":
        s0, s1 = (mp - lb[0]) / ub[0], (vp - lb[1]) / ub[1]
    dz0 = (dmp * ub[0]) * (s0 * (F32(1) - s0))
    dz1 = (dvp * ub[1]) * (s1 * (F32(1) - s1))
    return mp, vp, lossv, dz0, dz1


def head_inputs(w, h, value, variance, weight, weighted):
    p = params(w)
    z = head_z(h, p["fow"])
    x = z.astype(F32) + p["fob"][None]
    var = np.maximum(np.asarray(variance, F32).reshape(-1), F32(0.1))
    wt = np.asarray(weight, F32).reshape(-1) if weighted else np.ones(len(x), F32)
    return p, x, var, np.asarray(value, F32).reshape(-1), wt


def head_emulated(w, h, value, variance, weight, weighted, Bg, mutant=None):
    """k_head with a correctly rounded exp and log -> pred [B, 2], lossv [B], dz [B, 2]"""
    p, x, var, mean, wt = head_inputs(w, h, value, variance, weight, weighted)
    e = L.exp_rn(-x)
    t = (1 + e.astype(F64)).astype(F32)                    # the fused FFMA: 1 + expf's unrounded (exactly scaled) result, rounded once
    s = F32(1) / t
    vp = s[:, 1] * p["ub"][1] + p["lb"][1]
    l1, l2 = np.log(vp.astype(F64)).astype(F32), np.log(var.astype(F64)).astype(F32)
    mp, vp, lossv, dz0, dz1 = head_ops((s[:, 0], s[:, 1]), p["ub"], p["lb"], mean, var, wt, Bg, l1, l2, mutant)
    return np.stack([mp, vp], 1), lossv, np.stack([dz0, dz1], 1)


def head_checks(w, h, value, variance, weight, weighted, Bg, pred, lossv, dz):
    """pred, lossv and dz against every combination of expf (2 ulp) and logf (1 ulp) values -> [SetCheck]"""
    p, x, var, mean, wt = head_inputs(w, h, value, variance, weight, weighted)
    e_lo, e_hi = L.exp_range(-x)
    t_lo = (1 + _down(e_lo.astype(F64))).astype(F32)
    t_hi = (1 + _up(e_hi.astype(F64))).astype(F32)
    nt = (t_hi.view(np.int32) - t_lo.view(np.int32)).max(0)
    l2lo, l2hi = log_range(var)
    got = [np.asarray(pred, F32)[:, 0], np.asarray(pred, F32)[:, 1], np.asarray(lossv, F32).reshape(-1), np.asarray(dz, F32)[:, 0],
           np.asarray(dz, F32)[:, 1]]
    match = [np.zeros(len(x), bool) for _ in got]
    lo = [np.full(len(x), np.inf, F32) for _ in got]
    hi = [np.full(len(x), -np.inf, F32) for _ in got]

    def note(k, v):
        match[k] |= v == got[k]
        lo[k] = np.minimum(lo[k], v)
        hi[k] = np.maximum(hi[k], v)
    for i0 in range(int(nt[0]) + 1):
        s0 = F32(1) / _fp32_values(t_lo[:, 0], t_hi[:, 0], i0)
        for i1 in range(int(nt[1]) + 1):
            s1 = F32(1) / _fp32_values(t_lo[:, 1], t_hi[:, 1], i1)
            vp = s1 * p["ub"][1] + p["lb"][1]
            l1lo, l1hi = log_range(vp)
            for j1 in range(3):
                l1 = np.minimum(_step(l1lo, j1), l1hi)
                for j2 in range(3):
                    l2 = np.minimum(_step(l2lo, j2), l2hi)
                    r = head_ops((s0, s1), p["ub"], p["lb"], mean, var, wt, Bg, l1, l2)
                    for k in range(5):
                        note(k, r[k])
    names = ["pred.v", "pred.var", "lossv", "dz.v", "dz.var"]
    return [SetCheck(names[k], got[k], match[k], lo[k], hi[k]) for k in range(5)]


def _step(x, j):
    """x moved up by j fp32 values"""
    o = L.ordinal32(x) + j
    b = np.where(o < 0, (-o) | 0x80000000, o).astype(np.int64).astype(np.uint32)
    return b.view(F32)


# ---------------------------------------------------------------------------------------------------- loss, gradient norm, clip, Yogi
def fma64(a, b, c):
    """fma(a, b, c) in float64, exactly (Fraction), elementwise over 1-d arrays"""
    out = np.empty(len(a), F64)
    for i in range(len(a)):
        q = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        out[i] = _rn64(q)
    return out


def _rn64(q):
    """a Fraction -> the nearest float64, ties to even (float(Fraction) rounds correctly)"""
    return float(q)


def _tree(s):
    s = s.copy()
    d = 128
    while d > 0:
        s[:d] = s[:d] + s[d:2 * d]
        d >>= 1
    return s[0]


def _strided(x, n_threads=256):
    x = np.asarray(x, F64)
    pad = -len(x) % n_threads
    return np.concatenate([x, np.zeros(pad)]).reshape(-1, n_threads)


def std_mean(lossv):
    """k_std_mean: (mean, population std) in fp64, 256 strided sequential partials then the tree; the second pass is a DFMA chain"""
    x = np.asarray(lossv, F32).reshape(-1).astype(F64)
    n = len(x)
    mean = _tree(seqsum(np.concatenate([np.zeros((1, 256)), _strided(x)]), 0)) / n
    a = np.zeros(256, F64)
    for r0 in range(0, n, 256):
        xs = x[r0:r0 + 256]
        d = xs - mean
        a[:len(xs)] = fma64(d, d, a[:len(xs)])
    return mean, float(np.sqrt(_tree(a) / n))


def sumsq(g):
    """k_sumsq: per tensor, 256 strided sequential sums of g*g (exact products) then the tree -> float64 [10]"""
    g = np.asarray(g, F32).astype(F64)
    out = np.zeros(N_TENSORS, F64)
    for i in range(N_TENSORS):
        x = g[T_OFF[i]:T_OFF[i + 1]]
        out[i] = _tree(seqsum(np.concatenate([np.zeros((1, 256)), _strided(x * x)]), 0))
    return out


def grad_norm(ss):
    """the host's (and k_grad_norm's) sqrt(sum_i sqrt(ss_i)^2) in tensor order"""
    tot = 0.0
    for v in ss:
        nrm = float(np.sqrt(v))
        tot = tot + nrm * nrm
    return float(np.sqrt(tot))


def clip_coef(gn, clip):
    """clip / (gn + 1e-6) as fp32 when clipping applies (< 1), else None"""
    if clip <= 0:
        return None
    c = clip / (gn + 1e-6)
    return F32(c) if c < 1.0 else None


def clipped(g_raw, coef):
    return np.asarray(g_raw, F32) if coef is None else np.asarray(g_raw, F32) * coef


def next_step(step_before):
    """the step counter: state() reports -1 before the first step (or after set_state(-1)) -> (step, first)"""
    return (1, True) if step_before < 0 else (step_before + 1, False)


def yogi_const(step, first, lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-3, wd=1e-3):
    """YogiConst from the host's double arithmetic"""
    bc1, bc2 = 1.0 - beta1 ** float(step), 1.0 - beta2 ** float(step)
    return dict(beta1=F32(beta1), omb1=F32(1.0 - beta1), nomb2=F32(-(1.0 - beta2)), wd=F32(wd), eps=F32(eps),
                sqrt_bc2=F32(float(np.sqrt(bc2))), step_size=F32(lr / bc1), first=first)


YOGI_MUTANTS = ("step_off_by_one", "v0_decayed", "sign0_plus", "eps_in_sqrt")


def yogi(p, g, m, v, c, mutant=None):
    """k_yogi in numpy float32 -> (p, m, v)"""
    p, g, m, v = (np.array(x, F32) for x in (p, g, m, v))
    if c["first"]:
        m = np.zeros_like(m)
        v = g * g
    if c["wd"] != 0:
        g = g + c["wd"] * p
    if c["first"] and mutant == "v0_decayed":
        v = g * g
    m = m * c["beta1"] + c["omb1"] * g
    gs = g * g
    d = v - gs
    sg = np.where(d > 0, F32(1), np.where(d < 0, F32(-1), F32(1) if mutant == "sign0_plus" else F32(0)))
    v = v + c["nomb2"] * (sg * gs)
    if mutant == "eps_in_sqrt":
        denom = np.sqrt(v + c["eps"]) / c["sqrt_bc2"]
    else:
        denom = np.sqrt(v) / c["sqrt_bc2"] + c["eps"]
    p = p + (-c["step_size"]) * (m / denom)
    return p, m, v


def yogi_step(step_before, hyper=None, mutant=None):
    """YogiConst of the step after a state() that reported step_before; mutant step_off_by_one: the counter one ahead from step 100 on"""
    step, first = next_step(step_before)
    if mutant == "step_off_by_one" and step >= 100:
        step += 1
    return yogi_const(step, first, **(hyper or {}))


# ---------------------------------------------------------------------------------------------------- a whole step
def products(bf, w, grad, B):
    """name -> (A [M, K], Bm [K, N], bias, relu, got [M, N] or None, gradient offset or None) of the 12 products, from the buffers the
    kernels read (bf: name -> [B, row] fp32) and the fp32 gradient vector (or None)"""
    p = params(w)
    r = {k: np.asarray(v, F32).reshape(-1, {"col1": 9, "col2": 288, "col3": 288, "a1": 32, "a2": 32, "a3": 32, "dc3": 32, "da2": 32,
                                                "da1": 32, "dcol3": 288, "dcol2": 288}.get(k, np.asarray(v).shape[-1]))
         for k, v in bf.items() if k != "d_sumsq"}

    def gw(key, shape):
        return None if grad is None else np.asarray(grad, F32)[OFF[key]:OFF[key] + shape[0] * shape[1]].reshape(shape)
    return {"conv1": (r["col1"], p["c1w"].T, p["c1b"], True, r["a1"], None),
            "conv2": (r["col2"], p["c2w"].T, p["c2b"], True, r["a2"], None),
            "conv3": (r["col3"], p["c3w"].T, p["c3b"], True, r["a3"], None),
            "fc1": (r["flat"], p["f1w"].T, p["f1b"], True, r["h"], None),
            "fc_out_wgrad": (r["dz"].T, r["h"], None, False, gw("fow", (2, 256)), "fow"),
            "fc1_wgrad": (r["dh"].T, r["flat"], None, False, gw("f1w", (256, 1792)), "f1w"),
            "dflat": (r["dh"], p["f1w"], None, False, r["dflat"], None),
            "conv3_wgrad": (r["dc3"].T, r["col3"], None, False, gw("c3w", (32, 288)), "c3w"),
            "conv2_wgrad": (r["da2"].T, r["col2"], None, False, gw("c2w", (32, 288)), "c2w"),
            "conv1_wgrad": (r["da1"].T, r["col1"], None, False, gw("c1w", (32, 9)), "c1w"),
            "dcol3": (r["dc3"], p["c3w"], None, False, r["dcol3"], None),
            "dcol2": (r["da2"], p["c2w"], None, False, r["dcol2"], None)}


BIAS_GRADS = (("fob", "dz", 2), ("f1b", "dh", 256), ("c3b", "dc3", 32), ("c2b", "da2", 32), ("c1b", "da1", 32))


def step_checks(w, bf, B, kind, weighted, grad=None, grad64=None, Bg=None, x0=None, skip=()):
    """Every stage of one step from the buffers the kernels read -> [check] in stage order.  grad: the step's fp32 gradient before any
    clipping (None: the gradient stages are skipped); grad64: grad_rows_dev's unrounded fp64 slice gradient (the weight and bias
    gradients are then held before the last rounding); Bg: the whole batch's size (grad_rows_dev), else B; x0: the expected x0 (from the
    states or the gathered rows)."""
    out = []
    if x0 is not None:
        out.append(ExactCheck("x0", bf["x0"], x0))
    p = params(w)
    out.append(ExactCheck("col1 (k_im2col)", bf["col1"], im2col(bf["x0"], 20, 10, 1)))
    out.append(ExactCheck("col2 (k_im2col)", bf["col2"], im2col(bf["a1"], 18, 8, 32)))
    out.append(ExactCheck("col3 (k_im2col)", bf["col3"], im2col(bf["a2"], 16, 6, 32)))
    out.append(ExactCheck("flat (k_nhwc_to_flat)", bf["flat"], nhwc_to_flat(bf["a3"])))
    has_grad = "dz" in bf
    if has_grad:
        out += head_checks(w, bf["h"], bf["value"], bf["variance"], bf["weight"], weighted, Bg or B, bf["pred"], bf["lossv"], bf["dz"])
        out.append(ExactCheck("dh (k_dh)", bf["dh"], dh_of(bf["dz"], p["fow"], bf["h"])))
        out.append(ExactCheck("dc3 (k_flat_to_nhwc_relu)", bf["dc3"], flat_to_nhwc_relu(bf["dflat"], bf["flat"])))
        out.append(ExactCheck("da2 (k_col2im_relu)", bf["da2"], col2im_relu(bf["dcol3"], bf["a2"], 16, 6, 32)))
        out.append(ExactCheck("da1 (k_col2im_relu)", bf["da1"], col2im_relu(bf["dcol2"], bf["a1"], 18, 8, 32)))
    g = grad if grad64 is None else None
    for name, (A, Bm, bias, relu, got, goff) in products(bf, w, g, B).items():
        if name in skip or (goff is not None and grad is None and grad64 is None) or (not has_grad and name not in FORWARD):
            continue
        kk = "fp64" if name == "fc_out_wgrad" else kind
        kps = kps_of(name, B, kind)
        if goff is not None and grad64 is not None:
            n = A.shape[0] * Bm.shape[1]
            g64 = np.asarray(grad64, F64)[OFF[goff]:OFF[goff] + n].reshape(A.shape[0], Bm.shape[1])
            out.append(GemmCheck(name + " (fp64 slice)", kk, A, Bm, kps, got64=g64))
        else:
            out.append(GemmCheck(name, kk, A, Bm, kps, got=got, bias=bias, relu=relu))
    if has_grad and (grad is not None or grad64 is not None):
        for key, src, n in BIAS_GRADS:
            X = np.asarray(bf[src], F32).reshape(-1, n)
            if grad64 is not None:
                out.append(ExactCheck(key + " (k_colsum, fp64 slice)", np.asarray(grad64, F64)[OFF[key]:OFF[key] + n], colsum(X, True)))
            else:
                out.append(ExactCheck(key + " (k_colsum)", np.asarray(grad, F32)[OFF[key]:OFF[key] + n], colsum(X)))
    if grad is not None and "d_sumsq" in bf:
        out.append(ExactCheck("d_sumsq (k_sumsq)", bf["d_sumsq"], sumsq(grad)))
    return out


FORWARD = ("conv1", "conv2", "conv3", "fc1")
# deliberate defects of a step, for the tests that show the checks catch them (emulate_step's `mutant`)
STEP_MUTANTS = {"fp64": ("fp32_acc", "bias_before_round", "round_partials"),
                "tc": ("drop_tile", "partial_twice", "drop_cross", "bias_before_round"),
                "layout": ("im2col_swap", "col2im_wrong_mask", "flat_hwc"),
                "head": ("sigmoid_from_pred", "dz_own_B")}


def _tc_range(a, b, mutant):
    """the tc kind's partial of one k range, emulated: per 32-k tile a sequential fp32 sum truncated at every k (the three exact products
    of each k added in float64 first), the tile sums added to an fp32 accumulator with round-to-nearest"""
    (ab, as_), (bb, bs) = tf32_split(a), tf32_split(b)
    k = a.shape[1]
    nt = -(-k // TG_BK)
    pad = nt * TG_BK - k

    def tiles_a(x):
        return np.pad(x.astype(F64), ((0, 0), (0, pad))).reshape(len(x), nt, TG_BK)

    def tiles_b(x):
        return np.pad(x.astype(F64), ((0, pad), (0, 0))).reshape(nt, TG_BK, x.shape[1])
    pairs = [(as_, bb), (ab, bs), (ab, bb)]
    if mutant == "drop_cross":
        pairs = pairs[1:]
    pairs = [(tiles_a(x), tiles_b(y)) for x, y in pairs]
    d = np.zeros((nt, a.shape[0], b.shape[1]), F32)
    for kk in range(TG_BK):
        pk = sum(np.einsum("mt,tn->tmn", x[:, :, kk], y[:, kk, :]) for x, y in pairs)
        d = rz32(d.astype(F64) + pk)
    if mutant == "drop_tile":
        d = d[:-1]
    acc = np.zeros((a.shape[0], b.shape[1]), F32)
    for t in range(len(d)):
        acc = acc + d[t]
    return acc.astype(F64)


def emu_gemm(A, Bm, kps, kind, bias=None, relu=False, out64=False, mutant=None):
    """one product as a trainer of `kind` computes it (fp64: float64 accumulation per range), k_finish, the epilogue"""
    A, Bm = np.asarray(A, F32), np.asarray(Bm, F32)
    parts = []
    rs = ranges(A.shape[1], kps)
    for kb, ke in rs:
        a, b = A[:, kb:ke], Bm[kb:ke]
        if kind == "tc":
            parts.append(_tc_range(a, b, mutant if len(rs) > 1 or mutant == "drop_cross" else None))
            continue
        if mutant == "fp32_acc":
            acc = np.zeros((a.shape[0], b.shape[1]), F32)
            for kk in range(a.shape[1]):
                acc = acc + a[:, kk:kk + 1] * b[kk][None]
            parts.append(acc.astype(F64))
        else:
            parts.append(a.astype(F64) @ b.astype(F64))
        if mutant == "round_partials" and len(rs) > 1:
            parts[-1] = parts[-1].astype(F32).astype(F64)
    if mutant == "partial_twice" and len(rs) > 1:
        parts.append(parts[-1])
    s = fin(parts)
    if out64:
        return s
    if mutant == "bias_before_round" and bias is not None and (kind == "fp64" or len(rs) > 1):
        v = (s + np.asarray(bias, F32).astype(F64)[None]).astype(F32)
        return np.maximum(v, F32(0)) if relu else v
    return post(s.astype(F32), None if bias is None else np.asarray(bias, F32)[None], relu)


# which product each GEMM defect is built into
MUTANT_PRODUCTS = {"fp32_acc": ("conv2",), "bias_before_round": FORWARD, "round_partials": None, "drop_tile": None,
                   "partial_twice": None, "drop_cross": None}


def emulate_step(w, x0, value, variance, weight, weighted, kind, Bg=None, mutant=None, out64=False):
    """One step of a trainer of `kind` on the rows x0 [B, 200] (float), emulated -> (buffers, fp32 gradient, fp64 gradient or None).
    Bg: the whole batch's size (a grad_rows_dev slice).  mutant: one of STEP_MUTANTS, built into the stage it names."""
    B = len(x0)
    p = params(w)
    bf = dict(x0=np.asarray(x0, F32), value=np.asarray(value, F32), variance=np.asarray(variance, F32),
              weight=np.asarray(weight, F32) if weight is not None else np.zeros(B, F32))

    def mm(name, A, Bm, bias=None, relu=False, o64=False):
        m = mutant if mutant in MUTANT_PRODUCTS and (MUTANT_PRODUCTS[mutant] is None or name in MUTANT_PRODUCTS[mutant]) else None
        k = "fp64" if name == "fc_out_wgrad" else kind
        return emu_gemm(A, Bm, kps_of(name, B, kind), k, bias, relu, o64, m if k == kind else None)
    bf["col1"] = im2col(bf["x0"], 20, 10, 1)
    bf["a1"] = mm("conv1", bf["col1"], p["c1w"].T, p["c1b"], True)
    bf["col2"] = im2col(bf["a1"], 18, 8, 32, swap=mutant == "im2col_swap")
    bf["a2"] = mm("conv2", bf["col2"], p["c2w"].T, p["c2b"], True)
    bf["col3"] = im2col(bf["a2"], 16, 6, 32)
    bf["a3"] = mm("conv3", bf["col3"], p["c3w"].T, p["c3b"], True)
    bf["flat"] = nhwc_to_flat(bf["a3"], hwc=mutant == "flat_hwc")
    bf["h"] = mm("fc1", bf["flat"], p["f1w"].T, p["f1b"], True)
    pred, lossv, dz = head_emulated(w, bf["h"], value, variance, bf["weight"], weighted, B if mutant == "dz_own_B" else (Bg or B),
                                    "sigmoid_from_pred" if mutant == "sigmoid_from_pred" else None)
    bf.update(pred=pred, lossv=lossv[:, None], dz=dz)
    bf["dh"] = dh_of(dz, p["fow"], bf["h"])
    g = np.zeros(N_TRAIN, F32)
    g64 = np.zeros(N_TRAIN, F64) if out64 else None

    def wgrad(name, key, A, Bm):
        v = mm(name, A, Bm, o64=out64)
        if out64:
            g64[OFF[key]:OFF[key] + v.size] = v.ravel()
        else:
            g[OFF[key]:OFF[key] + v.size] = v.ravel()
    wgrad("fc_out_wgrad", "fow", dz.T, bf["h"])
    wgrad("fc1_wgrad", "f1w", bf["dh"].T, bf["flat"])
    bf["dflat"] = mm("dflat", bf["dh"], p["f1w"])
    bf["dc3"] = flat_to_nhwc_relu(bf["dflat"], bf["flat"]).reshape(B, -1)
    wgrad("conv3_wgrad", "c3w", bf["dc3"].reshape(-1, 32).T, bf["col3"])
    bf["dcol3"] = mm("dcol3", bf["dc3"].reshape(-1, 32), p["c3w"])
    bf["da2"] = col2im_relu(bf["dcol3"], bf["a1"].reshape(-1)[:B * 96 * 32] if mutant == "col2im_wrong_mask" else bf["a2"], 16, 6, 32)
    wgrad("conv2_wgrad", "c2w", bf["da2"].T, bf["col2"])
    bf["dcol2"] = mm("dcol2", bf["da2"], p["c2w"])
    bf["da1"] = col2im_relu(bf["dcol2"], bf["a1"], 18, 8, 32)
    wgrad("conv1_wgrad", "c1w", bf["da1"].T, bf["col1"])
    for key, src, n in BIAS_GRADS:
        X = bf[src].reshape(-1, n)
        if out64:
            g64[OFF[key]:OFF[key] + n] = colsum(X, True)
        else:
            g[OFF[key]:OFF[key] + n] = colsum(X)
    rows = {"col1": 144 * 9, "a1": 144 * 32, "col2": 96 * 288, "a2": 96 * 32, "col3": 56 * 288, "a3": 56 * 32, "dc3": 56 * 32,
            "dcol3": 56 * 288, "da2": 96 * 32, "dcol2": 96 * 288, "da1": 144 * 32}
    bf = {k: (v.reshape(B, rows[k]) if k in rows else v) for k, v in bf.items()}
    if not out64:
        bf["d_sumsq"] = sumsq(g)
    return bf, g, g64
