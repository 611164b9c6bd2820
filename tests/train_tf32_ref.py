"""Float64 restatement of the tf32 trainer kind (Trainer(kind="tf32"), B200_TRAIN_TF32: k_gemm_tf32 in tetris_mcts_b200/csrc/trainer.cu),
on top of tests/train_layer_ref.py.

The kind keeps no im2col / col2im buffers, so the checks rebuild the operands the kernel gathered from the buffers it did keep:
- the convolutions' A operand (OP_CONV) is im2col of the layer's NHWC input, k = ci*9 + ky*3 + kx; implicit_col restates the kernel's
  index arithmetic and equals train_layer_ref.im2col (tests/test_cpu_trainer_tf32.py), which the step checks then use;
- the conv weight gradients' col^T (OP_CONV_T) is the same gather transposed;
- the input gradients of conv3 / conv2 (OP_DGRAD x OP_DGRAD_W) are one product each, K = 288 in the order k = (ky*3 + kx)*32 + co:
  da[b][y][x][ci] = (act > 0) * sum_k dY[b][y-ky][x-kx][co] * W[co][ci][ky][kx] (taps outside dY are zero terms); dgrad_operands builds
  both operands, and in float64 their product equals col2im_relu(dY . W) up to the order of the sum.

Per element every product is held to range_interval (GemmCheck, train_layer_ref's check with this interval for the tf32 kind): the
exact products of the rna_tf32 operands, and the tc kind's accumulation bound with 32 adds per 32-k tile (one product per k).  The
masked input gradient must be exactly 0 where act <= 0 and lie in its set elsewhere.  Every other stage is held bit for bit as for the
other kinds.

emulate_step is the kind's step emulated in numpy (the tile sums truncated at every add, as the tc emulation), with deliberate defects
(MUTANTS) for the tests that show the checks catch them."""
import numpy as np

import train_layer_ref as T

F32, F64 = np.float32, np.float64
CONV_IN = {"conv1": (20, 10, 1), "conv2": (18, 8, 32), "conv3": (16, 6, 32)}      # each conv's input H, W, C
MUTANTS = ("3xtf32", "rz", "tap", "drop_tile", "no_mask")


def implicit_col(act, H, W, C, n):
    """k_gemm_tf32's OP_CONV accessor (im2col_at) at every (m, k) of n boards: its own index arithmetic -> [n*(H-2)*(W-2), C*9]"""
    a = np.asarray(act, F32).reshape(-1)
    OH, OW = H - 2, W - 2
    m = np.arange(n * OH * OW)[:, None]
    k = np.arange(C * 9)[None, :]
    b = m // (OH * OW)
    r = m - b * (OH * OW)
    y = r // OW
    x = r - y * OW
    ci = k // 9
    tap = k - ci * 9
    ky = tap // 3
    kx = tap - ky * 3
    return a[((b * H + y + ky) * W + x + kx) * C + ci]


def dgrad_operands(dY, Wt, H, W, swap=False):
    """OP_DGRAD's A [n*H*W, 288] from the output gradient dY [n*(H-2)*(W-2), 32] (zero where the tap leaves dY) and OP_DGRAD_W's B
    [288, C] from the layer's weight [32][C*9], both in the k order (ky*3 + kx)*32 + co; swap: ky and kx exchanged in A (a defect)"""
    OH, OW = H - 2, W - 2
    d = np.asarray(dY, F32).reshape(-1, OH, OW, 32)
    A = np.zeros((len(d), H, W, 9, 32), F32)
    for ky in range(3):
        for kx in range(3):
            A[:, ky:ky + OH, kx:kx + OW, (kx * 3 + ky) if swap else (ky * 3 + kx), :] = d
    w = np.asarray(Wt, F32).reshape(32, -1, 9)                              # [co][ci][tap]
    return A.reshape(-1, 288), np.ascontiguousarray(w.transpose(2, 0, 1).reshape(288, -1))


def dgrad_kps(B, H, W):
    return T.tc_kps(B * H * W, 32, 288, 32)


def rz_tf32(x):
    """tf32 rounded toward zero (the low 13 bits cleared; a defect in place of rna)"""
    b = np.asarray(x, F32).view(np.uint32)
    return np.where((b & 0x7F800000) == 0x7F800000, b, b & np.uint32(0xFFFFE000)).view(F32)


# ---------------------------------------------------------------------------------------------------- the checks
def range_interval(a, b, kind="tf32"):
    """train_layer_ref.range_interval for the tf32 kind (other kinds: that function): a [M, k], b [k, N] fp32 (one k range) -> (lo, hi,
    s, h) float64 [M, N].  The products of the rna_tf32 operands are exact; inside a 32-k tile each of at most 32 product adds loses less
    than 2^-23 of the tile's |term| sum (wgmma truncates), each FADD into the chunk accumulator at most 2^-24 of the chunk's, float64's
    own matmul stays within (k + 2) 2^-53 of the |term| sum, and the accumulator is an fp32 value."""
    if kind != "tf32":
        return T.range_interval(a, b, kind)
    k = a.shape[1]
    ab, bb = T.tf32_rna(a).astype(F64), T.tf32_rna(b).astype(F64)
    s = ab @ bb
    t = np.abs(ab) @ np.abs(bb)
    nt = -(-k // T.TG_BK)
    h = ((32 * 2.0 ** -23 + nt * 2.0 ** -24) * (1 + 2.0 ** -20) + (k + 2) * 2.0 ** -53) * t + (32 + nt) * 2.0 ** -149
    return T.L._ru32(T._down(s - h)).astype(F64), T.L._rd32(T._up(s + h)).astype(F64), s, h


class GemmCheck(T.GemmCheck):
    """train_layer_ref.GemmCheck with range_interval above (the same blocks, k_finish sum, epilogue and statistics)"""

    def __init__(self, name, kind, A, Bm, kps, got=None, bias=None, relu=False, got64=None, block=1 << 21):
        M, K = A.shape
        N = Bm.shape[1]
        self.name, self.kind, self.n = name, kind, M * N
        self.nbad, self.first, self.n_single, self.widest, self.used = 0, None, 0, 0, 0.0
        rs = T.ranges(K, kps)
        self.n_ranges = len(rs)
        mb = max(1, block // max(N, 1))
        for m0 in range(0, M, mb):
            m1 = min(M, m0 + mb)
            lo, hi, s, h = [], [], 0.0, 0.0
            for kb, ke in rs:
                l, u, sz, hz = range_interval(np.asarray(A[m0:m1, kb:ke], F32), np.asarray(Bm[kb:ke], F32), kind)
                lo.append(l); hi.append(u); s = s + sz; h = h + hz          # noqa: E702
            flo, fhi = T.fin(lo), T.fin(hi)
            if got64 is not None:
                g = np.asarray(got64[m0:m1], F64)
                self._note((g >= flo) & (g <= fhi), m0, g, flo, fhi, None)
                self.n_single += int((flo == fhi).sum())
                gu = g
            else:
                g = np.asarray(got[m0:m1], F32)
                xlo, xhi = flo.astype(F32), fhi.astype(F32)
                b = None if bias is None else np.asarray(bias, F32)[None, :]
                ok = self._admissible(g, xlo, xhi, b, relu)
                plo, phi = T.post(xlo, b, relu), T.post(xhi, b, relu)
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


def masked_check(name, A, Bm, kps, got, act):
    """an input gradient: exactly +0 where act <= 0 (ExactCheck), elsewhere in its set (GemmCheck; the masked elements are replaced by
    the rounded exact sum, which lies in every set)"""
    live = np.asarray(act, F32).reshape(got.shape) > 0
    got = np.asarray(got, F32)
    dead = np.where(live, F32(0), got)
    s = (T.tf32_rna(A).astype(F64) @ T.tf32_rna(Bm).astype(F64)).astype(F32)
    return [T.ExactCheck(name + " (0 where act <= 0)", dead, np.zeros_like(dead)),
            GemmCheck(name, "tf32", A, Bm, kps, got=np.where(live, got, s))]


def step_checks(w, bf, B, weighted, grad=None, grad64=None, Bg=None, x0=None):
    """train_layer_ref.step_checks for a tf32 trainer: the same stages from the buffers it keeps, the conv operands gathered here"""
    out = []
    if x0 is not None:
        out.append(T.ExactCheck("x0", bf["x0"], x0))
    p = T.params(w)
    out.append(T.ExactCheck("flat (k_nhwc_to_flat)", bf["flat"], T.nhwc_to_flat(bf["a3"])))
    has_grad = "dz" in bf
    r = {k: np.asarray(bf[k], F32).reshape(-1, 32) for k in ("a1", "a2", "a3", "dc3", "da2", "da1") if k in bf}
    col = {"conv1": T.im2col(bf["x0"], 20, 10, 1), "conv2": T.im2col(bf["a1"], 18, 8, 32), "conv3": T.im2col(bf["a2"], 16, 6, 32)}
    prods = [("conv1", col["conv1"], p["c1w"].T, p["c1b"], True, r["a1"], None),
             ("conv2", col["conv2"], p["c2w"].T, p["c2b"], True, r["a2"], None),
             ("conv3", col["conv3"], p["c3w"].T, p["c3b"], True, r["a3"], None),
             ("fc1", bf["flat"], p["f1w"].T, p["f1b"], True, bf["h"], None)]
    if has_grad:
        out += T.head_checks(w, bf["h"], bf["value"], bf["variance"], bf["weight"], weighted, Bg or B, bf["pred"], bf["lossv"], bf["dz"])
        out.append(T.ExactCheck("dh (k_dh)", bf["dh"], T.dh_of(bf["dz"], p["fow"], bf["h"])))
        out.append(T.ExactCheck("dc3 (k_flat_to_nhwc_relu)", bf["dc3"], T.flat_to_nhwc_relu(bf["dflat"], bf["flat"])))
        g = None if grad is None or grad64 is not None else np.asarray(grad, F32)

        def gw(key, shape):
            return None if g is None else g[T.OFF[key]:T.OFF[key] + shape[0] * shape[1]].reshape(shape)
        prods += [("fc_out_wgrad", np.asarray(bf["dz"], F32).T, bf["h"], None, False, gw("fow", (2, 256)), "fow"),
                  ("fc1_wgrad", np.asarray(bf["dh"], F32).T, bf["flat"], None, False, gw("f1w", (256, 1792)), "f1w"),
                  ("dflat", bf["dh"], p["f1w"], None, False, bf["dflat"], None),
                  ("conv3_wgrad", r["dc3"].T, col["conv3"], None, False, gw("c3w", (32, 288)), "c3w"),
                  ("conv2_wgrad", r["da2"].T, col["conv2"], None, False, gw("c2w", (32, 288)), "c2w"),
                  ("conv1_wgrad", r["da1"].T, col["conv1"], None, False, gw("c1w", (32, 9)), "c1w")]
        for name, dY, key, H, W, act in (("da2", "dc3", "c3w", 16, 6, "a2"), ("da1", "da2", "c2w", 18, 8, "a1")):
            A, Bm = dgrad_operands(r[dY], p[key], H, W)
            out += masked_check(name + " (implicit input gradient)", A, Bm, dgrad_kps(B, H, W), r[name], r[act])
    for name, A, Bm, bias, relu, got, goff in prods:
        if goff is not None and grad is None and grad64 is None:
            continue
        kind = "fp64" if name == "fc_out_wgrad" else "tf32"
        kps = T.kps_of(name, B, kind)
        if goff is not None and grad64 is not None:
            n = A.shape[0] * Bm.shape[1]
            g64 = np.asarray(grad64, F64)[T.OFF[goff]:T.OFF[goff] + n].reshape(A.shape[0], Bm.shape[1])
            out.append(GemmCheck(name + " (fp64 slice)", kind, A, Bm, kps, got64=g64))
        else:
            out.append(GemmCheck(name, kind, A, Bm, kps, got=got, bias=bias, relu=relu))
    if has_grad and (grad is not None or grad64 is not None):
        for key, src, n in T.BIAS_GRADS:
            X = np.asarray(bf[src], F32).reshape(-1, n)
            if grad64 is not None:
                out.append(T.ExactCheck(key + " (k_colsum, fp64 slice)", np.asarray(grad64, F64)[T.OFF[key]:T.OFF[key] + n], T.colsum(X, True)))
            else:
                out.append(T.ExactCheck(key + " (k_colsum)", np.asarray(grad, F32)[T.OFF[key]:T.OFF[key] + n], T.colsum(X)))
    if grad is not None and "d_sumsq" in bf:
        out.append(T.ExactCheck("d_sumsq (k_sumsq)", bf["d_sumsq"], T.sumsq(grad)))
    return out


# ---------------------------------------------------------------------------------------------------- emulation
def tf32_range(a, b, mutant=None):
    """one k range as k_gemm_tf32 computes it: per 32-k tile a sequential fp32 sum truncated at every k of the exact products of the
    rna_tf32 operands, the tile sums added to an fp32 accumulator with round-to-nearest.  mutant: "3xtf32" (tc's three products),
    "rz" (operands rounded toward zero), "drop_tile" (the range's last tile left out when it has several)"""
    if mutant == "3xtf32":
        return T._tc_range(a, b, None)
    cvt = rz_tf32 if mutant == "rz" else T.tf32_rna
    ab, bb = cvt(a).astype(F64), cvt(b).astype(F64)
    k = a.shape[1]
    nt = -(-k // T.TG_BK)
    pad = nt * T.TG_BK - k
    at = np.pad(ab, ((0, 0), (0, pad))).reshape(len(ab), nt, T.TG_BK)
    bt = np.pad(bb, ((0, pad), (0, 0))).reshape(nt, T.TG_BK, bb.shape[1])
    d = np.zeros((nt, a.shape[0], b.shape[1]), F32)
    for kk in range(T.TG_BK):
        d = T.rz32(d.astype(F64) + np.einsum("mt,tn->tmn", at[:, :, kk], bt[:, kk, :]))
    if mutant == "drop_tile" and nt > 1:
        d = d[:-1]
    acc = np.zeros((a.shape[0], b.shape[1]), F32)
    for t in range(len(d)):
        acc = acc + d[t]
    return acc.astype(F64)


def emu_gemm(A, Bm, kps, bias=None, relu=False, out64=False, mutant=None):
    A, Bm = np.asarray(A, F32), np.asarray(Bm, F32)
    s = T.fin([tf32_range(A[:, kb:ke], Bm[kb:ke], mutant) for kb, ke in T.ranges(A.shape[1], kps)])
    if out64:
        return s
    return T.post(s.astype(F32), None if bias is None else np.asarray(bias, F32)[None], relu)


def emulate_step(w, x0, value, variance, weight, weighted, Bg=None, mutant=None, out64=False):
    """One step of a tf32 trainer on the rows x0 [B, 200], emulated -> (buffers, fp32 gradient, fp64 gradient or None).  mutant: one of
    MUTANTS; "tap" exchanges ky and kx in conv2's gather and in da1's, "no_mask" leaves the ReLU mask out of both input gradients."""
    B = len(x0)
    p = T.params(w)
    gm = mutant if mutant in ("3xtf32", "rz", "drop_tile") else None
    bf = dict(x0=np.asarray(x0, F32), value=np.asarray(value, F32), variance=np.asarray(variance, F32),
              weight=np.asarray(weight, F32) if weight is not None else np.zeros(B, F32))

    def mm(name, A, Bm, bias=None, relu=False, o64=False):
        if name == "fc_out_wgrad":
            return T.emu_gemm(A, Bm, T.kps_of(name, B, "fp64"), "fp64", bias, relu, o64)
        return emu_gemm(A, Bm, T.kps_of(name, B, "tf32"), bias, relu, o64, gm)
    col1 = T.im2col(bf["x0"], 20, 10, 1)
    bf["a1"] = mm("conv1", col1, p["c1w"].T, p["c1b"], True)
    col2 = T.im2col(bf["a1"], 18, 8, 32, swap=mutant == "tap")
    bf["a2"] = mm("conv2", col2, p["c2w"].T, p["c2b"], True)
    col3 = T.im2col(bf["a2"], 16, 6, 32)
    bf["a3"] = mm("conv3", col3, p["c3w"].T, p["c3b"], True)
    bf["flat"] = T.nhwc_to_flat(bf["a3"])
    bf["h"] = mm("fc1", bf["flat"], p["f1w"].T, p["f1b"], True)
    pred, lossv, dz = T.head_emulated(w, bf["h"], value, variance, bf["weight"], weighted, Bg or B)
    bf.update(pred=pred, lossv=lossv[:, None], dz=dz)
    bf["dh"] = T.dh_of(dz, p["fow"], bf["h"])
    g = np.zeros(T.N_TRAIN, F32)
    g64 = np.zeros(T.N_TRAIN, F64) if out64 else None

    def wgrad(name, key, A, Bm):
        v = mm(name, A, Bm, o64=out64)
        (g64 if out64 else g)[T.OFF[key]:T.OFF[key] + v.size] = v.ravel()

    def dgrad(dY, key, H, W, act, swap):
        A, Bm = dgrad_operands(dY, p[key], H, W, swap)
        v = emu_gemm(A, Bm, dgrad_kps(B, H, W), mutant=gm)
        return v if mutant == "no_mask" else np.where(np.asarray(act, F32).reshape(v.shape) > 0, v, F32(0))
    wgrad("fc_out_wgrad", "fow", dz.T, bf["h"])
    wgrad("fc1_wgrad", "f1w", bf["dh"].T, bf["flat"])
    bf["dflat"] = mm("dflat", bf["dh"], p["f1w"])
    bf["dc3"] = T.flat_to_nhwc_relu(bf["dflat"], bf["flat"])
    wgrad("conv3_wgrad", "c3w", bf["dc3"].T, col3)
    bf["da2"] = dgrad(bf["dc3"], "c3w", 16, 6, bf["a2"], False)
    wgrad("conv2_wgrad", "c2w", bf["da2"].T, col2)
    bf["da1"] = dgrad(bf["da2"], "c2w", 18, 8, bf["a1"], mutant == "tap")
    wgrad("conv1_wgrad", "c1w", bf["da1"].T, col1)
    for key, src, n in T.BIAS_GRADS:
        X = bf[src].reshape(-1, n)
        if out64:
            g64[T.OFF[key]:T.OFF[key] + n] = T.colsum(X, True)
        else:
            g[T.OFF[key]:T.OFF[key] + n] = T.colsum(X)
    rows = {"a1": 144 * 32, "a2": 96 * 32, "a3": 56 * 32, "dc3": 56 * 32, "da2": 96 * 32, "da1": 144 * 32}
    bf = {k: (v.reshape(B, rows[k]) if k in rows else v) for k, v in bf.items()}
    if not out64:
        bf["d_sumsq"] = T.sumsq(g)
    return bf, g, g64
