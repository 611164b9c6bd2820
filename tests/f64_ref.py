"""Float64 restatement of the two value networks and the value-net training loss (CPU, torch float64), plus the board and
weight families the precision tests run them on.

Written from the architecture alone, independently of the product kernels and of the C oracle:
- valuenet: model/model_vv.py:13-52 Net — three valid 3x3 convs (1->32->32->32) with ReLU, NCHW flatten (1792 = 32 x 14 x 4),
  fc1 256 + ReLU, fc_out 2, sigmoid, then `* out_ubound + out_lbound`.
- distnet: model/model_distributional.py:18-52 Net — the 20x10 board under two empty rows (22x10 input), 4x4 conv 1->32, LeakyReLU(0.01),
  4x4 conv 32->32, LeakyReLU, flatten 2048 (32 x 16 x 4), fc1 128, LeakyReLU, fc_v `atoms`, softmax.
- train_loss_and_grads: Model_VV._loss (model_vv.py:136-153) with GaussianLL (:94-101), the target variance clamped at 0.1, the
  (weighted) std_mean(unbiased=False), and the gradients of the mean by autograd.
Weight vectors are in the state_dict order of include/b200_tetris_mcts.h (value net) and of DistValueSimOnline (distributional net)."""
import numpy as np
import torch
import torch.nn.functional as F

VN_SHAPES = (("conv1.weight", (32, 1, 3, 3)), ("conv1.bias", (32,)), ("conv2.weight", (32, 32, 3, 3)), ("conv2.bias", (32,)),
             ("conv3.weight", (32, 32, 3, 3)), ("conv3.bias", (32,)), ("fc1.weight", (256, 1792)), ("fc1.bias", (256,)),
             ("fc_out.weight", (2, 256)), ("fc_out.bias", (2,)), ("out_ubound", (2,)), ("out_lbound", (2,)))
N_VN = 478342
N_TRAIN = 478338          # everything before out_ubound


def dn_shapes(atoms):
    return (("conv1.weight", (32, 1, 4, 4)), ("conv1.bias", (32,)), ("conv2.weight", (32, 32, 4, 4)), ("conv2.bias", (32,)),
            ("fc1.weight", (128, 2048)), ("fc1.bias", (128,)), ("fc_v.weight", (atoms, 128)), ("fc_v.bias", (atoms,)))


def unpack(w, shapes, dtype=torch.float64):
    w = np.asarray(w, np.float32).ravel()
    out, off = {}, 0
    for name, shape in shapes:
        n = int(np.prod(shape))
        out[name] = torch.from_numpy(w[off:off + n].astype(np.float64)).reshape(shape).to(dtype)
        off += n
    assert off == w.size, (off, w.size)
    return out


def grads_size(name):
    return int(np.prod(dict(VN_SHAPES)[name]))


# the tensors the tensor-core path splits into two fp16 terms after scaling by 64 (biases and fc_out stay fp32)
SPLIT_VN = ("conv1.weight", "conv2.weight", "conv3.weight", "fc1.weight")
SPLIT_DN = ("conv1.weight", "conv2.weight", "fc1.weight")


def split_max(w, shapes=VN_SHAPES, names=SPLIT_VN):
    d = unpack(w, shapes)
    return max(float(d[k].abs().max()) for k in names)


def pack(d, shapes):
    return np.concatenate([np.asarray(d[name], np.float32).ravel() for name, _ in shapes])


def _x(states, dtype):
    return torch.from_numpy(np.asarray(states, np.int8).reshape(-1, 1, 20, 10).astype(np.float64)).to(dtype)


def _vn_forward(p, x):
    a = F.relu(F.conv2d(x, p["conv1.weight"], p["conv1.bias"]))
    a = F.relu(F.conv2d(a, p["conv2.weight"], p["conv2.bias"]))
    act3 = F.relu(F.conv2d(a, p["conv3.weight"], p["conv3.bias"])).flatten(1)
    h = F.relu(act3 @ p["fc1.weight"].T + p["fc1.bias"])
    out = torch.sigmoid(h @ p["fc_out.weight"].T + p["fc_out.bias"]) * p["out_ubound"] + p["out_lbound"]
    return out, act3, h


def valuenet(w, states, chunk=4096):
    """-> (v, var, act3) as float64 numpy; act3[k, c*56 + y*4 + x] is the flatten input of fc1 (the order b200_debug_act3 returns)."""
    p = unpack(w, VN_SHAPES)
    x = _x(states, torch.float64)
    outs, acts = [], []
    with torch.no_grad():
        for i in range(0, len(x), chunk):
            o, a, _ = _vn_forward(p, x[i:i + chunk])
            outs.append(o)
            acts.append(a)
    o, a = torch.cat(outs).numpy(), torch.cat(acts).numpy()
    return o[:, 0], o[:, 1], a


def valuenet_stats(w, states):
    """Largest magnitudes the fp16 x 2 split meets on these boards: conv activations, fc1 pre-activations, logits."""
    p = unpack(w, VN_SHAPES)
    x = _x(states, torch.float64)
    with torch.no_grad():
        a1 = F.relu(F.conv2d(x, p["conv1.weight"], p["conv1.bias"]))
        a2 = F.relu(F.conv2d(a1, p["conv2.weight"], p["conv2.bias"]))
        a3 = F.relu(F.conv2d(a2, p["conv3.weight"], p["conv3.bias"])).flatten(1)
        z1 = a3 @ p["fc1.weight"].T + p["fc1.bias"]
        lg = F.relu(z1) @ p["fc_out.weight"].T + p["fc_out.bias"]
    return dict(act=max(float(a1.abs().max()), float(a2.abs().max()), float(a3.abs().max())), fc1=float(z1.abs().max()),
                logit=float(lg.abs().max()), weight=float(max(p[k].abs().max() for k in p if k.endswith("weight"))))


# The two families a plain rtol 1e-5 does not fit, and the allowance each gets on top of it (every other family is held to 1e-5 alone):
# "saturated": a tiny output whose relative error is the absolute error of its logit -> the logit's fp32 rounding ("cond");
# "subnormal": an absolute error floor per activation -> that floor carried into the logit ("floor").
ALLOWANCE = {"saturated": "cond", "subnormal": "floor"}
ACT_FLOOR = 2.0 ** -26          # per act3 element: the absolute error the layer check allows on top of 2^-19 T3


def _sigma_max(m):
    return float(torch.linalg.matrix_norm(m, ord=2))


def valuenet_sensitivity(w, states, allowance=None):
    """Per output, the rounding allowance of an ill-conditioned family (see test_gpu_net_precision's docstring), |d out / d z_k| times
    "cond":  67 * 2^-24 S_out + 2^-18 S_fc1, where S_out = |h| . |w_out_k| + |b_out_k| bounds the terms of the logit z_k and
             S_fc1 = (|act3| . |W_fc1|^T + |b_fc1|) . |w_out_k| those of fc1 carried into z_k;
    "floor": 2^-24 ||w_out_k||_2 sigma_max(W_fc1), independent act3 errors of at most ACT_FLOOR carried into z_k;
    None: 0.  -> (sens_v, sens_var, T3 = |a2| * |W3| + |b3| per act3 element)."""
    p = unpack(w, VN_SHAPES)
    x = _x(states, torch.float64)
    with torch.no_grad():
        a1 = F.relu(F.conv2d(x, p["conv1.weight"], p["conv1.bias"]))
        a2 = F.relu(F.conv2d(a1, p["conv2.weight"], p["conv2.bias"]))
        t3 = F.conv2d(a2, p["conv3.weight"].abs(), p["conv3.bias"].abs()).flatten(1)       # sum of |terms| of each act3 element
        a3 = F.relu(F.conv2d(a2, p["conv3.weight"], p["conv3.bias"])).flatten(1)
        h = F.relu(a3 @ p["fc1.weight"].T + p["fc1.bias"])
        z = h @ p["fc_out.weight"].T + p["fc_out.bias"]
        s_out = h @ p["fc_out.weight"].abs().T + p["fc_out.bias"].abs()
        s_fc1 = (a3 @ p["fc1.weight"].abs().T + p["fc1.bias"].abs()) @ p["fc_out.weight"].abs().T
        floor = 2.0 ** -24 * p["fc_out.weight"].norm(dim=1) * _sigma_max(p["fc1.weight"])
        sg = torch.sigmoid(z)
        dz = {"cond": 67 * 2.0 ** -24 * s_out + 2.0 ** -18 * s_fc1, "floor": floor.expand_as(z), None: torch.zeros_like(z)}[allowance]
        sens = p["out_ubound"] * sg * (1 - sg) * dz
    return sens[:, 0].numpy(), sens[:, 1].numpy(), t3.numpy()


def valuenet_head(w, act3):
    """fc1 -> ReLU -> fc_out -> sigmoid -> bounds from a given act3 (torch order), float64: (v, var)"""
    p = unpack(w, VN_SHAPES)
    with torch.no_grad():
        a = torch.from_numpy(np.asarray(act3, np.float64))
        h = F.relu(a @ p["fc1.weight"].T + p["fc1.bias"])
        o = torch.sigmoid(h @ p["fc_out.weight"].T + p["fc_out.bias"]) * p["out_ubound"] + p["out_lbound"]
    return o[:, 0].numpy(), o[:, 1].numpy()


def split_act(a, terms=2):
    """An activation as the tensor-core path stores it: 16 a rounded to fp16 (x1) and the rest rounded to fp16 again (x2), over 16;
    terms=1 keeps x1 alone.  numpy's float16 has IEEE subnormals, as the device's has."""
    s = np.asarray(a, np.float32) * np.float32(16)
    x1 = s.astype(np.float16)
    out = x1.astype(np.float64)
    if terms == 2:
        out = out + (s - x1.astype(np.float32)).astype(np.float16).astype(np.float64)
    return out / 16


def distnet_sensitivity(w, states, atoms, allowance=None):
    """Per board, the rounding allowance of an ill-conditioned family on the logits, max over atoms (the terms of valuenet_sensitivity;
    k_tdc_fc sums 128 products per logit): "cond" 128 * 2^-24 S_v + 2^-18 S_fc1, "floor" 2^-24 ||w_v_a||_2 sigma_max(W_fc1), None 0."""
    p = unpack(w, dn_shapes(atoms))
    x = F.pad(_x(states, torch.float64), (0, 0, 2, 0))
    with torch.no_grad():
        a = F.leaky_relu(F.conv2d(x, p["conv1.weight"], p["conv1.bias"]), 0.01)
        a = F.leaky_relu(F.conv2d(a, p["conv2.weight"], p["conv2.bias"]), 0.01).flatten(1)
        h = F.leaky_relu(a @ p["fc1.weight"].T + p["fc1.bias"], 0.01)
        s_v = h.abs() @ p["fc_v.weight"].abs().T + p["fc_v.bias"].abs()
        s_fc1 = (a.abs() @ p["fc1.weight"].abs().T + p["fc1.bias"].abs()) @ p["fc_v.weight"].abs().T
        floor = 2.0 ** -24 * p["fc_v.weight"].norm(dim=1) * _sigma_max(p["fc1.weight"])
        dz = {"cond": 128 * 2.0 ** -24 * s_v + 2.0 ** -18 * s_fc1, "floor": floor.expand_as(s_v), None: torch.zeros_like(s_v)}[allowance]
        return dz.max(1).values.numpy()


def distnet(w, states, atoms, dtype=torch.float64):
    p = unpack(w, dn_shapes(atoms), dtype)
    x = F.pad(_x(states, dtype), (0, 0, 2, 0))                  # two empty rows on top: 22x10
    with torch.no_grad():
        a = F.leaky_relu(F.conv2d(x, p["conv1.weight"], p["conv1.bias"]), 0.01)
        a = F.leaky_relu(F.conv2d(a, p["conv2.weight"], p["conv2.bias"]), 0.01).flatten(1)
        h = F.leaky_relu(a @ p["fc1.weight"].T + p["fc1.bias"], 0.01)
        logits = h @ p["fc_v.weight"].T + p["fc_v.bias"]
        return torch.softmax(logits, 1).numpy(), logits.numpy()


def train_loss_and_grads(w, batch, weighted, dtype=torch.float64):
    """Model_VV._loss + backward on one batch [states, value, variance, weight]:
    -> dict(loss, loss_std, grad_norm, grads = {name: numpy}, grad_flat = state_dict-order float64 vector of the trainable tensors)."""
    p = unpack(w, VN_SHAPES, dtype)
    for k in p:
        if k not in ("out_ubound", "out_lbound"):
            p[k].requires_grad_(True)
    states, value, variance = batch[0], batch[1], batch[2]
    x = _x(states, dtype)
    mean = torch.from_numpy(np.asarray(value, np.float64).reshape(-1, 1)).to(dtype)
    var = torch.from_numpy(np.asarray(variance, np.float64).reshape(-1, 1)).to(dtype).clamp(min=0.1)
    out, _, _ = _vn_forward(p, x)
    mean_pred, var_pred = out[:, 0:1], out[:, 1:2]
    logl = var_pred.log() + ((mean - mean_pred) ** 2 + var) / var_pred - var.log() - 1
    if weighted:
        logl = torch.from_numpy(np.asarray(batch[3], np.float64).reshape(-1, 1)).to(dtype) * logl
    std, m = torch.std_mean(logl, unbiased=False)
    m.backward()
    m, std = m.detach(), std.detach()
    names = [n for n, _ in VN_SHAPES[:10]]
    grads = {n: p[n].grad.detach().to(torch.float64).numpy() for n in names}
    flat = np.concatenate([grads[n].ravel() for n in names])
    return dict(loss=float(m), loss_std=float(std), grad_norm=float(np.sqrt(sum(float((g ** 2).sum()) for g in grads.values()))),
                grads=grads, grad_flat=flat)


# ---------------------------------------------------------------------------------------------------- board families
def _settled(rng, n, top):
    """random settled cells below row `top`, about half full"""
    b = (rng.random((n, 20, 10)) < 0.5).astype(np.int8)
    b[:, :top] = 0
    return b


def impulse_boards():
    """400 boards: one settled cell at each of the 200 cells, then one falling-piece cell at each of the 200 cells."""
    b = np.zeros((400, 20, 10), np.int8)
    for c in range(200):
        b[c].flat[c] = 1
        b[200 + c].flat[c] = -1
    return b


def edge_boards(seed=0):
    """Named families of boards the key decoders and the conv taps must get right cell by cell."""
    rng = np.random.default_rng(seed)
    fam = {}
    e = np.zeros((4, 20, 10), np.int8)
    e[1, 0, 3:7] = -1                                               # I piece on an empty board
    e[2, 19, 9] = -1                                                # a single piece cell in the last cell
    e[3, 0, 0] = -1                                                 # ... and in the first
    fam["empty"] = e
    full = []
    for k in (1, 2, 3, 4, 8):                                       # full bottom rows (with holes above them)
        b = _settled(rng, 2, 20 - k - 4)
        b[:, 20 - k:] = 1
        b[1, 0:2, 4:6] = -1
        full.append(b)
    fam["full_rows"] = np.concatenate(full)
    pieces = []
    for r0 in range(16, 20):                                        # pieces in the bottom rows and in column 9
        for shape in ([(0, 0), (0, -1), (0, -2), (0, -3)], [(0, 0), (-1, 0), (0, -1), (-1, -1)], [(0, 0), (-1, 0), (-2, 0), (-3, 0)],
                      [(0, 0), (0, -1), (-1, -1), (-1, -2)]):
            for c0 in (9, int(rng.integers(3, 9))):
                b = _settled(rng, 1, 4)[0]
                cells = [(r0 + dr, c0 + dc) for dr, dc in shape if 0 <= r0 + dr < 20]
                for r, c in cells:
                    b[r, c] = -1
                pieces.append(b)
    for c0 in range(10):                                            # vertical I in every column, resting on the floor
        b = _settled(rng, 1, 8)[0]
        b[16:20, c0] = -1
        pieces.append(b)
    fam["bottom_and_col9"] = np.stack(pieces)
    part = []
    for ncell in (1, 2, 3):                                         # a piece partly above the board: 1-3 visible cells
        for _ in range(12):
            b = _settled(rng, 1, int(rng.integers(4, 14)))[0]
            r = int(rng.integers(0, 20 if ncell == 1 else 2))
            c = int(rng.integers(0, 11 - ncell))
            if rng.random() < 0.5:
                b[r, c:c + ncell] = -1
            else:
                b[max(0, r - ncell + 1):max(0, r - ncell + 1) + ncell, min(c, 9)] = -1
            part.append(b)
    fam["partial_piece"] = np.stack(part)
    return fam


def real_positions(n, seed, oracle):
    """positions of random-play games of the CPU oracle's Tetris (the observations pyTetris returns)"""
    rng = np.random.default_rng(seed)
    g = oracle.Game(seed=seed)
    out = []
    while len(out) < n:
        if g.end:
            g.reset()
        g.play(int(rng.integers(0, 7)))
        out.append(g.state())
    return np.stack(out).astype(np.int8)


def board_families(oracle, seed=0):
    fam = {"impulse": impulse_boards()}
    fam.update(edge_boards(seed))
    fam["real"] = real_positions(96, 5 + seed, oracle)
    return fam


# ---------------------------------------------------------------------------------------------------- weight families
def init_weights(seed):
    """U(+-1/sqrt(fan_in)) for weight and bias (torch's default init), out_ubound [1e2, 1e3], out_lbound [0, 0.1]"""
    rng = np.random.default_rng(seed)
    parts = []
    for (name, shape) in VN_SHAPES[:10]:
        fan_in = {"conv1": 9, "conv2": 288, "conv3": 288, "fc1": 1792, "fc_out": 256}[name.split(".")[0]]
        b = 1.0 / np.sqrt(fan_in)
        parts.append(rng.uniform(-b, b, size=shape).astype(np.float32).ravel())
    return np.concatenate(parts + [np.array([1e2, 1e3], np.float32), np.array([0.0, 1e-1], np.float32)])


def _rescale(w, conv, fc1, fc_out=None):
    """Scale conv layer l (weights and bias) by conv[l], fc1 by fc1, with the biases scaled by the running product, so that by the
    positive homogeneity of ReLU every activation is an exact power-of-two (or plain) multiple of the unscaled one; fc_out
    undoes the total (default) so that the logits are unchanged in exact arithmetic."""
    d = unpack(w, VN_SHAPES)
    run = 1.0
    for l, s in enumerate(conv):
        run *= s
        d["conv%d.weight" % (l + 1)] *= s
        d["conv%d.bias" % (l + 1)] *= run
    run *= fc1
    d["fc1.weight"] *= fc1
    d["fc1.bias"] *= run
    d["fc_out.weight"] *= (1.0 / run) if fc_out is None else fc_out
    return pack({k: v.numpy() for k, v in d.items()}, VN_SHAPES)


def weight_families(seed=0):
    """Deterministic variations of init_weights(seed), each aimed at one part of the fp16 x 2 working range."""
    w0 = init_weights(seed)
    fam = {"init": w0}
    # conv activations up to ~10^3 (16a stays below fp16's 65504), fc1 pre-activations ~10^3; logits unchanged
    fam["act_1e3"] = _rescale(w0, (8.0, 8.0, 32.0), 1.0)
    # activations in 2^-18 .. 2^-7 (94-100 % of the non-zero ones; medians 2^-11 .. 2^-14) and the conv1 / fc1 weights (96 % of the split
    # weights) below 2^-9: the high fp16 term is normal, the low one subnormal (an absolute error floor)
    fam["subnormal"] = _rescale(w0, (2.0 ** -9, 1.0, 1.0), 2.0 ** -4)
    d = unpack(w0, VN_SHAPES)
    dead = {k: v.clone() for k, v in d.items()}                   # most ReLUs dead: biases pushed well below zero
    for l in (1, 2, 3):
        dead["conv%d.bias" % l] -= {1: 0.5, 2: 0.2, 3: 0.05}[l]
    dead["fc1.bias"] -= 0.01
    fam["mostly_dead"] = pack({k: v.numpy() for k, v in dead.items()}, VN_SHAPES)
    live = {k: v.clone() for k, v in d.items()}                   # every ReLU live: biases above the largest negative input
    live["conv1.bias"] += 2.0
    live["conv2.bias"] += 5.0
    live["conv3.bias"] += 5.0
    live["fc1.bias"] += 8.0
    live["fc_out.weight"] *= 0.05
    fam["all_live"] = pack({k: v.numpy() for k, v in live.items()}, VN_SHAPES)
    sat = {k: v.clone() for k, v in d.items()}                    # logits of tens: v = ub * sigmoid(~-25) is tiny, var saturates at ub + lb
    sat["fc_out.weight"] *= 60.0
    sat["fc_out.bias"] = torch.tensor([-25.0, 25.0], dtype=torch.float64)
    fam["saturated"] = pack({k: v.numpy() for k, v in sat.items()}, VN_SHAPES)
    big = w0.copy()                                               # bounds of a trained model (out_ubound = max of the targets)
    big[N_TRAIN:N_TRAIN + 2] = [2e4, 5e6]
    fam["trained_bounds"] = big
    return fam


def dist_init_weights(seed, atoms):
    rng = np.random.default_rng(seed + 1000)
    parts = []
    for (name, shape) in dn_shapes(atoms):
        fan_in = {"conv1": 16, "conv2": 512, "fc1": 2048, "fc_v": 128}[name.split(".")[0]]
        b = 1.0 / np.sqrt(fan_in)
        parts.append(rng.uniform(-b, b, size=shape).astype(np.float32).ravel())
    return np.concatenate(parts)


def dist_weight_families(seed, atoms):
    """init; activations ~10^2-10^3 (logits unchanged); subnormal low terms; logits spread over +-60 (softmax saturated)."""
    sh = dn_shapes(atoms)
    w0 = dist_init_weights(seed, atoms)
    fam = {"init": w0}

    def scaled(s1, s2, sf, sv, bv=None):
        d = unpack(w0, sh)
        d["conv1.weight"] *= s1; d["conv1.bias"] *= s1                          # noqa: E702
        d["conv2.weight"] *= s2; d["conv2.bias"] *= s1 * s2                     # noqa: E702
        d["fc1.weight"] *= sf; d["fc1.bias"] *= s1 * s2 * sf                    # noqa: E702
        d["fc_v.weight"] *= sv
        if bv is not None:
            d["fc_v.bias"] = torch.from_numpy(bv)
        return pack({k: v.numpy() for k, v in d.items()}, sh)

    fam["act_1e3"] = scaled(16.0, 16.0, 1.0, 1.0 / 256)
    fam["subnormal"] = scaled(2.0 ** -9, 1.0, 2.0 ** -4, 2.0 ** 13)
    bv = np.linspace(-60.0, 60.0, atoms)                          # one atom far ahead of the rest; the last ones underflow to 0 in fp32
    fam["saturated"] = scaled(1.0, 1.0, 1.0, 1.0, bv)
    return fam
