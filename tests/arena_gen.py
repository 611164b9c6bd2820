"""Seeded synthetic search arenas in the reference's array layout (agents/agent.py:58-88), per SURVEY §8(d):
7-ary, depth 4-12, visit in [1,1000], value ~ U(0,50), variance ~ U(1,100), score non-decreasing along edges,
10-30 % duplicated observations among siblings."""
import numpy as np


def make_arena(seed, M=4096, max_depth=8, p_expand=0.6, p_dup=0.2, p_zero_child=0.1, unvisited=0.0, single_low=False):
    rng = np.random.default_rng(seed)
    child = np.zeros((M, 7), np.int32)
    score = np.zeros(M, np.float32)
    n2o = np.zeros(M, np.int32)
    depth = np.zeros(M, np.int32)
    nxt, nobs = 2, 2
    n2o[1] = 1
    score[1] = float(rng.integers(0, 500))
    frontier = [1]
    while frontier:
        n = frontier.pop(0)
        if depth[n] >= max_depth or nxt + 7 >= M:
            continue
        if n != 1 and rng.random() > p_expand:
            continue
        sib_obs = []
        for a in range(7):
            if rng.random() < p_zero_child:
                continue
            c = nxt
            nxt += 1
            child[n, a] = c
            depth[c] = depth[n] + 1
            score[c] = score[n] + float(rng.choice([0, 0, 0, 1, 2, 34, 100, 300]))
            if sib_obs and rng.random() < p_dup:
                n2o[c] = sib_obs[rng.integers(0, len(sib_obs))]
            else:
                n2o[c] = nobs
                nobs += 1
            sib_obs.append(n2o[c])
            frontier.append(c)
        if child[n].any() and rng.random() < 0.15:   # the same child in two slots
            nz = np.nonzero(child[n])[0]
            z = np.nonzero(child[n] == 0)[0]
            if len(z):
                child[n, z[0]] = child[n, nz[0]]
    visit = np.zeros(M, np.int32)
    value = np.zeros(M, np.float32)
    variance = np.zeros(M, np.float32)
    visit[1:nobs] = rng.integers(1, 1001, nobs - 1)
    value[1:nobs] = rng.uniform(0, 50, nobs - 1).astype(np.float32)
    variance[1:nobs] = rng.uniform(1, 100, nobs - 1).astype(np.float32)
    if unvisited > 0:
        mask = rng.random(nobs) < unvisited
        mask[:2] = False
        if single_low:   # at most one low observation per sibling set, so rand() % 1 == 0 whatever rand() returns
            for n in range(1, nxt):
                obs = sorted(set(int(n2o[c]) for c in child[n] if c))
                low = [o for o in obs if mask[o]]
                for o in low[1:]:
                    mask[o] = False
        idx = np.nonzero(mask)[0]
        visit[idx] = 0
        value[idx] = 0
        variance[idx] = 0
    return dict(child=child, visit=visit, value=value, variance=variance, score=score, n2o=n2o, n_nodes=nxt, n_obs=nobs)


def near_tie_arena(seed, M=64):
    """Root with seven children whose CLT scores differ in the last float bits: exercises core.h:94-101 rounding."""
    rng = np.random.default_rng(seed)
    a = dict(child=np.zeros((M, 7), np.int32), visit=np.zeros(M, np.int32), value=np.zeros(M, np.float32),
             variance=np.zeros(M, np.float32), score=np.zeros(M, np.float32), n2o=np.zeros(M, np.int32))
    a["n2o"][1] = 1
    a["score"][1] = 17.0
    base_v = np.float32(rng.uniform(10, 40))
    for i in range(7):
        c = 2 + i
        a["child"][1, i] = c
        a["n2o"][c] = 2 + i
        a["score"][c] = 17.0 + float(rng.integers(0, 3))
        a["visit"][2 + i] = int(rng.integers(5, 9))
        a["value"][2 + i] = np.nextafter(base_v, np.float32(100), dtype=np.float32) if rng.random() < 0.5 else base_v
        a["variance"][2 + i] = np.float32(rng.choice([4.0, 4.0000005, 3.9999998]))
    a["visit"][1] = 50
    a["n_nodes"], a["n_obs"] = 9, 9
    return a


def boards(n, seed):
    """tools/test.py:23-28 style inputs for the value network: random {0,1} cells, top rows cleared, four -1 cells."""
    rng = np.random.default_rng(seed)
    b = (rng.random((n, 20, 10)) < 0.45).astype(np.int8)
    for i in range(n):
        b[i, :rng.integers(2, 12)] = 0
        r, c = rng.integers(0, 3), rng.integers(0, 8)
        b[i, r:r + 2, c:c + 2] = -1
    return b


def state_to_obskey(s):
    """int8[20,10] observation -> SPEC §6 observation key (test helper for the synthetic evaluator)."""
    key = np.zeros(12, np.uint32)
    cells = []
    for r in range(20):
        row = 0
        for c in range(10):
            if s[r, c] == 1:
                row |= 1 << c
            elif s[r, c] == -1:
                cells.append(r * 10 + c)
        key[r >> 1] |= np.uint32(row << ((r & 1) * 16))
    cells.sort()
    key[10] = np.uint32(sum(v << (8 * i) for i, v in enumerate(cells[:4])))
    return key


def make_dist_arena(seed, M=512, bins=50, max_depth=6, unvisited=0.0):
    """Seeded node-indexed arena for the distributional cores: node_stats f32[M,5] = {visit, mean, reward, variance, M2},
    node_dist f32[M,bins] (rows sum to 1), child int32[M,7] (agents/core_distributional.py)."""
    a = make_arena(seed, M=M, max_depth=max_depth, p_dup=0.0)
    rng = np.random.default_rng(seed + 7)
    n = a["n_nodes"]
    ns = np.zeros((M, 5), np.float32)
    ns[1:n, 0] = rng.integers(1, 400, n - 1)
    ns[1:n, 1] = rng.uniform(0, 800, n - 1)
    ns[:, 2] = a["score"]
    ns[1:n, 3] = rng.uniform(1, 5000, n - 1)
    ns[1:n, 4] = ns[1:n, 3] * np.maximum(ns[1:n, 0] - 1, 1)
    if unvisited > 0:
        m = rng.random(M) < unvisited
        m[:2] = False
        ns[m, 0] = 0
    nd = rng.random((M, bins)).astype(np.float32) ** 4
    nd /= nd.sum(axis=1, keepdims=True)
    return dict(child=a["child"], node_stats=ns, node_dist=nd.astype(np.float32), n_nodes=n)


# ---- edge cases of the distributional backup (tests/golden/dist_edges_golden.npz, DESIGN §3)
DIST_EDGE_ATOMS = (2, 3, 31, 32, 33, 50, 56, 63, 64)                 # one / two bins per lane, the 64-float shared row
DIST_EDGE_RANGES = ((0.0, 5000.0), (0.0, 1000.0), (0.0, 45.0), (0.0, 200.0), (-300.0, 700.0))
DIST_EDGE_EXTRA = ((30, 0.0, 1000.0), (14, 0.0, 5000.0), (35, 0.0, 45.0), (28, 0.0, 5000.0), (60, 0.0, 1000.0), (44, 0.0, 200.0),
                   (58, -300.0, 700.0))                                # where integer x truncate one bin further (truncation_shifts)
DIST_EDGE_DEPTHS = (1, 5, 40)


def dist_edge_configs():
    """(atoms, vmin, vmax) of the edge goldens."""
    return [(a, lo, hi) for a in DIST_EDGE_ATOMS for lo, hi in DIST_EDGE_RANGES] + list(DIST_EDGE_EXTRA)


def truncation_shifts(bins, vmin, vmax, xmax, step=1.0):
    """x in [0, xmax] (multiples of step) for which shift_distribution's int(b + x / delta), clamped to the top bin, differs from
    b + int(x / delta) for some source bin b: x / delta lies just below an integer and adding b rounds the double sum up to it."""
    delta = (vmax - vmin) / bins
    x = np.arange(0.0, xmax + step / 2, step)
    bs = x / delta
    b = np.arange(bins, dtype=np.float64)[None, :]
    T = bins - 1
    differ = np.minimum(np.trunc(b + bs[:, None]), T) != np.minimum(b + np.trunc(bs)[:, None], T)
    return x[differ.any(axis=1)]


def edge_dists(bins, seed):
    """Histograms: random, one-hot at 0 (the game-over leaf), one-hot at the top bin, zero except one bin (not normalised)."""
    rng = np.random.default_rng(seed)
    r = rng.random(bins).astype(np.float32) ** 3
    r /= r.sum()
    one0, oneT, single = (np.zeros(bins, np.float32) for _ in range(3))
    one0[0], oneT[-1], single[bins // 2] = 1.0, 1.0, 0.37
    return np.stack([r.astype(np.float32), one0, oneT, single])


def edge_shifts(bins, vmin, vmax, seed):
    """x: 0, multiples of delta, truncation cases (up to five integer, four on a finer grid), at and beyond the range (all mass clamped
    into the top bin), random.  Returns (xs, the integer truncation cases)."""
    rng = np.random.default_rng(seed)
    w = vmax - vmin
    delta = w / bins
    spread = lambda a, k: a[np.unique(np.linspace(0, len(a) - 1, k).astype(int))] if len(a) else a      # noqa: E731
    near = spread(truncation_shifts(bins, vmin, vmax, 2 * w), 5)                                     # integer x (game scores)
    fine = spread(truncation_shifts(bins, vmin, vmax, w, delta / 64), 4)                             # x on a delta / 64 grid
    xs = [0.0, delta, 2 * delta, (bins // 2) * delta, (bins - 1) * delta] + list(near) + list(fine) + [vmax, w, 1.5 * w, 10 * w]
    xs += list(rng.uniform(0, w, 2)) + list(rng.integers(0, int(w) + 1, 2).astype(float))
    return np.array(xs, np.float64), near


def edge_backup_cases(bins, vmin, vmax, seed):
    """Traces of depth 1, 5 and 40 on nodes 1..D (node 0 untouched) at visit 0, 1 and many.  Each level's x = r - reward is an integer
    taken from edge_shifts (so the float32 reward holds it exactly): truncation cases, 0, clamped, random."""
    rng = np.random.default_rng(seed)
    xs, near = edge_shifts(bins, vmin, vmax, seed)
    pool = np.unique(np.round(xs))
    r = float(np.ceil(pool.max()) + 1000.0)
    dists = edge_dists(bins, bins)
    out = []
    for k, D in enumerate(DIST_EDGE_DEPTHS):
        M = D + 1
        ns = np.zeros((M, 5), np.float32)
        nd = np.zeros((M, bins), np.float32)
        trace = (rng.permutation(D) + 1).astype(np.int32)
        for t, idx in enumerate(trace):
            x = pool[(t * 7 + k) % len(pool)] if t % 3 else near[t % len(near)] if len(near) else 0.0
            n = (0, 1, 37, 2, 250)[t % 5]
            ns[idx] = (n, rng.uniform(0, vmax - vmin), r - x, 0, 0)
            if n:
                v = rng.uniform(1, 5000)
                ns[idx, 4] = v * max(n - 1, 0)
                ns[idx, 3] = v if n > 1 else 0
                row = rng.random(bins).astype(np.float32) ** 2
                nd[idx] = row / row.sum()
        dk = (1, 2, 0)[k]                                             # one-hot at 0 (game over), one-hot at the top bin, random
        out.append(dict(trace=trace, node_stats=ns, node_dist=nd, r=r, dist_k=dk, dist=dists[dk]))
    return out


def load_dist_edges(path):
    """The edge goldens as lists of cases: shift (cfg, dist, x, out), mean_variance (cfg, dist, mv), backup (cfg, trace, ..., bk_stats, bk_dist)."""
    z = np.load(path)
    cfgs = [tuple(c) for c in z["cfg"].tolist()]
    cfgs = [(int(a), lo, hi) for a, lo, hi in cfgs]
    dists = [z["dists_%d" % i] for i in range(len(cfgs))]
    shift = []
    off = z["sh_off"]
    for i, (c, k) in enumerate(z["sh_idx"].tolist()):
        shift.append(dict(cfg=cfgs[c], dist=dists[c][k], dist_k=k, x=float(z["sh_x"][i]), out=z["sh_out"][off[i]:off[i + 1]]))
    mv = [dict(cfg=cfgs[c], dist=dists[c][k], mv=z["mv_out"][i]) for i, (c, k) in enumerate(z["mv_idx"].tolist())]
    backup = []
    no, fo, to = z["tr_node_off"], z["tr_nd_off"], z["tr_off"]
    for i, (c, k) in enumerate(z["tr_idx"].tolist()):
        bins, ns, nd = cfgs[c][0], slice(no[i], no[i + 1]), slice(fo[i], fo[i + 1])
        backup.append(dict(cfg=cfgs[c], dist=dists[c][k], r=float(z["tr_r"][i]), trace=z["tr_trace"][to[i]:to[i + 1]],
                           node_stats=z["tr_ns"][ns], node_dist=z["tr_nd"][nd].reshape(-1, bins),
                           bk_stats=z["tr_bk_ns"][ns], bk_dist=z["tr_bk_nd"][nd].reshape(-1, bins)))
    return dict(cfgs=cfgs, shift=shift, mv=mv, backup=backup)


def assert_dist_close(got, want, what):
    """1e-5 relative (the reference is fastmath) and the same set of non-zero bins: a bin moved by one is a support difference."""
    got, want = np.asarray(got), np.asarray(want)
    sg, sw = got != 0, want != 0
    if not np.array_equal(sg, sw):
        first = np.argwhere(sg != sw)[0]
        raise AssertionError("%s: support differs first at %s: got %r, reference %r" % (what, tuple(first), got[tuple(first)], want[tuple(first)]))
    bad = ~np.isclose(got, want, rtol=1e-5, atol=1e-7)
    if bad.any():
        first = np.argwhere(bad)[0]
        raise AssertionError("%s: value differs first at %s: got %r, reference %r" % (what, tuple(first), got[tuple(first)], want[tuple(first)]))


def assert_mean_variance_close(got, want, what):
    """The variance is m2 - mean^2: for a one-hot histogram both terms are ~mean^2 and cancel exactly, and the fastmath reference
    leaves a residue of a few ulp of mean^2 there."""
    (m, v), (wm, wv) = got, want
    assert np.isclose(m, wm, rtol=1e-5) and abs(v - wv) <= 1e-5 * abs(wv) + 1e-15 * wm * wm, (what, got, want)
