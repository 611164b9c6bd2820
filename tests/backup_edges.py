"""Designed trees for the engine's backup (k_backup -> backup_game) at its window and repeat edges, and the reference's backup of each
of them (tests/golden/gen_backup_edges.py runs it on the reference's own core.cpp; the tests run it on the C oracle and the scalar twins).

A case is a chain: trace level d is node d + 1, its next level sits in one child slot, one or two more slots hold siblings.  backup_game
folds the trace 32 levels per round from the leaf (lanes 0..31 = levels top .. top - 31, top = D - 1 - 32 w), so every D is chosen for
where its window edges fall, and repeated observations are placed on the lanes the duplicate test has to see.

Modes (the engine's flags in parentheses):
  lp     core.h:303-381 backup_trace_obs_LP(mixture=False, averaged=True) with the never-written node `end` array of the Python path
         (ValueSimLP.py:29; SURVEY N1)                                                  (lp_end_from_obs 0, lp_var_gamma2 1)
  lpcpp  agent.cpp:530-562: the children initialised from end_obs, the average without gamma^2 and handed over as float; the trace is then
         folded by core.cpp's backup_trace_obs with those float arguments               (lp_end_from_obs 1, lp_var_gamma2 0)
  single ValueSim.py:80-95: backup_trace_obs with v = float32(leaf score + e), var = e (slot 7 of the evaluator outputs)
  vanilla Vanilla.py:40-56: backup_trace_obs with the rollout score and rollout_variance = 1e3
A terminal leaf (kind 0) backs up its own score with variance 0 in every mode."""
import numpy as np

KEYS = ("child", "n2o", "score", "visit", "value", "variance", "end", "trace", "ev")
MODES = ("lp", "lpcpp", "single", "vanilla")
GAMMAS = (1.0, 0.999, 0.9, 0.5)
DEPTHS = (1, 2, 31, 32, 33, 63, 64, 65, 96, 97, 200, 511, 512)
ROLLOUT_VARIANCE = 1e3
F32 = np.float32
SUB = float(np.float32(1e-40))          # a float32 subnormal
EDGE_EVALS = (0.0, -37.25, 1e30, SUB, float("inf"), float("-inf"), float("nan"))
EDGE_VISITS = (0, 1, (1 << 24) - 1, 1 << 24, (1 << 24) + 1, 3_000_000, 17_000_001)


def build(seed, D, mode, gamma, kind=1, same=(), leaf=None, leaf_scores=None, leaf_visits=None, ev=None, visits=None, rollout=None,
          transpose=(), tags=()):
    """One designed case.  same: groups of trace levels that share one observation; leaf: 7 slot specs of the leaf's children (0 = no
    child, ("new", t) = an observation of its own per tag t, ("trace", d) = the observation of trace level d); leaf_scores / leaf_visits:
    per slot / per tag overrides; ev: (value, variance) per slot (8 x 2); visits: {trace level: visit} overrides; transpose: (d, t) = one
    more child of trace level d whose observation is trace level t's (the same observation under another node of the path)."""
    rng = np.random.default_rng(seed)
    M = D + 2 * D + 16
    child = np.zeros((M, 7), np.int32)
    n2o = np.zeros(M, np.int32)
    score = np.zeros(M, np.float32)
    n_obs = [1]
    next_node = [D + 1]

    def new_obs():
        n_obs[0] += 1
        return n_obs[0] - 1

    def new_node(o, s):
        i = next_node[0]
        next_node[0] += 1
        n2o[i], score[i] = o, s
        return i

    lvl_obs = [new_obs() for _ in range(D)]
    for grp in same:
        for d in grp[1:]:
            lvl_obs[d] = lvl_obs[grp[0]]
    s = float(rng.integers(0, 50))
    for d in range(D):
        n2o[d + 1], score[d + 1] = lvl_obs[d], s
        s += float(rng.choice([0, 1, 2, 6, 20, 60, 120, 600]))
    for d in range(D - 1):
        slots = rng.permutation(7)
        child[d + 1, slots[0]] = d + 2
        for a in slots[1:1 + int(rng.integers(1, 3))]:
            child[d + 1, a] = new_node(new_obs(), score[d + 1] + float(rng.choice([0, 1, 6, 20, 120])))
    for d, t in transpose:
        a = int(np.nonzero(child[d + 1] == 0)[0][0])
        child[d + 1, a] = new_node(lvl_obs[t], score[d + 1] + 3.0)
    leaf_node = D
    if kind == 1:
        if leaf is None:
            leaf = [("new", a) for a in range(7)]
        tag_obs = {}
        for a, spec in enumerate(leaf):
            if spec == 0:
                continue
            if spec[0] == "trace":
                o = lvl_obs[spec[1]]
            else:
                o = tag_obs.setdefault(spec[1], None) or new_obs()
                tag_obs[spec[1]] = o
            sc = leaf_scores[a] if leaf_scores is not None else score[leaf_node] + float(rng.choice([0, 1, 6, 20, 120, 600]))
            child[leaf_node, a] = new_node(o, sc)
    n = n_obs[0]
    visit = np.zeros(M, np.int32)
    visit[1:n] = rng.integers(1, 400, n - 1)
    value = np.zeros(M, np.float32)
    value[1:n] = rng.uniform(-50, 3000, n - 1).astype(F32)
    variance = np.zeros(M, np.float32)
    variance[1:n] = rng.uniform(0, 2e5, n - 1).astype(F32)
    end = np.zeros(M, np.uint8)
    end[1:n] = rng.random(n - 1) < 0.25
    if kind == 1:
        for a, spec in enumerate(leaf):        # unvisited children by default every other slot: those the LP init writes
            if spec != 0 and spec[0] == "new":
                o = n2o[child[leaf_node, a]]
                visit[o] = (leaf_visits or {}).get(spec[1], 0 if (a + seed) % 2 else int(rng.integers(1, 50)))
    for d, v in (visits or {}).items():
        visit[lvl_obs[d]] = v
    evs = np.zeros((8, 2), np.float32)
    evs[:, 0] = rng.uniform(-20, 2500, 8)
    evs[:, 1] = rng.uniform(0, 5e4, 8)
    if ev is not None:
        evs[:] = np.asarray(ev, np.float32)
    ro = float(F32(rollout if rollout is not None else rng.integers(0, 20000)))   # the engine holds the rollout score as float
    return dict(child=child, n2o=n2o, score=score, visit=visit, value=value, variance=variance, end=end,
                trace=np.arange(1, D + 1, dtype=np.int32), ev=evs, rollout=ro, kind=int(kind), mode=mode, gamma=float(gamma),
                tags=list(tags))


def design():
    """The designed cases, in a fixed order (the golden's c<i>_ prefixes)."""
    cases = []
    k = 0

    def add(D, mode, gamma, **kw):
        nonlocal k
        cases.append(build(1000 + k, D, mode, gamma, **kw))
        k += 1

    # every depth, every mode, both leaf kinds
    for i, D in enumerate(DEPTHS):
        for j, mode in enumerate(MODES):
            add(D, mode, GAMMAS[(i + j) % 4], tags=["depth"])
        add(D, MODES[i % 4], GAMMAS[i % 4], kind=0, tags=["depth", "terminal"])
    # repeated observations on the trace (levels are absolute; lanes count from the leaf: lane l of window w = level D-1-32w-l)
    reps = [
        (40, [(20, 21)], "adjacent"), (100, [(99, 68)], "lanes0_31"), (100, [(67, 36)], "lanes0_31"),
        (96, [(31, 32)], "edge"), (96, [(63, 64)], "edge"), (100, [(67, 68)], "edge"), (65, [(0, 1)], "edge"), (33, [(0, 1)], "edge"),
        (97, [(0, 96)], "first_last"), (32, [(0, 31)], "first_last"), (200, [(3, 40, 41, 90, 150, 199)], "three"),
        (70, [tuple(range(70))], "all_same"), (64, [tuple(range(0, 64, 2)), tuple(range(1, 64, 2))], "three"),
        (130, [(5, 37, 69, 101)], "three"), (512, [(0, 31, 32, 255, 256, 511)], "three"),
    ]
    for i, (D, same, tag) in enumerate(reps):
        add(D, MODES[i % 4], GAMMAS[i % 4], same=same, tags=["repeat", tag])
        if i % 3 == 0:
            add(D, MODES[(i + 1) % 4], GAMMAS[(i + 2) % 4], same=same, kind=0, tags=["repeat", tag, "terminal"])
    # a sibling on the path whose observation is another trace level's (a transposition)
    for i, (D, tp) in enumerate([(40, [(5, 20)]), (40, [(20, 5)]), (40, [(0, 39)]), (100, [(10, 50), (60, 30), (97, 0)]),
                                 (70, [(3, 3 + 33)]), (64, [(31, 0), (1, 63)])]):
        add(D, ("lp", "lpcpp")[i % 2], GAMMAS[i % 4], transpose=tp, tags=["transposition"])
        add(D, ("lp", "lpcpp")[(i + 1) % 2], GAMMAS[(i + 1) % 4], transpose=tp, kind=0, tags=["transposition", "terminal"])
    # a leaf child whose observation is also a trace level's
    for i, (D, lvls) in enumerate([(40, (10,)), (40, (39,)), (70, (0, 38, 69)), (33, (1,))]):
        leaf = [("trace", lvls[a]) if a < len(lvls) else ("new", a) for a in range(7)]
        add(D, ("lp", "lpcpp")[i % 2], GAMMAS[i % 4], leaf=leaf, visits={lvls[0]: 0} if i == 3 else None, tags=["leaf_on_trace"])
    # leaf children: 1..7 unique, duplicates (unequal / equal scores), zero ids, visit 0 and > 0
    for kk in range(1, 8):
        leaf = [("new", a) if a < kk else 0 for a in range(7)]
        for mode in ("lp", "lpcpp"):
            add(45, mode, GAMMAS[kk % 4], leaf=leaf, tags=["k%d" % kk])
    dup_layouts = [
        ([("new", 0), ("new", 1), ("new", 0), ("new", 2), ("new", 1), ("new", 0), ("new", 3)], [5, 9, 7, 1, 9, 7, 2], "dup_unequal"),
        ([("new", 0), ("new", 0), ("new", 0), ("new", 1), ("new", 1), 0, ("new", 2)], [4, 4, 4, 8, 8, 0, 3], "dup_equal"),
        ([0, ("new", 0), 0, ("new", 1), ("new", 0), 0, 0], [0, 2, 0, 3, 6, 0, 0], "zero_ids"),
        ([("new", 0)] * 7, [1, 2, 3, 4, 5, 6, 7], "dup_unequal"),
        ([("new", 0)] * 7, [3] * 7, "dup_equal"),
    ]
    for i, (leaf, sc, tag) in enumerate(dup_layouts):
        for mode in ("lp", "lpcpp"):
            add(50, mode, GAMMAS[i % 4], leaf=leaf, leaf_scores=[1000.0 + x for x in sc], leaf_visits={0: 0, 1: 5, 2: 0, 3: 1},
                tags=["leaf_dups", tag])
    # evaluator outputs at the float edges, per mode; statistics at the visit edges
    for i, e in enumerate(EDGE_EVALS):
        ev = np.zeros((8, 2), np.float32)
        ev[:, 0] = e
        ev[:, 1] = abs(e) if e == e else e
        for mode in ("lp", "lpcpp", "single"):
            add(37, mode, GAMMAS[i % 4], ev=ev, leaf_visits={a: 0 for a in range(7)}, tags=["eval_edge"])
    for i in range(4):
        D = (33, 64, 97, 200)[i]
        visits = {d: EDGE_VISITS[(d + i) % len(EDGE_VISITS)] for d in range(D)}
        for mode in MODES:
            add(D, mode, GAMMAS[(i + 1) % 4], visits=visits, leaf_visits={a: EDGE_VISITS[a] for a in range(7)}, tags=["visit_edge"])
    add(60, "vanilla", 0.9, rollout=1e30, tags=["eval_edge"])
    add(60, "vanilla", 0.5, rollout=0.0, tags=["eval_edge"])
    return cases


def unique_children(index, child, score, n2o):
    """core.h:111-144 in Python: the first occurrence of each observation in slot order, represented by the child with the strictly
    largest score (earliest on ties); returns (nodes, observations, first slots)."""
    cn, co, slot = [], [], []
    for a in range(7):
        c = int(child[index, a])
        if c == 0:
            continue
        o = int(n2o[c])
        if o in co:
            j = co.index(o)
            if score[c] > score[cn[j]]:
                cn[j] = c
        else:
            cn.append(c)
            co.append(o)
            slot.append(a)
    return cn, co, slot


def lp_cpp_init(c, gamma, visit, value, variance):
    """agent.cpp:530-562 up to the backup call, on the per-observation arrays (mutated as agent.cpp mutates them): returns the float
    (_val_tmp, _var_tmp) that agent.cpp:562 hands to backup_obs_single."""
    cn, co, slot = unique_children(int(c["trace"][-1]), c["child"], c["score"], c["n2o"])
    val_tmp = var_tmp = 0.0                                  # agent.cpp:531-532 double
    for i, (n, o) in enumerate(zip(cn, co)):
        if visit[o] == 0:                                    # agent.cpp:536-545
            visit[o] += 1
            if c["end"][o]:                                  # end_obs[__o]: the observation's own flag
                value[o] = 0
                variance[o] = 0
            else:
                value[o] = c["ev"][slot[i], 0]
                variance[o] = c["ev"][slot[i], 1]
        val_tmp += float(c["score"][n]) + gamma * float(value[o])   # agent.cpp:547: float score + double gamma * float value
        var_tmp += float(variance[o])                        # agent.cpp:548
    val_tmp /= len(cn)                                       # agent.cpp:557-558
    var_tmp /= len(cn)
    return float(F32(val_tmp)), float(F32(var_tmp))          # agent.cpp:562 backup_obs_single(trace, float _val, float _var)


def run(c, core):
    """The reference's backup of case c on `core` (the reference's own core module, the C oracle or the device's scalar twins: the same
    call signatures).  Returns the per-observation (visit, value, variance) after it."""
    visit, value, variance = c["visit"].copy(), c["value"].copy(), c["variance"].copy()
    tr, g, leaf = c["trace"], c["gamma"], int(c["trace"][-1])
    leaf_score = float(c["score"][leaf])
    if c["kind"] == 0:
        if c["mode"] == "lp":
            core.backup_trace_obs_LP(tr, visit, value, variance, c["n2o"], c["score"], np.zeros(len(visit), bool), [], [],
                                     np.zeros(0, F32), np.zeros(0, F32), g, False, True)
        else:
            core.backup_trace_obs(tr, visit, value, variance, c["n2o"], c["score"], leaf_score, 0.0, g)
    elif c["mode"] == "lp":
        cn, co, slot = unique_children(leaf, c["child"], c["score"], c["n2o"])
        v = np.ascontiguousarray(c["ev"][slot, 0], F32)
        var = np.ascontiguousarray(c["ev"][slot, 1], F32)
        core.backup_trace_obs_LP(tr, visit, value, variance, c["n2o"], c["score"], np.zeros(len(visit), bool), cn, co, v, var, g,
                                 False, True)
    elif c["mode"] == "lpcpp":
        v, var = lp_cpp_init(c, g, visit, value, variance)
        core.backup_trace_obs(tr, visit, value, variance, c["n2o"], c["score"], v, var, g)
    elif c["mode"] == "single":
        v = F32(c["score"][leaf]) + F32(c["ev"][7, 0])      # ValueSim.py:86 int + np.float32 -> float32
        core.backup_trace_obs(tr, visit, value, variance, c["n2o"], c["score"], float(v), float(c["ev"][7, 1]), g)
    else:
        core.backup_trace_obs(tr, visit, value, variance, c["n2o"], c["score"], float(c["rollout"]), ROLLOUT_VARIANCE, g)
    return visit, value, variance


def digest(c):
    """A fingerprint of case c's inputs (arrays, mode, kind, gamma, rollout, tags): the golden stores it in place of the inputs, which
    design() regenerates."""
    import hashlib
    h = hashlib.sha256()
    for k in KEYS:
        a = np.ascontiguousarray(c[k])
        h.update(("%s %s %s;" % (k, a.dtype.str, a.shape)).encode())
        h.update(a.tobytes())
    h.update(("%s %d %r %s %s" % (c["mode"], c["kind"], c["gamma"], F32(c["rollout"]).tobytes().hex(), ",".join(c["tags"]))).encode())
    return np.frombuffer(h.digest()[:16], np.uint8)


def save(path, cases, outs):
    """The reference's outputs of every case: the observations whose (visit, value, variance) the backup changed, and those values, all
    cases concatenated (out_off[i] .. out_off[i+1]); plus each case's input digest.  The inputs are not stored: design() makes them.
    The zip is written with fixed timestamps, so that a regeneration is byte-identical."""
    import io
    import zipfile
    idx, vis, val, var, off = [], [], [], [], [0]
    for c, (v, x, y) in zip(cases, outs):
        changed = (v != c["visit"]) | (x.view(np.int32) != c["value"].view(np.int32)) | (y.view(np.int32) != c["variance"].view(np.int32))
        k = np.nonzero(changed)[0].astype(np.int32)
        idx.append(k); vis.append(v[k]); val.append(x[k]); var.append(y[k])
        off.append(off[-1] + len(k))
    arrays = {"n_cases": np.int32(len(cases)), "digest": np.stack([digest(c) for c in cases]), "out_off": np.asarray(off, np.int32),
              "out_idx": np.concatenate(idx), "out_visit": np.concatenate(vis), "out_value": np.concatenate(val),
              "out_variance": np.concatenate(var)}
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as z:
        for k in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(arrays[k]), allow_pickle=False)
            zi = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            zi.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(zi, buf.getvalue(), compresslevel=9)


def load(path):
    """design()'s cases, each with c["out"] = the reference's (visit, value, variance) after the backup (the inputs with the golden's
    changed entries written in) and c["digest_ok"] = its inputs are those the golden was made from."""
    z = np.load(path)
    cases = design()
    if len(cases) != int(z["n_cases"]):
        raise ValueError("%s holds %d cases, design() makes %d: regenerate it (tests/golden/gen_backup_edges.py)" % (path, int(z["n_cases"]), len(cases)))
    off = z["out_off"]
    for i, c in enumerate(cases):
        k = z["out_idx"][off[i]:off[i + 1]]
        out = [c["visit"].copy(), c["value"].copy(), c["variance"].copy()]
        for a, name in zip(out, ("out_visit", "out_value", "out_variance")):
            a[k] = z[name][off[i]:off[i + 1]]
        c["out"] = tuple(out)
        c["digest_ok"] = bool(np.array_equal(digest(c), z["digest"][i]))
    return cases


def same_bits(a, b):
    """Equal bit for bit, any NaN equal to any NaN (the device's NaN is canonical, x86 keeps the operand's)."""
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype.kind == "f":
        both_nan = np.isnan(a) & np.isnan(b)
        return bool(np.all(both_nan | (a.view(np.int32) == b.view(np.int32))))
    return bool(np.array_equal(a, b))
