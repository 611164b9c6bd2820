"""Designed trees for the engine's walk (k_select_expand -> select_trace, with and without the path cache) and its action choice
(k_root_stats), and the reference's own search on each of them (tests/golden/gen_select_edges.py runs it on the reference's compiled
core.cpp and agents/agent.py; the tests run the C oracle and the engine).

Every node without children is a terminal node, so a simulation is a walk (select_trace_obs, core.h:167-224) followed by the terminal
backup of the leaf's own score: backup_trace_obs_LP with an empty child list (mode lp) or backup_trace_obs(trace, score[leaf], 0) (mode
single).  A case runs `sims` such simulations from `root` with check_low's draws (core.h:76) on the xorshift32 stream seeded with `seed`,
then compute_stats / get_action (agent.py:153-185) on the root.  The statistics hold what whole searches never produce: exact q ties,
NaN and infinite q, negative and -0.0 variances, visit sums at the z(n) table edges and past 2^31, duplicate observations with NaN
scores, unvisited children under `low`, chains around the path cache's 8-level rounds and the trace's length limit, transpositions."""
import numpy as np

KEYS = ("child", "n2o", "score", "visit", "value", "variance", "end")
F32 = np.float32
NAN, INF = float("nan"), float("inf")
TRACE_MAX = 64          # the engines of the tests are made with this trace_max
LOWS = (0, 1, 5)
GAMMAS = (0.999, 0.5)


class Tree:
    """A tree in the reference's layout: node 0 and observation 0 are the reference's empty entries."""

    def __init__(self):
        self.child, self.n2o, self.score = [[0] * 7], [0], [0.0]
        self.visit, self.value, self.variance = [0], [0.0], [0.0]

    def obs(self, visit=1, value=0.0, variance=0.0):
        self.visit.append(int(visit)); self.value.append(float(value)); self.variance.append(float(variance))
        return len(self.visit) - 1

    def node(self, o, score=0.0):
        self.child.append([0] * 7); self.n2o.append(int(o)); self.score.append(float(score))
        return len(self.n2o) - 1

    def leaf(self, visit=1, value=0.0, variance=0.0, score=0.0):
        return self.node(self.obs(visit, value, variance), score)

    def link(self, parent, kids):
        """kids: up to 7 node ids in slot order (0 = empty slot)."""
        for a, c in enumerate(kids):
            self.child[parent][a] = int(c)

    def case(self, root, sims, low=1, gamma=0.999, mode="lp", seed=1, tags=()):
        M = len(self.n2o)
        visit = np.asarray(self.visit + [0] * (M - len(self.visit)), np.int64).astype(np.int32)
        f = lambda x: np.asarray(x + [0.0] * (M - len(x)), F32)
        return dict(child=np.asarray(self.child, np.int32), n2o=np.asarray(self.n2o, np.int32), score=f(self.score), visit=visit,
                    value=f(self.value), variance=f(self.variance), end=np.zeros(M, np.uint8), root=int(root), sims=int(sims),
                    low=int(low), gamma=float(gamma), mode=mode, seed=int(seed) & 0xffffffff, tags=list(tags))


def star(stats, scores=None, root_visit=None, dup=None):
    """A root whose children are leaves: stats = one (visit, value, variance) per slot (None = empty slot); scores per slot; dup = {slot:
    earlier slot} makes a slot's child another node of an earlier slot's observation."""
    t = Tree()
    kids, obs = [], {}
    for a, s in enumerate(stats):
        if s is None and not (dup and a in dup):
            kids.append(0)
            continue
        sc = scores[a] if scores is not None else 0.0
        if dup and a in dup:
            kids.append(t.node(obs[dup[a]], sc))
        else:
            obs[a] = t.obs(*s)
            kids.append(t.node(obs[a], sc))
    total = sum(s[0] for s in stats if s is not None)
    r = t.node(t.obs(root_visit if root_visit is not None else min(total + 1, 1 << 30), 0.0, 1.0), 0.0)
    t.link(r, kids)
    return t, r


def chain(D, rng, low_level=None, repick_level=None, same=(), transpose=()):
    """A path of D levels (root = level 0, the terminal leaf = level D - 1): level d's child in a random slot leads on (a high value), one or
    two sibling leaves are far worse.  low_level: two unvisited leaves there (check_low draws); repick_level: two equal leaves there that
    the walk alternates between; same: groups of levels whose nodes share one observation; transpose: (d, t) = a sibling at level d whose
    observation is level t's."""
    t = Tree()
    lvl_obs = [t.obs(10 + d, 1.0e4, 100.0) for d in range(D)]
    for grp in same:
        for d in grp[1:]:
            lvl_obs[d] = lvl_obs[grp[0]]
    nodes = [t.node(lvl_obs[d], 0.0) for d in range(D)]
    for d in range(D - 1):
        slots = rng.permutation(7)
        kids = [0] * 7
        kids[slots[0]] = nodes[d + 1]
        for a in slots[1:1 + int(rng.integers(1, 3))]:
            kids[a] = t.leaf(10, -1.0e6, 0.0, 0.0)
        if d == low_level:
            kids[slots[3]] = t.leaf(0, 0.0, 0.0, 1.0)
            kids[slots[4]] = t.leaf(2, 0.0, 0.0, 2.0)
        if d == repick_level:
            kids[slots[5]] = t.leaf(3, 2.0e4, 50.0, 0.0)
            kids[slots[6]] = t.leaf(4, 2.0e4, 50.0, 0.0)
        for dd, tt in transpose:
            if dd == d:
                kids[slots[6]] = t.node(lvl_obs[tt], 0.0)
        t.link(nodes[d], kids)
    return t, nodes[0]


def design():
    """The designed cases, in a fixed order."""
    rng = np.random.default_rng(20261017)
    cases = []

    def add(tr, sims, tags, low=1, gamma=GAMMAS[0], mode="lp"):
        t, r = tr
        cases.append(t.case(r, sims, low, gamma, mode, seed=0x9E3779B9 * (len(cases) + 1), tags=tags))

    # q ties
    add(star([(5, 10.0, 4.0)] * 7), 6, ["tie_all7"])
    add(star([(5, 10.0, 4.0), (5, 1.0, 4.0), (5, 1.0, 4.0), (5, 1.0, 4.0), (5, 1.0, 4.0), (5, 1.0, 4.0), (5, 10.0, 4.0)]), 4, ["tie_lanes_0_6"])
    add(star([(5, 1.0, 4.0), (5, 1.0, 4.0), (5, 1.0, 4.0), (5, 10.0, 4.0), (5, 10.0, 4.0), (5, 1.0, 4.0), None]), 4, ["tie_lanes_3_4"])
    add(star([(5, -0.0, 0.0), (5, 0.0, 0.0), (5, -0.0, 0.0), None, (5, 0.0, 0.0), None, None]), 4, ["signed_zero"], gamma=GAMMAS[1])
    # NaN q: first entry, a later entry, every entry
    add(star([(5, NAN, 4.0), (5, 10.0, 4.0), (5, 20.0, 4.0), None, None, None, None]), 4, ["nan_first"])
    add(star([(5, 10.0, 4.0), (5, 20.0, 4.0), (5, NAN, 4.0), (5, 30.0, 4.0), None, None, None]), 4, ["nan_later", "root_nan"])
    add(star([(5, NAN, 4.0), (5, NAN, 4.0), (5, NAN, 1.0), None, None, None, (5, NAN, 0.0)]), 3, ["nan_all", "root_nan"])
    add(star([(5, 30.0, 4.0), (5, 20.0, NAN), (5, 10.0, 4.0), None, None, None, None]), 3, ["nan_variance", "root_nan"])
    # infinite q
    add(star([(5, 1.0, 4.0), (5, INF, 4.0), (5, 2.0, 4.0), (5, INF, 4.0), (5, 3.0, 4.0), (5, INF, 1.0), None]), 3, ["inf_lanes", "root_inf"])
    add(star([(5, -INF, 4.0)] * 5 + [None, (5, -INF, 0.0)]), 3, ["neg_inf_all", "root_inf"])
    add(star([(5, 1.0, INF), (5, 1.0, 4.0), (5, -INF, INF), None, None, None, None]), 3, ["inf_variance"])
    # variance
    add(star([(5, 10.0, -4.0), (5, 9.0, 4.0), (5, 10.0, 4.0), (5, 8.0, -1e-30), None, None, None]), 3, ["neg_variance"])
    add(star([(5, 10.0, -0.0), (5, 10.0, 0.0), (5, 10.0, -0.0), None, None, None, None]), 3, ["negzero_variance"])
    # visit sums: 0 and 1 (z(n) is NaN), the shared-memory and global table edges, (float)N rounding, wrap past 2^31
    add(star([(0, 5.0, 4.0), (0, 7.0, 4.0), (0, 6.0, 1.0), None, None, None, None], root_visit=0), 4, ["visits_0_1"], low=0)
    add(star([(1, 5.0, 4.0), (0, 7.0, 4.0), None, None, None, None, None], root_visit=1), 3, ["visits_0_1"], low=0)
    add(star([(1000, 5.0, 40.0), (1000, 5.0, 30.0), (45, 5.2, 50.0), None, None, None, None]), 6, ["visits_2047_2048"])
    add(star([(600, 5.0, 40.0), (600, 5.0, 30.0), (600, 5.1, 50.0), (247, 5.2, 9.0), None, None, None]), 3, ["visits_2047_2048"], gamma=GAMMAS[1])
    add(star([(30000, 5.0, 40.0), (30000, 5.0, 30.0), (5533, 5.2, 50.0), None, None, None, None]), 6, ["visits_65535_65536"])
    add(star([(65534, 5.0, 40.0), None, None, None, None, None, None]), 4, ["visits_65535_65536"])
    big = (1 << 24) + 1
    add(star([(big, 5.0, 3.0e7), (big - 2, 5.0, 3.0e7), (1 << 24, 5.0, 3.0e7), (big + 2, 5.0, 3.0e7), None, None, None]), 4, ["visits_2p24"])
    add(star([(3, 5.0, 4.0), ((1 << 31) - 10, 9.0, 4.0), (1 << 30, 8.0, 4.0), None, None, None, None], root_visit=7), 4, ["visits_wrap"])
    add(star([(3, 5.0, 4.0), ((1 << 31) - 2, 9.0, 4.0), (1, 8.0, 4.0), (0, 1.0, 1.0), None, None, None], root_visit=7), 4, ["visits_wrap"],
        low=0)
    # duplicate observations in a child list: equal, unequal and NaN scores (the representative)
    add(star([(5, 1.0, 4.0), (5, 2.0, 4.0), None, None, (5, 3.0, 4.0), None, None], scores=[5, 0, 9, 9, 0, 3, 7], dup={2: 0, 3: 0, 5: 4, 6: 1}),
        4, ["dup_unequal", "dup_equal"])
    add(star([(5, 1.0, 4.0), (5, 2.0, 4.0), None, None, None, None, None], scores=[NAN, 0, 4, 2, 2, 2, 2], dup={2: 0, 3: 1, 4: 1, 5: 1, 6: 1}),
        4, ["dup_nan_score", "dup_equal"])
    add(star([(5, 1.0, 4.0), (5, 2.0, 4.0), None, None, None, None, None], scores=[3, 0, NAN, 0, 0, 0, 0], dup={2: 0, 3: 1}), 4, ["dup_nan_score"])
    # unvisited children under low: check_low draws (several such games share a warp in the tests)
    for i, low in enumerate((1, 5, 5, 1)):
        add(star([(0, 5.0, 4.0), (i, 7.0, 4.0), (0, 6.0, 1.0), (9, 9.0, 1.0), (0, 1.0, 1.0), None, (2, 3.0, 3.0)]), 8, ["low_draw"], low=low)
    # chains around the path cache's 8-level rounds (the terminal leaf at a round's last or first lane), trace_max and trace_max + 1
    for D in (7, 8, 9, 15, 16, 17, 23, 24, 25):
        add(chain(D, rng), 5, ["chain"], gamma=GAMMAS[D % 2])
    add(chain(TRACE_MAX, rng), 3, ["chain", "trace_max"])
    add(chain(TRACE_MAX + 1, rng), 1, ["chain", "trace_full"])
    # path-cache events
    add(chain(20, rng, repick_level=12), 8, ["chain", "repick"])
    add(chain(11, rng, repick_level=8), 8, ["chain", "repick"], gamma=GAMMAS[1])
    add(chain(18, rng, low_level=10), 8, ["chain", "low_bail"], low=5)
    add(chain(12, rng, low_level=7), 6, ["chain", "low_draw_repick"], low=1)
    add(chain(20, rng, same=[(2, 9)]), 5, ["chain", "twice_on_trace"])
    add(chain(20, rng, transpose=[(12, 3)]), 5, ["chain", "transposition"])
    add(chain(17, rng, transpose=[(4, 15)], same=[(1, 16)]), 5, ["chain", "transposition", "twice_on_trace"])
    # the single backup
    add(star([(5, 10.0, 4.0), (5, NAN, 4.0), (5, 1.0, -4.0), None, None, None, None]), 4, ["single", "root_nan"], mode="single")
    add(chain(16, rng), 4, ["chain", "single"], mode="single")
    add(star([(0, 5.0, 4.0), (2, 7.0, 4.0), (0, 6.0, 1.0), None, None, None, None]), 6, ["single", "low_draw"], low=5, mode="single")
    # root statistics: near ties for the action choice
    add(star([(1 << 20, 100.0, 4.0), (1 << 20, float(np.nextafter(F32(100.0), F32(200.0))), 4.0), (1 << 20, 100.0, 4.0), None, None, None,
              None]), 2, ["root_near_tie"])
    # the shared-memory z table's edge decides: q(slot 0) = 3.25387 lies between z(2047) and z(2048), q(slot 1) = z(n) at n = 2048
    add(star([(1024, 3.25387, 0.0), (1024, 0.0, 1024.0), None, None, None, None, None]), 2, ["z_2048_decides"])
    return cases


def zero_obs_case():
    """The operator-level case of the twin: a child whose observation id is 0 (never allocated in the engine's arena) under `low`: when
    check_low draws observation 0, core.h:202-205 falls through to policy_clt."""
    t = Tree()
    kids = [t.leaf(3, 9.0, 4.0), t.leaf(0, 5.0, 0.0), t.node(0, 0.0), 0, 0, 0, 0]   # policy_clt picks slot 0 (slots 1 and 2: NaN q)
    r = t.node(t.obs(4, 0.0, 1.0), 0.0)
    t.link(r, kids)
    return [t.case(r, 1, low=1, seed=s, tags=["obs0"]) for s in (1, 2, 3, 4, 5, 6, 7, 8)]


def xorshift32(s):
    s ^= (s << 13) & 0xffffffff
    s ^= s >> 17
    s ^= (s << 5) & 0xffffffff
    return s


def run(c, core, rng_seed, rng_next, compute_stats=None):
    """The reference's search of case c on `core` (the reference's own core module or the C oracle: the same call signatures).
    rng_seed(s) seeds check_low's stream, rng_next() returns its next value (the state after the run).  Returns (traces, per simulation the
    statistics after its backup, final (visit, value, variance), next stream value)."""
    visit, value, variance = c["visit"].copy(), c["value"].copy(), c["variance"].copy()
    rng_seed(c["seed"])
    traces, states = [], []
    for s in range(c["sims"]):
        tr = np.asarray(core.select_trace_obs(c["root"], c["child"], visit, value, variance, c["score"], c["n2o"], c["low"]), np.int32)
        traces.append(tr)
        if len(tr) > TRACE_MAX:              # the engine stops this walk (ST_TRACE_FULL) and backs nothing up
            break
        leaf = int(tr[-1])
        if c["mode"] == "lp":
            core.backup_trace_obs_LP(tr, visit, value, variance, c["n2o"], c["score"], np.zeros(len(visit), bool), [], [],
                                     np.zeros(0, F32), np.zeros(0, F32), c["gamma"], False, True)
        else:
            core.backup_trace_obs(tr, visit, value, variance, c["n2o"], c["score"], float(c["score"][leaf]), 0.0, c["gamma"])
        states.append((visit.copy(), value.copy(), variance.copy()))
    return traces, states, rng_next()


def pc_model(c, oracle):
    """The path-cache model (oracle.pc_replay) over case c's golden walks (an lp case): per simulation the levels the engine's walk serves
    from the cache, the cache's valid length after the backup and {re-picks on served levels, check_low stops at a cached level, walks that
    ended on a cached leaf}, and the number of stale reads the model found."""
    states = [(c["visit"], c["value"], c["variance"])] + list(c["states"])
    return oracle.pc_replay(c["child"], c["score"], c["n2o"], c["low"], c["traces"], states)


def root_stats(c, visit, value, variance):
    """compute_stats (agent.py:153-179) restated in numpy float32, and np.argmax of its value row (agent.py:185)."""
    r = c["root"]
    kids = c["child"][r]
    o = c["n2o"][kids]
    st = np.zeros((3, 7), F32)
    st[0] = visit[o]
    st[1] = value[o] + (c["score"][kids] - c["score"][r])
    st[2] = variance[o]
    return st, int(np.argmax(st[1]))


def digest(c):
    """A fingerprint of case c's inputs: the golden stores it in place of the inputs, which design() regenerates."""
    import hashlib
    h = hashlib.sha256()
    for k in KEYS:
        a = np.ascontiguousarray(c[k])
        h.update(("%s %s %s;" % (k, a.dtype.str, a.shape)).encode())
        h.update(a.tobytes())
    h.update(("%d %d %d %r %s %d %s" % (c["root"], c["sims"], c["low"], c["gamma"], c["mode"], c["seed"], ",".join(c["tags"]))).encode())
    return np.frombuffer(h.digest()[:16], np.uint8)


def save(path, cases, outs):
    """outs[i] = (traces, states, rng_after, stats[3,7], action).  Stored: every simulation's trace, the entries each backup changed, the
    final root statistics and action, the stream's next value and each case's input digest.  Fixed zip timestamps: a regeneration is
    byte-identical."""
    import io
    import zipfile
    tr, tr_off, sim_off = [], [0], [0]
    idx, vis, val, var, ch_off = [], [], [], [], [0]
    for c, (traces, states, _, _, _) in zip(cases, outs):
        prev = (c["visit"], c["value"], c["variance"])
        for t in traces:
            tr.append(t); tr_off.append(tr_off[-1] + len(t))
        for v, x, y in states:
            changed = (v != prev[0]) | (x.view(np.int32) != prev[1].view(np.int32)) | (y.view(np.int32) != prev[2].view(np.int32))
            k = np.nonzero(changed)[0].astype(np.int32)
            idx.append(k); vis.append(v[k]); val.append(x[k]); var.append(y[k])
            ch_off.append(ch_off[-1] + len(k))
            prev = (v, x, y)
        sim_off.append(sim_off[-1] + len(traces))
    arrays = {"n_cases": np.int32(len(cases)), "digest": np.stack([digest(c) for c in cases]), "sim_off": np.asarray(sim_off, np.int32),
              "trace_off": np.asarray(tr_off, np.int32), "trace": np.concatenate(tr).astype(np.int32), "change_off": np.asarray(ch_off, np.int32),
              "change_idx": np.concatenate(idx), "change_visit": np.concatenate(vis), "change_value": np.concatenate(val),
              "change_variance": np.concatenate(var), "rng_next": np.asarray([o[2] for o in outs], np.uint32),
              "stats": np.stack([o[3] for o in outs]).astype(F32), "action": np.asarray([o[4] for o in outs], np.int32)}
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as z:
        for k in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(arrays[k]), allow_pickle=False)
            zi = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            zi.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(zi, buf.getvalue(), compresslevel=9)


def load(path):
    """design()'s cases, each with the reference's results: c["traces"] (one per simulation), c["states"] (visit, value, variance after each
    backup), c["rng_next"], c["stats"], c["action"], and c["digest_ok"] = its inputs are those the golden was made from."""
    z = np.load(path)
    cases = design()
    if len(cases) != int(z["n_cases"]):
        raise ValueError("%s holds %d cases, design() makes %d: regenerate it (tests/golden/gen_select_edges.py)" % (path, int(z["n_cases"]), len(cases)))
    so, to, co = z["sim_off"], z["trace_off"], z["change_off"]
    first = 0                                # the change blocks of case i start here: one per backup
    for i, c in enumerate(cases):
        c["traces"] = [z["trace"][to[s]:to[s + 1]] for s in range(so[i], so[i + 1])]
        cur = [c["visit"].copy(), c["value"].copy(), c["variance"].copy()]
        c["states"] = []
        n_backups = len(c["traces"]) - (1 if len(c["traces"][-1]) > TRACE_MAX else 0)
        for s in range(first, first + n_backups):
            k = z["change_idx"][co[s]:co[s + 1]]
            for a, name in zip(cur, ("change_visit", "change_value", "change_variance")):
                a[k] = z[name][co[s]:co[s + 1]]
            c["states"].append(tuple(a.copy() for a in cur))
        first += n_backups
        c["rng_next"] = int(z["rng_next"][i])
        c["stats"], c["action"] = z["stats"][i], int(z["action"][i])
        c["digest_ok"] = bool(np.array_equal(digest(c), z["digest"][i]))
    return cases


def same_bits(a, b):
    """Equal bit for bit, any NaN equal to any NaN."""
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype.kind == "f":
        both_nan = np.isnan(a) & np.isnan(b)
        return bool(np.all(both_nan | (a.view(np.int32) == b.view(np.int32))))
    return bool(np.array_equal(a, b))
