"""Pin the C oracle's walk (mo_select_trace_obs with its xorshift32 stream) and backups to the reference's own core.cpp and agent.py on the
designed trees of tests/select_edges.py (tests/golden/select_edges_golden.npz), check that the golden holds the shapes it was designed
for, and run the path-cache model (mcts_oracle.c pc_*, mo_pc_replay) over each LP case's walks: it must find no stale read, and each
path-cache case must produce the event it was designed for (tests/test_gpu_select_edges.py holds the engine to the model's counts)."""
import os

import numpy as np
import pytest

import select_edges as SE

GOLD = os.path.join(os.path.dirname(__file__), "golden", "select_edges_golden.npz")


@pytest.fixture(scope="module")
def cases():
    return SE.load(GOLD)


class OracleCore:
    """The C oracle with the call signatures of the reference's core module; check_low draws from one xorshift32 stream."""

    def __init__(self, oracle):
        self.O, self.state = oracle, np.zeros(1, np.uint32)

    def seed(self, s):
        self.state[0] = s

    def next(self):
        return SE.xorshift32(int(self.state[0]))

    def select_trace_obs(self, index, child, visit, value, variance, score, n2o, low):
        return self.O.select_trace_obs(index, child, visit, value, variance, score, n2o, low, max_trace=SE.TRACE_MAX + 1,
                                       rng_state=self.state)

    def backup_trace_obs(self, *a):
        self.O.backup_trace_obs(*a)

    def backup_trace_obs_LP(self, *a):
        self.O.backup_trace_obs_LP(*a)


def test_golden_is_the_designed_cases(cases):
    bad = [i for i, c in enumerate(cases) if not c["digest_ok"]]
    assert not bad, "design() no longer makes the inputs the golden was generated from (cases %s): regenerate it" % bad


def test_oracle_matches_reference(oracle, cases):
    core = OracleCore(oracle)
    for i, c in enumerate(cases):
        traces, states, rng_next = SE.run(c, core, core.seed, core.next)
        assert len(traces) == len(c["traces"]), (i, c["tags"])
        for s, (t, w) in enumerate(zip(traces, c["traces"])):
            assert np.array_equal(t, w), (i, c["tags"], s, t, w)
        for s, (g, w) in enumerate(zip(states, c["states"])):
            for name, a, b in zip(("visit", "value", "variance"), g, w):
                assert SE.same_bits(a, b), (i, c["tags"], s, name)
        assert rng_next == c["rng_next"], (i, c["tags"])
        last = states[-1] if states else (c["visit"], c["value"], c["variance"])
        stats, action = SE.root_stats(c, *last)
        assert SE.same_bits(stats, c["stats"]) and action == c["action"], (i, c["tags"], stats, c["stats"], action, c["action"])


def _root_entries(c, visit, value, variance):
    """The root's child list as select_trace_obs sees it: (visit, value + score - root score, variance) per first occurrence."""
    r = c["root"]
    seen, out = [], []
    for a in range(7):
        k = int(c["child"][r, a])
        if k == 0:
            continue
        o = int(c["n2o"][k])
        if o in seen:
            continue
        seen.append(o)
        out.append((int(visit[o]), float(value[o]), float(variance[o])))
    return out


def test_designed_shapes(cases):
    found, sums, lens, lows = set(), set(), set(), set()
    for c in cases:
        lows.add(c["low"])
        befores = [(c["visit"], c["value"], c["variance"])] + list(c["states"])
        for t in c["traces"]:
            lens.add(len(t))
        for st in befores[:len(c["traces"])]:
            e = _root_entries(c, *st)
            n = np.int64(sum(x[0] for x in e))
            sums.add(int(n))
            vals = np.asarray([x[1] for x in e], np.float32)
            var = np.asarray([x[2] for x in e], np.float32)
            if n > (1 << 31) - 1:
                found.add("visits_wrap")
            if any(x[0] == (1 << 24) + 1 for x in e):
                found.add("visits_2p24")
            if np.isnan(vals[0]):
                found.add("nan_first")
            if np.isnan(vals[1:]).any() and not np.isnan(vals[0]):
                found.add("nan_later")
            if np.isnan(vals).all():
                found.add("nan_all")
            if np.sum(vals == np.inf) >= 2:
                found.add("inf_lanes")
            if np.all(vals == -np.inf):
                found.add("neg_inf_all")
            if np.any(var < 0):
                found.add("neg_variance")
            if np.any((var == 0) & np.signbit(var)):
                found.add("negzero_variance")
            if len(vals) == 7 and len(set(vals.tolist())) == 1 and len(set(var.tolist())) == 1:
                found.add("tie_all7")
            if any(x[0] < c["low"] for x in e):
                found.add("low_draw")
        r = c["root"]
        kids = c["child"][r][c["child"][r] != 0]
        obs = c["n2o"][kids]
        for o in set(obs.tolist()):
            sc = c["score"][kids[obs == o]]
            if len(sc) > 1:
                found.add("dup_nan_score" if np.isnan(sc).any() else ("dup_equal" if np.sum(sc == sc.max()) > 1 else "dup_unequal"))
        v = c["stats"][1]
        if np.isnan(v).any() and int(np.argmax(np.where(np.isnan(v), -np.inf, v))) != c["action"]:
            found.add("root_nan_decides")
        if np.isinf(v).any():
            found.add("root_inf")
    assert {0, 1, 2047, 2048, 65535, 65536} <= sums, sorted(sums)[:40]
    assert {7, 8, 9, 15, 16, 17, 23, 24, 25, SE.TRACE_MAX, SE.TRACE_MAX + 1} <= lens, sorted(lens)
    assert set(SE.LOWS) == lows
    want = {"visits_wrap", "visits_2p24", "nan_first", "nan_later", "nan_all", "inf_lanes", "neg_inf_all", "neg_variance",
            "negzero_variance", "tie_all7", "low_draw", "dup_nan_score", "dup_equal", "dup_unequal", "root_nan_decides", "root_inf"}
    assert want <= found, want - found
    tags = {t for c in cases for t in c["tags"]}
    assert {"repick", "low_bail", "transposition", "twice_on_trace", "trace_full", "single", "root_near_tie"} <= tags


def test_path_cache_model_on_the_designed_walks(oracle, cases):
    """Every cached level the model serves equals the arena (no stale read), and the designed path-cache events happen: chains are served
    from the cache up to their terminal leaf, the repick cases re-pick on a served level, the low case stops at a cached level because of
    check_low, and an observation twice on the trace or under another node of the path truncates the cache."""
    for i, c in enumerate(cases):
        if c["mode"] != "lp" or "trace_full" in c["tags"]:
            continue
        served, pcl, ev, err = SE.pc_model(c, oracle)
        tags, D = set(c["tags"]), [len(t) for t in c["traces"]]
        assert err == 0 and served[0] == 0, (i, c["tags"], err, served)
        assert np.all(served <= np.asarray(D)) and np.all(pcl <= np.asarray(D)), (i, c["tags"])
        if "chain" in tags and not tags & {"twice_on_trace", "transposition"}:
            assert np.all(served[1:] > 0), (i, c["tags"], served)
            assert ev[:, 2].any() or "low_bail" in tags, (i, c["tags"], ev)     # the low case stops above its leaf every time
        if tags & {"repick", "low_draw_repick"}:
            assert ev[:, 0].sum() > 0, (i, c["tags"], ev)
        if "low_bail" in tags:
            assert ev[:, 1].sum() > 0, (i, c["tags"], ev)
        if tags & {"twice_on_trace", "transposition"}:
            assert np.any(pcl < np.asarray(D)), (i, c["tags"], pcl, D)
