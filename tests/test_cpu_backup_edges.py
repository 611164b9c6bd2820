"""Pin the C oracle's backups (mo_backup_trace_obs*) to the reference's own core.cpp on the designed edge trees of tests/backup_edges.py
(tests/golden/backup_edges_golden.npz), and check that the golden holds the shapes it was designed for: every depth around the engine's
32-level windows, each pattern of repeated observations, each kind of leaf child list, the float and visit-count edges."""
import os

import numpy as np
import pytest

import backup_edges as BE

GOLD = os.path.join(os.path.dirname(__file__), "golden", "backup_edges_golden.npz")


@pytest.fixture(scope="module")
def cases():
    return BE.load(GOLD)


def test_golden_is_the_designed_cases(cases):
    """The golden stores the reference's outputs and a digest of each case's inputs; design() must regenerate exactly those inputs."""
    bad = [i for i, c in enumerate(cases) if not c["digest_ok"]]
    assert not bad, "design() no longer makes the inputs the golden was generated from (cases %s): regenerate it" % bad


def test_oracle_matches_reference(oracle, cases):
    for i, c in enumerate(cases):
        got = BE.run(c, oracle)
        for name, g, w in zip(("visit", "value", "variance"), got, c["out"]):
            assert BE.same_bits(g, w), (i, c["mode"], c["tags"], name)


def _obs(c):
    return c["n2o"][c["trace"]]


def _windows(D):
    """(top, bottom) of every 32-level window of the engine's backup, from the leaf up."""
    return [(top, max(top - 31, 0)) for top in range(D - 1, -1, -32)]


def test_depths_modes_gammas(cases):
    for D in BE.DEPTHS:
        for kind in (0, 1):
            assert any(len(c["trace"]) == D and c["kind"] == kind for c in cases), (D, kind)
        for mode in BE.MODES:
            assert any(len(c["trace"]) == D and c["mode"] == mode and c["kind"] == 1 for c in cases), (D, mode)
    assert {c["gamma"] for c in cases} == set(BE.GAMMAS)
    assert max(len(c["trace"]) for c in cases) == 512


def test_repeat_patterns(cases):
    found = set()
    for c in cases:
        o, D = _obs(c), len(c["trace"])
        if D < 2:
            continue
        if np.any(o[1:] == o[:-1]):
            found.add("adjacent")
        for top, bot in _windows(D):
            if top - bot == 31 and o[top] == o[bot]:
                found.add("lanes0_31")
            if bot > 0 and o[bot] == o[bot - 1]:
                found.add("across_edge")
        if D >= 33 and o[31] == o[32]:
            found.add("levels31_32")
        if D >= 65 and o[63] == o[64]:
            found.add("levels63_64")
        if o[0] == o[-1]:
            found.add("first_last")
        if np.max(np.unique(o, return_counts=True)[1]) >= 3:
            found.add("three_or_more")
        if np.all(o == o[0]):
            found.add("all_same")
        for d in range(D - 1):
            kids = c["child"][c["trace"][d]]
            sib = kids[(kids != 0) & (kids != c["trace"][d + 1])]
            if np.isin(c["n2o"][sib], o).any():
                found.add("transposition")
        if c["kind"] == 1:
            leaf_obs = c["n2o"][c["child"][c["trace"][-1]][c["child"][c["trace"][-1]] != 0]]
            if np.isin(leaf_obs, o).any():
                found.add("leaf_child_on_trace")
    assert found == {"adjacent", "lanes0_31", "across_edge", "levels31_32", "levels63_64", "first_last", "three_or_more", "all_same",
                     "leaf_child_on_trace", "transposition"}, found


def test_leaf_children(cases):
    ks, found = set(), set()
    for c in cases:
        if c["mode"] not in ("lp", "lpcpp"):
            continue
        if c["kind"] == 0:
            ks.add(0)
            continue
        leaf = int(c["trace"][-1])
        row = c["child"][leaf]
        cn, co, slot = BE.unique_children(leaf, c["child"], c["score"], c["n2o"])
        ks.add(len(cn))
        live = row[row != 0]
        if np.any(row == 0):
            found.add("zero_ids")
        obs, sc = c["n2o"][live], c["score"][live]
        for o in set(obs.tolist()):
            s = sc[obs == o]
            if len(s) > 1:
                found.add("dup_equal" if np.all(s == s.max()) or np.sum(s == s.max()) > 1 else "dup_unequal")
        vis = c["visit"][co]
        if np.any(vis == 0):
            found.add("visit0")
        if np.any(vis > 0):
            found.add("visit_pos")
    assert ks == set(range(8)), ks
    assert found == {"zero_ids", "dup_equal", "dup_unequal", "visit0", "visit_pos"}, found


def test_float_and_visit_edges(cases):
    evals, visits = [], set()
    for c in cases:
        if c["kind"] == 1 and c["mode"] in ("lp", "lpcpp"):
            _, co, slot = BE.unique_children(int(c["trace"][-1]), c["child"], c["score"], c["n2o"])
            evals += c["ev"][slot].ravel().tolist()
        elif c["kind"] == 1 and c["mode"] == "single":
            evals += c["ev"][7].tolist()
        visits |= set(c["visit"][_obs(c)].tolist())
    ev = np.asarray(evals, np.float32)
    assert np.any(ev == 0) and np.any(ev < 0) and np.any(ev == np.float32(1e30))
    assert np.any((ev != 0) & (np.abs(ev) < np.finfo(np.float32).tiny))
    assert np.any(ev == np.inf) and np.any(ev == -np.inf) and np.any(np.isnan(ev))
    assert {0, 1, (1 << 24) - 1, 1 << 24, (1 << 24) + 1} <= visits and max(visits) >= 1_000_000
    # the NaN / inf inputs reach the reference's outputs
    assert any(np.isnan(c["out"][1]).any() for c in cases) and any(np.isinf(c["out"][1]).any() for c in cases)
