"""Distributional cores (SURVEY §8a a16): the C oracle vs the reference's own numba functions (golden vectors; the
reference is compiled with fastmath, so floats are compared to 1e-5 relative, traces exactly)."""
import os

import numpy as np

GOLD = os.path.join(os.path.dirname(__file__), "golden", "dist_golden.npz")


def test_dist_oracle_matches_reference_numba(oracle):
    z = np.load(GOLD)
    for i in range(int(z["n_cases"])):
        p = "d%d_" % i
        assert np.allclose(oracle.shift_distribution(z[p + "dist"], float(z[p + "x"]), 0, 5000), z[p + "shift"], rtol=1e-5, atol=1e-7)
        m, v = oracle.mean_variance(z[p + "dist"], 0, 5000)
        assert np.allclose([m, v], z[p + "mv"], rtol=1e-5)
        tr = oracle.select_trace_distributional(1, z[p + "child"], z[p + "node_stats"], 0)
        assert np.array_equal(tr, z[p + "trace"]), i
        ns, nd = z[p + "node_stats"].copy(), z[p + "node_dist"].copy()
        oracle.backup_trace_distributional(z[p + "trace"], ns, nd, float(z[p + "r"]), z[p + "dist"], 0, 5000)
        assert np.allclose(ns, z[p + "bk_stats"], rtol=1e-5, atol=1e-5)
        assert np.allclose(nd, z[p + "bk_dist"], rtol=1e-5, atol=1e-7)


EDGES = os.path.join(os.path.dirname(__file__), "golden", "dist_edges_golden.npz")


def test_dist_oracle_matches_reference_edge_goldens(oracle):
    from arena_gen import assert_dist_close, assert_mean_variance_close, load_dist_edges
    z = load_dist_edges(EDGES)
    for c in z["shift"]:
        (bins, lo, hi), x = c["cfg"], c["x"]
        assert_dist_close(oracle.shift_distribution(c["dist"], x, lo, hi), c["out"], "atoms %d range (%g, %g) x %r dist %d" % (bins, lo, hi, x, c["dist_k"]))
    for c in z["mv"]:
        bins, lo, hi = c["cfg"]
        assert_mean_variance_close(oracle.mean_variance(c["dist"], lo, hi), c["mv"], c["cfg"])
    for i, c in enumerate(z["backup"]):
        bins, lo, hi = c["cfg"]
        ns, nd = c["node_stats"].copy(), c["node_dist"].copy()
        oracle.backup_trace_distributional(c["trace"], ns, nd, c["r"], c["dist"], lo, hi)
        what = "trace %d (atoms %d range (%g, %g) depth %d)" % (i, bins, lo, hi, len(c["trace"]))
        assert np.allclose(ns, c["bk_stats"], rtol=1e-5, atol=1e-5), what
        assert_dist_close(nd, c["bk_dist"], what)


def test_dist_edge_goldens_separate_the_two_bin_mappings():
    """The edge goldens would catch the mapping b + int(x / delta): emulated in numpy, it misplaces mass on truncation cases of several
    configurations (the rows of DESIGN §3's table among them), and on no other case."""
    from arena_gen import load_dist_edges
    z = load_dist_edges(EDGES)
    caught = set()
    for c in z["shift"]:
        (bins, lo, hi), x, d = c["cfg"], c["x"], c["dist"].astype(np.float64)
        bs = x / ((hi - lo) / bins)
        frac, T = bs - np.floor(bs), bins - 1
        lb = np.minimum(np.arange(bins) + int(min(bs, bins)), T)
        ub = np.minimum(lb + 1, T)
        emu = np.zeros(bins)
        np.add.at(emu, lb, d * (1 - frac))
        np.add.at(emu, ub, d * frac)
        if not np.array_equal(emu != 0, c["out"] != 0) or not np.allclose(emu, c["out"], rtol=1e-5, atol=1e-7):
            caught.add((bins, lo, hi, x))
    for row in ((30, 0.0, 1000.0, 500.0), (56, 0.0, 5000.0, 625.0), (14, 0.0, 5000.0, 2500.0), (35, 0.0, 45.0, 9.0)):
        assert row in caught, row
    assert len({k[:3] for k in caught}) >= 8, sorted(caught)
