"""The fp32 CUDA-core networks (eval_kind net: k_vn_conv / k_vn_fc, k_dn_conv / k_dn_fc) held stage by stage to tests/f32_net_ref.py:
every stage that b200_debug_net_acts exports must equal, bit for bit, the restatement from the kernel's own previous stage (NaN equals
NaN, zeros compare by value), and every output must lie in the set that expf's 2 ulp admit.  The export is itself held bit for bit to the
production paths: the value network's act3 to b200_debug_act3 and both networks' outputs to eng.valuenet / eng.distnet.

Covered: every weight family with hot swaps on one engine, plus a `huge` family (finite weights that only net accepts) whose sums
overflow to +-inf and NaN; the distributional network at 2 to 64 atoms; batches at every tile and pass edge of the four kernels, then a
small batch again; and two searches with eval_kind net whose steps cross the conv kernels' grid-stride passes, shadowed by the oracle."""
import time

import numpy as np
import pytest
import torch

import f32_net_ref as N
import f64_ref as R
from arena_gen import boards as random_boards

pytestmark = pytest.mark.gpu
ATOMS = 50
T0 = time.time()


@pytest.fixture(scope="module")
def n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def engine(dist, w, atoms=ATOMS):
    from tetris_mcts_b200.engine import BatchedEngine
    if dist:
        return BatchedEngine(1, max_nodes=64, mode="dist", eval_kind="net", dist_bins=atoms, dist_weights=w)
    return BatchedEngine(1, max_nodes=64, eval_kind="net", weights=w)


def shape(dist, layer, n, atoms):
    grid = N.DN_GRID if dist else N.VN_GRID
    if layer == 0 or (dist and layer == 4):
        return (n, atoms if dist else 2)
    if layer in grid:
        return (n, 32) + grid[layer]
    return (n, 128 if dist else 256)


def export(eng, dist, states, layer, atoms=ATOMS):
    from tetris_mcts_b200 import _lib as lib
    s = np.ascontiguousarray(np.asarray(states, np.int8).reshape(-1, 200))
    out = np.zeros(shape(dist, layer, len(s), atoms), np.float32)
    lib.check(lib.lib().b200_debug_net_acts(eng.h, int(dist), lib.ptr(s), len(s), layer, lib.ptr(out)))
    return out


def check(eng, w, states, dist, what, rows=None, atoms=ATOMS):
    """every stage of every board (or of `rows` of the batch) equal to its restatement, the outputs in their sets, and the export equal to
    the production paths bit for bit -> (median, largest head set width in ulps, fraction of non-finite elements per stage)"""
    from tetris_mcts_b200 import _lib as lib
    states = np.ascontiguousarray(np.asarray(states, np.int8).reshape(-1, 200))
    rows = np.arange(len(states)) if rows is None else rows
    stages = N.DN_STAGES if dist else N.VN_STAGES
    layer = {s: (0 if s == "out" else i + 1) for i, s in enumerate(stages)}
    got = {s: export(eng, dist, states, layer[s], atoms) for s in stages}
    label = "%s %s" % ("dist" if dist else "value", what)
    if dist:
        prod = eng.distnet(states)
    else:
        v, var = eng.valuenet(states)
        prod = np.stack([v, var], 1)
        a3 = np.zeros((len(states), 1792), np.float32)
        lib.check(lib.lib().b200_debug_act3(eng.h, lib.ptr(states), len(states), lib.ptr(a3)))
        assert np.array_equal(got["act3"].reshape(len(states), -1).view(np.uint32), a3.view(np.uint32)), "%s: act3 differs from the production path" % label
    assert np.array_equal(got["out"].view(np.uint32), prod.view(np.uint32)), "%s: outputs differ from the production path" % label
    c = N.StageCheck(w, states[rows], {s: got[s][rows] for s in stages}, dist)
    if c.total():
        pytest.fail(c.describe(label))
    nonfinite = {s: float((~np.isfinite(got[s][rows])).mean()) for s in stages}
    return float(np.median(c.width)), int(c.width.max()), nonfinite


def report(dist, what, r):
    wmed, wmax, nf = r
    bad = ", ".join("%s %.4f" % kv for kv in nf.items() if kv[1])
    print("\n[net %s] %-18s head set width %.1f / %d ulps (median / max)%s  (%.0f s)" % (
        "dist" if dist else "value", what, wmed, wmax, " | non-finite: " + bad if bad else "", time.time() - T0))


def families(dist):
    fam = dict(R.dist_weight_families(5, ATOMS) if dist else R.weight_families(0))
    fam["huge"] = N.huge_dist_weights(5, ATOMS) if dist else N.huge_value_weights(0)
    return fam


def fp32_reference(w, states, dist):
    """the reference network in torch fp32 (Model_VV / Model.inference precision) -> outputs"""
    if dist:
        return R.distnet(w, states, ATOMS, torch.float32)[0]
    p = R.unpack(w, R.VN_SHAPES, torch.float32)
    with torch.no_grad():
        return R._vn_forward(p, R._x(states, torch.float32))[0].numpy()


@pytest.mark.parametrize("dist", [False, True], ids=["value", "dist"])
def test_every_stage_on_every_weight_family_with_hot_swaps(gpu_lib, oracle, dist):
    """Every weight family plus `huge` x the impulse, edge and real-position boards and 64 random ones, on ONE engine with the weights
    swapped in between.  For `huge`, prints how the outputs compare with float64 and with the fp32 reference network, which overflow
    differently (float64 not at all; torch's ReLU keeps NaN where fmaxf gives 0)."""
    b = np.concatenate(list(R.board_families(oracle).values()) + [random_boards(64, 7)])
    wf = families(dist)
    eng = engine(dist, wf["init"])
    for wname, w in list(wf.items()) + [("init again", wf["init"])]:
        if dist:
            eng.load_dist_weights(w, ATOMS)
        else:
            eng.load_weights(w)
        report(dist, wname, check(eng, w, b, dist, wname))
        if wname == "huge":
            out = export(eng, dist, b, 0)
            f64 = R.distnet(w, b, ATOMS)[0] if dist else np.stack(R.valuenet(w, b)[:2], 1)
            f32 = fp32_reference(w, b, dist)
            fin = np.isfinite(out).all(1)
            print("[net %s] huge: boards with finite outputs %d / %d; float64 finite on %d, the fp32 reference on %d; net finite where the fp32 "
                  "reference is not: %d; largest relative difference from float64 where both are finite: %.3g" % (
                      "dist" if dist else "value", fin.sum(), len(b), np.isfinite(f64).all(1).sum(), np.isfinite(f32).all(1).sum(),
                      (fin & ~np.isfinite(f32).all(1)).sum(), float(np.max(np.abs(out[fin] - f64[fin]) / np.abs(f64[fin]))) if fin.any() else 0.0))
            nf = (~np.isfinite(export(eng, dist, b, 2 if dist else 3))).mean()
            assert nf > 0, "huge: no act2 / act3 sum overflowed"
    eng.close()


@pytest.mark.parametrize("atoms", [2, 3, 31, 32, 33, 50, 63, 64])
def test_every_stage_at_atoms(gpu_lib, oracle, atoms):
    """64 is the row stride of the logits in shared memory; above 32 atoms, 8 rows x atoms > 256 makes the fc_v task loop wrap."""
    b = np.concatenate([R.board_families(oracle)["real"][:40], random_boards(27, atoms)])
    w = R.dist_init_weights(atoms, atoms)
    eng = engine(True, w, atoms)
    report(True, "atoms %d" % atoms, check(eng, w, b, True, "atoms %d" % atoms, atoms=atoms))
    w = R.dist_weight_families(1, atoms)["saturated"]
    eng.load_dist_weights(w, atoms)
    report(True, "atoms %d saturated" % atoms, check(eng, w, b, True, "atoms %d saturated" % atoms, atoms=atoms))
    eng.close()


def _rows(n, periods, rng):
    """every row for small batches; else the rows on both sides of every multiple of each period, the first and last rows and 100 others"""
    if n <= 65:
        return np.arange(n)
    idx = {0, 1, 2, 3, n - 3, n - 2, n - 1}
    for p in periods:
        for k in range(p, n, p):
            idx.update((k - 1, k))
    return np.union1d(np.array(sorted(idx)), rng.choice(n, 100, replace=False))


@pytest.mark.parametrize("dist", [False, True], ids=["value", "dist"])
def test_every_stage_at_tile_and_pass_edges(gpu_lib, oracle, n_sm, dist):
    """S = SM count.  Batches 1, 3, 4, 5, 7, 8, 9, 63, 64, 65 (k_vn_conv's 4-board and k_dn_fc's 8-row tiles, k_vn_fc's 64-row tiles),
    2S +- 1 (k_dn_conv's pass: one board on each of 2S CTAs), 4S +- 1 (k_vn_conv's: 4-board tiles on S CTAs), 8S +- 1 (k_dn_fc's: 8 rows on
    S CTAs), one batch past 128S (k_vn_fc's: 64-row tiles on 2S CTAs), then 5 boards again (a stale tile or buffer would show there)."""
    S = n_sm
    sizes = [1, 3, 4, 5, 7, 8, 9, 63, 64, 65, 2 * S - 1, 2 * S + 1, 4 * S - 1, 4 * S + 1, 8 * S - 1, 8 * S + 1, 128 * S + 4 * S + 45, 5]
    periods = (64, 2 * S, 4 * S, 8 * S, 128 * S)
    pool = np.concatenate(list(R.board_families(oracle, 1).values()) + [random_boards(sizes[-2], 23)])
    w = R.dist_weight_families(2, ATOMS)["act_1e3"] if dist else R.weight_families(2)["trained_bounds"]
    eng = engine(dist, w)
    rng = np.random.default_rng(3)
    for n in sizes:
        s = pool[rng.permutation(len(pool))[:n]]
        report(dist, "batch %d" % n, check(eng, w, s, dist, "batch %d" % n, _rows(n, periods, rng)))
    eng.close()


def test_lp_search_across_the_conv_pass_is_exact(gpu_lib, oracle, n_sm):
    """ValueSimLP with eval_kind net and 160 games: a step evaluates up to 7 children per game, so its requests cross k_vn_conv's pass of
    4S boards.  The oracle agents get each leaf's outputs from a side engine (standalone network outputs, checked above)."""
    from test_gpu_engine import run_pair
    from tetris_mcts_b200.engine import BatchedEngine
    w = oracle.seeded_weights(0)
    side = BatchedEngine(1, max_nodes=64, eval_kind="net", weights=w)

    def cb(states):
        return side.valuenet(states)

    sims, moves = 12, 3
    c = run_pair(oracle, "lp", n=160, M=2048, sims=sims, moves=moves, eval_kind="net", weights=w, eval_cb=cb)
    side.close()
    per_step = c["eval_requests"] / (sims * moves)
    print("\n[net lp search] %.0f requests per step on average (4S = %d)" % (per_step, 4 * n_sm))
    assert per_step > 4 * n_sm, per_step


def test_dist_search_across_the_fc_pass_is_exact(gpu_lib, oracle, n_sm):
    """The distributional search with eval_kind net and more than 8S games (k_dn_fc's pass; k_dn_conv's is 2S), 16 of them shadowed by
    oracle agents fed by a side engine, as test_dist_bench_config_sampled_games_exact does for net_tc."""
    from test_gpu_dist_search import shadow
    from tetris_mcts_b200.engine import BatchedEngine
    from tetris_mcts_b200.agents.DistValueSimOnline import init_dist_weights
    n, M = 8 * n_sm + 77, 2048
    w = init_dist_weights(0, 50)
    side = BatchedEngine(1, max_nodes=64, mode="dist", eval_kind="net", dist_weights=w)
    sample = sorted(set([0, n - 1, 8 * n_sm - 1, 8 * n_sm] + list(np.random.default_rng(9).choice(n, 12, replace=False))))
    c, oc, _ = shadow(oracle, n=n, M=M, sims=40, moves=4, seed=321, eval_kind="net", dist_weights=w, eval_cb=side.distnet,
                      overflow_reset=True, headroom=M * 5 // 32, sample=sample)
    side.close()
    print("\n[net dist search] %d games (8S = %d), %d requests, %d collections" % (n, 8 * n_sm, c["eval_requests"], c["gcs"]))


def test_refusals(gpu_lib):
    """b200_debug_net_acts reads eval_kind net only; it refuses dist outside 0 / 1 and layers outside 0..4, returns NO_WEIGHTS for a
    network without weights, and answers the last layer of both networks."""
    from tetris_mcts_b200 import _lib as lib
    w = R.init_weights(0)
    s = np.zeros((1, 200), np.int8)
    out = np.zeros(4096, np.float32)
    fn = lib.lib().b200_debug_net_acts
    from tetris_mcts_b200.engine import BatchedEngine
    eng = BatchedEngine(1, max_nodes=64, eval_kind="net_tc", weights=w)
    assert fn(eng.h, 0, lib.ptr(s), 1, 1, lib.ptr(out)) == 1                                     # not eval_kind net
    eng.close()
    eng = engine(False, w)
    for dist, layer in ((0, 5), (0, -1), (2, 1), (-1, 0)):
        assert fn(eng.h, dist, lib.ptr(s), 1, layer, lib.ptr(out)) == 1, (dist, layer)
    assert fn(eng.h, 1, lib.ptr(s), 1, 1, lib.ptr(out)) == 5                                     # no distributional weights
    lib.check(fn(eng.h, 0, lib.ptr(s), 1, 4, lib.ptr(out)))
    eng.close()
    eng = engine(True, R.dist_init_weights(0, ATOMS))
    assert fn(eng.h, 1, lib.ptr(s), 1, 5, lib.ptr(out)) == 1
    assert fn(eng.h, 0, lib.ptr(s), 1, 1, lib.ptr(out)) == 5                                     # no value weights
    lib.check(fn(eng.h, 1, lib.ptr(s), 1, 4, lib.ptr(out)))
    eng.close()
