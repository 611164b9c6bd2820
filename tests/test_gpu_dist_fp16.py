"""eval_kind dist_fp16: the distributional network on the tensor cores with one fp16 term per operand (distnet_tc.cuh, NT = 1).

The network is held to the error contract tests/f16_dist_ref.py derives (act2 per element within 2^-10 of the board's largest |term| sum
plus the split's floor; probabilities within 2 e_z p + 1e-36) against the float64 reference of tests/f64_ref.py.  The search on its outputs
is held to the C oracle exactly, as for net_tc: the distributional search is deterministic given the evaluator and the piece sequence, so
oracle agents in mode 3 fed a dist_fp16 side engine's outputs must make the same decisions, statistics, node distributions and arenas.
net_tc shares the kernels through their template argument; its outputs and act2 are held bit for bit to tests/golden/dist_act2_golden.npz."""
import os

import numpy as np
import pytest

import f16_dist_ref as D
import f64_ref as R
from arena_gen import boards as random_boards

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "dist_act2_golden.npz")


def engine(kind, w, atoms=50, n=1, **kw):
    from tetris_mcts_b200.engine import BatchedEngine
    return BatchedEngine(n, max_nodes=64, mode="dist", eval_kind=kind, dist_bins=atoms, dist_weights=w, **kw)


def act2(eng, states):
    from tetris_mcts_b200 import _lib as L
    s = np.ascontiguousarray(np.asarray(states, np.int8).reshape(-1, 200))
    out = np.zeros((len(s), 2048), np.float32)
    L.check(L.lib().b200_debug_dist_act2(eng.h, L.ptr(s), len(s), L.ptr(out)))
    return out


def check_act2(eng, w, states, atoms, what):
    got = act2(eng, states)
    ref = D.act2(w, states, atoms)
    ratio = np.abs(got - ref) / D.act2_bound(w, states, atoms)
    assert np.isfinite(got).all(), what
    if ratio.max() > 1:
        b, e = np.unravel_index(int(np.argmax(ratio)), ratio.shape)
        pytest.fail("%s: act2 board %d channel %d pixel (%d, %d): got %.9g want %.9g (error / bound %.3g)" %
                    (what, b, e // 64, (e % 64) // 4, e % 4, got[b, e], ref[b, e], ratio.max()))
    return float(ratio.max())


def check_probs(got, w, states, atoms, what, allowance=None):
    ref, _ = R.distnet(w, states, atoms)
    ez = D.logit_bound(w, states, atoms, allowance)
    assert np.isfinite(got).all() and (got >= 0).all(), what
    assert np.abs(got.astype(np.float64).sum(1) - 1).max() < 1e-5, what
    r = D.prob_excess(got, ref, ez)
    if r > 1:
        ratio = np.abs(got - ref) / (2 * ez * ref + 1e-36)
        b, a = np.unravel_index(int(np.argmax(ratio)), ratio.shape)
        pytest.fail("%s: board %d atom %d got %.9g want %.9g (error / bound %.3g)" % (what, b, a, got[b, a], ref[b, a], r))
    return r


@pytest.fixture(scope="module")
def fam(oracle):
    return R.board_families(oracle)


@pytest.mark.parametrize("atoms", [2, 3, 33, 50, 64])
def test_every_weight_and_board_family_with_hot_swaps(gpu_lib, fam, atoms):
    """Every distributional weight family x every board family on ONE engine per atom count, the weights swapped in between."""
    wf = R.dist_weight_families(5, atoms)
    eng = engine("dist_fp16", wf["init"], atoms)
    allb = np.concatenate(list(fam.values()))
    for wname, w in list(wf.items()) + [("init again", wf["init"])]:
        eng.load_dist_weights(w, atoms)
        worst = 0.0
        for bname, b in fam.items():
            worst = max(worst, check_probs(eng.distnet(b), w, b, atoms, "%s / %s" % (wname, bname), R.ALLOWANCE.get(wname.split()[0])))
        r2 = check_act2(eng, w, allb, atoms, wname)
        print("\n[dist_fp16] atoms %d %-11s act2 error/bound %.3f  probabilities error/bound %.3g" % (atoms, wname, r2, worst))
    eng.close()


def test_batch_sizes_and_passes(gpu_lib, oracle):
    """Batches of 1, 7, 300 (not a multiple of 128) and more than one pass of k_tdc_fc over all SMs; every board's probabilities do not
    depend on the batch it is in, and a small batch after a large one (stale act2 tiles past it) gives the same bits."""
    import torch
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    Fp = n_sm * 128
    w = R.dist_init_weights(2, 50)
    big = Fp + n_sm * 16 + 45
    pool = np.concatenate(list(R.board_families(oracle, 1).values()) + [random_boards(big, 23)])[:big]
    eng = engine("dist_fp16", w)
    pb = eng.distnet(pool)
    rng = np.random.default_rng(1)
    sub = np.union1d(np.r_[0:4, Fp - 2:Fp + 2, big - 3:big], rng.choice(big, 400, replace=False))
    check_probs(pb[sub], w, pool[sub], 50, "batch %d" % big)
    for n in (1, 7, 300):
        idx = rng.permutation(big)[:n]
        s = pool[idx]
        p = eng.distnet(s)
        check_probs(p, w, s, 50, "batch %d" % n)
        check_act2(eng, w, s, 50, "batch %d" % n)
        assert np.array_equal(p, pb[idx]), n
    eng.close()


def test_batch_position_invariant(gpu_lib):
    """What the network shadow relies on (test_gpu_dist_search.py::test_dist_network_batch_position_invariant for net / net_tc): a board's
    output is the same bits alone and inside batches of 2 to 20000 boards, at several positions."""
    from tetris_mcts_b200.agents.DistValueSimOnline import init_dist_weights
    side = engine("dist_fp16", init_dist_weights(0, 50))
    probe = random_boards(5, 99)
    alone = np.stack([side.distnet(probe[i:i + 1])[0] for i in range(len(probe))])
    for n in (2, 3, 127, 129, 1000, 20000):
        batch = random_boards(n, n)
        for pos in sorted({0, n // 2, n - 1}):
            b = batch.copy()
            b[pos] = probe[pos % len(probe)]
            assert np.array_equal(side.distnet(b)[pos], alone[pos % len(probe)]), (n, pos)
    side.close()


def test_agrees_with_net_tc_within_the_fp16_bound(gpu_lib, oracle):
    """On random and real positions, dist_fp16 against net_tc (itself within 1e-5 of float64): within the fp16 contract, and not equal."""
    from tetris_mcts_b200.agents.DistValueSimOnline import init_dist_weights
    s = np.concatenate([random_boards(2000, 5), R.real_positions(2000, 11, oracle)])
    for name, w in (("init", init_dist_weights(0, 50)), ("act_1e3", R.dist_weight_families(4, 50)["act_1e3"])):
        e16, etc = engine("dist_fp16", w), engine("net_tc", w)
        p16, ptc = e16.distnet(s), etc.distnet(s)
        ez = D.logit_bound(w, s, 50)
        d = np.abs(p16.astype(np.float64) - ptc)
        assert np.all(d <= (2 * ez + 2e-5) * ptc + 1e-30), name
        big = ptc > 1e-30
        worst = float(np.max(d[big] / ptc[big]))
        assert worst > 0 and not np.array_equal(act2(e16, s[:64]), act2(etc, s[:64])), name   # one product per product is not the split
        print("\ndist_fp16 vs net_tc (%s), largest relative difference of a probability on %d positions: %.3g" % (name, len(s), worst))
        e16.close(); etc.close()


def test_net_tc_bits_are_unchanged(gpu_lib, oracle):
    """net_tc's probabilities and act2 bit for bit as tests/golden/gen_dist_act2.py recorded them."""
    from golden.gen_dist_act2 import cases, digest, engine as gen_engine, run
    z = np.load(GOLD)
    cs = cases(oracle)
    eng = gen_engine("net_tc", cs[0][1])
    for name, w, s in cs:
        d, a = run(eng, w, s)
        rows = z[name + "/rows"]
        assert np.array_equal(d[rows].view(np.uint32), z[name + "/dist"].view(np.uint32)), name
        assert np.array_equal(a[rows].view(np.uint32), z[name + "/act2"].view(np.uint32)), name
        bad = np.flatnonzero(digest(d) != z[name + "/digest_dist"])
        assert not len(bad), "%s: probabilities of %d boards differ, first %d" % (name, len(bad), bad[0])
        bad = np.flatnonzero(digest(a) != z[name + "/digest_act2"])
        assert not len(bad), "%s: act2 of %d boards differs, first %d" % (name, len(bad), bad[0])
    eng.close()


def test_refusals_keep_the_previous_weights(gpu_lib):
    """A non-distributional mode, b200_load_weights (no value network), and conv / fc1 weights out of fp16 range or NaN: BAD_ARG naming
    dist_fp16, with the weights loaded before still in use."""
    from tetris_mcts_b200 import _lib as L
    from tetris_mcts_b200.engine import BatchedEngine
    for mode in ("lp", "single", "vanilla"):
        with pytest.raises(L.B200Error) as ei:
            BatchedEngine(4, max_nodes=256, mode=mode, eval_kind="dist_fp16")
        assert ei.value.code == 1 and "dist_fp16" in str(ei.value) and "net_fp16" in str(ei.value), mode
    w = R.dist_init_weights(0, 50)
    states = random_boards(16, 1)
    eng = engine("dist_fp16", w)
    with pytest.raises(L.B200Error) as ei:
        eng.load_weights(R.init_weights(0))
    assert ei.value.code == 1 and "dist_fp16" in str(ei.value)
    fits = w.copy()
    fits[544 + 5] = 1023.0                                                 # conv2: 64 * 1023 = 65472 fits
    eng.load_dist_weights(fits, 50)
    loaded = eng.distnet(states)
    for off, x in ((7, -1100.0), (544 + 5, 1024.0), (16960 + 123456, 1100.0), (16960 + 7, np.nan), (3, np.nan)):   # conv1, conv2, fc1
        bad = w.copy()
        bad[off] = x
        with pytest.raises(L.B200Error) as ei:
            eng.load_dist_weights(bad, 50)
        assert ei.value.code == 1 and "65504" in str(ei.value) and "dist_fp16" in str(ei.value), off
        assert np.array_equal(loaded, eng.distnet(states)), off
    eng.close()


def test_search_is_exact_with_collections_and_drops(gpu_lib, oracle):
    """Oracle agents in mode 3 fed a dist_fp16 side engine's outputs shadow every game (test_gpu_dist_search.shadow): arenas small enough
    for collections, the head-room policy, one explicit remove_nodes() and overflow_reset tree drops."""
    from test_gpu_dist_search import shadow
    w = R.dist_init_weights(1, 33)
    side = engine("dist_fp16", w, 33)
    c, oc, _ = shadow(oracle, n=24, M=700, sims=40, moves=30, seed=57, bins=33, vmin=0.0, vmax=1000.0, low=1, eval_kind="dist_fp16",
                      dist_weights=w, eval_cb=side.distnet, headroom=150, overflow_reset=True, remove_at=(7,))
    assert c["gcs"] > 0 and c["tree_resets"] > 0, c
    side.close()


def test_bench_config_sampled_games_exact(gpu_lib, oracle):
    """configs[4] as bench.py runs it (2048 games, 1500 simulations per move, 32768 slots, init_dist_weights(0, 50), head-room
    32768 * 5 / 32, overflow_reset, play_move) on dist_fp16: games 0, n - 1 and 14 seeded others shadowed exactly, collections included."""
    from test_gpu_dist_search import shadow
    from tetris_mcts_b200.agents.DistValueSimOnline import init_dist_weights
    n, M = 2048, 32768
    w = init_dist_weights(0, 50)
    side = engine("dist_fp16", w)
    sample = sorted(set([0, n - 1] + list(np.random.default_rng(7).choice(n, 14, replace=False))))
    c, oc, _ = shadow(oracle, n=n, M=M, sims=1500, moves=5, seed=123, eval_kind="dist_fp16", dist_weights=w, eval_cb=side.distnet,
                      overflow_reset=True, headroom=M * 5 // 32, sample=sample)
    assert c["gcs"] > 0 and oc["gcs"] > 0, (c, oc)
    side.close()


def test_two_engines_with_the_same_seeds_are_identical(gpu_lib):
    from tetris_mcts_b200 import pyTetris as PT
    from tetris_mcts_b200.engine import BatchedEngine
    from tetris_mcts_b200.agents.DistValueSimOnline import init_dist_weights
    n, M, sims, seed = 512, 4096, 150, 5
    recs = PT.new_games(n, (1, 0, 0), np.arange(seed, seed + n, dtype=np.uint32))
    engs = []
    for _ in range(2):
        e = BatchedEngine(n, max_nodes=M, mode="dist", eval_kind="dist_fp16", dist_weights=init_dist_weights(3, 50), seed=seed,
                          overflow_reset=True)
        e.set_games(recs)
        e.set_gc_headroom(M * 5 // 32)
        engs.append(e)
    for mv in range(5):
        (a0, s0), (a1, s1) = [e.play_move(sims, auto_reset=True) for e in engs]
        assert a0.tobytes() == a1.tobytes() and s0.tobytes() == s1.tobytes(), mv
        assert engs[0].get_games().tobytes() == engs[1].get_games().tobytes(), mv
    for g in (0, n - 1):
        assert all(a.tobytes() == b.tobytes() for a, b in zip(engs[0].export_dist(g), engs[1].export_dist(g))), g
    assert engs[0].counters() == engs[1].counters()
    for e in engs:
        e.close()


def test_dist_value_sim_online_takes_dist_fp16(gpu_lib):
    """play.py's surface: getattr(import_module('agents.DistValueSimOnline'), 'DistValueSimOnline')(..., eval_kind='dist_fp16')."""
    from tetris_mcts_b200 import _lib as L
    from tetris_mcts_b200.agents import DistValueSimOnline as mod
    from tetris_mcts_b200.pyTetris import Tetris
    env_args = ((20, 10), 1, 0, 0)
    game = Tetris(*env_args)
    agent = getattr(mod, "DistValueSimOnline")(sims=80, env=Tetris, env_args=env_args, benchmark=True, online=False, min_visit=40,
                                               eval_kind="dist_fp16")
    assert agent._eng.eval_kind == L.EVAL_DIST_FP16
    agent.update_root(game)
    for _ in range(3):
        a = agent.play()
        assert 0 <= a < 7
        game.play(a)
        agent.update_root(game)
    m, v = agent.get_value()
    assert 0 <= m <= 5000 and v >= 0
    assert agent.counters()["sims"] == 240
    agent.close()
    default = getattr(mod, "DistValueSimOnline")(sims=10, env=Tetris, env_args=env_args, benchmark=True, online=False)
    assert default._eng.eval_kind == L.EVAL_NET                           # the default stays "net"
    default.close()
