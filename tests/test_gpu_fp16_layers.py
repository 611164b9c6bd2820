"""The tensor-core networks held layer by layer to tests/f16_layer_ref.py: every element of act1, act2 (and act3) that k_tc_conv /
k_tdc_conv write, read back by b200_debug_tc_acts, must lie in its admissible set given the kernel's own previous layer.  The one-term kinds
(net_fp16, dist_fp16) are held to a range of fp16 values that is a single value for most elements; net_tc (value and distributional) to a
canonical split whose sum lies in the same interval.  Then the fc stage (k_tc_fc / k_tdc_fc): fc1's fp32 accumulator to its interval given
the kernel's own last conv layer, and every output to the few fp32 values its head restatement admits given the kernel's own accumulator.
The export itself is held bit for bit to the production paths: its last conv layer to b200_debug_act3 / b200_debug_dist_act2 and its
outputs to the engine's valuenet / distnet."""
import numpy as np
import pytest

import f16_layer_ref as L
import f64_ref as R
from arena_gen import boards as random_boards

pytestmark = pytest.mark.gpu
ATOMS = 50
KINDS = [("net_fp16", False), ("net_tc", False), ("dist_fp16", True), ("net_tc", True)]
IDS = ["net_fp16", "net_tc-value", "dist_fp16", "net_tc-dist"]
FC1_LAYER = {False: 4, True: 3}              # b200_debug_tc_acts' layer index of fc1's accumulator


def engine(kind, dist, w):
    from tetris_mcts_b200.engine import BatchedEngine
    if dist:
        return BatchedEngine(1, max_nodes=64, mode="dist", eval_kind=kind, dist_bins=ATOMS, dist_weights=w)
    return BatchedEngine(1, max_nodes=64, eval_kind=kind, weights=w)


def export(eng, dist, states, layer, nt):
    from tetris_mcts_b200 import _lib as lib
    s = np.ascontiguousarray(np.asarray(states, np.int8).reshape(-1, 200))
    if layer == 0:
        shape = (len(s), ATOMS if dist else 2)
    elif layer == FC1_LAYER[dist]:
        shape = (len(s), L.FC1[dist][0])
    else:
        shape = (len(s), nt) + (32,) + L.GRID[dist][layer]
    out = np.zeros(shape, np.float32)
    lib.check(lib.lib().b200_debug_tc_acts(eng.h, int(dist), lib.ptr(s), len(s), layer, lib.ptr(out)))
    return out


def production(eng, dist, states):
    """(last conv layer in torch flatten order, outputs) from the production entry points"""
    from tetris_mcts_b200 import _lib as lib
    s = np.ascontiguousarray(np.asarray(states, np.int8).reshape(-1, 200))
    last = np.zeros((len(s), 2048 if dist else 1792), np.float32)
    fn = lib.lib().b200_debug_dist_act2 if dist else lib.lib().b200_debug_act3
    lib.check(fn(eng.h, lib.ptr(s), len(s), lib.ptr(last)))
    if dist:
        return last, eng.distnet(s)
    v, var = eng.valuenet(s)
    return last, np.stack([v, var], 1)


def check_kind(eng, kind, dist, w, states, what, rows=None):
    """every layer of every board (or of `rows` of the batch) in its admissible set, then fc1's accumulator and the outputs, and the export
    equal to the production paths bit for bit -> (fraction of elements with a single admissible value per conv layer, largest fraction of
    the fc1 bound used, median and largest width of the outputs' admissible sets in fp32 ulps)"""
    nt = 1 if kind.endswith("fp16") else 2
    label = "%s%s %s" % (kind, " (distributional)" if dist else "", what)
    states = np.asarray(states, np.int8).reshape(-1, 200)
    rows = np.arange(len(states)) if rows is None else rows
    n_layers = 2 if dist else 3
    got = []
    for l in range(1, n_layers + 1):
        a = export(eng, dist, states, l, nt)
        got.append([a[rows, s].astype(np.float64) for s in range(nt)])
    # b200_debug_act3 / b200_debug_dist_act2 add the terms to 0.f in fp32 in this order (so LeakyReLU's -0 reads back as +0)
    flat = (np.float32(0) + a[:, 1]) + a[:, 0] if nt == 2 else np.float32(0) + a[:, 0]
    out0 = export(eng, dist, states, 0, nt)
    last, out = production(eng, dist, states)
    assert np.array_equal(flat.reshape(len(states), -1).view(np.uint32), last.view(np.uint32)), "%s: last layer differs from the production path" % label
    assert np.array_equal(out0.view(np.uint32), out.view(np.uint32)), "%s: outputs differ from the production path" % label
    fr = []
    for c in L.check_stack(w, states[rows], got, dist):
        if c.bad():
            pytest.fail(c.describe(label))
        fr.append(float(c.single.mean()))
    d = export(eng, dist, states, FC1_LAYER[dist], nt)[rows]
    fc1 = L.Fc1Check(w, got[-1], d, dist)
    if fc1.bad():
        pytest.fail(fc1.describe(label))
    head = L.HeadCheck(w, d, out0[rows], dist)
    if head.bad():
        pytest.fail(head.describe(label))
    return fr, float(fc1.used.max()), float(np.median(head.width)), int(head.width.max())


def report(kind, dist, what, r):
    fr, used, wmed, wmax = r
    print("\n[%s%s] %-14s single admissible value: %s | fc1 bound used %.4f | head set width %.1f / %d ulps (median / max)" % (
        kind, " dist" if dist else "", what, " ".join("act%d %.3f" % (i + 1, f) for i, f in enumerate(fr)), used, wmed, wmax))


@pytest.mark.parametrize("kind,dist", KINDS, ids=IDS)
def test_every_layer_on_every_weight_and_board_family_with_hot_swaps(gpu_lib, oracle, kind, dist):
    """Every weight family x the impulse, edge and real-position boards on ONE engine, the weights swapped in between."""
    fam = R.board_families(oracle)
    b = np.concatenate(list(fam.values()) + [random_boards(64, 7)])
    wf = R.dist_weight_families(5, ATOMS) if dist else R.weight_families(0)
    eng = engine(kind, dist, wf["init"])
    for wname, w in list(wf.items()) + [("init again", wf["init"])]:
        if dist:
            eng.load_dist_weights(w, ATOMS)
        else:
            eng.load_weights(w)
        report(kind, dist, wname, check_kind(eng, kind, dist, w, b, wname))
    eng.close()


@pytest.mark.parametrize("kind,dist", KINDS, ids=IDS)
def test_every_layer_at_batch_sizes_and_passes(gpu_lib, oracle, kind, dist):
    """Batches of 1, 7, 300, one larger than a pass of 128-board tiles over all SMs (checked on its first and last boards, the boards on
    each side of every 128-board tile and of the pass, and 300 others), then a small batch again (a stale tile would show there)."""
    import torch
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    fp = n_sm * 128
    big = fp + n_sm * 16 + 45
    pool = np.concatenate(list(R.board_families(oracle, 1).values()) + [random_boards(big, 23)])[:big]
    w = R.dist_init_weights(2, ATOMS) if dist else R.weight_families(2)["trained_bounds"]
    eng = engine(kind, dist, w)
    rng = np.random.default_rng(3)
    for n in (1, 7, 300):
        report(kind, dist, "batch %d" % n, check_kind(eng, kind, dist, w, pool[rng.permutation(big)[:n]], "batch %d" % n))
    edges = np.arange(128, big, 128)
    rows = np.union1d(np.r_[0:4, fp - 2:fp + 2, big - 3:big, edges - 1, edges], rng.choice(big, 300, replace=False))
    report(kind, dist, "batch %d" % big, check_kind(eng, kind, dist, w, pool, "batch %d" % big, rows))
    report(kind, dist, "batch 5 after", check_kind(eng, kind, dist, w, pool[rng.permutation(big)[:5]], "batch 5 after the large one"))
    eng.close()


def test_refusals_past_the_fc1_layer(gpu_lib):
    """b200_debug_tc_acts refuses non-tensor-core kinds, the other network, negative layers and layers past fc1's accumulator (5 for the
    value network, 4 for the distributional one), and answers for fc1's accumulator itself."""
    from tetris_mcts_b200 import _lib as lib
    w = R.init_weights(0)
    s = np.zeros((1, 200), np.int8)
    out = np.zeros(4096, np.float32)
    eng = engine("net", False, w)
    assert lib.lib().b200_debug_tc_acts(eng.h, 0, lib.ptr(s), 1, 1, lib.ptr(out)) != 0          # not a tensor-core kind
    eng.close()
    eng = engine("net_fp16", False, w)
    for dist, layer in ((0, 5), (0, -1), (1, 1)):                                                  # no such layer; no distributional net
        assert lib.lib().b200_debug_tc_acts(eng.h, dist, lib.ptr(s), 1, layer, lib.ptr(out)) != 0
    lib.check(lib.lib().b200_debug_tc_acts(eng.h, 0, lib.ptr(s), 1, 4, lib.ptr(out)))             # fc1's accumulator, the last layer
    eng.close()
    eng = engine("dist_fp16", True, R.dist_init_weights(0, ATOMS))
    for dist, layer in ((1, 4), (1, -1), (0, 1)):                                                  # no such layer; no value net
        assert lib.lib().b200_debug_tc_acts(eng.h, dist, lib.ptr(s), 1, layer, lib.ptr(out)) != 0
    lib.check(lib.lib().b200_debug_tc_acts(eng.h, 1, lib.ptr(s), 1, 3, lib.ptr(out)))
    eng.close()
