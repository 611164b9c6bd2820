"""The tensor-core conv stacks held layer by layer to tests/f16_layer_ref.py: every element of act1, act2 (and act3) that k_tc_conv /
k_tdc_conv write, read back by b200_debug_tc_acts, must lie in its admissible set given the kernel's own previous layer.  The one-term kinds
(net_fp16, dist_fp16) are held to a range of fp16 values that is a single value for most elements; net_tc (value and distributional) to a
canonical split whose sum lies in the same interval.  The export itself is held bit for bit to the production paths: its last layer to
b200_debug_act3 / b200_debug_dist_act2 and its outputs to the engine's valuenet / distnet."""
import numpy as np
import pytest

import f16_layer_ref as L
import f64_ref as R
from arena_gen import boards as random_boards

pytestmark = pytest.mark.gpu
ATOMS = 50
KINDS = [("net_fp16", False), ("net_tc", False), ("dist_fp16", True), ("net_tc", True)]
IDS = ["net_fp16", "net_tc-value", "dist_fp16", "net_tc-dist"]


def engine(kind, dist, w):
    from tetris_mcts_b200.engine import BatchedEngine
    if dist:
        return BatchedEngine(1, max_nodes=64, mode="dist", eval_kind=kind, dist_bins=ATOMS, dist_weights=w)
    return BatchedEngine(1, max_nodes=64, eval_kind=kind, weights=w)


def export(eng, dist, states, layer, nt):
    from tetris_mcts_b200 import _lib as lib
    s = np.ascontiguousarray(np.asarray(states, np.int8).reshape(-1, 200))
    shape = (len(s), ATOMS if dist else 2) if layer == 0 else (len(s), nt) + (32,) + L.GRID[dist][layer]
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
    """every layer of every board (or of `rows` of the batch) in its admissible set, and the export equal to the production paths bit for
    bit -> fraction of elements with a single admissible value, per layer"""
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
    return fr


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
        fr = check_kind(eng, kind, dist, w, b, wname)
        print("\n[%s%s] %-14s single admissible value: %s" % (kind, " dist" if dist else "", wname, " ".join("act%d %.3f" % (i + 1, f) for i, f in enumerate(fr))))
    eng.close()


@pytest.mark.parametrize("kind,dist", KINDS, ids=IDS)
def test_every_layer_at_batch_sizes_and_passes(gpu_lib, oracle, kind, dist):
    """Batches of 1, 7, 300 and one larger than a pass of 128-board tiles over all SMs (checked on its first, last and pass-boundary boards
    and 300 others)."""
    import torch
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    fp = n_sm * 128
    big = fp + n_sm * 16 + 45
    pool = np.concatenate(list(R.board_families(oracle, 1).values()) + [random_boards(big, 23)])[:big]
    w = R.dist_init_weights(2, ATOMS) if dist else R.weight_families(2)["trained_bounds"]
    eng = engine(kind, dist, w)
    rng = np.random.default_rng(3)
    for n in (1, 7, 300):
        check_kind(eng, kind, dist, w, pool[rng.permutation(big)[:n]], "batch %d" % n)
    rows = np.union1d(np.r_[0:4, fp - 2:fp + 2, big - 3:big], rng.choice(big, 300, replace=False))
    check_kind(eng, kind, dist, w, pool, "batch %d" % big, rows)
    eng.close()


def test_refusals(gpu_lib):
    from tetris_mcts_b200 import _lib as lib
    w = R.init_weights(0)
    s = np.zeros((1, 200), np.int8)
    out = np.zeros(4096, np.float32)
    eng = engine("net", False, w)
    assert lib.lib().b200_debug_tc_acts(eng.h, 0, lib.ptr(s), 1, 1, lib.ptr(out)) != 0          # not a tensor-core kind
    eng.close()
    eng = engine("net_fp16", False, w)
    for dist, layer in ((0, 4), (0, -1), (1, 1)):                                                  # no such layer; no distributional net
        assert lib.lib().b200_debug_tc_acts(eng.h, dist, lib.ptr(s), 1, layer, lib.ptr(out)) != 0
    eng.close()
