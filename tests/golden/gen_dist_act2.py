"""Record the bits of the tensor-core distributional network (eval kind net_tc: k_tdc_conv<2> + k_tdc_fc<2>) into
tests/golden/dist_act2_golden.npz.

The kernels are shared with eval kind dist_fp16 through their term-count template argument; the two-term instantiation must keep every
product and every fp32 sum in the same order, so its outputs must stay bit for bit what is recorded here (tests/test_gpu_dist_fp16.py).
Recorded per case:
  digest_dist, digest_act2   a 32-bit hash of each board's probabilities (b200_distnet_forward) and of its act2 row
                             (b200_debug_dist_act2: the conv stack's output in torch order c*64 + y*4 + x)
  rows, dist, act2           full rows of one or two boards of the case, so that a mismatch there can be named by atom, channel and pixel
                             (the hashes keep the file small: a full act2 row is 8 KB)
Cases: every family of f64_ref.dist_weight_families(5, 50) (torch init, activations near 1e3, subnormal low terms, saturated softmax) on
impulse boards, edge boards and real game positions; and batch sizes on each side of a warpgroup's run of 4 boards, of a 128-board fc
tile, and one board past a whole k_tdc_fc pass (132 SMs x 128 boards).
Run on an H100:  python tests/golden/gen_dist_act2.py      (writes the npz next to this file)"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)
import f64_ref as R  # noqa: E402
from arena_gen import boards as random_boards  # noqa: E402

OUT = os.path.join(HERE, "dist_act2_golden.npz")
ATOMS = 50
BATCH_SIZES = (1, 4, 5, 127, 128, 129, 300, 16897)
N_FULL = {"family": 2, "batch": 1}           # boards per case whose rows are stored in full


def cases(oracle):
    """-> [(name, weights, boards)]"""
    allb = np.concatenate(list(R.board_families(oracle).values()))
    out = [("family_" + name, w, allb) for name, w in R.dist_weight_families(5, ATOMS).items()]
    pool = np.concatenate([random_boards(BATCH_SIZES[-1], 17), R.real_positions(512, 11, oracle)])
    rng = np.random.default_rng(0)
    w = R.dist_init_weights(2, ATOMS)
    for n in BATCH_SIZES:
        out.append(("batch_%d" % n, w, pool[rng.permutation(len(pool))[:n]]))
    return out


def full_rows(name, n):
    return np.unique(np.linspace(0, n - 1, min(n, N_FULL[name.split("_")[0]])).round().astype(np.int64))


def digest(a):
    return np.array([int.from_bytes(hashlib.blake2b(r.tobytes(), digest_size=4).digest(), "little") for r in a], np.uint32)


def act2_of(eng, states):
    from tetris_mcts_b200 import _lib as L
    s = np.ascontiguousarray(np.asarray(states, np.int8).reshape(-1, 200))
    out = np.zeros((len(s), 2048), np.float32)
    L.check(L.lib().b200_debug_dist_act2(eng.h, L.ptr(s), len(s), L.ptr(out)))
    return out


def run(eng, w, states):
    """-> (probabilities, act2) with weights w on the boards"""
    eng.load_dist_weights(w, ATOMS)
    return eng.distnet(states), act2_of(eng, states)


def engine(kind, w):
    from tetris_mcts_b200.engine import BatchedEngine
    return BatchedEngine(1, max_nodes=64, mode="dist", eval_kind=kind, dist_bins=ATOMS, dist_weights=w)


def main():
    import oracle_py
    oracle_py.build()
    cs = cases(oracle_py)
    eng = engine("net_tc", cs[0][1])
    rec = {}
    for name, w, s in cs:
        d, a = run(eng, w, s)
        rows = full_rows(name, len(s))
        rec.update({name + "/digest_dist": digest(d), name + "/digest_act2": digest(a), name + "/rows": rows,
                    name + "/dist": d[rows], name + "/act2": a[rows]})
        print("%-20s %5d boards" % (name, len(s)), flush=True)
    eng.close()
    np.savez_compressed(OUT, **rec)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
