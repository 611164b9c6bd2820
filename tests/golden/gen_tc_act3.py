"""Record the bits of the tensor-core value network (eval kind net_tc: k_tc_conv + k_tc_fc) into tests/golden/tc_act3_golden.npz.

k_tc_conv may be rescheduled (tile shapes, accumulator splits, operand layouts) only in ways that keep every product and every fp32
sum in the same order, so a rewrite must reproduce these outputs bit for bit (tests/test_gpu_tc_conv_bits.py).  Recorded per case:
  v, var       b200_valuenet_forward's outputs (float32)
  digest       a 64-bit hash of each board's act3 row (b200_debug_act3: the conv stack's output in torch order c*56 + y*4 + x)
  act3, rows   full act3 rows of a few boards of the case, so that a mismatch there can be named by channel and pixel
Cases: every weight family of f64_ref.weight_families(0) (torch init, activations near 1e3, subnormal low terms, mostly dead / all live
ReLUs, saturated logits, trained output bounds) on impulse boards, edge boards and real game positions; and batch sizes on each side of
a warpgroup's run of 4 boards, of a 128-row act3 tile and of a whole k_tc_conv pass (132 SMs x 4 warpgroups x 4 boards).
Run on an H100:  python tests/golden/gen_tc_act3.py      (writes the npz next to this file)"""
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

OUT = os.path.join(HERE, "tc_act3_golden.npz")
BATCH_SIZES = (1, 2, 3, 4, 5, 7, 8, 9, 127, 128, 129, 255, 256, 257, 2111, 2112, 2113, 4133)
N_FULL = {"family": 8, "batch": 2}            # boards per case whose act3 rows are stored in full


def cases(oracle):
    """-> [(name, weights, boards)]"""
    fam = R.board_families(oracle)
    allb = np.concatenate(list(fam.values()))
    out = [("family_" + name, w, allb) for name, w in R.weight_families(0).items()]
    pool = np.concatenate([random_boards(BATCH_SIZES[-1], 17), R.real_positions(512, 11, oracle)])
    rng = np.random.default_rng(0)
    w = R.weight_families(2)["trained_bounds"]
    for n in BATCH_SIZES:
        out.append(("batch_%d" % n, w, pool[rng.permutation(len(pool))[:n]]))
    return out


def full_rows(name, n):
    return np.unique(np.linspace(0, n - 1, min(n, N_FULL[name.split("_")[0]])).round().astype(np.int64))


def digest(act3):
    return np.array([int.from_bytes(hashlib.blake2b(r.tobytes(), digest_size=8).digest(), "little") for r in act3], np.uint64)


def act3_of(eng, states):
    from tetris_mcts_b200 import _lib as L
    s = np.ascontiguousarray(np.asarray(states, np.int8).reshape(-1, 200))
    out = np.zeros((len(s), 1792), np.float32)
    L.check(L.lib().b200_debug_act3(eng.h, L.ptr(s), len(s), L.ptr(out)))
    return out


def run(eng, w, states):
    """-> (v, var, act3) of net_tc with weights w on the boards"""
    eng.load_weights(w)
    v, var = eng.valuenet(states)
    return v, var, act3_of(eng, states)


def engine(w):
    from tetris_mcts_b200.engine import BatchedEngine
    return BatchedEngine(1, max_nodes=64, eval_kind="net_tc", weights=w)


def main():
    import oracle_py
    oracle_py.build()
    cs = cases(oracle_py)
    eng = engine(cs[0][1])
    rec = {}
    for name, w, s in cs:
        v, var, a = run(eng, w, s)
        rows = full_rows(name, len(s))
        rec.update({name + "/v": v, name + "/var": var, name + "/digest": digest(a), name + "/rows": rows, name + "/act3": a[rows]})
        print("%-24s %5d boards" % (name, len(s)), flush=True)
    eng.close()
    np.savez_compressed(OUT, **rec)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
