"""The tensor-core value network (net_tc) against its recorded bits (tests/golden/tc_act3_golden.npz, written by
tests/golden/gen_tc_act3.py): act3 and the outputs must be bit-identical, on every weight family, board family and batch size there.
A rewrite of k_tc_conv that changes the order of any product or fp32 sum fails here even when it stays within the float64 bounds of
test_gpu_net_precision.py."""
import importlib.util
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def _gen():
    spec = importlib.util.spec_from_file_location("gen_tc_act3", os.path.join(HERE, "golden", "gen_tc_act3.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


G = _gen()


@pytest.fixture(scope="module")
def golden():
    return np.load(G.OUT)


def first_difference(name, z, v, var, act3):
    """a message naming the first board (and, where its act3 row was recorded, the channel and pixel) that differs; None if none does"""
    dig = G.digest(act3)
    bad = np.nonzero((dig != z[name + "/digest"]) | (v.view(np.uint32) != z[name + "/v"].view(np.uint32)) |
                     (var.view(np.uint32) != z[name + "/var"].view(np.uint32)))[0]
    if len(bad) == 0:
        return None
    b = int(bad[0])
    msg = "%s: %d of %d boards differ; first board %d: v %.9g (want %.9g) var %.9g (want %.9g)" % (
        name, len(bad), len(v), b, v[b], z[name + "/v"][b], var[b], z[name + "/var"][b])
    rows = list(z[name + "/rows"])
    for r in [b] + [r for r in bad[1:] if r in rows][:1]:
        if r in rows:
            want, got = z[name + "/act3"][rows.index(r)], act3[r]
            e = np.nonzero(want.view(np.uint32) != got.view(np.uint32))[0]
            if len(e):
                c, y, x = e[0] // 56, (e[0] % 56) // 4, e[0] % 4
                msg += "; board %d act3 channel %d pixel (y %d, x %d): got %.9g want %.9g (%d elements differ)" % (
                    r, c, y, x, got[e[0]], want[e[0]], len(e))
            break
    return msg


def test_tc_outputs_and_act3_bit_identical(gpu_lib, oracle, golden):
    cs = G.cases(oracle)
    eng = G.engine(cs[0][1])
    fails = []
    for name, w, s in cs:
        v, var, a = G.run(eng, w, s)
        assert len(v) == len(golden[name + "/v"]), name
        m = first_difference(name, golden, v, var, a)
        if m:
            fails.append(m)
    eng.close()
    assert not fails, "\n".join(fails)
