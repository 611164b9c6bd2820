"""Generate tests/golden/select_edges_golden.npz: the reference's own agents/cppmodule/core.cpp (compiled unchanged -> oracle/_ref/core*.so,
oracle/Makefile) searching the designed trees of tests/select_edges.py (select_trace_obs, then the terminal backup, per simulation), with
check_low's rand() on each case's xorshift32 stream (oracle/_ref/librandshim.so preloaded, as gen_golden.py --agent-modes does), then
the reference's own agents/agent.py compute_stats / get_action on the root.  The golden keeps every trace, what each backup changed, the
root statistics and action, the stream's next value and a digest of each case's inputs; the tests regenerate the inputs with
select_edges.design().
Run:  python tests/golden/gen_select_edges.py      (needs `make -C oracle ref`; a regeneration is byte-identical)"""
import ctypes
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")]
import oracle_py as O  # noqa: E402
import select_edges as SE  # noqa: E402

OUT = os.path.join(HERE, "select_edges_golden.npz")
SHIM = os.path.join(ROOT, "oracle", "_ref", "librandshim.so")


def reference_action(c, visit, value, variance):
    """agent.py:153-185 as the reference has it, on a stand-in agent that holds the case's arrays (projection: statistics per observation)."""
    from agents.agent import TreeAgent
    a = types.SimpleNamespace(root=c["root"], n_actions=7, projection=True, node_to_obs=c["n2o"],
                              arrays=dict(child=c["child"], score=c["score"]), obs_arrays=dict(visit=visit, value=value, variance=variance))
    a.compute_stats = types.MethodType(TreeAgent.compute_stats, a)
    action = TreeAgent.get_action(a)
    return a.stats, int(action)


def main():
    shim = ctypes.CDLL(SHIM)
    shim.shim_next.restype = ctypes.c_uint32
    shim.shim_seed.argtypes = [ctypes.c_uint32]
    addr = lambda f: ctypes.cast(f, ctypes.c_void_p).value
    if addr(ctypes.CDLL(None).rand) != addr(shim.rand):
        raise RuntimeError("the reference's rand() must come from oracle/_ref/librandshim.so (LD_PRELOAD)")
    _, core = O.mount_reference()
    cases = SE.design()
    outs = []
    for c in cases:
        traces, states, rng_next = SE.run(c, core, shim.shim_seed, shim.shim_next)
        last = states[-1] if states else (c["visit"], c["value"], c["variance"])
        stats, action = reference_action(c, *last)
        outs.append((traces, states, rng_next, stats, action))
    SE.save(OUT, cases, outs)
    print("select_edges_golden: %d cases, %d simulations" % (len(cases), sum(len(o[0]) for o in outs)))


if __name__ == "__main__":
    if "librandshim" not in os.environ.get("LD_PRELOAD", ""):
        os.environ["LD_PRELOAD"] = SHIM + (":" + os.environ["LD_PRELOAD"] if os.environ.get("LD_PRELOAD") else "")
        os.execv(sys.executable, [sys.executable] + sys.argv)
    main()
