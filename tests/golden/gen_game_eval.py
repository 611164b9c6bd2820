"""Generate tests/golden/agent_type1_golden.npz by running the reference's OWN agents/cppmodule/agent.cpp (compiled unchanged ->
oracle/_ref/agent*.so) as MCTSAgent(sims, max_nodes, True, gamma, True, f, 1, False): the C++ agent with evaluator type 1, which hands a
copy of each expanded leaf game to f and backs (value, variance) up as they are (agent.cpp:449-455).  f is tests/game_eval_twins.evaluate on
the game's packed record, the evaluator the oracle and the engine are fed in the tests.  check_low's rand() draws from the xorshift32 stream
the engine gives game 0 of an engine seeded `engine_seed` (oracle/_ref/librandshim.so preloaded; the process re-executes itself so).

Pinned per move: the action, the game record after the move, and every record handed to f (in call order), so every simulation's walk is
pinned.  max_nodes is large enough that the reference's remove_nodes (SURVEY N2) never runs.
Run:  python tests/golden/gen_game_eval.py      (needs /root/reference and `make -C oracle`)"""
import ctypes
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")]
import oracle_py as O  # noqa: E402
from game_eval_twins import evaluate  # noqa: E402

# env_args = (actions_per_drop, scoring, randomizer); special: NaN / +-inf / negative outputs on a designed share of the leaves
CASES = [dict(name="vanillac", sims=30, moves=150, gamma=0.99, env=(1, 0, 0), seed=123, engine_seed=7, special=False),
         dict(name="gamma1", sims=20, moves=60, gamma=1.0, env=(1, 0, 0), seed=55, engine_seed=11, special=False),
         dict(name="env", sims=25, moves=60, gamma=0.99, env=(2, 1, 1), seed=9, engine_seed=3, special=False),
         dict(name="special", sims=25, moves=60, gamma=0.99, env=(1, 0, 0), seed=77, engine_seed=5, special=True)]
MAX_NODES = 100000


def stream_of_game0(engine_seed):
    """k_init_arena: game g's check_low stream starts at seed + 0x9E3779B9 * (g + 1) (0 -> 0x2545F491)"""
    s = (engine_seed + 0x9E3779B9) & 0xffffffff
    return s or 0x2545F491


def main():
    shim = ctypes.CDLL(os.path.join(ROOT, "oracle", "_ref", "librandshim.so"))
    shim.shim_seed.argtypes = [ctypes.c_uint32]
    if "librandshim" not in os.environ.get("LD_PRELOAD", ""):
        raise RuntimeError("run with LD_PRELOAD=oracle/_ref/librandshim.so (the script re-executes itself that way)")
    pt, _core = O.mount_reference()
    agent_mod = O.load_ref_module("agent")
    out = {"max_nodes": MAX_NODES, "n_cases": len(CASES)}
    for i, cs in enumerate(CASES):
        p = "c%d_" % i
        seen = []

        def f(game):                                       # agent.cpp:451-454: f(Tetris) -> [value, variance]
            rec = np.array(game.get_record(), np.uint32)
            seen.append(rec)
            v, var = evaluate(rec, cs["special"])
            return [v, var]

        game = pt.Tetris((20, 10), *cs["env"])
        game.seed(cs["seed"])
        shim.shim_seed(stream_of_game0(cs["engine_seed"]))
        ag = agent_mod.MCTSAgent(cs["sims"], MAX_NODES, True, cs["gamma"], True, f, 1, False)
        out[p + "start"] = np.array(game.get_record(), np.uint32)
        ag.update_root(game)
        acts, recs, calls, resets = [], [], [0], 0
        for mv in range(cs["moves"]):
            a = ag.play()
            acts.append(int(a))
            calls.append(len(seen))
            game.play(a)
            ag.update_root(game)
            if game.end:
                game.reset()
                ag.update_root(game)
                resets += 1
            recs.append(np.array(game.get_record(), np.uint32))
        for k in ("sims", "gamma", "engine_seed", "special"):
            out[p + k] = cs[k]
        out[p + "env"] = np.array(cs["env"], np.int32)
        out[p + "actions"], out[p + "records"] = np.array(acts, np.int32), np.stack(recs)
        out[p + "eval_off"], out[p + "eval_recs"] = np.array(calls, np.int64), np.stack(seen)
        out[p + "resets"] = resets
        print("%s: %d moves, %d evaluations, %d game overs" % (cs["name"], cs["moves"], len(seen), resets))
    np.savez_compressed(os.path.join(HERE, "agent_type1_golden.npz"), **out)


if __name__ == "__main__":
    O.build(ref=True)
    shim_path = os.path.join(ROOT, "oracle", "_ref", "librandshim.so")
    if "librandshim" not in os.environ.get("LD_PRELOAD", ""):
        os.environ["LD_PRELOAD"] = shim_path + (":" + os.environ["LD_PRELOAD"] if os.environ.get("LD_PRELOAD") else "")
        os.execv(sys.executable, [sys.executable] + sys.argv)
    main()
