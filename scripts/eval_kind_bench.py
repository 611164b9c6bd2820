"""net_tc against net_fp16 at the benchmarked configuration (bench.py's configs[2]: ValueSimLP, 16384 games x 500 simulations per move,
8192 slots per game, head-room 8192 * 5 // 32, overflow_reset, the path cache at its default, init_weights(0)).

  python scripts/eval_kind_bench.py [--runs 3] [--steps 3] [--warmup 2] [--agree_moves 20] [--agree_games 8192]

Speed: the two kinds run alternately, `runs` times each, on a fresh engine per run (the same seeds and games, so the same workload up to the
network's outputs): `warmup` moves, `steps` device-timed moves (CUDA events on the engine stream, as bench.py's `value`), then `steps`
moves with per-phase CUDA-event timing for the conv / fc milliseconds per simulation step and per launch.  The MMA work each kind issues per
board is read from the constants beside the kernels (csrc/valuenet_tc.cuh).

Decision agreement: one engine of each kind on the same games (the first `agree_games` of them: two engines of 16384 x 8192 slots do
not fit in 80 GB together).  Every move both search (run_sims), both report statistics, both play
net_tc's actions (env_step) and re-root (update_root), so the positions stay identical and only the searches differ.  Printed: the fraction
of (game, move) where net_fp16's argmax action is net_tc's, and the median / largest relative difference of the chosen child's value.

The card, its power limit and the SM clock are read with a read-only `nvidia-smi --query-gpu` in the same run.  Output goes to stdout only."""
import argparse
import json
import os
import re
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ENV_ARGS = ((20, 10), 1, 0, 0)
BASE_SEED = 123
KINDS = ("net_tc", "net_fp16")


def mma_flop_per_board():
    """{kind: (conv MFLOP, fc1 MFLOP)} issued per board, from the constants in valuenet_tc.cuh"""
    src = open(os.path.join(ROOT, "tetris_mcts_b200", "csrc", "valuenet_tc.cuh")).read()
    env = {}
    for name, expr in re.findall(r"constexpr int (TC_\w+) = ([^;]+);", src):
        env[name] = eval(expr, {"__builtins__": {}}, dict(env))
    conv = {2: env["TC_CONV_NUNITS_NT2"], 1: env["TC_CONV_NUNITS_NT1"]}
    return {"net_tc": (conv[2] * env["TC_NUNIT_FLOP"] / 1e6, 3 * env["TC_FC_FLOP_PER_PRODUCT"] / 1e6),
            "net_fp16": (conv[1] * env["TC_NUNIT_FLOP"] / 1e6, 1 * env["TC_FC_FLOP_PER_PRODUCT"] / 1e6)}


def gpu_query():
    q = "name,power.limit,clocks.sm,clocks.max.sm,power.draw,temperature.gpu"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0]],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = "nvidia-smi unavailable: %s" % e
    return dict(zip(q.split(","), [s.strip() for s in out.split(",")])) if "," in out else {"nvidia-smi": out}


def fresh_engine(kind, G, M, sims_headroom, recs, weights):
    from tetris_mcts_b200.engine import BatchedEngine
    e = BatchedEngine(G, max_nodes=M, mode="lp", eval_kind=kind, weights=weights, env_args=ENV_ARGS, seed=BASE_SEED,
                      rollout_variance=1e3, overflow_reset=True)
    e.set_games(recs)
    e.set_gc_headroom(sims_headroom)
    return e


def speed_run(kind, args, recs, weights):
    e = fresh_engine(kind, args.games, args.max_nodes, args.max_nodes * 5 // 32, recs, weights)
    for _ in range(args.warmup):
        e.play_move(args.sims, auto_reset=True, want_stats=False)
    e.sync()
    c0 = e.counters()
    e.timer_start()
    for _ in range(args.steps):
        e.play_move(args.sims, auto_reset=True, want_stats=False)
    ms = e.timer_stop()
    c1 = e.counters()
    clk = gpu_query().get("clocks.sm", "?")
    e.set_timing(True)
    for _ in range(args.steps):
        e.play_move(args.sims, auto_reset=True, want_stats=False)
    ph = e.phase_ms()
    e.set_timing(False)
    e.close()
    n_steps = args.steps * args.sims
    (conv_ms, conv_n), (fc_ms, fc_n) = ph["conv"], ph["fc"]
    return {"kind": kind, "msims_per_s": (c1["sims"] - c0["sims"]) / ms / 1e3, "ms_per_move": ms / args.steps,
            "evals_per_move": (c1["eval_requests"] - c0["eval_requests"]) / args.steps,
            "conv_ms_per_step": conv_ms / n_steps, "conv_ms_per_launch": conv_ms / max(conv_n, 1),
            "fc_ms_per_step": fc_ms / n_steps, "fc_ms_per_launch": fc_ms / max(fc_n, 1), "sm_clock_after": clk}


def agreement(args, recs, weights):
    G = args.agree_games
    engs = {k: fresh_engine(k, G, args.max_nodes, args.max_nodes * 5 // 32, recs[:G], weights) for k in KINDS}
    same, rel = [], []
    for _ in range(args.agree_moves):
        st = {}
        for k, e in engs.items():
            e.run_sims(args.sims)
        for k, e in engs.items():
            st[k] = e.get_stats()
        (s_tc, a_tc), (s_16, a_16) = st["net_tc"], st["net_fp16"]
        same.append(a_16 == a_tc)
        g = np.arange(G)
        v_tc, v_16 = s_tc[g, 1, a_tc].astype(np.float64), s_16[g, 1, a_tc].astype(np.float64)
        ok = np.abs(v_tc) > 0
        rel.append(np.abs(v_16[ok] - v_tc[ok]) / np.abs(v_tc[ok]))
        for e in engs.values():
            e.env_step(a_tc)
            e.update_root(auto_reset=True)
    for e in engs.values():
        e.close()
    same, rel = np.concatenate(same), np.concatenate(rel)
    return {"moves": args.agree_moves, "games": G, "argmax_agreement": float(same.mean()),
            "chosen_value_rel_diff_median": float(np.median(rel)), "chosen_value_rel_diff_max": float(rel.max())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--agree_moves", type=int, default=20)
    ap.add_argument("--agree_games", type=int, default=8192)
    ap.add_argument("--games", type=int, default=16384)
    ap.add_argument("--sims", type=int, default=500)
    ap.add_argument("--max_nodes", type=int, default=8192)
    args = ap.parse_args()
    from tetris_mcts_b200 import pyTetris as PT
    from tetris_mcts_b200.model.model_vv import init_weights
    recs = PT.new_games(args.games, ENV_ARGS, np.arange(BASE_SEED, BASE_SEED + args.games, dtype=np.uint32))
    weights = init_weights(0)
    flop = mma_flop_per_board()
    print("gpu:", json.dumps(gpu_query()), flush=True)
    for k in KINDS:
        print("%-8s issued MMA work per board: conv %.2f MFLOP, fc1 %.2f MFLOP" % (k, *flop[k]), flush=True)
    print("warm-up: one short run of each kind", flush=True)
    for k in KINDS:
        speed_run(k, argparse.Namespace(**{**vars(args), "steps": 1, "warmup": 1}), recs, weights)
    res = {k: [] for k in KINDS}
    t0 = time.time()
    for r in range(args.runs):
        for k in (KINDS if r % 2 == 0 else KINDS[::-1]):
            x = speed_run(k, args, recs, weights)
            res[k].append(x)
            print("run %d %-8s %6.2f M sims/s  %7.1f ms/move  conv %.4f ms/step %.4f ms/launch  fc %.4f ms/step %.4f ms/launch  "
                  "(evals/move %.0f, SM clock after %s)" % (r, k, x["msims_per_s"], x["ms_per_move"], x["conv_ms_per_step"],
                                                           x["conv_ms_per_launch"], x["fc_ms_per_step"], x["fc_ms_per_launch"],
                                                           x["evals_per_move"], x["sm_clock_after"]), flush=True)
    med = {k: float(np.median([x["msims_per_s"] for x in res[k]])) for k in KINDS}
    print("median M sims/s: net_tc %.2f, net_fp16 %.2f -> speed-up x%.3f  (%.0f s)" %
          (med["net_tc"], med["net_fp16"], med["net_fp16"] / med["net_tc"], time.time() - t0), flush=True)
    agr = agreement(args, recs, weights)
    print("decision agreement over %d moves x %d games: argmax %.4f, chosen child's value rel. diff median %.3g max %.3g" %
          (agr["moves"], agr["games"], agr["argmax_agreement"], agr["chosen_value_rel_diff_median"], agr["chosen_value_rel_diff_max"]), flush=True)
    print("gpu:", json.dumps(gpu_query()), flush=True)
    print(json.dumps({"median_msims_per_s": med, "speedup": med["net_fp16"] / med["net_tc"], "runs": res, "agreement": agr,
                      "mma_mflop_per_board": flop}), flush=True)


if __name__ == "__main__":
    main()
