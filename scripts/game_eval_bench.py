"""The caller's leaf-game evaluator (eval_kind "external_game") at BASELINE configs[1]: Vanilla, 4096 games x 300 simulations per move,
8192 slots per game, head-room 8192 * 5 // 32, overflow_reset.

  python scripts/game_eval_bench.py [--runs 3] [--steps 2] [--warmup 1]

Arms, alternating, `runs` times each, a fresh engine per run (same seeds and games): `warmup` moves, then `steps` timed moves.
  rollout     the built-in k_rollout (b200_play_move): random playouts over action ids 0..6, variance 1e3
  playout7    external_game + pyTetris.playout_evaluator(n_actions=7, variance=1e3): the same playout distribution through the split, so the
              difference to `rollout` is the split's own cost (one host synchronisation per step, the compaction, the record gather, the
              scatter) plus the evaluator's torch glue
  heuristic   external_game + a torch heuristic without a playout (score + filled cells): the split with a nearly free evaluator
  vanillac    VanillaC's default: low 1, playout_evaluator(n_actions=8, variance=1e5) (random_playout restated on the device)
Reported per arm: M sims/s, ms per move (host clock around moves that end in a device synchronisation), the evaluator's ms per move (CUDA
events around each call), rows per step, and the split kernels' ms per move (torch.profiler over one more move).  The card name and power
limit are read with a read-only `nvidia-smi --query-gpu` in the same run.  Output goes to stdout only."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.dirname(os.path.abspath(__file__))]
from external_eval_bench import Timed, gpu_query  # noqa: E402

ENV_ARGS = ((20, 10), 1, 0, 0)
BASE_SEED = 123
ARMS = ("rollout", "playout7", "heuristic", "vanillac")
SPLIT_KERNELS = ("k_ext_leaf_order", "k_ext_leaf_records", "k_ext_leaf_scatter", "k_game_playout", "k_rollout")


def heuristic(recs):
    import torch
    v = recs[:, 13].to(torch.float32) + (recs[:, :10] != 0).sum(1).to(torch.float32)
    return v, torch.full_like(v, 1e3)


def run_arm(arm, args, recs):
    from tetris_mcts_b200 import pyTetris as PT
    from tetris_mcts_b200.engine import BatchedEngine
    kind = "synthetic" if arm == "rollout" else "external_game"
    e = BatchedEngine(args.games, max_nodes=args.max_nodes, mode="vanilla", eval_kind=kind, low=1 if arm == "vanillac" else 5,
                      env_args=ENV_ARGS, seed=BASE_SEED, overflow_reset=True)
    e.set_games(recs)
    e.set_gc_headroom(args.max_nodes * 5 // 32)
    ev = None
    if arm == "playout7":
        ev = Timed(PT.playout_evaluator(n_actions=7, variance=1e3, seed=BASE_SEED))
    elif arm == "heuristic":
        ev = Timed(heuristic)
    elif arm == "vanillac":
        ev = Timed(PT.playout_evaluator(n_actions=8, variance=1e5, seed=BASE_SEED))
    for _ in range(args.warmup):
        e.play_move(args.sims, auto_reset=True, want_stats=False, game_evaluator=ev)
    e.sync()
    if ev:
        ev.ms()
    c0 = e.counters()
    t0 = time.perf_counter()
    for _ in range(args.steps):
        e.play_move(args.sims, auto_reset=True, want_stats=False, game_evaluator=ev)
    e.sync()
    ms = (time.perf_counter() - t0) * 1e3
    c1 = e.counters()
    res = {"arm": arm, "msims_per_s": (c1["sims"] - c0["sims"]) / ms / 1e3, "ms_per_move": ms / args.steps,
           "rows_per_step": (c1["eval_requests"] - c0["eval_requests"]) / (args.steps * args.sims),
           "rollout_steps_per_move": (c1["rollout_steps"] - c0["rollout_steps"]) / args.steps}
    if ev:
        res["evaluator_ms_per_move"] = ev.ms() / args.steps
    res.update(kernel_ms(e, args, ev))
    e.close()
    return res


def kernel_ms(e, args, ev):
    """the split's kernels (and k_rollout) over one move, from torch.profiler (CUDA activities), in ms per move"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        e.play_move(args.sims, auto_reset=True, want_stats=False, game_evaluator=ev)
        e.sync()
    if ev:
        ev.ms()
    tot = {k: 0.0 for k in SPLIT_KERNELS}
    for item in prof.key_averages():
        for k in tot:
            if k in item.key:
                tot[k] += item.device_time_total / 1e3
    return {k + "_ms": v for k, v in tot.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--games", type=int, default=4096)
    ap.add_argument("--sims", type=int, default=300)
    ap.add_argument("--max_nodes", type=int, default=8192)
    ap.add_argument("--arms", default=",".join(ARMS))
    args = ap.parse_args()
    from tetris_mcts_b200 import pyTetris as PT
    arms = args.arms.split(",")
    recs = PT.new_games(args.games, ENV_ARGS, np.arange(BASE_SEED, BASE_SEED + args.games, dtype=np.uint32))
    print("gpu:", json.dumps(gpu_query()), flush=True)
    res = {a: [] for a in arms}
    t0 = time.time()
    for r in range(args.runs):
        for a in (arms if r % 2 == 0 else arms[::-1]):
            x = run_arm(a, args, recs)
            res[a].append(x)
            print("run %d %-10s %7.3f M sims/s %9.1f ms/move  rows/step %.0f%s  order %.3f gather %.3f scatter %.3f playout %.1f rollout %.1f ms/move"
                  % (r, a, x["msims_per_s"], x["ms_per_move"], x["rows_per_step"],
                     "" if "evaluator_ms_per_move" not in x else "  evaluator %.1f ms/move" % x["evaluator_ms_per_move"],
                     x["k_ext_leaf_order_ms"], x["k_ext_leaf_records_ms"], x["k_ext_leaf_scatter_ms"], x["k_game_playout_ms"],
                     x["k_rollout_ms"]), flush=True)
    med = {a: {k: float(np.median([x[k] for x in res[a]])) for k in res[a][0] if k != "arm"} for a in arms}
    print("medians (%.0f s):" % (time.time() - t0), flush=True)
    for a in arms:
        print("  %-10s %s" % (a, "  ".join("%s %.3f" % kv for kv in med[a].items())), flush=True)
    print("gpu:", json.dumps(gpu_query()), flush=True)
    print(json.dumps({"median": med, "runs": res}), flush=True)


if __name__ == "__main__":
    main()
