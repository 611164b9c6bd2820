"""BASELINE configs[4]'s per-GPU share played through play_batched's game loop (--agent_type DistValueSimOnline: 2048 games x 1500
simulations per move, 32768 slots per game, head-room 32768 * 5 // 32, overflow_reset, init_dist_weights(0, 50)), with eval_kind net_tc and
dist_fp16, --save off and on, beside the engine alone (play_move in a plain loop, as scripts/dist_kind_bench.py times it).

  python scripts/dist_play_bench.py [--runs 3] [--moves 3] [--warmup 1]

Every arm runs `runs` times, the arms alternating in rotated order, each run on a fresh engine with the same seeds and games.  A play_batched
run plays `warmup` + `moves` moves (play_batched.run, --max_moves) in a temporary directory; the script wraps BatchedEngine.play_move and
BatchedEngine.dist_root_values (instrumentation only) to take a host timestamp at every move's start, and the time of every root-value read.
A move's time is the wall time from its start to the next move's start, one move more than timed being played (the search, the
statistics, --save's rows and the loop's own work; play_move synchronises the device before it returns), so M sims/s = games * sims / that time, over the moves after the warm-up.  The
root-value read (b200_dist_root_values_dev and the 32 KB copy of [2048, 2] doubles) is timed on the host around a synchronising call.  The
engine-only arm times the same moves with play_move(want_stats=False) between CUDA events on the engine stream (b200_timer_start / stop).

The card, its power limit and the SM clock are read with a read-only `nvidia-smi --query-gpu` in the same run.  Output goes to stdout; the
play_batched runs write only under a temporary directory."""
import argparse
import io
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from eval_kind_bench import gpu_query  # noqa: E402

ENV_ARGS = ((20, 10), 1, 0, 0)
BASE_SEED = 123
ATOMS = 50
ARMS = (("net_tc", "engine"), ("net_tc", "play"), ("net_tc", "play+save"), ("dist_fp16", "engine"), ("dist_fp16", "play"),
        ("dist_fp16", "play+save"))


class Probe:
    """host timestamps of every play_move start and the seconds of every dist_root_values call"""

    def __init__(self):
        from tetris_mcts_b200.engine import BatchedEngine
        self.cls, self.starts, self.reads = BatchedEngine, [], []
        self.play_move, self.root_values = BatchedEngine.play_move, BatchedEngine.dist_root_values
        probe = self

        def play_move(eng, *a, **k):
            probe.starts.append(time.perf_counter())
            return probe.play_move(eng, *a, **k)

        def dist_root_values(eng, *a, **k):
            t = time.perf_counter()
            r = probe.root_values(eng, *a, **k)
            probe.reads.append(time.perf_counter() - t)
            return r
        BatchedEngine.play_move, BatchedEngine.dist_root_values = play_move, dist_root_values

    def close(self):
        self.cls.play_move, self.cls.dist_root_values = self.play_move, self.root_values


def play_run(kind, save, args):
    from tetris_mcts_b200 import play_batched as PB
    argv = ["--agent_type", "DistValueSimOnline", "--n_parallel", str(args.games), "--max_nodes", str(args.max_nodes), "--mcts_sims",
            str(args.sims), "--seed", str(BASE_SEED), "--endless", "--ngames", "100000000", "--eval_kind", kind,
            "--max_moves", str(args.warmup + args.moves + 1)] + (["--save"] if save else [])
    probe = Probe()
    cwd = os.getcwd()
    try:
        with tempfile.TemporaryDirectory() as tmp:
            os.chdir(tmp)
            PB.run(PB.parse_args(argv), out=io.StringIO())
    finally:
        os.chdir(cwd)
        probe.close()
    per_move = np.diff(probe.starts)[args.warmup:]                                  # one more move than timed: its start ends the last
    reads = np.array(probe.reads[args.warmup:args.warmup + args.moves]) if save else np.zeros(0)
    s = float(per_move.mean())
    return {"msims_per_s": args.games * args.sims / s / 1e6, "ms_per_move": 1e3 * s,
            "root_read_ms": float(1e3 * reads.mean()) if len(reads) else None}


def engine_run(kind, args, recs, weights):
    from tetris_mcts_b200.engine import BatchedEngine
    e = BatchedEngine(args.games, max_nodes=args.max_nodes, mode="dist", eval_kind=kind, dist_weights=weights, dist_bins=ATOMS,
                      env_args=ENV_ARGS, seed=BASE_SEED, overflow_reset=True)
    e.set_games(recs)
    e.set_gc_headroom(args.max_nodes * 5 // 32)
    for _ in range(args.warmup):
        e.play_move(args.sims, auto_reset=True, want_stats=False)
    e.sync()
    e.timer_start()
    for _ in range(args.moves):
        e.play_move(args.sims, auto_reset=True, want_stats=False)
    ms = e.timer_stop()
    e.close()
    return {"msims_per_s": args.games * args.sims * args.moves / ms / 1e3, "ms_per_move": ms / args.moves, "root_read_ms": None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--moves", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--games", type=int, default=2048)
    ap.add_argument("--sims", type=int, default=1500)
    ap.add_argument("--max_nodes", type=int, default=32768)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("dist_play_bench measures on a CUDA device; none is visible")
    from tetris_mcts_b200 import pyTetris as PT
    from tetris_mcts_b200.agents.DistValueSimOnline import init_dist_weights
    recs = PT.new_games(args.games, ENV_ARGS, np.arange(BASE_SEED, BASE_SEED + args.games, dtype=np.uint32))
    weights = init_dist_weights(0, ATOMS)
    print("gpu:", json.dumps(gpu_query()), flush=True)
    print("configs[4] per-GPU share: %d games x %d sims/move, %d slots, warm-up %d + %d timed moves per run, %d runs per arm"
          % (args.games, args.sims, args.max_nodes, args.warmup, args.moves, args.runs), flush=True)
    res = {a: [] for a in ARMS}
    t0 = time.time()
    for r in range(args.runs):
        order = ARMS[r % len(ARMS):] + ARMS[:r % len(ARMS)]
        for kind, how in order:
            x = engine_run(kind, args, recs, weights) if how == "engine" else play_run(kind, how == "play+save", args)
            res[(kind, how)].append(x)
            print("run %d %-9s %-9s %6.3f M sims/s  %8.1f ms/move%s" % (r, kind, how, x["msims_per_s"], x["ms_per_move"],
                  "  root-value read %.3f ms" % x["root_read_ms"] if x["root_read_ms"] is not None else ""), flush=True)
    print("\n| kind | loop | M sims/s (runs) | median | ms / move (median) | root-value read, ms / move (median) |", flush=True)
    print("|---|---|---|---|---|---|")
    summary = {}
    for kind, how in ARMS:
        xs = res[(kind, how)]
        rates = [x["msims_per_s"] for x in xs]
        reads = [x["root_read_ms"] for x in xs if x["root_read_ms"] is not None]
        summary["%s/%s" % (kind, how)] = dict(median_msims_per_s=float(np.median(rates)), median_ms_per_move=float(np.median([x["ms_per_move"] for x in xs])),
                                              median_root_read_ms=float(np.median(reads)) if reads else None, runs=xs)
        s = summary["%s/%s" % (kind, how)]
        print("| %s | %s | %s | %.3f | %.1f | %s |" % (kind, how, " / ".join("%.3f" % v for v in rates), s["median_msims_per_s"],
                                                      s["median_ms_per_move"], "%.3f" % s["median_root_read_ms"] if reads else "-"), flush=True)
    print("(%.0f s)" % (time.time() - t0), flush=True)
    print("gpu:", json.dumps(gpu_query()), flush=True)
    print(json.dumps(summary), flush=True)


if __name__ == "__main__":
    main()
