"""Pipelined online self-play (play_batched --train_lag) on one GPU; prints one JSON line.

Each run is `play_batched --online` with ValueSimLP on the tensor-core network (eval_kind net_tc), --games games, --sims simulations per
move, --slots arena slots per game and the tf32 trainer (batch 1024, at most --iters steps per training, early stopping), stopped once --k
trainings have been installed into the search.  A first lag-0 run warms up (module loads, first allocations) and is not reported; its
(training time / search time per move) sets two lags around it.  Arms: train_lag 0 (the reference's serial loop) and the two lags with the
search's stream above the training's (OnlineTrainer's default), and the smaller lag with both streams at one priority and with the training
above the search; the arms alternate, --repeats runs each.  Per run: wall time, moves played, games finished, rows stored (what each
collection added to the memory), train_s and wait_s (play_batched's timing), the search's ms per move while a training is in flight and while
none is, and the trainer's ms per optimiser step over its intervals of 100 steps (Trainer.train_rows_dev, one synchronise each;
validation, checkpoints and set-up excluded): those that overlapped no move and those that spent at least a quarter of their time beside one.

The card's name and power limit are read in the same run.  Run from the repository root:
    python scripts/pipeline_bench.py [--games 4096] [--sims 100] [--slots 8192] [--k 8] [--iters 1000] [--repeats 3]
Files that play_batched writes (checkpoint) go to a temporary directory."""
import argparse
import io
import json
import os
import re
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    name, power = [s.strip() for s in q.splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power}


class _Stop(Exception):
    pass


PRIORITIES = {"search_high": (-1, 0), "equal": (0, 0), "train_high": (0, -1)}   # (OnlineTrainer.SEARCH_PRIORITY, TRAIN_PRIORITY)


def one_run(a, lag, priority="search_high"):
    from tetris_mcts_b200 import online
    from tetris_mcts_b200 import play_batched as PB
    from tetris_mcts_b200.engine import BatchedEngine
    from tetris_mcts_b200.model import model_vv as MV
    from tetris_mcts_b200.model.trainer import Trainer
    moves, intervals, trainer, mem = [], [], {}, dict(last=0, stored=0, shrank=0)

    class Timed(BatchedEngine):
        def play_move(self, *args, **kw):
            busy = trainer.get("t") is not None and trainer["t"]._pending is not None and trainer["t"]._pending["thread"].is_alive()
            t0 = time.perf_counter()
            out = super().play_move(*args, **kw)                   # ends in a synchronise of the engine's stream
            moves.append((t0, time.perf_counter(), busy))
            return out

        def replay_policy_step(self, ep):
            train_now, n = super().replay_policy_step(ep)          # n: the memory's rows since the last training
            mem["stored"] += n - mem["last"]
            mem["shrank"] += n < mem["last"]
            mem["last"] = n
            return train_now, n

        def replay_policy_trained(self, ep):
            super().replay_policy_trained(ep)                      # the memory counts from 0 again
            mem["last"] = 0

    class Counting(online.OnlineTrainer):
        def __init__(self, *args, **kw):
            super().__init__(*args, **kw)
            trainer["t"], trainer["installed"] = self, 0

        def install(self):
            done = super().install()
            trainer["installed"] += done
            if trainer["installed"] >= a.k:
                raise _Stop()
            return done

    Counting.SEARCH_PRIORITY, Counting.TRAIN_PRIORITY = PRIORITIES[priority]
    train_rows_dev, base = Trainer.train_rows_dev, online.OnlineTrainer

    def timed_train_rows_dev(self, rows_dev_ptr, n_train_rows, batch, iters, *args, **kw):
        t0 = time.perf_counter()
        log = train_rows_dev(self, rows_dev_ptr, n_train_rows, batch, iters, *args, **kw)    # ends in a synchronise of the trainer's stream
        intervals.append((t0, time.perf_counter(), int(iters)))
        return log

    PB.BatchedEngine, online.OnlineTrainer, Trainer.train_rows_dev = Timed, Counting, timed_train_rows_dev
    quiet = io.StringIO()
    PB.perr, MV.perr = dict(file=quiet, flush=True), dict(file=quiet, flush=True)
    out, timing = io.StringIO(), {}
    argv = ["--agent_type", "ValueSimLP", "--online", "--endless", "--eval_kind", "net_tc", "--train_kind", "tf32", "--n_parallel", str(a.games),
            "--mcts_sims", str(a.sims), "--max_nodes", str(a.slots), "--ngames", "100000000", "--train_max_iters", str(a.iters),
            "--train_lag", str(lag)]
    try:
        try:
            PB.run(PB.parse_args(argv), out=out, timing=timing)
        except _Stop:
            pass
    finally:
        PB.BatchedEngine, online.OnlineTrainer, Trainer.train_rows_dev = BatchedEngine, base, train_rows_dev
    busy = [t1 - t0 for t0, t1, b in moves if b]
    alone = [t1 - t0 for t0, t1, b in moves if not b]

    def beside(a0, a1):                                            # the share of [a0, a1) during which a move was being searched
        return sum(max(0.0, min(a1, t1) - max(a0, t0)) for t0, t1, _b in moves) / (a1 - a0)

    def ms_per_step(sel):
        steps = sum(it for _a0, _a1, it in sel)
        return (round(1e3 * sum(a1 - a0 for a0, a1, _it in sel) / steps, 3) if steps else None), steps
    shares = [(beside(a0, a1), (a0, a1, it)) for a0, a1, it in intervals]
    step_alone, n_alone = ms_per_step([iv for f, iv in shares if f == 0.0])
    step_beside, n_beside = ms_per_step([iv for f, iv in shares if f >= 0.25])
    return dict(lag=lag, priority=priority, wall_s=round(timing["total_s"], 3), moves=timing["moves"],
                games=len(re.findall("Episode:", out.getvalue())), rows_stored=int(mem["stored"]), memory_shrank=int(mem["shrank"]),
                trainings=timing["trainings"], installed=trainer["installed"],
                train_s=round(timing["train_s"], 3), wait_s=round(timing["wait_s"], 3), search_s=round(timing["search_s"], 3),
                search_ms_per_move_training=round(1e3 * float(np.mean(busy)), 2) if busy else None,
                search_ms_per_move_alone=round(1e3 * float(np.mean(alone)), 2) if alone else None,
                moves_during_training=len(busy),
                trainer_ms_per_step_alone=step_alone, steps_alone=n_alone, trainer_ms_per_step_beside_search=step_beside, steps_beside_search=n_beside)


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--games", type=int, default=4096)
    p.add_argument("--sims", type=int, default=100)
    p.add_argument("--slots", type=int, default=8192)
    p.add_argument("--k", type=int, default=8)
    p.add_argument("--iters", type=int, default=1000)
    p.add_argument("--repeats", type=int, default=3)
    p.add_argument("--lags", type=str, default=None, help="two lags, comma-separated (default: from the first lag-0 run)")
    a = p.parse_args()
    info = gpu_info()
    runs = []
    with tempfile.TemporaryDirectory() as d:
        os.chdir(d)
        warm = one_run(a, 0)                                       # module loads, first allocations; not reported
        ratio = (warm["train_s"] / max(warm["trainings"], 1)) / (warm["search_s"] / max(warm["moves"], 1))
        lags = [int(x) for x in a.lags.split(",")] if a.lags else [max(1, int(round(ratio / 2))), max(2, int(round(ratio * 1.5)))]
        arms = [(0, "search_high"), (lags[0], "search_high"), (lags[1], "search_high"), (lags[0], "equal"), (lags[0], "train_high")]
        for _ in range(a.repeats):
            for lag, priority in arms:
                runs.append(one_run(a, lag, priority))
                print(json.dumps(runs[-1]), file=sys.stderr, flush=True)
    summary = {}
    for lag, priority in arms:
        rs = [r for r in runs if (r["lag"], r["priority"]) == (lag, priority)]
        summary["%d %s" % (lag, priority)] = {k: [r[k] for r in rs] for k in rs[0] if k not in ("lag", "priority")}
    print(json.dumps(dict(info, games=a.games, sims=a.sims, slots=a.slots, k=a.k, iters=a.iters, ratio_train_to_move=round(ratio, 2), lags=lags,
                          arms=summary)))


if __name__ == "__main__":
    main()
