"""Online-training throughput on the GPU; prints one JSON line.

(1) Value-network training from device replay rows at batch 512 and 1024: the host loop of Trainer.step_rows_dev (indices drawn on the host,
    three synchronisations per step) against Trainer.train_rows_dev (indices drawn on the device, one synchronisation per call) on the same
    rows and the same indices; ms per iteration, samples/s, and whether both paths end with the same weights.
(2) The search / training time split of a short `play_batched --online` run (ValueSimLP, value network on the tensor-core kernels).

The card's name and power limit are read in the same run.  Run from the repository root:
    python scripts/train_bench.py [--iters 200] [--games 4096] [--moves 40]
Files that play_batched writes (checkpoint, dump) go to a temporary directory."""
import argparse
import io
import json
import os
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


def synthetic_rows(n, seed=0):
    from tetris_mcts_b200 import replay
    rng = np.random.default_rng(seed)
    states = rng.integers(-1, 2, (n, 20, 10))
    filled = (states > 0).sum(axis=(1, 2))
    return replay.memory_to_rows(states, 2.0 * filled + rng.normal(0, 5, n), 10.0 + filled, rng.integers(25, 500, n))


def bench_training(rows_dev, n_rows, batch, iters, warmup):
    from tetris_mcts_b200.model.model_vv import init_weights
    from tetris_mcts_b200.model.trainer import Trainer, sample_indices
    scale, seed = 1.0 / 250.0, 11
    a, b = Trainer(init_weights(0), max_batch=batch), Trainer(init_weights(0), max_batch=batch)
    for t in (a, b):
        t.set_out_ubound(100.0, 400.0)
    idx = [sample_indices(seed, it, batch, n_rows) for it in range(warmup + iters)]
    for it in range(warmup):
        a.step_rows_dev(rows_dev, n_rows, idx[it], scale)
    b.train_rows_dev(rows_dev, n_rows, batch, warmup, seed, 0, scale)
    t0 = time.perf_counter()
    for it in range(warmup, warmup + iters):
        a.step_rows_dev(rows_dev, n_rows, idx[it], scale)                 # each call ends in a stream synchronisation
    t_host = time.perf_counter() - t0
    t0 = time.perf_counter()
    b.train_rows_dev(rows_dev, n_rows, batch, iters, seed, warmup, scale)  # ends in a stream synchronisation
    t_dev = time.perf_counter() - t0
    same = bool(np.array_equal(a.weights(), b.weights()))
    a.close(); b.close()
    return {"batch": batch, "iters": iters,
            "step_rows_dev_ms_per_iter": 1e3 * t_host / iters, "step_rows_dev_samples_per_s": batch * iters / t_host,
            "train_rows_dev_ms_per_iter": 1e3 * t_dev / iters, "train_rows_dev_samples_per_s": batch * iters / t_dev,
            "same_final_weights": same}


def bench_online(games, moves, sims, max_nodes, train_max_iters):
    from tetris_mcts_b200 import play_batched as PB
    here = os.getcwd()
    with tempfile.TemporaryDirectory() as d:
        os.chdir(d)
        try:
            timing = {}
            args = PB.parse_args(["--agent_type", "ValueSimLP", "--online", "--endless", "--n_parallel", str(games), "--ngames", str(10 ** 9),
                                  "--mcts_sims", str(sims), "--max_nodes", str(max_nodes), "--max_moves", str(moves),
                                  "--train_max_iters", str(train_max_iters)])
            PB.run(args, out=io.StringIO(), timing=timing)
        finally:
            os.chdir(here)
    return {"games": games, "sims_per_move": sims, "max_nodes": max_nodes, "train_max_iters": train_max_iters, **timing,
            "train_share": timing["train_s"] / timing["total_s"]}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--iters", type=int, default=200)
    p.add_argument("--warmup", type=int, default=20)
    p.add_argument("--rows", type=int, default=200000)
    p.add_argument("--games", type=int, default=4096)
    p.add_argument("--moves", type=int, default=40)
    p.add_argument("--sims", type=int, default=100)
    p.add_argument("--max_nodes", type=int, default=8192)
    p.add_argument("--train_max_iters", type=int, default=2000)
    a = p.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("train_bench needs a CUDA device")
    from tetris_mcts_b200 import _lib
    _lib.lib()
    out = gpu_info()
    rows = torch.from_numpy(synthetic_rows(a.rows)).cuda()
    torch.cuda.synchronize()
    out["training"] = [bench_training(rows.data_ptr(), a.rows, b, a.iters, a.warmup) for b in (512, 1024)]
    del rows
    torch.cuda.empty_cache()
    out["online"] = bench_online(a.games, a.moves, a.sims, a.max_nodes, a.train_max_iters)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
