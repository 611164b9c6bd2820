"""Data-parallel training cost on the GPU; prints one JSON line per measurement.

(1) world 1: Trainer.grad_rows_dev over the whole batch + apply_grads_dev(n_parts=1) against Trainer.train_rows_dev, the two alternating on
    the same rows and indices, at --batches, both kinds: ms per step.  The difference is the cost of the fp64 gradient vector, the ordered
    sum and the extra launches.
(2) per-rank compute: grad_rows_dev of one slice of batch / R rows, R = 2, 4, 8, timed in one process.  With the exchange left out this is
    what bounds a step on R GPUs.
(3) the ordered sum and the apply for R parts (apply_grads_dev), R = 1, 2, 4, 8.
(4) under torchrun with WORLD_SIZE >= 2 (one GPU per rank, NCCL): the all-gather of one gradient vector per step (ms), and the search /
    training split of a short `play_batched --online` run.  With one process these are reported as not measured.

The card's name and power limit are read in the same run.  Run from the repository root:
    python scripts/dp_train_bench.py [--iters 50] [--repeats 3] [--batches 512,1024,4096]
    torchrun --nproc-per-node 8 scripts/dp_train_bench.py --exchange-only
Files that play_batched writes go to a temporary directory."""
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
    value = rng.uniform(0, 50, n).astype(np.float32)
    variance = rng.uniform(0.1, 30, n).astype(np.float32)
    visit = rng.integers(25, 400, n).astype(np.float32)
    return replay.memory_to_rows(states, value, variance, visit)


def emit(d, info):
    d.update(info)
    print(json.dumps(d), flush=True)


def timed(fn, iters):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn(iters)
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t0) / iters


def single_process(args, info):
    import torch
    from tetris_mcts_b200 import distributed as D
    from tetris_mcts_b200.model.model_vv import init_weights
    from tetris_mcts_b200.model.trainer import GRAD_VEC, Trainer
    n_rows = 50000
    rows = torch.from_numpy(synthetic_rows(n_rows)).cuda()
    torch.cuda.synchronize()
    batches = [int(b) for b in args.batches.split(",")]
    for kind in ("fp64", "tc"):
        for batch in batches:
            ref, dp = (Trainer(init_weights(0), max_batch=batch, kind=kind) for _ in range(2))
            part = torch.empty((8, GRAD_VEC), dtype=torch.float64, device="cuda")

            def run_ref(n, it0=[0]):
                ref.train_rows_dev(rows.data_ptr(), n_rows, batch, n, 1, it0[0], 1.0)
                it0[0] += n

            def run_dp(n, it0=[0]):
                for it in range(n):
                    dp.grad_rows_dev(rows.data_ptr(), n_rows, batch, 0, batch, 1, it0[0] + it, 1.0, part.data_ptr())
                    dp.apply_grads_dev(part.data_ptr(), 1, 0.0, it)
                dp.read_log(n)
                it0[0] += n

            run_ref(3); run_dp(3)                                   # warm-up of every shape
            r_ms, d_ms = [], []
            for _ in range(args.repeats):
                r_ms.append(timed(run_ref, args.iters))
                d_ms.append(timed(run_dp, args.iters))
            same = bool(np.array_equal(ref.weights(), dp.weights()))
            emit({"measure": "world1_slice_vs_train_rows_dev", "kind": kind, "batch": batch, "train_rows_dev_ms": r_ms, "slice_apply_ms": d_ms,
                  "overhead": float(np.median(d_ms) / np.median(r_ms) - 1), "same_weights": same}, info)
            for R in (2, 4, 8):
                lo, hi = D.batch_slice(batch, 0, R)

                def run_slice(n):
                    for it in range(n):
                        dp.grad_rows_dev(rows.data_ptr(), n_rows, batch, lo, hi, 1, it, 1.0, part.data_ptr())
                run_slice(2)
                ms = [timed(run_slice, args.iters) for _ in range(args.repeats)]
                emit({"measure": "per_rank_slice_grad", "kind": kind, "batch": batch, "R": R, "slice": hi - lo, "ms": ms,
                      "bound_speedup_vs_world1": float(np.median(r_ms) / np.median(ms))}, info)
            ref.close(); dp.close()
    t = Trainer(init_weights(0), max_batch=64)
    parts = torch.zeros((8, GRAD_VEC), dtype=torch.float64, device="cuda")
    parts[:, GRAD_VEC - 3] = 1.0
    for R in (1, 2, 4, 8):
        def run_apply(n):
            for it in range(n):
                t.apply_grads_dev(parts.data_ptr(), R, 0.0, it)
            t.read_log(n)
        run_apply(3)
        emit({"measure": "ordered_sum_and_apply", "R": R, "ms": [timed(run_apply, args.iters) for _ in range(args.repeats)]}, info)
    t.close()


def multi_process(args, info):
    import torch
    import torch.distributed as dist
    from tetris_mcts_b200 import distributed as D
    from tetris_mcts_b200 import play_batched as PB
    from tetris_mcts_b200.model.trainer import GRAD_VEC
    rank, local_rank, world = D.init(backend="nccl")
    dev = torch.device("cuda", local_rank)
    stream = torch.cuda.Stream(device=dev)
    local = torch.zeros(GRAD_VEC, dtype=torch.float64, device=dev)
    parts = torch.empty((world, GRAD_VEC), dtype=torch.float64, device=dev)

    def run_x(n):
        for _ in range(n):
            D.allgather_grads(local, parts, stream)
        stream.synchronize()
    run_x(5)
    ms = [timed(run_x, args.iters) for _ in range(args.repeats)]
    if rank == 0:
        emit({"measure": "exchange_allgather_grads", "world": world, "bytes_per_rank": GRAD_VEC * 8, "ms": ms}, info)
    with tempfile.TemporaryDirectory() as tmp:
        cwd = os.getcwd()
        os.chdir(tmp)
        try:
            timing = {}
            PB.run(PB.parse_args(["--agent_type", "ValueSimLP", "--online", "--endless", "--ngames", "1000000", "--n_parallel", str(args.games),
                                  "--max_moves", str(args.moves), "--train_kind", "tc", "--memory_growth_rate", "20000"]),
                   out=io.StringIO(), timing=timing)
        finally:
            os.chdir(cwd)
    if rank == 0:
        emit({"measure": "online_run_split", "world": world, "games": args.games, "moves": args.moves, **timing}, info)
    dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--batches", default="512,1024,4096")
    ap.add_argument("--games", type=int, default=4096, help="games of the --online run over all ranks (torchrun)")
    ap.add_argument("--moves", type=int, default=40)
    ap.add_argument("--exchange-only", action="store_true", help="under torchrun: skip the single-process measurements")
    args = ap.parse_args()
    info = gpu_info()
    from tetris_mcts_b200 import distributed as D
    world = D.env_world()[2]
    if world == 1 or (not args.exchange_only and D.env_world()[0] == 0):
        single_process(args, info)
    if world >= 2:
        multi_process(args, info)
    else:
        emit({"measure": "exchange_allgather_grads", "ms": "not measured (one process; run under torchrun with >= 2 GPUs)"}, info)
        emit({"measure": "online_run_split_multi_gpu", "ms": "not measured (one process; run under torchrun with >= 2 GPUs)"}, info)


if __name__ == "__main__":
    main()
