"""Online-training throughput on the GPU; prints one JSON line.

(1) Value-network training from device replay rows at batch 512 and 1024: the host loop of Trainer.step_rows_dev (indices drawn on the host,
    three synchronisations per step) against Trainer.train_rows_dev (indices drawn on the device, one synchronisation per call) on the same
    rows and the same indices; ms per iteration, samples/s, and whether both paths end with the same weights.
(2) Trainer kinds (--kinds fp64,tc,tf32): train_rows_dev of each kind in the same process on the same rows and the same device-drawn
    indices, the kinds alternating, --repeats times at each of --kind_batches; ms per step (median, min, max over the repeats), samples/s,
    the algorithmic FLOP/s (the GEMM work of a step, from the layer shapes, the same for every kind), speedup_<b>_over_<a> per repeat for
    each pair of kinds, and the HBM bytes of the explicit im2col buffers per step (fp64 and tc; tf32 has none).
(3) The search / training time split of a short `play_batched --online` run (ValueSimLP, value network on the tensor-core kernels) with
    --train_kind (default: the last of --kinds).

(4) --profile tc,tf32 (a run of its own, nothing else is measured): the per-kernel split of --profile_steps train_rows_dev steps of each
    kind at --profile_batch (default 1024), from torch.profiler's CUDA activities: us per step and share of the step's kernel time.

(5) --validation 2000 (a run of its own): each kind of --kinds trains that many train_rows_dev steps at batch 1024 from the same init on
    the same rows and batches (the first 90 % of the rows), then loss_rows_dev gives the weighted loss on the held-out 10 %.

The card's name and power limit are read in the same run.  Run from the repository root:
    python scripts/train_bench.py [--iters 200] [--kinds fp64,tc,tf32] [--repeats 3] [--games 4096] [--moves 40]
    python scripts/train_bench.py --profile tc,tf32
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


EXPLICIT_IM2COL = ("fp64", "tc")
# the value network's layers as GEMMs per sample: (output pixels, output channels, reduction length)
CONV = ((144, 32, 9), (96, 32, 288), (56, 32, 288))
FC = ((1, 256, 1792), (1, 2, 256))


def step_flops_per_sample():
    """multiply-adds x 2 of one training step per sample: forward, weight gradients (same work as the forward), input gradients of every
    layer but conv1"""
    fwd = sum(2 * p * n * k for p, n, k in CONV + FC)
    dgrad = sum(2 * p * n * k for p, n, k in CONV[1:] + FC)
    return 2 * fwd + dgrad


def im2col_bytes_per_sample():
    """HBM traffic of the explicit im2col buffers per sample and step: each col is written by k_im2col and read by the forward GEMM and
    the weight-gradient GEMM; dcol2 / dcol3 are written by the input-gradient GEMM and read by k_col2im_relu (fp32).  The fp64 and tc
    kinds only (EXPLICIT_IM2COL): the tf32 kind gathers its operands from the activations."""
    col = [4 * p * k for p, _, k in CONV]
    return 3 * sum(col) + 2 * sum(col[1:])


def bench_kinds(rows_dev, n_rows, kinds, batch, iters, warmup, repeats):
    from tetris_mcts_b200.model.model_vv import init_weights
    from tetris_mcts_b200.model.trainer import Trainer
    scale, seed = 1.0 / 250.0, 11
    ts = {k: Trainer(init_weights(0), max_batch=batch, kind=k) for k in kinds}
    times = {k: [] for k in kinds}
    for k, t in ts.items():
        t.set_out_ubound(100.0, 400.0)
        t.train_rows_dev(rows_dev, n_rows, batch, warmup, seed, 0, scale)
    first = warmup
    for _ in range(repeats):
        for k, t in ts.items():                                            # alternating kinds, the same iterations (indices) each
            t0 = time.perf_counter()
            t.train_rows_dev(rows_dev, n_rows, batch, iters, seed, first, scale)       # ends in a stream synchronisation
            times[k].append(1e3 * (time.perf_counter() - t0) / iters)
        first += iters
    for t in ts.values():
        t.close()
    flop, byts = step_flops_per_sample() * batch, im2col_bytes_per_sample() * batch
    out = {"batch": batch, "iters": iters, "repeats": repeats, "step_gflop": flop / 1e9, "im2col_gbytes_per_step": byts / 1e9,
           "im2col_kinds": [k for k in kinds if k in EXPLICIT_IM2COL]}
    for k in kinds:
        ms = np.array(times[k])
        out[k] = {"ms_per_step": [round(float(x), 4) for x in ms], "ms_median": float(np.median(ms)), "ms_min": float(ms.min()),
                  "ms_max": float(ms.max()), "samples_per_s": batch / (float(np.median(ms)) * 1e-3),
                  "algorithmic_tflop_s": flop / (float(np.median(ms)) * 1e-3) / 1e12}
    for i, a in enumerate(kinds):                                          # every pair, the later kind over the earlier one
        for b in kinds[i + 1:]:
            r = np.array(times[a]) / np.array(times[b])
            out["speedup_%s_over_%s" % (b, a)] = {"per_repeat": [round(float(x), 3) for x in r], "min": float(r.min()), "max": float(r.max())}
    return out


def profile_kinds(rows_dev, n_rows, kinds, batch, steps, warmup):
    """per-kernel device time of `steps` train_rows_dev steps of each kind (torch.profiler, CUDA activities) -> {kind: split}"""
    from torch.profiler import ProfilerActivity, profile
    from tetris_mcts_b200.model.model_vv import init_weights
    from tetris_mcts_b200.model.trainer import Trainer
    scale, seed = 1.0 / 250.0, 11
    out = {}
    for k in kinds:
        t = Trainer(init_weights(0), max_batch=batch, kind=k)
        t.set_out_ubound(100.0, 400.0)
        t.train_rows_dev(rows_dev, n_rows, batch, warmup, seed, 0, scale)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            t.train_rows_dev(rows_dev, n_rows, batch, steps, seed, warmup, scale)
        t.close()
        per = {}
        for e in prof.key_averages():
            us = float(getattr(e, "self_device_time_total", 0.0) or 0.0)
            if us <= 0:
                continue
            name = e.key.replace("void ", "").replace("(anonymous namespace)::", "").split("(")[0]
            c = per.setdefault(name, [0.0, 0])
            c[0] += us; c[1] += e.count
        total = sum(v[0] for v in per.values())
        rows = sorted(per.items(), key=lambda kv: -kv[1][0])
        out[k] = {"batch": batch, "steps": steps, "kernel_us_per_step": total / steps,
                  "kernels": [{"name": n, "us_per_step": round(v[0] / steps, 2), "launches_per_step": v[1] / steps,
                               "share": round(v[0] / total, 4)} for n, v in rows]}
    return out


def validation_loss(rows_dev, n_rows, kinds, steps, batch=1024):
    """{kind: held-out weighted loss after `steps` steps on the first 90 % of the rows} (same init, same device-drawn batches)"""
    from tetris_mcts_b200.model.model_vv import init_weights
    from tetris_mcts_b200.model.trainer import Trainer
    n_train = n_rows * 9 // 10
    scale, seed, out = 1.0 / 250.0, 11, {}
    for k in kinds:
        t = Trainer(init_weights(0), max_batch=4096, kind=k)
        mv, mvar, _ = t.rows_stats(rows_dev, n_train)                      # out_ubound from the training rows, as Model_VV.train_data
        t.set_out_ubound(mv, mvar)
        log = t.train_rows_dev(rows_dev, n_train, batch, steps, seed, 0, scale)
        tot, wsum = 0.0, 0.0
        for first in range(n_train, n_rows, 4096):
            loss, _, ws = t.loss_rows_dev(rows_dev, first, min(4096, n_rows - first), scale)
            tot, wsum = tot + loss * ws, wsum + ws
        out[k] = {"steps": steps, "batch": batch, "train_loss_last_20": float(np.mean(log[-20:, 0])), "validation_loss": tot / wsum}
        t.close()
    return out


def bench_online(games, moves, sims, max_nodes, train_max_iters, train_kind="fp64"):
    from tetris_mcts_b200 import play_batched as PB
    here = os.getcwd()
    with tempfile.TemporaryDirectory() as d:
        os.chdir(d)
        try:
            timing = {}
            args = PB.parse_args(["--agent_type", "ValueSimLP", "--online", "--endless", "--n_parallel", str(games), "--ngames", str(10 ** 9),
                                  "--mcts_sims", str(sims), "--max_nodes", str(max_nodes), "--max_moves", str(moves),
                                  "--train_max_iters", str(train_max_iters), "--train_kind", train_kind])
            PB.run(args, out=io.StringIO(), timing=timing)
        finally:
            os.chdir(here)
    return {"games": games, "sims_per_move": sims, "max_nodes": max_nodes, "train_max_iters": train_max_iters, "train_kind": train_kind, **timing,
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
    p.add_argument("--kinds", default="fp64", help="trainer kinds to time side by side, comma-separated (fp64, tc, tf32)")
    p.add_argument("--kind_batches", default="512,1024,4096")
    p.add_argument("--repeats", type=int, default=3)
    p.add_argument("--train_kind", default=None, help="trainer kind of the online run (default: the last of --kinds)")
    p.add_argument("--skip_online", action="store_true")
    p.add_argument("--profile", default=None, help="kinds to profile kernel by kernel, comma-separated (only this is run)")
    p.add_argument("--profile_batch", type=int, default=1024)
    p.add_argument("--profile_steps", type=int, default=20)
    p.add_argument("--validation", type=int, default=0, help="steps of the held-out loss comparison of --kinds (only this is run)")
    a = p.parse_args()
    kinds = [k for k in a.kinds.split(",") if k]
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("train_bench needs a CUDA device")
    from tetris_mcts_b200 import _lib
    _lib.lib()
    out = gpu_info()
    rows = torch.from_numpy(synthetic_rows(a.rows)).cuda()
    torch.cuda.synchronize()
    if a.profile:
        out["profile"] = profile_kinds(rows.data_ptr(), a.rows, [k for k in a.profile.split(",") if k], a.profile_batch, a.profile_steps, a.warmup)
        print(json.dumps(out), flush=True)
        return
    if a.validation:
        out["validation"] = validation_loss(rows.data_ptr(), a.rows, kinds, a.validation)
        print(json.dumps(out), flush=True)
        return
    out["training"] = [bench_training(rows.data_ptr(), a.rows, b, a.iters, a.warmup) for b in (512, 1024)]
    if len(kinds) > 1 or kinds != ["fp64"]:
        out["kinds"] = [bench_kinds(rows.data_ptr(), a.rows, kinds, int(b), a.iters, a.warmup, a.repeats) for b in a.kind_batches.split(",")]
    del rows
    torch.cuda.empty_cache()
    if not a.skip_online:
        out["online"] = bench_online(a.games, a.moves, a.sims, a.max_nodes, a.train_max_iters, a.train_kind or kinds[-1])
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
