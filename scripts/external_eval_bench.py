"""The caller-supplied evaluator (eval_kind "external") at the benchmarked configuration (scripts/eval_kind_bench.py's setup: ValueSimLP,
16384 games x 500 simulations per move, 8192 slots per game, head-room 8192 * 5 // 32, overflow_reset, the path cache on).

  python scripts/external_eval_bench.py [--runs 3] [--steps 2] [--warmup 1]

Arms, alternating, `runs` times each, a fresh engine per run (same seeds and games): `warmup` moves, then `steps` timed moves.
  net_tc         the built-in tensor-core value network (b200_play_move)
  torch_fp32     external: ValueNet below (Model_VV's architecture, init_weights(0) through weights_to_state_dict), fp32, TF32 off
  torch_bf16     external: the same module under torch.autocast(dtype=torch.bfloat16), outputs cast to fp32
  const          external: a constant evaluator (v = 1, var = 1): the cost of the split step itself (one host synchronisation per
                 simulation step, the ordering, the board gather and the scatter)
  synthetic      the built-in hash evaluator, the reference point of `const`
Reported per arm: M sims/s, ms per move (host clock around moves that end in a device synchronisation), the evaluator's ms per move (CUDA
events around each call, external arms), and the order / gather / scatter kernels' ms per move (torch.profiler over one more move, external
arms).  The card name and power limit are read with a read-only `nvidia-smi --query-gpu` in the same run.  Output goes to stdout only."""
import argparse
import json
import os
import subprocess
import sys
import time
from collections import OrderedDict

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ENV_ARGS = ((20, 10), 1, 0, 0)
BASE_SEED = 123
ARMS = ("net_tc", "torch_fp32", "torch_bf16", "const", "synthetic")


def value_net(weights, device):
    """A torch module of Model_VV's architecture (model/model_vv.py Net: three 3x3 convs with ReLU, fc1 + ReLU, fc_out, sigmoid, then
    x * out_ubound + out_lbound) holding `weights` (the C-ABI weight vector)."""
    import torch
    import torch.nn as nn
    from tetris_mcts_b200.model.model_vv import weights_to_state_dict

    class Net(nn.Module):
        def __init__(self):
            super().__init__()
            self.head = nn.Sequential(OrderedDict([
                ("conv1", nn.Conv2d(1, 32, 3)), ("act1", nn.ReLU()), ("conv2", nn.Conv2d(32, 32, 3)), ("act2", nn.ReLU()),
                ("conv3", nn.Conv2d(32, 32, 3)), ("act3", nn.ReLU()), ("flatten", nn.Flatten()), ("fc1", nn.Linear(1792, 256)),
                ("fc_act1", nn.ReLU()), ("fc_out", nn.Linear(256, 2)), ("act_out", nn.Sigmoid())]))
            self.out_ubound = nn.Parameter(torch.zeros(2), requires_grad=False)
            self.out_lbound = nn.Parameter(torch.zeros(2), requires_grad=False)

        def forward(self, x):
            return self.head(x) * self.out_ubound + self.out_lbound

    net = Net()
    net.load_state_dict(weights_to_state_dict(weights))
    return net.to(device).eval()


def module_evaluator(net, bf16=False):
    """A device evaluator around `net`: boards [n,1,20,10] float32 -> (v, var), each [n] float32"""
    import torch

    def ev(boards):
        with torch.no_grad():
            if bf16:
                with torch.autocast("cuda", dtype=torch.bfloat16):
                    out = net(boards)
            else:
                out = net(boards)
        out = out.float()
        return out[:, 0], out[:, 1]
    return ev


def const_evaluator(boards):
    import torch
    one = torch.ones(boards.shape[0], dtype=torch.float32, device=boards.device)
    return one, one


def gpu_query():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0]],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = "nvidia-smi unavailable: %s" % e
    return dict(zip(q.split(","), [s.strip() for s in out.split(",")])) if "," in out else {"nvidia-smi": out}


class Timed:
    """CUDA events around every call of a device evaluator (recorded on the engine's stream, which is current inside the call)"""

    def __init__(self, fn):
        self.fn, self.events = fn, []

    def __call__(self, boards):
        import torch
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = self.fn(boards)
        b.record()
        self.events.append((a, b))
        return out

    def ms(self):
        import torch
        torch.cuda.synchronize()
        t = sum(a.elapsed_time(b) for a, b in self.events)
        self.events = []
        return t


def run_arm(arm, args, recs, weights, net):
    from tetris_mcts_b200.engine import BatchedEngine
    external = arm in ("torch_fp32", "torch_bf16", "const")
    kind = "external" if external else arm
    e = BatchedEngine(args.games, max_nodes=args.max_nodes, mode="lp", eval_kind=kind, weights=None if external or arm == "synthetic" else weights,
                      env_args=ENV_ARGS, seed=BASE_SEED, overflow_reset=True, path_cache=True)
    e.set_games(recs)
    e.set_gc_headroom(args.max_nodes * 5 // 32)
    ev = None
    if external:
        ev = Timed(const_evaluator if arm == "const" else module_evaluator(net, bf16=arm == "torch_bf16"))
    for _ in range(args.warmup):
        e.play_move(args.sims, auto_reset=True, want_stats=False, evaluator=ev)
    e.sync()
    if ev:
        ev.ms()
    c0 = e.counters()
    t0 = time.perf_counter()
    for _ in range(args.steps):
        e.play_move(args.sims, auto_reset=True, want_stats=False, evaluator=ev)
    e.sync()
    ms = (time.perf_counter() - t0) * 1e3
    c1 = e.counters()
    res = {"arm": arm, "msims_per_s": (c1["sims"] - c0["sims"]) / ms / 1e3, "ms_per_move": ms / args.steps,
           "evals_per_move": (c1["eval_requests"] - c0["eval_requests"]) / args.steps}
    if ev:
        res["evaluator_ms_per_move"] = ev.ms() / args.steps
        res.update(kernel_ms(e, args, ev))
    e.close()
    return res


def kernel_ms(e, args, ev):
    """the split's own kernels over one move, from torch.profiler (CUDA activities), in ms per move"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        e.play_move(args.sims, auto_reset=True, want_stats=False, evaluator=ev)
        e.sync()
    ev.ms()
    tot = {"k_ext_order": 0.0, "k_ext_boards": 0.0, "k_ext_scatter": 0.0}
    for item in prof.key_averages():
        for k in tot:
            if k in item.key:
                tot[k] += item.device_time_total / 1e3
    return {k + "_ms_per_move": v for k, v in tot.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--games", type=int, default=16384)
    ap.add_argument("--sims", type=int, default=500)
    ap.add_argument("--max_nodes", type=int, default=8192)
    ap.add_argument("--arms", default=",".join(ARMS))
    args = ap.parse_args()
    import torch
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    from tetris_mcts_b200 import pyTetris as PT
    from tetris_mcts_b200.model.model_vv import init_weights
    arms = args.arms.split(",")
    recs = PT.new_games(args.games, ENV_ARGS, np.arange(BASE_SEED, BASE_SEED + args.games, dtype=np.uint32))
    weights = init_weights(0)
    net = value_net(weights, torch.device("cuda", 0))
    print("gpu:", json.dumps(gpu_query()), flush=True)
    res = {a: [] for a in arms}
    t0 = time.time()
    for r in range(args.runs):
        for a in (arms if r % 2 == 0 else arms[::-1]):
            x = run_arm(a, args, recs, weights, net)
            res[a].append(x)
            print("run %d %-10s %7.3f M sims/s %9.1f ms/move  evals/move %.0f%s" % (
                r, a, x["msims_per_s"], x["ms_per_move"], x["evals_per_move"],
                "" if "evaluator_ms_per_move" not in x else "  evaluator %.1f ms/move  order %.2f  gather %.2f  scatter %.2f ms/move" % (
                    x["evaluator_ms_per_move"], x["k_ext_order_ms_per_move"], x["k_ext_boards_ms_per_move"], x["k_ext_scatter_ms_per_move"])),
                flush=True)
    med = {a: {k: float(np.median([x[k] for x in res[a]])) for k in res[a][0] if k != "arm"} for a in arms}
    print("medians (%.0f s):" % (time.time() - t0), flush=True)
    for a in arms:
        print("  %-10s %s" % (a, "  ".join("%s %.3f" % kv for kv in med[a].items())), flush=True)
    print("gpu:", json.dumps(gpu_query()), flush=True)
    print(json.dumps({"median": med, "runs": res}), flush=True)


if __name__ == "__main__":
    main()
