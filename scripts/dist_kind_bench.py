"""net_tc against dist_fp16 on the distributional search at BASELINE configs[4]'s per-GPU share (DistValueSimOnline: 2048 games x 1500
simulations per move, 32768 slots per game, head-room 32768 * 5 // 32, overflow_reset, init_dist_weights(0, 50)).

  python scripts/dist_kind_bench.py [--runs 3] [--steps 2] [--warmup 1] [--agree_moves 20] [--agree_games 1024]

Speed: the two kinds run alternately, `runs` times each, on a fresh engine per run (the same seeds and games, so the same workload up to the
network's outputs): `warmup` moves, `steps` device-timed moves (CUDA events on the engine stream), then `steps` moves with per-phase
CUDA-event timing.  From the phase-timed moves: conv / fc milliseconds per launch, and the network's share of a move (conv + fc over the
sum of all phases).  The MMA work each kind issues per board is read from the constants beside the kernels (csrc/distnet_tc.cuh).

Decision agreement: one engine of each kind on the same games (the first `agree_games`: two engines of 2048 x 32768 slots do not fit in
80 GB together).  Every move both search (run_sims), both report statistics, both play net_tc's actions (env_step) and re-root
(update_root), so the positions stay identical and only the searches differ.  Printed: the fraction of (game, move) where dist_fp16's
argmax action is net_tc's, and the median / largest relative difference of the chosen child's value (the mean of its distribution).
The same is measured for `net` (fp32 CUDA cores, within 1e-5 of net_tc) against net_tc as a control: the distributional search samples
its descent, so any difference in an evaluation can change later choices.

The card, its power limit and the SM clock are read with a read-only `nvidia-smi --query-gpu` in the same run.  Output goes to stdout only."""
import argparse
import json
import os
import re
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from eval_kind_bench import gpu_query  # noqa: E402

ENV_ARGS = ((20, 10), 1, 0, 0)
BASE_SEED = 123
ATOMS = 50
KINDS = ("net_tc", "dist_fp16")
CONTROL = ("net_tc", "net")      # the fp32 CUDA-core network, within 1e-5 of net_tc: how far the search alone lets two close evaluators drift


def mma_flop_per_board():
    """{kind: (conv MFLOP, fc1 MFLOP)} issued per board, from the constants in distnet_tc.cuh and valuenet_tc.cuh"""
    env = {}
    for f in ("valuenet_tc.cuh", "distnet_tc.cuh"):
        src = open(os.path.join(ROOT, "tetris_mcts_b200", "csrc", f)).read()
        for name, expr in re.findall(r"constexpr int (T[CD][CF]?_\w+) = ([^;]+);", src):
            try:
                env[name] = eval(expr, {"__builtins__": {}}, dict(env))
            except Exception:
                pass
    return {"net_tc": (env["TDC_CONV_NUNITS_NT2"] * env["TC_NUNIT_FLOP"] / 1e6, 3 * env["TDF_FLOP_PER_PRODUCT"] / 1e6),
            "dist_fp16": (env["TDC_CONV_NUNITS_NT1"] * env["TC_NUNIT_FLOP"] / 1e6, 1 * env["TDF_FLOP_PER_PRODUCT"] / 1e6)}


def fresh_engine(kind, G, M, recs, weights):
    from tetris_mcts_b200.engine import BatchedEngine
    e = BatchedEngine(G, max_nodes=M, mode="dist", eval_kind=kind, dist_weights=weights, dist_bins=ATOMS, env_args=ENV_ARGS,
                      seed=BASE_SEED, overflow_reset=True)
    e.set_games(recs)
    e.set_gc_headroom(M * 5 // 32)
    return e


def speed_run(kind, args, recs, weights):
    e = fresh_engine(kind, args.games, args.max_nodes, recs, weights)
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
    (conv_ms, conv_n), (fc_ms, fc_n) = ph["conv"], ph["fc"]
    total = sum(v[0] for v in ph.values())
    return {"kind": kind, "msims_per_s": (c1["sims"] - c0["sims"]) / ms / 1e3, "ms_per_move": ms / args.steps,
            "evals_per_move": (c1["eval_requests"] - c0["eval_requests"]) / args.steps,
            "conv_ms_per_launch": conv_ms / max(conv_n, 1), "fc_ms_per_launch": fc_ms / max(fc_n, 1),
            "net_ms_per_timed_move": (conv_ms + fc_ms) / args.steps, "phase_ms_per_timed_move": total / args.steps,
            "net_share_of_move": (conv_ms + fc_ms) / total, "phases_ms": {k: v[0] / args.steps for k, v in ph.items()}, "sm_clock_after": clk}


def agreement(args, recs, weights, kinds=KINDS):
    G = args.agree_games
    engs = {k: fresh_engine(k, G, args.max_nodes, recs[:G], weights) for k in kinds}
    same, rel = [], []
    for _ in range(args.agree_moves):
        st = {}
        for k, e in engs.items():
            e.run_sims(args.sims)
        for k, e in engs.items():
            st[k] = e.get_stats()
        (s_tc, a_tc), (s_16, a_16) = st[kinds[0]], st[kinds[1]]
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
    return {"kinds": kinds, "moves": args.agree_moves, "games": G, "argmax_agreement": float(same.mean()),
            "chosen_value_rel_diff_median": float(np.median(rel)), "chosen_value_rel_diff_max": float(rel.max())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--agree_moves", type=int, default=20)
    ap.add_argument("--agree_games", type=int, default=1024)
    ap.add_argument("--games", type=int, default=2048)
    ap.add_argument("--sims", type=int, default=1500)
    ap.add_argument("--max_nodes", type=int, default=32768)
    args = ap.parse_args()
    from tetris_mcts_b200 import pyTetris as PT
    from tetris_mcts_b200.agents.DistValueSimOnline import init_dist_weights
    recs = PT.new_games(args.games, ENV_ARGS, np.arange(BASE_SEED, BASE_SEED + args.games, dtype=np.uint32))
    weights = init_dist_weights(0, ATOMS)
    flop = mma_flop_per_board()
    print("gpu:", json.dumps(gpu_query()), flush=True)
    for k in KINDS:
        print("%-9s issued MMA work per board: conv %.2f MFLOP, fc1 %.2f MFLOP" % (k, *flop[k]), flush=True)
    print("warm-up: one short run of each kind", flush=True)
    for k in KINDS:
        speed_run(k, argparse.Namespace(**{**vars(args), "steps": 1, "warmup": 0}), recs, weights)
    res = {k: [] for k in KINDS}
    t0 = time.time()
    for r in range(args.runs):
        for k in (KINDS if r % 2 == 0 else KINDS[::-1]):
            x = speed_run(k, args, recs, weights)
            res[k].append(x)
            print("run %d %-9s %6.3f M sims/s  %8.1f ms/move  conv %.4f ms/launch  fc %.4f ms/launch  network %.1f of %.1f ms per timed move "
                  "(%.1f %%)  (evals/move %.0f, SM clock after %s)" % (r, k, x["msims_per_s"], x["ms_per_move"], x["conv_ms_per_launch"],
                                                                      x["fc_ms_per_launch"], x["net_ms_per_timed_move"], x["phase_ms_per_timed_move"],
                                                                      100 * x["net_share_of_move"], x["evals_per_move"], x["sm_clock_after"]),
                  flush=True)
    med = {k: float(np.median([x["msims_per_s"] for x in res[k]])) for k in KINDS}
    share = {k: float(np.median([x["net_share_of_move"] for x in res[k]])) for k in KINDS}
    print("median M sims/s: net_tc %.3f, dist_fp16 %.3f -> speed-up x%.3f; network share of a move: net_tc %.1f %%, dist_fp16 %.1f %%  (%.0f s)" %
          (med["net_tc"], med["dist_fp16"], med["dist_fp16"] / med["net_tc"], 100 * share["net_tc"], 100 * share["dist_fp16"], time.time() - t0),
          flush=True)
    agr = [agreement(args, recs, weights, pair) for pair in (KINDS, CONTROL)]
    for a in agr:
        print("decision agreement %s against %s over %d moves x %d games: argmax %.4f, chosen child's value rel. diff median %.3g max %.3g" %
              (a["kinds"][1], a["kinds"][0], a["moves"], a["games"], a["argmax_agreement"], a["chosen_value_rel_diff_median"],
               a["chosen_value_rel_diff_max"]), flush=True)
    print("gpu:", json.dumps(gpu_query()), flush=True)
    print(json.dumps({"median_msims_per_s": med, "speedup": med["dist_fp16"] / med["net_tc"], "net_share_of_move": share, "runs": res,
                      "agreement": agr, "mma_mflop_per_board": flop}), flush=True)


if __name__ == "__main__":
    main()
