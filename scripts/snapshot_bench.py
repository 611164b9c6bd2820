"""Engine images (b200_engine_save / b200_engine_load) at two configurations:
  bench         bench.py's ValueSimLP workload: 16384 games x 8192 slots, head-room 1280, overflow_reset, the path cache on, net_tc,
                500 simulations per move
  play_batched  play_batched --online's defaults: 4096 games x 16384 slots, head-room 16384 * 5 // 32, overflow_reset, the path cache on,
                net_tc, 50 simulations per move, a 500 000-row replay memory under accumulation policy 3

  python scripts/snapshot_bench.py [--warmup 3] [--config bench play_batched] [--dir DIR]

After `warmup` moves: the image's size against the raw arena (every per-slot and per-table byte the engine allocates), the share of free
node and observation slots at that move boundary (read back from the image's game headers), and the seconds of save and load to DIR (default:
a temporary directory), wall clock and split into device pack / D2H / write and read / H2D / device unpack (b200_snapshot_timing).  The
engine is destroyed before the load, so that only one arena exists at a time.  The load reads a file just written: it comes from the page
cache where the host's memory holds it.  The card name and power limit are read with a read-only `nvidia-smi --query-gpu` in the same run."""
import argparse
import json
import os
import shutil
import struct
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CONFIGS = {"bench": dict(n=16384, M=8192, headroom=1280, sims=500, replay=False),
           "play_batched": dict(n=4096, M=16384, headroom=16384 * 5 // 32, sims=50, replay=True)}


def raw_arena_bytes(n, M):
    """row 128 + stat 16 + rec 80 + key 48 + two free lists 8 per slot, two tables of 1.5 M 8-byte entries per game (capi.cu engine_create)"""
    H = max(M + M // 2, 16)
    return n * M * (128 + 16 + 80 + 48 + 8) + n * H * 16


def free_shares(path):
    """(free node slots, free observation slots) / all slots over the image's games, from their headers (snapshot.cuh)"""
    with open(path, "rb") as f:
        data_off = 16
        while True:
            f.seek(data_off)
            fid, _z, nbytes = struct.unpack("<IIQ", f.read(16))
            if fid == 128:
                break
            data_off += 16 + nbytes + 8
        G = struct.unpack("<Q", f.read(8))[0]
        words = np.frombuffer(f.read(8 * G), np.uint64)
        base = data_off + 16 + 8 + 8 * G + 8
        offs = base + 4 * np.concatenate([[0], np.cumsum(words[:-1])]).astype(np.int64)
        nn = no = 0
        for o in offs:
            f.seek(int(o))
            _g, a, b = struct.unpack("<III", f.read(12))
            nn += a
            no += b
    return nn, no, G


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
    except Exception as exc:   # reported, not fatal: the numbers are still printed
        return "unknown (%s)" % exc


def run(name, cfg, warmup, directory):
    import tetris_mcts_b200._lib as L
    from tetris_mcts_b200 import pyTetris as PT
    from tetris_mcts_b200.engine import BatchedEngine
    from tetris_mcts_b200.model.model_vv import init_weights
    n, M = cfg["n"], cfg["M"]
    e = BatchedEngine(n, max_nodes=M, mode="lp", eval_kind="net_tc", weights=init_weights(0), env_args=((20, 10), 1, 0, 0), seed=123,
                      overflow_reset=True, path_cache=True)
    e.set_games(PT.new_games(n, (1, 0, 0), np.arange(123, 123 + n, dtype=np.uint32)))
    e.set_gc_headroom(cfg["headroom"])
    if cfg["replay"]:
        e.replay_enable(min_visits=25, capacity=500000)
        e.replay_policy(3, episodes_per_train=25, memory_growth_rate=5000)
    for _ in range(warmup):
        e.play_move(cfg["sims"], auto_reset=True, want_stats=False)
    e.sync()
    raw = raw_arena_bytes(n, M)
    free = shutil.disk_usage(directory).free
    if free < raw * 1.1:
        e.close()
        return dict(config=name, raw_arena_bytes=raw, image="not measured: %.1f GB free in %s" % (free / 1e9, directory))
    path = os.path.join(directory, "%s.img" % name)
    t0 = time.perf_counter()
    size = e.save(path)
    t_save = time.perf_counter() - t0
    sec = np.zeros(6, np.float64)
    L.check(L.lib().b200_snapshot_timing(L.ptr(sec)))
    e.close()
    nn, no, G = free_shares(path)
    t0 = time.perf_counter()
    b = BatchedEngine.load(path)
    b.sync()
    t_load = time.perf_counter() - t0
    sec2 = np.zeros(6, np.float64)
    L.check(L.lib().b200_snapshot_timing(L.ptr(sec2)))
    b.close()
    os.remove(path)
    return dict(config=name, games=n, max_nodes=M, warmup_moves=warmup, image_bytes=size, raw_arena_bytes=raw, image_over_raw=size / raw,
                free_node_share=nn / (G * M), free_obs_share=no / (G * M), save_s=t_save,
                save_split_s=dict(pack=sec[0], d2h=sec[1], write=sec[2]), load_s=t_load,
                load_split_s=dict(read=sec2[3], h2d=sec2[4], unpack=sec2[5]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--config", nargs="+", default=list(CONFIGS), choices=list(CONFIGS))
    ap.add_argument("--dir", default=None)
    args = ap.parse_args()
    directory = args.dir or tempfile.mkdtemp(prefix="b200_snapshot_")
    print(json.dumps({"card": card()}), flush=True)
    try:
        for name in args.config:
            print(json.dumps(run(name, CONFIGS[name], args.warmup, directory)), flush=True)
    finally:
        if not args.dir:
            shutil.rmtree(directory, ignore_errors=True)


if __name__ == "__main__":
    main()
