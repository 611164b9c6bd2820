"""play_batched.py — the game loop of the reference's play.py (play.py:115-181) for N games at once on the CUDA engine, emitting the
reference's own log / status wire formats (SURVEY §8f.4) so that web/parseLog.py and the dashboards keep working on batched runs:

  stdout  `Episode: {:>5} Score: {:>10} Lines Cleared: {:>10}`                      play.py:164 (--endless), parsed by web/parseLog.py:58-60
          `\rGames played:{:>3}    min/max/mean/std:...`                             play.py:26-37 (ScoreTracker.printStats, default mode)
  tmp/    board int8[20,10], combo int32[1], score int32[1], lines int32[1],        play.py:109-114 written every move play.py:143-148,
          line_stats int32[4] as numpy memmaps (--realtime_status)                   read by web/parseLog.py:34-38 (StatusParser)
  stderr  `Memory usage: a / b` after each move with a collection (--online)        agent.cpp:632 / parseLog.py:67 (queue_re)
          Model.train_data's `Training data size` / `Iteration:` lines when it trains  model/model.py:202,236, parseLog.py:61-66

--online closes the reference's self-play loop (OnlineMCTSAgent::remove_nodes, agent.cpp:619-708): the engine's collections store rows in the
device replay memory, the accumulation policy decides after each move whether to train, and the value network is then trained on the device
rows (Model_VV.train_rows), saved to ./pytorch_model/model_checkpoint and swapped into the running search.

  python -m tetris_mcts_b200.play_batched --agent_type ValueSimLP --mcts_sims 100 --ngames 1000 --n_parallel 4096 --endless
  torchrun --nproc-per-node 8 -m tetris_mcts_b200.play_batched --agent_type ValueSimLP --online --n_parallel 32768 --endless
  python -m tetris_mcts_b200.play_batched --agent_type ValueSimLP --evaluator mynets:make_evaluator --n_parallel 4096 --endless

--evaluator MODULE:FACTORY searches with the caller's network instead of the built-in one: FACTORY(device) returns a device evaluator
(BatchedEngine.run_sims: a torch tensor [n,1,20,10] of boards in, (v, var) out), and the engine runs eval_kind "external".

Flags are play.py's (play.py:46-70) plus --n_parallel / --max_nodes / --device / --watch / --seed and the online agent's memory and training
settings.  One "episode" is one finished game of any of the parallel games; episodes are numbered in the order (move, game index) they end."""
import argparse
import os
import sys
import time
from sys import stderr

import numpy as np

from . import pyTetris as PT
from .engine import BatchedEngine

perr = dict(file=stderr, flush=True)
EPISODE_FMT = 'Episode: {:>5} Score: {:>10} Lines Cleared: {:>10}'          # play.py:164
MODES = {"ValueSimLP": ("lp", 0.999, 1), "ValueSim": ("single", 0.999, 1), "Vanilla": ("vanilla", 0.99, 5)}


class ScoreTracker:                                                          # play.py:9-41
    def __init__(self):
        self.scores, self.lines = [], []

    def append(self, score, line):
        self.scores.append(score)
        self.lines.append(line)

    def printStats(self, file=sys.stdout):
        print('\rGames played:{:>3}    min/max/mean/std:{:5.2f}({:5.2f})/{:5.2f}'
              '({:5.2f})/{:5.2f}({:5.2f})/{:5.2f}({:5.2f})'.format(
                  len(self.scores), np.amin(self.scores), np.amin(self.lines), np.amax(self.scores), np.amax(self.lines),
                  np.mean(self.scores), np.mean(self.lines), np.std(self.scores), np.std(self.lines)), end='', flush=True, file=file)


class RealtimeStatus:
    """The five memmaps of play.py:109-114, refreshed from one watched game before every move (play.py:143-148)."""

    def __init__(self, directory='./tmp'):
        os.makedirs(directory, exist_ok=True)
        mm = lambda name, dtype, shape: np.memmap(os.path.join(directory, name), dtype=dtype, mode='w+', shape=shape)   # noqa: E731
        self.board, self.combo = mm('board', np.int8, (20, 10)), mm('combo', np.int32, (1,))
        self.score, self.lines, self.line_stats = mm('score', np.int32, (1,)), mm('lines', np.int32, (1,)), mm('line_stats', np.int32, (4,))

    def update(self, rec):
        g = PT.Tetris((20, 10), _record=rec)
        self.board[:] = g.getState()[:]
        self.combo[:] = g.combo
        self.lines[:] = g.line_clears
        self.score[:] = g.score
        self.line_stats[:] = g.line_stats[:]
        for m in (self.board, self.combo, self.score, self.lines, self.line_stats):
            m.flush()


def merge_finished(per_rank):
    """the games one move finished on every rank, [(global game, score, lines), ...] per rank -> one list in global game order, the order
    rank 0 numbers their episodes in (as one engine holding all games returns them)"""
    return sorted((f for fin in per_rank for f in fin), key=lambda f: f[0])


def save_suffix(rank, world):
    """--save under torchrun writes one file per rank: the single-process name, suffixed with the rank"""
    return "" if world == 1 else ".rank%d" % rank


def run(args, out=sys.stdout, timing=None):
    """timing: a dict, filled with moves, trainings and the wall-clock seconds of the run split into search (everything but training) and
    training (--online).

    Under a torch.distributed process group (main() under torchrun) rank r plays the games shard_range(n_parallel, r, world) on device
    LOCAL_RANK, with the piece seeds and search streams of their global indices, so every game plays as in a single-process run.  Finished
    games are all-gathered every move; rank 0 numbers the episodes and alone prints.  --online: rank 0's engine holds the replay memory and the
    accumulation policy; the other ranks' memories stage the rows of one move, which rank 0 appends in rank order; training is data-parallel
    over all ranks (Model_VV.train_rows)."""
    from . import distributed as D
    rank, world = D.rank_world()
    lo, hi = D.shard_range(args.n_parallel, rank, world)
    device = args.device if world == 1 else D.env_world()[1]
    mode, gamma, low = MODES[args.agent_type]
    env_args = ((20, 10), args.app, args.tetris_scoring, args.tetris_randomizer)           # play.py:75
    weights, evaluator = None, None
    if args.evaluator:
        import importlib
        import torch
        module, factory = args.evaluator.split(":", 1)
        evaluator = getattr(importlib.import_module(module), factory)(torch.device("cuda", device))
    elif mode != "vanilla":
        from .model.model_vv import init_weights, load_checkpoint_weights
        if rank == 0:
            weights = load_checkpoint_weights()                                             # agents/ValueSim.py:42-44
        else:                                                                               # the same file, without its message
            import contextlib
            with open(os.devnull, "w") as quiet, contextlib.redirect_stdout(quiet):
                weights = load_checkpoint_weights()
        if weights is None:
            weights = init_weights(0)
    # k_init_arena seeds game g's search stream with seed + 0x9E3779B9 * (g + 1): offset by the shard's first global index
    eng = BatchedEngine(hi - lo, max_nodes=args.max_nodes, mode=mode, gamma=gamma, low=low,
                        eval_kind="external" if evaluator else (args.eval_kind if mode != "vanilla" else "synthetic"), weights=weights, env_args=env_args,
                        seed=(args.seed + 0x9E3779B9 * lo) & 0xFFFFFFFF, device=device, overflow_reset=True)
    eng.set_games(PT.new_games(hi - lo, env_args, D.shard_seeds(args.seed, args.n_parallel, rank, world)))
    eng.set_gc_headroom(args.max_nodes * 5 // 32)
    online = args.online and not args.benchmark and mode != "vanilla"
    trainer, gcs, block = None, 0, None
    if online:                                                                             # ValueSim.py:21-37 memory, min_visits_to_store (25: ValueSimLP.py:11)
        from .online import OnlineTrainer
        eng.replay_enable(min_visits=25 if mode == "lp" else 10, capacity=args.memory_size)
        if rank == 0:
            eng.replay_policy(args.accumulation_policy, episodes_per_train=args.episodes_per_train, memory_growth_rate=args.memory_growth_rate)
        trainer = OnlineTrainer(eng, weights, args.memory_size, batch_size=args.train_batch_size, max_iters=args.train_max_iters,
                                train_kind=args.train_kind)   # ValueSim.py:180
        if world > 1:                                                                      # the rows one move's collections stored on this rank
            import torch
            block = torch.empty((args.memory_size, D.SAMPLE_BYTES), dtype=torch.uint8, device=trainer.buf.device)
    status = RealtimeStatus(args.status_dir) if args.realtime_status and (world == 1 or lo <= args.watch < hi) else None   # the watched game's owner
    saver = None
    if args.save:                                                                          # play.py:93-94, 131-132
        from .data import DataSaver, rows_from_move
        saver = DataSaver(args.save_dir, args.save_file, args.cycle, suffix=save_suffix(rank, world))
        episode_of = np.zeros(hi - lo, np.int32)                                           # play.py passes ngames: the episode a row belongs to
    tracker = ScoreTracker()
    ngames, moves = 0, 0
    t_start = time.perf_counter()
    try:
        while True:
            if status:
                status.update(eng.get_games()[args.watch - lo])
            before = eng.get_games() if saver else None
            actions, stats = eng.play_move(args.mcts_sims, auto_reset=True, want_stats=saver is not None,
                                           evaluator=evaluator)   # agent.play(); game.play(action); agent.update_root(game); reset
            if saver:
                saver.add_rows(rows_from_move(before, actions, stats, args.cycle, episode_of))
            moves += 1
            collected = online and eng.counters()["gcs"] != gcs                                # collections stored rows this move
            if collected:
                gcs = eng.counters()["gcs"]
            finished = [(g + lo, score, lines) for g, score, lines, _ep in eng.finished_games()]
            if world > 1:
                staged = eng.replay_drain_into(block.data_ptr(), args.memory_size) if collected and rank != 0 else 0
                moved = D.gather_objects((finished, collected, staged))
                finished = merge_finished([m[0] for m in moved])
                collected = any(m[1] for m in moved)
                if max(m[2] for m in moved) > 0:
                    _exchange_rows(eng, block, staged, max(m[2] for m in moved), rank)
            done = False
            for g, score, lines in finished:
                ngames += 1
                if saver and lo <= g < hi:
                    episode_of[g - lo] = ngames
                if rank == 0:
                    if args.endless:
                        print(EPISODE_FMT.format(ngames, int(score), int(lines)), flush=True, file=out)
                    else:
                        tracker.append(int(score), int(lines))
                        tracker.printStats(file=out)
                if ngames >= args.ngames:
                    done = True
                    break
            if collected:
                train_now, n = False, 0
                if rank == 0:
                    train_now, n = eng.replay_policy_step(ngames)                               # current_episode = finished games (all ranks)
                    print('Memory usage: {} / {}'.format(n, args.memory_size), **perr)        # agent.cpp:632
                if world > 1:
                    train_now, n = D.broadcast_ints([train_now, n])
                if train_now:
                    trainer.train(n, ngames)
            if done or (args.max_moves and moves >= args.max_moves):
                break
    finally:
        if rank == 0:
            print(flush=True, file=out)                                                     # play.py:179
        if timing is not None:
            total = time.perf_counter() - t_start
            timing.update(moves=moves, total_s=total, train_s=trainer.train_seconds if trainer else 0.0, trainings=trainer.n_trains if trainer else 0)
            timing["search_s"] = total - timing["train_s"]
        if trainer:
            trainer.close()
        eng.close()                                                                         # play.py:181
        if saver:
            saver.close()                                                                   # play.py:183-184
    return ngames, moves, tracker


def _exchange_rows(eng, block, staged, most, rank):
    """All-gather the rows the ranks staged this move (`most` rows at most per rank); rank 0 appends those of ranks 1.. in rank order to its
    memory, as its own collections would have stored them."""
    import torch
    from . import distributed as D
    part = block[:most] if D.on_device() else block[:most].cpu()
    rows, _counts = D.allgather_samples(part, staged)
    if rank == 0 and len(rows):
        rows = rows.to(block.device)
        torch.cuda.current_stream(block.device).synchronize()                           # the engine copies on its own stream
        eng.replay_append_dev(rows.data_ptr(), len(rows))


def parse_args(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument('--agent_type', default='ValueSimLP', choices=sorted(MODES))
    p.add_argument('--app', default=1, type=int)
    p.add_argument('--benchmark', default=False, action='store_true')
    p.add_argument('--endless', default=False, action='store_true')
    p.add_argument('--mcts_sims', default=50, type=int)
    p.add_argument('--ngames', default=50, type=int)
    p.add_argument('--online', default=False, action='store_true')
    p.add_argument('--realtime_status', default=False, action='store_true')
    p.add_argument('--save', default=False, action='store_true')
    p.add_argument('--save_dir', default='./data/', type=str)
    p.add_argument('--save_file', default='data', type=str)
    p.add_argument('--cycle', default=0, type=int)
    p.add_argument('--tetris_randomizer', default=0, type=int)
    p.add_argument('--tetris_scoring', default=0, type=int)
    p.add_argument('--n_parallel', default=4096, type=int, help='concurrent games on the device')
    p.add_argument('--max_nodes', default=16384, type=int)
    p.add_argument('--device', default=0, type=int)
    p.add_argument('--seed', default=123, type=int)
    p.add_argument('--watch', default=0, type=int, help='game whose status goes to the realtime memmaps')
    p.add_argument('--status_dir', default='./tmp')
    p.add_argument('--memory_size', default=500000, type=int)
    p.add_argument('--accumulation_policy', default=3, type=int, choices=(0, 1, 2, 3),
                   help='when to train (agent.cpp:619-708); 3 = ValueSim.train_nodes: memory_index >= min(n_trains * memory_growth_rate, memory_size)')
    p.add_argument('--episodes_per_train', default=25, type=int, help='finished games between trainings (policies 0-2)')
    p.add_argument('--memory_growth_rate', default=5000, type=int, help='rows the training threshold grows by per training (policy 3)')
    p.add_argument('--train_batch_size', default=1024, type=int, help='training batch size (--online)')
    p.add_argument('--train_max_iters', default=50000, type=int, help='most optimiser steps per training (--online; early stopping usually ends it)')
    p.add_argument('--train_kind', default='fp64', choices=('fp64', 'tc', 'tf32'),
                   help='trainer GEMMs (--online): fp64 CUDA cores, tc = Hopper tensor cores with the 3xTF32 split, or tf32 = one tf32 '
                        'term per operand with implicit-im2col convolutions (fastest, ~1e-3 of float64)')
    p.add_argument('--eval_kind', default='net_tc', choices=('net_tc', 'net_fp16'),
                   help='value network of the search (not Vanilla): net_tc = tensor cores within 1e-5 of fp32, net_fp16 = one fp16 product per '
                        'product, about a third of the tensor-core work (DESIGN §5).  --online trains in fp32 / fp64 either way')
    p.add_argument('--evaluator', default=None, metavar='MODULE:FACTORY',
                   help='search with the caller\'s network: FACTORY(device) returns a device evaluator (boards [n,1,20,10] -> (v, var)); '
                        'the engine runs eval_kind external.  Not with --online (the trainer trains the built-in network) nor Vanilla')
    p.add_argument('--max_moves', default=0, type=int)
    p.add_argument('--dist_backend', default='nccl', choices=('nccl', 'gloo'),
                   help='under torchrun: collectives over NCCL (one GPU per rank), or gloo through the host (several ranks may share a GPU)')
    args = p.parse_args(argv)
    if args.evaluator and args.online:
        p.error('--evaluator cannot be combined with --online: the online trainer trains the built-in Model_VV weights')
    if args.evaluator and args.agent_type == 'Vanilla':
        p.error('--evaluator cannot be combined with --agent_type Vanilla: Vanilla evaluates leaves by random rollout')
    if args.evaluator and ':' not in args.evaluator:
        p.error('--evaluator takes MODULE:FACTORY')
    return args


def main(argv=None, out=sys.stdout):
    """Under torchrun (WORLD_SIZE > 1) one process per rank joins a process group first."""
    from . import distributed as D
    args = parse_args(argv)
    if D.env_world()[2] == 1:
        return run(args, out=out)
    import torch.distributed as dist
    D.init(backend=args.dist_backend)
    try:
        return run(args, out=out)
    finally:
        dist.destroy_process_group()


if __name__ == '__main__':
    main()
