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


def run(args, out=sys.stdout, timing=None):
    """timing: a dict, filled with moves, trainings and the wall-clock seconds of the run split into search (everything but training) and
    training (--online)"""
    mode, gamma, low = MODES[args.agent_type]
    env_args = ((20, 10), args.app, args.tetris_scoring, args.tetris_randomizer)           # play.py:75
    weights = None
    if mode != "vanilla":
        from .model.model_vv import init_weights, load_checkpoint_weights
        weights = load_checkpoint_weights()                                                 # agents/ValueSim.py:42-44
        if weights is None:
            weights = init_weights(0)
    eng = BatchedEngine(args.n_parallel, max_nodes=args.max_nodes, mode=mode, gamma=gamma, low=low,
                        eval_kind="net_tc" if mode != "vanilla" else "synthetic", weights=weights, env_args=env_args, seed=args.seed,
                        device=args.device, overflow_reset=True)
    eng.set_games(PT.new_games(args.n_parallel, env_args, np.arange(args.seed, args.seed + args.n_parallel, dtype=np.uint32)))
    eng.set_gc_headroom(args.max_nodes * 5 // 32)
    online = args.online and not args.benchmark and mode != "vanilla"
    trainer, gcs = None, 0
    if online:                                                                             # ValueSim.py:21-37 memory, min_visits_to_store (25: ValueSimLP.py:11)
        from .online import OnlineTrainer
        eng.replay_enable(min_visits=25 if mode == "lp" else 10, capacity=args.memory_size)
        eng.replay_policy(args.accumulation_policy, episodes_per_train=args.episodes_per_train, memory_growth_rate=args.memory_growth_rate)
        trainer = OnlineTrainer(eng, weights, args.memory_size, batch_size=args.train_batch_size, max_iters=args.train_max_iters)   # ValueSim.py:180
    status = RealtimeStatus(args.status_dir) if args.realtime_status else None
    saver = None
    if args.save:                                                                          # play.py:93-94, 131-132
        from .data import DataSaver, rows_from_move
        saver = DataSaver(args.save_dir, args.save_file, args.cycle)
        episode_of = np.zeros(args.n_parallel, np.int32)                                    # play.py passes ngames: the episode a row belongs to
    tracker = ScoreTracker()
    ngames, moves = 0, 0
    t_start = time.perf_counter()
    try:
        while True:
            if status:
                status.update(eng.get_games()[args.watch])
            before = eng.get_games() if saver else None
            actions, stats = eng.play_move(args.mcts_sims, auto_reset=True, want_stats=saver is not None)   # agent.play(); game.play(action); agent.update_root(game); reset
            if saver:
                saver.add_rows(rows_from_move(before, actions, stats, args.cycle, episode_of))
            moves += 1
            done = False
            for g, score, lines, _ep in eng.finished_games():
                ngames += 1
                if saver:
                    episode_of[g] = ngames
                if args.endless:
                    print(EPISODE_FMT.format(ngames, int(score), int(lines)), flush=True, file=out)
                else:
                    tracker.append(int(score), int(lines))
                    tracker.printStats(file=out)
                if ngames >= args.ngames:
                    done = True
                    break
            if online and eng.counters()["gcs"] != gcs:                                        # collections stored rows this move
                gcs = eng.counters()["gcs"]
                train_now, n = eng.replay_policy_step(ngames)                                   # current_episode = finished games
                print('Memory usage: {} / {}'.format(n, args.memory_size), **perr)            # agent.cpp:632
                if train_now:
                    trainer.train(n, ngames)
            if done or (args.max_moves and moves >= args.max_moves):
                break
    finally:
        print(flush=True, file=out)                                                         # play.py:179
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
    p.add_argument('--max_moves', default=0, type=int)
    return p.parse_args(argv)


def main(argv=None, out=sys.stdout):
    return run(parse_args(argv), out=out)


if __name__ == '__main__':
    main()
