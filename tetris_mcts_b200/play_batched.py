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

--checkpoint_dir DIR writes a checkpoint there every --checkpoint_every moves (0: when the run ends), after the move's training: one engine image
per rank (BatchedEngine.save) and the run's own state, as one generation DIR/gen<moves> that DIR/latest names once it is complete; --resume
continues from that generation as the stopped processes would have gone on (DESIGN §4c: exactly so only where the run itself is
deterministic, one game per rank under --online):

  python -m tetris_mcts_b200.play_batched --agent_type ValueSimLP --online --endless --checkpoint_dir ckpt --checkpoint_every 100 --resume

--evaluator MODULE:FACTORY searches with the caller's network instead of the built-in one: FACTORY(device) returns a device evaluator
(BatchedEngine.run_sims: a torch tensor [n,1,20,10] of boards in, (v, var) out), and the engine runs eval_kind "external".

--trainer MODULE:FACTORY (with --online) trains with the caller's function instead of the built-in trainer (OnlineMCTSAgent's train callback,
online.CallbackTrainer): FACTORY(device) returns train(state, value, variance, visit, size), called with the memory's first `size` rows as
float32 torch tensors on the device (--trainer_host: numpy arrays) each time the accumulation policy says train.  With --evaluator it trains
that network in place and returns None; without, it returns new weights for the built-in network (a Model_VV state_dict or N_WEIGHTS floats),
or None to keep them:

  python -m tetris_mcts_b200.play_batched --agent_type ValueSimLP --online --evaluator mynets:make_evaluator --trainer mynets:make_trainer --endless
  python -m tetris_mcts_b200.play_batched --agent_type ValueSimLP --online --eval_kind net_fp16 --trainer mytraining:make_trainer --endless

--agent_type VanillaC is the C++ agent's rollout search (agents/VanillaC.py): check_low with low=1 and the leaf game scored by one random
playout over all eight action ids, backed up as (score, 1e5); the engine runs eval_kind "external_game".  --game_evaluator MODULE:FACTORY
(Vanilla or VanillaC) scores each step's leaf games with the caller's function instead: FACTORY(device) returns a device game evaluator
(BatchedEngine.run_sims: int32 packed records [n,20] in, (v, var) out; pyTetris.step_games_dev / states_of_dev / playout_dev work on them):

  python -m tetris_mcts_b200.play_batched --agent_type VanillaC --n_parallel 4096 --mcts_sims 300 --endless
  python -m tetris_mcts_b200.play_batched --agent_type Vanilla --game_evaluator mymod:make --n_parallel 4096 --mcts_sims 300 --endless

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
MODES = {"ValueSimLP": ("lp", 0.999, 1), "ValueSim": ("single", 0.999, 1), "Vanilla": ("vanilla", 0.99, 5), "VanillaC": ("vanilla", 0.99, 1)}


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


# flags a resumed run must share with the run that wrote the checkpoint (they change what the engine, the memory or the trainer hold)
RESUME_FLAGS = ("agent_type", "n_parallel", "max_nodes", "seed", "eval_kind", "train_kind", "online", "memory_size", "accumulation_policy",
                "episodes_per_train", "memory_growth_rate", "train_batch_size", "train_max_iters", "mcts_sims", "app", "tetris_scoring",
                "tetris_randomizer", "save", "cycle")


# A checkpoint is one generation: DIR/gen<moves>/ holds every rank's engine image and run state, each run state naming its image and the
# image's size.  DIR/latest names the newest complete generation; rank 0 replaces it (written aside, synced, renamed) only after every rank
# has written its files, and older generations are deleted only after that.  A run stopped at any point leaves `latest` on a generation
# whose files are all there.  DIR is shared by the ranks.
def generation_dir(directory, gen):
    return os.path.join(directory, "gen%09d" % gen)


def checkpoint_paths(directory, gen, rank):
    d = generation_dir(directory, gen)
    return os.path.join(d, "engine.rank%d" % rank), os.path.join(d, "run.rank%d" % rank)


def _write_synced(path, data):
    with open(path + ".tmp", "wb") as f:
        f.write(data)
        f.flush()
        os.fsync(f.fileno())
    os.replace(path + ".tmp", path)


def write_latest(directory, gen):
    _write_synced(os.path.join(directory, "latest"), b"%d\n" % gen)


def read_latest(directory):
    path = os.path.join(directory, "latest")
    if not os.path.isfile(path):
        raise ValueError("--resume: no checkpoint in %s (no %s)" % (directory, path))
    with open(path) as f:
        return int(f.read().strip())


def write_run_state(path, state):
    import pickle
    _write_synced(path, pickle.dumps(state))


def read_run_state(args, rank, world):
    """(run state, engine image path) of rank `rank` in the generation DIR/latest names.  Raises ValueError when the checkpoint is missing,
    when the run state and its image are not of one generation, when the checkpointed run had finished, or when it was written with other
    flags (the message names them)."""
    import pickle
    gen = read_latest(args.checkpoint_dir)
    image, path = checkpoint_paths(args.checkpoint_dir, gen, rank)
    if not os.path.isfile(path):
        raise ValueError("--resume: no run state at %s" % path)
    with open(path, "rb") as f:
        st = pickle.load(f)
    if st.get("generation") != gen or st.get("moves") != gen:
        raise ValueError("--resume: %s is the run state of move %s, not of generation %d" % (path, st.get("moves"), gen))
    if st.get("image") != os.path.basename(image) or not os.path.isfile(image) or os.path.getsize(image) != st.get("image_bytes"):
        raise ValueError("--resume: the engine image %s is not the one the run state %s names" % (image, path))
    if st.get("finished"):
        raise ValueError("--resume: the run checkpointed in %s had finished (--ngames reached)" % args.checkpoint_dir)
    differ = ["world size (%d, checkpoint %d)" % (world, st["world"])] if st["world"] != world else []
    differ += ["--%s (%r, checkpoint %r)" % (k, getattr(args, k), st["flags"].get(k)) for k in RESUME_FLAGS if st["flags"].get(k) != getattr(args, k)]
    if differ:
        raise ValueError("--resume: the checkpoint in %s was written with other settings: %s" % (args.checkpoint_dir, "; ".join(differ)))
    return st, image


def agree_on_generation(found):
    """found: every rank's (generation, None) or (None, error message) -> the one generation; raises ValueError (on every rank) when a rank
    failed or the ranks read different generations"""
    errors = ["rank %d: %s" % (r, err) for r, (_g, err) in enumerate(found) if err]
    if errors:
        raise ValueError("; ".join(errors))
    gens = [g for g, _e in found]
    if len(set(gens)) != 1:
        raise ValueError("--resume: the ranks found checkpoints of different moves: %s" % gens)
    return gens[0]


def drop_older_generations(directory, gen, rank):
    """this rank's files of every generation but `gen` (after `latest` names gen)"""
    for name in os.listdir(directory):
        if not name.startswith("gen") or name == os.path.basename(generation_dir(directory, gen)):
            continue
        d = os.path.join(directory, name)
        for f in ("engine.rank%d" % rank, "run.rank%d" % rank, "engine.rank%d.tmp" % rank, "run.rank%d.tmp" % rank):
            if os.path.exists(os.path.join(d, f)):
                os.remove(os.path.join(d, f))
        try:
            os.rmdir(d)
        except OSError:
            pass                                                                           # another rank's files are still there


def drop_later_chunks(file_name, chunk):
    """a resumed run rewrites the --save chunks from number `chunk` on: those the stopped run wrote after its checkpoint go"""
    import glob
    for f in glob.glob(glob.escape(file_name) + ".*.npy"):
        idx = f[len(file_name) + 1:-4]
        if idx.isdigit() and int(idx) >= chunk:
            os.remove(f)


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
    weights, evaluator, game_evaluator = None, None, None
    resumed = None
    if args.resume:
        try:
            resumed, image = read_run_state(args, rank, world)
            found = (resumed["generation"], None)
        except ValueError as exc:
            found = (None, str(exc))
        if world > 1:                                                                      # every rank resumes from the same generation, or none
            agree_on_generation(D.gather_objects(found))
        elif found[1]:
            raise ValueError(found[1])
    if args.evaluator:
        evaluator = _factory(args.evaluator)(_torch_device(device))
    elif args.game_evaluator:
        game_evaluator = _factory(args.game_evaluator)(_torch_device(device))
    elif args.agent_type == "VanillaC":                                                   # agents/VanillaC.py random_playout, on the device
        game_evaluator = PT.playout_evaluator(n_actions=8, variance=1e5, seed=args.seed + lo)
    elif mode != "vanilla" and resumed is not None:
        weights = resumed["trainer"]["weights"] if resumed["trainer"] else None               # the engine image holds the search's own
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
    if resumed is not None:                                                               # trees, games, memory and policy as they were saved
        eng = BatchedEngine.load(image, device=device)
    else:
        eng = BatchedEngine(hi - lo, max_nodes=args.max_nodes, mode=mode, gamma=gamma, low=low,
                            eval_kind="external" if evaluator else "external_game" if game_evaluator else (args.eval_kind if mode != "vanilla" else "synthetic"),
                            weights=weights,
                            env_args=env_args, seed=(args.seed + 0x9E3779B9 * lo) & 0xFFFFFFFF, device=device, overflow_reset=True)
        eng.set_games(PT.new_games(hi - lo, env_args, D.shard_seeds(args.seed, args.n_parallel, rank, world)))
        eng.set_gc_headroom(args.max_nodes * 5 // 32)
    online = args.online and not args.benchmark and mode != "vanilla"
    trainer, gcs, block = None, 0, None
    if online:                                                                             # ValueSim.py:21-37 memory, min_visits_to_store (25: ValueSimLP.py:11)
        from .online import CallbackTrainer, OnlineTrainer
        if resumed is None:
            eng.replay_enable(min_visits=25 if mode == "lp" else 10, capacity=args.memory_size)
            if rank == 0:
                eng.replay_policy(args.accumulation_policy, episodes_per_train=args.episodes_per_train, memory_growth_rate=args.memory_growth_rate)
        if args.trainer:
            trainer = CallbackTrainer(eng, weights, args.memory_size, _factory(args.trainer)(_torch_device(device)), host=args.trainer_host,
                                      external=evaluator is not None)
        else:
            trainer = OnlineTrainer(eng, weights, args.memory_size, batch_size=args.train_batch_size, max_iters=args.train_max_iters,
                                    train_kind=args.train_kind)   # ValueSim.py:180
        if resumed is not None and resumed["trainer"]:
            trainer.restore(resumed["trainer"])
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
    if resumed is not None:
        ngames, moves, gcs = resumed["ngames"], resumed["moves"], resumed["gcs"]
        tracker.scores, tracker.lines = list(resumed["scores"]), list(resumed["lines"])
        if saver:
            episode_of[:] = resumed["episode_of"]
            if not saver.hdf5:
                saver.chunk = resumed["saver_chunk"]
                drop_later_chunks(saver.file_name, saver.chunk)

    def checkpoint(finished):
        """after a completed move (and its training): every rank's engine image and run state in generation `moves`, then `latest`"""
        if saver:
            saver.flush()                                                                  # the rows so far are on disk: a resume appends the rest
        os.makedirs(generation_dir(args.checkpoint_dir, moves), exist_ok=True)
        if world > 1:
            D.barrier()
        image, state = checkpoint_paths(args.checkpoint_dir, moves, rank)
        size = eng.save(image)
        write_run_state(state, dict(world=world, flags={k: getattr(args, k) for k in RESUME_FLAGS}, generation=moves, ngames=ngames, moves=moves,
                                    gcs=gcs, image=os.path.basename(image), image_bytes=size, finished=bool(finished),
                                    scores=list(tracker.scores), lines=list(tracker.lines), trainer=trainer.state() if trainer else None,
                                    episode_of=episode_of.copy() if saver else None,
                                    saver_chunk=saver.chunk if saver and not saver.hdf5 else None))
        if world > 1:
            D.barrier()                                                                    # every rank's files of this generation are written
        if rank == 0:
            write_latest(args.checkpoint_dir, moves)
        if world > 1:
            D.barrier()
        drop_older_generations(args.checkpoint_dir, moves, rank)
    t_start = time.perf_counter()
    try:
        while True:
            if status:
                status.update(eng.get_games()[args.watch - lo])
            before = eng.get_games() if saver else None
            actions, stats = eng.play_move(args.mcts_sims, auto_reset=True, want_stats=saver is not None,
                                           evaluator=evaluator, game_evaluator=game_evaluator)   # agent.play(); game.play(action); agent.update_root(game); reset
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
                    if args.trainer and rank == 0:
                        print('Training complete.', **perr)                                   # agent.cpp:702
            last = done or (args.max_moves and moves >= args.max_moves)
            if args.checkpoint_dir and (last or (args.checkpoint_every and moves % args.checkpoint_every == 0)):
                checkpoint(done)
            if last:
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


def _factory(spec):
    """MODULE:FACTORY -> the callable FACTORY of the imported MODULE"""
    import importlib
    module, factory = spec.split(":", 1)
    return getattr(importlib.import_module(module), factory)


def _torch_device(device):
    import torch
    return torch.device("cuda", device)


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
                        'the engine runs eval_kind external.  Not with --online unless --trainer trains it, nor with Vanilla')
    p.add_argument('--game_evaluator', default=None, metavar='MODULE:FACTORY',
                   help='Vanilla / VanillaC: score each step\'s leaf games with the caller\'s function instead of the rollout: FACTORY(device) '
                        'returns a device game evaluator (int32 packed records [n,20] -> (v, var)); the engine runs eval_kind external_game')
    p.add_argument('--trainer', default=None, metavar='MODULE:FACTORY',
                   help='--online: train with the caller\'s function instead of the built-in trainer: FACTORY(device) returns '
                        'train(state, value, variance, visit, size), which trains the --evaluator network in place and returns None, or '
                        'returns new weights for the built-in network (a Model_VV state_dict or N_WEIGHTS floats) or None')
    p.add_argument('--trainer_host', default=False, action='store_true',
                   help='hand --trainer numpy arrays instead of torch tensors on the device')
    p.add_argument('--max_moves', default=0, type=int, help='stop after this many moves (counted from the start of the run, across --resume)')
    p.add_argument('--checkpoint_dir', default=None, help='write checkpoints here (one engine image per rank and the run state)')
    p.add_argument('--checkpoint_every', default=0, type=int, help='moves between checkpoints; 0 = only when the run ends')
    p.add_argument('--resume', default=False, action='store_true', help='continue the run checkpointed in --checkpoint_dir')
    p.add_argument('--dist_backend', default='nccl', choices=('nccl', 'gloo'),
                   help='under torchrun: collectives over NCCL (one GPU per rank), or gloo through the host (several ranks may share a GPU)')
    args = p.parse_args(argv)
    if args.trainer:
        if not args.online:
            p.error('--trainer needs --online: it is called when the online accumulation policy says train')
        if args.agent_type == 'Vanilla':
            p.error('--trainer cannot be combined with --agent_type Vanilla: Vanilla has no value network to train')
        if ':' not in args.trainer:
            p.error('--trainer takes MODULE:FACTORY')
        if args.checkpoint_dir:
            p.error('--checkpoint_dir cannot be combined with --trainer: the caller\'s training state is not part of the checkpoint')
        given = _given_flags(p, argv)
        clash = [f for f in ('train_kind', 'train_batch_size', 'train_max_iters') if f in given]
        if clash:
            p.error('--trainer cannot be combined with %s: they set the built-in trainer, which --trainer replaces'
                    % ', '.join('--' + f for f in clash))
    if args.trainer_host and not args.trainer:
        p.error('--trainer_host needs --trainer')
    if args.evaluator and args.online and not args.trainer:
        p.error('--evaluator cannot be combined with --online: the online trainer trains the built-in Model_VV weights')
    if args.evaluator and args.agent_type == 'Vanilla':
        p.error('--evaluator cannot be combined with --agent_type Vanilla: Vanilla evaluates leaves by random rollout')
    if args.evaluator and ':' not in args.evaluator:
        p.error('--evaluator takes MODULE:FACTORY')
    if (args.resume or args.checkpoint_every) and not args.checkpoint_dir:
        p.error('--resume and --checkpoint_every need --checkpoint_dir')
    if args.checkpoint_dir and args.evaluator:
        p.error('--checkpoint_dir cannot be combined with --evaluator: the caller\'s network is not part of the checkpoint')
    if args.game_evaluator:
        if args.agent_type not in ('Vanilla', 'VanillaC'):
            p.error('--game_evaluator needs --agent_type Vanilla or VanillaC: the other agents evaluate boards (see --evaluator)')
        if args.evaluator:
            p.error('--game_evaluator cannot be combined with --evaluator: the leaf games are scored by one of them')
        if args.online:
            p.error('--game_evaluator cannot be combined with --online: Vanilla has no value network to train')
        if ':' not in args.game_evaluator:
            p.error('--game_evaluator takes MODULE:FACTORY')
    if args.agent_type == 'VanillaC':
        if args.evaluator:
            p.error('--evaluator cannot be combined with --agent_type VanillaC: VanillaC scores leaf games (see --game_evaluator)')
        if args.trainer:
            p.error('--trainer cannot be combined with --agent_type VanillaC: VanillaC has no value network to train')
    if args.checkpoint_dir and (args.game_evaluator or args.agent_type == 'VanillaC'):
        p.error('--checkpoint_dir cannot be combined with --game_evaluator or --agent_type VanillaC: the playouts\' random state is not '
                'part of the checkpoint')
    if args.checkpoint_every < 0:
        p.error('--checkpoint_every takes a number of moves >= 0')
    return args


def _given_flags(p, argv):
    """the destinations of the flags argv sets itself (abbreviations included), whatever their values"""
    for a in p._actions:
        a.default = argparse.SUPPRESS
    return set(vars(p.parse_args(argv)))


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
