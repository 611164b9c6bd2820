"""Host logic of the data-parallel online loop, without a GPU: the batch slices of the ranks, the order rank 0 numbers the episodes of
every rank in, the stop decision every rank takes alike, and the per-rank --save file names."""
import numpy as np
import pytest

from tetris_mcts_b200 import distributed as D
from tetris_mcts_b200 import play_batched as PB


def test_batch_slices_cover_the_batch():
    for batch in (1, 2, 3, 8, 1000, 1024, 4097):
        for world in (1, 2, 3, 4, 8):
            if batch < world:
                with pytest.raises(ValueError):
                    D.batch_slice(batch, 0, world)
                continue
            edges = [D.batch_slice(batch, r, world) for r in range(world)]
            assert edges[0][0] == 0 and edges[-1][1] == batch
            assert all(edges[i][1] == edges[i + 1][0] and edges[i][0] < edges[i][1] for i in range(world - 1))
            assert edges == [D.shard_range(batch, r, world) for r in range(world)]
    assert D.batch_slice(1000, 0, 3) == (0, 334) and D.batch_slice(1000, 2, 3) == (667, 1000)


def test_episode_merge_order():
    """the games of all ranks, in global game order, as one engine holding them all lists them (a game may finish twice in a move)"""
    n, world = 10, 3
    rng = np.random.default_rng(1)
    games = sorted(rng.choice(n, 6, replace=False).tolist() + [4])
    one = [(g, 100 + g, i) for i, g in enumerate(games)]                    # one engine: sorted by game
    per_rank = []
    for r in range(world):
        lo, hi = D.shard_range(n, r, world)
        per_rank.append([f for f in one if lo <= f[0] < hi])
    assert PB.merge_finished(per_rank) == one
    assert PB.merge_finished(per_rank[::-1]) == one
    assert PB.merge_finished([[], []]) == []


def _stop_move(finished_per_move, ngames, max_moves):
    """the move at which play_batched's loop stops: every rank replays the same merged lists, so every rank stops on it"""
    total = 0
    for move, fin in enumerate(finished_per_move, 1):
        for _ in fin:
            total += 1
            if total >= ngames:
                return move, total
        if max_moves and move >= max_moves:
            return move, total
    return None, total


def test_global_stop_decision():
    rng = np.random.default_rng(2)
    n, world, moves = 12, 3, 40
    per_move = [sorted(rng.choice(n, rng.integers(0, 4), replace=False).tolist()) for _ in range(moves)]
    for ngames, max_moves in [(5, 0), (17, 0), (10 ** 6, 25), (3, 2)]:
        whole = _stop_move([[(g, 0, 0) for g in f] for f in per_move], ngames, max_moves)
        for r in range(world):                                                  # what rank r computes from the gathered lists
            lo, hi = D.shard_range(n, r, world)
            merged = [PB.merge_finished([[(g, 0, 0) for g in f if D.shard_range(n, q, world)[0] <= g < D.shard_range(n, q, world)[1]]
                                         for q in range(world)]) for f in per_move]
            assert _stop_move(merged, ngames, max_moves) == whole


def test_save_paths_per_rank(tmp_path):
    from tetris_mcts_b200.data import DataSaver
    assert PB.save_suffix(0, 1) == ""
    names = set()
    for r in range(4):
        s = DataSaver(str(tmp_path) + "/", "data", 3, suffix=PB.save_suffix(r, 4))
        names.add(s.file_name)
        assert s.file_name == str(tmp_path) + "/data3.rank%d" % r
        s.close()
    assert len(names) == 4


def test_dist_backend_flag():
    assert PB.parse_args([]).dist_backend == "nccl"
    assert PB.parse_args(["--dist_backend", "gloo"]).dist_backend == "gloo"
    with pytest.raises(SystemExit):
        PB.parse_args(["--dist_backend", "mpi"])
