"""CPU side of the online training loop: the new C-ABI entry points are exported, the numpy restatement of the device batch sampler
(include/b200_tetris_mcts.h b200_trainer_train_rows_dev) is deterministic, in range and equal to splitmix64 in plain integers, and
play_batched parses its online flags."""
import ctypes as C
import re
import subprocess

import numpy as np
import pytest

M64 = (1 << 64) - 1


def splitmix64(x):
    z = (x + 0x9E3779B97F4A7C15) & M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def test_online_training_symbols_exported():
    from tetris_mcts_b200 import _lib, build
    lib = build.build()
    names = {"b200_trainer_train_rows_dev", "b200_trainer_loss_rows_dev", "b200_rows_stats_dev"}
    assert names <= set(_lib.exported_symbols())
    nm = subprocess.run(["nm", "-D", "--defined-only", lib], capture_output=True, text=True).stdout
    L = C.CDLL(lib)
    for n in names:
        assert hasattr(L, n) and re.search(r"\bT %s\b" % n, nm), n


def test_sampler_restatement():
    from tetris_mcts_b200.model.trainer import sample_indices
    for seed, it, batch, n in [(0, 0, 64, 86), (12345, 200, 1024, 450000), (M64, 3, 7, 1), (2**40 + 3, 2**33, 300, 10)]:
        a = sample_indices(seed, it, batch, n)
        assert a.dtype == np.int32 and a.shape == (batch,) and a.min() >= 0 and a.max() < n
        assert np.array_equal(a, sample_indices(seed, it, batch, n))
        base = splitmix64((splitmix64(seed) + it) & M64)
        assert [splitmix64((base + i) & M64) % n for i in range(batch)] == a.tolist()
    assert not np.array_equal(sample_indices(1, 0, 64, 1000), sample_indices(1, 1, 64, 1000))
    assert not np.array_equal(sample_indices(1, 0, 64, 1000), sample_indices(2, 0, 64, 1000))
    # uniform over [0, n): every row is drawn about equally often
    counts = np.bincount(np.concatenate([sample_indices(9, it, 1000, 10) for it in range(50)]), minlength=10)
    assert counts.min() > 4500 and counts.max() < 5500


def test_play_batched_online_flags():
    from tetris_mcts_b200 import play_batched as PB
    a = PB.parse_args(["--online"])
    assert a.online and a.accumulation_policy == 3 and a.episodes_per_train == 25 and a.memory_growth_rate == 5000
    assert a.train_batch_size == 1024 and a.train_max_iters == 50000 and a.memory_size == 500000
    a = PB.parse_args(["--online", "--accumulation_policy", "1", "--episodes_per_train", "7", "--memory_growth_rate", "100",
                       "--train_batch_size", "512", "--train_max_iters", "300", "--memory_size", "1000"])
    assert (a.accumulation_policy, a.episodes_per_train, a.memory_growth_rate, a.train_batch_size, a.train_max_iters, a.memory_size) == (1, 7, 100, 512, 300, 1000)
    assert not hasattr(a, "drain_every")
    with pytest.raises(SystemExit):
        PB.parse_args(["--accumulation_policy", "4"])


def test_train_rows_refuses_unsupported_options():
    from tetris_mcts_b200.model import model_vv as MV
    assert MV._TRAIN_ROWS_FIXED["validation_fraction"] == 0.1 and MV._TRAIN_ROWS_FIXED["shuffle"] is False
    r = MV._combine_chunks([1.0, 3.0], [0.5, 0.5], [1.0, 1.0])
    assert r["loss"] == 2.0 and abs(r["loss_std"] - np.sqrt(0.25 + 1.0)) < 1e-12
