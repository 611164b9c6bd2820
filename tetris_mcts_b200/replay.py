"""Host side of the replay memory: the 212-byte sample rows the engine produces (k_gc's store_nodes, b200_collect_samples_dev,
the NCCL all-gather blocks of distributed.py) <-> the reference's `ValueSim.memory` arrays and its `./data/dump.npz` file.

Reference layout (agents/ValueSim.py:25-30): memory = [states f32[N,1,20,10], values f32[N,1], variance f32[N,1], weights f32[N,1]],
filled by store_nodes (ValueSim.py:122-159: state, value, variance, weight = visit count) and written by train_nodes as
np.savez('./data/dump', states=..., values=..., variance=..., weights=...) (ValueSim.py:176-177).  Pure re-layout, no arithmetic."""
import numpy as np

SAMPLE_BYTES = 212          # int8 state[200] | f32 value | f32 variance | f32 visit (include/b200_tetris_mcts.h)


def rows_to_memory(rows):
    """rows: uint8[n, 212] -> the four arrays of ValueSim.memory[:n] (ValueSim.py:25-30), same dtypes and shapes."""
    rows = np.ascontiguousarray(rows, dtype=np.uint8).reshape(-1, SAMPLE_BYTES)
    n = len(rows)
    states = rows[:, :200].view(np.int8).astype(np.float32).reshape(n, 1, 20, 10)
    tail = np.ascontiguousarray(rows[:, 200:212]).view(np.float32).reshape(n, 3)
    return [states, tail[:, 0:1].copy(), tail[:, 1:2].copy(), tail[:, 2:3].copy()]


def rows_to_memory_dev(rows):
    """The torch form of rows_to_memory: rows uint8 tensor [n, 212] (any device) -> four contiguous float32 tensors on that device, states
    [n,1,20,10] and value / variance / visit [n,1], bit for bit the arrays rows_to_memory returns.  Issued on torch's current stream."""
    import torch
    rows = rows.reshape(-1, SAMPLE_BYTES)
    n = rows.shape[0]
    states = rows[:, :200].view(torch.int8).to(torch.float32).reshape(n, 1, 20, 10)
    tail = rows[:, 200:212].contiguous().view(torch.float32)
    col = lambda j: tail[:, j:j + 1].clone(memory_format=torch.contiguous_format)    # noqa: E731
    return [states.contiguous(), col(0), col(1), col(2)]


def memory_to_rows(states, values, variance, weights):
    """The inverse (e.g. to feed samples stored by the reference into the all-gather format)."""
    n = len(states)
    rows = np.zeros((n, SAMPLE_BYTES), np.uint8)
    rows[:, :200] = np.asarray(states, np.float32).reshape(n, 200).astype(np.int8).view(np.uint8)
    tail = np.stack([np.asarray(values, np.float32).reshape(n), np.asarray(variance, np.float32).reshape(n),
                     np.asarray(weights, np.float32).reshape(n)], axis=1)
    rows[:, 200:212] = np.ascontiguousarray(tail).view(np.uint8)
    return rows


def dump(path, rows):
    """np.savez('./data/dump', states=, values=, variance=, weights=) of ValueSim.train_nodes (ValueSim.py:176-177)."""
    states, values, variance, weights = rows_to_memory(rows)
    np.savez(path, states=states, values=values, variance=variance, weights=weights)
