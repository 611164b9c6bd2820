"""An evaluator that is an integer-exact function of the board, written twice: in numpy (the oracle agents' eval_cb, and the host form) and
in torch on the device (the engine's eval_kind "external").  Batch-independent by construction: each row's outputs depend on its own board.

  h = sum over the 200 cells of (cell + 1) * W[cell]           (int64, W a fixed integer table)
  value modes: v = (h % 1000) / 8, var = (h // 1000 % 512 + 1) / 16                 (exact in float32)
  distributional: r_b = (h * (2b + 1)) % 97 + 1, p_b = float32(r_b / sum r)       (the quotient in float64, rounded once)"""
import numpy as np

W = ((np.arange(200, dtype=np.int64) * 7919 + 13) % 1009 + 1)


def _h_np(states):
    s = np.asarray(states).reshape(-1, 200).astype(np.int64)
    return (s + 1) @ W


def value_np(states):
    h = _h_np(states)
    return (h % 1000).astype(np.float32) / np.float32(8), ((h // 1000) % 512 + 1).astype(np.float32) / np.float32(16)


def dist_np(states, atoms):
    h = _h_np(states)
    r = (h[:, None] * (2 * np.arange(atoms, dtype=np.int64) + 1)) % 97 + 1
    return (r.astype(np.float64) / r.sum(1, keepdims=True).astype(np.float64)).astype(np.float32)


def _h_torch(boards):
    import torch
    w = torch.as_tensor(W, device=boards.device)
    return ((boards.reshape(boards.shape[0], 200).to(torch.int64) + 1) * w).sum(1)


def value_torch(boards):
    import torch
    h = _h_torch(boards)
    return (h % 1000).to(torch.float32) / 8, ((h // 1000) % 512 + 1).to(torch.float32) / 16


def dist_torch(atoms):
    import torch

    def ev(boards):
        h = _h_torch(boards)
        r = (h[:, None] * (2 * torch.arange(atoms, device=boards.device, dtype=torch.int64) + 1)) % 97 + 1
        return (r.to(torch.float64) / r.sum(1, keepdim=True).to(torch.float64)).to(torch.float32)
    return ev
