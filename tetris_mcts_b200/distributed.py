"""Multi-GPU plumbing: one process per GPU (torch.distributed, NCCL over NVLink), games sharded embarrassingly.

The reference has no distributed backend at all (SURVEY §2b: workers are `play.py &` processes exchanging HDF5 files,
cycle.sh:53-74).  The only exchange step of this build is the all-gather of fixed-size replay-sample blocks
(212-byte rows {int8 state[200], f32 value, f32 variance, f32 visit}; schema = ValueSim.memory, agents/ValueSim.py:25-30)
plus small counter reductions for reporting.  No data-path collective exists inside the search."""
import os

import numpy as np
import torch
import torch.distributed as dist

SAMPLE_BYTES = 212


def env_world():
    return int(os.environ.get("RANK", 0)), int(os.environ.get("LOCAL_RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))


def init(backend=None):
    rank, local_rank, world = env_world()
    if world > 1 and not dist.is_initialized():
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29511")
        if backend == "nccl":
            torch.cuda.set_device(local_rank)
        dist.init_process_group(backend=backend, rank=rank, world_size=world)
    return rank, local_rank, world


def shard_range(n_games, rank, world):
    """Contiguous block of games owned by `rank` (sizes differ by at most one)."""
    base, rem = divmod(n_games, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def shard_seeds(base_seed, n_games, rank, world):
    """Per-game piece seeds base_seed + global game id (SURVEY §8d), for this rank's block."""
    lo, hi = shard_range(n_games, rank, world)
    return (np.arange(lo, hi, dtype=np.uint64) + base_seed).astype(np.uint32)


def barrier():
    if dist.is_initialized():
        dist.barrier()


def max_over_ranks(x, device="cpu"):
    if not dist.is_initialized():
        return float(x)
    t = torch.tensor([float(x)], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def sum_over_ranks(values, device="cpu"):
    """values: dict name -> number; returns the element-wise sum over ranks."""
    keys = sorted(values)
    t = torch.tensor([float(values[k]) for k in keys], dtype=torch.float64, device=device)
    if dist.is_initialized():
        dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return {k: float(v) for k, v in zip(keys, t.tolist())}


def allgather_samples(block, count):
    """block: uint8 tensor [capacity, 212] (CUDA for NCCL, CPU for gloo) holding `count` valid rows.
    Returns (all_rows uint8 [sum(count), 212], counts list).  Fixed-size blocks + a count per rank, so every rank
    posts the same message size (no ragged collective)."""
    assert block.dtype == torch.uint8 and block.dim() == 2 and block.shape[1] == SAMPLE_BYTES
    if not dist.is_initialized():
        return block[:count].clone(), [int(count)]
    world = dist.get_world_size()
    cnt = torch.tensor([int(count)], dtype=torch.int32, device=block.device)
    counts = [torch.zeros_like(cnt) for _ in range(world)]
    dist.all_gather(counts, cnt)
    gathered = torch.empty((world,) + tuple(block.shape), dtype=torch.uint8, device=block.device)
    dist.all_gather_into_tensor(gathered, block.contiguous()) if hasattr(dist, "all_gather_into_tensor") and block.is_cuda else \
        dist.all_gather(list(gathered.unbind(0)), block.contiguous())
    counts = [int(c.item()) for c in counts]
    rows = torch.cat([gathered[r, :counts[r]] for r in range(world)], dim=0)
    return rows, counts


def decode_samples(rows):
    """uint8 [n,212] -> (states int8 [n,1,20,10], value f32[n,1], variance f32[n,1], weight f32[n,1]) — the four arrays of
    ValueSim.memory / the `./data/dump.npz` layout (agents/ValueSim.py:25-30,177)."""
    a = rows.cpu().numpy() if isinstance(rows, torch.Tensor) else np.asarray(rows)
    a = np.ascontiguousarray(a)
    states = a[:, :200].view(np.int8).reshape(-1, 1, 20, 10).copy()
    f = np.ascontiguousarray(a[:, 200:212]).view(np.float32).reshape(-1, 3)
    return states, f[:, 0:1].copy(), f[:, 1:2].copy(), f[:, 2:3].copy()
