"""The caller's training function (play_batched --trainer, online.CallbackTrainer) on the GPU; prints one JSON line.

(1) The handoff at --rows rows (default 500 000, a full default memory): b200_replay_peek_dev into the trainer's row buffer, then the re-layout
    into the reference's four float32 arrays, in the device form (replay.rows_to_memory_dev, torch tensors) and the host form (a device-to-host
    copy and replay.rows_to_memory).  Each timing ends in a device synchronise; median, min and max over --repeats.
(2) A --moves move `play_batched --online` run (ValueSimLP, --games games, --sims simulations per move, the value network on the tensor-core
    kernels), once with the built-in trainer (--train_kind tf32, batch 1024, at most --iters steps, early stopping) and once with a
    torch-trained Model_VV returning its state_dict (mode 2): the same network in torch modules (cuDNN convolutions), Gaussian negative log-
    likelihood weighted by visits, Adam, --iters steps of batch 1024.  The search / training seconds of each run, and the trainings.

The card's name and power limit are read in the same run.  Run from the repository root:
    python scripts/train_callback_bench.py [--rows 500000] [--games 4096] [--sims 100] [--moves 40] [--iters 1000]
Files that play_batched writes (checkpoint) go to a temporary directory."""
import argparse
import io
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
ITERS = [1000]


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    name, power = [s.strip() for s in q.splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power}


def synthetic_rows(n, seed=0):
    from tetris_mcts_b200 import replay
    rng = np.random.default_rng(seed)
    states = rng.integers(-1, 2, (n, 20, 10))
    filled = (states > 0).sum(axis=(1, 2))
    return replay.memory_to_rows(states, 2.0 * filled + rng.normal(0, 5, n), 10.0 + filled, rng.integers(25, 500, n))


def handoff(n, repeats):
    import torch
    from tetris_mcts_b200 import replay
    from tetris_mcts_b200.engine import BatchedEngine
    from tetris_mcts_b200.online import CallbackTrainer
    eng = BatchedEngine(1, max_nodes=64, eval_kind="synthetic")
    eng.replay_enable(min_visits=1, capacity=n)
    eng.replay_append(synthetic_rows(n))
    tr = CallbackTrainer(eng, None, n, lambda *a: None)
    dev = tr.buf.device
    res = {}
    for form in ("device", "host"):
        times = []
        for _ in range(repeats + 1):                             # the first, untimed, warms up the allocator
            torch.cuda.synchronize(dev)
            t0 = time.perf_counter()
            tr._peek(n)
            if form == "device":
                mem = replay.rows_to_memory_dev(tr.buf[:n])
                torch.cuda.synchronize(dev)
            else:
                mem = replay.rows_to_memory(tr.buf[:n].cpu().numpy())
            times.append(time.perf_counter() - t0)
            del mem
        t = np.array(times[1:]) * 1e3
        res[form] = {"ms_median": float(np.median(t)), "ms_min": float(t.min()), "ms_max": float(t.max())}
    tr.close(); eng.close()
    return res


def torch_model_vv(device):
    """Model_VV's network (model_vv.WEIGHT_KEYS) as torch modules"""
    import torch
    from torch import nn

    class Head(nn.Module):
        def __init__(self):
            super().__init__()
            self.conv1, self.conv2, self.conv3 = nn.Conv2d(1, 32, 3), nn.Conv2d(32, 32, 3), nn.Conv2d(32, 32, 3)
            self.fc1, self.fc_out = nn.Linear(1792, 256), nn.Linear(256, 2)

        def forward(self, x):
            x = torch.relu(self.conv3(torch.relu(self.conv2(torch.relu(self.conv1(x))))))
            return self.fc_out(torch.relu(self.fc1(x.flatten(1))))

    class Net(nn.Module):
        def __init__(self):
            super().__init__()
            self.head = Head()
            self.register_buffer("out_ubound", torch.tensor([1e2, 1e3]))
            self.register_buffer("out_lbound", torch.tensor([0.0, 1e-1]))

        def forward(self, x):
            out = torch.sigmoid(self.head(x)) * self.out_ubound + self.out_lbound
            return out[:, 0], out[:, 1]
    return Net().to(device)


def torch_trainer(device):
    """mode 2: train a torch Model_VV on the arrays, return its state_dict"""
    import torch
    from tetris_mcts_b200.model.model_vv import init_weights, weights_to_state_dict
    net = torch_model_vv(device)
    net.load_state_dict(weights_to_state_dict(init_weights(0)))       # play_batched's own initial weights
    opt = torch.optim.Adam(net.head.parameters(), lr=1e-3)
    gen = torch.Generator(device=device).manual_seed(0)

    def train(state, value, variance, visit, size):
        if size == 0:
            return None
        net.out_ubound.copy_(torch.stack([value.max(), variance.max()]))
        w = visit[:, 0] / visit.mean()
        for _ in range(ITERS[0]):
            idx = torch.randint(0, size, (1024,), device=device, generator=gen)
            v, var = net(state[idx])
            loss = ((0.5 * torch.log(var) + (value[idx, 0] - v) ** 2 / (2 * var)) * w[idx]).mean()
            opt.zero_grad(set_to_none=True)
            loss.backward()
            opt.step()
        return net.state_dict()
    return train


def online_run(extra, games, sims, moves):
    from tetris_mcts_b200 import play_batched as PB
    argv = ["--agent_type", "ValueSimLP", "--online", "--endless", "--ngames", "1000000000", "--n_parallel", str(games), "--mcts_sims",
            str(sims), "--max_moves", str(moves)] + extra
    timing, err = {}, io.StringIO()
    PB.perr = dict(file=err, flush=True)
    from tetris_mcts_b200.model import model_vv as MV
    MV.perr = PB.perr
    PB.run(PB.parse_args(argv), out=io.StringIO(), timing=timing)
    return {k: timing[k] for k in ("moves", "trainings", "total_s", "search_s", "train_s")}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--rows", type=int, default=500000)
    p.add_argument("--repeats", type=int, default=10)
    p.add_argument("--games", type=int, default=4096)
    p.add_argument("--sims", type=int, default=100)
    p.add_argument("--moves", type=int, default=40)
    p.add_argument("--iters", type=int, default=1000)
    a = p.parse_args()
    sys.modules.setdefault("train_callback_bench", sys.modules[__name__])   # play_batched --trainer imports this module by name
    ITERS[0] = a.iters
    out = dict(gpu_info())
    out["handoff_%d_rows" % a.rows] = handoff(a.rows, a.repeats)
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        os.chdir(tmp)
        try:
            out["online_builtin_tf32"] = online_run(["--train_kind", "tf32", "--train_max_iters", str(a.iters)], a.games, a.sims, a.moves)
            out["online_torch_trainer"] = online_run(["--trainer", "train_callback_bench:torch_trainer"], a.games, a.sims, a.moves)
        finally:
            os.chdir(cwd)
    out["config"] = dict(games=a.games, sims=a.sims, moves=a.moves, iters=a.iters, train_batch=1024)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
