"""The distributional agent's host side without a GPU: Net(atoms)'s state_dict <-> the engine's weight vector (model/model_distributional.py),
the checkpoint checks, Model_Dist's board forms, and play_batched's argument checks for --agent_type DistValueSimOnline."""
import os
from collections import OrderedDict

import numpy as np
import pytest

from tetris_mcts_b200.model import model_distributional as MD


def torch_net(atoms):
    """model/model_distributional.py:18-45 restated: Net(input_shape=(22, 10), atoms) as a torch nn.Sequential named seq"""
    import torch.nn as nn
    act = nn.LeakyReLU(inplace=True)
    seq = nn.Sequential(OrderedDict([("conv1", nn.Conv2d(1, 32, 4, 1)), ("act1", act), ("conv2", nn.Conv2d(32, 32, 4, 1)), ("act2", act),
                                     ("flatten", nn.Flatten()), ("fc1", nn.Linear(16 * 4 * 32, 128)), ("act3", act),
                                     ("fc_v", nn.Linear(128, atoms))]))
    net = nn.Module()
    net.seq = seq
    return net


@pytest.mark.parametrize("atoms", [2, 33, 50, 64])
def test_state_dict_round_trip_and_layout(atoms):
    import torch
    torch.manual_seed(atoms)
    sd = torch_net(atoms).state_dict()
    assert [(k, tuple(v.shape)) for k, v in sd.items()] == [(k, s) for k, s in MD.dist_weight_keys(atoms)]
    w = MD.state_dict_to_dist_weights(sd, atoms)
    assert w.dtype == np.float32 and w.size == MD.n_dist_weights(atoms) == 512 + 32 + 16384 + 32 + 128 * 2048 + 128 + atoms * 129
    back = MD.dist_weights_to_state_dict(w, atoms)
    assert list(back) == list(sd)
    for k in sd:
        assert torch.equal(back[k], sd[k]), k
    r = np.random.default_rng(atoms).standard_normal(w.size).astype(np.float32)
    assert np.array_equal(MD.state_dict_to_dist_weights(MD.dist_weights_to_state_dict(r, atoms), atoms).view(np.uint32), r.view(np.uint32))
    from tetris_mcts_b200.agents.DistValueSimOnline import init_dist_weights
    assert init_dist_weights(0, atoms).size == w.size


def test_value_network_and_other_atoms_are_refused_with_the_mismatch():
    from tetris_mcts_b200.model.model_vv import init_weights, weights_to_state_dict
    with pytest.raises(ValueError) as ei:
        MD.state_dict_to_dist_weights(weights_to_state_dict(init_weights(0)), 50)
    msg = str(ei.value)
    assert "missing seq.conv1.weight" in msg and "unexpected head.conv1.weight" in msg and "out_ubound" in msg
    sd = torch_net(33).state_dict()
    with pytest.raises(ValueError) as ei:
        MD.state_dict_to_dist_weights(sd, 50)
    assert "seq.fc_v.weight (33, 128)" in str(ei.value) and "(50, 128)" in str(ei.value)


def test_checkpoint_files(tmp_path, capsys):
    import torch
    from tetris_mcts_b200.model.model_vv import init_weights, weights_to_state_dict
    assert MD.load_checkpoint_dist_weights(str(tmp_path / "none"), 50) is None
    assert "Checkpoint not found, using default model" in capsys.readouterr().out
    vv = tmp_path / "vv"
    torch.save({"model_state_dict": weights_to_state_dict(init_weights(0)), "optimizer_state_dict": {}}, vv)
    with pytest.raises(ValueError) as ei:
        MD.load_checkpoint_dist_weights(str(vv), 50)
    assert str(vv) in str(ei.value) and "missing seq.conv1.weight" in str(ei.value)
    assert not MD.holds_dist_state_dict(str(vv), 50)
    dist = tmp_path / "dist"
    sd = torch_net(50).state_dict()
    torch.save({"model_state_dict": sd, "optimizer_state_dict": {}}, dist)
    assert MD.holds_dist_state_dict(str(dist), 50) and not MD.holds_dist_state_dict(str(dist), 33)
    w = MD.load_checkpoint_dist_weights(str(dist), 50)
    assert np.array_equal(w, MD.state_dict_to_dist_weights(sd, 50))


def test_board_forms():
    rng = np.random.default_rng(1)
    b = rng.integers(-1, 2, size=(5, 1, 20, 10)).astype(np.int8)
    assert np.array_equal(MD.boards_20x10(b), b.reshape(5, 200))
    padded = np.zeros((5, 1, 22, 10), np.float32)
    padded[:, :, 2:] = b
    assert np.array_equal(MD.boards_20x10(padded), b.reshape(5, 200))
    padded[3, 0, 1, 4] = 1
    with pytest.raises(ValueError, match="top two rows empty"):
        MD.boards_20x10(padded)
    for bad in (b.reshape(5, 20, 10), b.reshape(5, 1, 200), np.zeros((2, 1, 21, 10))):
        with pytest.raises(ValueError, match=r"\[n,1,20,10\]"):
            MD.boards_20x10(bad)
    with pytest.raises(ValueError, match="-1, 0 or 1"):
        MD.boards_20x10(b * 2)


def test_model_dist_does_not_train():
    with pytest.raises(NotImplementedError, match="training the distributional network is out of scope"):
        MD.Model_Dist.train(None)


def _refused(capsys, argv, *words):
    from tetris_mcts_b200 import play_batched as PB
    with pytest.raises(SystemExit) as ei:
        PB.parse_args(argv)
    assert ei.value.code == 2
    err = capsys.readouterr().err
    for w in words:
        assert w in err, err
    return err


@pytest.mark.parametrize("agent", ["DistValueSimOnline", "DistValueSim"])
def test_distributional_agent_arguments(capsys, agent):
    from tetris_mcts_b200 import play_batched as PB
    base = ["--agent_type", agent]
    for extra in (["--online"], ["--trainer", "m:f"], ["--online", "--trainer", "m:f"], ["--train_lag", "1"], ["--online", "--train_lag", "1"]):
        _refused(capsys, base + extra, "training the distributional network is not built")
    _refused(capsys, base + ["--eval_kind", "net_fp16"], "net_fp16 has no distributional network")
    _refused(capsys, base + ["--atoms", "65"], "--atoms")
    _refused(capsys, base + ["--vmin", "10", "--vmax", "10"], "--vmax")
    _refused(capsys, base + ["--evaluator", "m:f", "--dist_checkpoint", "x"], "--dist_checkpoint")
    for kind in ("net_tc", "dist_fp16", "net"):
        a = PB.parse_args(base + ["--eval_kind", kind, "--atoms", "33", "--vmax", "45"])
        assert (a.eval_kind, a.atoms, a.vmin, a.vmax) == (kind, 33, 0.0, 45.0)
    assert PB.MODES[agent] == ("dist", 0.999, 5)
    a = PB.parse_args(base + ["--save", "--checkpoint_dir", "c"])
    assert a.save and a.checkpoint_dir == "c"


def test_value_agents_refuse_the_distributional_settings(capsys):
    _refused(capsys, ["--agent_type", "ValueSimLP", "--eval_kind", "dist_fp16"], "dist_fp16", "DistValueSimOnline")
    _refused(capsys, ["--agent_type", "ValueSim", "--eval_kind", "dist_fp16"], "dist_fp16")
    _refused(capsys, ["--agent_type", "ValueSimLP", "--atoms", "33"], "--atoms")
    _refused(capsys, ["--agent_type", "ValueSimLP", "--dist_checkpoint", "x"], "--dist_checkpoint")
    from tetris_mcts_b200 import play_batched as PB
    assert PB.parse_args(["--agent_type", "ValueSimLP", "--eval_kind", "net"]).eval_kind == "net"


def test_resume_flags_cover_the_distributional_settings(tmp_path):
    """a resume with other --atoms / --vmin / --vmax / --dist_checkpoint is refused; checkpoints written before the flags existed read as
    their defaults"""
    from tetris_mcts_b200 import play_batched as PB
    d = str(tmp_path / "ckpt")
    os.makedirs(PB.generation_dir(d, 5))
    image, state = PB.checkpoint_paths(d, 5, 0)
    with open(image, "wb") as f:
        f.write(b"x" * 8)
    args = PB.parse_args(["--agent_type", "DistValueSimOnline", "--checkpoint_dir", d, "--resume"])
    flags = {k: getattr(args, k) for k in PB.RESUME_FLAGS}
    st = dict(world=1, flags=flags, generation=5, moves=5, image=os.path.basename(image), image_bytes=8, finished=False)
    PB.write_run_state(state, st)
    PB.write_latest(d, 5)
    assert PB.read_run_state(args, 0, 1)[0]["moves"] == 5
    for extra in (["--atoms", "33"], ["--vmin", "1"], ["--vmax", "45"], ["--dist_checkpoint", "x"]):
        other = PB.parse_args(["--agent_type", "DistValueSimOnline", "--checkpoint_dir", d, "--resume"] + extra)
        with pytest.raises(ValueError, match="--" + extra[0][2:]):
            PB.read_run_state(other, 0, 1)
    old = dict(st, flags={k: v for k, v in flags.items() if k not in ("atoms", "vmin", "vmax", "dist_checkpoint")})
    PB.write_run_state(state, old)
    assert PB.read_run_state(args, 0, 1)[0]["moves"] == 5
