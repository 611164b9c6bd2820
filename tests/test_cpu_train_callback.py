"""The caller's training function (OnlineMCTSAgent's train callback): play_batched --trainer's argument checks, ValueSim's train= switch, the
device form of the replay re-layout and the forms of weights a callback may return.  No device needed."""
import numpy as np
import pytest


def _error(capsys, argv):
    from tetris_mcts_b200 import play_batched as PB
    with pytest.raises(SystemExit):
        PB.parse_args(argv)
    return capsys.readouterr().err


ONLINE = ["--online", "--trainer", "mytraining:make_trainer"]


@pytest.mark.parametrize("extra,msg", [
    (["--trainer", "m:f"], "--trainer needs --online"),
    (ONLINE + ["--agent_type", "Vanilla"], "--trainer cannot be combined with --agent_type Vanilla"),
    (ONLINE + ["--checkpoint_dir", "ckpt"], "--checkpoint_dir cannot be combined with --trainer"),
    (["--online", "--trainer", "no_colon"], "--trainer takes MODULE:FACTORY"),
    (ONLINE + ["--train_kind", "tf32"], "--trainer cannot be combined with --train_kind"),
    (ONLINE + ["--train_kind", "fp64"], "--trainer cannot be combined with --train_kind"),           # the default value, set explicitly
    (ONLINE + ["--train_batch_size", "256"], "--trainer cannot be combined with --train_batch_size"),
    (ONLINE + ["--train_max_iters=100"], "--trainer cannot be combined with --train_max_iters"),
    (ONLINE + ["--train_k", "tc"], "--trainer cannot be combined with --train_kind"),                # an abbreviation argparse accepts
    (ONLINE + ["--train_batch_size", "8", "--train_max_iters", "9"], "--train_batch_size, --train_max_iters"),
    (["--online", "--trainer_host"], "--trainer_host needs --trainer"),
])
def test_trainer_refusals(capsys, extra, msg):
    assert msg in _error(capsys, extra)


def test_evaluator_with_online_stays_refused_without_trainer(capsys):
    err = _error(capsys, ["--evaluator", "m:f", "--online"])
    assert "--evaluator cannot be combined with --online: the online trainer trains the built-in Model_VV weights" in err
    assert "--checkpoint_dir cannot be combined with --trainer" in _error(capsys, ["--evaluator", "m:f", "--online", "--trainer", "a:b",
                                                                                  "--checkpoint_dir", "c"])


def test_trainer_accepted():
    from tetris_mcts_b200 import play_batched as PB
    a = PB.parse_args(ONLINE + ["--evaluator", "mynets:make_evaluator", "--trainer_host"])
    assert (a.trainer, a.evaluator, a.trainer_host, a.online) == ("mytraining:make_trainer", "mynets:make_evaluator", True, True)
    a = PB.parse_args(ONLINE + ["--eval_kind", "net_fp16", "--accumulation_policy", "2", "--memory_size", "100"])
    assert a.trainer and a.evaluator is None and a.train_kind == "fp64" and not a.trainer_host
    assert PB.parse_args(["--online"]).trainer is None


def test_valuesim_evaluator_online_without_train_is_refused():
    from tetris_mcts_b200.agents.ValueSim import ValueSim
    from tetris_mcts_b200.agents.ValueSimLP import ValueSimLP
    for cls in (ValueSim, ValueSimLP):
        with pytest.raises(ValueError) as ei:
            cls(online=True, evaluator=lambda b: None)
        assert str(ei.value) == "online=True trains the engine's Model_VV weights on the device, not the caller's evaluator: pass online=False"


def _extreme_rows(n, seed):
    from tetris_mcts_b200 import replay
    rng = np.random.default_rng(seed)
    rows = np.zeros((n, replay.SAMPLE_BYTES), np.uint8)
    rows[:, :200] = rng.integers(-1, 2, (n, 200)).astype(np.int8).view(np.uint8)
    special = np.array([np.nan, -np.nan, np.inf, -np.inf, 0.0, -0.0, 1e-45, -1e-45, 1.17e-38, 3.4028235e38, -3.4028235e38, 5.877e-39],
                       np.float32)
    tail = rng.normal(0, 1e3, (n, 3)).astype(np.float32)
    tail.ravel()[:min(tail.size, 3 * len(special))] = np.resize(special, min(tail.size, 3 * len(special)))
    bits = tail.view(np.uint32)
    bits[-1, :] = [0x7fc00001, 0xffbfffff, 0x00000001]       # NaN payloads and the smallest subnormal keep their bits
    rows[:, 200:212] = tail.view(np.uint8).reshape(n, 12)
    return rows


@pytest.mark.parametrize("n", [0, 1, 2, 37, 1000])
def test_device_relayout_is_rows_to_memory_bit_for_bit(n):
    import torch
    from tetris_mcts_b200 import replay
    rows = _extreme_rows(max(n, 1), n)[:n]
    if n >= 37:
        assert set(np.unique(rows[:, :200].view(np.int8))) == {-1, 0, 1}
    want = replay.rows_to_memory(rows)
    buf = torch.from_numpy(np.concatenate([rows, np.full((5, 212), 0xAB, np.uint8)]))   # a larger buffer, as the trainer's is
    got = replay.rows_to_memory_dev(buf[:n])
    assert len(got) == 4
    for g, w in zip(got, want):
        assert g.dtype == torch.float32 and g.is_contiguous() and tuple(g.shape) == w.shape
        assert g.numpy().tobytes() == w.tobytes()
    assert tuple(got[0].shape) == (n, 1, 20, 10) and all(tuple(g.shape) == (n, 1) for g in got[1:])


def test_returned_weights_forms():
    import torch
    from tetris_mcts_b200 import _lib as L
    from tetris_mcts_b200.model.model_vv import init_weights, weights_to_state_dict
    from tetris_mcts_b200.online import weights_vector
    w = init_weights(4)
    assert np.array_equal(weights_vector(w), w) and weights_vector(w) is not w
    assert np.array_equal(weights_vector(torch.from_numpy(w)), w)
    sd = weights_to_state_dict(w)
    assert np.array_equal(weights_vector(sd), w)
    sd["extra.buffer"] = torch.zeros(3)                             # keys outside Model_VV's are ignored, as Model.load ignores them
    assert np.array_equal(weights_vector(sd), w)
    bad_shape = dict(sd, **{"head.fc1.weight": torch.zeros(256, 1791)})
    no_bounds = {k: v for k, v in sd.items() if k != "out_lbound"}
    for bad, msg in ((w[:-1], "float32 weights of shape (%d,)" % L.N_WEIGHTS), (w.astype(np.float64), "float32 weights"),
                     (w.reshape(2, -1), "float32 weights"), (list(w[:3]), "got list"), (5, "got int"),
                     (bad_shape, "head.fc1.weight"), (no_bounds, "has no out_lbound")):
        with pytest.raises(ValueError) as ei:
            weights_vector(bad)
        assert msg in str(ei.value)
