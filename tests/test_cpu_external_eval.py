"""The caller-supplied evaluator (eval_kind "external") where no GPU is needed: the engine refuses to start without a device, the output
adapters, the test evaluator's batch independence, and play_batched's --evaluator flag."""
import numpy as np
import pytest

from ext_eval_twins import dist_np, value_np


def test_external_engine_needs_a_device():
    from tetris_mcts_b200 import _lib as L
    from tetris_mcts_b200.engine import BatchedEngine
    if L.lib().b200_device_count() > 0:
        pytest.skip("a CUDA device is present")
    with pytest.raises(L.B200Error) as e:
        BatchedEngine(4, max_nodes=256, mode="lp", eval_kind="external")
    assert e.value.code == 2                                                    # B200_ERR_CUDA


def test_host_output_adapters():
    from tetris_mcts_b200.engine import ext_output_parts
    n = 5
    v, var = np.arange(n, dtype=np.float32), np.ones(n, np.float32)
    for res in ((v, var), [v.reshape(n, 1), var.reshape(n, 1)], (v, var.reshape(n, 1))):
        parts = ext_output_parts(res, n, 2, dist=False, host=True)
        assert [p.shape for p in parts] == [(n, 1), (n, 1)]
        assert np.array_equal(parts[0].ravel(), v) and np.array_equal(parts[1].ravel(), var)
    p = np.full((n, 7), 1 / 7, np.float32)
    for res in (p, [p], (p,)):
        (q,) = ext_output_parts(res, n, 7, dist=True, host=True)
        assert q.shape == (n, 7) and np.array_equal(q, p)
    bad_value = [(v,), (v, var, var), v, (v[:-1], var), (v.reshape(1, n), var), (v.reshape(n, 1, 1), var), (v.astype(np.float64), var),
                 (list(v), var)]
    for res in bad_value:
        with pytest.raises(ValueError):
            ext_output_parts(res, n, 2, dist=False, host=True)
    for res in ([p, p], [], p[:, :6], p[:-1], p.ravel(), p.astype(np.float16)):
        with pytest.raises(ValueError):
            ext_output_parts(res, n, 7, dist=True, host=True)


def test_numpy_twin_is_batch_independent():
    rng = np.random.default_rng(3)
    boards = rng.integers(-1, 2, size=(300, 1, 20, 10)).astype(np.int8)
    v, var = value_np(boards)
    d = dist_np(boards, 50)
    assert v.dtype == var.dtype == d.dtype == np.float32 and np.allclose(d.sum(1), 1, atol=1e-5)
    for lo, hi in ((0, 1), (7, 8), (3, 130), (299, 300), (0, 300)):
        v2, var2 = value_np(boards[lo:hi])
        assert v2.tobytes() == v[lo:hi].tobytes() and var2.tobytes() == var[lo:hi].tobytes()
        assert dist_np(boards[lo:hi], 50).tobytes() == d[lo:hi].tobytes()
    perm = rng.permutation(300)
    assert value_np(boards[perm])[0].tobytes() == v[perm].tobytes()


@pytest.mark.parametrize("extra", [["--online"], ["--agent_type", "Vanilla"]])
def test_play_batched_rejects_evaluator_combinations(extra, capsys):
    from tetris_mcts_b200.play_batched import parse_args
    with pytest.raises(SystemExit):
        parse_args(["--evaluator", "mod:make"] + extra)
    assert "--evaluator" in capsys.readouterr().err
    assert parse_args(["--evaluator", "mod:make"]).evaluator == "mod:make"
