"""play_batched's --checkpoint_dir / --resume flag checks and run state, and the Python-side reading of engine image headers, without a GPU."""
import os
import struct

import numpy as np
import pytest


def _args(*extra):
    from tetris_mcts_b200 import play_batched as PB
    return PB.parse_args(["--online", "--checkpoint_dir", "ck"] + list(extra))


def test_resume_flags_need_a_checkpoint_dir():
    from tetris_mcts_b200 import play_batched as PB
    for argv in (["--resume"], ["--checkpoint_every", "5"]):
        with pytest.raises(SystemExit):
            PB.parse_args(argv)
    with pytest.raises(SystemExit):
        PB.parse_args(["--checkpoint_dir", "ck", "--checkpoint_every", "-1"])
    with pytest.raises(SystemExit):
        PB.parse_args(["--checkpoint_dir", "ck", "--evaluator", "m:f"])
    a = PB.parse_args(["--checkpoint_dir", "ck", "--checkpoint_every", "10", "--resume"])
    assert a.resume and a.checkpoint_every == 10 and a.checkpoint_dir == "ck"


def _state(args, world=1, moves=30, **over):
    from tetris_mcts_b200 import play_batched as PB
    st = dict(world=world, flags={k: getattr(args, k) for k in PB.RESUME_FLAGS}, generation=moves, ngames=7, moves=moves, gcs=12,
              image="engine.rank0", image_bytes=64, finished=False, scores=[1, 2], lines=[0, 1],
              trainer=dict(n_trains=2, train_seconds=1.5, weights=np.arange(4, dtype=np.float32), optimizer=None),
              episode_of=np.array([3, 0, 7], np.int32), saver_chunk=4)
    st.update(over)
    return st


def _write_generation(d, args, gen, rank=0, image_bytes=64, latest=True, **over):
    """a checkpoint generation as play_batched writes it: a stand-in image of image_bytes, the run state naming it, then `latest`"""
    from tetris_mcts_b200 import play_batched as PB
    os.makedirs(PB.generation_dir(d, gen), exist_ok=True)
    image, state = PB.checkpoint_paths(d, gen, rank)
    open(image, "wb").write(b"\0" * image_bytes)
    st = _state(args, moves=gen, image="engine.rank%d" % rank, image_bytes=image_bytes)
    st.update(over)
    PB.write_run_state(state, st)
    if latest:
        PB.write_latest(d, gen)
    return image, state, st


def test_run_state_round_trip(tmp_path):
    from tetris_mcts_b200 import play_batched as PB
    args = _args("--checkpoint_dir", str(tmp_path))
    image, _path, st = _write_generation(str(tmp_path), args, 30)
    got, img = PB.read_run_state(args, 0, 1)
    assert img == image
    assert got["moves"] == 30 and got["ngames"] == 7 and got["gcs"] == 12 and got["saver_chunk"] == 4
    assert np.array_equal(got["episode_of"], st["episode_of"]) and np.array_equal(got["trainer"]["weights"], st["trainer"]["weights"])
    # the resumed run may stop elsewhere and checkpoint at another rate
    assert PB.read_run_state(_args("--checkpoint_dir", str(tmp_path), "--max_moves", "99", "--checkpoint_every", "3"), 0, 1)[0]["moves"] == 30


def test_resume_refuses_a_missing_checkpoint_or_other_settings(tmp_path):
    from tetris_mcts_b200 import play_batched as PB
    args = _args("--checkpoint_dir", str(tmp_path))
    with pytest.raises(ValueError, match="no checkpoint"):
        PB.read_run_state(args, 0, 1)
    _write_generation(str(tmp_path), args, 30)
    for extra, names in ((["--n_parallel", "128"], ["--n_parallel"]), (["--seed", "5", "--max_nodes", "2048"], ["--seed", "--max_nodes"]),
                         (["--agent_type", "ValueSim"], ["--agent_type"]), (["--train_kind", "tf32", "--eval_kind", "net_fp16"],
                                                                            ["--train_kind", "--eval_kind"]),
                         (["--memory_size", "10", "--accumulation_policy", "0"], ["--memory_size", "--accumulation_policy"])):
        with pytest.raises(ValueError) as ei:
            PB.read_run_state(_args("--checkpoint_dir", str(tmp_path), *extra), 0, 1)
        for n in names:
            assert n in str(ei.value)
    with pytest.raises(ValueError, match="world size"):
        PB.read_run_state(args, 0, 2)


def test_resume_refuses_files_of_two_generations(tmp_path):
    """a stale run state next to a newer image, an image that is not the one its run state names, a run state of another move, and
    ranks that found different generations are all refused"""
    from tetris_mcts_b200 import play_batched as PB
    d = str(tmp_path)
    args = _args("--checkpoint_dir", d)
    image, state, _st = _write_generation(d, args, 30)
    open(image, "wb").write(b"\0" * 80)                                   # a newer image over the generation's own
    with pytest.raises(ValueError, match="not the one the run state"):
        PB.read_run_state(args, 0, 1)
    os.remove(image)
    with pytest.raises(ValueError, match="not the one the run state"):
        PB.read_run_state(args, 0, 1)
    _write_generation(d, args, 40, generation=30, moves=30)                # a run state of move 30 inside generation 40
    with pytest.raises(ValueError, match="not of generation 40"):
        PB.read_run_state(args, 0, 1)
    _write_generation(d, args, 50, latest=False)                           # written, but `latest` was never moved to it
    _write_generation(d, args, 40)
    assert PB.read_run_state(args, 0, 1)[0]["moves"] == 40
    assert PB.agree_on_generation([(40, None), (40, None)]) == 40
    with pytest.raises(ValueError, match="different moves"):
        PB.agree_on_generation([(40, None), (30, None)])
    with pytest.raises(ValueError, match="rank 1: boom"):
        PB.agree_on_generation([(40, None), (None, "boom")])


def test_resume_refuses_a_finished_run(tmp_path):
    from tetris_mcts_b200 import play_batched as PB
    args = _args("--checkpoint_dir", str(tmp_path))
    _write_generation(str(tmp_path), args, 30, finished=True)
    with pytest.raises(ValueError, match="had finished"):
        PB.read_run_state(args, 0, 1)


def test_checkpoint_housekeeping(tmp_path):
    """older generations go once `latest` names a newer one; a resumed run drops the --save chunks written after its checkpoint"""
    from tetris_mcts_b200 import play_batched as PB
    d = str(tmp_path)
    args = _args("--checkpoint_dir", d)
    _write_generation(d, args, 30)
    _write_generation(d, args, 40)
    _write_generation(d, args, 40, rank=1, latest=False)
    _write_generation(d, args, 30, rank=1, latest=False)
    PB.drop_older_generations(d, 40, 0)
    assert os.path.isdir(PB.generation_dir(d, 30)) and not os.path.exists(PB.checkpoint_paths(d, 30, 0)[1])
    PB.drop_older_generations(d, 40, 1)
    assert not os.path.exists(PB.generation_dir(d, 30)) and os.path.isfile(PB.checkpoint_paths(d, 40, 1)[0])
    base = os.path.join(d, "data0")
    for i in range(5):
        np.save("%s.%06d.npy" % (base, i), np.zeros(2))
    np.save("%s.rank0.%06d.npy" % (base, 4), np.zeros(2))
    PB.drop_later_chunks(base, 3)
    assert sorted(os.listdir(d)).count("data0.000002.npy") == 1 and not os.path.exists("%s.000003.npy" % base)
    assert not os.path.exists("%s.000004.npy" % base) and os.path.exists("%s.rank0.000004.npy" % base)


def _image(fields, version=1, magic=b"B200SNAP", arena=True):
    b = magic + struct.pack("<II", version, 0x01020304)
    for fid, payload in fields:
        b += struct.pack("<IIQ", fid, 0, len(payload)) + payload + b"\0" * 8
    if arena:
        b += struct.pack("<IIQ", 128, 0, 0)
    return b


def _config_fields(**over):
    from tetris_mcts_b200 import engine as E
    vals = dict(n_games=4, max_nodes=64, mode=0, low=1, lp_end_from_obs=0, lp_var_gamma2=1, stale_pop=1, overflow_reset=0, eval_kind=0,
                trace_max=512, actions_per_drop=1, scoring=0, randomizer=0, device=0, seed=123, gamma=0.999, rollout_variance=1e3, dist_bins=50,
                dist_vmin=0.0, dist_vmax=5000.0, path_cache=1)
    vals.update(over)
    out = []
    for fid, (name, real) in E.IMAGE_SCALARS.items():
        if name in vals:
            out.append((fid, struct.pack("<d" if real else "<q", vals[name])))
    return out


def test_image_header_parse(tmp_path):
    from tetris_mcts_b200.engine import read_image_fields
    p = tmp_path / "x.img"
    p.write_bytes(_image(_config_fields(n_games=9, gamma=0.5) + [(40, b"\0" * 16)]))   # a blob field is skipped
    f = read_image_fields(str(p))
    assert f["n_games"] == 9 and f["gamma"] == 0.5 and f["path_cache"] == 1 and f["seed"] == 123


@pytest.mark.parametrize("blob,msg", [
    (lambda: _image(_config_fields(), magic=b"NOTSNAP!"), "wrong magic"),
    (lambda: _image(_config_fields(), version=2), "format version 2"),
    (lambda: _image(_config_fields())[:30], "truncated"),
    (lambda: _image(_config_fields(), arena=False), "truncated"),
    (lambda: _image([f for f in _config_fields() if f[0] != 3]), "mode"),
    (lambda: b"B200", "truncated header"),
])
def test_image_header_refusals(tmp_path, blob, msg):
    from tetris_mcts_b200.engine import read_image_fields
    p = tmp_path / "bad.img"
    p.write_bytes(blob())
    with pytest.raises(ValueError, match=msg):
        read_image_fields(str(p))


def test_load_without_a_device_raises(tmp_path):
    """the image is read by the library: with no CUDA device that is an error, never a CPU path"""
    import tetris_mcts_b200._lib as L
    from tetris_mcts_b200.engine import BatchedEngine
    try:
        L.lib()
    except ImportError:
        pytest.skip("library not built")
    if L.lib().b200_device_count() > 0:
        pytest.skip("a CUDA device is present")
    p = tmp_path / "x.img"
    p.write_bytes(_image(_config_fields()) + struct.pack("<Q", 4) + b"\0" * 40)
    with pytest.raises(L.B200Error):
        BatchedEngine.load(str(p))
