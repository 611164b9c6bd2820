"""pyTetris.Tetris — drop-in for the (absent, third-party) hrpan/pyTetris module consumed by the reference:
play.py:1,75-76,150,169, agents/agent.py:70,103,114,143-144.  The object is a handle around the 80-byte packed
record of SPEC_PYTETRIS.md §6.  Construction, reset(), play() and getState() all run on the GPU through the C-ABI
(b200_tetris_new / b200_tetris_step / b200_tetris_state); no rule of the game is implemented on the host.

The `_dev` functions below work on records that stay on the device (torch int32 [n, 20], e.g. the leaf games an eval_kind
"external_game" engine hands to its game evaluator): they enqueue one kernel on the current torch stream and return."""
import ctypes as C

import numpy as np

from . import _lib as L


class Tetris:
    __slots__ = ("_rec", "_args")

    def __init__(self, boardsize=(20, 10), actions_per_drop=1, scoring=0, randomizer=0, _record=None):
        if tuple(boardsize) != (20, 10):
            raise ValueError("only 20x10 boards are supported (SPEC_PYTETRIS.md §1)")
        self._args = (int(actions_per_drop), int(scoring), int(randomizer))
        if _record is not None:
            self._rec = np.ascontiguousarray(_record, np.uint32).copy()
        else:
            self._rec = new_games(1, self._args, None)[0]

    # ---- state-changing calls: all on the device
    def play(self, action):
        a = np.array([int(action)], np.int32)
        L.check(L.lib().b200_tetris_step(L.ptr(self._rec), L.ptr(a), 1))

    def reset(self):
        L.check(L.lib().b200_tetris_new(L.ptr(self._rec), 1, *self._args, None, 1))

    def seed(self, s):
        self._rec = new_games(1, self._args, np.array([int(s) & 0xffffffff], np.uint32))[0]

    def copy_from(self, other):
        self._rec[:] = other._rec
        self._args = other._args

    def clone(self):
        return Tetris((20, 10), *self._args, _record=self._rec)

    def equiv(self, other):
        return bool(np.array_equal(self._rec, other._rec))

    def __eq__(self, other):
        return isinstance(other, Tetris) and bool(np.array_equal(self._rec, other._rec))

    def __hash__(self):
        return hash(self._rec.tobytes())

    def hash(self):
        return hash(self._rec.tobytes()) & 0xffffffffffffffff

    # ---- observation (agents/agent.py:116)
    def getState(self):
        out = np.zeros((20, 10), np.int8)
        L.check(L.lib().b200_tetris_state(L.ptr(self._rec), L.ptr(out), 1))
        return out

    def _getState(self):
        return self.getState().ravel().tolist()

    def printState(self):
        for row in self.getState():
            print("".join("." if v == 0 else ("#" if v > 0 else "o") for v in row))

    def getScore(self):
        return self.score

    def get_record(self):
        return self._rec.copy()

    def set_record(self, rec):
        self._rec[:] = np.asarray(rec, np.uint32)

    # ---- attributes read by play.py:144-148, util/Data.py:74-77 (decoded from the record, SPEC §6)
    @property
    def end(self):
        return bool((int(self._rec[10]) >> 21) & 1)

    @property
    def score(self):
        return int(np.int32(self._rec[13]))

    @property
    def combo(self):
        return int(self._rec[11]) >> 8

    @property
    def line_clears(self):
        return int(np.int32(self._rec[14]))

    @property
    def line_stats(self):
        return self._rec[15:19].astype(np.int32)


def new_games(n, env_args=(1, 0, 0), seeds=None):
    """n fresh packed games built on the device; seeds: uint32[n] or None (default seed)."""
    if len(env_args) == 4:
        env_args = env_args[1:]
    recs = np.zeros((n, L.REC_WORDS), np.uint32)
    s = None if seeds is None else np.ascontiguousarray(seeds, np.uint32)
    L.check(L.lib().b200_tetris_new(L.ptr(recs), int(n), int(env_args[0]), int(env_args[1]), int(env_args[2]), L.ptr(s), 0))
    return recs


def step_games(recs, actions):
    """Tetris.play over a batch of packed games (in place)."""
    recs = np.ascontiguousarray(recs, np.uint32)
    a = np.ascontiguousarray(actions, np.int32)
    L.check(L.lib().b200_tetris_step(L.ptr(recs), L.ptr(a), len(a)))
    return recs


def states_of(recs):
    recs = np.ascontiguousarray(recs, np.uint32).reshape(-1, L.REC_WORDS)
    out = np.zeros((len(recs), 20, 10), np.int8)
    L.check(L.lib().b200_tetris_state(L.ptr(recs), L.ptr(out), len(recs)))
    return out


# ---------------------------------------------------------------------------------------------------- games on the device
def _recs_dev(recs, name="recs"):
    import torch
    if not isinstance(recs, torch.Tensor) or recs.dtype != torch.int32 or recs.device.type != "cuda":
        raise ValueError("%s: a torch int32 tensor on a CUDA device; got %s" % (
            name, (recs.dtype, recs.device) if isinstance(recs, torch.Tensor) else type(recs).__name__))
    if recs.dim() != 2 or recs.shape[1] != L.REC_WORDS or not recs.is_contiguous() or recs.data_ptr() % 16:
        raise ValueError("%s: a contiguous, 16-byte aligned [n, %d] tensor; got shape %s" % (name, L.REC_WORDS, tuple(recs.shape)))
    return recs


def _same_device(t, recs, dtype, shape, name):
    import torch
    if not isinstance(t, torch.Tensor) or t.dtype != dtype or t.device != recs.device or tuple(t.shape) != shape or not t.is_contiguous():
        raise ValueError("%s: a contiguous %s tensor of shape %s on %s" % (name, dtype, shape, recs.device))
    return t


def _stream(recs):
    import torch
    return C.c_void_p(torch.cuda.current_stream(recs.device).cuda_stream)


def step_games_dev(recs, actions):
    """Tetris.play of every row of recs (torch int32 [n, 20] on a CUDA device, changed in place) with actions (int32 [n], same device;
    ids outside 0..6 move nothing), enqueued on the current stream."""
    import torch
    recs = _recs_dev(recs)
    actions = _same_device(actions, recs, torch.int32, (recs.shape[0],), "actions")
    L.check(L.lib().b200_tetris_step_dev(C.c_void_p(recs.data_ptr()), C.c_void_p(actions.data_ptr()), recs.shape[0], _stream(recs)))
    return recs


def states_of_dev(recs, dtype="float32", out=None):
    """getState() of every row of recs as a [n, 1, 20, 10] tensor ("float32" or "int8") on the records' device: the boards an eval_kind
    "external" engine hands to its evaluator (board bits, -1 on the falling piece), enqueued on the current stream."""
    import torch
    recs = _recs_dev(recs)
    tdt = {"float32": torch.float32, "int8": torch.int8}[dtype]
    n = recs.shape[0]
    out = torch.empty((n, 1, 20, 10), dtype=tdt, device=recs.device) if out is None else _same_device(out, recs, tdt, (n, 1, 20, 10), "out")
    kind = L.BOARD_F32 if dtype == "float32" else L.BOARD_INT8
    L.check(L.lib().b200_tetris_state_dev(C.c_void_p(recs.data_ptr()), C.c_void_p(out.data_ptr()), kind, n, _stream(recs)))
    return out


def playout_dev(recs, rng, n_actions=7, max_steps=2**31 - 1):
    """Random playouts of every row of recs in place (the rollout's loop): row i plays xorshift32(rng[i]) % n_actions (1..8; 8 includes the
    no-op 7, VanillaC's randint(0, 7)) until game over or after max_steps actions.  rng (int32 [n] xorshift32 states, same device) is
    advanced in place; a state of 0 starts as 0x2545F491.  Returns int32 [n], the actions each row played.  Enqueued on the current stream."""
    import torch
    recs = _recs_dev(recs)
    n = recs.shape[0]
    rng = _same_device(rng, recs, torch.int32, (n,), "rng")
    steps = torch.empty(n, dtype=torch.int32, device=recs.device)
    L.check(L.lib().b200_tetris_playout_dev(C.c_void_p(recs.data_ptr()), C.c_void_p(rng.data_ptr()), n, int(n_actions), int(max_steps),
                                            C.c_void_p(steps.data_ptr()), _stream(recs)))
    return steps


def record_fields(recs):
    """end, score, line_clears and combo of packed records (SPEC_PYTETRIS §6), decoded from their word offsets with torch bit operations:
    a dict of [n] int32 tensors on the records' device, or of numpy int32 arrays for a numpy [n, 20] uint32 / int32 input."""
    import torch
    host = isinstance(recs, np.ndarray)
    r = torch.from_numpy(np.ascontiguousarray(recs).reshape(-1, L.REC_WORDS).view(np.int32)) if host else recs
    out = {"end": (r[:, 10] >> 21) & 1, "score": r[:, 13], "line_clears": r[:, 14], "combo": (r[:, 11] >> 8) & 0xffffff}
    return {k: (v.numpy().astype(np.int32) if host else v) for k, v in out.items()}


def per_game(f):
    """A host game evaluator (BatchedEngine.run_sims(game_evaluator=, host=True)) from a reference-style f(Tetris) -> (value, variance),
    e.g. VanillaC's random_playout unchanged: f gets one Tetris per leaf record, built from a copy, and the results come back as float32.
    This is the drop-in for existing code, not a fast path: every Tetris.play is a device round trip."""
    def evaluate(recs):
        recs = np.asarray(recs, np.uint32).reshape(-1, L.REC_WORDS)
        v = np.zeros(len(recs), np.float32)
        var = np.zeros(len(recs), np.float32)
        for i, rec in enumerate(recs):
            v[i], var[i] = f(Tetris(_record=rec))
        return v, var
    return evaluate


def playout_evaluator(n_actions=7, variance=1e5, seed=0, max_steps=2**31 - 1):
    """A device game evaluator that scores each leaf record by one random playout (playout_dev) and returns (score, variance): with
    n_actions=8 and variance=1e5 it is VanillaC's random_playout, restated on the device.  Row i of the c-th call starts its stream from a
    hash of (seed, c, i, the record's piece-stream word), so two runs from the same start give the same playouts."""
    import torch
    calls = [0]

    def evaluate(recs):
        n = recs.shape[0]
        row = torch.arange(n, dtype=torch.int64, device=recs.device)
        x = (recs[:, 12].to(torch.int64) & 0xffffffff) ^ ((row * 0x9E3779B1 + calls[0] * 0x85EBCA77 + int(seed) * 0xC2B2AE3D) & 0xffffffff)
        x = ((x ^ (x >> 16)) * 0x45D9F3B) & 0xffffffff
        x = ((x ^ (x >> 16)) * 0x45D9F3B) & 0xffffffff
        x = x ^ (x >> 16)
        rng = torch.where(x >= 2**31, x - 2**32, x).to(torch.int32)       # the same 32 bits as int32
        calls[0] += 1
        games = recs.clone()
        playout_dev(games, rng, n_actions, max_steps)
        v = games[:, 13].to(torch.float32)
        return v, torch.full_like(v, float(variance))
    return evaluate
