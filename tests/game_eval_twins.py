"""Test helpers for eval_kind external_game: one deterministic leaf-game evaluator, stated once for numpy records (the reference's agent.cpp,
the C oracle and host evaluators) and once for torch records on the device, and CPU restatements of the device game calls.

evaluate(rec) = (v, var) of one packed record (SPEC_PYTETRIS §6):
  v   = score + popcount(board words) % 13 + 4 * line_clears
  var = 50 + 7 * piece + (score % 5)
and with special=True a designed share of the leaves, chosen by h = (popcount + piece word + rng word) % 11, gets
  h == 0: v = NaN;  h == 1: v = +inf;  h == 2: v = -inf;  h == 3: v = -v - 1;  h == 4: var = NaN;  h == 5: var = -var.
Every value is an integer below 2^24 or special, so float32 holds it exactly (the gamma = 1 golden's integer outputs).

GameEvalAgent drives an oracle agent (oracle_py.Agent, MODE_VANILLA) with such an evaluator in place of its rollout (tests/game_eval_oracle.c)."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

REC_WORDS = 20

# agent_type1_golden.npz: the first evaluation (global index in c<k>_eval_recs) at which the reference's agent.cpp walks differently from the
# oracle and the engine.  backup_obs_single (agent.cpp:496-513) carries the backed-up value in float, core.h:226-260 and k_backup in double,
# so at gamma 0.99 the statistics differ in low bits and, after enough simulations, a near tie in policy_clt resolves the other way.  With
# gamma 1 and integer outputs both chains are exact and the case agrees to its end, as does the NaN / inf case.  Up to these points every
# action, record and evaluator input agrees; a float-chain restatement of the same loop reproduces both cases to their ends.
FLOAT_CHAIN_DIVERGENCE = {0: 1428, 1: None, 2: 291, 3: None}


def golden_span(z, case):
    """(moves, evaluations) of golden case `case` that the double-chain search must reproduce: everything before the first diverging
    evaluation (all of it where there is none)"""
    p = "c%d_" % case
    off = z[p + "eval_off"]
    d = FLOAT_CHAIN_DIVERGENCE[case]
    if d is None:
        return len(z[p + "actions"]), int(off[-1])
    return int(np.searchsorted(off, d, side="right")) - 1, d


def _popcount32(x):
    x = x.astype(np.uint64)
    c = np.zeros(x.shape, np.int64)
    for b in range(32):
        c += ((x >> np.uint64(b)) & np.uint64(1)).astype(np.int64)
    return c


def evaluate_batch(recs, special=False):
    """numpy uint32 [n,20] -> (v float32 [n], var float32 [n])"""
    r = np.asarray(recs, np.uint32).reshape(-1, REC_WORDS)
    pop = _popcount32(r[:, :10]).sum(axis=1)
    score = r[:, 13].view(np.int32).astype(np.int64)
    lines = r[:, 14].view(np.int32).astype(np.int64)
    piece = (r[:, 10] & 7).astype(np.int64)
    v = (score + pop % 13 + 4 * lines).astype(np.float32)
    var = (50 + 7 * piece + score % 5).astype(np.float32)
    if special:
        h = (pop + r[:, 10].astype(np.int64) + r[:, 12].astype(np.int64)) % 11
        v = np.where(h == 0, np.float32(np.nan), np.where(h == 1, np.float32(np.inf), np.where(h == 2, np.float32(-np.inf),
                     np.where(h == 3, -v - 1, v)))).astype(np.float32)
        var = np.where(h == 4, np.float32(np.nan), np.where(h == 5, -var, var)).astype(np.float32)
    return v, var


def evaluate(rec, special=False):
    v, var = evaluate_batch(np.asarray(rec, np.uint32).reshape(1, REC_WORDS), special)
    return float(v[0]), float(var[0])


def evaluate_torch(recs, special=False):
    """the same on torch int32 [n,20] records on any device -> (v, var) float32 [n]"""
    import torch
    r = recs.to(torch.int64) & 0xffffffff
    pop = torch.zeros(r.shape[0], dtype=torch.int64, device=r.device)
    for b in range(32):
        pop += ((r[:, :10] >> b) & 1).sum(dim=1)
    score = recs[:, 13].to(torch.int64)
    lines = recs[:, 14].to(torch.int64)
    piece = r[:, 10] & 7
    v = (score + pop % 13 + 4 * lines).to(torch.float32)
    var = (50 + 7 * piece + torch.remainder(score, 5)).to(torch.float32)
    if special:
        h = (pop + r[:, 10] + r[:, 12]) % 11
        v = torch.where(h == 0, torch.full_like(v, float("nan")), torch.where(h == 1, torch.full_like(v, float("inf")),
                        torch.where(h == 2, torch.full_like(v, float("-inf")), torch.where(h == 3, -v - 1, v))))
        var = torch.where(h == 4, torch.full_like(var, float("nan")), torch.where(h == 5, -var, var))
    return v, var


def xorshift32(s):
    s ^= (s << 13) & 0xffffffff
    s ^= s >> 17
    s ^= (s << 5) & 0xffffffff
    return s


def playout_cpu(game_cls, rec, state, n_actions, max_steps):
    """CPU restatement of b200_tetris_playout_dev for one row on the oracle env: (final record, final stream, steps)."""
    g = game_cls(record=np.asarray(rec, np.uint32))
    s = int(state) & 0xffffffff or 0x2545F491
    k = 0
    while not g.end and k < max_steps:
        s = xorshift32(s)
        g.play(s % n_actions)
        k += 1
    return g.record(), s, k


# ---------------------------------------------------------------------------------------------------- the oracle agent with a game evaluator
HERE = os.path.dirname(os.path.abspath(__file__))
ORACLE = os.path.join(os.path.dirname(HERE), "oracle")
ORACLE_C = ("tetris_oracle.c", "valuenet_oracle.c", "dist_oracle.c", "distnet_oracle.c")   # oracle/Makefile's sources besides mcts_oracle.c
GAME_EVAL_CB = C.CFUNCTYPE(None, C.c_void_p, C.POINTER(C.c_uint32), C.POINTER(C.c_float), C.POINTER(C.c_float))
_ge_lib = None


def game_eval_lib():
    """tests/game_eval_oracle.c (which includes oracle/mcts_oracle.c) built with the oracle Makefile's CFLAGS into a temporary directory"""
    global _ge_lib
    if _ge_lib is None:
        so = os.path.join(tempfile.mkdtemp(prefix="game_eval_oracle"), "game_eval_oracle.so")
        subprocess.run(["gcc", "-O2", "-fPIC", "-std=c11", "-ffp-contract=off", "-shared", "-I", ORACLE, os.path.join(HERE, "game_eval_oracle.c")]
                       + [os.path.join(ORACLE, f) for f in ORACLE_C] + ["-o", so, "-lm"], check=True)
        L = C.CDLL(so)
        L.ge_agent_mcts.argtypes = [C.c_void_p, C.c_int, GAME_EVAL_CB, C.c_void_p]
        L.ge_agent_rng.argtypes = [C.c_void_p]
        L.ge_agent_rng.restype = C.c_uint32
        _ge_lib = L
    return _ge_lib


class GameEvalAgent:
    """An oracle_py.Agent in mode 2 (Vanilla) whose mcts() scores each expanded leaf with f(rec uint32[20]) -> (value, variance), as
    agent.cpp's evaluator type 1 does, instead of rolling it out.  Every other method is the wrapped agent's."""

    def __init__(self, agent, f):
        self.agent = agent

        def tramp(ctx, rec, v, var):
            rv, rvar = f(np.ctypeslib.as_array(rec, shape=(REC_WORDS,)).copy())
            v[0], var[0] = float(rv), float(rvar)
        self._cb = GAME_EVAL_CB(tramp)

    def mcts(self, sims):
        rc = game_eval_lib().ge_agent_mcts(self.agent.h, int(sims), self._cb, None)
        if rc != 0:
            raise RuntimeError("oracle agent with a game evaluator: rc=%d" % rc)

    def rng(self):
        return int(game_eval_lib().ge_agent_rng(self.agent.h))

    def __getattr__(self, name):
        return getattr(self.agent, name)
