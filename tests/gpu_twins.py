"""numpy-in / numpy-out wrappers over the C-ABI twins of agents/cppmodule/core.cpp:20-26 (used by the -m gpu tests)."""
import ctypes as C

import numpy as np

from tetris_mcts_b200 import _lib as L


def select_trace_obs(index, child, visit, value, variance, score, n2o, low, rng_state=None, max_trace=512):
    tr = np.zeros(max_trace, np.int32)
    n = np.zeros(1, np.int32)
    L.check(L.lib().b200_select_trace_obs(int(index), L.ptr(child), L.ptr(visit), L.ptr(value), L.ptr(variance), L.ptr(score),
                                          L.ptr(n2o), child.shape[0], int(low), L.ptr(rng_state), L.ptr(tr), max_trace, L.ptr(n)))
    return tr[:int(n[0])].copy()


def backup_trace_obs(trace, visit, value, variance, n2o, score, v, var, gamma):
    trace = np.ascontiguousarray(trace, np.int32)
    L.check(L.lib().b200_backup_trace_obs(L.ptr(trace), len(trace), L.ptr(visit), L.ptr(value), L.ptr(variance), L.ptr(n2o),
                                          L.ptr(score), len(visit), float(v), float(var), float(gamma)))


def backup_trace_obs_LP(trace, visit, value, variance, n2o, score, end, c_nodes, c_obs, v, var, gamma, mixture, averaged):
    trace = np.ascontiguousarray(trace, np.int32)
    cn = np.ascontiguousarray(c_nodes, np.int32)
    co = np.ascontiguousarray(c_obs, np.int32)
    v = np.ascontiguousarray(v, np.float32)
    var = np.ascontiguousarray(var, np.float32)
    end = np.ascontiguousarray(end, np.uint8)
    L.check(L.lib().b200_backup_trace_obs_LP(L.ptr(trace), len(trace), L.ptr(visit), L.ptr(value), L.ptr(variance), L.ptr(n2o),
                                             L.ptr(score), L.ptr(end), len(visit), L.ptr(cn), L.ptr(co), len(cn), L.ptr(v),
                                             L.ptr(var), float(gamma), int(mixture), int(averaged)))


def get_unique_child_obs(index, child, score, n2o):
    cn = np.zeros(7, np.int32)
    co = np.zeros(7, np.int32)
    k = np.zeros(1, np.int32)
    L.check(L.lib().b200_get_unique_child_obs(int(index), L.ptr(child), L.ptr(score), L.ptr(n2o), child.shape[0], L.ptr(cn),
                                              L.ptr(co), L.ptr(k)))
    return cn[:int(k[0])].copy(), co[:int(k[0])].copy()


def get_all_childs(index, child):
    mark = np.zeros(child.shape[0], np.uint8)
    L.check(L.lib().b200_get_all_childs(int(index), L.ptr(child), child.shape[0], L.ptr(mark)))
    return set(np.nonzero(mark)[0].tolist())


def debug_backup(eng, c, pc_len=None):
    """The production k_backup on case c (tests/backup_edges.py layout) through b200_debug_backup on the one-game engine `eng`.
    Returns (visit, value, variance) and, with pc_len given (the path cache on), a dict of what the backup left in the cache."""
    visit, value, variance = c["visit"].copy(), c["value"].copy(), c["variance"].copy()
    child = np.ascontiguousarray(c["child"], np.int32)
    M, D = child.shape[0], len(c["trace"])
    ev = np.ascontiguousarray(c["ev"], np.float32)
    pc = None
    if pc_len is not None:
        pc = dict(pc_len=np.array([pc_len], np.int32), own=np.zeros((D, 4), np.int32), sib=np.zeros((D, 8), np.uint16),
                  ent=np.zeros((D, 8, 4), np.int32), var=np.zeros((D, 8), np.int32))
    g = pc or {}
    L.check(L.lib().b200_debug_backup(eng.h, M, L.ptr(child), L.ptr(np.ascontiguousarray(c["n2o"], np.int32)),
                                      L.ptr(np.ascontiguousarray(c["score"], np.float32)), L.ptr(visit), L.ptr(value), L.ptr(variance),
                                      L.ptr(np.ascontiguousarray(c["end"], np.uint8)), L.ptr(np.ascontiguousarray(c["trace"], np.int32)), D,
                                      int(c["kind"]), L.ptr(ev), float(c["rollout"]), L.ptr(g.get("pc_len")), L.ptr(g.get("own")),
                                      L.ptr(g.get("sib")), L.ptr(g.get("ent")), L.ptr(g.get("var"))))
    return (visit, value, variance), pc


def ztab(n):
    """The walk's z(n) on the device (search_dev.cuh ztab) for an int32 array of n."""
    n = np.ascontiguousarray(n, np.int32)
    out = np.empty(len(n), np.float32)
    L.check(L.lib().b200_debug_ztab(L.ptr(n), len(n), L.ptr(out)))
    return out


def debug_load_tree(eng, game, c):
    """Game `game` of engine `eng` set to the tree of case c (tests/select_edges.py layout) through b200_debug_load_tree: root c["root"],
    check_low stream c["seed"], every childless node terminal."""
    L.check(L.lib().b200_debug_load_tree(eng.h, int(game), len(c["n2o"]), L.ptr(c["child"]), L.ptr(c["n2o"]), L.ptr(c["score"]),
                                         L.ptr(c["visit"]), L.ptr(c["value"]), L.ptr(c["variance"]), L.ptr(c["end"]), int(c["root"]),
                                         int(c["seed"])))


def debug_game_state(eng, game):
    """(check_low stream state, path cache valid length) of one game."""
    rng, pcl = np.zeros(1, np.uint32), np.zeros(1, np.int32)
    L.check(L.lib().b200_debug_game_state(eng.h, int(game), L.ptr(rng), L.ptr(pcl)))
    return int(rng[0]), int(pcl[0])
