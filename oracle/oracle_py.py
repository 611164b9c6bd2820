"""ctypes face of oracle/liboracle.so — TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import this.
The functions mirror oracle/mcts_oracle.h and oracle/tetris_oracle.h (which cite the reference file:line).
"""
import ctypes as C
import os
import subprocess
import sys
import types
import importlib.util

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
NA = 7
REC_WORDS = 20
KEY_WORDS = 12
NW = 478342

_lib = None


def build(ref=False):
    """Compile the C restatement (and, when /root/reference is present and ref=True, oracle/_ref)."""
    target = ["liboracle.so"] + (["ref"] if ref else [])
    subprocess.run(["make", "-C", HERE, "-s"] + target, check=True)


def lib():
    global _lib
    if _lib is None:
        path = os.path.join(HERE, "liboracle.so")
        if not os.path.exists(path):
            build()
        _lib = C.CDLL(path)
        _sig(_lib)
    return _lib


class MoConfig(C.Structure):
    _fields_ = [
        ("max_nodes", C.c_int), ("mode", C.c_int), ("gamma", C.c_double), ("low", C.c_int),
        ("lp_end_from_obs", C.c_int), ("lp_var_gamma2", C.c_int), ("rollout_variance", C.c_double),
        ("eval_mode", C.c_int), ("weights", C.c_void_p), ("eval_cb", C.c_void_p), ("eval_ctx", C.c_void_p),
        ("search_seed", C.c_uint32), ("stale_pop", C.c_int), ("dist_bins", C.c_int), ("dist_vmin", C.c_double), ("dist_vmax", C.c_double),
        ("replay_min_visits", C.c_int), ("replay_cap", C.c_int), ("overflow_reset", C.c_int),
    ]


EVAL_CB = C.CFUNCTYPE(None, C.c_void_p, C.POINTER(C.c_int8), C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_float))


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def _sig(L):
    L.mo_norm_quantile.restype = C.c_double
    L.mo_norm_quantile.argtypes = [C.c_double]
    L.mo_norm_quantile_f32.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    L.mo_pc_replay.restype = C.c_long
    L.mo_pc_replay.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int] + [C.c_void_p] * 8
    L.mo_agent_create.restype = C.c_void_p
    L.mo_agent_create.argtypes = [C.POINTER(MoConfig), C.c_int, C.c_int, C.c_int]
    L.mo_agent_destroy.argtypes = [C.c_void_p]
    L.mo_agent_update_root.argtypes = [C.c_void_p, C.c_void_p]
    L.mo_agent_mcts.argtypes = [C.c_void_p, C.c_int]
    L.mo_agent_get_action.argtypes = [C.c_void_p, C.c_void_p]
    L.mo_agent_root.argtypes = [C.c_void_p]
    L.mo_agent_episode.argtypes = [C.c_void_p]
    L.mo_agent_counter.restype = C.c_long
    L.mo_agent_counter.argtypes = [C.c_void_p, C.c_int]
    L.mo_agent_export.argtypes = [C.c_void_p] + [C.c_void_p] * 10
    L.mo_agent_last_trace.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    L.mo_select_trace_obs.argtypes = [C.c_int] + [C.c_void_p] * 6 + [C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    L.mo_backup_trace_obs.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 5 + [C.c_double] * 3
    L.mo_backup_trace_mixture_obs.argtypes = L.mo_backup_trace_obs.argtypes
    L.mo_backup_trace_obs_LP.argtypes = ([C.c_void_p, C.c_int] + [C.c_void_p] * 8 + [C.c_int, C.c_void_p, C.c_void_p,
                                         C.c_double, C.c_int, C.c_int])
    L.mo_unique_child_obs.argtypes = [C.c_int] + [C.c_void_p] * 5
    L.mo_get_all_childs.argtypes = [C.c_int, C.c_void_p, C.c_int, C.c_void_p]
    L.mo_synthetic_eval.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    L.vo_forward.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    L.to_play_records.argtypes = [C.c_void_p, C.c_void_p, C.c_int]


# ----------------------------------------------------------------------------- env
class ToGame(C.Structure):
    _fields_ = [("rows", C.c_uint16 * 20), ("piece", C.c_int), ("rot", C.c_int), ("px", C.c_int), ("py", C.c_int),
                ("bag", C.c_uint32), ("dropcnt", C.c_int), ("end", C.c_int), ("app", C.c_int), ("scoring", C.c_int),
                ("randomizer", C.c_int), ("combo", C.c_int), ("rng", C.c_uint32), ("score", C.c_int32),
                ("line_clears", C.c_int32), ("line_stats", C.c_int32 * 4)]


class Game:
    """Single oracle game (SPEC_PYTETRIS.md)."""

    def __init__(self, app=1, scoring=0, randomizer=0, seed=None, record=None):
        self.g = ToGame()
        L = lib()
        L.to_init(C.byref(self.g), app, scoring, randomizer)
        if seed is not None:
            L.to_seed(C.byref(self.g), C.c_uint32(seed))
        if record is not None:
            L.to_unpack(C.byref(self.g), _p(np.ascontiguousarray(record, dtype=np.uint32)))

    def play(self, a):
        lib().to_play(C.byref(self.g), int(a))

    def reset(self):
        lib().to_reset(C.byref(self.g))

    def record(self):
        w = np.zeros(REC_WORDS, np.uint32)
        lib().to_pack(C.byref(self.g), _p(w))
        return w

    def obskey(self):
        k = np.zeros(KEY_WORDS, np.uint32)
        lib().to_obskey(C.byref(self.g), _p(k))
        return k

    def state(self):
        s = np.zeros((20, 10), np.int8)
        lib().to_state(C.byref(self.g), _p(s))
        return s

    @property
    def end(self):
        return bool(self.g.end)

    @property
    def score(self):
        return int(self.g.score)

    @property
    def line_clears(self):
        return int(self.g.line_clears)


def fresh_records(n, base_seed=123, app=1, scoring=0, randomizer=0):
    """n fresh games, game i seeded with base_seed + i (SURVEY §8d: base 123 echoes agent.cpp:23)."""
    out = np.zeros((n, REC_WORDS), np.uint32)
    for i in range(n):
        out[i] = Game(app, scoring, randomizer, seed=base_seed + i).record()
    return out


def play_records(recs, actions):
    recs = np.ascontiguousarray(recs, dtype=np.uint32).copy()
    actions = np.ascontiguousarray(actions, dtype=np.int32)
    lib().to_play_records(_p(recs), _p(actions), len(actions))
    return recs


def obskey_to_state(key):
    key = np.asarray(key, np.uint32)
    s = np.zeros(200, np.int8)
    for r in range(20):
        row = (int(key[r >> 1]) >> ((r & 1) * 16)) & 0x3ff
        for c in range(10):
            s[r * 10 + c] = (row >> c) & 1
    for j in range(4):
        s[(int(key[10]) >> (8 * j)) & 0xff] = -1
    return s.reshape(20, 10)


# ----------------------------------------------------------------------------- core twins
def norm_quantile_f32(n):
    """z(n) of policy_clt (special.h:26-33 narrowed to float, core.h:93) with the host libm, for an int32 array of n."""
    n = np.ascontiguousarray(n, np.int32)
    out = np.empty(len(n), np.float32)
    lib().mo_norm_quantile_f32(_p(n), len(n), _p(out))
    return out


def pc_replay(child, score, n2o, low, traces, states):
    """The path-cache model (mcts_oracle.c pc_*) over given walks on a fixed tree whose childless nodes are terminal, from an empty cache:
    traces[s] is simulation s's walk, states[s] = (visit, value, variance) before it and states[s + 1] after its backup.  Returns
    (served[S], pc_len[S], events[S, 3], stale reads): the levels the engine's phase 1 serves, the valid length after each backup, and
    per simulation {served levels whose pick changed, stops at a cached level because of check_low, the walk ended on a cached leaf}."""
    S, M = len(traces), len(n2o)
    tr = np.ascontiguousarray(np.concatenate(traces), np.int32)
    off = np.zeros(S + 1, np.int32)
    off[1:] = np.cumsum([len(t) for t in traces])
    vis, val, var = (np.ascontiguousarray(np.stack([st[k] for st in states[:S + 1]]), dt) for k, dt in ((0, np.int32), (1, np.float32), (2, np.float32)))
    served, pcl, ev = np.zeros(S, np.int32), np.zeros(S, np.int32), np.zeros((S, 3), np.int32)
    err = lib().mo_pc_replay(M, _p(np.ascontiguousarray(child, np.int32)), _p(np.ascontiguousarray(score, np.float32)),
                             _p(np.ascontiguousarray(n2o, np.int32)), int(low), S, _p(tr), _p(off), _p(vis), _p(val), _p(var),
                             _p(served), _p(pcl), _p(ev))
    return served, pcl, ev, int(err)


def select_trace_obs(index, child, visit, value, variance, score, n2o, low, max_trace=512, rng_state=None):
    """rng_state: uint32[1] array -> check_low draws come from xorshift32 on it (as in the device twin);
    None -> libc rand() like the reference (core.h:76)."""
    tr = np.zeros(max_trace, np.int32)
    fn = ctx = None
    if rng_state is not None:
        fn = C.cast(lib().mo_xorshift32, C.c_void_p)
        ctx = _p(rng_state)
    D = lib().mo_select_trace_obs(int(index), _p(child), _p(visit), _p(value), _p(variance), _p(score), _p(n2o),
                                  int(low), _p(tr), max_trace, fn, ctx)
    assert D > 0
    return tr[:D].copy()


def backup_trace_obs(trace, visit, value, variance, n2o, score, v, var, gamma, mixture=False):
    f = lib().mo_backup_trace_mixture_obs if mixture else lib().mo_backup_trace_obs
    trace = np.ascontiguousarray(trace, np.int32)
    f(_p(trace), len(trace), _p(visit), _p(value), _p(variance), _p(n2o), _p(score), float(v), float(var), float(gamma))


def backup_trace_obs_LP(trace, visit, value, variance, n2o, score, end, c_nodes, c_obs, v, var, gamma, mixture, averaged):
    trace = np.ascontiguousarray(trace, np.int32)
    cn = np.ascontiguousarray(c_nodes, np.int32)
    co = np.ascontiguousarray(c_obs, np.int32)
    v = np.ascontiguousarray(v, np.float32)
    var = np.ascontiguousarray(var, np.float32)
    end = np.ascontiguousarray(end, np.uint8)
    lib().mo_backup_trace_obs_LP(_p(trace), len(trace), _p(visit), _p(value), _p(variance), _p(n2o), _p(score), _p(end),
                                 _p(cn), _p(co), len(cn), _p(v), _p(var), float(gamma), int(mixture), int(averaged))


def get_unique_child_obs(index, child, score, n2o):
    cn = np.zeros(NA, np.int32)
    co = np.zeros(NA, np.int32)
    k = lib().mo_unique_child_obs(int(index), _p(child), _p(score), _p(n2o), _p(cn), _p(co))
    return cn[:k].copy(), co[:k].copy()


def get_all_childs(index, child):
    M = child.shape[0]
    mark = np.zeros(M, np.uint8)
    lib().mo_get_all_childs(int(index), _p(child), M, _p(mark))
    return set(np.nonzero(mark)[0].tolist())


def synthetic_eval(key):
    v = C.c_float()
    var = C.c_float()
    key = np.ascontiguousarray(key, np.uint32)
    lib().mo_synthetic_eval(_p(key), C.byref(v), C.byref(var))
    return v.value, var.value


def valuenet_forward(weights, states):
    states = np.ascontiguousarray(states, np.int8).reshape(-1, 200)
    w = np.ascontiguousarray(weights, np.float32)
    assert w.size == NW
    k = states.shape[0]
    v = np.zeros(k, np.float32)
    var = np.zeros(k, np.float32)
    lib().vo_forward(_p(w), _p(states), k, _p(v), _p(var))
    return v, var


# ----------------------------------------------------------------------------- agent
class Agent:
    MODE_LP, MODE_SINGLE, MODE_VANILLA = 0, 1, 2

    def __init__(self, max_nodes=100000, mode=0, gamma=0.999, low=1, eval_mode=0, weights=None, eval_cb=None,
                 lp_end_from_obs=0, lp_var_gamma2=1, rollout_variance=1e3, search_seed=0, stale_pop=1,
                 app=1, scoring=0, randomizer=0, dist_bins=50, dist_vmin=0.0, dist_vmax=5000.0, replay_min_visits=0, replay_cap=0,
                 overflow_reset=0):
        cfg = MoConfig()
        cfg.overflow_reset = int(overflow_reset)
        cfg.replay_min_visits, cfg.replay_cap = replay_min_visits, replay_cap
        cfg.dist_bins, cfg.dist_vmin, cfg.dist_vmax = dist_bins, dist_vmin, dist_vmax
        self.dist_bins = dist_bins
        cfg.max_nodes, cfg.mode, cfg.gamma, cfg.low = max_nodes, mode, gamma, low
        cfg.lp_end_from_obs, cfg.lp_var_gamma2, cfg.rollout_variance = lp_end_from_obs, lp_var_gamma2, rollout_variance
        cfg.eval_mode = eval_mode
        self._w = None
        if weights is not None:
            self._w = np.ascontiguousarray(weights, np.float32)
            cfg.weights = self._w.ctypes.data
        self._cb = None
        if eval_cb is not None:
            def tramp(ctx, states, k, v, var):
                st = np.ctypeslib.as_array(states, shape=(k * 200,)).reshape(k, 1, 20, 10)
                if mode == 3:                                         # distributional: eval_cb(states) -> f32[k, dist_bins]
                    p = np.ravel(np.asarray(eval_cb(st), np.float32))
                    for i in range(k * dist_bins):
                        v[i] = float(p[i])
                    return
                rv, rvar = eval_cb(st)
                for i in range(k):
                    v[i] = float(np.ravel(rv)[i])
                    var[i] = float(np.ravel(rvar)[i])
            self._cb = EVAL_CB(tramp)
            cfg.eval_cb = C.cast(self._cb, C.c_void_p)
        cfg.search_seed, cfg.stale_pop = search_seed, stale_pop
        self.M = max_nodes
        self.h = lib().mo_agent_create(C.byref(cfg), app, scoring, randomizer)

    def close(self):
        if self.h:
            lib().mo_agent_destroy(self.h)
            self.h = None

    __del__ = close

    def update_root(self, rec):
        rec = np.ascontiguousarray(rec, np.uint32)
        lib().mo_agent_update_root(self.h, _p(rec))

    def mcts(self, sims):
        rc = lib().mo_agent_mcts(self.h, sims)
        if rc != 0:
            raise RuntimeError("oracle agent: rc=%d (arena overflow / trace too deep)" % rc)

    def get_action(self):
        st = np.zeros((3, NA), np.float32)
        a = lib().mo_agent_get_action(self.h, _p(st))
        return a, st

    def remove_nodes(self):                                           # agents/agent.py:246-257, called explicitly
        lib().mo_agent_remove_nodes.argtypes = [C.c_void_p]
        lib().mo_agent_remove_nodes(self.h)

    @property
    def n_free(self):                                                 # len(self.available)
        lib().mo_agent_n_free.argtypes = [C.c_void_p]
        return lib().mo_agent_n_free(self.h)

    @property
    def root(self):
        return lib().mo_agent_root(self.h)

    def counter(self, which):
        return lib().mo_agent_counter(self.h, which)

    def export(self):
        M = self.M
        d = dict(child=np.zeros((M, NA), np.int32), score=np.zeros(M, np.float32), episode=np.zeros(M, np.int32),
                 n2o=np.zeros(M, np.int32), visit=np.zeros(M, np.int32), value=np.zeros(M, np.float32),
                 variance=np.zeros(M, np.float32), obs_end=np.zeros(M, np.uint8),
                 game=np.zeros((M, REC_WORDS), np.uint32), obs_key=np.zeros((M, KEY_WORDS), np.uint32))
        lib().mo_agent_export(self.h, _p(d["child"]), _p(d["score"]), _p(d["episode"]), _p(d["n2o"]), _p(d["visit"]),
                              _p(d["value"]), _p(d["variance"]), _p(d["obs_end"]), _p(d["game"]), _p(d["obs_key"]))
        return d

    def replay(self, max_rows=1 << 20):
        rows = np.zeros((max_rows, 212), np.uint8)
        lib().mo_agent_replay.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        n = lib().mo_agent_replay(self.h, _p(rows), max_rows)
        return rows[:n].copy()

    def export_dist(self):
        ns = np.zeros((self.M, 5), np.float32)
        nd = np.zeros((self.M, self.dist_bins), np.float32)
        lib().mo_agent_export_dist.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        lib().mo_agent_export_dist(self.h, _p(ns), _p(nd))
        return ns, nd

    def pc_enable(self, on=True):                                     # CPU model of the engine's path cache (diagnostic)
        lib().mo_agent_pc_enable.argtypes = [C.c_void_p, C.c_int]
        lib().mo_agent_pc_enable(self.h, int(on))

    def pc_stats(self):
        out = np.zeros(7, np.int64)
        lib().mo_agent_pc_stats.argtypes = [C.c_void_p, C.c_void_p]
        lib().mo_agent_pc_stats(self.h, _p(out))
        return dict(zip(("errors", "irregular", "shared", "levels", "sims", "full_walks", "len"), out.tolist()))

    def last_trace(self):
        tr = np.zeros(512, np.int32)
        D = lib().mo_agent_last_trace(self.h, _p(tr), 512)
        return tr[:D].copy()


# ----------------------------------------------------------------------------- weights
def seeded_weights(seed=0):
    """Value-net weights with the reference's default-init distribution (torch kaiming_uniform(a=sqrt 5) ==
    U(-1/sqrt(fan_in), 1/sqrt(fan_in)) for weight and bias, model_vv.py:31-43), drawn from numpy's PCG64 so
    both boxes regenerate the same 478342 floats without shipping a checkpoint (SURVEY §6: none matches)."""
    rng = np.random.default_rng(seed)
    parts = []
    for shape, fan_in in (((32, 1, 3, 3), 9), ((32,), 9), ((32, 32, 3, 3), 288), ((32,), 288), ((32, 32, 3, 3), 288),
                          ((32,), 288), ((256, 1792), 1792), ((256,), 1792), ((2, 256), 256), ((2,), 256)):
        b = 1.0 / np.sqrt(fan_in)
        parts.append(rng.uniform(-b, b, size=shape).astype(np.float32).ravel())
    parts.append(np.array([1e2, 1e3], np.float32))     # out_ubound, model_vv.py:45
    parts.append(np.array([0.0, 1e-1], np.float32))    # out_lbound, model_vv.py:46
    w = np.concatenate(parts)
    assert w.size == NW
    return w


WEIGHT_KEYS = (("head.conv1.weight", (32, 1, 3, 3)), ("head.conv1.bias", (32,)), ("head.conv2.weight", (32, 32, 3, 3)),
               ("head.conv2.bias", (32,)), ("head.conv3.weight", (32, 32, 3, 3)), ("head.conv3.bias", (32,)),
               ("head.fc1.weight", (256, 1792)), ("head.fc1.bias", (256,)), ("head.fc_out.weight", (2, 256)),
               ("head.fc_out.bias", (2,)), ("out_ubound", (2,)), ("out_lbound", (2,)))


def weights_to_state_dict(w):
    out, off = {}, 0
    for name, shape in WEIGHT_KEYS:
        n = int(np.prod(shape))
        out[name] = np.asarray(w[off:off + n], np.float32).reshape(shape)
        off += n
    return out


# ----------------------------------------------------------------------------- reference modules (oracle/_ref)
def load_ref_module(name):
    """Import oracle/_ref/<name>*.so (core / agent = the reference's own C++ compiled unchanged; pyTetris = oracle env)."""
    d = os.path.join(HERE, "_ref")
    for f in sorted(os.listdir(d)) if os.path.isdir(d) else []:
        if f.startswith(name + ".") and f.endswith(".so"):
            if name in sys.modules:
                return sys.modules[name]
            spec = importlib.util.spec_from_file_location(name, os.path.join(d, f))
            m = importlib.util.module_from_spec(spec)
            sys.modules[name] = m
            spec.loader.exec_module(m)
            return m
    raise ImportError("oracle/_ref/%s*.so missing: run `make -C oracle ref` where /root/reference exists" % name)


def mount_reference(ref="/root/reference"):
    """Make the reference's own Python agents importable UNMODIFIED in this container (SURVEY §8c work-around:
    a site-packages package named `agents` shadows the namespace package; cppimport is absent)."""
    if not os.path.isdir(ref):
        raise ImportError("reference tree absent")
    pt = load_ref_module("pyTetris")
    core = load_ref_module("core")
    m = types.ModuleType("agents")
    m.__path__ = [os.path.join(ref, "agents")]
    sys.modules["agents"] = m
    sys.modules["agents.helper"] = types.ModuleType("agents.helper")
    cm = types.ModuleType("agents.cppmodule")
    cm.__path__ = []
    sys.modules["agents.cppmodule"] = cm
    sys.modules["agents.cppmodule.core"] = core
    try:
        sys.modules["agents.cppmodule.agent"] = load_ref_module("agent")
    except ImportError:
        pass
    if ref not in sys.path:
        sys.path.insert(0, ref)
    return pt, core


# ----------------------------------------------------------------------------- distributional cores (a16)
def _dsig():
    L = lib()
    if getattr(L, "_dsig", False):
        return L
    L.do_shift_distribution.argtypes = [C.c_void_p, C.c_int, C.c_double, C.c_double, C.c_double, C.c_void_p]
    L.do_mean_dist.restype = C.c_double
    L.do_mean_dist.argtypes = [C.c_void_p, C.c_int, C.c_double, C.c_double]
    L.do_mean_variance.argtypes = [C.c_void_p, C.c_int, C.c_double, C.c_double, C.c_void_p, C.c_void_p]
    L.do_policy_dist.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_double, C.c_void_p]
    L.do_select_trace_distributional.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    L.do_backup_trace_distributional.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_double, C.c_void_p, C.c_double, C.c_double]
    L._dsig = True
    return L


def shift_distribution(dist, x, vmin, vmax):
    dist = np.ascontiguousarray(dist, np.float32)
    out = np.zeros_like(dist)
    _dsig().do_shift_distribution(_p(dist), len(dist), float(x), float(vmin), float(vmax), _p(out))
    return out


def mean_variance(dist, vmin, vmax):
    dist = np.ascontiguousarray(dist, np.float32)
    m, v = C.c_double(), C.c_double()
    _dsig().do_mean_variance(_p(dist), len(dist), float(vmin), float(vmax), C.byref(m), C.byref(v))
    return m.value, v.value


def policy_dist(child_nodes, node_stats, curr_reward):
    cn = np.ascontiguousarray(child_nodes, np.int32)
    q = np.zeros(len(cn), np.float64)
    c = _dsig().do_policy_dist(_p(cn), len(cn), _p(node_stats), float(curr_reward), _p(q))
    return c, q


def select_trace_distributional(index, child, node_stats, low, rng_state=None, max_trace=512):
    tr = np.zeros(max_trace, np.int32)
    fn = C.cast(lib().mo_xorshift32, C.c_void_p)
    st = rng_state if rng_state is not None else np.array([1], np.uint32)
    D = _dsig().do_select_trace_distributional(int(index), _p(child), _p(node_stats), int(low), _p(tr), max_trace, fn, _p(st))
    assert D > 0
    return tr[:D].copy()


def backup_trace_distributional(trace, node_stats, node_dist, r, dist, vmin, vmax):
    trace = np.ascontiguousarray(trace, np.int32)
    dist = np.ascontiguousarray(dist, np.float32)
    _dsig().do_backup_trace_distributional(_p(trace), len(trace), _p(node_stats), _p(node_dist), node_dist.shape[1], float(r), _p(dist), float(vmin), float(vmax))


def synthetic_dist(key, bins=50):
    key = np.ascontiguousarray(key, np.uint32)
    out = np.zeros(bins, np.float32)
    lib().mo_synthetic_dist.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    lib().mo_synthetic_dist(_p(key), bins, _p(out))
    return out


DIST_WEIGHT_KEYS = (("seq.conv1.weight", (32, 1, 4, 4)), ("seq.conv1.bias", (32,)), ("seq.conv2.weight", (32, 32, 4, 4)),
                    ("seq.conv2.bias", (32,)), ("seq.fc1.weight", (128, 2048)), ("seq.fc1.bias", (128,)),
                    ("seq.fc_v.weight", (50, 128)), ("seq.fc_v.bias", (50,)))


def seeded_dist_weights(seed=0, atoms=50):
    """Default-init-distributed weights of model/model_distributional.py:18-45 Net (22x10 input, flatten 2048), numpy PCG64."""
    rng = np.random.default_rng(seed + 1000)
    parts = []
    for shape, fan_in in (((32, 1, 4, 4), 16), ((32,), 16), ((32, 32, 4, 4), 512), ((32,), 512), ((128, 2048), 2048), ((128,), 2048),
                          ((atoms, 128), 128), ((atoms,), 128)):
        b = 1.0 / np.sqrt(fan_in)
        parts.append(rng.uniform(-b, b, size=shape).astype(np.float32).ravel())
    return np.concatenate(parts)


def dist_weights_to_state_dict(w, atoms=50):
    out, off = {}, 0
    for name, shape in DIST_WEIGHT_KEYS:
        if name.startswith("seq.fc_v"):
            shape = (atoms,) + tuple(shape[1:])
        n = int(np.prod(shape))
        out[name] = np.asarray(w[off:off + n], np.float32).reshape(shape)
        off += n
    return out


def distnet_forward(weights, states, bins=50):
    states = np.ascontiguousarray(states, np.int8).reshape(-1, 200)
    w = np.ascontiguousarray(weights, np.float32)
    out = np.zeros((len(states), bins), np.float32)
    lib().dn_forward.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    lib().dn_forward(_p(w), _p(states), len(states), bins, _p(out))
    return out
