"""ctypes face of the device trainer (tetris_mcts_b200/csrc/trainer.cu, include/b200_tetris_mcts.h b200_trainer_*): one optimiser step of the
reference's value network — Model_VV._loss (model/model_vv.py:136-153, GaussianLL :94-101), Model.train (model/model.py:95-119), Yogi.step
(model/yogi.py:39-90) — entirely on the GPU.  No CPU path: without the library / a device the calls raise.

kind: "fp64" runs the contractions on CUDA cores with fp64 accumulation (the reference kind); "tc" runs them on Hopper tensor cores with
the 3xTF32 split (trainer.cu header, include/b200_tetris_mcts.h B200_TRAIN_TC).  Weights and optimiser state are the same in both kinds."""
import ctypes as C

import numpy as np

from .. import _lib as L

N_TRAIN = 478338            # trainable floats (state_dict order without out_ubound / out_lbound)
KINDS = {"fp64": 0, "tc": 1}  # B200_TRAIN_FP64, B200_TRAIN_TC
P = C.c_void_p
_sig_done = False


def _lib():
    global _sig_done
    lib = L.lib()
    if not _sig_done:
        lib.b200_trainer_last_error.restype = C.c_char_p
        lib.b200_trainer_create.argtypes = [C.c_int, P, C.c_int, C.POINTER(P)]
        lib.b200_trainer_create_kind.argtypes = [C.c_int, P, C.c_int, C.c_int, C.POINTER(P)]
        lib.b200_trainer_destroy.argtypes = [P]
        lib.b200_trainer_set_hyper.argtypes = [P] + [C.c_double] * 5
        lib.b200_trainer_set_out_ubound.argtypes = [P, C.c_float, C.c_float]
        lib.b200_trainer_get_weights.argtypes = [P, P]
        lib.b200_trainer_set_weights.argtypes = [P, P]
        lib.b200_trainer_get_state.argtypes = [P, P, P, P]
        lib.b200_trainer_set_state.argtypes = [P, P, P, C.c_int64]
        lib.b200_trainer_get_grads.argtypes = [P, P]
        lib.b200_trainer_loss.argtypes = [P, P, P, P, P, C.c_int, C.c_int, P, P, P]
        lib.b200_trainer_step.argtypes = [P, P, P, P, P, C.c_int, C.c_int, C.c_double, P, P, P]
        lib.b200_trainer_step_rows_dev.argtypes = [P, P, C.c_int, P, C.c_int, C.c_float, C.c_int, C.c_double, P, P, P]
        lib.b200_trainer_train_rows_dev.argtypes = [P, P, C.c_int, C.c_int, C.c_int, C.c_uint64, C.c_int64, C.c_float, C.c_int, C.c_double, P]
        lib.b200_trainer_loss_rows_dev.argtypes = [P, P, C.c_int, C.c_int, C.c_float, C.c_int, P, P, P]
        lib.b200_rows_stats_dev.argtypes = [P, P, C.c_int, P, P, P]
        _sig_done = True
    return lib


_M64 = np.uint64(0xFFFFFFFFFFFFFFFF)


def _splitmix64(x):
    with np.errstate(over="ignore"):
        z = (x + np.uint64(0x9E3779B97F4A7C15)) & _M64
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def sample_indices(seed, iteration, batch, n_rows):
    """The batch Trainer.train_rows_dev draws on the device for one iteration (include/b200_tetris_mcts.h b200_trainer_train_rows_dev),
    restated in numpy: idx[i] = splitmix64(splitmix64(splitmix64(seed) + iteration) + i) mod n_rows."""
    base = _splitmix64(np.array([seed], np.uint64))[0]
    with np.errstate(over="ignore"):
        base = _splitmix64(np.array([base + np.uint64(iteration)], np.uint64))[0]
        keys = _splitmix64(base + np.arange(batch, dtype=np.uint64))
    return (keys % np.uint64(n_rows)).astype(np.int32)


def _check(rc):
    if rc != 0:
        raise L.B200Error(rc, _lib().b200_trainer_last_error().decode())


def _batch(batch):
    """[states (n,1,20,10) or (n,20,10) in {-1,0,1}, value (n,1), variance (n,1), weight (n,1)] -> contiguous host arrays"""
    states, value, variance = batch[0], batch[1], batch[2]
    s = np.ascontiguousarray(np.asarray(states).reshape(-1, 200), np.int8)
    v = np.ascontiguousarray(np.asarray(value, np.float32).reshape(-1))
    var = np.ascontiguousarray(np.asarray(variance, np.float32).reshape(-1))
    w = np.ascontiguousarray(np.asarray(batch[3], np.float32).reshape(-1)) if len(batch) > 3 and batch[3] is not None else None
    if not (len(s) == len(v) == len(var)) or (w is not None and len(w) != len(s)):
        raise ValueError("batch arrays differ in length")
    return s, v, var, w


class Trainer:
    def __init__(self, weights, max_batch=4096, device=0, lr=1e-3, betas=(0.9, 0.999), eps=1e-3, weight_decay=1e-3, kind="fp64"):
        if kind not in KINDS:
            raise ValueError("trainer kind must be one of %s, not %r" % (sorted(KINDS), kind))
        self.kind = kind
        w = np.ascontiguousarray(weights, np.float32).ravel()
        if w.size != L.N_WEIGHTS:
            raise ValueError("expected %d floats (state_dict order)" % L.N_WEIGHTS)
        self.h, self.max_batch, self.device = P(), int(max_batch), int(device)
        _check(_lib().b200_trainer_create_kind(int(device), L.ptr(w), int(max_batch), KINDS[kind], C.byref(self.h)))
        _check(_lib().b200_trainer_set_hyper(self.h, lr, betas[0], betas[1], eps, weight_decay))     # Yogi(lr=1e-3, eps=1e-3, weight_decay=1e-3), model_vv.py:132

    def close(self):
        if getattr(self, "h", None):
            _lib().b200_trainer_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_out_ubound(self, ub_value, ub_variance):              # model_vv.py:227-231
        _check(_lib().b200_trainer_set_out_ubound(self.h, float(ub_value), float(ub_variance)))

    def weights(self):
        w = np.zeros(L.N_WEIGHTS, np.float32)
        _check(_lib().b200_trainer_get_weights(self.h, L.ptr(w)))
        return w

    def set_weights(self, weights):
        w = np.ascontiguousarray(weights, np.float32).ravel()
        _check(_lib().b200_trainer_set_weights(self.h, L.ptr(w)))

    def state(self):
        m, v, step = np.zeros(N_TRAIN, np.float32), np.zeros(N_TRAIN, np.float32), np.zeros(1, np.int64)
        _check(_lib().b200_trainer_get_state(self.h, L.ptr(m), L.ptr(v), L.ptr(step)))
        return m, v, int(step[0])

    def set_state(self, exp_avg, exp_avg_sq, step):
        if step is None or step < 0:
            _check(_lib().b200_trainer_set_state(self.h, None, None, -1))
            return
        m, v = np.ascontiguousarray(exp_avg, np.float32).ravel(), np.ascontiguousarray(exp_avg_sq, np.float32).ravel()
        _check(_lib().b200_trainer_set_state(self.h, L.ptr(m), L.ptr(v), int(step)))

    def grads(self):
        g = np.zeros(N_TRAIN, np.float32)
        _check(_lib().b200_trainer_get_grads(self.h, L.ptr(g)))
        return g

    def loss(self, batch, weighted=False, want_pred=False):
        """Model_VV._loss under no_grad on one chunk: (mean, population std[, pred (n,2)])"""
        s, v, var, w = _batch(batch)
        out = np.zeros(2, np.float64)
        pred = np.zeros((len(s), 2), np.float32) if want_pred else None
        _check(_lib().b200_trainer_loss(self.h, L.ptr(s), L.ptr(v), L.ptr(var), L.ptr(w), len(s), int(bool(weighted)),
                                        out[0:1].ctypes.data_as(P), out[1:2].ctypes.data_as(P), L.ptr(pred)))
        return (out[0], out[1], pred) if want_pred else (out[0], out[1])

    def step(self, batch, weighted=False, grad_clip=0.0):
        """Model.train (model/model.py:95-119) -> dict(loss, loss_std, grad_norm)"""
        s, v, var, w = _batch(batch)
        out = np.zeros(3, np.float64)
        _check(_lib().b200_trainer_step(self.h, L.ptr(s), L.ptr(v), L.ptr(var), L.ptr(w), len(s), int(bool(weighted)), float(grad_clip),
                                        out[0:1].ctypes.data_as(P), out[1:2].ctypes.data_as(P), out[2:3].ctypes.data_as(P)))
        return {"loss": float(out[0]), "loss_std": float(out[1]), "grad_norm": float(out[2])}

    def step_rows_dev(self, rows_dev_ptr, n_rows, idx, weight_scale, weighted=True, grad_clip=0.0):
        """The same step on a batch gathered on the device from 212-byte replay rows (engine.replay_drain_into / the all-gather block)."""
        idx = np.ascontiguousarray(idx, np.int32)
        out = np.zeros(3, np.float64)
        _check(_lib().b200_trainer_step_rows_dev(self.h, P(int(rows_dev_ptr)), int(n_rows), L.ptr(idx), len(idx), float(weight_scale),
                                                 int(bool(weighted)), float(grad_clip), out[0:1].ctypes.data_as(P), out[1:2].ctypes.data_as(P),
                                                 out[2:3].ctypes.data_as(P)))
        return {"loss": float(out[0]), "loss_std": float(out[1]), "grad_norm": float(out[2])}

    def train_rows_dev(self, rows_dev_ptr, n_train_rows, batch, iters, seed, first_iter, weight_scale, weighted=True, grad_clip=0.0):
        """`iters` steps of step_rows_dev on batches drawn on the device (sample_indices(seed, first_iter + it, batch, n_train_rows)), one host
        synchronisation in all -> float64 [iters, 3] = per-step (loss, loss_std, grad_norm)."""
        log = np.zeros((int(iters), 3), np.float64)
        _check(_lib().b200_trainer_train_rows_dev(self.h, P(int(rows_dev_ptr)), int(n_train_rows), int(batch), int(iters), int(seed) & 0xFFFFFFFFFFFFFFFF,
                                                  int(first_iter), float(weight_scale), int(bool(weighted)), float(grad_clip), L.ptr(log)))
        return log

    def loss_rows_dev(self, rows_dev_ptr, first, n, weight_scale, weighted=True):
        """Model_VV._loss under no_grad on device rows [first, first + n) -> (mean, population std, sum of the weights)"""
        out = np.zeros(3, np.float64)
        _check(_lib().b200_trainer_loss_rows_dev(self.h, P(int(rows_dev_ptr)), int(first), int(n), float(weight_scale), int(bool(weighted)),
                                                 out[0:1].ctypes.data_as(P), out[1:2].ctypes.data_as(P), out[2:3].ctypes.data_as(P)))
        return float(out[0]), float(out[1]), float(out[2])

    def rows_stats(self, rows_dev_ptr, n):
        """(max value, max variance, fp64 sum of visits) of device rows [0, n)"""
        mx, s = np.zeros(2, np.float32), np.zeros(1, np.float64)
        _check(_lib().b200_rows_stats_dev(self.h, P(int(rows_dev_ptr)), int(n), mx[0:1].ctypes.data_as(P), mx[1:2].ctypes.data_as(P), L.ptr(s)))
        return float(mx[0]), float(mx[1]), float(s[0])
