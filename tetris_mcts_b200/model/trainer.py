"""ctypes face of the device trainer (tetris_mcts_b200/csrc/trainer.cu, include/b200_tetris_mcts.h b200_trainer_*): one optimiser step of the
reference's value network — Model_VV._loss (model/model_vv.py:136-153, GaussianLL :94-101), Model.train (model/model.py:95-119), Yogi.step
(model/yogi.py:39-90) — entirely on the GPU.  No CPU path: without the library / a device the calls raise.

kind: "fp64" runs the contractions on CUDA cores with fp64 accumulation (the reference kind); "tc" runs them on Hopper tensor cores with
the 3xTF32 split (trainer.cu header, include/b200_tetris_mcts.h B200_TRAIN_TC); "tf32" on tensor cores with one tf32 term per operand and
implicit-im2col convolutions (B200_TRAIN_TF32: faster, ~1e-3 instead of 1e-5 of float64).  Weights and optimiser state are the same in
every kind.  A tf32 trainer has no col* / dcol* buffers (NO_BUFFERS); debug_buffer refuses those names."""
import ctypes as C

import numpy as np

from .. import _lib as L

N_TRAIN = 478338            # trainable floats (state_dict order without out_ubound / out_lbound)
GRAD_VEC = N_TRAIN + 3      # doubles of one data-parallel gradient slice: the fp64 gradient, then the slice's loss {count, mean, M2}
KINDS = {"fp64": 0, "tc": 1, "tf32": 2}  # B200_TRAIN_FP64, B200_TRAIN_TC, B200_TRAIN_TF32
# floats per batch row of each buffer b200_trainer_debug_buffer reads (include/b200_tetris_mcts.h)
DEBUG_ROWS = {"x0": 200, "value": 1, "variance": 1, "weight": 1, "col1": 144 * 9, "a1": 144 * 32, "col2": 96 * 288, "a2": 96 * 32,
              "col3": 56 * 288, "a3": 56 * 32, "flat": 1792, "h": 256, "pred": 2, "lossv": 1, "dz": 2, "dh": 256, "dflat": 1792,
              "dc3": 56 * 32, "dcol3": 56 * 288, "da2": 96 * 32, "dcol2": 96 * 288, "da1": 144 * 32}
NO_BUFFERS = {"tf32": ("col1", "col2", "col3", "dcol3", "dcol2")}    # the buffers a trainer of that kind does not allocate
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
        lib.b200_trainer_set_stream.argtypes = [P, P]
        lib.b200_trainer_grad_rows_dev.argtypes = [P, P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_uint64, C.c_int64, C.c_float, C.c_int, P]
        lib.b200_trainer_apply_grads_dev.argtypes = [P, P, C.c_int, C.c_double, C.c_int]
        lib.b200_trainer_read_log.argtypes = [P, C.c_int, P]
        lib.b200_trainer_debug_buffer.argtypes = [P, C.c_char_p, C.c_int, P]
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

    def debug_buffer(self, name, n):
        """test aid: batch buffer `name` (DEBUG_ROWS) as the last step / loss / step_rows_dev / grad_rows_dev left it, rows [0, n) ->
        float32 [n, row]; "d_sumsq": the last step's per-tensor gradient sums of squares, float64 [10]"""
        if name == "d_sumsq":
            out = np.zeros(10, np.float64)
        else:
            out = np.zeros((max(int(n), 0), DEBUG_ROWS.get(name, 1)), np.float32)
        _check(_lib().b200_trainer_debug_buffer(self.h, name.encode(), int(n), L.ptr(out)))
        return out

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

    def set_stream(self, stream_ptr):
        """All later work runs on the CUDA stream `stream_ptr` (e.g. torch.cuda.Stream().cuda_stream; 0 / None: a private stream again)."""
        _check(_lib().b200_trainer_set_stream(self.h, P(int(stream_ptr)) if stream_ptr else None))

    def grad_rows_dev(self, rows_dev_ptr, n_train_rows, batch, lo, hi, seed, iteration, weight_scale, grad_dev_ptr, weighted=True):
        """Rows [lo, hi) of train_rows_dev's batch of iteration `iteration`: their fp64 gradient (scaled by 1 / batch) and loss moments ->
        GRAD_VEC doubles at grad_dev_ptr (device).  Asynchronous on the trainer's stream."""
        _check(_lib().b200_trainer_grad_rows_dev(self.h, P(int(rows_dev_ptr)), int(n_train_rows), int(batch), int(lo), int(hi),
                                                 int(seed) & 0xFFFFFFFFFFFFFFFF, int(iteration), float(weight_scale), int(bool(weighted)),
                                                 P(int(grad_dev_ptr))))

    def apply_grads_dev(self, parts_dev_ptr, n_parts, grad_clip=0.0, log_slot=0):
        """Sum n_parts GRAD_VEC slices (device, rank order) left to right in fp64, round once, clip and take the Yogi step; the step's
        (loss, loss_std, grad_norm) go to log slot `log_slot` (read_log).  Asynchronous."""
        _check(_lib().b200_trainer_apply_grads_dev(self.h, P(int(parts_dev_ptr)), int(n_parts), float(grad_clip), int(log_slot)))

    def read_log(self, n):
        """log slots [0, n) -> float64 [n, 3] = (loss, loss_std, grad_norm); synchronises the trainer's stream"""
        log = np.zeros((int(n), 3), np.float64)
        _check(_lib().b200_trainer_read_log(self.h, int(n), L.ptr(log)))
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
