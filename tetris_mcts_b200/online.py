"""The training half of the online agent's remove_nodes on the device (agents/ValueSim.py:101-115,161-185; OnlineMCTSAgent::remove_nodes
agent.cpp:619-708): once the engine's replay policy says train, the rows of the device replay memory are copied to a device buffer
(b200_replay_peek_dev), Model_VV.train_rows trains the value network on them without a host copy, the engine searches on with the new
weights, and the policy is told that the memory was trained on.  Used by agents.ValueSim (online=True) and play_batched --online.

Under a torch.distributed process group (play_batched under torchrun) rank 0's engine holds the memory and the policy: rank 0 copies the rows
out and broadcasts them into every rank's buffer, and all ranks train data-parallel on them (Model_VV.train_rows).

OnlineTrainer trains on a thread of its own (start), and the new weights reach the search when install() is called: at once (train,
train_lag 0), or train_lag moves later while the search plays on (play_batched --train_lag).

CallbackTrainer hands the same rows to a caller-supplied training function instead (OnlineMCTSAgent's train callback, agent.cpp:698)."""
import os
import time

from . import distributed, replay
from .model.model_vv import EXP_PATH


class OnlineTrainer:
    """train_lag L (moves): the weights of a training started after move s are installed into the search after move s + L (start / due /
    install); with L > 0 the search plays on while the trainer trains, on the same device, and evaluates with weights up to L moves older
    than the reference's would be.  Everything the run computes depends on its seeds and L alone, not on how long a training takes."""
    # train_lag > 0: the CUDA stream priorities of the search engine and of the training (lower is higher)
    SEARCH_PRIORITY, TRAIN_PRIORITY = -1, 0

    def __init__(self, eng, weights, capacity, batch_size=1024, iters_per_val=100, max_iters=50000, checkpoint=EXP_PATH + "model_checkpoint",
                 train_kind="fp64", train_lag=0):
        from .model.trainer import KINDS
        if train_kind not in KINDS:
            raise ValueError("train_kind must be one of %s, not %r" % (sorted(KINDS), train_kind))
        if int(train_lag) < 0:
            raise ValueError("train_lag counts moves: >= 0, not %r" % (train_lag,))
        self.train_kind, self.train_lag = train_kind, int(train_lag)
        self._pending, self._train_stream, self._streamed, self._search_stream = None, None, None, None
        self.move, self.wait_seconds = 0, 0.0                      # the last completed move (after_move); seconds blocked in join / install
        self.eng, self.weights = eng, weights
        self.kw = dict(batch_size=int(batch_size), iters_per_val=int(iters_per_val), max_iters=int(max_iters), checkpoint=checkpoint)
        self.model, self.n_trains, self.train_seconds, self.last_rows = None, 0, 0.0, None
        self.rank = distributed.rank_world()[0]
        self.buf = self._row_buffer(int(capacity))
        if self.train_lag > 0:
            self._search_on_own_stream()

    def _row_buffer(self, capacity):
        """the rows a training reads: `capacity` replay rows on the engine's device (not torch's current one)"""
        import torch
        dev = torch.device("cuda", int(self.eng.cfg.device))
        buf = torch.empty((capacity, replay.SAMPLE_BYTES), dtype=torch.uint8, device=dev)
        torch.cuda.synchronize(dev)                                # the engine copies on its own stream: nothing of torch's may be pending on buf
        return buf

    def _search_on_own_stream(self):
        """the search engine's work on a non-blocking stream of priority SEARCH_PRIORITY, beside the training's (_stream)"""
        import torch
        self._search_stream = torch.cuda.Stream(device=self.buf.device, priority=self.SEARCH_PRIORITY)
        self.eng.set_stream(self._search_stream)

    def _model(self):
        if self.model is None:
            from .model.model_vv import Model_VV
            self.model = Model_VV(device=int(self.eng.cfg.device), eval_kind="net", train_kind=self.train_kind)
            self.model.weights = self.weights
            self.model._eng.load_weights(self.weights)
        return self.model

    def _peek(self, n_rows):
        """the first n_rows rows of rank 0's memory -> buf[:n_rows] on every rank, in place when this returns"""
        if self.rank == 0:
            self.eng.replay_peek_into(self.buf.data_ptr(), n_rows)  # synchronises the engine's stream
        distributed.broadcast_rows(self.buf, n_rows)               # world > 1: rank 0's rows on every rank

    def train(self, n_rows, current_episode, dump_path=None):
        """Train on the first n_rows rows of the engine's memory (ValueSim.py:176-183 / agent.cpp:697-701): install() the training in flight,
        if any, start() this one after the move after_move() last named, and with train_lag 0 install() it at once, so that the search goes
        on with the new weights.  Returns False (memory untouched, still collecting) when there are too few rows for a validation split."""
        self.install()
        if not self.start(n_rows, current_episode, dump_path):
            return False
        if self.due(self.move):
            self.install()
        return True

    def after_move(self, move):
        """Move `move` is complete: install the training in flight if train_lag moves have passed since it started"""
        self.move = int(move)
        if self.due(self.move):
            self.install()

    def start(self, n_rows, current_episode, dump_path=None, move=None):
        """The first half of train(), which returns before the training ends: the first n_rows rows of the memory are copied to the
        trainer's buffer, dumped when dump_path is given (np.savez(dump_path, states=, values=, variance=, weights=), ValueSim.py:176-177;
        the host rows are kept in last_rows), the memory is marked trained, and Model_VV.train_rows trains on them on a thread of its own.
        The search keeps its weights until install(); due(m) says whether they are to be installed after move m: from move + train_lag on
        (move None: the move after_move() last named).
        At most one training is in flight: the caller installs the previous one first.  Returns False, with nothing started, when there
        are too few rows for a validation split."""
        import threading
        from .model.model_vv import rows_validation_size
        if self._pending is not None:
            raise RuntimeError("OnlineTrainer.start: the previous training is not installed (install() first)")
        t0 = time.perf_counter()
        self._peek(n_rows)
        self.last_rows = None
        enough = rows_validation_size(n_rows) > 0                  # train_rows skips fewer rows: decided here, before anything starts
        if dump_path and enough and self.rank == 0:
            self.last_rows = self.buf[:n_rows].cpu().numpy()
            os.makedirs(os.path.dirname(dump_path) or ".", exist_ok=True)
            replay.dump(dump_path, self.last_rows)
        if not enough:
            return False
        if self.rank == 0:
            self.eng.replay_policy_trained(current_episode)        # ++n_trains; memory_index = 0; last_training_episode (agent.cpp:697-701)
        seed = self.n_trains
        self.n_trains += 1
        job = dict(move=(self.move if move is None else int(move)) + self.train_lag, weights=None, error=None)
        job["thread"] = threading.Thread(target=self._train, args=(job, int(n_rows), seed, t0), name="b200-train", daemon=True)
        self._pending = job
        job["thread"].start()
        return True

    def _train(self, job, n_rows, seed, t0):
        """The training thread: Model_VV's trainer and validation engine, and torch, on the engine's device and on a stream of their own"""
        import torch
        try:
            with torch.cuda.device(self.buf.device), torch.cuda.stream(self._stream()):
                m = self._model()
                t = m._trainer_obj()
                if m._dp is None and self._streamed is not t:     # data-parallel training orders its exchange on a stream of its own
                    t.set_stream(self._stream().cuda_stream)
                    self._streamed = t
                m.train_rows(self.buf.data_ptr(), n_rows, seed=seed, **self.kw)
                job["weights"] = m.weights.copy()
        except BaseException as exc:                               # noqa: BLE001 (raised by install(), on the caller's thread)
            job["error"] = exc
        self.train_seconds += time.perf_counter() - t0

    def _stream(self):
        """the training's CUDA stream: non-blocking, of priority TRAIN_PRIORITY"""
        import torch
        if self._train_stream is None:
            self._train_stream = torch.cuda.Stream(device=self.buf.device, priority=self.TRAIN_PRIORITY)
        return self._train_stream

    def due(self, move):
        """whether the training in flight is to be installed now that move `move` is complete"""
        return self._pending is not None and move >= self._pending["move"]

    def join(self):
        """Wait for the training in flight, if any; it stays pending (not installed).  Raises what the training raised."""
        job = self._pending
        if job is None:
            return
        t0 = time.perf_counter()
        job["thread"].join()
        self.wait_seconds += time.perf_counter() - t0
        if job["error"] is not None:
            self._pending = None
            raise job["error"]

    def install(self):
        """Wait for the training in flight, if any, and load its weights into the engine's search.  Returns whether there was one."""
        if self._pending is None:
            return False
        self.join()
        self.weights = self._pending["weights"]
        self._pending = None
        self.eng.load_weights(self.weights)                        # the search now evaluates with the trained network
        return True

    def state(self):
        """What a resumed run needs to train on exactly as this one would: n_trains (it seeds the batch draws), train_seconds, the search's
        weights, once the trainer exists its Yogi state (exp_avg, exp_avg_sq, step), and a training not yet installed as pending: its
        install move and weights (the training in flight is joined first, so the trainer's state includes it)."""
        self.join()
        st = dict(n_trains=self.n_trains, train_seconds=self.train_seconds, weights=None if self.weights is None else self.weights.copy(),
                  optimizer=None, pending=None)
        if self._pending is not None:
            st["pending"] = dict(move=self._pending["move"], weights=self._pending["weights"].copy())
        if self.model is not None and self.model._trainer is not None:
            m, v, step = self.model._trainer.state()
            st["optimizer"] = (m, v, step)
        return st

    def restore(self, state):
        """The inverse of state(): weights into the engine's search and the trainer (created here if the state has optimiser moments); a
        pending training is installed when due() says so."""
        self.n_trains, self.train_seconds = int(state["n_trains"]), float(state["train_seconds"])
        if state["weights"] is not None:
            self.weights = state["weights"]
            self.eng.load_weights(self.weights)
        pending = state.get("pending")
        trained = self.weights if pending is None else pending["weights"]
        if state["optimizer"] is not None:
            m = self._model()
            m.weights = trained
            m._eng.load_weights(trained)
            t = m._trainer_obj()
            t.set_weights(trained)
            t.set_state(*state["optimizer"])
        if pending is not None:
            self._pending = dict(move=int(pending["move"]), weights=pending["weights"], error=None, thread=_Finished())

    def close(self):
        """Waits for a training in flight (its error, if any, is dropped: close runs when the run ends, also on an error of its own)."""
        if self._pending is not None:
            self._pending["thread"].join()
            self._pending = None
        if self.model is not None:
            self.model.close()
            self.model = None


class _Finished:
    """the thread of a restored pending training, which ended before the checkpoint"""

    def join(self):
        pass


class CallbackTrainer(OnlineTrainer):
    """OnlineTrainer's interface around the caller's training function: OnlineMCTSAgent(..., train=) (agent.cpp:588-616), called where
    remove_nodes calls train(m_state, m_value, m_variance, m_visit, memory_index) (agent.cpp:698).

    train(state, value, variance, visit, size) receives the first `size` rows of the memory as the reference's arrays: float32 states
    [size,1,20,10] and value / variance / visit [size,1].  host=False: contiguous torch tensors on the engine's device, re-laid out from the
    device rows (replay.rows_to_memory_dev) and valid until the call returns; host=True: numpy arrays (replay.rows_to_memory), so that a
    ValueSimC-style training() runs as it is.

    external=True (eval_kind "external"): the caller's network searches and the callback updates it in place; it returns None.  Otherwise
    the engine's own network kernels search, and the callback returns the new weights (a Model_VV state_dict with out_ubound / out_lbound,
    or a flat float32 array of N_WEIGHTS), which the engine loads, or None to keep the current ones.

    A callback that raises, or weights the engine refuses (wrong form, or out of a tensor-core kind's limits), raise here before the memory
    is marked trained or the search's weights change.  Under a process group every rank's callback receives rank 0's rows; rank 0's returned
    weights are broadcast and loaded on every rank.  A caller's network (external) is the caller's to keep in step across ranks."""

    def __init__(self, eng, weights, capacity, train, host=False, external=False):
        super().__init__(eng, weights, capacity)
        self.fn, self.host, self.external = train, bool(host), bool(external)

    def train(self, n_rows, current_episode, dump_path=None):
        import torch
        t0 = time.perf_counter()
        self._peek(n_rows)
        rows = self.buf[:n_rows]
        self.last_rows = rows.cpu().numpy() if self.host or (dump_path and self.rank == 0) else None
        if dump_path and self.rank == 0:
            os.makedirs(os.path.dirname(dump_path) or ".", exist_ok=True)
            replay.dump(dump_path, self.last_rows)
        memory = replay.rows_to_memory(self.last_rows) if self.host else replay.rows_to_memory_dev(rows)
        result = self.fn(*memory, int(n_rows))
        torch.cuda.synchronize(self.buf.device)                   # the caller's work on torch's streams ends before the engine's stream searches on
        if self.external and result is not None:
            raise ValueError("with the caller's evaluator (eval_kind external) the training callback updates that network in place and returns "
                             "None, not weights")
        if not self.external:
            self._load(result)
        if self.rank == 0:
            self.eng.replay_policy_trained(current_episode)        # ++n_trains; memory_index = 0; last_training_episode (agent.cpp:699-701)
        self.n_trains += 1
        self.train_seconds += time.perf_counter() - t0
        return True

    def _load(self, result):
        """rank 0's returned weights into every rank's engine (None: keep them).  Refused weights raise on every rank and change nothing."""
        code, w, err = 0, None, None                               # 0 keep, 1 load w, 2 refused
        if self.rank == 0 and result is not None:
            try:
                w = weights_vector(result)
                self.eng.load_weights(w)                           # checks a tensor-core kind's limits before it changes anything
                code = 1
            except Exception as exc:                               # noqa: BLE001 (re-raised below, after the other ranks have heard of it)
                code, err = 2, exc
        if distributed.rank_world()[1] > 1:
            code = distributed.broadcast_ints([code])[0]
            if code == 1:
                w = distributed.broadcast_weights(w)
                if self.rank != 0:
                    self.eng.load_weights(w)
        if code == 2:
            raise err if err is not None else ValueError("rank 0's training callback returned weights its engine refused")
        if code == 1:
            self.weights = w


def weights_vector(w):
    """A training callback's weights -> the engine's float32 vector: a Model_VV state_dict (model_vv.WEIGHT_KEYS, torch tensors or arrays)
    or a flat float32 array / tensor of N_WEIGHTS.  Anything else raises ValueError."""
    import numpy as np
    from . import _lib as L
    from .model.model_vv import WEIGHT_KEYS, state_dict_to_weights
    if hasattr(w, "keys"):
        missing = [k for k, _shape in WEIGHT_KEYS if k not in w]
        if missing:
            raise ValueError("the returned state_dict has no %s" % ", ".join(missing))
        return state_dict_to_weights(w)
    if hasattr(w, "detach"):
        w = w.detach().cpu().numpy()
    if not isinstance(w, np.ndarray) or w.dtype != np.float32 or w.shape != (L.N_WEIGHTS,):
        raise ValueError("a training callback returns None, a Model_VV state_dict or float32 weights of shape (%d,); got %s" % (
            L.N_WEIGHTS, (w.dtype, w.shape) if isinstance(w, np.ndarray) else type(w).__name__))
    return w.copy()
