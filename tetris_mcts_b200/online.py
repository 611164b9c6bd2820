"""The training half of the online agent's remove_nodes on the device (agents/ValueSim.py:101-115,161-185; OnlineMCTSAgent::remove_nodes
agent.cpp:619-708): once the engine's replay policy says train, the rows of the device replay memory are copied to a device buffer
(b200_replay_peek_dev), Model_VV.train_rows trains the value network on them without a host copy, the engine searches on with the new
weights, and the policy is told that the memory was trained on.  Used by agents.ValueSim (online=True) and play_batched --online.

Under a torch.distributed process group (play_batched under torchrun) rank 0's engine holds the memory and the policy: rank 0 copies the rows
out and broadcasts them into every rank's buffer, and all ranks train data-parallel on them (Model_VV.train_rows)."""
import os
import time

from . import distributed, replay
from .model.model_vv import EXP_PATH


class OnlineTrainer:
    def __init__(self, eng, weights, capacity, batch_size=1024, iters_per_val=100, max_iters=50000, checkpoint=EXP_PATH + "model_checkpoint",
                 train_kind="fp64"):
        import torch
        from .model.trainer import KINDS
        if train_kind not in KINDS:
            raise ValueError("train_kind must be one of %s, not %r" % (sorted(KINDS), train_kind))
        self.train_kind = train_kind
        dev = torch.device("cuda", int(eng.cfg.device))            # the engine's device, not torch's current one
        self.buf = torch.empty((int(capacity), replay.SAMPLE_BYTES), dtype=torch.uint8, device=dev)
        torch.cuda.synchronize(dev)                                # the engine copies on its own stream: nothing of torch's may be pending on buf
        self.eng, self.weights = eng, weights
        self.kw = dict(batch_size=int(batch_size), iters_per_val=int(iters_per_val), max_iters=int(max_iters), checkpoint=checkpoint)
        self.model, self.n_trains, self.train_seconds, self.last_rows = None, 0, 0.0, None
        self.rank = distributed.rank_world()[0]

    def _model(self):
        if self.model is None:
            from .model.model_vv import Model_VV
            self.model = Model_VV(device=int(self.eng.cfg.device), eval_kind="net", train_kind=self.train_kind)
            self.model.weights = self.weights
            self.model._eng.load_weights(self.weights)
        return self.model

    def train(self, n_rows, current_episode, dump_path=None):
        """Train on the first n_rows rows of the engine's memory (ValueSim.py:176-183 / agent.cpp:697-701).  dump_path: also write them as
        np.savez(dump_path, states=, values=, variance=, weights=) (ValueSim.py:176-177); the host rows are kept in last_rows.  Returns False
        (memory untouched, still collecting) when there are too few rows for a validation split."""
        t0 = time.perf_counter()
        if self.rank == 0:
            self.eng.replay_peek_into(self.buf.data_ptr(), n_rows)  # synchronises the engine's stream
        distributed.broadcast_rows(self.buf, n_rows)               # world > 1: rank 0's rows on every rank
        self.last_rows = None
        if dump_path and n_rows >= 10 and self.rank == 0:                             # fewer rows leave no validation split: train_rows skips them
            self.last_rows = self.buf[:n_rows].cpu().numpy()
            os.makedirs(os.path.dirname(dump_path) or ".", exist_ok=True)
            replay.dump(dump_path, self.last_rows)
        m = self._model()
        if not m.train_rows(self.buf.data_ptr(), n_rows, seed=self.n_trains, **self.kw):
            return False
        self.weights = m.weights
        self.eng.load_weights(self.weights)                        # the search now evaluates with the trained network
        if self.rank == 0:
            self.eng.replay_policy_trained(current_episode)        # ++n_trains; memory_index = 0; last_training_episode (agent.cpp:697-701)
        self.n_trains += 1
        self.train_seconds += time.perf_counter() - t0
        return True

    def close(self):
        if self.model is not None:
            self.model.close()
            self.model = None
