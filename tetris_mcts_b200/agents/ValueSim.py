"""agents.ValueSim — agents/ValueSim.py:12-99 (leaf itself evaluated, gamma=0.999, max_nodes=100000)."""
from sys import stderr

import numpy as np

from .agent import TreeAgent
from ..model.model_vv import init_weights, load_checkpoint_weights

perr = dict(file=stderr, flush=True)


class ValueSim(TreeAgent):
    _mode = "single"

    def __init__(self, online=True, memory_size=500000, min_visits_to_store=10, gamma=0.999, memory_growth_rate=5000, weights=None,
                 train_kind="fp64", **kwargs):
        kwargs.pop("max_nodes", None)
        if kwargs.get("evaluator") is not None and online and not kwargs.get("benchmark", False):
            raise ValueError("online=True trains the engine's Model_VV weights on the device, not the caller's evaluator: pass online=False")
        if weights is None and kwargs.get("evaluator") is None:
            # ValueSim.py:42-44: self.model = Model(); self.model.load(); self.model.training(False).  Model.load (model/model.py:163-174)
            # reads ./pytorch_model/model_checkpoint when it exists and otherwise keeps the default-initialised network.
            weights = load_checkpoint_weights()
            if weights is None:
                weights = init_weights(0)
        super().__init__(max_nodes=100000, gamma=gamma, low=1, weights=weights, **kwargs)   # ValueSim.py:16
        self.online, self.min_visits_to_store = online, min_visits_to_store
        self.memory_size, self.memory_growth_rate, self.n_trains = memory_size, memory_growth_rate, 0   # ValueSim.py:21-37
        self._weights, self._online = np.asarray(weights, np.float32), None
        if online and not self.benchmark:                         # ValueSim.py:21-37: the replay memory lives on the device (k_gc fills it)
            from ..online import OnlineTrainer
            self._eng.replay_enable(min_visits=min_visits_to_store, capacity=memory_size)
            # accumulation policy 3 is train_nodes' rule: train once memory_index >= min(n_trains * memory_growth_rate, memory_size)
            self._eng.replay_policy(3, memory_growth_rate=memory_growth_rate)
            self._online = OnlineTrainer(self._eng, self._weights, memory_size, batch_size=1024, iters_per_val=100, max_iters=50000,
                                         train_kind=train_kind)   # ValueSim.py:180
            self._gcs = 0
            print('online: freed observations are stored on the device as in ValueSim.store_nodes (ValueSim.py:122-159) and the value network '
                  'is trained on them after the collections that fill the memory (train_nodes, ValueSim.py:161-185)', **perr)

    @property
    def model(self):
        return self._online.model if self._online else None

    def _after_collections(self):
        """remove_nodes' store_nodes + train_nodes (ValueSim.py:101-115) after a call in which the engine collected (gcs counter moved)"""
        if self._online is None:
            return
        gcs = self._eng.counters()["gcs"]
        if gcs != self._gcs:
            self._gcs = gcs
            self.train_nodes()

    def play(self):
        action = super().play()
        self._after_collections()
        return action

    def update_root(self, game):
        super().update_root(game)
        self._after_collections()

    def remove_nodes(self):
        super().remove_nodes()
        self._after_collections()

    def train_nodes(self, dump_data=True, path='./data/dump'):    # ValueSim.py:161-185
        """When memory_index >= min(n_trains * memory_growth_rate, memory_size): dump the memory (np.savez('./data/dump', ...),
        ValueSim.py:176-177), run Model_VV.train_rows on the device rows (ValueSim.py:180: iters_per_val=100, batch_size=1024,
        max_iters=50000) and hot-swap the search network.  Returns the memory arrays used for training, or None while still collecting
        (ValueSim.py:170-172)."""
        from .. import replay
        if self._online is None:
            return None
        print('Training...', **perr)
        train_now, d_size = self._eng.replay_policy_step(self.episode)
        m_size = min(self.n_trains * self.memory_growth_rate, self.memory_size)
        if not train_now:
            print('Not enough training data ({} < {}), collecting more data.'.format(d_size, m_size), **perr)
            return None
        print('Enough training data ({} >= {}), proceed to training.'.format(d_size, m_size), **perr)
        if not self._online.train(d_size, self.episode, dump_path=path if dump_data else None):
            return None
        if not dump_data:
            self._online.last_rows = self._online.buf[:d_size].cpu().numpy()
        self.n_trains += 1
        self._weights = self._online.weights
        print('Training complete.', **perr)
        return replay.rows_to_memory(self._online.last_rows)

    def close(self):
        if self._online is not None:
            self._online.close()
        super().close()

    def evaluate_state(self, state):                              # ValueSim.py:46-50
        v, var = self._eng.valuenet(state[None])
        return v[0], var[0]
