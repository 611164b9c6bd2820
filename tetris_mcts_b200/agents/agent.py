"""agents.agent — the Agent / TreeAgent surface of the reference (agents/agent.py:10-307) over the CUDA engine.

play.py (unchanged) constructs `Agent(sims=, env=, env_args=, benchmark=, online=, min_visit=)` (play.py:83-89) and calls
update_root(game), play(), close() and, through util/Data.py:65-89, get_prob(), get_stats(), get_value_and_variance().
The tree lives in HBM; `arrays`, `obs_arrays`, `node_to_obs` and `game_arr` are read-only snapshots downloaded on demand
in the reference's layout (agents/agent.py:58-88)."""
from sys import stderr

import numpy as np

from .. import _lib as L
from ..engine import BatchedEngine
from ..pyTetris import Tetris

perr = dict(file=stderr, flush=True)


class Agent:                                                     # agents/agent.py:10-31
    def __init__(self, n_actions=7, benchmark=False, **kwargs):
        self.episode = 0
        self.n_actions = n_actions
        self.benchmark = benchmark

    def play(self):
        raise NotImplementedError('update_root not implemented')

    def get_action(self):
        raise NotImplementedError('get_action not implemented')

    def get_prob(self):
        raise NotImplementedError('get_action not implemented')

    def update_root(self, game):
        raise NotImplementedError('update_root not implemented')

    def close(self):
        raise NotImplementedError('close not implemented')


class _GameArr:
    """game_arr[idx] -> a Tetris handle of node idx (agents/agent.py:70), built from the downloaded record."""

    def __init__(self, agent):
        self._agent = agent

    def __getitem__(self, idx):
        rec = self._agent._snapshot()["game"][idx]
        return Tetris((20, 10), int(rec[11]) & 0xff, (int(rec[10]) >> 22) & 1, (int(rec[10]) >> 23) & 1, _record=rec)

    def __len__(self):
        return self._agent.max_nodes


class TreeAgent(Agent):                                          # agents/agent.py:34-307
    _mode = "lp"

    def __init__(self, sims=100, max_nodes=500000, env=None, env_args=None, node_saver=None, projection=True, min_visits=30,
                 gamma=0.999, low=1, eval_kind="net_tc", weights=None, device=0, overflow_reset=False, evaluator=None,
                 evaluator_on_device=False, **kwargs):
        """evaluator: the reference's evaluator callback (OnlineMCTSAgent(..., evaluator=, evaluation_type=0), agents/ValueSimC.py;
        ValueSimLP's self.model.inference): the engine then runs eval_kind "external" and mcts() hands every simulation step's boards to
        it.  evaluator_on_device=False: int8 ndarray [n,1,20,10] in, [v (n,1), var (n,1)] or [probs (n, atoms)] out (Model_VV.inference
        as it is); True: a torch tensor on the engine's device in, torch float32 out (BatchedEngine.run_sims)."""
        super().__init__(**kwargs)
        if not projection:
            raise NotImplementedError("only projection=True is live in the reference (SURVEY N4)")
        self.sims, self.max_nodes = sims, int(max_nodes) & ~3
        self.env, self.env_args = env, env_args if env_args is not None else ((20, 10), 1, 0, 0)
        self.episode, self.min_visits, self.node_saver, self.projection = 0, min_visits, node_saver, projection
        self.gamma = gamma
        self._evaluator, self._evaluator_on_device = evaluator, bool(evaluator_on_device)
        if evaluator is not None:
            eval_kind, weights = "external", None
        self.stats = np.zeros((3, self.n_actions), np.float32)
        self._eng = BatchedEngine(1, max_nodes=self.max_nodes, mode=self._mode, gamma=gamma, low=low, eval_kind=eval_kind, weights=weights,
                                  env_args=self.env_args, device=device, overflow_reset=overflow_reset, **self._engine_kwargs())
        self._snap = None
        self.game_arr = _GameArr(self)

    def _engine_kwargs(self):
        return {}

    # ---- snapshots in the reference layout
    def _snapshot(self):
        if self._snap is None:
            self._snap = self._eng.export_game(0)
        return self._snap

    @property
    def root(self):
        return self._snapshot()["root"]

    @property
    def arrays(self):
        s = self._snapshot()
        z = np.zeros(self.max_nodes, np.float32)
        return {"child": s["child"], "visit": np.zeros(self.max_nodes, np.int32), "value": z, "variance": z.copy(), "episode": s["episode"],
                "score": s["score"], "end": np.zeros(self.max_nodes, bool)}     # node-indexed stats are never written (SURVEY N1)

    @property
    def obs_arrays(self):
        s = self._snapshot()
        from ..pyTetris import states_of  # noqa: F401
        return {"visit": s["visit"], "value": s["value"], "variance": s["variance"], "end": s["obs_end"].astype(bool), "key": s["obs_key"]}

    @property
    def node_to_obs(self):
        return self._snapshot()["n2o"]

    # ---- the calls play.py makes
    def update_root(self, game):                                  # agents/agent.py:296-301
        self._snap = None
        self._eng.set_games(game.get_record().reshape(1, L.REC_WORDS))
        if game.end:
            self.episode += 1

    def mcts(self, root_index=None, sims=None):                   # agents/agent.py:132 (overridden per agent type)
        self._snap = None
        self._eng.run_sims(self.sims if sims is None else sims, evaluator=self._evaluator, host=not self._evaluator_on_device)

    def play(self):                                               # agents/agent.py:147-151
        self.mcts(None, self.sims)
        return self.get_action()

    def compute_stats(self, idx=None):                            # agents/agent.py:153-179
        if idx is None:
            stats, _ = self._eng.get_stats()
            return stats[0]
        s = self._snapshot()
        out = np.zeros((3, self.n_actions), np.float32)
        for i, c in enumerate(s["child"][idx]):
            o = s["n2o"][c]
            out[0, i] = s["visit"][o]
            out[1, i] = s["value"][o] + (s["score"][c] - s["score"][idx])
            out[2, i] = s["variance"][o]
        return out

    def get_action(self):                                         # agents/agent.py:181-185
        self.stats = self.compute_stats()
        return int(np.argmax(self.stats[1]))

    def get_prob(self):
        return self.stats[0] / np.sum(self.stats[0])

    def get_stats(self):
        return np.copy(self.stats)

    def get_value_and_variance(self, node=None):                  # agents/agent.py:195-204
        s = self._snapshot()
        o = s["n2o"][s["root"] if node is None else node]
        return s["value"][o], s["variance"][o]

    def remove_nodes(self):                                       # agents/agent.py:246-257 (also run on the device where new_node needs it, :96-97)
        self._snap = None                                         # the collection frees and zeroes slots: snapshots are stale
        self._eng.remove_nodes()

    def counters(self):
        return self._eng.counters()

    def close(self):                                              # agents/agent.py:303-307
        if self.node_saver:
            self.node_saver.close()
        self._eng.close()
