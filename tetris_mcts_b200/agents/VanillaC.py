"""agents.VanillaC — agents/VanillaC.py: the C++ agent's rollout MCTS (MCTSAgent(sims, max_nodes, projection, gamma, benchmark,
random_playout, 1, False), agents/cppmodule/agent.cpp:415-460): selection_obs(1), the leaf game evaluated by a game evaluator and backed up
as it returns it.  The engine runs eval_kind "external_game" in mode "vanilla"."""
from ..pyTetris import playout_evaluator
from .agent import TreeAgent


class VanillaC(TreeAgent):
    _mode = "vanilla"

    def __init__(self, sims=100, max_nodes=500000, projection=True, gamma=0.99, benchmark=False, LP=False, game_evaluator=None,
                 game_evaluator_on_device=True, **kwargs):
        """game_evaluator: f(recs) -> (v, var) in place of random_playout (BatchedEngine.run_sims(game_evaluator=)): on the device (int32
        records [n,20] in, torch float32 out) or, with game_evaluator_on_device=False, numpy uint32 records in and numpy float32 out
        (pyTetris.per_game(random_playout) is the reference's own function on that form).  None: random_playout restated on the device,
        playout_dev with n_actions=8 (randint(0, 7), the no-op 7 included) and (score, 1e5).  LP is ignored, as agent.cpp ignores it for
        evaluator type 1."""
        kwargs.pop("online", None)
        kwargs.pop("min_visit", None)
        if kwargs.get("evaluator") is not None:
            raise ValueError("VanillaC evaluates leaf games; pass game_evaluator=, not evaluator=")
        super().__init__(sims=sims, max_nodes=max_nodes, projection=projection, gamma=gamma, low=1, eval_kind="external_game",
                         benchmark=benchmark, **kwargs)                    # agent.cpp:417 selection_obs(1)
        self._game_evaluator = game_evaluator if game_evaluator is not None else playout_evaluator(n_actions=8, variance=1e5)
        self._game_host = game_evaluator is not None and not game_evaluator_on_device

    def mcts(self, root_index=None, sims=None):
        self._snap = None
        self._eng.run_sims(self.sims if sims is None else sims, game_evaluator=self._game_evaluator, host=self._game_host)
