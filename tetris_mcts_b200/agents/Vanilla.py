"""agents.Vanilla — agents/Vanilla.py:8-64 (random-rollout MCTS: low=5, gamma=0.99, rollout variance 1e3)."""
from .agent import TreeAgent


class Vanilla(TreeAgent):
    _mode = "vanilla"

    def __init__(self, gamma=0.99, **kwargs):
        kwargs.pop("online", None)
        kwargs.pop("min_visit", None)
        if kwargs.get("evaluator") is not None:
            raise ValueError("Vanilla evaluates leaves by random rollout; it takes no evaluator")
        super().__init__(projection=True, gamma=gamma, low=5, **kwargs)   # Vanilla.py:11, :27
