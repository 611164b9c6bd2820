"""agents.DistValueSimOnline — the distributional agent of agents/DistValueSimOnline.py:11-116 (atoms=50, vmin=0, vmax=5000).
Upstream the file is not runnable (it imports a module that does not exist and calls undefined functions, SURVEY §2 row 7);
the search loop it sketches (:36-75) is driven here on the reference's distributional cores
(agents/core_distributional.py:82-124) by the CUDA engine in B200_MODE_DIST.  play.py does
getattr(module, 'DistValueSimOnline') (play.py:82), so the class is exported under both names."""
import os
from collections.abc import Mapping

import numpy as np

from .. import _lib as L
from .agent import TreeAgent


def init_dist_weights(seed=0, atoms=50):
    """Default-init-distributed weights of model/model_distributional.py:18-45 Net (22x10 input, flatten 2048), numpy PCG64."""
    rng = np.random.default_rng(seed + 1000)
    parts = []
    for shape, fan_in in (((32, 1, 4, 4), 16), ((32,), 16), ((32, 32, 4, 4), 512), ((32,), 512), ((128, 2048), 2048), ((128,), 2048),
                          ((atoms, 128), 128), ((atoms,), 128)):
        b = 1.0 / np.sqrt(fan_in)
        parts.append(rng.uniform(-b, b, size=shape).astype(np.float32).ravel())
    return np.concatenate(parts)


def _dist_weight_vector(w, atoms):
    """a state_dict or a checkpoint path -> the weight vector (model/model_distributional.py); a vector passes as it is"""
    from ..model.model_distributional import load_checkpoint_dist_weights, state_dict_to_dist_weights
    if isinstance(w, (str, bytes, os.PathLike)):
        if not os.path.isfile(w):
            raise ValueError("no distributional checkpoint at %s" % (w,))
        return load_checkpoint_dist_weights(w, atoms)
    if isinstance(w, Mapping):
        return state_dict_to_dist_weights(w, atoms)
    return w


class DistValueSim(TreeAgent):
    _mode = "dist"

    def __init__(self, atoms=50, vmin=0, vmax=5000, dist_weights=None, **kwargs):          # DistValueSimOnline.py:13
        """dist_weights: None (init_dist_weights(0, atoms)), the flat weight vector, a Net(atoms) state_dict or the path of a checkpoint
        Model_Dist.save / the reference's Model.save wrote (model/model_distributional.py)."""
        kwargs.pop("max_nodes", None)
        kwargs.pop("online", None)
        kwargs.pop("min_visit", None)
        self.atoms, self.vrange = atoms, (vmin, vmax)
        super().__init__(max_nodes=100000, low=5, eval_kind=kwargs.pop("eval_kind", "net"), **kwargs)
        if self._eng.eval_kind not in (L.EVAL_SYNTHETIC, L.EVAL_EXTERNAL):
            self._eng.load_dist_weights(init_dist_weights(0, atoms) if dist_weights is None else _dist_weight_vector(dist_weights, atoms), atoms)

    def _engine_kwargs(self):
        return dict(dist_bins=self.atoms, dist_vmin=self.vrange[0], dist_vmax=self.vrange[1])

    def get_value(self, node=None):                                                         # DistValueSimOnline.py:106-116
        ns, nd = self._eng.export_dist(0)
        idx = self.root if node is None else node
        from .core_distributional import mean_variance
        return mean_variance(nd[idx], *self.vrange)


DistValueSimOnline = DistValueSim
