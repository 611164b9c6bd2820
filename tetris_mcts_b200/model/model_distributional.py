"""Model_Dist — host-side mirror of the reference's distributional network wrapper (model/model_distributional.py:18-102 on model/model.py)
for the calls an agent makes: Model_Dist().load(); .training(False); .inference(batch) -> [probs (k, atoms)]; .save().  The forward pass
runs on the GPU through the C-ABI (b200_distnet_forward, the kernels of the engine's eval_kind); weights are the reference's state_dict
tensors seq.conv1.weight ... seq.fc_v.bias concatenated in that order (b200_load_dist_weights).  Training the distributional network is
not built: Model_Dist has no train."""
import os
from collections import OrderedDict

import numpy as np

EXP_PATH = "./pytorch_model/"          # model/model_distributional.py:13 (the same directory as Model_VV's, model/model.py:11)


def dist_weight_keys(atoms=50):
    """(name, shape) of Net(atoms)'s state_dict (model_distributional.py:18-45: 22x10 input, two 4x4 convolutions, flatten 2048), in its order"""
    return (("seq.conv1.weight", (32, 1, 4, 4)), ("seq.conv1.bias", (32,)), ("seq.conv2.weight", (32, 32, 4, 4)), ("seq.conv2.bias", (32,)),
            ("seq.fc1.weight", (128, 2048)), ("seq.fc1.bias", (128,)), ("seq.fc_v.weight", (int(atoms), 128)), ("seq.fc_v.bias", (int(atoms),)))


def n_dist_weights(atoms=50):
    return sum(int(np.prod(s)) for _n, s in dist_weight_keys(atoms))


def _check_state_dict(sd, atoms):
    """ValueError naming every key of Net(atoms) that sd lacks or holds with another shape, and every key it has beyond them"""
    want = OrderedDict(dist_weight_keys(atoms))
    missing = [k for k in want if k not in sd]
    shapes = ["%s %s (Net(atoms=%d) has %s)" % (k, tuple(sd[k].shape), atoms, want[k]) for k in want if k in sd and tuple(sd[k].shape) != want[k]]
    extra = [k for k in sd if k not in want]
    if missing or shapes or extra:
        parts = (["missing " + ", ".join(missing)] if missing else []) + (["shape " + "; ".join(shapes)] if shapes else []) + \
                (["unexpected " + ", ".join(extra)] if extra else [])
        raise ValueError("not a state_dict of the distributional network Net(atoms=%d) (model_distributional.py): %s"
                         % (atoms, " | ".join(parts)))


def state_dict_to_dist_weights(sd, atoms=50):
    """A Net(atoms) state_dict (torch tensors or arrays) -> the float32 vector b200_load_dist_weights takes.  Any other state_dict (a
    Model_VV one, another atoms) raises ValueError naming the mismatch."""
    _check_state_dict(sd, int(atoms))
    parts = []
    for name, _shape in dist_weight_keys(atoms):
        t = sd[name]
        a = t.detach().cpu().numpy() if hasattr(t, "detach") else np.asarray(t)
        parts.append(np.ascontiguousarray(a, np.float32).ravel())
    return np.concatenate(parts)


def dist_weights_to_state_dict(w, atoms=50):
    """The weight vector as Net(atoms)'s state_dict (torch tensors, keys and shapes of model_distributional.py:18-45, in its order)"""
    import torch
    w = np.asarray(w, np.float32).ravel()
    if w.size != n_dist_weights(atoms):
        raise ValueError("expected %d floats for atoms=%d, got %d" % (n_dist_weights(atoms), atoms, w.size))
    sd, off = OrderedDict(), 0
    for name, shape in dist_weight_keys(atoms):
        n = int(np.prod(shape))
        sd[name] = torch.from_numpy(w[off:off + n].reshape(shape).copy())
        off += n
    return sd


def load_checkpoint_dist_weights(filename=EXP_PATH + "model_checkpoint", atoms=50):
    """Model.load (model/model.py:163-174) for Model_Dist: the checkpoint's model_state_dict as the weight vector, or None (after the
    reference's own message) when the file does not exist.  A checkpoint of another network (Model_VV writes the same path) raises
    ValueError naming the mismatch."""
    if os.path.isfile(filename):
        import torch
        print("Loading model...", flush=True)
        ck = torch.load(filename, map_location="cpu", weights_only=False)
        if not isinstance(ck, dict) or "model_state_dict" not in ck:
            raise ValueError("%s: not a checkpoint of model/model.py's layout (no model_state_dict)" % filename)
        try:
            return state_dict_to_dist_weights(ck["model_state_dict"], atoms)
        except ValueError as exc:
            raise ValueError("%s: %s" % (filename, exc)) from None
    print("Checkpoint not found, using default model", flush=True)
    return None


def holds_dist_state_dict(filename, atoms=50):
    """True when `filename` is a checkpoint whose model_state_dict is Net(atoms)'s (no message, no exception otherwise)"""
    if not os.path.isfile(filename):
        return False
    import torch
    try:
        ck = torch.load(filename, map_location="cpu", weights_only=False)
        _check_state_dict(ck["model_state_dict"], int(atoms))
        return True
    except Exception:
        return False


def boards_20x10(batch):
    """inference's input -> int8 [n, 200]: [n,1,20,10] boards, or the reference's own [n,1,22,10] input when its top two rows are empty (the
    kernels pad a 20x10 board with exactly those two rows); anything else raises ValueError"""
    b = np.asarray(batch)
    if b.ndim == 4 and b.shape[1:] == (1, 22, 10):
        if np.any(b[:, :, :2]):
            raise ValueError("a [n,1,22,10] board must have its top two rows empty: the network pads 20x10 boards with two empty rows")
        b = b[:, :, 2:]
    if b.ndim != 4 or b.shape[1:] != (1, 20, 10):
        raise ValueError("inference takes boards [n,1,20,10] (or [n,1,22,10] with the top two rows empty), got shape %s" % (b.shape,))
    if not np.all((b == -1) | (b == 0) | (b == 1)):
        raise ValueError("board cells are -1, 0 or 1 (Tetris.getState)")
    return np.ascontiguousarray(b, np.int8).reshape(-1, 200)


class Model_Dist:
    """Model_Dist(atoms).load(); .training(flag); .inference(batch); .save()  (model/model_distributional.py:60-102 on model/model.py).
    eval_kind: the kernels of the forward pass, as the engine's ("net" fp32 CUDA cores, "net_tc" tensor cores within 1e-5 of fp32,
    "dist_fp16" one fp16 term per operand).  Weights start as init_dist_weights(0, atoms)."""

    def __init__(self, atoms=50, device=0, eval_kind="net", weights=None):
        from ..agents.DistValueSimOnline import init_dist_weights
        from ..engine import BatchedEngine
        self.atoms, self.device, self.eval_kind = int(atoms), device, eval_kind
        self._eng = BatchedEngine(1, max_nodes=64, mode="dist", eval_kind=eval_kind, dist_bins=self.atoms, device=device)
        self._set(init_dist_weights(0, self.atoms) if weights is None else weights)
        self._training = False

    def _set(self, w):
        w = np.ascontiguousarray(w, np.float32).ravel()
        self._eng.load_dist_weights(w, self.atoms)
        self.weights = w

    def load(self, filename=EXP_PATH + "model_checkpoint"):           # model/model.py:163-174
        w = load_checkpoint_dist_weights(filename, self.atoms)
        if w is not None:
            self._set(w)

    def save(self, filename=EXP_PATH + "model_checkpoint", verbose=True):   # model/model.py:143-160: the same file layout, no optimiser state
        import torch
        if verbose:
            print("Saving model...", flush=True)
        d = os.path.dirname(filename) or "."
        if not os.path.isdir(d):
            if verbose:
                print("Export path does not exist, creating a new one...", flush=True)
            os.mkdir(d)
        torch.save({"model_state_dict": dist_weights_to_state_dict(self.weights, self.atoms),
                    "optimizer_state_dict": {"state": {}, "param_groups": []}}, filename)

    def state_dict(self):
        return dist_weights_to_state_dict(self.weights, self.atoms)

    def training(self, mode=True):                                    # model/model.py:121-126 (no train/eval-dependent layers)
        self._training = bool(mode)

    def inference(self, batch):                                       # model_distributional.py:95-102
        return [self._eng.distnet(boards_20x10(batch))]

    def train(self, *args, **kwargs):
        raise NotImplementedError("training the distributional network is out of scope: Model_Dist loads, saves and evaluates it only")

    train_data = train

    def close(self):
        self._eng.close()
