"""Model_VV — host-side mirror of the reference value-network wrapper (model/model_vv.py:104-231, base model/model.py:39-255)
for the calls the agents make: Model_VV().load(); .training(False); .inference(batch) -> [v (k,1), var (k,1)].
The forward pass runs on the GPU through the C-ABI (b200_valuenet_forward); weights are the reference's state_dict
tensors (head.conv1.weight ... head.fc_out.bias, out_ubound, out_lbound) concatenated in that order."""
import os
import sys
from collections import OrderedDict
from sys import stderr

import numpy as np

from .. import _lib as L

perr = dict(file=stderr, flush=True)

EXP_PATH = "./pytorch_model/"          # model/model.py:11
WEIGHT_KEYS = (("head.conv1.weight", (32, 1, 3, 3)), ("head.conv1.bias", (32,)), ("head.conv2.weight", (32, 32, 3, 3)),
               ("head.conv2.bias", (32,)), ("head.conv3.weight", (32, 32, 3, 3)), ("head.conv3.bias", (32,)),
               ("head.fc1.weight", (256, 1792)), ("head.fc1.bias", (256,)), ("head.fc_out.weight", (2, 256)),
               ("head.fc_out.bias", (2,)), ("out_ubound", (2,)), ("out_lbound", (2,)))


def init_weights(seed=0):
    """Random weights with the reference's default-init distribution (torch Conv2d/Linear: U(-1/sqrt(fan_in), +1/sqrt(fan_in))
    for weight and bias; out_ubound=[1e2,1e3], out_lbound=[0,1e-1], model_vv.py:45-46).  numpy PCG64 so that every box
    regenerates the same floats; no checkpoint of the current architecture ships with the reference (SURVEY §6)."""
    rng = np.random.default_rng(seed)
    parts = []
    for shape, fan_in in (((32, 1, 3, 3), 9), ((32,), 9), ((32, 32, 3, 3), 288), ((32,), 288), ((32, 32, 3, 3), 288),
                          ((32,), 288), ((256, 1792), 1792), ((256,), 1792), ((2, 256), 256), ((2,), 256)):
        b = 1.0 / np.sqrt(fan_in)
        parts.append(rng.uniform(-b, b, size=shape).astype(np.float32).ravel())
    parts.append(np.array([1e2, 1e3], np.float32))
    parts.append(np.array([0.0, 1e-1], np.float32))
    return np.concatenate(parts)


def state_dict_to_weights(sd):
    """Flatten a reference checkpoint's model_state_dict (torch tensors or arrays) into the C-ABI weight vector."""
    parts = []
    for name, shape in WEIGHT_KEYS:
        t = sd[name]
        a = t.detach().cpu().numpy() if hasattr(t, "detach") else np.asarray(t)
        if tuple(a.shape) != shape:
            raise ValueError("%s: expected %s, checkpoint has %s (SURVEY §6: old checkpoints do not match the live Net)" % (name, shape, a.shape))
        parts.append(a.astype(np.float32).ravel())
    return np.concatenate(parts)


def weights_to_state_dict(w):
    """The C-ABI weight vector as the reference's model_state_dict (torch tensors, model/model.py:152-156)."""
    import torch
    w = np.asarray(w, np.float32).ravel()
    sd, off = OrderedDict(), 0
    for name, shape in WEIGHT_KEYS:
        n = int(np.prod(shape))
        sd[name] = torch.from_numpy(w[off:off + n].reshape(shape).copy())
        off += n
    return sd


def optimizer_state_to_dict(exp_avg, exp_avg_sq, step):
    """torch.optim.Optimizer.state_dict() layout of the reference's Yogi (model/yogi.py:56-61: step, exp_avg, exp_avg_sq per trainable
    parameter; model/model.py:154): params are numbered in model.parameters() order, the two bound vectors (requires_grad=False) have no state."""
    import torch
    state = {}
    if exp_avg is not None and step is not None and step >= 0:
        off = 0
        for i, (name, shape) in enumerate(WEIGHT_KEYS[:10]):
            n = int(np.prod(shape))
            state[i] = {"step": int(step), "exp_avg": torch.from_numpy(np.asarray(exp_avg[off:off + n], np.float32).reshape(shape).copy()),
                        "exp_avg_sq": torch.from_numpy(np.asarray(exp_avg_sq[off:off + n], np.float32).reshape(shape).copy())}
            off += n
    return {"state": state, "param_groups": [{"lr": 1e-3, "betas": (0.9, 0.999), "eps": 1e-3, "weight_decay": 1e-3, "params": list(range(12))}]}


def optimizer_state_from_dict(d):
    if not d or not d.get("state"):
        return None
    m, v, step = [], [], 0
    for i, (name, shape) in enumerate(WEIGHT_KEYS[:10]):
        st = d["state"].get(i)
        if st is None:
            return None
        m.append(np.asarray(st["exp_avg"], np.float32).ravel())
        v.append(np.asarray(st["exp_avg_sq"], np.float32).ravel())
        step = int(st["step"])
    return np.concatenate(m), np.concatenate(v), step


def load_checkpoint_weights(filename=EXP_PATH + "model_checkpoint"):
    """Model.load (model/model.py:163-174): the checkpoint's model_state_dict as the C-ABI weight vector, or None (after the
    reference's own message) when the file does not exist — the agent then keeps its default-initialised network."""
    if os.path.isfile(filename):
        import torch
        print("Loading model...", flush=True)
        ck = torch.load(filename, map_location="cpu", weights_only=False)
        return state_dict_to_weights(ck["model_state_dict"])
    print("Checkpoint not found, using default model", flush=True)
    return None


def _combine_chunks(loss, std, bsize):
    """Model.compute_loss's combination of per-chunk (mean, std, size) into one (model/model.py:67-83)"""
    loss, std, bsize = np.array(loss), np.nan_to_num(np.array(std)), np.array(bsize)
    d_size = bsize.sum()
    combined = float(np.sum(loss * bsize) / d_size)
    std_combined = float(np.sqrt(np.sum(bsize * std ** 2 + bsize * (loss ** 2 - combined ** 2)) / d_size))
    return {"loss": combined, "loss_std": std_combined}


# Model.train_data's options as its callers pass them (ValueSim.py:180); train_rows implements these values only
_TRAIN_ROWS_FIXED = dict(validation_fraction=0.1, sample_replacement=True, oversampling=False, weighted=True, early_stopping=True,
                         early_stopping_patience=10, early_stopping_threshold=1., shuffle=False)


def rows_validation_size(n_rows):
    """train_rows' validation split of n_rows rows; 0 (after the message) means too few rows to train on, and train_rows skips them.  It
    depends on n_rows alone, so a pipelined trainer (online.OnlineTrainer.start) decides the skip before its training starts."""
    validation_size = int(int(n_rows) * _TRAIN_ROWS_FIXED["validation_fraction"])
    if validation_size == 0:
        print("Not enough training data ({} < {}), collecting more data.".format(int(n_rows), int(np.ceil(1 / _TRAIN_ROWS_FIXED["validation_fraction"]))), **perr)
    return validation_size


class Model_VV:
    """Model_VV().load(); .training(flag); .inference(batch); .train(batch); .train_data(data); .save()  (model/model_vv.py:104-231 on
    model/model.py:39-255).  Inference runs through the engine's network kernels, training through the device trainer."""

    def __init__(self, device=0, seed=0, train_kind="fp64", **kwargs):
        from ..engine import BatchedEngine
        from .trainer import KINDS
        if train_kind not in KINDS:
            raise ValueError("train_kind must be one of %s, not %r" % (sorted(KINDS), train_kind))
        self.weights = init_weights(seed)
        self.device, self.train_kind = device, train_kind
        self._eng = BatchedEngine(1, max_nodes=64, eval_kind=kwargs.get("eval_kind", "net"), device=device)
        self._eng.load_weights(self.weights)
        self._trainer = None
        self._dp = None                                            # data-parallel buffers: (stream, own gradient slice, every rank's)
        self._opt_state = None                                     # (exp_avg, exp_avg_sq, step) loaded from a checkpoint before the trainer exists
        self._training = False

    # ------------------------------------------------------------------ trainer plumbing
    def _trainer_obj(self):
        if self._trainer is None:
            from .trainer import Trainer
            self._trainer = Trainer(self.weights, max_batch=4096, device=self.device, kind=self.train_kind)    # Yogi(lr=1e-3, eps=1e-3, weight_decay=1e-3), model_vv.py:132
            if self._opt_state is not None:
                self._trainer.set_state(*self._opt_state)
        return self._trainer

    def _publish(self):
        """weights of the trainer -> the inference kernels (the reference shares one torch module between both)"""
        self.weights = self._trainer.weights()
        self._eng.load_weights(self.weights)

    def load(self, filename=EXP_PATH + "model_checkpoint"):       # model/model.py:163-174
        if os.path.isfile(filename):
            import torch
            print("Loading model...", flush=True)
            ck = torch.load(filename, map_location="cpu", weights_only=False)
            self.weights = state_dict_to_weights(ck["model_state_dict"])
            self._eng.load_weights(self.weights)
            self._opt_state = optimizer_state_from_dict(ck.get("optimizer_state_dict"))
            if self._trainer is not None:
                self._trainer.set_weights(self.weights)
                self._trainer.set_state(*(self._opt_state or (None, None, -1)))
        else:
            print("Checkpoint not found, using default model", flush=True)

    def save(self, filename=EXP_PATH + "model_checkpoint", verbose=True):   # model/model.py:143-160
        import torch
        if verbose:
            print("Saving model...", flush=True)
        d = os.path.dirname(filename) or "."
        if not os.path.isdir(d):
            if verbose:
                print("Export path does not exist, creating a new one...", flush=True)
            os.mkdir(d)
        if self._trainer is not None:
            self.weights = self._trainer.weights()
            m, v, step = self._trainer.state()
        else:
            m, v, step = self._opt_state or (None, None, -1)
        torch.save({"model_state_dict": weights_to_state_dict(self.weights), "optimizer_state_dict": optimizer_state_to_dict(m, v, step)}, filename)

    def reset_optimizer(self):                                    # model/model.py:134-135
        self._opt_state = None
        if self._trainer is not None:
            self._trainer.set_state(None, None, -1)

    def training(self, mode=True):                                # model/model.py:121-126 (the network has no train/eval-dependent layers)
        self._training = bool(mode)

    # ------------------------------------------------------------------ inference (model_vv.py:210-217)
    def inference(self, batch):
        b = np.asarray(batch)
        v, var = self._eng.valuenet(b.reshape(-1, 20, 10))
        return [v.reshape(-1, 1), var.reshape(-1, 1)]

    # ------------------------------------------------------------------ training (model/model.py:52-119,176-249; model_vv.py:136-153,227-231)
    def compute_loss(self, batch, weighted, chunksize=1024):      # model/model.py:52-83
        t = self._trainer_obj()
        loss, std, bsize = [], [], []
        for c in range(0, len(batch[0]), chunksize):
            b = [d[c:c + chunksize] for d in batch]
            mean, sd = t.loss(b, weighted=weighted)
            loss.append(mean); std.append(sd)
            bsize.append(float(np.sum(b[-1])) if weighted else float(len(b[0])))
        return _combine_chunks(loss, std, bsize)

    def train(self, batch, grad_clip=0., g_norm_warn=1e3, weighted=False):   # model/model.py:95-119
        r = self._trainer_obj().step(batch, weighted=weighted, grad_clip=grad_clip)
        if r["grad_norm"] > g_norm_warn:
            print("Large gradient ({}) detected".format(r["grad_norm"]), **perr)
        return r

    def train_data(self, data, batch_size=128, iters_per_val=500, validation_fraction=0.1, sample_replacement=True, oversampling=False,
                   weighted=True, early_stopping=True, early_stopping_patience=10, early_stopping_threshold=1., shuffle=False,
                   max_iters=100000, checkpoint=EXP_PATH + "model_checkpoint"):
        """Model_VV.train_data (model_vv.py:227-231) + Model.train_data (model/model.py:176-249): out_ubound from the data, validation split,
        weights / mean, random batches, validation every iters_per_val iterations, early stopping with the best model saved and re-loaded.
        Log lines as the reference prints them (stderr; parsed by web/parseLog.py:61-66)."""
        data = [np.asarray(d) for d in data]
        t = self._trainer_obj()
        t.set_out_ubound(float(data[1].max()), float(data[2].max()))                         # model_vv.py:228-229
        data_size = len(data[0])
        validation_size = int(data_size * validation_fraction)
        data[-1] = (data[-1] / data[-1].mean()).astype(np.float32)                           # model/model.py:186-187
        if shuffle:
            idx = np.random.permutation(data_size)
            data = [d[idx] for d in data]
        batch_training = [d[:-validation_size] for d in data]
        batch_validation = [d[-validation_size:] for d in data]
        p = np.squeeze(batch_training[-1] / batch_training[-1].sum()) if oversampling else None
        print("Training data size: {}    Validation data size: {}".format(data_size - validation_size, validation_size), **perr)
        fails, loss_val_min = 0, float("inf")
        loss_avg = g_norm_avg = 0
        self.training(True)
        for iters in range(max_iters):
            b_idx = np.random.choice(data_size - validation_size, size=batch_size, replace=sample_replacement, p=p)
            loss = self.train([b[b_idx] for b in batch_training], weighted=weighted)
            loss_avg += loss["loss"]
            g_norm_avg += loss["grad_norm"]
            if (iters + 1) % iters_per_val == 0:
                loss_val = self.compute_loss(batch_validation, weighted=weighted)
                loss_val_mean, loss_val_std = loss_val["loss"], loss_val["loss_std"] / validation_size ** 0.5
                suffix = ""
                stop = False
                if early_stopping:
                    if loss_val_mean - loss_val_min < loss_val_std * early_stopping_threshold:
                        fails = 0
                        if loss_val_mean < loss_val_min:
                            suffix = "*"
                            self.save(checkpoint, verbose=False)
                            loss_val_min = loss_val_mean
                    else:
                        fails += 1
                        stop = fails >= early_stopping_patience
                if stop:
                    break
                print("Iteration:{:7d}  training loss:{:6.4f}  validation loss:{:6.4f}±{:6.4f}  gradient norm:{:6.3f}    {}"
                      .format(iters + 1, loss_avg / iters_per_val, loss_val_mean, loss_val_std, g_norm_avg / iters_per_val, suffix), **perr)
                loss_avg = g_norm_avg = 0
        if early_stopping:
            self.load(checkpoint)                                                            # model/model.py:240-241: back to the best model
        else:
            self.save(checkpoint)
        self._publish()
        self.training(False)

    def train_rows(self, rows_dev_ptr, n_rows, batch_size=128, iters_per_val=500, max_iters=100000, checkpoint=EXP_PATH + "model_checkpoint",
                   seed=0, chunksize=1024, **options):
        """train_data on 212-byte replay rows that stay on the device (the engine's memory, b200_replay_peek_dev): out_ubound and the weight
        mean come from b200_rows_stats_dev, batches are drawn on the device (Trainer.train_rows_dev, seeded by `seed`; the reference's draw is
        np.random.choice), a validation interval runs with one synchronisation, and the validation loss is computed chunk by chunk on the device
        and combined as compute_loss combines it.  Same split (the last 10 % of the rows, no shuffle), early stopping, checkpoint and log lines
        as train_data.  Returns False without training when the split leaves no validation rows (the reference fails on d[:-0]).

        Under a torch.distributed process group of world > 1 (play_batched under torchrun) every rank holds the same rows and trains data-
        parallel: each step, rank r computes the gradient of rows shard_range(batch_size, r, world) of the batch, the fp64 gradients are all-
        gathered and every rank adds them in rank order and applies the same update (Trainer.apply_grads_dev), so all ranks keep bit-identical
        weights.  Everything else (row statistics, validation, early stopping) runs redundantly on every rank; rank 0 alone prints and writes
        the checkpoint, the other ranks keep the best weights and optimiser state in memory."""
        bad = {k: v for k, v in options.items() if k not in _TRAIN_ROWS_FIXED or v != _TRAIN_ROWS_FIXED[k]}
        if bad:
            raise ValueError("train_rows implements train_data with %s only; got %s" % (_TRAIN_ROWS_FIXED, bad))
        n_rows = int(n_rows)
        validation_size = rows_validation_size(n_rows)
        if validation_size == 0:
            return False
        from .. import distributed as D
        rank, world = D.rank_world()
        if world > 1:
            lo, hi = D.batch_slice(int(batch_size), rank, world)
        def say(msg, **where):                                    # rank 0 alone prints
            if rank == 0:
                print(msg, **(where or perr))
        best = None
        t = self._trainer_obj()
        max_value, max_variance, visit_sum = t.rows_stats(rows_dev_ptr, n_rows)
        t.set_out_ubound(max_value, max_variance)                                             # model_vv.py:228-229
        scale = float(n_rows / visit_sum)                                                     # weights / weights.mean(), model/model.py:186-187
        n_train = n_rows - validation_size
        say("Training data size: {}    Validation data size: {}".format(n_train, validation_size))
        patience, threshold = _TRAIN_ROWS_FIXED["early_stopping_patience"], _TRAIN_ROWS_FIXED["early_stopping_threshold"]
        fails, loss_val_min = 0, float("inf")
        self.training(True)
        for it0 in range(0, int(max_iters), int(iters_per_val)):
            k = min(int(iters_per_val), int(max_iters) - it0)
            if world > 1:
                log = self._train_interval_dp(rows_dev_ptr, n_train, batch_size, lo, hi, k, seed, it0, scale)
            else:
                log = t.train_rows_dev(rows_dev_ptr, n_train, batch_size, k, seed, it0, scale, weighted=True)
            loss_avg = g_norm_avg = 0
            for loss, _std, g_norm in log:
                if g_norm > 1e3:
                    say("Large gradient ({}) detected".format(g_norm))             # Model.train's g_norm_warn (model/model.py:103-105)
                loss_avg += loss
                g_norm_avg += g_norm
            if k < iters_per_val:
                break                                                                         # no validation after a partial interval
            loss_val = self._loss_rows(rows_dev_ptr, n_train, n_rows, scale, chunksize)
            loss_val_mean, loss_val_std = loss_val["loss"], loss_val["loss_std"] / validation_size ** 0.5
            suffix = ""
            if loss_val_mean - loss_val_min < loss_val_std * threshold:
                fails = 0
                if loss_val_mean < loss_val_min:
                    suffix = "*"
                    if rank == 0:
                        self.save(checkpoint, verbose=False)
                    if world > 1:
                        best = (t.weights(), t.state())
                    loss_val_min = loss_val_mean
            else:
                fails += 1
                if fails >= patience:
                    break
            say("Iteration:{:7d}  training loss:{:6.4f}  validation loss:{:6.4f}±{:6.4f}  gradient norm:{:6.3f}    {}"
                .format(it0 + k, loss_avg / iters_per_val, loss_val_mean, loss_val_std, g_norm_avg / iters_per_val, suffix))
        if world > 1:                                                                         # back to the best model, from memory on every rank
            say("Loading model...", file=sys.stdout, flush=True)
            if best is not None:
                t.set_weights(best[0])
                t.set_state(*best[1])
        else:
            self.load(checkpoint)                                                             # model/model.py:240-241: back to the best model
        self._publish()
        self.training(False)
        return True

    def _train_interval_dp(self, rows_dev_ptr, n_train, batch, lo, hi, iters, seed, first_iter, weight_scale):
        """`iters` data-parallel steps (rows [lo, hi) of each batch on this rank) -> the [iters, 3] log train_rows_dev returns"""
        import torch
        from .. import distributed as D
        from .trainer import GRAD_VEC
        t = self._trainer_obj()
        if self._dp is None:
            dev = torch.device("cuda", int(self.device))
            stream = torch.cuda.Stream(device=dev)
            t.set_stream(stream.cuda_stream)                     # the exchange is ordered on the trainer's own stream
            self._dp = (stream, torch.empty(GRAD_VEC, dtype=torch.float64, device=dev),
                        torch.empty((D.rank_world()[1], GRAD_VEC), dtype=torch.float64, device=dev))
        stream, local, parts = self._dp
        for it in range(int(iters)):
            t.grad_rows_dev(rows_dev_ptr, n_train, batch, lo, hi, seed, first_iter + it, weight_scale, local.data_ptr())
            D.allgather_grads(local, parts, stream)
            t.apply_grads_dev(parts.data_ptr(), parts.shape[0], 0.0, it)
        return t.read_log(iters)

    def _loss_rows(self, rows_dev_ptr, first, end, weight_scale, chunksize=1024):
        """compute_loss(weighted=True) on device rows [first, end)"""
        t = self._trainer_obj()
        loss, std, bsize = [], [], []
        for c in range(first, end, chunksize):
            mean, sd, wsum = t.loss_rows_dev(rows_dev_ptr, c, min(chunksize, end - c), weight_scale, weighted=True)
            loss.append(mean); std.append(sd); bsize.append(wsum)
        return _combine_chunks(loss, std, bsize)

    def close(self):
        if self._trainer is not None:
            self._trainer.close()
        self._eng.close()
