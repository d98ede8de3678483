"""Training of the consensus GRU on the H100: the counterpart of medaka/training.py and the training half of
medaka/torch_ext.py (run_epoch, ClipGrad, the learning-rate schedules).

``GRUTrainer`` drives an ``mdk_trainer`` (csrc/gru_train.cu): forward with saved activations, cross-entropy, BPTT,
gradient reductions, norm / clip / skip and the optimizer step all run in the library's CUDA kernels in fp32; the weights,
their gradient and the optimizer state stay on the device.  Mixed precision (``amp=True``) and the read-level
LatentSpaceLSTM are not implemented here.  The learning-rate schedule is a plain function of the step, computed on the host.

``RLTrainer`` does the same for the read-level LatentSpaceLSTM through an ``mdk_rl_trainer`` (csrc/rl_train.cu), with
batch-statistics BatchNorm as in ``model.train()``.
"""
import csv
import functools
import logging
import math
import os
import tomllib

import numpy as np

from medaka_b200 import libmedaka as _lm

# the reference's optimizer defaults (medaka/training.py run_training)
DEFAULT_OPTIM_ARGS = {
    "nadam": {"lr": 0.002, "betas": (0.9, 0.99), "eps": 1e-07},
    "adam": {"lr": 0.0001, "betas": (0.9, 0.99), "eps": 1e-07},
    "rmsprop": {"lr": 0.001, "alpha": 0.9, "eps": 1e-07, "momentum": 0.0},
    "sgd": {"lr": 0.001},
}
# the arguments each rule implements, with torch.optim's defaults; any other argument is a ValueError
_OPTIM_KEYS = {
    "rmsprop": {"lr": 0.01, "alpha": 0.99, "eps": 1e-08, "weight_decay": 0.0, "momentum": 0.0, "centered": False},
    "adam": {"lr": 0.001, "betas": (0.9, 0.999), "eps": 1e-08, "weight_decay": 0.0, "amsgrad": False},
    "nadam": {"lr": 0.002, "betas": (0.9, 0.999), "eps": 1e-08, "weight_decay": 0.0, "momentum_decay": 0.004},
    "sgd": {"lr": 0.001, "momentum": 0.0, "dampening": 0.0, "weight_decay": 0.0, "nesterov": False},
}
# arguments accepted only at the value that means "off"
_OFF_ONLY = {"centered": False, "amsgrad": False}
_KINDS = {"rmsprop": 0, "adam": 1, "nadam": 2, "sgd": 3}

DEFAULT_MODEL_DICT = {"type": "GRUModel", "kwargs": {"num_features": 10, "num_classes": 5, "gru_size": 256}}


def optimizer_args(optimizer, optim_args=None):
    """The full argument set of ``optimizer`` (torch.optim defaults completed by ``optim_args``, or the reference's
    defaults when None); ValueError for an unknown optimizer or an argument the kernels do not implement."""
    if optimizer not in _OPTIM_KEYS:
        raise ValueError("Unknown optimizer: {}".format(optimizer))
    given = dict(DEFAULT_OPTIM_ARGS[optimizer] if optim_args is None else optim_args)
    args = dict(_OPTIM_KEYS[optimizer])
    for k, v in given.items():
        if k not in args or (k in _OFF_ONLY and v != _OFF_ONLY[k]):
            raise ValueError("optimizer argument {}={!r} is not implemented for {}".format(k, v, optimizer))
        args[k] = v
    return args


def _optim_desc(optimizer, args):
    od = _lm.ffi.new("mdk_optim_desc *")
    od.kind = _KINDS[optimizer]
    od.alpha = args.get("alpha", 0.0)
    b1, b2 = args.get("betas", (0.0, 0.0))
    od.beta1, od.beta2 = b1, b2
    od.eps = args.get("eps", 0.0)
    od.weight_decay = args.get("weight_decay", 0.0)
    od.momentum = args.get("momentum", 0.0)
    od.dampening = args.get("dampening", 0.0)
    od.momentum_decay = args.get("momentum_decay", 0.0)
    od.nesterov = 1 if args.get("nesterov", False) else 0
    return od


# ---------------------------------------------------------------------------------------------- schedules and clipping
def linear_schedule(y0, y1):
    return lambda t: y0 + (y1 - y0) * t


def cosine_decay_schedule(y0, y1):
    return lambda t: y1 + 0.5 * (y0 - y1) * (np.cos(t * np.pi) + 1.0)


def piecewise_schedule(knots, funcs):
    def f(t):
        i = np.searchsorted(knots, t)
        t0 = 0.0 if i == 0 else knots[i - 1]
        t1 = 1.0 if i == len(knots) else knots[i]
        return funcs[i]((t - t0) / (t1 - t0))
    return f


class FuncScheduler(object):
    """The learning rate of torch's LambdaLR over ``func`` (torch_ext.func_scheduler) as a host-side counter:
    ``get_last_lr()`` and ``step()`` as the reference's run_epoch uses them."""

    def __init__(self, base_lr, func, total_steps, warmup_steps=None, warmup_ratio=0.1, start_step=0):
        if warmup_steps:
            y0 = func(0.0)
            func = piecewise_schedule([warmup_steps / total_steps], [linear_schedule(warmup_ratio * y0, y0), func])
        self.base_lr = base_lr
        self.factor = lambda step: func((step + start_step) / total_steps)
        self.last_epoch = 0

    def lr_at(self, step):
        return self.base_lr * self.factor(step)

    def get_last_lr(self):
        return [self.lr_at(self.last_epoch)]

    def step(self):
        self.last_epoch += 1


def linear_warmup_cosine_decay(end_ratio=0.01, warmup_steps=500, **kwargs):
    """Linear warmup, cosine decay (torch_ext.linear_warmup_cosine_decay): called with (base_lr, steps per epoch,
    epochs, last_epoch) where the reference passes (optimizer, train_loader, epochs, last_epoch)."""
    return lambda base_lr, steps_per_epoch, epochs, last_epoch: FuncScheduler(
        base_lr, cosine_decay_schedule(1.0, end_ratio), epochs * steps_per_epoch, warmup_steps=warmup_steps,
        start_step=last_epoch * steps_per_epoch)


def no_schedule(warmup_steps=None, **kwargs):
    """Constant learning rate after an optional linear warmup (torch_ext.no_schedule)."""
    return lambda base_lr, steps_per_epoch, epochs, last_epoch: FuncScheduler(
        base_lr, lambda x: 1.0, epochs * steps_per_epoch, warmup_steps=warmup_steps,
        start_step=last_epoch * steps_per_epoch)


class ClipGrad(object):
    """Gradient clipping by quantile (torch_ext.ClipGrad): the threshold is ``factor`` times the ``quantile`` of the
    last ``buffer_size`` gradient norms.  ``max_norm()`` is the threshold of the next step, ``append`` records its
    pre-clip norm (NaN norms are not recorded)."""

    def __init__(self, quantile=0.5, factor=2.0, buffer_size=100):
        self.buffer = np.full(buffer_size, fill_value=1e6)
        self.quantile = quantile
        self.factor = factor
        self.i = 0

    def append(self, grad_norm):
        self.buffer[self.i] = grad_norm
        self.i = (self.i + 1) % len(self.buffer)

    def max_norm(self):
        return self.factor * np.quantile(self.buffer, self.quantile)

    def record(self, grad_norm):
        if not math.isnan(grad_norm):
            self.append(grad_norm)
        return grad_norm


class FixedClip(object):
    """clip_grad_norm_ at a fixed threshold: run_training's clipping with quantile_grad_clip=False (the reference's
    clip_grad_fn, max_norm=2.0)."""

    def __init__(self, max_norm=2.0):
        self._max_norm = max_norm

    def max_norm(self):
        return self._max_norm

    def record(self, grad_norm):
        return grad_norm


# ---------------------------------------------------------------------------------------------------------- trainer
def state_dict_keys(n_layers=2):
    keys = []
    for layer in range(n_layers):
        for sfx in ("", "_reverse"):
            keys += ["gru.%s_l%d%s" % (k, layer, sfx) for k in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]
    return keys + ["linear.weight", "linear.bias"]


class GRUTrainer(object):
    """The consensus GRUModel (gru.py) under training on an H100, fp32 (the reference's amp=False)."""

    def __init__(self, num_features=10, num_classes=5, gru_size=256, n_layers=2, bidirectional=True, device=0,
                 optimizer="rmsprop", optim_args=None, amp=False):
        if amp:
            raise NotImplementedError("mixed-precision training (amp=True) is not implemented: training runs in fp32")
        if num_classes != 5 or n_layers != 2 or not bidirectional:
            raise NotImplementedError("only the 2-layer bidirectional GRU with 5 classes is implemented")
        self.num_features, self.gru_size, self.num_classes = num_features, gru_size, num_classes
        self.n_layers, self.bidirectional = n_layers, bidirectional
        self._device = int(device)
        self._tr = None
        lib = _lm.load()
        _lm.require_gpu(self._device)
        desc = _lm.ffi.new("mdk_model_desc *")
        desc.num_features, desc.gru_size, desc.n_layers = num_features, gru_size, 2
        desc.bidirectional, desc.num_classes = 1, 5
        pt = _lm.ffi.new("mdk_trainer **")
        _lm.check(lib.mdk_trainer_create(self._device, desc, pt))
        self._tr = pt[0]
        n = _lm.ffi.new("int64_t *")
        _lm.check(lib.mdk_trainer_num_params(self._tr, n))
        self.n_params = int(n[0])
        self.shapes = self._shapes()
        self.set_optimizer(optimizer, optim_args)

    def _shapes(self):
        H, F = self.gru_size, self.num_features
        out = {}
        for layer in range(2):
            n_in = F if layer == 0 else 2 * H
            for sfx in ("", "_reverse"):
                out["gru.weight_ih_l%d%s" % (layer, sfx)] = (3 * H, n_in)
                out["gru.weight_hh_l%d%s" % (layer, sfx)] = (3 * H, H)
                out["gru.bias_ih_l%d%s" % (layer, sfx)] = (3 * H,)
                out["gru.bias_hh_l%d%s" % (layer, sfx)] = (3 * H,)
        out["linear.weight"] = (5, 2 * H)
        out["linear.bias"] = (5,)
        return {k: out[k] for k in state_dict_keys()}

    def close(self):
        if self._tr is not None and _lm.lib is not None:
            _lm.lib.mdk_trainer_destroy(self._tr)
        self._tr = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_optimizer(self, optimizer="rmsprop", optim_args=None):
        """One of 'rmsprop', 'adam', 'nadam', 'sgd' with torch.optim's arguments (the reference's defaults when
        ``optim_args`` is None); resets the optimizer state."""
        args = optimizer_args(optimizer, optim_args)
        _lm.check(_lm.lib.mdk_trainer_set_optimizer(self._tr, _optim_desc(optimizer, args)))
        self.optimizer, self.optim_args, self.lr = optimizer, args, float(args["lr"])

    def set_bptt_windows(self, nb):
        """Schedule hook for tests and benchmarks: windows per CTA of the BPTT kernel (1, 2, 4 or 8), or 0 to choose
        from the batch size.  The gradients do not depend on it."""
        _lm.check(_lm.lib.mdk_trainer_set_bptt_windows(self._tr, int(nb)))

    def bptt_windows(self, B):
        """Windows per CTA the BPTT kernel runs at for a batch of B windows, under the current setting."""
        nb = _lm.ffi.new("int *")
        _lm.check(_lm.lib.mdk_trainer_bptt_windows(self._tr, int(B), nb))
        return int(nb[0])

    def load_state_dict(self, state_dict):
        """torch state-dict layout (GRUModel.state_dict()); resets the optimizer state."""
        missing = [k for k in self.shapes if k not in state_dict]
        unexpected = [k for k in state_dict if k not in self.shapes]
        if missing or unexpected:
            raise RuntimeError("Error(s) in loading state_dict: missing {}, unexpected {}".format(missing, unexpected))
        sd = {}
        for k, shape in self.shapes.items():
            v = state_dict[k]
            if hasattr(v, "detach"):
                v = v.detach().cpu().numpy()
            a = np.ascontiguousarray(v, dtype=np.float32)
            if a.shape != shape:
                raise RuntimeError("size mismatch for {}: expected {}, got {}".format(k, shape, a.shape))
            sd[k] = a
        ptr = lambda a: _lm.ffi.cast("const float *", _lm.ffi.from_buffer(a))   # noqa: E731
        for layer in range(2):
            for d, sfx in enumerate(("", "_reverse")):
                _lm.check(_lm.lib.mdk_trainer_load_gru(
                    self._tr, layer, d, *(ptr(sd["gru.%s_l%d%s" % (k, layer, sfx)])
                                          for k in ("weight_ih", "weight_hh", "bias_ih", "bias_hh"))))
        _lm.check(_lm.lib.mdk_trainer_load_linear(self._tr, ptr(sd["linear.weight"]), ptr(sd["linear.bias"])))
        return self

    def _unflatten(self, flat):
        out, o = {}, 0
        for k, shape in self.shapes.items():
            n = int(np.prod(shape))
            out[k] = flat[o:o + n].reshape(shape)
            o += n
        return out

    def flat_params(self):
        out = np.empty(self.n_params, np.float32)
        _lm.check(_lm.lib.mdk_trainer_read_params(self._tr, _lm.ffi.cast("float *", _lm.ffi.from_buffer(out)),
                                                  self.n_params))
        return out

    def state_dict(self):
        """The current weights as numpy float32 arrays, torch state-dict keys and order."""
        return self._unflatten(self.flat_params())

    def grads(self):
        """The gradients of the last train_step, before clipping, as a state dict."""
        out = np.empty(self.n_params, np.float32)
        _lm.check(_lm.lib.mdk_trainer_read_grads(self._tr, _lm.ffi.cast("float *", _lm.ffi.from_buffer(out)),
                                                 self.n_params))
        return self._unflatten(out)

    @staticmethod
    def _batch_arrays(batch):
        feats = batch.counts_matrix if hasattr(batch, "counts_matrix") else batch[0]
        labels = batch.labels if hasattr(batch, "labels") else batch[1]
        if hasattr(feats, "detach"):
            feats = feats.detach().cpu().numpy()
        if hasattr(labels, "detach"):
            labels = labels.detach().cpu().numpy()
        feats = np.ascontiguousarray(feats, dtype=np.float32)
        labels = np.asarray(labels)
        if labels.ndim == 3 and labels.shape[-1] == 1:      # encoded_labels_to_training_vectors' sparse one-hot
            labels = labels[..., 0]
        if feats.ndim != 3 or labels.shape != feats.shape[:2]:
            raise ValueError("features must be [B, T, F] and labels [B, T]")
        return feats, np.ascontiguousarray(labels, dtype=np.int32)

    @staticmethod
    def _metrics(stats, batch):
        metrics = {"n_model_correct": int(stats.n_correct)}
        mvp = getattr(batch, "majority_vote_probs", None)
        if mvp is not None:
            labels = GRUTrainer._batch_arrays(batch)[1]
            mvp = mvp.detach().cpu().numpy() if hasattr(mvp, "detach") else np.asarray(mvp)
            metrics["n_argmax_correct"] = int((mvp.argmax(-1) == labels).sum())
        metrics["n_positions"] = int(stats.n_positions)
        return metrics

    def _checked(self, feats, labels=None):
        """The kernels read B x T x num_features floats: features of another width are refused, not misread."""
        if feats.ndim != 3 or feats.shape[2] != self.num_features:
            raise ValueError("expected features of shape [B, T, {}], got {}".format(self.num_features, feats.shape))
        return feats, labels

    def train_step(self, batch, lr=None, max_norm=None):
        """One step (forward, loss, backward, clip, update) at learning rate ``lr`` (the optimizer's when None),
        clipping at ``max_norm`` (none when None).  Returns (loss, metrics, grad_norm, skipped); a non-finite gradient
        skips the update."""
        feats, labels = self._checked(*self._batch_arrays(batch))
        B, T = labels.shape
        st = _lm.ffi.new("mdk_train_stats *")
        _lm.check(_lm.lib.mdk_trainer_step(
            self._tr, _lm.ffi.cast("const float *", _lm.ffi.from_buffer(feats)),
            _lm.ffi.cast("const int32_t *", _lm.ffi.from_buffer(labels)), B, T,
            float(self.lr if lr is None else lr), float(max_norm) if max_norm is not None else 0.0, st))
        return float(st.loss), self._metrics(st, batch), float(st.grad_norm), bool(st.skipped)

    def process_batch(self, batch, want_probs=False):
        """Loss and metrics of a batch without a backward pass (the reference's process_batch under no_grad):
        (loss, {'n_model_correct', ['n_argmax_correct',] 'n_positions'}), plus the probabilities with want_probs."""
        feats, labels = self._checked(*self._batch_arrays(batch))
        B, T = labels.shape
        st = _lm.ffi.new("mdk_train_stats *")
        probs = np.empty((B, T, 5), np.float32) if want_probs else None
        pp = _lm.ffi.cast("float *", _lm.ffi.from_buffer(probs)) if want_probs else _lm.ffi.NULL
        _lm.check(_lm.lib.mdk_trainer_eval(
            self._tr, _lm.ffi.cast("const float *", _lm.ffi.from_buffer(feats)),
            _lm.ffi.cast("const int32_t *", _lm.ffi.from_buffer(labels)), B, T, pp, _lm.ffi.NULL, st))
        out = (float(st.loss), self._metrics(st, batch))
        return out + (probs,) if want_probs else out

    def forward_arrays(self, feats):
        """(probs, logits) float32 [B, T, 5] of the training forward, without labels."""
        feats, _ = self._checked(np.ascontiguousarray(feats, dtype=np.float32))
        B, T = feats.shape[:2]
        probs, logits = np.empty((B, T, 5), np.float32), np.empty((B, T, 5), np.float32)
        _lm.check(_lm.lib.mdk_trainer_eval(
            self._tr, _lm.ffi.cast("const float *", _lm.ffi.from_buffer(feats)), _lm.ffi.NULL, B, T,
            _lm.ffi.cast("float *", _lm.ffi.from_buffer(probs)), _lm.ffi.cast("float *", _lm.ffi.from_buffer(logits)),
            _lm.ffi.NULL))
        return probs, logits

    def stage_ms(self):
        """Device times of the last train_step: forward, head (loss + head backward), BPTT, reductions, optimizer."""
        ms = _lm.ffi.new("float[5]")
        _lm.check(_lm.lib.mdk_trainer_stage_ms(self._tr, ms))
        return dict(zip(("forward", "head", "bptt", "reductions", "optimizer"), [float(x) for x in ms]))


def workspace_bytes(num_features, gru_size, B, T):
    """(device bytes a train_step of B x T needs, the budget beyond which it is refused)."""
    lib = _lm.load()
    desc = _lm.ffi.new("mdk_model_desc *")
    desc.num_features, desc.gru_size, desc.n_layers, desc.bidirectional, desc.num_classes = num_features, gru_size, 2, 1, 5
    b, budget = _lm.ffi.new("size_t *"), _lm.ffi.new("size_t *")
    _lm.check(lib.mdk_trainer_workspace_bytes(desc, B, T, b, budget))
    return int(b[0]), int(budget[0])


RL_BUFFERS = ("read_level_conv.convs.2.running_mean", "read_level_conv.convs.2.running_var",
              "read_level_conv.convs.5.running_mean", "read_level_conv.convs.5.running_var")
RL_NBT = ("read_level_conv.convs.2.num_batches_tracked", "read_level_conv.convs.5.num_batches_tracked")


def rl_param_shapes(lstm_size=128, cnn_size=128, use_dwells=False):
    """named_parameters() of the reference's LatentSpaceLSTM (bidirectional, kernel sizes 1 and 17): name -> shape."""
    H, C, nin = lstm_size, cnn_size, 6 + 1 + (1 if use_dwells else 0)
    out = {"base_embedder.weight": (6, 6), "strand_embedder.weight": (3, 6),
           "read_level_conv.convs.0.weight": (C, nin, 1), "read_level_conv.convs.0.bias": (C,),
           "read_level_conv.convs.2.weight": (C,), "read_level_conv.convs.2.bias": (C,),
           "read_level_conv.convs.3.weight": (C, C, 17), "read_level_conv.convs.3.bias": (C,),
           "read_level_conv.convs.5.weight": (C,), "read_level_conv.convs.5.bias": (C,),
           "read_level_conv.expansion_layer.weight": (H, C), "read_level_conv.expansion_layer.bias": (H,),
           "pre_pool_expansion_layer.weight": (H, C), "pre_pool_expansion_layer.bias": (H,)}
    for layer in range(2):
        for sfx in ("", "_reverse"):
            n_in = H if layer == 0 else 2 * H
            out["lstm.weight_ih_l%d%s" % (layer, sfx)] = (4 * H, n_in)
            out["lstm.weight_hh_l%d%s" % (layer, sfx)] = (4 * H, H)
            out["lstm.bias_ih_l%d%s" % (layer, sfx)] = (4 * H,)
            out["lstm.bias_hh_l%d%s" % (layer, sfx)] = (4 * H,)
    out["linear.weight"] = (5, 2 * H)
    out["linear.bias"] = (5,)
    return out


def rl_state_dict_keys(lstm_size=128, use_dwells=False):
    """state_dict() keys of the reference's LatentSpaceLSTM: parameters with each BatchNorm's buffers after its own."""
    keys = []
    for k in rl_param_shapes(lstm_size, use_dwells=use_dwells):
        keys.append(k)
        if k.endswith(("convs.2.bias", "convs.5.bias")):
            base = k[:-len("bias")]
            keys += [base + "running_mean", base + "running_var", base + "num_batches_tracked"]
    return keys


def _rl_features(x):
    """int8 [B, P, D, F] features: collated batches are uint8 (torch_ext.Batch.collate), whose strand -1 reads back as
    255; the unsafe cast restores it, as the read-level engine's wrapper does."""
    if hasattr(x, "detach"):
        x = x.detach().cpu().numpy()
    x = np.asarray(x)
    out = np.empty(x.shape, np.int8)
    np.copyto(out, x, casting="unsafe")
    if out.ndim != 4:
        raise ValueError("read-level features must be [B, P, D, F]")
    return out


class RLTrainer(object):
    """The read-level LatentSpaceLSTM (latent_space_lstm.py) under training on an H100, fp32 (the reference's
    amp=False): lstm_size 128 or 384, cnn_size 128, with or without dwells."""

    STAGES = ("stats", "forward", "lstm", "head", "bptt", "read_backward", "reductions", "optimizer")

    def __init__(self, lstm_size=128, cnn_size=128, use_dwells=False, num_classes=5, kernel_sizes=(1, 17),
                 pooler_type="mean", bidirectional=True, device=0, optimizer="rmsprop", optim_args=None, amp=False,
                 **unused):
        if amp:
            raise NotImplementedError("mixed-precision training (amp=True) is not implemented: training runs in fp32")
        if (num_classes != 5 or list(kernel_sizes) != [1, 17] or pooler_type != "mean" or not bidirectional
                or cnn_size != 128 or lstm_size not in (128, 384)):
            raise NotImplementedError("only the bidirectional, mean-pooled LatentSpaceLSTM with kernel sizes [1, 17], "
                                      "cnn_size 128, lstm_size 128 or 384 and 5 classes is implemented")
        self.lstm_size, self.cnn_size, self.use_dwells = lstm_size, cnn_size, bool(use_dwells)
        self.shapes = rl_param_shapes(lstm_size, cnn_size, use_dwells)
        self._device = int(device)
        self._tr = None
        lib = _lm.load()
        _lm.require_gpu(self._device)
        pt = _lm.ffi.new("mdk_rl_trainer **")
        _lm.check(lib.mdk_rl_trainer_create(self._device, lstm_size, cnn_size, 1 if use_dwells else 0, 5, pt))
        self._tr = pt[0]
        n = _lm.ffi.new("int64_t *")
        _lm.check(lib.mdk_rl_trainer_num_params(self._tr, n))
        self.n_params = int(n[0])
        self.set_optimizer(optimizer, optim_args)

    def close(self):
        if self._tr is not None and _lm.lib is not None:
            _lm.lib.mdk_rl_trainer_destroy(self._tr)
        self._tr = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_optimizer(self, optimizer="rmsprop", optim_args=None):
        """As GRUTrainer.set_optimizer."""
        args = optimizer_args(optimizer, optim_args)
        _lm.check(_lm.lib.mdk_rl_trainer_set_optimizer(self._tr, _optim_desc(optimizer, args)))
        self.optimizer, self.optim_args, self.lr = optimizer, args, float(args["lr"])

    def set_bptt_windows(self, nb):
        """Schedule hook for tests and benchmarks: windows per CTA of the LSTM BPTT kernel (1, 2, 4 or 8), or 0 to
        choose from the batch size.  The gradients do not depend on it."""
        _lm.check(_lm.lib.mdk_rl_trainer_set_bptt_windows(self._tr, int(nb)))

    def bptt_windows(self, B):
        """Windows per CTA the BPTT kernel runs at for a batch of B windows, under the current setting."""
        nb = _lm.ffi.new("int *")
        _lm.check(_lm.lib.mdk_rl_trainer_bptt_windows(self._tr, int(B), nb))
        return int(nb[0])

    def set_slice_rows(self, rows):
        """Schedule hook for tests and benchmarks: cap the (window, read) rows of one slice of the forward and read
        backward passes at ``rows``, or 0 for the automatic length (what the per-read scratch holds).  Only the fp32
        order of the sums across slices depends on it."""
        _lm.check(_lm.lib.mdk_rl_trainer_set_slice_rows(self._tr, int(rows)))

    def load_state_dict(self, state_dict):
        """The reference's state dict (parameters, BatchNorm buffers, the unused expansion_layer); resets the
        optimizer state."""
        keys = rl_state_dict_keys(self.lstm_size, self.use_dwells)
        missing = [k for k in keys if k not in state_dict]
        unexpected = [k for k in state_dict if k not in keys]
        if missing or unexpected:
            raise RuntimeError("Error(s) in loading state_dict: missing {}, unexpected {}".format(missing, unexpected))
        for k in keys:
            v = state_dict[k]
            if hasattr(v, "detach"):
                v = v.detach().cpu().numpy()
            a = np.ascontiguousarray(np.asarray(v, dtype=np.float32).reshape(-1))
            shape = self.shapes.get(k, (1,) if k in RL_NBT else (self.cnn_size,))
            if a.size != int(np.prod(shape)):
                raise RuntimeError("size mismatch for {}: expected {}, got {}".format(k, shape, np.shape(v)))
            _lm.check(_lm.lib.mdk_rl_trainer_load(self._tr, k.encode(), _lm.ffi.cast("const float *", _lm.ffi.from_buffer(a)),
                                                  a.size))
        return self

    def _unflatten(self, flat):
        out, o = {}, 0
        for k, shape in self.shapes.items():
            n = int(np.prod(shape))
            out[k] = flat[o:o + n].reshape(shape)
            o += n
        return out

    def flat_params(self):
        out = np.empty(self.n_params, np.float32)
        _lm.check(_lm.lib.mdk_rl_trainer_read_params(self._tr, _lm.ffi.cast("float *", _lm.ffi.from_buffer(out)),
                                                     self.n_params))
        return out

    def buffers(self):
        """The BatchNorm buffers: running statistics (float32) and num_batches_tracked (int64 scalars)."""
        out = np.empty(4 * self.cnn_size, np.float32)
        nbt = _lm.ffi.new("int64_t[2]")
        _lm.check(_lm.lib.mdk_rl_trainer_read_buffers(self._tr, _lm.ffi.cast("float *", _lm.ffi.from_buffer(out)),
                                                      out.size, nbt))
        res = {k: out[i * self.cnn_size:(i + 1) * self.cnn_size] for i, k in enumerate(RL_BUFFERS)}
        res.update({k: np.array(int(nbt[i]), np.int64) for i, k in enumerate(RL_NBT)})
        return res

    def state_dict(self):
        """Weights and buffers as numpy arrays in the reference's state-dict keys and order."""
        sd = self._unflatten(self.flat_params())
        sd.update(self.buffers())
        return {k: sd[k] for k in rl_state_dict_keys(self.lstm_size, self.use_dwells)}

    def grads(self):
        """The gradients of the last train_step, before clipping; expansion_layer, which gets none, is left out."""
        out = np.empty(self.n_params, np.float32)
        _lm.check(_lm.lib.mdk_rl_trainer_read_grads(self._tr, _lm.ffi.cast("float *", _lm.ffi.from_buffer(out)),
                                                    self.n_params))
        return {k: v for k, v in self._unflatten(out).items() if not k.startswith("read_level_conv.expansion_layer")}

    @staticmethod
    def _batch_arrays(batch):
        x = batch.read_level_features if hasattr(batch, "read_level_features") else batch[0]
        labels = batch.labels if hasattr(batch, "labels") else batch[1]
        x = _rl_features(x)
        if hasattr(labels, "detach"):
            labels = labels.detach().cpu().numpy()
        labels = np.asarray(labels)
        if labels.ndim == 3 and labels.shape[-1] == 1:
            labels = labels[..., 0]
        if labels.shape != x.shape[:2]:
            raise ValueError("features must be [B, P, D, F] and labels [B, P]")
        return x, np.ascontiguousarray(labels, dtype=np.int32)

    def _call(self, fn, x, *args):
        B, P, D, F = x.shape
        return fn(self._tr, _lm.ffi.cast("const int8_t *", _lm.ffi.from_buffer(x)), *args[:1], B, P, D, F, *args[1:])

    def train_step(self, batch, lr=None, max_norm=None):
        """As GRUTrainer.train_step, on read-level batches (read_level_features int8 / uint8 [B, P, D, F])."""
        x, labels = self._batch_arrays(batch)
        st = _lm.ffi.new("mdk_train_stats *")
        _lm.check(self._call(_lm.lib.mdk_rl_trainer_step, x, _lm.ffi.cast("const int32_t *", _lm.ffi.from_buffer(labels)),
                             float(self.lr if lr is None else lr), float(max_norm) if max_norm is not None else 0.0, st))
        return float(st.loss), GRUTrainer._metrics(st, batch), float(st.grad_norm), bool(st.skipped)

    def process_batch(self, batch, want_probs=False):
        """The reference's validation (model.eval(): running statistics) without a backward pass."""
        x, labels = self._batch_arrays(batch)
        B, P = labels.shape
        st = _lm.ffi.new("mdk_train_stats *")
        probs = np.empty((B, P, 5), np.float32) if want_probs else None
        pp = _lm.ffi.cast("float *", _lm.ffi.from_buffer(probs)) if want_probs else _lm.ffi.NULL
        _lm.check(self._call(_lm.lib.mdk_rl_trainer_eval, x, _lm.ffi.cast("const int32_t *", _lm.ffi.from_buffer(labels)),
                             pp, _lm.ffi.NULL, st))
        metrics = {"n_model_correct": int(st.n_correct), "n_positions": int(st.n_positions)}
        return (float(st.loss), metrics) + ((probs,) if want_probs else ())

    def forward_arrays(self, x):
        """(probs, logits) float32 [B, P, 5] of the validation forward, without labels."""
        x = _rl_features(x)
        B, P = x.shape[:2]
        probs, logits = np.empty((B, P, 5), np.float32), np.empty((B, P, 5), np.float32)
        _lm.check(self._call(_lm.lib.mdk_rl_trainer_eval, x, _lm.ffi.NULL,
                             _lm.ffi.cast("float *", _lm.ffi.from_buffer(probs)),
                             _lm.ffi.cast("float *", _lm.ffi.from_buffer(logits)), _lm.ffi.NULL))
        return probs, logits

    def stage_ms(self):
        """Device times of the last train_step by stage (STAGES)."""
        ms = _lm.ffi.new("float[8]")
        _lm.check(_lm.lib.mdk_rl_trainer_stage_ms(self._tr, ms))
        return dict(zip(self.STAGES, [float(v) for v in ms]))


def rl_workspace_bytes(lstm_size, B, P, D, F):
    """(device bytes a read-level train_step of B x P x D x F needs, the budget beyond which it is refused)."""
    lib = _lm.load()
    b, budget = _lm.ffi.new("size_t *"), _lm.ffi.new("size_t *")
    _lm.check(lib.mdk_rl_trainer_workspace_bytes(lstm_size, B, P, D, F, b, budget))
    return int(b[0]), int(budget[0])


# ---------------------------------------------------------------------------------------------------------- batching
def encoded_labels_to_training_vectors(enc_labels):
    """HaploidLabelScheme.encoded_labels_to_training_vectors (labels.py): sparse one-hot [n, 1]; legacy labels with two
    fields (base, run length) map base codes past the four lowercase ones onto the classes."""
    enc_labels = np.asarray(enc_labels)
    if enc_labels.dtype.names is not None and len(enc_labels.dtype) == 2:
        enc_labels = np.array([max(0, x[0] - 4) for x in enc_labels], dtype="int64")
    return np.expand_dims(enc_labels, axis=1)


class TrainBatch(object):
    """What a training step reads of torch_ext.Batch: counts_matrix [B, T, F] or read_level_features int8
    [B, P, D, F], labels [B, T] and, when a caller has them, majority_vote_probs [B, T, 5] (n_argmax_correct)."""

    def __init__(self, counts_matrix=None, labels=None, majority_vote_probs=None, read_level_features=None):
        self.counts_matrix, self.labels, self.majority_vote_probs = counts_matrix, labels, majority_vote_probs
        if read_level_features is not None:
            self.read_level_features = read_level_features


def pad_to_max_depth(read_level_features):
    """Batch.collate's padding of read-level samples [P, D_i, F] to the batch's maximum depth: int8 [B, P, Dmax, F],
    zeros past each sample's reads."""
    depths = [f.shape[1] for f in read_level_features]
    B, (P, _, F) = len(read_level_features), read_level_features[0].shape
    out = np.zeros((B, P, max(depths), F), np.int8)
    for i, f in enumerate(read_level_features):
        np.copyto(out[i, :, :depths[i], :], np.asarray(f), casting="unsafe")
    return out


class TrainBatcher(object):
    """Training and validation batches from this package's DataStores (medaka/training.py TrainBatcher)."""

    def __init__(self, features, validation=0.2, seed=0, batch_size=500, max_samples=None, max_valid_samples=None):
        from medaka_b200 import datastore
        self.logger = logging.getLogger("TrainBatcher")
        self.seed, self.batch_size = seed, batch_size
        self.samples = self._index(features)
        with datastore.DataStore(self.samples[0][1]) as ds:
            self.label_scheme = ds.get_meta("label_scheme")
            self.feature_encoder = ds.get_meta("feature_encoder")
            self.feature_shape = ds.load_sample(self.samples[0][0]).features.shape
        if len(self.feature_shape) not in (2, 3):
            raise NotImplementedError("training reads counts-matrix or read-level features only")
        self.read_level = len(self.feature_shape) == 3
        generator = np.random.default_rng(self.seed)
        if isinstance(validation, float):
            generator.shuffle(self.samples)
            n_train = int((1 - validation) * len(self.samples))
            self.train_samples, self.valid_samples = self.samples[:n_train], self.samples[n_train:]
        else:
            self.train_samples, self.valid_samples = self.samples, self._index(validation)
        if max_samples is not None and max_samples < len(self.train_samples):
            np.random.default_rng(self.seed).shuffle(self.train_samples)
            self.train_samples = self.train_samples[:max_samples]
        if max_valid_samples is not None and max_valid_samples < len(self.valid_samples):
            np.random.default_rng(self.seed).shuffle(self.valid_samples)
            self.valid_samples = self.valid_samples[:max_valid_samples]

    @staticmethod
    def _index(files):
        from medaka_b200 import datastore
        out = []
        for f in files:
            with datastore.DataStore(f) as ds:
                out += [(s, f) for s in sorted(ds.sample_registry)]
        return out

    def n_batches(self, which="train"):
        return len(self.train_samples if which == "train" else self.valid_samples) // self.batch_size

    def batches(self, which="train", rng=None):
        """Full batches (drop_last) of the training samples (shuffled with ``rng``) or the validation samples.  Like
        the reference's collate, which never sets majority_vote_probs for counts features, the batches carry none, so
        the epoch metrics have no n_argmax_correct."""
        from medaka_b200 import datastore
        samples = list(self.train_samples if which == "train" else self.valid_samples)
        if rng is not None:
            rng.shuffle(samples)
        for i in range(len(samples) // self.batch_size):
            feats, labels = [], []
            for key, fname in samples[i * self.batch_size:(i + 1) * self.batch_size]:
                with datastore.DataStore(fname) as ds:
                    s = ds.load_sample(key)
                feats.append(np.asarray(s.features) if self.read_level else np.asarray(s.features, np.float32))
                labels.append(encoded_labels_to_training_vectors(s.labels)[:, 0])
            labels = np.stack(labels).astype(np.int64)
            if self.read_level:
                yield TrainBatch(labels=labels, read_level_features=pad_to_max_depth(feats))
            else:
                yield TrainBatch(np.stack(feats), labels)


# ---------------------------------------------------------------------------------------------------------- the loop
class CSVLogger(object):
    """medaka/training.py CSVLogger: one header row from the first row's keys, '-' for absent values."""

    def __init__(self, filename):
        self.fh = open(filename, "a", newline="")
        self.writer = csv.writer(self.fh)
        self.columns = None

    def append(self, row):
        if self.columns is None:
            self.columns = list(row.keys())
            self.writer.writerow(self.columns)
        self.writer.writerow([row.get(k, "-") for k in self.columns])

    def __enter__(self):
        return self

    def __exit__(self, *args):
        self.fh.close()


def _model_dict(model_fp, batcher=None):
    from medaka_b200 import datastore
    if model_fp is None:
        # the default consensus model at the width of the store's counts (one to four datatypes: F = 10 to 40)
        if batcher is None or getattr(batcher, "read_level", False):
            return DEFAULT_MODEL_DICT, None
        kwargs = dict(DEFAULT_MODEL_DICT["kwargs"], num_features=int(batcher.feature_shape[-1]))
        return dict(DEFAULT_MODEL_DICT, kwargs=kwargs), None
    if model_fp.endswith(".gz"):
        store = datastore.ModelStoreTGZ(model_fp)
        return store.model_kwargs(), store._unpack()._weights
    if model_fp.endswith("toml"):
        with open(model_fp, "rb") as fh:
            return tomllib.load(fh), None
    raise ValueError("Unknown model file type: {}".format(model_fp))


def _init_state_dict(num_features, gru_size, seed):
    """torch.nn.GRU / nn.Linear default initialisation: U(-1/sqrt(H), 1/sqrt(H)), U(-1/sqrt(2H), 1/sqrt(2H))."""
    import torch
    torch.manual_seed(seed)
    gru = torch.nn.GRU(num_features, gru_size, num_layers=2, bidirectional=True, batch_first=True)
    lin = torch.nn.Linear(2 * gru_size, 5)
    sd = {"gru." + k: v.detach().numpy() for k, v in gru.state_dict().items()}
    sd.update({"linear." + k: v.detach().numpy() for k, v in lin.state_dict().items()})
    return sd


def _init_rl_state_dict(kwargs, seed):
    """A fresh LatentSpaceLSTM's state dict: torch's modules built in the reference's construction order under
    torch.manual_seed(seed), so the weights equal model_from_dict's under the same seed."""
    import torch
    H, C = int(kwargs.get("lstm_size", 128)), int(kwargs.get("cnn_size", 128))
    nin = 6 + 1 + (1 if kwargs.get("use_dwells", False) else 0)
    torch.manual_seed(seed)
    mods = [("base_embedder.", torch.nn.Embedding(6, 6)), ("strand_embedder.", torch.nn.Embedding(3, 6)),
            ("read_level_conv.convs.0.", torch.nn.Conv1d(nin, C, kernel_size=1, padding=0)),
            ("read_level_conv.convs.2.", torch.nn.BatchNorm1d(C)),
            ("read_level_conv.convs.3.", torch.nn.Conv1d(C, C, kernel_size=17, padding=8)),
            ("read_level_conv.convs.5.", torch.nn.BatchNorm1d(C)),
            ("read_level_conv.expansion_layer.", torch.nn.Linear(C, H)),
            ("pre_pool_expansion_layer.", torch.nn.Linear(C, H)),
            ("lstm.", torch.nn.LSTM(H, H, num_layers=2, bidirectional=True, batch_first=True)),
            ("linear.", torch.nn.Linear(2 * H, 5))]
    sd = {}
    for prefix, m in mods:
        sd.update({prefix + k: v.detach().numpy() for k, v in m.state_dict().items()})
    return sd


def run_epoch(trainer, batches, clip_grad=None, lr_scheduler=None, loss_log=None, is_training_epoch=False):
    """torch_ext.run_epoch: (mean batch loss, metrics) with the reference's metric names.  As there, the learning-rate
    schedule advances once per batch of a validation epoch too, when one is given."""
    from time import perf_counter
    total = {"n_model_correct": 0, "n_positions": 0}
    sum_loss, n_batches, n_samples, t0 = 0.0, 0, 0, perf_counter()
    for batch in batches:
        n_samples += np.shape(batch.labels)[0]
        if is_training_epoch:
            lr = lr_scheduler.get_last_lr()[0] if lr_scheduler is not None else trainer.lr
            max_norm = clip_grad.max_norm() if clip_grad is not None else None
            loss, metrics, grad_norm, _ = trainer.train_step(batch, lr=lr, max_norm=max_norm)
            if clip_grad is not None:
                clip_grad.record(grad_norm)
        else:
            loss, metrics = trainer.process_batch(batch)
            lr, grad_norm = None, 0
        sum_loss += loss
        n_batches += 1
        for k, v in metrics.items():
            total[k] = total.get(k, 0) + v
        if loss_log is not None:
            loss_log.append({
                "samples": n_samples, "time": perf_counter() - t0, "grad_norm": grad_norm, "lr": lr, "loss": loss,
                "model_correct": metrics["n_model_correct"] / metrics["n_positions"],
                "argmax_correct": metrics.get("n_argmax_correct", 0) / metrics["n_positions"],
                "n_positions": metrics["n_positions"]})
        if lr_scheduler is not None:
            lr_scheduler.step()
    n_pos = max(total["n_positions"], 1)
    epoch_metrics = {"model_tot_acc": total["n_model_correct"] / n_pos,
                     "argmax_tot_acc": total.get("n_argmax_correct", 0) / n_pos}
    epoch_metrics.update(total)
    return sum_loss / max(n_batches, 1), epoch_metrics


def run_training(train_name, batcher, model_fp=None, epochs=10, optimizer="rmsprop", optim_args=None, loss_args=None,
                 use_lr_schedule=True, samples_per_training_epoch=None, quantile_grad_clip=True, amp=False, device=0,
                 seed=0):
    """medaka/training.py run_training on the H100: per epoch a training pass (losses_{n}.csv), a validation pass, a
    row of training.csv, model-{n}.tar.gz and model-best_*.tar.gz archives (ModelStoreTGZ, loadable by the reference);
    stops after 20 epochs without a better validation loss.  As in the reference, the schedule spans epochs x the
    training batches of the whole store (samples_per_training_epoch only ends an epoch early), it advances on
    validation batches too, and quantile_grad_clip=False clips at a fixed norm of 2.  The reference's optim_{n}.pt is
    not written."""
    from medaka_b200 import datastore
    if loss_args:
        raise ValueError("loss argument(s) {} are not implemented: the loss is CrossEntropyLoss()".format(
            ", ".join(sorted(loss_args))))
    os.makedirs(train_name, exist_ok=True)
    model_dict, weights = _model_dict(model_fp, batcher)
    kw = model_dict.get("kwargs", {})
    if model_dict.get("type") == "LatentSpaceLSTM":
        from medaka_b200 import read_level
        import types
        read_level.LatentSpaceLSTM.check_feature_encoder_compatibility(
            types.SimpleNamespace(use_dwells=bool(kw.get("use_dwells", False))), batcher.feature_encoder)
        trainer = RLTrainer(device=device, optimizer=optimizer, optim_args=optim_args, amp=amp, **kw)
        trainer.load_state_dict(weights if weights is not None else _init_rl_state_dict(kw, seed))
    elif model_dict.get("type") == "GRUModel":
        num_features, gru_size = int(kw.get("num_features", 10)), int(kw.get("gru_size", 128))
        trainer = GRUTrainer(num_features=num_features, num_classes=int(kw.get("num_classes", 5)), gru_size=gru_size,
                             device=device, optimizer=optimizer, optim_args=optim_args, amp=amp)
        trainer.load_state_dict(weights if weights is not None else _init_state_dict(num_features, gru_size, seed))
    else:
        raise NotImplementedError("only the consensus GRUModel and the read-level LatentSpaceLSTM are trained")
    meta = {"model_function": functools.partial(datastore._ref_model_from_dict, model_dict),
            "label_scheme": batcher.label_scheme, "feature_encoder": batcher.feature_encoder}
    clip_grad = ClipGrad() if quantile_grad_clip else FixedClip(2.0)
    n_train = batcher.n_batches("train")
    steps = n_train
    if samples_per_training_epoch is not None:
        steps = min(steps, max(1, samples_per_training_epoch // batcher.batch_size))
    sched = linear_warmup_cosine_decay() if use_lr_schedule else no_schedule(warmup_steps=None)
    lr_scheduler = sched(trainer.lr, n_train, epochs, 0)
    rng = np.random.default_rng(seed)
    best_val_loss, best_epoch = np.inf, -1
    best_metrics = {"val_model_tot_acc": 0}

    def save(tag):
        datastore.ModelStoreTGZ.write(os.path.join(train_name, "model-{}.tar.gz".format(tag)), trainer.state_dict(), meta)

    with CSVLogger(os.path.join(train_name, "training.csv")) as training_log:
        for n in range(epochs):
            train_batches = (b for i, b in enumerate(batcher.batches("train", rng)) if i < steps)
            with CSVLogger(os.path.join(train_name, "losses_{}.csv".format(n))) as loss_log:
                train_loss, train_metrics = run_epoch(trainer, train_batches, clip_grad, lr_scheduler, loss_log,
                                                      is_training_epoch=True)
            val_loss, val_metrics = run_epoch(trainer, batcher.batches("valid"), lr_scheduler=lr_scheduler)
            all_metrics = {**{"train_" + k: v for k, v in train_metrics.items()},
                           **{"val_" + k: v for k, v in val_metrics.items()}}
            training_log.append({"epoch": n, "train_loss": train_loss, "val_loss": val_loss, **all_metrics})
            save(n)
            for k in best_metrics:
                if all_metrics[k] > best_metrics[k]:
                    save("best_{}".format(k))
                    best_metrics[k] = all_metrics[k]
            if val_loss < best_val_loss:
                save("best_val_loss")
                best_val_loss, best_epoch = val_loss, n
            if n >= best_epoch + 20:
                break
    return trainer
