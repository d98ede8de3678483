"""Model seam: a drop-in for the reference's GRUModel / TorchModel backed by libmedaka_b200.

Mirrors medaka/architectures/gru.py:13-72 (constructor arguments, ``forward``) and
medaka/models.py:277-383 (``TorchModel``: ``predict_on_batch``, ``device``, ``half``,
``eval``, ``load_state_dict``, ``to_dict``, ``check_feature_encoder_compatibility``),
so ``prediction.run_prediction`` (medaka/prediction.py:44-52) runs unchanged on top of it.
PyTorch tensors are used only as host containers for weights and for the returned CPU
tensor; all arithmetic runs in the CUDA library.  No CPU fallback.
"""
import collections
import inspect
import logging
import warnings

import numpy as np

from medaka_b200 import libmedaka as _lm

ForwardOutput = collections.namedtuple("ForwardOutput", ["probs", "logits", "labels"])

# mdk_engine_set_precision's modes (MDK_PREC_*); "half" and "full" are the names half() and float() stand for
_PRECISIONS = {"tc": 0, "half": 0, "fp32": 1, "full": 1, "fp16": 2}


def _as_f32(x):
    """numpy float32 C-contiguous view/copy of a torch tensor or array-like."""
    if hasattr(x, "detach"):
        x = x.detach().cpu().numpy()
    return np.ascontiguousarray(x, dtype=np.float32)


class PinnedArray(object):
    """A numpy array living in CUDA page-locked host memory (mdk_host_alloc)."""

    def __init__(self, shape, dtype):
        lib = _lm.load()
        self.shape = tuple(int(s) for s in shape)
        self.dtype = np.dtype(dtype)
        self.nbytes = int(np.prod(self.shape)) * self.dtype.itemsize
        pp = _lm.ffi.new("void **")
        _lm.check(lib.mdk_host_alloc(max(self.nbytes, 1), pp))
        self._ptr = pp[0]
        buf = _lm.ffi.buffer(self._ptr, max(self.nbytes, 1))
        self.array = np.frombuffer(buf, dtype=self.dtype, count=int(np.prod(self.shape))).reshape(self.shape)

    def close(self):
        if getattr(self, "_ptr", None) is not None and _lm.lib is not None:
            self.array = None
            _lm.lib.mdk_host_free(self._ptr)
            self._ptr = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def pinned_array(cache, key, shape, dtype):
    """A view of shape ``shape`` on the page-locked array ``cache[key]``, which is (re)allocated when it is too small."""
    need = int(np.prod(shape))
    cur = cache.get(key)
    if cur is None or cur.dtype != np.dtype(dtype) or int(np.prod(cur.shape)) < need:
        if cur is not None:
            cur.close()
        cur = PinnedArray((need,), dtype)
        cache[key] = cur
    return cur.array[:need].reshape(shape)


class AsyncResult(object):
    """Handle of one asynchronous call: ``result()`` waits for it, then returns the probabilities as a CPU tensor and
    leaves the argmax labels on ``.labels`` and on the model's ``last_labels`` (copies of the page-locked staging)."""

    def __init__(self, model, wait, probs, labels):
        self._model, self._wait, self._probs, self._labels = model, wait, probs, labels

    def result(self):
        import torch
        self._wait()
        self._model.last_labels = self.labels = self._labels.copy()
        return torch.from_numpy(self._probs.copy())


class GRUModel(object):
    """Bidirectional GRU consensus model (gru.py:10-72) executing on an H100.

    The constructor signature is the reference's, so ``model_from_dict``-style
    configs (medaka/models.py:392-400) instantiate it directly.
    """

    def __init__(self, num_features=10, num_classes=5, gru_size=128, n_layers=2,
                 bidirectional=True, time_steps=None, classify_activation=None, device=0):
        if time_steps is not None:
            warnings.warn("timesteps is no longer required to be specified")
        if classify_activation is not None:
            warnings.warn("classify_activation is no longer used")
        self.gru_size = gru_size
        self.num_classes = num_classes
        self.num_features = num_features
        self.n_layers = n_layers
        self.bidirectional = bidirectional
        self.normalise = True
        self.half_precision = False
        self.logger = logging.getLogger("B200Model")
        self._device = int(device)
        self._state = {}
        self._pinned = {}
        self._engine = None
        lib = _lm.load()
        _lm.require_gpu(self._device)
        desc = _lm.ffi.new("mdk_model_desc *")
        desc.num_features = num_features
        desc.gru_size = gru_size
        desc.n_layers = n_layers
        desc.bidirectional = 1 if bidirectional else 0
        desc.num_classes = num_classes
        pe = _lm.ffi.new("mdk_engine **")
        _lm.check(lib.mdk_engine_create(self._device, desc, pe))
        self._engine = pe[0]

    # ------------------------------------------------------------------ torch.nn.Module look-alikes
    def eval(self):
        return self

    def to(self, device=None):
        return self

    def device(self):
        """Device where the model has been loaded (medaka/models.py:291-296)."""
        import torch
        return torch.device("cuda", self._device)

    def half(self):
        """TorchModel.half (models.py:298-301): tensor-core path (fp16 hi/lo split operands)."""
        self.half_precision = True
        self.set_precision("tc")
        return self

    def float(self):
        self.half_precision = False
        self.set_precision("fp32")
        return self

    def set_precision(self, mode):
        """'tc' (wgmma, default: three fp16 products per contraction, fp32-faithful), 'fp16' (wgmma, one product hi.hi
        per contraction: what medaka runs on a GPU without --full_precision) or 'fp32' (CUDA-core FFMA, the
        --full_precision path).  half() keeps selecting 'tc'.  The mode travels with the model to every entry point;
        windows submitted before a change run in the old mode."""
        if mode not in _PRECISIONS:
            raise ValueError("precision must be one of %s, got %r" % (", ".join(_PRECISIONS), mode))
        _lm.check(_lm.lib.mdk_engine_set_precision(self._engine, _PRECISIONS[mode]))

    def parameters(self):
        return iter(self._state.values())

    def count_parameters(self):
        return int(sum(v.size for v in self._state.values()))

    def state_dict(self):
        import torch
        return collections.OrderedDict((k, torch.from_numpy(v.copy())) for k, v in self._state.items())

    def load_state_dict(self, state_dict, strict=True):
        """torch state-dict layout (SURVEY.md 3.4); mirrors datastore.py:150-152."""
        lib = _lm.lib
        H, F = self.gru_size, self.num_features
        ndir = 2 if self.bidirectional else 1
        expected = {}
        for layer in range(self.n_layers):
            n_in = F if layer == 0 else H * ndir
            for sfx in [""] + (["_reverse"] if self.bidirectional else []):
                expected["gru.weight_ih_l%d%s" % (layer, sfx)] = (3 * H, n_in)
                expected["gru.weight_hh_l%d%s" % (layer, sfx)] = (3 * H, H)
                expected["gru.bias_ih_l%d%s" % (layer, sfx)] = (3 * H,)
                expected["gru.bias_hh_l%d%s" % (layer, sfx)] = (3 * H,)
        expected["linear.weight"] = (5, H * ndir)
        expected["linear.bias"] = (5,)
        missing = [k for k in expected if k not in state_dict]
        unexpected = [k for k in state_dict if k not in expected]
        if missing or (strict and unexpected):
            raise RuntimeError("Error(s) in loading state_dict: missing {}, unexpected {}".format(
                missing, unexpected))
        sd = {}
        for k, shape in expected.items():
            a = _as_f32(state_dict[k])
            if a.shape != shape:
                raise RuntimeError("size mismatch for {}: expected {}, got {}".format(k, shape, a.shape))
            sd[k] = a
        ptr = lambda a: _lm.ffi.cast("const float *", _lm.ffi.from_buffer(a))   # noqa: E731
        for layer in range(self.n_layers):
            for d, sfx in enumerate([""] + (["_reverse"] if self.bidirectional else [])):
                _lm.check(lib.mdk_engine_load_gru(
                    self._engine, layer, d,
                    ptr(sd["gru.weight_ih_l%d%s" % (layer, sfx)]), ptr(sd["gru.weight_hh_l%d%s" % (layer, sfx)]),
                    ptr(sd["gru.bias_ih_l%d%s" % (layer, sfx)]), ptr(sd["gru.bias_hh_l%d%s" % (layer, sfx)])))
        _lm.check(lib.mdk_engine_load_linear(self._engine, ptr(sd["linear.weight"]), ptr(sd["linear.bias"])))
        self._state = sd
        return self

    # ------------------------------------------------------------------ TorchModel interface
    def get_model_input_features(self, batch):
        """CountsMatrixModel (medaka/architectures/base_classes.py:9-11)."""
        return batch.counts_matrix

    def check_feature_encoder_compatibility(self, fenc):
        """base_classes.py:13-20: counts-matrix models need a counts encoder of matching width."""
        fvl = getattr(fenc, "feature_vector_length", None)
        if fvl is not None and int(fvl) != int(self.num_features):
            raise ValueError("Feature encoder produces {} features, model expects {}".format(fvl, self.num_features))

    def to_dict(self):
        """models.py:343-361."""
        kwargs = inspect.signature(self.__class__.__init__).parameters
        out = {}
        for k in kwargs:
            if k in ("self", "device"):
                continue
            out[k] = getattr(self, k, kwargs[k].default)
        return {"type": "GRUModel", "kwargs": out}

    def pinned(self, key, shape, dtype):
        """Reusable page-locked staging array, grown on demand."""
        return pinned_array(self._pinned, key, shape, dtype)

    def forward_arrays(self, feats, want_logits=False, want_labels=True):
        """feats float32 [B,T,F] (host) -> ForwardOutput of numpy arrays (copies out of pinned staging)."""
        feats = np.asarray(feats)
        if feats.ndim != 3 or feats.shape[2] != self.num_features:
            raise ValueError("expected features of shape [B, T, {}], got {}".format(self.num_features, feats.shape))
        B, T, F = feats.shape
        self._last_shape = (B, T)
        lib, ffi = _lm.lib, _lm.ffi
        x = self.pinned("feats", (B, T, F), np.float32)
        np.copyto(x, feats, casting="same_kind")
        probs = self.pinned("probs", (B, T, 5), np.float32)
        logits = self.pinned("logits", (B, T, 5), np.float32) if want_logits else None
        labels = self.pinned("labels", (B, T), np.uint8) if want_labels else None
        _lm.check(lib.mdk_engine_forward(
            self._engine, ffi.cast("const float *", ffi.from_buffer(x)), B, T,
            ffi.cast("float *", ffi.from_buffer(probs)),
            ffi.cast("float *", ffi.from_buffer(logits)) if want_logits else ffi.NULL,
            ffi.cast("uint8_t *", ffi.from_buffer(labels)) if want_labels else ffi.NULL))
        return ForwardOutput(probs.copy(), logits.copy() if want_logits else None,
                             labels.copy() if want_labels else None)

    def submit_arrays(self, feats_pinned, probs_out, labels_out=None, logits_out=None):
        """Queue one forward on host arrays WITHOUT waiting (mdk_engine_submit); returns a ticket for ``wait``.

        All arrays must stay alive and untouched until ``wait(ticket)``; page-locked arrays (``pinned``)
        make the copies asynchronous so consecutive calls overlap H2D, compute and D2H.
        """
        B, T, F = feats_pinned.shape
        lib, ffi = _lm.lib, _lm.ffi
        ticket = ffi.new("int64_t *")
        _lm.check(lib.mdk_engine_submit(
            self._engine, ffi.cast("const float *", ffi.from_buffer(feats_pinned)), B, T,
            ffi.cast("float *", ffi.from_buffer(probs_out)),
            ffi.cast("float *", ffi.from_buffer(logits_out)) if logits_out is not None else ffi.NULL,
            ffi.cast("uint8_t *", ffi.from_buffer(labels_out)) if labels_out is not None else ffi.NULL, ticket))
        self._last_shape = (B, T)
        return int(ticket[0])

    def submit_decoded(self, feats_pinned, labels_out, quals_out=None):
        """Queue one forward whose outputs are the decoded calls (mdk_engine_submit_decoded); returns a ticket.

        ``labels_out`` / ``quals_out`` receive uint8 [B, T] argmax labels and phred+33 quality bytes: numpy arrays,
        or device addresses (int) of B * T bytes.  ``quals_out`` may be None.  Everything must stay alive and untouched
        until ``wait(ticket)`` (or ``sync``).
        """
        B, T, F = feats_pinned.shape
        lib, ffi = _lm.lib, _lm.ffi

        def u8(x):
            if x is None:
                return ffi.NULL
            return ffi.cast("uint8_t *", x) if isinstance(x, int) else ffi.cast("uint8_t *", ffi.from_buffer(x))

        ticket = ffi.new("int64_t *")
        _lm.check(lib.mdk_engine_submit_decoded(
            self._engine, ffi.cast("const float *", ffi.from_buffer(feats_pinned)), B, T, u8(labels_out), u8(quals_out),
            ticket))
        self._last_shape = (B, T)
        return int(ticket[0])

    def submit_variant_decoded(self, feats, ref_bytes, calls_out, pred_q_out, ref_q_out):
        """Queue one forward whose outputs are what variant decoding needs (mdk_engine_submit_variant_decoded); returns
        a ticket.

        ``feats`` float32 [B, T, F] and ``ref_bytes`` uint8 [B, T] (the draft's label code per column, 0x80 on insertion
        columns) are numpy arrays (page-locked for an asynchronous copy) or CUDA tensors.  ``calls_out`` uint8 [B, T]
        and ``pred_q_out`` / ``ref_q_out`` float32 [B, T] are numpy arrays or device addresses (int).  Everything must
        stay alive and untouched until ``wait(ticket)`` (or ``sync``).
        """
        B, T, F = feats.shape
        if tuple(ref_bytes.shape) != (B, T):
            raise ValueError("ref_bytes must be [B, T] = [{}, {}], got {}".format(B, T, tuple(ref_bytes.shape)))
        lib, ffi = _lm.lib, _lm.ffi

        def ptr(x, ctype):
            if isinstance(x, int):
                return ffi.cast(ctype, x)
            if hasattr(x, "data_ptr"):
                if not x.is_contiguous():
                    raise ValueError("tensors must be contiguous")
                return ffi.cast(ctype, x.data_ptr())
            return ffi.cast(ctype, ffi.from_buffer(x))

        ticket = ffi.new("int64_t *")
        _lm.check(lib.mdk_engine_submit_variant_decoded(
            self._engine, ptr(feats, "const float *"), B, T, ptr(ref_bytes, "const uint8_t *"),
            ptr(calls_out, "uint8_t *"), ptr(pred_q_out, "float *"), ptr(ref_q_out, "float *"), ticket))
        self._last_shape = (B, T)
        return int(ticket[0])

    def sync(self):
        """Wait for every call queued on the engine (mdk_engine_sync)."""
        _lm.check(_lm.lib.mdk_engine_sync(self._engine))

    def wait(self, ticket):
        _lm.check(_lm.lib.mdk_engine_wait(self._engine, ticket))

    def predict_async(self, batch, slots=2):
        """Asynchronous predict_on_batch: returns a handle whose ``result()`` is the CPU tensor [B,T,5].

        Up to ``slots`` calls may be in flight (each owns one set of page-locked staging arrays).  The engine
        packs consecutive batches of the same window length into one-wave groups window by window (mdk_engine_submit;
        a batch may straddle two groups), so ``run_prediction`` keeps about three groups of batches queued: the
        reference's default 200-window batches then run as 1056-window groups, one computing at a time, with the
        PCIe copies of the neighbouring groups under the compute.
        """
        x = _as_f32(self.get_model_input_features(batch))
        B, T, F = x.shape
        slot = getattr(self, "_async_n", 0) % max(int(slots), 1)
        self._async_n = getattr(self, "_async_n", 0) + 1
        xin = self.pinned("afeats%d" % slot, (B, T, F), np.float32)
        np.copyto(xin, x)
        probs = self.pinned("aprobs%d" % slot, (B, T, 5), np.float32)
        labels = self.pinned("alabels%d" % slot, (B, T), np.uint8)
        ticket = self.submit_arrays(xin, probs, labels)
        return AsyncResult(self, lambda: self.wait(ticket), probs, labels)

    def lookahead(self, batch_size, window_len=None):
        """How many ``predict_async`` calls of ``batch_size`` windows to keep in flight (four coalesced groups, one per
        big staging lane: two computing, one copying in, one copying out)."""
        pref = self.preferred_batch_size()
        if window_len is not None and batch_size * window_len <= (1 << 18):
            return 14                                   # small forwards rotate over the engine's small lanes
        return int(max(2, min(64, 4 * ((pref + batch_size - 1) // max(batch_size, 1)) + 1)))

    def reserve(self, windows, window_len):
        """Size the engine's compute lanes for coalesced groups of up to ``windows`` windows (mdk_engine_reserve)."""
        _lm.check(_lm.lib.mdk_engine_reserve(self._engine, int(windows), int(window_len)))

    def flush(self):
        _lm.check(_lm.lib.mdk_engine_flush(self._engine))

    def set_rec_mode(self, mode):
        """'auto' | 'one' | 'pp': tiles per CTA of the recurrent kernels (mdk_engine_set_rec_mode).  'auto' runs two
        tiles per CTA for every forward with at most 16 features, so that a group's layer 1 runs beside the next group's
        layer 0, and otherwise one tile per CTA up to one wave of windows, two beyond.  At gru_size 256 the recurrence
        has one kernel and only 'auto' is accepted."""
        code = {"auto": _lm.lib.MDK_REC_AUTO, "one": _lm.lib.MDK_REC_ONE_TILE, "pp": _lm.lib.MDK_REC_PINGPONG}[mode]
        _lm.check(_lm.lib.mdk_engine_set_rec_mode(self._engine, code))

    def set_group_windows(self, windows):
        _lm.check(_lm.lib.mdk_engine_set_group_windows(self._engine, int(windows)))

    def forward(self, x):
        """gru.py:58-72 on host tensors: returns probabilities (or logits if normalise is off)."""
        import torch
        out = self.forward_arrays(_as_f32(x), want_logits=not self.normalise, want_labels=False)
        return torch.from_numpy(out.probs if self.normalise else out.logits)

    def predict_on_batch(self, batch):
        """TorchModel.predict_on_batch (models.py:303-313): returns a CPU float32 tensor [B,T,5].

        The argmax labels of the same call are kept on ``self.last_labels`` (uint8 [B,T]) so the
        decode stage need not recompute them (north-star: softmax/argmax on the GPU).
        """
        import torch
        out = self.forward_arrays(_as_f32(self.get_model_input_features(batch)), want_logits=False,
                                  want_labels=True)
        self.last_labels = out.labels
        return torch.from_numpy(out.probs)

    # ------------------------------------------------------------------ diagnostics
    def last_timings(self):
        t = _lm.ffi.new("mdk_timings *")
        _lm.check(_lm.lib.mdk_engine_last_timings(self._engine, t))
        return {k: getattr(t, k) for k in ("h2d_ms", "inproj0_ms", "rec0_ms", "inproj1_ms", "rec1_ms",
                                             "head_ms", "d2h_ms", "total_ms", "launches")}

    def read_activation(self, which, first=0, count=None):
        """Layer output [count,T,2*gru_size] of windows first .. first + count - 1 (default: all B) of the last forward
        (0 = layer 0, 1 = layer 1) for layer-wise parity."""
        t = self.last_timings()  # syncs
        del t
        shape = self._last_shape
        count = shape[0] - first if count is None else count
        out = np.empty((count, shape[1], 2 * self.gru_size), dtype=np.float32)
        _lm.check(_lm.lib.mdk_engine_read_activation_windows(
            self._engine, which, first, count, _lm.ffi.cast("float *", _lm.ffi.from_buffer(out)), out.size))
        return out

    def read_plog(self):
        """Partial logits of the last forward on the fused-head path, float32 [2 directions][tiles][T][5 classes][16
        windows] (mdk_debug_read_plog): what the layer-1 recurrence writes in place of h1."""
        t = self.last_timings()  # syncs
        del t
        B, T = self._last_shape
        out = np.empty((2, (B + 15) // 16, T, 5, 16), dtype=np.float32)
        _lm.check(_lm.lib.mdk_debug_read_plog(self._engine, _lm.ffi.cast("float *", _lm.ffi.from_buffer(out)), out.size))
        return out

    def launch_count(self):
        return int(_lm.lib.mdk_engine_launch_count(self._engine))

    def keep_activations(self, keep=True):
        """Debugging: keep the layer-1 output in HBM for ``read_activation(1)`` (runs the head as its own kernel)."""
        _lm.check(_lm.lib.mdk_engine_keep_activations(self._engine, 1 if keep else 0))

    def preferred_batch_size(self):
        """Windows per batch that fill the device in one wave (1056 on an H100 at gru_size 128, 240 at 256);
        ``batch_size="auto"`` in ``prediction.run_prediction`` / ``predict_regions`` resolves to this."""
        return int(_lm.lib.mdk_engine_preferred_windows(self._engine))

    @property
    def engine(self):
        return self._engine

    def close(self):
        if self._engine is not None and _lm.lib is not None:
            _lm.lib.mdk_engine_destroy(self._engine)
            self._engine = None
        for p in self._pinned.values():
            p.close()
        self._pinned = {}

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def model_from_dict(d, time_steps=None, device=0):
    """medaka/models.py:392-400 for the architectures this engine implements."""
    name, kwargs = d["type"], dict(d["kwargs"])
    kwargs.pop("read_majority_threshold", None)
    if name == "LatentSpaceLSTM":
        from medaka_b200 import read_level
        return read_level.LatentSpaceLSTM(device=device, **kwargs)
    if name != "GRUModel":
        raise NotImplementedError("medaka_b200 implements GRUModel and LatentSpaceLSTM; got {}".format(name))
    return GRUModel(device=device, **kwargs)


def build_model_torch(feature_len, num_classes, gru_size=128, classify_activation="softmax", time_steps=None,
                      device=0):
    """Legacy model function (medaka/models.py:403-431) -> the same GRUModel."""
    return GRUModel(num_features=feature_len, num_classes=num_classes, gru_size=gru_size, device=device)
