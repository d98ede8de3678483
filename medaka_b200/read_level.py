"""Read-level consensus model behind the reference's model seam.

Mirror of ``medaka.architectures.latent_space_lstm.LatentSpaceLSTM`` (latent_space_lstm.py:34-207) as far as inference
needs it: constructor keywords, ``load_state_dict`` with the reference's parameter names, ``predict_on_batch`` on a batch
whose ``read_level_features`` is the int8 tensor [batch, positions, reads, features] of
``ReadAlignmentFeatureEncoder`` (``ReadLevelFeaturesModel.get_model_input_features``, base_classes.py:29-36), the
compatibility check of :209-236.  The arithmetic runs in libmedaka_b200 (``mdk_rl_*``, csrc/readlevel.cu).
"""
import warnings

import numpy as np

from medaka_b200 import libmedaka as _lm


class LatentSpaceLSTM(object):

    def __init__(self, num_classes=5, lstm_size=128, cnn_size=128, kernel_sizes=(1, 17), pooler_type="mean",
                 pooler_args=None, use_dwells=False, bases_alphabet_size=6, bases_embedding_size=6, bidirectional=True,
                 time_steps=None, device=0):
        if time_steps is not None:
            warnings.warn("timesteps is no longer required to be specified")
        if list(kernel_sizes) != [1, 17] or pooler_type != "mean" or not bidirectional or bases_alphabet_size != 6 \
                or bases_embedding_size != 6:
            raise NotImplementedError("the engine implements the bidirectional, mean-pooled, kernel_sizes=[1, 17] model")
        self.num_classes, self.lstm_size, self.cnn_size = num_classes, lstm_size, cnn_size
        self.kernel_sizes, self.pooler_type, self.pooler_args = list(kernel_sizes), pooler_type, pooler_args or {}
        self.use_dwells = use_dwells
        self.bases_alphabet_size, self.bases_embedding_size = bases_alphabet_size, bases_embedding_size
        self.bidirectional = bidirectional
        self.normalise = True
        self.device_index = device
        lib, ffi = _lm.load(), _lm.ffi
        _lm.require_gpu(device)
        pe = ffi.new("mdk_rl_engine **")
        _lm.check(lib.mdk_rl_create(device, lstm_size, cnn_size, 1 if use_dwells else 0, num_classes, pe))
        self._engine = pe[0]
        self.max_cells = 1 << 26            # positions x reads per device call
        self.max_bytes = 8 << 30            # forward_arrays' call size in scratch_bytes_per_window units, bytes
        self._fp32_conv = False
        self._pinned = {}
        self._async_n = 0

    # ---- TorchModel interface (medaka/models.py:233-313) ----
    def load_state_dict(self, state_dict, strict=True):
        lib, ffi = _lm.lib, _lm.ffi
        for name, t in state_dict.items():
            if name.endswith("num_batches_tracked"):
                continue
            a = np.ascontiguousarray(t.detach().cpu().numpy() if hasattr(t, "detach") else t, dtype=np.float32)
            _lm.check(lib.mdk_rl_load(self._engine, name.encode(), ffi.cast("const float *", ffi.from_buffer(a)), a.size))
        return self

    def set_conv(self, tensor_cores=True, lstm_tensor_cores=None):
        """k = 17 convolution / LSTM recurrences on the tensor cores (default, three fp16 products per contraction) or on
        the fp32 CUDA cores (validation)."""
        if lstm_tensor_cores is None:
            lstm_tensor_cores = tensor_cores
        _lm.check(_lm.lib.mdk_rl_set_conv(self._engine, (1 if tensor_cores else 0) | (2 if lstm_tensor_cores else 0)))
        self._fp32_conv = not tensor_cores

    PRECISIONS = {"tc": 3, "fp16": 7, "fp32": 0}      # mdk_rl_set_conv's bits

    def set_precision(self, mode):
        """'tc' (default: wgmma, three fp16 products per contraction, fp32-faithful), 'fp16' (wgmma, one product hi.hi
        per contraction: what medaka runs on a GPU without --full_precision) or 'fp32' (the CUDA-core twins).  The mode
        travels with the model to every entry point; windows submitted before a change run in the old mode."""
        if mode not in self.PRECISIONS:
            raise ValueError("precision must be one of %s, got %r" % (", ".join(self.PRECISIONS), mode))
        _lm.check(_lm.lib.mdk_rl_set_conv(self._engine, self.PRECISIONS[mode]))
        self._fp32_conv = mode == "fp32"

    STAGES = ("convolution", "projection_0", "recurrence_0", "projection_1", "recurrence_1", "head")

    def set_timing(self, on=True):
        """Record per-stage device times (CUDA events) in the forwards that follow; read them with stage_ms()."""
        _lm.check(_lm.lib.mdk_rl_set_timing(self._engine, 1 if on else 0))

    def stage_ms(self):
        """Device time of each stage of the last device call, in ms, keyed by the names in STAGES."""
        ms = _lm.ffi.new("float[6]")
        _lm.check(_lm.lib.mdk_rl_stage_ms(self._engine, ms))
        return dict(zip(self.STAGES, (float(v) for v in ms)))

    def scratch_bytes_per_window(self, P, D, F):
        """Bytes per window that windows_per_call budgets against max_bytes: every intermediate of the window at once
        (features, conv partial sums, z, gi, h0, h1, probabilities).  The engine no longer holds them all: a call's
        convolution runs in slices of a fixed 2 GiB scratch and the group buffers take 52 H + 21 bytes per position
        (DESIGN §4).  The formula is kept so that forward_arrays cuts batches into the same calls as before."""
        H, groups = self.lstm_size, -(-D // 4)
        per_pos = D * F + groups * 512 + 4 * H + 32 * H + 16 * H + 20 + (D * 512 if self._fp32_conv else 0)
        return P * per_pos + D

    def eval(self):
        return self

    def half(self):
        return self

    def device(self):
        return "cuda:%d" % self.device_index

    def get_model_input_features(self, batch):
        return batch.read_level_features

    def check_feature_encoder_compatibility(self, fenc):
        """latent_space_lstm.py:209-236."""
        from medaka_b200 import features
        if not isinstance(fenc, features.ReadAlignmentFeatureEncoder):
            raise ValueError("LatentSpaceLSTM expects a ReadAlignmentFeatureEncoder.")
        if len(fenc.dtypes) > 1:
            raise NotImplementedError("LatentSpaceLSTM is currently only implemented for one dtype.")
        if self.use_dwells and not getattr(fenc, "include_dwells", False):
            raise ValueError("Model expects dwells, however include_dwells not set in the feature encoder.")

    def forward_arrays(self, x):
        """x int8 [B, P, D, F] -> probabilities float32 [B, P, 5]."""
        x = np.ascontiguousarray(x.detach().cpu().numpy() if hasattr(x, "detach") else x)
        if x.dtype != np.int8:
            x = x.astype(np.int8)
        if x.ndim != 4:
            raise ValueError("expected read-level features [batch, positions, reads, features]")
        B, P, D, F = x.shape
        lib, ffi = _lm.lib, _lm.ffi
        probs = np.empty((B, P, 5), dtype=np.float32)
        step = self.windows_per_call(P, D, F)
        self._last_call = None
        for b0 in range(0, B, step):
            xb = np.ascontiguousarray(x[b0:b0 + step])
            pb = probs[b0:b0 + step]
            _lm.check(lib.mdk_rl_forward(self._engine, ffi.cast("const int8_t *", ffi.from_buffer(xb)), len(xb), P, D, F,
                                         ffi.cast("float *", ffi.from_buffer(pb))))
            self._last_call = (len(xb), P)
        return probs

    MAX_WINDOWS_PER_CALL = 65535            # mdk_rl_forward's limit on B

    def windows_per_call(self, P, D, F):
        """Windows per device call of forward_arrays: bounded in cells (max_cells), in scratch bytes (max_bytes; at
        lstm_size 384, gi alone takes 12 KiB per position) and by mdk_rl_forward's B <= 65535.  The windows are
        independent, so the split does not change the outputs."""
        step = min(int(self.max_cells // max(P * D, 1)), int(self.max_bytes // self.scratch_bytes_per_window(P, D, F)))
        return max(1, min(step, self.MAX_WINDOWS_PER_CALL))

    STAGE_INDEX = {"z": 0, "h0": 1, "h1": 2}

    def read_stage(self, name):
        """An intermediate of the last device call, float32: "z" [B, P, H] (pooled pre_pool_expansion_layer output, the
        LSTM input), "h0" / "h1" [B, P, 2H] (the LSTM layers' outputs, forward direction in the first H columns).

        B and P are those of the last mdk_rl_forward call, so this covers the whole batch only when the last
        forward_arrays ran as ONE device call (B <= windows_per_call(P, D, F)); otherwise it holds the last slice."""
        last = getattr(self, "_last_call", None)
        if last is None:
            raise RuntimeError("read_stage: no forward has completed on this model")
        B, P = last
        width = self.lstm_size if name == "z" else 2 * self.lstm_size
        out = np.empty((B, P, width), dtype=np.float32)
        _lm.check(_lm.lib.mdk_rl_debug_read(self._engine, self.STAGE_INDEX[name],
                                            _lm.ffi.cast("float *", _lm.ffi.from_buffer(out)), out.size))
        return out

    # ---- packed asynchronous calls (mdk_rl_submit / wait / flush / reserve) ----
    def pinned(self, key, shape, dtype):
        """Reusable page-locked staging array, grown on demand."""
        from medaka_b200 import models
        return models.pinned_array(self._pinned, key, shape, dtype)

    def predict_async(self, batch, slots=2):
        """Asynchronous predict_on_batch: returns a handle whose ``result()`` is the CPU tensor [B, P, 5] and which then
        carries the argmax labels (uint8 [B, P]) as ``.labels``.

        Up to ``slots`` calls may be in flight, each with its own page-locked staging for the int8 features and the
        outputs.  The engine runs each call's convolution when it is submitted and packs the calls' windows into groups
        of ``preferred_batch_size()`` windows whose LSTM runs once (mdk_rl_submit), so the reference's 100-window
        batches share recurrence waves instead of paying the P-step chain each.
        """
        slot = self._async_n % max(int(slots), 1)
        self._async_n += 1
        return self._submit(batch, "a%d" % slot)

    def _submit(self, batch, key):
        """Submit the batch's features through the page-locked staging arrays named `key`; returns the handle."""
        from medaka_b200 import models
        x = self.get_model_input_features(batch)
        x = x.detach().cpu().numpy() if hasattr(x, "detach") else np.asarray(x)
        if x.ndim != 4:
            raise ValueError("expected read-level features [batch, positions, reads, features]")
        B, P, D, F = x.shape
        lib, ffi = _lm.lib, _lm.ffi
        self._last_call = None                               # this call's group overwrites the stages read_stage reads
        xin = self.pinned(key + "feats", (B, P, D, F), np.int8)
        np.copyto(xin, x, casting="unsafe")                  # collated batches are uint8 (torch_ext.Batch.collate)
        probs = self.pinned(key + "probs", (B, P, 5), np.float32)
        labels = self.pinned(key + "labels", (B, P), np.uint8)
        ticket = ffi.new("int64_t *")
        _lm.check(lib.mdk_rl_submit(self._engine, ffi.cast("const int8_t *", ffi.from_buffer(xin)), B, P, D, F,
                                    ffi.cast("float *", ffi.from_buffer(probs)),
                                    ffi.cast("uint8_t *", ffi.from_buffer(labels)), ticket))
        ticket = int(ticket[0])
        return models.AsyncResult(self, lambda: _lm.check(_lm.lib.mdk_rl_wait(self._engine, ticket)), probs, labels)

    @staticmethod
    def _ptr(x, ctype):
        """cffi pointer to a numpy array or to a device address (int)."""
        ffi = _lm.ffi
        if x is None:
            return ffi.NULL
        return ffi.cast(ctype, x) if isinstance(x, int) else ffi.cast(ctype, ffi.from_buffer(x))

    def _features(self, feats):
        feats = np.asarray(feats)
        if feats.ndim != 4 or feats.dtype != np.int8:
            raise ValueError("expected int8 read-level features [batch, positions, reads, features], got {} {}".format(
                feats.dtype, feats.shape))
        if not feats.flags.c_contiguous:
            raise ValueError("features must be contiguous")
        self._last_call = None                               # the call's group overwrites the stages read_stage reads
        return feats.shape

    def submit_decoded(self, feats, labels_out, quals_out=None):
        """Queue one forward whose outputs are the decoded calls (mdk_rl_submit_decoded); returns a ticket for ``wait``.

        ``feats`` int8 [B, P, D, F] host array (page-locked, ``pinned``, for an asynchronous copy).  ``labels_out`` /
        ``quals_out`` receive uint8 [B, P] argmax labels and phred+33 quality bytes: numpy arrays, or device addresses
        (int) of B * P bytes.  ``quals_out`` may be None.  Everything must stay alive and untouched until
        ``wait(ticket)`` (or ``sync``).
        """
        B, P, D, F = self._features(feats)
        ticket = _lm.ffi.new("int64_t *")
        _lm.check(_lm.lib.mdk_rl_submit_decoded(self._engine, self._ptr(feats, "const int8_t *"), B, P, D, F,
                                                self._ptr(labels_out, "uint8_t *"), self._ptr(quals_out, "uint8_t *"),
                                                ticket))
        return int(ticket[0])

    def submit_variant_decoded(self, feats, ref_bytes, calls_out, pred_q_out, ref_q_out):
        """Queue one forward whose outputs are what variant decoding needs (mdk_rl_submit_variant_decoded); returns a
        ticket.

        ``feats`` int8 [B, P, D, F] host array; ``ref_bytes`` uint8 [B, P] (the draft's label code per column, 0x80 on
        insertion columns) a numpy array or a device address.  ``calls_out`` uint8 [B, P] and ``pred_q_out`` /
        ``ref_q_out`` float32 [B, P] are numpy arrays or device addresses (int).  Everything must stay alive and
        untouched until ``wait(ticket)`` (or ``sync``).
        """
        B, P, D, F = self._features(feats)
        if not isinstance(ref_bytes, int) and tuple(ref_bytes.shape) != (B, P):
            raise ValueError("ref_bytes must be [B, P] = [{}, {}], got {}".format(B, P, tuple(ref_bytes.shape)))
        ticket = _lm.ffi.new("int64_t *")
        _lm.check(_lm.lib.mdk_rl_submit_variant_decoded(
            self._engine, self._ptr(feats, "const int8_t *"), B, P, D, F, self._ptr(ref_bytes, "const uint8_t *"),
            self._ptr(calls_out, "uint8_t *"), self._ptr(pred_q_out, "float *"), self._ptr(ref_q_out, "float *"), ticket))
        return int(ticket[0])

    def wait(self, ticket):
        """Wait for a submitted call (mdk_rl_wait)."""
        _lm.check(_lm.lib.mdk_rl_wait(self._engine, int(ticket)))

    def sync(self):
        """Launch the open group and wait for every call queued on the engine (mdk_rl_sync)."""
        _lm.check(_lm.lib.mdk_rl_sync(self._engine))

    def preferred_batch_size(self):
        """Windows one packed group holds at the reference's 10 000-position chunks (mdk_rl_preferred_windows: one
        recurrence wave within the group buffers' memory budget, 112 at lstm_size 384 on an H100);
        ``batch_size="auto"`` in ``prediction.run_prediction`` resolves to this."""
        return int(_lm.lib.mdk_rl_preferred_windows(self._engine))

    def lookahead(self, batch_size, window_len=None):
        """How many ``predict_async`` calls of ``batch_size`` windows to keep in flight: enough to fill the group that
        computes and to start filling the next one (its convolutions queue behind the group in flight)."""
        pref = self.preferred_batch_size()
        return int(max(2, min(64, 2 * ((pref + batch_size - 1) // max(batch_size, 1)) + 1)))

    def reserve(self, windows, window_len):
        """Size the group buffers for packed groups of up to ``windows`` windows (mdk_rl_reserve)."""
        _lm.check(_lm.lib.mdk_rl_reserve(self._engine, int(windows), int(window_len)))

    def flush(self):
        _lm.check(_lm.lib.mdk_rl_flush(self._engine))

    def predict_on_batch(self, batch):
        """TorchModel.predict_on_batch (models.py:303-313): CPU float32 tensor [B, P, 5].  Runs through the packed path
        (one submit, then wait), and keeps the argmax labels of the call on ``self.last_labels`` (uint8 [B, P])."""
        return self._submit(batch, "sync").result()

    def to_dict(self):
        return {"type": "LatentSpaceLSTM", "kwargs": {
            "num_classes": self.num_classes, "lstm_size": self.lstm_size, "cnn_size": self.cnn_size,
            "kernel_sizes": self.kernel_sizes, "pooler_type": self.pooler_type, "pooler_args": self.pooler_args,
            "use_dwells": self.use_dwells, "bases_alphabet_size": self.bases_alphabet_size,
            "bases_embedding_size": self.bases_embedding_size, "bidirectional": self.bidirectional}}

    def close(self):
        if getattr(self, "_engine", None) is not None and _lm.lib is not None:
            _lm.lib.mdk_rl_destroy(self._engine)
            self._engine = None
        for p in getattr(self, "_pinned", {}).values():
            p.close()
        self._pinned = {}

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
