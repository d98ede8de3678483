"""Oracle for the read-level consensus network: LatentSpaceLSTM restated with plain torch modules.

TEST INFRASTRUCTURE (see oracle/__init__.py).  Follows medaka/architectures/latent_space_lstm.py:34-207 (bidirectional
variant), read_level_modules.py:7-100 (make_1dconv_layers, ReadLevelConv, MeanPooler).  Parameter names are the
reference's state-dict keys, so one state dict drives the reference class (tests/golden/make_rl_golden.py), this
restatement and the engine.
"""
import numpy as np
import torch


def synth_rl_state_dict(seed=0, lstm_size=128, cnn_size=128, use_dwells=False, gain=1.0):
    """Seeded random parameters in torch's own initialisation ranges, with non-trivial BatchNorm statistics."""
    rs = np.random.RandomState(seed)

    def u(shape, bound):
        return torch.from_numpy(rs.uniform(-bound, bound, size=shape).astype(np.float32))
    nin = 6 + 1 + (1 if use_dwells else 0)
    sd = {"base_embedder.weight": torch.from_numpy(rs.randn(6, 6).astype(np.float32)),
          "strand_embedder.weight": torch.from_numpy(rs.randn(3, 6).astype(np.float32))}
    for idx, (cin, k) in (("0", (nin, 1)), ("3", (cnn_size, 17))):
        bound = 1.0 / np.sqrt(cin * k)
        sd["read_level_conv.convs.%s.weight" % idx] = u((cnn_size, cin, k), bound * gain)
        sd["read_level_conv.convs.%s.bias" % idx] = u((cnn_size,), bound)
    for idx in ("2", "5"):
        sd["read_level_conv.convs.%s.weight" % idx] = torch.from_numpy(rs.uniform(0.5, 1.5, cnn_size).astype(np.float32))
        sd["read_level_conv.convs.%s.bias" % idx] = u((cnn_size,), 0.3)
        sd["read_level_conv.convs.%s.running_mean" % idx] = u((cnn_size,), 0.3)
        sd["read_level_conv.convs.%s.running_var" % idx] = torch.from_numpy(rs.uniform(0.3, 1.5, cnn_size).astype(np.float32))
        sd["read_level_conv.convs.%s.num_batches_tracked" % idx] = torch.tensor(7, dtype=torch.long)
    b = 1.0 / np.sqrt(cnn_size)
    sd["read_level_conv.expansion_layer.weight"] = u((lstm_size, cnn_size), b)      # present in the class, unused by forward
    sd["read_level_conv.expansion_layer.bias"] = u((lstm_size,), b)
    sd["pre_pool_expansion_layer.weight"] = u((lstm_size, cnn_size), b)
    sd["pre_pool_expansion_layer.bias"] = u((lstm_size,), b)
    k = 1.0 / np.sqrt(lstm_size)
    for layer in (0, 1):
        cin = lstm_size if layer == 0 else 2 * lstm_size
        for sfx in ("", "_reverse"):
            sd["lstm.weight_ih_l%d%s" % (layer, sfx)] = u((4 * lstm_size, cin), k)
            sd["lstm.weight_hh_l%d%s" % (layer, sfx)] = u((4 * lstm_size, lstm_size), k * gain)
            sd["lstm.bias_ih_l%d%s" % (layer, sfx)] = u((4 * lstm_size,), k)
            sd["lstm.bias_hh_l%d%s" % (layer, sfx)] = u((4 * lstm_size,), k)
    sd["linear.weight"] = u((5, 2 * lstm_size), 1.0 / np.sqrt(2 * lstm_size) * 24)
    sd["linear.bias"] = u((5,), 0.1)
    return sd


def synth_rl_features(B, P, D, use_dwells=False, seed=0, empty_rows=3, ragged=True):
    """Read-level feature tensors int8 [B, P, D, F] the way the featuriser + Batch.collate padding produce them:
    base 0 = no read, 1-4 ACGT, 5 deletion; quality 0-60; strand 0 / 1 (after the clip); mapQ; dwell; trailing reads
    empty (padding to the batch's maximum depth)."""
    rs = np.random.RandomState(seed)
    F = 5 if use_dwells else 4
    x = np.zeros((B, P, D, F), dtype=np.int8)
    for b in range(B):
        depth = D - (rs.randint(0, empty_rows + 1) if empty_rows else 0)
        for d in range(depth):
            lo = rs.randint(0, max(1, P // 3)) if ragged else 0
            hi = P - (rs.randint(0, max(1, P // 3)) if ragged else 0)
            n = hi - lo
            base = rs.choice([1, 2, 3, 4, 5], size=n, p=[0.23, 0.23, 0.23, 0.23, 0.08])
            x[b, lo:hi, d, 0] = base
            x[b, lo:hi, d, 1] = np.where(base == 5, 0, rs.randint(1, 55, n))
            x[b, lo:hi, d, 2] = rs.randint(0, 2)
            x[b, lo:hi, d, 3] = rs.randint(1, 61)
            if use_dwells:
                x[b, lo:hi, d, 4] = np.where(base == 5, 0, rs.randint(1, 30, n))
    return x


class LatentSpaceLSTM(torch.nn.Module):
    def __init__(self, lstm_size=128, cnn_size=128, use_dwells=False, num_classes=5):
        super().__init__()
        self.use_dwells = use_dwells
        self.lstm_size = lstm_size
        nin = 6 + 1 + (1 if use_dwells else 0)
        self.base_embedder = torch.nn.Embedding(6, 6)
        self.strand_embedder = torch.nn.Embedding(3, 6)
        rlc = torch.nn.Module()
        rlc.convs = torch.nn.Sequential(
            torch.nn.Conv1d(nin, cnn_size, kernel_size=1, padding=0), torch.nn.ReLU(), torch.nn.BatchNorm1d(cnn_size),
            torch.nn.Conv1d(cnn_size, cnn_size, kernel_size=17, padding=8), torch.nn.ReLU(), torch.nn.BatchNorm1d(cnn_size))
        rlc.expansion_layer = torch.nn.Linear(cnn_size, lstm_size)
        self.read_level_conv = rlc
        self.pre_pool_expansion_layer = torch.nn.Linear(cnn_size, lstm_size)
        self.lstm = torch.nn.LSTM(lstm_size, lstm_size, num_layers=2, bidirectional=True, batch_first=True)
        self.linear = torch.nn.Linear(2 * lstm_size, num_classes)

    def forward(self, x):
        mask = x.sum((1, -1)) != 0                                       # latent_space_lstm.py:163-165
        e = self.base_embedder(x[:, :, :, 0].long()) + self.strand_embedder(x[:, :, :, 2].long() + 1)
        q = (x[:, :, :, 1] / 25 - 1).unsqueeze(-1)
        parts = [e, q]
        if self.use_dwells:
            parts.append(x[:, :, :, 4].unsqueeze(-1))
        h = torch.cat(parts, dim=-1).permute(0, 2, 3, 1)                 # b, d, f, p
        b, d, f, p = h.shape
        h = self.read_level_conv.convs(h.flatten(0, 1)).permute(0, 2, 1)
        h = self.pre_pool_expansion_layer(h).view(b, d, p, self.lstm_size)
        h = (h * mask[..., None, None]).sum(dim=1) / mask.sum(-1)[..., None, None]      # MeanPooler
        h = self.lstm(h)[0]
        return torch.softmax(self.linear(h), dim=-1)


def build(state_dict, use_dwells=False):
    m = LatentSpaceLSTM(lstm_size=int(state_dict["lstm.weight_hh_l0"].shape[1]), use_dwells=use_dwells)
    m.load_state_dict(state_dict)
    m.eval()
    return m


def predict(model, x, threads=8):
    torch.set_num_threads(threads)
    with torch.inference_mode():
        return model(torch.from_numpy(np.asarray(x))).numpy()


# ---------------------------------------------------------------------------------------------- layer-wise reference
def _layer_lstms(model):
    """The two layers of model.lstm as single-layer bidirectional modules (same weights; torch runs a stacked LSTM
    layer by layer, so the outputs are those of the stacked module)."""
    if getattr(model, "_layers", None) is None:
        H = model.lstm.hidden_size
        layers = []
        for layer in (0, 1):
            m = torch.nn.LSTM(H if layer == 0 else 2 * H, H, num_layers=1, bidirectional=True, batch_first=True)
            m.load_state_dict({k.replace("_l%d" % layer, "_l0"): v for k, v in model.lstm.state_dict().items()
                               if "_l%d" % layer in k})
            layers.append(m.to(next(model.parameters()).dtype))
        object.__setattr__(model, "_layers", layers)           # not a submodule: keeps model.state_dict() unchanged
    return model._layers


def _lstm_layer_rounded_h(lstm, x):
    """One bidirectional layer as an explicit cell loop that feeds h back through fp16 (the recurrent product without
    h's low half); the layer's output keeps the unrounded h."""
    outs = []
    for sfx, reverse in (("_l0", False), ("_l0_reverse", True)):
        w_ih, w_hh = getattr(lstm, "weight_ih" + sfx), getattr(lstm, "weight_hh" + sfx)
        gi = x @ w_ih.T + getattr(lstm, "bias_ih" + sfx) + getattr(lstm, "bias_hh" + sfx)
        B, P, H = x.shape[0], x.shape[1], w_hh.shape[1]
        h = x.new_zeros(B, H)
        c = x.new_zeros(B, H)
        out = x.new_empty(B, P, H)
        for t in (range(P - 1, -1, -1) if reverse else range(P)):
            g = gi[:, t] + h.half().to(x.dtype) @ w_hh.T
            i, f, gg, o = g.chunk(4, -1)
            c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(gg)
            h = torch.sigmoid(o) * torch.tanh(c)
            out[:, t] = h
        outs.append(out)
    return torch.cat(outs, -1)


def stages(model, x, dtype=torch.float32, round_h=False, round_y1=False, threads=8):
    """The intermediates of LatentSpaceLSTM.forward, window by window (a P = 10 000, D = 100 window's convolution output
    alone is 0.5 GB): {"z": [B, P, H] pooled pre_pool_expansion_layer output, "h0" / "h1": [B, P, 2H] LSTM layer
    outputs, "probs": [B, P, 5]} as numpy arrays of dtype.  The arithmetic is forward's: the same mask over every feature
    column, the Linear before the mean, the same sum-then-divide pooling.  dtype runs it in float64 for a tighter
    reference; round_h / round_y1 are the ablations of ablate()."""
    import copy
    torch.set_num_threads(threads)
    m = model
    if dtype != torch.float32:
        m = copy.deepcopy(model).to(dtype)
        object.__setattr__(m, "_layers", None)
    layers = _layer_lstms(m)
    out = {"z": [], "h0": [], "h1": [], "probs": []}
    with torch.inference_mode():
        for b in range(len(x)):
            xb = torch.from_numpy(np.asarray(x[b:b + 1]))
            mask = xb.sum((1, -1)) != 0
            e = m.base_embedder(xb[:, :, :, 0].long()) + m.strand_embedder(xb[:, :, :, 2].long() + 1)
            parts = [e, (xb[:, :, :, 1].to(dtype) / 25 - 1).unsqueeze(-1)]
            if m.use_dwells:
                parts.append(xb[:, :, :, 4].to(dtype).unsqueeze(-1))
            h = torch.cat(parts, dim=-1).permute(0, 2, 3, 1)
            _, d, _, p = h.shape
            convs = m.read_level_conv.convs
            y1 = convs[2](convs[1](convs[0](h.flatten(0, 1))))
            if round_y1:
                y1 = y1.half().to(dtype)
            h = convs[5](convs[4](convs[3](y1))).permute(0, 2, 1)
            h = m.pre_pool_expansion_layer(h).view(1, d, p, m.lstm_size)
            z = (h * mask[..., None, None]).sum(dim=1) / mask.sum(-1)[..., None, None]
            if round_h:
                h0 = _lstm_layer_rounded_h(layers[0], z)
                h1 = _lstm_layer_rounded_h(layers[1], h0)
            else:
                h0 = layers[0](z)[0]
                h1 = layers[1](h0)[0]
            probs = torch.softmax(m.linear(h1), dim=-1)
            for k, v in (("z", z), ("h0", h0), ("h1", h1), ("probs", probs)):
                out[k].append(v[0].numpy())
    return {k: np.stack(v) for k, v in out.items()}


ABLATIONS = ("w_hh", "w_ih", "conv17", "h", "y1")


def ablate(state_dict, which):
    """A precision ablation: what a tensor-core kernel computes when it loses one of its three fp16 products
    (hi.hi + hi.lo + lo.hi, DESIGN §3).  Returns (state_dict, keyword arguments for stages()).
      w_hh / w_ih / conv17  the LSTM recurrent / input weights or the k = 17 convolution weights rounded to fp16 (the
                            weights' lo plane dropped)
      h                     h fed back through fp16 at every step (the recurrence's h lo plane dropped)
      y1                    the k = 17 convolution's input rounded to fp16 (the activations' lo plane dropped)"""
    sd = dict(state_dict)
    keys = {"w_hh": "lstm.weight_hh", "w_ih": "lstm.weight_ih", "conv17": "read_level_conv.convs.3.weight"}
    if which in keys:
        for k in sd:
            if k.startswith(keys[which]):
                sd[k] = sd[k].half().float()
        return sd, {}
    if which == "h":
        return sd, {"round_h": True}
    if which == "y1":
        return sd, {"round_y1": True}
    raise ValueError("unknown ablation %r (one of %s)" % (which, ", ".join(ABLATIONS)))


def featuriser_like_rl_features(B, P, D, F=5, seed=0, empty_rows=True, dwell_sat=0.07):
    """Read-level features int8 [B, P, D, F] with the properties of real windows (ReadAlignmentFeatureEncoder output
    after the wrapper's clip to >= 0 and Batch.collate padding), which synth_rl_features does not have:
      - each row holds several reads separated by >= 5 empty positions (the read matrix's row packing); some reads start
        in the first 8 positions and some end in the last 8 (the k = 17 convolution's zero padding); long reads cross
        the 128-position tiles of the convolution
      - base 1-4, deletions (base 5, quality 0), reads without qualities (quality 0 throughout), quality up to 93
      - strand 0 / 1, mapQ 0-60
      - F >= 5: column 4 holds dwells 0-127 (0 on deletions) with a fraction dwell_sat saturated at 127, the read
        matrix's clip; F = 6: column 5 the haplotype tag 0-2
      - empty rows in the middle of the window (empty_rows): a run of 4 aligned to a 4-read group of the convolution
        and a few single ones."""
    rs = np.random.RandomState(seed)
    x = np.zeros((B, P, D, F), dtype=np.int8)
    for b in range(B):
        empty = set()
        if empty_rows and D >= 12:
            g = rs.randint(1, D // 4 - 1)
            empty.update(range(4 * g, 4 * g + 4))
            empty.update(int(d) for d in rs.choice(D - 1, size=max(1, D // 25), replace=False))
        for d in range(D):
            if d in empty:
                continue
            p = rs.randint(0, 8) if rs.rand() < 0.3 else rs.randint(0, max(1, P // 4))
            while p < P:
                n = min(P - p, rs.randint(max(1, P // 20), max(2, P // 2)))
                if p + n > P - 8 and rs.rand() < 0.5:
                    n = max(1, P - p - rs.randint(0, 8))            # end in the last 8 positions
                base = rs.choice([1, 2, 3, 4, 5], size=n, p=[0.23, 0.23, 0.23, 0.23, 0.08])
                qual = np.zeros(n, dtype=np.int64) if rs.rand() < 0.1 else rs.randint(0, 94, n)
                sl = slice(p, p + n)
                x[b, sl, d, 0] = base
                x[b, sl, d, 1] = np.where(base == 5, 0, qual)
                x[b, sl, d, 2] = rs.randint(0, 2)
                x[b, sl, d, 3] = rs.randint(0, 61)
                if F >= 5:
                    dw = np.minimum(rs.exponential(12.0, n).astype(np.int64), 127)
                    dw[rs.rand(n) < dwell_sat] = 127
                    x[b, sl, d, 4] = np.where(base == 5, 0, dw)
                if F >= 6:
                    x[b, sl, d, 5] = rs.randint(0, 3)
                p += n + 5 + rs.geometric(0.05)                      # >= 5 empty positions to the next read
    return x
