"""Oracle for the model forward: the reference's GRUModel restated in plain torch (CPU fp32).

TEST INFRASTRUCTURE (see oracle/__init__.py).

Follows medaka/architectures/gru.py:46-72 (nn.GRU(F,H,2,bidirectional,batch_first)
-> nn.Linear(2H,5) -> softmax(-1)) and medaka/models.py:303-313 (predict_on_batch:
inference_mode, returns a CPU tensor).  On CPU the reference always runs fp32
(medaka/prediction.py:146-148 forces full_precision), which is the parity target.

``manual_forward`` is a second, loop-level restatement of the same arithmetic
(gate order r,z,n; n = tanh(gi_n + r*(gh_n + b_hn))) used to cross-check
intermediate tensors of the CUDA path layer by layer.
"""
import numpy as np
import torch


class GRUOracle(torch.nn.Module):
    """medaka/architectures/gru.py:13-72 without the medaka base classes."""

    def __init__(self, num_features=10, num_classes=5, gru_size=128, n_layers=2,
                 bidirectional=True):
        super().__init__()
        self.gru = torch.nn.GRU(num_features, gru_size, num_layers=n_layers,
                                bidirectional=bidirectional, batch_first=True)
        # gru.py:53-55: the head is hard-coded to 5 outputs
        self.linear = torch.nn.Linear(2 * gru_size if bidirectional else gru_size, 5)
        self.normalise = True

    def forward(self, x, return_logits=False):
        y = self.gru(x)[0]
        logits = self.linear(y)
        probs = torch.softmax(logits, dim=-1)
        if return_logits:
            return probs, logits
        return probs


def build(state_dict, num_features=10, gru_size=128, n_layers=2, bidirectional=True):
    m = GRUOracle(num_features, 5, gru_size, n_layers, bidirectional)
    m.load_state_dict({k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in state_dict.items()})
    m.eval()
    return m


def predict_on_batch(model, feats, threads=None):
    """feats float32 [B,T,F] (numpy or torch) -> (probs [B,T,5], logits [B,T,5]) numpy fp32.

    Mirrors TorchModel.predict_on_batch (medaka/models.py:303-313) on CPU.
    """
    if threads is not None:
        torch.set_num_threads(int(threads))
    x = torch.as_tensor(feats, dtype=torch.float32)
    with torch.inference_mode():
        probs, logits = model(x, return_logits=True)
    return probs.numpy(), logits.numpy()


def labels_from_probs(probs):
    """argmax as decode_consensus does it (medaka/labels.py:1063): first max wins."""
    return np.argmax(probs, -1).astype(np.uint8)


def manual_forward(state_dict, feats, gru_size=128, n_layers=2):
    """Loop-level fp32 restatement; returns dict of intermediates (numpy).

    out['h0'] / out['h1']: layer outputs [B,T,2H]; out['logits'], out['probs'].
    """
    x = torch.as_tensor(feats, dtype=torch.float32)
    B, T, _ = x.shape
    H = gru_size
    out = {}
    sd = {k: torch.as_tensor(v) for k, v in state_dict.items()}
    inp = x
    for layer in range(n_layers):
        ys = []
        for sfx in ("", "_reverse"):
            w_ih = sd["gru.weight_ih_l%d%s" % (layer, sfx)]
            w_hh = sd["gru.weight_hh_l%d%s" % (layer, sfx)]
            b_ih = sd["gru.bias_ih_l%d%s" % (layer, sfx)]
            b_hh = sd["gru.bias_hh_l%d%s" % (layer, sfx)]
            gi = inp @ w_ih.T + b_ih  # [B,T,3H]
            h = torch.zeros(B, H)
            hs = [None] * T
            order = range(T) if sfx == "" else range(T - 1, -1, -1)
            for t in order:
                gh = h @ w_hh.T + b_hh
                r = torch.sigmoid(gi[:, t, 0:H] + gh[:, 0:H])
                z = torch.sigmoid(gi[:, t, H:2 * H] + gh[:, H:2 * H])
                n = torch.tanh(gi[:, t, 2 * H:] + r * gh[:, 2 * H:])
                h = (1 - z) * n + z * h
                hs[t] = h
            ys.append(torch.stack(hs, 1))
        inp = torch.cat(ys, -1)
        out["h%d" % layer] = inp.numpy()
    logits = inp @ sd["linear.weight"].T + sd["linear.bias"]
    out["logits"] = logits.numpy()
    out["probs"] = torch.softmax(logits, -1).numpy()
    return out


# ---------------------------------------------------------------------------------------------- stage-wise reference
def _gru_direction(gi, w_hh, b_hh, reverse, round_h):
    """One direction of one layer: gi [B, T, 3H] (input part with b_ih) -> h [B, T, H].  round_h feeds h back through
    fp16 (the recurrent product without h's lo plane); the output keeps the unrounded h."""
    B, T, G = gi.shape
    H = G // 3
    h = gi.new_zeros(B, H)
    out = gi.new_empty(B, T, H)
    for t in (range(T - 1, -1, -1) if reverse else range(T)):
        hin = h.half().to(gi.dtype) if round_h else h
        gh = torch.addmm(b_hh, hin, w_hh.T)
        g = gi[:, t]
        rz = torch.sigmoid(g[:, :2 * H] + gh[:, :2 * H])
        n = torch.tanh(g[:, 2 * H:] + rz[:, :H] * gh[:, 2 * H:])
        h = n + rz[:, H:] * (h - n)               # (1 - z) n + z h
        out[:, t] = h
    return out


def stages(state_dict, feats, dtype=torch.float64, round_h=False, round_x=False, round_h0=False):
    """The intermediates of the forward, with manual_forward's arithmetic (gate order r, z, n;
    n = tanh(gi_n + r (gh_n + b_hn))), vectorised over windows and looped over T:
      h0, h1  [B, T, 2H] layer outputs (columns direction * H + unit)
      plog    [B, T, 2, 5] per-direction partial logits without the bias, h1[..., dH:(d+1)H] @ W_lin[:, dH:(d+1)H]^T:
              what the layer-1 recurrence with the fused head writes (the device's [dir][tile][T][class][16 windows])
      logits  [B, T, 5] = plog summed over directions + bias;  probs [B, T, 5]
    as numpy arrays of dtype.  round_h / round_x / round_h0 are the ablations of ablate()."""
    sd = {k: torch.as_tensor(np.asarray(v)).to(dtype) for k, v in state_dict.items()}
    x = torch.as_tensor(np.asarray(feats)).to(dtype)
    H = sd["gru.weight_hh_l0"].shape[1]
    out = {}
    inp = x.half().to(dtype) if round_x else x
    with torch.inference_mode():
        for layer in (0, 1):
            if layer == 1 and round_h0:
                inp = inp.half().to(dtype)
            ys = []
            for sfx in ("", "_reverse"):
                gi = inp @ sd["gru.weight_ih_l%d%s" % (layer, sfx)].T + sd["gru.bias_ih_l%d%s" % (layer, sfx)]
                ys.append(_gru_direction(gi, sd["gru.weight_hh_l%d%s" % (layer, sfx)],
                                         sd["gru.bias_hh_l%d%s" % (layer, sfx)], sfx == "_reverse", round_h))
            out["h%d" % layer] = torch.cat(ys, -1)
            inp = out["h%d" % layer]
        w = sd["linear.weight"]
        h1 = out["h1"]
        plog = torch.stack([h1[..., :H] @ w[:, :H].T, h1[..., H:] @ w[:, H:].T], -2)
        logits = plog.sum(-2) + sd["linear.bias"]
        out.update(plog=plog, logits=logits, probs=torch.softmax(logits, -1))
    return {k: v.numpy() for k, v in out.items()}


ABLATIONS = ("w_hh", "w_ih0", "w_ih1", "x", "h", "h0")


def ablate(state_dict, which):
    """A precision ablation: what a tensor-core kernel computes when it loses one of its three fp16 products
    (hi.hi + hi.lo + lo.hi, DESIGN §3).  Returns (state_dict, keyword arguments for stages()).
      w_hh    W_hh of both layers rounded to fp16: the recurrences without W_lo.h_hi
      w_ih0   layer-0 W_ih rounded: the fused x projection without W_lo.x_hi
      w_ih1   layer-1 W_ih rounded: the layer-1 input projection (gemm_tc_kernel) without W_lo.h0_hi
      x       the features rounded to fp16: the fused x projection without W_hi.x_lo
      h       h fed back through fp16 at every step: the recurrences without W_hi.h_lo
      h0      the layer-1 input rounded to fp16: the layer-1 input projection without W_hi.h0_lo"""
    sd = dict(state_dict)
    keys = {"w_hh": ("gru.weight_hh_l0", "gru.weight_hh_l1"), "w_ih0": ("gru.weight_ih_l0",),
            "w_ih1": ("gru.weight_ih_l1",)}
    if which in keys:
        for k in sd:
            if k.startswith(keys[which]):
                sd[k] = np.asarray(sd[k], dtype=np.float32).astype(np.float16).astype(np.float32)
        return sd, {}
    kw = {"x": "round_x", "h": "round_h", "h0": "round_h0"}
    if which in kw:
        return sd, {kw[which]: True}
    raise ValueError("unknown ablation %r (one of %s)" % (which, ", ".join(ABLATIONS)))


def featuriser_like_features(B, T, F=10, seed=0, gaps=4):
    """Features float32 [B, T, F] as the counts featuriser makes them, which synth_features (Dirichlet rows) is not:
    raw counts from synth.synth_counts through features_oracle.post_process_pileup, cut into windows of T columns.
    F = 10: one datatype, "total" normalisation; F = 20, 30, 40: two to four datatypes, "fwd_rev".  Major columns are
    one-hot-like (the true base on both strands), insertion (minor) columns sparse and small, and each window of T >= 100
    has `gaps` runs of 5-60 columns without coverage (all-zero rows)."""
    from oracle import features_oracle, synth
    if F not in (10, 20, 30, 40):
        raise ValueError("F must be 10, 20, 30 or 40")
    ndt = F // 10
    n = B * T
    # 15 reads per datatype at three and four datatypes, as at two: strand groups of a few reads would make most
    # normalised values quarters and halves, which fp16 holds exactly
    depth = 30 if ndt <= 2 else 15 * ndt
    counts, pos = synth.synth_counts(n, seed=seed, num_dtypes=ndt, mean_depth=depth, max_depth=4 * depth)
    rs = np.random.RandomState(seed + 1)
    for b in range(B):
        for _ in range(gaps if T >= 100 else 0):
            a = b * T + rs.randint(0, T)
            e = min(a + rs.randint(5, 61), n)
            while e < n and pos["minor"][e] > 0:        # a minor column takes its major column's depth: drop it too
                e += 1
            counts[a:e] = 0
    if ndt == 1:
        f, _ = features_oracle.post_process_pileup(counts, pos, "total")
    else:
        f, _ = features_oracle.post_process_pileup(counts, pos, "fwd_rev", dtypes=tuple("dt%d" % k for k in range(ndt)))
    return np.ascontiguousarray(f.reshape(B, T, F), dtype=np.float32)
