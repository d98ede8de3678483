"""Float64 target of the read-level engine's fp16 mode (LatentSpaceLSTM.set_precision("fp16"), mdk_rl_set_conv bit 2).

TEST INFRASTRUCTURE.  The arithmetic of oracle/rl_oracle.stages (LatentSpaceLSTM.forward window by window: the same
mask over every feature column, the Linear before the mean, sum-then-divide pooling) in float64, with the operands the
mode rounds to the nearest fp16 rounded here too, and the LSTM layers as explicit cell loops.
"""
import copy

import numpy as np
import torch

# The operands the fp16 mode rounds to fp16: the k = 17 convolution's weights and input y1, W_hh and the h fed back at
# every step, and at lstm_size 384, where the input projections run on the tensor cores, W_ih and the projections'
# inputs x (z for layer 0, h0 for layer 1).  At lstm_size 128 the projections stay fp32 (gemm_fp32_kernel).
FP16_OPERANDS = ("conv17", "y1", "w_hh", "h", "w_ih", "x")


def operands(lstm_size):
    return FP16_OPERANDS if lstm_size == 384 else FP16_OPERANDS[:4]


def _fp16(t):
    return t.half().to(t.dtype)


def _layer(lstm, layer, x, round_h, round_x, fed):
    """One bidirectional layer of lstm (torch gate order i, f, g, o) as an explicit cell loop.  round_h feeds h back
    through fp16, round_x rounds the input projection's input; the layer's output keeps the unrounded h.  fed
    [B, P, 2H]: the h fed back at each step is fed's previous step instead of the loop's own (c stays the loop's)."""
    if round_x:
        x = _fp16(x)
    outs = []
    for d, (sfx, reverse) in enumerate((("", False), ("_reverse", True))):
        name = "_l%d%s" % (layer, sfx)
        w_ih, w_hh = getattr(lstm, "weight_ih" + name), getattr(lstm, "weight_hh" + name)
        gi = x @ w_ih.T + getattr(lstm, "bias_ih" + name) + getattr(lstm, "bias_hh" + name)
        B, P, H = x.shape[0], x.shape[1], w_hh.shape[1]
        h = x.new_zeros(B, H)
        c = x.new_zeros(B, H)
        out = x.new_empty(B, P, H)
        for t in (range(P - 1, -1, -1) if reverse else range(P)):
            if fed is not None:
                tp = t + 1 if reverse else t - 1
                h = fed[:, tp, d * H:(d + 1) * H] if 0 <= tp < P else x.new_zeros(B, H)
            g = gi[:, t] + (_fp16(h) if round_h else h) @ w_hh.T
            i, f, gg, o = g.chunk(4, -1)
            c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(gg)
            h = torch.sigmoid(o) * torch.tanh(c)
            out[:, t] = h
        outs.append(out)
    return torch.cat(outs, -1)


def stages(model, x, keep=(), feed=None, device=None, threads=8):
    """{"z", "h0", "h1", "probs"} of an oracle/rl_oracle.LatentSpaceLSTM on int8 features x [B, P, D, F], float64, with
    the operands of operands(lstm_size) rounded to fp16 as the fp16 mode rounds them.

    keep: operands left unrounded (one of them: a single-rounding effect; all of them: the float64 forward).
    feed: {"z", "h0", "h1"} [B, P, ...] arrays of the engine's stages on the same windows.  Each LSTM layer then takes the
    fed input (z, h0) and, at every step, the fed previous h of its own output (h0, h1): the engine's fp32 values, which
    are rounded here exactly as the engine rounds them.  Free-running, an fp32-level difference in h that lands on an
    fp16 rounding boundary moves the rounded h by a whole fp16 unit, and such flips, not the arithmetic, would dominate
    a comparison over thousands of steps.
    device: where the arithmetic runs (e.g. "cuda"); the outputs are host arrays."""
    torch.set_num_threads(threads)
    dtype = torch.float64
    rnd = set(operands(model.lstm_size)) - set(keep)
    m = copy.deepcopy(model).to(dtype)
    with torch.no_grad():
        for name, p in m.named_parameters():
            if ("conv17" in rnd and name == "read_level_conv.convs.3.weight" or
                    "w_hh" in rnd and name.startswith("lstm.weight_hh") or
                    "w_ih" in rnd and name.startswith("lstm.weight_ih")):
                p.copy_(_fp16(p))
    dev = device or "cpu"
    m = m.to(dev)
    out = {"z": [], "h0": [], "h1": [], "probs": []}
    with torch.inference_mode():
        for b in range(len(x)):
            xb = torch.from_numpy(np.asarray(x[b:b + 1])).to(dev)
            mask = xb.sum((1, -1)) != 0
            e = m.base_embedder(xb[:, :, :, 0].long()) + m.strand_embedder(xb[:, :, :, 2].long() + 1)
            parts = [e, (xb[:, :, :, 1].to(dtype) / 25 - 1).unsqueeze(-1)]
            if m.use_dwells:
                parts.append(xb[:, :, :, 4].to(dtype).unsqueeze(-1))
            h = torch.cat(parts, dim=-1).permute(0, 2, 3, 1)
            _, d, _, p = h.shape
            convs = m.read_level_conv.convs
            y1 = convs[2](convs[1](convs[0](h.flatten(0, 1))))
            if "y1" in rnd:
                y1 = _fp16(y1)
            h = convs[5](convs[4](convs[3](y1))).permute(0, 2, 1)
            h = m.pre_pool_expansion_layer(h).view(1, d, p, m.lstm_size)
            z = (h * mask[..., None, None]).sum(dim=1) / mask.sum(-1)[..., None, None]
            fed = None
            if feed is not None:
                fed = {k: torch.from_numpy(np.asarray(feed[k][b:b + 1])).to(dev, dtype) for k in ("z", "h0", "h1")}
            h0 = _layer(m.lstm, 0, fed["z"] if fed else z, "h" in rnd, "x" in rnd, fed["h0"] if fed else None)
            h1 = _layer(m.lstm, 1, fed["h0"] if fed else h0, "h" in rnd, "x" in rnd, fed["h1"] if fed else None)
            probs = torch.softmax(m.linear(h1), dim=-1)
            for k, v in (("z", z), ("h0", h0), ("h1", h1), ("probs", probs)):
                out[k].append(v[0].cpu().numpy())
    return {k: np.stack(v) for k, v in out.items()}
