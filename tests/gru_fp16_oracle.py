"""Float64 target of the consensus engine's fp16 mode (GRUModel.set_precision("fp16"), MDK_PREC_FP16).

TEST INFRASTRUCTURE.  The arithmetic of oracle/gru_oracle.stages (gate order r, z, n; n = tanh(gi_n + r (gh_n + b_hn)))
in float64, with the operands the mode rounds to fp16 rounded here exactly as the kernels round them.  The tensor-core
weights are rounded after the exp2 gate scale is folded in (gru_pack.cuh: hi = fp16(w * gate_scale(gate)) in fp32), so
the weight a product sees is fp16(s w) / s, not fp16(w): the two differ by as much as the effects the bars resolve.
"""
import numpy as np
import torch

from oracle import gru_oracle

# common.cuh GATE_SCALE_RZ, GATE_SCALE_N (fp32)
GATE_SCALE = (np.float32(-1.4426950408889634), np.float32(-1.4426950408889634), np.float32(2.8853900817779268))

# The operands the fp16 mode rounds to fp16: W_hh of both layers and the h fed back at every step (the recurrences),
# the layer-1 projection's W_ih and its input h0 (gemm_fp16_kernel, gemm256_fp16_kernel), and at gru_size 128 with
# F <= 16, where layer 0's projection is fused into the recurrence's MMAs, W_ih0 and the features x.  The CUDA-core
# layer-0 projection (F > 16 at 128, every F at 256) stays fp32.
FP16_OPERANDS = ("w_hh", "h", "w_ih1", "h0", "w_ih0", "x")


def operands(gru_size, F):
    return FP16_OPERANDS if gru_size == 128 and F <= 16 else FP16_OPERANDS[:4]


def round_weight(w):
    """A [3H, K] weight as the fp16 mode's product sees it: fp16(s w) / s per gate, s the gate's exp2 scale (fp32)."""
    w = np.asarray(w, dtype=np.float32)
    H = w.shape[0] // 3
    s = np.repeat(np.array(GATE_SCALE, dtype=np.float32), H)[:, None]
    hi = (w * s).astype(np.float16)
    return hi.astype(np.float64) / s.astype(np.float64)


def _fp16(t):
    return t.half().to(t.dtype)


def _direction(gi, w_hh, b_hh, reverse, round_h, fed):
    """One direction of one layer: gi [B, T, 3H] -> h [B, T, H].  round_h feeds h back through fp16; fed [B, T, H]: the
    h fed back at each step (product and z h term) is fed's previous step instead of the loop's own."""
    B, T, G = gi.shape
    H = G // 3
    h = gi.new_zeros(B, H)
    out = gi.new_empty(B, T, H)
    for t in (range(T - 1, -1, -1) if reverse else range(T)):
        if fed is not None:
            tp = t + 1 if reverse else t - 1
            h = fed[:, tp] if 0 <= tp < T else gi.new_zeros(B, H)
        gh = torch.addmm(b_hh, _fp16(h) if round_h else h, w_hh.T)
        g = gi[:, t]
        rz = torch.sigmoid(g[:, :2 * H] + gh[:, :2 * H])
        n = torch.tanh(g[:, 2 * H:] + rz[:, :H] * gh[:, 2 * H:])
        h = n + rz[:, H:] * (h - n)
        out[:, t] = h
    return out


def stages(state_dict, feats, keep=(), feed=None, device=None):
    """{"h0", "h1", "plog", "logits", "probs"} (gru_oracle.stages' layouts) of the fp16 mode in float64, host arrays.

    keep: operands left unrounded (one of them: a single-rounding effect; all of them: the float64 forward, equal to
    gru_oracle.stages).
    feed: {"h0", "h1"} [B, T, 2H] arrays of the engine's layer outputs on the same windows.  Each recurrence then takes,
    at every step, the fed previous h of its own output, and layer 1 takes the fed h0 as its input; the engine's fp32
    values are rounded here exactly as the engine rounds them.  Free-running over 10 000 steps, an fp32-level difference
    in h that lands on an fp16 rounding boundary moves the rounded h by a whole fp16 unit, and such flips, not the
    arithmetic, would dominate any comparison.
    device: where the arithmetic runs (e.g. "cuda")."""
    dt = torch.float64
    dev = device or "cpu"
    sd = {k: np.asarray(v, dtype=np.float32) for k, v in state_dict.items()}
    H = sd["gru.weight_hh_l0"].shape[1]
    F = np.asarray(feats).shape[-1]
    unknown = set(keep) - set(FP16_OPERANDS)
    if unknown:
        raise ValueError("unknown operands %s" % sorted(unknown))
    rnd = set(operands(H, F)) - set(keep)

    def weight(name, rounded):
        w = round_weight(sd[name]) if rounded else sd[name]
        return torch.as_tensor(np.asarray(w, dtype=np.float64), device=dev)

    def vec(name):
        return torch.as_tensor(sd[name].astype(np.float64), device=dev)

    fed = None
    if feed is not None:
        fed = {k: torch.as_tensor(np.asarray(feed[k]), device=dev).to(dt) for k in ("h0", "h1")}
    x = torch.as_tensor(np.asarray(feats), device=dev).to(dt)
    out = {}
    with torch.inference_mode():
        for layer in (0, 1):
            if layer == 0:
                inp = _fp16(x) if "x" in rnd else x
            else:
                inp = fed["h0"] if fed is not None else out["h0"]
                inp = _fp16(inp) if "h0" in rnd else inp
            ys = []
            for d, sfx in enumerate(("", "_reverse")):
                name = "_l%d%s" % (layer, sfx)
                w_ih = weight("gru.weight_ih" + name, "w_ih%d" % layer in rnd)
                w_hh = weight("gru.weight_hh" + name, "w_hh" in rnd)
                gi = inp @ w_ih.T + vec("gru.bias_ih" + name)
                own = fed["h%d" % layer][..., d * H:(d + 1) * H] if fed is not None else None
                ys.append(_direction(gi, w_hh, vec("gru.bias_hh" + name), d == 1, "h" in rnd, own))
            out["h%d" % layer] = torch.cat(ys, -1)
        w = torch.as_tensor(sd["linear.weight"].astype(np.float64), device=dev)
        h1 = out["h1"]
        plog = torch.stack([h1[..., :H] @ w[:, :H].T, h1[..., H:] @ w[:, H:].T], -2)
        logits = plog.sum(-2) + vec("linear.bias")
        out.update(plog=plog, logits=logits, probs=torch.softmax(logits, -1))
    return {k: v.cpu().numpy() for k, v in out.items()}


def float64(state_dict, feats):
    """The float64 forward (nothing rounded): gru_oracle.stages."""
    return gru_oracle.stages(state_dict, feats)
