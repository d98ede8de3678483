"""Oracle for training the read-level LatentSpaceLSTM: float64 torch autograd on oracle/rl_oracle.py's restatement in
training mode (batch-statistics BatchNorm), with the optimizer rules of oracle/train_oracle.py.

TEST INFRASTRUCTURE (see oracle/__init__.py).  The loss is CrossEntropyLoss() over all B*P positions of the logits
(normalise = False, as the reference's run_epoch trains); the strand index is int8 strand + 1, as the engine reads it.

With an ``ablation`` the forward is restated (the k = 17 convolution as an autograd Function with its backward written
out, the LSTM per step) so that one backward term can go wrong the way a kernel bug would, while the forward's values
stay the true ones: where autograd cannot express the wrong term directly, the value comes from the true op and the
gradient from the ablated one (straight-through).  The GPU tests' bars are shown to see each of them.
"""
import numpy as np
import torch

from oracle import rl_oracle, train_oracle

ABLATIONS = ("bn1_stats_const", "bn2_stats_const", "dgrad_unflipped", "dw17_tap_shift", "pool_over_D",
             "lstm_h_t_in_dwhh", "lstm_no_forget_carry")


def build(state_dict, use_dwells=False, dtype=torch.float64):
    """rl_oracle.LatentSpaceLSTM in training mode carrying state_dict (parameters and buffers)."""
    H = int(np.shape(state_dict["lstm.weight_hh_l0"])[1])
    m = rl_oracle.LatentSpaceLSTM(lstm_size=H, use_dwells=use_dwells).to(dtype)
    m.load_state_dict({k: torch.as_tensor(np.asarray(v)).to(dtype if np.asarray(v).dtype.kind == "f" else torch.int64)
                       for k, v in state_dict.items()})
    m.train()
    return m


def logits(m, x, ablation=None, restated=None, flip=None):
    """LatentSpaceLSTM.forward without the softmax, in the model's dtype.  restated (default: with an ablation) runs
    the restatement that carries the ablations; without one it equals the modules' forward."""
    if ablation is not None and ablation not in ABLATIONS:
        raise ValueError("unknown ablation %r" % ablation)
    restated = ablation is not None or flip is not None if restated is None else restated
    x = x if torch.is_tensor(x) else torch.as_tensor(np.asarray(x, np.int8))
    dtype = m.linear.weight.dtype
    mask = x.sum((1, -1)) != 0
    e = m.base_embedder(x[:, :, :, 0].long()) + m.strand_embedder(x[:, :, :, 2].long() + 1)
    parts = [e, (x[:, :, :, 1].to(dtype) / 25 - 1).unsqueeze(-1)]
    if m.use_dwells:
        parts.append(x[:, :, :, 4].to(dtype).unsqueeze(-1))
    h = torch.cat(parts, dim=-1).permute(0, 2, 3, 1)
    b, d, _, p = h.shape
    if restated:
        h = _convs(m.read_level_conv.convs, h.flatten(0, 1), ablation, flip).permute(0, 2, 1)
    else:
        h = m.read_level_conv.convs(h.flatten(0, 1)).permute(0, 2, 1)
    h = m.pre_pool_expansion_layer(h).view(b, d, p, m.lstm_size)
    pooled = (h * mask[..., None, None]).sum(dim=1)
    h = pooled / mask.sum(-1)[..., None, None]
    if ablation == "pool_over_D":                 # the backward of the mean divides by D, not by the reads
        h = _straight_through(h, pooled / d)
    return m.linear(lstm(m.lstm, h, ablation) if restated else m.lstm(h)[0])


def _straight_through(value, grad_from):
    """value's value, grad_from's gradient"""
    return value.detach() + (grad_from - grad_from.detach())


def _batch_norm(bn, h, ablation):
    """training-mode BatchNorm1d (running statistics move); stats_const: the batch mean and variance are constants in
    the backward"""
    y = bn(h)
    if ablation is None:
        return y
    mean = h.mean((0, 2), keepdim=True).detach()
    var = h.var((0, 2), unbiased=False, keepdim=True).detach()
    const = (h - mean) / torch.sqrt(var + bn.eps) * bn.weight[:, None] + bn.bias[:, None]
    return _straight_through(y, const)


class _Conv17(torch.autograd.Function):
    """Conv1d(k = 17, padding 8) with its backward written out: dy1 is the convolution of dout with the weights
    transposed and the taps flipped, dW17[t] pairs dout with y1 shifted by t - 8."""

    @staticmethod
    def forward(ctx, y1, w, bias, ablation):
        ctx.save_for_backward(y1, w)
        ctx.ablation = ablation
        return torch.nn.functional.conv1d(y1, w, bias, padding=8)

    @staticmethod
    def backward(ctx, dout):
        y1, w = ctx.saved_tensors
        k, P = w.shape[-1], y1.shape[-1]
        wt = w.transpose(0, 1)
        dy1 = torch.nn.functional.conv1d(dout, wt if ctx.ablation == "dgrad_unflipped" else wt.flip(-1), padding=8)
        lo = 7 if ctx.ablation == "dw17_tap_shift" else 8            # tap t pairs with y1[p + t - lo]
        ypad = torch.nn.functional.pad(y1, (lo, k - 1 - lo))
        dw = torch.stack([torch.einsum("nop,nip->oi", dout, ypad[:, :, t:t + P]) for t in range(k)], -1)
        return dy1, dw, dout.sum((0, 2)), None


def _relu(v, flip):
    """ReLU; flip (a bool tensor like v, or None): elements whose derivative takes the other side of zero"""
    r = torch.relu(v)
    if flip is None:
        return r
    g = ((v > 0) ^ flip).to(v.dtype)
    return _straight_through(r, v * g)


def _convs(convs, h, ablation, flip=None):
    """read_level_conv.convs: conv1, ReLU, BN1, conv17, ReLU, BN2"""
    flip = flip or {}
    h = _batch_norm(convs[2], _relu(convs[0](h), flip.get("conv1")), ablation if ablation == "bn1_stats_const" else None)
    h = _Conv17.apply(h, convs[3].weight, convs[3].bias, ablation)
    return _batch_norm(convs[5], _relu(h, flip.get("conv17")), ablation if ablation == "bn2_stats_const" else None)


def relu_margins(m, x):
    """{'conv1', 'conv17': |pre-activation| / sum |w x| + |b| per element [B*D, C, P]} of a forward of m (which moves
    its running statistics): how far each ReLU's input lies from zero relative to what fp32 rounding can move it"""
    convs, seen = m.read_level_conv.convs, []
    hooks = [convs[i].register_forward_hook(lambda mod, inp, out: seen.append((mod, inp[0].detach(), out.detach())))
             for i in (0, 3)]
    try:
        with torch.no_grad():
            logits(m, x)
    finally:
        for h in hooks:
            h.remove()
    out = {}
    for name, (mod, inp, v) in zip(("conv1", "conv17"), seen):
        s = torch.nn.functional.conv1d(inp.abs(), mod.weight.abs(), mod.bias.abs(), padding=mod.padding)
        out[name] = v.abs() / s
    return out


def lstm(mod, h, ablation=None):
    """torch.nn.LSTM (2 layers, bidirectional, batch_first, gates i, f, g, o) restated per step:
    lstm_h_t_in_dwhh      dW_hh pairs the gate gradients with h_t instead of h_{t-1}
    lstm_no_forget_carry  the cell gradient carried to c_{t-1} is dc instead of dc f"""
    B, P, H = h.shape[0], h.shape[1], mod.hidden_size
    for layer in range(mod.num_layers):
        outs = []
        if ablation == "lstm_h_t_in_dwhh":
            with torch.no_grad():
                h_true = _lstm_layer(mod, h, layer, None)
        for d, sfx in enumerate(("", "_reverse")):
            w_ih, w_hh, b_ih, b_hh = (getattr(mod, "%s_l%d%s" % (k, layer, sfx))
                                      for k in ("weight_ih", "weight_hh", "bias_ih", "bias_hh"))
            gi = h @ w_ih.T + b_ih + b_hh
            hp, c = h.new_zeros(B, H), h.new_zeros(B, H)
            out = [None] * P
            for t in (range(P - 1, -1, -1) if d else range(P)):
                if ablation == "lstm_h_t_in_dwhh":
                    ht = h_true[:, t, d * H:(d + 1) * H]
                    g = gi[:, t] + hp @ w_hh.detach().T + (ht @ w_hh.T - (ht @ w_hh.T).detach())
                else:
                    g = gi[:, t] + hp @ w_hh.T
                i, f = torch.sigmoid(g[:, :H]), torch.sigmoid(g[:, H:2 * H])
                gg, o = torch.tanh(g[:, 2 * H:3 * H]), torch.sigmoid(g[:, 3 * H:])
                cn = f * c + i * gg
                if ablation == "lstm_no_forget_carry":         # value unchanged, d c_{t-1} = dc
                    cn = cn + (c - c.detach()) * (1 - f.detach())
                c = cn
                hp = o * torch.tanh(c)
                out[t] = hp
            outs.append(torch.stack(out, 1))
        h = torch.cat(outs, -1)
    return h


def _lstm_layer(mod, h, layer, ablation):
    """one layer of lstm(): its [B, P, 2H] output"""
    one = torch.nn.LSTM(mod.input_size if layer == 0 else 2 * mod.hidden_size, mod.hidden_size, num_layers=1,
                        bidirectional=True, batch_first=True).to(h.dtype)
    for k in ("weight_ih", "weight_hh", "bias_ih", "bias_hh"):
        for sfx in ("", "_reverse"):
            getattr(one, "%s_l0%s" % (k, sfx)).data.copy_(getattr(mod, "%s_l%d%s" % (k, layer, sfx)))
    return lstm(one, h, ablation)


def loss_and_grads(m, x, labels, ablation=None, restated=None, flip=None):
    """(loss, {parameter: float64 gradient}, n_correct) of one training forward and backward of model m (which moves
    its running statistics, as a training forward does).  Parameters without a gradient are left out.  ablation: one
    of ABLATIONS or None:
      bn1_stats_const       BN1's batch mean and variance treated as constants in the backward
      bn2_stats_const       the same for BN2
      dgrad_unflipped       dy1 from the conv17 weights transposed, the taps not flipped
      dw17_tap_shift        dW17 tap t paired with y1 shifted by t - 7 instead of t - 8
      pool_over_D           the masked mean's backward divides by D instead of the non-empty reads
      lstm_h_t_in_dwhh      dW_hh against h_t instead of h_{t-1}
      lstm_no_forget_carry  the cell gradient carried to c_{t-1} is dc instead of dc f
    restated: as logits().  flip: {'conv1' | 'conv17': bool [B*D, C, P]}, ReLU derivatives taken on the other side of
    zero (values unchanged), for pre-activations fp32 cannot place (relu_margins)."""
    m.zero_grad()
    lg = logits(m, x, ablation, restated, flip)
    y = torch.as_tensor(np.asarray(labels), dtype=torch.int64)
    loss = torch.nn.CrossEntropyLoss()(lg.flatten(0, 1), y.flatten())
    loss.backward()
    grads = {k: p.grad.detach().double().numpy().copy() for k, p in m.named_parameters() if p.grad is not None}
    return float(loss.detach()), grads, int((lg.detach().argmax(-1) == y).sum())


def train_steps(state_dict, batches, use_dwells=False, steps_per_epoch=1000, lr=0.001):
    """Three (or len(batches)) steps of run_training's defaults: ClipGrad, RMSprop (alpha 0.9, eps 1e-7),
    linear_warmup_cosine_decay; a non-finite gradient norm skips the update.  Returns (per-step [loss, norm, threshold,
    lr, n_correct], step-1 gradients, final state dict as float64 arrays)."""
    from medaka_b200 import training
    m = build(state_dict, use_dwells)
    names = [k for k, _ in m.named_parameters()]
    opt = train_oracle.Optimizer("rmsprop", lr=lr, alpha=0.9, eps=1e-7)
    clip = training.ClipGrad()
    sched = training.linear_warmup_cosine_decay()(lr, steps_per_epoch, 1, 0)
    rows, g0 = [], None
    for s, (x, y) in enumerate(batches):
        loss, grads, correct = loss_and_grads(m, x, y)
        if g0 is None:
            g0 = grads
        keys = [k for k in names if k in grads]
        flat = train_oracle.flatten(grads, keys)
        norm = float(np.sqrt((flat ** 2).sum()))
        threshold = clip.max_norm()
        step_lr = sched.get_last_lr()[0]
        if np.isfinite(norm):
            flat = flat * train_oracle.clip_coef(norm, threshold)
            p = train_oracle.flatten({k: v.detach().numpy() for k, v in m.named_parameters()}, keys)
            newp = train_oracle.unflatten(opt.step(p, flat, lr=step_lr), grads, keys)
            with torch.no_grad():
                for k, v in m.named_parameters():
                    if k in newp:
                        v.copy_(torch.from_numpy(newp[k]))
        clip.record(norm)
        sched.step()
        rows.append([loss, norm, threshold, step_lr, correct])
    sd = {k: v.detach().double().numpy() if v.is_floating_point() else v.numpy() for k, v in m.state_dict().items()}
    return np.array(rows), g0, sd
