"""Oracle for training the read-level LatentSpaceLSTM: float64 torch autograd on oracle/rl_oracle.py's restatement in
training mode (batch-statistics BatchNorm), with the optimizer rules of oracle/train_oracle.py.

TEST INFRASTRUCTURE (see oracle/__init__.py).  The loss is CrossEntropyLoss() over all B*P positions of the logits
(normalise = False, as the reference's run_epoch trains); the strand index is int8 strand + 1, as the engine reads it.
"""
import numpy as np
import torch

from oracle import rl_oracle, train_oracle


def build(state_dict, use_dwells=False, dtype=torch.float64):
    """rl_oracle.LatentSpaceLSTM in training mode carrying state_dict (parameters and buffers)."""
    H = int(np.shape(state_dict["lstm.weight_hh_l0"])[1])
    m = rl_oracle.LatentSpaceLSTM(lstm_size=H, use_dwells=use_dwells).to(dtype)
    m.load_state_dict({k: torch.as_tensor(np.asarray(v)).to(dtype if np.asarray(v).dtype.kind == "f" else torch.int64)
                       for k, v in state_dict.items()})
    m.train()
    return m


def logits(m, x):
    """LatentSpaceLSTM.forward without the softmax, in the model's dtype."""
    x = x if torch.is_tensor(x) else torch.as_tensor(np.asarray(x, np.int8))
    dtype = m.linear.weight.dtype
    mask = x.sum((1, -1)) != 0
    e = m.base_embedder(x[:, :, :, 0].long()) + m.strand_embedder(x[:, :, :, 2].long() + 1)
    parts = [e, (x[:, :, :, 1].to(dtype) / 25 - 1).unsqueeze(-1)]
    if m.use_dwells:
        parts.append(x[:, :, :, 4].to(dtype).unsqueeze(-1))
    h = torch.cat(parts, dim=-1).permute(0, 2, 3, 1)
    b, d, _, p = h.shape
    h = m.read_level_conv.convs(h.flatten(0, 1)).permute(0, 2, 1)
    h = m.pre_pool_expansion_layer(h).view(b, d, p, m.lstm_size)
    h = (h * mask[..., None, None]).sum(dim=1) / mask.sum(-1)[..., None, None]
    return m.linear(m.lstm(h)[0])


def loss_and_grads(m, x, labels):
    """(loss, {parameter: float64 gradient}, n_correct) of one training forward and backward of model m (which moves
    its running statistics, as a training forward does).  Parameters without a gradient are left out."""
    m.zero_grad()
    lg = logits(m, x)
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
