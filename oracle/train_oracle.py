"""Oracle for training the consensus GRU: float64 loss and gradients by explicit BPTT, the four optimizer rules, and
ablations that each drop one term of the backward pass.

TEST INFRASTRUCTURE (see oracle/__init__.py).

The forward is gru_oracle.manual_forward's arithmetic (gate order r, z, n; n = tanh(gi_n + r (W_hn h + b_hn)));
the loss is CrossEntropyLoss() (mean over B*T positions) of the logits, which is what the reference's run_epoch trains
(it sets model.normalise = False).  The backward pass is written out term by term, so that ``ablate`` can remove one
term and the GPU tests can show their bars are tight enough to see it.
"""
import numpy as np
import torch

ABLATIONS = ("r_factor", "dgh_is_dgi", "h_t_in_dwhh", "no_z_carry", "bhn_outside_r", "no_dx1")


def _t(a):
    return torch.as_tensor(np.asarray(a), dtype=torch.float64)


def loss_and_grads(state_dict, feats, labels, ablation=None):
    """(loss, grads {state-dict key: float64 array}, logits [B, T, 5]) of CrossEntropyLoss over all B*T positions.
    ablation: one of ABLATIONS or None:
      r_factor       dr without the r (1 - r) factor
      dgh_is_dgi     the hidden-side gate gradient's n third is dn instead of dn r (dW_hh, db_hh and the carry)
      h_t_in_dwhh    dW_hh against h_t instead of h_{t-1}
      no_z_carry     the carry into h_{t-1} without dh z
      bhn_outside_r  b_hn treated as outside r: dr from W_hn h_{t-1} alone, db_hh_n = sum dn
      no_dx1         no gradient from layer 1 into layer 0"""
    if ablation is not None and ablation not in ABLATIONS:
        raise ValueError("unknown ablation %r" % ablation)
    sd = {k: _t(v) for k, v in state_dict.items()}
    x = _t(feats)
    y = torch.as_tensor(np.asarray(labels), dtype=torch.int64)
    B, T, _ = x.shape
    H = sd["gru.weight_hh_l0"].shape[1]
    cache, inp = [], x
    for layer in (0, 1):
        outs, lc = [], []
        for d, sfx in enumerate(("", "_reverse")):
            w_ih, w_hh = sd["gru.weight_ih_l%d%s" % (layer, sfx)], sd["gru.weight_hh_l%d%s" % (layer, sfx)]
            b_ih, b_hh = sd["gru.bias_ih_l%d%s" % (layer, sfx)], sd["gru.bias_hh_l%d%s" % (layer, sfx)]
            gi = inp @ w_ih.T + b_ih
            h = x.new_zeros(B, H)
            r_, z_, n_, ghn_, hp_, ho_ = (x.new_zeros(B, T, H) for _ in range(6))
            for t in (range(T - 1, -1, -1) if d else range(T)):
                gh = h @ w_hh.T + b_hh
                r = torch.sigmoid(gi[:, t, :H] + gh[:, :H])
                z = torch.sigmoid(gi[:, t, H:2 * H] + gh[:, H:2 * H])
                n = torch.tanh(gi[:, t, 2 * H:] + r * gh[:, 2 * H:])
                hp_[:, t] = h
                h = (1 - z) * n + z * h
                r_[:, t], z_[:, t], n_[:, t], ghn_[:, t], ho_[:, t] = r, z, n, gh[:, 2 * H:], h
            outs.append(ho_)
            lc.append(dict(r=r_, z=z_, n=n_, ghn=ghn_, hp=hp_, h=ho_, w_hh=w_hh, b_hn=b_hh[2 * H:]))
        cache.append((inp, lc))
        inp = torch.cat(outs, -1)
    h1 = inp
    logits = h1 @ sd["linear.weight"].T + sd["linear.bias"]
    logp = torch.log_softmax(logits, -1)
    P = B * T
    loss = -logp.gather(-1, y[..., None]).sum() / P
    dlogits = (torch.softmax(logits, -1) - torch.nn.functional.one_hot(y, 5).to(torch.float64)) / P
    grads = {"linear.weight": torch.einsum("btc,btk->ck", dlogits, h1), "linear.bias": dlogits.sum((0, 1))}
    dh_out = dlogits @ sd["linear.weight"]
    for layer in (1, 0):
        inp, lc = cache[layer]
        dinp = torch.zeros_like(inp)
        for d, sfx in enumerate(("", "_reverse")):
            c = lc[d]
            dho = dh_out[..., d * H:(d + 1) * H]
            carry = x.new_zeros(B, H)
            dgi = x.new_zeros(B, T, 3 * H)
            dgh = x.new_zeros(B, T, 3 * H)
            w_hh = c["w_hh"]
            for t in (range(T) if d else range(T - 1, -1, -1)):
                r, z, n, ghn, hp = c["r"][:, t], c["z"][:, t], c["n"][:, t], c["ghn"][:, t], c["hp"][:, t]
                if ablation == "bhn_outside_r":
                    ghn = ghn - c["b_hn"]
                dh = dho[:, t] + carry
                dn = dh * (1 - z) * (1 - n * n)
                dz = dh * (hp - n) * z * (1 - z)
                dr = dn * ghn if ablation == "r_factor" else dn * ghn * r * (1 - r)
                dgi[:, t] = torch.cat([dr, dz, dn], -1)
                dgh[:, t] = torch.cat([dr, dz, dn if ablation == "dgh_is_dgi" else dn * r], -1)
                carry = dgh[:, t] @ w_hh
                if ablation != "no_z_carry":
                    carry = carry + dh * z
            hx = c["h"] if ablation == "h_t_in_dwhh" else c["hp"]
            grads["gru.weight_ih_l%d%s" % (layer, sfx)] = torch.einsum("btg,btk->gk", dgi, inp)
            grads["gru.bias_ih_l%d%s" % (layer, sfx)] = dgi.sum((0, 1))
            grads["gru.weight_hh_l%d%s" % (layer, sfx)] = torch.einsum("btg,btk->gk", dgh, hx)
            bhh = dgh.sum((0, 1))
            if ablation == "bhn_outside_r":
                bhh[2 * H:] = dgi[..., 2 * H:].sum((0, 1))
            grads["gru.bias_hh_l%d%s" % (layer, sfx)] = bhh
            dinp = dinp + dgi @ sd["gru.weight_ih_l%d%s" % (layer, sfx)]
        dh_out = torch.zeros_like(dinp) if ablation == "no_dx1" else dinp
    return float(loss), {k: grads[k].numpy() for k in state_dict}, logits.numpy()


def loss_and_grads_chunked(state_dict, feats, labels, windows=10):
    """loss_and_grads over slices of ``windows`` windows at a time, so that a training batch's activations never exist
    at once (100 x 10 000 columns at gru_size 256 would hold over 100 GB of float64 activations).  The windows are
    independent, and the loss is a mean over all B*T positions: each slice's loss and gradients are weighted by its
    share of the positions and added up.  Returns (loss, grads, logits [B, T, 5]) as loss_and_grads does.

    At 100 x 10 000 on 8 CPU cores it took 299 s at gru_size 256 and 177 s at gru_size 128 (349 s and 234 s on
    another 8-core host), with a peak of 9.8 GB at the default 10 windows per slice."""
    feats, labels = np.asarray(feats), np.asarray(labels)
    B, T = labels.shape
    loss, grads, logits = 0.0, {}, np.empty((B, T, 5))
    for b0 in range(0, B, windows):
        b1 = min(B, b0 + windows)
        share = (b1 - b0) / B
        l_, g, logits[b0:b1] = loss_and_grads(state_dict, feats[b0:b1], labels[b0:b1])
        loss += share * l_
        for k, v in g.items():
            grads[k] = grads.get(k, 0.0) + share * v
    return loss, grads, logits


def autograd_loss_and_grads(state_dict, feats, labels):
    """The same loss and gradients from torch autograd on gru_oracle.GRUOracle in float64."""
    from oracle import gru_oracle
    H = np.asarray(state_dict["gru.weight_hh_l0"]).shape[1]
    F = np.asarray(state_dict["gru.weight_ih_l0"]).shape[1]
    m = gru_oracle.GRUOracle(num_features=F, gru_size=H).double()
    m.load_state_dict({k: _t(v) for k, v in state_dict.items()})
    x = _t(feats)
    y = torch.as_tensor(np.asarray(labels), dtype=torch.int64)
    _, logits = m(x, return_logits=True)
    loss = torch.nn.CrossEntropyLoss()(logits.flatten(0, 1), y.flatten())
    loss.backward()
    sdp = dict(m.named_parameters())
    return float(loss), {k: sdp[k].grad.numpy() for k in state_dict}


# ---------------------------------------------------------------------------------------------- optimizer rules
class Optimizer(object):
    """torch.optim's update rules (RMSprop, Adam, NAdam, SGD; single-tensor form) in float64 on flat arrays."""

    def __init__(self, kind, **args):
        self.kind, self.args, self.t, self.mu_product = kind, args, 0, 1.0
        self.s1 = self.s2 = None

    def step(self, p, g, lr=None):
        a = self.args
        lr = a["lr"] if lr is None else lr
        p, g = np.asarray(p, np.float64).copy(), np.asarray(g, np.float64).copy()
        if self.s1 is None:
            self.s1, self.s2 = np.zeros_like(p), np.zeros_like(p)
        self.t += 1
        t = self.t
        if a.get("weight_decay", 0.0):
            g = g + a["weight_decay"] * p
        if self.kind == "rmsprop":
            self.s1 = self.s1 * a["alpha"] + (1 - a["alpha"]) * g * g
            avg = np.sqrt(self.s1) + a["eps"]
            if a.get("momentum", 0.0) > 0:
                self.s2 = self.s2 * a["momentum"] + g / avg
                return p - lr * self.s2
            return p - lr * g / avg
        if self.kind in ("adam", "nadam"):
            b1, b2 = a["betas"]
            self.s1 = self.s1 + (g - self.s1) * (1 - b1)
            self.s2 = self.s2 * b2 + (1 - b2) * g * g
            bc2 = 1 - b2 ** t
            if self.kind == "adam":
                denom = np.sqrt(self.s2) / np.sqrt(bc2) + a["eps"]
                return p - lr / (1 - b1 ** t) * self.s1 / denom
            md = a.get("momentum_decay", 0.004)
            mu = b1 * (1 - 0.5 * 0.96 ** (t * md))
            mu_next = b1 * (1 - 0.5 * 0.96 ** ((t + 1) * md))
            # torch keeps the product in a float32 scalar tensor
            self.mu_product = float(np.float32(self.mu_product) * np.float32(mu))
            denom = np.sqrt(self.s2 / bc2) + a["eps"]
            p = p - lr * (1 - mu) / (1 - self.mu_product) * g / denom
            return p - lr * mu_next / (1 - self.mu_product * mu_next) * self.s1 / denom
        if self.kind == "sgd":
            m = a.get("momentum", 0.0)
            if m:
                self.s1 = g.copy() if t == 1 else self.s1 * m + (1 - a.get("dampening", 0.0)) * g
                g = g + m * self.s1 if a.get("nesterov", False) else self.s1
            return p - lr * g
        raise ValueError(self.kind)


def clip_coef(norm, max_norm):
    """clip_grad_norm_'s scale: max_norm / (norm + 1e-6) when below 1, else 1"""
    c = max_norm / (norm + 1e-6)
    return c if c < 1 else 1.0


def flatten(sd, keys):
    return np.concatenate([np.asarray(sd[k], np.float64).ravel() for k in keys])


def unflatten(flat, like, keys):
    out, o = {}, 0
    for k in keys:
        n = np.asarray(like[k]).size
        out[k] = flat[o:o + n].reshape(np.asarray(like[k]).shape)
        o += n
    return out
