"""Training of the consensus GRU at the shape `medaka train` runs by default: 100 windows x 10 000 columns, F = 10, at
gru_size 256 (the model it builds) and 128.  tests/test_training_gpu.py checks gradients on batches of at most
8 x 10 000; this shape takes paths those never reach: the BPTT kernel at 2 windows per CTA (and, forced, at 1, 4 and
8, with a ragged last CTA at gru_size 256), and split-M reductions whose fp32 partial sums each run over tens of
thousands of rows.

The oracle is the float64 BPTT of oracle/train_oracle.py over slices of windows (loss_and_grads_chunked); it takes a
few minutes of CPU per width.  Next to it runs torch's own fp32 training step on the same batch (nn.GRU + nn.Linear +
CrossEntropyLoss on cuDNN, TF32 off: the arithmetic of the reference's training loop), and the trainer's worst
per-tensor error may not exceed twice torch's.  Argmax-correct counts equal the oracle's except on positions whose
float64 top-two logit margin is below MARGIN, where fp32 may pick either class.  Measured values are in DESIGN.md's
training section ("train-prod" lines).
"""
import functools
import os
import time

import numpy as np
import pytest

from oracle import gru_oracle, synth, train_oracle
from tests.test_training_gpu import GRAD_BAR, LOSS_BAR, _case, _trainer, grad_errors

F, B, T = 10, 100, 10000
# float64 top-two logit margin below which fp32 may pick either class: 10x the largest logit error measured at either
# width on the production batch
MARGIN = 4e-6


@functools.lru_cache(maxsize=None)
def production_batch(H):
    """(state dict, features, labels) at the production shape.  Features as the counts featuriser makes them; at
    gru_size 256 each column's label is its majority class (*ACGT from dD, aA, cC, gG, tT), 2 % of them replaced by
    uniform draws, which gives the gradient sums a strong signal; at 128 the labels are uniform."""
    x = gru_oracle.featuriser_like_features(B, T, F, seed=5)
    rs = np.random.RandomState(6)
    if H == 256:
        votes = np.stack([x[..., 8] + x[..., 9]] + [x[..., c] + x[..., c + 4] for c in range(4)], -1)
        y = np.where(rs.uniform(size=(B, T)) < 0.02, rs.randint(0, 5, size=(B, T)), votes.argmax(-1))
    else:
        y = rs.randint(0, 5, size=(B, T))
    return synth.synth_state_dict(0, num_features=F, gru_size=H), x, y


def expected_windows(nb_sm, B_):
    """The BPTT schedule the trainer documents: the fewest windows per CTA (1, 2, 4) whose CTAs of both directions fit
    one wave, else 8"""
    for nb in (1, 2, 4):
        if -(-B_ // nb) * 2 <= nb_sm:
            return nb
    return 8


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def torch_fp32_grads(sd, x, y, H):
    """Loss and gradients of torch's fp32 training step on the GPU (tools/train_bench.py's setup, TF32 off)."""
    import torch
    flags = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        dev = torch.device("cuda")
        gru = torch.nn.GRU(x.shape[2], H, num_layers=2, bidirectional=True, batch_first=True).to(dev)
        lin = torch.nn.Linear(2 * H, 5).to(dev)
        gru.load_state_dict({k[4:]: torch.from_numpy(v) for k, v in sd.items() if k.startswith("gru.")})
        lin.load_state_dict({k[7:]: torch.from_numpy(v) for k, v in sd.items() if k.startswith("linear.")})
        xt, yt = torch.from_numpy(x).to(dev), torch.from_numpy(np.asarray(y, np.int64)).to(dev)
        loss = torch.nn.CrossEntropyLoss()(lin(gru(xt)[0]).flatten(0, 1), yt.flatten())
        loss.backward()
        grads = {"gru." + k: p.grad.double().cpu().numpy() for k, p in gru.named_parameters()}
        grads.update({"linear." + k: p.grad.double().cpu().numpy() for k, p in lin.named_parameters()})
        out = float(loss.item())
        del gru, lin, xt, yt, loss
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = flags
        torch.cuda.empty_cache()
    return out, grads


class Argmax(object):
    """The forward's argmax and the step's argmax-correct count against the oracle's.  Positions whose float64 top-two
    margin is below MARGIN are near ties: ``flips`` counts the others whose argmax differs from the oracle's, and the
    count must lie between the oracle's correct positions among the others and that plus the near ties."""

    def __init__(self, n_correct, logits, want_logits, y):
        top2 = np.sort(want_logits, -1)[..., -2:]
        near = top2[..., 1] - top2[..., 0] < MARGIN
        self.near = int(near.sum())
        self.flips = int((logits.argmax(-1) != want_logits.argmax(-1))[~near].sum())
        self.low = int((want_logits.argmax(-1) == y)[~near].sum())
        self.n_correct = n_correct
        self.logit_err = float(np.abs(logits - want_logits).max())

    def check(self):
        assert self.flips == 0, self.flips
        assert self.low <= self.n_correct <= self.low + self.near, (self.n_correct, self.low, self.near)


def _worst(err):
    k = max(err, key=err.get)
    return k, err[k]


@pytest.mark.gpu
@pytest.mark.parametrize("H", [256, 128])
def test_production_step_matches_the_oracle(H):
    sd, x, y = production_batch(H)
    tr = _trainer(sd, F, H)
    nb = tr.bptt_windows(B)
    sms = sm_count()
    assert nb == expected_windows(sms, B)
    if sms == 132:
        assert nb == 2
    loss, metrics, norm, skipped = tr.train_step((x, y), lr=0.0)
    got = tr.grads()
    _, logits = tr.forward_arrays(x)
    tr.close()              # the 29.5 GB workspace goes before torch's step
    assert not skipped and metrics["n_positions"] == B * T
    torch_loss, torch_grads = torch_fp32_grads(sd, x, y, H)
    t0 = time.perf_counter()
    want_loss, want, want_logits = train_oracle.loss_and_grads_chunked(sd, x, y)
    oracle_s = time.perf_counter() - t0
    err, err_t = grad_errors(got, want), grad_errors(torch_grads, want)
    (k, e), (kt, et) = _worst(err), _worst(err_t)
    lerr = abs(loss - want_loss) / abs(want_loss)
    am = Argmax(metrics["n_model_correct"], logits, want_logits, y)
    want_norm = np.sqrt(sum((v ** 2).sum() for v in want.values()))
    print("train-prod H=%d B=%d T=%d: %d windows/CTA (%d SMs); worst gradient ours %s %.3g, torch fp32 %s %.3g; "
          "loss ours %.3g torch %.3g; norm %.3g; %d near-tie positions (margin < %g), %d flips outside them, max "
          "logit error %.3g; oracle %.0f s on %d CPUs" % (H, B, T, nb, sms, k, e, kt, et, lerr,
                                                         abs(torch_loss - want_loss) / abs(want_loss),
                                                         abs(norm / want_norm - 1), am.near, MARGIN, am.flips,
                                                         am.logit_err, oracle_s, os.cpu_count()))
    for key in want:
        print("train-prod H=%d   %-28s ours %.3g  torch %.3g" % (H, key, err[key], err_t[key]))
    am.check()
    assert abs(norm - want_norm) <= 1e-4 * want_norm
    assert lerr < LOSS_BAR
    assert e < GRAD_BAR, err
    assert e <= max(2 * et, 1e-6), (k, e, kt, et)


def _grads_at(tr, x, y, nb):
    tr.set_bptt_windows(nb)
    tr.train_step((x, y), lr=0.0)
    return tr.grads()


def _assert_identical(a, b, what):
    for k in a:
        assert np.array_equal(a[k], b[k]), (what, k)


@pytest.mark.gpu
@pytest.mark.parametrize("H", [256, 128])
def test_production_schedules_are_bit_identical(H):
    """1 window per CTA puts 200 CTAs (two waves) on a 132-SM card, 4 and 8 leave most SMs idle: only the schedule
    changes, and setting 0 returns to the automatic choice"""
    sd, x, y = production_batch(H)
    tr = _trainer(sd, F, H)
    auto_nb = tr.bptt_windows(B)
    auto = _grads_at(tr, x, y, 0)
    for nb in (n for n in (1, 2, 4, 8) if n != auto_nb):
        _assert_identical(auto, _grads_at(tr, x, y, nb), nb)
        assert tr.bptt_windows(B) == nb
    tr.set_bptt_windows(0)
    assert tr.bptt_windows(B) == auto_nb
    _assert_identical(auto, _grads_at(tr, x, y, 0), 0)
    tr.close()


@pytest.mark.gpu
def test_ragged_bptt_ctas_at_gru_size_256():
    """B = 37: the last CTA holds 1 window at 2 and 4 per CTA and 5 at 8; every schedule gives the automatic one's
    gradients, which match the oracle"""
    H, B_, T_ = 256, 37, 300
    sd, x, y = _case(H, F, B_, T_)
    tr = _trainer(sd, F, H)
    assert tr.bptt_windows(B_) == expected_windows(sm_count(), B_)
    tr.set_bptt_windows(0)
    loss, metrics, norm, skipped = tr.train_step((x, y), lr=0.0)
    auto = tr.grads()
    _, logits = tr.forward_arrays(x)
    for nb in (1, 2, 4, 8):
        _assert_identical(auto, _grads_at(tr, x, y, nb), nb)
    tr.close()
    want_loss, want, want_logits = train_oracle.loss_and_grads(sd, x, y)
    err = grad_errors(auto, want)
    k, e = _worst(err)
    lerr = abs(loss - want_loss) / abs(want_loss)
    am = Argmax(metrics["n_model_correct"], logits, want_logits, y)
    print("train-ragged H=%d B=%d T=%d: loss %.3g, worst gradient %s %.3g, %d near-tie positions, max logit error %.3g"
          % (H, B_, T_, lerr, k, e, am.near, am.logit_err))
    want_norm = np.sqrt(sum((v ** 2).sum() for v in want.values()))
    am.check()
    assert not skipped
    assert abs(norm - want_norm) <= 1e-4 * want_norm
    assert lerr < LOSS_BAR
    assert e < GRAD_BAR, err


@pytest.mark.gpu
@pytest.mark.parametrize("H", [256, 128])
def test_production_forward_equals_engine_fp32(H):
    """run_training's validation pass (GRUTrainer.forward_arrays) is the engine's fp32 path bit for bit at the
    production shape"""
    from medaka_b200 import models
    sd, x, _ = production_batch(H)
    tr = _trainer(sd, F, H)
    probs, logits = tr.forward_arrays(x)
    tr.close()
    m = models.GRUModel(num_features=F, gru_size=H)
    m.load_state_dict(sd)
    m.set_precision("fp32")
    out = m.forward_arrays(x, want_logits=True)
    m.close()
    assert np.array_equal(out.logits, logits)
    assert np.array_equal(out.probs, probs)
