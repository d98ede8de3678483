"""Read-level training on the H100 at the schedules a real training run takes, which the small batches of
tests/test_rl_training_gpu.py never reach: BPTT kernels at 2, 4 and 8 windows per CTA, forward and read backward passes
over many slices of (window, read) rows, every optimizer rule, and steps skipped between good ones.

RLTrainer.set_bptt_windows and RLTrainer.set_slice_rows force a schedule on small batches; the automatic schedules are
also run at batch sizes that choose them (B = 100, 150, 300) and at depths that cut slices by themselves (the grid's
65 535-row limit and the per-read scratch).

Bars, calibrated on an H100 80GB HBM3 (SXM, 700 W) from the printed lines:
  SLICE_BAR   gradients of a many-slice step against the single-slice step, per tensor max |d| / max |ref|.  Only the
              fp32 order of the additions into the pooled sums and dW17 differs ("rl-train-slices" lines).
  STEP_BAR    three optimizer steps against the oracle's float64 rule fed the kernel's own gradients, beyond one ulp of
              the fp32 weight, over the largest change ("rl-train-3-steps" lines).
The values behind them are in DESIGN.md's training section.
"""
import numpy as np
import pytest
import torch

from oracle import rl_train_oracle, train_oracle
from tests.test_rl_training_gpu import GRAD_BAR, LOSS_BAR, batch, check_buffers, grad_error, sd_for, trainer
from tests.test_training_gpu import OPTIMIZER_CASES

# worst observed: 1.0e-6 over the forced slices, 3.5e-6 for the scratch cut; GRAD_BAR / 10
SLICE_BAR = 5e-6
# worst observed: 6.6e-5 (NAdam at both sizes); a wrong term of a rule moves the update by 1e-3 of a step or more
STEP_BAR = 2e-4


def _batch(x, y):
    from medaka_b200 import training
    return training.TrainBatch(labels=y, read_level_features=x)


def _step(tr, x, y, **kw):
    loss, _, _, skipped = tr.train_step(_batch(x, y), lr=0.0, **kw)
    assert not skipped
    return loss, tr.grads()


def _oracle(H, dw, sd, x, y):
    m = rl_train_oracle.build(sd, dw)
    loss, g, _ = rl_train_oracle.loss_and_grads(m, x, y)
    return m, loss, g


def _against_oracle(tag, tr, m, loss_ref, g_ref, loss, got):
    err, which = grad_error(got, g_ref)
    lerr = abs(loss / loss_ref - 1)
    print("%s: grad %.2e (%s) loss %.2e" % (tag, err, which, lerr))
    assert err < GRAD_BAR, (which, err)
    assert lerr < LOSS_BAR
    check_buffers(tr, m)


# ---------------------------------------------------------------------------------------------- BPTT windows per CTA
@pytest.mark.gpu
@pytest.mark.parametrize("H", [128, 384])
def test_bptt_windows_per_cta_give_identical_gradients(H):
    """At B = 11, 2, 4 and 8 windows per CTA each leave a partial last CTA; each window's arithmetic does not depend on
    how many share a CTA, so every instantiation equals the automatic one bit for bit.  A hook set and reset to 0 gives
    the automatic step again."""
    sd = sd_for(H, False)
    x, y = batch(11, 24, 3, False)
    tr = trainer(H, False, sd)
    assert tr.bptt_windows(11) == 1
    _, auto = _step(tr, x, y)
    for nb in (1, 2, 4, 8):
        tr.set_bptt_windows(nb)
        assert tr.bptt_windows(11) == nb
        _, got = _step(tr, x, y)
        for k in auto:
            assert np.array_equal(auto[k], got[k]), (nb, k)
    tr.set_slice_rows(4)
    _step(tr, x, y)
    tr.set_bptt_windows(0)
    tr.set_slice_rows(0)
    _, got = _step(tr, x, y)
    for k in auto:
        assert np.array_equal(auto[k], got[k]), k
    tr.close()


@pytest.mark.gpu
def test_schedule_hooks_refuse_bad_values():
    from medaka_b200 import libmedaka
    tr = trainer(128, False, sd_for(128, False))
    for nb in (-1, 3, 16):
        with pytest.raises(libmedaka.MedakaB200Error):
            tr.set_bptt_windows(nb)
    with pytest.raises(libmedaka.MedakaB200Error):
        tr.set_slice_rows(-1)
    tr.close()


def _expected_nb(B):
    """bptt_nb's rule: the fewest windows per CTA whose CTAs (both directions) fit one wave"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for nb in (1, 2, 4):
        if -(-B // nb) * 2 <= sms:
            return nb
    return 8


# The fp32 step and the float64 oracle can put a conv pre-activation that lies within fp32 rounding of zero on opposite
# sides of its ReLU.  That moves one element's dpre2 (or dpre1), which moves dW17, db17 and every gradient below it by
# about 1 / sqrt(B D P) of their largest values: at B = 300, P = 16, D = 3 with dwells, the conv17 input of read 687,
# channel 6, position 12 lies 3.5e-8 of its sum of |terms| from zero, and the step taking its other side moved dW17 (taps 0
# to 11, the taps position 12 reaches) by 1.2e-2.  So the automatic-NB cases compare with the oracle whose undecidable
# ReLUs (margin below RELU_FP32, rl_train_oracle.relu_margins) take the step's side: each candidate flip's effect on the
# convolution-side gradients is computed, the step's difference from the oracle is fitted by them, and the oracle is
# run again with the flips whose fitted weight exceeds 1/2.  A kernel error that is not such a flip is left in full.
RELU_FP32 = 1e-6


def _fp32_relu_oracle(H, dw, sd, x, y, got):
    """(model, loss, grads, flips taken) of the oracle with the step's side of every undecidable ReLU"""
    m, loss, g = _oracle(H, dw, sd, x, y)
    margins = rl_train_oracle.relu_margins(rl_train_oracle.build(sd, dw), x)
    cands = [(name, tuple(i)) for name, v in margins.items() for i in torch.nonzero(v < RELU_FP32).tolist()]
    if not cands:
        return m, loss, g, []
    keys = [k for k in g if k.startswith(("read_level_conv", "base_embedder", "strand_embedder"))]
    scale = {k: max(np.abs(g[k]).max(), 1e-30) for k in keys}

    def vec(d):
        return np.concatenate([(np.asarray(d[k], np.float64) - g[k]).ravel() / scale[k] for k in keys])

    def flips(which):
        f = {}
        for name, i in which:
            f.setdefault(name, torch.zeros(margins[name].shape, dtype=torch.bool))[i] = True
        return f

    cols = [vec(rl_train_oracle.loss_and_grads(rl_train_oracle.build(sd, dw), x, y, flip=flips([c]))[1]) for c in cands]
    w = np.linalg.lstsq(np.stack(cols, 1), vec(got), rcond=None)[0]
    taken = [c for c, v in zip(cands, w) if v > 0.5]
    if taken:
        m = rl_train_oracle.build(sd, dw)
        loss, g, _ = rl_train_oracle.loss_and_grads(m, x, y, flip=flips(taken))
    print("rl-train-relu %d undecidable ReLU inputs, the step's side differs at %s" % (len(cands), taken))
    return m, loss, g, taken


# (lstm_size, use_dwells, B, P, D, windows per CTA on a 132-SM H100)
AUTO_NB_CASES = [(128, False, 100, 16, 3, 2), (384, False, 150, 16, 3, 4), (128, True, 300, 16, 3, 8)]


@pytest.mark.gpu
@pytest.mark.parametrize("case", AUTO_NB_CASES)
def test_automatic_bptt_windows_at_training_batch_sizes(case):
    """The batch sizes training runs choose 2, 4 and 8 windows per CTA by themselves; against the float64 oracle."""
    H, dw, B, P, D, nb = case
    assert _expected_nb(B) == nb, "this card's SM count moves the case off the instantiation it is meant to cover"
    sd = sd_for(H, dw)
    x, y = batch(B, P, D, dw)
    tr = trainer(H, dw, sd)
    assert tr.bptt_windows(B) == nb
    loss, got = _step(tr, x, y)
    m, loss_ref, g_ref, _ = _fp32_relu_oracle(H, dw, sd, x, y, got)
    _against_oracle("rl-train-auto-nb H=%d dw=%d B=%d nb=%d" % (H, dw, B, nb), tr, m, loss_ref, g_ref, loss, got)
    tr.close()


# ------------------------------------------------------------------------------------------------------- slices
def _slice_case(H, dw, rows):
    """B = 3, D = 5, P = 40 at slices of ``rows`` (window, read) rows, against the oracle and the single-slice step"""
    sd = sd_for(H, dw)
    x, y = batch(3, 40, 5, dw)
    one = trainer(H, dw, sd)
    _, g_one = _step(one, x, y)
    one.close()
    tr = trainer(H, dw, sd)
    tr.set_slice_rows(rows)
    loss, got = _step(tr, x, y)
    m, loss_ref, g_ref = _oracle(H, dw, sd, x, y)
    _against_oracle("rl-train-slices-oracle H=%d dw=%d rows=%d" % (H, dw, rows), tr, m, loss_ref, g_ref, loss, got)
    err, which = grad_error(got, {k: v.astype(np.float64) for k, v in g_one.items()})
    print("rl-train-slices H=%d dw=%d rows=%d: against one slice %.2e (%s)" % (H, dw, rows, err, which))
    assert err < SLICE_BAR, (which, err)
    tr.close()


@pytest.mark.gpu
@pytest.mark.parametrize("rows", [1, 2, 4, 5, 6, 11, 14])
def test_forced_slices_match_the_oracle_and_one_slice(rows):
    """Slices shorter than a window (5 reads), one window, just longer, and lengths that are no multiple of it: a
    window's reads add into the pooled sums, BN2's sums and dW17 across slices."""
    _slice_case(128, False, rows)


@pytest.mark.gpu
def test_forced_slices_at_lstm_size_384_with_dwells():
    _slice_case(384, True, 4)


@pytest.mark.gpu
def test_the_grid_limit_cuts_a_window_without_the_hook():
    """B = 2, P = 1, D = 33 000: 66 000 rows, so the automatic slice (65 535 rows, the grid's y limit) ends inside
    window 1.  Reads of one position are also shorter than the 17-tap kernel.  With 33 000 reads behind each of two
    positions the convolutions' gradients are sums that cancel almost entirely, so fp32 cannot hold them to GRAD_BAR:
    torch's own fp32 forward and backward of the same batch miss the float64 oracle by about 2.7e-2.  The step must do
    no worse than that, and its loss and running statistics hold the usual bars."""
    sd = sd_for(128, False)
    x, y = batch(2, 1, 33000, False)
    tr = trainer(128, False, sd)
    loss, got = _step(tr, x, y)
    m, loss_ref, g_ref = _oracle(128, False, sd, x, y)
    _, g32, _ = rl_train_oracle.loss_and_grads(rl_train_oracle.build(sd, False, dtype=torch.float32), x, y)
    err32, which32 = grad_error(g32, g_ref)
    err, which = grad_error(got, g_ref)
    lerr = abs(loss / loss_ref - 1)
    print("rl-train-grid-cut B=2 P=1 D=33000: grad %.2e (%s), torch fp32 %.2e (%s), loss %.2e"
          % (err, which, err32, which32, lerr))
    assert err < max(GRAD_BAR, err32), (which, err, err32)
    assert lerr < LOSS_BAR
    check_buffers(tr, m)
    tr.close()


@pytest.mark.gpu
def test_the_scratch_cuts_slices_without_the_hook():
    """B = 1, P = 10 000, D = 250: the per-read scratch holds 209 rows, so the automatic step runs 2 slices; against
    the same batch at 50-row slices."""
    sd = sd_for(128, False)
    x, y = batch(1, 10000, 250, False)
    tr = trainer(128, False, sd)
    _, auto = _step(tr, x, y)
    tr.close()
    tr = trainer(128, False, sd)
    tr.set_slice_rows(50)
    _, got = _step(tr, x, y)
    tr.close()
    err, which = grad_error(got, {k: v.astype(np.float64) for k, v in auto.items()})
    print("rl-train-slices scratch cut B=1 P=10000 D=250 rows=50: against 2 slices %.2e (%s)" % (err, which))
    assert err < SLICE_BAR, (which, err)


# ------------------------------------------------------------------------------------------------ optimizer rules
def _f32(v):
    if isinstance(v, tuple):
        return tuple(_f32(u) for u in v)
    return float(np.float32(v)) if isinstance(v, float) else v


def _grad_keys(H, dw):
    from medaka_b200 import training
    return [k for k in training.rl_param_shapes(H, use_dwells=dw) if not k.startswith("read_level_conv.expansion_layer")]


def _step_error(got, p, p0):
    """beyond one ulp of the fp32 weight (an update next to a rounding boundary rounds either way), over the largest
    change"""
    ulp = np.spacing(np.abs(got).astype(np.float32)).astype(np.float64)
    return np.maximum(np.abs(got - p) - ulp, 0).max() / np.abs(p - p0).max()


@pytest.mark.gpu
@pytest.mark.parametrize("H", [128, 384])
@pytest.mark.parametrize("kind,optim_args", OPTIMIZER_CASES)
def test_three_steps_match_the_oracle(H, kind, optim_args):
    """The update rules over three steps of ClipGrad and the warmup / cosine schedule: the oracle's float64 rule fed the
    kernel's own pre-clip gradients and norms and the hyper-parameters in fp32, the weights kept in fp32 between steps.
    The rule runs over two ranges around read_level_conv.expansion_layer, which stays as loaded."""
    from medaka_b200 import training
    dw = False
    sd = sd_for(H, dw, seed=4)
    keys = _grad_keys(H, dw)
    args = training.optimizer_args(kind, optim_args)
    tr = training.RLTrainer(lstm_size=H, use_dwells=dw, optimizer=kind, optim_args=optim_args).load_state_dict(sd)
    clip = training.ClipGrad(buffer_size=2)
    sched = training.linear_warmup_cosine_decay(warmup_steps=2)(args["lr"], 3, 1, 0)
    opt = train_oracle.Optimizer(kind, **{k: _f32(v) for k, v in args.items()})
    p0 = train_oracle.flatten(sd, keys)
    p = p0
    for step in range(3):
        x, y = batch(2, 30, 4, dw, seed=10 + step)
        lr, max_norm = sched.get_last_lr()[0], clip.max_norm()
        _, _, norm, skipped = tr.train_step(_batch(x, y), lr=lr, max_norm=max_norm)
        assert not skipped
        clip.record(norm)
        sched.step()
        gf = train_oracle.flatten(tr.grads(), keys)
        p = opt.step(p, gf * train_oracle.clip_coef(norm, max_norm), lr=_f32(lr))
        p = p.astype(np.float32).astype(np.float64)
    sd3 = tr.state_dict()
    tr.close()
    err = _step_error(train_oracle.flatten(sd3, keys), p, p0)
    print("rl-train-3-steps H=%d %s %s: max (|w - w_ref| - ulp) / max |step| = %.3g" % (H, kind, optim_args, err))
    assert err < STEP_BAR
    for k in ("read_level_conv.expansion_layer.weight", "read_level_conv.expansion_layer.bias"):
        assert np.array_equal(sd3[k], sd[k]), k


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["adam", "nadam"])
def test_a_skipped_step_does_not_count(kind):
    """good step, a window without reads (NaN loss: skipped), good step: the weights are the rule's at t = 1 and 2, so
    the skip advanced neither Adam's bias correction nor NAdam's mu_product"""
    from medaka_b200 import training
    sd = sd_for(128, False, seed=4)
    keys = _grad_keys(128, False)
    args = training.optimizer_args(kind, None)
    tr = training.RLTrainer(lstm_size=128, optimizer=kind).load_state_dict(sd)
    opt = train_oracle.Optimizer(kind, **{k: _f32(v) for k, v in args.items()})
    p0 = train_oracle.flatten(sd, keys)
    p = p0
    bad, yb = batch(2, 30, 4, False, seed=20)
    bad[1] = 0
    for x, y, skip in (batch(2, 30, 4, False, seed=10) + (False,), (bad, yb, True),
                       batch(2, 30, 4, False, seed=11) + (False,)):
        _, _, norm, skipped = tr.train_step(_batch(x, y), lr=1e-3, max_norm=2.0)
        assert skipped == skip
        if not skip:
            gf = train_oracle.flatten(tr.grads(), keys)
            p = opt.step(p, gf * train_oracle.clip_coef(norm, 2.0), lr=_f32(1e-3))
            p = p.astype(np.float32).astype(np.float64)
    got = train_oracle.flatten(tr.state_dict(), keys)
    tr.close()
    err = _step_error(got, p, p0)
    print("rl-train-skip %s: max (|w - w_ref| - ulp) / max |step| = %.3g" % (kind, err))
    assert err < STEP_BAR
