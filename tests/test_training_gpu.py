"""Training of the consensus GRU on the H100 (medaka_b200/training.py, csrc/gru_train.cu), against the float64 BPTT
oracle (oracle/train_oracle.py, itself checked against torch autograd in tests/test_training.py).

Gradient parity: per tensor, max |d| / max |ref| over the tensor's elements, the worst tensor of a step against
GRAD_BAR; the loss relative to the oracle's against LOSS_BAR.  Calibrated on an H100 80GB HBM3 (SXM, 700 W power
limit, 1980 MHz max SM clock) over every case of test_gradients_match_the_oracle ("train-parity" lines):
  worst gradient error   1.03e-6  (gru_size 128, F = 10, B = 3, T = 1: weight_ih_l0_reverse); 5.4e-7 on 8 x 10 000,
                         9.3e-7 at gru_size 256
  worst loss error       6.7e-8   (the same case); 3.9e-9 on 8 x 10 000
  smallest ablation      3.86e-2  (h_t in place of h_{t-1} in dW_hh; the other five terms move some tensor by 0.25 to
                         1.8), measured by tests/test_training.py::test_ablations_exceed_the_bars on the oracle at
                         gru_size 128, 2 x 60; 2.31e-2 at gru_size 256, 2 x 200
The same bars hold at the default training batch, 100 x 10 000, in tests/test_training_production.py.
GRAD_BAR = 1e-5 is 9.7x the worst error and 1/3860 of the smallest ablation effect; LOSS_BAR = 1e-6 is 15x the worst
loss error.  A kernel that drops any term of the backward pass fails the bar by orders of magnitude; fp32 reordering
of the sums does not come near it.  Three optimizer steps against the oracle's float64 rules move the weights within
2.8e-4 of a step's size (Adam, the worst rule); that bar is 1e-2.

The reference's own loop pins the rest: tests/golden/train_steps.npz (tests/golden/make_train_golden.py) holds three
steps of the unmodified reference GRUModel (process_batch, ClipGrad, RMSprop with run_training's defaults,
linear_warmup_cosine_decay) at gru_size 128 and 256 in fp32.  GOLDEN_BARS are about 10x what separates the float64
oracle from it on the CPU (tests/test_training.py::test_oracle_reproduces_the_reference_golden): loss and pre-clip norm
1.2e-7 / 5.0e-7 relative, gradient and weight checksums 1.7e-7 relative, the three-step weight change 4.0e-5 (sum of
squares) and 8.6e-6 (sum, scaled by sqrt(n x sum of squares)).  Clip threshold, learning rate and argmax-correct counts
are exact.
"""
import os

import numpy as np
import pytest

from oracle import synth, train_oracle

GRAD_BAR = 1e-5
LOSS_BAR = 1e-6

# (gru_size, F, B, T)
CASES = [(128, 10, 4, 200), (128, 1, 3, 120), (128, 40, 3, 120), (128, 21, 3, 120), (256, 10, 3, 150),
         (128, 10, 1, 50), (128, 10, 3, 1), (128, 10, 37, 40)]
LONG = (128, 10, 8, 10000)

GOLDEN_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "train_steps.npz")
GOLDEN_BARS = {"loss": 1e-6, "norm": 5e-6, "grad_sum": 1e-6, "grad_sumsq": 1e-6, "weight_sum": 1e-6,
               "weight_sumsq": 1e-6, "delta_sum": 1e-4, "delta_sumsq": 4e-4}


def golden():
    """(npz, seed, F, B, T, steps, steps per epoch, state-dict keys) of the reference's three training steps"""
    g = np.load(GOLDEN_PATH)
    seed, F, B, T, steps, spe = [int(v) for v in g["args"]]
    return g, seed, F, B, T, steps, spe, [str(k) for k in g["keys"]]


def golden_batch(step, F, B, T):
    x = synth.synth_features(B, T, F, seed=10 + step)
    y = np.random.RandomState(20 + step).randint(0, 5, size=(B, T))
    return x, y


def golden_errors(H, steps, grads0, w0, w3):
    """Errors against the golden of per-step (loss, norm, threshold, lr, n_correct), the step-1 gradients and the
    weights before and after the three steps (state dicts).  Asserts the exact quantities, returns the others."""
    g, _, _, _, _, _, _, keys = golden()
    ref = g["h%d_steps" % H]
    steps = np.asarray(steps, np.float64)
    assert np.array_equal(steps[:, 2], ref[:, 2]), "clip thresholds"
    np.testing.assert_allclose(steps[:, 3], ref[:, 3], rtol=1e-12, atol=0, err_msg="learning rates")
    assert np.array_equal(steps[:, 4], ref[:, 4]), "argmax-correct counts"

    def sums(sd):
        a = [np.asarray(sd[k], np.float64) for k in keys]
        return np.array([v.sum() for v in a]), np.array([(v * v).sum() for v in a]), np.array([v.size for v in a])

    err = {"loss": np.abs(steps[:, 0] / ref[:, 0] - 1).max(), "norm": np.abs(steps[:, 1] / ref[:, 1] - 1).max()}
    for name, sd in (("grad", grads0), ("weight", w3), ("delta", {k: np.asarray(w3[k], np.float64) - w0[k] for k in keys})):
        s_, sq, n = sums(sd)
        err[name + "_sum"] = (np.abs(s_ - g["h%d_%s_sum" % (H, name)]) / np.sqrt(sq * n)).max()
        err[name + "_sumsq"] = (np.abs(sq / g["h%d_%s_sumsq" % (H, name)] - 1)).max()
    return err


def ablation_case():
    """The shape the ablation effects are measured at: the first parity case, shortened for the CPU."""
    H, F, B, T = 128, 10, 2, 60
    return _case(H, F, B, T)


def _case(H, F, B, T, seed=0):
    sd = synth.synth_state_dict(seed, num_features=F, gru_size=H)
    x = synth.synth_features(B, T, F, seed=seed + 10)
    y = np.random.RandomState(seed + 20).randint(0, 5, size=(B, T))
    return sd, x, y


def grad_errors(got, ref):
    return {k: float(np.abs(np.asarray(got[k], np.float64) - ref[k]).max() / max(np.abs(ref[k]).max(), 1e-30))
            for k in ref}


def zero_like_state_dict(F, H):
    return {k: np.zeros(v.shape, np.float32) for k, v in synth.synth_state_dict(0, num_features=F, gru_size=H).items()}


def _trainer(sd, F, H, **kw):
    from medaka_b200 import training
    tr = training.GRUTrainer(num_features=F, gru_size=H, **kw)
    tr.load_state_dict(sd)
    return tr


@pytest.mark.gpu
@pytest.mark.parametrize("H,F", [(128, 10), (128, 21), (256, 10)])
def test_training_forward_equals_engine_fp32(H, F):
    from medaka_b200 import models
    sd, x, _ = _case(H, F, 5, 300)
    tr = _trainer(sd, F, H)
    probs, logits = tr.forward_arrays(x)
    m = models.GRUModel(num_features=F, gru_size=H)
    m.load_state_dict(sd)
    m.set_precision("fp32")
    out = m.forward_arrays(x, want_logits=True)
    m.close()
    tr.close()
    assert np.array_equal(out.logits, logits)
    assert np.array_equal(out.probs, probs)


def _parity(H, F, B, T):
    sd, x, y = _case(H, F, B, T)
    tr = _trainer(sd, F, H)
    loss, metrics, norm, skipped = tr.train_step((x, y), lr=0.0)
    got = tr.grads()
    tr.close()
    want_loss, want, logits = train_oracle.loss_and_grads(sd, x, y)
    err = grad_errors(got, want)
    worst = max(err, key=err.get)
    lerr = abs(loss - want_loss) / abs(want_loss)
    print("train-parity H=%d F=%d B=%d T=%d: loss %.3g, worst gradient %s %.3g" % (H, F, B, T, lerr, worst, err[worst]))
    assert not skipped
    assert metrics["n_positions"] == B * T
    assert metrics["n_model_correct"] == int((logits.argmax(-1) == y).sum())
    want_norm = np.sqrt(sum((v.astype(np.float64) ** 2).sum() for v in want.values()))
    assert abs(norm - want_norm) <= 1e-4 * want_norm
    assert lerr < LOSS_BAR
    assert err[worst] < GRAD_BAR, err


@pytest.mark.gpu
@pytest.mark.parametrize("H,F,B,T", CASES)
def test_gradients_match_the_oracle(H, F, B, T):
    _parity(H, F, B, T)


@pytest.mark.gpu
def test_gradients_match_the_oracle_long():
    _parity(*LONG)


@pytest.mark.gpu
@pytest.mark.parametrize("nb", [2, 4, 8])
def test_bptt_windows_per_cta_give_identical_gradients(nb):
    """The BPTT kernel's windows per CTA change the schedule, not the arithmetic: every instantiation against the
    automatic choice (1 window per CTA at B = 11)"""
    sd, x, y = _case(128, 10, 11, 30)
    tr = _trainer(sd, 10, 128)
    tr.train_step((x, y), lr=0.0)
    auto = tr.grads()
    tr.set_bptt_windows(nb)
    tr.train_step((x, y), lr=0.0)
    got = tr.grads()
    tr.close()
    for k in auto:
        assert np.array_equal(auto[k], got[k]), k


@pytest.mark.gpu
def test_identical_steps_are_bit_identical():
    sd, x, y = _case(128, 10, 9, 700)
    outs = []
    for _ in range(2):
        tr = _trainer(sd, 10, 128)
        tr.train_step((x, y), lr=1e-3, max_norm=0.5)
        outs.append((tr.grads(), tr.state_dict()))
        tr.close()
    for k in sd:
        assert np.array_equal(outs[0][0][k], outs[1][0][k]), k
        assert np.array_equal(outs[0][1][k], outs[1][1][k]), k


OPTIMIZER_CASES = [
    ("rmsprop", None), ("rmsprop", {"lr": 0.01, "alpha": 0.99, "eps": 1e-08, "momentum": 0.9, "weight_decay": 0.01}),
    ("adam", None), ("adam", {"lr": 0.01, "betas": (0.8, 0.999), "eps": 1e-08, "weight_decay": 0.1}),
    ("nadam", None), ("nadam", {"lr": 0.002, "betas": (0.9, 0.999), "eps": 1e-08, "momentum_decay": 0.01,
                                "weight_decay": 0.05}),
    ("sgd", {"lr": 0.01, "momentum": 0.9, "dampening": 0.1, "weight_decay": 0.01}),
    ("sgd", {"lr": 0.01, "momentum": 0.9, "nesterov": True}),
]
# The error beyond one ulp of the fp32 weight, over the largest three-step change, printed as "train-3-steps"; without
# the ulp allowance the worst case over OPTIMIZER_CASES on the card above was 2.5e-5 (NAdam) apart from Adam at lr 1e-4
# (1.8e-4, one ulp); with it the worst is 2.3e-5, so the bar is 4.4x that.  A wrong term in a rule moves the update by
# 1e-3 of a step or more.
STEP_BAR = 1e-4


@pytest.mark.gpu
@pytest.mark.parametrize("H", [128, 256])
@pytest.mark.parametrize("kind,optim_args", OPTIMIZER_CASES)
def test_three_steps_match_the_oracle(H, kind, optim_args):
    """The kernel's update rules over three steps of ClipGrad and the warmup / cosine schedule.  The oracle's float64
    rule is fed the kernel's own pre-clip gradients and norms, the hyper-parameters as the kernel holds them (fp32) and
    keeps the weights in fp32 between steps, as the kernel's master weights are: the difference left is the update's
    fp32 arithmetic, and a wrong term of any rule (a momentum_decay, a dampening, a weight decay) shows far above it."""
    from medaka_b200 import training
    F, B, T = 10, 3, 80
    sd, _, _ = _case(H, F, B, T, seed=4)
    keys = training.state_dict_keys()
    args = training.optimizer_args(kind, optim_args)
    tr = _trainer(sd, F, H, optimizer=kind, optim_args=optim_args)
    clip = training.ClipGrad(buffer_size=2)
    sched = training.linear_warmup_cosine_decay(warmup_steps=2)(args["lr"], 3, 1, 0)
    f32 = lambda v: tuple(f32(u) for u in v) if isinstance(v, tuple) else (   # noqa: E731
        float(np.float32(v)) if isinstance(v, float) else v)
    opt = train_oracle.Optimizer(kind, **{k: f32(v) for k, v in args.items()})
    p = train_oracle.flatten(sd, keys)
    for step in range(3):
        _, x, y = _case(H, F, B, T, seed=10 + step)
        lr, max_norm = sched.get_last_lr()[0], clip.max_norm()
        _, _, norm, _ = tr.train_step((x, y), lr=lr, max_norm=max_norm)
        clip.record(norm)
        sched.step()
        gf = train_oracle.flatten(tr.grads(), keys)
        p = opt.step(p, gf * train_oracle.clip_coef(norm, max_norm), lr=f32(lr))
        p = p.astype(np.float32).astype(np.float64)
    got = train_oracle.flatten(tr.state_dict(), keys)
    tr.close()
    moved = np.abs(p - train_oracle.flatten(sd, keys)).max()
    # beyond the last store's rounding: an update that lands next to a rounding boundary of the fp32 weight can round
    # either way (one ulp, which is 2e-4 of the three steps of Adam at lr 1e-4)
    ulp = np.spacing(np.abs(got).astype(np.float32)).astype(np.float64)
    err = np.maximum(np.abs(got - p) - ulp, 0).max() / moved
    print("train-3-steps H=%d %s %s: max (|w - w_ref| - ulp) / max |step| = %.3g" % (H, kind, optim_args, err))
    assert err < STEP_BAR


@pytest.mark.gpu
@pytest.mark.parametrize("H", [128, 256])
def test_three_steps_match_the_reference_golden(H):
    """The reference's loop (make_train_golden.py) on the trainer: process_batch, ClipGrad, RMSprop with run_training's
    defaults and linear_warmup_cosine_decay() over an epoch of the golden's length."""
    from medaka_b200 import training
    g, seed, F, B, T, nsteps, spe, keys = golden()
    sd = synth.synth_state_dict(seed, num_features=F, gru_size=H)
    tr = _trainer(sd, F, H)             # RMSprop with the reference's defaults
    clip = training.ClipGrad()
    sched = training.linear_warmup_cosine_decay()(tr.lr, spe, 1, 0)
    steps, grads0 = [], None
    for s_ in range(nsteps):
        x, y = golden_batch(s_, F, B, T)
        lr, thr = sched.get_last_lr()[0], clip.max_norm()
        loss, metrics, norm, skipped = tr.train_step((x, y), lr=lr, max_norm=thr)
        assert not skipped
        if s_ == 0:
            grads0 = tr.grads()
        clip.record(norm)
        sched.step()
        steps.append([loss, norm, thr, lr, metrics["n_model_correct"]])
    w3 = tr.state_dict()
    tr.close()
    err = golden_errors(H, steps, grads0, sd, w3)
    print("train-golden H=%d: %s" % (H, " ".join("%s=%.2g" % kv for kv in err.items())))
    for k, v in err.items():
        assert v < GOLDEN_BARS[k], (k, v)


@pytest.mark.gpu
def test_loading_some_weights_keeps_the_trained_rest():
    """A load after training replaces the tensors it names and keeps the trained values of the others."""
    sd, x, y = _case(128, 10, 3, 40)
    tr = _trainer(sd, 10, 128)
    tr.train_step((x, y), lr=1e-2)
    trained = tr.state_dict()
    new_w = np.full((5, 256), 0.01, np.float32)
    new_b = np.arange(5, dtype=np.float32)
    from medaka_b200 import libmedaka as lm
    ptr = lambda a: lm.ffi.cast("const float *", lm.ffi.from_buffer(a))   # noqa: E731
    lm.check(lm.lib.mdk_trainer_load_linear(tr._tr, ptr(new_w), ptr(new_b)))
    tr.train_step((x, y), lr=0.0)        # uploads the host image again
    got = tr.state_dict()
    tr.close()
    assert np.array_equal(got["linear.weight"], new_w) and np.array_equal(got["linear.bias"], new_b)
    for k in sd:
        if not k.startswith("linear."):
            assert np.array_equal(got[k], trained[k]), k
            assert not np.array_equal(got[k], sd[k]), k


@pytest.mark.gpu
def test_non_finite_gradient_skips_the_step():
    sd, x, y = _case(128, 10, 3, 50)
    tr = _trainer(sd, 10, 128, optimizer="adam")
    tr.train_step((x, y), lr=1e-3)
    before = tr.flat_params()
    bad = x.copy()
    bad[1, 7, 3] = np.nan
    _, _, norm, skipped = tr.train_step((bad, y), lr=1e-3)
    assert skipped and not np.isfinite(norm)
    assert np.array_equal(tr.flat_params(), before)
    _, _, norm, skipped = tr.train_step((x, y), lr=1e-3)       # the next good batch steps again
    assert not skipped and np.isfinite(norm)
    assert not np.array_equal(tr.flat_params(), before)
    tr.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["adam", "nadam"])
def test_a_skipped_step_does_not_count(kind):
    """good step, a NaN feature (skipped), good step: the weights are the rule's at t = 1 and 2, so the skip advanced
    neither Adam's bias correction nor NAdam's mu_product"""
    from medaka_b200 import training
    F, H = 10, 128
    sd, _, _ = _case(H, F, 3, 50, seed=4)
    keys = training.state_dict_keys()
    args = training.optimizer_args(kind, None)
    tr = _trainer(sd, F, H, optimizer=kind)
    f32 = lambda v: tuple(f32(u) for u in v) if isinstance(v, tuple) else (   # noqa: E731
        float(np.float32(v)) if isinstance(v, float) else v)
    opt = train_oracle.Optimizer(kind, **{k: f32(v) for k, v in args.items()})
    p0 = train_oracle.flatten(sd, keys)
    p = p0
    _, bad, yb = _case(H, F, 3, 50, seed=11)
    bad = bad.copy()
    bad[1, 7, 3] = np.nan
    for x, y, skip in (_case(H, F, 3, 50, seed=10)[1:] + (False,), (bad, yb, True),
                       _case(H, F, 3, 50, seed=12)[1:] + (False,)):
        _, _, norm, skipped = tr.train_step((x, y), lr=1e-3, max_norm=2.0)
        assert skipped == skip
        if not skip:
            gf = train_oracle.flatten(tr.grads(), keys)
            p = opt.step(p, gf * train_oracle.clip_coef(norm, 2.0), lr=f32(1e-3))
            p = p.astype(np.float32).astype(np.float64)
    got = train_oracle.flatten(tr.state_dict(), keys)
    tr.close()
    ulp = np.spacing(np.abs(got).astype(np.float32)).astype(np.float64)
    err = np.maximum(np.abs(got - p) - ulp, 0).max() / np.abs(p - p0).max()
    print("train-skip %s: max (|w - w_ref| - ulp) / max |step| = %.3g" % (kind, err))
    assert err < STEP_BAR


@pytest.mark.gpu
def test_bad_labels_and_budget_are_argument_errors():
    from medaka_b200 import libmedaka, training
    sd, x, y = _case(128, 10, 2, 20)
    tr = _trainer(sd, 10, 128)
    bad = y.copy()
    bad[0, 3] = 5
    with pytest.raises(libmedaka.MedakaB200Error) as e:
        tr.train_step((x, bad))
    assert e.value.code == -1
    need, budget = training.workspace_bytes(10, 256, 100, 10000)
    assert need < budget < 80e9
    print("training workspace at 100 x 10000, gru_size 256: %.1f GB" % (need / 1e9))
    assert training.workspace_bytes(10, 256, 300, 10000)[0] > budget
    tr.close()


def _write_store(path, n, T, seed):
    """A counts store whose labels are learnable: the label is the argmax of the first five features."""
    from medaka_b200 import common, datastore, features, labels
    rs = np.random.RandomState(seed)
    with datastore.DataStore(path, "w") as ds:
        ds.set_meta(labels.HaploidLabelScheme(), "label_scheme")
        ds.set_meta(features.CountsFeatureEncoder(), "feature_encoder")
        for i in range(n):
            f = rs.dirichlet(np.full(10, 0.3), size=T).astype(np.float32)
            pos = np.zeros(T, dtype=[("major", int), ("minor", int)])
            pos["major"] = i * T + np.arange(T)
            ds.write_sample(common.Sample(ref_name="c", features=f, labels=f[:, :5].argmax(-1).astype(np.int64),
                                          ref_seq=None, positions=pos, label_probs=None, depth=None))
    return path


@pytest.mark.gpu
def test_run_training_end_to_end(tmp_path):
    import glob
    import os
    from medaka_b200 import datastore, training
    store = _write_store(str(tmp_path / "train.npzstore"), 300, 100, 0)
    batcher = training.TrainBatcher([store], validation=0.2, seed=1, batch_size=20)
    out = str(tmp_path / "run")
    model_fp = str(tmp_path / "model.toml")
    with open(model_fp, "w") as fh:
        fh.write('type = "GRUModel"\n[kwargs]\nnum_features = 10\nnum_classes = 5\ngru_size = 128\n')
    trainer = training.run_training(out, batcher, model_fp=model_fp, epochs=3, optimizer="rmsprop",
                                    use_lr_schedule=False)
    for name in ("training.csv", "losses_0.csv", "losses_2.csv", "model-0.tar.gz", "model-2.tar.gz",
                 "model-best_val_loss.tar.gz", "model-best_val_model_tot_acc.tar.gz"):
        assert os.path.exists(os.path.join(out, name)), name
    assert not glob.glob("optim_*.pt")
    rows = list(np.genfromtxt(os.path.join(out, "training.csv"), delimiter=",", names=True))
    val = [r["val_loss"] for r in rows]
    print("run_training val_loss per epoch", val)
    assert val[-1] < val[0]
    model = datastore.ModelStoreTGZ(os.path.join(out, "model-2.tar.gz")).load_model()
    model.set_precision("fp32")
    x = np.stack([np.random.RandomState(9).dirichlet(np.full(10, 0.3), size=100).astype(np.float32)] * 2)
    got = model.forward_arrays(x).probs
    model.close()
    want, _ = trainer.forward_arrays(x)
    trainer.close()
    assert np.array_equal(got, want)
