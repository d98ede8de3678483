"""Training of the consensus GRU, CPU half: the float64 BPTT oracle (oracle/train_oracle.py) against torch autograd,
its optimizer rules against torch.optim, the host-side schedules and ClipGrad against the reference's own test
literals (medaka/test/test_torch_ext.py, copied as data), the argument checks of run_training, and the proof that the
GPU file's gradient bars see every term of the backward pass (each ablation moves some tensor by more than 3x its bar).
"""
import functools
import tarfile

import numpy as np
import pytest
import torch

from oracle import synth, train_oracle
from tests import test_training_gpu as gpu


def _case(H=16, F=10, B=3, T=9, seed=0):
    sd = synth.synth_state_dict(seed, num_features=F, gru_size=H)
    x = synth.synth_features(B, T, F, seed=seed + 10)
    y = np.random.RandomState(seed + 20).randint(0, 5, size=(B, T))
    return sd, x, y


@pytest.mark.parametrize("H,F,B,T", [(16, 10, 3, 9), (8, 1, 1, 5), (12, 21, 2, 1), (16, 40, 4, 6)])
def test_oracle_gradients_equal_autograd(H, F, B, T):
    sd, x, y = _case(H, F, B, T)
    loss, g, _ = train_oracle.loss_and_grads(sd, x, y)
    want_loss, want = train_oracle.autograd_loss_and_grads(sd, x, y)
    assert abs(loss - want_loss) <= 1e-12 * abs(want_loss)
    for k in sd:
        np.testing.assert_allclose(g[k], want[k], rtol=1e-9, atol=1e-13, err_msg=k)


def test_ablations_change_the_oracle_and_are_named():
    sd, x, y = _case()
    _, ref, _ = train_oracle.loss_and_grads(sd, x, y)
    for which in train_oracle.ABLATIONS:
        _, g, _ = train_oracle.loss_and_grads(sd, x, y, ablation=which)
        assert any(not np.allclose(g[k], ref[k], rtol=1e-6, atol=0) for k in sd), which
    with pytest.raises(ValueError):
        train_oracle.loss_and_grads(sd, x, y, ablation="nope")


def _ablations_exceed_the_bars(H, sd, x, y):
    _, ref, _ = train_oracle.loss_and_grads(sd, x, y)
    for which in train_oracle.ABLATIONS:
        _, g, _ = train_oracle.loss_and_grads(sd, x, y, ablation=which)
        err = gpu.grad_errors(g, ref)
        worst = max(err, key=err.get)
        print("train-ablation H=%d %-14s max per-tensor effect %.3g (%.0fx the bar, %s)"
              % (H, which, err[worst], err[worst] / gpu.GRAD_BAR, worst))
        assert err[worst] > 3 * gpu.GRAD_BAR, (which, err[worst])


def test_ablations_exceed_the_bars():
    """Every dropped term moves some gradient tensor by more than 3x the GPU file's bar, at one of its shapes."""
    _ablations_exceed_the_bars(128, *gpu.ablation_case())


def test_ablations_exceed_the_bars_at_gru_size_256():
    """The same at the width medaka train builds by default, on a batch the CPU oracle runs in seconds"""
    _ablations_exceed_the_bars(256, *gpu._case(256, 10, 2, 200))


def test_chunked_oracle_equals_the_whole_batch():
    """Slices of 3 windows out of 7 (the last one short), weighted by their share of the positions, give the
    whole batch's loss, gradients and logits"""
    sd, x, y = _case(H=16, F=10, B=7, T=9)
    loss, g, logits = train_oracle.loss_and_grads(sd, x, y)
    c_loss, c_g, c_logits = train_oracle.loss_and_grads_chunked(sd, x, y, windows=3)
    assert abs(c_loss - loss) <= 1e-12 * abs(loss)
    err = gpu.grad_errors(c_g, g)
    assert max(err.values()) < 1e-12, err
    np.testing.assert_allclose(c_logits, logits, rtol=1e-12, atol=0)


OPTIMIZERS = [
    ("rmsprop", {"lr": 0.001, "alpha": 0.9, "eps": 1e-07, "momentum": 0.0}),
    ("rmsprop", {"lr": 0.01, "alpha": 0.99, "eps": 1e-08, "momentum": 0.9, "weight_decay": 0.01}),
    ("adam", {"lr": 0.0001, "betas": (0.9, 0.99), "eps": 1e-07}),
    ("adam", {"lr": 0.01, "betas": (0.8, 0.999), "eps": 1e-08, "weight_decay": 0.1}),
    ("nadam", {"lr": 0.002, "betas": (0.9, 0.99), "eps": 1e-07}),
    ("nadam", {"lr": 0.002, "betas": (0.9, 0.999), "eps": 1e-08, "momentum_decay": 0.01, "weight_decay": 0.05}),
    ("sgd", {"lr": 0.001}),
    ("sgd", {"lr": 0.01, "momentum": 0.9, "dampening": 0.1, "weight_decay": 0.01}),
    ("sgd", {"lr": 0.01, "momentum": 0.9, "nesterov": True}),
]
TORCH_OPT = {"rmsprop": torch.optim.RMSprop, "adam": torch.optim.Adam, "nadam": torch.optim.NAdam,
             "sgd": torch.optim.SGD}


@pytest.mark.parametrize("kind,args", OPTIMIZERS)
def test_optimizer_rules_equal_torch_optim(kind, args):
    """20 steps of the same gradients through the oracle's rule and torch.optim, float64 on the CPU."""
    rs = np.random.RandomState(1)
    p0 = rs.randn(257)
    grads = [rs.randn(257) * 10.0 ** rs.uniform(-3, 1) for _ in range(20)]
    w = torch.nn.Parameter(torch.tensor(p0))
    opt = TORCH_OPT[kind]([w], **args)
    mine = train_oracle.Optimizer(kind, **args)
    p = p0
    for g in grads:
        w.grad = torch.tensor(g)
        opt.step()
        p = mine.step(p, g)
        np.testing.assert_allclose(p, w.detach().numpy(), rtol=1e-12, atol=1e-15)


def test_optimizer_args_complete_and_reject():
    from medaka_b200 import training
    assert training.optimizer_args("rmsprop") == {"lr": 0.001, "alpha": 0.9, "eps": 1e-07, "weight_decay": 0.0,
                                                  "momentum": 0.0, "centered": False}
    assert training.optimizer_args("adam", {"lr": 0.1})["betas"] == (0.9, 0.999)
    for kind, bad in (("rmsprop", {"centered": True}), ("adam", {"amsgrad": True}), ("adam", {"foreach": True}),
                      ("nadam", {"decoupled_weight_decay": True}), ("sgd", {"maximize": True})):
        with pytest.raises(ValueError, match=list(bad)[0]):
            training.optimizer_args(kind, bad)
    with pytest.raises(ValueError, match="Unknown optimizer"):
        training.optimizer_args("adagrad")


def test_run_training_rejects_loss_args_and_amp():
    from medaka_b200 import training
    with pytest.raises(ValueError, match="label_smoothing"):
        training.run_training("unused", batcher=None, loss_args={"label_smoothing": 0.1})
    with pytest.raises(NotImplementedError):
        training.GRUTrainer(amp=True)


# the reference's scheduler tests: RMSprop default lr 0.01, 10 batches per epoch, one epoch
def _lrs(sched, n=10, base_lr=0.01):
    s = sched(base_lr, n, 1, 0)
    out = []
    for _ in range(n):
        out.append(s.get_last_lr()[0])
        s.step()
    return out


def test_no_schedule():
    from medaka_b200 import training
    assert _lrs(training.no_schedule()) == [0.01] * 10


def test_warmup_schedule():
    from medaka_b200 import training
    np.testing.assert_allclose(_lrs(training.no_schedule(warmup_steps=3)), [0.001, 0.004, 0.007] + [0.01] * 7,
                               rtol=0, atol=1e-7)


def test_cosine_schedule():
    from medaka_b200 import training
    want = 0.01 * 0.01 + 0.5 * (1 - 0.01) * 0.01 * (1 + np.cos(np.linspace(0, 1, 11) * np.pi))
    np.testing.assert_allclose(_lrs(training.linear_warmup_cosine_decay(end_ratio=0.01, warmup_steps=0)), want[:10],
                               rtol=0, atol=1e-7)


def test_warmup_cosine_schedule():
    from medaka_b200 import training
    want = [0.001, 0.004, 0.007] + list(0.0001 + 0.5 * 0.0099 * (1 + np.cos(np.arange(0, 7) * np.pi / 7.)))
    np.testing.assert_allclose(_lrs(training.linear_warmup_cosine_decay(end_ratio=0.01, warmup_steps=3)), want,
                               rtol=0, atol=1e-7)


def test_clip_grad_threshold():
    """ClipGrad(quantile=0.5, factor=2) over a buffer of ones clips a gradient of norm 1000 sqrt(10) to <= 2, as the
    reference's test_013_clip_grad checks through clip_grad_norm_."""
    from medaka_b200 import training
    clip = training.ClipGrad(quantile=0.5, factor=2)
    assert clip.max_norm() == 2e6
    for _ in range(len(clip.buffer)):
        clip.append(1.0)
    g = 1000 * np.ones(10)
    norm = float(np.linalg.norm(g))
    clipped = g * train_oracle.clip_coef(norm, clip.max_norm())
    assert np.linalg.norm(clipped) <= 2 * 1.0
    assert clip.record(norm) == norm and clip.buffer[0] == norm
    clip.record(float("nan"))
    assert clip.i == 1


def test_encoded_labels_to_training_vectors():
    from medaka_b200 import training
    plain = np.array([0, 3, 4, 1])
    assert training.encoded_labels_to_training_vectors(plain).tolist() == [[0], [3], [4], [1]]
    legacy = np.array([(5, 1), (2, 1), (8, 2)], dtype=[("base", "i8"), ("run_length", "i8")])
    assert training.encoded_labels_to_training_vectors(legacy).tolist() == [[1], [0], [4]]


def test_model_meta_unpickles_as_the_reference_wrote_it(tmp_path):
    """The meta.pkl of an archive run_training writes (ModelStoreTGZ.write with a model_from_dict partial) unpickles
    with ref_loads under the reference's module paths."""
    from medaka_b200 import datastore, features, labels, training
    meta = {"model_function": functools.partial(datastore._ref_model_from_dict, training.DEFAULT_MODEL_DICT),
            "label_scheme": labels.HaploidLabelScheme(), "feature_encoder": features.CountsFeatureEncoder()}
    sd = gpu.zero_like_state_dict(10, 256)
    fp = str(tmp_path / "model-0.tar.gz")
    datastore.ModelStoreTGZ.write(fp, sd, meta)
    with tarfile.open(fp) as tar:
        raw = tar.extractfile("model/meta.pkl").read()
    assert b"medaka.models" in raw and b"medaka.labels" in raw
    got = datastore.ref_loads(raw)
    assert got["model_function"].args[0] == training.DEFAULT_MODEL_DICT
    assert datastore.ModelStoreTGZ(fp).model_kwargs()["kwargs"]["gru_size"] == 256


def test_oracle_reproduces_the_reference_golden():
    """The float64 oracle with this package's ClipGrad and schedule through the reference's three recorded steps
    (tests/golden/make_train_golden.py); prints the errors GOLDEN_BARS are derived from."""
    from medaka_b200 import training
    g, seed, F, B, T, nsteps, spe, keys = gpu.golden()
    for H in (128, 256):
        sd = synth.synth_state_dict(seed, num_features=F, gru_size=H)
        clip = training.ClipGrad()
        sched = training.linear_warmup_cosine_decay()(0.001, spe, 1, 0)
        opt = train_oracle.Optimizer("rmsprop", **training.optimizer_args("rmsprop"))
        p = train_oracle.flatten(sd, keys)
        steps, grads0 = [], None
        for s in range(nsteps):
            x, y = gpu.golden_batch(s, F, B, T)
            loss, gr, logits = train_oracle.loss_and_grads(train_oracle.unflatten(p, sd, keys), x, y)
            gf = train_oracle.flatten(gr, keys)
            norm, thr, lr = float(np.linalg.norm(gf)), clip.max_norm(), sched.get_last_lr()[0]
            grads0 = gr if s == 0 else grads0
            steps.append([loss, norm, thr, lr, int((logits.argmax(-1) == y).sum())])
            clip.record(norm)
            sched.step()
            p = opt.step(p, gf * train_oracle.clip_coef(norm, thr), lr=lr)
        err = gpu.golden_errors(H, steps, grads0, sd, train_oracle.unflatten(p, sd, keys))
        print("oracle-golden H=%d: %s" % (H, " ".join("%s=%.2g" % kv for kv in err.items())))
        for k, v in err.items():
            assert v < gpu.GOLDEN_BARS[k] / 3, (H, k, v)


class _FakeTrainer(object):
    """Records what run_training asks of a GRUTrainer, without a GPU."""

    def __init__(self, num_features=10, gru_size=128, optimizer="rmsprop", optim_args=None, **kw):
        from medaka_b200 import training
        self.lr = training.optimizer_args(optimizer, optim_args)["lr"]
        self.sd = gpu.zero_like_state_dict(num_features, gru_size)
        self.calls = []

    def load_state_dict(self, sd):
        return self

    def state_dict(self):
        return self.sd

    def train_step(self, batch, lr=None, max_norm=None):
        self.calls.append(("train", lr, max_norm))
        n = batch.labels.size
        return 1.0, {"n_model_correct": 0, "n_positions": n}, 1.0, False

    def process_batch(self, batch):
        self.calls.append(("valid", None, None))
        return 1.0, {"n_model_correct": 0, "n_positions": batch.labels.size}


class _FakeBatcher(object):
    from medaka_b200 import features, labels
    label_scheme, feature_encoder = labels.HaploidLabelScheme(), features.CountsFeatureEncoder()
    batch_size = 2

    def __init__(self, n_train, n_valid):
        self.n = {"train": n_train, "valid": n_valid}

    def n_batches(self, which="train"):
        return self.n[which]

    def batches(self, which="train", rng=None):
        from medaka_b200 import training
        for _ in range(self.n[which]):
            yield training.TrainBatch(np.zeros((2, 5, 10), np.float32), np.zeros((2, 5), np.int64))


@pytest.mark.parametrize("quantile_grad_clip", [True, False])
def test_run_training_follows_the_reference_schedule_and_clip(tmp_path, monkeypatch, quantile_grad_clip):
    """As medaka/training.py + torch_ext.run_epoch: the schedule spans epochs x the whole training loader (however
    many batches samples_per_training_epoch lets an epoch run), advances on validation batches too, and without the
    quantile clipper the clip threshold is 2.0."""
    from medaka_b200 import training
    made = []
    monkeypatch.setattr(training, "GRUTrainer", lambda **kw: made.append(_FakeTrainer(**kw)) or made[-1])
    model_fp = str(tmp_path / "m.toml")
    with open(model_fp, "w") as fh:
        fh.write('type = "GRUModel"\n[kwargs]\nnum_features = 10\nnum_classes = 5\ngru_size = 128\n')
    n_train, n_valid, epochs = 6, 2, 3
    training.run_training(str(tmp_path / "run"), _FakeBatcher(n_train, n_valid), model_fp=model_fp, epochs=epochs,
                          samples_per_training_epoch=8, quantile_grad_clip=quantile_grad_clip)
    calls = made[0].calls
    assert [c[0] for c in calls] == (["train"] * 4 + ["valid"] * n_valid) * epochs
    sched = training.linear_warmup_cosine_decay()(0.001, n_train, epochs, 0)
    want = []
    for _ in range(epochs):
        for _ in range(4):
            want.append(sched.get_last_lr()[0])
            sched.step()
        for _ in range(n_valid):
            sched.step()
    np.testing.assert_allclose([c[1] for c in calls if c[0] == "train"], want, rtol=1e-15, atol=0)
    thresholds = {c[2] for c in calls if c[0] == "train"}
    assert thresholds == ({2e6} if quantile_grad_clip else {2.0})
    assert (tmp_path / "run" / "model-best_val_loss.tar.gz").exists()


def test_metrics_count_majority_vote_when_a_batch_carries_it():
    """process_batch's metrics: n_argmax_correct only for batches with majority_vote_probs (the reference's
    process_batch); TrainBatcher's batches carry none, as the reference's collate never sets them for counts."""
    from medaka_b200 import training

    class _Stats:
        n_correct, n_positions = 3, 4
    labels = np.array([[0, 1, 2, 3]])
    mvp = np.eye(5)[[[0, 1, 4, 4]]]
    with_mvp = training.GRUTrainer._metrics(_Stats, training.TrainBatch(np.zeros((1, 4, 10)), labels, mvp))
    assert with_mvp == {"n_model_correct": 3, "n_argmax_correct": 2, "n_positions": 4}
    assert training.GRUTrainer._metrics(_Stats, training.TrainBatch(np.zeros((1, 4, 10)), labels)) == \
        {"n_model_correct": 3, "n_positions": 4}
