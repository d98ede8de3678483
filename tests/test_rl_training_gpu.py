"""Read-level training on the H100 (RLTrainer, csrc/rl_train.cu) against the float64 autograd oracle
(oracle/rl_train_oracle.py, itself checked against the reference's own loop in tests/test_rl_training.py) and the
reference golden tests/golden/rl_train_steps.npz.

Gradient parity: per tensor, max |d| / max |ref| over the tensor's elements; the worst tensor of a step against
GRAD_BAR, the loss relative to the oracle's against LOSS_BAR.  Calibrated on an H100 80GB HBM3 (SXM, 700 W) over every
case of test_gradients_match_the_oracle ("rl-train-parity" lines): the worst gradient error is 5.4e-6
(read_level_conv.convs.3.weight, the single-read window), 2.1e-6 on 4 x 2 000 x 30; the worst loss error 8.0e-8.
GRAD_BAR = 5e-5 is 9.3x the worst gradient error, LOSS_BAR = 1e-6 12x the worst loss error.  The smallest of the
oracle's seven ablations of the backward pass (tests/test_rl_training.py::test_rl_ablations_exceed_the_bars, at the
first of CASES) moves some tensor by 9.0e-2, 1 800x GRAD_BAR: dW_hh against h_t instead of h_{t-1}; a dropped BatchNorm
statistics term, an unflipped dgrad, a shifted dW17 tap and a pooled mean over D instead of the reads move some tensor by
0.1 to 13, and no forget-gate
factor on the cell carry moves one by 1.3e6.  The golden bars are
those of the oracle against the same golden on the CPU (tests/test_rl_training.py); the trainer's worst observed
errors are 8.2e-7 (loss), 1.9e-5 (norm), 1.9e-6 (gradient checksums) and 3.9e-6 (weight checksums), at lstm_size 384.
"""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

import make_rl_train_golden as mk  # noqa: E402
from oracle import rl_oracle, rl_train_oracle  # noqa: E402
from tests.test_rl_training import case_state_dict, checksum_errors  # noqa: E402

GRAD_BAR = 5e-5
LOSS_BAR = 1e-6

# (lstm_size, use_dwells, B, P, D)
CASES = [(128, False, 3, 60, 6), (384, False, 2, 50, 5), (128, True, 3, 60, 6), (128, False, 1, 40, 4),
         (128, False, 2, 9, 5), (128, False, 3, 30, 1), (384, True, 2, 12, 3)]
LONG = (128, False, 4, 2000, 30)


def trainer(H, dw, sd):
    from medaka_b200 import training
    return training.RLTrainer(lstm_size=H, use_dwells=dw).load_state_dict(sd)


def sd_for(H, dw, seed=3):
    return {k: v.numpy() for k, v in rl_oracle.synth_rl_state_dict(seed, lstm_size=H, use_dwells=dw).items()}


def batch(B, P, D, dw, seed=1, single=False):
    x = rl_oracle.synth_rl_features(B, P, D, use_dwells=dw, seed=seed, empty_rows=min(2, D - 1))
    x[..., 2] = np.where((x[..., 0] != 0) & (x[..., 2] == 0), -1, x[..., 2])
    if single:                                   # window 0 with a single non-empty read
        x[0, :, 1:] = 0
    y = np.random.RandomState(seed + 7).randint(0, 5, size=(B, P))
    return x, y


def ablation_case(P=None):
    """(state dict, use_dwells, (x, y)) of the shape the ablation effects are measured at: the first of CASES
    (P shortened when given)."""
    H, dw, B, P0, D = CASES[0]
    return sd_for(H, dw), dw, batch(B, P or P0, D, dw)


def grad_error(got, ref):
    worst, which = 0.0, None
    for k, r in ref.items():
        e = np.abs(np.asarray(got[k], np.float64).reshape(r.shape) - r).max() / max(np.abs(r).max(), 1e-30)
        if e > worst:
            worst, which = e, k
    return worst, which


def check_case(H, dw, B, P, D, single=False):
    from medaka_b200 import training
    sd = sd_for(H, dw)
    x, y = batch(B, P, D, dw, single=single)
    m = rl_train_oracle.build(sd, dw)
    loss_ref, g_ref, _ = rl_train_oracle.loss_and_grads(m, x, y)
    tr = trainer(H, dw, sd)
    loss, _, _, _ = tr.train_step(training.TrainBatch(labels=y, read_level_features=x), lr=0.0)
    err, which = grad_error(tr.grads(), g_ref)
    lerr = abs(loss / loss_ref - 1)
    print("rl-train-parity H=%d dw=%d B=%d P=%d D=%d: grad %.2e (%s) loss %.2e" % (H, dw, B, P, D, err, which, lerr))
    assert err < GRAD_BAR, (which, err)
    assert lerr < LOSS_BAR
    check_buffers(tr, m)
    tr.close()


def check_buffers(tr, m):
    """All four BatchNorm running statistics within 1e-4 of the oracle's (relative to max(max |ref|, 1)) after its
    training forward, and num_batches_tracked equal to the oracle's."""
    from medaka_b200 import training
    buf, ref = tr.buffers(), m.state_dict()
    errs = []
    for k in training.RL_BUFFERS:
        r = ref[k].numpy()
        errs.append(np.abs(buf[k] - r).max() / max(np.abs(r).max(), 1.0))
        assert errs[-1] <= 1e-4, (k, errs[-1])
    print("rl-train-buffers: %s" % " ".join("%.2e" % e for e in errs))
    for k in training.RL_NBT:
        assert int(buf[k]) == int(ref[k]), k


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_gradients_match_the_oracle(case):
    check_case(*case)


@pytest.mark.gpu
def test_gradients_match_the_oracle_with_a_single_read_window():
    check_case(128, False, 2, 40, 5, single=True)


@pytest.mark.gpu
def test_gradients_match_the_oracle_on_a_long_batch():
    check_case(*LONG)


@pytest.mark.gpu
@pytest.mark.parametrize("case", mk.CASES, ids=[c[0] for c in mk.CASES])
def test_three_steps_match_the_reference_golden(case):
    from medaka_b200 import training
    name, H, dw, _, _ = case
    tr = trainer(H, dw, case_state_dict(case))
    clip = training.ClipGrad()
    sched = training.linear_warmup_cosine_decay()(0.001, mk.STEPS_PER_EPOCH, 1, 0)
    steps, g0 = [], None
    for s in range(mk.STEPS):
        x, y = mk.rl_batch(case, s)
        threshold, lr = clip.max_norm(), sched.get_last_lr()[0]
        loss, metrics, norm, _ = tr.train_step(training.TrainBatch(labels=y, read_level_features=x), lr=lr,
                                               max_norm=threshold)
        clip.record(norm)
        sched.step()
        if g0 is None:
            g0 = tr.grads()
        steps.append([loss, norm, threshold, lr, metrics["n_model_correct"]])
    err, dcorrect = checksum_errors(case, steps, g0, tr.state_dict())
    print("rl-train-golden", name, {k: "%.2e" % v for k, v in err.items()})
    for k, bar in {"loss": 1e-5, "norm": 1e-4, "grad": 1e-4, "weight": 1e-5}.items():
        assert err[k] < bar, (k, err[k])
    assert dcorrect <= 1
    sd = tr.state_dict()
    for k in ("read_level_conv.convs.2.num_batches_tracked", "read_level_conv.convs.5.num_batches_tracked"):
        assert int(sd[k]) == 7 + mk.STEPS


@pytest.mark.gpu
def test_identical_steps_are_bit_identical_and_expansion_layer_stays():
    from medaka_b200 import training
    sd = sd_for(128, False)
    x, y = batch(3, 70, 6, False)
    b = training.TrainBatch(labels=y, read_level_features=x)
    outs = []
    for _ in range(2):
        tr = trainer(128, False, sd)
        tr.train_step(b, lr=1e-3, max_norm=2.0)
        tr.train_step(b, lr=1e-3, max_norm=2.0)
        outs.append((tr.grads(), tr.state_dict()))
        tr.close()
    for k in outs[0][0]:
        assert np.array_equal(outs[0][0][k], outs[1][0][k]), k
    for k in outs[0][1]:
        assert np.array_equal(outs[0][1][k], outs[1][1][k]), k
    for k in ("read_level_conv.expansion_layer.weight", "read_level_conv.expansion_layer.bias"):
        assert np.array_equal(outs[0][1][k], sd[k]), k


@pytest.mark.gpu
def test_a_window_without_reads_skips_the_step_but_moves_the_running_statistics():
    from medaka_b200 import training
    sd = sd_for(128, False)
    x, y = batch(2, 30, 4, False)
    x[1] = 0
    tr = trainer(128, False, sd)
    w0, b0 = tr.flat_params(), tr.buffers()
    loss, _, norm, skipped = tr.train_step(training.TrainBatch(labels=y, read_level_features=x), lr=1e-3, max_norm=2.0)
    assert np.isnan(loss) and skipped and not np.isfinite(norm)
    assert np.array_equal(tr.flat_params(), w0)
    b1 = tr.buffers()
    assert not np.array_equal(b1["read_level_conv.convs.2.running_mean"], b0["read_level_conv.convs.2.running_mean"])
    assert int(b1["read_level_conv.convs.2.num_batches_tracked"]) == int(b0["read_level_conv.convs.2.num_batches_tracked"]) + 1


@pytest.mark.gpu
@pytest.mark.parametrize("H", [128, 384])
def test_process_batch_equals_the_engines_fp32_path_bit_for_bit(H):
    from medaka_b200 import read_level, training
    sd = sd_for(H, False)
    x, y = batch(3, 50, 6, False)
    tr = trainer(H, False, sd)
    tr.train_step(training.TrainBatch(labels=y, read_level_features=x), lr=1e-3, max_norm=2.0)
    loss, metrics, probs = tr.process_batch(training.TrainBatch(labels=y, read_level_features=x), want_probs=True)
    m = read_level.LatentSpaceLSTM(lstm_size=H)
    m.load_state_dict(tr.state_dict())
    m.set_conv(tensor_cores=False)
    ref = m.forward_arrays(x)
    assert np.array_equal(probs, ref)
    ll = -np.log(np.take_along_axis(probs.astype(np.float64), y[..., None], -1)).mean()
    assert abs(loss / ll - 1) < 1e-5
    assert metrics["n_positions"] == y.size


@pytest.mark.gpu
def test_workspace_and_argument_errors():
    from medaka_b200 import libmedaka, training
    # past the bounded per-read scratch, only the int8 features and the read mask grow with D
    b1, budget = training.rl_workspace_bytes(128, 4, 10000, 1000, 4)
    b2, _ = training.rl_workspace_bytes(128, 4, 10000, 2000, 4)
    assert 0 < b2 - b1 <= 4 * 10000 * 1000 * 4 + 4 * 1000 + 64
    assert training.rl_workspace_bytes(384, 100000, 10000, 10, 5)[0] > budget
    tr = trainer(128, False, sd_for(128, False))
    x, y = batch(2, 20, 3, False)
    with pytest.raises(libmedaka.MedakaB200Error):
        tr.train_step(training.TrainBatch(labels=np.full_like(y, 5), read_level_features=x))
    with pytest.raises(libmedaka.MedakaB200Error):
        tr.train_step(training.TrainBatch(labels=y, read_level_features=np.zeros((2, 20, 3, 3), np.int8)))
    trd = trainer(128, True, sd_for(128, True))
    with pytest.raises(libmedaka.MedakaB200Error):
        trd.train_step(training.TrainBatch(labels=y, read_level_features=x))


@pytest.mark.gpu
def test_run_training_on_a_created_read_level_store_writes_loadable_archives(tmp_path):
    """create_samples' read-level store through TrainBatcher and one run_training epoch; the archive loads through
    ModelStoreTGZ.load_model into the read-level engine, whose default tensor-core path predicts within the read-level
    bar of the trainer's validation forward."""
    from medaka_b200 import datastore, features, training
    from tests.test_training_samples import _synth_bams
    rpath, tpath, _, _ = _synth_bams(str(tmp_path), 4)
    store = str(tmp_path / "rl.npzstore")
    features.create_samples(rpath, store, truth=tpath, chunk_len=500, chunk_ovlp=50,
                            feature_encoder=features.ReadAlignmentFeatureEncoder())
    batcher = training.TrainBatcher([store], validation=0.25, seed=1, batch_size=4)
    assert batcher.read_level and batcher.n_batches("train") >= 2 and batcher.n_batches("valid") >= 1
    b = next(batcher.batches("valid"))
    assert b.read_level_features.dtype == np.int8 and b.read_level_features.ndim == 4
    model_fp = str(tmp_path / "model.toml")
    with open(model_fp, "w") as fh:
        fh.write('type = "LatentSpaceLSTM"\n[kwargs]\nnum_classes = 5\nlstm_size = 128\ncnn_size = 128\n')
    out = str(tmp_path / "run")
    tr = training.run_training(out, batcher, model_fp=model_fp, epochs=1, use_lr_schedule=False)
    rows = np.genfromtxt(os.path.join(out, "training.csv"), delimiter=",", names=True)
    assert np.isfinite(rows["train_loss"]) and np.isfinite(rows["val_loss"])
    model = datastore.ModelStoreTGZ(os.path.join(out, "model-0.tar.gz")).load_model()
    probs = model.forward_arrays(b.read_level_features)
    _, _, ref = tr.process_batch(b, want_probs=True)
    assert np.abs(probs - ref).max() < 2e-5
