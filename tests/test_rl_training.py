"""Read-level training on the CPU: the float64 oracle (oracle/rl_train_oracle.py) against the unmodified reference's
three training steps (tests/golden/rl_train_steps.npz, tests/golden/make_rl_train_golden.py), its restatement against
torch's modules, the proof that the GPU file's gradient bar sees every ablated term of the backward pass (each moves some
tensor by more than 3x the bar), the trainer's state-dict layout, read-level batching and the argument errors raised
before the library loads."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

import make_rl_train_golden as mk  # noqa: E402
from medaka_b200 import training  # noqa: E402
from oracle import rl_oracle, rl_train_oracle  # noqa: E402

GOLDEN = np.load(os.path.join(HERE, "golden", "rl_train_steps.npz"))
# the float64 oracle against the reference's fp32 loop: relative errors
ORACLE_BARS = {"loss": 1e-5, "norm": 1e-4, "grad": 1e-4, "weight": 1e-5}


def case_state_dict(case):
    _, H, dw, _, _ = case
    return {k: v.numpy() for k, v in rl_oracle.synth_rl_state_dict(mk.SEED, lstm_size=H, use_dwells=dw).items()}


def checksum_errors(case, steps, g0, w3):
    """(relative errors of the per-step values, grad sums, weight sums) against the golden; exact quantities asserted"""
    name = case[0]
    ref = GOLDEN[name + "_steps"]
    steps = np.asarray(steps, np.float64)
    np.testing.assert_allclose(steps[:, 2], ref[:, 2], rtol=1e-12)
    np.testing.assert_allclose(steps[:, 3], ref[:, 3], rtol=1e-12)
    err = {"loss": np.abs(steps[:, 0] / ref[:, 0] - 1).max(), "norm": np.abs(steps[:, 1] / ref[:, 1] - 1).max()}
    gk = [str(k) for k in GOLDEN[name + "_grad_keys"]]
    gs = np.array([np.asarray(g0[k], np.float64).sum() for k in gk])
    gq = np.array([(np.asarray(g0[k], np.float64) ** 2).sum() for k in gk])
    n = np.array([np.asarray(g0[k]).size for k in gk])
    err["grad"] = max((np.abs(gs - GOLDEN[name + "_grad_sum"]) / np.sqrt(gq * n)).max(),
                      np.abs(gq / GOLDEN[name + "_grad_sumsq"] - 1).max())
    keys = [str(k) for k in GOLDEN[name + "_keys"]]
    ws = np.array([np.asarray(w3[k], np.float64).sum() for k in keys])
    wq = np.array([(np.asarray(w3[k], np.float64) ** 2).sum() for k in keys])
    n = np.array([max(np.asarray(w3[k]).size, 1) for k in keys])
    scale = np.sqrt(np.maximum(wq, 1e-30) * n)
    err["weight"] = max((np.abs(ws - GOLDEN[name + "_weight_sum"]) / scale).max(),
                        np.abs((wq + 1e-30) / (GOLDEN[name + "_weight_sumsq"] + 1e-30) - 1).max())
    return err, np.abs(steps[:, 4] - ref[:, 4]).max()


@pytest.mark.parametrize("case", mk.CASES, ids=[c[0] for c in mk.CASES])
def test_oracle_reproduces_the_reference_golden(case):
    batches = [mk.rl_batch(case, s) for s in range(mk.STEPS)]
    steps, g0, w3 = rl_train_oracle.train_steps(case_state_dict(case), batches, use_dwells=case[2],
                                                steps_per_epoch=mk.STEPS_PER_EPOCH)
    err, dcorrect = checksum_errors(case, steps, g0, w3)
    print("rl-oracle-golden", case[0], {k: "%.2e" % v for k, v in err.items()})
    for k, bar in ORACLE_BARS.items():
        assert err[k] < bar, (k, err[k])
    assert dcorrect <= 1
    for k in ("read_level_conv.convs.2.num_batches_tracked", "read_level_conv.convs.5.num_batches_tracked"):
        assert int(w3[k]) == 7 + mk.STEPS


@pytest.mark.parametrize("H", [128, 384])
def test_restated_lstm_equals_torch(H):
    """The per-step LSTM that carries the LSTM ablations is torch.nn.LSTM without one (float64, 1e-12)."""
    torch.manual_seed(H)
    mod = torch.nn.LSTM(H, H, num_layers=2, bidirectional=True, batch_first=True).double()
    h = torch.randn(3, 17, H, dtype=torch.float64, requires_grad=True)
    want = mod(h)[0]
    got = rl_train_oracle.lstm(mod, h)
    assert (got - want).abs().max() <= 1e-12 * want.abs().max()
    gw = torch.autograd.grad((want * torch.cos(want)).sum(), [h] + list(mod.parameters()))
    gg = torch.autograd.grad((got * torch.cos(got)).sum(), [h] + list(mod.parameters()))
    for a, b in zip(gw, gg):
        assert (a - b).abs().max() <= 1e-12 * a.abs().max()


@pytest.mark.parametrize("H,dw", [(128, False), (384, True)])
def test_restated_oracle_equals_the_modules(H, dw):
    """The whole restatement (k = 17 convolution with its backward written out, BatchNorm, per-step LSTM) without an
    ablation: loss, gradients and running statistics of torch's modules."""
    from tests.test_rl_training_gpu import batch, sd_for
    sd = sd_for(H, dw)
    x, y = batch(2, 20, 4, dw)
    m0, m1 = rl_train_oracle.build(sd, dw), rl_train_oracle.build(sd, dw)
    l0, g0, c0 = rl_train_oracle.loss_and_grads(m0, x, y)
    l1, g1, c1 = rl_train_oracle.loss_and_grads(m1, x, y, restated=True)
    assert abs(l1 / l0 - 1) <= 1e-12 and c0 == c1
    assert sorted(g0) == sorted(g1)
    for k in g0:
        assert np.abs(g1[k] - g0[k]).max() <= 1e-12 * np.abs(g0[k]).max(), k
    b0, b1 = m0.state_dict(), m1.state_dict()
    for k in training.RL_BUFFERS + training.RL_NBT:
        assert torch.equal(b0[k], b1[k]), k


def test_a_flipped_relu_keeps_the_values_and_moves_the_gradient_at_one_element():
    """oracle flips (the side of an undecidable ReLU): the loss and running statistics stay, the gradient changes by
    one element's dpre2, so db17 moves in the flipped channel only"""
    from tests.test_rl_training_gpu import ablation_case
    sd, dw, (x, y) = ablation_case(P=20)
    m0, m1 = rl_train_oracle.build(sd, dw), rl_train_oracle.build(sd, dw)
    l0, g0, _ = rl_train_oracle.loss_and_grads(m0, x, y, restated=True)
    r = rl_train_oracle.relu_margins(rl_train_oracle.build(sd, dw), x)["conv17"]
    flip = torch.zeros(r.shape, dtype=torch.bool)
    flip[tuple(torch.nonzero(r == r.min())[0].tolist())] = True
    l1, g1, _ = rl_train_oracle.loss_and_grads(m1, x, y, flip={"conv17": flip})
    assert abs(l1 / l0 - 1) <= 1e-15
    for k in training.RL_BUFFERS:
        assert torch.equal(m0.state_dict()[k], m1.state_dict()[k]), k
    c = int(torch.nonzero(flip)[0, 1])
    d = np.abs(g1["read_level_conv.convs.3.bias"] - g0["read_level_conv.convs.3.bias"])
    assert d[c] > 1e-6 * np.abs(g0["read_level_conv.convs.3.bias"]).max()
    assert np.delete(d, c).max() <= 1e-12 * np.abs(g0["read_level_conv.convs.3.bias"]).max()


def test_rl_ablations_change_the_oracle_and_are_named():
    from tests.test_rl_training_gpu import ablation_case
    sd, dw, (x, y) = ablation_case(P=20)
    _, ref, _ = rl_train_oracle.loss_and_grads(rl_train_oracle.build(sd, dw), x, y)
    for which in rl_train_oracle.ABLATIONS:
        _, g, _ = rl_train_oracle.loss_and_grads(rl_train_oracle.build(sd, dw), x, y, ablation=which)
        assert any(not np.allclose(g[k], ref[k], rtol=1e-6, atol=0) for k in ref), which
    with pytest.raises(ValueError):
        rl_train_oracle.loss_and_grads(rl_train_oracle.build(sd, dw), x, y, ablation="nope")


def test_rl_ablations_exceed_the_bars():
    """Every ablated term moves some gradient tensor by more than 3x the GPU file's bar, at its first parity case."""
    from tests import test_rl_training_gpu as gpu
    sd, dw, (x, y) = gpu.ablation_case()
    _, ref, _ = rl_train_oracle.loss_and_grads(rl_train_oracle.build(sd, dw), x, y)
    for which in rl_train_oracle.ABLATIONS:
        _, g, _ = rl_train_oracle.loss_and_grads(rl_train_oracle.build(sd, dw), x, y, ablation=which)
        worst, k = gpu.grad_error(g, ref)
        print("rl-train-ablation %-20s max per-tensor effect %.3g (%.0fx the bar, %s)"
              % (which, worst, worst / gpu.GRAD_BAR, k))
        assert worst > 3 * gpu.GRAD_BAR, (which, worst)


@pytest.mark.parametrize("case", mk.CASES, ids=[c[0] for c in mk.CASES])
def test_state_dict_layout_is_the_references(case):
    name, H, dw, _, _ = case
    assert training.rl_state_dict_keys(H, dw) == [str(k) for k in GOLDEN[name + "_keys"]]
    shapes = training.rl_param_shapes(H, use_dwells=dw)
    sd = case_state_dict(case)
    for k, shape in shapes.items():
        assert tuple(sd[k].shape) == shape, k
    assert [k for k in shapes if "read_level_conv.expansion_layer" not in k] == [str(k) for k in GOLDEN[name + "_grad_keys"]]


@pytest.mark.parametrize("case", mk.CASES, ids=[c[0] for c in mk.CASES])
def test_seeded_initial_weights_equal_model_from_dicts(case):
    name, H, dw, _, _ = case
    sd = training._init_rl_state_dict(mk.model_dict(case)["kwargs"], mk.SEED)
    keys = [str(k) for k in GOLDEN[name + "_keys"]]
    s = np.array([np.asarray(sd[k], np.float64).sum() for k in keys])
    q = np.array([(np.asarray(sd[k], np.float64) ** 2).sum() for k in keys])
    np.testing.assert_allclose(s, GOLDEN[name + "_init_sum"], rtol=1e-12, atol=1e-9)
    np.testing.assert_allclose(q, GOLDEN[name + "_init_sumsq"], rtol=1e-12, atol=1e-9)


def test_pad_to_max_depth_pads_reads_with_zeros_into_int8():
    rs = np.random.RandomState(0)
    feats = [rs.randint(-1, 60, size=(7, d, 4)).astype(np.int8) for d in (3, 5, 1)]
    feats[1] = feats[1].astype(np.uint8)                  # collated stores may hold uint8: -1 reads back as 255
    out = training.pad_to_max_depth(feats)
    assert out.dtype == np.int8 and out.shape == (3, 7, 5, 4)
    for i, f in enumerate(feats):
        d = f.shape[1]
        assert np.array_equal(out[i, :, :d], f.astype(np.int8))
        assert not out[i, :, d:].any()


def test_read_level_features_are_int8_with_the_strand_restored():
    x = np.zeros((1, 2, 1, 4), np.uint8)
    x[0, 0, 0, 2] = 255
    assert training._rl_features(x)[0, 0, 0, 2] == -1
    with pytest.raises(ValueError):
        training._rl_features(np.zeros((2, 3, 4), np.int8))


@pytest.mark.parametrize("kw", [{"amp": True}, {"lstm_size": 256}, {"cnn_size": 64}, {"kernel_sizes": [1, 9]},
                                {"num_classes": 4}, {"bidirectional": False}, {"pooler_type": "max"}])
def test_unsupported_configurations_raise_before_the_library_loads(kw):
    with pytest.raises(NotImplementedError):
        training.RLTrainer(**kw)
