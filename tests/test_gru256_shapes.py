"""The consensus GRU at gru_size = 256 at the shapes and feature widths beyond tests/test_gru256.py's one wave at F = 10:
the models `medaka train` builds from stores of one to four datatypes (F = 10 to 40) and every other width the engine
accepts, ragged calls, calls that span several groups, groups of several cluster waves, and the engine's state across
weight reloads, refused state dicts and a refused workspace.

  F        layer-0 input projection at gru_size 256 (both precisions; tile-interleaved, pre-scaled rows on tc)
  10, 20   inproj0_kernel<10 | 20, 256>: the weights of six columns in registers per thread
  others   inproj0_generic_kernel<256>: the weights streamed from L1 / L2

Every device stage is held to test_gru256's float64 bars (BARS) against oracle/gru_oracle.stages; windows, whatever
group, tile or cluster wave they run in, give bit-identical outputs; and the trainer's forward at 256 is the engine's
fp32 forward bit for bit.  The ablation test shows on the CPU that the bars still see a lost tensor-core product at
each width the GPU tests use.
"""
import numpy as np
import pytest

from oracle import gru_oracle
from tests.test_feature_widths import _features
from tests.test_gru256 import ABLATIONS, BARS, H, STAGES, WEIGHTS, _decided, _model, _scaled, _sd
from tests.test_gru_stages import _need_memory
from tests.test_training_gpu import GRAD_BAR, LOSS_BAR, _case, _parity  # noqa: F401  (the bars _parity asserts)

LONG_T = 10000
# featuriser_like_features: one to four datatypes; _features: unnormalised cubed uniforms (not fp16-exact)
COUNTS_WIDTHS = (20, 30, 40)
UNIFORM_WIDTHS = (1, 3, 9, 16, 17, 21, 64, 129, 1024)
LONG_WIDTHS = {40: "counts", 17: "uniform"}
# At 10 000 steps with hot weights the tc path's probabilities at F = 17 and 40 are up to 4.0e-6 from the oracle, where
# BARS["probs"] (2.6e-6) was set at 1.3x the worst error at F = 10.  As there, no probs bar can be both 4x the tc error
# and a third of the smallest ablation effect; these widths' bar keeps the 1.3x margin and the other stages, at BARS,
# carry the discrimination (DESIGN section 2).
LONG_BARS = dict(BARS, probs=5.2e-6)


def _x(F, B, T, seed):
    if F in COUNTS_WIDTHS:
        return gru_oracle.featuriser_like_features(B, T, F, seed=seed)
    return _features(B, T, F, seed)


# ---------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("weights", list(WEIGHTS))
@pytest.mark.parametrize("F", COUNTS_WIDTHS + UNIFORM_WIDTHS)
def test_ablations_exceed_the_bars_at_every_width(F, weights):
    """Each tensor-core product the 256 path can lose moves some stage by more than 3x its bar, at every width the GPU
    tests run: at the long windows' 10 000 steps for F = 17 and 40, on 2 windows x 2 000 steps otherwise."""
    T = LONG_T if F in LONG_WIDTHS else 2000
    sd = _sd(30 + F, F, **WEIGHTS[weights])
    x = _x(F, 2, T, seed=F)
    want = gru_oracle.stages(sd, x)
    smallest = np.inf
    for which in ABLATIONS:
        asd, kw = gru_oracle.ablate(sd, which)
        got = gru_oracle.stages(asd, x, **kw)
        effect = {k: float(_scaled(k, got[k], want[k]).max()) for k in STAGES}
        ratio = {k: effect[k] / BARS[k] for k in STAGES}
        print("gru256 ablation F=%d %s/%s: %s" % (F, weights, which, " ".join("%s=%.3g" % (k, effect[k])
                                                                            for k in STAGES)))
        smallest = min(smallest, max(ratio.values()))
        assert max(ratio.values()) > 3, (F, weights, which, effect)
    print("gru256 smallest ablation F=%d %s: %.1fx its bar" % (F, weights, smallest))


class _Batcher(object):
    read_level = False

    def __init__(self, F):
        self.feature_shape = (100, F)


@pytest.mark.parametrize("F", [10, 20, 40])
def test_default_model_takes_the_width_of_the_store(F):
    """run_training with no model file trains DEFAULT_MODEL_DICT (gru_size 256) at the store's feature width, so a store
    of two to four datatypes gives an F = 20 to 40 model whose archive builds that model."""
    from medaka_b200 import training
    d, weights = training._model_dict(None, _Batcher(F))
    assert weights is None
    assert d == {"type": "GRUModel", "kwargs": {"num_features": F, "num_classes": 5, "gru_size": 256}}
    assert training.DEFAULT_MODEL_DICT["kwargs"]["num_features"] == 10


def test_trainer_refuses_features_of_another_width():
    """The trainer's kernels read B x T x num_features floats: a batch of another width is an error, not a misread."""
    from medaka_b200 import training
    tr = object.__new__(training.GRUTrainer)           # the check runs before any device call
    tr.num_features, tr._tr = 10, None
    x = np.zeros((2, 50, 20), np.float32)
    y = np.zeros((2, 50), np.int64)
    for call in (lambda: tr.train_step((x, y)), lambda: tr.process_batch((x, y)), lambda: tr.forward_arrays(x)):
        with pytest.raises(ValueError, match=r"\[B, T, 10\]"):
            call()


# ---------------------------------------------------------------------------------------------- GPU: stage bars
def _wave():
    from medaka_b200 import models
    m = models.GRUModel(num_features=10, gru_size=H)
    try:
        return m.preferred_batch_size()
    finally:
        m.close()


def _check(got, want, label, bars=BARS):
    """got: device stages of some windows (h0 / h1 optional); want: the oracle's of the same windows."""
    err = {k: float(_scaled(k, got[k], want[k]).max()) for k in STAGES if k in got}
    print("gru256-shapes %s: %s" % (label, " ".join("%s=%.3g" % kv for kv in err.items())))
    for k, e in err.items():
        assert np.isfinite(got[k]).all(), (label, k)
        assert e <= bars[k], (label, k, e, bars[k])
    decided = _decided(want["probs"])
    assert np.array_equal(got["labels"][decided], np.argmax(want["probs"], -1)[decided]), label


def _device(sd, F, precision, x, windows, activations=True):
    """The forward of all of x; stages of `windows` (h0 and h1 only for a call of one group)."""
    m = _model(sd, F, precision)
    try:
        out = m.forward_arrays(x, want_logits=True, want_labels=True)
        assert np.array_equal(out.labels, np.argmax(out.probs, -1))
        got = {"logits": out.logits[windows], "probs": out.probs[windows], "labels": out.labels[windows]}
        if activations:
            got["h0"] = np.concatenate([m.read_activation(0, w, 1) for w in windows])
            got["h1"] = np.concatenate([m.read_activation(1, w, 1) for w in windows])
    finally:
        m.close()
    return got


RAGGED = [(F, B, T) for F in (1, 3, 9, 16, 17, 20, 21, 30, 40, 64, 129, 1024) for B in (1, 15, 17, 37)
          for T in (1, 2, 129) if F < 1024 or B <= 17]


@pytest.mark.gpu
@pytest.mark.parametrize("F,B,T", RAGGED)
def test_ragged_at_every_width(F, B, T):
    """A partial last 16-window tile (15, 17, 37), a partial last 8-window CTA of the fp32 recurrence (15, 17, 37),
    T = 1 (no prefetch step), and every layer-0 kernel at 256: inproj0_kernel<20> and the generic one."""
    sd = _sd(50 + F, F)
    x = _x(F, B, T, seed=1000 * F + T)
    windows = list(range(B))
    want = gru_oracle.stages(sd, x)
    for precision in ("tc", "fp32"):
        _check(_device(sd, F, precision, x, windows), want, "ragged F=%d B=%d T=%d %s" % (F, B, T, precision))


@pytest.fixture(scope="module")
def long_case():
    """long_case(F, weights): one wave x 10 000 columns, the windows test_gru256's one-wave test checks and their
    float64 stages (the latest case only is kept)."""
    cache = {}

    def get(F, weights):
        if (F, weights) not in cache:
            cache.clear()
            B = _wave()
            sd = _sd(60 + F, F, **WEIGHTS[weights])
            x = _x(F, B, LONG_T, seed=60 + F)
            picks = sorted({0, 15, 16, B // 2 - 1, B // 2, B - 16, B - 1})
            cache[F, weights] = sd, x, picks, gru_oracle.stages(sd, x[picks])
        return cache[F, weights]
    yield get
    cache.clear()


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["tc", "fp32"])
@pytest.mark.parametrize("weights", list(WEIGHTS))
@pytest.mark.parametrize("F", sorted(LONG_WIDTHS))
def test_long_windows_at_new_widths(long_case, F, weights, precision):
    """10 000 steps at F = 40 (four datatypes, the generic projection on featuriser-like counts) and F = 17 (the
    generic projection on unnormalised input)."""
    _need_memory(25)
    sd, x, picks, want = long_case(F, weights)
    _check(_device(sd, F, precision, x, picks), want, "long F=%d %s %s" % (F, weights, precision), LONG_BARS)


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["tc", "fp32"])
@pytest.mark.parametrize("extra", [-1, 0, 1, None], ids=["wave-1", "wave", "wave+1", "2wave+1"])
def test_across_the_wave_and_the_group(extra, precision):
    """Calls of one wave minus one, one wave, one wave plus one and two waves plus one (239 to 481 windows on an H100)
    are cut into one-wave groups: the windows on both sides of every group boundary against the oracle."""
    wave = _wave()
    B = 2 * wave + 1 if extra is None else wave + extra
    windows = sorted({w for w in (0, wave - 1, wave, 2 * wave - 1, 2 * wave, B - 1) if w < B})
    sd = _sd(70, 10)
    x = _features(B, 300, 10, seed=70 + B)
    want = gru_oracle.stages(sd, x[windows])
    _check(_device(sd, 10, precision, x, windows, activations=B <= wave), want, "B=%d %s" % (B, precision))


# ---------------------------------------------------------------------------------------------- GPU: placement
def _same(a, b, what):
    for k in ("probs", "logits", "labels"):
        if a.get(k) is not None and b.get(k) is not None:
            assert np.array_equal(a[k], b[k]), (what, k)


def _outs(out, idx):
    return {"probs": out.probs[idx], "logits": out.logits[idx], "labels": out.labels[idx]}


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["tc", "fp32"])
def test_windows_equal_wherever_they_run(precision):
    """Windows alone, in default one-wave groups, in one group of several cluster waves (3 x wave + 7 windows), and in a
    call of 2 x wave + 3 windows through forward_arrays, predict_async (batches that straddle groups) and
    mdk_engine_forward_dev (cut into one-wave groups, not run as one forward): bit for bit the same outputs."""
    from medaka_b200 import libmedaka as lm
    from tests.test_forward_dev import DevCall
    T = 300
    sd = _sd(80, 10)
    m = _model(sd, 10, precision)
    c = None
    try:
        wave = m.preferred_batch_size()
        x = _features(3 * wave + 7, T, 10, seed=80)
        idx = sorted({0, 15, 16, wave - 1, wave, wave + 1, 2 * wave - 1, 2 * wave + 2, 3 * wave + 6})
        alone = {w: _outs(m.forward_arrays(x[[w]], want_logits=True), 0) for w in idx}
        grouped = m.forward_arrays(x, want_logits=True)                       # one-wave groups
        m.set_group_windows(3 * wave + 7)
        big = m.forward_arrays(x, want_logits=True)                           # one group of several cluster waves
        m.set_group_windows(0)
        n = 2 * wave + 3
        part = m.forward_arrays(x[:n], want_logits=True)
        for w in idx:
            _same(alone[w], _outs(grouped, w), "one-wave group, window %d" % w)
            _same(alone[w], _outs(big, w), "3 x wave + 7 group, window %d" % w)
            if w < n:
                _same(alone[w], _outs(part, w), "2 x wave + 3 call, window %d" % w)

        m.reserve(wave, T)                  # groups collect calls up to one wave, so batches straddle them
        sizes = [70] * (n // 70) + [n % 70]
        starts = np.cumsum([0] + sizes)
        handles = []
        for s0, s1 in zip(starts[:-1], starts[1:]):
            class _B:
                counts_matrix = x[s0:s1]
            handles.append(m.predict_async(_B(), slots=len(sizes)))
        probs = np.concatenate([h.result().numpy() for h in handles])
        labels = np.concatenate([h.labels for h in handles])
        assert np.array_equal(probs, part.probs) and np.array_equal(labels, part.labels)

        per_forward = m.last_timings()["launches"]
        c = DevCall(np.ascontiguousarray(x[:n]), True)
        n0 = m.launch_count()
        c.run(m.engine)
        lm.check(lm.lib.mdk_engine_sync(m.engine))
        groups = (m.launch_count() - n0) / per_forward
        assert groups == -(-n // wave), "forward_dev ran %s groups, not %d one-wave groups" % (groups, -(-n // wave))
        dprobs, dlogits, dlabels = c.results()
        assert np.array_equal(dprobs, part.probs) and np.array_equal(dlogits, part.logits)
        assert np.array_equal(dlabels, part.labels)
    finally:
        if c is not None:
            c.free()
        m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["tc", "fp32"])
def test_decoded_heads_across_a_group_boundary_at_f40(precision):
    from tests.test_one_pass import _decode, _decoded
    from tests.test_one_pass_variants import _random_ref, _variant_decoded, _vd_of_probs
    F, T = 40, 137
    sd = _sd(81, F)
    m = _model(sd, F, precision)
    try:
        B = m.preferred_batch_size() + 9
        x = gru_oracle.featuriser_like_features(B, T, F, seed=81)
        probs = m.forward_arrays(x, want_labels=False).probs
        labels, quals = _decoded(m, x)
        want_l, want_q = _decode(probs)
        assert np.array_equal(labels, want_l) and np.array_equal(quals, want_q)
        ref = _random_ref(B, T, seed=3)
        calls, pq, rq = _variant_decoded(m, x, ref)
        wc, wpq, wrq = _vd_of_probs(probs, ref)
        assert np.array_equal(calls, wc)
        assert np.array_equal(pq, wpq) and np.array_equal(rq, wrq)
    finally:
        m.close()


# ---------------------------------------------------------------------------------------------- GPU: engine state
@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["tc", "fp32"])
@pytest.mark.parametrize("F", [10, 40])
def test_weight_reload(F, precision):
    """Model B loaded over model A after a forward: bit for bit a fresh model B's forward, activations included (the
    engine packs B's hi / lo planes again)."""
    sd_a, sd_b = _sd(1, F), _sd(2, F)
    x = _x(F, 37, 65, seed=9)

    def forward_b(first):
        m = _model(first, F, precision)
        try:
            if first is not sd_b:
                m.forward_arrays(x, want_logits=True)
                m.load_state_dict(sd_b)
            out = m.forward_arrays(x, want_logits=True, want_labels=True)
            return out.probs, out.logits, out.labels, m.read_activation(0), m.read_activation(1)
        finally:
            m.close()

    for reloaded, fresh in zip(forward_b(sd_a), forward_b(sd_b)):
        assert np.array_equal(reloaded, fresh)


@pytest.mark.gpu
@pytest.mark.parametrize("F,other", [(40, "F=10"), (40, "gru_size=128"), (10, "gru_size=128")])
def test_refused_state_dict_keeps_the_weights(F, other):
    from oracle import synth
    bad = (synth.synth_state_dict(101, num_features=10, gru_size=H) if other == "F=10"
           else synth.synth_state_dict(101, num_features=F, gru_size=128))
    m = _model(_sd(100, F), F)
    x = _x(F, 37, 65, seed=100)
    try:
        before = m.forward_arrays(x, want_logits=True)
        with pytest.raises(RuntimeError, match="size mismatch"):
            m.load_state_dict(bad)
        after = m.forward_arrays(x, want_logits=True)
    finally:
        m.close()
    for k in ("probs", "logits", "labels"):
        assert np.array_equal(getattr(before, k), getattr(after, k)), k


@pytest.mark.gpu
def test_workspace_budget_is_an_argument_error():
    """A 600 x 10 000 group asks for about 57 GiB of workspace: refused before any allocation, with the budget named.
    The engine then runs as before, and its timings cover only the groups that ran."""
    from medaka_b200 import libmedaka as lm
    from tests.test_forward_dev import _timings
    sd = _sd(110)
    small = _features(37, 300, 10, seed=110)
    m = _model(sd, 10)
    try:
        m.forward_arrays(small, want_logits=True)
        m.set_group_windows(600)
        with pytest.raises(lm.MedakaB200Error, match="48 GiB"):
            m.forward_arrays(_features(600, LONG_T, 10, seed=111))
        m.set_group_windows(0)
        got = m.forward_arrays(small, want_logits=True)
        two, many = _timings(m, 2), _timings(m, 8)
    finally:
        m.close()
    assert two == many, "a refused group was counted as a recorded forward"
    assert all(np.isfinite(v) and v >= 0 for v in many.values()), many
    fresh = _model(sd, 10)
    try:
        want = fresh.forward_arrays(small, want_logits=True)
    finally:
        fresh.close()
    for k in ("probs", "logits", "labels"):
        assert np.array_equal(getattr(got, k), getattr(want, k)), k


# ---------------------------------------------------------------------------------------------- GPU: trained models
@pytest.mark.gpu
@pytest.mark.parametrize("F,B,T", [(1, 3, 120), (21, 3, 120), (40, 3, 120), (10, 37, 40)])
def test_gradients_match_the_oracle(F, B, T):
    _parity(H, F, B, T)


@pytest.mark.gpu
@pytest.mark.parametrize("F", [1, 40])
def test_training_forward_equals_engine_fp32(F):
    from tests.test_training_gpu import test_training_forward_equals_engine_fp32 as check
    check(H, F)


def _write_store(path, n, T, F, seed):
    """A store of two-datatype counts (F = 20) whose labels are learnable: the argmax of the summed datatypes' first
    five features."""
    from medaka_b200 import common, datastore, features, labels
    x = gru_oracle.featuriser_like_features(n, T, F, seed=seed)
    with datastore.DataStore(path, "w") as ds:
        ds.set_meta(labels.HaploidLabelScheme(), "label_scheme")
        ds.set_meta(features.CountsFeatureEncoder(normalise="fwd_rev", dtypes=("r9", "r10")), "feature_encoder")
        for i in range(n):
            pos = np.zeros(T, dtype=[("major", int), ("minor", int)])
            pos["major"] = i * T + np.arange(T)
            y = (x[i, :, :5] + x[i, :, 10:15]).argmax(-1).astype(np.int64)
            ds.write_sample(common.Sample(ref_name="c", features=x[i], labels=y, ref_seq=None, positions=pos,
                                          label_probs=None, depth=None))
    return path


@pytest.mark.gpu
def test_run_training_default_model_at_f20(tmp_path):
    """No model file: DEFAULT_MODEL_DICT at the store's width (F = 20, gru_size 256), two epochs; model-1.tar.gz loads
    as that model, its fp32 forward is the trainer's bit for bit, and its tc forward is within the bars of the float64
    oracle on the trained weights."""
    import os
    from medaka_b200 import datastore, training
    F = 20
    store = _write_store(str(tmp_path / "train.npzstore"), 200, 100, F, 0)
    batcher = training.TrainBatcher([store], validation=0.2, seed=1, batch_size=20)
    out = str(tmp_path / "run")
    trainer = training.run_training(out, batcher, epochs=2, use_lr_schedule=False)
    try:
        assert (trainer.num_features, trainer.gru_size) == (F, H)
        trained = trainer.state_dict()
        x = gru_oracle.featuriser_like_features(3, 100, F, seed=9)
        want_probs, want_logits = trainer.forward_arrays(x)
    finally:
        trainer.close()
    m = datastore.ModelStoreTGZ(os.path.join(out, "model-1.tar.gz")).load_model()
    try:
        assert (m.num_features, m.gru_size) == (F, H)
        m.set_precision("fp32")
        got = m.forward_arrays(x, want_logits=True)
        assert np.array_equal(got.probs, want_probs) and np.array_equal(got.logits, want_logits)
        m.set_precision("tc")
        tc = m.forward_arrays(x, want_logits=True, want_labels=True)
        dev = {"logits": tc.logits, "probs": tc.probs, "labels": tc.labels, "h0": m.read_activation(0),
               "h1": m.read_activation(1)}
    finally:
        m.close()
    _check(dev, gru_oracle.stages(trained, x), "trained F=20 tc")
