"""Consensus GRU at feature widths other than the production ones: every F from 1 to 1024 is accepted by
mdk_engine_create, and F picks layer 0's input projection.

  F        tc path                                           fp32 path
  1 - 16   fused into rec_tc_kernel (FUSE_X: x staged as an  inproj0_generic_kernel (inproj0_kernel<10> at F = 10)
           fp16 hi / lo B tile, W_ih packed as w_x_tm, K
           zero-padded to 16)
  20       inproj0_kernel<20>, gi in the quad layout         inproj0_kernel<20>
  others   inproj0_generic_kernel, gi in the quad layout     inproj0_generic_kernel, gi in rows

The fused path has F-dependent logic that F = 10 cannot check: thread entry q = tid + 256 m stages (window q / F,
feature q % F), features 8-15 go to the second k-group, at two tiles per CTA the second entry is partly populated, the
feature strides of the first load and of the next step's prefetch are multiples of F, and W_ih and the x tile are
zero beyond F.  So the fused widths cover one feature, each side of the k-group boundary, a partly populated second
entry (F = 15: 480 of 512) and a full K = 16 tile; the generic widths cover the first width past the fused path
(17), widths under 10 on the fp32 path (3), a width that is not a multiple of 4 (21), widths in the hundreds and the
ABI's maximum (1024, at small shapes only).

Every device stage is held to the bars of tests/test_gru_stages.py against the float64 oracle.  The features are
unnormalised cubed uniforms: at small F, row-normalised counts are fp16-exact (at F = 1 every x is 1) and a kernel
that lost the x lo plane would not show.
"""
import numpy as np
import pytest

from oracle import gru_oracle, synth
from tests import test_gpu_parity, test_gru_pack
from tests.test_gru_pack import driver  # noqa: F401  (the packer's native driver, a fixture)
from tests.test_gru_stages import (BARS, PROD_B, PROD_T, PROD_WINDOWS, STAGES, _check, _device, _errors, _model,
                                   _need_memory, _sd)

FUSED = (1, 2, 7, 8, 9, 11, 15, 16)
GENERIC = (3, 17, 21, 64, 129, 1024)
WIDTHS = FUSED + GENERIC
PATHS = [("tc", "one"), ("tc", "pp"), ("fp32", "auto")]
PATH_IDS = ["tc-one_tile", "tc-two_tiles", "fp32"]


def _features(B, T, F, seed):
    """float32 [B, T, F]: cubed uniforms in [0, 1), not normalised (most of them fp16 cannot hold at any F), with 2 % of
    the columns all zero (coverage gaps)."""
    rng = np.random.default_rng(seed)
    x = rng.random((B, T, F), dtype=np.float32)
    x *= x * x
    x[rng.random((B, T)) < 0.02] = 0.0
    return x


# ---------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("F", WIDTHS)
def test_features_are_not_fp16_exact(F):
    """Rounding these features to fp16 is a visible error at every width, so the x hi / lo split is exercised."""
    x = _features(8, 300, F, seed=F)
    assert x.shape == (8, 300, F) and x.dtype == np.float32 and x.min() >= 0 and x.max() < 1
    assert (x.sum(-1) == 0).any() and (x.sum(-1) > 0).mean() > 0.9
    v = x[x > 0]
    assert (v.astype(np.float16).astype(np.float32) != v).mean() > 0.9
    if F > 1:
        assert np.abs(x.sum(-1)[x.sum(-1) > 0] - 1).max() > 0.1          # not row-normalised


@pytest.mark.parametrize("weights", ["default", "hot"])
@pytest.mark.parametrize("F", FUSED)
def test_ablations_exceed_the_bars_fused(F, weights):
    """At every fused width each lost product of the tensor-core path (gru_oracle.ablate, all six apply: the layer-0
    projection runs on the tensor cores) moves some stage by more than 3x its bar, on 4 windows x 2000 steps."""
    sd = _sd(weights, F=F)
    x = _features(4, 2000, F, seed=3)
    ref = gru_oracle.stages(sd, x)
    for which in gru_oracle.ABLATIONS:
        sd_a, kw = gru_oracle.ablate(sd, which)
        err = _errors(gru_oracle.stages(sd_a, x, **kw), ref)
        ratio = {k: err[k] / BARS[k] for k in STAGES}
        print("gru-ablation F=%-2d %-7s %-5s %s" % (F, weights, which, " ".join("%s=%.3g (%.1fx)" % (k, err[k], ratio[k])
                                                                                for k in STAGES)))
        assert max(ratio.values()) > 3, (F, weights, which, err)


@pytest.mark.parametrize("F", [1, 9, 16, 17])
def test_gru_pack_layouts_at_unusual_widths(driver, tmp_path, F):  # noqa: F811
    """The host packer: every array bit for bit as test_gru_pack checks it; w_x_tm exists exactly when F <= 16, is zero
    beyond F, and its hi + lo is W_ih * gate_scale to the precision of an fp16 pair."""
    test_gru_pack.test_gru_pack_layouts(driver, tmp_path, F)
    sd = synth.synth_state_dict(3, num_features=F)
    w_x_tm = test_gru_pack._pack(driver, sd, F, tmp_path)[0]["w_x_tm"]
    assert (w_x_tm.size > 0) == (F <= 16)
    if F > 16:
        return
    w = w_x_tm.reshape(2, 2, 3, test_gru_pack.H, 16).astype(np.float64)
    assert not w[..., F:].any()
    want = np.stack([sd["gru.weight_ih_l0%s" % s].astype(np.float64).reshape(3, test_gru_pack.H, F)
                     * test_gru_pack.SCALE[:, None, None] for s in ("", "_reverse")])
    d = np.abs(w[:, 0, ..., :F] + w[:, 1, ..., :F] - want)
    assert (d <= 2.0 ** -21 * np.abs(want) + 2.0 ** -25).all(), float(d.max())
    assert (w[:, 1, ..., :F] != 0).mean() > 0.9                         # the lo plane carries the residual


# ---------------------------------------------------------------------------------------------- GPU: stage bars
def _ragged_windows(B):
    """All windows of the 37-window call; at 1217 windows a tile's first and last, the next tile and the call's last."""
    return tuple(range(37)) if B == 37 else (0, 15, 16, 1200, 1215, 1216)


@pytest.mark.gpu
@pytest.mark.parametrize("T", [1, 2, 129])
@pytest.mark.parametrize("B", [37, 1217])
@pytest.mark.parametrize("F", WIDTHS)
def test_ragged_at_every_width(F, B, T):
    """Partial tiles (37 windows: the last tile holds 5), 1217 windows (77 tiles: at two tiles per CTA the last CTA has
    no second tile), T = 1 (no prefetch step), T = 2 and T = 129, both directions; tc at one and two tiles per CTA,
    fused head and kept activations (h1 and the head as its own kernel), and the fp32 path."""
    if F == 1024 and B * T > 37 * 129:
        pytest.skip("F = 1024 runs at small shapes only")
    windows = _ragged_windows(B)
    sd = _sd("default", F=F, seed=50 + F)
    x = _features(B, T, F, seed=1000 * F + T)
    want = gru_oracle.stages(sd, x[list(windows)])
    for path, rec, keep in (("tc", "one", False), ("tc", "one", True), ("tc", "pp", False), ("tc", "pp", True),
                            ("fp32", "auto", False)):
        m = _model(sd, F, path, rec, keep)
        try:
            got = _device(m, x, windows, path == "tc" and not keep)
        finally:
            m.close()
        _check(got, want, "ragged F=%d B=%d T=%d %s %s keep=%d" % (F, B, T, path, rec, keep))


@pytest.fixture(scope="module")
def long_case():
    """long_case(F, weights): 300 windows x 10 000 columns and the float64 stages of four of them (the latest case
    only is kept: the tests that share one run back to back)."""
    cache = {}

    def get(F, weights):
        if (F, weights) not in cache:
            cache.clear()
            windows = (0, 17, 150, 299)
            sd = _sd(weights, F=F, seed=60 + F)
            x = _features(300, 10000, F, seed=60 + F)
            cache[F, weights] = sd, x, windows, gru_oracle.stages(sd, x[list(windows)])
        return cache[F, weights]
    yield get
    cache.clear()


def _run_kept_and_not(sd, F, x, windows, want, label, path, rec):
    for keep in (False, True):
        m = _model(sd, F, path, rec, keep)
        try:
            got = _device(m, x, windows, path == "tc" and not keep)
        finally:
            m.close()
        _check(got, want, "%s %s %s keep=%d" % (label, path, rec, keep))


@pytest.mark.gpu
@pytest.mark.parametrize("path,rec", PATHS, ids=PATH_IDS)
@pytest.mark.parametrize("weights", ["default", "hot"])
@pytest.mark.parametrize("F", [9, 16, 17])
def test_long_windows(long_case, F, weights, path, rec):
    """10 000 steps on each side of the fused / generic boundary, with and without kept activations."""
    _need_memory(20)
    sd, x, windows, want = long_case(F, weights)
    _run_kept_and_not(sd, F, x, windows, want, "long F=%d %s" % (F, weights), path, rec)


@pytest.fixture(scope="module")
def full_group_f16():
    cache = {}

    def get():
        if not cache:
            sd = _sd("default", F=16, seed=70)
            x = _features(PROD_B, PROD_T, 16, seed=70)
            cache["v"] = sd, x, gru_oracle.stages(sd, x[list(PROD_WINDOWS)])
        return cache["v"]
    yield get
    cache.clear()


@pytest.mark.gpu
@pytest.mark.parametrize("rec", ["one", "pp"], ids=["one_tile", "two_tiles"])
def test_full_group_f16(full_group_f16, rec):
    """One group of 1056 windows x 10 000 columns at F = 16, the widest fused x tile (both k-groups full)."""
    _need_memory(60)
    sd, x, want = full_group_f16()
    _run_kept_and_not(sd, 16, x, PROD_WINDOWS, want, "full F=16", "tc", rec)


# ---------------------------------------------------------------------------------------------- GPU: placement
GROUP = 1056
PLACED = (0, 17, 520, 530, 1055)      # tiles 0, 1, 32, 33 and 65: both tile slots of a CTA, and the last CTA
FILL = 20                             # windows ahead of the target in the ragged call: window 4 of a 5-window tile


def _placed(m, x, idx):
    m.set_group_windows(len(x))
    out = m.forward_arrays(x, want_logits=False, want_labels=True)
    plog = m.read_plog()
    return [{"h0": m.read_activation(0, i, 1)[0], "plog": plog[:, i // 16, :, :, i % 16], "labels": out.labels[i]}
            for i in idx]


@pytest.mark.gpu
@pytest.mark.parametrize("rec", ["one", "pp"])
@pytest.mark.parametrize("T", [1, 2, 9, 129])
@pytest.mark.parametrize("F", [9, 16])
def test_placement_independence(F, T, rec):
    """As tests/test_rec_step.py at F = 10: a window's h0, partial logits and labels are bit-identical alone, at slot 4
    of a ragged tile and inside a full group, and the group's h0 and plog are within the bars."""
    sd = synth.synth_state_dict(80 + F, num_features=F)
    x = _features(GROUP, T, F, seed=80 + F + T)
    m = _model(sd, F, "tc", rec)
    try:
        group = _placed(m, x, PLACED)
        for k, w in enumerate(PLACED):
            alone = _placed(m, x[[w]], [0])[0]
            ragged = _placed(m, np.concatenate([x[1030:1030 + FILL], x[[w]]]), [FILL])[0]
            for name in ("h0", "plog", "labels"):
                assert np.array_equal(alone[name], group[k][name]), (w, name, "alone")
                assert np.array_equal(ragged[name], group[k][name]), (w, name, "ragged")
    finally:
        m.close()
    want = gru_oracle.stages(sd, x[list(PLACED)])
    got = {"h0": np.stack([g["h0"] for g in group]),
           "plog": np.stack([g["plog"].transpose(1, 0, 2) for g in group])}
    for name, v in got.items():
        err = float(np.abs(v.astype(np.float64) - want[name]).max() / np.abs(want[name]).max())
        assert err <= BARS[name], (F, T, rec, name, err)


# ---------------------------------------------------------------------------------------------- GPU: engine plumbing
def _gru(F, seed, precision="tc"):
    from medaka_b200 import models
    m = models.GRUModel(num_features=F)
    m.load_state_dict(synth.synth_state_dict(seed, num_features=F))
    m.set_precision(precision)
    return m


@pytest.mark.gpu
@pytest.mark.parametrize("F", [16, 17])
def test_pipelined_groups(F):
    """forward_dev and decoded calls packed into 48-window groups across group boundaries, a T change, a small-lane
    call and a workspace regrowth: every call bit-identical to its lone forward.  At F = 16 layer 0 is fused and runs
    beside the previous group's layer 1; at F = 17 its generic projection waits for it."""
    from tests.test_layer_overlap import _pipelined
    m = _gru(F, 90 + F)
    try:
        _pipelined(m, [(100, 3000), (90, 3000), (1, 500), (120, 2700), (70, 3000), (60, 3200)], 90 + F,
                   decoded=(1, 4))
    finally:
        m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["tc", "fp32"])
def test_calls_beyond_the_staging_capacity_at_f1024(precision):
    """At F = 1024 a lane's staging holds a few windows only: calls that do not fit what is left of the open group are
    split across groups, and a call larger than the whole reservation regrows it.  Every call equals its lone forward
    bit for bit, and the split call is within the bars."""
    from medaka_b200 import libmedaka as lm
    from tests.test_forward_dev import DevCall
    F, T = 1024, 200
    m = _gru(F, 99, precision)
    plan = [(6, T), (11, T), (3, T), (9, T), (4, 150)]
    feats = [_features(b, t, F, seed=990 + i) for i, (b, t) in enumerate(plan)]
    calls = []
    try:
        want = [m.forward_arrays(x, want_logits=True) for x in feats]
        m.reserve(8, T)
        m.set_group_windows(64)
        calls = [DevCall(x, True) for x in feats]
        for c in calls:
            c.run(m.engine)
        lm.check(lm.lib.mdk_engine_sync(m.engine))
        for i, (c, w) in enumerate(zip(calls, want)):
            probs, logits, labels = c.results()
            assert np.array_equal(probs, w.probs), "call %d: probabilities differ" % i
            assert np.array_equal(logits, w.logits), "call %d: logits differ" % i
            assert np.array_equal(labels, w.labels), "call %d: labels differ" % i
        probs, logits, labels = calls[1].results()
        sd = synth.synth_state_dict(99, num_features=F)
        _check({"probs": probs, "logits": logits, "labels": labels}, gru_oracle.stages(sd, feats[1]),
               "split F=1024 %s" % precision)
    finally:
        for c in calls:
            c.free()
        m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp32", "tc"])
@pytest.mark.parametrize("F", [9, 17])
def test_weight_reload(F, precision):
    """A model loaded over another: bit for bit a fresh model's forward, activations included."""
    test_gpu_parity.test_weight_reload_matches_fresh_model(precision, F)


@pytest.mark.gpu
@pytest.mark.parametrize("F,other", [(16, 17), (17, 16), (9, 10), (1, 1024)])
def test_state_dict_of_another_width_is_refused(F, other):
    """Loading a state dict of another feature width raises, and the engine keeps the weights it had: its forward is
    bit for bit the one before the attempt."""
    m = _gru(F, 100)
    x = _features(37, 65, F, seed=100)
    try:
        before = m.forward_arrays(x, want_logits=True)
        with pytest.raises(RuntimeError, match="size mismatch"):
            m.load_state_dict(synth.synth_state_dict(101, num_features=other))
        after = m.forward_arrays(x, want_logits=True)
    finally:
        m.close()
    for k in ("probs", "logits", "labels"):
        assert np.array_equal(getattr(before, k), getattr(after, k)), k
