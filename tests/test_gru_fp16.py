"""Consensus GRU in the fp16 mode (GRUModel.set_precision("fp16"), MDK_PREC_FP16): one fp16 product per tensor-core
contraction, the arithmetic medaka runs on a GPU without --full_precision.

Every stage is compared with tests/gru_fp16_oracle.stages, float64 with the mode's operands rounded to fp16 as the
kernels round them, fed the engine's own h0 and h1 (so fp16 rounding flips of h over 10 000 steps do not dominate), in
the scaling of tests/test_gru_stages.py (h0, h1, plog: max|d| / max|ref|; logits: per position / max_c|logit_c|;
probs: max|d|).  The bars sit between the device's error and every single-rounding effect (the oracle with one operand
left unrounded): a kernel that keeps a lo plane, or rounds an operand the mode leaves fp32, fails them.
"""
import numpy as np
import pytest
import torch

from oracle import gru_oracle, synth
from tests import gru_fp16_oracle
from tests.test_gru_stages import PROD_B, PROD_T, PROD_WINDOWS, WEIGHTS, _features, _need_memory, _plog_windows, _scaled

# Calibrated on an H100 80GB HBM3 (SXM, 700 W power limit) over every GPU case of this file; DESIGN §2 "GRU fp16 stage
# bars" has the table of worst device errors and smallest single-rounding effects.
# Each bar is at most a third of its stage's smallest single-rounding effect except at logits and probs, where the
# device's worst error (5.2e-6 at gru_size 256, F = 40; 6.3e-7) leaves a narrower window: there the other stages carry
# the discrimination, and test_single_rounding_effects_exceed_the_bars checks that they do.
BARS = {"h0": 9e-6, "h1": 9e-6, "plog": 7.5e-6, "logits": 1.6e-5, "probs": 2e-6}
STAGES = ("h0", "h1", "plog", "logits", "probs")
MARGIN = 1e-5


def _sd(weights, F=10, H=128, seed=21):
    return synth.synth_state_dict(seed, num_features=F, gru_size=H, **WEIGHTS[weights])


def _errors(got, want):
    return {k: float(_scaled(k, got[k], want[k]).max()) for k in STAGES if k in got and k in want}


def _check(got, want, label):
    err = _errors(got, want)
    print("gru-fp16 %s %s" % (label, " ".join("%s=%.3g" % (k, err[k]) for k in STAGES if k in err)))
    for k in err:
        assert np.isfinite(got[k]).all(), k
    for k, e in err.items():
        assert e <= BARS[k], (label, k, e, BARS[k])
    top2 = np.sort(want["probs"], -1)[..., -2:]
    decided = (top2[..., 1] - top2[..., 0]) > MARGIN
    assert np.array_equal(got["labels"][decided], np.argmax(want["probs"], -1)[decided]), label


def _model(sd, F, H=128, precision="fp16", rec="auto", keep=False):
    from medaka_b200 import models
    m = models.GRUModel(num_features=F, gru_size=H)
    m.load_state_dict(sd)
    m.set_precision(precision)
    if H == 128:
        m.set_rec_mode(rec)
    m.keep_activations(keep)
    return m


def _device(m, feats, windows, H):
    """One forward of all windows; h0, h1, logits, probs, labels of `windows`, and at gru_size 128 plog of the fused
    head (then a second forward keeping h1: its h0 must be bit-identical)."""
    m.set_group_windows(len(feats))
    out = m.forward_arrays(feats, want_logits=True, want_labels=True)
    w = list(windows)
    got = {"logits": out.logits[w], "probs": out.probs[w], "labels": out.labels[w]}
    got["h0"] = np.concatenate([m.read_activation(0, i, 1) for i in w])
    if H == 128:
        got["plog"] = _plog_windows(m.read_plog(), w)
        m.keep_activations(True)
        m.forward_arrays(feats)
        assert np.array_equal(np.concatenate([m.read_activation(0, i, 1) for i in w]), got["h0"])
        m.keep_activations(False)
    got["h1"] = np.concatenate([m.read_activation(1, i, 1) for i in w])
    return got


def _fed(sd, x, got):
    return gru_fp16_oracle.stages(sd, x, feed={"h0": got["h0"], "h1": got["h1"]}, device="cuda")


# ---------------------------------------------------------------------------------------------- CPU
def test_nothing_rounded_is_the_float64_forward():
    for H, F in ((128, 10), (128, 20), (256, 10)):
        sd = _sd("default", F, H, seed=4)
        x = gru_oracle.featuriser_like_features(2, 150, F, seed=4)
        got = gru_fp16_oracle.stages(sd, x, keep=gru_fp16_oracle.FP16_OPERANDS)
        want = gru_oracle.stages(sd, x)
        for k in STAGES:
            assert np.abs(got[k] - want[k]).max() <= 1e-12, (H, F, k)
        # fed its own stages, the oracle reproduces them
        ref = gru_fp16_oracle.stages(sd, x)
        fed = gru_fp16_oracle.stages(sd, x, feed=ref)
        for k in STAGES:
            assert np.abs(fed[k] - ref[k]).max() <= 1e-12, (H, F, k)


def test_operands_follow_the_kernels():
    """W_hh, h, W_ih1 and h0 at both widths; W_ih0 and x only where layer 0's projection runs on the tensor cores
    (gru_size 128, F <= 16).  Each listed operand changes the result, and the unlisted ones do not exist for the mode."""
    assert gru_fp16_oracle.operands(128, 10) == ("w_hh", "h", "w_ih1", "h0", "w_ih0", "x")
    assert gru_fp16_oracle.operands(128, 16) == gru_fp16_oracle.operands(128, 10)
    for H, F in ((128, 17), (128, 20), (256, 10), (256, 40)):
        assert gru_fp16_oracle.operands(H, F) == ("w_hh", "h", "w_ih1", "h0")
    for H, F in ((128, 10), (128, 20), (256, 10)):
        sd = _sd("default", F, H, seed=5)
        x = gru_oracle.featuriser_like_features(1, 60, F, seed=5)
        ref = gru_fp16_oracle.stages(sd, x)
        for op in gru_fp16_oracle.FP16_OPERANDS:
            alt = gru_fp16_oracle.stages(sd, x, keep=(op,))
            moved = np.abs(alt["h1"] - ref["h1"]).max() > 0
            assert moved == (op in gru_fp16_oracle.operands(H, F)), (H, F, op)
    # the weight rounding folds the gate scale in first: fp16(s w) / s, which is not fp16(w)
    w = np.random.RandomState(0).randn(384, 16).astype(np.float32) * 0.3
    r = gru_fp16_oracle.round_weight(w)
    assert np.abs(r - w.astype(np.float16).astype(np.float64)).max() > 0
    with pytest.raises(ValueError):
        gru_fp16_oracle.stages(sd, x, keep=("w_lo",))


def _effects(sd, x, H, F):
    """{operand: stage errors} of leaving one operand unrounded, each recurrence fed the mode's own stages (as the
    device comparisons are fed the engine's)."""
    ref = gru_fp16_oracle.stages(sd, x)
    return {op: _errors(gru_fp16_oracle.stages(sd, x, keep=(op,), feed=ref), ref)
            for op in gru_fp16_oracle.operands(H, F)}


@pytest.mark.parametrize("weights", sorted(WEIGHTS))
@pytest.mark.parametrize("H,F", [(128, 10), (128, 20), (256, 10), (256, 40)])
def test_single_rounding_effects_exceed_the_bars(H, F, weights):
    """Every single-rounding effect (a kernel that keeps one lo plane, i.e. runs tc under the fp16 name, or that rounds
    an operand one product fewer) moves some stage by more than 3x its bar, on 4 featuriser-like windows x 2000 steps."""
    sd = _sd(weights, F, H)
    x = gru_oracle.featuriser_like_features(4, 2000, F, seed=3)
    for op, err in _effects(sd, x, H, F).items():
        ratio = {k: err[k] / BARS[k] for k in err}
        print("gru-fp16-effect H=%d F=%d %-7s %-5s %s" % (H, F, weights, op, " ".join(
            "%s=%.3g (%.1fx)" % (k, err[k], ratio[k]) for k in STAGES if k in err)))
        assert max(ratio.values()) > 3, (H, F, weights, op, err)


# ---------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def production():
    """production(H, F, weights, rec): the fp16 engine's stages on a production group (gru_size 128: 1056 windows, 300
    at F = 20; 256: one wave) of 10 000 columns, with the features and state dict; computed once per case."""
    cache = {}

    def get(H, F, weights, rec="auto"):
        key = (H, F, weights, rec)
        if key not in cache:
            sd = _sd(weights, F, H, seed=31)
            if H == 128:
                B, windows = (PROD_B, PROD_WINDOWS) if F == 10 else (300, (0, 17, 150, 299))
            else:
                m = _model(sd, F, H)
                B = m.preferred_batch_size()
                m.close()
                windows = (0, 15, 16, B // 2, B - 16, B - 1)
            x = _features(B, PROD_T, F, windows, seed=31)
            m = _model(sd, F, H, rec=rec)
            got = _device(m, x, windows, H)
            m.close()
            cache[key] = sd, x[list(windows)], got
        return cache[key]
    yield get
    cache.clear()


@pytest.mark.gpu
@pytest.mark.parametrize("weights", sorted(WEIGHTS))
@pytest.mark.parametrize("rec", ["one", "pp"])
@pytest.mark.parametrize("F", [10, 20])
def test_stages_at_production_shapes_128(production, F, rec, weights):
    """gru_size 128, 10 000 columns: one and two tiles per CTA, F = 10 (layer 0's projection fused into the recurrence)
    and F = 20 (the CUDA-core projection)."""
    _need_memory(60)
    sd, x, got = production(128, F, weights, rec)
    _check(got, _fed(sd, x, got), "H=128 F=%d %s %s" % (F, rec, weights))


@pytest.mark.gpu
@pytest.mark.parametrize("weights", sorted(WEIGHTS))
@pytest.mark.parametrize("F", [10, 40])
def test_stages_at_production_shapes_256(production, F, weights):
    """gru_size 256: one wave of the cluster recurrence x 10 000 columns."""
    _need_memory(40)
    sd, x, got = production(256, F, weights)
    _check(got, _fed(sd, x, got), "H=256 F=%d %s" % (F, weights))


@pytest.mark.gpu
@pytest.mark.parametrize("H", [128, 256])
@pytest.mark.parametrize("B,T,F", [(37, 129, 17), (19, 2, 10), (21, 1, 10)])
def test_ragged_calls(H, B, T, F):
    """B not a multiple of 16, short T, and a generic feature width (17: layer 0 unfused at 128)."""
    sd = _sd("default", F, H, seed=33)
    x = synth.synth_features_fast(B, T, F, seed=33)
    windows = tuple(range(B))
    for rec in (("one", "pp") if H == 128 else ("auto",)):
        m = _model(sd, F, H, rec=rec)
        got = _device(m, x, windows, H)
        m.close()
        _check(got, _fed(sd, x, got), "ragged H=%d B=%d T=%d F=%d %s" % (H, B, T, F, rec))


@pytest.mark.gpu
@pytest.mark.parametrize("H", [128, 256])
def test_no_worse_than_the_reference_under_autocast(production, H):
    """The reference's class on CUDA under torch.autocast(float16), on the same windows: against the float64 forward the
    fp16 mode's max |dprob| is no larger than autocast's, and its labels equal float64's wherever the float64 top-2
    margin exceeds twice that max |dprob|."""
    sd, x, got = production(H, 10, "default", "one" if H == 128 else "auto")
    f64 = gru_fp16_oracle.stages(sd, x, keep=gru_fp16_oracle.FP16_OPERANDS, device="cuda")["probs"]
    ref = gru_oracle.build(sd, num_features=10, gru_size=H).cuda()
    with torch.inference_mode(), torch.autocast("cuda", dtype=torch.float16):
        half = ref(torch.as_tensor(x, device="cuda")).float().cpu().numpy()
    err16 = float(np.abs(got["probs"].astype(np.float64) - f64).max())
    err_ac = float(np.abs(half.astype(np.float64) - f64).max())
    top2 = np.sort(f64, -1)[..., -2:]
    decided = (top2[..., 1] - top2[..., 0]) > 2 * err16
    flips = int((got["labels"] != np.argmax(f64, -1))[decided].sum())
    flips_ac = int((np.argmax(half, -1) != np.argmax(f64, -1))[decided].sum())
    print("gru-fp16 vs float64 H=%d: fp16 mode %.3g (%d label flips), autocast %.3g (%d label flips)" % (
        H, err16, flips, err_ac, flips_ac))
    assert err16 <= err_ac
    assert flips == 0


@pytest.mark.gpu
@pytest.mark.parametrize("H,F", [(128, 10), (128, 20), (256, 10)])
def test_windows_are_independent_of_packing(H, F):
    """A window's fp16 outputs are bit-identical alone, packed in one group, across group boundaries, and through the
    host, device-resident and submit entry points."""
    from tests.test_forward_dev import DevCall
    from medaka_b200 import libmedaka as lm
    B, T = 40, 300
    x = synth.synth_features_fast(B, T, F, seed=50 + F)
    m = _model(_sd("default", F, H, seed=50), F, H)
    try:
        alone = [m.forward_arrays(x[i:i + 1], want_logits=True) for i in range(B)]
        want = {k: np.concatenate([getattr(a, k) for a in alone]) for k in ("probs", "logits", "labels")}
        whole = m.forward_arrays(x, want_logits=True)
        for k in want:
            assert np.array_equal(getattr(whole, k), want[k]), k
        m.reserve(B, T)
        m.set_group_windows(16)                                        # groups of 16: calls cut at 16 and 32
        assert np.array_equal(m.forward_arrays(x).probs, want["probs"])
        probs = [m.pinned("p%d" % i, (n, T, 5), np.float32) for i, n in enumerate((5, 20, 15))]
        feats = [m.pinned("x%d" % i, (n, T, F), np.float32) for i, n in enumerate((5, 20, 15))]
        tickets, lo = [], 0
        for xin, p in zip(feats, probs):                                # calls straddling the boundaries
            np.copyto(xin, x[lo:lo + len(xin)])
            tickets.append(m.submit_arrays(xin, p))
            lo += len(xin)
        for t in tickets:
            m.wait(t)
        assert np.array_equal(np.concatenate(probs), want["probs"])
        calls = [DevCall(x[a:b], True) for a, b in ((0, 7), (7, 33), (33, 40))]
        for c in calls:
            c.run(m.engine)
        lm.check(lm.lib.mdk_engine_sync(m.engine))
        got = [c.results() for c in calls]
        for c in calls:
            c.free()
        for i, k in enumerate(("probs", "logits", "labels")):
            assert np.array_equal(np.concatenate([g[i] for g in got]), want[k]), k
    finally:
        m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("H,F", [(128, 10), (128, 20), (256, 10)])
def test_decoded_heads_equal_decode_of_fp16_probabilities(H, F):
    """Quality bytes, call bytes and phreds of the decoded and variant-decoded heads in the fp16 mode are the decode of
    the fp16 probabilities."""
    from tests.test_one_pass import _decode, _decoded
    from tests.test_one_pass_variants import _random_ref, _variant_decoded, _vd_of_probs
    B, T = 19, 137
    x = synth.synth_features_fast(B, T, F, seed=60 + F)
    ref = _random_ref(B, T, seed=61)
    m = _model(_sd("default", F, H, seed=60), F, H)
    try:
        probs = m.forward_arrays(x).probs
        labels, quals = _decoded(m, x)
        want_labels, want_quals = _decode(probs)
        assert np.array_equal(labels, want_labels) and np.array_equal(quals, want_quals)
        for g, w in zip(_variant_decoded(m, x, ref), _vd_of_probs(probs, ref)):
            assert np.array_equal(g, w)
    finally:
        m.close()


@pytest.mark.gpu
def test_predict_consensus_and_variants_equal_two_pass_in_fp16(tmp_path):
    """predict_consensus and predict_variants with an fp16 model equal predict_regions + sequence / variants."""
    from medaka_b200 import common, features
    from tests.test_one_pass import _both, _draft, _pileup_source
    from tests.test_one_pass_variants import CONFIGS, _check as _check_variants
    m = _model(synth.synth_state_dict(2), 10)
    enc = features.CountsFeatureEncoder(normalise="total", pileup_source=_pileup_source)
    R = common.Region
    lengths = {"long": 7000, "gappy": 4200, "tiny": 600, "nodata": 300}
    bam_regions = [R("long", 0, 7000), R("gappy", 0, 4200), R("tiny", 0, 600)]
    try:
        for cfg in ({}, {"regions": ["long:1500-5200", R("tiny", None, None), "nodata"]}):
            (a, bed_a), (b, bed_b) = _both(str(tmp_path), m, enc, None, bam_regions, _draft(lengths), **cfg)
            assert len(a) > 1000 and a == b and bed_a == bed_b, cfg
        vdir = tmp_path / "variants"
        vdir.mkdir()
        _check_variants(m, enc, None, bam_regions, lengths, CONFIGS[:2], str(vdir))
    finally:
        m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("H", [128, 256])
def test_switching_precision(H):
    """tc -> fp16 -> tc on one engine gives tc results bit-identical to before; windows submitted before a switch run
    in the mode they were submitted in; a weight reload in fp16 equals a fresh fp16 engine; unknown modes are refused."""
    from medaka_b200 import libmedaka as lm
    B, T = 5, 200
    sd, sd2 = _sd("default", 10, H, seed=70), _sd("hot", 10, H, seed=71)
    x = synth.synth_features_fast(B, T, 10, seed=70)
    m = _model(sd, 10, H, precision="tc")
    try:
        with pytest.raises(ValueError, match="fp16"):
            m.set_precision("bf16")
        mode = lm.ffi.new("int *")
        assert lm.lib.mdk_engine_set_precision(m.engine, 3) == lm.lib.MDK_ERR_ARG
        lm.check(lm.lib.mdk_engine_get_precision(m.engine, mode))
        assert mode[0] == lm.lib.MDK_PREC_TC
        want_tc = m.forward_arrays(x).probs
        m.set_precision("fp16")
        lm.check(lm.lib.mdk_engine_get_precision(m.engine, mode))
        assert mode[0] == lm.lib.MDK_PREC_FP16 == 2
        want_fp16 = m.forward_arrays(x).probs
        assert not np.array_equal(want_tc, want_fp16)
        m.set_precision("tc")
        assert np.array_equal(m.forward_arrays(x).probs, want_tc)
        # queued: each 5-window call waits in the open group while the mode changes
        m.reserve(64, T)
        m.set_group_windows(64)
        feats = [m.pinned("q%d" % i, (B, T, 10), np.float32) for i in range(3)]
        probs = [m.pinned("qp%d" % i, (B, T, 5), np.float32) for i in range(3)]
        tickets = []
        for i, mode_name in enumerate(("fp16", "tc", "fp16")):
            np.copyto(feats[i], x)
            tickets.append(m.submit_arrays(feats[i], probs[i]))
            m.set_precision(mode_name)
        for t in tickets:
            m.wait(t)
        assert np.array_equal(probs[0], want_tc)
        assert np.array_equal(probs[1], want_fp16)
        assert np.array_equal(probs[2], want_tc)
        # weight reload in fp16
        m.load_state_dict(sd2)
        reloaded = m.forward_arrays(x).probs
        fresh = _model(sd2, 10, H)
        assert np.array_equal(reloaded, fresh.forward_arrays(x).probs)
        fresh.close()
    finally:
        m.close()
