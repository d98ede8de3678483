"""Read-level models in the fp16 mode (LatentSpaceLSTM.set_precision("fp16"), mdk_rl_set_conv bit 2): every
tensor-core contraction takes the single product hi.hi, operands rounded to the nearest fp16 with fp32 accumulation -
the arithmetic of medaka's own GPU default (model.half() under autocast), with fp32 activations in between.

Its target is rl_fp16_oracle.stages(..., feed=the engine's stages): float64 arithmetic on the operands the mode
rounds, each LSTM layer fed the engine's own input and previous h.  A free-running target would not do: an fp32-level
difference in h that lands on an fp16 rounding boundary moves the rounded h by a whole fp16 unit, and at 10 000 steps
such flips moved h1 and probs as much as leaving h unrounded does (1e-4).  Stages are compared as in
test_read_level_production.py (z, h0, h1 as max|d| / max|ref|, probs as max|d|), against bars of their own:
  - each bar is at most a third of the smallest single-rounding effect at its stage (one operand left unrounded, judged
    the way the engine is: test_single_roundings_exceed_the_bars), so a kernel that kept a product it should drop, or
    dropped a rounding, fails;
  - the fp16 oracle lies far outside the fp32-faithful path's bars (test_fp16_oracle_lies_outside_the_tc_bars), and a
    kernel that silently ran three products fails this file's bars.
"""
import numpy as np
import pytest

from oracle import rl_oracle
from tests import rl_fp16_oracle
from tests.test_read_level_production import BARS as TC_BARS
from tests.test_read_level_production import MODELS, PROD_D, PROD_P, STAGES, _block_report, _errors

# Calibrated on an H100 80GB HBM3 (SXM, 700 W power limit) over every GPU case of this file (DESIGN §2 "Read-level fp16
# bars").  Worst device error z / h0 / h1 (relative) / probs (absolute): 3.9e-6 / 1.0e-6 / 1.3e-6 / 5.9e-7.  Smallest
# single-rounding effects: z 6.7e-5 (y1), h0 8.9e-5 (h at 384), h1 5.6e-5 (W_hh at 128), probs 1.6e-5 (W_hh at 128).
# Each bar is at least 3x the worst error and at most a third of the smallest effect.
BARS = {"z": 1.5e-5, "h0": 1e-5, "h1": 8e-6, "probs": 4e-6}
PROD_B = 17                             # a full 16-window tile and a partial one
PROD_WINDOWS = (0, 15, 16)


def _check(got, want, label=""):
    err = _errors(got, want)
    print("rl-fp16 %s %s" % (label, " ".join("%s=%.3g" % (k, err[k]) for k in STAGES if k in err)))
    for k, e in err.items():
        assert np.isfinite(got[k]).all(), k
        assert e <= BARS[k], (k, e, BARS[k])
    return err


def _sd(H, seed, use_dwells=True):
    return rl_oracle.synth_rl_state_dict(seed, lstm_size=H, use_dwells=use_dwells)


def _model(sd, H, use_dwells=True, precision="fp16"):
    from medaka_b200 import read_level
    m = read_level.LatentSpaceLSTM(lstm_size=H, use_dwells=use_dwells)
    m.load_state_dict(sd)
    m.set_precision(precision)
    return m


# ---------------------------------------------------------------------------------------------- CPU
def _reduced(H):
    """A reduced production case: one window of 2 000 positions x 40 featuriser-like reads, dwell model."""
    sd = _sd(H, 31)
    return rl_oracle.build(sd, use_dwells=True), rl_oracle.featuriser_like_rl_features(1, 2000, 40, F=5, seed=H)


def _judged(m, x, got):
    """got's errors against the fp16 oracle fed got's stages: how the GPU tests judge the engine."""
    return _errors(got, rl_fp16_oracle.stages(m, x, feed=got))


@pytest.mark.parametrize("H", [128, 384])
def test_fp16_oracle_lies_outside_the_tc_bars(H):
    """The fp32 forward (what a three-product kernel computes) judged against the fp16 oracle: beyond 5x the tc bar at
    every stage, and beyond 3x this file's bar at every stage of the LSTM, so a kernel that ran three products in the fp16
    mode fails here."""
    m, x = _reduced(H)
    err = _judged(m, x, rl_oracle.stages(m, x))
    print("rl-fp16 oracle vs fp32 H=%d %s" % (H, " ".join("%s=%.3g" % (k, err[k]) for k in STAGES)))
    assert all(err[k] > 5 * TC_BARS[k] for k in STAGES), err
    assert all(err[k] > 3 * BARS[k] for k in STAGES), err


@pytest.mark.parametrize("H", [128, 384])
def test_single_roundings_exceed_the_bars(H):
    """Each operand the mode rounds, left unrounded on its own, moves some stage by more than 3x its bar, judged as the
    engine is."""
    m, x = _reduced(H)
    for op in rl_fp16_oracle.operands(H):
        err = _judged(m, x, rl_fp16_oracle.stages(m, x, keep=(op,)))
        ratio = {k: err[k] / BARS[k] for k in STAGES}
        print("rl-fp16 keep H=%d %-6s %s" % (H, op, " ".join("%s=%.3g (%.1fx)" % (k, err[k], ratio[k]) for k in STAGES)))
        assert max(ratio.values()) > 3, (op, err)


def test_oracle_operands_follow_the_kernels():
    """At lstm_size 128 the input projections stay fp32 (gemm_fp32_kernel): W_ih and their inputs are not rounded."""
    assert set(rl_fp16_oracle.operands(128)) == {"conv17", "y1", "w_hh", "h"}
    assert set(rl_fp16_oracle.operands(384)) == {"conv17", "y1", "w_hh", "h", "w_ih", "x"}


# ---------------------------------------------------------------------------------------------- GPU
def _f64_target(sd, dw, x, got):
    """The fp16 oracle of x, its LSTM layers fed the engine's inputs and h (rl_fp16_oracle.stages)."""
    return rl_fp16_oracle.stages(rl_oracle.build(sd, use_dwells=dw), x, device="cuda", feed=got)


@pytest.fixture(scope="module")
def production():
    """production(H, model): 17 windows of 10 000 positions x 100 featuriser-like reads through one fp16 device call;
    the device's stages of PROD_WINDOWS with the fp16 oracle's, the float64 forward's and the reference class's
    probabilities under torch.autocast.  Computed once per (H, model)."""
    cache = {}

    def get(H, model):
        if (H, model) not in cache:
            import torch
            dw, F = MODELS[model]
            sd = _sd(H, 31, dw)
            x = rl_oracle.featuriser_like_rl_features(PROD_B, PROD_P, PROD_D, F=F, seed=H + F + 7 * dw)
            m = _model(sd, H, dw)
            assert m.windows_per_call(PROD_P, PROD_D, F) >= PROD_B
            probs = m.forward_arrays(x)
            w = list(PROD_WINDOWS)
            got = {k: m.read_stage(k)[w] for k in ("z", "h0", "h1")}
            got["probs"] = probs[w]
            m.close()
            ref = rl_oracle.build(sd, use_dwells=dw)
            want = rl_fp16_oracle.stages(ref, x[w], device="cuda", feed=got)
            f64 = rl_fp16_oracle.stages(ref, x[w], keep=rl_fp16_oracle.FP16_OPERANDS, device="cuda")["probs"]
            half = []
            ref = ref.cuda()
            with torch.inference_mode(), torch.autocast("cuda", dtype=torch.float16):
                for b in w:
                    half.append(ref(torch.from_numpy(x[b:b + 1]).cuda()).float().cpu().numpy()[0])
            cache[H, model] = got, want, f64, np.stack(half)
            torch.cuda.empty_cache()
        return cache[H, model]
    yield get
    cache.clear()


@pytest.mark.gpu
@pytest.mark.parametrize("model", sorted(MODELS))
@pytest.mark.parametrize("case", ["small", "production"])
@pytest.mark.parametrize("H", [128, 384])
def test_stages_match_fp16_oracle(production, H, case, model):
    """z, h0, h1 and the probabilities of one fp16 device call against the fp16 oracle: 18 windows of 300 positions x 97
    reads (a full tile and a partial one), or windows 0, 15 and 16 of 17 at the production shape."""
    label = "stages H=%d %s %s" % (H, case, model)
    if case == "production":
        got, want, _, _ = production(H, model)
        _block_report(got, want, label)
    else:
        dw, F = MODELS[model]
        sd = _sd(H, 41, dw)
        x = rl_oracle.featuriser_like_rl_features(18, 300, 97, F=F, seed=41 + H)
        m = _model(sd, H, dw)
        probs = m.forward_arrays(x)
        got = {k: m.read_stage(k) for k in ("z", "h0", "h1")}
        got["probs"] = probs
        m.close()
        want = _f64_target(sd, dw, x, got)
    _check(got, want, label)


@pytest.mark.gpu
@pytest.mark.parametrize("model", sorted(MODELS))
@pytest.mark.parametrize("H", [128, 384])
def test_no_worse_than_the_reference_under_autocast(production, H, model):
    """The reference's own half path - its class on CUDA under torch.autocast(float16) - on the same windows: against
    the float64 forward, the fp16 mode's max |dprob| is no larger than autocast's, and its labels equal float64's
    wherever the float64 top-2 margin exceeds twice that max |dprob|.  (The mode's own roundings move the
    probabilities by up to 4e-4 at lstm_size 384, so below that margin they may flip a label, as autocast's do.)"""
    got, _, f64, half = production(H, model)
    err16 = float(np.abs(got["probs"].astype(np.float64) - f64).max())
    err_ac = float(np.abs(half.astype(np.float64) - f64).max())
    top2 = np.sort(f64, -1)[..., -2:]
    decided = (top2[..., 1] - top2[..., 0]) > 2 * err16
    flips = int((np.argmax(got["probs"], -1) != np.argmax(f64, -1))[decided].sum())
    flips_ac = int((np.argmax(half, -1) != np.argmax(f64, -1))[decided].sum())
    print("rl-fp16 vs float64 H=%d %s: fp16 mode %.3g (%d label flips), autocast %.3g (%d label flips)" % (
        H, model, err16, flips, err_ac, flips_ac))
    assert err16 <= err_ac
    assert flips == 0


@pytest.mark.gpu
@pytest.mark.parametrize("H", [128, 384])
def test_windows_are_independent_of_packing(H):
    """Windows give bit-identical fp16 results run alone, packed across calls into 16-window groups (calls split
    across groups), and in ragged calls of another read depth."""
    from tests.test_read_level_one_pass import _submit_probs
    P = 150
    sd = _sd(H, 50)
    xa = rl_oracle.featuriser_like_rl_features(37, P, 9, F=5, seed=50)
    xb = rl_oracle.featuriser_like_rl_features(6, P, 4, F=5, seed=51)
    m = _model(sd, H)
    try:
        alone_a = np.concatenate([m.forward_arrays(xa[i:i + 1]) for i in range(len(xa))])
        alone_b = np.concatenate([m.forward_arrays(xb[i:i + 1]) for i in range(len(xb))])
        assert np.array_equal(m.forward_arrays(xa), alone_a)                    # one ragged 37-window call
        m.reserve(16, P)
        handles, cuts = [], [0, 5, 16, 19, 30, 37]
        for i, (lo, hi) in enumerate(zip(cuts[:-1], cuts[1:])):
            handles.append(m.predict_async(_Batch(xa[lo:hi]), slots=8))
            if i == 1:
                handles.append(m.predict_async(_Batch(xb), slots=8))            # another D between them
        res = [h.result().numpy() for h in handles]
        assert np.array_equal(np.concatenate(res[:2] + res[3:]), alone_a)
        assert np.array_equal(res[2], alone_b)
        probs, labels = _submit_probs(m, xb)
        assert np.array_equal(probs, alone_b) and np.array_equal(labels, np.argmax(alone_b, -1))
    finally:
        m.close()


class _Batch(object):
    def __init__(self, x):
        self.read_level_features = x


@pytest.mark.gpu
@pytest.mark.parametrize("dwells", [True, False], ids=["dwells", "nodwells"])
@pytest.mark.parametrize("H", [128, 384])
def test_decoded_heads_equal_decode_of_fp16_probabilities(H, dwells):
    """Labels, quality bytes, call bytes and phreds of the decoded and variant-decoded heads in the fp16 mode are the
    decode of the fp16 probabilities."""
    from tests.test_one_pass import _decode
    from tests.test_one_pass_variants import _random_ref, _vd_of_probs
    from tests.test_read_level_one_pass import _pinned, _submit_probs
    B, P, D = 7, 230, 9
    x = rl_oracle.synth_rl_features(B, P, D, use_dwells=dwells, seed=H + dwells, empty_rows=3, ragged=True)
    ref = _random_ref(B, P, seed=B * P + H)
    m = _model(_sd(H, 3, dwells), H, dwells)
    try:
        probs, labels = _submit_probs(m, x)
        want_labels, want_quals = _decode(probs)
        assert np.array_equal(labels, want_labels)
        xin = _pinned(m, "feats", x)
        got_labels, got_quals = np.empty((B, P), np.uint8), np.empty((B, P), np.uint8)
        m.wait(m.submit_decoded(xin, got_labels, got_quals))
        assert np.array_equal(got_labels, want_labels) and np.array_equal(got_quals, want_quals)
        calls, pq, rq = np.empty((B, P), np.uint8), np.empty((B, P), np.float32), np.empty((B, P), np.float32)
        m.wait(m.submit_variant_decoded(xin, _pinned(m, "ref", ref), calls, pq, rq))
        for g, w in zip((calls, pq, rq), _vd_of_probs(probs, ref)):
            assert np.array_equal(g, w)
    finally:
        m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("H", [128, 384])
def test_predict_consensus_equals_two_pass_in_fp16(H, tmp_path):
    """predict_consensus with an fp16 model writes the FASTQ and gap bed of predict_regions + sequence, byte for byte."""
    from medaka_b200 import common
    from tests.test_one_pass import _both, _draft
    from tests.test_read_level_one_pass import _encoder
    sd = _sd(H, 2)
    sd["linear.bias"][0] -= 6.0                      # as test_read_level_one_pass: few deletions, long sequences
    m = _model(sd, H)
    R = common.Region
    try:
        (a, bed_a), (b, bed_b) = _both(str(tmp_path), m, _encoder(True), None,
                                       [R("long", 0, 7000), R("gappy", 0, 4200), R("tiny", 0, 600)],
                                       _draft({"long": 7000, "gappy": 4200, "tiny": 600, "nodata": 300}))
        assert len(a) > 1000 and a == b and bed_a == bed_b
    finally:
        m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("H", [128, 384])
def test_switching_precision(H):
    """tc -> fp16 -> tc on one engine gives tc results bit-identical to a fresh engine's; windows queued before a switch
    run in the old mode."""
    from medaka_b200 import read_level
    P = 120
    sd = _sd(H, 52)
    x = rl_oracle.featuriser_like_rl_features(5, P, 7, F=5, seed=52)
    fresh = _model(sd, H, precision="tc")
    want_tc = fresh.forward_arrays(x)
    fresh.set_precision("fp16")
    want_fp16 = fresh.forward_arrays(x)
    fresh.close()
    assert not np.array_equal(want_tc, want_fp16)
    m = read_level.LatentSpaceLSTM(lstm_size=H, use_dwells=True)
    m.load_state_dict(sd)
    try:
        with pytest.raises(ValueError):
            m.set_precision("bf16")
        assert np.array_equal(m.forward_arrays(x), want_tc)                     # tc is the default
        m.set_precision("fp16")
        assert np.array_equal(m.forward_arrays(x), want_fp16)
        m.set_precision("tc")
        assert np.array_equal(m.forward_arrays(x), want_tc)
        # queued: a 5-window call waits in the open group (16 windows) while the mode changes
        m.reserve(16, P)
        first = m.predict_async(_Batch(x), slots=4)
        m.set_precision("fp16")
        second = m.predict_async(_Batch(x), slots=4)
        m.set_precision("tc")
        third = m.predict_async(_Batch(x), slots=4)
        assert np.array_equal(first.result().numpy(), want_tc)
        assert np.array_equal(second.result().numpy(), want_fp16)
        assert np.array_equal(third.result().numpy(), want_tc)
    finally:
        m.close()
