"""The consensus GRU at gru_size = 256, the width `medaka train` builds by default (DEFAULT_MODEL_DICT of the reference's
medaka/models.py).  Its own kernels (medaka_b200/csrc/gru256.cu, the width-templated layer-0 projection, fp32 recurrence
and head) are checked against:
  * the reference itself (tests/golden/gru256_forward.npz, tests/golden/make_gru256_golden.py): the 1e-3 scale-aware
    logit bar of tests/test_gpu_parity.py and identical labels wherever the top-2 margin exceeds 1e-5, both precisions;
  * oracle/gru_oracle.stages in float64, stage by stage, at one wave x 10 000 featuriser-like columns, with bars that can
    tell three fp16 products from two (test_ablations_exceed_the_bars proves that on the CPU);
  * the engine's own contracts: placement independence, asynchronous and decoded calls, one-pass consensus and variant
    calling, and model archives with the reference's default model function.
"""
import functools
import os
import subprocess
import tempfile

import numpy as np
import pytest

from oracle import gru_oracle, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H = 256
SCALE = np.array([-1.4426950408889634, -1.4426950408889634, 2.8853900817779268], np.float32)   # gate_scale(r, z, n)
F32 = ["w_in_packed", "bias_gi", "b_hn", "bias_gi_tc", "b_hn_tc", "w_hh_t"]
F16 = ["w_hh_tm", "w_x_tm", "w_in_tc"]
LOGIT_TOL = 1e-3
MARGIN = 1e-5
DEFAULT_MODEL_DICT = {"type": "GRUModel", "kwargs": {"num_features": 10, "num_classes": 5, "gru_size": 256}}

# Stage bars at H = 256 (h0 / h1: max|d| / max|ref|; logits: max |d| / max_c |logit_c|; probs: max |d|), calibrated on
# an H100 80GB HBM3 (SXM, 700 W power limit) over every GPU stage case of this file (DESIGN §2 has the table).  Worst
# device error, h0 / h1 / logits / probs:
#   fp32 path   5.6e-7 / 7.6e-7 / 6.4e-7 / 5.1e-7
#   tc path     1.8e-6 / 4.7e-6 / 4.7e-6 / 2.1e-6
# Smallest ablation effects (test_ablations_exceed_the_bars prints them): h0 5.8e-5 (h), h1 7.4e-5 (h), logits 8.1e-5
# (w_hh), probs 7.9e-6 (w_hh), all with default weights.  Each bar is at most a third of that stage's smallest effect, so
# a kernel that lost a product fails it, and at h0, h1 and logits at least 4.7x the worst error of either path.  At probs
# the window is narrower than the tc path's error allows (2.6e-6 is 1.3x its worst error); the other stages carry the
# discrimination there.
BARS = {"h0": 1.5e-5, "h1": 2.2e-5, "logits": 2.5e-5, "probs": 2.6e-6}
STAGES = ("h0", "h1", "logits", "probs")
# The tensor-core products a kernel at H = 256 can lose.  Layer 0's input projection runs in fp32 on the CUDA cores at
# this width (inproj0_kernel), so the x and w_ih0 ablations do not apply.
ABLATIONS = ("w_hh", "w_ih1", "h", "h0")
WEIGHTS = {"default": {}, "hot": dict(rec_gain=2.5, head_gain=24.0)}
LONG_T = 10000


def _sd(seed, F=10, **kw):
    return synth.synth_state_dict(seed, num_features=F, gru_size=H, **kw)


def _model(sd, F=10, precision="tc"):
    from medaka_b200 import models
    m = models.GRUModel(num_features=F, gru_size=H)
    m.load_state_dict(sd)
    m.set_precision(precision)
    return m


def _scaled(k, got, want):
    d = np.abs(got.astype(np.float64) - want)
    if k == "probs":
        return d
    if k == "logits":
        return d / np.abs(want).max(-1, keepdims=True)
    return d / float(np.abs(want).max())


def _decided(probs):
    top2 = np.sort(probs, -1)[..., -2:]
    return (top2[..., 1] - top2[..., 0]) > MARGIN


# ------------------------------------------------------------------------------------------------ CPU
@pytest.fixture(scope="module")
def pack_driver(tmp_path_factory):
    import __graft_entry__
    exe = str(tmp_path_factory.mktemp("gru256_pack") / "gru256_pack_check")
    subprocess.run([__graft_entry__._nvcc(), "-std=c++17", "-O1", "-o", exe,
                    os.path.join(ROOT, "tests", "native", "gru256_pack_check.cu")], check=True, capture_output=True)
    return exe


def _pack(exe, sd, F, tmp_path):
    src, dst = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    with open(src, "wb") as f:
        for layer in range(2):
            for sfx in ("", "_reverse"):
                for name in ("weight_ih", "weight_hh", "bias_ih", "bias_hh"):
                    f.write(np.ascontiguousarray(sd["gru.%s_l%d%s" % (name, layer, sfx)], np.float32).tobytes())
    r = subprocess.run([exe, str(F), src, dst], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    raw, off, layers = open(dst, "rb").read(), 0, []
    for _ in range(2):
        arrays = {}
        for name in F32 + F16:
            n = int(np.frombuffer(raw, np.int64, 1, off)[0])
            dt = np.float32 if name in F32 else np.float16
            arrays[name] = np.frombuffer(raw, dt, n, off + 8)
            off += 8 + n * np.dtype(dt).itemsize
        layers.append(arrays)
    assert off == len(raw)
    return layers


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint16 if a.dtype == np.float16 else np.uint32)


def _hi_lo(x):
    hi = x.astype(np.float16)
    return np.stack([hi, (x - hi.astype(np.float32)).astype(np.float16)])


@pytest.mark.parametrize("F", [10, 20])
def test_gru256_pack_layouts(pack_driver, tmp_path, F):
    """Every array the 256-wide kernels read, bit for bit: the H = 128 layouts with H = 256 in place (gru_pack.cuh)."""
    sd = _sd(3, F)
    layers = _pack(pack_driver, sd, F, tmp_path)
    for layer, got in enumerate(layers):
        nin = F if layer == 0 else 2 * H
        w_ih = [sd["gru.weight_ih_l%d%s" % (layer, s)] for s in ("", "_reverse")]
        w_hh = [sd["gru.weight_hh_l%d%s" % (layer, s)] for s in ("", "_reverse")]
        b_ih = [sd["gru.bias_ih_l%d%s" % (layer, s)] for s in ("", "_reverse")]
        b_hh = [sd["gru.bias_hh_l%d%s" % (layer, s)] for s in ("", "_reverse")]
        assert np.array_equal(_bits(got["w_in_packed"].reshape(6 * H, nin)), _bits(np.concatenate(w_ih)))
        bias = np.concatenate([np.concatenate([bi[:2 * H] + bh[:2 * H], bi[2 * H:]]) for bi, bh in zip(b_ih, b_hh)])
        b_hn = np.stack([bh[2 * H:] for bh in b_hh])
        assert np.array_equal(_bits(got["bias_gi"]), _bits(bias))
        assert np.array_equal(_bits(got["b_hn"].reshape(2, H)), _bits(b_hn))
        assert np.array_equal(_bits(got["bias_gi_tc"].reshape(2, 3, H)), _bits(bias.reshape(2, 3, H) * SCALE[:, None]))
        assert np.array_equal(_bits(got["b_hn_tc"].reshape(2, H)), _bits(b_hn * SCALE[2]))
        assert np.array_equal(_bits(got["w_hh_t"].reshape(2, H, 3 * H)), _bits(np.stack([w.T for w in w_hh])))
        w_hh_tm = np.stack([_hi_lo(w.reshape(3, H, H) * SCALE[:, None, None]) for w in w_hh])
        assert np.array_equal(_bits(got["w_hh_tm"].reshape(2, 2, 3, H, H)), _bits(w_hh_tm))
        assert got["w_x_tm"].size == 0            # no fused layer-0 projection at this width
        if layer == 1:
            w_in_tc = np.stack([_hi_lo(w.reshape(3, H, nin)[g] * SCALE[g]) for w in w_ih for g in range(3)])
            assert np.array_equal(_bits(got["w_in_tc"].reshape(6, 2, H, nin)), _bits(w_in_tc))
        else:
            assert got["w_in_tc"].size == 0


@pytest.mark.parametrize("gru_size", [64, 192, 384])
def test_engine_refuses_other_widths(gru_size):
    """mdk_engine_create checks the model description before it touches a device."""
    from medaka_b200 import libmedaka as lm
    lib, ffi = lm.load(), lm.ffi
    desc = ffi.new("mdk_model_desc *")
    desc.num_features, desc.gru_size, desc.n_layers, desc.bidirectional, desc.num_classes = 10, gru_size, 2, 1, 5
    pe = ffi.new("mdk_engine **")
    assert lib.mdk_engine_create(0, desc, pe) == lib.MDK_ERR_UNSUPPORTED
    assert ffi.string(lib.mdk_last_error()).decode() == "engine_create: gru_size must be 128 or 256"


def _write_default_archive(path, sd):
    from medaka_b200 import datastore
    # what the reference stores: partial(medaka.models.model_from_dict, DEFAULT_MODEL_DICT)
    meta = {"model_function": functools.partial(datastore._ref_model_from_dict, DEFAULT_MODEL_DICT)}
    datastore.ModelStoreTGZ.write(path, sd, meta)


def test_default_model_archive_resolves_to_gru_size_256(tmp_path):
    from medaka_b200 import datastore
    path = str(tmp_path / "default_model_pt.tar.gz")
    _write_default_archive(path, _sd(0))
    kw = datastore.ModelStoreTGZ(path).model_kwargs()
    assert kw == DEFAULT_MODEL_DICT


@pytest.mark.parametrize("weights", list(WEIGHTS))
def test_ablations_exceed_the_bars(weights):
    """Every tensor-core product the H = 256 path can lose moves every stage it reaches by at least 3x that stage's bar,
    at the shape of the GPU stage test (10 000 featuriser-like columns; two windows)."""
    sd = synth.synth_state_dict(21, gru_size=H, **WEIGHTS[weights])
    x = gru_oracle.featuriser_like_features(2, LONG_T, 10, seed=5)
    want = gru_oracle.stages(sd, x)
    smallest = {k: np.inf for k in STAGES}
    for which in ABLATIONS:
        asd, kw = gru_oracle.ablate(sd, which)
        got = gru_oracle.stages(asd, x, **kw)
        effect = {k: float(_scaled(k, got[k], want[k]).max()) for k in STAGES}
        print("gru256 ablation %s/%s: %s" % (weights, which, " ".join("%s=%.3g" % (k, effect[k]) for k in STAGES)))
        for k in STAGES:
            if effect[k] > 0:            # w_ih1 and h0 act after layer 0
                smallest[k] = min(smallest[k], effect[k])
    print("gru256 smallest effects %s: %s" % (weights, " ".join(
        "%s=%.3g (%.1fx its bar)" % (k, smallest[k], smallest[k] / BARS[k]) for k in STAGES)))
    for k in STAGES:
        assert smallest[k] >= 3 * BARS[k], (k, smallest[k], BARS[k])


# ------------------------------------------------------------------------------------------------ GPU
def _golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "gru256_forward.npz"))


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["tc", "fp32"])
@pytest.mark.parametrize("case", ["default", "f20", "ragged", "t1", "short", "hot"])
def test_forward_matches_reference_golden(case, precision):
    g = _golden()
    seed, B, T, F, head_gain, rec_gain = g[case + "_args"]
    sd = _sd(int(seed), int(F), head_gain=head_gain, rec_gain=rec_gain)
    feats = synth.synth_features(int(B), int(T), int(F), seed=100 + int(seed))
    m = _model(sd, int(F), precision)
    try:
        out = m.forward_arrays(feats, want_logits=True, want_labels=True)
    finally:
        m.close()
    ref_logits, ref_probs = g[case + "_logits"], g[case + "_probs"]
    err = float(_scaled("logits", out.logits, ref_logits).max())
    decided = _decided(ref_probs)
    flips = int(((out.labels != np.argmax(ref_probs, -1)) & decided).sum())
    print("gru256 %s/%s: scaled logit err %.3e, prob err %.3e, label mismatches %d/%d" % (
        case, precision, err, np.abs(out.probs - ref_probs).max(), flips, out.labels.size))
    assert err <= LOGIT_TOL
    assert flips == 0
    assert np.array_equal(out.labels, np.argmax(out.probs, -1))


@pytest.fixture(scope="module")
def wave():
    """One wave of the 256 recurrence x 10 000 featuriser-like columns, and the windows checked stage by stage: a
    tile's first and last window, the next tile, the middle and the last tile's edges."""
    from medaka_b200 import models
    m = models.GRUModel(num_features=10, gru_size=H)
    B = m.preferred_batch_size()
    m.close()
    x = gru_oracle.featuriser_like_features(B, LONG_T, 10, seed=3)
    picks = sorted({0, 15, 16, B // 2 - 1, B // 2, B - 16, B - 1})
    return x, picks


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["tc", "fp32"])
@pytest.mark.parametrize("weights", list(WEIGHTS))
def test_stages_at_one_wave(wave, weights, precision):
    x, picks = wave
    sd = synth.synth_state_dict(21, gru_size=H, **WEIGHTS[weights])
    m = _model(sd, 10, precision)
    try:
        out = m.forward_arrays(x, want_logits=True, want_labels=True)
        got = {"h0": np.concatenate([m.read_activation(0, w, 1) for w in picks]),
               "h1": np.concatenate([m.read_activation(1, w, 1) for w in picks]),
               "logits": out.logits[picks], "probs": out.probs[picks], "labels": out.labels[picks]}
        t = m.last_timings()
    finally:
        m.close()
    want = gru_oracle.stages(sd, x[picks])
    err = {k: float(_scaled(k, got[k], want[k]).max()) for k in STAGES}
    print("gru256-stages %s/%s B=%d: %s  (rec0 %.1f ms, rec1 %.1f ms)" % (
        weights, precision, len(x), " ".join("%s=%.3g" % (k, err[k]) for k in STAGES), t["rec0_ms"], t["rec1_ms"]))
    for k in STAGES:
        assert np.isfinite(got[k]).all(), k
        assert err[k] <= BARS[k], (k, err[k], BARS[k])
    decided = _decided(want["probs"])
    assert np.array_equal(got["labels"][decided], np.argmax(want["probs"], -1)[decided])
    assert np.array_equal(out.labels, np.argmax(out.probs, -1))


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["tc", "fp32"])
def test_windows_in_a_group_equal_windows_alone(precision):
    """A window's outputs do not depend on its neighbours or its place in a tile or a group."""
    sd = _sd(7)
    x = synth.synth_features(45, 300, 10, seed=8)
    m = _model(sd, 10, precision)
    try:
        group = m.forward_arrays(x, want_logits=True, want_labels=True)
        for w in (0, 15, 16, 31, 44):
            alone = m.forward_arrays(x[w:w + 1], want_logits=True, want_labels=True)
            assert np.array_equal(alone.probs[0], group.probs[w]), w
            assert np.array_equal(alone.logits[0], group.logits[w]), w
            assert np.array_equal(alone.labels[0], group.labels[w]), w
        h1 = m.read_activation(1)
        assert h1.shape == (1, 300, 2 * H)
    finally:
        m.close()


@pytest.mark.gpu
def test_engine_sizing_and_modes():
    from medaka_b200 import libmedaka as lm
    m = _model(_sd(1))
    try:
        pref = m.preferred_batch_size()
        assert pref >= 16 and pref % 16 == 0
        assert m.lookahead(200, 10000) >= 2
        m.reserve(pref, 1000)
        m.reserve(10 * pref, 10000)         # capped at one group: 240 x 10 000 positions stay inside the budget
        m.set_rec_mode("auto")
        for mode in ("one", "pp"):
            with pytest.raises(lm.MedakaB200Error, match="only MDK_REC_AUTO"):
                m.set_rec_mode(mode)
    finally:
        m.close()


@pytest.mark.gpu
def test_predict_async_equals_predict_on_batch():
    sd = _sd(9)
    m = _model(sd)
    try:
        batches = []
        for i in range(5):
            x = synth.synth_features(23 + i, 200, 10, seed=30 + i)

            class _B:
                counts_matrix = x
            batches.append(_B())
        handles = [m.predict_async(b, slots=5) for b in batches]
        got = [h.result().numpy() for h in handles]
        for b, g in zip(batches, got):
            want = m.predict_on_batch(b).numpy()
            assert np.array_equal(g, want)
    finally:
        m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["tc", "fp32"])
def test_decoded_heads_equal_decode_of_probabilities(precision):
    from tests.test_one_pass import _decode, _decoded
    from tests.test_one_pass_variants import _random_ref, _variant_decoded, _vd_of_probs
    sd = _sd(4)
    x = synth.synth_features(19, 137, 10, seed=11)
    m = _model(sd, 10, precision)
    try:
        probs = m.forward_arrays(x, want_labels=False).probs
        labels, quals = _decoded(m, x)
        want_l, want_q = _decode(probs)
        assert np.array_equal(labels, want_l) and np.array_equal(quals, want_q)
        ref = _random_ref(19, 137, seed=2)
        calls, pq, rq = _variant_decoded(m, x, ref)
        wc, wpq, wrq = _vd_of_probs(probs, ref)
        assert np.array_equal(calls, wc)
        assert np.array_equal(pq, wpq) and np.array_equal(rq, wrq)
    finally:
        m.close()


@pytest.mark.gpu
def test_predict_consensus_equals_two_pass():
    from medaka_b200 import common, features
    from tests.test_one_pass import _both, _draft, _pileup_source
    model = _model(_sd(2))
    enc = features.CountsFeatureEncoder(normalise="total", pileup_source=_pileup_source)
    lengths = {"long": 7000, "gappy": 4200, "tiny": 600}
    draft = _draft(lengths)
    R = common.Region
    bam_regions = [R("long", 0, 7000), R("gappy", 0, 4200), R("tiny", 0, 600)]
    try:
        with tempfile.TemporaryDirectory() as d:
            for cfg in ({}, {"min_depth": 25}, {"fill_char": "N", "qualities": False}):
                (a, bed_a), (b, bed_b) = _both(d, model, enc, None, bam_regions, draft, **cfg)
                assert len(a) > 1000, cfg
                assert a == b and bed_a == bed_b, cfg
    finally:
        model.close()


@pytest.mark.gpu
def test_predict_variants_on_a_bam_through_the_fused_featuriser():
    from medaka_b200 import common, features
    from tests import bamutil
    from tests.test_one_pass_variants import _check
    recs = synth.synth_reads(160, 4000, seed=9, mean_len=500)
    recs.sort(key=lambda r: r["pos"])
    for r in recs:
        r["ref"] = 0
    sd = _sd(6)
    sd["linear.bias"][0] -= 6.0
    model = _model(sd)
    try:
        with tempfile.TemporaryDirectory() as d:
            path = os.path.join(d, "r.bam")
            bamutil.write_bam(path, [("ctg", 4000)], recs)
            enc = features.CountsFeatureEncoder(normalise="total")
            _check(model, enc, path, [common.Region("ctg", 0, 4000)], {"ctg": 4000}, [{}, {"return_all": True}], d,
                   min_records=20)
    finally:
        model.close()


@pytest.mark.gpu
def test_default_model_archive_loads_and_runs(tmp_path):
    from medaka_b200 import datastore
    g = _golden()
    sd = _sd(0, 10)
    path = str(tmp_path / "default_model_pt.tar.gz")
    _write_default_archive(path, sd)
    m = datastore.ModelStoreTGZ(path).load_model()
    try:
        assert m.gru_size == H
        feats = synth.synth_features(3, 500, 10, seed=100)

        class _B:
            counts_matrix = feats
        probs = m.predict_on_batch(_B()).numpy()
    finally:
        m.close()
    assert np.abs(probs - g["default_probs"]).max() <= 1e-3
    decided = _decided(g["default_probs"])
    assert np.array_equal(np.argmax(probs, -1)[decided], np.argmax(g["default_probs"], -1)[decided])
