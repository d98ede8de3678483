"""One-pass consensus on the GPU: the engine's decoded outputs (mdk_engine_submit_decoded), the stitch from a device
arena of labels and qualities (mdk_stitch_labels_dev), and predict_consensus against predict_regions + sequence()."""
import os
import tempfile

import numpy as np
import pytest

from oracle import synth

pytestmark = pytest.mark.gpu


def _lib():
    from medaka_b200 import libmedaka as lm
    return lm.load(), lm.ffi, lm


def _decode(probs):
    lib, ffi, lm = _lib()
    p = np.ascontiguousarray(probs.reshape(-1, 5), dtype=np.float32)
    labels = np.empty(len(p), np.uint8)
    quals = np.empty(len(p), np.uint8)
    lm.check(lib.mdk_decode_consensus(0, ffi.cast("const float *", ffi.from_buffer(p)), len(p),
                                      ffi.cast("uint8_t *", ffi.from_buffer(labels)),
                                      ffi.cast("uint8_t *", ffi.from_buffer(quals))))
    return labels.reshape(probs.shape[:-1]), quals.reshape(probs.shape[:-1])


def _model(sd, F, precision="tc", rec_mode="auto", keep=False):
    from medaka_b200 import models
    m = models.GRUModel(num_features=F)
    m.load_state_dict(sd)
    m.set_precision(precision)
    m.set_rec_mode(rec_mode)
    m.keep_activations(keep)
    return m


def _decoded(m, feats, quals=True):
    x = m.pinned("tfeats", feats.shape, np.float32)
    np.copyto(x, feats)
    labels = np.empty(feats.shape[:2], np.uint8)
    q = np.empty(feats.shape[:2], np.uint8) if quals else None
    m.wait(m.submit_decoded(x, labels, q))
    return labels, q


CASES = [
    # (precision, rec_mode, keep_activations, F, B, T, state dict)
    ("tc", "auto", False, 10, 19, 37, "plain"),
    ("tc", "one", False, 10, 19, 37, "plain"),
    ("tc", "pp", False, 10, 35, 64, "plain"),
    ("tc", "auto", True, 10, 19, 37, "plain"),
    ("tc", "auto", False, 20, 21, 50, "plain"),
    ("fp32", "auto", False, 10, 19, 37, "plain"),
    ("fp32", "auto", False, 20, 3, 5, "plain"),
    ("tc", "auto", False, 10, 6, 400, "neartie"),
    ("fp32", "auto", False, 10, 6, 400, "neartie"),
]


@pytest.mark.parametrize("precision,rec_mode,keep,F,B,T,kind", CASES)
def test_head_quals_equal_decode_of_probabilities(precision, rec_mode, keep, F, B, T, kind):
    if kind == "neartie":
        sd, feats = synth.synth_state_dict_neartie(5), synth.synth_features(B, T, F, seed=105)
    else:
        sd, feats = synth.synth_state_dict(3, num_features=F), synth.synth_features(B, T, F, seed=B + T)
    m = _model(sd, F, precision, rec_mode, keep)
    try:
        ref = m.forward_arrays(feats)
        ref_labels, ref_quals = _decode(ref.probs)
        assert np.array_equal(ref.labels, ref_labels)
        labels, quals = _decoded(m, feats)
        assert np.array_equal(labels, ref_labels)
        assert np.array_equal(quals, ref_quals)
        labels_only, _ = _decoded(m, feats, quals=False)
        assert np.array_equal(labels_only, ref_labels)
    finally:
        m.close()


@pytest.mark.parametrize("precision,keep", [("tc", False), ("tc", True), ("fp32", False)])
def test_decoded_and_ordinary_calls_share_a_group_and_device_outputs(precision, keep):
    from medaka_b200 import libmedaka as lm
    lib, ffi = lm.load(), lm.ffi
    T = 200
    sd = synth.synth_state_dict(4)
    m = _model(sd, 10, precision, keep=keep)
    sizes = (5, 7, 9)           # decoded to host, ordinary, decoded to device: the ordinary piece sits mid-group
    feats = [synth.synth_features(b, T, 10, seed=b) for b in sizes]
    try:
        n0 = m.launch_count()
        alone = [m.forward_arrays(f) for f in feats]
        per_forward = (m.launch_count() - n0) // len(feats)
        expect = [_decode(a.probs) for a in alone]
        # staging for one group of all 21 windows: the three calls coalesce into it, and it launches once full
        m.set_group_windows(64)
        m.reserve(sum(sizes), T)
        xs = [m.pinned("mix%d" % i, f.shape, np.float32) for i, f in enumerate(feats)]
        for x, f in zip(xs, feats):
            np.copyto(x, f)
        labels0 = np.empty((5, T), np.uint8)
        quals0 = np.empty((5, T), np.uint8)
        probs1 = np.empty((7, T, 5), np.float32)
        labels1 = np.empty((7, T), np.uint8)
        n2 = 9 * T
        pp = ffi.new("void **")
        lm.check(lib.mdk_dev_alloc(0, 2 * n2, pp))
        dev = int(ffi.cast("uintptr_t", pp[0]))
        try:
            n0 = m.launch_count()
            t0 = m.submit_decoded(xs[0], labels0, quals0)
            t1 = m.submit_arrays(xs[1], probs1, labels1)
            t2 = m.submit_decoded(xs[2], dev, dev + n2)
            for t in (t0, t1, t2):
                m.wait(t)
            m.sync()
            assert m.launch_count() - n0 == per_forward           # one forward ran all three calls
            back = np.empty(2 * n2, np.uint8)
            lm.check(lib.mdk_memcpy_d2h(0, ffi.cast("void *", ffi.from_buffer(back)), pp[0], 2 * n2))
        finally:
            lib.mdk_dev_free(0, pp[0])
        assert np.array_equal(labels0, expect[0][0]) and np.array_equal(quals0, expect[0][1])
        assert np.array_equal(probs1, alone[1].probs) and np.array_equal(labels1, alone[1].labels)
        assert np.array_equal(back[:n2].reshape(9, T), expect[2][0])
        assert np.array_equal(back[n2:].reshape(9, T), expect[2][1])
    finally:
        m.close()


def _stitch_probs(probs_segments):
    from medaka_b200 import libmedaka as lm
    lib, ffi = lm.load(), lm.ffi
    ptrs = ffi.new("const float *[]", len(probs_segments))
    rows = np.array([len(p) for p in probs_segments], np.int64)
    for k, p in enumerate(probs_segments):
        ptrs[k] = ffi.cast("const float *", ffi.from_buffer(p))
    seq = np.empty(int(rows.sum()), np.uint8)
    qual = np.empty(int(rows.sum()), np.uint8)
    off = np.empty(len(rows) + 1, np.int64)
    lm.check(lib.mdk_stitch_consensus(0, ptrs, ffi.cast("const int64_t *", ffi.from_buffer(rows)), len(rows),
                                      ffi.cast("uint8_t *", ffi.from_buffer(seq)),
                                      ffi.cast("uint8_t *", ffi.from_buffer(qual)),
                                      ffi.cast("int64_t *", ffi.from_buffer(off))))
    return seq[:off[-1]].tobytes(), qual[:off[-1]].tobytes(), off


@pytest.mark.parametrize("seed", [0, 1])
def test_stitch_labels_dev_equals_stitch_of_probabilities(seed):
    from medaka_b200 import libmedaka as lm, stitch
    lib, ffi = lm.load(), lm.ffi
    rs = np.random.RandomState(seed)
    n = 5000
    logits = rs.standard_normal((n, 5)).astype(np.float32) * 3
    logits[1000:1400, 0] += 20                  # a run of gap calls
    probs = np.exp(logits)
    probs = (probs / probs.sum(1, keepdims=True)).astype(np.float32)
    labels, quals = _decode(probs)
    # shuffled, overlapping, single-row, all-gap and multi-block segments
    segs = [(0, 1), (4000, 1000), (1000, 400), (1100, 2500), (17, 3), (4999, 1), (0, 5000), (1200, 30), (300, 2000)]
    order = rs.permutation(len(segs))
    segs = [segs[i] for i in order]
    pp = ffi.new("void **")
    lm.check(lib.mdk_dev_alloc(0, 2 * n, pp))
    try:
        both = np.concatenate([labels, quals])
        lm.check(lib.mdk_memcpy_h2d(0, pp[0], ffi.cast("void *", ffi.from_buffer(both)), 2 * n))
        dev = int(ffi.cast("uintptr_t", pp[0]))
        seqs, quals_out = stitch.decode_label_pieces(dev, dev + n, [a for a, _ in segs], [r for _, r in segs])
        seqs_nq, none = stitch.decode_label_pieces(dev, None, [a for a, _ in segs], [r for _, r in segs])
    finally:
        lib.mdk_dev_free(0, pp[0])
    ref_seq, ref_qual, off = _stitch_probs([np.ascontiguousarray(probs[a:a + r]) for a, r in segs])
    assert "".join(seqs).encode() == ref_seq and "".join(quals_out).encode() == ref_qual
    assert [len(s) for s in seqs] == list(np.diff(off))
    assert seqs_nq == seqs and none is None
    assert seqs[[k for k, s in enumerate(segs) if s == (1000, 400)][0]] == ""


# ------------------------------------------------------------------------------------------- predict_consensus


def _pileup_source(region, bam, encoder):
    # deterministic per contig, with a coverage gap on "gappy"
    n_ref = region.end - region.start
    seed = sum(map(ord, region.ref_name))
    counts, pos = synth.synth_counts(int(n_ref * 1.18) + 8, seed=seed, start_major=region.start)
    keep = pos["major"] < region.end
    counts, pos = counts[keep], pos[keep]
    if region.ref_name == "gappy":
        hole = (pos["major"] >= region.start + 2000) & (pos["major"] < region.start + 2600)
        counts[hole] = 0
    return [(counts, pos)]


def _draft(lengths, seed=7):
    rs = np.random.RandomState(seed)
    return {k: "".join(rs.choice(list("ACGT"), n)) for k, n in lengths.items()}


def _both(tmp, model, enc, bam, bam_regions, draft, **kw):
    from medaka_b200 import prediction, stitch
    run = dict(chunk_len=kw.pop("chunk_len", 1000), chunk_ovlp=kw.pop("chunk_ovlp", 100),
               batch_size=kw.pop("batch_size", 4), bam_chunk=kw.pop("bam_chunk", 3000))
    store = os.path.join(tmp, "p%d.npzstore" % len(os.listdir(tmp)))
    a, b = os.path.join(tmp, "a.fastq"), os.path.join(tmp, "b.fastq")
    prediction.predict_regions(store, bam, bam_regions, model, enc, **run)
    stitch.sequence(store, draft, a, **kw)
    prediction.predict_consensus(bam, bam_regions, model, enc, draft, b, **run, **kw)
    out = []
    for p in (a, b):
        with open(p, "rb") as fh:
            text = fh.read()
        bed = None
        if os.path.exists(p + ".gaps_in_draft_coords.bed"):
            with open(p + ".gaps_in_draft_coords.bed", "rb") as fh:
                bed = fh.read()
            os.remove(p + ".gaps_in_draft_coords.bed")
        os.remove(p)
        out.append((text, bed))
    return out


@pytest.mark.parametrize("precision", ["tc", "fp32"])
def test_predict_consensus_equals_two_pass(precision):
    from medaka_b200 import common, features
    sd = synth.synth_state_dict(2)
    model = _model(sd, 10, precision)
    enc = features.CountsFeatureEncoder(normalise="total", pileup_source=_pileup_source)
    lengths = {"long": 7000, "gappy": 4200, "tiny": 600, "nodata": 300}
    draft = _draft(lengths)
    R = common.Region
    bam_regions = [R("long", 0, 7000), R("gappy", 0, 4200), R("tiny", 0, 600)]
    configs = [
        {},
        {"min_depth": 25},
        {"regions": ["long:1500-5200", R("tiny", None, None), "nodata"]},
        {"fillgaps": False},
        {"fill_char": "N", "qualities": False},
    ]
    try:
        with tempfile.TemporaryDirectory() as d:
            for cfg in configs:
                (a, bed_a), (b, bed_b) = _both(d, model, enc, None, bam_regions, draft, **cfg)
                assert len(a) > 1000, cfg
                assert a == b, cfg
                assert bed_a == bed_b, cfg
    finally:
        model.close()


def test_predict_consensus_on_a_bam_through_the_fused_featuriser():
    from medaka_b200 import common, features
    from tests import bamutil
    recs = synth.synth_reads(160, 4000, seed=9, mean_len=500)
    recs.sort(key=lambda r: r["pos"])
    for r in recs:
        r["ref"] = 0
    sd = synth.synth_state_dict(6)
    sd["linear.bias"][0] -= 6.0          # fewer gap calls on real pileup features, so that most columns reach the output
    model = _model(sd, 10)
    try:
        with tempfile.TemporaryDirectory() as d:
            path = os.path.join(d, "r.bam")
            bamutil.write_bam(path, [("ctg", 4000)], recs)
            enc = features.CountsFeatureEncoder(normalise="total")
            draft = _draft({"ctg": 4000}, seed=3)
            (a, bed_a), (b, bed_b) = _both(d, model, enc, path, [common.Region("ctg", 0, 4000)], draft)
            assert len(a) > 1000 and a == b and bed_a == bed_b
    finally:
        model.close()


def test_predict_consensus_refuses_read_level_models_and_several_ranks():
    from medaka_b200 import prediction

    class ReadLevel(object):
        pass

    with pytest.raises(NotImplementedError, match="predict_regions"):
        prediction.predict_consensus(None, [], ReadLevel(), None, {}, "x")
    model = _model(synth.synth_state_dict(1), 10)
    try:
        with pytest.raises(NotImplementedError):
            prediction.predict_consensus(None, [], model, None, {}, "x", world_size=2)
    finally:
        model.close()


def test_predict_consensus_across_many_arena_slabs(monkeypatch):
    """Slabs of two 4 x 1000 batches: the windows of a stitch region lie in several slabs, each stitched on its own."""
    from medaka_b200 import common, features, prediction
    monkeypatch.setattr(prediction._LabelArena.__init__, "__defaults__", (8192,))
    model = _model(synth.synth_state_dict(2), 10)
    enc = features.CountsFeatureEncoder(normalise="total", pileup_source=_pileup_source)
    draft = _draft({"long": 7000, "gappy": 4200, "tiny": 600})
    R = common.Region
    try:
        with tempfile.TemporaryDirectory() as d:
            for cfg in ({}, {"min_depth": 25}):
                (a, bed_a), (b, bed_b) = _both(d, model, enc, None, [R("long", 0, 7000), R("gappy", 0, 4200),
                                                                     R("tiny", 0, 600)], draft, **cfg)
                assert len(a) > 1000 and a == b and bed_a == bed_b, cfg
    finally:
        model.close()
