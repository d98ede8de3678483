"""Labelled training samples (`medaka features --truth`): truth alignments, their filters and labels, create_samples.

CPU: the oracle against its golden (cut from the reference's truth_to_ref.bam / test_reads.bam by
tests/golden/make_truth_golden.py), the host encoding against the oracle, the truth filters on hand-built alignments
with hand-derived spans, argument errors.  GPU: mdk_truth_labels and create_samples against the oracle, and a store from
create_samples through one training epoch.
"""
import os
import pickle

import numpy as np
import pytest

from medaka_b200 import bam, common, labels
from oracle import pileup_oracle, synth, truth_oracle
from tests.bamutil import write_bam
from tests.test_oracle import SIMPLE_CALLS

R = common.Region
TEST_030_TRUTH = dict(query_name="truth", pos=0, cigar="4=1I3=2I1=", seq="ACATAGATCTG", flag=0, tags={"MD": "8"})
TEST_030_FEATURES = np.array([
    [0.5, 0., 0., 0., 0.5, 0., 0., 0., 0., 0.], [0., 0.5, 0., 0., 0., 0.5, 0., 0., 0., 0.],
    [0.5, 0., 0., 0., 0.5, 0., 0., 0., 0., 0.], [0., 0.25, 0., 0.25, 0., 0., 0., 0.25, 0., 0.25],
    [0.25, 0., 0., 0., 0., 0., 0., 0., 0., 0.], [0., 0., 0.5, 0., 0., 0., 0.5, 0., 0., 0.],
    [0.5, 0., 0., 0., 0.5, 0., 0., 0., 0., 0.], [0., 0., 0., 0.5, 0., 0., 0., 0.5, 0., 0.],
    [0., 0., 0.5, 0., 0., 0., 0.5, 0., 0., 0.]], dtype=np.float32)


def _golden(golden_dir):
    return np.load(os.path.join(golden_dir, "truth_labels.npz"))


def _golden_truth(g):
    return labels.TruthRecord("utg000001l", int(g["truth_pos"]), g["truth_cigar"], g["truth_seq"], int(g["truth_l_seq"]),
                              {"MD": str(g["truth_md"])}, int(g["truth_flag"]), "truth")


def _golden_reads(g):
    return bam.RecordBatch(pos=g["pos"], flag=g["flag"], mapq=g["mapq"], dtype=g["dtype"], cigar=g["cigar"],
                           cigar_off=g["cigar_off"], seq=g["seq"], seq_off=g["seq_off"], l_seq=g["l_seq"], names=None,
                           tags=None)


def _as_dict(rec):
    """A TruthRecord as the oracle's dict record."""
    ops = "MIDNSHP=X"
    return dict(pos=rec.reference_start, cigar="".join("%d%s" % (int(c) >> 4, ops[int(c) & 15]) for c in rec.cigar),
                seq=rec.query_sequence, flag=rec.flag, tags=rec.tags)


def _record(d, ref_name="ref"):
    """A dict record (pos, cigar, seq, tags) as a TruthRecord."""
    return labels.TruthRecord.from_batch(bam.records_from_dicts([d]), ref_name)[0]


def _synth_truth(rs, pos=50):
    """A random truth: hard and soft clips at both ends, M/=/X, insertion runs (consecutive I, I right after D or N),
    deletions, skips; ACGT only."""
    ops = []
    if rs.uniform() < 0.5:
        ops.append((int(rs.randint(1, 9)), "H"))
    if rs.uniform() < 0.6:
        ops.append((int(rs.randint(1, 9)), "S"))
    ops.append((int(rs.randint(1, 12)), "M"))
    for _ in range(int(rs.randint(3, 30))):
        kind = rs.choice(["M", "=", "X", "I", "II", "D", "N", "DI", "ID", "NI"])
        for op in kind:
            ops.append((int(rs.randint(1, 6)) if op in "IDN" else int(rs.randint(1, 12)), op))
        ops.append((int(rs.randint(1, 12)), "M"))
    if rs.uniform() < 0.6:
        ops.append((int(rs.randint(1, 9)), "S"))
    if rs.uniform() < 0.5:
        ops.append((int(rs.randint(1, 9)), "H"))
    qlen = sum(n for n, op in ops if op in "MIS=X")
    seq = "".join("ACGT"[k] for k in rs.randint(0, 4, qlen))
    return dict(pos=pos, cigar="".join("%d%s" % o for o in ops), seq=seq, flag=0, tags={})


def _clip_candidates(d):
    """Window bounds worth testing: inside deletions / skips, at and behind positions with an insertion run, around
    the ends of the alignment."""
    pairs = truth_oracle.get_aligned_pairs(d)
    out = {d["pos"] - 3, d["pos"], d["pos"] + truth_oracle.reference_length(d) + 2}
    for (q, r), nxt in zip(pairs, pairs[1:] + [(None, None)]):
        if r is not None and q is None:
            out.add(r)
        if r is not None and nxt[0] is not None and nxt[1] is None:
            out.update((r, r + 1))
    return sorted(out)


def _columns(d, rs):
    """Pileup-like columns: every truth position over a wide window, minors beyond each run, majors outside."""
    t = truth_oracle.Truth(d)
    t.start, t.end = d["pos"] - 5, t.reference_end + 5
    pos = set(truth_oracle.alignment_to_labels(t))
    for major, minor in list(pos):
        pos.add((major, minor + 1))
        pos.add((major, minor + int(rs.randint(2, 5))))
    for m in rs.randint(d["pos"] - 10, t.reference_end + 10, 20):
        pos.add((int(m), 0))
        pos.add((int(m), int(rs.randint(1, 4))))
    return np.array(sorted(pos), dtype=[("major", "<i8"), ("minor", "<i8")])


def _truth_from_draft(draft, start, end, rs, p_edit=0.01, query_name="truth", tags=None):
    """A truth aligned to draft[start:end) with ~p_edit mismatches, insertions and deletions, and its MD tag."""
    ops, seq, md, run = [], [], [], 0

    def push(op, n=1):
        if ops and ops[-1][1] == op:
            ops[-1][0] += n
        else:
            ops.append([n, op])
    p = start
    while p < end:
        u = rs.uniform()
        if u < p_edit / 3 and 0 < p - start and ops[-1][1] == "M":
            b = "ACGT"[rs.randint(4)]
            push("I")
            seq.append(b)
            continue
        if u < 2 * p_edit / 3 and 0 < p - start < end - start - 5 and ops[-1][1] == "M":
            n = int(rs.randint(1, 4))
            push("D", n)
            md.append("%d^%s" % (run, draft[p:p + n]))
            run = 0
            p += n
            continue
        push("M")
        if u < p_edit:
            b = "ACGT".replace(draft[p], "")[rs.randint(3)]
            seq.append(b)
            md.append("%d%s" % (run, draft[p]))
            run = 0
        else:
            seq.append(draft[p])
            run += 1
        p += 1
    md.append(str(run))
    t = dict(tags or {})
    t["MD"] = "".join(md)
    return dict(query_name=query_name, pos=start, cigar="".join("%d%s" % (n, op) for n, op in ops), seq="".join(seq),
                flag=0, mapq=60, tags=t)


# ------------------------------------------------------------------------------------------------------------ CPU
def test_oracle_reproduces_golden(golden_dir):
    """The oracle on the fixture gives the labelled samples it was stored with; make_truth_golden.py asserts the
    reference's test_030 / test_031 numbers and the hand-derived truth spans of utg000001l."""
    g = _golden(golden_dir)
    truth = _as_dict(_golden_truth(g))
    samples = truth_oracle.bams_to_training_samples(
        [truth], pileup_oracle.records_from_batch(_golden_reads(g)), "utg000001l", int(g["start"]), int(g["end"]))
    assert [len(p) for p, _ in samples] == g["sample_len"].tolist()
    assert np.array_equal(np.concatenate([p["major"] for p, _ in samples]), g["major"])
    assert np.array_equal(np.concatenate([p["minor"] for p, _ in samples]), g["minor"])
    assert np.array_equal(np.concatenate([lb for _, lb in samples]), g["labels"])


def test_oracle_test_030_literals():
    (pos, lab), = truth_oracle.bams_to_training_samples([TEST_030_TRUTH], SIMPLE_CALLS, "ref", 0, 100, min_length=0)
    assert lab.tolist() == [1, 2, 1, 4, 1, 3, 1, 4, 3]
    assert lab.dtype == np.int64


def test_encode_matches_oracle(golden_dir):
    """HaploidLabelScheme.encode (host) equals the oracle's pair loop: the real truth in its fixture window and
    seeded synthetic truths in windows that start or end inside deletions or at insertion runs."""
    scheme = labels.HaploidLabelScheme()
    g = _golden(golden_dir)
    cases = [(_golden_truth(g), int(g["start"]), int(g["end"]))]
    rs = np.random.RandomState(7)
    for _ in range(40):
        d = _synth_truth(rs)
        cand = _clip_candidates(d)
        for _ in range(3):
            s, e = sorted(rs.choice(cand, 2))
            cases.append((_record(d), int(s), int(e)))
    for rec, s, e in cases:
        ta = labels.TruthAlignment(rec)
        ta.start, ta.end = s, e
        to = truth_oracle.Truth(_as_dict(rec))
        to.start, to.end = s, e
        pos, codes = scheme.encode((ta,))
        want_pos, want = truth_oracle.encode(to)
        assert [tuple(p) for p in pos.tolist()] == want_pos
        assert np.array_equal(codes, want) and codes.dtype == np.int64


def test_reference_sequence_from_md():
    d = dict(pos=10, cigar="2S3M2D2M1I3M1S", seq="TTACGTAGCCGT", flag=0, tags={"MD": "1G1^CC2T2"})
    rec = _record(d)
    assert rec.get_reference_sequence() == truth_oracle.get_reference_sequence(d) == "AGGCCTATCG"
    assert rec.reference_end == 10 + 10
    with pytest.raises(ValueError):
        _record(dict(d, tags={})).get_reference_sequence()
    with pytest.raises(ValueError):
        _record(dict(d, tags={"MD": "9"})).get_reference_sequence()


def test_scheme_encoding_and_pickle():
    scheme = labels.HaploidLabelScheme()
    assert scheme._encoding == {('*',): 0, ('A',): 1, ('C',): 2, ('G',): 3, ('T',): 4}
    assert scheme.padding_vector == 0 and scheme.num_classes == 5
    assert scheme._labels_to_encoded_labels([('A',), ('*',), ('T',)]).tolist() == [1, 0, 4]
    assert scheme.__getstate__() == {}
    assert pickle.loads(pickle.dumps(scheme)).__dict__.keys() == scheme.__dict__.keys()


def _draft(n, seed=3):
    rs = np.random.RandomState(seed)
    return "".join("ACGT"[k] for k in rs.randint(0, 4, n))


def _perfect(draft, start, end, name, **kw):
    return dict(query_name=name, pos=start, cigar="%dM" % (end - start), seq=draft[start:end], flag=kw.pop("flag", 2064),
                mapq=60, tags=dict({"MD": str(end - start)}, **kw.pop("tags", {})), **kw)


@pytest.fixture(scope="module")
def filter_bam(tmp_path_factory):
    """One contig per filter case, truth records with hand-chosen spans (flag 2064 like the reference's truth)."""
    L = 20000
    d = _draft(L)
    cases = {
        "case1": [(1000, 3000), (1500, 3500)],
        "case2": [(1000, 3000), (2500, 4500)],
        "case3": [(1000, 6000), (5000, 6500)],
        "case4": [(1000, 6000), (5800, 7300)],
        "case4later": [(1000, 2500), (2300, 7300)],
        "misc": [],
        "haps": [],
    }
    refs = [(name, L) for name in cases]
    recs = []
    for ti, (name, spans) in enumerate(cases.items()):
        for k, (s, e) in enumerate(spans):
            recs.append(dict(_perfect(d, s, e, "%s_%d" % (name, k)), ref=ti))
    misc = refs.index(("misc", L))
    amb = _perfect(d, 1000, 3000, "ambiguous_query")
    amb["seq"] = amb["seq"][:700] + "N" + amb["seq"][701:]
    amb_ref = _perfect(d, 4000, 6000, "ambiguous_ref")
    amb_ref["seq"] = amb_ref["seq"][:500] + ("A" if d[4500] != "A" else "C") + amb_ref["seq"][501:]
    amb_ref["tags"]["MD"] = "500N1499"
    recs += [dict(amb, ref=misc), dict(amb_ref, ref=misc), dict(_perfect(d, 7000, 7900, "short"), ref=misc),
             dict(_perfect(d, 8000, 11000, "long"), ref=misc), dict(_perfect(d, 12000, 14000, "unmapped", flag=4), ref=misc),
             dict(_perfect(d, 15000, 17000, "secondary", flag=256), ref=misc)]
    haps = refs.index(("haps", L))
    for name, s, e, hp in (("a", 1000, 5000, 1), ("x", 1500, 4000, 2), ("y", 3500, 6000, 2), ("b", 7000, 9000, 1)):
        recs.append(dict(_perfect(d, s, e, name, tags={"HP": hp}), ref=haps))
    recs.sort(key=lambda r: (r["ref"], r["pos"]))
    path = str(tmp_path_factory.mktemp("truth") / "truth.bam")
    write_bam(path, refs, recs)
    return path


def _spans(path, region, **kw):
    return [tuple((a.start, a.end) for a in g) for g in labels.TruthAlignment.bam_to_alignments(path, region, **kw)]


@pytest.mark.parametrize("ctg, want", [
    ("case1", []),                                                  # similar lengths, large overlap: both dropped
    ("case2", [((1000, 2500),), ((3000, 4500),)]),                  # similar lengths, small overlap: trimmed to abut
    ("case3", [((1000, 6000),)]),                                   # ratio >= 2, large overlap: shorter dropped
    ("case4", [((1000, 6000),), ((6000, 7300),)]),                  # ratio >= 2, small overlap: later one starts behind
    ("case4later", [((1000, 2500),), ((2500, 7300),)]),             # ... even when the later one is the longer
])
def test_truth_filter_cases(filter_bam, ctg, want):
    assert _spans(filter_bam, R(ctg, 0, 20000), min_length=1000) == want


def test_truth_filter_ambiguity_min_length_and_trim(filter_bam):
    # ambiguous query / MD-reconstructed reference dropped, 900 bases < min_length, unmapped and secondary not fetched
    assert _spans(filter_bam, R("misc", 0, 20000)) == [((8000, 11000),)]
    assert _spans(filter_bam, R("misc", 0, 20000), min_length=900) == [((7000, 7900),), ((8000, 11000),)]
    assert _spans(filter_bam, R("misc", 9000, 10500)) == [((9000, 10500),)]     # trimmed to the region
    assert _spans(filter_bam, R("misc", 10500, 12000)) == []                     # 500 bases left: too short
    assert _spans(filter_bam, R("misc", 10500, 12000), min_length=500) == [((10500, 11000),)]


def test_truth_haplotype_grouping(filter_bam):
    """x and y (haplotype 2) are trimmed to abut first (3500 / 4000); a (haplotype 1) overlaps x the most, so the
    pair is cut to x's window; b has no haplotype-2 partner and is skipped."""
    assert _spans(filter_bam, R("haps", 0, 20000), haplotag="HP") == [((1500, 3500), (1500, 3500))]
    from medaka_b200 import features
    with pytest.raises(ValueError):
        features.CountsFeatureEncoder().bams_to_training_samples(filter_bam, filter_bam, R("haps", 0, 20000),
                                                                 labels.HaploidLabelScheme(), truth_haplotag="HP")


def test_truth_without_md_raises(tmp_path):
    d = _draft(3000)
    rec = dict(_perfect(d, 100, 2000, "no_md", tags={}), ref=0)
    del rec["tags"]["MD"]
    path = str(tmp_path / "nomd.bam")
    write_bam(path, [("ref", 3000)], [rec])
    with pytest.raises(ValueError):
        labels.TruthAlignment.bam_to_alignments(path, R("ref", 0, 3000))


def test_create_samples_argument_errors(tmp_path):
    from medaka_b200 import features
    out = str(tmp_path / "out.npzstore")
    with pytest.raises(ValueError):
        features.create_samples("reads.bam", out, chunk_len=1000, chunk_ovlp=1000)
    for name in ("DiploidLabelScheme", "RLELabelScheme"):
        with pytest.raises(NotImplementedError):
            features.create_samples("reads.bam", out, truth="truth.bam", label_scheme=name)
    with pytest.raises(NotImplementedError):
        features.CountsFeatureEncoder().bams_to_training_samples("t.bam", "r.bam", R("ref", 0, 10), object())
    assert not os.path.exists(out)


# ------------------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
def test_gpu_test_030(tmp_path):
    """medaka/test/test_counts.py:73-115: features, positions and labels of the reference's simple case."""
    from medaka_b200 import features
    reads, truth = str(tmp_path / "reads.bam"), str(tmp_path / "truth.bam")
    write_bam(reads, [("ref", 8)], [dict(r, ref=0) for r in SIMPLE_CALLS])
    write_bam(truth, [("ref", 8)], [dict(TEST_030_TRUTH, ref=0)])
    enc = features.CountsFeatureEncoder(normalise='total')
    result = enc.bams_to_training_samples(truth, reads, R('ref', 0, 100), labels.HaploidLabelScheme(), min_length=0)[0]
    assert result.labels.tolist() == [1, 2, 1, 4, 1, 3, 1, 4, 3] and result.labels.dtype == np.int64
    assert [tuple(p) for p in result.positions.tolist()] == [(0, 0), (1, 0), (2, 0), (3, 0), (3, 1), (4, 0), (5, 0),
                                                             (6, 0), (7, 0)]
    np.testing.assert_equal(result.features, TEST_030_FEATURES)


@pytest.mark.gpu
def test_gpu_truth_labels_real_slice(golden_dir):
    from medaka_b200 import features
    g = _golden(golden_dir)
    ta = labels.TruthAlignment(_golden_truth(g))
    ta.start, ta.end = int(g["start"]), int(g["end"])
    _, _, pos = features.pileup_features_from_batch(_golden_reads(g), ta.start, ta.end)
    assert np.array_equal(pos["major"], g["major"]) and np.array_equal(pos["minor"], g["minor"])
    got = labels.HaploidLabelScheme().label_columns((ta,), pos)
    assert np.array_equal(got, g["labels"]) and got.dtype == np.int64


@pytest.mark.gpu
def test_gpu_truth_labels_synthetic():
    """mdk_truth_labels equals the oracle's dictionary join on seeded truths with every CIGAR op, windows that start or
    end inside deletions or at insertion runs, minors beyond the runs, and 0 or 1 columns."""
    rs = np.random.RandomState(11)
    n_checked = 0
    for _ in range(60):
        d = _synth_truth(rs, pos=int(rs.randint(0, 200)))
        rec = _record(d)
        cand = _clip_candidates(d)
        cols = _columns(d, rs)
        for _ in range(4):
            s, e = (int(x) for x in sorted(rs.choice(cand, 2)))
            ta, to = labels.TruthAlignment(rec), truth_oracle.Truth(d)
            ta.start, ta.end = to.start, to.end = s, e
            for c in (cols, cols[:0], cols[rs.randint(len(cols)):][:1]):
                got = labels.truth_labels(ta, c)
                assert np.array_equal(got, truth_oracle.join_labels(to, c)), (d["cigar"], s, e)
                n_checked += len(c)
    assert n_checked > 10000


def _synth_bams(tmp, seed, num_dtypes=1, L=30000):
    rs = np.random.RandomState(seed)
    draft = _draft(L, seed)
    truths = [_truth_from_draft(draft, 200, 9000, rs, query_name="t0"),
              _truth_from_draft(draft, 8800, 19500, rs, query_name="t1"),        # small overlap: trimmed
              _truth_from_draft(draft, 20500, 21200, rs, query_name="t2"),       # too short
              _truth_from_draft(draft, 21500, 29900, rs, query_name="t3")]
    for t in truths:
        t["flag"] = 2064
    reads = synth.synth_reads(300, L, seed=seed, mean_len=2500, num_dtypes=num_dtypes)
    rpath, tpath = os.path.join(tmp, "reads.bam"), os.path.join(tmp, "truth.bam")
    write_bam(rpath, [("ctg", L)], [dict(r, ref=0) for r in reads])
    write_bam(tpath, [("ctg", L)], [dict(t, ref=0) for t in truths])
    return rpath, tpath, truths, reads


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["counts", "counts2", "read_level"])
def test_gpu_create_samples_matches_oracle(tmp_path, monkeypatch, kind):
    """create_samples over 12 kb pieces (the last overlapping the one before, like Region.split's at 1 Mb): the sample
    names of the oracle, labels equal to it, features bit-identical to bam_to_sample's over the truth spans."""
    from medaka_b200 import datastore, features
    num_dtypes = 2 if kind == "counts2" else 1
    rpath, tpath, truths, reads = _synth_bams(str(tmp_path), 5 + num_dtypes, num_dtypes)
    dts = ("dt0", "dt1") if num_dtypes == 2 else ("",)
    enc = (features.ReadAlignmentFeatureEncoder(dtypes=dts) if kind == "read_level"
           else features.CountsFeatureEncoder(dtypes=dts))
    monkeypatch.setattr(features, "MAX_REGION_SIZE", 12000)
    out = str(tmp_path / "train.npzstore")
    n = features.create_samples(rpath, out, truth=tpath, feature_encoder=enc, chunk_len=1000, chunk_ovlp=100)
    want = truth_oracle.create_samples(truths, reads, "ctg", 30000, chunk_len=1000, chunk_ovlp=100, max_size=12000,
                                       dtypes=list(dts) if num_dtypes > 1 else None)
    expect_feats = {}
    for s0, s1 in ((0, 12000), (12000, 24000), (18000, 30000)):
        for g in truth_oracle.bam_to_alignments(truths, "ctg", s0, s1):
            for src in enc.bam_to_sample(rpath, R("ctg", g[0].start, g[0].end)):
                if src.size >= 1000:
                    for c in src.chunks(1000, 100):
                        expect_feats.setdefault(c.name, c.features)
    with datastore.DataStore(out) as ds:
        assert n == len(want) > 20 and ds.sample_registry == set(want)
        assert type(ds.get_meta("feature_encoder")) is type(enc)
        assert isinstance(ds.get_meta("label_scheme"), labels.HaploidLabelScheme)
        for name, (pos, lab) in want.items():
            s = ds.load_sample(name)
            assert np.array_equal(s.positions["major"], pos["major"]) and np.array_equal(s.positions["minor"], pos["minor"])
            assert np.array_equal(s.labels, lab) and s.labels.dtype == np.int64
            assert np.array_equal(s.features, expect_feats[name])


@pytest.mark.gpu
def test_gpu_create_samples_unlabelled_and_empty(tmp_path):
    from medaka_b200 import datastore, features
    rpath, tpath, _, _ = _synth_bams(str(tmp_path), 3)
    out = str(tmp_path / "plain.npzstore")
    n = features.create_samples(rpath, out, chunk_len=1000, chunk_ovlp=100)
    with datastore.DataStore(out) as ds:
        assert n > 20 and all(ds.load_sample(k).labels is None for k in list(ds.sample_registry)[:5])
    empty = str(tmp_path / "empty.npzstore")
    assert features.create_samples(rpath, empty, regions=["ctg:20500-21200"], truth=tpath, chunk_len=1000,
                                   chunk_ovlp=100) == 0
    assert not os.path.exists(empty)


@pytest.mark.gpu
def test_gpu_created_store_trains(tmp_path):
    """A store from create_samples through TrainBatcher and one run_training epoch."""
    from medaka_b200 import features, training
    rpath, tpath, _, _ = _synth_bams(str(tmp_path), 4)
    store = str(tmp_path / "train.npzstore")
    features.create_samples(rpath, store, truth=tpath, chunk_len=500, chunk_ovlp=50)
    batcher = training.TrainBatcher([store], validation=0.25, seed=1, batch_size=8)
    assert batcher.n_batches("train") >= 2 and batcher.n_batches("valid") >= 1
    out = str(tmp_path / "run")
    model_fp = str(tmp_path / "model.toml")
    with open(model_fp, "w") as fh:
        fh.write('type = "GRUModel"\n[kwargs]\nnum_features = 10\nnum_classes = 5\ngru_size = 128\n')
    training.run_training(out, batcher, model_fp=model_fp, epochs=1, use_lr_schedule=False)
    rows = np.genfromtxt(os.path.join(out, "training.csv"), delimiter=",", names=True)
    assert np.isfinite(rows["train_loss"]) and np.isfinite(rows["val_loss"])
    for name in ("model-0.tar.gz", "model-best_val_loss.tar.gz"):
        assert os.path.exists(os.path.join(out, name))
