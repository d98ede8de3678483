"""Counts models with three and four datatypes (F = 30 and 40), the widest the C ABI accepts (1..4 datatypes).

Every part a three- or four-datatype model runs that F = 10 and 20 do not: normalise_kernel<3> / <4>, the pileup's
datatype indices 2 and 3, inproj0_generic_kernel (the layer-0 input projection of every F other than 10 and 20, quad
layout on the tc path, plain rows on fp32), the engine's per-F staging, and the packing, decoded heads and layer overlap
at those widths.  Pinned to the reference through tests/golden/multi_dtype.npz (tests/golden/make_multi_dtype_golden.py
runs the reference's own CountsFeatureEncoder and GRUModel), and to the oracle at the bars the suite uses for F = 10, 20.
"""
import os
import re
import tempfile
from timeit import default_timer as now

import numpy as np
import pytest

from oracle import features_oracle, gru_oracle, pileup_oracle, read_matrix_oracle, synth
from tests import test_gpu_parity, test_gru_pack
from tests.test_gpu_parity import label_parity
from tests.test_gru_pack import driver  # noqa: F401  (the packer's native driver, a fixture)
from tests.test_gru_stages import BARS, STAGES, _check, _device, _errors, _features, _model, _need_memory, _sd

DTYPES = {3: ("r9", "r10", "x"), 4: ("r9", "r10", "x", "y")}
NORM_NAMES = ["%s%d" % (k, nd) for nd in (3, 4) for k in ("synth", "minor_start", "deep", "empty_dt", "wrap")]
MODES = ["total", "fwd_rev", None]
FORWARD_CASES = ["f30", "f40", "f40_b1", "f40_hot"]


@pytest.fixture(scope="module")
def gold(golden_dir):
    return np.load(os.path.join(golden_dir, "multi_dtype.npz"))


def _norm_case(gold, name):
    counts = gold["norm_%s_counts" % name].copy()
    pos = np.empty(len(counts), dtype=[("major", "<i8"), ("minor", "<i8")])
    pos["major"], pos["minor"] = gold["norm_%s_major" % name], gold["norm_%s_minor" % name]
    return counts, pos, DTYPES[counts.shape[1] // 10]


def _forward_case(gold, name):
    seed, B, T, F, head_gain, rec_gain = gold["fwd_%s_args" % name]
    sd = synth.synth_state_dict(int(seed), num_features=int(F), head_gain=head_gain, rec_gain=rec_gain)
    return sd, synth.synth_features(int(B), int(T), int(F), seed=100 + int(seed)), int(F)


def _pieces(positions):
    """[a, b) bounds of the gap-free pieces (the reference normalises each on its own, features.py:125-134)."""
    cuts = np.where(np.ediff1d(positions["major"]) > 1)[0] + 1
    bounds = [0] + cuts.tolist() + [len(positions)]
    return list(zip(bounds[:-1], bounds[1:]))


def _oracle_features(counts, positions, normalise, dtypes, sym=False):
    f = np.empty(counts.shape, np.float32)
    d = np.empty(len(counts), np.int64)
    for a, b in _pieces(positions):
        f[a:b], d[a:b] = features_oracle.post_process_pileup(counts[a:b].copy(), positions[a:b], normalise,
                                                             dtypes=dtypes, sym_indels=sym)
    return f, d


# ---------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("name", NORM_NAMES)
def test_oracle_reproduces_post_processing_golden(gold, name):
    counts, pos, dtypes = _norm_case(gold, name)
    for norm in MODES:
        for sym in (False, True):
            key = "norm_%s_%s_%d" % (name, norm, int(sym))
            f, d = features_oracle.post_process_pileup(counts.copy(), pos, norm, dtypes=dtypes, sym_indels=sym)
            assert np.array_equal(f, gold[key + "_features"]), key
            assert np.array_equal(d.astype(np.int64), gold[key + "_depth"].astype(np.int64)), key
    if name.startswith("empty_dt"):      # a (datatype, strand) group without reads: np.maximum(1, 0) in fwd_rev
        assert not counts[30:90, 10:20].any() and counts[30:90].any()
    if name.startswith("wrap"):          # the sym_indels fill wrapped around in uint64
        assert (gold["norm_%s_None_1_features" % name] > 1e18).any()


def test_norm_indices_golden(gold):
    for nd, dtypes in DTYPES.items():
        got = features_oracle.pileup_counts_norm_indices(list(dtypes))
        keys = [k for k in gold.files if k.startswith("idx_%s|" % ",".join(dtypes))]
        assert len(keys) == len(got) == 2 * nd
        for (dt, rev), v in got.items():
            assert np.array_equal(v, gold["idx_%s|%s|%d" % (",".join(dtypes), dt, int(rev))])


@pytest.mark.parametrize("name", FORWARD_CASES)
def test_oracle_reproduces_forward_golden(gold, name):
    sd, feats, F = _forward_case(gold, name)
    probs, logits = gru_oracle.predict_on_batch(gru_oracle.build(sd, num_features=F), feats)
    assert np.abs(probs - gold["fwd_%s_probs" % name]).max() <= 2e-6
    assert np.abs(logits - gold["fwd_%s_logits" % name]).max() <= 2e-6


@pytest.mark.parametrize("F", [30, 40])
def test_gru_pack_layouts_wide(driver, tmp_path, F):  # noqa: F811
    """The host packer at F = 30 / 40: layer 0 has no tensor-core x weights (F > 16), everything else as at F = 10."""
    test_gru_pack.test_gru_pack_layouts(driver, tmp_path, F)


@pytest.mark.parametrize("F", [30, 40])
def test_featuriser_like_features_wide(F):
    """The properties test_gru_stages checks of featuriser-like windows, per datatype: coverage gaps, major columns whose
    strand groups are each normalised to 1 and one-hot-like, sparse small minors, values fp16 cannot hold."""
    nd, T = F // 10, 3000
    x = gru_oracle.featuriser_like_features(4, T, F, seed=5)
    assert x.shape == (4, T, F) and x.dtype == np.float32 and x.min() >= 0
    s = x.sum(-1)
    empty = s == 0
    assert empty.any(1).all() and empty.mean() < 0.2
    minor_any = np.zeros_like(empty)
    for dt in range(nd):
        groups = [[dt * 10 + i for i in g] for g in ([0, 1, 2, 3, 8], [4, 5, 6, 7, 9])]
        gs = np.stack([x[..., g].sum(-1) for g in groups], -1)
        major = (np.abs(gs - 1) < 1e-5).all(-1)
        assert 0.55 < major.mean() < 0.95, (dt, major.mean())
        xd = x[..., dt * 10:(dt + 1) * 10]
        top = np.sort(xd[major], -1)[:, -2:].sum(-1) / 2          # the true base on each strand
        assert np.median(top) > 0.85, dt
        minor = ~empty & (gs < 1 - 1e-5).all(-1) & (gs.sum(-1) > 0)
        minor_any |= minor
        assert (xd[minor] == 0).mean() > 0.5 and np.median(xd[minor].sum(-1)) / 2 < 0.5, dt
    assert minor_any.mean() > 0.05
    v = x[x > 0]
    assert (v.astype(np.float16).astype(np.float32) != v).mean() > 0.3


@pytest.mark.parametrize("weights", ["default", "hot"])
def test_ablations_exceed_the_bars_at_f40(weights):
    """At F > 16 the layer-0 projection is fp32 (no x / w_ih0 products to lose); every ablation of the products the
    unfused path still has moves some stage by more than 3x its bar."""
    sd = _sd(weights, F=40)
    x = gru_oracle.featuriser_like_features(4, 2000, 40, seed=3)
    ref = gru_oracle.stages(sd, x)
    for which in ("w_hh", "w_ih1", "h", "h0"):
        sd_a, kw = gru_oracle.ablate(sd, which)
        err = _errors(gru_oracle.stages(sd_a, x, **kw), ref)
        ratio = {k: err[k] / BARS[k] for k in STAGES}
        print("gru-ablation f40 %-7s %-5s %s" % (weights, which, " ".join("%s=%.3g (%.1fx)" % (k, err[k], ratio[k])
                                                                            for k in STAGES)))
        assert max(ratio.values()) > 3, (which, err)


# ---------------------------------------------------------------------------------------------- GPU: normalisation
def _lm():
    from medaka_b200 import libmedaka
    libmedaka.load()
    return libmedaka


def _normalise_dev(counts, pos, nd, norm, sym):
    """mdk_normalise_counts_dev on device copies of counts and positions."""
    from medaka_b200 import features
    from tests.test_forward_dev import DevBuf
    lm = _lm()
    n = len(counts)
    bufs = [DevBuf(counts.nbytes).upload(np.ascontiguousarray(counts, np.uint64)),
            DevBuf(8 * n).upload(np.ascontiguousarray(pos["major"], np.int64)),
            DevBuf(8 * n).upload(np.ascontiguousarray(pos["minor"], np.int64)),
            DevBuf(4 * n * 10 * nd).upload(np.full((n, 10 * nd), -1, np.float32)),
            DevBuf(8 * n).upload(np.full(n, -1, np.int64))]
    try:
        lm.check(lm.lib.mdk_normalise_counts_dev(0, bufs[0].cast("const uint64_t *"), bufs[1].cast("const int64_t *"),
                                                 bufs[2].cast("const int64_t *"), n, nd, features._NORM_MODES[norm],
                                                 int(sym), bufs[3].cast("float *"), bufs[4].cast("int64_t *")))
        return bufs[3].download((n, 10 * nd), np.float32), bufs[4].download(n, np.int64)
    finally:
        for b in bufs:
            b.free()


def _normalise_host(counts, pos, dtypes, norm, sym):
    from medaka_b200 import common, features
    enc = features.CountsFeatureEncoder(normalise=norm, dtypes=dtypes, sym_indels=sym)
    s = enc._post_process_pileup(counts.copy(), pos,
                                 common.Region("ref", int(pos["major"][0]), int(pos["major"][-1]) + 1))
    return s.features, np.asarray(s.depth).astype(np.int64)


@pytest.mark.gpu
@pytest.mark.parametrize("name", NORM_NAMES)
def test_normalise_golden_bit_exact(gold, name):
    counts, pos, dtypes = _norm_case(gold, name)
    for norm in MODES:
        for sym in (False, True):
            key = "norm_%s_%s_%d" % (name, norm, int(sym))
            want_f, want_d = gold[key + "_features"], gold[key + "_depth"].astype(np.int64)
            for how, (f, d) in (("host", _normalise_host(counts, pos, dtypes, norm, sym)),
                                ("dev", _normalise_dev(counts, pos, len(dtypes), norm, sym))):
                assert f.dtype == np.float32 and np.array_equal(f, want_f), (key, how)
                assert np.array_equal(d, want_d), (key, how)


@pytest.mark.gpu
@pytest.mark.parametrize("nd", [3, 4])
def test_normalise_large_and_single_column(nd):
    counts, pos = synth.synth_counts(2000000, seed=130 + nd, num_dtypes=nd)
    for norm, sym in (("fwd_rev", True), ("total", False)):
        ef, ed = features_oracle.post_process_pileup(counts.copy(), pos, norm, dtypes=DTYPES[nd], sym_indels=sym)
        f, d = _normalise_host(counts, pos, DTYPES[nd], norm, sym)
        assert np.array_equal(f, ef) and np.array_equal(d, ed.astype(np.int64)), norm
    one = counts[:1].copy()
    one[0, 10:20] = 0                                # one datatype without reads
    for norm in MODES:
        for sym in (False, True):
            ef, ed = features_oracle.post_process_pileup(one.copy(), pos[:1], norm, dtypes=DTYPES[nd], sym_indels=sym)
            for f, d in (_normalise_host(one, pos[:1], DTYPES[nd], norm, sym),
                         _normalise_dev(one, pos[:1], nd, norm, sym)):
                assert np.array_equal(f, ef) and np.array_equal(d, ed.astype(np.int64)), (norm, sym)


# ---------------------------------------------------------------------------------------------- GPU: pileup
def _dt_names(nd):
    return ["dt%d" % k for k in range(nd)]


@pytest.mark.gpu
@pytest.mark.parametrize("seed,nd,p_skip,ins_after_skip", [(20, 3, 0.0, False), (21, 4, 0.0, False),
                                                           (22, 3, 0.05, True), (23, 4, 0.08, True)])
def test_pileup_counts_random_reads(seed, nd, p_skip, ins_after_skip):
    from medaka_b200 import bam, features
    recs = synth.synth_reads(300, 4000, seed=seed, mean_len=800, p_skip=p_skip, num_dtypes=nd,
                             ins_after_skip=ins_after_skip)
    assert {r["tags"]["DT"] for r in recs} == set(_dt_names(nd))
    batch = bam.records_from_dicts(recs, _dt_names(nd))
    for s, e, mq in [(0, 4000, 1), (1000, 2500, 1), (500, 600, 20), (3990, 4000, 1)]:
        c, p = features.pileup_counts_from_batch(batch, s, e, num_dtypes=nd, min_mapq=mq)
        ec, ep = pileup_oracle.pileup_counts(recs, s, e, dtypes=_dt_names(nd), min_mapq=mq)
        assert c.shape[1] == 10 * nd
        assert np.array_equal(p, ep), (s, e)
        assert np.array_equal(c, ec), (s, e)
        if e - s > 1000:
            assert all(c[:, 10 * k:10 * (k + 1)].any() for k in range(nd))


@pytest.mark.gpu
@pytest.mark.parametrize("nd", [3, 4])
def test_pileup_counts_long_operations_over_all_datatypes(nd):
    """The long-operation reads of test_pileup (a 5 kb match, a 3 kb deletion, a 2 kb skip then an insertion) and 1500
    random reads, datatypes assigned round-robin; a stretch [6000, 7000) covered by the last datatype only."""
    from medaka_b200 import bam, features
    rs = np.random.RandomState(5)
    seq = lambda n: "".join(rs.choice(list("ACGT"), n))  # noqa: E731
    recs = [dict(query_name="longM", pos=10, cigar="5000M", seq=seq(5000), flag=0, mapq=60, tags={}),
            dict(query_name="longD", pos=500, cigar="100M3000D100M", seq=seq(200), flag=16, mapq=60, tags={}),
            dict(query_name="skipI", pos=700, cigar="50M2000N4I60M", seq=seq(114), flag=0, mapq=60, tags={})]
    recs += synth.synth_reads(1500, 9000, seed=9, mean_len=2500, p_skip=0.01, ins_after_skip=True)
    names = _dt_names(nd)
    keep = []
    for i, r in enumerate(recs):
        r["tags"] = {"DT": names[i % nd]}
        ref_len = sum(int(n) for n, op in re.findall(r"(\d+)([MDN=X])", r["cigar"]))
        if r["pos"] < 7000 and r["pos"] + ref_len > 6000 and r["tags"]["DT"] != names[-1]:
            continue                       # only the last datatype covers [6000, 7000)
        keep.append(r)
    recs = sorted(keep, key=lambda r: r["pos"])
    batch = bam.records_from_dicts(recs, names)
    for s, e in [(0, 9000), (2040, 4100), (4095, 4097), (5900, 7100)]:
        c, p = features.pileup_counts_from_batch(batch, s, e, num_dtypes=nd)
        ec, ep = pileup_oracle.pileup_counts(recs, s, e, dtypes=names)
        assert np.array_equal(p, ep), (s, e)
        assert np.array_equal(c, ec), (s, e)
        assert int(c.sum()) > 0
    only = (p["major"] >= 6000) & (p["major"] < 7000)
    assert only.any() and not c[only, :10 * (nd - 1)].any() and c[only, 10 * (nd - 1):].any()


@pytest.mark.gpu
@pytest.mark.parametrize("nd", [3, 4])
def test_fused_pileup_features_match_two_step(nd):
    """mdk_pileup_features against oracle pileup + oracle post-processing per gap-free piece, every mode x sym_indels."""
    from medaka_b200 import bam, features
    from tests.test_pileup import _clip_cigar
    recs = synth.synth_reads(200, 2400, seed=40 + nd, mean_len=300, num_dtypes=nd)
    recs = [r for r in recs if not (900 <= r["pos"] < 1100)]
    for r in recs:
        if r["pos"] < 900:
            r["cigar"] = _clip_cigar(r["cigar"], 900 - r["pos"])
    names = _dt_names(nd)
    batch = bam.records_from_dicts(recs, dtypes=names)
    ec, ep = pileup_oracle.pileup_counts(recs, 100, 2300, dtypes=names)
    assert (np.ediff1d(ep["major"]) > 1).any()
    for normalise in MODES:
        for sym in (False, True):
            feats, depth, pos = features.pileup_features_from_batch(batch, 100, 2300, nd, 1, normalise, sym)
            assert np.array_equal(pos, ep)
            ef, ed = _oracle_features(ec, ep, normalise, names, sym)
            assert np.array_equal(feats, ef), (normalise, sym)
            assert np.array_equal(depth, ed), (normalise, sym)


def _bam_reads(nd, seed, n_reads=160, ref_len=4000, hole=(1400, 1500)):
    """Reads of nd datatypes (DT tags) on contig 0, none covering [hole[0], hole[1]): a coverage gap."""
    from tests.test_pileup import _clip_cigar
    recs = synth.synth_reads(n_reads, ref_len, seed=seed, mean_len=500, num_dtypes=nd)
    recs = [r for r in recs if not (hole[0] <= r["pos"] < hole[1])]
    for r in recs:
        if r["pos"] < hole[0]:
            r["cigar"] = _clip_cigar(r["cigar"], hole[0] - r["pos"])
            r["seq"] = r["seq"][:sum(int(n) for n, op in re.findall(r"(\d+)([MIS=X])", r["cigar"]))]
    recs.sort(key=lambda r: r["pos"])
    for r in recs:
        r["ref"] = 0
    return recs


@pytest.mark.gpu
def test_bam_to_sample_three_datatypes(tmp_path):
    """CountsFeatureEncoder(dtypes=<3 names>).bam_to_sample on a BAM with DT tags (native reader -> fused featuriser)
    equals the two-step path and the oracle, sample by sample."""
    from medaka_b200 import common, features
    from tests import bamutil
    names = _dt_names(3)
    recs = _bam_reads(3, seed=8, n_reads=150, ref_len=3000)
    path = str(tmp_path / "r.bam")
    bamutil.write_bam(path, [("ctg", 3000)], recs)
    region = common.Region("ctg", 0, 3000)
    ec, ep = pileup_oracle.pileup_counts(recs, 0, 3000, dtypes=names)
    for normalise, sym in (("total", True), ("fwd_rev", False), ("fwd_rev", True), (None, False)):
        enc = features.CountsFeatureEncoder(normalise=normalise, dtypes=tuple(names), sym_indels=sym)
        fused = enc.bam_to_sample(path, region)
        two = [enc._post_process_pileup(c, p, region) for c, p in enc._pileup_function(region, path)]
        assert len(fused) == len(two) == len(_pieces(ep)) >= 2
        ef, ed = _oracle_features(ec, ep, normalise, names, sym)
        for a, b, (lo, hi) in zip(fused, two, _pieces(ep)):
            assert a.features.shape[1] == 30
            assert np.array_equal(a.positions, b.positions) and np.array_equal(a.positions, ep[lo:hi])
            assert np.array_equal(a.features, b.features) and np.array_equal(a.features, ef[lo:hi])
            assert np.array_equal(np.asarray(a.depth), np.asarray(b.depth))
            assert np.array_equal(np.asarray(a.depth), ed[lo:hi])


@pytest.mark.gpu
def test_five_datatypes_are_refused(tmp_path):
    from medaka_b200 import bam, common, features
    from medaka_b200.libmedaka import MedakaB200Error
    from tests import bamutil
    names = _dt_names(5)
    recs = _bam_reads(5, seed=11, n_reads=60, ref_len=2000)
    path = str(tmp_path / "r.bam")
    bamutil.write_bam(path, [("ctg", 2000)], recs)
    region = common.Region("ctg", 0, 2000)
    enc = features.CountsFeatureEncoder(normalise="total", dtypes=tuple(names))
    got = None
    with pytest.raises(MedakaB200Error, match=r"1\.\.4 dtypes"):
        got = enc.bam_to_sample(path, region)
    assert got is None
    with pytest.raises(MedakaB200Error, match=r"1\.\.4 dtypes"):
        enc._pileup_function(region, path)
    with pytest.raises(MedakaB200Error, match=r"1\.\.4 dtypes"):
        features.pileup_counts_from_batch(bam.records_from_dicts(recs, names), 0, 2000, num_dtypes=5)
    counts, pos = synth.synth_counts(100, seed=1, num_dtypes=5)
    with pytest.raises(MedakaB200Error, match=r"1\.\.4 dtypes"):
        enc._post_process_pileup(counts, pos, common.Region("ctg", 0, int(pos["major"][-1]) + 1))


# ---------------------------------------------------------------------------------------------- GPU: forward
def _make(sd, F, precision="tc", rec="auto", keep=False):
    return _model(sd, F, precision, rec, keep)


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp32", "tc"])
@pytest.mark.parametrize("name", FORWARD_CASES)
def test_forward_matches_reference_golden(gold, name, precision):
    sd, feats, F = _forward_case(gold, name)
    m = _make(sd, F, precision)
    out = m.forward_arrays(feats, want_logits=True, want_labels=True)
    m.close()
    ref_logits, ref_probs = gold["fwd_%s_logits" % name], gold["fwd_%s_probs" % name]
    err = float((np.abs(out.logits - ref_logits) / np.abs(ref_logits).max(-1, keepdims=True)).max())
    perr = float(np.abs(out.probs - ref_probs).max())
    flips, tie_flips, ties = label_parity(out.labels, ref_probs)
    print("%s/%s: scaled logit err %.3e, prob err %.3e, label mismatches %d/%d (+%d among %d near-ties)" % (
        name, precision, err, perr, flips, out.labels.size, tie_flips, ties))
    assert err <= test_gpu_parity.LOGIT_TOL and perr <= 1e-3 and flips == 0
    assert np.array_equal(out.labels, np.argmax(out.probs, -1))


PATHS = [("tc", "one"), ("tc", "pp"), ("fp32", "auto")]
PATH_IDS = ["tc-one_tile", "tc-two_tiles", "fp32"]


def _run_paths(sd, F, x, windows, want, label, path, rec):
    for keep in (False, True):
        m = _make(sd, F, path, rec, keep)
        t0 = now()
        got = _device(m, x, windows, path == "tc" and not keep)
        t = now() - t0
        timings = m.last_timings()
        m.close()
        print("%s %s %s keep=%d: %.2f s, inproj0 %.2f ms" % (label, path, rec, keep, t, timings.get("inproj0_ms", -1)))
        _check(got, want, "%s %s %s keep=%d" % (label, path, rec, keep))


@pytest.fixture(scope="module")
def wide_case():
    """wide_case(F): 300 windows x 10 000 columns, featuriser-like at (0, 17, 150, 299), and their float64 stages."""
    cache = {}

    def get(F):
        if F not in cache:
            windows = (0, 17, 150, 299)
            sd = _sd("default", F=F, seed=35 + F)
            x = _features(300, 10000, F, windows, seed=35 + F)
            cache[F] = sd, x, windows, gru_oracle.stages(sd, x[list(windows)])
        return cache[F]
    yield get
    cache.clear()


@pytest.mark.gpu
@pytest.mark.parametrize("path,rec", PATHS, ids=PATH_IDS)
@pytest.mark.parametrize("F", [30, 40])
def test_stage_bars_wide(wide_case, F, path, rec):
    """Layer 0 unfused, inproj0_generic_kernel writing gi (quad layout on tc, plain rows on fp32); every stage within the
    F = 10 bars, with and without keep_activations."""
    _need_memory(20)
    sd, x, windows, want = wide_case(F)
    _run_paths(sd, F, x, windows, want, "f%d" % F, path, rec)


@pytest.mark.gpu
@pytest.mark.parametrize("rec", ["one", "pp"])
@pytest.mark.parametrize("T", [1, 129])
@pytest.mark.parametrize("B", [37, 1217])
@pytest.mark.parametrize("F", [30, 40])
def test_ragged_wide(F, B, T, rec):
    windows = tuple(range(37)) if B == 37 else (0, 15, 16, 1200, 1215, 1216)
    sd = _sd("default", F=F, seed=36)
    x = _features(B, T, F, windows, seed=36 + T)
    want = gru_oracle.stages(sd, x[list(windows)])
    for path, keep in (("tc", False), ("tc", True), ("fp32", False), ("fp32", True)):
        m = _make(sd, F, path, rec, keep)
        got = _device(m, x, windows, path == "tc" and not keep)
        m.close()
        _check(got, want, "ragged F=%d B=%d T=%d %s %s keep=%d" % (F, B, T, path, rec, keep))


@pytest.fixture(scope="module")
def full_group():
    cache = {}

    def get():
        if not cache:
            from tests.test_gru_stages import PROD_B, PROD_T, PROD_WINDOWS
            sd = _sd("default", F=40, seed=37)
            x = _features(PROD_B, PROD_T, 40, PROD_WINDOWS, seed=37)
            cache["v"] = sd, x, PROD_WINDOWS, gru_oracle.stages(sd, x[list(PROD_WINDOWS)])
        return cache["v"]
    yield get
    cache.clear()


@pytest.mark.gpu
@pytest.mark.parametrize("path,rec", PATHS, ids=PATH_IDS)
def test_full_group_f40(full_group, path, rec):
    """One group at the shape bench.py runs, 1056 windows x 10 000 columns, at F = 40."""
    _need_memory(70)
    sd, x, windows, want = full_group()
    _run_paths(sd, 40, x, windows, want, "full f40", path, rec)


# ---------------------------------------------------------------------------------------------- GPU: engine plumbing
@pytest.mark.gpu
def test_pipelined_groups_f40():
    """Mixed-B submits over ten and more 48-window groups, a T change, a small-lane call and decoded calls in between:
    every call bit-identical to its lone forward."""
    from tests.test_layer_overlap import _pipelined
    m = _make(synth.synth_state_dict(16, num_features=40), 40)
    try:
        _pipelined(m, [(100, 3000), (90, 3000), (1, 500), (120, 2700), (70, 3000), (90, 3200), (60, 3200)], 70,
                   decoded=(1, 4))
    finally:
        m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["tc", "fp32"])
def test_forward_dev_packed_f40(precision):
    """forward_dev calls packed into 48-window groups (a call larger than a group, a T change, calls on both sides of the
    small-lane threshold) equal the same windows run alone, bit for bit."""
    from medaka_b200 import libmedaka as lm
    from tests.test_forward_dev import DevCall
    m = _make(synth.synth_state_dict(17, num_features=40), 40, precision)
    plan = [(30, 2000, True), (60, 2000, False), (1, 2000, True), (150, 2000, True), (20, 2000, False),
            (25, 1500, True), (60, 1500, False), (5, 1500, True)]
    feats = [synth.synth_features_fast(b, t, 40, seed=80 + i) for i, (b, t, _) in enumerate(plan)]
    try:
        want = [m.forward_arrays(x, want_logits=True) for x in feats]
        m.reserve(48, 2000)
        m.set_group_windows(48)
        calls = [DevCall(x, lg) for x, (_, _, lg) in zip(feats, plan)]
        for c in calls:
            c.run(m.engine)
        lm.check(lm.lib.mdk_engine_sync(m.engine))
        for i, (c, w) in enumerate(zip(calls, want)):
            probs, logits, labels = c.results()
            c.free()
            assert np.array_equal(probs, w.probs), "call %d: probabilities differ" % i
            assert np.array_equal(labels, w.labels), "call %d: labels differ" % i
            if logits is not None:
                assert np.array_equal(logits, w.logits), "call %d: logits differ" % i
    finally:
        m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("precision,rec,keep", [("tc", "auto", False), ("tc", "pp", False), ("tc", "auto", True),
                                                ("fp32", "auto", False)])
def test_decoded_heads_f40(precision, rec, keep):
    """submit_decoded and submit_variant_decoded outputs are mdk_decode_consensus / mdk_decode_variants of the ordinary
    forward's probabilities, bit for bit."""
    from tests.test_one_pass import _decode, _decoded
    from tests.test_one_pass_variants import _random_ref, _variant_decoded, _vd_of_probs
    B, T = 21, 50
    feats = synth.synth_features(B, T, 40, seed=B + T)
    ref = _random_ref(B, T, seed=B * T)
    m = _make(synth.synth_state_dict(3, num_features=40), 40, precision, rec, keep)
    try:
        probs = m.forward_arrays(feats).probs
        labels, quals = _decoded(m, feats)
        want_labels, want_quals = _decode(probs)
        assert np.array_equal(labels, want_labels) and np.array_equal(quals, want_quals)
        for g, w in zip(_variant_decoded(m, feats, ref), _vd_of_probs(probs, ref)):
            assert np.array_equal(g, w)
    finally:
        m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp32", "tc"])
def test_weight_reload_f40(precision):
    """An F = 40 model loaded over another: bit for bit a fresh model's forward, activations included."""
    test_gpu_parity.test_weight_reload_matches_fresh_model(precision, 40)


# ---------------------------------------------------------------------------------------------- GPU: end to end
def _e2e_model(F):
    sd = synth.synth_state_dict(6, num_features=F)
    sd["linear.bias"][0] -= 6.0          # fewer gap calls on real pileup features, so that most columns reach the output
    return _make(sd, F), sd


@pytest.mark.gpu
def test_end_to_end_three_datatypes():
    """A 3-datatype BAM and an F = 30 model: predict_consensus / predict_variants equal predict_regions + sequence() /
    variants(); the stored features are the oracle's and the stored probabilities within the forward bar of the oracle
    chain (pileup -> post-processing -> gru_oracle)."""
    from medaka_b200 import common, datastore, features, prediction
    from tests import bamutil
    from tests.test_one_pass import _both, _draft
    from tests.test_one_pass_variants import RUN, _check as check_variants
    names = _dt_names(3)
    recs = _bam_reads(3, seed=19, n_reads=200, ref_len=4000, hole=(2000, 2100))
    model, sd = _e2e_model(30)
    enc = features.CountsFeatureEncoder(normalise="fwd_rev", dtypes=tuple(names))
    regions = [common.Region("ctg", 0, 4000)]
    try:
        with tempfile.TemporaryDirectory() as d:
            path = os.path.join(d, "r.bam")
            bamutil.write_bam(path, [("ctg", 4000)], recs)
            (a, bed_a), (b, bed_b) = _both(d, model, enc, path, regions, _draft({"ctg": 4000}, seed=3))
            assert len(a) > 1000 and a == b and bed_a == bed_b
            check_variants(model, enc, path, regions, {"ctg": 4000}, [{}, {"return_all": True}], d, min_records=20)
            store = os.path.join(d, "feats.npzstore")
            prediction.predict_regions(store, path, regions, model, enc, save_features=True, **RUN)
            ds = datastore.DataStore(store, "r")
            samples = [ds.load_sample(k) for k in sorted(ds.sample_registry)]
            ds.close()
    finally:
        model.close()
    ec, ep = pileup_oracle.pileup_counts(recs, 0, 4000, dtypes=names)
    ef, _ = _oracle_features(ec, ep, "fwd_rev", names)
    row = {(int(a), int(b)): i for i, (a, b) in enumerate(zip(ep["major"], ep["minor"]))}
    oracle = gru_oracle.build(sd, num_features=30)
    assert len(samples) >= 4
    worst, flips = 0.0, 0
    for s in samples:
        rows = [row[(int(a), int(b))] for a, b in zip(s.positions["major"], s.positions["minor"])]
        x = ef[rows]
        if s.features is not None:
            assert np.array_equal(np.asarray(s.features), x)
        want, _ = gru_oracle.predict_on_batch(oracle, x[None])
        worst = max(worst, float(np.abs(np.asarray(s.label_probs) - want[0]).max()))
        flips += label_parity(np.argmax(np.asarray(s.label_probs), -1), want[0])[0]
    print("end to end F=30: %d windows, prob err %.3e, decided label flips %d" % (len(samples), worst, flips))
    assert worst <= 1e-3 and flips == 0


# ---------------------------------------------------------------------------------------------- GPU: read matrix
@pytest.mark.gpu
@pytest.mark.parametrize("nd", [3, 4])
def test_read_matrix_datatype_column(nd):
    from medaka_b200 import bam
    from tests.test_read_matrix import _device as read_matrix_device
    rs = np.random.RandomState(50 + nd)
    names = _dt_names(nd)
    recs = synth.synth_reads(260, 3000, seed=50 + nd, mean_len=500, num_dtypes=nd)
    for i, r in enumerate(recs):
        r["query_name"] = "read_%d" % i
        r["qual"] = rs.randint(0, 60, len(r["seq"])).tolist()
        if rs.uniform() < 0.7:
            r["tags"]["HP"] = int(rs.randint(0, 3))
        if rs.uniform() < 0.8:
            mv = [5] + (rs.uniform(size=3 * len(r["seq"])) < 0.34).astype(int).tolist()
            mv[1] = 1
            r["tags"]["mv"] = mv
    kw = dict(include_dwells=True, include_haplotype=True)
    want, wpos, wl, wr = read_matrix_oracle.read_alignment(recs, 400, 2600, dtypes=names, **kw)
    got, gpos, gl, gr = read_matrix_device(bam.records_from_dicts(recs, names), 400, 2600, num_dtypes=nd, **kw)
    assert got.shape == want.shape and got.shape[2] == 7
    assert np.array_equal(gpos, wpos) and np.array_equal(got, want) and gl == wl and gr == wr
    assert set(np.unique(got[..., -1])) >= set(range(nd))


@pytest.mark.gpu
def test_read_level_model_refuses_several_datatypes():
    """As the reference (latent_space_lstm.py:219): read-level models take one datatype only."""
    from medaka_b200 import features, read_level
    m = read_level.LatentSpaceLSTM()
    try:
        m.check_feature_encoder_compatibility(features.ReadAlignmentFeatureEncoder())
        for nd in (2, 3, 4):
            with pytest.raises(NotImplementedError, match="one dtype"):
                m.check_feature_encoder_compatibility(features.ReadAlignmentFeatureEncoder(dtypes=tuple(_dt_names(nd))))
    finally:
        m.close()
