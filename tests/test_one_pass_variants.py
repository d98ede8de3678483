"""One-pass variant calling: the engine's variant-decoded outputs (mdk_engine_submit_variant_decoded), the join cuts and
decode over device-resident rows (mdk_variant_join_cuts, mdk_decode_variants_dev), and predict_variants against
predict_regions + variant.variants."""
import os
import tempfile

import numpy as np
import pytest

from oracle import synth
from tests.test_one_pass import CASES, _model, _pileup_source


def _vd_of_probs(probs, ref):
    """What mdk_decode_variants computes from probabilities, as the call byte and the two phreds."""
    from medaka_b200 import labels
    ins = (ref & 0x80) != 0
    codes = ref & 0x07
    d = labels.decode_variant_arrays(probs.reshape(-1, 5), ins.reshape(-1).astype(np.int64), codes.reshape(-1))
    pred = d['pred'].reshape(ref.shape)
    calls = pred | ((pred != codes).astype(np.uint8) << 6) | (ref & 0x80)
    return calls, d['pred_q'].reshape(ref.shape), d['ref_q'].reshape(ref.shape)


def _random_ref(B, T, seed):
    rs = np.random.RandomState(seed)
    codes = rs.randint(0, 7, size=(B, T)).astype(np.uint8)          # '*ACGT', N (5) and other symbols (6)
    ins = rs.rand(B, T) < 0.2
    ins[0, 0] = False                                                # mdk_decode_variants starts on a major column
    codes[ins] = 0
    return codes | (ins.astype(np.uint8) << 7)


def _variant_decoded(m, feats, ref):
    x = m.pinned("vfeats", feats.shape, np.float32)
    np.copyto(x, feats)
    r = m.pinned("vref", ref.shape, np.uint8)
    np.copyto(r, ref)
    calls = np.empty(ref.shape, np.uint8)
    pq, rq = np.empty(ref.shape, np.float32), np.empty(ref.shape, np.float32)
    m.wait(m.submit_variant_decoded(x, r, calls, pq, rq))
    return calls, pq, rq


@pytest.mark.gpu
@pytest.mark.parametrize("precision,rec_mode,keep,F,B,T,kind", CASES)
def test_head_variant_outputs_equal_decode_of_probabilities(precision, rec_mode, keep, F, B, T, kind):
    if kind == "neartie":
        sd, feats = synth.synth_state_dict_neartie(5), synth.synth_features(B, T, F, seed=105)
    else:
        sd, feats = synth.synth_state_dict(3, num_features=F), synth.synth_features(B, T, F, seed=B + T)
    ref = _random_ref(B, T, seed=B * T)
    m = _model(sd, F, precision, rec_mode, keep)
    try:
        want = _vd_of_probs(m.forward_arrays(feats).probs, ref)
        got = _variant_decoded(m, feats, ref)
        for g, w in zip(got, want):
            assert np.array_equal(g, w)
    finally:
        m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("precision,keep", [("tc", False), ("tc", True), ("fp32", False)])
def test_ordinary_decoded_and_variant_decoded_calls_share_a_group(precision, keep):
    from medaka_b200 import libmedaka as lm
    from tests.test_one_pass import _decode
    lib, ffi = lm.load(), lm.ffi
    T = 200
    m = _model(synth.synth_state_dict(4), 10, precision, keep=keep)
    sizes = (5, 7, 9, 4)        # variant to host, ordinary, consensus-decoded to device, variant to device
    feats = [synth.synth_features(b, T, 10, seed=b) for b in sizes]
    refs = [_random_ref(b, T, seed=10 + b) for b in sizes]
    try:
        n0 = m.launch_count()
        alone = [m.forward_arrays(f) for f in feats]
        per_forward = (m.launch_count() - n0) // len(feats)
        m.set_group_windows(64)
        m.reserve(sum(sizes), T)
        xs = [m.pinned("mix%d" % i, f.shape, np.float32) for i, f in enumerate(feats)]
        rb = [m.pinned("mixr%d" % i, r.shape, np.uint8) for i, r in enumerate(refs)]
        for x, f, r, b in zip(xs, feats, rb, refs):
            np.copyto(x, f)
            np.copyto(r, b)
        v0 = (np.empty((5, T), np.uint8), np.empty((5, T), np.float32), np.empty((5, T), np.float32))
        probs1, labels1 = np.empty((7, T, 5), np.float32), np.empty((7, T), np.uint8)
        n2, n3 = 9 * T, 4 * T
        pp = ffi.new("void **")
        lm.check(lib.mdk_dev_alloc(0, 2 * n2 + 9 * n3, pp))
        dev = int(ffi.cast("uintptr_t", pp[0]))
        d3 = dev + 2 * n2
        try:
            n0 = m.launch_count()
            tickets = [m.submit_variant_decoded(xs[0], rb[0], *v0),
                       m.submit_arrays(xs[1], probs1, labels1),
                       m.submit_decoded(xs[2], dev, dev + n2),
                       m.submit_variant_decoded(xs[3], rb[3], d3, d3 + n3, d3 + 5 * n3)]
            for t in tickets:
                m.wait(t)
            m.sync()
            assert m.launch_count() - n0 == per_forward           # one forward ran all four calls
            back = np.empty(2 * n2 + 9 * n3, np.uint8)
            lm.check(lib.mdk_memcpy_d2h(0, ffi.cast("void *", ffi.from_buffer(back)), pp[0], len(back)))
        finally:
            lib.mdk_dev_free(0, pp[0])
        for g, w in zip(v0, _vd_of_probs(alone[0].probs, refs[0])):
            assert np.array_equal(g, w)
        assert np.array_equal(probs1, alone[1].probs) and np.array_equal(labels1, alone[1].labels)
        lab2, q2 = _decode(alone[2].probs)
        assert np.array_equal(back[:n2].reshape(9, T), lab2) and np.array_equal(back[n2:2 * n2].reshape(9, T), q2)
        tail = back[2 * n2:]
        got3 = (tail[:n3].reshape(4, T), tail[n3:5 * n3].view(np.float32).reshape(4, T),
                tail[5 * n3:].view(np.float32).reshape(4, T))
        for g, w in zip(got3, _vd_of_probs(alone[3].probs, refs[3])):
            assert np.array_equal(g, w)
    finally:
        m.close()


# ------------------------------------------------------------------------------- join and decode on device rows


def _windows(d, chunk_len, overlap):
    from medaka_b200 import common
    n = len(d['positions'])
    step = chunk_len - overlap
    ranges = [(lo, lo + chunk_len) for lo in range(0, n - chunk_len + 1, step)]
    if not ranges or ranges[-1][1] < n:
        ranges.append((max(0, n - chunk_len), n))
    return [common.Sample(d['ref_name'], None, None, None, d['positions'][a:b], d['label_probs'][a:b], None)
            for a, b in ranges], ranges


def _device_records(d, samples, ranges, arena_half, ambig_ref, return_all, verbose, seed=0):
    """The windows' variant-decoded rows (from their probabilities) in a real arena, placed in shuffled order across
    slabs; then the one-pass join / decode of the whole contig."""
    from medaka_b200 import common, labels, libmedaka as lm, prediction, stitch
    lib, ffi = lm.load(), lm.ffi
    ls = labels.HaploidLabelScheme()
    ls.verbose = verbose
    pos = d['positions']
    ins = pos['minor'] != 0
    ref = ls.reference_codes(pos, d['ref_seq']) | (ins.astype(np.uint8) << 7)
    calls, pq, rq = _vd_of_probs(d['label_probs'], ref)
    arena = prediction._LabelArena(0, prediction.VARIANT_ROW_BYTES, arena_half)
    views = {}
    try:
        for k in np.random.RandomState(seed).permutation(len(ranges)):
            a, b = ranges[k]
            slab, row = arena.take(b - a)
            for f, arr in enumerate((calls, pq, rq)):
                part = np.ascontiguousarray(arr[a:b])
                lm.check(lib.mdk_memcpy_h2d(0, ffi.cast("void *", arena.addr(slab, f, row)),
                                            ffi.cast("void *", ffi.from_buffer(part)), part.nbytes))
            s = samples[k]
            views[s.name] = (prediction._stitch_view(s, 0), slab, row)
        assert len(arena.slabs) >= 2
        samples_d = dict(views)
        index = stitch.sample_index(samples_d)
        region = common.Region(d['ref_name'], None, None)
        out = prediction._variants_of_region(region, samples_d, index, arena, ls, d['ref_seq'].upper(), ambig_ref,
                                             return_all)
        # the cuts: the joined samples' sizes equal join_samples'
        vs = [samples_d[n][0] for n in index[d['ref_name']]]
        pieces = stitch.plan_pieces(vs)
        inner = [p for p in pieces if not p.last]
        cuts = np.full(len(pieces), -1, np.int64)
        cuts[[k for k, p in enumerate(pieces) if not p.last]] = labels.variant_join_cuts(
            [arena.addr(samples_d[vs[p.sample].name][1], 0, samples_d[vs[p.sample].name][2] + p.lo) for p in inner],
            [p.hi - p.lo for p in inner])
        from medaka_b200 import variant
        sizes = [sum(hi - lo for _, lo, hi in g) for g in variant.joined_pieces(vs, pieces, cuts)]
    finally:
        arena.free()
    return out, sizes


def _host_records(d, samples, ambig_ref, return_all, verbose):
    from medaka_b200 import labels, variant
    ls = labels.HaploidLabelScheme()
    ls.verbose = verbose
    ref_seq = d['ref_seq'].upper()
    out, sizes = [], []
    for joined in variant.join_samples(variant.trimmed_samples(samples), ref_seq, ls):
        sizes.append(len(joined.positions))
        out.extend(variant.sort_records(ls.decode_variants(joined, ref_seq, ambig_ref=ambig_ref,
                                                           return_all=return_all)))
    return out, sizes


def _golden_cases():
    from tests.test_variants import golden
    for name, rec in sorted(golden().items()):
        kw = dict(rec['kwargs'])
        if name.startswith("join"):
            yield name, kw, rec['chunk_len'], rec['overlap']
        else:
            yield name, kw, 300, 60


@pytest.mark.gpu
@pytest.mark.parametrize("ambig_ref,return_all,verbose", [(False, False, False), (True, False, True),
                                                          (False, True, False), (True, True, True)])
def test_device_join_and_decode_equal_host(ambig_ref, return_all, verbose):
    n_cases = 0
    for name, kw, chunk_len, overlap in _golden_cases():
        d = synth.synth_variant_pileup(**kw)
        samples, ranges = _windows(d, chunk_len, overlap)
        if len(ranges) < 2:
            continue
        want, want_sizes = _host_records(d, samples, ambig_ref, return_all, verbose)
        got, sizes = _device_records(d, samples, ranges, 2 * chunk_len, ambig_ref, return_all, verbose)
        assert sizes == want_sizes, name
        assert got == want, name
        n_cases += 1
    assert n_cases >= 5


@pytest.mark.gpu
def test_device_join_and_decode_equal_host_at_scale():
    """The 0.6 M-major pileup of test_gpu_decode_variants_large_matches_oracle, phred-edge rows included, as 10 000 /
    1 000 windows."""
    from medaka_b200 import labels
    from tests.test_stitch import PHRED_EDGE_P, phred_edge_rows
    d = synth.synth_variant_pileup(seed=77, n_major=600000, p_mut=0.01, n_frac=0.001)
    ls = labels.HaploidLabelScheme()
    codes = ls.reference_codes(d['positions'], d['ref_seq'])
    is_major = d['positions']['minor'] == 0
    edge = np.flatnonzero(is_major & (codes >= 1) & (codes <= 4))[:len(PHRED_EDGE_P)]
    d['label_probs'][edge] = phred_edge_rows(codes[edge])
    samples, ranges = _windows(d, 10000, 1000)
    for ambig_ref, return_all, verbose in ((False, False, False), (True, True, True)):
        want, want_sizes = _host_records(d, samples, ambig_ref, return_all, verbose)
        got, sizes = _device_records(d, samples, ranges, 200000, ambig_ref, return_all, verbose, seed=3)
        assert sizes == want_sizes
        assert len(want) > 1000 and got == want


# ------------------------------------------------------------------------------------------- predict_variants


def _draft_from_calls(store, lengths, seed, iupac=True):
    """The two-pass run's own calls on major columns, with ~1 % of positions mutated and some N (and IUPAC) symbols."""
    from medaka_b200 import datastore
    rs = np.random.RandomState(seed)
    draft = {k: np.array(list(rs.choice(list("ACGT"), n))) for k, n in lengths.items()}
    ds = datastore.DataStore(store, 'r')
    try:
        for name in ds.sample_registry:
            s = ds.load_sample(name)
            lab = np.argmax(np.asarray(s.label_probs), -1)
            keep = (s.positions['minor'] == 0) & (lab > 0)
            draft[s.ref_name][s.positions['major'][keep]] = np.array(list("*ACGT"))[lab[keep]]
    finally:
        ds.close()
    for k, seq in draft.items():
        n = len(seq)
        for i in rs.choice(n, max(1, n // 100), replace=False):
            seq[i] = rs.choice([c for c in "ACGT" if c != seq[i]])
        seq[rs.choice(n, max(1, n // 500), replace=False)] = "N"
        at = rs.choice(n, max(1, n // 500), replace=False)
        if iupac:
            seq[at] = rs.choice(list("RYKM"))
        draft[k] = "".join(seq).lower() if k == "gappy" else "".join(seq)     # soft-masked draft: upper()ed
    return draft


def _two_pass(tmp, model, enc, bam, bam_regions, run):
    from medaka_b200 import prediction
    store = os.path.join(tmp, "p%d.npzstore" % len(os.listdir(tmp)))
    prediction.predict_regions(store, bam, bam_regions, model, enc, **run)
    return store


RUN = dict(chunk_len=1000, chunk_ovlp=100, batch_size=4, bam_chunk=3000)


def _check(model, enc, bam, bam_regions, draft_lengths, configs, store_dir, min_records=50, **extra):
    from medaka_b200 import prediction, variant
    store = _two_pass(store_dir, model, enc, bam, bam_regions, RUN)
    drafts = [_draft_from_calls(store, draft_lengths, seed=5, iupac=i) for i in (True, False)]
    for cfg in configs:
        # ambig_ref refuses draft symbols outside '*ACGTN' inside a variant run (labels.py), in both paths alike
        draft = drafts[bool(cfg.get("ambig_ref"))]
        if cfg.get("ambig_ref"):
            with pytest.raises(KeyError) as a:
                variant.variants(store, drafts[0], **cfg)
            with pytest.raises(KeyError) as b:
                prediction.predict_variants(bam, bam_regions, model, enc, drafts[0], **RUN, **cfg, **extra)
            assert str(a.value) == str(b.value)
        want = variant.variants(store, draft, **cfg)
        got = prediction.predict_variants(bam, bam_regions, model, enc, draft, **RUN, **cfg, **extra)
        assert len(want) > min_records, cfg
        assert got == want, cfg
        assert [(v.chrom, v.pos) for v in got] == [(v.chrom, v.pos) for v in want]


CONFIGS = [
    {},
    {"regions": ["long:1500-5200", "tiny", "nodata", "gappy"]},
    {"ambig_ref": True, "verbose": True},
    {"return_all": True},
]


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["tc", "fp32"])
def test_predict_variants_equals_two_pass(precision):
    from medaka_b200 import common, features
    model = _model(synth.synth_state_dict(2), 10, precision)
    enc = features.CountsFeatureEncoder(normalise="total", pileup_source=_pileup_source)
    R = common.Region
    bam_regions = [R("long", 0, 7000), R("gappy", 0, 4200), R("tiny", 0, 600)]
    try:
        with tempfile.TemporaryDirectory() as d:
            _check(model, enc, None, bam_regions, {"long": 7000, "gappy": 4200, "tiny": 600, "nodata": 300},
                   CONFIGS, d)
    finally:
        model.close()


@pytest.mark.gpu
def test_predict_variants_on_a_bam_through_the_fused_featuriser():
    from medaka_b200 import common, features
    from tests import bamutil
    recs = synth.synth_reads(160, 4000, seed=9, mean_len=500)
    recs.sort(key=lambda r: r["pos"])
    for r in recs:
        r["ref"] = 0
    sd = synth.synth_state_dict(6)
    sd["linear.bias"][0] -= 6.0
    model = _model(sd, 10)
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
def test_predict_variants_across_arena_slabs_and_passes(monkeypatch):
    """Slabs of two 4 x 1000 batches and a budget below any contig: joined samples span slabs, every contig is a pass."""
    from medaka_b200 import common, features, prediction
    monkeypatch.setattr(prediction._LabelArena.__init__, "__defaults__", (8192,))
    passes = []
    plan = prediction.plan_passes
    monkeypatch.setattr(prediction, "plan_passes", lambda *a, **k: passes.append(plan(*a, **k)) or passes[-1])
    model = _model(synth.synth_state_dict(2), 10)
    enc = features.CountsFeatureEncoder(normalise="total", pileup_source=_pileup_source)
    R = common.Region
    bam_regions = [R("long", 0, 7000), R("gappy", 0, 4200), R("tiny", 0, 600), R("unasked", 0, 2000)]
    try:
        with tempfile.TemporaryDirectory() as d:
            _check(model, enc, None, bam_regions, {"long": 7000, "gappy": 4200, "tiny": 600, "unasked": 2000},
                   [{"regions": ["tiny", "long", "gappy:100-3000"]}, {"regions": ["long:0-100", "gappy", "long"],
                                                                      "return_all": True}],
                   d, arena_bytes=1)
        assert passes[0] == [["tiny"], ["long"], ["gappy"]] and passes[1] == [["long"], ["gappy"]]
    finally:
        model.close()


@pytest.mark.gpu
def test_predict_variants_refuses_read_level_models_and_several_ranks():
    from medaka_b200 import prediction

    class ReadLevel(object):
        pass

    with pytest.raises(NotImplementedError, match="predict_regions"):
        prediction.predict_variants(None, [], ReadLevel(), None, {})
    model = _model(synth.synth_state_dict(1), 10)
    try:
        with pytest.raises(NotImplementedError):
            prediction.predict_variants(None, [], model, None, {}, world_size=2)
    finally:
        model.close()


# ------------------------------------------------------------------------------------------------ CPU


def test_plan_passes_order_budget_oversized_and_unrequested_contigs():
    from medaka_b200 import prediction
    from medaka_b200.common import Region as R
    per_base = prediction.estimated_columns(1000, 1000, 100) * 9 / 1000.0      # bytes per draft base, roughly
    bam = [R("a", 0, 1000), R("b", 0, 1000), R("b", 1000, 2000), R("c", 0, 10000), R("d", 0, 1000), R("e", 0, 500)]
    budget = int(2600 * per_base)
    # the order the variant regions name the contigs in; "e" is not asked for, "x" has no bam regions
    vreg = [R("d", None, None), R("a", 0, 10), R("x", None, None), R("b", None, None), R("a", 5, 20),
            R("c", None, None)]
    passes = prediction.plan_passes(vreg, bam, budget, 1000, 100)
    assert passes == [["d", "a"], ["b"], ["c"]]
    for p in passes[:-1]:
        need = sum(prediction.estimated_columns(sum(r.size for r in bam if r.ref_name == c), 1000, 100) * 9 for c in p)
        assert need <= budget
    assert prediction.plan_passes(vreg, bam, 1, 1000, 100) == [["d"], ["a"], ["b"], ["c"]]
    assert prediction.plan_passes(vreg, bam, 1 << 40, 1000, 100) == [["d", "a", "b", "c"]]
