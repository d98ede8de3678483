"""One-pass consensus and variant calling with read-level models: the read-level engine's decoded outputs
(mdk_rl_submit_decoded / mdk_rl_submit_variant_decoded), and predict_consensus / predict_variants with LatentSpaceLSTM
against predict_regions + stitch.sequence / variant.variants."""
import os
import tempfile

import numpy as np
import pytest

from oracle import rl_oracle, synth
from tests.test_one_pass import _both, _decode, _draft
from tests.test_one_pass_variants import CONFIGS, _check, _random_ref, _vd_of_probs

# (lstm_size, tensor cores for the convolution and the LSTM, dwells)
MATRIX = [(H, tc, dw) for H in (128, 384) for tc in (True, False) for dw in (True, False)]
MATRIX_IDS = ["H%d-%s-%s" % (H, "tc" if tc else "fp32", "dwells" if dw else "nodwells") for H, tc, dw in MATRIX]


def _model(H, tc, use_dwells, seed=3, bias0=0.0):
    from medaka_b200 import read_level
    sd = rl_oracle.synth_rl_state_dict(seed, lstm_size=H, use_dwells=use_dwells)
    sd["linear.bias"][0] += bias0
    m = read_level.LatentSpaceLSTM(lstm_size=H, use_dwells=use_dwells)
    m.load_state_dict(sd)
    m.set_conv(tc)
    return m


def _ptr(x, ctype):
    from medaka_b200 import libmedaka as lm
    return lm.ffi.cast(ctype, lm.ffi.from_buffer(x))


def _submit_probs(m, x):
    """Probabilities and labels of x through mdk_rl_submit + wait."""
    from medaka_b200 import libmedaka as lm
    B, P, D, F = x.shape
    probs, labels = np.empty((B, P, 5), np.float32), np.empty((B, P), np.uint8)
    t = lm.ffi.new("int64_t *")
    lm.check(lm.lib.mdk_rl_submit(m._engine, _ptr(x, "const int8_t *"), B, P, D, F, _ptr(probs, "float *"),
                                  _ptr(labels, "uint8_t *"), t))
    m.wait(int(t[0]))
    return probs, labels


def _pinned(m, key, a):
    x = m.pinned(key, a.shape, a.dtype)
    np.copyto(x, a)
    return x


# ------------------------------------------------------------------------------------------------ decoded heads


@pytest.mark.gpu
@pytest.mark.parametrize("H,tc,dwells", MATRIX, ids=MATRIX_IDS)
def test_decoded_heads_equal_decode_of_probabilities(H, tc, dwells):
    """Labels and quality bytes, call bytes and both phreds of the read-level heads (rl_head768_kernel at 384,
    head_kernel at 128) are bit-equal to the decode of the probabilities mdk_rl_submit returns for the same features:
    ragged reads, empty rows, random reference bytes with codes 5 and 6 and insertion columns."""
    B, P, D = 7, 230, 9
    x = rl_oracle.synth_rl_features(B, P, D, use_dwells=dwells, seed=H + 2 * tc + dwells, empty_rows=3, ragged=True)
    ref = _random_ref(B, P, seed=B * P + H)
    m = _model(H, tc, dwells)
    try:
        probs, labels = _submit_probs(m, x)
        want_labels, want_quals = _decode(probs)
        assert np.array_equal(labels, want_labels)
        xin = _pinned(m, "feats", x)
        got_labels, got_quals = np.empty((B, P), np.uint8), np.empty((B, P), np.uint8)
        m.wait(m.submit_decoded(xin, got_labels, got_quals))
        assert np.array_equal(got_labels, want_labels)
        assert np.array_equal(got_quals, want_quals)
        labels_only = np.empty((B, P), np.uint8)
        m.wait(m.submit_decoded(xin, labels_only))
        assert np.array_equal(labels_only, want_labels)
        calls, pq, rq = np.empty((B, P), np.uint8), np.empty((B, P), np.float32), np.empty((B, P), np.float32)
        m.wait(m.submit_variant_decoded(xin, _pinned(m, "ref", ref), calls, pq, rq))
        for g, w in zip((calls, pq, rq), _vd_of_probs(probs, ref)):
            assert np.array_equal(g, w)
    finally:
        m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("H,tc,dwells", MATRIX, ids=MATRIX_IDS)
def test_ordinary_decoded_and_variant_decoded_calls_share_groups(H, tc, dwells):
    """Calls of different B and D packed into 16-window groups: ordinary to host, variant-decoded to host, decoded to
    device (split across the two groups), decoded to host, variant-decoded with reference bytes and outputs in device
    memory.  Each group holds three kinds of call.  Each call's outputs equal those of the same call run alone."""
    from medaka_b200 import libmedaka as lm
    lib, ffi = lm.load(), lm.ffi
    P = 150
    shapes = [(5, 11), (3, 8), (9, 14), (4, 6), (6, 5)]
    xs = [rl_oracle.featuriser_like_rl_features(B, P, D, F=5 if dwells else 4, seed=40 + i)
          for i, (B, D) in enumerate(shapes)]
    refs = [_random_ref(B, P, seed=60 + i) for i, (B, _) in enumerate(shapes)]
    m = _model(H, tc, dwells, seed=5)
    try:
        alone = [m.forward_arrays(x) for x in xs]
        m.reserve(16, P)
        pins = [_pinned(m, "mix%d" % i, x) for i, x in enumerate(xs)]
        n2, n4 = 9 * P, 6 * P
        # device: labels + quals of call 2, then ref bytes, calls, pred_q, ref_q of call 4
        pp = ffi.new("void **")
        lm.check(lib.mdk_dev_alloc(0, 2 * n2 + 10 * n4, pp))
        dev = int(ffi.cast("uintptr_t", pp[0]))
        d4 = dev + 2 * n2
        try:
            lm.check(lib.mdk_memcpy_h2d(0, ffi.cast("void *", d4), _ptr(refs[4], "void *"), n4))
            probs0, labels0 = np.empty((5, P, 5), np.float32), np.empty((5, P), np.uint8)
            t = ffi.new("int64_t *")
            lm.check(lib.mdk_rl_submit(m._engine, _ptr(pins[0], "const int8_t *"), 5, P, 11, pins[0].shape[3],
                                       _ptr(probs0, "float *"), _ptr(labels0, "uint8_t *"), t))
            tickets = [int(t[0])]
            v1 = (np.empty((3, P), np.uint8), np.empty((3, P), np.float32), np.empty((3, P), np.float32))
            tickets.append(m.submit_variant_decoded(pins[1], _pinned(m, "ref1", refs[1]), *v1))
            tickets.append(m.submit_decoded(pins[2], dev, dev + n2))          # 8 windows in group 1, 1 in group 2
            lab3, q3 = np.empty((4, P), np.uint8), np.empty((4, P), np.uint8)
            tickets.append(m.submit_decoded(pins[3], lab3, q3))
            tickets.append(m.submit_variant_decoded(pins[4], d4, d4 + n4, d4 + 2 * n4, d4 + 6 * n4))
            for t in tickets:
                m.wait(t)
            m.sync()
            back = np.empty(2 * n2 + 10 * n4, np.uint8)
            lm.check(lib.mdk_memcpy_d2h(0, _ptr(back, "void *"), pp[0], len(back)))
        finally:
            lib.mdk_dev_free(0, pp[0])
        assert np.array_equal(probs0, alone[0])
        assert np.array_equal(labels0, _decode(alone[0])[0])
        for got, want in zip(v1, _vd_of_probs(alone[1], refs[1])):
            assert np.array_equal(got, want)
        for got, want in zip((back[:n2].reshape(9, P), back[n2:2 * n2].reshape(9, P)), _decode(alone[2])):
            assert np.array_equal(got, want)
        for got, want in zip((lab3, q3), _decode(alone[3])):
            assert np.array_equal(got, want)
        tail = back[2 * n2:]
        assert np.array_equal(tail[:n4].reshape(6, P), refs[4])                 # the input is left as it was
        got4 = (tail[n4:2 * n4].reshape(6, P), tail[2 * n4:6 * n4].view(np.float32).reshape(6, P),
                tail[6 * n4:].view(np.float32).reshape(6, P))
        for got, want in zip(got4, _vd_of_probs(alone[4], refs[4])):
            assert np.array_equal(got, want)
    finally:
        m.close()


# -------------------------------------------------------------------------------- predict_consensus / variants

_SOURCE_CACHE = {}


def _rl_pileup_source(region, bam, encoder):
    """Seeded read-level features per region: insertion columns after ~12 % of the majors, a read depth that differs
    from region to region (so batches differ in D), and a coverage gap on "gappy" (two chunks)."""
    F = encoder.feature_vector_length
    key = (region.ref_name, region.start, region.end, F)
    if key not in _SOURCE_CACHE:
        seed = sum(map(ord, region.ref_name)) * 131 + region.start
        rs = np.random.RandomState(seed)
        n_ins = np.where(rs.rand(region.end - region.start) < 0.12, rs.randint(1, 3, region.end - region.start), 0)
        width = 1 + n_ins
        major = np.repeat(np.arange(region.start, region.end, dtype=np.int64), width)
        minor = np.arange(len(major), dtype=np.int64) - np.repeat(np.cumsum(width) - width, width)
        pos = np.empty(len(major), dtype=[('major', '<i8'), ('minor', '<i8')])
        pos['major'], pos['minor'] = major, minor
        x = rl_oracle.featuriser_like_rl_features(1, len(pos), 6 + seed % 11, F=F, seed=seed % (1 << 31))[0]
        chunks = [(x, pos)]
        hole = np.flatnonzero((major >= 2000) & (major < 2600)) if region.ref_name == "gappy" else []
        if len(hole):
            lo, hi = hole[0], hole[-1] + 1
            chunks = [c for c in ((x[:lo], pos[:lo]), (x[hi:], pos[hi:])) if len(c[1])]
        _SOURCE_CACHE[key] = chunks
    return _SOURCE_CACHE[key]


def _encoder(dwells):
    from medaka_b200 import features
    return features.ReadAlignmentFeatureEncoder(include_dwells=dwells, pileup_source=_rl_pileup_source)


@pytest.mark.gpu
@pytest.mark.parametrize("H,tc,dwells", MATRIX, ids=MATRIX_IDS)
def test_predict_consensus_equals_two_pass(H, tc, dwells):
    from medaka_b200 import common
    model = _model(H, tc, dwells, seed=2, bias0=-6.0)
    R = common.Region
    lengths = {"long": 7000, "gappy": 4200, "tiny": 600, "nodata": 300}
    draft = _draft(lengths)
    bam_regions = [R("long", 0, 7000), R("gappy", 0, 4200), R("tiny", 0, 600)]
    configs = [
        {},
        {"min_depth": 9},
        {"regions": ["long:1500-5200", R("tiny", None, None), "nodata"]},
        {"fillgaps": False},
        {"fill_char": "N", "qualities": False},
    ]
    try:
        with tempfile.TemporaryDirectory() as d:
            for cfg in configs:
                (a, bed_a), (b, bed_b) = _both(d, model, _encoder(dwells), None, bam_regions, draft, **cfg)
                assert len(a) > 1000, cfg
                assert a == b, cfg
                assert bed_a == bed_b, cfg
    finally:
        model.close()


@pytest.mark.gpu
@pytest.mark.parametrize("H,tc,dwells", MATRIX, ids=MATRIX_IDS)
def test_predict_variants_equals_two_pass(H, tc, dwells):
    from medaka_b200 import common
    model = _model(H, tc, dwells, seed=2, bias0=-6.0)
    R = common.Region
    bam_regions = [R("long", 0, 7000), R("gappy", 0, 4200), R("tiny", 0, 600)]
    try:
        with tempfile.TemporaryDirectory() as d:
            _check(model, _encoder(dwells), None, bam_regions, {"long": 7000, "gappy": 4200, "tiny": 600, "nodata": 300},
                   CONFIGS, d)
    finally:
        model.close()


def _bam_with_moves(path, ref_len=4000, seed=9):
    from tests import bamutil
    rs = np.random.RandomState(seed)
    recs = synth.synth_reads(120, ref_len, seed=seed, mean_len=500)
    recs.sort(key=lambda r: r["pos"])
    for i, r in enumerate(recs):
        r["query_name"], r["ref"] = "q%d" % i, 0
        r["qual"] = rs.randint(1, 50, len(r["seq"])).tolist()
        mv = [5] + (rs.uniform(size=3 * len(r["seq"])) < 0.34).astype(int).tolist()
        mv[1] = 1
        r["tags"] = {"mv": mv}
    bamutil.write_bam(path, [("ctg", ref_len)], recs)


@pytest.mark.gpu
@pytest.mark.parametrize("H", [128, 384])
def test_one_pass_on_a_bam_through_the_read_level_featuriser(H):
    """Reads with move tables through the read-level featuriser with dwells: both entry points equal the two-pass
    path."""
    from medaka_b200 import common, features
    model = _model(H, True, True, seed=6, bias0=-6.0)
    try:
        with tempfile.TemporaryDirectory() as d:
            path = os.path.join(d, "r.bam")
            _bam_with_moves(path)
            enc = features.ReadAlignmentFeatureEncoder(include_dwells=True)
            regions = [common.Region("ctg", 0, 4000)]
            (a, bed_a), (b, bed_b) = _both(d, model, enc, path, regions, _draft({"ctg": 4000}, seed=3))
            assert len(a) > 1000 and a == b and bed_a == bed_b
            _check(model, enc, path, regions, {"ctg": 4000}, [{}, {"return_all": True}], d, min_records=20)
    finally:
        model.close()


@pytest.mark.gpu
@pytest.mark.parametrize("H", [128, 384])
def test_one_pass_across_many_arena_slabs_and_passes(H, monkeypatch):
    """Slabs of two 4 x 1000 batches: stitch regions and joined samples span several slabs; a budget below any contig
    runs every contig as a pass of its own."""
    from medaka_b200 import common, prediction
    monkeypatch.setattr(prediction._LabelArena.__init__, "__defaults__", (8192,))
    passes = []
    plan = prediction.plan_passes
    monkeypatch.setattr(prediction, "plan_passes", lambda *a, **k: passes.append(plan(*a, **k)) or passes[-1])
    model = _model(H, True, H == 384, seed=2, bias0=-6.0)
    enc = _encoder(H == 384)
    R = common.Region
    bam_regions = [R("long", 0, 7000), R("gappy", 0, 4200), R("tiny", 0, 600)]
    try:
        with tempfile.TemporaryDirectory() as d:
            for cfg in ({}, {"min_depth": 9}):
                (a, bed_a), (b, bed_b) = _both(d, model, enc, None, bam_regions,
                                               _draft({"long": 7000, "gappy": 4200, "tiny": 600}), **cfg)
                assert len(a) > 1000 and a == b and bed_a == bed_b, cfg
            _check(model, enc, None, bam_regions, {"long": 7000, "gappy": 4200, "tiny": 600},
                   [{"regions": ["tiny", "long", "gappy:100-3000"]}], d, arena_bytes=1)
        assert passes[0] == [["tiny"], ["long"], ["gappy"]]
    finally:
        model.close()


# ------------------------------------------------------------------------------------------------------- CPU


class _FakeReadLevelModel(object):
    """The read-level model interface _run_decoded uses, recording what it is given."""

    def __init__(self):
        self.buffers, self.calls, self.waited, self.reserved = {}, [], set(), []
        self.key_ticket = {}           # pinned key -> ticket of the call that last used it

    def get_model_input_features(self, batch):
        return batch.read_level_features

    def preferred_batch_size(self):
        return 3

    def lookahead(self, batch_size, window_len=None):
        return 2

    def reserve(self, windows, window_len):
        self.reserved.append((windows, window_len))

    def pinned(self, key, shape, dtype):
        t = self.key_ticket.get(key)
        assert t is None or t in self.waited, "slot %s reused before its call %d was waited for" % (key, t)
        self._key = key
        self.buffers[key] = np.zeros(shape, dtype)
        return self.buffers[key]

    def submit(self, x, data, slot, slab, row):
        ticket = len(self.calls)
        self.key_ticket[self._key] = ticket
        self.calls.append(dict(x=x.copy(), dtype=x.dtype, names=[s.name for s in data], slot=slot, slab=slab, row=row,
                               depth=max(s.features.shape[1] for s in data), feats=[s.features for s in data]))
        return ticket

    def wait(self, ticket):
        self.waited.add(ticket)


class _FakeArena(object):
    def __init__(self, half):
        self.half, self.slab, self.used = half, -1, half

    def take(self, n):
        if self.used + n > self.half:
            self.slab, self.used = self.slab + 1, 0
        at = self.used
        self.used += n
        return self.slab, at


def test_run_decoded_stages_read_level_batches_as_int8_of_their_depth():
    from medaka_b200 import common, prediction
    model = _FakeReadLevelModel()
    arena = _FakeArena(2500)
    samples = {}
    R = common.Region
    regions = [R("long", 0, 7000), R("gappy", 0, 4200), R("other", 0, 3000)]
    rem = prediction._run_decoded(samples, arena, None, regions, model, _encoder(True), 500, 50, lambda s: s,
                                  model.submit, batch_size=3, bam_workers=1)
    assert rem == []
    assert len(model.calls) >= 10 and model.waited == set(range(len(model.calls)))
    assert len({c["depth"] for c in model.calls}) >= 3                  # the batches differ in D
    for k, c in enumerate(model.calls):
        nb = len(c["names"])
        assert c["dtype"] == np.int8 and c["x"].shape == (nb, 500, c["depth"], 5)
        for i, f in enumerate(c["feats"]):                                # padded with empty reads to the batch's D
            assert np.array_equal(c["x"][i, :, :f.shape[1]], f.astype(np.int8))
            assert not c["x"][i, :, f.shape[1]:].any()
        assert c["slot"] == k % 3
    # the window -> (slab, row) map: the rows arena.take handed out, window after window
    n = 0
    for c in model.calls:
        for i, name in enumerate(c["names"]):
            view, slab, row = samples[name]
            assert (slab, row) == (c["slab"], c["row"] + i * 500) and view.name == name
            n += 1
    assert n == len(samples)
    assert max(c["slab"] for c in model.calls) >= 2


def test_device_index_of_both_model_kinds():
    import torch
    from medaka_b200 import prediction

    class Model(object):
        def __init__(self, dev):
            self.dev = dev

        def device(self):
            return self.dev
    assert prediction._device_index(Model("cuda:3")) == 3                     # LatentSpaceLSTM.device()
    assert prediction._device_index(Model(torch.device("cuda", 2))) == 2      # GRUModel.device()
