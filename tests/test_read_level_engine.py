"""Packed asynchronous read-level calls (mdk_rl_submit / wait / flush / reserve, LatentSpaceLSTM.predict_async).

Each submitted call's convolution runs on its own windows; the LSTM and the head run once per group of windows.  Every
window is its own grid slice of the convolution kernels, its own column of the projections and its own MMA column of the
recurrences, so packing must not change a single bit: the probabilities of a packed window equal those of the same
window run alone through mdk_rl_forward at the same read depth.
"""
import numpy as np
import pytest

from oracle import rl_oracle
from tests.test_read_level_production import _check

# (windows, reads) of the submitted calls at P = 300: 161 windows, so a 112-window group (one wave at lstm_size 384
# on an H100) is split inside the sixth call, a 64-window group inside the fifth
CALLS = [(1, 9), (7, 33), (16, 100), (25, 50), (40, 71), (40, 100), (25, 12), (7, 9)]
P0, P1 = 300, 257
TAIL = [(5, 20), (3, 40)]          # calls with another P: the first seals the open group, the second stays open


def _model(H, seed, use_dwells=True):
    from medaka_b200 import read_level
    sd = rl_oracle.synth_rl_state_dict(seed, lstm_size=H, use_dwells=use_dwells)
    m = read_level.LatentSpaceLSTM(lstm_size=H, use_dwells=use_dwells)
    m.load_state_dict(sd)
    return sd, m


class _Calls(object):
    """Host buffers of a stream of submitted calls (outputs pre-filled with NaN / 255: untouched until written)."""

    def __init__(self, shapes, seed):
        self.x = [rl_oracle.featuriser_like_rl_features(B, P, D, F=5, seed=seed + i) for i, (B, P, D) in enumerate(shapes)]
        self.probs = [np.full((B, P, 5), np.nan, dtype=np.float32) for B, P, _ in shapes]
        self.labels = [np.full((B, P), 255, dtype=np.uint8) for B, P, _ in shapes]
        self.tickets = []

    def submit(self, m, i):
        from medaka_b200 import libmedaka as lm
        ffi = lm.ffi
        x = self.x[i]
        B, P, D, F = x.shape
        t = ffi.new("int64_t *")
        lm.check(lm.lib.mdk_rl_submit(m._engine, ffi.cast("const int8_t *", ffi.from_buffer(x)), B, P, D, F,
                                      ffi.cast("float *", ffi.from_buffer(self.probs[i])),
                                      ffi.cast("uint8_t *", ffi.from_buffer(self.labels[i])), t))
        self.tickets.append(int(t[0]))
        return int(t[0])


def _wait(m, ticket):
    from medaka_b200 import libmedaka as lm
    lm.check(lm.lib.mdk_rl_wait(m._engine, ticket))


def _alone(m, x):
    """Each window of x through mdk_rl_forward by itself."""
    return np.concatenate([m.forward_arrays(x[b:b + 1]) for b in range(len(x))])


@pytest.mark.gpu
@pytest.mark.parametrize("H", [128, 384])
def test_packing_is_invisible(H):
    """Mixed B and D at one P, packed into groups of `gw` windows (at 384 one recurrence wave, mdk_rl_preferred_windows,
    112 on an H100; at 128 the wave is 1056 windows, so the group buffers are reserved for 64): bit-identical to every
    window alone, labels the argmax of the probabilities.  Covers a call split across two groups, a P change sealing a
    group, a wait on an open group launching it, and tickets completing in order."""
    from medaka_b200 import libmedaka as lm
    sd, m = _model(H, 51 + H)
    pref = m.preferred_batch_size()
    gw = pref if H == 384 else 64
    if H == 384:
        assert pref % 16 == 0 and 100 < pref <= 128, pref
    m.reserve(gw, P0)
    shapes = [(B, P0, D) for B, D in CALLS] + [(B, P1, D) for B, D in TAIL]
    calls = _Calls(shapes, seed=7 * H)
    total = sum(B for B, _ in CALLS)
    assert total > gw
    # the call whose windows cross the first group boundary
    ends = np.cumsum([B for B, _ in CALLS])
    split = int(np.flatnonzero(ends > gw)[0])
    assert ends[split] - CALLS[split][0] < gw < ends[split]
    for i in range(len(CALLS)):
        calls.submit(m, i)
    # the first group filled up inside call `split` and was launched: the calls before it complete without any wait
    # once a later ticket has been waited for
    calls.submit(m, len(CALLS))                          # another P: seals the open (second) group
    _wait(m, calls.tickets[split])                       # the split call completes with the second group
    for i in range(split + 1):
        assert not np.isnan(calls.probs[i]).any(), i      # tickets complete in order
        assert (calls.labels[i] != 255).all(), i
    # the last call stays in an open group until its ticket is waited for
    t_last = calls.submit(m, len(CALLS) + 1)
    assert np.isnan(calls.probs[-1]).all()
    _wait(m, t_last)                                     # launches the open group
    for t in calls.tickets:
        _wait(m, t)
    for i, x in enumerate(calls.x):
        want = _alone(m, x)
        assert np.array_equal(calls.probs[i], want, equal_nan=True), (i, float(np.nanmax(np.abs(calls.probs[i] - want))))
        assert np.array_equal(calls.labels[i], np.argmax(calls.probs[i], -1)), i
    with pytest.raises(lm.MedakaB200Error):
        _wait(m, calls.tickets[-1] + 10 ** 6)            # never issued
    m.close()


@pytest.mark.gpu
def test_predict_async_handles_and_flush():
    """predict_async on uint8 batches (what Batch.collate makes): result() is the probability tensor, .labels the
    argmax; flush launches the open group without waiting; predict_on_batch sets last_labels."""
    import torch
    sd, m = _model(128, 61, use_dwells=False)
    xs = [rl_oracle.featuriser_like_rl_features(B, 120, D, F=5, seed=B) for B, D in ((3, 14), (9, 40), (2, 5))]

    class Batch(object):
        def __init__(self, x):
            self.read_level_features = torch.from_numpy(x.astype(np.uint8))
    handles = [m.predict_async(Batch(x), slots=4) for x in xs]
    m.flush()
    for x, h in zip(xs, handles):
        p = h.result().numpy()
        assert np.array_equal(p, _alone(m, x))
        assert np.array_equal(h.labels, np.argmax(p, -1))
    out = m.predict_on_batch(Batch(xs[1])).numpy()
    assert np.array_equal(out, _alone(m, xs[1]))
    assert np.array_equal(m.last_labels, np.argmax(out, -1))
    m.close()


@pytest.mark.gpu
def test_released_shape_one_wave_lstm384():
    """One full wave at lstm_size 384 (preferred_batch_size: 16 windows per cluster that fits the device at once, both
    directions; 112 windows on an H100, whose 132 SMs hold 14 clusters of 8 CTAs) of 10 000 positions x 100
    featuriser-like reads with dwells, submitted as 100 + the rest.  Windows 0, 15, 16 and the last (both ends of the
    first tile, the next tile, the last window) are bit-identical to the same window alone through mdk_rl_forward, whose
    z / h0 / h1 / probabilities are within the per-stage bars of the oracle with its decided labels; every label is the
    argmax of its probabilities."""
    H, P, D = 384, 10000, 100
    sd, m = _model(H, 31)
    gw = m.preferred_batch_size()
    assert gw % 16 == 0 and 100 < gw <= 128, gw
    picks = (0, 15, 16, gw - 1)
    x = rl_oracle.featuriser_like_rl_features(gw, P, D, F=5, seed=71)
    m.reserve(gw, P)
    calls = _Calls([], 0)
    calls.x = [x[:100], x[100:]]
    calls.probs = [np.full((n, P, 5), np.nan, dtype=np.float32) for n in (100, gw - 100)]
    calls.labels = [np.full((n, P), 255, dtype=np.uint8) for n in (100, gw - 100)]
    calls.submit(m, 0)
    calls.submit(m, 1)                                   # fills the group: launched without a wait
    for t in calls.tickets:
        _wait(m, t)
    probs, labels = np.concatenate(calls.probs), np.concatenate(calls.labels)
    assert np.array_equal(labels, np.argmax(probs, -1))
    want = rl_oracle.stages(rl_oracle.build(sd, use_dwells=True), x[list(picks)])
    for i, b in enumerate(picks):
        alone = m.forward_arrays(x[b:b + 1])
        assert np.array_equal(probs[b:b + 1], alone), b
        got = {k: m.read_stage(k) for k in ("z", "h0", "h1")}
        got["probs"] = alone
        _check(got, {k: v[i:i + 1] for k, v in want.items()}, "engine wave H=384 window %d" % b)
    m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("H", [128, 384])
def test_reserve_is_capped_at_the_group_limit(H):
    """reserve(50 x preferred, 10 000) allocates no more than one group at the group limit (24 GiB budget; unclamped it
    would need terabytes), and a submit of 4 x preferred windows of a shorter P afterwards runs in full groups and
    matches the windows run alone."""
    import torch
    sd, m = _model(H, 81, use_dwells=False)
    pref = m.preferred_batch_size()
    torch.cuda.init()
    free0, _ = torch.cuda.mem_get_info()
    m.reserve(50 * pref, 10000)
    free1, _ = torch.cuda.mem_get_info()
    per_window = 10000 * (52 * H + 21)
    assert free0 - free1 <= pref * per_window + (256 << 20), (free0 - free1, pref * per_window)
    assert free0 - free1 <= (24 << 30) + (256 << 20)
    x = rl_oracle.featuriser_like_rl_features(4 * pref, 40, 3, F=5, seed=H)
    calls = _Calls([], 0)
    calls.x = [x]
    calls.probs = [np.full((len(x), 40, 5), np.nan, dtype=np.float32)]
    calls.labels = [np.full((len(x), 40), 255, dtype=np.uint8)]
    _wait(m, calls.submit(m, 0))
    for b in (0, pref - 1, pref, 4 * pref - 1):
        assert np.array_equal(calls.probs[0][b:b + 1], m.forward_arrays(x[b:b + 1])), b
    assert np.array_equal(calls.labels[0], np.argmax(calls.probs[0], -1))
    m.close()


@pytest.mark.gpu
def test_stages_are_not_read_after_a_submit():
    """read_stage / mdk_rl_debug_read return the stages of the last mdk_rl_forward only while nothing has overwritten
    them: a submit that opens a group writes z, so the stages are refused instead of mixing two calls."""
    from medaka_b200 import libmedaka as lm
    sd, m = _model(128, 82, use_dwells=False)
    x = rl_oracle.featuriser_like_rl_features(3, 50, 6, F=5, seed=82)
    m.forward_arrays(x)
    assert m.read_stage("z").shape == (3, 50, 128)
    calls = _Calls([(2, 50, 6)], 83)
    calls.submit(m, 0)                                   # opens a group: its convolution writes z
    out = np.empty((3, 50, 128), dtype=np.float32)
    rc = lm.lib.mdk_rl_debug_read(m._engine, 0, lm.ffi.cast("float *", lm.ffi.from_buffer(out)), out.size)
    assert rc == lm.lib.MDK_ERR_STATE
    _wait(m, calls.tickets[0])
    m.forward_arrays(x[:1])
    assert m.read_stage("h1").shape == (1, 50, 256)     # a new forward is readable again
    m.reserve(64, 50)                                    # regrows the group buffers
    with pytest.raises(lm.MedakaB200Error):
        m.read_stage("z")
    m.close()


class _Synchronous(object):
    """The model without its asynchronous interface: run_prediction takes the predict_on_batch path."""

    def __init__(self, model):
        self._m = model

    def predict_on_batch(self, batch):
        import torch
        return torch.from_numpy(self._m.forward_arrays(self._m.get_model_input_features(batch)))

    def __getattr__(self, name):
        if name in ("predict_async", "lookahead", "reserve", "flush", "preferred_batch_size", "last_labels"):
            raise AttributeError(name)
        return getattr(self._m, name)


@pytest.mark.gpu
@pytest.mark.parametrize("H", [128, 384])
def test_pipeline_auto_batch_matches_synchronous(tmp_path, H):
    """predict_regions with batch_size="auto" (predict_async, look-ahead) stores the same label_probs as the synchronous
    predict_on_batch path, and the argmax labels beside them."""
    from medaka_b200 import common, datastore, features, prediction
    from oracle import synth
    from tests import bamutil
    rs = np.random.RandomState(5)
    recs = synth.synth_reads(120, 4100, seed=23, mean_len=700)
    recs.sort(key=lambda r: r["pos"])
    for i, r in enumerate(recs):
        r["query_name"], r["ref"], r["tags"] = "q%d" % i, 0, {}
        r["qual"] = rs.randint(1, 50, len(r["seq"])).tolist()
    bam = str(tmp_path / "reads.bam")
    bamutil.write_bam(bam, [("ctg", 4100)], recs)
    sd, m = _model(H, 9, use_dwells=False)
    enc = features.ReadAlignmentFeatureEncoder(include_dwells=False)
    region = [common.Region("ctg", 0, 4100)]
    out_async, out_sync = str(tmp_path / "async.npzstore"), str(tmp_path / "sync.npzstore")
    prediction.predict_regions(out_async, bam, region, m, enc, chunk_len=500, chunk_ovlp=100, batch_size="auto",
                               bam_chunk=100000)
    prediction.predict_regions(out_sync, bam, region, _Synchronous(m), enc, chunk_len=500, chunk_ovlp=100,
                               batch_size="auto", bam_chunk=100000)
    m.close()
    with datastore.DataStore(out_async, "r") as da, datastore.DataStore(out_sync, "r") as ds:
        names = sorted(da.sample_registry)
        assert names == sorted(ds.sample_registry) and len(names) >= 5
        for name in names:
            a, s = da.load_sample(name), ds.load_sample(name)
            assert np.array_equal(a.positions, s.positions)
            assert np.array_equal(a.label_probs, s.label_probs), name
            assert a.labels is not None and np.array_equal(a.labels, np.argmax(a.label_probs, -1)), name
