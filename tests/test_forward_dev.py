"""Device-resident forwards (mdk_engine_forward_dev) are packed into groups like submitted batches: results must equal
the same windows run one call at a time through the host path, bit for bit, and the timing API must cope with fewer
launched groups than calls."""
import numpy as np
import pytest

from oracle import synth

pytestmark = pytest.mark.gpu

SMALL_POS = 1 << 18        # calls up to this many positions take the engine's small lanes


class DevBuf(object):
    """Raw device memory of the engine's device (mdk_dev_alloc)."""

    def __init__(self, nbytes):
        from medaka_b200 import libmedaka as lm
        self.lm = lm
        pp = lm.ffi.new("void **")
        lm.check(lm.lib.mdk_dev_alloc(0, nbytes, pp))
        self.ptr, self.nbytes = pp[0], nbytes

    def upload(self, a):
        a = np.ascontiguousarray(a)
        assert a.nbytes == self.nbytes
        self.lm.check(self.lm.lib.mdk_memcpy_h2d(0, self.ptr, self.lm.ffi.from_buffer(a), a.nbytes))
        return self

    def download(self, shape, dtype):
        out = np.empty(shape, dtype=dtype)
        assert out.nbytes == self.nbytes
        self.lm.check(self.lm.lib.mdk_memcpy_d2h(0, self.lm.ffi.from_buffer(out), self.ptr, out.nbytes))
        return out

    def cast(self, ctype):
        return self.lm.ffi.cast(ctype, self.ptr)

    def free(self):
        self.lm.check(self.lm.lib.mdk_dev_free(0, self.ptr))


class DevCall(object):
    """One forward_dev call: its features and its own output buffers in HBM."""

    def __init__(self, feats, want_logits, want_labels=True):
        B, T, _ = feats.shape
        self.feats = feats
        self.d_feats = DevBuf(feats.nbytes).upload(feats)
        self.d_probs = DevBuf(B * T * 5 * 4).upload(np.full((B, T, 5), -1.0, dtype=np.float32))
        self.d_logits = DevBuf(B * T * 5 * 4).upload(np.full((B, T, 5), -1.0, dtype=np.float32)) if want_logits else None
        self.d_labels = DevBuf(B * T).upload(np.full((B, T), 255, dtype=np.uint8)) if want_labels else None

    def run(self, eng):
        from medaka_b200 import libmedaka as lm
        B, T, _ = self.feats.shape
        lm.check(lm.lib.mdk_engine_forward_dev(
            eng, self.d_feats.cast("const float *"), B, T, self.d_probs.cast("float *"),
            self.d_logits.cast("float *") if self.d_logits else lm.ffi.NULL,
            self.d_labels.cast("uint8_t *") if self.d_labels else lm.ffi.NULL))

    def results(self):
        B, T, _ = self.feats.shape
        probs = self.d_probs.download((B, T, 5), np.float32)
        logits = self.d_logits.download((B, T, 5), np.float32) if self.d_logits else None
        labels = self.d_labels.download((B, T), np.uint8) if self.d_labels else None
        return probs, logits, labels

    def free(self):
        for b in (self.d_feats, self.d_probs, self.d_logits, self.d_labels):
            if b is not None:
                b.free()


def _model(seed):
    from medaka_b200 import models
    m = models.GRUModel(num_features=10)
    m.load_state_dict(synth.synth_state_dict(seed))
    return m


def _timings(m, n):
    from medaka_b200 import libmedaka as lm
    t = lm.ffi.new("mdk_timings *")
    lm.check(lm.lib.mdk_engine_mean_timings(m.engine, n, t))
    return {k: float(getattr(t, k)) for k in ("inproj0_ms", "rec0_ms", "inproj1_ms", "rec1_ms", "head_ms", "total_ms")}


@pytest.mark.parametrize("group_windows", [48, 0])
def test_forward_dev_packed_matches_host_forwards(group_windows):
    """A ragged sequence of device calls: calls that straddle group boundaries, a call larger than a group (48), a T
    change mid-sequence, logits for some calls only, calls on both sides of the small-lane threshold.  Every call's
    outputs must equal its windows run alone through the host path, bit for bit (windows never interact, and groups of
    up to one wave run the same one-tile kernel with the fused head as the single calls)."""
    from medaka_b200 import libmedaka as lm
    m = _model(6)
    gw = group_windows or m.preferred_batch_size()
    # (windows, columns, want_logits)
    plan = [(150, 2000, False), (30, 2000, True), (40, 2000, False), (1, 2000, True), (400, 2000, True),
            (500, 2000, False), (20, 2000, True),
            (200, 1500, True), (25, 1500, False), (60, 1500, True), (5, 1500, False)]
    assert any(b * t <= SMALL_POS for b, t, _ in plan) and any(b * t > SMALL_POS for b, t, _ in plan)
    assert sum(b for b, t, _ in plan if t == 2000) > gw           # some call straddles a group boundary
    feats = [synth.synth_features_fast(b, t, 10, seed=40 + i) for i, (b, t, _) in enumerate(plan)]
    want = [m.forward_arrays(x, want_logits=True) for x in feats]
    m.reserve(gw, 2000)
    m.set_group_windows(group_windows)
    calls = [DevCall(x, lg) for x, (_, _, lg) in zip(feats, plan)]
    for c in calls:
        c.run(m.engine)
    lm.check(lm.lib.mdk_engine_sync(m.engine))
    for i, (c, w) in enumerate(zip(calls, want)):
        probs, logits, labels = c.results()
        assert np.array_equal(probs, w.probs), "call %d: probabilities differ" % i
        assert np.array_equal(labels, w.labels), "call %d: labels differ" % i
        if logits is not None:
            assert np.array_equal(logits, w.logits), "call %d: logits differ" % i
        c.free()
    m.close()


def test_forward_dev_larger_than_group_runs_whole():
    """A call of more windows than a group holds is one forward (one set of kernel launches), not several groups."""
    from medaka_b200 import libmedaka as lm
    m = _model(7)
    x = synth.synth_features_fast(100, 1000, 10, seed=3)
    want = m.forward_arrays(x, want_logits=True)                     # also prepares the weights
    per_forward = m.last_timings()["launches"]
    m.set_group_windows(48)
    c = DevCall(x, True)
    n0 = m.launch_count()
    c.run(m.engine)
    lm.check(lm.lib.mdk_engine_sync(m.engine))
    assert m.launch_count() - n0 == per_forward
    probs, logits, labels = c.results()
    assert np.array_equal(probs, want.probs) and np.array_equal(logits, want.logits) and np.array_equal(labels, want.labels)
    c.free()
    m.close()


def test_mean_timings_with_fewer_groups_than_requested():
    """Two calls of 30 windows under 48-window groups: one full group launches, 12 windows stay open.  mean_timings(32)
    launches the open group and averages the two groups that exist."""
    from medaka_b200 import libmedaka as lm
    m = _model(8)
    t = lm.ffi.new("mdk_timings *")
    assert lm.lib.mdk_engine_mean_timings(m.engine, 4, t) == lm.lib.MDK_ERR_STATE     # nothing recorded yet
    xs = [synth.synth_features_fast(30, 1000, 10, seed=10 + i) for i in range(2)]
    want = [m.forward_arrays(x) for x in xs]                       # prepares the weights; two groups recorded
    per_forward = m.last_timings()["launches"]
    m.reserve(48, 1000)
    m.set_group_windows(48)
    calls = [DevCall(x, False) for x in xs]
    n0 = m.launch_count()
    for c in calls:
        c.run(m.engine)
    assert m.launch_count() - n0 == per_forward                      # the full group only
    mean_all = _timings(m, 32)                                       # launches the open group first
    assert m.launch_count() - n0 == 2 * per_forward
    assert m.last_timings()["launches"] == per_forward
    mean_two, last = _timings(m, 2), _timings(m, 1)
    for k, v in mean_two.items():
        assert np.isfinite(v) and v >= 0.0
    assert mean_two["rec0_ms"] > 0.0 and last["rec0_ms"] > 0.0 and mean_two["total_ms"] > 0.0
    assert mean_all == _timings(m, 4)            # four groups in all (two host forwards, two packed groups)
    lm.check(lm.lib.mdk_engine_sync(m.engine))
    for c, w in zip(calls, want):
        probs, _, labels = c.results()
        assert np.array_equal(probs, w.probs) and np.array_equal(labels, w.labels)
        c.free()
    m.close()
