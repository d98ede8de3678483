"""A group's layer-1 recurrence and head run on a stream of their own, beside the next group's layer 0, and AUTO runs two
window tiles per CTA for every forward with the fused layer-0 projection.  Every result must still equal its windows run
alone, bit for bit, and the timed region must cover every group's layer 1."""
import numpy as np
import pytest

from oracle import synth
from tests.test_forward_dev import DevCall

pytestmark = pytest.mark.gpu


def _model(seed, F=10):
    from medaka_b200 import models
    m = models.GRUModel(num_features=F)
    m.load_state_dict(synth.synth_state_dict(seed, num_features=F))
    return m


def _same(a, b):
    return np.array_equal(a.probs, b.probs) and np.array_equal(a.logits, b.logits) and np.array_equal(a.labels, b.labels)


def test_auto_equals_two_tiles_per_cta():
    """Under AUTO at F = 10 a window's outputs are those of the two-tile kernel, alone, in ragged groups and in a full
    1056-window group."""
    m = _model(11)
    x = synth.synth_features_fast(1056, 40, 10, seed=5)
    outs = {}
    for B in (1, 40, 48, 1056):
        m.set_rec_mode("auto")
        a = m.forward_arrays(x[:B], want_logits=True)
        m.set_rec_mode("pp")
        b = m.forward_arrays(x[:B], want_logits=True)
        assert _same(a, b), "B = %d: AUTO differs from two tiles per CTA" % B
        outs[B] = a
    for B in (40, 48, 1056):
        assert np.array_equal(outs[B].probs[:1], outs[1].probs) and np.array_equal(outs[B].labels[:1], outs[1].labels)
    m.close()


def _pipelined(m, plan, seed0, decoded=()):
    """Run plan [(B, T)] as forward_dev calls (the indices in `decoded` as submit_decoded) under 48-window groups after a
    reservation for short windows, without waiting in between, and check each call against its lone run."""
    from medaka_b200 import libmedaka as lm
    F = m.num_features
    feats = [synth.synth_features_fast(b, t, F, seed=seed0 + i) for i, (b, t) in enumerate(plan)]
    want = [m.forward_arrays(x, want_logits=True) for x in feats]
    m.reserve(48, 1000)                      # the later, longer windows regrow the workspace while groups are queued
    m.set_group_windows(48)
    calls = []
    for i, x in enumerate(feats):
        if i in decoded:
            xp = m.pinned("dx%d" % i, x.shape, np.float32)
            np.copyto(xp, x)
            lab = np.full(x.shape[:2], 255, dtype=np.uint8)
            m.submit_decoded(xp, lab)
            calls.append(lab)
        else:
            c = DevCall(x, want_logits=True)
            c.run(m.engine)
            calls.append(c)
    lm.check(lm.lib.mdk_engine_sync(m.engine))
    for i, (c, w) in enumerate(zip(calls, want)):
        if i in decoded:
            assert np.array_equal(c, w.labels), "call %d: decoded labels differ" % i
            continue
        probs, logits, labels = c.results()
        assert np.array_equal(probs, w.probs), "call %d: probabilities differ" % i
        assert np.array_equal(logits, w.logits), "call %d: logits differ" % i
        assert np.array_equal(labels, w.labels), "call %d: labels differ" % i
        c.free()


def test_pipelined_groups_match_lone_runs():
    """Ten and more 48-window groups queued back to back on the big lanes: a T change between groups, a workspace
    regrowth while earlier groups' layer 1 may still run, decoded calls and a small-lane call in between."""
    m = _model(12)
    plan = [(100, 3000), (90, 3000), (1, 500), (120, 2700), (70, 3000), (90, 3200), (60, 3200)]
    _pipelined(m, plan, 60, decoded=(1, 4))
    m.close()


def test_pipelined_groups_unfused_layer0():
    """F = 20: layer 0 reads gi, so its input projection waits for the previous group's layer 1."""
    m = _model(13, F=20)
    plan = [(100, 3000), (60, 2800), (90, 3000)]
    _pipelined(m, plan, 80)
    m.close()


def test_activations_of_the_last_pipelined_forward():
    """keep_activations(1): after several queued groups, h0 and h1 of the last forward equal those of a lone run."""
    from medaka_b200 import libmedaka as lm
    m = _model(14)
    lm.check(lm.lib.mdk_engine_keep_activations(m.engine, 1))
    xs = [synth.synth_features_fast(96, 3000, 10, seed=90), synth.synth_features_fast(48, 5500, 10, seed=91)]
    m.forward_arrays(xs[1])
    want = (m.read_activation(0), m.read_activation(1))
    m.reserve(48, 3000)
    m.set_group_windows(48)
    calls = [DevCall(x, want_logits=False) for x in xs]
    for c in calls:
        c.run(m.engine)                     # three groups; the 5500-column call is the last, a group of its own
    lm.check(lm.lib.mdk_engine_sync(m.engine))
    assert np.array_equal(m.read_activation(0), want[0])
    assert np.array_equal(m.read_activation(1), want[1])
    for c in calls:
        c.free()
    m.close()


def test_timer_covers_every_layer1():
    """timer_stop's end event follows the last group's layer 1 and head, which run on the layer-1 stream."""
    from medaka_b200 import libmedaka as lm
    m = _model(15)
    xs = [synth.synth_features_fast(48, 6000, 10, seed=7 + i) for i in range(3)]
    m.forward_arrays(xs[0][:1])
    m.reserve(48, 6000)
    m.set_group_windows(48)
    calls = [DevCall(x, want_logits=False) for x in xs]
    ms = lm.ffi.new("float *")
    lm.check(lm.lib.mdk_engine_timer_start(m.engine))
    for c in calls:
        c.run(m.engine)                     # three full 48-window groups on the big lanes
    lm.check(lm.lib.mdk_engine_timer_stop(m.engine, ms))
    tl = lm.ffi.new("float[24]")
    lm.check(lm.lib.mdk_debug_timeline(m.engine, 3, tl))
    latest = max(tl[i] for i in range(24))
    assert latest > 0.0 and float(ms[0]) >= latest - 1e-3, (float(ms[0]), latest)
    for c in calls:
        c.free()
    m.close()
