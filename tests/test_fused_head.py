"""The linear head fused into the layer-1 recurrence (fp32 on the CUDA cores, partial logits per direction) in the
two-tile kernel (NT = 2, N = 32 windows per CTA): against the unfused head (h1 through HBM, separate head kernel), and
independent of a window's slot in the tile."""
import numpy as np
import pytest

from oracle import synth

pytestmark = pytest.mark.gpu

NEAR_TIE = 1e-5


def _make_model(sd, rec_mode="auto"):
    from medaka_b200 import models
    m = models.GRUModel(num_features=10)
    m.load_state_dict(sd)
    m.set_precision("tc")
    m.set_rec_mode(rec_mode)
    return m


def _scaled_err(got, ref):
    scale = np.abs(ref).max(axis=-1, keepdims=True)
    return float((np.abs(got - ref) / scale).max())


def _decided_mismatches(labels, probs):
    top2 = np.sort(probs, -1)[..., -2:]
    decided = (top2[..., 1] - top2[..., 0]) > NEAR_TIE
    return int(((labels != np.argmax(probs, -1)) & decided).sum())


def test_two_tile_fused_and_unfused_head_agree():
    """B = 1217 (77 tiles, the last one ragged: 1 window of 16), the two-tile kernel selected explicitly; the unfused
    side runs the layer-1 recurrence without the head and the separate head kernel."""
    sd = synth.synth_state_dict(5)
    feats = synth.synth_features(1217, 257, 10, seed=78)
    m = _make_model(sd, "pp")
    fused = m.forward_arrays(feats, want_logits=True, want_labels=True)
    m.keep_activations(True)
    plain = m.forward_arrays(feats, want_logits=True, want_labels=True)
    err = _scaled_err(fused.logits, plain.logits)
    print("two-tile fused vs unfused head: scaled logit diff %.3e" % err)
    assert err < 1e-5
    assert _decided_mismatches(fused.labels, plain.probs) == 0
    m.close()


def test_two_tile_fused_head_slot_independent():
    """A window's logits do not depend on its slot (tile, column) in the two-tile kernel: bit-identical."""
    sd = synth.synth_state_dict(6)
    feats = synth.synth_features(40, 300, 10, seed=5)
    m = _make_model(sd, "pp")
    out = m.forward_arrays(feats, want_logits=True)
    pick = [37, 2, 16, 31, 0, 20, 9]
    sub = m.forward_arrays(feats[pick], want_logits=True)
    assert np.array_equal(sub.logits, out.logits[pick])
    m.close()
