"""Where a window runs does not change what the tensor-core recurrences compute for it.

A window's h0 (the layer-0 output, read back from the projection GEMM's operand tiles), its partial logits (what the
layer-1 recurrence writes) and its labels are bit-identical whether it is forwarded alone (a ragged one-window tile), at
slot 4 of a ragged last tile, or inside a full 1056-window group.  The step counts cover T = 1 and odd T (which of the
double-buffered h tiles holds the last step) and T that put the 16-row blocks of a window tile at many offsets inside
the 128-row operand tiles; both tile counts per CTA and both directions (h0 columns 0-127 / 128-255, plog[0] / plog[1])
are covered.  The group's h0 and plog are also checked against the float64 oracle, so the identity is not one of
unwritten outputs.
"""
import numpy as np
import pytest

from oracle import gru_oracle, synth
from tests.test_gru_stages import BARS

GROUP = 1056
# tiles 0, 1, 32, 33 and 65 of the group: at two tiles per CTA both tile slots of a CTA, and the last CTA
WINDOWS = (0, 17, 520, 530, 1055)
FILL = 20           # windows ahead of the target in the ragged call: it is window 4 of a 5-window second tile


def _run(m, x, idx):
    """One forward of all of x; h0, plog [dir][T][class] and labels of windows idx."""
    m.set_group_windows(len(x))
    out = m.forward_arrays(x, want_logits=False, want_labels=True)
    plog = m.read_plog()
    return [{"h0": m.read_activation(0, i, 1)[0], "plog": plog[:, i // 16, :, :, i % 16], "labels": out.labels[i]}
            for i in idx]


@pytest.mark.gpu
@pytest.mark.parametrize("rec", ["one", "pp"])
@pytest.mark.parametrize("T", [1, 2, 3, 8, 9, 129])
def test_window_outputs_do_not_depend_on_placement(T, rec):
    from medaka_b200 import models
    sd = synth.synth_state_dict(41, num_features=10)
    x = synth.synth_features_fast(GROUP, T, 10, seed=41 + T)
    x[list(WINDOWS)] = gru_oracle.featuriser_like_features(len(WINDOWS), T, 10, seed=41 + T)
    m = models.GRUModel(num_features=10)
    m.load_state_dict(sd)
    m.set_precision("tc")
    m.set_rec_mode(rec)
    try:
        group = _run(m, x, WINDOWS)
        for k, w in enumerate(WINDOWS):
            alone = _run(m, x[[w]], [0])[0]
            ragged = _run(m, np.concatenate([x[1030:1030 + FILL], x[[w]]]), [FILL])[0]
            for name in ("h0", "plog", "labels"):
                assert np.array_equal(alone[name], group[k][name]), (w, name, "alone")
                assert np.array_equal(ragged[name], group[k][name]), (w, name, "ragged")
    finally:
        m.close()
    want = gru_oracle.stages(sd, x[list(WINDOWS)])
    got = {"h0": np.stack([g["h0"] for g in group]),
           "plog": np.stack([g["plog"].transpose(1, 0, 2) for g in group])}    # -> [window][T][dir][class]
    for name, v in got.items():
        err = float(np.abs(v.astype(np.float64) - want[name]).max() / np.abs(want[name]).max())
        assert err <= BARS[name], (name, err)
