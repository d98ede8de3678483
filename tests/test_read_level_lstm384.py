"""Read-level network at lstm_size = 384, the width of every released read-level model (``..._rl_lstm384_...``).

Goldens = outputs of the reference's own LatentSpaceLSTM(lstm_size=384) on seeded parameters
(tests/golden/make_rl384_golden.py; the other constructor arguments are the class defaults).  Bar as in
test_read_level.py: probabilities within 2e-5 absolute of the reference, labels identical wherever the reference's top-2
margin exceeds 1e-4.  Every device test runs on both paths: wgmma (cluster recurrence + projection GEMM) and the fp32
CUDA-core twins."""
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import rl_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "rl_forward_lstm384.npz")
H = 384
TOL = 2e-5
CASES = ["small", "deep", "dwells", "hot", "long"]


def _oracle(sd, use_dwells=False):
    m = rl_oracle.LatentSpaceLSTM(lstm_size=H, use_dwells=use_dwells)
    m.load_state_dict(sd)
    m.eval()
    return m


def _case(g, name):
    seed, B, P, D, dw, gain = g[name + "_args"]
    sd = rl_oracle.synth_rl_state_dict(int(seed), lstm_size=H, use_dwells=bool(dw), gain=float(gain))
    x = rl_oracle.synth_rl_features(int(B), int(P), int(D), use_dwells=bool(dw), seed=100 + int(seed))
    return sd, x, bool(dw), g[name + "_probs"]


def _check(got, want):
    assert got.shape == want.shape and np.isfinite(got).all()
    assert np.abs(got - want).max() < TOL, np.abs(got - want).max()
    top2 = np.sort(want, -1)[..., -2:]
    decided = (top2[..., 1] - top2[..., 0]) > 1e-4
    assert np.array_equal(np.argmax(got, -1)[decided], np.argmax(want, -1)[decided])


def _model(sd, path, use_dwells=False):
    from medaka_b200 import read_level
    m = read_level.LatentSpaceLSTM(lstm_size=H, use_dwells=use_dwells)
    m.load_state_dict(sd)
    m.set_conv(path == "tc")
    return m


# ---------------------------------------------------------------------------------------------- CPU

@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference_class_lstm384(name):
    g = np.load(GOLD)
    sd, x, dw, want = _case(g, name)
    got = rl_oracle.predict(_oracle(sd, dw), x)
    assert np.abs(got - want).max() < 2e-6


def test_golden_cases_cover_a_long_window():
    g = np.load(GOLD)
    assert max(int(g[n + "_args"][2]) for n in CASES) >= 2000
    assert int(g["deep_args"][3]) == 40 and bool(g["dwells_args"][4]) and float(g["hot_args"][5]) == 2.5


def test_model_archive_roundtrip_lstm384(tmp_path):
    """A read-level archive with lstm_size = 384 written and reloaded through ModelStoreTGZ yields those kwargs (what
    load_model hands to model_from_dict)."""
    from medaka_b200 import datastore
    sd = rl_oracle.synth_rl_state_dict(4, lstm_size=H)
    kwargs = {"num_classes": 5, "lstm_size": H, "cnn_size": 128, "kernel_sizes": [1, 17], "pooler_type": "mean",
              "use_dwells": False, "bidirectional": True}
    meta = {"model_function": {"type": "LatentSpaceLSTM", "kwargs": kwargs},
            "feature_encoder": {"type": "ReadAlignmentFeatureEncoder", "kwargs": {"include_dwells": False}},
            "label_scheme": "HaploidLabelScheme"}
    path = str(tmp_path / "rl_lstm384_model_pt.tar.gz")
    datastore.ModelStoreTGZ.write(path, sd, meta)
    with datastore.ModelStoreTGZ(path) as ms:
        assert ms.model_kwargs() == {"type": "LatentSpaceLSTM", "kwargs": kwargs}
        w = ms._unpack()._weights
        assert tuple(w["lstm.weight_hh_l1_reverse"].shape) == (4 * H, H)
        assert tuple(w["linear.weight"].shape) == (5, 2 * H)


def _kernel_sass(sass, name):
    """The SASS text of one kernel (cuobjdump -sass prints a 'Function : <mangled name>' header per kernel)."""
    blocks = sass.split("Function : ")
    hits = [b for b in blocks if b.split("\n", 1)[0].strip().startswith("_ZN3mdk%d%s" % (len(name), name))]
    assert len(hits) == 1, name
    return hits[0]


@pytest.mark.parametrize("kernel", ["rl_lstm384_tc_kernel", "rl_proj_tc_kernel"])
def test_sass_lstm384_kernels_are_wgmma_without_spills(kernel):
    sys.path.insert(0, ROOT)
    import __graft_entry__
    lib = __graft_entry__.build()
    sass = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True).stdout
    body = _kernel_sass(sass, kernel)
    assert "HGMMA" in body
    assert "STL" not in body and "LDL" not in body          # no local-memory traffic: nothing spilled


# ---------------------------------------------------------------------------------------------- GPU

@pytest.mark.gpu
@pytest.mark.parametrize("path", ["tc", "fp32"])
@pytest.mark.parametrize("name", CASES)
def test_device_matches_reference_class_lstm384(name, path):
    g = np.load(GOLD)
    sd, x, dw, want = _case(g, name)
    m = _model(sd, path, use_dwells=dw)
    _check(m.forward_arrays(x), want)
    m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["tc", "fp32"])
@pytest.mark.parametrize("B,P,D,max_cells", [(1, 1, 1, None), (2, 17, 1, None), (19, 65, 5, 2000), (33, 40, 3, None),
                                             (5, 301, 9, 3000)])
def test_device_matches_oracle_ragged_shapes_lstm384(B, P, D, max_cells, path):
    """P = 1 and 17, single reads, windows off the 16-window tile, windows split over several device calls."""
    sd = rl_oracle.synth_rl_state_dict(15, lstm_size=H)
    x = rl_oracle.synth_rl_features(B, P, D, seed=B * 1000 + P, empty_rows=min(2, D - 1))
    want = rl_oracle.predict(_oracle(sd), x)
    m = _model(sd, path)
    if max_cells:
        m.max_cells = max_cells
    _check(m.forward_arrays(x), want)
    m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["tc", "fp32"])
def test_device_more_clusters_than_fit_lstm384(path):
    """640 windows = 40 tiles x 2 directions = 80 clusters of 8 CTAs: more than an H100 runs at once (one CTA per SM),
    so clusters run in several waves."""
    sd = rl_oracle.synth_rl_state_dict(16, lstm_size=H)
    x = rl_oracle.synth_rl_features(640, 24, 2, seed=640, empty_rows=1)
    want = rl_oracle.predict(_oracle(sd), x)
    m = _model(sd, path)
    m.max_bytes = 1 << 40                    # one device call
    _check(m.forward_arrays(x), want)
    m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["tc", "fp32"])
def test_predict_on_batch_lstm384(path):
    sd = rl_oracle.synth_rl_state_dict(17, lstm_size=H)
    feats = rl_oracle.synth_rl_features(3, 80, 6, seed=3)
    m = _model(sd, path)

    class Batch(object):
        read_level_features = feats
    out = m.predict_on_batch(Batch)
    assert tuple(out.shape) == (3, 80, 5)
    _check(out.numpy(), rl_oracle.predict(_oracle(sd), feats))
    m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["tc", "fp32"])
def test_read_level_prediction_end_to_end_lstm384(tmp_path, path):
    """BAM file -> native reader -> mdk_read_matrix -> windows -> Batch.collate -> the 384 engine -> store, against the
    oracles driven over the same reads."""
    from medaka_b200 import common, datastore, features, prediction
    from oracle import read_matrix_oracle, synth
    from tests import bamutil
    rs = np.random.RandomState(3)
    recs = synth.synth_reads(90, 2600, seed=21, mean_len=700)
    recs.sort(key=lambda r: r["pos"])
    for i, r in enumerate(recs):
        r["query_name"], r["ref"], r["tags"] = "q%d" % i, 0, {}
        r["qual"] = rs.randint(1, 50, len(r["seq"])).tolist()
    bam = str(tmp_path / "reads.bam")
    bamutil.write_bam(bam, [("ctg", 2600)], recs)
    sd = rl_oracle.synth_rl_state_dict(9, lstm_size=H)
    model = _model(sd, path)
    enc = features.ReadAlignmentFeatureEncoder(include_dwells=False)
    out = str(tmp_path / "probs.npzstore")
    prediction.predict_regions(out, bam, [common.Region("ctg", 0, 2600)], model, enc, chunk_len=500, chunk_ovlp=100,
                               batch_size=3, bam_chunk=100000)
    mat, pos, _, _ = read_matrix_oracle.read_alignment(recs, 0, 2600)
    oracle_model = _oracle(sd)
    n = 0
    with datastore.DataStore(out, "r") as ds:
        for name in sorted(ds.sample_registry):
            s = ds.load_sample(name)
            a = int(np.flatnonzero((pos["major"] == s.positions["major"][0]) & (pos["minor"] == s.positions["minor"][0]))[0])
            b = a + len(s.positions)
            assert np.array_equal(pos[a:b], s.positions)
            want = rl_oracle.predict(oracle_model, mat[a:b][None].astype(np.int8))[0]
            assert np.abs(s.label_probs - want).max() < TOL
            n += 1
    assert n >= 5
    model.close()


@pytest.mark.gpu
def test_stage_times_lstm384():
    sd = rl_oracle.synth_rl_state_dict(18, lstm_size=H)
    m = _model(sd, "tc")
    m.set_timing(True)
    m.forward_arrays(rl_oracle.synth_rl_features(17, 300, 8, seed=5))
    ms = m.stage_ms()
    assert list(ms) == list(m.STAGES) and all(v > 0 for v in ms.values())
    m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("lstm_size,cnn_size", [(256, 128), (128, 384), (384, 384)])
def test_unsupported_sizes_raise(lstm_size, cnn_size):
    from medaka_b200 import libmedaka, read_level
    with pytest.raises(libmedaka.MedakaB200Error, match="lstm_size 128 or 384 with cnn_size 128"):
        read_level.LatentSpaceLSTM(lstm_size=lstm_size, cnn_size=cnn_size)
