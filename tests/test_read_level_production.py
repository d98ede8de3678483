"""Read-level network at the shapes and on the inputs the released models run: windows of 10 000 positions x 100 reads
(medaka.py's chunk_len / max_reads defaults), featuriser-like reads (several per row, dwells saturated at 127, absent
qualities, empty rows), both lstm_size 128 and 384 (every released model), both device paths (tc: wgmma with fp16 hi / lo
operand pairs; fp32: the CUDA-core twins).

Parity is checked per stage against oracle/rl_oracle.py (fp32 torch, window by window):
  z  the pooled pre_pool_expansion_layer output (the LSTM input), h0 / h1 the two LSTM layers' outputs: max|d| / max|ref|
  probs: max|d| absolute, and labels identical wherever the reference's top-2 margin exceeds 1e-4.
The probabilities alone cannot tell a three-product kernel (hi.hi + hi.lo + lo.hi, DESIGN §3) from one that lost a
product: near 1/3 the softmax shrinks the error.  The intermediates show it 3-10x more clearly, so the bars are set per
stage, and test_ablations_exceed_the_bars checks (on the CPU) that every lost product or fp16 rounding of rl_oracle.ablate
lands above 3x the bar at one stage or more.
"""
import numpy as np
import pytest

from oracle import rl_oracle

# One set of bars for every path, calibrated on an H100 80GB HBM3 (SXM, 400 W power limit) over every GPU case of this
# file (DESIGN §2 "Read-level stage bars" has the table).  Worst device error, z / h0 / h1 (relative) / probs (absolute):
#   fp32 path  9.7e-7 / 1.4e-6 / 1.2e-6 / 9.2e-7
#   tc path    1.6e-6 / 4.8e-6 / 2.9e-6 / 2.4e-6
# Smallest ablation effects (rl_oracle.ablate, P = 1 000-3 000, D = 40-100): z 4.3e-5 (y1), h0 6.1e-5 (h),
# h1 3.8e-5 (y1), probs 9.9e-6 (w_hh at 384).
# Each bar is at most a third of that stage's smallest ablation effect, so a kernel that lost a product fails it, and at
# least 3x the worst error of both paths at z, h0 and h1.  At probs the window is narrower than the tc path's error
# allows: the bar (3.2e-6) is 3.5x the fp32 path's worst error but only 1.3x the tc path's; z, h0 and h1 carry the
# discrimination there.
BARS = {"z": 1.4e-5, "h0": 2e-5, "h1": 1.2e-5, "probs": 3.2e-6}
STAGES = ("z", "h0", "h1", "probs")
MARGIN = 1e-4
PROD_P, PROD_D, PROD_B = 10000, 100, 18
PROD_WINDOWS = (0, 15, 16, 17)          # a full 16-window tile's first and last window, the partial tile


def _errors(got, want):
    """{stage: error} with the scaling of BARS (relative to max|ref| for z, h0, h1; absolute for probs)."""
    out = {}
    for k in got:
        d = float(np.abs(got[k].astype(np.float64) - want[k]).max())
        out[k] = d if k == "probs" else d / float(np.abs(want[k]).max())
    return out


def _check(got, want, label=""):
    """got / want: dicts of stages (any subset of STAGES) with [B, P, ...] arrays.  One set of bars for every path."""
    bars = BARS
    err = _errors(got, want)
    print("rl-parity %s %s" % (label, " ".join("%s=%.3g" % (k, err[k]) for k in STAGES if k in err)))
    for k, e in err.items():
        assert np.isfinite(got[k]).all(), k
        assert e <= bars[k], (k, e, bars[k])
    if "probs" in got:
        top2 = np.sort(want["probs"], -1)[..., -2:]
        decided = (top2[..., 1] - top2[..., 0]) > MARGIN
        assert np.array_equal(np.argmax(got["probs"], -1)[decided], np.argmax(want["probs"], -1)[decided])


def _block_report(got, want, label, block=1000):
    """Max error per block of positions along the recurrence (printed: the log shows whether it grows with P)."""
    for k in ("h1", "probs"):
        if k not in got:
            continue
        d = np.abs(got[k].astype(np.float64) - want[k]).max(axis=tuple(i for i in range(got[k].ndim) if i != 1))
        blocks = [float(d[i:i + block].max()) for i in range(0, len(d), block)]
        print("rl-blocks %s %s per %d positions: %s" % (label, k, block, " ".join("%.2g" % b for b in blocks)))


def _sd(H, seed, use_dwells=False):
    return rl_oracle.synth_rl_state_dict(seed, lstm_size=H, use_dwells=use_dwells)


def _model(sd, H, path, use_dwells=False):
    from medaka_b200 import read_level
    m = read_level.LatentSpaceLSTM(lstm_size=H, use_dwells=use_dwells)
    m.load_state_dict(sd)
    if isinstance(path, tuple):
        m.set_conv(*path)
    else:
        m.set_conv(path == "tc")
    return m


# ---------------------------------------------------------------------------------------------- shared cases
# "dwells": a use_dwells=True model on F = 5 features;  "f5": a non-dwell model on the default encoder's F = 5 (the dwell
# column is there and counts for the read mask, but the model does not read it)
MODELS = {"dwells": (True, 5), "f5": (False, 5)}


@pytest.fixture(scope="module")
def production():
    """production(H, model): B = 18 windows of P = 10 000 x D = 100 featuriser-like reads and the oracle's stages of
    windows PROD_WINDOWS, computed once per (H, model) and shared by both paths; freed when the module ends."""
    cache = {}

    def get(H, model):
        if (H, model) not in cache:
            dw, F = MODELS[model]
            sd = _sd(H, 31, dw)
            x = rl_oracle.featuriser_like_rl_features(PROD_B, PROD_P, PROD_D, F=F, seed=H + F + 7 * dw)
            cache[H, model] = sd, x, rl_oracle.stages(rl_oracle.build(sd, use_dwells=dw), x[list(PROD_WINDOWS)])
        return cache[H, model]
    yield get
    cache.clear()


def _small(H, seed=41):
    """One device call: 18 windows (a full tile and a partial one) of 300 positions x 97 reads, dwell model."""
    sd = _sd(H, seed, True)
    x = rl_oracle.featuriser_like_rl_features(18, 300, 97, F=5, seed=seed)
    return sd, x, rl_oracle.stages(rl_oracle.build(sd, use_dwells=True), x)


# ---------------------------------------------------------------------------------------------- CPU
def test_featuriser_like_features_have_the_properties_of_real_windows():
    D = 100
    x = rl_oracle.featuriser_like_rl_features(3, 2000, D, F=6, seed=3)
    assert x.shape == (3, 2000, D, 6) and x.dtype == np.int8 and x.min() >= 0
    base, qual, strand, mapq, dwell, hap = (x[..., i] for i in range(6))
    present = base > 0
    assert set(np.unique(base[present])) == {1, 2, 3, 4, 5}
    assert (qual[base == 5] == 0).all() and (qual[(base > 0) & (base < 5)] == 0).any() and qual.max() == 93
    assert set(np.unique(strand[present])) == {0, 1} and mapq[present].min() == 0 and mapq.max() == 60
    assert (dwell[base == 5] == 0).all() and dwell.max() == 127
    assert (dwell[(base > 0) & (base < 5)] == 127).mean() >= 0.05
    assert set(np.unique(hap[present])) == {0, 1, 2}
    n_starts = n_heads = n_tails = n_tile_cross = 0
    for b in range(3):
        rows = present[b].any(0)
        empty = np.flatnonzero(~rows)
        assert len(empty) and empty.min() < D - 1                      # empty rows in the middle, not only at the end
        assert any((~rows[4 * g:4 * g + 4]).all() for g in range(D // 4))   # 4 empty rows = one 4-read conv group
        for d in np.flatnonzero(rows):
            occ = np.concatenate([[0], present[b, :, d].astype(np.int8), [0]])
            starts, ends = np.flatnonzero(np.diff(occ) == 1), np.flatnonzero(np.diff(occ) == -1)
            assert ((starts[1:] - ends[:-1]) >= 5).all()                # reads of a row separated by >= 5 positions
            n_starts += len(starts)
            n_heads += int(starts[0] < 8)
            n_tails += int(2000 - 8 <= ends[-1] < 2000)
            n_tile_cross += int(((starts // 128) != ((ends - 1) // 128)).sum())
    assert n_starts > 2 * 3 * (D - 8) and n_heads > 0 and n_tails > 0 and n_tile_cross > 0


def test_stages_match_predict():
    """stages() restates forward: the probabilities of each window equal predict() on that window."""
    for H in (128, 384):
        sd = _sd(H, 8, True)
        x = rl_oracle.featuriser_like_rl_features(2, 150, 13, F=5, seed=8)
        m = rl_oracle.build(sd, use_dwells=True)
        got = rl_oracle.stages(m, x)
        want = np.concatenate([rl_oracle.predict(m, x[b:b + 1]) for b in range(2)])
        assert got["z"].shape == (2, 150, H) and got["h1"].shape == (2, 150, 2 * H)
        assert np.abs(got["probs"] - want).max() <= 1e-7


@pytest.mark.parametrize("H", [128, 384])
def test_ablations_exceed_the_bars(H):
    """Every precision ablation (a kernel that lost one of its three fp16 products, or rounds an operand to fp16) moves
    some stage by more than 3x its bar on a reduced production case, so the bars can tell the products apart."""
    sd = _sd(H, 31, True)
    x = rl_oracle.featuriser_like_rl_features(1, 2000, 40, F=5, seed=H)
    ref = rl_oracle.stages(rl_oracle.build(sd, use_dwells=True), x)
    for which in rl_oracle.ABLATIONS:
        sd_a, kw = rl_oracle.ablate(sd, which)
        err = _errors(rl_oracle.stages(rl_oracle.build(sd_a, use_dwells=True), x, **kw), ref)
        ratio = {k: err[k] / BARS[k] for k in STAGES}
        print("rl-ablation H=%d %-6s %s" % (H, which, " ".join("%s=%.3g (%.1fx)" % (k, err[k], ratio[k]) for k in STAGES)))
        assert max(ratio.values()) > 3, (which, err)


def test_windows_per_call_is_capped():
    """mdk_rl_forward takes at most 65 535 windows; forward_arrays splits bigger batches of short windows."""
    from medaka_b200 import read_level
    m = object.__new__(read_level.LatentSpaceLSTM)          # no engine: pure arithmetic
    m.lstm_size, m._fp32_conv, m.max_cells, m.max_bytes = 128, False, 1 << 26, 8 << 30
    assert m.windows_per_call(1, 1, 4) == 65535
    assert m.windows_per_call(2, 1, 4) == 65535
    assert m.windows_per_call(10000, 100, 5) == min((1 << 26) // (10000 * 100),
                                                     (8 << 30) // m.scratch_bytes_per_window(10000, 100, 5))
    m.max_bytes = 1
    assert m.windows_per_call(10000, 100, 5) == 1


# ---------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("model", sorted(MODELS))
@pytest.mark.parametrize("path", ["tc", "fp32"])
@pytest.mark.parametrize("H", [128, 384])
def test_production_windows(production, H, path, model):
    """18 windows of 10 000 positions x 100 reads through forward_arrays with its default limits: a full 16-window tile
    plus a partial one, 78 convolution tiles of 128 positions plus a 16-position tail."""
    dw, _ = MODELS[model]
    sd, x, want = production(H, model)
    m = _model(sd, H, path, use_dwells=dw)
    probs = m.forward_arrays(x)
    m.close()
    got = {"probs": probs[list(PROD_WINDOWS)]}
    label = "production H=%d %s %s" % (H, path, model)
    _block_report(got, want, label)
    _check(got, {"probs": want["probs"]}, label)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["small", "production"])
@pytest.mark.parametrize("path", ["tc", "fp32"])
@pytest.mark.parametrize("H", [128, 384])
def test_stages_match_oracle(production, H, path, case):
    """z, h0, h1 and the probabilities of one device call, read back with read_stage."""
    if case == "small":
        sd, x, want = _small(H)
    else:                                                   # window 0 of the production case, alone
        sd, xs, ws = production(H, "dwells")
        x, want = xs[:1], {k: v[:1] for k, v in ws.items()}
    m = _model(sd, H, path, use_dwells=True)
    probs = m.forward_arrays(x)
    got = {k: m.read_stage(k) for k in ("z", "h0", "h1")}
    got["probs"] = probs
    m.close()
    label = "stages H=%d %s %s" % (H, path, case)
    _block_report(got, want, label)
    _check(got, want, label)


@pytest.mark.gpu
@pytest.mark.parametrize("path", [(True, False), (False, True)], ids=["conv_tc-lstm_fp32", "conv_fp32-lstm_tc"])
@pytest.mark.parametrize("H", [128, 384])
def test_mixed_paths(H, path):
    """The convolution on one path and the LSTM on the other, on a ragged case: 19 windows, 301 positions, 9 reads."""
    sd = _sd(H, 43, True)
    x = rl_oracle.featuriser_like_rl_features(19, 301, 9, F=5, seed=43)
    want = rl_oracle.stages(rl_oracle.build(sd, use_dwells=True), x)
    m = _model(sd, H, path, use_dwells=True)
    probs = m.forward_arrays(x)
    got = {k: m.read_stage(k) for k in ("z", "h0", "h1")}
    got["probs"] = probs
    m.close()
    _check(got, want, "mixed H=%d %s" % (H, path))


@pytest.mark.gpu
@pytest.mark.parametrize("F", [5, 6])
@pytest.mark.parametrize("path", ["tc", "fp32"])
@pytest.mark.parametrize("H", [128, 384])
def test_read_mask_covers_every_column(H, path, F):
    """A non-dwell model on the default encoder's F = 5 (F = 6 with the haplotype tag): rows whose only non-zero entries
    are in columns 4-5 count as reads (the reference's mask is x.sum((1, -1)) != 0 over every column)."""
    sd = _sd(H, 44)
    x = rl_oracle.featuriser_like_rl_features(3, 400, 12, F=F, seed=44 + F)
    x[:, :, 2:4, :4] = 0                           # rows 2, 3: nothing but dwells / haplotype tags
    x[1, :, 5:9] = 0
    x[1, 50:90, 6, F - 1] = 3                      # window 1, row 6: one non-zero column
    want = rl_oracle.stages(rl_oracle.build(sd), x)
    m = _model(sd, H, path)
    probs = m.forward_arrays(x)
    got = {k: m.read_stage(k) for k in ("z", "h0", "h1")}
    got["probs"] = probs
    m.close()
    _check(got, want, "mask H=%d %s F=%d" % (H, path, F))


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["tc", "fp32"])
@pytest.mark.parametrize("H", [128, 384])
def test_window_without_reads(H, path):
    """Window 5 of 18 has no reads: the reference divides 0 by 0 in MeanPooler, so the whole window is NaN.  The device
    gives NaN at the same places, and the other 17 windows (window 5's tile-mates included) are bit-identical to a run
    without window 5."""
    sd = _sd(H, 45, True)
    x = rl_oracle.featuriser_like_rl_features(18, 200, 13, F=5, seed=45)
    x[5] = 0
    want = rl_oracle.predict(rl_oracle.build(sd, use_dwells=True), x[5:6])
    assert np.isnan(want).all()
    m = _model(sd, H, path, use_dwells=True)
    got = m.forward_arrays(x)
    rest = m.forward_arrays(np.delete(x, 5, axis=0))
    m.close()
    assert np.isnan(got[5]).all()
    others = np.delete(got, 5, axis=0)
    assert not np.isnan(others).any()
    assert np.array_equal(others, rest)


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["tc", "fp32"])
def test_more_lstm_tiles_than_sms_lstm128(path):
    """2 200 windows in one call: 138 tiles x 2 directions of the H = 128 recurrence, more CTAs than an H100 has SMs."""
    H = 128
    sd = _sd(H, 46)
    x = rl_oracle.synth_rl_features(2200, 40, 3, seed=46, empty_rows=1)
    want = rl_oracle.predict(rl_oracle.build(sd), x)
    m = _model(sd, H, path)
    assert m.windows_per_call(40, 3, 4) >= 2200
    got = m.forward_arrays(x)
    m.close()
    _check({"probs": got}, {"probs": want}, "tiles H=128 %s" % path)


@pytest.mark.gpu
def test_more_than_65535_windows_are_split():
    """70 000 windows of 2 positions: more than mdk_rl_forward takes in one call, so forward_arrays splits them."""
    H = 128
    sd = _sd(H, 47)
    x = rl_oracle.synth_rl_features(70000, 2, 1, seed=47, empty_rows=0)
    want = rl_oracle.predict(rl_oracle.build(sd), x)
    m = _model(sd, H, "tc")
    got = m.forward_arrays(x)
    m.close()
    _check({"probs": got}, {"probs": want}, "70000 windows")


@pytest.mark.gpu
@pytest.mark.parametrize("H,B,D", [(384, 128, 2), (128, 220, 1)])
def test_beyond_2_31_elements(H, B, D):
    """One device call whose LSTM pre-activations gi hold more than 2^31 floats (B x 10 000 x 8H): windows 0, 64 and
    the last are bit-identical to the same windows run alone, and window 0 is within the bars of the oracle."""
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < (40 << 30):
        pytest.skip("needs 40 GB of free device memory, %.1f GB free" % (free / 2 ** 30))
    P = PROD_P
    assert B * P * 8 * H > 2 ** 31
    sd = _sd(H, 48, True)
    x = rl_oracle.featuriser_like_rl_features(B, P, D, F=5, seed=48)
    m = _model(sd, H, "tc", use_dwells=True)
    m.max_bytes = 1 << 40                          # one device call
    assert m.windows_per_call(P, D, 5) >= B
    got = m.forward_arrays(x)
    alone = {b: m.forward_arrays(x[b:b + 1])[0] for b in (0, 64, B - 1)}
    m.close()
    for b, p in alone.items():
        assert np.array_equal(got[b], p), b
    want = rl_oracle.stages(rl_oracle.build(sd, use_dwells=True), x[:1])
    _check({"probs": got[:1]}, {"probs": want["probs"]}, "2^31 H=%d" % H)
