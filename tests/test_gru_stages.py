"""Consensus GRU stage by stage, at the shapes bench.py runs: groups of 1056 windows x 10 000 columns (one wave of the
one-tile recurrence), featuriser-like features, both tile counts of the tensor-core recurrences, both device paths (tc:
wgmma with fp16 hi / lo operand pairs; fp32: the CUDA-core twins).

Every stage is compared with oracle/gru_oracle.stages in float64:
  h0, h1  the layer outputs (read_activation), max|d| / max|ref|
  plog    the per-direction partial logits the layer-1 recurrence writes on the fused-head path (read_plog), the only
          view into the production layer-1 kernel, max|d| / max|ref|
  logits  max over positions of |d| / max_c|logit_c| (the scaling of the 1e-3 parity bar of tests/test_gpu_parity.py)
  probs   max|d|
and labels are identical wherever the reference's top-2 probability margin exceeds 1e-5.
The 1e-3 logit bar is the contract with the reference; it cannot tell a tensor-core kernel that computes all three fp16
products (hi.hi + hi.lo + lo.hi, DESIGN §3) from one that lost one: every lost product stays 3-17x under it.  These bars
can: test_ablations_exceed_the_bars checks (on the CPU) that every ablation of gru_oracle.ablate lands above 3x the bar
at one stage or more.
"""
import numpy as np
import pytest
import torch

from oracle import gru_oracle, synth

# One set of bars for every path and tile count, calibrated on an H100 80GB HBM3 (SXM, 700 W power limit) over every GPU
# case of this file (DESIGN §2 "GRU stage bars" has the table).  Worst device error, h0 / h1 / plog / logits / probs:
#   fp32 path           3.7e-7 / 5.0e-7 / -      / 6.6e-7 / 4.8e-7
#   tc path, one tile   1.1e-6 / 1.7e-6 / 1.6e-6 / 2.4e-6 / 1.3e-6
#   tc path, two tiles  1.5e-6 / 2.2e-6 / 2.0e-6 / 2.9e-6 / 1.4e-6
# Smallest ablation effects (test_ablations_exceed_the_bars prints them): h0 6.0e-5 (h), h1 5.6e-5 (x, hot weights),
# plog 6.9e-5 (w_ih0), logits 8.8e-5 (w_ih0), probs 9.5e-6 (x).
# Each bar is at most a third of that stage's smallest ablation effect, so a kernel that lost a product fails it, and at
# h0, h1, plog and logits at least 5x the worst error of either path.  At probs the window is narrower than the tc
# path's error allows (3e-6 is 2.1x its worst error); the other stages carry the discrimination there.
BARS = {"h0": 1e-5, "h1": 1.1e-5, "plog": 1.2e-5, "logits": 1.6e-5, "probs": 3e-6}
STAGES = ("h0", "h1", "plog", "logits", "probs")
MARGIN = 1e-5
WEIGHTS = {"default": {}, "hot": dict(rec_gain=2.5, head_gain=24.0)}
PROD_B, PROD_T = 1056, 10000
PROD_WINDOWS = (0, 15, 16, 527, 1040, 1055)    # a tile's first and last window, the next tile, the middle, the last tile


def _sd(weights, F=10, seed=21):
    return synth.synth_state_dict(seed, num_features=F, **WEIGHTS[weights])


def _scaled(k, got, want):
    """Element-wise error of stage k in the scaling of BARS."""
    d = np.abs(got.astype(np.float64) - want)
    if k == "probs":
        return d
    if k == "logits":
        return d / np.abs(want).max(-1, keepdims=True)
    return d / float(np.abs(want).max())


def _errors(got, want):
    return {k: float(_scaled(k, got[k], want[k]).max()) for k in STAGES if k in got}


def _check(got, want, label):
    """got: any subset of STAGES (+ "labels") for the same windows as want, arrays [windows, T, ...]."""
    err = _errors(got, want)
    print("gru-stages %s %s" % (label, " ".join("%s=%.3g" % (k, err[k]) for k in STAGES if k in err)))
    _block_report(got, want, label)
    for k in err:
        assert np.isfinite(got[k]).all(), k
    for k, e in err.items():
        assert e <= BARS[k], (label, k, e, BARS[k])
    top2 = np.sort(want["probs"], -1)[..., -2:]
    decided = (top2[..., 1] - top2[..., 0]) > MARGIN
    ref = np.argmax(want["probs"], -1)
    assert np.array_equal(got["labels"][decided], ref[decided]), label


def _block_report(got, want, label, block=1000):
    """Max error per block of steps along T, scaled like BARS (printed: the log shows whether error grows with T)."""
    T = want["probs"].shape[1]
    if T < 2 * block:
        return
    for k in STAGES:
        if k not in got:
            continue
        e = _scaled(k, got[k], want[k])
        e = e.max(axis=tuple(i for i in range(e.ndim) if i != 1))
        print("gru-blocks %s %s per %d steps: %s" % (label, k, block,
                                                      " ".join("%.2g" % e[i:i + block].max() for i in range(0, T, block))))


def _features(B, T, F, windows, seed):
    """B windows of T columns: featuriser-like at `windows` (the ones that get checked), synth_features_fast elsewhere
    (windows are independent: tests/test_gpu_parity.py::test_full_size_window_properties)."""
    x = synth.synth_features_fast(B, T, F, seed=seed)
    x[list(windows)] = gru_oracle.featuriser_like_features(len(windows), T, F, seed=seed)
    return x


def _model(sd, F, path, rec="auto", keep=False):
    from medaka_b200 import models
    m = models.GRUModel(num_features=F)
    m.load_state_dict(sd)
    m.set_precision(path)
    m.set_rec_mode(rec)
    m.keep_activations(keep)
    return m


def _plog_windows(plog, windows):
    """Device plog [dir][tile][T][class][16 windows] -> [windows, T, dir, class] (the oracle's layout)."""
    return np.stack([plog[:, w // 16, :, :, w % 16].transpose(1, 0, 2) for w in windows])


def _device(m, feats, windows, fused):
    """One forward; the stages it exposes, for `windows`: h0, logits, probs, labels, and plog (fused: the tc path's
    layer-1 recurrence with the head) or h1 (the fp32 path, or tc keeping its activations)."""
    m.set_group_windows(len(feats))         # one forward of all windows (a group holds 1056 by default)
    out = m.forward_arrays(feats, want_logits=True, want_labels=True)
    w = list(windows)
    got = {"logits": out.logits[w], "probs": out.probs[w], "labels": out.labels[w]}
    got["h0"] = np.concatenate([m.read_activation(0, i, 1) for i in w])
    if fused:
        got["plog"] = _plog_windows(m.read_plog(), w)
    else:
        got["h1"] = np.concatenate([m.read_activation(1, i, 1) for i in w])
    return got


def _need_memory(gb):
    free, _ = torch.cuda.mem_get_info()
    if free < (gb << 30):
        pytest.skip("needs %d GB of free device memory, %.1f GB free" % (gb, free / 2 ** 30))


# ---------------------------------------------------------------------------------------------- CPU
def test_stages_match_predict_and_manual_forward():
    """stages() in float32 restates the forward: predict_on_batch's logits and probabilities (nn.GRU) and
    manual_forward's h0 / h1; plog summed over directions plus the bias is the logits."""
    sd = _sd("default", seed=4)
    x = gru_oracle.featuriser_like_features(3, 300, 10, seed=4)
    st = gru_oracle.stages(sd, x, dtype=torch.float32)
    probs, logits = gru_oracle.predict_on_batch(gru_oracle.build(sd), x)
    man = gru_oracle.manual_forward(sd, x)
    assert st["h0"].shape == (3, 300, 256) and st["plog"].shape == (3, 300, 2, 5) and st["h0"].dtype == np.float32
    assert np.abs(st["logits"] - logits).max() <= 1e-5 and np.abs(st["probs"] - probs).max() <= 1e-6
    for k in ("h0", "h1"):
        assert np.abs(st[k] - man[k]).max() <= 1e-6
    assert np.abs(st["plog"].sum(-2) + sd["linear.bias"] - st["logits"]).max() <= 1e-5
    st64 = gru_oracle.stages(sd, x)
    assert st64["h1"].dtype == np.float64 and np.abs(st64["logits"] - logits).max() <= 1e-5


@pytest.mark.parametrize("F", [10, 20])
def test_featuriser_like_features_have_the_properties_of_real_windows(F):
    T = 3000
    x = gru_oracle.featuriser_like_features(4, T, F, seed=5)
    assert x.shape == (4, T, F) and x.dtype == np.float32 and x.min() >= 0
    s = x.sum(-1)
    empty = s == 0
    assert empty.any(1).all() and empty.mean() < 0.2                      # coverage gaps in every window
    groups = [[0, 1, 2, 3, 8], [4, 5, 6, 7, 9]]                            # (reverse, forward) strand of a datatype
    if F == 20:
        groups += [[i + 10 for i in g] for g in groups]
    gs = np.stack([x[..., g].sum(-1) for g in groups], -1)
    major = (np.abs(gs - 1) < 1e-5).all(-1) if F == 20 else np.abs(s - 1) < 1e-5
    minor = ~empty & ~major
    assert 0.6 < major.mean() < 0.95 and minor.mean() > 0.05
    # major columns one-hot-like: the true base on each strand carries most of the strand's reads
    top = np.sort(x[major], -1)[:, -(F // 5):].sum(-1) / (F // 10)
    assert np.median(top) > 0.85
    # minor (insertion) columns sparse and small (F = 20: each of the 4 strand groups is normalised to 1 on majors)
    assert (x[minor] == 0).mean() > 0.5 and np.median(s[minor]) / (1 if F == 10 else 4) < 0.5
    # fp16 cannot hold most of them: rounding x is a visible error
    v = x[x > 0]
    assert (v.astype(np.float16).astype(np.float32) != v).mean() > 0.3


@pytest.mark.parametrize("weights", sorted(WEIGHTS))
def test_ablations_exceed_the_bars(weights):
    """Every precision ablation (a kernel that lost one of its three fp16 products) moves some stage by more than 3x its
    bar on a reduced production case (4 featuriser-like windows x 2000 steps), so the bars can tell the products apart."""
    sd = _sd(weights)
    x = gru_oracle.featuriser_like_features(4, 2000, 10, seed=3)
    ref = gru_oracle.stages(sd, x)
    for which in gru_oracle.ABLATIONS:
        sd_a, kw = gru_oracle.ablate(sd, which)
        err = _errors(gru_oracle.stages(sd_a, x, **kw), ref)
        ratio = {k: err[k] / BARS[k] for k in STAGES}
        print("gru-ablation %-7s %-5s %s" % (weights, which, " ".join("%s=%.3g (%.1fx)" % (k, err[k], ratio[k])
                                                                        for k in STAGES)))
        assert max(ratio.values()) > 3, (which, err)


# ---------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def production():
    """production(weights): one bench.py group, 1056 windows x 10 000 columns x F = 10, and the float64 stages of
    PROD_WINDOWS; computed once per weight set and shared by every path."""
    cache = {}

    def get(weights):
        if weights not in cache:
            sd = _sd(weights, seed=31)
            x = _features(PROD_B, PROD_T, 10, PROD_WINDOWS, seed=31)
            cache[weights] = sd, x, gru_oracle.stages(sd, x[list(PROD_WINDOWS)])
        return cache[weights]
    yield get
    cache.clear()


@pytest.mark.gpu
@pytest.mark.parametrize("weights", sorted(WEIGHTS))
@pytest.mark.parametrize("path,rec", [("tc", "auto"), ("tc", "pp"), ("fp32", "auto")],
                         ids=["tc-one_tile", "tc-two_tiles", "fp32"])
def test_production_group(production, path, rec, weights):
    """A full group: on the tc path "auto" runs the one-tile kernels (fused x projection, fused head) and "pp" the
    two-tile kernels.  tc then runs again keeping h1 (the head as its own kernel): h0 is bit-identical, h1 in the bars."""
    _need_memory(60)
    sd, x, want = production(weights)
    label = "production %s %s %s" % (path, rec, weights)
    m = _model(sd, 10, path, rec)
    got = _device(m, x, PROD_WINDOWS, path == "tc")
    if path == "tc":
        m.keep_activations(True)
        kept = _device(m, x, PROD_WINDOWS, False)
        assert np.array_equal(kept["h0"], got["h0"])
        got["h1"] = kept["h1"]
    m.close()
    _check(got, want, label)


@pytest.mark.gpu
@pytest.mark.parametrize("path,rec", [("tc", "one"), ("tc", "pp"), ("fp32", "auto")],
                         ids=["tc-one_tile", "tc-two_tiles", "fp32"])
def test_f20_unfused_layer0(path, rec):
    """F = 20 (two datatypes, fwd_rev normalisation): layer 0 runs unfused, inproj0 writing gi in the quad layout."""
    _need_memory(20)
    B, T, windows = 300, 10000, (0, 17, 150, 299)
    sd = _sd("default", F=20, seed=32)
    x = _features(B, T, 20, windows, seed=32)
    want = gru_oracle.stages(sd, x[list(windows)])
    for keep in ((False, True) if path == "tc" else (False,)):
        m = _model(sd, 20, path, rec, keep)
        _check(_device(m, x, windows, path == "tc" and not keep), want, "f20 %s %s keep=%d" % (path, rec, keep))
        m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("rec", ["one", "pp"])
@pytest.mark.parametrize("T", [1, 129])
@pytest.mark.parametrize("B", [37, 1217])
def test_ragged(B, T, rec):
    """Partial tiles (37 windows: 3 tiles, the last of 5 windows) and 1217 windows (77 tiles: at two tiles per CTA the
    last CTA's second tile does not exist), T = 1 and T = 129 (not a multiple of the GEMM's 128-row tiles)."""
    windows = tuple(range(37)) if B == 37 else (0, 15, 16, 1200, 1215, 1216)
    sd = _sd("default", seed=33)
    x = _features(B, T, 10, windows, seed=33 + T)
    want = gru_oracle.stages(sd, x[list(windows)])
    for path, keep in (("tc", False), ("tc", True), ("fp32", False)):
        m = _model(sd, 10, path, rec, keep)
        _check(_device(m, x, windows, path == "tc" and not keep), want, "ragged B=%d T=%d %s %s keep=%d" % (B, T, path, rec, keep))
        m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("rec", ["one", "pp"])
def test_kept_and_fused_head_runs(rec):
    """The layer-1 recurrence writing h1 (OUT_ROWS, the head as its own kernel) and writing partial logits (the fused
    head) on the same input: layer 0 is the same computation, so h0 is bit-identical; both runs are within the bars."""
    windows = tuple(range(45))
    sd = _sd("hot", seed=34)
    x = gru_oracle.featuriser_like_features(45, 2000, 10, seed=34)
    want = gru_oracle.stages(sd, x)
    m = _model(sd, 10, "tc", rec)
    fused = _device(m, x, windows, True)
    m.keep_activations(True)
    kept = _device(m, x, windows, False)
    m.close()
    assert np.array_equal(fused["h0"], kept["h0"])
    _check(fused, want, "fused %s" % rec)
    _check(kept, want, "kept %s" % rec)
