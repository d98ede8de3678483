"""Golden vectors for counts models with three and four datatypes (F = 30 and 40), from the REAL reference classes.

Run:  python tests/golden/make_multi_dtype_golden.py   (needs /root/reference; writes tests/golden/multi_dtype.npz)

Imports the reference unmodified behind make_golden.install_stubs() and records:
  * medaka.features.CountsFeatureEncoder._post_process_pileup with 3 and 4 datatypes, every normalise mode x sym_indels,
    on synthetic counts, a chunk that starts on a minor column, a deep pileup, a stretch where one datatype has no reads
    (its per-(datatype, strand) depth is 0), and minor columns whose sym_indels fill wraps around in uint64;
  * medaka.features.pileup_counts_norm_indices for 3 and 4 datatypes;
  * medaka.architectures.gru.GRUModel(num_features = 30 / 40) through predict_on_batch: probabilities and logits.
Before writing, it asserts that the oracle (oracle/features_oracle.py, oracle/gru_oracle.py) reproduces every recorded
output: the post-processing bit for bit, the forward to 2e-6.  The tests read only the .npz.
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden  # noqa: E402  (puts the repository root on sys.path)

DTYPES = {3: ("r9", "r10", "x"), 4: ("r9", "r10", "x", "y")}
# (name, seed, B, T, F, head_gain, rec_gain)
FORWARD_CASES = [("f30", 50, 3, 300, 30, 8.0, 1.0),
                 ("f40", 51, 2, 1000, 40, 8.0, 1.0),
                 ("f40_b1", 52, 1, 777, 40, 8.0, 1.0),
                 ("f40_hot", 53, 2, 300, 40, 24.0, 2.5)]


def norm_inputs():
    """{name: (counts uint64 [n, 10 nd], positions, dtypes)} for nd = 3 and 4."""
    import numpy as np
    from oracle import synth
    out = {}
    for nd in (3, 4):
        dts = DTYPES[nd]
        out["synth%d" % nd] = synth.synth_counts(120, seed=60 + nd, num_dtypes=nd) + (dts,)
        out["minor_start%d" % nd] = synth.synth_counts(80, seed=62 + nd, num_dtypes=nd, start_on_minor=True,
                                                       start_major=1000) + (dts,)
        out["deep%d" % nd] = synth.synth_counts(30, seed=64 + nd, num_dtypes=nd, mean_depth=20000,
                                                max_depth=100000) + (dts,)
        # datatype 1 has no reads over columns 30..89, datatype nd - 1 none on its reverse strand over 110..139
        counts, pos = synth.synth_counts(160, seed=66 + nd, num_dtypes=nd)
        counts[30:90, 10:20] = 0
        counts[110:140, [10 * (nd - 1) + k for k in (0, 1, 2, 3, 8)]] = 0
        out["empty_dt%d" % nd] = (counts, pos, dts)
        # some minor columns carry more reads of one datatype than their major column: the sym_indels fill
        # (major group depth - minor group depth) wraps around in uint64
        counts, pos = synth.synth_counts(100, seed=68 + nd, num_dtypes=nd)
        rs = np.random.RandomState(70 + nd)
        minors = np.flatnonzero(pos["minor"] > 0)
        for i in rs.choice(minors, len(minors) // 3, replace=False):
            counts[i, 10 * rs.randint(0, nd) + rs.choice([0, 5])] += np.uint64(200)
        out["wrap%d" % nd] = (counts, pos, dts)
    return out


def main():
    make_golden.install_stubs()
    import numpy as np
    import torch
    import medaka.architectures.gru as ref_gru
    import medaka.common as ref_common
    import medaka.features as ref_features
    from oracle import features_oracle, gru_oracle, synth

    torch.set_num_threads(8)
    meta = "medaka v%s, torch %s, numpy %s" % (__import__('medaka').__version__, torch.__version__, np.__version__)
    print(meta)
    out = {}

    # ---------------------------------------------------------------- normalisation
    region = ref_common.Region('ref', 0, 8)
    for name, (counts, pos, dtypes) in norm_inputs().items():
        out["norm_%s_counts" % name] = counts
        out["norm_%s_major" % name] = pos['major']
        out["norm_%s_minor" % name] = pos['minor']
        for norm in ('total', 'fwd_rev', None):
            for sym in (False, True):
                enc = ref_features.CountsFeatureEncoder(normalise=norm, dtypes=dtypes, sym_indels=sym)
                s = enc._post_process_pileup(counts.copy(), pos, region)
                key = "norm_%s_%s_%d" % (name, norm, int(sym))
                feats, depth = s.features, np.asarray(s.depth)
                ef, ed = features_oracle.post_process_pileup(counts.copy(), pos, norm, dtypes=dtypes, sym_indels=sym)
                assert feats.dtype == np.float32 and np.array_equal(feats, ef), key
                assert np.array_equal(depth.astype(np.int64), ed.astype(np.int64)), key
                out[key + "_features"] = feats
                out[key + "_depth"] = depth
        if name.startswith("wrap"):
            assert (features_oracle.post_process_pileup(counts.copy(), pos, None, dtypes=dtypes, sym_indels=True)[0]
                    > 1e18).any(), "no sym_indels fill wrapped around"
        print("normalisation", name, counts.shape)
    for nd, dtypes in DTYPES.items():
        got = ref_features.pileup_counts_norm_indices(list(dtypes))
        assert got == features_oracle.pileup_counts_norm_indices(list(dtypes))
        for (dt, rev), v in got.items():
            out["idx_%s|%s|%d" % (",".join(dtypes), dt, int(rev))] = np.array(v)

    # ---------------------------------------------------------------- forward pass
    for name, seed, B, T, F, head_gain, rec_gain in FORWARD_CASES:
        sd = synth.synth_state_dict(seed, num_features=F, head_gain=head_gain, rec_gain=rec_gain)
        model = ref_gru.GRUModel(num_features=F)
        model.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
        model.eval()
        feats = synth.synth_features(B, T, F, seed=100 + seed)

        class _Batch:
            counts_matrix = torch.from_numpy(feats)

        probs = model.predict_on_batch(_Batch())           # medaka/models.py:303-313
        assert probs.device.type == 'cpu' and probs.dtype == torch.float32
        model.normalise = False                             # gru.py:68-71 -> logits
        logits = model.predict_on_batch(_Batch())
        probs, logits = probs.numpy(), logits.numpy()
        op, ol = gru_oracle.predict_on_batch(gru_oracle.build(sd, num_features=F), feats)
        assert np.abs(op - probs).max() <= 2e-6 and np.abs(ol - logits).max() <= 2e-6, name
        out["fwd_%s_probs" % name] = probs
        out["fwd_%s_logits" % name] = logits
        out["fwd_%s_args" % name] = np.array([seed, B, T, F, head_gain, rec_gain], dtype=np.float64)
        print("forward", name, probs.shape, float(probs.max()))
    np.savez_compressed(os.path.join(HERE, "multi_dtype.npz"), meta=meta, **out)
    print("golden vectors written to", os.path.join(HERE, "multi_dtype.npz"))


if __name__ == "__main__":
    main()
