#!/usr/bin/env python
"""On-device measurement of the fp16 product sets (VERDICT r01 item 2): for each set of products per contraction
{hi.hi} / {hi.hi + W_hi.x_lo} / {hi.hi + W_lo.x_hi} / {all three} the real kernels (fused layer-0 projection, both
recurrences, the layer-1 GEMM; the fused linear head is fp32 on the CUDA cores whatever the set) are run on the golden
cases, a T = 10 000 batch and two "hot" recurrent-gain models, against the fp32 CPU reference.  Writes markdown to
stdout."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import gru_oracle, synth  # noqa: E402

SETS = [(7, "hi.hi + hi.lo + lo.hi (default)"), (3, "hi.hi + W_hi.x_lo  (weights rounded to fp16)"),
        (5, "hi.hi + W_lo.x_hi  (activations rounded to fp16)"), (1, "hi.hi only")]
NEAR = 1e-5


def main():
    from medaka_b200 import models
    g = np.load(os.path.join(ROOT, "tests", "golden", "gru_forward.npz"))
    cases = []
    for case in ("small", "long", "hot", "f20", "b1", "neartie"):
        seed, B, T, F, hg, rg = g[case + "_args"]
        maker = synth.synth_state_dict_neartie if case == "neartie" else synth.synth_state_dict
        sd = maker(int(seed), num_features=int(F), head_gain=hg, rec_gain=rg)
        feats = synth.synth_features(int(B), int(T), int(F), seed=100 + int(seed))
        cases.append(("golden:" + case, sd, feats, int(F), g[case + "_probs"], g[case + "_logits"]))
    for name, kw, B, T in (("T=10000 (16 windows)", {}, 16, 10000), ("hot rec_gain=2 (8 x 3000)", dict(rec_gain=2.0), 8, 3000),
                           ("hot rec_gain=3 (8 x 3000)", dict(rec_gain=3.0), 8, 3000),
                           ("wave 1184 x 512 (ping-pong kernels)", {}, 1184, 512)):
        sd = synth.synth_state_dict(0, **kw)
        feats = synth.synth_features_fast(B, T, 10, seed=21)
        p, l = gru_oracle.predict_on_batch(gru_oracle.build(sd), feats, threads=8)
        cases.append((name, sd, feats, 10, p, l))
    rows = []
    for name, sd, feats, F, ref_p, ref_l in cases:
        for mask, label in SETS:
            m = models.GRUModel(num_features=F)
            m.load_state_dict(sd)
            m.set_products(mask)
            out = m.forward_arrays(feats, want_logits=True)
            t = m.last_timings()
            m.close()
            scale = np.abs(ref_l).max(-1, keepdims=True)
            d = np.abs(out.logits - ref_l)
            top2 = np.sort(ref_p, -1)[..., -2:]
            near = (top2[..., 1] - top2[..., 0]) <= NEAR
            mism = out.labels != np.argmax(ref_p, -1)
            rows.append(dict(case=name, products=label, mask=mask, positions=int(mism.size),
                             scaled=float((d / scale).max()), elementwise=float((d / np.maximum(np.abs(ref_l), 1e-30)).max()),
                             flips_decided=int((mism & ~near).sum()), flips_near=int((mism & near).sum()),
                             near=int(near.sum()), rec_ms=t["rec0_ms"] + t["rec1_ms"], gemm_ms=t["inproj1_ms"]))
            print(json.dumps(rows[-1]), file=sys.stderr, flush=True)
    print("| case | products per contraction | positions | scaled logit err | element-wise rel err | decided-label flips | "
          "near-tie flips / near ties | rec ms | GEMM ms |")
    print("|---|---|---|---|---|---|---|---|---|")
    for r in rows:
        print("| %s | %s | %d | %.2e | %.2e | %d | %d / %d | %.2f | %.2f |" % (
            r["case"], r["products"], r["positions"], r["scaled"], r["elementwise"], r["flips_decided"], r["flips_near"],
            r["near"], r["rec_ms"], r["gemm_ms"]))


if __name__ == "__main__":
    main()
