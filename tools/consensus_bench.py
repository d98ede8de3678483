#!/usr/bin/env python
"""Consensus from pileups to FASTQ, two ways, on synthetic pileups (the pileup_source of tools/pipeline_bench.py) and
a seeded random draft of --mb megabases:

    (a) two-pass: prediction.predict_regions -> directory store (label_probs, 20 B per column) -> stitch.sequence
    (b) one-pass: prediction.predict_consensus (decoded calls stay on the device, 2 B per column)

    python tools/consensus_bench.py [--mb 20] [--repeats 2]

The two are run alternately in one process, (a) first, after one warm-up of each.  Per run one JSON line: wall clock
from the first region to the closed output, pileup columns / s, bytes copied device -> host (engine outputs, counted
from the calls' shapes, plus the stitched bytes returned), and whether the FASTQ and bed equal the other path's.
"""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mb", type=float, default=20.0, help="draft megabases")
    ap.add_argument("--region-mb", type=float, default=1.0, help="length of each draft contig")
    ap.add_argument("--batch-size", type=int, default=200)
    ap.add_argument("--workers", type=int, default=8)
    ap.add_argument("--repeats", type=int, default=2)
    args = ap.parse_args()
    from medaka_b200 import common, features, libmedaka as lm, models, prediction, stitch
    from oracle import synth      # seeded synthetic weights / counts only
    lm.require_gpu(0)

    base_counts, base_pos = synth.synth_counts(int(args.region_mb * 1e6 * 1.18) + 8, seed=11)

    def pileup_source(region, bam, encoder):
        n_ref = region.end - region.start
        pos = base_pos.copy()
        keep = pos["major"] < n_ref
        pos = pos[keep]
        pos["major"] += region.start
        return [(base_counts[keep], pos)]

    model = models.GRUModel(num_features=10)
    model.load_state_dict(synth.synth_state_dict(0))
    enc = features.CountsFeatureEncoder(normalise="total", pileup_source=pileup_source)
    n_ctg = max(1, int(round(args.mb / args.region_mb)))
    ctg_len = int(args.region_mb * 1e6)
    rs = np.random.RandomState(5)
    draft = {"ctg%d" % i: np.frombuffer(b"ACGT", np.uint8)[rs.randint(0, 4, ctg_len)].tobytes().decode()
             for i in range(n_ctg)}
    regions = [common.Region(name, 0, ctg_len) for name in draft]
    cols = n_ctg * int((base_pos["major"] < ctg_len).sum())
    run = dict(chunk_len=10000, chunk_ovlp=1000, batch_size=args.batch_size, bam_chunk=1000000,
               bam_workers=args.workers)

    # device -> host bytes: the engine's outputs from the calls' shapes, the stitch's from what it returns
    d2h = [0]
    sub_arrays, sub_decoded, split_text = model.submit_arrays, model.submit_decoded, stitch._split_text

    def count_arrays(feats, probs_out, labels_out=None, logits_out=None):
        d2h[0] += probs_out.nbytes + (labels_out.nbytes if labels_out is not None else 0)
        return sub_arrays(feats, probs_out, labels_out, logits_out)

    def count_decoded(feats, labels_out, quals_out=None):
        d2h[0] += sum(x.nbytes for x in (labels_out, quals_out) if isinstance(x, np.ndarray))
        return sub_decoded(feats, labels_out, quals_out)

    def count_split(seq, qual, off):
        d2h[0] += 2 * int(off[-1]) + 8 * len(off)
        return split_text(seq, qual, off)

    model.submit_arrays, model.submit_decoded, stitch._split_text = count_arrays, count_decoded, count_split

    tmp = tempfile.mkdtemp(prefix="mdk_cons_")

    def two_pass(out, regs, drf):
        store = out + ".npzstore"
        prediction.predict_regions(store, None, regs, model, enc, **run)
        stitch.sequence(store, drf, out)
        shutil.rmtree(store, ignore_errors=True)

    def one_pass(out, regs, drf):
        prediction.predict_consensus(None, regs, model, enc, drf, out, **run)

    def read(out):
        with open(out, "rb") as fh, open(out + ".gaps_in_draft_coords.bed", "rb") as fb:
            return fh.read(), fb.read()

    try:
        warm_draft = {"warm": draft["ctg0"][:200000]}
        for fn in (two_pass, one_pass):
            fn(os.path.join(tmp, "warm.fastq"), [common.Region("warm", 0, 200000)], warm_draft)
        last = {}
        for rep in range(args.repeats):
            for name, fn in (("two-pass", two_pass), ("one-pass", one_pass)):
                out = os.path.join(tmp, "%s.fastq" % name)
                d2h[0] = 0
                t0 = time.perf_counter()
                fn(out, regions, draft)
                dt = time.perf_counter() - t0
                last[name] = read(out)
                other = last.get("two-pass" if name == "one-pass" else "one-pass")
                print(json.dumps({
                    "metric": "pileup columns/s from regions to closed FASTQ ({})".format(name),
                    "value": cols / dt, "unit": "columns/s", "seconds": dt, "columns": cols,
                    "d2h_bytes": d2h[0], "draft_mb": n_ctg * ctg_len / 1e6, "repeat": rep,
                    "identical": None if other is None else other == last[name],
                    "timing": "host wall clock"}), flush=True)
    finally:
        model.close()
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
