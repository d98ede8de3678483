#!/usr/bin/env python
"""Read-level consensus from pileups to FASTQ, two ways, with an lstm_size 384 model with dwells (the width of every
released read-level model; seeded weights, gap class biased down) on seeded featuriser-like read-level features
(rl_oracle) over a random draft of --mb megabases:

    (a) two-pass: prediction.predict_regions -> directory store (label_probs, 20 B per column) -> stitch.sequence
    (b) one-pass: prediction.predict_consensus (decoded calls stay on the device, 2 B per column)

    python tools/rl_one_pass_bench.py [--mb 3] [--depth 16] [--repeats 2]

One warm-up of each arm, then the two alternate in one process, (a) first.  Per run one JSON line: wall clock from the
first region to the closed output, pileup positions / s, whether the FASTQ and gap bed equal the other arm's latest,
and the GPU's name, power limit and maximum SM clock (read-only nvidia-smi query at the start of the run).  The features
of one contig are generated once and reused, shifted, for every contig, so that the host's feature generation does not
pace the run.
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_card():
    """(name, power limit, max SM clock) of GPU 0 as nvidia-smi reports them (a read-only query), or Nones."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                              "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit, clock = [x.strip() for x in out.split(",")[:3]]
        return name, limit, clock
    except Exception:
        return None, None, None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mb", type=float, default=3.0, help="draft megabases")
    ap.add_argument("--region-mb", type=float, default=1.0, help="length of each draft contig")
    ap.add_argument("--depth", type=int, default=16, help="read rows per window")
    ap.add_argument("--batch-size", default="auto", help="windows per batch ('auto': the engine's one-wave group)")
    ap.add_argument("--workers", type=int, default=4)
    ap.add_argument("--repeats", type=int, default=2)
    args = ap.parse_args()
    from medaka_b200 import common, features, libmedaka as lm, prediction, read_level, stitch
    from oracle import rl_oracle      # seeded synthetic weights / features only
    lm.require_gpu(0)
    card, power, clock = gpu_card()
    batch_size = args.batch_size if args.batch_size == "auto" else int(args.batch_size)

    # one contig's read-level features: majors with insertion columns after ~12 % of them, read rows as the featuriser
    # packs them (rl_oracle.featuriser_like_rl_features), dwells in column 4
    ctg_len = int(args.region_mb * 1e6)
    rs = np.random.RandomState(11)
    n_ins = np.where(rs.rand(ctg_len) < 0.12, rs.randint(1, 3, ctg_len), 0)
    width = 1 + n_ins
    base_pos = np.empty(int(width.sum()), dtype=[('major', '<i8'), ('minor', '<i8')])
    base_pos['major'] = np.repeat(np.arange(ctg_len, dtype=np.int64), width)
    base_pos['minor'] = np.arange(len(base_pos), dtype=np.int64) - np.repeat(np.cumsum(width) - width, width)
    t0 = time.perf_counter()
    base_x = rl_oracle.featuriser_like_rl_features(1, len(base_pos), args.depth, F=5, seed=12)[0]
    t_feats = time.perf_counter() - t0

    def pileup_source(region, bam, encoder):
        keep = (base_pos['major'] >= region.start) & (base_pos['major'] < region.end)
        return [(base_x[keep], base_pos[keep])]

    model = read_level.LatentSpaceLSTM(lstm_size=384, use_dwells=True)
    sd = rl_oracle.synth_rl_state_dict(0, lstm_size=384, use_dwells=True)
    # the seeded weights call a gap almost everywhere; with the gap class biased down the consensus is about as long as
    # the draft, as a real model's is, so the two-pass arm's host decode and FASTQ are full size
    sd["linear.bias"][0] -= 6.0
    model.load_state_dict(sd)
    enc = features.ReadAlignmentFeatureEncoder(include_dwells=True, pileup_source=pileup_source)
    n_ctg = max(1, int(round(args.mb / args.region_mb)))
    draft = {"ctg%d" % i: np.frombuffer(b"ACGT", np.uint8)[rs.randint(0, 4, ctg_len)].tobytes().decode()
             for i in range(n_ctg)}
    regions = [common.Region(name, 0, ctg_len) for name in draft]
    positions = n_ctg * len(base_pos)
    run = dict(chunk_len=10000, chunk_ovlp=1000, batch_size=batch_size, bam_chunk=1000000, bam_workers=args.workers)
    tmp = tempfile.mkdtemp(prefix="mdk_rl1p_")

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
        warm = {"warm": draft["ctg0"][:200000]}
        for fn in (two_pass, one_pass):
            fn(os.path.join(tmp, "warm.fastq"), [common.Region("warm", 0, 200000)], warm)
        last = {}
        for rep in range(args.repeats):
            for name, fn in (("two-pass", two_pass), ("one-pass", one_pass)):
                out = os.path.join(tmp, "%s.fastq" % name)
                t0 = time.perf_counter()
                fn(out, regions, draft)
                dt = time.perf_counter() - t0
                last[name] = read(out)
                other = last.get("two-pass" if name == "one-pass" else "one-pass")
                print(json.dumps({
                    "metric": "read-level pileup positions/s from regions to closed FASTQ ({})".format(name),
                    "arm": name, "value": positions / dt, "unit": "positions/s", "seconds": dt,
                    "positions": positions, "draft_mb": n_ctg * ctg_len / 1e6, "depth": args.depth,
                    "lstm_size": 384, "dwells": True, "batch_size": batch_size, "repeat": rep,
                    "fastq_bytes": len(last[name][0]),
                    "identical": None if other is None else other == last[name],
                    "feature_generation_s": t_feats, "gpu": card, "power_limit": power, "max_sm_clock": clock,
                    "timing": "host wall clock"}), flush=True)
    finally:
        model.close()
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
