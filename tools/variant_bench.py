#!/usr/bin/env python
"""Variant calling from pileups to variant records, two ways, on synthetic pileups (the pileup_source of
tools/consensus_bench.py) and a draft of --mb megabases:

    (a) two-pass: prediction.predict_regions -> directory store (label_probs, 20 B per column) -> variant.variants
    (b) one-pass: prediction.predict_variants (call bytes and phreds stay on the device, 9 B per column)

    python tools/variant_bench.py [--mb 50] [--repeats 2]

Every contig gets the same pileup, so the network's calls are the same on every contig: the draft is those calls
(from one warm-up run), with ~1 % of the positions of every contig mutated (seeded), so that variants are sparse.  The
two paths are run alternately in one process, (a) first, after one warm-up of each.  Per run one JSON line: wall clock
from the first region to the last record, pileup columns / s, bytes copied device -> host and host -> device (counted
from the shapes of what the engine and the decode entry points are given and return), the peak arena bytes of the
one-pass run, the number of records and whether they equal the other path's.  The GPU's name and power limit are
recorded in every line.
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
    """(name, power limit) of GPU 0 as nvidia-smi reports them (a read-only query), or None where it is absent."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = [x.strip() for x in out.split(",")[:2]]
        return name, limit
    except Exception:
        return None, None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mb", type=float, default=50.0, help="draft megabases")
    ap.add_argument("--region-mb", type=float, default=1.0, help="length of each draft contig")
    ap.add_argument("--batch-size", type=int, default=200)
    ap.add_argument("--workers", type=int, default=8)
    ap.add_argument("--repeats", type=int, default=2)
    args = ap.parse_args()
    from medaka_b200 import common, datastore, features, labels, libmedaka as lm, models, prediction, variant
    from oracle import synth      # seeded synthetic weights / counts only
    lm.require_gpu(0)
    card, power = gpu_card()

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
    regions = [common.Region("ctg%d" % i, 0, ctg_len) for i in range(n_ctg)]
    cols = n_ctg * int((base_pos["major"] < ctg_len).sum())
    run = dict(chunk_len=10000, chunk_ovlp=1000, batch_size=args.batch_size, bam_chunk=1000000,
               bam_workers=args.workers)

    # bytes over PCIe, from the shapes of the engine calls and of the decode entry points
    d2h, h2d, peak = [0], [0], [0]
    orig = dict(sub_arrays=model.submit_arrays, sub_var=model.submit_variant_decoded, dec=labels.decode_arrays,
                dva=labels.decode_variant_arrays, cuts=labels.variant_join_cuts, dvs=labels.decode_variant_segments,
                free=prediction._LabelArena.free)

    def count_arrays(feats, probs_out, labels_out=None, logits_out=None):
        h2d[0] += feats.nbytes
        d2h[0] += probs_out.nbytes + (labels_out.nbytes if labels_out is not None else 0)
        return orig["sub_arrays"](feats, probs_out, labels_out, logits_out)

    def count_var(feats, ref, calls, pq, rq):
        h2d[0] += feats.nbytes + ref.nbytes
        d2h[0] += sum(x.nbytes for x in (calls, pq, rq) if isinstance(x, np.ndarray))
        return orig["sub_var"](feats, ref, calls, pq, rq)

    def count_dec(label_probs, device=0, with_qualities=True):
        out = orig["dec"](label_probs, device, with_qualities)
        h2d[0] += np.asarray(label_probs).nbytes
        d2h[0] += sum(x.nbytes for x in out if x is not None)
        return out

    def count_dva(label_probs, minor, ref_codes, device=0, want_quals=True):
        out = orig["dva"](label_probs, minor, ref_codes, device, want_quals)
        h2d[0] += np.asarray(label_probs).nbytes // np.asarray(label_probs).itemsize * 4 + 9 * len(minor)
        d2h[0] += sum(x.nbytes for x in out.values() if x is not None)
        return out

    def count_cuts(seg_calls, seg_rows, device=0):
        h2d[0] += 16 * len(seg_calls)
        d2h[0] += 8 * len(seg_calls)
        return orig["cuts"](seg_calls, seg_rows, device)

    def count_dvs(*a, **k):
        out = orig["dvs"](*a, **k)
        h2d[0] += 33 * len(a[0])
        d2h[0] += sum(x.nbytes for x in out.values() if x is not None)
        return out

    def free(self):
        peak[0] = max(peak[0], self.peak)
        return orig["free"](self)

    model.submit_arrays, model.submit_variant_decoded = count_arrays, count_var
    labels.decode_arrays, labels.decode_variant_arrays = count_dec, count_dva
    labels.variant_join_cuts, labels.decode_variant_segments = count_cuts, count_dvs
    prediction._LabelArena.free = free

    tmp = tempfile.mkdtemp(prefix="mdk_var_")
    t_start = time.perf_counter()

    def progress(what):
        print("[{:8.1f} s] {}".format(time.perf_counter() - t_start, what), file=sys.stderr, flush=True)

    def two_pass(regs, drf):
        store = os.path.join(tmp, "p.npzstore")
        prediction.predict_regions(store, None, regs, model, enc, **run)
        try:
            return variant.variants(store, drf)
        finally:
            shutil.rmtree(store, ignore_errors=True)

    def one_pass(regs, drf):
        return prediction.predict_variants(None, regs, model, enc, drf, **run)

    try:
        # the draft: the calls on one contig's major columns (the same on every contig), mutated per contig
        store = os.path.join(tmp, "calls.npzstore")
        prediction.predict_regions(store, None, [common.Region("c", 0, ctg_len)], model, enc, **run)
        rs = np.random.RandomState(5)
        calls = np.frombuffer(b"ACGT", np.uint8)[rs.randint(0, 4, ctg_len)].copy()
        ds = datastore.DataStore(store, "r")
        for name in ds.sample_registry:
            s = ds.load_sample(name)
            lab = np.argmax(np.asarray(s.label_probs), -1)
            keep = (s.positions["minor"] == 0) & (lab > 0)
            calls[s.positions["major"][keep]] = np.frombuffer(b"*ACGT", np.uint8)[lab[keep]]
        ds.close()
        shutil.rmtree(store, ignore_errors=True)
        acgt = np.frombuffer(b"ACGT", np.uint8)
        index_of = np.zeros(256, np.int64)
        index_of[acgt] = np.arange(4)
        draft = {}
        for r in regions:
            seq = calls.copy()
            at = rs.choice(ctg_len, ctg_len // 100, replace=False)
            seq[at] = acgt[(index_of[seq[at]] + rs.randint(1, 4, len(at))) % 4]      # a different base
            draft[r.ref_name] = seq.tobytes().decode()
        progress("draft ready")
        warm = [common.Region(regions[0].ref_name, 0, min(ctg_len, 200000))]
        for fn in (two_pass, one_pass):
            progress("warm-up: {} records".format(len(fn(warm, draft))))
        last = {}
        for rep in range(args.repeats):
            for name, fn in (("two-pass", two_pass), ("one-pass", one_pass)):
                d2h[0] = h2d[0] = peak[0] = 0
                progress("{} run {}".format(name, rep))
                t0 = time.perf_counter()
                recs = fn(regions, draft)
                dt = time.perf_counter() - t0
                last[name] = recs
                other = last.get("two-pass" if name == "one-pass" else "one-pass")
                print(json.dumps({
                    "metric": "pileup columns/s from regions to variant records ({})".format(name),
                    "value": cols / dt, "unit": "columns/s", "seconds": dt, "columns": cols,
                    "d2h_bytes": d2h[0], "h2d_bytes": h2d[0],
                    "peak_arena_bytes": peak[0] if name == "one-pass" else None,
                    "records": len(recs), "draft_mb": n_ctg * ctg_len / 1e6, "repeat": rep,
                    "identical": None if other is None else other == recs,
                    "gpu": card, "power_limit": power, "timing": "host wall clock"}), flush=True)
    finally:
        model.close()
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
