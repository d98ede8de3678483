#!/usr/bin/env python
"""Drives every HBM-bound kernel of the path at a realistic size through the C ABI (a workload for a kernel profiler),
and prints wall-clock figures of the host-pointer calls (copies included) plus the pileup rate next to the CPU
restatement (oracle/pileup_oracle.py).

    python tools/hbm_bench.py [--n 4000000] [--reads 20000] [--cpu-pileup]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def timed(fn, reps=3):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return min(ts)


def pileup_ops(rec):
    """(length, op) of the reference-consuming CIGAR operations of a synthetic record."""
    cig = rec["cigar"]
    if isinstance(cig, str):
        import re
        cig = [(int(l), o) for l, o in re.findall(r"(\d+)([MIDNSHP=X])", cig)]
    return [(l, o) for l, o in cig if o in "MDN=X"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=4000000, help="pileup columns for the per-column kernels")
    ap.add_argument("--reads", type=int, default=20000)
    ap.add_argument("--read-len", type=int, default=5000)
    ap.add_argument("--cpu-pileup", action="store_true", help="also time the CPU restatement of calculate_pileup")
    args = ap.parse_args()
    from medaka_b200 import libmedaka as lm, models, labels as mlabels, features as mfeatures
    from oracle import synth
    lib, ffi = lm.load(), lm.ffi
    dev = 0
    lm.require_gpu(dev)
    n = args.n
    res = {}

    def dalloc(nbytes):
        pp = ffi.new("void **")
        lm.check(lib.mdk_dev_alloc(dev, nbytes, pp))
        return pp[0]

    def h2d(arr):
        d = dalloc(arr.nbytes)
        lm.check(lib.mdk_memcpy_h2d(dev, d, ffi.from_buffer(arr), arr.nbytes))
        return d

    def dev_time(fn, reps=5):
        fn()
        lm.check(lib.mdk_device_synchronize(dev))
        t0 = time.perf_counter()
        for _ in range(reps):
            fn()
        lm.check(lib.mdk_device_synchronize(dev))
        return (time.perf_counter() - t0) / reps

    # ---- a3 normalise (counts -> features): 144 B / column (F = 10), device-resident ----
    for nd, mode, name in ((1, lib.MDK_NORM_TOTAL, "normalise total F=10"), (2, lib.MDK_NORM_FWD_REV, "normalise fwd_rev F=20")):
        counts, pos = synth.synth_counts(n, seed=5, num_dtypes=nd)
        major = np.ascontiguousarray(pos["major"]).astype(np.int64)
        minor = np.ascontiguousarray(pos["minor"]).astype(np.int64)
        F = 10 * nd
        d_counts, d_major, d_minor = h2d(counts), h2d(major), h2d(minor)
        d_feats, d_depth = dalloc(n * F * 4), dalloc(n * 8)
        t = dev_time(lambda: lm.check(lib.mdk_normalise_counts_dev(
            dev, ffi.cast("const uint64_t *", d_counts), ffi.cast("const int64_t *", d_major),
            ffi.cast("const int64_t *", d_minor), n, nd, mode, 0, ffi.cast("float *", d_feats),
            ffi.cast("int64_t *", d_depth))))
        bytes_alg = n * (8 * F + 16 + 4 * F + 8)
        res[name] = {"columns": n, "call_ms": t * 1e3, "algorithmic_GBps": bytes_alg / t / 1e9, "bytes_per_column": bytes_alg // n}
        for d in (d_counts, d_major, d_minor, d_feats, d_depth):
            lm.check(lib.mdk_dev_free(dev, d))

    # ---- a9 decode (probs -> labels + quals): 22 B / column ----
    rs = np.random.RandomState(3)
    probs = rs.dirichlet(np.ones(5) * 0.3, size=n).astype(np.float32)
    d_probs = h2d(probs)
    d_lab, d_q = dalloc(n), dalloc(n)
    t = dev_time(lambda: lm.check(lib.mdk_decode_consensus_dev(dev, ffi.cast("const float *", d_probs), n,
                                                               ffi.cast("uint8_t *", d_lab), ffi.cast("uint8_t *", d_q))))
    res["decode_consensus"] = {"columns": n, "call_ms": t * 1e3, "algorithmic_GBps": n * 22 / t / 1e9, "bytes_per_column": 22}

    # ---- f1 stitch (kept row ranges -> sequence + qualities): 20 B in, <= 2 B out per row ----
    seg = 9000
    seg_base = np.arange(0, n, seg, dtype=np.int64)
    seg_off = np.zeros(len(seg_base) + 1, dtype=np.int64)
    d_seq, d_qual = dalloc(n), dalloc(n)
    t = dev_time(lambda: lm.check(lib.mdk_stitch_consensus_dev(
        dev, ffi.cast("const float *", d_probs), n, ffi.cast("const int64_t *", ffi.from_buffer(seg_base)), len(seg_base),
        ffi.cast("uint8_t *", d_seq), ffi.cast("uint8_t *", d_qual), ffi.cast("int64_t *", ffi.from_buffer(seg_off)))))
    res["stitch_consensus_dev"] = {"rows": n, "segments": int(len(seg_base)), "call_ms": t * 1e3,
                                   "algorithmic_GBps": (n * 20 + 2 * int(seg_off[-1])) / t / 1e9,
                                   "kept_bases": int(seg_off[-1])}

    # ---- f2 variant decode (host pointers: copies included in the call) ----
    vminor = (rs.uniform(size=n) < 0.12).astype(np.int64)
    vminor[0] = 0
    vref = np.where(vminor == 0, rs.randint(1, 5, n), 0).astype(np.uint8)
    out = {}
    t = timed(lambda: out.update(mlabels.decode_variant_arrays(probs, vminor, vref, dev, want_quals=True)))
    res["decode_variants (host buffers)"] = {"columns": n, "call_ms": t * 1e3, "runs": int(len(out["run_start"])),
                                             "columns_per_s": n / t}

    # ---- a1 pileup counts from packed records (host pointers) ----
    # (the record generator is a Python loop: 2000 reads are generated and tiled along the reference)
    from medaka_b200 import bam as mbam
    base_n = min(args.reads, 2000)
    reps = max(1, args.reads // base_n)
    span0 = max(100000, base_n * args.read_len // 30)             # ~30x coverage
    recs = synth.synth_reads(base_n, span0, seed=9, mean_len=args.read_len)
    b0 = mbam.records_from_dicts(recs)
    span = span0 * reps
    args.reads = base_n * reps
    batch = mbam.RecordBatch(
        pos=np.concatenate([b0.pos + k * span0 for k in range(reps)]).astype(np.int32), flag=np.tile(b0.flag, reps),
        mapq=np.tile(b0.mapq, reps), dtype=np.tile(b0.dtype, reps), cigar=np.tile(b0.cigar, reps),
        cigar_off=np.concatenate([b0.cigar_off[:-1] + k * b0.cigar_off[-1] for k in range(reps)] + [[reps * b0.cigar_off[-1]]]).astype(np.int64),
        seq=np.tile(b0.seq, reps),
        seq_off=np.concatenate([b0.seq_off[:-1] + k * b0.seq_off[-1] for k in range(reps)] + [[reps * b0.seq_off[-1]]]).astype(np.int64),
        l_seq=np.tile(b0.l_seq, reps), names=None, tags=None)
    aligned = reps * int(sum(l for r in recs for l, op in pileup_ops(r)))
    holder = {}

    def run_plp():
        holder["out"] = mfeatures.pileup_counts_from_batch(batch, 0, span, num_dtypes=1, min_mapq=1, device=dev)
    t = timed(run_plp)
    counts, positions = holder["out"]
    res["pileup_counts (host buffers)"] = {"reads": args.reads, "span": span, "columns": int(len(positions)),
                                           "call_ms": t * 1e3, "reads_per_s": args.reads / t,
                                           "columns_per_s": len(positions) / t,
                                           "aligned_bases_per_s": aligned / t}
    def run_fused():
        holder["fused"] = mfeatures.pileup_features_from_batch(batch, 0, span, 1, 1, "total", False, dev)
    t = timed(run_fused)
    res["pileup_features fused (host buffers)"] = {"reads": args.reads, "columns": int(len(holder["fused"][2])),
                                                   "call_ms": t * 1e3, "reads_per_s": args.reads / t,
                                                   "columns_per_s": len(holder["fused"][2]) / t,
                                                   "aligned_bases_per_s": aligned / t}

    def run_two_step():
        c, p = mfeatures.pileup_counts_from_batch(batch, 0, span, num_dtypes=1, min_mapq=1, device=dev)
        enc = mfeatures.CountsFeatureEncoder(normalise="total", device=dev)

        class R(object):
            ref_name, start, end = "x", 0, span
        holder["two"] = enc._post_process_pileup(c, p, R)
    t = timed(run_two_step)
    res["pileup_counts + normalise, two calls (host buffers)"] = {"call_ms": t * 1e3, "columns_per_s": len(positions) / t}

    # ---- a11 read-level feature matrix over the same reads (host pointers; row bookkeeping on the host) ----
    rbatch = batch._replace(names=["r%d" % i for i in range(args.reads)],
                            qual=np.tile(b0.qual, reps) if b0.qual is not None else None)

    def run_rm():
        holder["rm"] = mfeatures.read_matrix_from_batch(rbatch, 0, span, max_reads=100, device=dev)
    t = timed(run_rm, reps=2)
    rm = holder["rm"][0]
    res["read_matrix (host buffers)"] = {"reads": args.reads, "columns": int(rm.shape[0]), "rows": int(rm.shape[1]),
                                         "call_ms": t * 1e3, "reads_per_s": args.reads / t,
                                         "cells_per_s": rm.shape[0] * rm.shape[1] / t}
    if args.cpu_pileup:
        from oracle import pileup_oracle
        sub_span = span0 // 8                              # bounded sample of the same reads
        sub_recs = [r for r in recs if r["pos"] < sub_span]
        t0 = time.perf_counter()
        c2, p2 = pileup_oracle.pileup_counts(sub_recs, 0, sub_span)
        tc = time.perf_counter() - t0
        res["pileup_counts cpu restatement (python, bounded sample)"] = {
            "reads": len(sub_recs), "columns": int(len(p2)), "seconds": tc, "reads_per_s": len(sub_recs) / tc,
            "columns_per_s": len(p2) / tc}

    # ---- a8 head (partial logits -> probs + labels) runs inside a forward ----
    m = models.GRUModel(num_features=10)
    m.load_state_dict(synth.synth_state_dict(0))
    feats = synth.synth_features_fast(592, 2000, 10, seed=3)
    m.forward_arrays(feats, want_labels=True)
    m.forward_arrays(feats, want_labels=True)
    res["forward 592x2000 stage ms"] = m.last_timings()
    m.close()
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
