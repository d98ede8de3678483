"""Throughput of `medaka features` (create_samples) with and without truth labels, and of the label kernels.

A synthetic draft of --mb Mb, reads from oracle.synth.synth_reads at depth ~--depth, and one truth alignment per 1 Mb
region with ~1 % edits (mismatches, insertions, deletions; MD tags) are written as indexed BAMs under a temporary
directory.  Reported, one JSON line each, with the card's name and power limit read in the same call:
  * create_samples positions/s (draft positions over wall time, store writes included) without and with --truth;
  * mdk_truth_labels over the columns of one 1 Mb region: the call (host copies in and out) by a host clock around it,
    and the device time of its kernels (truth_*) from torch.profiler;
  * the oracle's labelling rate (pair loop + dictionary join, oracle/truth_oracle.py) on a --oracle-kb slice.
    python tools/features_bench.py [--mb 10] [--depth 30] [--steps 5] [--out DIR]
"""
import argparse
import bisect
import json
import os
import shutil
import struct
import subprocess
import sys
import tempfile
import time
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import bamutil  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True)
    except OSError:
        return "unknown"
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def member(data):
    """One BGZF member (bamutil._member at zlib level 1: the reads BAM is hundreds of MB)."""
    co = zlib.compressobj(1, zlib.DEFLATED, -15)
    comp = co.compress(data) + co.flush()
    return (b"\x1f\x8b\x08\x04\x00\x00\x00\x00\x00\xff\x06\x00BC\x02\x00" + struct.pack("<H", len(comp) + 25) + comp +
            struct.pack("<II", zlib.crc32(data) & 0xffffffff, len(data)))


def write_bam(path, refs, records, member_size=65280):
    """bamutil.write_bam for many records: 64 KiB members and a bisect for the index's virtual offsets."""
    header = b"BAM\x01" + struct.pack("<i", 0) + struct.pack("<i", len(refs))
    for name, length in refs:
        header += struct.pack("<i", len(name) + 1) + name.encode() + b"\x00" + struct.pack("<i", length)
    parts, rec_u, spans, u = [header], [], [], len(header)
    for rec in records:
        enc, ref_len = bamutil.encode_record(rec, rec["ref"])
        rec_u.append(u)
        spans.append(ref_len)
        parts.append(enc)
        u += len(enc)
    stream = b"".join(parts)
    out, f_starts, u_starts = bytearray(), [], []
    for u0 in range(0, len(stream), member_size):
        f_starts.append(len(out))
        u_starts.append(u0)
        out += member(stream[u0:u0 + member_size])
    out += member(b"")
    with open(path, "wb") as fh:
        fh.write(out)

    def voff(upos):
        k = bisect.bisect_right(u_starts, upos) - 1
        return (f_starts[k] << 16) | (upos - u_starts[k])
    bai = b"BAI\x01" + struct.pack("<i", len(refs))
    for tid in range(len(refs)):
        bins, linear = {}, {}
        for i, rec in enumerate(records):
            if rec["ref"] != tid:
                continue
            beg, end = rec["pos"], rec["pos"] + max(spans[i], 1)
            v0 = voff(rec_u[i])
            v1 = voff(rec_u[i + 1]) if i + 1 < len(records) else (len(out) - 28) << 16
            bins.setdefault(bamutil.reg2bin(beg, end), []).append((v0, v1))
            for w in range(beg >> 14, ((end - 1) >> 14) + 1):
                if w not in linear:
                    linear[w] = v0
        bai += struct.pack("<i", len(bins))
        for b, chunks in sorted(bins.items()):
            bai += struct.pack("<Ii", b, len(chunks)) + b"".join(
                struct.pack("<QQ", a, e) for a, e in chunks)
        n_intv = (max(linear) + 1) if linear else 0
        bai += struct.pack("<i", n_intv)
        last = 0
        for w in range(n_intv):
            last = linear.get(w, last)
            bai += struct.pack("<Q", last)
    with open(path + ".bai", "wb") as fh:
        fh.write(bai)


def truth_record(draft, start, end, rs, p_edit=0.01):
    """A truth over draft[start:end) with ~p_edit edits (a third each mismatches, insertions, deletions) and its MD."""
    ops, seq, md, run, p = [], [], [], 0, start

    def push(op, n=1):
        if ops and ops[-1][1] == op:
            ops[-1][0] += n
        else:
            ops.append([n, op])
    u = rs.uniform(size=end - start + 1)
    i = 0
    while p < end:
        x = u[i % len(u)]
        i += 1
        if x < p_edit / 3 and ops and ops[-1][1] == "M":
            push("I")
            seq.append("ACGT"[int(x * 1e6) % 4])
            continue
        if x < 2 * p_edit / 3 and ops and ops[-1][1] == "M" and p < end - 5:
            n = 1 + int(x * 1e6) % 3
            push("D", n)
            md.append("%d^%s" % (run, draft[p:p + n]))
            run, p = 0, p + n
            continue
        push("M")
        if x < p_edit:
            seq.append("ACGT".replace(draft[p], "")[int(x * 1e6) % 3])
            md.append("%d%s" % (run, draft[p]))
            run = 0
        else:
            seq.append(draft[p])
            run += 1
        p += 1
    md.append(str(run))
    return dict(query_name="truth_%d" % start, pos=start, cigar="".join("%d%s" % (n, op) for n, op in ops),
                seq="".join(seq), flag=0, mapq=60, tags={"MD": "".join(md)}, ref=0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mb", type=int, default=10)
    ap.add_argument("--depth", type=float, default=30)
    ap.add_argument("--mean-len", type=int, default=5000)
    ap.add_argument("--steps", type=int, default=5, help="timed calls of the label kernels")
    ap.add_argument("--oracle-kb", type=int, default=50)
    ap.add_argument("--out", default=None, help="directory for the profiler trace (default: none written)")
    args = ap.parse_args()

    from medaka_b200 import common, features, labels
    from oracle import synth, truth_oracle
    info = card()
    L = args.mb * 1000000
    rs = np.random.RandomState(0)
    draft = "".join("ACGT"[k] for k in rs.randint(0, 4, L))
    tmp = tempfile.mkdtemp(prefix="features_bench_")
    t0 = time.perf_counter()
    n_reads = int(args.depth * L / args.mean_len)
    reads = synth.synth_reads(n_reads, L, seed=1, mean_len=args.mean_len)
    truths = [truth_record(draft, s + 500, min(s + 1000000, L) - 500, rs) for s in range(0, L, 1000000)]
    rpath, tpath = os.path.join(tmp, "reads.bam"), os.path.join(tmp, "truth.bam")
    write_bam(rpath, [("ctg", L)], [dict(r, ref=0) for r in reads])
    write_bam(tpath, [("ctg", L)], truths)
    print(json.dumps({"setup_s": round(time.perf_counter() - t0, 1), "reads": n_reads, "draft_mb": args.mb,
                      "card": info}), flush=True)

    # warm-up: library load, device context, cached device buffers
    features.create_samples(rpath, os.path.join(tmp, "warm.npzstore"), regions=["ctg:0-200000"], truth=tpath)
    for label, truth in (("create_samples", None), ("create_samples_truth", tpath)):
        out = os.path.join(tmp, label + ".npzstore")
        t0 = time.perf_counter()
        n = features.create_samples(rpath, out, truth=truth)
        dt = time.perf_counter() - t0
        print(json.dumps({"measure": label, "draft_positions": L, "samples": n, "wall_s": round(dt, 3),
                          "positions_per_s": round(L / dt), "card": info}), flush=True)

    # the label kernels over the columns of one 1 Mb region
    region = common.Region("ctg", 1000000, 2000000)
    (aln,), = labels.TruthAlignment.bam_to_alignments(tpath, region)
    enc = features.CountsFeatureEncoder()
    pos = np.concatenate([s.positions for s in enc.bam_to_sample(rpath, common.Region("ctg", aln.start, aln.end))])
    labels.truth_labels(aln, pos)
    t0 = time.perf_counter()
    for _ in range(args.steps):
        got = labels.truth_labels(aln, pos)
    call_ms = (time.perf_counter() - t0) / args.steps * 1e3
    kernel_ms = None
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            labels.truth_labels(aln, pos)
        torch.cuda.synchronize()
    ev = [e for e in prof.key_averages() if "truth_" in e.key and "kernel" in e.key]
    if ev:
        kernel_ms = sum(e.device_time_total for e in ev) / args.steps / 1e3
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        prof.export_chrome_trace(os.path.join(args.out, "truth_labels_trace.json"))
    print(json.dumps({"measure": "truth_labels_1mb", "columns": len(pos), "cigar_ops": len(aln.aln.cigar),
                      "call_ms": round(call_ms, 3), "kernels_ms": None if kernel_ms is None else round(kernel_ms, 4),
                      "columns_per_s_kernels": None if not kernel_ms else round(len(pos) / kernel_ms * 1e3),
                      "non_gap_labels": int((got != 0).sum()), "card": info}), flush=True)

    # the oracle's labelling rate on a slice of the same region
    d = dict(pos=aln.aln.reference_start, seq=aln.aln.query_sequence, flag=0, tags=aln.aln.tags,
             cigar="".join("%d%s" % (int(c) >> 4, "MIDNSHP=X"[int(c) & 15]) for c in aln.aln.cigar))
    t = truth_oracle.Truth(d)
    t.start, t.end = aln.start, aln.start + args.oracle_kb * 1000
    sl = pos[(pos["major"] >= t.start) & (pos["major"] < t.end)]
    t0 = time.perf_counter()
    want = truth_oracle.join_labels(t, sl)
    dt = time.perf_counter() - t0
    assert np.array_equal(want, got[(pos["major"] >= t.start) & (pos["major"] < t.end)])
    print(json.dumps({"measure": "oracle_labels_cpu", "columns": len(sl), "wall_s": round(dt, 3),
                      "columns_per_s": round(len(sl) / dt)}), flush=True)
    shutil.rmtree(tmp)


if __name__ == "__main__":
    main()
