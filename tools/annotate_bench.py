#!/usr/bin/env python
"""Variant annotation with spanning reads (`annotate(..., dpsp=True)`) on a seeded synthetic contig and BAM:

    python tools/annotate_bench.py [--variants 20000] [--depth 200] [--read-len 1000] [--repeats 3] [--cpu-variants 40]

Variants every --spacing bases (60 % SNVs, 15 % insertions and 15 % deletions of 1-50 bases, 10 % two-ALT records);
reads are copies of the contig with 2 % substitutions, on both strands, --depth deep; pad 25.  The BAM is written
into a temporary directory (numpy + zlib, with no index, so each chunk's fetch streams the file).

Per run one JSON line:
  device       mdk_annotate over the whole contig as one chunk, records already in host memory: CUDA-event time of the
               call's kernels (pileup, trimming, alignments, reductions), variants / s and alignment cells / s
               (cells = trimmed read length x haplotype length, summed over every read-haplotype pair);
  end_to_end   `annotate` from the BAM path: fetch, inflate, staging, kernels and the INFO strings, wall clock;
  cpu          the tests' numpy restatement (tests/annotate_oracle.py, NOT parasail, which is not installed) on the
               first --cpu-variants variants, variants / s, and whether its INFO equals the GPU's on them;
and the GPU's name, power limit and maximum SM clock (read-only nvidia-smi query).
"""
import argparse
import json
import os
import struct
import subprocess
import sys
import tempfile
import time
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

NT = np.frombuffer(b"=ACMGRSVTWYHKDBN", dtype=np.uint8)


def gpu_card():
    """(name, power limit, max SM clock) of GPU 0 as nvidia-smi reports them (a read-only query), or Nones."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                              "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
        return tuple(x.strip() for x in out.split(",")[:3])
    except Exception:
        return None, None, None


def synth(n_var, depth, read_len, spacing, seed):
    rng = np.random.default_rng(seed)
    length = n_var * spacing + 4000
    contig = np.frombuffer(b"ACGT", dtype=np.uint8)[rng.integers(0, 4, length)]
    n_reads = depth * length // read_len
    pos = np.sort(rng.integers(0, length - read_len // 2, n_reads)).astype(np.int32)
    lens = np.minimum(rng.integers(read_len * 7 // 10, read_len * 13 // 10, n_reads), length - pos).astype(np.int32)
    flag = np.where(rng.random(n_reads) < 0.5, 16, 0).astype(np.uint16)
    var_pos = (np.arange(n_var) * spacing + 2000 + rng.integers(0, spacing // 2, n_var)).astype(np.int64)
    kinds = rng.random(n_var)
    variants = []
    from medaka_b200.variant import Variant
    text = contig.tobytes().decode()
    for p, k in zip(var_pos.tolist(), kinds.tolist()):
        base = text[p]
        if k < 0.6:
            variants.append(Variant("ctg", p, base, alt=["ACGT"[("ACGT".index(base) + 1) % 4]]))
        elif k < 0.75:
            ins = "".join("ACGT"[x] for x in rng.integers(0, 4, rng.integers(1, 51)))
            variants.append(Variant("ctg", p, base, alt=[base + ins]))
        elif k < 0.9:
            variants.append(Variant("ctg", p, text[p:p + int(rng.integers(2, 52))], alt=[base]))
        else:
            variants.append(Variant("ctg", p, base, alt=["ACGT"[("ACGT".index(base) + 1) % 4], base + "A"]))
    return text, pos, lens, flag, variants, rng


def write_bam(path, contig, pos, lens, flag, rng, block=60000):
    """Single-M records (contig copies with 2 % substitutions) as a BAM stream, BGZF members of `block` bytes."""
    chunks = [b"BAM\x01" + struct.pack("<ii", 0, 1) + struct.pack("<i", 4) + b"ctg\x00" + struct.pack("<i", len(contig))]
    cbytes = np.frombuffer(contig.encode(), dtype=np.uint8)
    code = np.zeros(256, dtype=np.uint8)
    code[NT] = np.arange(16, dtype=np.uint8)
    for i in range(len(pos)):
        p, n = int(pos[i]), int(lens[i])
        s = code[cbytes[p:p + n]].copy()
        err = rng.random(n) < 0.02
        s[err] = np.array([1, 2, 4, 8], dtype=np.uint8)[rng.integers(0, 4, int(err.sum()))]
        if n % 2:
            s = np.append(s, 0)
        packed = ((s[0::2] << 4) | s[1::2]).astype(np.uint8).tobytes()
        name = b"r%d\x00" % i
        body = struct.pack("<iiBBHHHiiii", 0, p, len(name), 60, 4680, 1, int(flag[i]), n, -1, -1, 0)
        body += name + struct.pack("<I", (n << 4) | 0) + packed + b"\xff" * n
        chunks.append(struct.pack("<i", len(body)) + body)
    stream = b"".join(chunks)
    out = bytearray()
    for u in range(0, len(stream), block):
        data = stream[u:u + block]
        co = zlib.compressobj(6, zlib.DEFLATED, -15)
        comp = co.compress(data) + co.flush()
        out += (b"\x1f\x8b\x08\x04\x00\x00\x00\x00\x00\xff\x06\x00BC\x02\x00" + struct.pack("<H", len(comp) + 25) + comp +
                struct.pack("<II", zlib.crc32(data) & 0xffffffff, len(data)))
    out += b"\x1f\x8b\x08\x04\x00\x00\x00\x00\x00\xff\x06\x00BC\x02\x00\x1b\x00\x03\x00\x00\x00\x00\x00\x00\x00\x00\x00"
    with open(path, "wb") as fh:
        fh.write(bytes(out))


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--variants", type=int, default=20000)
    ap.add_argument("--depth", type=int, default=200)
    ap.add_argument("--read-len", type=int, default=1000)
    ap.add_argument("--spacing", type=int, default=100)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--cpu-variants", type=int, default=40)
    ap.add_argument("--seed", type=int, default=1)
    args = ap.parse_args()

    from medaka_b200 import annotate as mann
    from medaka_b200 import bam as mbam
    from medaka_b200 import libmedaka
    libmedaka.require_gpu(0)
    card = gpu_card()
    contig, pos, lens, flag, variants, rng = synth(args.variants, args.depth, args.read_len, args.spacing, args.seed)
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "synth.bam")
        t0 = time.perf_counter()
        write_bam(path, contig, pos, lens, flag, rng)
        build_s = time.perf_counter() - t0
        ref = {"ctg": contig}
        with mbam.BamFile(path) as fh:
            batch = fh.fetch("ctg", 0, len(contig), min_mapq=mann.MIN_MAPQ)
        mann.annotate_chunk(batch, contig, variants, pad=25, dpsp=True)           # warm-up
        dev = [mann.annotate_chunk(batch, contig, variants, pad=25, dpsp=True) for _ in range(args.repeats)]
        mann.annotate(variants[:100], ref, path, pad=25, dpsp=True)               # warm-up
        e2e, got = [], None
        for _ in range(args.repeats):
            t0 = time.perf_counter()
            got = mann.annotate(variants, ref, path, pad=25, dpsp=True)
            e2e.append(time.perf_counter() - t0)

        # CPU arm: the numpy restatement on the first variants, over the records that reach their windows
        from tests import annotate_oracle as ao
        sub = variants[:args.cpu_variants]
        hi = max(v.pos + len(v.ref) for v in sub) + 25
        keep = np.flatnonzero(pos < hi)
        recs = []
        for i in keep.tolist():
            s0, s1 = int(batch.seq_off[i]), int(batch.seq_off[i + 1])
            nib = np.empty(2 * (s1 - s0), dtype=np.uint8)
            nib[0::2], nib[1::2] = batch.seq[s0:s1] >> 4, batch.seq[s0:s1] & 15
            recs.append(dict(ref="ctg", pos=int(batch.pos[i]), cigar="%dM" % int(batch.l_seq[i]), flag=int(batch.flag[i]),
                             mapq=int(batch.mapq[i]), tags={}, seq=NT[nib[:int(batch.l_seq[i])]].tobytes().decode()))
        t0 = time.perf_counter()
        want = ao.annotate(sub, ref, recs, pad=25, dpsp=True)
        cpu_s = time.perf_counter() - t0

    ms = sorted(r.kernel_ms for r in dev)
    e2e.sort()
    res = dev[0]
    print(json.dumps({
        "workload": "annotate dpsp", "variants": len(variants), "depth": args.depth, "read_len": args.read_len,
        "reads": int(len(pos)), "pairs": res.pairs, "cells": res.cells,
        "device": {"kernel_ms": [round(x, 3) for x in ms], "variants_per_s": round(len(variants) / (ms[len(ms) // 2] / 1e3)),
                   "cells_per_s": float("%.4g" % (res.cells / (ms[len(ms) // 2] / 1e3)))},
        "end_to_end": {"seconds": [round(x, 3) for x in e2e],
                       "variants_per_s": round(len(variants) / e2e[len(e2e) // 2])},
        "cpu_numpy_restatement": {"variants": len(sub), "seconds": round(cpu_s, 3),
                                  "variants_per_s": round(len(sub) / cpu_s, 2),
                                  "matches_gpu": [g.info for g in got[:len(sub)]] == want},
        "repeat_identical": all(np.array_equal(r.sc, res.sc) and np.array_equal(r.sr, res.sr) for r in dev),
        "bam_build_s": round(build_s, 1), "gpu": card[0], "power_limit": card[1], "max_sm_clock": card[2]}))


if __name__ == "__main__":
    main()
