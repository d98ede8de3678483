"""CPU restatement of `medaka tools annotate` (medaka/vcf.py:1158-1385).  TEST INFRASTRUCTURE ONLY.

Restates, over plain dict records (the ``oracle.pileup_oracle`` format: 'pos', 'cigar' string, 'seq', 'flag', 'mapq',
'tags'):
  * get_padded_haplotypes  vcf.py:1305-1327
  * trim_read              src/medaka_trimbam.c:101-246 with partial = false, base by base as the C walks the CIGAR,
                           and the keep rules of retrieve_trimmed_reads (:320-348: qstart, qend >= 0, qend - qstart > 1,
                           the forward-strand query [qstart, qend)); reads filtered like src/medaka_bamiter.c:17-45 with
                           min_mapq = 1 and the read group (features.get_trimmed_reads, medaka/features.py:561-565)
  * sw_scores              parasail sw_trace_striped_32's score: local alignment, a gap of length k costs
                           open + (k - 1) extend.  numpy, row by row over a batch of alignments, with the horizontal
                           gap state as a running maximum (exact for open >= extend).  Not parasail (not installed).
  * align_reads_to_haps    vcf.py:1356-1385
  * annotate               vcf.py:1243-1301: DP / DPS from oracle.pileup_oracle's counts at the variant's major column
                           (normalise='fwd_rev' index groups), the rest from the above.
The substitution scores are medaka_b200.annotate.SCORE_TABLE, the table the kernel takes.
"""
import collections
import re
import struct

import numpy as np

from medaka_b200 import bam as mbam
from medaka_b200.annotate import GAP_EXTEND, GAP_OPEN, SCORE_TABLE, check_ref, nt16_code
from oracle import pileup_oracle

_CIGAR_RE = re.compile(r"(\d+)([MIDNSHP=X])")
_NEG = -(1 << 28)


def read_bam(path):
    """(references [(name, length)], records) of a BAM file, by a plain parse of the inflated stream (SAM spec 4.2)."""
    with open(path, "rb") as fh:
        data = mbam.bgzf_decompress(fh.read(), threads=1)
    assert data[:4] == b"BAM\x01"
    l_text = struct.unpack_from("<i", data, 4)[0]
    off = 8 + l_text
    n_ref = struct.unpack_from("<i", data, off)[0]
    off += 4
    refs = []
    for _ in range(n_ref):
        l_name = struct.unpack_from("<i", data, off)[0]
        name = data[off + 4:off + 4 + l_name - 1].decode()
        refs.append((name, struct.unpack_from("<i", data, off + 4 + l_name)[0]))
        off += 8 + l_name
    records = []
    while off < len(data):
        block = struct.unpack_from("<i", data, off)[0]
        (tid, pos, l_rn, mapq, _bin, n_cig, flag, l_seq, _nt, _np, _tl) = struct.unpack_from("<iiBBHHHiiii", data, off + 4)
        p = off + 36
        name = data[p:p + l_rn - 1].decode()
        p += l_rn
        ops = struct.unpack_from("<%dI" % n_cig, data, p)
        p += 4 * n_cig
        packed = data[p:p + (l_seq + 1) // 2]
        p += (l_seq + 1) // 2 + l_seq
        seq = "".join(mbam_nt16(packed, i) for i in range(l_seq))
        tags = mbam._parse_tags(data[p:off + 4 + block])
        records.append(dict(ref=refs[tid][0] if tid >= 0 else None, pos=pos, query_name=name, mapq=mapq, flag=flag,
                            cigar="".join("%d%s" % (o >> 4, "MIDNSHP=X"[o & 15]) for o in ops), seq=seq, tags=tags))
        off += 4 + block
    return refs, records


def mbam_nt16(packed, i):
    b = packed[i >> 1]
    return "=ACMGRSVTWYHKDBN"[(b >> 4) if i % 2 == 0 else (b & 15)]


def get_padded_haplotypes(var, ref_seq, pad):
    """vcf.py:1305-1327: ((padded ref, padded alt 1, ...), (start, end)); ValueError when REF disagrees."""
    check_ref(var, ref_seq)
    left_start = max(0, var.pos - pad)
    right_start = var.pos + len(var.ref)
    right_end = min(len(ref_seq), right_start + pad)
    pad_left, pad_right = ref_seq[left_start:var.pos], ref_seq[right_start:right_end]
    return tuple(pad_left + h + pad_right for h in [var.ref] + list(var.alt)), (left_start, right_end)


def trim_read(rec, rstart, rend):
    """trim_read (src/medaka_trimbam.c:101-246), partial = false: (qstart, qend) or None."""
    if rec["pos"] > rstart:
        return None
    qstart = qend = -1
    found_start = found_end = False
    read_pos, ref_pos = 0, rec["pos"]
    for n, op in _CIGAR_RE.findall(rec["cigar"]):
        aligned, read_inc, ref_inc = False, 0, 0
        if op in "M=X":
            aligned, read_inc, ref_inc = True, 1, 1
        elif op == "D":
            ref_inc = 1
        elif op in "IS":
            read_inc = 1
        elif op == "H":
            pass
        else:                       # N and P: "Unhandled cigar op"
            return None
        if found_start and found_end:
            continue                # the rest of the walk only checks the operations
        for _ in range(int(n)):
            if aligned:
                if not found_start:
                    if ref_pos == rstart:
                        qstart, found_start = read_pos, True
                    elif ref_pos > rstart:
                        qstart, found_start = read_pos - 1, True
                if not found_end:
                    if ref_pos == rend:
                        qend, found_end = read_pos, True
                    elif ref_pos > rend:
                        qend, found_end = read_pos - 1, True
            read_pos += read_inc
            ref_pos += ref_inc
    if qstart < 0 or qend < 0:
        return None
    return qstart, qend


def get_trimmed_reads(records, region, read_group=None, min_mapq=1):
    """[(is_rev, trimmed forward-strand sequence)] of the records spanning region = (start, end), in record order."""
    out = []
    for rec in records:
        if not pileup_oracle.read_passes(rec, min_mapq=min_mapq, read_group=read_group):
            continue
        t = trim_read(rec, region[0], region[1])
        if t is None or t[1] - t[0] <= 1:
            continue
        out.append((bool(rec.get("flag", 0) & 16), rec["seq"][t[0]:t[1]]))
    return out


def sw_scores(pairs, go=GAP_OPEN, ge=GAP_EXTEND, table=SCORE_TABLE, cells_per_batch=1 << 21):
    """Local-alignment scores of (read, haplotype) string pairs, int64 [len(pairs)]."""
    out = np.zeros(len(pairs), dtype=np.int64)
    order = sorted(range(len(pairs)), key=lambda k: (len(pairs[k][1]), len(pairs[k][0])))
    tab = np.asarray(table, dtype=np.int32)
    k = 0
    while k < len(order):
        n_max = len(pairs[order[k]][1])
        group = []
        while k < len(order) and (len(group) + 1) * max(n_max, len(pairs[order[k]][1])) <= max(cells_per_batch, n_max):
            n_max = max(n_max, len(pairs[order[k]][1]))
            group.append(order[k])
            k += 1
        reads = [pairs[g][0] for g in group]
        haps = [pairs[g][1] for g in group]
        B, M, N = len(group), max(len(r) for r in reads), max(len(h) for h in haps)
        a = np.full((B, M), 15, dtype=np.int64)
        b = np.full((B, N), 15, dtype=np.int64)
        for x, (r, h) in enumerate(zip(reads, haps)):
            a[x, :len(r)] = [nt16_code(c) for c in r]
            b[x, :len(h)] = [nt16_code(c) for c in h]
        m_len = np.array([len(r) for r in reads])
        col_ok = np.arange(N)[None, :] < np.array([len(h) for h in haps])[:, None]
        ramp = ge * np.arange(N, dtype=np.int64)
        h_prev = np.zeros((B, N + 1), dtype=np.int64)       # H of the row above, column -1 first
        f_prev = np.full((B, N), _NEG, dtype=np.int64)
        best = np.zeros(B, dtype=np.int64)
        for i in range(M):
            diag = h_prev[:, :-1] + tab[a[:, i][:, None], b]
            f = np.maximum(f_prev - ge, h_prev[:, 1:] - go)
            base = np.maximum(np.maximum(diag, f), 0)
            # E[j] = max(E[j-1] - ge, H[j-1] - go) = max over k < j of base[k] - go - ge (j - 1 - k), since go >= ge
            run = np.maximum.accumulate(base + ramp, axis=1)
            e = np.full((B, N), _NEG, dtype=np.int64)
            e[:, 1:] = run[:, :-1] - go - ramp[:-1][None, :]
            h = np.maximum(base, e)
            ok = col_ok & (i < m_len)[:, None]
            best = np.maximum(best, np.where(ok, h, 0).max(axis=1))
            h_prev[:, 1:] = h
            f_prev = f
        out[group] = best
    return out


def align_read_to_haps(read, haps, go=GAP_OPEN, ge=GAP_EXTEND):
    """vcf.py:1388-1403."""
    return [int(s) for s in sw_scores([(read, h) for h in haps], go, ge)]


def align_reads_to_haps(reads, haps, go=GAP_OPEN, ge=GAP_EXTEND):
    """vcf.py:1356-1385 over [(is_rev, seq)]: (Counter (is_rev, best hap or None), Counter (is_rev, hap) of scores)."""
    scores = sw_scores([(seq, h) for _, seq in reads for h in haps], go, ge).reshape(len(reads), len(haps))
    hap_counts, total = collections.Counter(), collections.Counter()
    for (is_rev, _), row in zip(reads, scores):
        best = None if len(set(row.tolist())) == 1 else int(np.argmax(row))
        hap_counts[(is_rev, best)] += 1
        for h, s in enumerate(row):
            total[(is_rev, h)] += int(s)
    return hap_counts, total


def annotate(variants, ref, records, read_group=None, pad=25, dpsp=False):
    """INFO dicts (string values, the reference's formats) of ``variants`` (medaka_b200.variant.Variant), in order.
    ``ref``: dict contig -> sequence; ``records``: dict records with 'ref' naming their contig."""
    by_chrom = collections.defaultdict(list)
    for rec in records:
        by_chrom[rec.get("ref")].append(rec)
    depth = {}
    for chrom in set(v.chrom for v in variants):
        ps = [v.pos for v in variants if v.chrom == chrom]
        counts, positions = pileup_oracle.pileup_counts(by_chrom[chrom], min(ps), max(ps) + 1, min_mapq=1,
                                                        read_group=read_group)
        for row, (major, minor) in zip(counts, positions):
            if minor == 0:
                rev = int(row[[0, 1, 2, 3, 8]].sum())
                fwd = int(row[[4, 5, 6, 7, 9]].sum())
                depth[chrom, int(major)] = (fwd, rev)
    # a read can only span [start, end) when it starts at or before start and its reference end passes end: the records
    # of a window are looked up among those (in record order), the rules above decide
    ends = {c: [r["pos"] + sum(int(n) for n, op in _CIGAR_RE.findall(r["cigar"]) if op in "MDN=X") for r in recs]
            for c, recs in by_chrom.items()}
    out = []
    for v in variants:
        ref_seq = ref[v.chrom].upper()
        fwd, rev = depth.get((v.chrom, v.pos), (0, 0))
        info = {'DP': str(fwd + rev), 'DPS': '{},{}'.format(fwd, rev)}
        if dpsp:
            haps, region = get_padded_haplotypes(v, ref_seq, pad)
            haps = tuple(h.upper() for h in haps)
            recs = [r for r, e in zip(by_chrom[v.chrom], ends[v.chrom]) if r["pos"] <= region[0] and e > region[1]]
            reads = get_trimmed_reads(recs, region, read_group=read_group)
            counts, scores = align_reads_to_haps(reads, haps)
            info['DPSP'] = str(sum(counts.values()))
            sr, sc = [], []
            for hap in range(len(haps)):
                for is_rev in (False, True):
                    sr.append(counts[(is_rev, hap)])
                    sc.append(scores[(is_rev, hap)])
            info['SR'] = ','.join(map(str, sr))
            info['SC'] = ','.join(map(str, sc))
            info['AR'] = '{},{}'.format(*[counts[(is_rev, None)] for is_rev in (False, True)])
        out.append(info)
    return out


def parse_info(text):
    """'K=V;K=V' -> dict of strings (how the reference's VCFReader holds INFO)."""
    return dict(kv.split('=', 1) for kv in text.split(';') if kv)
