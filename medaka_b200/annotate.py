"""Read support of variant records: `medaka tools annotate` (medaka/vcf.py:1158-1302) on the GPU.

``annotate`` adds to every record the INFO fields of the reference's annotation, with its keys and string formats:

* ``DP`` / ``DPS``: the pileup depth at the variant's position, and that depth split by strand (fwd, rev), from the
  pileup counts of the reads that pass the read-group and mapping-quality (>= 1) filters.  The htslib depth cap the
  reference's header text mentions (~8000) is not modelled (DESIGN.md section 7).
* with ``dpsp``: ``DPSP``, the reads that span the variant +- ``pad``; every such read is trimmed to the padded window and
  aligned (affine Smith-Waterman, NUC.4.4 scores, gap open 5 / extend 3) to the padded REF and ALT haplotypes.  ``SR``
  counts the reads whose best haplotype is each allele (ref fwd, ref rev, alt1 fwd, ...), ``AR`` the reads that score
  all alleles equally (fwd, rev), ``SC`` sums the scores per allele and strand.

One BAM fetch and one ``mdk_annotate`` call per chunk of ``chunk_size`` bases of a contig: the trimming, the alignments,
their reduction and the pileup all run on the device (csrc/annotate.cu).  Every input record is annotated exactly once,
and its values do not depend on the chunking (DESIGN.md section 7 on the reference's overlapping chunks).  VCF text I/O
stays out of scope, as for the rest of the variant path.
"""
import collections
import os

import numpy as np

from medaka_b200 import bam as mbam
from medaka_b200 import libmedaka as _lm
from medaka_b200 import stitch
from medaka_b200.features import _record_args
from medaka_b200.variant import Variant

GAP_OPEN = 5
GAP_EXTEND = 3
MIN_MAPQ = 1            # features.get_trimmed_reads and CountsFeatureEncoder default (medaka/features.py:564, :816)

# NUC.4.4 (EDNAFULL), the public nucleotide matrix parasail ships as `dnafull`.  Only the A/C/G/T block (match 5,
# mismatch -4) is pinned by the reference (vcf.py:1167-1176 asserts it, test_vcf.py:711-782 and the annotated fixture
# depend on it); no reference literal exercises the ambiguity codes, so those entries are the published matrix's.
_NUC44_COLS = "ATGCSWRYKMBVHDN"
_NUC44 = """
A   5  -4  -4  -4  -4   1   1  -4  -4   1  -4  -1  -1  -1  -2
T  -4   5  -4  -4  -4   1  -4   1   1  -4  -1  -4  -1  -1  -2
G  -4  -4   5  -4   1  -4   1  -4   1  -4  -1  -1  -4  -1  -2
C  -4  -4  -4   5   1  -4  -4   1  -4   1  -1  -1  -1  -4  -2
S  -4  -4   1   1  -1  -4  -2  -2  -2  -2  -1  -1  -3  -3  -1
W   1   1  -4  -4  -4  -1  -2  -2  -2  -2  -3  -3  -1  -1  -1
R   1  -4   1  -4  -2  -2  -1  -4  -2  -2  -3  -1  -3  -1  -1
Y  -4   1  -4   1  -2  -2  -4  -1  -2  -2  -1  -3  -1  -3  -1
K  -4   1   1  -4  -2  -2  -2  -2  -1  -4  -1  -3  -3  -1  -1
M   1  -4  -4   1  -2  -2  -2  -2  -4  -1  -3  -1  -1  -3  -1
B  -4  -1  -1  -1  -1  -3  -3  -1  -1  -3  -1  -2  -2  -2  -1
V  -1  -4  -1  -1  -1  -3  -1  -3  -3  -1  -2  -1  -2  -2  -1
H  -1  -1  -4  -1  -3  -1  -3  -1  -3  -1  -2  -2  -1  -2  -1
D  -1  -1  -1  -4  -3  -1  -1  -3  -1  -3  -2  -2  -2  -1  -1
N  -2  -2  -2  -2  -1  -1  -1  -1  -1  -1  -1  -1  -1  -1  -1
"""
NT16 = "=ACMGRSVTWYHKDBN"       # htslib's 4-bit codes: the alphabet of BAM sequences


def nt16_code(ch):
    """The 4-bit code of a sequence character (either case); anything outside NT16 is N (15)."""
    i = NT16.find(ch.upper())
    return 15 if i < 0 else i


def _score_table():
    rows = {}
    for line in _NUC44.strip().splitlines():
        parts = line.split()
        rows[parts[0]] = dict(zip(_NUC44_COLS, (int(x) for x in parts[1:])))
    table = np.zeros((16, 16), dtype=np.int8)
    for a, ca in enumerate(NT16):
        for b, cb in enumerate(NT16):
            # '=' (a base equal to the reference, BAM code 0) carries no base of its own: scored as N
            table[a, b] = rows["N" if ca == "=" else ca]["N" if cb == "=" else cb]
    return table


# [16][16] substitution scores over NT16 codes (read code, haplotype code): the one table the kernel and the tests'
# CPU restatement share
SCORE_TABLE = _score_table()


def annotation_meta(pad=25):
    """The six INFO header entries of the annotation (vcf.py:1178-1202): (kind, id, number, type, description)."""
    match, mismatch = int(SCORE_TABLE[1, 1]), int(SCORE_TABLE[1, 2])
    return [
        ('INFO', 'DP', 1, 'Integer',
         'Depth of reads at position, calculated from read pileup, capped to ~8000.'),
        ('INFO', 'DPS', 2, 'Integer',
         'Depth of reads at position by strand (fwd, rev), calculated from read pileup, capped to ~8000 total.'),
        ('INFO', 'DPSP', 1, 'Integer',
         'Depth of reads spanning pos +-{}. This is not capped as in the case of DP and DPS.'.format(pad)),
        ('INFO', 'SR', '.', 'Integer',
         'Depth of spanning reads by strand which best align to each allele (ref fwd, ref rev, alt1 fwd, alt1 rev, '
         'etc.). This is not capped as in the case of DP and DPS.'),
        ('INFO', 'AR', 2, 'Integer',
         'Depth of ambiguous spanning reads by strand which align equally well to all alleles (fwd, rev). This is not '
         'capped as in the case of DP and DPS.'),
        ('INFO', 'SC', '.', 'Integer',
         'Total alignment score to each allele of spanning reads by strand (ref fwd, ref rev, alt1 fwd, alt1 rev, '
         'etc.) aligned with parasail: match {}, mismatch {}, open {}, extend {}'.format(
             match, mismatch, GAP_OPEN, GAP_EXTEND)),
    ]


def check_ref(var, ref_seq):
    """The REF check of get_padded_haplotypes (vcf.py:1315-1318)."""
    got = ref_seq[var.pos:var.pos + len(var.ref)].upper()
    if var.ref != got:
        raise ValueError('Ref sequences {} and {} differ at {}:{}, check your files.'.format(
            var.ref, got, var.chrom, var.pos))


ChunkResult = collections.namedtuple("ChunkResult", ["dp", "sr", "ar", "sc", "hap_off", "cells", "pairs", "kernel_ms"])


def annotate_chunk(batch, ref_seq, variants, pad=25, dpsp=False, device=0):
    """One ``mdk_annotate`` call: ``variants`` of one contig (sequence ``ref_seq``, REF already checked) against the
    records of ``batch`` (read-group filtered, sorted by position, covering every padded window).  Returns the raw
    integer arrays: dp [n][3] (DP, fwd, rev); sr / sc [haplotypes][2] and ar [n][2] with dpsp; hap_off [n + 1]."""
    lib, ffi = _lm.load(), _lm.ffi
    n = len(variants)
    pos = np.array([v.pos for v in variants], dtype=np.int32)
    ref_len = np.array([len(v.ref) for v in variants], dtype=np.int32)
    alleles = [[v.ref] + [a.upper() for a in v.alt] for v in variants]
    hap_off = np.zeros(n + 1, dtype=np.int64)
    np.cumsum([len(a) for a in alleles], out=hap_off[1:])
    flat = [s.encode() for a in alleles for s in a]
    allele_off = np.zeros(len(flat) + 1, dtype=np.int64)
    np.cumsum([len(s) for s in flat], out=allele_off[1:])
    allele_bytes = np.frombuffer(b"".join(flat) or b"\x00", dtype=np.uint8)
    contig_start = int(max(0, pos.min() - pad)) if n else 0
    contig_end = int(min(len(ref_seq), (pos + ref_len).max() + pad)) if n else 0
    contig = np.frombuffer(ref_seq[contig_start:contig_end].encode() or b"\x00", dtype=np.uint8)
    n_hap = int(hap_off[-1])
    dp = np.zeros((n, 3), dtype=np.int64)
    sr = np.zeros((n_hap, 2), dtype=np.int64)
    sc = np.zeros((n_hap, 2), dtype=np.int64)
    ar = np.zeros((n, 2), dtype=np.int64)
    stats = np.zeros(2, dtype=np.int64)
    ms = ffi.new("float *")
    records = _record_args(batch)

    def buf(ctype, a):
        return ffi.cast(ctype, ffi.from_buffer(a))

    _lm.check(lib.mdk_annotate(
        device, len(batch.pos), *records, buf("uint8_t *", contig), contig_start, contig_end - contig_start,
        len(ref_seq), n, buf("int32_t *", pos), buf("int32_t *", ref_len), buf("int64_t *", hap_off),
        buf("int64_t *", allele_off), buf("uint8_t *", allele_bytes), int(pad), MIN_MAPQ, 1 if dpsp else 0,
        buf("int8_t *", SCORE_TABLE), GAP_OPEN, GAP_EXTEND, buf("int64_t *", dp), buf("int64_t *", sr),
        buf("int64_t *", ar), buf("int64_t *", sc), buf("int64_t *", stats), ms))
    return ChunkResult(dp, sr, ar, sc, hap_off, int(stats[0]), int(stats[1]), float(ms[0]))


def _info(res, k, dpsp):
    """INFO values of variant k of a chunk, in the reference's string formats (vcf.py:1277-1301)."""
    info = {'DP': str(int(res.dp[k, 0])), 'DPS': '{},{}'.format(int(res.dp[k, 1]), int(res.dp[k, 2]))}
    if dpsp:
        h0, h1 = int(res.hap_off[k]), int(res.hap_off[k + 1])
        sr, sc, ar = res.sr[h0:h1], res.sc[h0:h1], res.ar[k]
        info['DPSP'] = str(int(sr.sum() + ar.sum()))
        info['SR'] = ','.join(str(int(x)) for x in sr.reshape(-1))
        info['SC'] = ','.join(str(int(x)) for x in sc.reshape(-1))
        info['AR'] = '{},{}'.format(int(ar[0]), int(ar[1]))
    return info


def annotate(variants, ref, bam, read_group=None, pad=25, dpsp=False, chunk_size=500000, device=0):
    """Annotated copies of ``variants`` (``Variant`` records, any order), in their order.

    :param ref: FASTA path, or a dict contig name -> sequence.
    :param bam: BAM path (indexed) or a ``medaka_b200.bam.BamFile``.
    :param read_group: only reads of this RG count, for the depth and the spanning reads alike.
    :param pad: flank of the padded haplotypes either side of the variant.
    :param dpsp: also DPSP, SR, AR and SC (the alignments); otherwise DP and DPS only.
    :param chunk_size: bases of a contig per BAM fetch and device call (memory, not results).
    :raises ValueError: a record's REF differs from the reference sequence.
    """
    if chunk_size < 1:
        raise ValueError("chunk_size must be positive")
    if isinstance(ref, (str, bytes, os.PathLike)):
        ref = stitch.read_fasta(ref)
    own_bam = not isinstance(bam, mbam.BamFile)
    if own_bam:
        bam = mbam.BamFile(bam)
    try:
        by_chrom = collections.OrderedDict()
        for i, v in enumerate(variants):
            by_chrom.setdefault(v.chrom, []).append(i)
        out = [None] * len(variants)
        for chrom, idx in by_chrom.items():
            if chrom not in ref:
                raise ValueError("contig {} is not in the reference".format(chrom))
            ref_seq = ref[chrom].upper()
            for i in idx:
                check_ref(variants[i], ref_seq)
            idx.sort(key=lambda i: variants[i].pos)
            first = variants[idx[0]].pos
            chunks = collections.OrderedDict()
            for i in idx:
                chunks.setdefault((variants[i].pos - first) // chunk_size, []).append(i)
            for members in chunks.values():
                vs = [variants[i] for i in members]
                lo = max(0, min(v.pos for v in vs) - pad)
                hi = min(len(ref_seq), max(v.pos + len(v.ref) for v in vs) + pad)
                batch = bam.fetch(chrom, lo, max(hi, lo + 1), read_group=read_group, min_mapq=MIN_MAPQ)
                res = annotate_chunk(batch, ref_seq, vs, pad=pad, dpsp=dpsp, device=device)
                for k, (i, v) in enumerate(zip(members, vs)):
                    info = dict(v.info)
                    info.update(_info(res, k, dpsp))
                    out[i] = Variant(v.chrom, v.pos, v.ref, alt=list(v.alt), ident=v.ident, qual=v.qual, filt=v.filt,
                                     info=info, genotype_data=v.genotype_data or None)
        return out
    finally:
        if own_bam:
            bam.close()
