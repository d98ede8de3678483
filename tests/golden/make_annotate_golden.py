"""Annotation fixture: the reference's real amplicon BAM and its expected annotation, checked against the CPU restatement.

`python tests/golden/make_annotate_golden.py [--copy-from <medaka checkout>]`

With --copy-from, copies medaka/test/data/test_annotate.{bam,bam.bai,vcf} and test_annotate_ref.fasta (data only) into
tests/golden/annotate/.  Then, always, asserts that tests/annotate_oracle.py reproduces the reference's literals:
  * medaka/test/test_vcf.py:796-808: the full INFO (DP, DPS, DPSP, SR, AR, SC) of all six records, the three of
    MN908947.3 and their copies on the "Duplicate" contig, with RG nCoV-2019_2 and pad 25;
  * test_vcf.py:656-687: get_padded_haplotypes, including the REF mismatch;
  * test_vcf.py:711-721: scores of one read against four haplotypes, from match / mismatch / open / extend;
  * test_vcf.py:723-782: best-haplotype counts of four reads against two and three haplotypes.  The reference computes
    the expected scores of that case with parasail at test time; here they are the restatement's own values (SCORES).
"""
import argparse
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

DATA = os.path.join(HERE, "annotate")
FILES = ("test_annotate.bam", "test_annotate.bam.bai", "test_annotate.vcf", "test_annotate_ref.fasta")
READ_GROUP = "nCoV-2019_2"
PAD = 25

# test_vcf.py:796-808 (0-based positions, as the reference's Variant holds them)
EXPECTED = [
    ('MN908947.3', 29748, 'ACGATCGAGTG', 'A',
     'AR=0,0;DP=200;DPS=100,100;DPSP=199;SC=19484,20327,22036,23215;SR=1,2,98,98'),
    ('MN908947.3', 29764, 'TGAACAATGCT', 'A',
     'AR=0,0;DP=200;DPS=100,100;DPSP=199;SC=19970,21140,15773,16751;SR=99,100,0,0'),
    ('MN908947.3', 29788, 'TATATGGAAGA', 'A',
     'AR=0,0;DP=199;DPS=99,100;DPSP=197;SC=26174,28129,19085,20315;SR=96,100,1,0'),
]
EXPECTED = EXPECTED + [('Duplicate',) + e[1:] for e in EXPECTED]

# test_vcf.py:656-680: ((pos, ref, alt), pad, padded ref, padded alt, start, end) on 'ATGCTACTGC'
PADDED_REF = 'ATGCTACTGC'
PADDED_CASES = [
    ((4, 'T', 'G'), 2, 'GCTAC', 'GCGAC', 2, 7),
    ((4, 'T', 'TA'), 2, 'GCTAC', 'GCTAAC', 2, 7),
    ((4, 'T', 'GA'), 2, 'GCTAC', 'GCGAAC', 2, 7),
    ((4, 'TA', 'T'), 2, 'GCTACT', 'GCTCT', 2, 8),
    ((4, 'TA', 'G'), 2, 'GCTACT', 'GCGCT', 2, 8),
    ((0, 'A', 'G'), 2, 'ATG', 'GTG', 0, 3),
    ((0, 'A', 'AG'), 2, 'ATG', 'AGTG', 0, 3),
    ((0, 'AT', 'T'), 2, 'ATGC', 'TGC', 0, 4),
    ((9, 'C', 'G'), 2, 'TGC', 'TGG', 7, 10),
    ((9, 'C', 'CG'), 2, 'TGC', 'TGCG', 7, 10),
    ((8, 'GC', 'G'), 2, 'CTGC', 'CTG', 6, 10),
]

# test_vcf.py:711-717 with match 5, mismatch -4, open 5, extend 3
ALIGN_READ = 'ATGCTTTTTGCTAC'
ALIGN_HAPS = [('ATGCTTTTTGCTAC', 14 * 5), ('ATGCTTaTTGCTAC', 13 * 5 - 4), ('ATGCTTTT*GCTAC', 13 * 5 - 5),
              ('ATGCTTT**GCTAC', 12 * 5 - 5 - 3)]

# test_vcf.py:727-782
HAPS3 = ['ATGCTTTTT*GCTAC', 'ATGCTTaTT*GCTAC', 'ATGCTTTTTTGCTAC']
READS4 = ['AaGCTTTTT*GCcAC', 'ATcCTTaTT*GCTgC', 'ATGgTTTTTTGCcAC', 'ATGCTTgTT*GCTAC']
BEST_OF_TWO = [0, 1, 0, None]
BEST_OF_THREE = {0: 2, 1: 1, 2: 1}
# scores of READS4 against HAPS3[:2] (parasail at the reference's test time; the restatement's values here)
SCORES = [[52, 43], [43, 52], [47, 38], [61, 61]]


def strip(s):
    return s.upper().replace('*', '')


def read_vcf(path):
    """The data lines of a VCF as medaka_b200.variant.Variant (0-based pos, INFO as a dict of strings)."""
    from medaka_b200.variant import Variant
    from tests.annotate_oracle import parse_info
    out = []
    with open(path) as fh:
        for line in fh:
            if line.startswith('#') or not line.strip():
                continue
            f = line.rstrip('\n').split('\t')
            gd = dict(zip(f[8].split(':'), f[9].split(':'))) if len(f) > 9 else None
            out.append(Variant(f[0], int(f[1]) - 1, f[3], alt=f[4], ident=f[2], qual=f[5], filt=f[6],
                               info=parse_info(f[7]) if f[7] not in ('', '.') else {}, genotype_data=gd))
    return out


def expected_info():
    from tests.annotate_oracle import parse_info
    return [parse_info(e[4]) for e in EXPECTED]


def check():
    from medaka_b200 import stitch
    from medaka_b200.variant import Variant
    from tests import annotate_oracle as ao

    variants = read_vcf(os.path.join(DATA, "test_annotate.vcf"))
    assert [(v.chrom, v.pos, v.ref, v.alt) for v in variants] == [e[:3] + ([e[3]],) for e in EXPECTED]
    ref = stitch.read_fasta(os.path.join(DATA, "test_annotate_ref.fasta"))
    _, records = ao.read_bam(os.path.join(DATA, "test_annotate.bam"))
    got = ao.annotate(variants, ref, records, read_group=READ_GROUP, pad=PAD, dpsp=True)
    assert got == expected_info(), got

    for (pos, r, a), pad, pref, palt, start, end in PADDED_CASES:
        haps, region = ao.get_padded_haplotypes(Variant('my_chrom', pos, r, alt=a), PADDED_REF, pad)
        assert (haps[0], haps[1], region) == (pref, palt, (start, end)), (pos, r, a)
    try:
        ao.get_padded_haplotypes(Variant('my_chrom', 2, 'GT', alt='G'), PADDED_REF, 2)
        raise AssertionError("REF mismatch not detected")
    except ValueError:
        pass

    assert ao.align_read_to_haps(ALIGN_READ, [strip(h) for h, _ in ALIGN_HAPS]) == [s for _, s in ALIGN_HAPS]

    haps = [strip(h) for h in HAPS3]
    reads = [strip(r) for r in READS4]
    for is_rev in (False, True):
        for read, best, scores in zip(reads, BEST_OF_TWO, SCORES):
            counts, totals = ao.align_reads_to_haps([(is_rev, read)], haps[:2])
            assert counts == {(is_rev, best): 1}, (read, counts)
            assert totals == {(is_rev, h): s for h, s in enumerate(scores)}, (read, totals)
    counts, _ = ao.align_reads_to_haps([(False, r) for r in reads], haps)
    assert counts == {(False, h): n for h, n in BEST_OF_THREE.items()}, counts
    return got


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--copy-from", help="a medaka source checkout to copy the fixture files from")
    args = ap.parse_args(argv)
    if args.copy_from:
        os.makedirs(DATA, exist_ok=True)
        for name in FILES:
            shutil.copyfile(os.path.join(args.copy_from, "medaka", "test", "data", name), os.path.join(DATA, name))
    for info, e in zip(check(), EXPECTED):
        print(e[0], e[1], info)
    print("annotate golden OK")


if __name__ == "__main__":
    main()
