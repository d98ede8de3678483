"""Pin the truth-label oracle on the reference's own training-sample tests and its REAL truth BAM (build container only).

Run:  python tests/golden/make_truth_golden.py     (needs /root/reference; writes tests/golden/truth_labels.npz)

Reads /root/reference/medaka/test/data/{truth_to_ref,test_reads}.bam with medaka_b200.bam (no htslib, no pysam) and
runs oracle/truth_oracle.py.  Asserted:
1. test_030_bams_to_training_samples_simple (medaka/test/test_counts.py:73-115, truth from mock_data.py:24-31): labels
   [1,2,1,4,1,3,1,4,3] at (0..3,0),(3,1),(4..7,0); the truth's two insertions after position 6 that no read covers are
   dropped.
2. test_031_bams_to_training_samples_regression (:118-133): over utg000001l:149744-318288 the first sample has 177 981
   columns.
3. The truth filter on all of utg000001l, derived by hand from the rules of TruthAlignment._filter_alignments: 18
   records fetched (every one has flag 2064, supplementary + reverse), 17 kept: 417732-422799 overlaps 318288-417741 by
   9 bases, length ratio >= 2 and overlap fraction < 0.5 (case 4), so its start moves to 417 741; the 333-base
   919073-919406 falls to min_length; 149744-318288 and 318288-417741 touch without overlapping.  The package's own
   TruthAlignment.bam_to_alignments gives the same spans.
Stores the truth record 149744-318288, the read records over utg000001l:200000-203000 and the oracle's labelled
samples of that region as the fixture the CPU and GPU tests replay.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from medaka_b200 import bam, common, labels  # noqa: E402
from oracle import pileup_oracle, truth_oracle  # noqa: E402
from tests.test_oracle import SIMPLE_CALLS  # noqa: E402

DATA = "/root/reference/medaka/test/data"
CONTIG = "utg000001l"


def truth_dicts(batch):
    recs = pileup_oracle.records_from_batch(batch)
    for r, tags in zip(recs, batch.tags):
        r["tags"] = tags
    return recs


def main():
    # 1. test_030
    truth = dict(pos=0, cigar="4=1I3=2I1=", seq="ACATAGATCTG", flag=0, tags={"MD": "8"})
    (pos, lab), = truth_oracle.bams_to_training_samples([truth], SIMPLE_CALLS, "ref", 0, 100, min_length=0)
    assert lab.tolist() == [1, 2, 1, 4, 1, 3, 1, 4, 3]
    assert [tuple(p) for p in pos] == [(0, 0), (1, 0), (2, 0), (3, 0), (3, 1), (4, 0), (5, 0), (6, 0), (7, 0)]
    print("test_030 literals reproduced")

    tb = bam.BamFile(os.path.join(DATA, "truth_to_ref.bam"))
    rb = bam.BamFile(os.path.join(DATA, "test_reads.bam"))
    tbatch = tb.fetch(CONTIG, None, None, exclude_flags=labels.TRUTH_EXCLUDE_FLAGS, min_mapq=0, with_tags=True,
                      with_names=True)
    trecs = truth_dicts(tbatch)

    # 3. the filter over the whole contig
    assert len(trecs) == 18 and set(int(f) for f in tbatch.flag) == {2064}
    assert len(tb.fetch(CONTIG, None, None)[0]) == 0          # the pileup's flag filter would drop every record
    length = tb.lengths[tb.references.index(CONTIG)]
    spans = [(g[0].start, g[0].end) for g in truth_oracle.bam_to_alignments(trecs, CONTIG, 0, length)]
    assert len(spans) == 17
    assert (149744, 318288) in spans and (318288, 417741) in spans
    assert (417741, 422799) in spans and not any(s[0] == 417732 for s in spans)
    assert not any(s[0] == 919073 for s in spans)
    got = [(g[0].start, g[0].end) for g in labels.TruthAlignment.bam_to_alignments(
        tb, common.Region(CONTIG, 0, length))]
    assert got == spans
    print("truth filter: 18 fetched, 17 kept, case-4 trim to 417741 reproduced")

    # 2. test_031
    start, end = 149744, 318288
    reads = pileup_oracle.records_from_batch(rb.fetch(CONTIG, start, end))
    first_pos, _ = truth_oracle.bams_to_training_samples(trecs, reads, CONTIG, start, end)[0]
    assert len(first_pos) == 177981, len(first_pos)
    print("test_031 width reproduced: 177981 columns")

    # the fixture
    k = [i for i, r in enumerate(trecs) if r["pos"] == 149744][0]
    s0, s1 = 200000, 203000
    rbatch = rb.fetch(CONTIG, s0, s1)
    samples = truth_oracle.bams_to_training_samples([trecs[k]], pileup_oracle.records_from_batch(rbatch), CONTIG, s0, s1)
    major = np.concatenate([p["major"] for p, _ in samples])
    minor = np.concatenate([p["minor"] for p, _ in samples])
    lab = np.concatenate([lb for _, lb in samples])
    c0, c1 = tbatch.cigar_off[k], tbatch.cigar_off[k + 1]
    q0, q1 = tbatch.seq_off[k], tbatch.seq_off[k + 1]
    np.savez_compressed(
        os.path.join(HERE, "truth_labels.npz"),
        meta="truth_to_ref.bam record at %s:149744 and test_reads.bam records over %s:%d-%d" % (CONTIG, CONTIG, s0, s1),
        start=s0, end=s1, truth_pos=int(tbatch.pos[k]), truth_cigar=tbatch.cigar[c0:c1], truth_seq=tbatch.seq[q0:q1],
        truth_l_seq=int(tbatch.l_seq[k]), truth_md=tbatch.tags[k]["MD"], truth_flag=int(tbatch.flag[k]),
        pos=rbatch.pos, flag=rbatch.flag, mapq=rbatch.mapq, dtype=rbatch.dtype, cigar=rbatch.cigar,
        cigar_off=rbatch.cigar_off, seq=rbatch.seq, seq_off=rbatch.seq_off, l_seq=rbatch.l_seq,
        sample_len=np.array([len(p) for p, _ in samples]), major=major, minor=minor, labels=lab)
    print("fixture:", len(rbatch.pos), "read records,", len(major), "labelled columns,",
          int((lab != 0).sum()), "non-gap labels")


if __name__ == "__main__":
    main()
