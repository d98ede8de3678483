"""Oracle for the training-label half of `medaka features --truth`.  TEST INFRASTRUCTURE (see oracle/__init__.py).

A loop-based restatement of TruthAlignment (medaka/labels.py:27-266), _alignments_to_labels / encode
(:422-567), the encoding half of HaploidLabelScheme (:703-771), bams_to_training_samples
(medaka/features.py:937-994) and the training half of SampleGenerator / create_samples (:1208-1414), over plain
dict records ('pos', 'cigar' string, 'seq' string, 'flag', 'tags' with 'MD').  Pairs are generated one by one and
labels are joined to pileup columns through a dictionary: nothing is shared with the device path (no scans, no
binary search).  Pileup columns come from oracle/pileup_oracle.py.
"""
import re

import numpy as np

from oracle import common_oracle, pileup_oracle

_CIGAR_RE = re.compile(r"(\d+)([MIDNSHP=X])")
SYMBOLS = "*ACGT"
ENCODING = {(s,): i for i, s in enumerate(SYMBOLS)}


def cigar_ops(rec):
    return [(op, int(n)) for n, op in _CIGAR_RE.findall(rec["cigar"])]


def reference_length(rec):
    return sum(n for op, n in cigar_ops(rec) if op in "MDN=X")


def get_aligned_pairs(rec):
    """pysam's AlignedSegment.get_aligned_pairs(): list of (qpos or None, rpos or None)."""
    pairs = []
    q, r = 0, rec["pos"]
    for op, n in cigar_ops(rec):
        for _ in range(n):
            if op in "M=X":
                pairs.append((q, r))
                q += 1
                r += 1
            elif op in "IS":
                pairs.append((q, None))
                q += 1
            elif op in "DN":
                pairs.append((None, r))
                r += 1
            # H and P: nothing
    return pairs


def get_reference_sequence(rec):
    """pysam's get_reference_sequence(): the aligned reference from the query and the MD tag (upper case)."""
    md = rec.get("tags", {}).get("MD")
    if md is None:
        raise ValueError("MD tag not present")
    seq = rec["seq"]
    aligned = []            # one entry per M/=/X/D reference base: the query base, or '-' for a deletion
    q = 0
    for op, n in cigar_ops(rec):
        for _ in range(n):
            if op in "M=X":
                aligned.append(seq[q])
                q += 1
            elif op in "IS":
                q += 1
            elif op == "D":
                aligned.append("-")
    i = 0
    k = 0
    while k < len(md):
        if md[k].isdigit():
            j = k
            while j < len(md) and md[j].isdigit():
                j += 1
            i += int(md[k:j])
            k = j
        elif md[k] == "^":
            k += 1
            while k < len(md) and md[k].isalpha():
                if aligned[i] != "-":
                    raise ValueError("MD deletion on an aligned base")
                aligned[i] = md[k].upper()
                i += 1
                k += 1
        else:
            if aligned[i] == "-":
                raise ValueError("MD mismatch on a deleted base")
            aligned[i] = md[k].upper()
            i += 1
            k += 1
    if i != len(aligned):
        raise ValueError("MD does not cover the alignment")
    return "".join(aligned).upper()


class Truth(object):
    def __init__(self, rec):
        self.rec = rec
        self.reference_start = rec["pos"]
        self.reference_length = reference_length(rec)
        self.reference_end = self.reference_start + self.reference_length
        self.start = self.reference_start
        self.end = self.reference_end
        self.is_kept = True

    def copy(self):
        t = Truth(self.rec)
        t.start, t.end, t.is_kept = self.start, self.end, self.is_kept
        return t


def filter_alignments(alignments, region_start, region_end, min_length=1000, length_ratio=2.0, overlap_fraction=0.5):
    """TruthAlignment._filter_alignments (labels.py:53-136)."""
    out = []
    for a in alignments:
        ref = get_reference_sequence(a.rec)
        ok = all(c in "ACGT" for c in ref) and all(c in "ACGT" for c in a.rec["seq"].upper())
        if ok:
            out.append(a.copy())
    for i in range(len(out)):
        for j in range(i + 1, len(out)):
            ai, aj = out[i], out[j]
            if aj.reference_start < ai.reference_start:
                first, second = aj, ai
            else:
                first, second = ai, aj
            if not first.reference_end > second.reference_start:
                continue
            ovlp_start, ovlp_end = second.reference_start, first.reference_end
            if aj.reference_length < ai.reference_length:
                shorter, longer = aj, ai
            else:
                shorter, longer = ai, aj
            ratio = longer.reference_length / shorter.reference_length
            frac = (ovlp_end - ovlp_start) / shorter.reference_length
            if ratio < length_ratio:
                if frac >= overlap_fraction:
                    shorter.is_kept = False
                    longer.is_kept = False
                else:
                    first.end = ovlp_start
                    second.start = ovlp_end
            else:
                if frac >= overlap_fraction:
                    shorter.is_kept = False
                else:
                    second.start = ovlp_end
    for a in out:
        if region_start > 0:
            a.start = max(region_start, a.start)
        if region_end is not None:
            a.end = min(region_end, a.end)
    out = [a for a in out if a.is_kept and a.end - a.start >= min_length]
    out.sort(key=lambda a: a.start)
    return out


def group_and_trim(by_hap):
    """TruthAlignment._group_and_trim_by_haplotype (labels.py:170-234); ties of the overlap go to the earliest start."""
    haps = sorted(by_hap)
    if len(haps) == 1:
        return [(a,) for a in by_hap[haps[0]]]
    grouped = []
    for a in by_hap[haps[0]]:
        group = [a]
        cs, ce = a.start, a.end
        for h in haps[1:]:
            best, best_ovl = None, None
            for o in by_hap[h]:
                if o.start < o.end and o.start < ce and o.end > cs:
                    ovl = min(ce, o.end) - max(cs, o.start)
                    if best is None or ovl > best_ovl:
                        best, best_ovl = o, ovl
            if best is None:
                break
            cs, ce = max(cs, best.start), min(ce, best.end)
            group.append(best)
        if len(group) != len(haps):
            continue
        for g in group:
            g.start, g.end = cs, ce
        grouped.append(tuple(group))
    return grouped


def bam_to_alignments(truth_records, ref_name, region_start, region_end, haplotag=None, min_length=1000):
    """TruthAlignment.bam_to_alignments: of the records overlapping the region (what pysam's fetch returns), the
    unmapped and secondary ones are skipped."""
    by_hap = {}
    for rec in truth_records:
        if rec.get("flag", 0) & (0x4 | 0x100):
            continue
        if not (rec["pos"] < region_end and rec["pos"] + reference_length(rec) > region_start):
            continue
        hap = rec["tags"][haplotag] if haplotag is not None else None
        by_hap.setdefault(hap, []).append(Truth(rec))
    for h in by_hap:
        by_hap[h].sort(key=lambda a: a.start)
    by_hap = {h: filter_alignments(a, region_start, region_end, min_length) for h, a in by_hap.items()}
    if not by_hap:
        return []
    return group_and_trim(by_hap)


def alignment_to_labels(truth):
    """_alignments_to_labels (labels.py:422-483) for one haplotype: {(major, minor): symbol}."""
    seq = truth.rec["seq"]
    pos_to_symbol = {}
    dropping = True
    ins_count = 0
    current_pos = None
    for qpos, rpos in get_aligned_pairs(truth.rec):
        if dropping:
            if rpos is None or rpos < truth.start:
                continue
            dropping = False
        if rpos is not None and rpos >= truth.end:
            break
        if rpos is None:
            ins_count += 1
        else:
            ins_count = 0
            current_pos = rpos
        pos_to_symbol[(current_pos, ins_count)] = seq[qpos].upper() if qpos is not None else "*"
    return pos_to_symbol


def encode(truth):
    """HaploidLabelScheme.encode: (sorted positions [(major, minor)], int64 codes)."""
    m = alignment_to_labels(truth)
    positions = sorted(m)
    return positions, np.array([ENCODING[(m[p],)] for p in positions], dtype=np.int64)


def join_labels(truth, positions):
    """bams_to_training_samples' padding + np.in1d join (features.py:979-992) for one sample's positions."""
    m = alignment_to_labels(truth)
    out = np.zeros(len(positions), dtype=np.int64)
    for i, (major, minor) in enumerate(zip(positions["major"], positions["minor"])):
        key = (int(major), int(minor))
        if key in m:
            out[i] = ENCODING[(m[key],)]
    return out


def split_on_gaps(positions):
    """Index ranges of the pieces of a pileup between coverage gaps."""
    if len(positions) == 0:
        return []
    bounds = [0]
    for i in range(1, len(positions)):
        if positions["major"][i] - positions["major"][i - 1] > 1:
            bounds.append(i)
    bounds.append(len(positions))
    return list(zip(bounds[:-1], bounds[1:]))


def bams_to_training_samples(truth_records, read_records, ref_name, region_start, region_end, min_length=1000,
                             haplotag=None, dtypes=None):
    """Labelled pileups of a region: list of (positions, labels) per gap-free piece of the reads' pileup over each
    trimmed truth span."""
    out = []
    for group in bam_to_alignments(truth_records, ref_name, region_start, region_end, haplotag, min_length):
        if len(group) != 1:
            raise ValueError("{} alignments were passed to HaploidLabelScheme, requires 1".format(len(group)))
        truth = group[0]
        _, positions = pileup_oracle.pileup_counts(read_records, truth.start, truth.end, dtypes=dtypes)
        for a, b in split_on_gaps(positions):
            out.append((positions[a:b], join_labels(truth, positions[a:b])))
    return out


def sample_name(ref_name, positions):
    return "{}:{}.{}-{}.{}".format(ref_name, positions["major"][0], positions["minor"][0], positions["major"][-1],
                                   positions["minor"][-1])


def create_samples(truth_records, read_records, ref_name, ref_len, chunk_len=10000, chunk_ovlp=1000, min_length=1000,
                   max_size=1000000, dtypes=None):
    """create_samples for one contig: {sample name: (positions, labels)} of every chunk that would be written."""
    written = {}
    for start, end in common_oracle.region_split(0, ref_len, max_size):
        for positions, labels in bams_to_training_samples(truth_records, read_records, ref_name, start, end,
                                                          min_length, dtypes=dtypes):
            if len(positions) < chunk_len:
                continue
            for a, b in common_oracle.chunk_ranges(len(positions), chunk_len, chunk_ovlp):
                name = sample_name(ref_name, positions[a:b])
                if name not in written:
                    written[name] = (positions[a:b], labels[a:b])
    return written
