"""Decode seam: per-position label decode on the GPU; and the training-label half: truth alignments and their labels.

Mirrors ``HaploidLabelScheme.decode_consensus`` (medaka/labels.py:1053-1085) and ``_phred``
(:387-401).  The array work - argmax (first maximum wins), probability of the chosen class,
``uint8(min(70, -10*log10(clip(1-p, 1e-7, 1)))) + 33`` - runs in libmedaka_b200
(mdk_decode_consensus); gap removal and string building, which are O(n) byte shuffles on
the result, stay on the host.

Training labels (medaka/labels.py:27-266, :422-567, :703-771): ``TruthAlignment`` selects and trims the truth
alignments of a region (host bookkeeping over a handful of records); the label of every pileup column - the reference's
per-pair dictionary joined to the sample positions - comes from the GPU (mdk_truth_labels).
"""
import collections
import copy
import itertools
import re

import numpy as np

from medaka_b200 import libmedaka as _lm


def decode_arrays(label_probs, device=0, with_qualities=True):
    """float32 probabilities [..., 5] -> (labels uint8 [...], quals uint8 [...] or None)."""
    lib = _lm.load()
    label_probs = label_probs.detach().cpu().numpy() if hasattr(label_probs, "detach") else np.asarray(label_probs)
    # numpy decodes in the array's own precision: float64 stays float64, everything else runs as float32
    f64 = label_probs.dtype == np.float64
    p = np.ascontiguousarray(label_probs, dtype=np.float64 if f64 else np.float32)
    if p.shape[-1] != 5:
        raise ValueError("expected label probabilities with 5 classes, got shape {}".format(p.shape))
    n = int(np.prod(p.shape[:-1]))
    labels = np.empty(p.shape[:-1], dtype=np.uint8)
    quals = np.empty(p.shape[:-1], dtype=np.uint8) if with_qualities else None
    ffi = _lm.ffi
    fn, ctype = (lib.mdk_decode_consensus_f64, "const double *") if f64 else (lib.mdk_decode_consensus, "const float *")
    _lm.check(fn(
        device, ffi.cast(ctype, ffi.from_buffer(p)), n,
        ffi.cast("uint8_t *", ffi.from_buffer(labels)),
        ffi.cast("uint8_t *", ffi.from_buffer(quals)) if with_qualities else ffi.NULL))
    return labels, quals


def variant_columns(minor, reference, prediction, device=0):
    """Which pileup columns belong to a variant run - ``HaploidLabelScheme._find_variants``
    (medaka/labels.py:869-887 -> libmedaka.lib.variant_columns, src/medaka_rnn_variants.c:28-55) on the GPU.

    :param minor: pileup minor indices; :param reference, prediction: per-column symbols (str, '|U1' / '|S1'
        arrays or uint8 label codes) including gaps.  :returns: bool array.
    """
    lib, ffi = _lm.load(), _lm.ffi

    def codes(x):
        a = np.asarray(list(x) if isinstance(x, str) else x)
        if a.dtype.kind == 'U':
            a = np.array([ord(c) for c in a.tolist()], dtype=np.uint32)
        elif a.dtype.kind == 'S':
            a = np.frombuffer(a.tobytes(), dtype=np.uint8)
        if a.size and int(a.max()) > 255:
            raise ValueError("symbols must fit one byte")
        return np.ascontiguousarray(a, dtype=np.uint8)

    mn = np.ascontiguousarray(minor, dtype=np.int64)
    r, p = codes(reference), codes(prediction)
    if not (len(mn) == len(r) == len(p)):
        raise ValueError("minor, reference and prediction must have the same length")
    out = np.zeros(len(mn), dtype=np.uint8)
    _lm.check(lib.mdk_variant_columns(device, ffi.cast("const int64_t *", ffi.from_buffer(mn)),
                                      ffi.cast("const uint8_t *", ffi.from_buffer(r)),
                                      ffi.cast("const uint8_t *", ffi.from_buffer(p)),
                                      ffi.cast("uint8_t *", ffi.from_buffer(out)), len(mn)))
    return out.astype(bool)


def decode_variant_arrays(label_probs, minor, ref_codes, device=0, want_quals=True):
    """The array half of ``decode_variants`` on the GPU (libmedaka_b200 ``mdk_decode_variants``).

    :param label_probs: float [n, 5]; :param minor: pileup minor indices [n]; :param ref_codes: uint8 [n], the draft
        with gaps as label codes (0..4 '*ACGT', 5 'N', 6 other).
    :returns: dict(pred uint8 [n], is_var bool [n], pred_q / ref_q float32 [n], run_start / run_len int64 [r],
        run_pred_q / run_ref_q float32 [r]).
    """
    lib, ffi = _lm.load(), _lm.ffi
    p = np.ascontiguousarray(label_probs.detach().cpu().numpy() if hasattr(label_probs, "detach") else label_probs,
                             dtype=np.float32)
    n = len(p)
    mn = np.ascontiguousarray(minor, dtype=np.int64)
    rc = np.ascontiguousarray(ref_codes, dtype=np.uint8)
    if p.ndim != 2 or p.shape[1] != 5 or len(mn) != n or len(rc) != n:
        raise ValueError("label_probs [n,5], minor [n] and ref_codes [n] expected")
    pred = np.empty(n, dtype=np.uint8)
    is_var = np.empty(n, dtype=np.uint8)
    pq = np.empty(n, dtype=np.float32) if want_quals else None
    rq = np.empty(n, dtype=np.float32) if want_quals else None
    max_runs = max(16, n // 8)
    n_runs = ffi.new("int64_t *")
    while True:
        rs, rl = np.empty(max_runs, dtype=np.int64), np.empty(max_runs, dtype=np.int64)
        rp, rr = np.empty(max_runs, dtype=np.float32), np.empty(max_runs, dtype=np.float32)
        code = lib.mdk_decode_variants(
            device, ffi.cast("const float *", ffi.from_buffer(p)), ffi.cast("const int64_t *", ffi.from_buffer(mn)),
            ffi.cast("const uint8_t *", ffi.from_buffer(rc)), n, ffi.cast("uint8_t *", ffi.from_buffer(pred)),
            ffi.cast("uint8_t *", ffi.from_buffer(is_var)),
            ffi.cast("float *", ffi.from_buffer(pq)) if want_quals else ffi.NULL,
            ffi.cast("float *", ffi.from_buffer(rq)) if want_quals else ffi.NULL, max_runs,
            ffi.cast("int64_t *", ffi.from_buffer(rs)), ffi.cast("int64_t *", ffi.from_buffer(rl)),
            ffi.cast("float *", ffi.from_buffer(rp)), ffi.cast("float *", ffi.from_buffer(rr)), n_runs)
        if code == lib.MDK_ERR_NOMEM and int(n_runs[0]) > max_runs:
            max_runs = int(n_runs[0])            # enlarge and retry, like enlarge_plp_data for the pileup
            continue
        _lm.check(code)
        break
    r = int(n_runs[0])
    return dict(pred=pred, is_var=is_var.astype(bool), pred_q=pq, ref_q=rq, run_start=rs[:r], run_len=rl[:r],
                run_pred_q=rp[:r], run_ref_q=rr[:r])


def _run_index(run_start, run_len):
    """Columns of the runs, back to back: run k's are run_start[k] .. run_start[k] + run_len[k] - 1."""
    run_len = np.asarray(run_len, dtype=np.int64)
    if len(run_len) == 0:
        return np.zeros(0, dtype=np.int64)
    off = np.cumsum(run_len) - run_len
    return np.repeat(np.asarray(run_start, dtype=np.int64) - off, run_len) + np.arange(int(run_len.sum()))


def variant_join_cuts(seg_calls, seg_rows, device=0):
    """Per trimmed piece of variant-decoded calls on the device (libmedaka_b200 ``mdk_variant_join_cuts``): the index of
    its last insertion-free column whose call equals the draft, or -1 when ``join_samples`` finds every column
    different.

    :param seg_calls: device addresses (int) of the pieces' first call bytes; :param seg_rows: their lengths.
    :returns: int64 array.
    """
    n = len(seg_calls)
    cut = np.empty(n, dtype=np.int64)
    if n == 0:
        return cut
    lib, ffi = _lm.load(), _lm.ffi
    ptrs = ffi.new("const uint8_t *[]", [ffi.cast("const uint8_t *", int(a)) for a in seg_calls])
    rows = np.ascontiguousarray(seg_rows, dtype=np.int64)
    _lm.check(lib.mdk_variant_join_cuts(device, ptrs, ffi.cast("const int64_t *", ffi.from_buffer(rows)), n,
                                        ffi.cast("int64_t *", ffi.from_buffer(cut))))
    return cut


def decode_variant_segments(seg_calls, seg_pred_q, seg_ref_q, seg_rows, sample_seg, device=0, want_quals=False,
                            want_ref_q=False):
    """The array half of ``decode_variants`` for joined samples whose variant-decoded calls are already on the device
    (libmedaka_b200 ``mdk_decode_variants_dev``).

    :param seg_calls, seg_pred_q, seg_ref_q: device addresses (int) of each piece's first call byte and phreds.
    :param seg_rows: the pieces' lengths.  :param sample_seg: joined sample s is pieces [sample_seg[s], sample_seg[s+1]).
    :returns: dict(run_sample, run_start (column within its sample), run_len int64 [r], run_pred_q / run_ref_q float32
        [r], run_pred uint8 [run columns], run_col_pred_q / run_col_ref_q float32 [run columns] (want_quals, else None),
        ref_q float32 [all columns of all samples] (want_ref_q, else None)).
    """
    lib, ffi = _lm.load(), _lm.ffi
    n_seg, n_samples = len(seg_calls), len(sample_seg) - 1
    rows = np.ascontiguousarray(seg_rows, dtype=np.int64)
    sseg = np.ascontiguousarray(sample_seg, dtype=np.int64)
    n = int(rows.sum())

    def table(ctype, addrs):
        return ffi.new(ctype + "[]", [ffi.cast(ctype, int(a)) for a in addrs]) if n_seg else ffi.NULL

    calls, pqs, rqs = (table("const uint8_t *", seg_calls), table("const float *", seg_pred_q),
                       table("const float *", seg_ref_q))
    ref_q = np.empty(n, dtype=np.float32) if want_ref_q else None
    max_runs, max_cols = max(16, n // 64), max(64, n // 16)
    n_runs, n_cols = ffi.new("int64_t *"), ffi.new("int64_t *")

    def out(a, ctype):
        return ffi.cast(ctype, ffi.from_buffer(a)) if a is not None else ffi.NULL

    while True:
        rsmp, rs, rl = (np.empty(max_runs, dtype=np.int64) for _ in range(3))
        rp, rr = np.empty(max_runs, dtype=np.float32), np.empty(max_runs, dtype=np.float32)
        cp = np.empty(max_cols, dtype=np.uint8)
        cpq = np.empty(max_cols, dtype=np.float32) if want_quals else None
        crq = np.empty(max_cols, dtype=np.float32) if want_quals else None
        code = lib.mdk_decode_variants_dev(
            device, calls, pqs, rqs, out(rows, "const int64_t *"), n_seg, out(sseg, "const int64_t *"), n_samples,
            max_runs, out(rsmp, "int64_t *"), out(rs, "int64_t *"), out(rl, "int64_t *"), out(rp, "float *"),
            out(rr, "float *"), max_cols, out(cp, "uint8_t *"), out(cpq, "float *"), out(crq, "float *"),
            out(ref_q, "float *"), n_runs, n_cols)
        if code == lib.MDK_ERR_NOMEM and (int(n_runs[0]) > max_runs or int(n_cols[0]) > max_cols):
            max_runs, max_cols = max(max_runs, int(n_runs[0])), max(max_cols, int(n_cols[0]))   # enlarge and retry
            continue
        _lm.check(code)
        break
    r, c = int(n_runs[0]), int(n_cols[0])
    return dict(run_sample=rsmp[:r], run_start=rs[:r], run_len=rl[:r], run_pred_q=rp[:r], run_ref_q=rr[:r],
                run_pred=cp[:c], run_col_pred_q=cpq[:c] if want_quals else None,
                run_col_ref_q=crq[:c] if want_quals else None, ref_q=ref_q)


# ---------------------------------------------------------------------------------------------------------
# Truth alignments
_OP_REF = np.array([c in "MDN=X" for c in "MIDNSHP=X"] + [False] * 7)     # by BAM op code
_OP_QRY = np.array([c in "MIS=X" for c in "MIDNSHP=X"] + [False] * 7)
_OP_MATCH = np.array([c in "M=X" for c in "MIDNSHP=X"] + [False] * 7)
_OP_D = 2
_NT16 = np.frombuffer(b"=ACMGRSVTWYHKDBN", dtype=np.uint8)
_NT16_LABEL = np.full(16, -1, dtype=np.int64)          # 4-bit base -> '*ACGT' code
_NT16_LABEL[[1, 2, 4, 8]] = [1, 2, 3, 4]
_MD_TOKEN = re.compile(r"(\d+)|(\^[A-Za-z]+)|([A-Za-z])")
TRUTH_EXCLUDE_FLAGS = 0x4 | 0x100          # UNMAP | SECONDARY: supplementary truth alignments are kept


class TruthRecord(object):
    """One truth alignment in BAM's packed encodings (CIGAR ops, 4-bit sequence) with the ``pysam.AlignedSegment``
    properties the truth filters read."""

    def __init__(self, reference_name, pos, cigar, seq, l_seq, tags=None, flag=0, query_name=None):
        self.reference_name = reference_name
        self.reference_start = int(pos)
        self.cigar = np.ascontiguousarray(cigar, dtype=np.uint32)
        self.seq = np.ascontiguousarray(seq, dtype=np.uint8)
        self.l_seq = int(l_seq)
        self.tags = dict(tags or {})
        self.flag = int(flag)
        self.query_name = query_name
        ops, lens = self.cigar & 0xF, (self.cigar >> 4).astype(np.int64)
        self.reference_length = int(lens[_OP_REF[ops]].sum())
        self.reference_end = self.reference_start + self.reference_length

    @classmethod
    def from_batch(cls, batch, reference_name):
        """Records of a ``RecordBatch`` fetched with tags and names."""
        return [cls(reference_name, batch.pos[i], batch.cigar[batch.cigar_off[i]:batch.cigar_off[i + 1]],
                    batch.seq[batch.seq_off[i]:batch.seq_off[i + 1]], batch.l_seq[i],
                    batch.tags[i] if batch.tags is not None else None, batch.flag[i],
                    batch.names[i] if batch.names is not None else None) for i in range(len(batch.pos))]

    def _nibbles(self):
        nib = np.empty(2 * len(self.seq), dtype=np.uint8)
        nib[0::2], nib[1::2] = self.seq >> 4, self.seq & 0xF
        return nib[:self.l_seq]

    @property
    def query_sequence(self):
        return _NT16[self._nibbles()].tobytes().decode()

    def aligned_pairs(self):
        """(query position, reference position) of every pair ``get_aligned_pairs`` yields, -1 for None: M, = and X
        give both, I and S the query position, D and N the reference position, H and P nothing."""
        ops, lens = self.cigar & 0xF, (self.cigar >> 4).astype(np.int64)
        r0 = self.reference_start + np.concatenate([[0], np.cumsum(np.where(_OP_REF[ops], lens, 0))[:-1]])
        q0 = np.concatenate([[0], np.cumsum(np.where(_OP_QRY[ops], lens, 0))[:-1]])
        n = np.where(_OP_REF[ops] | _OP_QRY[ops], lens, 0)
        op_of = np.repeat(np.arange(len(ops)), n)
        k = np.arange(int(n.sum())) - np.repeat(np.cumsum(n) - n, n)
        qpos = np.where(_OP_QRY[ops][op_of], q0[op_of] + k, -1)
        rpos = np.where(_OP_REF[ops][op_of], r0[op_of] + k, -1)
        return qpos, rpos

    def get_reference_sequence(self):
        """The reference under the alignment, rebuilt from the query and the MD tag like pysam's (upper case; skipped
        reference has no bases in MD and none here).  ValueError when MD is absent or does not fit the CIGAR."""
        md = self.tags.get("MD")
        if md is None:
            raise ValueError("MD tag not present")
        ops, lens = self.cigar & 0xF, (self.cigar >> 4).astype(np.int64)
        qpos, rpos = self.aligned_pairs()
        op_of = np.repeat(np.arange(len(ops)), np.where(_OP_REF[ops] | _OP_QRY[ops], lens, 0))
        aligned = (rpos >= 0) & (ops[op_of] != 3)               # M, =, X and D: the positions MD describes
        is_del = ops[op_of][aligned] == _OP_D
        ref = _NT16[self._nibbles()][np.where(is_del, 0, qpos[aligned])]
        ref[is_del] = ord("-")
        at = 0
        for num, dele, mism in _MD_TOKEN.findall(md):
            if num:
                at += int(num)
            else:
                bases = (dele[1:] if dele else mism).upper().encode()
                if at + len(bases) > len(ref) or bool(is_del[at:at + len(bases)].all()) != bool(dele):
                    raise ValueError("MD tag {} does not fit the CIGAR of {}".format(md, self.query_name))
                ref[at:at + len(bases)] = np.frombuffer(bases, dtype=np.uint8)
                at += len(bases)
        if at != len(ref):
            raise ValueError("MD tag {} does not fit the CIGAR of {}".format(md, self.query_name))
        return ref.tobytes().decode()


class TruthAlignment(object):
    """A truth alignment and the window [start, end) of it that is used (medaka/labels.py:27-266)."""

    def __init__(self, alignment):
        self.aln = alignment
        self.start = alignment.reference_start
        self.end = alignment.reference_end
        self.is_kept = True

    def _valid_symbols(self):
        """Neither the query nor the reference under it has a symbol other than A, C, G, T."""
        acgt = set("ACGT")
        return set(self.aln.get_reference_sequence().upper()) <= acgt and set(self.aln.query_sequence.upper()) <= acgt

    @staticmethod
    def _filter_alignments(alignments, region, min_length=1000, length_ratio=2.0, overlap_fraction=0.5):
        """The alignments suitable for training, trimmed to the region and sorted by start.

        Alignments with an ambiguous symbol go first.  Then every overlapping pair (over the untrimmed alignment
        spans) is resolved: of similar lengths (ratio < length_ratio), a large overlap (>= overlap_fraction of the
        shorter) drops both and a small one trims both to abut; otherwise a large overlap drops the shorter and a small
        one moves the start of the later one behind the overlap.  Last the region trim and ``min_length``.
        """
        kept = [copy.copy(a) for a in alignments if a._valid_symbols()]
        for a, b in itertools.combinations(kept, 2):
            first, second = sorted((a, b), key=lambda t: t.aln.reference_start)
            ovl_start, ovl_end = second.aln.reference_start, first.aln.reference_end
            if ovl_end <= ovl_start:
                continue
            shorter, longer = sorted((a, b), key=lambda t: t.aln.reference_length)
            large = (ovl_end - ovl_start) / shorter.aln.reference_length >= overlap_fraction
            if longer.aln.reference_length / shorter.aln.reference_length < length_ratio:
                if large:
                    a.is_kept = b.is_kept = False
                else:
                    first.end, second.start = ovl_start, ovl_end
            elif large:
                shorter.is_kept = False
            else:
                second.start = ovl_end
        for al in kept:
            if region.start is not None:
                al.start = max(region.start, al.start)
            if region.end is not None:
                al.end = min(region.end, al.end)
        kept = [al for al in kept if al.is_kept and al.end - al.start >= min_length]
        kept.sort(key=lambda t: t.start)
        return kept

    @staticmethod
    def _load_alignments(truth_bam, region, haplotag=None):
        """{haplotype: [TruthAlignment]} of the mapped, primary or supplementary truth records overlapping the region,
        sorted by start.  A record without the ``haplotag`` tag raises KeyError."""
        from medaka_b200 import bam as mbam
        bf = truth_bam if isinstance(truth_bam, mbam.BamFile) else mbam.BamFile(truth_bam)
        batch = bf.fetch(region.ref_name, region.start, region.end, exclude_flags=TRUTH_EXCLUDE_FLAGS, min_mapq=0,
                         with_tags=True, with_names=True)
        alignments = collections.defaultdict(list)
        for rec in TruthRecord.from_batch(batch, region.ref_name):
            alignments[rec.tags[haplotag] if haplotag is not None else None].append(TruthAlignment(rec))
        for algns in alignments.values():
            algns.sort(key=lambda t: t.start)
        return alignments

    @staticmethod
    def bam_to_alignments(truth_bam, region, haplotag=None, min_length=1000):
        """Filtered truth alignments of a region, as tuples of one ``TruthAlignment`` per haplotype trimmed to a
        common window."""
        algns = TruthAlignment._load_alignments(truth_bam, region, haplotag)
        algns = {h: TruthAlignment._filter_alignments(a, region=region, min_length=min_length)
                 for h, a in algns.items()}
        if not algns:
            return []
        return TruthAlignment._group_and_trim_by_haplotype(algns)

    @staticmethod
    def _group_and_trim_by_haplotype(alignments):
        """{haplotype: [TruthAlignment]} -> tuples, one alignment per haplotype (in sorted haplotype order), trimmed to
        their common window.  Each alignment of the first haplotype is taken in turn; in every other haplotype the
        alignment overlapping the window built so far the most (the first of equals) joins it; an alignment that finds
        no partner in some haplotype is skipped."""
        haplotypes = sorted(alignments.keys())
        if len(haplotypes) == 1:
            return [(a,) for a in alignments[haplotypes[0]]]
        grouped = []
        for a in alignments[haplotypes[0]]:
            group, lo, hi = [a], a.start, a.end
            for h in haplotypes[1:]:
                cands = [o for o in alignments[h] if o.start < o.end and o.start < hi and o.end > lo]
                if not cands:
                    break
                best = max(cands, key=lambda o: min(hi, o.end) - max(lo, o.start))
                lo, hi = max(lo, best.start), min(hi, best.end)
                group.append(best)
            if len(group) != len(haplotypes):
                continue
            for al in group:
                al.start, al.end = lo, hi
            grouped.append(tuple(group))
        return grouped


def truth_labels(truth, positions, device=0):
    """Label codes (int64, '*ACGT' -> 0..4, 0 where the truth has no such position) of the pileup columns at
    ``positions`` from one ``TruthAlignment``, on the GPU (mdk_truth_labels)."""
    lib, ffi = _lm.load(), _lm.ffi
    rec = truth.aln
    major = np.ascontiguousarray(positions['major'], dtype=np.int64)
    minor = np.ascontiguousarray(positions['minor'], dtype=np.int64)
    out = np.empty(len(major), dtype=np.int64)

    def ptr(ctype, a):
        return ffi.cast(ctype, ffi.from_buffer(a)) if a.size else ffi.NULL
    _lm.check(lib.mdk_truth_labels(
        device, rec.reference_start, ptr("const uint32_t *", rec.cigar), len(rec.cigar), ptr("const uint8_t *", rec.seq),
        rec.l_seq, int(truth.start), int(truth.end), len(major), ptr("const int64_t *", major),
        ptr("const int64_t *", minor), ptr("int64_t *", out)))
    return out


def from_name(name):
    """A label scheme by its class name; the diploid and run-length schemes are not implemented."""
    if name == 'HaploidLabelScheme':
        return HaploidLabelScheme()
    if name in ('DiploidLabelScheme', 'DiploidZygosityLabelScheme', 'RLELabelScheme'):
        raise NotImplementedError("label scheme {} is not implemented".format(name))
    raise ValueError("unknown label scheme {}".format(name))


class HaploidLabelScheme(object):
    """The reference's HaploidLabelScheme (labels.py:703-1085): decoding, and the encoding of haploid truth labels."""

    symbols = '*ACGT'     # labels.py:342
    n_elements = 1

    def __init__(self, device=0):
        self.device = device
        self.verbose = False
        # draft symbol -> label code; 5 = 'N' (its own symbol when compared, the gap class when scored), 6 = other
        self._ref_table = np.full(256, 6, dtype=np.uint8)
        for i, c in enumerate(self.symbols):
            self._ref_table[ord(c)] = i
        self._ref_table[ord('N')] = 5

    # pickles as an attribute-less object, like the reference's label scheme (plain object pickling of a class whose
    # instances carry no state); the lookup table and the device are rebuilt on load
    def __getstate__(self):
        return {}

    def __setstate__(self, state):
        self.__init__()
        self.__dict__.update(state)

    @staticmethod
    def _pfmt(p, dp=3):
        """labels.py:404-416."""
        if isinstance(p, np.ndarray):
            return np.char.mod("%.{}f".format(dp), p)
        return '{:.{dp}f}'.format(round(p, dp), dp=dp)

    def decode_labels(self, sample):
        """argmax label codes (uint8, gaps kept) of a sample - the integer form of decode_consensus(with_gaps=True)."""
        return decode_arrays(sample.label_probs, self.device, with_qualities=False)[0]

    def encode_reference(self, ref_seq, majors):
        """Label codes of the draft at the given major positions."""
        majors = np.asarray(majors, dtype=np.int64)
        if len(majors) == 0:
            return np.zeros(0, dtype=np.uint8)
        lo, hi = int(majors[0]), int(majors[-1]) + 1
        window = np.frombuffer(ref_seq[lo:hi].encode('ascii', 'replace'), dtype=np.uint8)
        return self._ref_table[window[majors - lo]]

    def reference_codes(self, positions, ref_seq):
        """The draft with '*' on insertion columns as label codes (labels.py:920): uint8 [n]."""
        is_major = positions['minor'] == 0
        ref_codes = np.zeros(len(positions), dtype=np.uint8)
        ref_codes[is_major] = self.encode_reference(ref_seq, positions['major'][is_major])
        return ref_codes

    def decode_variants(self, sample, ref_seq, ambig_ref=False, return_all=False):
        """Convert network output in sample to variant records (medaka/labels.py:889-1014).

        The consensus with gaps, the variant columns, the per-column qualities and the per-run sums come from the GPU
        (``mdk_decode_variants``); the records are built by ``variant_records``.  Returns a list of
        ``medaka_b200.variant.Variant``.
        """
        pos = sample.positions
        if pos['minor'][0] != 0:
            raise ValueError("The first position of a sample must not be an insertion.")
        ref_codes = self.reference_codes(pos, ref_seq)
        d = decode_variant_arrays(sample.label_probs, pos['minor'], ref_codes, self.device)
        idx = _run_index(d['run_start'], d['run_len'])
        return self.variant_records(
            sample.ref_name, pos, ref_codes, ref_seq, d['run_start'], d['run_len'], d['run_pred_q'], d['run_ref_q'],
            d['pred'][idx], d['pred_q'][idx] if self.verbose else None, d['ref_q'][idx] if self.verbose else None,
            d['ref_q'][pos['minor'] == 0] if return_all else None, ambig_ref=ambig_ref, return_all=return_all)

    def variant_records(self, ref_name, pos, ref_codes, ref_seq, run_start, run_len, run_pred_q, run_ref_q, run_pred,
                        run_col_pred_q=None, run_col_ref_q=None, major_ref_q=None, ambig_ref=False, return_all=False):
        """The host half of ``decode_variants`` (medaka/labels.py:927-1012): the decoded runs of one joined sample ->
        list of ``medaka_b200.variant.Variant``.

        :param pos, ref_codes: the sample's positions and ``reference_codes``.
        :param run_start, run_len, run_pred_q, run_ref_q: the variant runs (columns of the sample) and their sums.
        :param run_pred: the labels of all run columns back to back; ``run_col_pred_q`` / ``run_col_ref_q`` their
            phreds (needed when ``self.verbose``).  :param major_ref_q: the reference phred of every major column
            (needed with ``return_all``).
        Covers string spelling, the ref == alt and ambiguous-draft filters, ``ambig_ref``, the verbose info, the gVCF
        records and the VCF normalisation.
        """
        from medaka_b200.variant import Variant
        sym = np.frombuffer((self.symbols + 'N?').encode(), dtype=np.uint8)
        variants = []
        o = 0
        for rstart, rlen, spq, srq in zip(run_start, run_len, run_pred_q, run_ref_q):
            rstart, rend, o0 = int(rstart), int(rstart + rlen), o
            o += int(rlen)
            codes = ref_codes[rstart:rend]
            if np.any(codes == 6):
                # spell the run's draft from the sequence itself (any IUPAC symbol)
                ref_g = ''.join(ref_seq[int(m)] if mi == 0 else '*' for m, mi in zip(pos['major'][rstart:rend],
                                                                                     pos['minor'][rstart:rend]))
            else:
                ref_g = sym[codes].tobytes().decode()
            pred_g = sym[run_pred[o0:o]].tobytes().decode()
            var_ref, var_pred = ref_g.replace('*', ''), pred_g.replace('*', '')
            if var_ref == var_pred:          # deletion followed by insertion of the same base (labels.py:942-944)
                continue
            if not set(var_ref).issubset(set(self.symbols)):
                if not ambig_ref:
                    continue
                if set(var_ref) - set(self.symbols) - {'N'}:
                    raise KeyError("draft symbol outside '*ACGTN' in a variant run at {}:{}".format(
                        ref_name, int(pos['major'][rstart])))
            qual = np.float32(spq) - np.float32(srq)          # log likelihood ratio (labels.py:974-975), float32
            info = {}
            if self.verbose:
                info = {'ref_seq': ref_g, 'pred_seq': pred_g,
                        'ref_qs': ','.join(self._pfmt(float(q)) for q in run_col_ref_q[o0:o]),
                        'pred_qs': ','.join(self._pfmt(float(q)) for q in run_col_pred_q[o0:o]),
                        'ref_q': self._pfmt(float(srq)), 'pred_q': self._pfmt(float(spq)), 'n_cols': rend - rstart}
            genotype = {'GT': '1', 'GQ': self._pfmt(float(qual), 0)}
            var_pos = int(pos['major'][rstart])
            if pos['minor'][rstart] != 0:    # variant starts on an insertion column: prepend the draft base
                var_ref = ref_seq[var_pos] + var_ref
                var_pred = ref_seq[var_pos] + var_pred
            v = Variant(ref_name, var_pos, var_ref, alt=var_pred, filt='PASS', info=info,
                        qual=self._pfmt(float(qual)), genotype_data=genotype)
            variants.append(v.normalize(reference=ref_seq))
        if return_all:
            # one record per reference position (labels.py:991-1012)
            is_major = pos['minor'] == 0
            quals = np.asarray(major_ref_q)
            qf, qi = np.char.mod("%.3f", quals), np.char.mod("%d", np.rint(quals))
            bases = [ref_seq[int(m)] for m in pos['major'][is_major]]
            for p_, base, f_, i_ in zip(pos['major'][is_major], bases, qf, qi):
                variants.append(Variant(ref_name, int(p_), base, alt='.', filt='.', info={}, qual=str(f_),
                                        genotype_data={'GT': '0', 'GQ': str(i_)}))
            variants.sort(key=lambda x: x.pos)
        return variants

    @property
    def num_classes(self):
        return len(self.symbols)

    # ---- encoding (labels.py:422-567, :730-756)
    @property
    def _encoding(self):
        """label tuple -> integer: ('*',) 0, ('A',) 1, ('C',) 2, ('G',) 3, ('T',) 4."""
        return {(s,): i for i, s in enumerate(self.symbols)}

    def _labels_to_encoded_labels(self, labels):
        enc = self._encoding
        return np.fromiter((enc[x] for x in labels), dtype=np.int64, count=len(labels))

    @property
    def padding_vector(self):
        """The code of a column the truth has no base for: the gap's."""
        return self._labels_to_encoded_labels([('*',)])[0]

    def _check_truth(self, truth_alns):
        if len(truth_alns) != self.n_elements:
            raise ValueError('{} alignments were passed to {}, requires {}'.format(
                len(truth_alns), type(self).__name__, self.n_elements))

    def encode(self, truth_alns):
        """Truth positions (structured major / minor) and their codes (int64) of a 1-tuple of ``TruthAlignment``.

        The alignment's pairs are taken from the first one on a reference position >= start up to the first one on a
        position >= end: a reference position gets (pos, 0) and the base or '*', each query-only pair behind it (pos,
        k) for the k-th of its run - so a trailing soft clip becomes insertions, a leading one is dropped.
        """
        self._check_truth(truth_alns)
        aln = truth_alns[0]
        qpos, rpos = aln.aln.aligned_pairs()
        inside = rpos >= aln.start
        first = int(np.argmax(inside)) if inside.any() else len(rpos)
        beyond = rpos >= aln.end
        beyond[:first] = False
        stop = int(np.argmax(beyond)) if beyond.any() else len(rpos)
        qpos, rpos = qpos[first:stop], rpos[first:stop]
        idx = np.arange(len(rpos))
        last_ref = np.maximum.accumulate(np.where(rpos >= 0, idx, 0))
        positions = np.empty(len(rpos), dtype=[('major', '<i8'), ('minor', '<i8')])
        positions['major'] = rpos[last_ref]
        positions['minor'] = idx - last_ref
        codes = np.zeros(len(rpos), dtype=np.int64)
        has_q = qpos >= 0
        codes[has_q] = _NT16_LABEL[aln.aln._nibbles()[qpos[has_q]]]
        if np.any(codes < 0):
            raise KeyError("truth base outside 'ACGT' in {}".format(aln.aln.query_name))
        return positions, codes

    def label_columns(self, truth_alns, positions):
        """Labels of a sample's columns from a 1-tuple of ``TruthAlignment``: ``encode`` joined to the sample's
        positions, the padding vector where the truth has no position, computed on the GPU (mdk_truth_labels)."""
        self._check_truth(truth_alns)
        return truth_labels(truth_alns[0], positions, self.device)

    @staticmethod
    def _phred(err, cap=70.0):
        """Host restatement kept for API compatibility (labels.py:387-401); not used on the hot path."""
        err = np.clip(err, 10 ** (-cap / 10.0), 1)
        return np.minimum(-10 * np.log10(err), cap)

    @staticmethod
    def _find_variants(minor, reference, prediction):
        """labels.py:869-887."""
        return variant_columns(minor, reference, prediction)

    def decode_consensus(self, sample, with_gaps=False, dtype=None, with_qualities=False):
        """Convert network output to consensus sequence by argmax decoding.

        :param sample: object with a ``label_probs`` array [n, 5].
        :param with_gaps: include gap ("*") characters in output.
        :returns: str, consensus sequence, optionally: qualities
        """
        mp, quals = decode_arrays(sample.label_probs, self.device, with_qualities=with_qualities)
        if not with_gaps:
            keep = mp != self.symbols.index('*')
            mp = mp[keep]
            if with_qualities:
                quals = quals[keep]
        if dtype is None:
            table = np.frombuffer(self.symbols.encode(), dtype=np.uint8)
            seq = table[mp].tobytes().decode()
        else:
            seq = np.fromiter(self.symbols, dtype=dtype)[mp]
        if with_qualities:
            return seq, quals.tobytes().decode()
        return seq
