"""Featuriser seam: counts post-processing / normalisation on the GPU, and window generation.

Mirrors the inference half of medaka/features.py: ``pileup_counts_norm_indices`` (:647-687),
``CountsFeatureEncoder`` (:813-935; ``_post_process_pileup`` is the part that runs on the
device through mdk_normalise_counts) and ``SampleGenerator`` (:1208-1313).  Raw pileup
counts come from ``_pileup_function`` - in the reference that is htslib's multi-pileup walked
by src/medaka_counts.c; here it is pluggable (``pileup_source``) because no BAM decoder is
part of the reference tree; ``pileup_counts`` below is the GPU replacement (BAM inflate/parse on the
host in medaka_b200/bam.py, per-base counting in csrc/pileup.cu), and a custom ``pileup_source`` can
still be plugged in (the benchmark's synthetic source does).

The training half (``bams_to_training_samples`` :937-994, the truth arguments of ``SampleGenerator``,
``create_samples`` :1316-1414) labels the samples of both encoders from truth alignments (medaka_b200/labels.py).
"""
import inspect
from collections import defaultdict
from timeit import default_timer as now

import concurrent.futures

import numpy as np

from medaka_b200 import common
from medaka_b200 import libmedaka as _lm

_NORM_MODES = {'total': 0, 'fwd_rev': 1, None: 2}


def pileup_counts_norm_indices(dtypes, num_qstrat=1):
    """Per (datatype, is_rev) column indices of the counts matrix (medaka/features.py:647-687)."""
    lib = _lm.load()
    codes = _lm.ffi.string(lib.mdk_plp_bases()).decode()
    featlen = int(lib.mdk_featlen())
    assert len(codes) == featlen
    indices = defaultdict(list)
    for dti, dt in enumerate(dtypes):
        for qindex in range(num_qstrat):
            for base_i, code in enumerate(codes):
                indices[dt, code.islower()].append(base_i + featlen * (dti * num_qstrat + qindex))
    return dict(indices)


def _split_on_gaps(counts, positions):
    """First pass of __enforce_pileup_chunk_contiguity (medaka/features.py:111-164): a jump of the major
    coordinate by more than one starts a new chunk.  (The second pass - re-joining abutting sub-region results -
    is moot here because the GPU featuriser processes a region in one piece instead of 100 kb slices.)"""
    if len(positions) == 0:
        return []
    cuts = np.where(np.ediff1d(positions['major']) > 1)[0] + 1
    bounds = [0] + cuts.tolist() + [len(positions)]
    return [(counts[a:b], positions[a:b]) for a, b in zip(bounds[:-1], bounds[1:])]


def pileup_counts(region, bam, dtype_prefixes=None, region_split=100000, workers=8, tag_name=None,
                  tag_value=None, keep_missing=False, num_qstrat=1, weibull_summation=False, read_group=None,
                  min_mapq=1, device=0):
    """Create pileup counts feature array for region - the reference's ``pileup_counts``
    (medaka/features.py:199-255) with the per-base work on the GPU (mdk_pileup_counts).

    :param bam: a ``medaka_b200.bam.BamFile`` (or a path to a BAM file).
    :returns: list of (counts uint64 [n, 10*len(dtypes)], positions) chunks, split at coverage gaps.
    ``region_split`` / ``workers`` are accepted for signature compatibility; the device processes the whole
    region at once.  Quality stratification / Weibull summation (legacy RLE models) are not supported.
    """
    from medaka_b200 import bam as mbam
    if num_qstrat != 1 or weibull_summation:
        raise NotImplementedError("q-score stratification / Weibull summation belong to the legacy RLE models")
    if tag_name is not None and len(tag_name) != 2:
        raise ValueError("'tag_name' must be a length-2 string.")
    if not isinstance(bam, mbam.BamFile):
        bam = mbam.BamFile(bam)
    multi = not (dtype_prefixes is None or isinstance(dtype_prefixes, str) or len(dtype_prefixes) == 1)
    num_dtypes = len(dtype_prefixes) if multi else 1
    # the read filter in the reference's order (src/medaka_bamiter.c:17-45): flags and mapping quality first, natively,
    # so that the tag / read-group / datatype tests only ever see reads the reference would have looked at too
    batch = bam.fetch(region.ref_name, region.start, region.end, dtypes=dtype_prefixes if multi else None,
                      tag_name=tag_name, tag_value=tag_value, keep_missing=keep_missing, read_group=read_group,
                      min_mapq=min_mapq)
    counts, positions = pileup_counts_from_batch(batch, region.start, region.end, num_dtypes, min_mapq, device)
    return _split_on_gaps(counts, positions)


def _record_args(batch):
    """The eight record arrays of a ``RecordBatch`` as the featuriser entry points take them, in ABI order (pos, flag,
    mapq, dtype, cigar, cigar_off, seq, seq_off).  Each is a typed cffi buffer that keeps its numpy array alive for as
    long as the returned list is referenced, so hold the list until the call returns."""
    ffi = _lm.ffi
    return [ffi.from_buffer(ctype + "[]", np.ascontiguousarray(getattr(batch, name), dtype))
            for name, ctype, dtype in (("pos", "int32_t", np.int32), ("flag", "uint16_t", np.uint16),
                                       ("mapq", "uint8_t", np.uint8), ("dtype", "uint8_t", np.uint8),
                                       ("cigar", "uint32_t", np.uint32), ("cigar_off", "int64_t", np.int64),
                                       ("seq", "uint8_t", np.uint8), ("seq_off", "int64_t", np.int64))]


def _positions(major, minor, n):
    """The (major, minor) positions array of the first n columns."""
    positions = np.empty(n, dtype=[('major', '<i8'), ('minor', '<i8')])
    positions['major'] = major[:n]
    positions['minor'] = minor[:n]
    return positions


def pileup_counts_from_batch(batch, start, end, num_dtypes=1, min_mapq=1, device=0):
    """Run the GPU pileup over a ``RecordBatch``; returns (counts, positions) for [start, end)."""
    lib, ffi = _lm.load(), _lm.ffi
    n_rec = len(batch.pos)
    F = 10 * num_dtypes
    max_cols = max(2 * (end - start), 16)          # the reference's initial guess (medaka_counts.c:245)
    records = _record_args(batch)
    n_cols = ffi.new("int64_t *")
    for _ in range(2):
        # (np.empty: untouched pages of the reference-style over-allocation cost nothing; the library writes n rows)
        counts = np.empty((max_cols, F), dtype=np.uint64)
        major = np.empty(max_cols, dtype=np.int64)
        minor = np.empty(max_cols, dtype=np.int64)
        rc = lib.mdk_pileup_counts(
            device, n_rec, *records, int(start), int(end), num_dtypes, int(min_mapq), max_cols,
            ffi.cast("uint64_t *", ffi.from_buffer(counts)), ffi.cast("int64_t *", ffi.from_buffer(major)),
            ffi.cast("int64_t *", ffi.from_buffer(minor)), n_cols)
        if rc == lib.MDK_ERR_NOMEM and n_cols[0] > max_cols:
            max_cols = int(n_cols[0])       # like enlarge_plp_data: retry with room for every column
            continue
        _lm.check(rc)
        break
    n = int(n_cols[0])
    positions = _positions(major, minor, n)
    return counts[:n], positions


def pileup_features_from_batch(batch, start, end, num_dtypes=1, min_mapq=1, normalise='total', sym_indels=False,
                               device=0):
    """calculate_pileup + _post_process_pileup in one device pass (mdk_pileup_features): the counts never leave the
    GPU.  Returns (features float32 [n, 10*num_dtypes], depth int64 [n], positions) for [start, end)."""
    lib, ffi = _lm.load(), _lm.ffi
    n_rec = len(batch.pos)
    F = 10 * num_dtypes
    max_cols = max(2 * (end - start), 16)
    records = _record_args(batch)
    n_cols = ffi.new("int64_t *")
    for _ in range(2):
        feats = np.empty((max_cols, F), dtype=np.float32)
        depth = np.empty(max_cols, dtype=np.int64)
        major = np.empty(max_cols, dtype=np.int64)
        minor = np.empty(max_cols, dtype=np.int64)
        rc = lib.mdk_pileup_features(
            device, n_rec, *records, int(start), int(end), num_dtypes, int(min_mapq), _NORM_MODES[normalise],
            1 if sym_indels else 0, max_cols,
            ffi.cast("float *", ffi.from_buffer(feats)), ffi.cast("int64_t *", ffi.from_buffer(depth)),
            ffi.cast("int64_t *", ffi.from_buffer(major)), ffi.cast("int64_t *", ffi.from_buffer(minor)), n_cols)
        if rc == lib.MDK_ERR_NOMEM and n_cols[0] > max_cols:
            max_cols = int(n_cols[0])
            continue
        _lm.check(rc)
        break
    n = int(n_cols[0])
    positions = _positions(major, minor, n)
    return feats[:n], depth[:n], positions


class CountsFeatureEncoder(object):
    """Create a pileup array of counts of observed bases (medaka/features.py:813-935)."""

    _norm_modes_ = ['total', 'fwd_rev', None]
    feature_dtype = np.float32

    def __init__(self, normalise='total', dtypes=('',), tag_name=None, tag_value=None,
                 tag_keep_missing=False, read_group=None, min_mapq=1, sym_indels=False,
                 pileup_source=None, device=0):
        self.normalise = normalise
        self.dtypes = dtypes
        self.feature_indices = pileup_counts_norm_indices(self.dtypes)
        self.tag_name = tag_name
        self.tag_value = tag_value
        self.tag_keep_missing = tag_keep_missing
        self.read_group = read_group
        self.min_mapq = min_mapq
        self.sym_indels = sym_indels
        self.pileup_source = pileup_source
        self.device = device
        if self.normalise not in self._norm_modes_:
            raise ValueError('normalise={} is not one of {}'.format(self.normalise, self._norm_modes_))
        self.logger = common.get_named_logger('Feature')

    # pickled like the reference's encoder (medaka/features.py:800-810): the attribute set of its __init__ (:819-846),
    # no logger; nothing device- or source-specific crosses the fence
    _state_fields = ('normalise', 'dtypes', 'feature_indices', 'tag_name', 'tag_value', 'tag_keep_missing',
                     'read_group', 'min_mapq', 'sym_indels')

    def __getstate__(self):
        return {k: getattr(self, k) for k in self._state_fields}

    def __setstate__(self, state):
        self.__dict__.update(state)
        self.__dict__.setdefault('pileup_source', None)
        self.__dict__.setdefault('device', 0)
        self.logger = common.get_named_logger('Feature')

    def to_dict(self):
        """Return dictionary of keyword arguments."""
        opts = inspect.signature(self.__class__.__init__).parameters
        kwargs = {k: getattr(self, k) for k in opts if k not in ('self', 'pileup_source', 'device')}
        return {'type': self.__class__.__name__, 'kwargs': kwargs}

    @property
    def feature_vector_length(self):
        """Length of a neural network input at a single time point."""
        return len(self.dtypes) * int(_lm.load().mdk_featlen())

    def _pileup_function(self, region, bam):
        """Raw counts for a region: list of (counts uint64 [n,F], positions) chunks (features.py:863-869)."""
        if self.pileup_source is not None:
            return self.pileup_source(region, bam, self)
        return pileup_counts(
            region, bam, dtype_prefixes=self.dtypes, tag_name=self.tag_name, tag_value=self.tag_value,
            keep_missing=self.tag_keep_missing, read_group=self.read_group, min_mapq=self.min_mapq,
            device=self.device)

    def _post_process_pileup(self, counts, positions, region):
        """Normalise counts on the GPU (features.py:871-935) and wrap them in a Sample."""
        start, end = positions['major'][0], positions['major'][-1]
        if start != region.start or end + 1 != region.end:
            self.logger.warning(
                'Pileup counts do not span requested region, requested {}, '
                'received {}-{}.'.format(region, start, end))
        lib, ffi = _lm.load(), _lm.ffi
        n, F = counts.shape
        num_dtypes = len(self.dtypes)
        if F != 10 * num_dtypes:
            raise ValueError("counts have {} columns, encoder expects {}".format(F, 10 * num_dtypes))
        counts = np.ascontiguousarray(counts, dtype=np.uint64)
        major = np.ascontiguousarray(positions['major'], dtype=np.int64)
        minor = np.ascontiguousarray(positions['minor'], dtype=np.int64)
        feats = np.empty((n, F), dtype=np.float32)
        depth = np.empty(n, dtype=np.int64)
        _lm.check(lib.mdk_normalise_counts(
            self.device, ffi.cast("const uint64_t *", ffi.from_buffer(counts)),
            ffi.cast("const int64_t *", ffi.from_buffer(major)),
            ffi.cast("const int64_t *", ffi.from_buffer(minor)), n, num_dtypes,
            _NORM_MODES[self.normalise], 1 if self.sym_indels else 0,
            ffi.cast("float *", ffi.from_buffer(feats)), ffi.cast("int64_t *", ffi.from_buffer(depth))))
        return common.Sample(
            ref_name=region.ref_name, features=feats, labels=None, ref_seq=None,
            positions=positions, label_probs=None, depth=depth)

    _fused_featuriser = True     # counts -> features in one device pass (subclasses with other features switch it off)

    def _fused_samples(self, reads_bam, region):
        """bam_to_sample through mdk_pileup_features: fetch, pileup + normalise on the device, split at coverage gaps.
        Same Samples as the two-step path (a minor column and its major never sit on different sides of a gap)."""
        from medaka_b200 import bam as mbam
        bam = reads_bam if isinstance(reads_bam, mbam.BamFile) else mbam.BamFile(reads_bam)
        if self.tag_name is not None and len(self.tag_name) != 2:
            raise ValueError("'tag_name' must be a length-2 string.")
        dts = self.dtypes
        multi = not (dts is None or isinstance(dts, str) or len(dts) == 1)
        batch = bam.fetch(region.ref_name, region.start, region.end, dtypes=dts if multi else None, tag_name=self.tag_name,
                          tag_value=self.tag_value, keep_missing=self.tag_keep_missing, read_group=self.read_group,
                          min_mapq=self.min_mapq)
        feats, depth, positions = pileup_features_from_batch(
            batch, region.start, region.end, len(dts) if multi else 1, self.min_mapq, self.normalise, self.sym_indels,
            self.device)
        if len(positions) == 0:
            return None
        cuts = np.where(np.ediff1d(positions['major']) > 1)[0] + 1
        bounds = [0] + cuts.tolist() + [len(positions)]
        samples = []
        for a, b in zip(bounds[:-1], bounds[1:]):
            p = positions[a:b]
            if p['major'][0] != region.start or p['major'][-1] + 1 != region.end:
                self.logger.warning('Pileup counts do not span requested region, requested {}, received {}-{}.'.format(
                    region, p['major'][0], p['major'][-1]))
            samples.append(common.Sample(ref_name=region.ref_name, features=feats[a:b], labels=None, ref_seq=None,
                                         positions=p, label_probs=None, depth=depth[a:b]))
        return samples

    def bam_to_sample(self, reads_bam, region):
        """Convert a section of an alignment pileup to samples (features.py:770-798)."""
        if self._fused_featuriser and self.pileup_source is None:
            fused = self._fused_samples(reads_bam, region)
            if fused is not None:
                return fused
        samples = []
        for counts, positions in self._pileup_function(region, reads_bam):
            if len(counts) == 0:
                self.logger.warning(
                    'Pileup-feature is zero-length for {} indicating no reads in this region.'.format(region))
                samples.append(common.Sample(
                    ref_name=region.ref_name, features=None, labels=None, ref_seq=None,
                    positions=positions, label_probs=None, depth=None))
                continue
            samples.append(self._post_process_pileup(counts, positions, region))
        return samples

    def bams_to_training_samples(self, truth_bam, bam, region, label_scheme, truth_haplotag=None, min_length=1000):
        """Labelled samples of a region (medaka/features.py:937-994): per filtered truth alignment, the samples of the
        reads over its trimmed span, each column labelled from the truth on the GPU (0, the padding vector, where the
        truth has no position; truth positions without a column are dropped).

        :param truth_bam: BAM (path or ``bam.BamFile``) of the truth aligned to the draft.
        :param bam: BAM of the reads.  :param label_scheme: a ``labels.HaploidLabelScheme``.
        :param truth_haplotag: tag grouping the truth alignments by haplotype.
        :param min_length: shortest truth alignment kept.
        :returns: tuple of ``common.Sample`` with int64 labels.
        """
        from medaka_b200 import labels
        if not isinstance(label_scheme, labels.HaploidLabelScheme):
            raise NotImplementedError("training labels are implemented for the HaploidLabelScheme only")
        alns = labels.TruthAlignment.bam_to_alignments(truth_bam, region, haplotag=truth_haplotag,
                                                       min_length=min_length)
        if len(alns) == 0:
            self.logger.info("Filtering and grouping removed all alignments of truth to ref from {}.".format(region))
        for aln in alns:
            if len(aln) != label_scheme.n_elements:
                raise ValueError('{} alignments were passed to {}, requires {}'.format(
                    len(aln), type(label_scheme).__name__, label_scheme.n_elements))
        samples = []
        for aln in alns:
            for sample in self.bam_to_sample(bam, common.Region(region.ref_name, aln[0].start, aln[0].end)):
                samples.append(sample.amend(labels=label_scheme.label_columns(aln, sample.positions)))
        return tuple(samples)


# ---------------------------------------------------------------------------------------------------------
# Read-level features (medaka/features.py:258-560, 1100-1205): one int8 vector per (pileup column, read row).

def read_matrix_from_batch(batch, start, end, num_dtypes=1, min_mapq=1, row_per_read=False, include_dwells=False,
                           include_haplotype=False, max_reads=100, device=0):
    """calculate_read_alignment over a ``RecordBatch`` fetched with names, qualities and raw aux fields
    (mdk_read_matrix).  Returns (matrix int8 [n_cols, n_reads, featlen] - not clipped -, positions,
    (read_ids_left, read_ids_right)) like ``_read_matrix_data_to_numpy`` (medaka/features.py:322-389)."""
    lib, ffi = _lm.load(), _lm.ffi
    n_rec = len(batch.pos)
    featlen = 4 + (1 if include_dwells else 0) + (1 if include_haplotype else 0) + (1 if num_dtypes > 1 else 0)
    names = batch.names if batch.names is not None else ["r%d" % i for i in range(n_rec)]
    enc = [nm.encode() for nm in names]
    name_off = np.zeros(n_rec + 1, dtype=np.int64)
    np.cumsum([len(b) for b in enc], out=name_off[1:])
    names_raw = b"".join(enc) or b"\x00"
    l_seq = np.ascontiguousarray(batch.l_seq, np.int64)
    qual_off = np.zeros(n_rec + 1, dtype=np.int64)
    np.cumsum(l_seq, out=qual_off[1:])
    qual = batch.qual if batch.qual is not None else np.full(int(qual_off[-1]), 0xFF, dtype=np.uint8)
    aux = batch.aux if batch.aux is not None else np.zeros(0, dtype=np.uint8)
    aux_off = batch.aux_off if batch.aux_off is not None else np.zeros(n_rec + 1, dtype=np.int64)
    records = _record_args(batch)
    arrs = dict(qual=np.ascontiguousarray(qual, np.uint8), qoff=qual_off,
                aux=np.ascontiguousarray(aux, np.uint8) if len(aux) else np.zeros(1, dtype=np.uint8),
                aoff=np.ascontiguousarray(aux_off, np.int64))
    n_cols, n_reads = ffi.new("int64_t *"), ffi.new("int32_t *")
    max_cols, max_reads_buf = 0, 0                  # first call sizes the outputs (enlarge_read_aln_data_*), second fills
    matrix = major = minor = left = right = None
    for _ in range(3):
        matrix = np.zeros((max_cols, max_reads_buf, featlen), dtype=np.int8)
        major = np.zeros(max_cols, dtype=np.int64)
        minor = np.zeros(max_cols, dtype=np.int64)
        left = np.full(max(max_reads_buf, 1), -2, dtype=np.int32)
        right = np.full(max(max_reads_buf, 1), -2, dtype=np.int32)
        rc = lib.mdk_read_matrix(
            device, n_rec, *records,
            ffi.cast("const uint8_t *", ffi.from_buffer(arrs["qual"])),
            ffi.cast("const int64_t *", ffi.from_buffer(arrs["qoff"])),
            ffi.cast("const uint8_t *", ffi.from_buffer(arrs["aux"])),
            ffi.cast("const int64_t *", ffi.from_buffer(arrs["aoff"])),
            ffi.from_buffer(names_raw), ffi.cast("const int64_t *", ffi.from_buffer(name_off)),
            int(start), int(end), num_dtypes, int(min_mapq), 1 if row_per_read else 0, 1 if include_dwells else 0,
            1 if include_haplotype else 0, int(max_reads), max_cols, matrix.size,
            ffi.cast("int8_t *", ffi.from_buffer(matrix)) if matrix.size else ffi.NULL,
            ffi.cast("int64_t *", ffi.from_buffer(major)) if max_cols else ffi.NULL,
            ffi.cast("int64_t *", ffi.from_buffer(minor)) if max_cols else ffi.NULL, n_cols, n_reads,
            ffi.cast("int32_t *", ffi.from_buffer(left)), ffi.cast("int32_t *", ffi.from_buffer(right)))
        if rc == lib.MDK_ERR_NOMEM and (n_cols[0] != max_cols or n_reads[0] != max_reads_buf):
            max_cols, max_reads_buf = int(n_cols[0]), int(n_reads[0])
            continue
        _lm.check(rc)
        break
    n, d = int(n_cols[0]), int(n_reads[0])
    positions = _positions(major, minor, n)
    matrix = matrix[:n, :d]

    def ids(idx):
        out, blanks = [], 0
        for i in idx[:d]:
            if i >= 0:
                out.append(enc[int(i)])
            elif i == -1:
                blanks += 1
                out.append(("__blank_%d" % blanks).encode())
            else:
                out.append(b"")
        return np.array(out, dtype="S") if out else np.zeros(0, dtype="S1")
    return matrix, positions, (ids(left), ids(right))


def _align_rows(chunks, read_ids):
    """Rows of consecutive sub-region results lined up on read identity (the reference's ``_reorder_reads``,
    medaka/features.py:411-467): a read that leaves chunk n-1 through row r enters chunk n in row r; rows of chunk n that
    continue nothing fill the vacated rows in ascending order, the rest are appended."""
    if len(chunks) == 1:
        return chunks
    ids_in = [list(r[0]) for r in read_ids]
    ids_out = [list(r[1]) for r in read_ids]
    aligned = [chunks[0]]
    for n in range(1, len(chunks)):
        chunk, leaving, entering = chunks[n], ids_out[n - 1], ids_in[n]
        where = {}
        for j, rid in enumerate(entering):
            where.setdefault(rid, j)                    # first match wins
        src = np.array([where.get(rid, -1) for rid in leaving], dtype=np.int64)
        vacant = [i for i, j in enumerate(src) if j == -1]
        used = set(int(j) for j in src if j != -1)
        unplaced = [j for j in range(len(entering)) if j not in used]
        for i, j in zip(vacant, unplaced):
            src[i] = j
        if len(unplaced) > len(vacant):
            src = np.concatenate([src, np.array(unplaced[len(vacant):], dtype=np.int64)])
        out = np.zeros((chunk.shape[0], max(len(leaving), len(entering)), chunk.shape[2]), dtype=chunk.dtype)
        out[:, src != -1, :] = chunk[:, src[src != -1], :]
        aligned.append(out)
        if n < len(chunks) - 1:
            renamed, k = [], 1
            for j in src:
                if j == -1:
                    renamed.append(("__inserted_%d" % k).encode())
                    k += 1
                else:
                    renamed.append(ids_out[n][int(j)])
            ids_out[n] = renamed
    return aligned


def _pad_rows(chunks):
    depth = max(c.shape[1] for c in chunks)
    return [np.concatenate([c, np.zeros((c.shape[0], depth - c.shape[1], c.shape[2]), dtype=c.dtype)], axis=1)
            for c in chunks]


def _join_read_matrix_chunks(results):
    """Split sub-region results at coverage gaps and join abutting ones (the reference's
    ``__enforce_read_matrix_chunk_contiguity``, medaka/features.py:470-557)."""
    pieces = []
    for matrix, positions, read_ids in results:
        cuts = np.where(np.ediff1d(positions['major']) > 1)[0] + 1
        if len(cuts) == 0:
            pieces.append((matrix, positions, read_ids))
            continue
        # (the reference names the placeholders after the LAST sub-region's read ids seen so far; only their count and
        # mutual distinctness matter: placeholders never match a real read name)
        holder = np.array([("__placeholder_%d" % m).encode() for m in range(len(read_ids[0]))])
        bounds = [0] + cuts.tolist() + [len(positions)]
        for k, (a, b) in enumerate(zip(bounds[:-1], bounds[1:])):
            first, last = k == 0, k == len(bounds) - 2
            pieces.append((matrix[a:b], positions[a:b], (read_ids[0] if first else holder, read_ids[1] if last else holder)))
    joined, buf, last_major = [], [], None

    def flush():
        mats = _pad_rows(_align_rows([b[0] for b in buf], [b[2] for b in buf]))
        joined.append((np.concatenate(mats), np.concatenate([b[1] for b in buf])))
    for matrix, positions, read_ids in pieces:
        if len(positions) == 0:
            continue
        if buf and positions['major'][0] - last_major != 1:
            flush()
            buf = []
        buf.append((matrix, positions, read_ids))
        last_major = positions['major'][-1]
    if buf:
        flush()
    return joined


def read_alignment_matrix(region, bam, dtype_prefixes=None, region_split=100000, workers=8, tag_name=None, tag_value=None,
                          keep_missing=False, read_group=None, min_mapq=1, row_per_read=False, include_dwells=False,
                          include_haplotype=False, max_reads=100, clip_to_zero=True, device=0):
    """Read-level feature array for a region - the reference's ``read_alignment_matrix`` (medaka/features.py:258-319):
    the region is cut into ``region_split`` sub-regions exactly as the reference does (the row bookkeeping restarts in
    each, so the cut points are part of the result), each is built on the GPU (mdk_read_matrix), and abutting
    sub-region results are joined on read identity.  Returns a list of (matrix, positions) chunks."""
    from medaka_b200 import bam as mbam
    if tag_name is not None and len(tag_name) != 2:
        raise ValueError("'tag_name' must be a length-2 string.")
    if not isinstance(bam, mbam.BamFile):
        bam = mbam.BamFile(bam)
    multi = not (dtype_prefixes is None or isinstance(dtype_prefixes, str) or len(dtype_prefixes) == 1)
    num_dtypes = len(dtype_prefixes) if multi else 1

    def one(reg):
        batch = bam.fetch(reg.ref_name, reg.start, reg.end, dtypes=dtype_prefixes if multi else None, tag_name=tag_name,
                          tag_value=tag_value, keep_missing=keep_missing, read_group=read_group, min_mapq=min_mapq,
                          with_names=True, with_qual=True, with_aux=True)
        matrix, positions, read_ids = read_matrix_from_batch(
            batch, reg.start, reg.end, num_dtypes, min_mapq, row_per_read, include_dwells, include_haplotype, max_reads,
            device)
        if clip_to_zero:
            matrix = np.maximum(matrix, 0)
        return matrix, positions, read_ids
    regions = region.split(region_split, fixed_size=False)
    with concurrent.futures.ThreadPoolExecutor(max_workers=max(1, workers)) as ex:
        results = list(ex.map(one, regions))
    return _join_read_matrix_chunks(results)


class ReadAlignmentFeatureEncoder(CountsFeatureEncoder):
    """Read-level feature tensors (positions, reads, features) - medaka/features.py:1100-1205.  Features per read and
    position: [base, baseQ, strand, mapQ (, dwell) (, haplotype) (, datatype)]; bases 0-5 = [pad, A, C, G, T, deletion]."""

    feature_dtype = np.int8
    _fused_featuriser = False

    def __init__(self, dtypes=('',), tag_name=None, tag_value=None, tag_keep_missing=False, read_group=None,
                 min_mapq=1, max_reads=100, row_per_read=False, include_dwells=True, include_haplotype=False,
                 pileup_source=None, device=0):
        self.max_reads = max_reads
        self.row_per_read = row_per_read
        self.include_dwells = include_dwells
        self.include_haplotype = include_haplotype
        super().__init__(normalise=None, dtypes=dtypes, tag_name=tag_name, tag_value=tag_value,
                         tag_keep_missing=tag_keep_missing, read_group=read_group, min_mapq=min_mapq,
                         pileup_source=pileup_source, device=device)

    _state_fields = CountsFeatureEncoder._state_fields + ('max_reads', 'row_per_read', 'include_dwells',
                                                          'include_haplotype')

    @property
    def feature_vector_length(self):
        return 4 + (1 if self.include_dwells else 0) + (1 if self.include_haplotype else 0) + (
            1 if len(self.dtypes) > 1 else 0)

    def _pileup_function(self, region, bam):
        if self.pileup_source is not None:
            return self.pileup_source(region, bam, self)
        return read_alignment_matrix(
            region, bam, dtype_prefixes=self.dtypes, tag_name=self.tag_name, tag_value=self.tag_value,
            keep_missing=self.tag_keep_missing, read_group=self.read_group, min_mapq=self.min_mapq,
            row_per_read=self.row_per_read, include_dwells=self.include_dwells,
            include_haplotype=self.include_haplotype, max_reads=self.max_reads, device=self.device)

    def _post_process_pileup(self, features, positions, region):
        if features.ndim == 2:
            depth = np.count_nonzero(features, axis=-1)
        elif features.ndim == 3:
            depth = np.count_nonzero(features[..., 0], axis=-1)
        else:
            raise ValueError("Unknown feature dimension size of {}. Should be either 2 (counts matrices) or 3 "
                             "(for read level features).".format(features.ndim))
        return common.Sample(ref_name=region.ref_name, features=features, labels=None, ref_seq=None,
                             positions=positions, label_probs=None, depth=depth)


class SampleGenerator(object):
    """Chunked inference or training samples for one region (medaka/features.py:1208-1313).  With ``truth_bam`` the
    samples are labelled (``bams_to_training_samples`` of the encoder with ``label_scheme``, ``truth_haplotag`` and
    ``min_truth_length``)."""

    def __init__(self, bam, region, feature_encoder, chunk_len=1000, chunk_overlap=200,
                 enable_chunking=True, truth_bam=None, label_scheme=None, truth_haplotag=None, min_truth_length=1000):
        self.logger = common.get_named_logger("Sampler")
        self.fencoder = feature_encoder
        self.bam = bam
        self.region = region
        self.chunk_len = chunk_len
        self.chunk_overlap = chunk_overlap
        self.enable_chunking = enable_chunking
        self.truth_bam = truth_bam
        self.label_scheme = label_scheme
        self.truth_haplotag = truth_haplotag
        self.min_truth_length = min_truth_length
        self._source = None
        self._quarantined = list()     # (Region, pileup width) of sources narrower than chunk_len
        if self.truth_bam is not None and self.label_scheme is None:
            raise ValueError("A `LabelScheme` must be given to create training data.")

    def _fill_features(self):
        if self._source is None:
            t0 = now()
            if self.truth_bam is not None:
                self._source = self.fencoder.bams_to_training_samples(
                    self.truth_bam, self.bam, self.region, self.label_scheme, truth_haplotag=self.truth_haplotag,
                    min_length=self.min_truth_length)
            else:
                self._source = self.fencoder.bam_to_sample(self.bam, self.region)
            self.logger.debug("Took {:.2f}s to make features.".format(now() - t0))

    @property
    def samples(self):
        """List of (possibly) chunked samples; short sources are quarantined (features.py:1283-1313)."""
        self._fill_features()
        self._quarantined = list()
        out = []
        for source in self._source:
            if source.is_empty:
                continue
            if not self.enable_chunking:
                out.append(source)
                continue
            if source.size < self.chunk_len:
                start, end = source.first_pos[0], source.last_pos[0] + 1
                self._quarantined.append((common.Region(source.ref_name, start, end), source.size))
                continue
            out.extend(source.chunks(chunk_len=self.chunk_len, overlap=self.chunk_overlap))
        return out


def _bam_regions(bam, regions=None):
    """The regions to process, with integer bounds clipped to the contigs (medaka/common.py:762-790): every contig of
    the BAM, or the given ``Region``s / region strings.  KeyError for a contig the BAM does not have."""
    from medaka_b200 import bam as mbam
    bf = bam if isinstance(bam, mbam.BamFile) else mbam.BamFile(bam)
    lengths = dict(bf.get_regions())
    if regions is None:
        return [common.Region(name, 0, length) for name, length in lengths.items()]
    out = []
    for r in regions:
        r = common.Region.from_string(r) if isinstance(r, str) else r
        if r.ref_name not in lengths:
            raise KeyError('Contig {} is not one of the bam references.'.format(r.ref_name))
        start = max(0, r.start) if r.start is not None else 0
        end = min(r.end, lengths[r.ref_name]) if r.end is not None else lengths[r.ref_name]
        out.append(common.Region(r.ref_name, start, end))
    return out


MAX_REGION_SIZE = 1000000     # regions are processed in pieces of this size (medaka/features.py:1390)


def create_samples(bam, output, regions=None, truth=None, truth_haplotag=None, feature_encoder=None,
                   label_scheme='HaploidLabelScheme', chunk_len=10000, chunk_ovlp=1000, min_region_size=0):
    """`medaka features`: chunked samples of the regions, labelled from the truth alignments in ``truth`` when it is
    given, written to a ``DataStore`` with ``feature_encoder`` and ``label_scheme`` meta (medaka/features.py:1316-1414).

    :param bam: BAM of the reads.  :param output: the store to write (deleted again when no sample is written).
    :param regions: ``Region``s or region strings (default: every contig of ``bam``); each is processed in 1 Mb
        pieces (``Region.split``, whose last piece overlaps the one before; a sample already written is not written
        again).  Regions shorter than ``min_region_size`` are skipped.
    :param truth: BAM of the truth aligned to the draft, or None for unlabelled samples.
    :param feature_encoder: a ``CountsFeatureEncoder`` or ``ReadAlignmentFeatureEncoder`` (default: counts, total
        normalisation).  :param label_scheme: a ``labels.HaploidLabelScheme`` or its class name.
    :param chunk_len, chunk_ovlp: sample length and overlap; sources shorter than ``chunk_len`` are not written.
    :returns: the number of samples in the store.
    """
    import os
    import shutil
    from medaka_b200 import datastore, labels
    logger = common.get_named_logger('Prepare')
    if chunk_ovlp >= chunk_len:
        raise ValueError('chunk_ovlp {} is not smaller than chunk_len {}'.format(chunk_ovlp, chunk_len))
    if isinstance(label_scheme, str):
        label_scheme = labels.from_name(label_scheme)
    if feature_encoder is None:
        feature_encoder = CountsFeatureEncoder()
    pieces = []
    for r in _bam_regions(bam, regions):
        if r.size < min_region_size:
            logger.warning("Region {} is smaller than min region size {}, skipping.".format(r, min_region_size))
            continue
        pieces.extend(r.split(MAX_REGION_SIZE))
    if truth is None:
        logger.warning('Running medaka features without a truth bam, unlabelled data will be produced.')
    with datastore.DataStore(output, 'w') as ds:
        ds.set_meta(feature_encoder, 'feature_encoder')
        ds.set_meta(label_scheme, 'label_scheme')
        for reg in pieces:
            samples = SampleGenerator(bam, reg, feature_encoder, chunk_len=chunk_len, chunk_overlap=chunk_ovlp,
                                      truth_bam=truth, label_scheme=label_scheme,
                                      truth_haplotag=truth_haplotag).samples
            logger.info("Writing {} samples for region {}".format(len(samples), reg))
            for sample in samples:
                ds.write_sample(sample)
        n_samples = ds.n_samples
    if n_samples == 0:
        logger.critical("Warning: No training data was written to file, deleting output.")
        if os.path.isdir(output):
            shutil.rmtree(output)
        elif os.path.exists(output):
            os.remove(output)
    return n_samples
