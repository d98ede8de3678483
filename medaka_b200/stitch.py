"""Consensus stitching: network outputs of a region -> contiguous sequences (medaka/stitch.py).

The reference streams `Sample` views through four generators (trim overlaps -> trim to region -> depth filter ->
trim again, medaka/common.py:495-644) and decodes each surviving view on the CPU (stitch.py:33-85).  None of the
views ever changes a probability, so here the stream is reduced to a *plan*: a list of `Piece(sample, lo, hi)` row
ranges plus the contig breaks, computed from positions / depths only.  The ranges of a whole region then go to the
GPU in one call (libmedaka_b200 `mdk_stitch_consensus`): only the kept rows are copied in, decoded (argmax + phred),
gap calls are removed by a stable compaction, and the bytes that come back are the FASTA/FASTQ text.

``sequence`` is `medaka sequence` (medaka/stitch.py:197-309) over this package's stores; ``write_consensus`` is its
body, shared with the one-pass ``prediction.predict_consensus``, whose decoded calls never leave the device
(``decode_label_pieces``, libmedaka_b200 `mdk_stitch_labels_dev`).
"""
import collections
import functools
import itertools

import numpy as np

from medaka_b200 import libmedaka as _lm
from medaka_b200.common import OverlapException, Region, Relationship, Sample, get_named_logger

# stitch regions are at most this long (medaka/stitch.py:219)
MAX_REGION_SIZE = int(1e6)

Piece = collections.namedtuple('Piece', 'sample lo hi last heuristic')
Piece.__doc__ = "rows [lo, hi) of samples[sample]; `last` closes a contig; `heuristic` = junction search was used"

# a junction is only searched for when both sides of the overlap span more than this many major positions
_MIN_JUNCTION_MAJORS = 3


def _keys(positions):
    """(major, minor) -> one sortable int64 per column."""
    return (positions['major'].astype(np.int64) << 24) | positions['minor'].astype(np.int64)


def _key(major, minor):
    return (int(major) << 24) | int(minor)


def junction(pos1, pos2):
    """Cut points for two forward-overlapping position arrays (semantics of medaka/common.py:327-427).

    :returns: (end1, start2, heuristic) such that pos1[:end1] followed by pos2[start2:] has no overlap and no gap.

    When both samples list the same columns across the overlap the cut is its mid-point.  Otherwise (the pileups
    disagreed on insertion columns) the cut goes to the major position closest to the middle of the overlap - trying
    mid+1, mid-1, mid+2, ... - that carries the same number of columns in both samples.
    """
    k1, k2 = _keys(pos1), _keys(pos2)
    a = int(np.searchsorted(k1, k2[0], side='left'))       # first column of pos1 inside the overlap
    b = int(np.searchsorted(k2, k1[-1], side='right'))     # one past the last column of pos2 inside it
    n = len(k1) - a
    if n == b and np.array_equal(pos1['minor'][a:], pos2['minor'][:b]):
        half = n // 2
        return a + half, b - (n - half), False
    maj1, maj2 = pos1['major'], pos2['major']
    ov1, ov2 = maj1[a:], maj2[:b]
    # majors are sorted, so the number of distinct ones is 1 + the number of steps
    if (1 + np.count_nonzero(np.diff(ov1)) > _MIN_JUNCTION_MAJORS
            and 1 + np.count_nonzero(np.diff(ov2)) > _MIN_JUNCTION_MAJORS):
        mid = int(ov1[0]) + (int(ov1[-1]) - int(ov1[0])) // 2
        top, bottom = int(maj1[-1]), int(maj2[0])
        for step in itertools.count(1):
            if mid + step > top and mid - step < bottom:
                break
            for major in (mid + step, mid - step):
                l0, l1 = np.searchsorted(maj1, [major, major + 1])
                r0, r1 = np.searchsorted(maj2, [major, major + 1])
                if l1 - l0 == r1 - r0:
                    if l1 == l0:
                        raise OverlapException("junction search left both samples at major {}".format(major))
                    return int(l0), int(r0), True
    raise OverlapException("Could not find viable junction")


def _trim_overlaps(views):
    """views: list of (sample_index, lo, hi, Sample-like with positions/ref_name restricted to [lo,hi)).

    Removes the overlap between consecutive views and marks contig ends; yields Piece tuples.
    """
    pieces = []
    if not views:
        return pieces
    cur = views[0]
    cur_lo = 0
    for nxt in views[1:] + [None]:
        heuristic, last, nxt_lo = False, False, 0
        idx, lo, hi, s = cur
        n = hi - lo
        cur_hi = n
        if nxt is None:
            last = True
        else:
            rel = Sample.relative_position(s, nxt[3])
            if rel is Relationship.s2_within_s1:
                continue
            if rel is Relationship.forward_gapped:
                last = True
            elif rel is Relationship.forward_abutted:
                pass
            elif rel is Relationship.forward_overlap:
                cur_hi, nxt_lo, heuristic = junction(s.positions, nxt[3].positions)
            else:
                raise OverlapException("Cannot overlap samples {} and {} with relationship {!r}".format(
                    s.name, nxt[3].name, rel))
        pieces.append(Piece(idx, lo + cur_lo, lo + cur_hi, last, heuristic))
        cur, cur_lo = nxt, nxt_lo
    return pieces


def _view(samples, idx, lo, hi):
    s = samples[idx]
    if lo == 0 and hi == len(s.positions):
        return (idx, lo, hi, s)
    return (idx, lo, hi, Sample(ref_name=s.ref_name, features=None, labels=None, ref_seq=None,
                                positions=s.positions[lo:hi], label_probs=None, depth=None))


def plan_pieces(samples, start=None, end=None, min_depth=0):
    """Which rows of which samples make up the consensus of [start, end) - everything `_stitch_samples` decides before
    it decodes (medaka/stitch.py:48-52).

    :param samples: list of Sample (same reference sequence, in genomic order as stored).
    :returns: list of Piece, in output order.
    """
    samples = list(samples)
    pieces = _trim_overlaps([_view(samples, i, 0, len(s.positions)) for i, s in enumerate(samples)])
    clipped = []
    for p in pieces:
        major = samples[p.sample].positions['major']
        lo, hi = p.lo, p.hi
        if hi <= lo:
            raise OverlapException("empty sample after overlap trimming: {}".format(samples[p.sample].name))
        if start is not None:
            if major[hi - 1] < start:
                continue
            if major[lo] < start:
                lo += int(np.searchsorted(major[lo:hi], start, side='left'))
        if end is not None:
            if major[lo] >= end:
                break
            if major[hi - 1] >= end:
                hi = lo + int(np.searchsorted(major[lo:hi], end, side='left'))
        if hi > lo:
            clipped.append(p._replace(lo=lo, hi=hi))
    if not min_depth:
        return clipped
    # depth filter: runs of sufficient depth become views of their own and the contig breaks are recomputed from
    # how those runs sit relative to each other (abutting -> same contig, gap -> new contig)
    views = []
    for p in clipped:
        ok = np.asarray(samples[p.sample].depth[p.lo:p.hi]) >= min_depth
        edges = np.flatnonzero(np.diff(ok.astype(np.int8))) + 1
        bounds = np.concatenate(([0], edges, [len(ok)]))
        for a, b in zip(bounds[:-1], bounds[1:]):
            if ok[a]:
                views.append(_view(samples, p.sample, p.lo + int(a), p.lo + int(b)))
    return _trim_overlaps(views)


def decode_pieces(samples, pieces, device=0, with_qualities=True):
    """Decode + gap-strip all pieces in one device call.  -> (list of str, list of str or None), one per piece."""
    if not pieces:
        return [], ([] if with_qualities else None)
    lib, ffi = _lm.load(), _lm.ffi
    keep = []          # arrays whose memory the pointer table refers to
    ptrs = ffi.new("const float *[]", len(pieces))
    rows = np.empty(len(pieces), dtype=np.int64)
    for k, p in enumerate(pieces):
        probs = samples[p.sample].label_probs
        probs = probs.detach().cpu().numpy() if hasattr(probs, "detach") else np.asarray(probs)
        if probs.ndim != 2 or probs.shape[1] != 5:
            raise ValueError("expected label probabilities [n, 5], got shape {}".format(probs.shape))
        part = np.ascontiguousarray(probs[p.lo:p.hi], dtype=np.float32)
        keep.append(part)
        ptrs[k] = ffi.cast("const float *", ffi.from_buffer(part))
        rows[k] = part.shape[0]
    total = int(rows.sum())
    seq = np.empty(total, dtype=np.uint8)
    qual = np.empty(total, dtype=np.uint8) if with_qualities else None
    off = np.empty(len(pieces) + 1, dtype=np.int64)
    _lm.check(lib.mdk_stitch_consensus(
        device, ptrs, ffi.cast("const int64_t *", ffi.from_buffer(rows)), len(pieces),
        ffi.cast("uint8_t *", ffi.from_buffer(seq)),
        ffi.cast("uint8_t *", ffi.from_buffer(qual)) if with_qualities else ffi.NULL,
        ffi.cast("int64_t *", ffi.from_buffer(off))))
    return _split_text(seq, qual, off)


def decode_label_pieces(labels_dev, quals_dev, seg_start, seg_rows, device=0):
    """Gap-strip row ranges of decoded calls already on the device (mdk_stitch_labels_dev).

    :param labels_dev, quals_dev: device addresses (int) of the uint8 labels and phred+33 bytes (quals_dev may be None).
    :param seg_start, seg_rows: range k is rows [seg_start[k], seg_start[k] + seg_rows[k]) of both arrays.
    :returns: (list of str, list of str or None), one per range.
    """
    n = len(seg_start)
    if n == 0:
        return [], ([] if quals_dev is not None else None)
    lib, ffi = _lm.load(), _lm.ffi
    starts = np.ascontiguousarray(seg_start, dtype=np.int64)
    rows = np.ascontiguousarray(seg_rows, dtype=np.int64)
    total = int(rows.sum())
    seq = np.empty(total, dtype=np.uint8)
    qual = np.empty(total, dtype=np.uint8) if quals_dev is not None else None
    off = np.empty(n + 1, dtype=np.int64)
    _lm.check(lib.mdk_stitch_labels_dev(
        device, ffi.cast("const uint8_t *", labels_dev),
        ffi.cast("const uint8_t *", quals_dev) if quals_dev is not None else ffi.NULL,
        ffi.cast("const int64_t *", ffi.from_buffer(starts)), ffi.cast("const int64_t *", ffi.from_buffer(rows)), n,
        ffi.cast("uint8_t *", ffi.from_buffer(seq)),
        ffi.cast("uint8_t *", ffi.from_buffer(qual)) if qual is not None else ffi.NULL,
        ffi.cast("int64_t *", ffi.from_buffer(off))))
    return _split_text(seq, qual, off)


def _split_text(seq, qual, off):
    """The stitch's concatenated output -> one str per range (and the qualities, or None)."""
    n = len(off) - 1
    seq_txt = seq[:off[-1]].tobytes().decode('ascii')
    seqs = [seq_txt[off[k]:off[k + 1]] for k in range(n)]
    quals = None
    if qual is not None:
        qual_txt = qual[:off[-1]].tobytes().decode('ascii')
        quals = [qual_txt[off[k]:off[k + 1]] for k in range(n)]
    return seqs, quals


def stitch_samples(samples, label_scheme=None, region=None, min_depth=0, device=0, decode=None):
    """Drop-in for `medaka.stitch._stitch_samples` (stitch.py:33-85).

    :param samples: iterable of Sample with positions, label_probs (and depth when min_depth is used).
    :param label_scheme: accepted for signature compatibility (the haploid '*ACGT' decoding is what the library does).
    :param region: object with .start / .end (either may be None) or None.
    :param decode: ``decode(samples, pieces) -> (seqs, quals)``; default ``decode_pieces`` on the samples' label_probs.
    :returns: list of ((ref_name, first major, last major), [sequence parts], [quality parts]).
    """
    samples = list(samples)
    start = getattr(region, 'start', None)
    end = getattr(region, 'end', None)
    pieces = plan_pieces(samples, start, end, min_depth)
    seqs, quals = (decode or functools.partial(decode_pieces, device=device))(samples, pieces)
    logger = get_named_logger('Stitch')
    logger.debug("Used heuristic {} times for {}.".format(sum(p.heuristic for p in pieces), region))
    contigs = []
    first = 0
    for k, p in enumerate(pieces):
        if p.last or k == len(pieces) - 1:
            s0, s1 = samples[pieces[first].sample], samples[p.sample]
            name = (s1.ref_name, int(s0.positions['major'][pieces[first].lo]), int(s1.positions['major'][p.hi - 1]))
            contigs.append((name, seqs[first:k + 1], quals[first:k + 1]))
            first = k + 1
    return contigs


def collapse_neighbours(contigs):
    """Join contigs that continue each other (stitch.py:168-196): same reference, start == previous stop + 1."""
    merged = None
    for (ref, start, stop), seq_parts, qual_parts in contigs:
        if merged is not None and merged[0][0] == ref and start == merged[0][2] + 1:
            merged = ((ref, merged[0][1], stop), merged[1] + list(seq_parts), merged[2] + list(qual_parts))
            continue
        if merged is not None:
            yield merged
        merged = ((ref, start, stop), list(seq_parts), list(qual_parts))
    if merged is not None:
        yield merged


def fill_gaps(contigs, draft, fill_char=None):
    """Pad the stitched pieces of every reference to full length (stitch.py:109-165).

    :param contigs: iterable of ((ref_name, start, stop inclusive), sequence parts, quality parts).
    :param draft: dict ref_name -> draft sequence (str).
    :param fill_char: None / '' -> fill with draft sequence, else the first character is repeated.
    :returns: (list of ((ref_name, 0, length), seq parts, qual parts), dict ref_name -> list of (gap start, gap end)).
    """
    fill_char = None if fill_char in (None, "") else str(fill_char)[0]
    by_ref = collections.OrderedDict()
    for (ref, start, stop), seq_parts, qual_parts in contigs:
        by_ref.setdefault(ref, []).append((int(start), int(stop) + 1, seq_parts, qual_parts))
    out, gaps = [], {}
    for ref, items in by_ref.items():
        text = draft[ref]
        items.sort(key=lambda x: x[0])
        seqs, quals, cursor, holes = [], [], 0, []

        def pad(a, b):
            holes.append((a, b))
            seqs.append(text[a:b] if fill_char is None else fill_char * (b - a))
            quals.append('!' * (b - a))

        for start, stop, seq_parts, qual_parts in items:
            if start > cursor:
                pad(cursor, start)
            seqs.extend(seq_parts)
            quals.extend(qual_parts)
            cursor = max(cursor, stop)
        if cursor < len(text):
            pad(cursor, len(text))
        out.append(((ref, 0, len(text)), seqs, quals))
        gaps[ref] = holes
    return out, gaps


def write_fastx_segment(fh, contig, qualities=True):
    """(name, sequence parts, quality parts) -> one FASTA or FASTQ record (stitch.py:16-31)."""
    fh.write('{}{}\n{}\n'.format('@' if qualities else '>', contig[0], ''.join(contig[1])))
    if qualities:
        fh.write('+\n{}\n'.format(''.join(contig[2])))


def read_fasta(path):
    """Minimal FASTA reader -> OrderedDict name -> sequence (stands in for pysam.FastaFile in fill_gaps)."""
    seqs = collections.OrderedDict()
    name, parts = None, []
    with open(path) as fh:
        for line in fh:
            line = line.rstrip('\n')
            if line.startswith('>'):
                if name is not None:
                    seqs[name] = ''.join(parts)
                name, parts = line[1:].split()[0], []
            elif line:
                parts.append(line)
    if name is not None:
        seqs[name] = ''.join(parts)
    return seqs


def sample_index(names):
    """Sample names -> OrderedDict ref_name -> list of sample names in stitch order (medaka/datastore.py:453-485):
    reference names sorted, a reference's samples by start (major, minor), then by descending end."""
    by_ref = collections.defaultdict(list)
    for name in names:
        d = Sample.decode_sample_name(name)
        if d is not None:
            by_ref[d['ref_name']].append((name, d['start'], d['end']))

    def major_minor(x):
        return tuple(int(i) for i in x.split('.'))

    def sorter(item):
        return major_minor(item[1]) + tuple(-i for i in major_minor(item[2]))

    return collections.OrderedDict((ref, [x[0] for x in sorted(by_ref[ref], key=sorter)]) for ref in sorted(by_ref))


def select_samples(index, region):
    """Names of the indexed samples overlapping ``region``, in index order (medaka/datastore.py:504-515): a sample
    covers the draft positions [int(start major), int(end major) + 1)."""
    out = []
    for name in index.get(region.ref_name, ()):
        d = Sample.decode_sample_name(name)
        if Region(d['ref_name'], int(float(d['start'])), int(float(d['end'])) + 1).overlaps(region):
            out.append(name)
    return out


def plan_regions(index, draft_lengths, regions=None):
    """The stitch regions of a run (medaka/stitch.py:206-233) and the requested contigs without samples.

    :param regions: Regions or region strings to stitch; default every draft contig.  A missing start / end means the
        contig's start / end.
    :returns: (list of Region of at most MAX_REGION_SIZE, in request order; list of contig names absent from the index).
    """
    if regions is None:
        regions = [Region(name, None, None) for name in draft_lengths]
    todo, missing = [], []
    for r in regions:
        ref, start, end = Region.from_string(r) if isinstance(r, str) else r
        if ref not in index:
            if ref not in missing:
                missing.append(ref)
            continue
        start = 0 if start is None else start
        end = draft_lengths[ref] if end is None else end
        todo.extend(Region(ref, start, end).split(MAX_REGION_SIZE, overlap=0, fixed_size=False))
    return todo, missing


def write_bed(gaps, path):
    """Gap intervals -> bed (medaka/common.py write_intervaltrees_to_bed): contigs sorted, intervals sorted."""
    with open(path, 'w') as fh:
        for ref in sorted(gaps):
            for a, b in sorted(gaps[ref]):
                fh.write("{}\t{}\t{}\n".format(ref, a, b))


def write_consensus(index, load, draft, output, regions=None, min_depth=0, fillgaps=True, fill_char=None,
                    qualities=True, decode=None, device=0):
    """The serial body of `medaka sequence` (medaka/stitch.py:197-309) over any sample source.

    :param index: ``sample_index`` of the available samples.
    :param load: list of sample names -> list of Sample (positions, depth, and whatever ``decode`` reads).
    :param draft: FASTA path or mapping name -> sequence.
    :param decode: as in ``stitch_samples``.
    Writes ``output`` (FASTQ, or FASTA without ``qualities``) and, with ``fillgaps``,
    ``output + '.gaps_in_draft_coords.bed'``.
    """
    if isinstance(draft, str):
        draft = read_fasta(draft)
    todo, missing = plan_regions(index, {k: len(v) for k, v in draft.items()}, regions)
    logger = get_named_logger('Stitcher')

    def pieces():
        for region in todo:
            logger.debug("Stitching {}".format(region))
            yield from stitch_samples(load(select_samples(index, region)), region=region, min_depth=min_depth,
                                      device=device, decode=decode)

    contigs = collapse_neighbours(pieces())
    with open(output, 'w') as fh:
        if fillgaps:
            contigs, gaps = fill_gaps(contigs, draft, fill_char)
            for (ref, _, _), seq_parts, qual_parts in contigs:
                write_fastx_segment(fh, (ref, seq_parts, qual_parts), qualities=qualities)
            # requested contigs without any sample are copied verbatim, as one gap each
            for ref in missing:
                logger.info("Copying contig '{}' verbatim from input.".format(ref))
                seq = draft[ref]
                write_fastx_segment(fh, (ref, [seq], ['!' * len(seq)]), qualities=qualities)
                gaps[ref] = [(0, len(seq))]
        else:
            last, k = None, 0
            for (ref, start, stop), seq_parts, qual_parts in contigs:
                k = k + 1 if ref == last else 0
                write_fastx_segment(fh, ("{}_{} {}-{}".format(ref, k, start, stop + 1), seq_parts, qual_parts),
                                    qualities=qualities)
                last = ref
    if fillgaps:
        write_bed(gaps, output + ".gaps_in_draft_coords.bed")


def sequence(stores, draft, output, regions=None, min_depth=0, fillgaps=True, fill_char=None, qualities=True,
             device=0):
    """`medaka sequence` (medaka/stitch.py:197-309, serial path) over stores written by ``prediction.predict_regions``.

    :param stores: one store path or several (a sample name found in more than one is read from the first).
    :param draft: FASTA path or mapping name -> sequence.
    :param regions: Regions or region strings to stitch (default: every draft contig).
    """
    from medaka_b200 import datastore
    if isinstance(stores, str):
        stores = [stores]
    opened = [datastore.DataStore(path, 'r') for path in stores]
    try:
        owner = {}
        for ds in opened:
            for name in ds.sample_registry:
                owner.setdefault(name, ds)
        write_consensus(sample_index(owner), lambda names: [owner[n].load_sample(n) for n in names], draft, output,
                        regions=regions, min_depth=min_depth, fillgaps=fillgaps, fill_char=fill_char,
                        qualities=qualities, device=device)
    finally:
        for ds in opened:
            ds.close()
