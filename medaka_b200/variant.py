"""Variant calling from network outputs: the `medaka vcf` path up to the variant records (medaka/variant.py:30-119,
180-244) - the consumer of BASELINE config 4's model (SURVEY.md section 8 row f2).

Stored samples of a region are trimmed at their overlaps (the plan of medaka_b200/stitch.py), re-cut so that no
variant straddles a sample edge (``join_samples``), and every joined sample is decoded on the GPU
(``HaploidLabelScheme.decode_variants`` -> libmedaka_b200 ``mdk_decode_variants``).  Writing VCF text is out of scope
(SURVEY.md section 2); ``Variant`` carries what a VCF line needs.

``variants`` is `medaka vcf` (the serial body of medaka/variant.py:180-244) over stores written by
``prediction.predict_regions``; ``joined_pieces`` is ``join_samples`` replayed on positions and per-piece cuts, for the
one-pass ``prediction.predict_variants``, whose calls never leave the device.
"""
import collections

import numpy as np

from medaka_b200 import stitch
from medaka_b200.common import Sample


class Variant(object):
    """The fields of medaka.vcf.Variant this path fills (medaka/vcf.py:159-214) plus its normalisation (:338-415)."""

    def __init__(self, chrom, pos, ref, alt='.', ident='.', qual='.', filt='.', info='.', genotype_data=None):
        self.chrom = chrom
        self.pos = int(pos)
        self.ref = ref.upper()
        self.alt = alt.split(',') if isinstance(alt, str) else list(alt)
        self.ident = str(ident)
        self.qual = float(qual) if qual != '.' else qual
        self.filt = filt
        self.info = info if isinstance(info, dict) else {}
        gd = collections.OrderedDict()
        if genotype_data is not None:       # GT first (vcf.py:146-156)
            gd['GT'] = genotype_data['GT']
            gd.update((k, v) for k, v in genotype_data.items() if k != 'GT')
        self.genotype_data = gd

    def __eq__(self, other):
        return all(getattr(self, f) == getattr(other, f) for f in
                   ('chrom', 'pos', 'ident', 'ref', 'alt', 'qual', 'filt', 'info', 'genotype_data'))

    def __repr__(self):
        return "Variant({}:{} {}>{} Q{})".format(self.chrom, self.pos, self.ref, ','.join(self.alt), self.qual)

    def trim(self, reference=None):
        """Minimal REF / ALT, left-aligned when the contig sequence is given (vcf.py:338-402)."""
        pos, seqs = self.pos, [self.ref] + list(self.alt)
        if reference is None:
            while min(len(s) for s in seqs) > 1 and len(set(s[-1] for s in seqs)) == 1:
                seqs = [s[:-1] for s in seqs]
        else:
            changed = True
            while changed:
                changed = False
                if all(len(s) > 0 for s in seqs) and len(set(s[-1] for s in seqs)) == 1:
                    seqs = [s[:-1] for s in seqs]
                    changed = True
                if any(len(s) == 0 for s in seqs):
                    if pos == 0:   # multi-base deletion at the start of the contig: pad on the right instead
                        seqs = [s + reference[len(seqs[0])] for s in seqs]
                        break
                    pos -= 1
                    seqs = [reference[pos] + s for s in seqs]
                    changed = True
        lead = 0
        shortest = min(len(s) for s in seqs)
        while lead < shortest - 1 and len(set(s[lead] for s in seqs)) == 1:
            lead += 1
        seqs = [s[lead:] for s in seqs]
        return Variant(self.chrom, pos + lead, seqs[0], alt=seqs[1:], ident=self.ident, qual=self.qual, filt=self.filt,
                       info=dict(self.info), genotype_data=self.genotype_data)

    def normalize(self, reference):
        """vcf.py:404-415."""
        if all(x == self.ref for x in self.alt):
            return self
        return self.trim(reference=reference)


def trimmed_samples(samples):
    """Sample.trim_samples (medaka/common.py:495-557) as a list: (Sample view, is_last_in_contig, heuristic)."""
    samples = list(samples)
    return [(samples[p.sample].slice(slice(p.lo, p.hi)), p.last, p.heuristic) for p in stitch.plan_pieces(samples)]


def join_samples(sample_gen, ref_seq, label_scheme):
    """Re-cut a stream of trimmed samples so that no variant is split across two of them (medaka/variant.py:30-119).

    :param sample_gen: iterable of (Sample, is_last_in_contig, heuristic).
    :yields: Sample
    """
    queue = []
    s = None
    for s, is_last_in_contig, _ in sample_gen:
        if is_last_in_contig:
            queue.append(s)
            yield Sample.from_samples(queue)
            queue = []
            continue
        # the call with gaps kept (argmax on the device) against the draft with gaps on insertion columns
        call = label_scheme.decode_labels(s)
        pos = s.positions
        is_major = pos['minor'] == 0
        ref_codes = np.zeros(len(pos), dtype=np.uint8)
        ref_codes[is_major] = label_scheme.encode_reference(ref_seq, pos['major'][is_major])
        # a column is "different" when call and draft disagree, or when both are a gap (variant.py:66-71)
        is_var = (call != ref_codes) | ((call == 0) & (ref_codes == 0))
        if np.all(is_var):
            queue.append(s)
            continue
        major_pos = pos['major'][is_major]
        major_same = call[is_major] == ref_codes[is_major]
        # the last major position whose call equals the draft, looking from the end (variant.py:84-93)
        rev = major_same[::-1]
        offset = int(np.argmax(rev)) if rev.any() else len(rev) - 1
        last_non_var_pos = major_pos[len(major_pos) - 1 - offset]
        cut = int(np.searchsorted(pos['major'], last_non_var_pos, side='left'))
        to_yield = queue + ([s.slice(slice(None, cut))] if cut > 0 else [])
        if to_yield:
            yield Sample.from_samples(to_yield)
        queue = [s.slice(slice(cut, None))]
    if queue:
        raise ValueError('Reached end of generator at {} without is_last_in_contig being True'.format(s.name))


def variants_from_samples(samples, ref_seq, label_scheme=None, ambig_ref=False, return_all=False):
    """The per-region body of variants_from_hdf (medaka/variant.py:215-237): trimmed -> joined -> decoded."""
    from medaka_b200 import labels
    if label_scheme is None:
        label_scheme = labels.HaploidLabelScheme()
    out = []
    for joined in join_samples(trimmed_samples(samples), ref_seq, label_scheme):
        out.extend(label_scheme.decode_variants(joined, ref_seq, ambig_ref=ambig_ref, return_all=return_all))
    return out


def sort_records(records):
    """The order ``VCFWriter.write_variants(sort=True)`` writes one joined sample's records in (medaka/vcf.py:509-516):
    a stable sort on 'chrom-pos' as loose versions, which for records of one contig is a stable sort on pos."""
    return sorted(records, key=lambda v: v.pos)


def joined_pieces(views, pieces, cuts):
    """``join_samples`` on positions only: how the trimmed pieces are re-cut and grouped into joined samples.

    :param views: list of Sample with positions (the pieces' samples); :param pieces: ``stitch.plan_pieces(views)``.
    :param cuts: per piece, the index (within the piece) of its last insertion-free column whose call equals the draft,
        or -1 when every column differs (``HaploidLabelScheme`` / ``mdk_variant_join_cuts``); ignored for pieces that
        end a contig.
    :yields: lists of (sample index, lo, hi) row ranges, one list per joined sample.
    """
    queue = []
    p = None
    for p, c in zip(pieces, cuts):
        if p.last:
            queue.append((p.sample, p.lo, p.hi))
            yield queue
            queue = []
            continue
        if c < 0:
            queue.append((p.sample, p.lo, p.hi))
            continue
        major = views[p.sample].positions['major'][p.lo:p.hi]
        cut = int(np.searchsorted(major, major[int(c)], side='left'))
        to_yield = queue + ([(p.sample, p.lo, p.lo + cut)] if cut > 0 else [])
        if to_yield:
            yield to_yield
        queue = [(p.sample, p.lo + cut, p.hi)]
    if queue:
        raise ValueError('Reached end of generator at {} without is_last_in_contig being True'.format(
            views[p.sample].name))


def _ref_seq(draft, ref_name):
    return draft[ref_name].upper()


def variants(stores, draft, regions=None, ambig_ref=False, return_all=False, verbose=False, device=0):
    """`medaka vcf` (medaka/variant.py:180-244, serial path) over stores written by ``prediction.predict_regions``.

    :param stores: one store path or several (a sample name found in more than one is read from the first).
    :param draft: FASTA path or mapping name -> sequence.
    :param regions: Regions or region strings (default: every indexed contig, in index order).  As in `medaka vcf`, a
        region selects the samples overlapping it; their variants are not clipped to it.
    :param ambig_ref: decode variants at ambiguous draft positions; :param return_all: also one record per draft
        position (gVCF); :param verbose: per-run info fields.
    :returns: list of Variant, in the order `medaka vcf` writes them: region by region, each joined sample's records
        sorted by position.
    """
    from medaka_b200 import datastore, labels
    if isinstance(stores, str):
        stores = [stores]
    if isinstance(draft, str):
        draft = stitch.read_fasta(draft)
    scheme = labels.HaploidLabelScheme(device)
    scheme.verbose = verbose
    opened = [datastore.DataStore(path, 'r') for path in stores]
    out = []
    try:
        owner = {}
        for ds in opened:
            for name in ds.sample_registry:
                owner.setdefault(name, ds)
        index = stitch.sample_index(owner)
        for reg in variant_regions(index, regions):
            ref_seq = _ref_seq(draft, reg.ref_name)
            samples = [owner[n].load_sample(n) for n in stitch.select_samples(index, reg)]
            for joined in join_samples(trimmed_samples(samples), ref_seq, scheme):
                out.extend(sort_records(scheme.decode_variants(joined, ref_seq, ambig_ref=ambig_ref,
                                                               return_all=return_all)))
    finally:
        for ds in opened:
            ds.close()
    return out


def variant_regions(index, regions=None):
    """The regions of a `medaka vcf` run: as given (strings parsed), or every indexed contig in index order
    (DataIndex.regions, medaka/datastore.py:446-451)."""
    from medaka_b200.common import Region
    if regions is None:
        return [Region(name, None, None) for name in index]
    return [Region.from_string(r) if isinstance(r, str) else r for r in regions]
