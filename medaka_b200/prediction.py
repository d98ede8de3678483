"""Inference orchestration: region scheduling, batching, the per-batch hot loop, output.

Host-side mirror of medaka/prediction.py: ``run_prediction`` (:14-81), the region triage of
``predict`` (:95-110, :180-215) and ``DataLoader`` (:225-370) with the same observable
behaviour (batch / sample / remainder counts are those of medaka/test/test_dataloader.py),
plus the one thing the reference leaves to the user (README.md:294-330): dealing regions to
the GPUs of a box, one process per GPU, each writing its own output store.

The body of the loop - ``model.predict_on_batch(batch)`` - is the engine call; everything in
this file is scheduling.
"""
import collections
import queue
import threading
from timeit import default_timer as now

import numpy as np

from medaka_b200 import common, datastore, features, libmedaka as _lm, torch_ext


def triage_regions(bam_regions, chunk_len, bam_chunk, chunk_ovlp):
    """Split regions into (long regions to batch, remainder regions) like predict() (:95-110)."""
    regions, remainders = [], []
    for region in bam_regions:
        if region.size < chunk_len:
            remainders.append(region)
        elif region.size > bam_chunk:
            regions.extend(region.split(bam_chunk, overlap=chunk_ovlp, fixed_size=False))
        else:
            regions.append(region)
    return regions, remainders


def shard_regions(regions, world_size):
    """Deal regions to ranks, longest first onto the least-loaded rank (SURVEY.md 8e).

    Returns a list of ``world_size`` lists.  Regions are independent units (no cross-window
    state: each window starts from h0 = 0), so no data-path collective is needed.
    """
    shards = [[] for _ in range(world_size)]
    load = [0] * world_size
    order = sorted(range(len(regions)), key=lambda i: (-regions[i].size, i))
    for i in order:
        r = min(range(world_size), key=lambda k: (load[k], k))
        shards[r].append(regions[i])
        load[r] += regions[i].size
    return shards


class DataLoader(object):
    """Threads + bounded queues feeding inference batches (cf. medaka/prediction.py:225-370).

    Iterating yields ``(list of Samples, Batch)``.  ``bam_workers`` threads turn regions into
    chunked samples, one batcher thread groups and collates them.  Sources narrower than
    ``chunk_len`` end up in ``self.remainders`` as ``(Region, width)``.
    """

    _STOP = object()

    def __init__(self, bam, regions, batch_size, batch_cache_size=8, bam_workers=2, **kwargs):
        self.logger = common.get_named_logger('DLoader')
        self.bam = bam
        self.batch_size = batch_size
        self.bam_workers = bam_workers
        self.kwargs = kwargs
        self._samples = queue.Queue(maxsize=batch_cache_size * batch_size)
        self._batches = queue.Queue(maxsize=batch_cache_size)
        self._regions = queue.Queue()
        for r in regions:
            self._regions.put(r)
        self.remainders = list()
        self._remainder_lock = threading.Lock()
        self._error = None
        self._workers = []
        for i in range(bam_workers):
            t = threading.Thread(target=self._region_worker, name="Sample-{}".format(i), daemon=True)
            t.start()
            self._workers.append(t)
        self._bthread = threading.Thread(target=self._batch_worker, name="Batcher", daemon=True)
        self._bthread.start()

    def __iter__(self):
        return self

    def __next__(self):
        item = self._batches.get()
        if item is self._STOP:
            if self._error is not None:
                raise self._error
            raise StopIteration
        return item

    def _region_worker(self):
        try:
            while True:
                try:
                    region = self._regions.get_nowait()
                except queue.Empty:
                    break
                gen = features.SampleGenerator(self.bam, region, **self.kwargs)
                for sample in gen.samples:
                    self._samples.put(sample)
                with self._remainder_lock:
                    self.remainders.extend(gen._quarantined)
        except BaseException as e:  # surfaced by __next__
            self._error = e
        finally:
            self._samples.put(self._STOP)

    def _iter_samples(self):
        stops = 0
        while stops < self.bam_workers:
            item = self._samples.get()
            if item is self._STOP:
                stops += 1
            else:
                yield item

    def _batch_worker(self):
        try:
            for data in common.grouper(self._iter_samples(), self.batch_size):
                self._batches.put((data, torch_ext.Batch.collate(data)))
        except BaseException as e:
            self._error = e
        finally:
            self._batches.put(self._STOP)


def run_prediction(output, bam, regions, model, feature_encoder, chunk_len, chunk_ovlp, batch_size=200,
                   save_features=False, enable_chunking=True, bam_workers=2):
    """Inference worker (medaka/prediction.py:14-81): returns the remainder regions."""
    logger = common.get_named_logger('PWorker')
    if batch_size == "auto":   # the engine's one-wave batch instead of the reference's CLI default
        batch_size = model.preferred_batch_size() if hasattr(model, "preferred_batch_size") else 200
    loader = DataLoader(
        bam, regions, batch_size, batch_cache_size=8, bam_workers=bam_workers,
        feature_encoder=feature_encoder, chunk_len=chunk_len, chunk_overlap=chunk_ovlp,
        enable_chunking=enable_chunking)
    total_region_mbases = sum(r.size for r in regions) / 1e6
    logger.info("Running inference for {:.1f}M draft bases.".format(total_region_mbases))
    n_batches, n_positions = 0, 0
    t0 = now()
    def _store(ds, data, batch, class_probs, labels=None):
        # label_probs as the reference stores them, plus the engine's argmax labels (uint8 [T]) in the Sample's
        # `labels` field: `medaka sequence` / `medaka vcf` read label_probs and ignore it, the GPU stitch / variant
        # decode of this package can skip the argmax (SURVEY.md 8b, decode seam)
        for i, (sample, prob, feat) in enumerate(zip(data, class_probs, batch.features)):
            feats = feat if save_features else None
            extra = {} if labels is None else {"labels": labels[i]}
            # (no defensive copy: the probabilities / labels are this batch's private arrays - predict_async copies
            # them out of its pinned slot -, positions and depth are slices of the region's arrays that nobody rewrites)
            ds.write_sample(sample.amend(label_probs=prob, features=feats, **extra), copy=False)

    with datastore.DataStore(output, 'a') as ds:
        # look-ahead: enough batches are queued on the engine for it to coalesce them into device-filling groups
        # and to keep a second group's copies and compute under the first (mdk_engine_submit); results are collected
        # in order, so PCIe traffic and the store's writer thread overlap the GPU work
        pending = collections.deque()
        use_async = hasattr(model, "predict_async")
        depth = None

        def _collect():
            data0, batch0, handle = pending.popleft()
            probs = handle.result()
            _store(ds, data0, batch0, probs, getattr(handle, "labels", None))

        for data, batch in loader:
            n_batches += 1
            n_positions += int(batch.features.shape[0]) * int(batch.features.shape[1])
            if not use_async:
                _store(ds, data, batch, model.predict_on_batch(batch), getattr(model, "last_labels", None))
                continue
            if depth is None:
                nb, nt = int(batch.features.shape[0]), int(batch.features.shape[1])
                depth = model.lookahead(batch_size, nt) if hasattr(model, "lookahead") else 2
                if hasattr(model, "reserve") and enable_chunking and nb * nt > (1 << 18):
                    # coalescing needs the lanes sized for a whole group up front
                    model.reserve(max(model.preferred_batch_size(), nb), nt)
            while len(pending) >= depth:
                _collect()
            pending.append((data, batch, model.predict_async(batch, slots=depth + 1)))
        while pending:
            _collect()
    dt = max(now() - t0, 1e-9)
    logger.info("Processed {} batches, {} positions in {:.2f}s ({:.3e} positions/s)".format(
        n_batches, n_positions, dt, n_positions / dt))
    logger.info("All done, {} remainder regions.".format(len(loader.remainders)))
    return loader.remainders


def predict_regions(output, bam, bam_regions, model, feature_encoder, chunk_len=10000, chunk_ovlp=1000,
                    batch_size=200, bam_chunk=int(1e6), save_features=False, bam_workers=2,
                    rank=0, world_size=1):
    """The body of ``predict`` (medaka/prediction.py:84-222) for already-opened model and encoder.

    With ``world_size > 1`` each rank keeps its share of the regions (``shard_regions``) and should
    be given its own ``output`` (``medaka sequence`` accepts several stores, medaka.py:703-704).
    """
    logger = common.get_named_logger('Predict')
    model.check_feature_encoder_compatibility(feature_encoder)
    regions, remainder_regions = triage_regions(bam_regions, chunk_len, bam_chunk, chunk_ovlp)
    if world_size > 1:
        regions = shard_regions(regions, world_size)[rank]
        remainder_regions = shard_regions(remainder_regions, world_size)[rank]
    if len(regions) > 0:
        logger.info("Processing {} long region(s) with batching.".format(len(regions)))
        rem = run_prediction(output, bam, regions, model, feature_encoder, chunk_len, chunk_ovlp,
                             batch_size=batch_size, save_features=save_features, bam_workers=bam_workers)
        remainder_regions.extend([r[0] for r in rem])
    if len(remainder_regions) > 0:
        logger.info("Processing {} short region(s).".format(len(remainder_regions)))
        new_remainders = run_prediction(
            output, bam, remainder_regions, model, feature_encoder, chunk_len, chunk_ovlp,
            batch_size=1, save_features=save_features, enable_chunking=False)
        if len(new_remainders) > 0:
            logger.warning("{} regions were not processed: {}.".format(
                len(new_remainders), [x[0] for x in new_remainders]))
    logger.info("Finished processing all regions.")


class _LabelArena(object):
    """Device memory for the decoded outputs of a one-pass run: ``row_bytes[f]`` bytes of field f per computed column,
    e.g. (1, 1) for the labels and quality bytes of ``predict_consensus``, (1, 4, 4) for the call bytes and the two
    phreds of ``predict_variants``.

    Slabs from mdk_dev_alloc hold ``half`` rows of every field, field after field.  A row is (slab index, offset); every
    stitch call reads from one slab.  ``reset`` hands the slabs out again from the first (for a run in passes).
    """

    def __init__(self, device, row_bytes, half=1 << 28):
        self.device, self.half = device, int(half)
        self.row_bytes = tuple(int(b) for b in row_bytes)
        self.field_at = [self.half * sum(self.row_bytes[:f]) for f in range(len(self.row_bytes))]
        self.slabs = []          # device addresses
        self.cur = -1            # slab rows are taken from
        self.used = self.half    # rows taken from it
        self.peak = 0            # most slabs held at once, in bytes

    def take(self, n):
        """Room for n rows -> (slab index, offset of the first row)."""
        if n > self.half:
            raise ValueError("a batch of {} columns does not fit a {}-row arena slab".format(n, self.half))
        if self.used + n > self.half:
            self.cur += 1
            if self.cur == len(self.slabs):
                lib, ffi = _lm.load(), _lm.ffi
                pp = ffi.new("void **")
                _lm.check(lib.mdk_dev_alloc(self.device, self.half * sum(self.row_bytes), pp))
                self.slabs.append(int(ffi.cast("uintptr_t", pp[0])))
                self.peak = max(self.peak, len(self.slabs) * self.half * sum(self.row_bytes))
            self.used = 0
        at = self.used
        self.used += n
        return self.cur, at

    def addr(self, slab, field, row=0):
        """Device address of field ``field`` of row ``row`` of slab ``slab``."""
        return self.slabs[slab] + self.field_at[field] + row * self.row_bytes[field]

    def reset(self):
        self.cur, self.used = -1, self.half

    def free(self):
        lib, ffi = _lm.load(), _lm.ffi
        while self.slabs:
            _lm.check(lib.mdk_dev_free(self.device, ffi.cast("void *", self.slabs.pop())))
        self.reset()


def _device_index(model):
    """CUDA device index of a model: ``GRUModel.device()`` is a torch.device, ``LatentSpaceLSTM.device()`` the string
    "cuda:<index>"."""
    dev = model.device()
    return int(dev.rsplit(":", 1)[1]) if isinstance(dev, str) else dev.index


def _stitch_view(sample, min_depth):
    """What the stitch plan reads of a window, in the smallest exact form: positions as (int32 major unless a major
    needs more, unsigned minor of the width its largest value needs), and, only when the run filters on depth, depth
    clipped to min_depth (``depth >= min_depth`` is unchanged).  About 5 B per column instead of the 24 B of the
    window's int64 positions and depth."""
    major, minor = sample.positions['major'], sample.positions['minor']
    big = len(major) and int(major[-1]) >= np.iinfo(np.int32).max
    pos = np.empty(len(major), dtype=[('major', np.int64 if big else np.int32),
                                      ('minor', np.min_scalar_type(int(minor.max()) if len(minor) else 0))])
    pos['major'], pos['minor'] = major, minor
    depth = None
    if min_depth:
        depth = np.minimum(np.asarray(sample.depth), min_depth).astype(np.min_scalar_type(min_depth))
    return common.Sample(ref_name=sample.ref_name, features=None, labels=None, ref_seq=None, positions=pos,
                         label_probs=None, depth=depth)


def _run_decoded(samples, arena, bam, regions, model, feature_encoder, chunk_len, chunk_ovlp, view, submit,
                 batch_size=200, enable_chunking=True, bam_workers=2):
    """``run_prediction`` for the one-pass runs: ``submit(features, data, slot, slab, row)`` queues every batch with its
    decoded outputs going to the arena (``slot`` numbers the page-locked buffers it may reuse) and returns a ticket;
    ``samples[name] = (view(window), arena slab, row in the slab)`` is kept for each window (the first window of a name
    wins, as in a store).  Returns the remainder regions."""
    logger = common.get_named_logger('PWorker')
    if batch_size == "auto":
        batch_size = model.preferred_batch_size()
    loader = DataLoader(
        bam, regions, batch_size, batch_cache_size=8, bam_workers=bam_workers,
        feature_encoder=feature_encoder, chunk_len=chunk_len, chunk_overlap=chunk_ovlp,
        enable_chunking=enable_chunking)
    logger.info("Running one-pass inference for {:.1f}M draft bases.".format(sum(r.size for r in regions) / 1e6))
    pending = collections.deque()
    depth = None
    n_calls = 0
    for data, batch in loader:
        x = model.get_model_input_features(batch)
        x = x.detach().cpu().numpy() if hasattr(x, "detach") else x
        # counts features float32 [nb, nt, F]; read-level features int8 [nb, nt, D, F], D the batch's deepest window
        # (collated batches are uint8, cast like LatentSpaceLSTM's own submit)
        nb, nt = x.shape[:2]
        read_level = x.ndim == 4
        if depth is None:
            depth = model.lookahead(batch_size, nt)
            if enable_chunking and nb * nt > (1 << 18):
                model.reserve(max(model.preferred_batch_size(), nb), nt)
        while len(pending) >= depth:
            model.wait(pending.popleft())
        for s in data:
            if len(s.positions) != nt:
                raise ValueError("sample {} has {} columns in a batch of {}".format(s.name, len(s.positions), nt))
        # the page-locked slots are reused once the call that last used them has been waited for
        slot = n_calls % (depth + 1)
        xin = model.pinned("dfeats%d" % slot, x.shape, np.int8 if read_level else np.float32)
        np.copyto(xin, x, casting="unsafe" if read_level else "same_kind")
        n_calls += 1
        slab, row = arena.take(nb * nt)
        pending.append(submit(xin, data, slot, slab, row))
        for i, s in enumerate(data):
            name = s.name
            if name not in samples:
                samples[name] = (view(s), slab, row + i * nt)
    while pending:
        model.wait(pending.popleft())
    return loader.remainders


def _run_one_pass(samples, arena, bam, long_regions, remainder_regions, model, feature_encoder, chunk_len, chunk_ovlp,
                  view, submit, batch_size, bam_workers):
    """The long regions batched, then the remainder regions one window at a time (``predict_regions``), into the arena;
    returns once the engine has finished."""
    logger = common.get_named_logger('Predict')
    remainder_regions = list(remainder_regions)
    if long_regions:
        logger.info("Processing {} long region(s) with batching.".format(len(long_regions)))
        rem = _run_decoded(samples, arena, bam, long_regions, model, feature_encoder, chunk_len, chunk_ovlp, view,
                           submit, batch_size=batch_size, bam_workers=bam_workers)
        remainder_regions.extend([r[0] for r in rem])
    if remainder_regions:
        logger.info("Processing {} short region(s).".format(len(remainder_regions)))
        new_rem = _run_decoded(samples, arena, bam, remainder_regions, model, feature_encoder, chunk_len, chunk_ovlp,
                               view, submit, batch_size=1, enable_chunking=False)
        if new_rem:
            logger.warning("{} regions were not processed: {}.".format(len(new_rem), [x[0] for x in new_rem]))
    model.sync()


def predict_consensus(bam, bam_regions, model, feature_encoder, draft, output, chunk_len=10000, chunk_ovlp=1000,
                      batch_size=200, bam_chunk=int(1e6), bam_workers=2, regions=None, min_depth=0, fillgaps=True,
                      fill_char=None, qualities=True, world_size=1):
    """`medaka inference` followed by `medaka sequence` in one pass: the FASTQ / FASTA (and gap bed) that
    ``predict_regions`` + ``stitch.sequence`` write, without the probabilities ever leaving the GPU.

    The engine decodes every window in its head (labels and quality bytes, ``submit_decoded`` of ``GRUModel`` or of the
    read-level ``LatentSpaceLSTM``) into a device arena; per window only its name, positions and (with ``min_depth``)
    depth stay on the host.  At the end the windows are indexed, trimmed and stitched exactly as ``stitch.sequence``
    does (``stitch.write_consensus``), the kept rows compacted on the device (``stitch.decode_label_pieces``).

    The arena holds 2 B per computed column (every column of every window, overlaps included) until the output is
    written, and is freed on return, also on error: about (draft bases) x (1 + insertion column share) x chunk_len /
    (chunk_len - chunk_ovlp) x 2 B, e.g. an estimated 7-8 GB for a 3.1 Gb draft with ~15 % insertion columns and
    10 000 / 1 000 windows.  On the host each window keeps its positions as int32 major and (usually) uint8 minor, and
    with ``min_depth`` a clipped depth of (usually) 1 B: about 5-6 B per computed column, an estimated 20-25 GB for
    the same draft.

    :param draft: FASTA path or mapping name -> sequence.
    :param regions: Regions or region strings to stitch (default: every draft contig); ``bam_regions`` are the regions
        to run inference on, as in ``predict_regions``.
    """
    if not hasattr(model, "submit_decoded"):
        raise NotImplementedError(
            "predict_consensus runs models with decoded outputs (GRUModel, LatentSpaceLSTM) only; for {} use "
            "predict_regions followed by stitch.sequence".format(type(model).__name__))
    if world_size != 1:
        raise NotImplementedError("predict_consensus runs on one GPU; for several, use predict_regions with one "
                                  "store per rank, then stitch.sequence over the stores")
    from medaka_b200 import stitch
    logger = common.get_named_logger('Predict')
    model.check_feature_encoder_compatibility(feature_encoder)
    long_regions, remainder_regions = triage_regions(bam_regions, chunk_len, bam_chunk, chunk_ovlp)
    arena = _LabelArena(_device_index(model), (1, 1))
    samples = collections.OrderedDict()
    try:
        _run_one_pass(samples, arena, bam, long_regions, remainder_regions, model, feature_encoder, chunk_len,
                      chunk_ovlp, lambda s: _stitch_view(s, min_depth),
                      lambda x, data, slot, slab, row: model.submit_decoded(x, arena.addr(slab, 0, row),
                                                                            arena.addr(slab, 1, row)),
                      batch_size, bam_workers)

        def decode(views, pieces):
            # one stitch call per arena slab the pieces lie in, results back in piece order
            where = [samples[views[p.sample].name][1:] for p in pieces]
            seqs, quals = [None] * len(pieces), [None] * len(pieces)
            for slab in sorted({w[0] for w in where}):
                ks = [k for k, w in enumerate(where) if w[0] == slab]
                got = stitch.decode_label_pieces(arena.addr(slab, 0), arena.addr(slab, 1),
                                                 [where[k][1] + pieces[k].lo for k in ks],
                                                 [pieces[k].hi - pieces[k].lo for k in ks], device=arena.device)
                for k, s, q in zip(ks, *got):
                    seqs[k], quals[k] = s, q
            return seqs, quals

        stitch.write_consensus(stitch.sample_index(samples), lambda names: [samples[n][0] for n in names], draft, output, regions=regions,
                               min_depth=min_depth, fillgaps=fillgaps, fill_char=fill_char, qualities=qualities,
                               decode=decode, device=arena.device)
    finally:
        try:
            model.sync()
        finally:
            arena.free()
    logger.info("Finished one-pass consensus of {} windows.".format(len(samples)))


# bytes of arena per computed column of a variant run: the call byte and the two float32 phreds
VARIANT_ROW_BYTES = (1, 4, 4)


def estimated_columns(bases, chunk_len, chunk_ovlp, insertion_share=0.15):
    """Computed columns (overlaps included) for ``bases`` draft bases: bases x (1 + insertion column share) x
    chunk_len / (chunk_len - chunk_ovlp)."""
    return int(bases * (1.0 + insertion_share) * chunk_len / max(chunk_len - chunk_ovlp, 1)) + 1


def plan_passes(variant_regions, bam_regions, arena_bytes, chunk_len, chunk_ovlp, row_bytes=sum(VARIANT_ROW_BYTES)):
    """Contigs of a ``predict_variants`` run grouped into passes whose estimated arena fits ``arena_bytes``.

    Contigs come in the order the variant regions first name them, and only those with bam regions (the others have no
    samples).  A pass never splits a contig; a contig whose estimate alone exceeds the budget gets a pass of its own.
    The estimate is ``estimated_columns`` of the contig's bam region bases times ``row_bytes``.
    :returns: list of lists of contig names.
    """
    bases = collections.OrderedDict()
    for r in bam_regions:
        bases[r.ref_name] = bases.get(r.ref_name, 0) + r.size
    order = []
    for r in variant_regions:
        if r.ref_name in bases and r.ref_name not in order:
            order.append(r.ref_name)
    passes, cur, cur_bytes = [], [], 0
    for name in order:
        need = estimated_columns(bases[name], chunk_len, chunk_ovlp) * row_bytes
        if cur and cur_bytes + need > arena_bytes:
            passes.append(cur)
            cur, cur_bytes = [], 0
        cur.append(name)
        cur_bytes += need
    if cur:
        passes.append(cur)
    return passes


def _variants_of_region(region, samples, index, arena, scheme, ref_seq, ambig_ref, return_all):
    """``variant.variants`` for one region, on the calls in the arena: trimmed pieces (host, positions), join cuts and
    decode (device), records (host)."""
    from medaka_b200 import labels, stitch, variant
    names = stitch.select_samples(index, region)
    views = [samples[n][0] for n in names]
    where = [samples[n][1:] for n in names]

    def addr(field, k, lo):
        slab, row = where[k]
        return arena.addr(slab, field, row + lo)

    pieces = stitch.plan_pieces(views)
    inner = [p for p in pieces if not p.last]
    cuts = np.full(len(pieces), -1, dtype=np.int64)
    got = labels.variant_join_cuts([addr(0, p.sample, p.lo) for p in inner], [p.hi - p.lo for p in inner],
                                   device=arena.device)
    cuts[[k for k, p in enumerate(pieces) if not p.last]] = got
    groups = list(variant.joined_pieces(views, pieces, cuts))
    if not groups:
        return []
    segs, sample_seg, joined = [], [0], []
    for g in groups:
        parts = [common.Sample(ref_name=views[k].ref_name, features=None, labels=None, ref_seq=None,
                               positions=views[k].positions[lo:hi], label_probs=None, depth=None) for k, lo, hi in g]
        pos = common.Sample.from_samples(parts).positions
        if pos['minor'][0] != 0:
            raise ValueError("The first position of a sample must not be an insertion.")
        joined.append(pos)
        segs.extend((addr(0, k, lo), addr(1, k, lo), addr(2, k, lo), hi - lo) for k, lo, hi in g)
        sample_seg.append(len(segs))
    d = labels.decode_variant_segments([s[0] for s in segs], [s[1] for s in segs], [s[2] for s in segs],
                                       [s[3] for s in segs], sample_seg, device=arena.device,
                                       want_quals=scheme.verbose, want_ref_q=return_all)
    run_edges = np.searchsorted(d['run_sample'], np.arange(len(joined) + 1), side='left')
    col_edges = np.concatenate(([0], np.cumsum(d['run_len'])))
    out, col0 = [], 0
    for smp, pos in enumerate(joined):
        r0, r1 = int(run_edges[smp]), int(run_edges[smp + 1])
        c0, c1 = int(col_edges[r0]), int(col_edges[r1])
        qs = (d['run_col_pred_q'][c0:c1], d['run_col_ref_q'][c0:c1]) if scheme.verbose else (None, None)
        major_ref_q = d['ref_q'][col0:col0 + len(pos)][pos['minor'] == 0] if return_all else None
        col0 += len(pos)
        out.extend(variant.sort_records(scheme.variant_records(
            region.ref_name, pos, scheme.reference_codes(pos, ref_seq), ref_seq, d['run_start'][r0:r1],
            d['run_len'][r0:r1], d['run_pred_q'][r0:r1], d['run_ref_q'][r0:r1], d['run_pred'][c0:c1], *qs,
            major_ref_q=major_ref_q, ambig_ref=ambig_ref, return_all=return_all)))
    return out


def predict_variants(bam, bam_regions, model, feature_encoder, draft, regions=None, ambig_ref=False, return_all=False,
                     verbose=False, chunk_len=10000, chunk_ovlp=1000, batch_size=200, bam_chunk=int(1e6), bam_workers=2,
                     arena_bytes=8 << 30, world_size=1):
    """`medaka inference` followed by `medaka vcf` in one pass: the records ``predict_regions`` + ``variant.variants``
    return, in the same order, without the probabilities ever leaving the GPU.

    The engine decodes every window in its head (``submit_variant_decoded`` of ``GRUModel`` or of the read-level
    ``LatentSpaceLSTM``: a call byte and the phreds of the winning and of the draft's class, 9 B per column) into a
    device arena; per window only its name and positions stay on the host.  The join cuts and the variant runs are computed on the device (``labels.variant_join_cuts``,
    ``labels.decode_variant_segments``); only the runs come back.

    The run goes in passes (``plan_passes``): contigs are grouped, in the order of the variant regions, so that a pass's
    estimated arena fits ``arena_bytes``; each pass runs inference on its contigs' ``bam_regions``, then joins and decodes
    its variant regions and hands the arena to the next.  A contig is never split; bam regions on contigs no variant
    region asks for are skipped.  The arena is freed on return, also on error.

    :param draft: FASTA path or mapping name -> sequence.
    :param regions: Regions or region strings to call (default: every contig with samples, in index order).
    """
    if not hasattr(model, "submit_variant_decoded"):
        raise NotImplementedError(
            "predict_variants runs models with decoded outputs (GRUModel, LatentSpaceLSTM) only; for {} use "
            "predict_regions followed by variant.variants".format(type(model).__name__))
    from medaka_b200 import labels, stitch, variant
    scheme_of_model = getattr(model, "label_scheme", None)
    if scheme_of_model is not None and not isinstance(scheme_of_model, labels.HaploidLabelScheme):
        raise NotImplementedError("predict_variants decodes haploid label schemes only; use predict_regions followed "
                                  "by variant.variants")
    if world_size != 1:
        raise NotImplementedError("predict_variants runs on one GPU; for several, use predict_regions with one store "
                                  "per rank, then variant.variants over the stores")
    logger = common.get_named_logger('Predict')
    model.check_feature_encoder_compatibility(feature_encoder)
    if isinstance(draft, str):
        draft = stitch.read_fasta(draft)
    scheme = labels.HaploidLabelScheme(_device_index(model))
    scheme.verbose = verbose
    # every contig with samples, in index order: the contigs of the bam regions, sorted (stitch.sample_index)
    vregions = variant.variant_regions(sorted({r.ref_name for r in bam_regions}), regions)
    passes = plan_passes(vregions, bam_regions, arena_bytes, chunk_len, chunk_ovlp)
    ref_seqs = {}

    def ref_seq(name):
        if name not in ref_seqs:
            ref_seqs[name] = draft[name].upper()
        return ref_seqs[name]

    arena = _LabelArena(_device_index(model), VARIANT_ROW_BYTES)

    def submit(x, data, slot, slab, row):
        nb, nt = x.shape[:2]
        ref = model.pinned("vref%d" % slot, (nb, nt), np.uint8)
        for i, s in enumerate(data):
            ins = s.positions['minor'] != 0
            ref[i] = scheme.reference_codes(s.positions, ref_seq(s.ref_name)) | (ins.astype(np.uint8) << 7)
        return model.submit_variant_decoded(x, ref, arena.addr(slab, 0, row), arena.addr(slab, 1, row),
                                            arena.addr(slab, 2, row))

    records = [None] * len(vregions)
    n_windows = 0
    try:
        for k, contigs in enumerate(passes):
            logger.info("Pass {} of {}: {} contig(s).".format(k + 1, len(passes), len(contigs)))
            wanted = set(contigs)
            long_regions, remainder_regions = triage_regions([r for r in bam_regions if r.ref_name in wanted],
                                                             chunk_len, bam_chunk, chunk_ovlp)
            samples = collections.OrderedDict()
            arena.reset()
            _run_one_pass(samples, arena, bam, long_regions, remainder_regions, model, feature_encoder, chunk_len,
                          chunk_ovlp, lambda s: _stitch_view(s, 0), submit, batch_size, bam_workers)
            n_windows += len(samples)
            index = stitch.sample_index(samples)
            for i, reg in enumerate(vregions):
                if reg.ref_name in wanted:
                    records[i] = _variants_of_region(reg, samples, index, arena, scheme, ref_seq(reg.ref_name),
                                                     ambig_ref, return_all)
    finally:
        try:
            model.sync()
        finally:
            arena.free()
    logger.info("Finished one-pass variant calling of {} windows in {} pass(es).".format(n_windows, len(passes)))
    return [v for recs in records if recs for v in recs]
