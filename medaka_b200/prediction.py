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
    """Device memory for the decoded calls of a one-pass run (``predict_consensus``): 2 B per computed column.

    Slabs of ``2 * half`` bytes from mdk_dev_alloc hold labels in their first half and quality bytes at the same offset
    in the second.  A row is (slab index, offset); every stitch call reads from one slab.
    """

    def __init__(self, device, half=1 << 28):
        self.device, self.half = device, int(half)
        self.slabs = []          # device addresses
        self.used = self.half    # bytes taken from the newest slab's halves

    def take(self, n):
        """Room for n rows -> (slab index, offset of the first row)."""
        if n > self.half:
            raise ValueError("a batch of {} columns does not fit a {} B arena slab".format(n, self.half))
        if self.used + n > self.half:
            lib, ffi = _lm.load(), _lm.ffi
            pp = ffi.new("void **")
            _lm.check(lib.mdk_dev_alloc(self.device, 2 * self.half, pp))
            self.slabs.append(int(ffi.cast("uintptr_t", pp[0])))
            self.used = 0
        at = self.used
        self.used += n
        return len(self.slabs) - 1, at

    def labels(self, slab):
        return self.slabs[slab]

    def quals(self, slab):
        return self.slabs[slab] + self.half

    def free(self):
        lib, ffi = _lm.load(), _lm.ffi
        while self.slabs:
            _lm.check(lib.mdk_dev_free(self.device, ffi.cast("void *", self.slabs.pop())))


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


def _run_decoded(samples, arena, bam, regions, model, feature_encoder, chunk_len, chunk_ovlp, min_depth,
                 batch_size=200, enable_chunking=True, bam_workers=2):
    """``run_prediction`` for ``predict_consensus``: every batch's decoded calls go to the arena, and
    ``samples[name] = (_stitch_view of the window, arena slab, row in the slab)`` is kept for each window (the first
    window of a name wins, as in a store).  Returns the remainder regions."""
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
        nb, nt, nf = x.shape
        if depth is None:
            depth = model.lookahead(batch_size, nt)
            if enable_chunking and nb * nt > (1 << 18):
                model.reserve(max(model.preferred_batch_size(), nb), nt)
        while len(pending) >= depth:
            model.wait(pending.popleft())
        # the page-locked feature slot is reused once the call that last used it has been waited for
        xin = model.pinned("dfeats%d" % (n_calls % (depth + 1)), (nb, nt, nf), np.float32)
        np.copyto(xin, x, casting="same_kind")
        n_calls += 1
        slab, row = arena.take(nb * nt)
        pending.append(model.submit_decoded(xin, arena.labels(slab) + row, arena.quals(slab) + row))
        for i, s in enumerate(data):
            if len(s.positions) != nt:
                raise ValueError("sample {} has {} columns in a batch of {}".format(s.name, len(s.positions), nt))
            name = s.name
            if name not in samples:
                samples[name] = (_stitch_view(s, min_depth), slab, row + i * nt)
    while pending:
        model.wait(pending.popleft())
    return loader.remainders


def predict_consensus(bam, bam_regions, model, feature_encoder, draft, output, chunk_len=10000, chunk_ovlp=1000,
                      batch_size=200, bam_chunk=int(1e6), bam_workers=2, regions=None, min_depth=0, fillgaps=True,
                      fill_char=None, qualities=True, world_size=1):
    """`medaka inference` followed by `medaka sequence` in one pass: the FASTQ / FASTA (and gap bed) that
    ``predict_regions`` + ``stitch.sequence`` write, without the probabilities ever leaving the GPU.

    The engine decodes every window in its head (labels and quality bytes, ``GRUModel.submit_decoded``) into a
    device arena; per window only its name, positions and (with ``min_depth``) depth stay on the host.  At the end the
    windows are indexed,
    trimmed and stitched exactly as ``stitch.sequence`` does (``stitch.write_consensus``), the kept rows compacted on
    the device (``stitch.decode_label_pieces``).

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
            "predict_consensus runs consensus (GRUModel) models only; for {} use predict_regions followed by "
            "stitch.sequence".format(type(model).__name__))
    if world_size != 1:
        raise NotImplementedError("predict_consensus runs on one GPU; for several, use predict_regions with one "
                                  "store per rank, then stitch.sequence over the stores")
    from medaka_b200 import stitch
    logger = common.get_named_logger('Predict')
    model.check_feature_encoder_compatibility(feature_encoder)
    long_regions, remainder_regions = triage_regions(bam_regions, chunk_len, bam_chunk, chunk_ovlp)
    arena = _LabelArena(model.device().index)
    samples = collections.OrderedDict()
    try:
        if long_regions:
            logger.info("Processing {} long region(s) with batching.".format(len(long_regions)))
            rem = _run_decoded(samples, arena, bam, long_regions, model, feature_encoder, chunk_len, chunk_ovlp,
                               min_depth, batch_size=batch_size, bam_workers=bam_workers)
            remainder_regions.extend([r[0] for r in rem])
        if remainder_regions:
            logger.info("Processing {} short region(s).".format(len(remainder_regions)))
            new_rem = _run_decoded(samples, arena, bam, remainder_regions, model, feature_encoder, chunk_len,
                                   chunk_ovlp, min_depth, batch_size=1, enable_chunking=False)
            if new_rem:
                logger.warning("{} regions were not processed: {}.".format(len(new_rem), [x[0] for x in new_rem]))
        model.sync()

        def decode(views, pieces):
            # one stitch call per arena slab the pieces lie in, results back in piece order
            where = [samples[views[p.sample].name][1:] for p in pieces]
            seqs, quals = [None] * len(pieces), [None] * len(pieces)
            for slab in sorted({w[0] for w in where}):
                ks = [k for k, w in enumerate(where) if w[0] == slab]
                got = stitch.decode_label_pieces(arena.labels(slab), arena.quals(slab),
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
