/*
 * medaka_b200.h - C ABI of libmedaka_b200.so, the sm_90a engine behind medaka's
 * inference hot path (medaka/prediction.py:44-52).
 *
 * Plain C: opaque handles, pointers + sizes, int return codes (0 = MDK_OK).  No torch
 * types, no exit(): every failure returns a negative code and leaves a message in
 * mdk_last_error() (the reference's C layer calls exit(1) on error,
 * src/medaka_common.c:19-26; a drop-in library must not).
 *
 * Each entry point cites the reference interface it replaces.  The cffi binding a
 * medaka maintainer would add is in INTEGRATION.md; medaka_b200/libmedaka.py is
 * that binding (it cdef()s this file minus the '#' lines, like the reference's
 * build.py:71-82 does for libmedaka).
 *
 * Conventions
 *   - "host" pointers are ordinary host memory (pinned memory from mdk_host_alloc makes
 *     the copies asynchronous); "dev" pointers are CUDA device pointers on the engine's
 *     device (e.g. torch tensor .data_ptr()).
 *   - feats   float32 [B][T][F] row-major (torch_ext.Batch.counts_matrix, torch_ext.py:155)
 *   - probs   float32 [B][T][5]  (GRUModel.forward output, gru.py:58-72)
 *   - logits  float32 [B][T][5]  (pre-softmax, gru.py:67)            - optional (NULL)
 *   - labels  uint8   [B][T]     (argmax, first max wins, labels.py:1063) - optional
 *   - weights: torch state-dict layout (gate order r,z,n): w_ih [3H][in], w_hh [3H][H],
 *     b_ih [3H], b_hh [3H]; linear w [5][2H], b [5]   (SURVEY.md section 3.4)
 */
#ifndef MEDAKA_B200_H
#define MEDAKA_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MDK_OK 0
#define MDK_ERR_ARG -1
#define MDK_ERR_CUDA -2
#define MDK_ERR_STATE -3
#define MDK_ERR_UNSUPPORTED -4
#define MDK_ERR_NOMEM -5

/* precision modes of the GRU gate matmuls */
#define MDK_PREC_TC 0    /* wgmma tensor cores, fp16 hi/lo split operands (3 MMAs), fp32 accumulate */
#define MDK_PREC_FP32 1  /* CUDA-core fp32 FFMA path: validation / --full_precision */
#define MDK_PREC_FP16 2  /* wgmma tensor cores, one fp16 product per contraction (hi.hi), fp32 accumulate: the arithmetic
                            medaka itself runs on a GPU without --full_precision (the model in half precision).  Rounded
                            to fp16: W_hh and the h fed back at every step, the layer-1 projection's W_ih and its input h0,
                            and at gru_size 128 with F <= 16 (fused layer-0 projection) W_ih0 and the features.  fp32 as
                            on MDK_PREC_TC: the CUDA-core layer-0 projection (F > 16 at 128, every F at 256), the biases,
                            the gate math and h state, the head.  Same kernels' bodies, tile choice and workspaces as
                            MDK_PREC_TC; h0 keeps ~22 bits (read_activation(0) reads it as on MDK_PREC_TC). */

/* how many 16-window tiles each CTA of the tensor-core recurrences runs (mdk_engine_set_rec_mode) */
#define MDK_REC_AUTO 0      /* two whatever the batch size when F <= 16 (a group's layer-1 recurrence then runs on half the
                               SMs beside the next group's layer 0); otherwise two once the tiles of both directions
                               outnumber the SMs (beyond one wave), else one */
#define MDK_REC_ONE_TILE 1  /* one tile per CTA, over several waves when the batch needs more CTAs than there are SMs */
#define MDK_REC_PINGPONG 2  /* two tiles per CTA (one N = 32 MMA chain), whatever the batch size */

/* count normalisation modes: CountsFeatureEncoder._norm_modes_ (medaka/features.py:816) */
#define MDK_NORM_TOTAL 0
#define MDK_NORM_FWD_REV 1
#define MDK_NORM_NONE 2

typedef struct mdk_engine mdk_engine;
typedef struct mdk_bam mdk_bam;              /* an open BAM file (+ its .bai index when present) */
typedef struct mdk_bam_batch mdk_bam_batch;  /* the records of one region, in BAM's packed encodings */

/* GRUModel constructor arguments (medaka/architectures/gru.py:13-21). */
typedef struct mdk_model_desc {
    int32_t num_features;   /* F = 10 * len(dtypes) */
    int32_t gru_size;       /* H: 128 (every shipped counts-matrix model) or 256 (what `medaka train` builds by default,
                               DEFAULT_MODEL_DICT); any other width fails with MDK_ERR_UNSUPPORTED */
    int32_t n_layers;       /* 2 */
    int32_t bidirectional;  /* 1 */
    int32_t num_classes;    /* linear head is hard-coded to 5 outputs (gru.py:53-55) */
} mdk_model_desc;

/* per-stage device timings of the last mdk_engine_forward* call, milliseconds (CUDA events) */
typedef struct mdk_timings {
    float h2d_ms;
    float inproj0_ms;   /* layer-0 input projection */
    float rec0_ms;      /* layer-0 recurrence (both directions) */
    float inproj1_ms;   /* layer-1 input projection GEMM */
    float rec1_ms;      /* layer-1 recurrence */
    float head_ms;      /* linear + softmax + argmax */
    float d2h_ms;
    float total_ms;
    int32_t launches;   /* kernels launched by the call */
} mdk_timings;

/* constants the Python layer reads from the library, like libmedaka.lib.plp_bases etc.
 * (src/medaka_counts.h:19-22; read at medaka/common.py:29-35, medaka/features.py:860,902-904) */
const char *mdk_plp_bases(void);   /* "acgtACGTdD" */
size_t mdk_featlen(void);          /* 10 */
size_t mdk_fwd_del(void);          /* 9 */
size_t mdk_rev_del(void);          /* 8 */

const char *mdk_last_error(void);  /* thread-local message of the last failing call */
const char *mdk_version(void);
int mdk_device_count(int *count);
/* sm major*10+minor of `device`, SM count, bytes of global memory */
int mdk_device_info(int device, int *sm_arch, int *sm_count, size_t *total_mem);

/* pinned host memory for batch staging (replaces the pageable .to(device) / .cpu() copies of
 * TorchModel.predict_on_batch, medaka/models.py:309,312) */
int mdk_host_alloc(size_t bytes, void **out);
int mdk_host_free(void *p);
/* raw device memory + copies, for callers that keep inputs resident in HBM (bench, tests) */
int mdk_dev_alloc(int device, size_t bytes, void **out);
int mdk_dev_free(int device, void *p);
int mdk_memcpy_h2d(int device, void *dst_dev, const void *src_host, size_t bytes);
int mdk_memcpy_d2h(int device, void *dst_host, const void *src_dev, size_t bytes);
int mdk_dev_memset(int device, void *dst_dev, int value, size_t bytes);
int mdk_device_synchronize(int device);

/* ---- model seam: replaces ModelStoreTGZ.load_model + TorchModel.predict_on_batch --------------
 * (medaka/datastore.py:135-157, medaka/models.py:303-313) */
int mdk_engine_create(int device, const mdk_model_desc *desc, mdk_engine **out);
int mdk_engine_destroy(mdk_engine *e);
/* load_state_dict for one (layer, direction) of gru.* ; direction 1 = "_reverse" */
int mdk_engine_load_gru(mdk_engine *e, int layer, int direction, const float *w_ih,
                        const float *w_hh, const float *b_ih, const float *b_hh);
int mdk_engine_load_linear(mdk_engine *e, const float *w, const float *b);
/* TorchModel.half() / --full_precision (medaka/prediction.py:164-168): MDK_PREC_*; any other value fails with
 * MDK_ERR_ARG.  The mode is read when a group is launched: a call that changes it launches the open group first, so no
 * group mixes modes and windows submitted before the change run in the mode they were submitted in. */
int mdk_engine_set_precision(mdk_engine *e, int mode);
int mdk_engine_get_precision(mdk_engine *e, int *mode);
/* MDK_REC_*: tiles per CTA of the recurrent kernels (A/B measurements; AUTO is the default).  At gru_size 256 the
 * recurrence has one kernel (one 4-CTA cluster per 16-window tile and direction) and only MDK_REC_AUTO is accepted. */
int mdk_engine_set_rec_mode(mdk_engine *e, int mode);
/* pre-size the compute lanes (workspace + staging) for groups of up to B windows of T columns (otherwise grown on
 * demand, to the size of the batch that opens a group - i.e. without a reserve call nothing is coalesced).  At gru_size
 * 256 B is capped at the group size (no group holds more) and the workspace (gi, h0, h1 in fp32: 10 KiB per position)
 * has a budget of 48 GiB; a reserve beyond it fails with MDK_ERR_ARG. */
int mdk_engine_reserve(mdk_engine *e, int64_t B, int64_t T);
/* predict_on_batch with HOST buffers: H2D feats, forward, D2H probs (+logits, +labels when
 * non-NULL); returns when outputs are in host memory. */
int mdk_engine_forward(mdk_engine *e, const float *feats_host, int64_t B, int64_t T,
                       float *probs_host, float *logits_host, uint8_t *labels_host);
/* asynchronous form of the same call: returns once the batch is queued.  Host buffers must stay valid (and should be
 * page-locked) until mdk_engine_wait(ticket) returns.
 * Batches are COALESCED: consecutive submits with the same T collect in a group (their features are copied to the
 * device as they arrive, behind the previous group's compute) and the group runs as ONE forward over all of its
 * windows - the reference's default batches (medaka/prediction.py:14, 100-200 windows) are a fraction of what fills an
 * H100.  A group is launched when it is full (one wave of windows, mdk_engine_preferred_windows, or as far as the
 * buffers sized by mdk_engine_reserve reach), when a batch with another T arrives, or when somebody waits for one of
 * its tickets.  Groups rotate over the staging lanes and compute on one workspace (a one-wave group fills every SM),
 * so the copies of the neighbouring groups run under the compute; small forwards (<= 2^18 positions: the B = 1 remainder
 * regions of prediction.py:196-209) rotate over 14 more lanes and run concurrently.  Results are identical to
 * uncoalesced forwards: windows never interact. */
int mdk_engine_submit(mdk_engine *e, const float *feats_host, int64_t B, int64_t T,
                      float *probs_host, float *logits_host, uint8_t *labels_host, int64_t *ticket);
int mdk_engine_wait(mdk_engine *e, int64_t ticket);
/* one-pass consensus: the same forward, but what leaves the engine is the decoded call per position instead of the
 * probabilities - labels_out uint8 [B][T] (argmax, first max wins) and quals_out uint8 [B][T] (phred+33 byte of the
 * winning probability, min(70, -10 log10(clip(1 - p_max, 1e-7, 1))), or NULL), 2 B instead of 20 B per position.  Both
 * are computed by the engine's head from the fp32 probability it produces, and are bit-identical to
 * mdk_decode_consensus on the probabilities mdk_engine_submit returns for the same features.  feats and the outputs
 * may each be host or device memory.  Packed like mdk_engine_submit (decoded and ordinary calls share groups);
 * complete after mdk_engine_wait(ticket) or mdk_engine_sync. */
int mdk_engine_submit_decoded(mdk_engine *e, const float *feats, int64_t B, int64_t T,
                              uint8_t *labels_out, uint8_t *quals_out, int64_t *ticket);
/* one-pass variant calling: the same forward, but what leaves the engine is what variant decoding needs per position,
 * 9 B instead of 20 B.  ref_bytes uint8 [B][T] in: the draft's label code per position (0..4 = '*ACGT', 0 on insertion
 * columns; 5 = 'N'; 6 = any other symbol) in the low 3 bits, 0x80 on insertion columns (minor != 0).  Out: calls_out
 * uint8 [B][T] = argmax label (first max wins) in the low 3 bits | 0x40 when it differs from the ref code | the ref
 * byte's 0x80; pred_q_out / ref_q_out float [B][T] = min(70, -10 log10(clip(1 - p, 1e-7, 1))) of the winning class's
 * and of the reference class's probability (codes 5 and 6 are scored as class 0).  Bit-identical to what
 * mdk_decode_variants computes from the probabilities mdk_engine_submit returns for the same features (pred, pred !=
 * ref code, pred_q, ref_q).  feats, ref_bytes and the outputs may each be host or device memory.  Packed like
 * mdk_engine_submit (ordinary, decoded and variant-decoded calls share groups); complete after mdk_engine_wait(ticket)
 * or mdk_engine_sync. */
int mdk_engine_submit_variant_decoded(mdk_engine *e, const float *feats, int64_t B, int64_t T, const uint8_t *ref_bytes,
                                      uint8_t *calls_out, float *pred_q_out, float *ref_q_out, int64_t *ticket);
/* launch the group that is still collecting batches (if any) without waiting for it */
int mdk_engine_flush(mdk_engine *e);
/* most windows coalesced into one group; 0 (default) = one wave, 1 = never coalesce */
int mdk_engine_set_group_windows(mdk_engine *e, int64_t windows);
/* same forward with DEVICE buffers (inputs resident in HBM); asynchronous, complete after mdk_engine_sync().  Calls are
 * packed into groups exactly like submitted batches: the features are copied into the open group's staging when the
 * call is made, a call that does not fit what is left of the group is split, and the group is launched when full, when
 * T changes, or on flush / sync; results are copied from the staging into the call's own buffers (each output buffer is
 * written only by the pieces of its call).  So the tail of one call (say 55 windows) runs together with the head of
 * the next instead of as a forward that fills a few SMs for as long as a full one.  A call of more windows than a
 * group holds runs as one forward of its own (at gru_size 128; at 256 it is cut into groups, whose workspace is bounded).
 * feats_dev and the outputs must stay untouched until the sync; give
 * calls that may be in flight together distinct output buffers. */
int mdk_engine_forward_dev(mdk_engine *e, const float *feats_dev, int64_t B, int64_t T,
                           float *probs_dev, float *logits_dev, uint8_t *labels_dev);
int mdk_engine_sync(mdk_engine *e);
/* mdk_engine_mean_timings(e, 1, out) */
int mdk_engine_last_timings(mdk_engine *e, mdk_timings *out);
/* mean per-stage device times over the last min(n_last, groups launched) forwards, n_last <= 32.  A "forward" here is
 * one launched group (one pass of the kernels over all of its windows), not one call: there can be fewer groups than
 * calls.  A group that is still open is launched first, as mdk_engine_sync does. */
int mdk_engine_mean_timings(mdk_engine *e, int n_last, mdk_timings *out);
/* bracket a timed region on the engine stream with CUDA events (bench.py) */
int mdk_engine_timer_start(mdk_engine *e);
int mdk_engine_timer_stop(mdk_engine *e, float *elapsed_ms);
/* debugging / layer-wise parity: copy an internal activation of the last forward to host.
 * which: 0 = layer-0 output [B][T][2H] fp32, 1 = layer-1 output [B][T][2H] fp32 */
int mdk_engine_read_activation(mdk_engine *e, int which, float *out_host, int64_t n_floats);
/* the same for windows first .. first + count - 1 only: out_host is [count][T][2H] (a full 1056 x 10 000 group's layer
 * output is 10.8 GB) */
int mdk_engine_read_activation_windows(mdk_engine *e, int which, int64_t first, int64_t count, float *out_host,
                                       int64_t n_floats);
/* keep != 0: leave the layer-1 output in HBM (for mdk_engine_read_activation(e, 1, ...)) by running the 5-class head as
 * its own kernel; default 0: the tensor-core path fuses the head into the layer-1 recurrence (at gru_size 128 only: at
 * 256 the head always runs as its own kernel and the layer-1 output is always kept) */
int mdk_engine_keep_activations(mdk_engine *e, int keep);
/* number of kernels launched by this engine since creation (bench.py "gpu_launches") */
int64_t mdk_engine_launch_count(mdk_engine *e);
/* Number of windows per predict_on_batch call that fills the device exactly once: the recurrent kernel runs one CTA per
 * (16-window tile, direction), so 16 * (SMs / 2) windows = 1056 on an H100 is one full wave (the reference's --batch_size
 * default, medaka/prediction.py:14 / medaka.py, is sized for its own GPUs' memory; a 200-window batch uses 26 of 132 SMs).
 * At gru_size 256 it runs one 4-CTA cluster per (tile, direction): 16 windows per two clusters that are resident at once
 * (240 on an H100 SXM).  Callers that own the batching (run_prediction) should coalesce to this size. */
int64_t mdk_engine_preferred_windows(mdk_engine *e);

/* ---- featuriser seam: replaces CountsFeatureEncoder._post_process_pileup --------------------
 * (medaka/features.py:871-935): depth = sum of counts, minor columns take the depth of their
 * major column (np.searchsorted side='left'), optional sym_indels fill, normalisation by
 * `mode`, float64 divide then cast to float32.  counts is what calculate_pileup returns
 * (size_t matrix, src/medaka_counts.h:5-14): uint64 [n][F], F = 10 * num_dtypes.
 * feats_out float32 [n][F]; depth_out int64 [n] (may be NULL).
 * Host-buffer version stages through the device; *_dev works on device pointers. */
int mdk_normalise_counts(int device, const uint64_t *counts, const int64_t *major,
                         const int64_t *minor, int64_t n, int32_t num_dtypes, int32_t mode,
                         int32_t sym_indels, float *feats_out, int64_t *depth_out);
int mdk_normalise_counts_dev(int device, const uint64_t *counts_dev, const int64_t *major_dev,
                             const int64_t *minor_dev, int64_t n, int32_t num_dtypes,
                             int32_t mode, int32_t sym_indels, float *feats_out_dev,
                             int64_t *depth_out_dev);

/* ---- featuriser seam, raw counts: replaces calculate_pileup (src/medaka_counts.c:199-372, declared
 * src/medaka_counts.h:105-108) for num_homop == 1.  htslib's BGZF/BAM decoding stays on the host
 * (medaka_b200/bam.py); the records arrive in BAM's own packed encodings:
 *   pos[n] 0-based reference start, flag[n], mapq[n], dtype[n] (datatype index, 0 when num_dtypes == 1),
 *   cigar[] uint32 (len << 4 | op) with cigar_off[n+1] (op index of each read's first op),
 *   seq[] 4-bit codes, two per byte, high nibble first, with seq_off[n+1] (byte offset of each read).
 * Region is [start, end) 0-based on one contig; reads failing the flag / min_mapQ filter of
 * src/medaka_bamiter.c:19-21 are skipped on the device (tag / RG filters are the reader's job).
 * Outputs like the plp_data struct (src/medaka_counts.h:5-14): counts uint64 [n_cols][10*num_dtypes] in
 * 'acgtACGTdD' order, major / minor [n_cols].  *n_cols_out is always set; if it exceeds max_cols the call
 * returns MDK_ERR_NOMEM without writing counts and the caller retries with larger buffers
 * (enlarge_plp_data, medaka_counts.c:266-271).  All pointers are HOST pointers. */
int mdk_pileup_counts(int device, int64_t n_rec, const int32_t *pos, const uint16_t *flag,
                      const uint8_t *mapq, const uint8_t *dtype, const uint32_t *cigar,
                      const int64_t *cigar_off, const uint8_t *seq, const int64_t *seq_off,
                      int32_t start, int32_t end, int32_t num_dtypes, int32_t min_mapq,
                      int64_t max_cols, uint64_t *counts_out, int64_t *major_out, int64_t *minor_out,
                      int64_t *n_cols_out);

/* calculate_pileup + _post_process_pileup in one device pass (src/medaka_counts.c:199-372 followed by
 * medaka/features.py:871-935): the records of mdk_pileup_counts in, the normalised float32 features [n_cols][10*num_dtypes],
 * depth [n_cols] (may be NULL) and positions out; the uint64 counts stay on the device.  mode / sym_indels as for
 * mdk_normalise_counts.  Normalising a region before it is split at coverage gaps (medaka/features.py:125-134) gives the
 * same numbers as normalising the pieces: an insertion column and its parent never sit on different sides of a gap.
 * *n_cols_out is always set; MDK_ERR_NOMEM (nothing written) when it exceeds max_cols. */
int mdk_pileup_features(int device, int64_t n_rec, const int32_t *pos, const uint16_t *flag,
                        const uint8_t *mapq, const uint8_t *dtype, const uint32_t *cigar,
                        const int64_t *cigar_off, const uint8_t *seq, const int64_t *seq_off,
                        int32_t start, int32_t end, int32_t num_dtypes, int32_t min_mapq, int32_t mode,
                        int32_t sym_indels, int64_t max_cols, float *feats_out, int64_t *depth_out,
                        int64_t *major_out, int64_t *minor_out, int64_t *n_cols_out);

/* ---- featuriser seam, read-level features: replaces calculate_read_alignment (src/medaka_read_matrix.c:277-615,
 * declared src/medaka_read_matrix.h:124-129) for one region of one contig.  Records as for mdk_pileup_counts plus
 *   qual[] base qualities (l_seq bytes per read, 0xff = absent) with qual_off[n+1],
 *   aux[] the raw optional fields with aux_off[n+1] (read for the `mv` move table -> dwell channel, calculate_dwells
 *   :154-213, and the `HP` haplotag, :405-414; may be NULL when neither channel is requested),
 *   names[] query names with name_off[n+1] (alignments of one name share a row, :386-388).
 * Output like read_aln_data (src/medaka_read_matrix.h:5-17) after the Python wrapper's `[:, :n_reads]` cut
 * (medaka/features.py:337-347): matrix int8 [n_cols][n_reads][featlen], featlen = 4 (+1 dwells) (+1 haplotype)
 * (+1 datatype when num_dtypes > 1): base 1..4 = ACGT / 5 = deletion / -1 other, base quality, strand +1 / -1, mapping
 * quality, ... ; cells no read touches are 0.  Values are NOT clipped (the wrapper's np.maximum(.., 0) is the caller's).
 * Rows follow the reference's bookkeeping (first row whose previous read ended >= 5 positions ago, or a new row;
 * row_per_read: always a new row; rows >= max_reads are dropped); n_reads = min(max_reads, deepest column) or the
 * number of rows used with row_per_read.  left_read_out / right_read_out [n_reads] (may both be NULL): index of the read
 * whose name the reference reports as read_ids_left / read_ids_right for that row, -1 = "__blank_<k>", -2 = NULL id.
 * *n_cols_out and *n_reads_out are always set; if n_cols > max_cols or n_cols * n_reads * featlen > max_cells the call
 * returns MDK_ERR_NOMEM without data and the caller retries with larger buffers (enlarge_read_aln_data_*, :85-138).
 * Known divergence: a read that finds no free row is dropped for good; the reference can let such a read alias a row
 * that is pushed after a later growth of its buffer (reads another read's struct - undefined behaviour, not reproduced).
 * All pointers are HOST pointers. */
int mdk_read_matrix(int device, int64_t n_rec, const int32_t *pos, const uint16_t *flag, const uint8_t *mapq,
                    const uint8_t *dtype, const uint32_t *cigar, const int64_t *cigar_off, const uint8_t *seq,
                    const int64_t *seq_off, const uint8_t *qual, const int64_t *qual_off, const uint8_t *aux,
                    const int64_t *aux_off, const char *names, const int64_t *name_off, int32_t start, int32_t end,
                    int32_t num_dtypes, int32_t min_mapq, int32_t row_per_read, int32_t include_dwells,
                    int32_t include_haplotype, int32_t max_reads, int64_t max_cols, int64_t max_cells,
                    int8_t *matrix_out, int64_t *major_out, int64_t *minor_out, int64_t *n_cols_out,
                    int32_t *n_reads_out, int32_t *left_read_out, int32_t *right_read_out);

/* ---- training labels: HaploidLabelScheme.encode joined to a sample's columns (medaka/labels.py:422-484,
 * medaka/features.py:979-992) for one truth alignment.  The truth record in BAM's packed encodings: pos 0-based
 * reference start, cigar[n_cigar] (len << 4 | op), seq 4-bit codes (two per byte, high nibble first) of l_seq bases,
 * every one of them A, C, G or T, and the CIGAR's query length equal to l_seq.  [clip_start, clip_end) is the window
 * the alignment was trimmed to.  labels_out[i] (int64, the dtype the reference stores) is the code ('*ACGT' -> 0..4) of
 * the truth at (major[i], minor[i]): the base aligned to major[i] (minor 0; 0 on a deletion or skip), or the minor[i]-th
 * base of the query-only run (I ops, a trailing soft clip) behind major[i]; 0 (the padding vector) where the truth has
 * no such position or major[i] lies outside the window.  MDK_ERR_ARG for a non-ACGT base or a CIGAR that does not
 * fit the sequence.  All pointers are HOST pointers. */
int mdk_truth_labels(int device, int32_t pos, const uint32_t *cigar, int64_t n_cigar, const uint8_t *seq,
                     int64_t l_seq, int32_t clip_start, int32_t clip_end, int64_t n_cols, const int64_t *major,
                     const int64_t *minor, int64_t *labels_out);

/* ---- read-level model seam: LatentSpaceLSTM (medaka/architectures/latent_space_lstm.py:34-207, the model class of the
 * `rl_` consensus models) behind TorchModel.predict_on_batch (medaka/models.py:303-313) with
 * ReadLevelFeaturesModel.get_model_input_features = batch.read_level_features (base_classes.py:29-36).
 *   mdk_rl_create   lstm_size 128 (the class default) or 384 (every released `rl_lstm384_` model) with cnn_size = 128,
 *                   5 classes, kernel sizes [1, 17], mean pooling, bidirectional; anything else -> MDK_ERR_UNSUPPORTED.
 *                   At 384 the recurrence runs on 8-CTA thread-block clusters: the first forward fails with
 *                   MDK_ERR_UNSUPPORTED if no such cluster fits the device
 *   mdk_rl_load     one state-dict tensor by its torch name ("base_embedder.weight", "read_level_conv.convs.0.weight",
 *                   "read_level_conv.convs.2.running_mean", "lstm.weight_ih_l0_reverse", "linear.bias", ...), host float32,
 *                   torch's own layouts; tensors the forward does not use (num_batches_tracked,
 *                   read_level_conv.expansion_layer.*) may be skipped
 *   mdk_rl_forward  x int8 [B][P][D][F] host (the padded read-level feature tensor, torch_ext.py:127-136: F = 4, or 5 with
 *                   dwells) -> probs float32 [B][P][5] host (softmax output, normalise = True as at inference); returns
 *                   when the probabilities are in host memory.  It is mdk_rl_submit + mdk_rl_wait, except that the open
 *                   group is launched first and the call runs as one group of its own, whatever its B */
typedef struct mdk_rl_engine mdk_rl_engine;
int mdk_rl_create(int device, int32_t lstm_size, int32_t cnn_size, int32_t use_dwells, int32_t num_classes,
                  mdk_rl_engine **out);
int mdk_rl_destroy(mdk_rl_engine *e);
int mdk_rl_load(mdk_rl_engine *e, const char *name, const float *data, int64_t n);
/* which parts run on wgmma with fp16 hi/lo operand pairs (bit set) or on the fp32 CUDA cores (validation twins):
 * bit 0 = the k = 17 convolution (99 % of the network's FLOPs at lstm_size 128), bit 1 = the LSTM recurrences (at
 * lstm_size 384 also the LSTM input projections).  Default 3: three fp16 products per contraction
 * (hi.hi + hi.lo + lo.hi), fp32-faithful.
 * bit 2 = the fp16 mode, medaka's own GPU default (the model in half precision under autocast): every contraction that
 * bits 0 and 1 put on the tensor cores takes the single product hi.hi, operands rounded to the nearest fp16 with fp32
 * accumulation: the k = 17 convolution (weights and its input y1), at lstm_size 384 the LSTM input projections (W_ih and
 * their input, z or h0), and the recurrences (W_hh and the h fed back).  Everything else is unchanged: embedding, k = 1
 * convolution, BatchNorm, ReLU, pooling and pre_pool_expansion_layer, gate math, c and h, head and softmax; at lstm_size
 * 128 the input projections stay fp32 (gemm_fp32_kernel).  The fp32 twins ignore bit 2.  So 7 = fp16, 3 = tc, 0 = fp32.
 * The mode is read when a window is staged and when its group is launched: a call that changes it launches the open
 * group first, so no group mixes modes and windows submitted before the change run in the old mode. */
int mdk_rl_set_conv(mdk_rl_engine *e, int tensor_cores);
int mdk_rl_forward(mdk_rl_engine *e, const int8_t *x_host, int64_t B, int64_t P, int64_t D, int64_t F,
                   float *probs_host);
/* asynchronous form of mdk_rl_forward: returns once the call is queued; labels_host uint8 [B][P] (may be NULL) receives
 * the argmax of each position's probabilities, first maximum wins (labels.py:1063).  x_host, probs_host and labels_host
 * must stay valid and untouched until mdk_rl_wait(ticket) returns (page-locked memory from mdk_host_alloc makes the
 * copies asynchronous).
 * Calls are PACKED: each call's convolution (which depends on its read depth D) runs when it is submitted, in slices of
 * a fixed scratch budget, and leaves the pooled LSTM input of its windows in the open group; the LSTM input
 * projections, both recurrences and the head then run ONCE per group over all of its windows - the recurrences take as
 * long for one window as for a full wave, so a 100-window batch that runs alone pays the whole 2 x P-step chain.  Calls
 * of different D share a group; a call with another P seals the group first; a call that does not fit what is left of
 * the group is split, and its ticket follows its last piece.  A group is launched when it is full
 * (mdk_rl_preferred_windows at P = 10 000, in general one recurrence wave capped by a 24 GiB budget for the group
 * buffers), when P changes, on mdk_rl_flush, or when somebody waits for one of its tickets.  Without mdk_rl_reserve a
 * group collects calls only as far as the group buffers reach (they grow to the call that opens a group).  Groups
 * complete, and tickets with them, in submission order.  Results are bit-identical to each window run alone through
 * mdk_rl_forward: windows never interact. */
int mdk_rl_submit(mdk_rl_engine *e, const int8_t *x_host, int64_t B, int64_t P, int64_t D, int64_t F,
                  float *probs_host, uint8_t *labels_host, int64_t *ticket);
/* one-pass consensus with a read-level model: the same forward, but what leaves the engine is the decoded call per
 * position instead of the probabilities - labels_out uint8 [B][P] (argmax, first max wins) and quals_out uint8 [B][P]
 * (phred+33 byte of the winning probability, as mdk_engine_submit_decoded, or NULL).  Both are computed by the engine's
 * head from the fp32 probability it produces, and are bit-identical to mdk_decode_consensus on the probabilities
 * mdk_rl_submit returns for the same features.  x_host is host memory as for mdk_rl_submit; the outputs may be host or
 * device memory.  Packed like mdk_rl_submit (ordinary and decoded calls share groups); complete after
 * mdk_rl_wait(ticket) or mdk_rl_sync. */
int mdk_rl_submit_decoded(mdk_rl_engine *e, const int8_t *x_host, int64_t B, int64_t P, int64_t D, int64_t F,
                          uint8_t *labels_out, uint8_t *quals_out, int64_t *ticket);
/* one-pass variant calling with a read-level model: ref_bytes uint8 [B][P] in, calls_out uint8 [B][P] and pred_q_out /
 * ref_q_out float [B][P] out, with the encodings of mdk_engine_submit_variant_decoded and bit-identical to what
 * mdk_decode_variants computes from the probabilities mdk_rl_submit returns for the same features.  x_host is host
 * memory; ref_bytes and the outputs may be host or device memory.  Packed like mdk_rl_submit (ordinary, decoded and
 * variant-decoded calls share groups); complete after mdk_rl_wait(ticket) or mdk_rl_sync. */
int mdk_rl_submit_variant_decoded(mdk_rl_engine *e, const int8_t *x_host, int64_t B, int64_t P, int64_t D, int64_t F,
                                  const uint8_t *ref_bytes, uint8_t *calls_out, float *pred_q_out, float *ref_q_out,
                                  int64_t *ticket);
int mdk_rl_wait(mdk_rl_engine *e, int64_t ticket);
/* launch the open group (if any) and wait for everything queued on the engine */
int mdk_rl_sync(mdk_rl_engine *e);
/* launch the group that is still collecting calls (if any) without waiting for it */
int mdk_rl_flush(mdk_rl_engine *e);
/* size the group buffers for groups of up to min(windows, the group limit at P) windows of P positions (launches the
 * open group first): a submitted group never holds more, so the reservation stays within the 24 GiB budget */
int mdk_rl_reserve(mdk_rl_engine *e, int64_t windows, int64_t P);
/* windows one group holds at P = 10 000 (the reference's chunk_len): one wave of the tensor-core recurrence (16 windows
 * per CTA at lstm_size 128, 16 per 8-CTA cluster at 384, both directions), capped by the group buffers' 24 GiB budget -
 * 112 at 384 (14 clusters of 8 CTAs fit an H100 at once) and 384 at 128.  Callers that own the batching should coalesce to this size. */
int64_t mdk_rl_preferred_windows(mdk_rl_engine *e);
/* per-stage device times of the groups that follow mdk_rl_set_timing(e, 1) (CUDA events on the engine's compute
 * stream); mdk_rl_stage_ms writes the last launched group's 6 times in ms: convolution (mask, k = 1 and k = 17
 * convolutions, pooling Linear, of all of the group's calls), layer-0 projection, layer-0 recurrence, layer-1
 * projection, layer-1 recurrence, head */
int mdk_rl_set_timing(mdk_rl_engine *e, int on);
int mdk_rl_stage_ms(mdk_rl_engine *e, float *ms);

/* ---- alignment access: what calculate_pileup gets from htslib (create_bam_fset src/medaka_bamiter.c:52-63,
 * bam_itr_querys src/medaka_counts.c:233, the flag / mapQ part of read_bam src/medaka_bamiter.c:19-21).  Native BGZF
 * inflate (zlib, a thread pool over the independent members), BAI-indexed region fetch (bins + linear index; without an
 * index the file is streamed once in bounded memory), CG-tag long CIGARs resolved like htslib does.
 *   mdk_bam_open     index_path NULL = "<path>.bai" (or "<stem>.bai") when it exists
 *   mdk_bam_fetch    records of reference `tid` overlapping [start, end) whose flag has none of `exclude_flags` and
 *                    whose mapping quality is >= min_mapq, in file (coordinate) order
 *   mdk_bam_batch_arrays   pos[n], flag[n], mapq[n], l_seq[n]; cigar[] (len << 4 | op) with cigar_off[n+1]; seq[] 4-bit
 *                    codes with seq_off[n+1] (bytes); aux[] the raw optional fields with aux_off[n+1] (tag / read-group /
 *                    datatype filters are the caller's); names[] with name_off[n+1].  Any pointer may be NULL.  The
 *                    arrays live until mdk_bam_batch_free.
 * One handle may be used from several threads (reads are serialised on it). */
int mdk_bam_open(const char *path, const char *index_path, mdk_bam **out);
int mdk_bam_close(mdk_bam *b);
int mdk_bam_n_refs(mdk_bam *b);
const char *mdk_bam_ref_name(mdk_bam *b, int i);
int32_t mdk_bam_ref_len(mdk_bam *b, int i);
int mdk_bam_has_index(mdk_bam *b);
int mdk_bam_fetch(mdk_bam *b, int tid, int32_t start, int32_t end, uint32_t exclude_flags, int min_mapq, int threads,
                  mdk_bam_batch **out);
int64_t mdk_bam_batch_size(mdk_bam_batch *x);
int mdk_bam_batch_arrays(mdk_bam_batch *x, const int32_t **pos, const uint16_t **flag, const uint8_t **mapq,
                         const int32_t **l_seq, const uint32_t **cigar, const int64_t **cigar_off,
                         const uint8_t **seq, const int64_t **seq_off, const uint8_t **aux, const int64_t **aux_off,
                         const char **names, const int64_t **name_off);
/* base qualities as stored (bam_get_qual, src/medaka_read_matrix.c:428): l_seq bytes per read, 0xff when absent;
 * qual_off[n+1] */
int mdk_bam_batch_qual(mdk_bam_batch *x, const uint8_t **qual, const int64_t **qual_off);
int mdk_bam_batch_free(mdk_bam_batch *x);

/* ---- annotation seam: replaces the per-variant body of annotate_vcf_n_reads (medaka/vcf.py:1230-1302, `medaka tools
 * annotate`) for one chunk of one contig.
 *   records      as for mdk_pileup_counts, SORTED by position; the read-group filter is the caller's (the flag / min_mapq
 *                filter of src/medaka_bamiter.c:19-21 runs on the device)
 *   contig       bytes of the contig from contig_start, contig_n of them, covering every variant's padded window (may be
 *                NULL when dpsp == 0); contig_len is the contig's full length (the windows are clipped to it)
 *   variants     var_pos[n_var] 0-based, var_ref_len[n_var]; variant v's alleles (REF first, then the ALTs) are
 *                hap_off[v] .. hap_off[v + 1] - 1, allele k's bytes alleles[allele_off[k] .. allele_off[k + 1])
 *   score        int8 [16][16] substitution scores over htslib's 4-bit codes "=ACMGRSVTWYHKDBN" (read code, haplotype
 *                code), each in [-8, 7]; haplotype bytes outside that alphabet score as N.  Gap of length k costs
 *                gap_open + (k - 1) gap_extend (parasail's sw_trace_striped_32 convention), gap_open >= gap_extend.
 * Out (host): dp_out [n_var][3] = DP, DPS fwd, DPS rev: the pileup counts (min_mapq, no depth cap) at the variant's major
 * column, 0 without coverage.  With dpsp != 0 every read that spans the padded window [max(0, pos - pad),
 * min(contig_len, pos + ref_len + pad)) is trimmed to it (trim_read, src/medaka_trimbam.c:101-246, partial = false; reads
 * of trimmed length <= 1 dropped) and aligned (exact int32 affine Smith-Waterman) to every padded haplotype:
 * sr_out [n_hap][2] reads whose first best haplotype it is, per strand (fwd, rev); sc_out [n_hap][2] their summed
 * scores; ar_out [n_var][2] reads whose scores are all equal.  stats_out [2] (may be NULL) = alignment cells, pairs;
 * kernel_ms (may be NULL) = device time of the call's kernels (CUDA events). */
int mdk_annotate(int device, int64_t n_rec, const int32_t *pos, const uint16_t *flag, const uint8_t *mapq,
                 const uint8_t *dtype, const uint32_t *cigar, const int64_t *cigar_off, const uint8_t *seq,
                 const int64_t *seq_off, const uint8_t *contig, int32_t contig_start, int32_t contig_n,
                 int32_t contig_len, int64_t n_var, const int32_t *var_pos, const int32_t *var_ref_len,
                 const int64_t *hap_off, const int64_t *allele_off, const uint8_t *alleles, int32_t pad,
                 int32_t min_mapq, int32_t dpsp, const int8_t *score, int32_t gap_open, int32_t gap_extend,
                 int64_t *dp_out, int64_t *sr_out, int64_t *ar_out, int64_t *sc_out, int64_t *stats_out,
                 float *kernel_ms);

/* ---- decode seam: replaces the array part of HaploidLabelScheme.decode_consensus ------------
 * (medaka/labels.py:1053-1085 with _phred :387-401): labels = argmax (first max wins),
 * quals = uint8(min(70, -10*log10(clip(1-p_max, 1e-7, 1)))) + 33.  probs float32 [n][5].
 * Gap removal / string building stays on the host.  quals may be NULL. */
int mdk_decode_consensus(int device, const float *probs, int64_t n, uint8_t *labels_out,
                         uint8_t *quals_out);
int mdk_decode_consensus_dev(int device, const float *probs_dev, int64_t n,
                             uint8_t *labels_out_dev, uint8_t *quals_out_dev);
/* same for float64 probabilities: all arithmetic in double, as numpy does for a float64 label_probs array */
int mdk_decode_consensus_f64(int device, const double *probs, int64_t n, uint8_t *labels_out,
                             uint8_t *quals_out);

/* Consensus stitching (medaka/stitch.py:33-85 `_stitch_samples`: per trimmed sample decode_consensus(with_qualities)
 * -> gap removal -> append).  The caller plans the kept row ranges (overlap trimming medaka/common.py:327-427,495-557,
 * region trimming :560-609, depth filter :612-644) and passes one pointer per range; the library copies only those
 * rows in, decodes them, removes gap calls and returns the concatenated ASCII bases / phred+33 quality characters.
 *   seg_probs[k]   host float32 [seg_rows[k]][5], first kept row of range k;  seg_rows[k] > 0
 *   seq_out/qual_out  host, capacity sum(seg_rows) bytes (qual_out may be NULL)
 *   seg_out_off    host [n_seg + 1]: range k produced seq_out[seg_out_off[k] : seg_out_off[k+1]]
 * The _dev form takes the ranges already back to back on the device (probs_dev [n_rows][5], 16-byte aligned) with
 * seg_base[k] = first row of range k (host array, strictly increasing from 0); seq/qual outputs are device pointers
 * of capacity n_rows, seg_out_off stays a host array. */
int mdk_stitch_consensus(int device, const float *const *seg_probs, const int64_t *seg_rows, int64_t n_seg,
                         uint8_t *seq_out, uint8_t *qual_out, int64_t *seg_out_off);
int mdk_stitch_consensus_dev(int device, const float *probs_dev, int64_t n_rows, const int64_t *seg_base,
                             int64_t n_seg, uint8_t *seq_out_dev, uint8_t *qual_out_dev, int64_t *seg_out_off);
/* The same stitch on decoded outputs already on the device (mdk_engine_submit_decoded): segment k is the rows
 * [seg_start[k], seg_start[k] + seg_rows[k]) of labels_dev / quals_dev (quals_dev may be NULL), seg_rows[k] > 0; every
 * row lies inside the allocations labels_dev and quals_dev point into.
 * Segments may come in any order and overlap.  seg_start, seg_rows and seg_out_off are host arrays; seq_out / qual_out
 * are host buffers of capacity sum(seg_rows) (qual_out may be NULL).  Runs on the legacy stream: the engine that wrote
 * the arena must have been synchronised (mdk_engine_sync).  Equal byte for byte to mdk_stitch_consensus on the
 * probabilities the labels / quals were derived from. */
int mdk_stitch_labels_dev(int device, const uint8_t *labels_dev, const uint8_t *quals_dev,
                          const int64_t *seg_start, const int64_t *seg_rows, int64_t n_seg,
                          uint8_t *seq_out, uint8_t *qual_out, int64_t *seg_out_off);
/* Join and decode on the outputs of mdk_engine_submit_variant_decoded already on the device.  A piece k is the rows
 * [0, seg_rows[k]) at the device addresses seg_calls[k] (call bytes) and seg_pred_q[k] / seg_ref_q[k] (phreds);
 * seg_rows[k] > 0.  The pointer tables and every other array are host memory.  Both run on the legacy stream: the engine
 * that wrote the outputs must have been synchronised (mdk_engine_sync).
 * mdk_variant_join_cuts: per trimmed piece, cut_out[k] = the index of its last insertion-free column whose call equals
 * the draft, or -1 when no column has call == draft != '*' - what join_samples (medaka/variant.py:84-93) reads of the
 * labels.
 * mdk_decode_variants_dev: mdk_decode_variants over joined samples; joined sample s is the pieces
 * [sample_seg[s], sample_seg[s + 1]) back to back (sample_seg[0] = 0, sample_seg[n_samples] = n_seg, none empty).
 * Neither the variant-column rule nor a run crosses a joined sample's edge.  Per run (in sample, then column order):
 * run_sample, run_start (column within its sample), run_len and the two float32 left-to-right sums.  run_pred receives
 * the labels of all run columns back to back (run k's at the sum of the earlier runs' lengths), run_col_pred_q /
 * run_col_ref_q (both or neither may be NULL) their phreds, ref_q_out (or NULL) the reference phred of every column of
 * every sample, back to back.  When more than max_runs runs or max_run_cols run columns are found, returns
 * MDK_ERR_NOMEM with *n_runs_out / *n_run_cols_out set (retry with larger buffers).  MDK_ERR_ARG when a joined sample
 * starts on an insertion column (labels.py:909-911). */
int mdk_variant_join_cuts(int device, const uint8_t *const *seg_calls, const int64_t *seg_rows, int64_t n_seg,
                          int64_t *cut_out);
int mdk_decode_variants_dev(int device, const uint8_t *const *seg_calls, const float *const *seg_pred_q,
                            const float *const *seg_ref_q, const int64_t *seg_rows, int64_t n_seg,
                            const int64_t *sample_seg, int64_t n_samples, int64_t max_runs, int64_t *run_sample,
                            int64_t *run_start, int64_t *run_len, float *run_pred_q, float *run_ref_q,
                            int64_t max_run_cols, uint8_t *run_pred, float *run_col_pred_q, float *run_col_ref_q,
                            float *ref_q_out, int64_t *n_runs_out, int64_t *n_run_cols_out);

/* variant_columns (src/medaka_rnn_variants.h:26, called at medaka/labels.py:869-887): which pileup columns belong
 * to a variant run.  minor [len] pileup minor indices; reference / prediction [len] one byte per column (the
 * symbol or label code incl. the gap - the reference passes wchar_t strings, any 1-byte coding with the same
 * equalities works); out [len] 0/1.  Host pointers. */
int mdk_variant_columns(int device, const int64_t *minor, const uint8_t *reference,
                        const uint8_t *prediction, uint8_t *out, int64_t len);

/* Variant decoding (medaka/labels.py:889-1014 `HaploidLabelScheme.decode_variants`, the array half): for one joined
 * sample of n pileup columns
 *   pred[i]      = argmax label of probs[i] (gaps kept; labels.py:917)
 *   is_var[i]    = variant_columns(minor, reference-with-gaps, prediction)   (src/medaka_rnn_variants.c:28-55)
 *   pred_q[i]    = phred(1 - probs[i][pred[i]]),  ref_q[i] = phred(1 - probs[i][ref_code[i]])   (labels.py:387-401,
 *                  float32; 'N' is scored as the gap class, labels.py:949-952)
 *   runs         = maximal runs of variant columns (common.rle, labels.py:928-930): first column, length and the
 *                  left-to-right float32 sums of pred_q / ref_q over the run (labels.py:957-975; the variant's
 *                  quality is run_pred_q - run_ref_q)
 * ref_code[i]: 0..4 = '*ACGT' with 0 on insertion columns (minor != 0), 5 = 'N', 6+ = any other draft symbol.
 * Strings, the ref == alt / ambiguous-reference filters and VCF normalisation stay on the host (medaka_b200/labels.py).
 * Host pointers; pred_q_out / ref_q_out may be NULL.  *n_runs_out is always set; if it exceeds max_runs the call
 * returns MDK_ERR_NOMEM without run data and the caller retries with larger buffers. */
int mdk_decode_variants(int device, const float *probs, const int64_t *minor, const uint8_t *ref_code, int64_t n,
                        uint8_t *pred_out, uint8_t *is_var_out, float *pred_q_out, float *ref_q_out, int64_t max_runs,
                        int64_t *run_start, int64_t *run_len, float *run_pred_q, float *run_ref_q,
                        int64_t *n_runs_out);

/* ---- self test of the wgmma building block (one 128xN tile GEMM), used by tests ------------
 * Computes D[128][N] = A[128][K] * B[N][K]^T with the same smem layouts, descriptors and
 * fp16 hi/lo split the GRU kernels use.  A, B, D are host fp32.  variant must be 0 (the
 * production descriptor encoding). */
int mdk_selftest_umma(int device, const float *A, const float *B, float *D, int N, int K,
                      int variant);

/* ---- diagnostics -------------------------------------------------------------------------
 * completion times (ms after mdk_engine_timer_start's event) of the eight stage events of the last n_last launched
 * groups, oldest first: out is float[n_last][8] = start, features in, inproj0, rec0, inproj1, rec1, head, end.  Shows
 * how the lanes' kernels actually interleaved.  An open group is launched first. */
int mdk_debug_timeline(mdk_engine *e, int n_last, float *out);
/* partial logits of the last forward on the fused-head path: float32 [2 directions][tiles][T][5 classes][16 windows]
 * (what the layer-1 recurrence writes instead of h1); per-direction parity checks of the fused linear head */
int mdk_debug_read_plog(mdk_engine *e, float *out_host, int64_t n_floats);
/* layer-wise parity of the read-level network: copy one intermediate of the LAST mdk_rl_forward call (B, P of that call)
 * from the engine's scratch to host.  which: 0 = z [B][P][H] (the pooled pre_pool_expansion_layer output, the LSTM
 * input), 1 = h0 [B][P][2H] (layer-0 output, columns direction * H + unit), 2 = h1 [B][P][2H] (layer-1 output).
 * MDK_ERR_STATE before the first completed forward, MDK_ERR_ARG when n_floats is not the stage's size. */
int mdk_rl_debug_read(mdk_rl_engine *e, int which, float *out_host, int64_t n_floats);

/* ---- training seam: replaces the GRUModel forward / backward, CrossEntropyLoss, clip_grad_norm_ and the torch.optim
 * step of medaka train (medaka/torch_ext.py run_epoch, medaka/models.py process_batch) for the consensus GRU of
 * mdk_model_desc (2 layers, bidirectional, gru_size 128 or 256, 5 classes).  fp32 throughout, the arithmetic of
 * MDK_PREC_FP32: the forward's logits and probabilities equal mdk_engine_forward's at MDK_PREC_FP32 bit for bit.
 * An mdk_trainer is separate from any mdk_engine; it keeps fp32 master weights, their gradient and the optimizer state
 * on the device.  Weights: the flat array of mdk_trainer_read_params is the state dict in torch order (per layer and
 * direction weight_ih, weight_hh, bias_ih, bias_hh; then linear.weight, linear.bias), mdk_trainer_num_params floats. */
typedef struct mdk_trainer mdk_trainer;

#define MDK_OPT_RMSPROP 0   /* torch.optim.RMSprop (alpha, eps, weight_decay, momentum; not centered) */
#define MDK_OPT_ADAM 1      /* torch.optim.Adam (beta1, beta2, eps, weight_decay; not amsgrad) */
#define MDK_OPT_NADAM 2     /* torch.optim.NAdam (beta1, beta2, eps, weight_decay, momentum_decay) */
#define MDK_OPT_SGD 3       /* torch.optim.SGD (momentum, dampening, weight_decay, nesterov) */

typedef struct mdk_optim_desc {
    int32_t kind;           /* MDK_OPT_* */
    float alpha, beta1, beta2, eps, weight_decay, momentum, dampening, momentum_decay;
    int32_t nesterov;
} mdk_optim_desc;

typedef struct mdk_train_stats {
    double loss;            /* CrossEntropyLoss() of the batch: mean over the B*T positions */
    int64_t n_correct;      /* positions whose argmax (first maximum) of the logits is the label */
    int64_t n_positions;
    float grad_norm;        /* L2 norm of all gradients before clipping (mdk_trainer_step only); NaN or inf when
                               a gradient is not finite */
    int32_t skipped;        /* the update was skipped (non-finite gradient): weights and optimizer state unchanged */
} mdk_train_stats;

int mdk_trainer_create(int device, const mdk_model_desc *desc, mdk_trainer **out);
int mdk_trainer_destroy(mdk_trainer *tr);
/* as mdk_engine_load_gru / mdk_engine_load_linear; a load resets the optimizer state and leaves the tensors it does not
 * name at their current (trained) values */
int mdk_trainer_load_gru(mdk_trainer *tr, int layer, int direction, const float *w_ih, const float *w_hh,
                         const float *b_ih, const float *b_hh);
int mdk_trainer_load_linear(mdk_trainer *tr, const float *w, const float *b);
/* the optimizer and its hyper-parameters (the learning rate is per step); resets its state.  Default: RMSprop with
 * the reference's arguments (alpha 0.9, eps 1e-7, momentum 0) */
int mdk_trainer_set_optimizer(mdk_trainer *tr, const mdk_optim_desc *opt);
/* One training step on B windows of T columns (host buffers: feats float32 [B][T][F], labels int32 [B][T] in [0, 5),
 * MDK_ERR_ARG otherwise): forward, loss, backward, then - unless the gradient norm is not finite, which skips the
 * update as GradScaler.step does - the gradients scaled by max_norm / (norm + 1e-6) when that is below 1
 * (clip_grad_norm_; max_norm <= 0 means no clipping) and one optimizer step at learning rate lr.  Returns once the
 * statistics are on the host.  The stored gradient (mdk_trainer_read_grads) is the unclipped one. */
int mdk_trainer_step(mdk_trainer *tr, const float *feats, const int32_t *labels, int64_t B, int64_t T, float lr,
                     float max_norm, mdk_train_stats *stats);
/* forward and loss without a backward pass (validation).  labels may be NULL (no loss); probs / logits (host float32
 * [B][T][5]) may be NULL. */
int mdk_trainer_eval(mdk_trainer *tr, const float *feats, const int32_t *labels, int64_t B, int64_t T, float *probs,
                     float *logits, mdk_train_stats *stats);
int mdk_trainer_num_params(mdk_trainer *tr, int64_t *n);
int mdk_trainer_read_params(mdk_trainer *tr, float *out_host, int64_t n);
int mdk_trainer_read_grads(mdk_trainer *tr, float *out_host, int64_t n);
/* device bytes a step of B windows x T columns needs (about 28 gru_size floats per position), and the budget above
 * which a step fails with MDK_ERR_ARG (64 GiB) */
int mdk_trainer_workspace_bytes(const mdk_model_desc *desc, int64_t B, int64_t T, size_t *bytes, size_t *budget);
/* device times of the last step in ms (CUDA events): forward (with the feature and label copies), loss and head
 * backward, BPTT recurrences, gradient reductions (and layer 1's dX), optimizer step (norm, update, weight repack) */
int mdk_trainer_stage_ms(mdk_trainer *tr, float *ms);
/* windows per CTA of the BPTT kernel: 1, 2, 4 or 8, or 0 (default) to choose from B (the fewest whose CTAs still fill
 * no more than one wave).  The gradients do not depend on it.  For tests and measurements. */
int mdk_trainer_set_bptt_windows(mdk_trainer *tr, int nb);
/* windows per CTA the BPTT kernel runs at for a batch of B windows, under the current setting */
int mdk_trainer_bptt_windows(mdk_trainer *tr, int64_t B, int *nb);

/* ---- read-level training: medaka train for the LatentSpaceLSTM the read-level engine accepts (bidirectional, mean
 * pooling, kernel sizes 1 and 17, cnn_size 128, lstm_size 128 or 384, 5 classes, with or without dwells), fp32.  The
 * model is in training mode: both BatchNorm layers normalise with the batch's statistics over all B*D*P elements of the
 * padded batch (empty and padding reads included) and update their running statistics (momentum 0.1, unbiased
 * variance) at every step, a skipped one included.  Per-read activations live only in a bounded scratch: device
 * memory grows with B*P and the int8 features, not with the read depth.
 * Weights: the flat array of mdk_rl_trainer_read_params is named_parameters() in order (read_level_conv.
 * expansion_layer included: the forward never uses it, so it gets no gradient and no update).  The BatchNorm running
 * statistics and num_batches_tracked are kept apart (mdk_rl_trainer_read_buffers). */
typedef struct mdk_rl_trainer mdk_rl_trainer;

int mdk_rl_trainer_create(int device, int32_t lstm_size, int32_t cnn_size, int32_t use_dwells, int32_t num_classes,
                          mdk_rl_trainer **out);
int mdk_rl_trainer_destroy(mdk_rl_trainer *tr);
/* one tensor by its torch state-dict name (parameters and buffers; num_batches_tracked as one float); resets the
 * optimizer state, and the tensors it does not name keep their current values */
int mdk_rl_trainer_load(mdk_rl_trainer *tr, const char *name, const float *data, int64_t n);
int mdk_rl_trainer_set_optimizer(mdk_rl_trainer *tr, const mdk_optim_desc *opt);
/* One training step on x int8 [B][P][D][F] (strand + 1 clamped to [0, 2], as the engine reads it) and labels int32
 * [B][P] in [0, 5): as mdk_trainer_step.  F is 5 with dwells, 4 or more without (MDK_ERR_ARG otherwise). */
int mdk_rl_trainer_step(mdk_rl_trainer *tr, const int8_t *x, const int32_t *labels, int64_t B, int64_t P, int64_t D,
                        int64_t F, float lr, float max_norm, mdk_train_stats *stats);
/* validation (model.eval()): the running statistics, the read-level engine's fp32 kernels (probabilities equal the
 * engine's fp32 path bit for bit); labels, probs, logits may be NULL */
int mdk_rl_trainer_eval(mdk_rl_trainer *tr, const int8_t *x, const int32_t *labels, int64_t B, int64_t P, int64_t D,
                        int64_t F, float *probs, float *logits, mdk_train_stats *stats);
int mdk_rl_trainer_num_params(mdk_rl_trainer *tr, int64_t *n);
int mdk_rl_trainer_read_params(mdk_rl_trainer *tr, float *out_host, int64_t n);
/* out: running_mean, running_var of convs.2, then of convs.5 (n = 4 cnn_size); num_batches_tracked[2] may be NULL */
int mdk_rl_trainer_read_buffers(mdk_rl_trainer *tr, float *out_host, int64_t n, int64_t *num_batches_tracked);
int mdk_rl_trainer_read_grads(mdk_rl_trainer *tr, float *out_host, int64_t n);
/* device bytes a step on B x P x D x F needs, and the budget above which a step fails with MDK_ERR_ARG (64 GiB) */
int mdk_rl_trainer_workspace_bytes(int32_t lstm_size, int64_t B, int64_t P, int64_t D, int64_t F, size_t *bytes,
                                   size_t *budget);
/* device times of the last step in ms: stats pass, forward pass (with the copies), LSTM forward, loss and head
 * backward, BPTT, read backward pass, reductions, optimizer step */
int mdk_rl_trainer_stage_ms(mdk_rl_trainer *tr, float *ms);
/* windows per CTA of the LSTM BPTT kernel: 1, 2, 4 or 8, or 0 (default) to choose from B as mdk_trainer_set_bptt_windows
 * does.  The gradients do not depend on it.  For tests and measurements. */
int mdk_rl_trainer_set_bptt_windows(mdk_rl_trainer *tr, int nb);
/* the (window, read) rows of one slice of the forward and read backward passes: rows >= 1 caps the slice at
 * min(rows, the automatic length), 0 (default) takes the automatic length (the per-read scratch's capacity, at most
 * 65535 rows).  The workspace is sized for the automatic length.  For tests and measurements. */
int mdk_rl_trainer_set_slice_rows(mdk_rl_trainer *tr, int64_t rows);
/* windows per CTA the BPTT kernel runs at for a batch of B windows, under the current setting */
int mdk_rl_trainer_bptt_windows(mdk_rl_trainer *tr, int64_t B, int *nb);

#ifdef __cplusplus
}
#endif
#endif /* MEDAKA_B200_H */
