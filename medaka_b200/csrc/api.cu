// C ABI of libmedaka_b200 (include/medaka_b200.h): the consensus (GRU) engine - life-cycle, weight loading (host copies,
// packed on the host by gru_pack.cuh and uploaded before the first forward after a load), the forward pipeline - and the
// device utilities, error reporting and cached device blobs the other entry points share.  Host orchestration only - the
// engine's kernels live in misc.cu, gru_fp32.cu and gru_wg.cu.  The featuriser entry points are in pileup.cu, the decode
// entry points in decode.cu, the read-level engine in readlevel.cu.
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <new>

#include "common.cuh"
#include "gru_pack.cuh"

namespace mdk {

static thread_local std::string g_last_error;

void set_error(const std::string &msg) { g_last_error = msg; }

int cuda_fail(cudaError_t err, const char *what, const char *file, int line) {
    char buf[512];
    snprintf(buf, sizeof(buf), "CUDA error %d (%s) at %s:%d: %s", (int)err, cudaGetErrorString(err), file, line, what);
    g_last_error = buf;
    if (err == cudaErrorMemoryAllocation) {
        cudaGetLastError();
        return MDK_ERR_NOMEM;
    }
    return MDK_ERR_CUDA;
}

struct CachedBlob {
    int device = -1;
    uint8_t *buf = nullptr;
    size_t cap = 0;
    ~CachedBlob() {
        if (buf) cudaFree(buf);
    }
};
static thread_local CachedBlob g_blob[2];     // indexed by Blob

cudaError_t cached_blob(Blob role, size_t bytes, uint8_t **out) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    CachedBlob &b = g_blob[(int)role];
    if (b.device != dev || b.cap < bytes) {
        if (b.buf) cudaFree(b.buf);
        b.buf = nullptr;
        b.cap = 0;
        const size_t want = bytes + bytes / 4 + (1 << 20);
        e = cudaMalloc(&b.buf, want);
        if (e != cudaSuccess) return e;
        b.cap = want;
        b.device = dev;
    }
    *out = b.buf;
    return cudaSuccess;
}

template <typename T>
static int dev_alloc(T **p, size_t n_elems) {
    MDK_CUDA(cudaMalloc(reinterpret_cast<void **>(p), n_elems * sizeof(T)));
    return MDK_OK;
}
template <typename T>
static void dev_free(T *&p) {
    if (p) cudaFree(p);
    p = nullptr;
}

// Both streams of a workspace: what its buffers are read or written by
static cudaError_t ws_sync(mdk_ws &ws) {
    cudaError_t err = cudaStreamSynchronize(ws.stream);
    return err == cudaSuccess ? cudaStreamSynchronize(ws.l1_stream) : err;
}

static int in_features(const mdk_engine *e, int layer) { return layer == 0 ? e->desc.num_features : 2 * e->desc.gru_size; }

// At gru_size 256 the workspace holds gi, h0 and h1 as fp32 rows: 6H + 2H + 2H floats, 10 KiB per position (24.6 GB
// for one wave of 240 windows x 10 000 columns on an H100 SXM).  Groups are cut to one wave and mdk_engine_reserve caps
// its windows at a group, so only longer windows or a larger mdk_engine_set_group_windows can ask for more; beyond this
// budget the forward fails instead of taking the whole card.
constexpr int64_t WS256_BYTES_PER_POS = (int64_t)(GI256_COLS + 2 * H2_256) * sizeof(float);
constexpr int64_t WS256_BUDGET = (int64_t)48 << 30;

// The weights as the kernels read them, packed on the host (gru_pack.cuh) and uploaded once after each load.
static int prepare_weights(mdk_engine *e) {
    if (e->prepared) return MDK_OK;
    for (int l = 0; l < 2; ++l) {
        MDK_REQUIRE(!e->layer[l].w_ih[0].empty() && !e->layer[l].w_ih[1].empty(), MDK_ERR_STATE,
                    "engine: GRU weights not loaded for every (layer, direction)");
    }
    MDK_REQUIRE(!e->lin_w_host.empty(), MDK_ERR_STATE, "engine: linear head weights not loaded");
    DeviceWeights &dw = e->weights;
    int rc;
    for (int l = 0; l < 2; ++l) {
        LayerWeights &lw = e->layer[l];
        const PackedLayer p = pack_layer(lw, in_features(e, l), l, e->desc.gru_size);
        if ((rc = dw.upload(e->stream, &lw.w_in_packed, p.w_in_packed)) || (rc = dw.upload(e->stream, &lw.bias_gi, p.bias_gi)) ||
            (rc = dw.upload(e->stream, &lw.b_hn, p.b_hn)) || (rc = dw.upload(e->stream, &lw.bias_gi_tc, p.bias_gi_tc)) ||
            (rc = dw.upload(e->stream, &lw.b_hn_tc, p.b_hn_tc)) || (rc = dw.upload(e->stream, &lw.w_hh_t, p.w_hh_t)) ||
            (rc = dw.upload(e->stream, &lw.w_hh_tm, p.w_hh_tm)) || (rc = dw.upload(e->stream, &lw.w_x_tm, p.w_x_tm)) ||
            (rc = dw.upload(e->stream, &lw.w_in_tc, p.w_in_tc)))
            return rc;
    }
    if ((rc = dw.upload(e->stream, &e->lin_w, e->lin_w_host)) || (rc = dw.upload(e->stream, &e->lin_b, e->lin_b_host)))
        return rc;
    e->prepared = true;
    return MDK_OK;
}

static int ensure_workspace(mdk_engine *e, mdk_ws &ws, int64_t B, int64_t T) {
    // rows of the tile-interleaved intermediates (>= B*T: the last window tile is padded to 16 windows)
    const int64_t rows = tiled_rows(B, T);
    const int64_t need = ((rows + XT_ROWS - 1) / XT_ROWS) * XT_ROWS;
    if (need <= ws.cap_pos) return MDK_OK;
    const bool wide = e->desc.gru_size == H256;
    MDK_REQUIRE(!wide || need * WS256_BYTES_PER_POS <= WS256_BUDGET, MDK_ERR_ARG,
                "engine: at gru_size 256 a forward of this many positions exceeds the 48 GiB workspace budget (10 KiB "
                "per position)");
    MDK_CUDA(ws_sync(ws));
    dev_free(ws.gi);
    if (ws.h0) { cudaFree(ws.h0); ws.h0 = nullptr; }
    dev_free(ws.h1);
    ws.cap_h1 = 0;
    dev_free(ws.plog);
    ws.cap_pos = 0;
    int rc;
    if ((rc = dev_alloc(&ws.gi, (size_t)need * (wide ? GI256_COLS : GI_COLS)))) return rc;
    MDK_CUDA(cudaMalloc(&ws.h0, (size_t)need * (wide ? H2_256 : H2) * sizeof(float)));
    if (!wide && (rc = dev_alloc(&ws.plog, (size_t)NDIR * (need / WT) * PLOG_TS_FLOATS))) return rc;
    ws.cap_pos = need;
    return MDK_OK;
}

// h1 (the layer-1 output, 1 KiB / position, 2 KiB at gru_size 256) only exists on the unfused-head paths: allocated on
// first use
static int ensure_h1(mdk_ws &ws, int width) {
    if (ws.cap_h1 >= ws.cap_pos && ws.h1) return MDK_OK;
    MDK_CUDA(ws_sync(ws));
    dev_free(ws.h1);
    ws.cap_h1 = 0;
    int rc;
    if ((rc = dev_alloc(&ws.h1, (size_t)ws.cap_pos * width))) return rc;
    ws.cap_h1 = ws.cap_pos;
    return MDK_OK;
}

static int ensure_io(mdk_engine *e, mdk_lane &ln, int64_t B, int64_t T) {
    const int64_t P = B * T;
    const int64_t feats = P * e->desc.num_features;
    if (P <= ln.cap_io && feats <= ln.cap_feats) return MDK_OK;
    MDK_CUDA(ws_sync(*ln.ws));
    MDK_CUDA(cudaStreamSynchronize(e->copy_in));
    MDK_CUDA(cudaStreamSynchronize(e->copy_out.stream));
    ln.cap_io = 0; ln.cap_feats = 0; ln.cap_quals = 0; ln.cap_var = 0;
    dev_free(ln.d_feats); dev_free(ln.d_probs); dev_free(ln.d_logits); dev_free(ln.d_labels); dev_free(ln.d_quals);
    dev_free(ln.d_ref); dev_free(ln.d_calls); dev_free(ln.d_pred_q); dev_free(ln.d_ref_q);
    int rc;
    if ((rc = dev_alloc(&ln.d_feats, (size_t)feats))) return rc;
    if ((rc = dev_alloc(&ln.d_probs, (size_t)P * NCLS))) return rc;
    if ((rc = dev_alloc(&ln.d_logits, (size_t)P * NCLS))) return rc;
    if ((rc = dev_alloc(&ln.d_labels, (size_t)P))) return rc;
    ln.cap_io = P; ln.cap_feats = feats;
    return MDK_OK;
}

// d_quals (1 B / position) only exists on lanes that have run a decoded call (mdk_engine_submit_decoded): allocated
// when the group being launched needs it.  The lane's previous group has left it (acquire_lane), and ensure_io, which
// frees it on growth, synchronises first.
static int ensure_quals(mdk_lane &ln) {
    if (ln.cap_quals >= ln.cap_io && ln.d_quals) return MDK_OK;
    dev_free(ln.d_quals);
    ln.cap_quals = 0;
    int rc;
    if ((rc = dev_alloc(&ln.d_quals, (size_t)ln.cap_io))) return rc;
    ln.cap_quals = ln.cap_io;
    return MDK_OK;
}

// The variant-decoded calls' buffers (mdk_engine_submit_variant_decoded, 10 B / position): the reference bytes, staged
// next to the features, and the call bytes and phreds the head writes.  Allocated like d_quals, but when the first
// variant piece is staged (its reference bytes go in then): a lane never frees them while a group collects, because
// ensure_io only runs when a group opens.
static int ensure_var(mdk_lane &ln) {
    if (ln.cap_var >= ln.cap_io && ln.d_ref) return MDK_OK;
    dev_free(ln.d_ref); dev_free(ln.d_calls); dev_free(ln.d_pred_q); dev_free(ln.d_ref_q);
    ln.cap_var = 0;
    int rc;
    if ((rc = dev_alloc(&ln.d_ref, (size_t)ln.cap_io))) return rc;
    if ((rc = dev_alloc(&ln.d_calls, (size_t)ln.cap_io))) return rc;
    if ((rc = dev_alloc(&ln.d_pred_q, (size_t)ln.cap_io))) return rc;
    if ((rc = dev_alloc(&ln.d_ref_q, (size_t)ln.cap_io))) return rc;
    ln.cap_var = ln.cap_io;
    return MDK_OK;
}

// The forward at gru_size 256, on the same streams and events as run_forward: the layer-0 input projection, the layer-0
// recurrence and the layer-1 projection on ws.stream, the layer-1 recurrence and the head on ws.l1_stream.  Every
// stage reads or writes gi, so each forward's first kernel waits for the previous forward's layer 1.
static int run_forward256(mdk_engine *e, mdk_ws &ws, const float *feats_dev, int64_t B, int64_t T, float *probs_dev,
                          float *logits_dev, uint8_t *labels_dev, uint8_t *quals_dev, const HeadVariant *var) {
    int rc;
    if ((rc = ensure_h1(ws, H2_256))) return rc;
    const int64_t P = B * T;
    cudaStream_t s = ws.stream, s1 = ws.l1_stream;
    const bool tc = e->precision != MDK_PREC_FP32, fp16 = e->precision == MDK_PREC_FP16;
    const LayerWeights &l0 = e->layer[0], &l1 = e->layer[1];
    float *h0 = static_cast<float *>(ws.h0);
    MDK_CUDA(cudaStreamWaitEvent(s, ws.l1_done, 0));
    MDK_CUDA(cudaEventRecord(e->ev[1], s));
    MDK_CUDA(launch_inproj0(feats_dev, l0.w_in_packed, l0.bias_gi, ws.gi, P, e->desc.num_features,
                            T, tc ? 1 : 0, s, H256));
    MDK_CUDA(cudaEventRecord(e->ev[2], s));
    if (tc) MDK_CUDA(launch_rec256_tc(ws.gi, l0.w_hh_tm, l0.b_hn_tc, h0, B, T, fp16, s));
    else MDK_CUDA(launch_rec_fp32(ws.gi, l0.w_hh_t, l0.b_hn, h0, B, T, s, H256));
    MDK_CUDA(cudaEventRecord(e->ev[3], s));
    if (tc) MDK_CUDA(launch_gemm256_tc(h0, l1.w_in_tc, l1.bias_gi_tc, ws.gi, tiled_rows(B, T), fp16, s));
    else MDK_CUDA(launch_gemm_fp32(h0, l1.w_in_packed, l1.bias_gi, ws.gi, P, H2_256, GI256_COLS, s));
    MDK_CUDA(cudaEventRecord(e->ev[4], s));
    MDK_CUDA(cudaStreamWaitEvent(s1, e->ev[4], 0));
    if (tc) MDK_CUDA(launch_rec256_tc(ws.gi, l1.w_hh_tm, l1.b_hn_tc, ws.h1, B, T, fp16, s1));
    else MDK_CUDA(launch_rec_fp32(ws.gi, l1.w_hh_t, l1.b_hn, ws.h1, B, T, s1, H256));
    MDK_CUDA(cudaEventRecord(e->ev[5], s1));
    MDK_CUDA(cudaEventRecord(ws.l1_done, s1));
    MDK_CUDA(launch_head(ws.h1, e->lin_w, e->lin_b, B, T, tc ? 1 : 0, probs_dev, logits_dev, labels_dev, s1, quals_dev,
                         var, H2_256));
    MDK_CUDA(cudaEventRecord(e->ev[6], s1));
    e->launches += 5;
    e->last.launches = 5;
    ws.last_fused_head = false;
    ws.last_B = B; ws.last_T = T; ws.last_precision = e->precision;
    e->last_ws = (int)(&ws - e->ws);
    return MDK_OK;
}

// The forward pipeline on the workspace's two streams: [layer-0 input projection,] layer 0 and the layer-1 projection on
// ws.stream, layer 1 and the head on ws.l1_stream.  ev[1..6] bracket the stages for mdk_timings; the wait for the previous
// forward's layer 1 falls into h2d_ms (unfused layer 0) or rec0_ms (fused), and with the fused layer 0 the rec0_ms and
// rec1_ms of consecutive forwards overlap in wall time.
static int run_forward(mdk_engine *e, mdk_ws &ws, const float *feats_dev, int64_t B, int64_t T, float *probs_dev,
                       float *logits_dev, uint8_t *labels_dev, uint8_t *quals_dev, const HeadVariant *var) {
    int rc;
    if ((rc = prepare_weights(e))) return rc;
    if ((rc = ensure_workspace(e, ws, B, T))) return rc;
    if (e->desc.gru_size == H256)
        return run_forward256(e, ws, feats_dev, B, T, probs_dev, logits_dev, labels_dev, quals_dev, var);
    const int64_t P = B * T;
    cudaStream_t s = ws.stream, s1 = ws.l1_stream;
    // tc: the tensor-core kernels, in the fp16 mode's one-product form or the three-product default
    const bool tc = e->precision != MDK_PREC_FP32, fp16 = e->precision == MDK_PREC_FP16;
    int launches = 0;
    const bool fuse_x = tc && e->layer[0].w_x_tm != nullptr;     // F <= 16
    // Recurrent kernels of the tensor-core path.  With the fused layer-0 projection AUTO runs two tiles per CTA (one
    // N = 32 MMA chain) for every forward: a group's layer 1 then takes half the SMs and the next group's layer 0 the
    // other half, which does a group's two recurrences in less SM time than one tile per CTA on all of them in turn.
    // It does not depend on B, so a window's outputs are the same whether it is packed into a group or runs alone.
    // Otherwise layer 0 reads gi and cannot overlap the previous layer 1: one 16-window tile per CTA (a single dependent
    // chain per SM) while the tiles of both directions fit the SMs, two beyond.  The linear head rides inside the layer-1
    // recurrence, fp32 on the CUDA cores (40 B/position of partial logits reach HBM instead of the 1 KiB/position h1
    // round trip), unless h1 is to be kept.
    const int64_t tiles = (B + WT - 1) / WT;
    const int tiles_per_cta = e->rec_mode == MDK_REC_PINGPONG ? 2
                            : e->rec_mode == MDK_REC_ONE_TILE ? 1
                            : fuse_x || tiles * NDIR > (int64_t)e->sm_count ? 2 : 1;
    const bool fuse_head = tc && !e->keep_act;
    if (!fuse_head && (rc = ensure_h1(ws, H2))) return rc;
    // gi is still read by the previous forward's layer 1: its first writer here waits for it
    if (!fuse_x) MDK_CUDA(cudaStreamWaitEvent(s, ws.l1_done, 0));
    MDK_CUDA(cudaEventRecord(e->ev[1], s));
    if (!fuse_x) {
        MDK_CUDA(launch_inproj0(feats_dev, e->layer[0].w_in_packed, e->layer[0].bias_gi, ws.gi, P,
                                e->desc.num_features, T, tc ? 1 : 0, s));
        launches++;
    }
    MDK_CUDA(cudaEventRecord(e->ev[2], s));
    if (tc) {
        const RecX fx{feats_dev, e->layer[0].w_x_tm, e->layer[0].bias_gi_tc, e->desc.num_features};
        MDK_CUDA(launch_rec_tc(ws.gi, fuse_x ? &fx : nullptr, e->layer[0].w_hh_tm, e->layer[0].b_hn_tc, tiles_per_cta,
                               OUT_TILES, ws.h0, nullptr, B, T, fp16, s));
    } else {
        MDK_CUDA(launch_rec_fp32(ws.gi, e->layer[0].w_hh_t, e->layer[0].b_hn, (float *)ws.h0, B, T, s));
    }
    launches++;
    if (fuse_x) MDK_CUDA(cudaStreamWaitEvent(s, ws.l1_done, 0));
    MDK_CUDA(cudaEventRecord(e->ev[3], s));
    if (tc)
        MDK_CUDA(launch_gemm_tc(ws.h0, e->layer[1].w_in_tc, e->layer[1].bias_gi_tc, ws.gi, tiled_rows(B, T), e->sm_count,
                                fp16, s));
    else MDK_CUDA(launch_gemm_fp32((const float *)ws.h0, e->layer[1].w_in_packed, e->layer[1].bias_gi, ws.gi, P, H2, GI_COLS, s));
    launches++;
    MDK_CUDA(cudaEventRecord(e->ev[4], s));
    // layer 1 after the projection; the lane's features and reference bytes reached s before it (ev_in)
    MDK_CUDA(cudaStreamWaitEvent(s1, e->ev[4], 0));
    if (tc) {
        MDK_CUDA(launch_rec_tc(ws.gi, nullptr, e->layer[1].w_hh_tm, e->layer[1].b_hn_tc, tiles_per_cta,
                               fuse_head ? OUT_LOGITS : OUT_ROWS, fuse_head ? (void *)ws.plog : ws.h1, e->lin_w, B, T, fp16,
                               s1));
    } else {
        MDK_CUDA(launch_rec_fp32(ws.gi, e->layer[1].w_hh_t, e->layer[1].b_hn, ws.h1, B, T, s1));
    }
    launches++;
    MDK_CUDA(cudaEventRecord(e->ev[5], s1));
    MDK_CUDA(cudaEventRecord(ws.l1_done, s1));
    if (fuse_head) MDK_CUDA(launch_head_plog(ws.plog, e->lin_b, B, T, probs_dev, logits_dev, labels_dev, s1, quals_dev, var));
    else MDK_CUDA(launch_head(ws.h1, e->lin_w, e->lin_b, B, T, tc ? 1 : 0, probs_dev, logits_dev, labels_dev, s1, quals_dev,
                              var));
    launches++;
    MDK_CUDA(cudaEventRecord(e->ev[6], s1));
    e->launches += launches;
    e->last.launches = launches;
    ws.last_fused_head = fuse_head;
    ws.last_B = B; ws.last_T = T; ws.last_precision = e->precision;
    e->last_ws = (int)(&ws - e->ws);
    return MDK_OK;
}

// Next lane for a forward of P positions, round robin within its size class; the lane's previous group must have left
// the device before its buffers are reused.
static int acquire_lane(mdk_engine *e, int64_t P, int *out) {
    int idx;
    if (P > mdk_engine::SMALL_POS) {
        idx = e->next_big;
        e->next_big = (e->next_big + 1) % mdk_engine::BIG_LANES;
    } else {
        idx = mdk_engine::BIG_LANES + e->next_small;
        e->next_small = (e->next_small + 1) % mdk_engine::SMALL_LANES;
    }
    mdk_lane &ln = e->lane[idx];
    if (ln.busy) {
        MDK_CUDA(cudaEventSynchronize(ln.ev_out));
        ln.busy = false;
    }
    *out = idx;
    return MDK_OK;
}

// The engine's side of the packing core (packing.h) for one call of B windows of T columns, features at feats (host or
// device memory), and for a variant-decoded call its reference bytes at ref.  Launching alone (flush, sync, waits) needs
// no call.
struct GruCall {
    mdk_engine *e;
    const float *feats = nullptr;
    int64_t B = 0, T = 0;
    const uint8_t *ref = nullptr;

    int open(int64_t windows) {
        // size class of the CALL: the tail piece of a split call stays with the big lanes
        const int rc = acquire_lane(e, B * T, &e->open_lane);
        // the staging grows to this call (at most one group of it); a reserved lane is already larger and keeps
        // collecting further calls up to its size
        return rc ? rc : ensure_io(e, e->lane[e->open_lane], windows, T);
    }
    int64_t capacity(int64_t len) {
        const mdk_lane &ln = e->lane[e->open_lane];
        return std::min(ln.cap_io / len, ln.cap_feats / (len * e->desc.num_features));
    }
    // copy-in stream: features into the staging (asynchronous for device and page-locked host memory), behind the
    // group's earlier pieces
    int stage(int64_t first, int64_t n, int64_t at) {
        const size_t w = (size_t)T * e->desc.num_features;
        mdk_lane &ln = e->lane[e->open_lane];
        MDK_CUDA(cudaMemcpyAsync(ln.d_feats + at * w, feats + first * w, n * w * sizeof(float), cudaMemcpyDefault,
                                 e->copy_in));
        if (ref) {
            int rc;
            if ((rc = ensure_var(ln))) return rc;
            MDK_CUDA(cudaMemcpyAsync(ln.d_ref + at * T, ref + first * T, n * T, cudaMemcpyDefault, e->copy_in));
        }
        return MDK_OK;
    }
    // the sealed group on its lane: one forward over all of its windows, then the results back to each call's buffers
    int launch() {
        mdk_lane &ln = e->lane[e->open_lane];
        const Packing &pk = e->pk;
        bool logits = false, labels = false, quals = false, var = false;      // whether any call wants them
        for (const Packing::Piece &p : pk.pieces) {
            logits = logits || p.logits; labels = labels || (p.labels && !p.ref); quals = quals || p.quals;
            var = var || p.ref;
        }
        const HeadVariant hv{ln.d_ref, ln.d_calls, ln.d_pred_q, ln.d_ref_q};
        int rc;
        if (quals && (rc = ensure_quals(ln))) return rc;
        // a group the workspace cannot take (the budget at gru_size 256) is refused before it claims a slot of the
        // event ring: the timings then cover the groups that ran, and the next forward records into the same slots
        if ((rc = prepare_weights(e)) || (rc = ensure_workspace(e, *ln.ws, pk.windows, pk.len))) return rc;
        cudaStream_t s = ln.ws->stream;
        e->ev = e->evr[e->fwd_count % mdk_engine::EV_RING];
        e->fwd_count++;
        MDK_CUDA(cudaEventRecord(e->ev[0], s));
        MDK_CUDA(cudaEventRecord(ln.ev_in, e->copy_in));      // every feature copy of the group was queued on copy_in
        MDK_CUDA(cudaStreamWaitEvent(s, ln.ev_in, 0));
        if ((rc = run_forward(e, *ln.ws, ln.d_feats, pk.windows, pk.len, ln.d_probs, logits ? ln.d_logits : nullptr,
                              labels ? ln.d_labels : nullptr, quals ? ln.d_quals : nullptr, var ? &hv : nullptr)))
            return rc;
        // the outputs are written by the head, on the layer-1 stream
        MDK_CUDA(cudaEventRecord(e->ev[7], ln.ws->l1_stream));
        if ((rc = copy_back(e->copy_out, pk, ln.ws->l1_stream, ln.d_probs, ln.d_logits, ln.d_labels, ln.d_quals, &hv)))
            return rc;
        MDK_CUDA(cudaEventRecord(ln.ev_out, e->copy_out.stream));
        ln.busy = true;
        return MDK_OK;
    }
};

static int launch_group(mdk_engine *e) { return e->pk.launch(GruCall{e}); }

// Most windows one group collects: one wave unless mdk_engine_set_group_windows says otherwise.
static int64_t group_limit(mdk_engine *e) {
    return e->group_windows > 0 ? e->group_windows : mdk_engine_preferred_windows(e);
}

static float ev_ms(cudaEvent_t a, cudaEvent_t b) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, a, b) != cudaSuccess) { cudaGetLastError(); return -1.f; }
    return ms;
}

static int check_shapes(const mdk_engine *e, const void *feats, int64_t B, int64_t T, const void *probs) {
    MDK_REQUIRE(e != nullptr, MDK_ERR_ARG, "engine is NULL");
    MDK_REQUIRE(feats != nullptr && probs != nullptr, MDK_ERR_ARG, "forward: feats/probs must not be NULL");
    MDK_REQUIRE(B >= 1 && T >= 1, MDK_ERR_ARG, "forward: need B >= 1 and T >= 1");
    MDK_REQUIRE(B * T < (int64_t)1 << 40, MDK_ERR_ARG, "forward: B*T too large");
    return MDK_OK;
}

}  // namespace mdk

using namespace mdk;

extern "C" {

const char *mdk_plp_bases(void) { return "acgtACGTdD"; }
size_t mdk_featlen(void) { return 10; }
size_t mdk_fwd_del(void) { return 9; }
size_t mdk_rev_del(void) { return 8; }
const char *mdk_last_error(void) { return g_last_error.c_str(); }
const char *mdk_version(void) { return "medaka_b200 0.1.0 (sm_90a)"; }

int mdk_device_count(int *count) {
    MDK_REQUIRE(count, MDK_ERR_ARG, "count is NULL");
    cudaError_t err = cudaGetDeviceCount(count);
    if (err != cudaSuccess) { *count = 0; return cuda_fail(err, "cudaGetDeviceCount", __FILE__, __LINE__); }
    return MDK_OK;
}

int mdk_device_info(int device, int *sm_arch, int *sm_count, size_t *total_mem) {
    cudaDeviceProp prop;
    MDK_CUDA(cudaGetDeviceProperties(&prop, device));
    if (sm_arch) *sm_arch = prop.major * 10 + prop.minor;
    if (sm_count) *sm_count = prop.multiProcessorCount;
    if (total_mem) *total_mem = prop.totalGlobalMem;
    return MDK_OK;
}

int mdk_host_alloc(size_t bytes, void **out) {
    MDK_REQUIRE(out, MDK_ERR_ARG, "out is NULL");
    MDK_CUDA(cudaHostAlloc(out, bytes ? bytes : 1, cudaHostAllocPortable));
    return MDK_OK;
}
int mdk_host_free(void *p) {
    if (p) MDK_CUDA(cudaFreeHost(p));
    return MDK_OK;
}
int mdk_dev_alloc(int device, size_t bytes, void **out) {
    MDK_REQUIRE(out, MDK_ERR_ARG, "out is NULL");
    MDK_CUDA(cudaSetDevice(device));
    MDK_CUDA(cudaMalloc(out, bytes ? bytes : 1));
    return MDK_OK;
}
int mdk_dev_free(int device, void *p) {
    MDK_CUDA(cudaSetDevice(device));
    if (p) MDK_CUDA(cudaFree(p));
    return MDK_OK;
}
int mdk_memcpy_h2d(int device, void *dst_dev, const void *src_host, size_t bytes) {
    MDK_CUDA(cudaSetDevice(device));
    MDK_CUDA(cudaMemcpy(dst_dev, src_host, bytes, cudaMemcpyHostToDevice));
    return MDK_OK;
}
int mdk_memcpy_d2h(int device, void *dst_host, const void *src_dev, size_t bytes) {
    MDK_CUDA(cudaSetDevice(device));
    MDK_CUDA(cudaMemcpy(dst_host, src_dev, bytes, cudaMemcpyDeviceToHost));
    return MDK_OK;
}
int mdk_dev_memset(int device, void *dst_dev, int value, size_t bytes) {
    MDK_CUDA(cudaSetDevice(device));
    MDK_CUDA(cudaMemset(dst_dev, value, bytes));
    return MDK_OK;
}
int mdk_device_synchronize(int device) {
    MDK_CUDA(cudaSetDevice(device));
    MDK_CUDA(cudaDeviceSynchronize());
    return MDK_OK;
}

int mdk_engine_create(int device, const mdk_model_desc *desc, mdk_engine **out) {
    MDK_REQUIRE(desc && out, MDK_ERR_ARG, "engine_create: NULL argument");
    MDK_REQUIRE(desc->gru_size == H || desc->gru_size == H256, MDK_ERR_UNSUPPORTED,
                "engine_create: gru_size must be 128 or 256");
    MDK_REQUIRE(desc->n_layers == 2 && desc->bidirectional == 1, MDK_ERR_UNSUPPORTED,
                "engine_create: only the 2-layer bidirectional GRU is supported");
    MDK_REQUIRE(desc->num_features >= 1 && desc->num_features <= 1024, MDK_ERR_ARG, "engine_create: bad num_features");
    int ndev = 0;
    MDK_CUDA(cudaGetDeviceCount(&ndev));
    MDK_REQUIRE(device >= 0 && device < ndev, MDK_ERR_ARG, "engine_create: no such CUDA device");
    cudaDeviceProp prop;
    MDK_CUDA(cudaGetDeviceProperties(&prop, device));
    MDK_REQUIRE(prop.major == 9 && prop.minor == 0, MDK_ERR_UNSUPPORTED,
                "engine_create: this library is built for sm_90a (Hopper H100) only");
    MDK_CUDA(cudaSetDevice(device));
    mdk_engine *e = new (std::nothrow) mdk_engine();
    MDK_REQUIRE(e, MDK_ERR_NOMEM, "engine_create: out of host memory");
    e->device = device;
    e->desc = *desc;
    e->sm_count = prop.multiProcessorCount;
    if (desc->gru_size == H256) {     // one wave of the cluster recurrence: one 4-CTA cluster per (tile, direction)
        int clusters = 0;
        cudaError_t err = rec256_max_clusters(&clusters);
        if (err != cudaSuccess) { delete e; return cuda_fail(err, "rec256_max_clusters", __FILE__, __LINE__); }
        if (clusters < 1) {
            delete e;
            set_error("engine_create: gru_size 256 needs a cluster of 4 CTAs with 150 KiB of shared memory each; none "
                      "fits this device");
            return MDK_ERR_UNSUPPORTED;
        }
        e->wave256 = (int64_t)WT * std::max(1, clusters / NDIR);
    }
    for (auto &ws : e->ws) {
        cudaError_t err = cudaStreamCreateWithFlags(&ws.stream, cudaStreamNonBlocking);
        if (err == cudaSuccess) err = cudaStreamCreateWithFlags(&ws.l1_stream, cudaStreamNonBlocking);
        if (err == cudaSuccess) err = cudaEventCreateWithFlags(&ws.l1_done, cudaEventDisableTiming);
        if (err != cudaSuccess) { mdk_engine_destroy(e); return cuda_fail(err, "cudaStreamCreate", __FILE__, __LINE__); }
    }
    for (int i = 0; i < mdk_engine::N_LANES; ++i) {
        mdk_lane &ln = e->lane[i];
        ln.ws = i < mdk_engine::BIG_LANES ? &e->ws[i % mdk_engine::BIG_WS]
                                          : &e->ws[mdk_engine::BIG_WS + (i - mdk_engine::BIG_LANES)];
        cudaEventCreateWithFlags(&ln.ev_in, cudaEventDisableTiming);
        cudaEventCreateWithFlags(&ln.ev_out, cudaEventDisableTiming);
    }
    e->stream = e->ws[0].stream;
    for (auto &set : e->evr) for (auto &ev : set) cudaEventCreate(&ev);
    cudaStreamCreateWithFlags(&e->copy_in, cudaStreamNonBlocking);
    for (auto &ev : e->ev_timer) cudaEventCreate(&ev);
    cudaEventCreateWithFlags(&e->ev_join, cudaEventDisableTiming);
    cudaError_t err = create_copy_out(e->copy_out);
    if (err != cudaSuccess) { mdk_engine_destroy(e); return cuda_fail(err, "create_copy_out", __FILE__, __LINE__); }
    *out = e;
    return MDK_OK;
}

int mdk_engine_destroy(mdk_engine *e) {
    if (!e) return MDK_OK;
    cudaSetDevice(e->device);
    for (auto &ws : e->ws) {
        if (ws.stream) cudaStreamSynchronize(ws.stream);
        if (ws.l1_stream) cudaStreamSynchronize(ws.l1_stream);
    }
    destroy_copy_out(e->copy_out);
    for (auto &ws : e->ws) {
        dev_free(ws.gi); dev_free(ws.h1); dev_free(ws.plog);
        if (ws.h0) cudaFree(ws.h0);
        if (ws.stream) cudaStreamDestroy(ws.stream);
        if (ws.l1_stream) cudaStreamDestroy(ws.l1_stream);
        if (ws.l1_done) cudaEventDestroy(ws.l1_done);
    }
    for (auto &ln : e->lane) {
        dev_free(ln.d_feats); dev_free(ln.d_probs); dev_free(ln.d_logits); dev_free(ln.d_labels); dev_free(ln.d_quals);
        dev_free(ln.d_ref); dev_free(ln.d_calls); dev_free(ln.d_pred_q); dev_free(ln.d_ref_q);
        if (ln.ev_in) cudaEventDestroy(ln.ev_in);
        if (ln.ev_out) cudaEventDestroy(ln.ev_out);
    }
    if (e->copy_in) cudaStreamDestroy(e->copy_in);
    for (auto &set : e->evr) for (auto &ev : set) if (ev) cudaEventDestroy(ev);
    for (auto &ev : e->ev_timer) if (ev) cudaEventDestroy(ev);
    if (e->ev_join) cudaEventDestroy(e->ev_join);
    delete e;     // and with it the weights (DeviceWeights)
    cudaGetLastError();
    return MDK_OK;
}

// weights are read by every lane: quiesce all of them, so that the calls made before a load run with the weights they
// were made with and no forward is in flight when prepare_weights rewrites the device copies
static int quiesce(mdk_engine *e) {
    int rc = launch_group(e);
    if (rc) return rc;
    for (auto &ws : e->ws) MDK_CUDA(ws_sync(ws));
    return MDK_OK;
}

int mdk_engine_load_gru(mdk_engine *e, int layer, int direction, const float *w_ih, const float *w_hh,
                        const float *b_ih, const float *b_hh) {
    MDK_REQUIRE(e, MDK_ERR_ARG, "engine is NULL");
    MDK_REQUIRE(layer >= 0 && layer < 2 && direction >= 0 && direction < 2, MDK_ERR_ARG, "load_gru: bad layer/direction");
    MDK_REQUIRE(w_ih && w_hh && b_ih && b_hh, MDK_ERR_ARG, "load_gru: NULL weight pointer");
    MDK_CUDA(cudaSetDevice(e->device));
    { int rcq = quiesce(e); if (rcq) return rcq; }
    LayerWeights &lw = e->layer[layer];
    const int g3 = 3 * e->desc.gru_size;
    lw.w_ih[direction].assign(w_ih, w_ih + (size_t)g3 * in_features(e, layer));
    lw.w_hh[direction].assign(w_hh, w_hh + (size_t)g3 * e->desc.gru_size);
    lw.b_ih[direction].assign(b_ih, b_ih + g3);
    lw.b_hh[direction].assign(b_hh, b_hh + g3);
    e->prepared = false;
    return MDK_OK;
}

int mdk_engine_load_linear(mdk_engine *e, const float *w, const float *b) {
    MDK_REQUIRE(e && w && b, MDK_ERR_ARG, "load_linear: NULL argument");
    MDK_CUDA(cudaSetDevice(e->device));
    { int rcq = quiesce(e); if (rcq) return rcq; }
    e->lin_w_host.assign(w, w + NCLS * 2 * e->desc.gru_size);
    e->lin_b_host.assign(b, b + NCLS);
    e->prepared = false;
    return MDK_OK;
}

int mdk_engine_set_precision(mdk_engine *e, int mode) {
    MDK_REQUIRE(e, MDK_ERR_ARG, "engine is NULL");
    MDK_REQUIRE(mode == MDK_PREC_TC || mode == MDK_PREC_FP32 || mode == MDK_PREC_FP16, MDK_ERR_ARG,
                "set_precision: unknown mode");
    if (mode != e->precision) {
        // the open group's windows were submitted in the old mode: they run in it
        MDK_CUDA(cudaSetDevice(e->device));
        const int rc = launch_group(e);
        if (rc) return rc;
    }
    e->precision = mode;
    return MDK_OK;
}
int mdk_engine_get_precision(mdk_engine *e, int *mode) {
    MDK_REQUIRE(e && mode, MDK_ERR_ARG, "NULL argument");
    *mode = e->precision;
    return MDK_OK;
}

int mdk_engine_set_rec_mode(mdk_engine *e, int mode) {
    MDK_REQUIRE(e, MDK_ERR_ARG, "engine is NULL");
    MDK_REQUIRE(mode == MDK_REC_AUTO || mode == MDK_REC_ONE_TILE || mode == MDK_REC_PINGPONG, MDK_ERR_ARG,
                "set_rec_mode: unknown mode");
    MDK_REQUIRE(mode == MDK_REC_AUTO || e->desc.gru_size == H, MDK_ERR_UNSUPPORTED,
                "set_rec_mode: at gru_size 256 the recurrence has one kernel; only MDK_REC_AUTO applies");
    e->rec_mode = mode;
    return MDK_OK;
}

int mdk_engine_set_group_windows(mdk_engine *e, int64_t windows) {
    MDK_REQUIRE(e && windows >= 0, MDK_ERR_ARG, "set_group_windows: bad arguments");
    e->group_windows = windows;
    return MDK_OK;
}

// Reserve = size the big workspaces and the big lanes' staging for groups of up to B windows of T columns.  This is also
// what switches coalescing on: a group collects calls only as far as its lane's staging buffers reach.
int mdk_engine_reserve(mdk_engine *e, int64_t B, int64_t T) {
    MDK_REQUIRE(e && B >= 1 && T >= 1, MDK_ERR_ARG, "reserve: bad arguments");
    MDK_CUDA(cudaSetDevice(e->device));
    int rc;
    if ((rc = launch_group(e))) return rc;
    if (e->desc.gru_size == H256) B = std::min(B, group_limit(e));   // no group at 256 holds more (forward_dev cuts too)
    const bool big = B * T > mdk_engine::SMALL_POS;
    const int l0 = big ? 0 : mdk_engine::BIG_LANES, l1 = big ? mdk_engine::BIG_LANES : mdk_engine::N_LANES;
    for (int i = l0; i < l1; ++i) {
        mdk_lane &ln = e->lane[i];
        if (ln.busy) { MDK_CUDA(cudaEventSynchronize(ln.ev_out)); ln.busy = false; }
        if ((rc = ensure_workspace(e, *ln.ws, B, T))) return rc;
        if ((rc = ensure_io(e, ln, B, T))) return rc;
    }
    return MDK_OK;
}

int mdk_engine_forward_dev(mdk_engine *e, const float *feats_dev, int64_t B, int64_t T, float *probs_dev,
                           float *logits_dev, uint8_t *labels_dev) {
    int rc;
    if ((rc = check_shapes(e, feats_dev, B, T, probs_dev))) return rc;
    MDK_CUDA(cudaSetDevice(e->device));
    int64_t gmax = group_limit(e);
    // A call of more than one group's windows was sized by its caller (one full wave of the two-tile kernel is 2112
    // windows on an H100): it runs as one forward of its own instead of being cut into groups that each fill part of
    // the device.  At gru_size 256 a group is already a full wave and the workspace is bounded: the call is cut.
    if (B > gmax && e->desc.gru_size == H) {
        if ((rc = launch_group(e))) return rc;
        gmax = B;
    }
    return e->pk.enqueue(GruCall{e, feats_dev, B, T}, B, T, probs_dev, logits_dev, labels_dev, gmax, nullptr);
}

int mdk_engine_submit(mdk_engine *e, const float *feats_host, int64_t B, int64_t T, float *probs_host,
                      float *logits_host, uint8_t *labels_host, int64_t *ticket) {
    int rc;
    if ((rc = check_shapes(e, feats_host, B, T, probs_host))) return rc;
    MDK_REQUIRE(ticket, MDK_ERR_ARG, "submit: ticket is NULL");
    MDK_CUDA(cudaSetDevice(e->device));
    return e->pk.enqueue(GruCall{e, feats_host, B, T}, B, T, probs_host, logits_host, labels_host, group_limit(e), ticket);
}

int mdk_engine_submit_decoded(mdk_engine *e, const float *feats, int64_t B, int64_t T, uint8_t *labels_out,
                              uint8_t *quals_out, int64_t *ticket) {
    MDK_REQUIRE(e != nullptr, MDK_ERR_ARG, "engine is NULL");
    MDK_REQUIRE(feats != nullptr && labels_out != nullptr, MDK_ERR_ARG, "submit_decoded: feats/labels must not be NULL");
    MDK_REQUIRE(B >= 1 && T >= 1, MDK_ERR_ARG, "submit_decoded: need B >= 1 and T >= 1");
    MDK_REQUIRE(B * T < (int64_t)1 << 40, MDK_ERR_ARG, "submit_decoded: B*T too large");
    MDK_REQUIRE(ticket, MDK_ERR_ARG, "submit_decoded: ticket is NULL");
    MDK_CUDA(cudaSetDevice(e->device));
    return e->pk.enqueue(GruCall{e, feats, B, T}, B, T, nullptr, nullptr, labels_out, group_limit(e), ticket, quals_out);
}

int mdk_engine_submit_variant_decoded(mdk_engine *e, const float *feats, int64_t B, int64_t T, const uint8_t *ref_bytes,
                                      uint8_t *calls_out, float *pred_q_out, float *ref_q_out, int64_t *ticket) {
    MDK_REQUIRE(e != nullptr, MDK_ERR_ARG, "engine is NULL");
    MDK_REQUIRE(feats && ref_bytes && calls_out && pred_q_out && ref_q_out, MDK_ERR_ARG,
                "submit_variant_decoded: NULL input or output");
    MDK_REQUIRE(B >= 1 && T >= 1, MDK_ERR_ARG, "submit_variant_decoded: need B >= 1 and T >= 1");
    MDK_REQUIRE(B * T < (int64_t)1 << 40, MDK_ERR_ARG, "submit_variant_decoded: B*T too large");
    MDK_REQUIRE(ticket, MDK_ERR_ARG, "submit_variant_decoded: ticket is NULL");
    MDK_CUDA(cudaSetDevice(e->device));
    GruCall call{e, feats, B, T, ref_bytes};
    return e->pk.enqueue(call, B, T, nullptr, nullptr, calls_out, group_limit(e), ticket, nullptr, ref_bytes,
                         pred_q_out, ref_q_out);
}

int mdk_engine_flush(mdk_engine *e) {
    MDK_REQUIRE(e, MDK_ERR_ARG, "engine is NULL");
    MDK_CUDA(cudaSetDevice(e->device));
    return launch_group(e);
}

int mdk_engine_wait(mdk_engine *e, int64_t ticket) {
    MDK_REQUIRE(e, MDK_ERR_ARG, "engine is NULL");
    MDK_REQUIRE(ticket >= 0 && ticket < e->pk.tickets, MDK_ERR_ARG, "wait: unknown ticket");
    MDK_CUDA(cudaSetDevice(e->device));
    return wait_ticket(e->copy_out, e->pk, GruCall{e}, ticket);
}

int mdk_engine_forward(mdk_engine *e, const float *feats_host, int64_t B, int64_t T, float *probs_host,
                       float *logits_host, uint8_t *labels_host) {
    int64_t ticket = -1;
    int rc = mdk_engine_submit(e, feats_host, B, T, probs_host, logits_host, labels_host, &ticket);
    if (rc) return rc;
    return mdk_engine_wait(e, ticket);
}

int mdk_engine_sync(mdk_engine *e) {
    MDK_REQUIRE(e, MDK_ERR_ARG, "engine is NULL");
    MDK_CUDA(cudaSetDevice(e->device));
    int rc = launch_group(e);
    if (rc) return rc;
    MDK_CUDA(cudaStreamSynchronize(e->copy_in));
    for (auto &ws : e->ws) MDK_CUDA(ws_sync(ws));
    MDK_CUDA(cudaStreamSynchronize(e->copy_out.stream));
    for (auto &ln : e->lane) ln.busy = false;
    return MDK_OK;
}

static void stage_times(cudaEvent_t *ev, mdk_timings *t) {
    t->h2d_ms = ev_ms(ev[0], ev[1]);
    t->inproj0_ms = ev_ms(ev[1], ev[2]);
    t->rec0_ms = ev_ms(ev[2], ev[3]);
    t->inproj1_ms = ev_ms(ev[3], ev[4]);
    t->rec1_ms = ev_ms(ev[4], ev[5]);
    t->head_ms = ev_ms(ev[5], ev[6]);
    t->d2h_ms = ev_ms(ev[6], ev[7]);
    t->total_ms = ev_ms(ev[0], ev[7]);
}

int mdk_engine_last_timings(mdk_engine *e, mdk_timings *out) { return mdk_engine_mean_timings(e, 1, out); }

// Calls are packed into groups, so there may be fewer groups than calls: the mean is over the last
// min(n_last, groups launched) groups.  The open group is launched first so that its events are not read stale.
int mdk_engine_mean_timings(mdk_engine *e, int n_last, mdk_timings *out) {
    MDK_REQUIRE(e && out, MDK_ERR_ARG, "NULL argument");
    MDK_REQUIRE(n_last >= 1 && n_last <= mdk_engine::EV_RING, MDK_ERR_ARG, "mean_timings: n_last out of range");
    MDK_CUDA(cudaSetDevice(e->device));
    int rc = launch_group(e);
    if (rc) return rc;
    MDK_REQUIRE(e->fwd_count >= 1, MDK_ERR_STATE, "mean_timings: no forward recorded");
    n_last = (int)std::min<int64_t>(n_last, e->fwd_count);
    for (auto &ws : e->ws) MDK_CUDA(ws_sync(ws));
    mdk_timings acc{};
    for (int i = 0; i < n_last; ++i) {
        mdk_timings t{};
        stage_times(e->evr[(e->fwd_count - 1 - i) % mdk_engine::EV_RING], &t);
        acc.h2d_ms += t.h2d_ms; acc.inproj0_ms += t.inproj0_ms; acc.rec0_ms += t.rec0_ms;
        acc.inproj1_ms += t.inproj1_ms; acc.rec1_ms += t.rec1_ms; acc.head_ms += t.head_ms;
        acc.d2h_ms += t.d2h_ms; acc.total_ms += t.total_ms;
    }
    const float inv = 1.0f / (float)n_last;
    acc.h2d_ms *= inv; acc.inproj0_ms *= inv; acc.rec0_ms *= inv; acc.inproj1_ms *= inv; acc.rec1_ms *= inv;
    acc.head_ms *= inv; acc.d2h_ms *= inv; acc.total_ms *= inv;
    acc.launches = e->last.launches;
    *out = acc;
    return MDK_OK;
}

// Diagnostics: completion times (ms after the timer's start event) of the eight stage events of the last n launched
// groups, oldest first - the schedule the lanes actually ran.  The open group is launched first, as in mean_timings.
int mdk_debug_timeline(mdk_engine *e, int n_last, float *out) {
    MDK_REQUIRE(e && out, MDK_ERR_ARG, "NULL argument");
    MDK_CUDA(cudaSetDevice(e->device));
    int rc = launch_group(e);
    if (rc) return rc;
    MDK_REQUIRE(n_last >= 1 && n_last <= mdk_engine::EV_RING && e->fwd_count >= n_last, MDK_ERR_ARG, "timeline: bad n_last");
    for (auto &ws : e->ws) MDK_CUDA(ws_sync(ws));
    for (int i = 0; i < n_last; ++i) {
        cudaEvent_t *ev = e->evr[(e->fwd_count - n_last + i) % mdk_engine::EV_RING];
        for (int k = 0; k < 8; ++k) MDK_CUDA(cudaEventElapsedTime(out + i * 8 + k, e->ev_timer[0], ev[k]));
    }
    return MDK_OK;
}

// The timed region spans every lane: the start event goes on lane 0 after all lanes have drained, the stop event on
// lane 0 after it has been made to wait for every other stream of every workspace and for the copy-out stream.
int mdk_engine_timer_start(mdk_engine *e) {
    MDK_REQUIRE(e, MDK_ERR_ARG, "engine is NULL");
    MDK_CUDA(cudaSetDevice(e->device));
    int rc = mdk_engine_sync(e);
    if (rc) return rc;
    MDK_CUDA(cudaEventRecord(e->ev_timer[0], e->stream));
    // work queued on the other lanes / copy streams after this point must not start before the start event
    for (int i = 0; i < mdk_engine::N_WS; ++i) {
        if (i) MDK_CUDA(cudaStreamWaitEvent(e->ws[i].stream, e->ev_timer[0], 0));
        MDK_CUDA(cudaStreamWaitEvent(e->ws[i].l1_stream, e->ev_timer[0], 0));
    }
    MDK_CUDA(cudaStreamWaitEvent(e->copy_in, e->ev_timer[0], 0));
    return MDK_OK;
}
int mdk_engine_timer_stop(mdk_engine *e, float *elapsed_ms) {
    MDK_REQUIRE(e && elapsed_ms, MDK_ERR_ARG, "NULL argument");
    MDK_CUDA(cudaSetDevice(e->device));
    int rc = launch_group(e);
    if (rc) return rc;
    // every layer-1 stream, ws[0]'s included: the last group's layer 1 and head run there after ws[0].stream is done
    for (int i = 0; i < mdk_engine::N_WS; ++i) {
        if (i) {
            MDK_CUDA(cudaEventRecord(e->ev_join, e->ws[i].stream));
            MDK_CUDA(cudaStreamWaitEvent(e->stream, e->ev_join, 0));
        }
        MDK_CUDA(cudaEventRecord(e->ev_join, e->ws[i].l1_stream));
        MDK_CUDA(cudaStreamWaitEvent(e->stream, e->ev_join, 0));
    }
    MDK_CUDA(cudaEventRecord(e->ev_join, e->copy_out.stream));     // the end event must follow every copy-out still in flight
    MDK_CUDA(cudaStreamWaitEvent(e->stream, e->ev_join, 0));
    MDK_CUDA(cudaEventRecord(e->ev_timer[1], e->stream));
    MDK_CUDA(cudaEventSynchronize(e->ev_timer[1]));
    MDK_CUDA(cudaEventElapsedTime(elapsed_ms, e->ev_timer[0], e->ev_timer[1]));
    return MDK_OK;
}

int mdk_engine_read_activation(mdk_engine *e, int which, float *out_host, int64_t n_floats) {
    MDK_REQUIRE(e, MDK_ERR_ARG, "engine is NULL");
    return mdk_engine_read_activation_windows(e, which, 0, e->ws[e->last_ws].last_B, out_host, n_floats);
}

int mdk_engine_read_activation_windows(mdk_engine *e, int which, int64_t first, int64_t count, float *out_host,
                                       int64_t n_floats) {
    MDK_REQUIRE(e && out_host, MDK_ERR_ARG, "NULL argument");
    MDK_REQUIRE(which == 0 || which == 1, MDK_ERR_ARG, "read_activation: which must be 0 or 1");
    mdk_ws &ln = e->ws[e->last_ws];
    MDK_REQUIRE(ln.last_B > 0 && ln.last_T > 0, MDK_ERR_STATE, "read_activation: no forward recorded");
    MDK_REQUIRE(first >= 0 && count > 0 && first + count <= ln.last_B, MDK_ERR_ARG,
                "read_activation: windows first .. first + count - 1 must lie in the last forward's B windows");
    const int width = 2 * e->desc.gru_size;
    MDK_REQUIRE(n_floats == count * ln.last_T * width, MDK_ERR_ARG, "read_activation: size must be count*T*2*gru_size");
    MDK_REQUIRE(!(which == 1 && ln.last_fused_head), MDK_ERR_STATE,
                "read_activation(1): the last forward fused the head into layer 1 (h1 never reached HBM); call "
                "mdk_engine_keep_activations(e, 1) before the forward");
    MDK_CUDA(cudaSetDevice(e->device));
    MDK_CUDA(ws_sync(ln));
    if (ln.last_precision == MDK_PREC_FP32) {
        const float *src = (which == 1 ? ln.h1 : reinterpret_cast<const float *>(ln.h0)) + first * ln.last_T * width;
        MDK_CUDA(cudaMemcpy(out_host, src, (size_t)n_floats * sizeof(float), cudaMemcpyDeviceToHost));
    } else {
        // tensor-core path: rows are tile-interleaved (and at gru_size 128 layer 0 is stored as fp16 hi/lo operand tiles)
        float *tmp = nullptr;
        MDK_CUDA(cudaMalloc(&tmp, (size_t)n_floats * sizeof(float)));
        const float *rows = which == 1 ? ln.h1 : static_cast<const float *>(ln.h0);
        cudaError_t err = which == 0 && width == H2 ? launch_unpack_h0(ln.h0, tmp, first, count, ln.last_T, ln.stream)
                                                    : launch_untile_rows(rows, tmp, first, count, ln.last_T, ln.stream, width);
        if (err == cudaSuccess) err = cudaStreamSynchronize(ln.stream);
        if (err == cudaSuccess) err = cudaMemcpy(out_host, tmp, (size_t)n_floats * sizeof(float), cudaMemcpyDeviceToHost);
        cudaFree(tmp);
        e->launches++;
        if (err != cudaSuccess) return cuda_fail(err, "read_activation", __FILE__, __LINE__);
    }
    return MDK_OK;
}


int mdk_debug_read_plog(mdk_engine *e, float *out_host, int64_t n_floats) {
    MDK_REQUIRE(e && out_host, MDK_ERR_ARG, "NULL argument");
    mdk_ws &ln = e->ws[e->last_ws];
    MDK_REQUIRE(ln.last_fused_head, MDK_ERR_STATE, "read_plog: the last forward did not run the fused head");
    const int64_t tiles = (ln.last_B + WT - 1) / WT;
    MDK_REQUIRE(n_floats == NDIR * tiles * ln.last_T * PLOG_TS_FLOATS, MDK_ERR_ARG, "read_plog: size must be 2*tiles*T*80");
    MDK_CUDA(cudaSetDevice(e->device));
    MDK_CUDA(ws_sync(ln));
    MDK_CUDA(cudaMemcpy(out_host, ln.plog, (size_t)n_floats * sizeof(float), cudaMemcpyDeviceToHost));
    return MDK_OK;
}

int64_t mdk_engine_launch_count(mdk_engine *e) { return e ? e->launches : 0; }

int mdk_engine_keep_activations(mdk_engine *e, int keep) {
    MDK_REQUIRE(e, MDK_ERR_ARG, "NULL engine");
    e->keep_act = keep != 0;
    return MDK_OK;
}

int64_t mdk_engine_preferred_windows(mdk_engine *e) {
    if (e && e->desc.gru_size == H256) return e->wave256;
    const int sms = e ? e->sm_count : 132;
    return (int64_t)mdk::WT * (sms / mdk::NDIR);
}

int mdk_selftest_umma(int device, const float *A, const float *B, float *D, int N, int K, int variant) {
    MDK_REQUIRE(A && B && D, MDK_ERR_ARG, "selftest_umma: NULL pointer");
    return selftest_umma(device, A, B, D, N, K, variant);
}


}  // extern "C"
