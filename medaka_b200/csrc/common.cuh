// Shared declarations of libmedaka_b200: engine state, error plumbing, kernel launchers.
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>

#include <cstdint>
#include <cstdio>
#include <string>
#include <vector>

#include "../../include/medaka_b200.h"
#include "packing.h"

namespace mdk {

constexpr int H = 128;        // gru_size of every shipped counts-matrix model (gru.py:18)
constexpr int G3 = 3 * H;     // gate rows per direction (r,z,n)
constexpr int NDIR = 2;
constexpr int GI_COLS = NDIR * G3;  // 768: input-projection row [fwd r z n | rev r z n]
constexpr int H2 = NDIR * H;        // 256: layer output width
constexpr int NCLS = 5;             // gru.py:53-55
// gru_size 256, the width `medaka train` builds by default (gru256.cu)
constexpr int H256 = 256;
constexpr int G3_256 = 3 * H256;
constexpr int GI256_COLS = NDIR * G3_256;   // 1536
constexpr int H2_256 = NDIR * H256;         // 512

void set_error(const std::string &msg);
int cuda_fail(cudaError_t err, const char *what, const char *file, int line);

// Device memory of the featuriser and decode entry points, cached per host thread and grown on demand: the loader
// threads call them concurrently, per region and per contig, and a cudaMalloc / cudaFree pair per call costs more than
// their kernels.  One blob per role that can be live on a thread at once: STAGING holds a call's copies of the host
// arrays and its results, SCRATCH the kernels' intermediates under it (the column plan, or the stitch scratch under
// mdk_stitch_consensus's staging).
enum class Blob { STAGING, SCRATCH };
cudaError_t cached_blob(Blob role, size_t bytes, uint8_t **out);

// One call's arrays in a cached blob.  in() and take() name them (with and without host data to copy in); alloc() lays
// them out in that order, 256-byte aligned, points the named pointers at them and queues the copies of the host data on
// the legacy stream, ahead of the call's kernels (from page-locked memory the transfer overlaps the staging of the next
// array); out() copies results back synchronously, after everything queued before it.  The first CUDA error ends the
// chain, and result() reports it under the entry point's name.
class Staging {
  public:
    Staging(Blob role, const char *what) : role_(role), what_(what) {}
    template <class T> void take(T **dev, size_t n) { add(dev, &point<T>, nullptr, n * sizeof(T)); }
    template <class T> void in(const T **dev, const T *host, size_t n) { add(dev, &point<const T>, host, n * sizeof(T)); }
    bool alloc() {
        uint8_t *base = nullptr;
        check(cached_blob(role_, size_, &base));
        for (const Array &a : arrays_) {
            if (!ok()) break;
            a.point(a.dev, base + a.off);
            if (a.host && a.bytes) check(cudaMemcpyAsync(base + a.off, a.host, a.bytes, cudaMemcpyHostToDevice, 0));
        }
        return ok();
    }
    template <class T> void out(T *host, const T *dev, size_t n) {
        if (n) check(cudaMemcpy(host, dev, n * sizeof(T), cudaMemcpyDeviceToHost));
    }
    void check(cudaError_t err) { if (ok()) err_ = err; }
    bool ok() const { return err_ == cudaSuccess; }
    int result(int rc = MDK_OK) const { return ok() ? rc : cuda_fail(err_, what_, __FILE__, __LINE__); }

  private:
    struct Array {
        void *dev;
        void (*point)(void *dev, uint8_t *at);
        const void *host;
        size_t off, bytes;
    };
    template <class T> static void point(void *dev, uint8_t *at) { *static_cast<T **>(dev) = reinterpret_cast<T *>(at); }
    void add(void *dev, void (*pt)(void *, uint8_t *), const void *host, size_t bytes) {
        arrays_.push_back(Array{dev, pt, host, size_, bytes});
        size_ += (bytes + 255) / 256 * 256;
    }
    Blob role_;
    const char *what_;
    cudaError_t err_ = cudaSuccess;
    size_t size_ = 0;
    std::vector<Array> arrays_;
};

#define MDK_CUDA(call)                                                        \
    do {                                                                      \
        cudaError_t _e = (call);                                              \
        if (_e != cudaSuccess) return ::mdk::cuda_fail(_e, #call, __FILE__, __LINE__); \
    } while (0)

#define MDK_REQUIRE(cond, code, msg)  \
    do {                              \
        if (!(cond)) {                \
            ::mdk::set_error(msg);    \
            return (code);            \
        }                             \
    } while (0)

// An engine's device weights, freed with the engine.  upload() allocates an array on its first upload and reuses it on a
// reload (the model fixes its size); an empty source leaves it absent (nullptr).  The copy is queued on the engine's
// compute stream, which is then synchronised: a plain cudaMemcpy from pageable memory can return before its DMA lands,
// and the engines' streams are non-blocking (they do not wait for the legacy stream), so the first forward could read
// stale weights (seen as run-to-run 3e-6 differences in the GRU's layer-0 outputs).
struct DeviceWeights {
    std::vector<void *> allocs;
    template <class T> int upload(cudaStream_t s, T **dst, const std::vector<T> &src) {
        const size_t bytes = src.size() * sizeof(T);
        if (!bytes) return MDK_OK;
        if (!*dst) {
            void *p = nullptr;
            MDK_CUDA(cudaMalloc(&p, bytes));
            allocs.push_back(p);
            *dst = static_cast<T *>(p);
        }
        MDK_CUDA(cudaMemcpyAsync(*dst, src.data(), bytes, cudaMemcpyHostToDevice, s));
        MDK_CUDA(cudaStreamSynchronize(s));
        return MDK_OK;
    }
    ~DeviceWeights() {
        for (void *p : allocs) cudaFree(p);
    }
};

// Geometry of the fp16 hi/lo operand tiles the wgmma kernels consume (K-major, no swizzle:
// [k-group][row][8 halfs]; see ptx.cuh make_smem_desc).
constexpr int XT_ROWS = 128;                       // positions per activation tile
constexpr int XT_K = H2;                           // 256
constexpr int XT_PLANE_BYTES = XT_ROWS * XT_K * 2; // one plane (hi or lo) of a tile: 64 KiB
constexpr int XT_TILE_BYTES = 2 * XT_PLANE_BYTES;  // hi plane then lo plane

// Tile-interleaved row order of the tensor-core path's intermediates (gi, h0 tiles, h1): windows are grouped in
// tiles of WT = 16 (the recurrent kernel's N) and rows run  p' = ((w / 16) * T + t) * 16 + w % 16 , i.e. the 16
// windows of a tile are adjacent for a given time step.  A thread's windows are then `base + c * const` apart
// (immediate offsets, no per-element address arithmetic, no ragged-edge predicates: padding windows are real rows
// that are simply never copied out), and one tile-step of gi is a single contiguous 48 KiB block.
constexpr int WT = 16;
__host__ __device__ inline int64_t tiled_rows(int64_t B, int64_t T) { return ((B + WT - 1) / WT) * WT * T; }
__host__ __device__ inline int64_t tiled_row(int64_t w, int64_t t, int64_t T) { return ((w / WT) * T + t) * WT + (w % WT); }

// gi (gate pre-activations) on the tensor-core path is stored in QUAD layout: per tile-step ts = tiled row / 16 (the 16
// windows of a tile at one time step) a 48 KiB block  [blk = dir*3 + gate (6)][cg = window quad (4)][j (128)][w4 (4)]
// of floats.  A recurrent-kernel thread (hidden unit j, window quad cg) then reads its 3 gates x 4 windows as three
// 16-byte loads that are contiguous across the warp (512 B per load), the projection GEMM's epilogue thread (row j of
// block blk) writes 16-byte vectors that are contiguous across its warp, and the (ts, dir) block a CTA needs next is
// one contiguous 24 KiB range for the L2 prefetch.
constexpr int GI_TS_FLOATS = 6 * 4 * H * 4;   // 12288 floats per tile-step
__host__ __device__ inline int64_t gi_quad_index(int64_t tiled_row, int col) {
    const int64_t ts = tiled_row >> 4;
    const int w = (int)(tiled_row & 15), blk = col / H, j = col % H;
    return ((((ts * 6 + blk) * 4 + (w >> 2)) * H + j) << 2) + (w & 3);
}

// sigmoid(a) = 1 / (1 + 2^(-log2e * a)),  tanh(x) = (2^(2 log2e * x) - 1) / (2^(2 log2e * x) + 1)
constexpr float GATE_SCALE_RZ = -1.4426950408889634f;
constexpr float GATE_SCALE_N = 2.8853900817779268f;
__host__ __device__ inline float gate_scale(int gate) { return gate < 2 ? GATE_SCALE_RZ : GATE_SCALE_N; }

struct LayerWeights {
    // as loaded (host, torch layout; empty until mdk_engine_load_gru)
    std::vector<float> w_ih[NDIR];  // [3H][in]
    std::vector<float> w_hh[NDIR];  // [3H][H]
    std::vector<float> b_ih[NDIR], b_hh[NDIR];
    // device arrays the kernels read, packed on the host from the above (gru_pack.cuh) and uploaded by prepare_weights
    float *w_in_packed = nullptr;   // [768][in] fp32: rows = dir*384 + gate*128 + j
    float *bias_gi = nullptr;       // [768]: r,z: b_ih+b_hh ; n: b_ih
    float *b_hn = nullptr;          // [2][128]
    // tensor-core path: the activations' exp2 scale factors are folded into everything that feeds a gate pre-activation
    // (rows of W_hh / W_ih and the biases of the r and z gates times -log2 e, of the n gate times 2 log2 e), so the gate
    // math goes straight from the accumulators into ex2 - see gate_scale() and rec_tc_kernel
    float *bias_gi_tc = nullptr;    // [768] = bias_gi * gate_scale
    float *b_hn_tc = nullptr;       // [2][128] = b_hn * gate_scale(n)
    float *w_hh_t = nullptr;        // [2][128(k)][384] fp32 (transposed) for the FFMA path
    __half *w_hh_tm = nullptr;      // [2][hi/lo][gate][row128][k128] fp16 row-major: source of the recurrent kernel's A operand
    __half *w_x_tm = nullptr;       // layer 0, F <= 16: [2][hi/lo][gate][row128][16] fp16 (K zero-padded): fused input projection
    __half *w_in_tc = nullptr;      // layer 1 only: [6 blocks][hi/lo][row128][k256] fp16 row-major: source of the
                                    // gemm_tc shared-memory A operand
};

// The copy-out side of packing.h in both engines: one copy-out stream per engine, so groups' results reach their calls'
// buffers in serial order; ev[g % RING] marks those of group g until group g + RING reuses it.  RING is above the groups
// a caller keeps in flight (run_prediction's look-ahead keeps at most 64 calls; in the remainder phase 14 calls of
// distinct lengths, each sealing a group of its own), so a wait is on its own group's event and the small lanes' groups
// keep running side by side.
struct CopyOut {
    static constexpr int RING = 128;
    cudaStream_t stream = nullptr;
    cudaEvent_t done = nullptr;    // compute stream -> copy-out stream
    cudaEvent_t ev[RING] = {};
};
inline cudaError_t create_copy_out(CopyOut &co) {
    cudaError_t err = cudaStreamCreateWithFlags(&co.stream, cudaStreamNonBlocking);
    if (err == cudaSuccess) err = cudaEventCreateWithFlags(&co.done, cudaEventDisableTiming);
    for (int i = 0; i < CopyOut::RING && err == cudaSuccess; ++i)
        err = cudaEventCreateWithFlags(&co.ev[i], cudaEventDisableTiming);
    return err;
}

inline void destroy_copy_out(CopyOut &co) {
    if (co.stream) { cudaStreamSynchronize(co.stream); cudaStreamDestroy(co.stream); }
    if (co.done) cudaEventDestroy(co.done);
    for (cudaEvent_t ev : co.ev) if (ev) cudaEventDestroy(ev);
}

// What a variant-decoded forward adds to the head (phred.cuh): per position p the reference byte ref[p] in, the call
// byte calls[p] and the phreds of the winning and of the reference class out
struct HeadVariant {
    const uint8_t *ref;
    uint8_t *calls;
    float *pred_q, *ref_q;
};

// Once the work queued on `compute` is done, per piece of the group being launched: the probabilities, logits, labels
// and qualities the piece has, from the group's buffers to the call's (host or device), and for a variant-decoded piece
// the call bytes (into its labels) and phreds; then ev[pk.serial].
inline int copy_back(CopyOut &co, const Packing &pk, cudaStream_t compute, const float *probs, const float *logits,
                     const uint8_t *labels, const uint8_t *quals = nullptr, const HeadVariant *var = nullptr) {
    MDK_CUDA(cudaEventRecord(co.done, compute));
    MDK_CUDA(cudaStreamWaitEvent(co.stream, co.done, 0));
    int64_t w0 = 0;
    for (const Packing::Piece &p : pk.pieces) {
        const size_t n = (size_t)p.n * pk.len, dst = (size_t)p.first * pk.len, src = (size_t)w0 * pk.len;
        const size_t bytes = n * NCLS * sizeof(float);
        if (p.probs) MDK_CUDA(cudaMemcpyAsync(p.probs + dst * NCLS, probs + src * NCLS, bytes, cudaMemcpyDefault, co.stream));
        if (p.logits) MDK_CUDA(cudaMemcpyAsync(p.logits + dst * NCLS, logits + src * NCLS, bytes, cudaMemcpyDefault, co.stream));
        if (p.labels)
            MDK_CUDA(cudaMemcpyAsync(p.labels + dst, (p.ref ? var->calls : labels) + src, n, cudaMemcpyDefault, co.stream));
        if (p.quals) MDK_CUDA(cudaMemcpyAsync(p.quals + dst, quals + src, n, cudaMemcpyDefault, co.stream));
        if (p.ref) {
            MDK_CUDA(cudaMemcpyAsync(p.pred_q + dst, var->pred_q + src, n * sizeof(float), cudaMemcpyDefault, co.stream));
            MDK_CUDA(cudaMemcpyAsync(p.ref_q + dst, var->ref_q + src, n * sizeof(float), cudaMemcpyDefault, co.stream));
        }
        w0 += p.n;
    }
    MDK_CUDA(cudaEventRecord(co.ev[pk.serial % CopyOut::RING], co.stream));
    return MDK_OK;
}

// Wait for ticket's group g (Packing::settle) on ev[g % RING]: it was last recorded for g or, once reused, for a later
// group, whose copies leave the copy-out stream after g's.
template <class Eng>
int wait_ticket(CopyOut &co, Packing &pk, Eng &&eng, int64_t ticket) {
    int64_t g = 0;
    const int rc = pk.settle(eng, ticket, &g);
    if (rc) return rc;
    MDK_CUDA(cudaEventSynchronize(co.ev[g % CopyOut::RING]));
    return MDK_OK;
}

}  // namespace mdk

// The engine runs GROUPS of windows (packing.h).  A workspace (mdk_ws) is a compute stream plus the intermediates of one
// forward; a lane (mdk_lane) is the device-side staging of one group of calls - submitted host batches and forward_dev
// calls alike (features in, probabilities / labels out) - bound to one workspace.  There are more big lanes than big
// workspaces: while one group computes, others receive their features or drain their results, so the copies never hold
// the workspace (43 GB for a 1056 x 10 000 group, 4 KiB per position) idle.  One big workspace: a one-wave group already
// fills every SM, and a second 43 GB workspace would not fit beside it in 80 GB.  Small forwards (the B = 1 remainder
// regions of medaka/prediction.py:196-209) spread over the small lanes, each with a workspace of its own.
struct mdk_ws {
    cudaStream_t stream = nullptr;      // [layer-0 input projection,] layer-0 recurrence, layer-1 projection
    // layer-1 recurrence and head: on a stream of their own, so that on the tensor-core path with the fused layer-0
    // projection the next group's layer 0 (which writes only h0, already consumed by this group's projection) runs on
    // the SMs beside this group's layer 1.  l1_done marks the last layer 1 queued: every writer of gi waits for it.
    cudaStream_t l1_stream = nullptr;
    cudaEvent_t l1_done = nullptr;
    int64_t cap_pos = 0;       // capacity in positions (rounded up to XT_ROWS)
    float *gi = nullptr;       // [cap_pos][768]
    void *h0 = nullptr;        // fp32 [cap_pos][256]  or  fp16 hi/lo tiles (same byte size)
    float *h1 = nullptr;       // [cap_pos][256], allocated on first use (unfused head only)
    int64_t cap_h1 = 0;
    float *plog = nullptr;     // fused head: per-direction partial logits [dir][tile-step][class 5][16 windows]
    // geometry of the last forward run here (mdk_engine_read_activation)
    int64_t last_B = 0, last_T = 0;
    int last_precision = -1;
    bool last_fused_head = false;
};

struct mdk_lane {
    mdk_ws *ws = nullptr;      // where the lane's groups compute (fixed at engine creation)
    // device staging of the group's calls (their buffers may be host or device memory)
    int64_t cap_io = 0;        // positions
    int64_t cap_quals = 0;     // positions of d_quals (allocated for decoded calls only)
    int64_t cap_var = 0;       // positions of d_ref, d_calls, d_pred_q, d_ref_q (variant-decoded calls only)
    int64_t cap_feats = 0;     // floats
    float *d_feats = nullptr, *d_probs = nullptr, *d_logits = nullptr;
    uint8_t *d_labels = nullptr, *d_quals = nullptr;
    uint8_t *d_ref = nullptr, *d_calls = nullptr;
    float *d_pred_q = nullptr, *d_ref_q = nullptr;
    cudaEvent_t ev_in = nullptr, ev_out = nullptr;
    bool busy = false;         // ev_out marks a group the lane has not been reclaimed from
};

struct mdk_engine {
    int device = 0;
    mdk_model_desc desc{};
    int precision = MDK_PREC_TC;  // MDK_PREC_*: read when a group is launched (set_precision launches the open one first)
    int sm_count = 132;
    int rec_mode = MDK_REC_AUTO;  // tiles per CTA of the tensor-core recurrences (MDK_REC_*)
    int64_t wave256 = 0;          // gru_size 256: windows of one wave of the cluster recurrence (16 per 2 clusters)
    static constexpr int BIG_WS = 1, BIG_LANES = 4, SMALL_LANES = 14;
    static constexpr int N_LANES = BIG_LANES + SMALL_LANES, N_WS = BIG_WS + SMALL_LANES;
    static constexpr int64_t SMALL_POS = 1 << 18;   // forwards up to this many positions run on the small lanes
    mdk_ws ws[N_WS];              // [0, BIG_WS): big groups; then one per small lane
    mdk_lane lane[N_LANES];       // big lane j computes on ws[j % BIG_WS], small lane i on ws[BIG_WS + i]
    int next_big = 0, next_small = 0;
    mdk::Packing pk;
    int open_lane = -1;           // lane of the open (or last launched) group
    int last_ws = 0;              // workspace of the most recent forward
    int64_t group_windows = 0;    // most windows coalesced into one group (0 = one wave, mdk_engine_preferred_windows)
    cudaStream_t stream = nullptr;       // == ws[0].stream: weight uploads, timers (waits for every other stream)
    static constexpr int EV_RING = 32;   // per-group event sets kept for mdk_engine_mean_timings
    cudaEvent_t evr[EV_RING][8] = {};
    cudaEvent_t *ev = evr[0];            // event set of the group being launched
    int64_t fwd_count = 0;               // groups launched
    cudaEvent_t ev_timer[2] = {};
    cudaEvent_t ev_join = nullptr;
    mdk::LayerWeights layer[2];
    std::vector<float> lin_w_host, lin_b_host;     // as loaded: [5][256], [5]
    float *lin_w = nullptr, *lin_b = nullptr;
    mdk::DeviceWeights weights;   // every device array of layer[] and lin_w / lin_b
    bool keep_act = false;        // debugging: keep h1 (layer-1 output) in HBM, i.e. run the unfused head
    bool prepared = false;
    cudaStream_t copy_in = nullptr;
    mdk::CopyOut copy_out;
    mdk_timings last{};
    int64_t launches = 0;
};

namespace mdk {

// ---- launchers (each returns cudaGetLastError() of its launch) -------------------------------
// misc.cu
// tiled != 0: gi rows are written / h1 rows are read in tile-interleaved order (T = window length)
// hs: the GRU width (H or H256); gi has 6 hs columns
cudaError_t launch_inproj0(const float *feats, const float *w_packed, const float *bias, float *gi,
                           int64_t P, int F, int64_t T, int tiled, cudaStream_t s, int hs = H);
enum { HEAD_PLAIN = 0, HEAD_QUALS = 1, HEAD_VARIANT = 2 };     // the heads' instantiations
// quals (may be null): phred bytes of the argmax class (phred.cuh), from the probability the head writes; var (may be
// null): the variant outputs, from the same probabilities
cudaError_t launch_head(const float *h1, const float *lin_w, const float *lin_b, int64_t B, int64_t T, int tiled,
                        float *probs, float *logits, uint8_t *labels, cudaStream_t s, uint8_t *quals = nullptr,
                        const HeadVariant *var = nullptr, int width = H2);     // width: h1 row width, H2 or H2_256
cudaError_t launch_untile_rows(const float *src_tiled, float *dst, int64_t w0, int64_t nw, int64_t T, cudaStream_t s,
                               int width = H2);
cudaError_t launch_unpack_h0(const void *h0_tiles, float *out, int64_t w0, int64_t nw, int64_t T, cudaStream_t s);
// gru_fp32.cu
// save (training): also r, z, n and W_hn.h_{t-1} + b_hn per position, direction and unit (gru_fp32.cu)
cudaError_t launch_rec_fp32(const float *gi, const float *w_hh_t, const float *b_hn, float *h_out, int64_t B,
                            int64_t T, cudaStream_t s, int hs = H, float *save = nullptr);
// C[M][N] = A[M][K] . W[N][K]^T + bias[N], fp32 (K % 16 == 0, N % 128 == 0)
cudaError_t launch_gemm_fp32(const float *A, const float *W, const float *bias, float *C, int64_t M, int K, int N,
                             cudaStream_t s);
// gru_wg.cu
struct RecX {               // fused layer-0 input projection (rec_tc_kernel FUSE_X, F <= 16)
    const float *feats;     // [B][T][F]
    const __half *w_x;      // LayerWeights::w_x_tm: [dir][part][gate][row 128][16] fp16, K zero-padded to 16
    const float *bias;      // LayerWeights::bias_gi_tc: [768]: r,z: b_ih + b_hh ; n: b_ih
    int F;
};
// what the recurrent kernel writes: h as the fp16 hi/lo operand tiles of the layer-1 GEMM (layer 0), h as fp32 tiled rows
// [row][256] (layer 1, unfused head), or the partial logits of the 5-class linear head (fp32 W_lin [5][256] in lin_w),
// which runs inside the layer-1 recurrence in fp32 on the CUDA cores (plog layout)
enum { OUT_TILES = 0, OUT_ROWS = 1, OUT_LOGITS = 2 };
// one layer's recurrence, both directions, tiles_per_cta (1 or 2) 16-window tiles per CTA.  xin: the fused layer-0 input
// projection (OUT_TILES only), or nullptr to read the pre-activations from gi.  out: h0 tiles, h1 rows or plog (out_kind).
// fp16: the fp16 mode's kernels (one product per contraction, rec_fp16_kernel), else the three-product ones.
cudaError_t launch_rec_tc(const float *gi, const RecX *xin, const __half *w_hh_tm, const float *b_hn, int tiles_per_cta,
                          int out_kind, void *out, const float *lin_w, int64_t B, int64_t T, bool fp16, cudaStream_t s);
// head on the partial logits of the fused path: sum of the two directions + bias -> softmax / argmax (/ quals / var,
// as launch_head)
cudaError_t launch_head_plog(const float *plog, const float *lin_b, int64_t B, int64_t T, float *probs, float *logits,
                             uint8_t *labels, cudaStream_t s, uint8_t *quals = nullptr,
                             const HeadVariant *var = nullptr);
constexpr int PLOG_TS_FLOATS = NCLS * WT;     // 80 floats per (tile-step, direction)
cudaError_t launch_gemm_tc(const void *x_tiles, const __half *w_in_tm, const float *bias, float *gi, int64_t P,
                           int sm_count, bool fp16, cudaStream_t s);
int selftest_umma(int device, const float *A, const float *B, float *D, int N, int K, int variant);
// gru256.cu: the tensor-core path at gru_size 256.  gi [tiled rows][1536] and h [tiled rows][512] fp32 (gru256.cu).
// One layer's recurrence, both directions, one 4-CTA cluster per (16-window tile, direction); fp16 as launch_rec_tc's:
cudaError_t launch_rec256_tc(const float *gi, const __half *w_hh_tm, const float *b_hn, float *h_out, int64_t B,
                             int64_t T, bool fp16, cudaStream_t s);
// clusters of the recurrence that are resident at once (one wave)
cudaError_t rec256_max_clusters(int *clusters);
// layer-1 input projection over M tiled rows (w_in_tm: LayerWeights::w_in_tc at 256)
cudaError_t launch_gemm256_tc(const float *h0, const __half *w_in_tm, const float *bias, float *gi, int64_t M, bool fp16,
                              cudaStream_t s);
// pileup.cu
// exclusive scan of n per-block counts, in place, by one block: counts[i] = sum of counts[0, i), counts[n] = the total
cudaError_t launch_scan_blocks(int64_t *counts, int64_t n, cudaStream_t s);
// The eight BAM record arrays of a featuriser call (host or device copies); cigar_off / seq_off hold n_rec + 1 offsets.
struct Records {
    const int32_t *pos;
    const uint16_t *flag;
    const uint8_t *mapq, *dtype;
    const uint32_t *cigar;
    const int64_t *cigar_off;
    const uint8_t *seq;
    const int64_t *seq_off;
};
// Counts of a region (device pointers in, device pointers out; the column plan lives in the SCRATCH blob until the call
// returns).  Returns the number of columns through *n_cols_host; if it exceeds max_cols the outputs are incomplete and
// the caller re-runs with a larger buffer.
int pileup_counts_dev(int64_t n_rec, const Records &d, int64_t n_ops, int32_t start, int32_t end, int num_dtypes,
                      int min_mapq, int64_t max_cols, uint64_t *counts, int64_t *major, int64_t *minor,
                      int64_t *n_cols_host, cudaStream_t s);

}  // namespace mdk
