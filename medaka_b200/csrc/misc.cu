// The GRU path's small kernels: layer-0 input projection, linear head + softmax + argmax, and the debug unpacking of
// the tiled intermediates.  All are coalesced / vectorised streaming kernels; none is GEMM-shaped.
#include "common.cuh"
#include "phred.cuh"
#include "ptx.cuh"

namespace mdk {

// =====================================================================================
// Layer-0 input projection: gi[p][c] = sum_f x[p][f] * W[c][f] + bias[c],  c in [0, 6 HS)
// K = F (10 or 20) is far too thin for the tensor cores; the kernel is bound by the 3 KiB/position
// (6 KiB at HS = 256) write of gi.  256 threads, each owns 3 (6) of the 768 (1536) columns with its weights in registers.
// =====================================================================================
// Column c of position p into gi: plain rows (fp32 path), or, on the tensor-core path, pre-scaled for the exp2-based gate
// math (common.cuh gate_scale) in the quad layout (HS = 128, common.cuh) or as tile-interleaved rows (HS = 256, gru256.cu)
template <int HS>
__device__ __forceinline__ void store_gi(float *gi, int64_t p, int64_t T, int c, float a, int tiled) {
    if (!tiled) {
        gi[p * (6 * HS) + c] = a;
        return;
    }
    const int64_t orow = tiled_row(p / T, p % T, T);
    const float v = a * gate_scale((c % (3 * HS)) / HS);
    if (HS == H) gi[gi_quad_index(orow, c)] = v;
    else gi[orow * (6 * HS) + c] = v;
}

template <int F, int HS>
__global__ void __launch_bounds__(256) inproj0_kernel(const float *__restrict__ feats, const float *__restrict__ w,
                                                      const float *__restrict__ bias, float *__restrict__ gi,
                                                      int64_t P, int64_t T, int tiled) {
    constexpr int PT = 64;   // positions per block
    constexpr int NQ = 6 * HS / 256;   // columns per thread
    __shared__ float xs[PT * F];
    const int tid = threadIdx.x;
    const int64_t p0 = (int64_t)blockIdx.x * PT;
    const int np = (int)min((int64_t)PT, P - p0);
    for (int i = tid; i < np * F; i += 256) xs[i] = feats[p0 * F + i];
    float wr[NQ][F], b[NQ];
#pragma unroll
    for (int q = 0; q < NQ; ++q) {
        const int c = tid + 256 * q;
        b[q] = bias[c];
#pragma unroll
        for (int f = 0; f < F; ++f) wr[q][f] = w[c * F + f];
    }
    __syncthreads();
    for (int p = 0; p < np; ++p) {
        float a[NQ];
#pragma unroll
        for (int q = 0; q < NQ; ++q) a[q] = b[q];
#pragma unroll
        for (int f = 0; f < F; ++f) {
            const float x = xs[p * F + f];   // smem broadcast
#pragma unroll
            for (int q = 0; q < NQ; ++q) a[q] = fmaf(x, wr[q][f], a[q]);
        }
        const int64_t pp = p0 + p;
#pragma unroll
        for (int q = 0; q < NQ; ++q) store_gi<HS>(gi, pp, T, tid + 256 * q, a[q], tiled);
    }
}

// generic F (weights streamed from L1/L2)
template <int HS>
__global__ void __launch_bounds__(256) inproj0_generic_kernel(const float *__restrict__ feats,
                                                              const float *__restrict__ w,
                                                              const float *__restrict__ bias, float *__restrict__ gi,
                                                              int64_t P, int F, int64_t T, int tiled) {
    const int64_t p = blockIdx.x;
    if (p >= P) return;
    for (int c = threadIdx.x; c < 6 * HS; c += 256) {
        float a = bias[c];
        for (int f = 0; f < F; ++f) a = fmaf(feats[p * F + f], w[c * F + f], a);
        store_gi<HS>(gi, p, T, c, a, tiled);
    }
}

template <int HS>
static cudaError_t launch_inproj0_hs(const float *feats, const float *w_packed, const float *bias, float *gi, int64_t P,
                                     int F, int64_t T, int tiled, cudaStream_t s) {
    const unsigned blocks = (unsigned)((P + 63) / 64);
    if (F == 10) inproj0_kernel<10, HS><<<blocks, 256, 0, s>>>(feats, w_packed, bias, gi, P, T, tiled);
    else if (F == 20) inproj0_kernel<20, HS><<<blocks, 256, 0, s>>>(feats, w_packed, bias, gi, P, T, tiled);
    else inproj0_generic_kernel<HS><<<(unsigned)P, 256, 0, s>>>(feats, w_packed, bias, gi, P, F, T, tiled);
    return cudaGetLastError();
}

cudaError_t launch_inproj0(const float *feats, const float *w_packed, const float *bias, float *gi, int64_t P,
                           int F, int64_t T, int tiled, cudaStream_t s, int hs) {
    if (P == 0) return cudaSuccess;
    return hs == H256 ? launch_inproj0_hs<H256>(feats, w_packed, bias, gi, P, F, T, tiled, s)
                      : launch_inproj0_hs<H>(feats, w_packed, bias, gi, P, F, T, tiled, s);
}

// =====================================================================================
// Head: logits = h1 . W^T + b (gru.py:67), probs = softmax (gru.py:71), label = argmax (labels.py:1063)
// One warp per position, 8 of the 256 inputs per lane; 1 KiB read + 41 B written per position.
// =====================================================================================
// Outputs always go to position p = w*T + t; on the tensor-core path the h1 row of that position is the
// tile-interleaved row(w, t).  Each warp handles 4 positions per iteration: 8 of the 256 inputs per lane, the
// 4 x 5 (padded to 4 x 8) partial dot products are reduced with a transposing butterfly (31 shuffles for all 32
// values instead of 5 per value), after which lane L owns logit (position L/8, class L%8) and the softmax / argmax
// run across the 8-lane groups - one expf per lane instead of five per lane.  HEAD_QUALS: also the phred byte of the
// winning probability (consensus-decoded forwards); HEAD_VARIANT: also the call byte and the phreds of the winning and of
// the reference class (variant-decoded forwards, phred.cuh), and the phred byte where quals is given.  HEAD_PLAIN is the
// kernel of the ordinary forward.
template <int MODE, int K>
__global__ void __launch_bounds__(256) head_kernel(const float *__restrict__ h1, const float *__restrict__ lin_w,
                                                   const float *__restrict__ lin_b, int64_t P, int64_t B, int64_t T,
                                                   int tiled, float *__restrict__ probs, float *__restrict__ logits,
                                                   uint8_t *__restrict__ labels, uint8_t *__restrict__ quals,
                                                   HeadVariant var) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    constexpr int NI = K / 32;                     // inputs per lane: 8 (H = 128) or 16 (H = 256)
    float w[NCLS][NI];
#pragma unroll
    for (int c = 0; c < NCLS; ++c)
#pragma unroll
        for (int v = 0; v < NI / 4; ++v) {
            const float4 a = *reinterpret_cast<const float4 *>(lin_w + c * K + lane * NI + 4 * v);
            w[c][4 * v] = a.x; w[c][4 * v + 1] = a.y; w[c][4 * v + 2] = a.z; w[c][4 * v + 3] = a.w;
        }
    const int cls = lane & 7;                      // class owned by this lane after the reduction
    const float my_bias = cls < NCLS ? lin_b[cls] : 0.f;
    constexpr int PU = 4;
    // Each warp walks a CONTIGUOUS chunk of row quads of h1 (rows = the tensor-core path's tile-interleaved order, or plain
    // position order): the row -> (window, t) -> output position mapping is then one 64-bit division per warp and an
    // increment per iteration, where a grid-stride loop paid two divisions per position (the kernel is instruction-bound:
    // 170 instructions per position before this change, profiles/r01f_ncu_full.md).
    const int64_t rows = tiled ? tiled_rows(B, T) : P;            // multiple of 16 when tiled
    const int64_t quads = (rows + PU - 1) / PU;
    const int64_t per_warp = (quads + nwarps - 1) / nwarps;
    const int64_t q0 = warp * per_warp, q1 = min(quads, q0 + per_warp);
    // position of the first row of the chunk: tiled row r = ((w / 16) * T + t) * 16 + w % 16
    int64_t wt = 0, t = 0;      // window tile, time step
    int wl = 0;                 // window within the tile (multiple of 4 at quad granularity)
    if (tiled && q0 < q1) {
        const int64_t r0 = q0 * PU;
        wt = r0 / (T * WT);
        const int64_t rem = r0 - wt * (T * WT);
        t = rem / WT;
        wl = (int)(rem - t * WT);
    }
    for (int64_t q = q0; q < q1; ++q) {
        const int64_t rb = q * PU;                 // first row of the quad
        float4 va[PU][NI / 4];
#pragma unroll
        for (int u = 0; u < PU; ++u) {
            const int64_t r = min(rb + u, rows - 1);
#pragma unroll
            for (int v = 0; v < NI / 4; ++v) va[u][v] = ld_stream4(h1 + r * K + lane * NI + 4 * v);
        }
        float v[32];
#pragma unroll
        for (int u = 0; u < PU; ++u) {
            float x[NI];
#pragma unroll
            for (int i = 0; i < NI / 4; ++i) {
                x[4 * i] = va[u][i].x; x[4 * i + 1] = va[u][i].y; x[4 * i + 2] = va[u][i].z; x[4 * i + 3] = va[u][i].w;
            }
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                float s = 0.f;
                if (c < NCLS) {
#pragma unroll
                    for (int i = 0; i < NI; ++i) s = fmaf(x[i], w[c][i], s);
                }
                v[u * 8 + c] = s;
            }
        }
        // transposing butterfly: after the step with mask m a lane keeps the half of its values selected by (lane & m)
#pragma unroll
        for (int m = 16, cnt = 16; m >= 1; m >>= 1, cnt >>= 1) {
            const bool hi = (lane & m) != 0;
#pragma unroll
            for (int i = 0; i < cnt; ++i) {
                const float send = hi ? v[i] : v[i + cnt];
                const float keep = hi ? v[i + cnt] : v[i];
                v[i] = keep + __shfl_xor_sync(0xffffffffu, send, m);
            }
        }
        // lane L: logit of position pb + L/8, class L%8 (classes 5..7 are padding)
        const float logit = cls < NCLS ? v[0] + my_bias : -INFINITY;
        float mx = logit;
#pragma unroll
        for (int m = 4; m >= 1; m >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, m));
        const float e = cls < NCLS ? expf(logit - mx) : 0.f;
        float e0 = __shfl_sync(0xffffffffu, e, (lane & 24) + 0), e1 = __shfl_sync(0xffffffffu, e, (lane & 24) + 1),
              e2 = __shfl_sync(0xffffffffu, e, (lane & 24) + 2), e3 = __shfl_sync(0xffffffffu, e, (lane & 24) + 3),
              e4 = __shfl_sync(0xffffffffu, e, (lane & 24) + 4);
        const float sum = (((e0 + e1) + e2) + e3) + e4;          // class order, like a sequential softmax
        const float pr = e / sum;
        // argmax over the 5 probabilities, first maximum wins (np.argmax, labels.py:1063)
        float best = cls < NCLS ? pr : -1.f;
        int arg = cls;
#pragma unroll
        for (int m = 4; m >= 1; m >>= 1) {
            const float ob = __shfl_xor_sync(0xffffffffu, best, m);
            const int oa = __shfl_xor_sync(0xffffffffu, arg, m);
            if (ob > best || (ob == best && oa < arg)) { best = ob; arg = oa; }
        }
        // output position of this lane's row (quad row lane >> 3)
        int64_t p;
        bool ok;
        if (tiled) {
            const int64_t win = wt * WT + wl + (lane >> 3);
            p = win * T + t;
            ok = win < B;                            // padding windows of a ragged last tile are real rows, never copied out
            wl += PU;
            if (wl == WT) {
                wl = 0;
                if (++t == T) { t = 0; ++wt; }
            }
        } else {
            p = rb + (lane >> 3);
            ok = p < P;
        }
        uint8_t ref = 0;
        float p_ref = 0.f;
        if (MODE == HEAD_VARIANT) {             // the reference class's probability from its lane of the 8-lane group
            if (ok) ref = var.ref[p];
            p_ref = __shfl_sync(0xffffffffu, pr, (lane & 24) + ref_class(ref));
        }
        if (ok) {
            if (cls < NCLS) {
                probs[p * NCLS + cls] = pr;
                if (logits) logits[p * NCLS + cls] = logit;
            }
            if (labels && cls == 0) labels[p] = (uint8_t)arg;
            if (MODE == HEAD_QUALS && cls == 0) quals[p] = phred_char(best);
            if (MODE == HEAD_VARIANT && cls == 0) {
                if (quals) quals[p] = phred_char(best);
                var.calls[p] = variant_call(arg, ref);
                var.pred_q[p] = phred_f32(best);
                var.ref_q[p] = phred_f32(p_ref);
            }
        }
    }
}

template <int K>
static cudaError_t launch_head_k(const float *h1, const float *lin_w, const float *lin_b, int64_t B, int64_t T, int tiled,
                                 float *probs, float *logits, uint8_t *labels, cudaStream_t s, uint8_t *quals,
                                 const HeadVariant *var) {
    const int64_t P = B * T;
    int64_t blocks = (P + 31) / 32;            // 8 warps per block, 4 positions per warp per iteration
    if (blocks > 132 * 8) blocks = 132 * 8;    // persistent-ish grid: multiple of the SM count
    const dim3 g((unsigned)blocks);
    if (var) head_kernel<HEAD_VARIANT, K><<<g, 256, 0, s>>>(h1, lin_w, lin_b, P, B, T, tiled, probs, logits, labels, quals, *var);
    else if (quals) head_kernel<HEAD_QUALS, K><<<g, 256, 0, s>>>(h1, lin_w, lin_b, P, B, T, tiled, probs, logits, labels, quals, {});
    else head_kernel<HEAD_PLAIN, K><<<g, 256, 0, s>>>(h1, lin_w, lin_b, P, B, T, tiled, probs, logits, labels, nullptr, {});
    return cudaGetLastError();
}

cudaError_t launch_head(const float *h1, const float *lin_w, const float *lin_b, int64_t B, int64_t T, int tiled,
                        float *probs, float *logits, uint8_t *labels, cudaStream_t s, uint8_t *quals,
                        const HeadVariant *var, int width) {
    if (B * T == 0) return cudaSuccess;
    return width == H2_256 ? launch_head_k<H2_256>(h1, lin_w, lin_b, B, T, tiled, probs, logits, labels, s, quals, var)
                           : launch_head_k<H2>(h1, lin_w, lin_b, B, T, tiled, probs, logits, labels, s, quals, var);
}

// Head of the fused path (gru.py:53-55,67-71): logits = fwd partial + rev partial + bias, softmax, first-max argmax.
// One thread per (window of the tile, time step); blockIdx.y = window tile.  41 B written per position, 40 B read.
// MODE as in head_kernel.
template <int MODE>
__global__ void __launch_bounds__(256) head_plog_kernel(const float *__restrict__ plog, const float *__restrict__ lin_b,
                                                        int64_t B, int64_t T, int64_t n_ts, float *__restrict__ probs,
                                                        float *__restrict__ logits, uint8_t *__restrict__ labels,
                                                        uint8_t *__restrict__ quals, HeadVariant var) {
    const int64_t wt = blockIdx.y;
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;   // t * 16 + w
    const int64_t t = i >> 4;
    const int w = (int)(i & 15);
    if (t >= T) return;
    const int64_t win = wt * WT + w;
    const float *p0 = plog + (wt * T + t) * PLOG_TS_FLOATS + w;
    const float *p1 = p0 + n_ts * PLOG_TS_FLOATS;
    float lg[NCLS];
#pragma unroll
    for (int c = 0; c < NCLS; ++c) lg[c] = (ldg_stream(p0 + c * WT) + ldg_stream(p1 + c * WT)) + lin_b[c];
    if (win >= B) return;                          // padding windows of a ragged last tile
    float mx = lg[0];
#pragma unroll
    for (int c = 1; c < NCLS; ++c) mx = fmaxf(mx, lg[c]);
    float e[NCLS], sum = 0.f;
#pragma unroll
    for (int c = 0; c < NCLS; ++c) { e[c] = expf(lg[c] - mx); sum += e[c]; }   // class order, like a sequential softmax
    const int64_t p = win * T + t;
    float best = -1.f, p_ref = 0.f;
    int arg = 0;
    const uint8_t ref = MODE == HEAD_VARIANT ? var.ref[p] : 0;
    const int rc = ref_class(ref);
#pragma unroll
    for (int c = 0; c < NCLS; ++c) {
        const float pr = e[c] / sum;
        probs[p * NCLS + c] = pr;
        if (logits) logits[p * NCLS + c] = lg[c];
        if (pr > best) { best = pr; arg = c; }     // first maximum wins (np.argmax, labels.py:1063)
        if (MODE == HEAD_VARIANT && c == rc) p_ref = pr;
    }
    if (labels) labels[p] = (uint8_t)arg;
    if (MODE == HEAD_QUALS) quals[p] = phred_char(best);
    if (MODE == HEAD_VARIANT) {
        if (quals) quals[p] = phred_char(best);
        var.calls[p] = variant_call(arg, ref);
        var.pred_q[p] = phred_f32(best);
        var.ref_q[p] = phred_f32(p_ref);
    }
}

cudaError_t launch_head_plog(const float *plog, const float *lin_b, int64_t B, int64_t T, float *probs, float *logits,
                             uint8_t *labels, cudaStream_t s, uint8_t *quals, const HeadVariant *var) {
    if (B == 0 || T == 0) return cudaSuccess;
    const int64_t tiles = (B + WT - 1) / WT;
    dim3 grid((unsigned)((T * WT + 255) / 256), (unsigned)tiles);
    const int64_t n_ts = tiles * T;
    if (var) head_plog_kernel<HEAD_VARIANT><<<grid, 256, 0, s>>>(plog, lin_b, B, T, n_ts, probs, logits, labels, quals, *var);
    else if (quals) head_plog_kernel<HEAD_QUALS><<<grid, 256, 0, s>>>(plog, lin_b, B, T, n_ts, probs, logits, labels, quals, {});
    else head_plog_kernel<HEAD_PLAIN><<<grid, 256, 0, s>>>(plog, lin_b, B, T, n_ts, probs, logits, labels, nullptr, {});
    return cudaGetLastError();
}

// fp16 hi/lo activation tiles (tile-interleaved rows) -> fp32 [nw*T][256] in position order: windows w0 .. w0 + nw - 1
// (debug / layer-wise parity)
__global__ void unpack_h0_kernel(const __half *__restrict__ tiles, float *__restrict__ out, int64_t w0, int64_t nw,
                                 int64_t T) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= nw * T * H2) return;
    const int64_t p = w0 * T + i / H2;
    const int k = (int)(i % H2);
    const int64_t row = tiled_row(p / T, p % T, T);
    const int64_t tile = row / XT_ROWS;
    const int r = (int)(row % XT_ROWS);
    const __half *base = tiles + tile * (XT_TILE_BYTES / 2);
    const int64_t off = (int64_t)(k / 8) * (XT_ROWS * 8) + r * 8 + (k % 8);
    out[i] = __half2float(base[off]) + __half2float(base[XT_PLANE_BYTES / 2 + off]);
}

cudaError_t launch_unpack_h0(const void *h0_tiles, float *out, int64_t w0, int64_t nw, int64_t T, cudaStream_t s) {
    const int64_t n = nw * T * H2;
    if (n == 0) return cudaSuccess;
    unpack_h0_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(reinterpret_cast<const __half *>(h0_tiles), out, w0, nw, T);
    return cudaGetLastError();
}

// fp32 [rows'][width] in tile-interleaved order -> [nw*T][width] in position order: windows w0 .. w0 + nw - 1 (debug /
// layer-wise parity)
__global__ void untile_rows_kernel(const float *__restrict__ src, float *__restrict__ dst, int64_t w0, int64_t nw,
                                   int64_t T, int width) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= nw * T * width) return;
    const int64_t p = w0 * T + i / width;
    dst[i] = src[tiled_row(p / T, p % T, T) * width + (i % width)];
}

cudaError_t launch_untile_rows(const float *src_tiled, float *dst, int64_t w0, int64_t nw, int64_t T, cudaStream_t s,
                               int width) {
    const int64_t n = nw * T * width;
    if (n == 0) return cudaSuccess;
    untile_rows_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(src_tiled, dst, w0, nw, T, width);
    return cudaGetLastError();
}

}  // namespace mdk
