// HBM-bound kernels of the hot path: count normalisation, layer-0 input projection,
// linear head + softmax + argmax, consensus decode (argmax + phred), weight packing.
// All are coalesced / vectorised streaming kernels; none is GEMM-shaped.
#include "common.cuh"
#include "ptx.cuh"

namespace mdk {

// =====================================================================================
// Count normalisation  (CountsFeatureEncoder._post_process_pileup, medaka/features.py:871-935)
// One thread per pileup column.  Algorithmic bytes per column (F=10): read 80 (counts) + 16
// (major, minor), write 40 (features) + 8 (depth) = 144 B.
// =====================================================================================
// index helpers for the per-(dtype, strand) groups of medaka/features.py:647-687:
// feature order per dtype is 'acgtACGTdD' (src/medaka_counts.h:19): reverse = {0,1,2,3,8}, forward = {4,5,6,7,9}
__device__ __forceinline__ bool feat_is_rev(int f10) { return f10 < 4 || f10 == 8; }

__device__ __forceinline__ int64_t lower_bound_major(const int64_t *__restrict__ major, int64_t n, int64_t key) {
    int64_t lo = 0, hi = n;
    while (lo < hi) {
        int64_t mid = (lo + hi) >> 1;
        if (major[mid] < key) lo = mid + 1; else hi = mid;
    }
    return lo;
}

template <int ND>
__global__ void __launch_bounds__(256) normalise_kernel(const uint64_t *__restrict__ counts,
                                                        const int64_t *__restrict__ major,
                                                        const int64_t *__restrict__ minor, int64_t n, int mode,
                                                        int sym_indels, float *__restrict__ feats,
                                                        int64_t *__restrict__ depth_out) {
    constexpr int F = 10 * ND;
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint64_t c[F];
    {
        const ulonglong2 *src = reinterpret_cast<const ulonglong2 *>(counts + i * F);
#pragma unroll
        for (int q = 0; q < F / 2; ++q) {
            ulonglong2 v = src[q];
            c[2 * q] = v.x;
            c[2 * q + 1] = v.y;
        }
    }
    const int64_t mn = minor[i];
    // group sums of this column: gs[dt][0] = reverse strand, gs[dt][1] = forward strand
    uint64_t gs_i[ND][2];
#pragma unroll
    for (int dt = 0; dt < ND; ++dt) {
        gs_i[dt][0] = c[dt * 10 + 0] + c[dt * 10 + 1] + c[dt * 10 + 2] + c[dt * 10 + 3] + c[dt * 10 + 8];
        gs_i[dt][1] = c[dt * 10 + 4] + c[dt * 10 + 5] + c[dt * 10 + 6] + c[dt * 10 + 7] + c[dt * 10 + 9];
    }
    uint64_t gs_p[ND][2];      // group sums of the parent (major) column, ORIGINAL counts
    uint64_t del_p[ND][2];     // parent's original deletion counts (needed only if the parent is a minor column)
    int64_t parent_minor = 0;
    if (mn > 0) {
        // np.searchsorted(positions['major'], major, side='left'): first column with this major.  Columns of one
        // major are contiguous with minors counting up from the first one, so the parent is normally mn columns back
        // (two loads to confirm); anything else (a chunk cut inside an insertion run, repeated majors) takes the search.
        const int64_t mj = major[i];
        int64_t j = i - mn;
        if (j < 0 || major[j] != mj || (j > 0 && major[j - 1] == mj)) j = lower_bound_major(major, n, mj);
        parent_minor = minor[j];
        const ulonglong2 *src = reinterpret_cast<const ulonglong2 *>(counts + j * F);
        uint64_t p[F];
#pragma unroll
        for (int q = 0; q < F / 2; ++q) {
            ulonglong2 v = src[q];
            p[2 * q] = v.x;
            p[2 * q + 1] = v.y;
        }
#pragma unroll
        for (int dt = 0; dt < ND; ++dt) {
            gs_p[dt][0] = p[dt * 10 + 0] + p[dt * 10 + 1] + p[dt * 10 + 2] + p[dt * 10 + 3] + p[dt * 10 + 8];
            gs_p[dt][1] = p[dt * 10 + 4] + p[dt * 10 + 5] + p[dt * 10 + 6] + p[dt * 10 + 7] + p[dt * 10 + 9];
            del_p[dt][0] = p[dt * 10 + 8];
            del_p[dt][1] = p[dt * 10 + 9];
        }
    } else {
#pragma unroll
        for (int dt = 0; dt < ND; ++dt) {
            gs_p[dt][0] = gs_i[dt][0];
            gs_p[dt][1] = gs_i[dt][1];
            del_p[dt][0] = c[dt * 10 + 8];
            del_p[dt][1] = c[dt * 10 + 9];
        }
    }
    // depth = row sum of the parent column's original counts (features.py:889-890)
    uint64_t depth = 0;
#pragma unroll
    for (int dt = 0; dt < ND; ++dt) depth += gs_p[dt][0] + gs_p[dt][1];
    if (depth_out) depth_out[i] = (int64_t)depth;

    if (sym_indels && mn > 0) {
        // features.py:892-908: reads spanning the insertion site without the insertion count as deletions
#pragma unroll
        for (int dt = 0; dt < ND; ++dt) {
            c[dt * 10 + 8] = gs_p[dt][0] - gs_i[dt][0];   // uint64 wrap-around like numpy
            c[dt * 10 + 9] = gs_p[dt][1] - gs_i[dt][1];
        }
    }
    float out[F];
    if (mode == MDK_NORM_TOTAL) {
        const double d = (double)(depth > 1 ? depth : 1);
#pragma unroll
        for (int f = 0; f < F; ++f) out[f] = __double2float_rn((double)c[f] / d);   // f64 divide then cast (features.py:914,926)
    } else if (mode == MDK_NORM_FWD_REV) {
        // features.py:915-923: per (dtype, strand) depth, recomputed from the (possibly sym_indels-modified)
        // counts; minor columns take their parent's group depth.
#pragma unroll
        for (int dt = 0; dt < ND; ++dt) {
#pragma unroll
            for (int st = 0; st < 2; ++st) {
                uint64_t g;
                if (mn > 0) {
                    g = gs_p[dt][st];
                    // parent itself a minor column (chunk cut inside an insertion run): its own deletion
                    // slot was overwritten by the sym_indels fill (with gs_p - gs_p = 0)
                    if (sym_indels && parent_minor > 0) g -= del_p[dt][st];
                } else {
                    g = gs_i[dt][st];
                }
                const double d = (double)(g > 1 ? g : 1);
#pragma unroll
                for (int b = 0; b < 10; ++b) {
                    if (feat_is_rev(b) == (st == 0)) out[dt * 10 + b] = __double2float_rn((double)c[dt * 10 + b] / d);
                }
            }
        }
    } else {
#pragma unroll
        for (int f = 0; f < F; ++f) out[f] = (float)c[f];
    }
    float2 *dst = reinterpret_cast<float2 *>(feats + i * F);
#pragma unroll
    for (int q = 0; q < F / 2; ++q) dst[q] = make_float2(out[2 * q], out[2 * q + 1]);
}

cudaError_t launch_normalise(const uint64_t *counts, const int64_t *major, const int64_t *minor, int64_t n,
                             int num_dtypes, int mode, int sym_indels, float *feats, int64_t *depth,
                             cudaStream_t s) {
    if (n == 0) return cudaSuccess;
    const int threads = 256;
    const unsigned blocks = (unsigned)((n + threads - 1) / threads);
    switch (num_dtypes) {
        case 1: normalise_kernel<1><<<blocks, threads, 0, s>>>(counts, major, minor, n, mode, sym_indels, feats, depth); break;
        case 2: normalise_kernel<2><<<blocks, threads, 0, s>>>(counts, major, minor, n, mode, sym_indels, feats, depth); break;
        case 3: normalise_kernel<3><<<blocks, threads, 0, s>>>(counts, major, minor, n, mode, sym_indels, feats, depth); break;
        case 4: normalise_kernel<4><<<blocks, threads, 0, s>>>(counts, major, minor, n, mode, sym_indels, feats, depth); break;
        default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}

// =====================================================================================
// Consensus decode (labels.py:1053-1085, _phred :387-401).  41 B per position.
// =====================================================================================
__global__ void __launch_bounds__(256) decode_kernel(const float *__restrict__ probs, int64_t n,
                                                     uint8_t *__restrict__ labels, uint8_t *__restrict__ quals) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float *p = probs + i * NCLS;
    float best = p[0];
    int arg = 0;
#pragma unroll
    for (int c = 1; c < NCLS; ++c) {
        const float v = p[c];
        if (v > best) { best = v; arg = c; }   // strict '>' : first maximum wins, as np.argmax
    }
    labels[i] = (uint8_t)arg;
    if (quals) {
        float err = 1.0f - best;                              // float32 arithmetic, like numpy on f32 probs
        err = fminf(fmaxf(err, 1e-7f), 1.0f);                 // np.clip(err, 10**-7, 1)
        const float l = __double2float_rn(log10((double)err));  // correctly rounded float32 log10
        float q = -10.0f * l;
        q = fminf(q, 70.0f);
        quals[i] = (uint8_t)((int)q + 33);                    // astype('u1') truncation, +33
    }
}

// float64 probabilities (what numpy computes when label_probs is a float64 array, e.g. the reference's own
// test literals medaka/test/test_labels.py:252-266): every step in double, like numpy would.
__global__ void __launch_bounds__(256) decode_f64_kernel(const double *__restrict__ probs, int64_t n,
                                                         uint8_t *__restrict__ labels, uint8_t *__restrict__ quals) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double *p = probs + i * NCLS;
    double best = p[0];
    int arg = 0;
#pragma unroll
    for (int c = 1; c < NCLS; ++c) {
        const double v = p[c];
        if (v > best) { best = v; arg = c; }
    }
    labels[i] = (uint8_t)arg;
    if (quals) {
        double err = 1.0 - best;
        err = fmin(fmax(err, 1e-7), 1.0);
        double q = -10.0 * log10(err);
        q = fmin(q, 70.0);
        quals[i] = (uint8_t)((int)q + 33);
    }
}

cudaError_t launch_decode_f64(const double *probs, int64_t n, uint8_t *labels, uint8_t *quals, cudaStream_t s) {
    if (n == 0) return cudaSuccess;
    decode_f64_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(probs, n, labels, quals);
    return cudaGetLastError();
}

cudaError_t launch_decode(const float *probs, int64_t n, uint8_t *labels, uint8_t *quals, cudaStream_t s) {
    if (n == 0) return cudaSuccess;
    decode_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(probs, n, labels, quals);
    return cudaGetLastError();
}

// =====================================================================================
// Variant columns (src/medaka_rnn_variants.c:28-55, called from labels.py:869-887): a major column is variant when
// reference and prediction differ there; the minor (insertion) columns that follow it are variant when ANY column of
// the group - the major or one of its minors - differs.  The reference walks the columns sequentially; here every
// column finds its group (insertion runs are short) and reduces over it.  ~10 B per column.
// =====================================================================================
__global__ void __launch_bounds__(256) variant_columns_kernel(const int64_t *__restrict__ minor,
                                                              const uint8_t *__restrict__ ref,
                                                              const uint8_t *__restrict__ pred, int64_t n,
                                                              uint8_t *__restrict__ out) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const bool mism = ref[i] != pred[i];
    if (i == 0 || minor[i] == 0) {          // the first column is taken as a major ("assume start on major")
        out[i] = mism;
        return;
    }
    bool any = mism;
    for (int64_t j = i - 1; j >= 0 && !any; --j) {      // back to (and including) the group's major column
        any = ref[j] != pred[j];
        if (j == 0 || minor[j] == 0) break;
    }
    for (int64_t j = i + 1; j < n && !any && minor[j] != 0; ++j) any = ref[j] != pred[j];
    out[i] = any;
}

cudaError_t launch_variant_columns(const int64_t *minor, const uint8_t *ref, const uint8_t *pred, int64_t n,
                                   uint8_t *out, cudaStream_t s) {
    if (n == 0) return cudaSuccess;
    variant_columns_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(minor, ref, pred, n, out);
    return cudaGetLastError();
}

// =====================================================================================
// Layer-0 input projection: gi[p][c] = sum_f x[p][f] * W[c][f] + bias[c],  c in [0,768)
// K = F (10 or 20) is far too thin for the tensor cores; the kernel is bound by the 3 KiB/position
// write of gi.  256 threads, each owns 3 of the 768 columns with its weights in registers.
// =====================================================================================
template <int F>
__global__ void __launch_bounds__(256) inproj0_kernel(const float *__restrict__ feats, const float *__restrict__ w,
                                                      const float *__restrict__ bias, float *__restrict__ gi,
                                                      int64_t P, int64_t T, int tiled) {
    constexpr int PT = 64;   // positions per block
    __shared__ float xs[PT * F];
    const int tid = threadIdx.x;
    const int64_t p0 = (int64_t)blockIdx.x * PT;
    const int np = (int)min((int64_t)PT, P - p0);
    for (int i = tid; i < np * F; i += 256) xs[i] = feats[p0 * F + i];
    float wr[3][F], b[3];
#pragma unroll
    for (int q = 0; q < 3; ++q) {
        const int c = tid + 256 * q;
        b[q] = bias[c];
#pragma unroll
        for (int f = 0; f < F; ++f) wr[q][f] = w[c * F + f];
    }
    __syncthreads();
    for (int p = 0; p < np; ++p) {
        float a0 = b[0], a1 = b[1], a2 = b[2];
#pragma unroll
        for (int f = 0; f < F; ++f) {
            const float x = xs[p * F + f];   // smem broadcast
            a0 = fmaf(x, wr[0][f], a0);
            a1 = fmaf(x, wr[1][f], a1);
            a2 = fmaf(x, wr[2][f], a2);
        }
        const int64_t pp = p0 + p;
        if (tiled) {   // tensor-core path: quad layout (common.cuh)
            const int64_t orow = tiled_row(pp / T, pp % T, T);
            // (pre-scaled for the exp2-based gate math of rec_tc_kernel, common.cuh gate_scale)
            gi[gi_quad_index(orow, tid)] = a0 * gate_scale((tid % G3) / H);
            gi[gi_quad_index(orow, tid + 256)] = a1 * gate_scale(((tid + 256) % G3) / H);
            gi[gi_quad_index(orow, tid + 512)] = a2 * gate_scale(((tid + 512) % G3) / H);
        } else {
            float *row = gi + pp * GI_COLS;
            row[tid] = a0;
            row[tid + 256] = a1;
            row[tid + 512] = a2;
        }
    }
}

// generic F (weights streamed from L1/L2)
__global__ void __launch_bounds__(256) inproj0_generic_kernel(const float *__restrict__ feats,
                                                              const float *__restrict__ w,
                                                              const float *__restrict__ bias, float *__restrict__ gi,
                                                              int64_t P, int F, int64_t T, int tiled) {
    const int64_t p = blockIdx.x;
    if (p >= P) return;
    const int64_t orow = tiled ? tiled_row(p / T, p % T, T) : p;
    for (int c = threadIdx.x; c < GI_COLS; c += 256) {
        float a = bias[c];
        for (int f = 0; f < F; ++f) a = fmaf(feats[p * F + f], w[c * F + f], a);
        if (tiled) gi[gi_quad_index(orow, c)] = a * gate_scale((c % G3) / H);
        else gi[orow * GI_COLS + c] = a;
    }
}

cudaError_t launch_inproj0(const float *feats, const float *w_packed, const float *bias, float *gi, int64_t P,
                           int F, int64_t T, int tiled, cudaStream_t s) {
    if (P == 0) return cudaSuccess;
    const unsigned blocks = (unsigned)((P + 63) / 64);
    if (F == 10) inproj0_kernel<10><<<blocks, 256, 0, s>>>(feats, w_packed, bias, gi, P, T, tiled);
    else if (F == 20) inproj0_kernel<20><<<blocks, 256, 0, s>>>(feats, w_packed, bias, gi, P, T, tiled);
    else inproj0_generic_kernel<<<(unsigned)P, 256, 0, s>>>(feats, w_packed, bias, gi, P, F, T, tiled);
    return cudaGetLastError();
}

// =====================================================================================
// Head: logits = h1 . W^T + b (gru.py:67), probs = softmax (gru.py:71), label = argmax (labels.py:1063)
// One warp per position, 8 of the 256 inputs per lane; 1 KiB read + 41 B written per position.
// =====================================================================================
// Outputs always go to position p = w*T + t; on the tensor-core path the h1 row of that position is the
// tile-interleaved row(w, t).  Each warp handles 4 positions per iteration: 8 of the 256 inputs per lane, the
// 4 x 5 (padded to 4 x 8) partial dot products are reduced with a transposing butterfly (31 shuffles for all 32
// values instead of 5 per value), after which lane L owns logit (position L/8, class L%8) and the softmax / argmax
// run across the 8-lane groups - one expf per lane instead of five per lane.
__global__ void __launch_bounds__(256) head_kernel(const float *__restrict__ h1, const float *__restrict__ lin_w,
                                                   const float *__restrict__ lin_b, int64_t P, int64_t B, int64_t T,
                                                   int tiled, float *__restrict__ probs, float *__restrict__ logits,
                                                   uint8_t *__restrict__ labels) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    float w[NCLS][8];
#pragma unroll
    for (int c = 0; c < NCLS; ++c) {
        const float4 a = *reinterpret_cast<const float4 *>(lin_w + c * H2 + lane * 8);
        const float4 b = *reinterpret_cast<const float4 *>(lin_w + c * H2 + lane * 8 + 4);
        w[c][0] = a.x; w[c][1] = a.y; w[c][2] = a.z; w[c][3] = a.w;
        w[c][4] = b.x; w[c][5] = b.y; w[c][6] = b.z; w[c][7] = b.w;
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
        float4 va[PU], vb[PU];
#pragma unroll
        for (int u = 0; u < PU; ++u) {
            const int64_t r = min(rb + u, rows - 1);
            va[u] = ld_stream4(h1 + r * H2 + lane * 8);
            vb[u] = ld_stream4(h1 + r * H2 + lane * 8 + 4);
        }
        float v[32];
#pragma unroll
        for (int u = 0; u < PU; ++u) {
            const float x[8] = {va[u].x, va[u].y, va[u].z, va[u].w, vb[u].x, vb[u].y, vb[u].z, vb[u].w};
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                float s = 0.f;
                if (c < NCLS) {
#pragma unroll
                    for (int i = 0; i < 8; ++i) s = fmaf(x[i], w[c][i], s);
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
        if (ok) {
            if (cls < NCLS) {
                probs[p * NCLS + cls] = pr;
                if (logits) logits[p * NCLS + cls] = logit;
            }
            if (labels && cls == 0) labels[p] = (uint8_t)arg;
        }
    }
}

cudaError_t launch_head(const float *h1, const float *lin_w, const float *lin_b, int64_t B, int64_t T, int tiled,
                        float *probs, float *logits, uint8_t *labels, cudaStream_t s) {
    const int64_t P = B * T;
    if (P == 0) return cudaSuccess;
    int64_t blocks = (P + 31) / 32;            // 8 warps per block, 4 positions per warp per iteration
    if (blocks > 132 * 8) blocks = 132 * 8;    // persistent-ish grid: multiple of the SM count
    head_kernel<<<(unsigned)blocks, 256, 0, s>>>(h1, lin_w, lin_b, P, B, T, tiled, probs, logits, labels);
    return cudaGetLastError();
}

// =====================================================================================
// Weight packing (runs once per load_state_dict)
// =====================================================================================
__global__ void pack_layer_kernel(const float *w_ih0, const float *w_ih1, const float *w_hh0, const float *w_hh1,
                                  const float *b_ih0, const float *b_ih1, const float *b_hh0, const float *b_hh1,
                                  int in_features, float *w_in_packed, float *bias_gi, float *b_hn, float *w_hh_t,
                                  __half *w_hh_tm, __half *w_x_tm, __half *w_in_tc, float *bias_gi_tc, float *b_hn_tc) {
    const int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    const float *w_ih[2] = {w_ih0, w_ih1}, *w_hh[2] = {w_hh0, w_hh1};
    const float *b_ih[2] = {b_ih0, b_ih1}, *b_hh[2] = {b_hh0, b_hh1};
    // input weights packed [768][in]
    for (int64_t i = tid; i < (int64_t)GI_COLS * in_features; i += stride) {
        const int row = (int)(i / in_features), k = (int)(i % in_features);
        const int d = row / G3, r = row % G3;
        w_in_packed[i] = w_ih[d][(int64_t)r * in_features + k];
    }
    for (int64_t i = tid; i < GI_COLS; i += stride) {
        const int d = (int)i / G3, r = (int)i % G3;
        bias_gi[i] = (r < 2 * H) ? (b_ih[d][r] + b_hh[d][r]) : b_ih[d][r];
        bias_gi_tc[i] = bias_gi[i] * gate_scale(r / H);
    }
    for (int64_t i = tid; i < NDIR * H; i += stride) {
        const int d = (int)i / H, j = (int)i % H;
        b_hn[i] = b_hh[d][2 * H + j];
        b_hn_tc[i] = b_hn[i] * GATE_SCALE_N;
    }
    // recurrent weights, transposed fp32 [d][k][384] and fp16 hi/lo blocks [d][part][gate][kg][row][8]
    for (int64_t i = tid; i < (int64_t)NDIR * G3 * H; i += stride) {
        const int d = (int)(i / (G3 * H));
        const int rem = (int)(i % (G3 * H));
        const int c = rem / H, k = rem % H;          // c = gate row, k = input unit
        const float v = w_hh[d][c * H + k];
        w_hh_t[((int64_t)d * H + k) * G3 + c] = v;
        const int g = c / H, j = c % H;
        __half hi, lo;
        split_f16(v * gate_scale(g), hi, lo);
        const int64_t blk_halfs = (int64_t)H * H;   // 128x128 block
        w_hh_tm[(((int64_t)d * 2 + 0) * 3 + g) * blk_halfs + j * H + k] = hi;
        w_hh_tm[(((int64_t)d * 2 + 1) * 3 + g) * blk_halfs + j * H + k] = lo;
    }
    if (w_x_tm) {   // layer 0, in_features <= 16: [d][part][gate][row j][16], K zero-padded
        for (int64_t i = tid; i < (int64_t)NDIR * G3 * 16; i += stride) {
            const int d = (int)(i / (G3 * 16));
            const int rem = (int)(i % (G3 * 16));
            const int c = rem / 16, k = rem % 16;
            const float v = (k < in_features) ? w_ih[d][(int64_t)c * in_features + k] : 0.f;
            const int g = c / H, j = c % H;
            __half hi, lo;
            split_f16(v * gate_scale(g), hi, lo);
            w_x_tm[((((int64_t)d * 2 + 0) * 3 + g) * H + j) * 16 + k] = hi;
            w_x_tm[((((int64_t)d * 2 + 1) * 3 + g) * H + j) * 16 + k] = lo;
        }
    }
    if (w_in_tc) {   // layer 1: [blk = dir*3+gate][part][row j][k] row-major
        for (int64_t i = tid; i < (int64_t)GI_COLS * H2; i += stride) {
            const int row = (int)(i / H2), k = (int)(i % H2);
            const int d = row / G3, r = row % G3;
            const float v = w_ih[d][(int64_t)r * H2 + k];
            __half hi, lo;
            split_f16(v * gate_scale(r / H), hi, lo);
            const int blk = row / H, j = row % H;
            const int64_t plane = (int64_t)H * H2;   // 128 x 256 halfs
            w_in_tc[((int64_t)blk * 2 + 0) * plane + (int64_t)j * H2 + k] = hi;
            w_in_tc[((int64_t)blk * 2 + 1) * plane + (int64_t)j * H2 + k] = lo;
        }
    }
}

cudaError_t launch_prepare_layer(const LayerWeights &lw, int in_features, bool build_in_tc, cudaStream_t s) {
    pack_layer_kernel<<<296, 256, 0, s>>>(lw.w_ih[0], lw.w_ih[1], lw.w_hh[0], lw.w_hh[1], lw.b_ih[0], lw.b_ih[1],
                                          lw.b_hh[0], lw.b_hh[1], in_features, lw.w_in_packed, lw.bias_gi,
                                          lw.b_hn, lw.w_hh_t, lw.w_hh_tm, lw.w_x_tm, build_in_tc ? lw.w_in_tc : nullptr,
                                          lw.bias_gi_tc, lw.b_hn_tc);
    return cudaGetLastError();
}

// Head of the fused path (gru.py:53-55,67-71): logits = fwd partial + rev partial + bias, softmax, first-max argmax.
// One thread per (window of the tile, time step); blockIdx.y = window tile.  41 B written per position, 40 B read.
__global__ void __launch_bounds__(256) head_plog_kernel(const float *__restrict__ plog, const float *__restrict__ lin_b,
                                                        int64_t B, int64_t T, int64_t n_ts, float *__restrict__ probs,
                                                        float *__restrict__ logits, uint8_t *__restrict__ labels) {
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
    float best = -1.f;
    int arg = 0;
#pragma unroll
    for (int c = 0; c < NCLS; ++c) {
        const float pr = e[c] / sum;
        probs[p * NCLS + c] = pr;
        if (logits) logits[p * NCLS + c] = lg[c];
        if (pr > best) { best = pr; arg = c; }     // first maximum wins (np.argmax, labels.py:1063)
    }
    if (labels) labels[p] = (uint8_t)arg;
}

cudaError_t launch_head_plog(const float *plog, const float *lin_b, int64_t B, int64_t T, float *probs, float *logits,
                             uint8_t *labels, cudaStream_t s) {
    if (B == 0 || T == 0) return cudaSuccess;
    const int64_t tiles = (B + WT - 1) / WT;
    dim3 grid((unsigned)((T * WT + 255) / 256), (unsigned)tiles);
    head_plog_kernel<<<grid, 256, 0, s>>>(plog, lin_b, B, T, tiles * T, probs, logits, labels);
    return cudaGetLastError();
}

// fp16 hi/lo activation tiles (tile-interleaved rows) -> fp32 [B*T][256] in position order (debug / layer-wise parity)
__global__ void unpack_h0_kernel(const __half *__restrict__ tiles, float *__restrict__ out, int64_t B, int64_t T) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= B * T * H2) return;
    const int64_t p = i / H2;
    const int k = (int)(i % H2);
    const int64_t row = tiled_row(p / T, p % T, T);
    const int64_t tile = row / XT_ROWS;
    const int r = (int)(row % XT_ROWS);
    const __half *base = tiles + tile * (XT_TILE_BYTES / 2);
    const int64_t off = (int64_t)(k / 8) * (XT_ROWS * 8) + r * 8 + (k % 8);
    out[i] = __half2float(base[off]) + __half2float(base[XT_PLANE_BYTES / 2 + off]);
}

cudaError_t launch_unpack_h0(const void *h0_tiles, float *out, int64_t B, int64_t T, cudaStream_t s) {
    const int64_t n = B * T * H2;
    if (n == 0) return cudaSuccess;
    unpack_h0_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(reinterpret_cast<const __half *>(h0_tiles), out, B, T);
    return cudaGetLastError();
}

// fp32 [rows'][256] in tile-interleaved order -> [B*T][256] in position order (debug / layer-wise parity)
__global__ void untile_rows_kernel(const float *__restrict__ src, float *__restrict__ dst, int64_t B, int64_t T) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= B * T * H2) return;
    const int64_t p = i / H2;
    dst[i] = src[tiled_row(p / T, p % T, T) * H2 + (i % H2)];
}

cudaError_t launch_untile_rows(const float *src_tiled, float *dst, int64_t B, int64_t T, cudaStream_t s) {
    const int64_t n = B * T * H2;
    if (n == 0) return cudaSuccess;
    untile_rows_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(src_tiled, dst, B, T);
    return cudaGetLastError();
}

}  // namespace mdk
