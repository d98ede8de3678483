// Training of the read-level LatentSpaceLSTM (medaka train with a LatentSpaceLSTM model dict): the mdk_rl_trainer
// object of include/medaka_b200.h.  fp32 on the CUDA cores throughout; BatchNorm normalises with batch statistics
// (model.train()), taken over all B*D*P elements of the padded batch, empty and padding reads included.  One step:
//   stats pass     embedding + k = 1 convolution + ReLU over every element: BN1's per-channel sum and sum of squares
//                  (rlt_conv1_stats_kernel), then mean, invstd and the running statistics (rlt_bn_stats_kernel)
//   forward pass   per slice of (window, read) rows: BN1's output rebuilt from the int8 features into the slice's
//                  scratch (rlt_y1_kernel), the k = 17 convolution + ReLU (rlt_conv17_kernel<FWD>): BN2's sums and the
//                  masked sum over reads per (window, position).  BN2 and pre_pool_expansion_layer are affine, so they
//                  apply to the pooled mean (rlt_pool_bn_kernel + gemm_fp32): no [B*D*P][C] tensor exists
//   LSTM           gemm_fp32 input projections, rl_lstm_fp32<SAVE> (readlevel.cu) keeping i, f, g, o, c per position
//   head           logits, cross-entropy (mean over B*P), dlogits, head backward (train_common.cuh)
//   BPTT           per layer, both directions (rlt_bptt_kernel); split-M weight / bias reductions; dX by gemm_fp32
//   read backward  BN2's two backward sums over (window, position) (rlt_bn2_sums_kernel); then per slice: y1 again,
//                  the convolution again with dpre2 = ReLU'-masked BN2 backward (rlt_conv17_kernel<BWD>), dW17 as 17
//                  shifted wgrad reductions, dy1 by the same convolution with the weights transposed and the taps
//                  flipped (<DGRAD>), and the per-channel sums that make BN1 -> ReLU -> conv1 -> embedding's backward
//                  linear (rlt_bn1_sums_kernel); rlt_bn1_final_kernel turns them into dW1, db1, dgamma1, dbeta1 and
//                  both embeddings' gradients
//   step           global norm, non-finite skip, clip, optimizer rule (train_common.cuh), weight repack on the device
// Every reduction adds partial sums in a fixed order (no float atomics): two identical steps give bit-identical
// gradients, weights and running statistics.  Device memory grows with B*P (and the int8 features), not with D: the
// per-read tensors live only in a scratch of at most RLT_SCRATCH bytes.
#include <cmath>
#include <cstring>
#include <new>
#include <string>
#include <vector>

#include "rl_common.cuh"
#include "train_common.cuh"

namespace mdk {
namespace {

constexpr int RLT_NQ = 56;                           // BN1 backward sums per channel (rlt_bn1_sums_kernel)
constexpr size_t RLT_SCRATCH = (size_t)2 << 30;      // per-read scratch of one slice (y1 and dpre2), bytes
constexpr int64_t RLT_WS_BUDGET = (int64_t)64 << 30;
constexpr double BN_EPS = 1e-5, BN_MOMENTUM = 0.1;

// the k = 1 convolution's input at one element: base and strand embeddings, q / 25 - 1, dwell (as the engine reads it)
__device__ __forceinline__ void rlt_inputs(const int8_t *v, const float *emb_base, const float *emb_strand,
                                           int use_dwells, float *in, int &base, int &strand) {
    base = min(max((int)v[0], 0), 5);
    strand = min(max((int)v[2] + 1, 0), 2);
    for (int i = 0; i < RL_EMB; ++i) in[i] = emb_base[base * RL_EMB + i] + emb_strand[strand * RL_EMB + i];
    in[RL_EMB] = (float)v[1] / 25.0f - 1.0f;
    in[RL_EMB + 1] = use_dwells ? (float)v[4] : 0.f;
}

struct RltIn {
    const int8_t *x;          // [B][P][D][F]
    const float *emb_base, *emb_strand, *w1, *b1;
    int64_t P;
    int D, F, use_dwells;
};

// element e = row * P + p of the (window, read) rows: its feature vector
__device__ __forceinline__ const int8_t *rlt_x(const RltIn &a, int64_t row, int64_t p) {
    const int64_t b = row / a.D, d = row % a.D;
    return a.x + ((b * a.P + p) * a.D + d) * a.F;
}

// BN1's statistics: per-block sums of ReLU(conv1) and its square over elements [0, n) in chunks of 32
__global__ void __launch_bounds__(RL_C) rlt_conv1_stats_kernel(RltIn a, int64_t n, double *__restrict__ part) {
    const int c = threadIdx.x, nin = RL_EMB + 1 + (a.use_dwells ? 1 : 0);
    __shared__ float in[32][RL_EMB + 2];
    float w[RL_EMB + 2];
    for (int k = 0; k < nin; ++k) w[k] = a.w1[c * nin + k];
    const float bias = a.b1[c];
    double s = 0.0, ss = 0.0;
    for (int64_t q = blockIdx.x; q * 32 < n; q += gridDim.x) {
        __syncthreads();
        if (c < 32 && q * 32 + c < n) {
            const int64_t e = q * 32 + c;
            int base, strand;
            rlt_inputs(rlt_x(a, e / a.P, e % a.P), a.emb_base, a.emb_strand, a.use_dwells, in[c], base, strand);
        }
        __syncthreads();
        const int m = (int)min((int64_t)32, n - q * 32);
        for (int i = 0; i < m; ++i) {
            float acc = bias;
            for (int k = 0; k < nin; ++k) acc = fmaf(w[k], in[i][k], acc);
            const double r = fmaxf(acc, 0.f);
            s += r;
            ss += r * r;
        }
    }
    part[(int64_t)blockIdx.x * 2 * RL_C + c] = s;
    part[(int64_t)blockIdx.x * 2 * RL_C + RL_C + c] = ss;
}

// tot[i] += sum_j part[j * n + i], j in order
__global__ void __launch_bounds__(256) rlt_accum_kernel(const double *__restrict__ part, int64_t nparts, int n,
                                                        double *__restrict__ tot) {
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    double s = 0.0;
    for (int64_t j = 0; j < nparts; ++j) s += part[j * n + i];
    tot[i] += s;
}

// dst[e] += sum_s part[s][e] in order s = 0, 1, ...
__global__ void __launch_bounds__(256) rlt_accum_partials_kernel(const float *__restrict__ part, int splits,
                                                                 int64_t count, float *__restrict__ dst) {
    const int64_t e = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (e >= count) return;
    float s = 0.f;
    for (int i = 0; i < splits; ++i) s += part[(int64_t)i * count + e];
    dst[e] += s;
}

// Batch statistics from the sums tot [2][C] over N elements: mean, 1 / sqrt(biased var + eps); the running statistics
// move by momentum 0.1 towards the mean and the unbiased variance
__global__ void rlt_bn_stats_kernel(const double *__restrict__ tot, double N, float *__restrict__ mean,
                                    float *__restrict__ invstd, float *__restrict__ run_mean, float *__restrict__ run_var) {
    const int c = threadIdx.x;
    const double m = tot[c] / N;
    const double var = fmax(tot[RL_C + c] / N - m * m, 0.0);
    mean[c] = (float)m;
    invstd[c] = (float)(1.0 / sqrt(var + BN_EPS));
    run_mean[c] = (float)((1.0 - BN_MOMENTUM) * (double)run_mean[c] + BN_MOMENTUM * m);
    const double unbiased = N > 1.0 ? var * N / (N - 1.0) : NAN;
    run_var[c] = (float)((1.0 - BN_MOMENTUM) * (double)run_var[c] + BN_MOMENTUM * unbiased);
}

// inference BatchNorm's invstd from the running variance, as the engine computes it
__global__ void rlt_invstd_kernel(const float *__restrict__ var, float *__restrict__ invstd) {
    invstd[threadIdx.x] = 1.0f / sqrtf(var[threadIdx.x] + 1e-5f);
}

// reads[b] = non-empty reads of window b, inv_n[b] = 1 / reads (inf for none: the window's mean is NaN, as the reference's)
__global__ void rlt_reads_kernel(const uint8_t *__restrict__ mask, int64_t B, int D, float *__restrict__ reads) {
    const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    int n = 0;
    for (int d = 0; d < D; ++d) n += mask[b * D + d];
    reads[b] = (float)n;
}

// y1 = BN1(ReLU(conv1(inputs))) with the batch statistics, rows r0 .. r0 + gridDim.y - 1 -> y1 [row - r0][P][C]
__global__ void __launch_bounds__(RL_C) rlt_y1_kernel(RltIn a, const float *__restrict__ mean, const float *__restrict__ invstd,
                                                      const float *__restrict__ gamma, const float *__restrict__ beta,
                                                      int64_t r0, float *__restrict__ y1) {
    const int c = threadIdx.x, nin = RL_EMB + 1 + (a.use_dwells ? 1 : 0);
    const int64_t row = r0 + blockIdx.y, p0 = (int64_t)blockIdx.x * 32;
    float w[RL_EMB + 2];
    for (int k = 0; k < nin; ++k) w[k] = a.w1[c * nin + k];
    const float bias = a.b1[c], mu = mean[c], is = invstd[c], g = gamma[c], bt = beta[c];
    __shared__ float in[32][RL_EMB + 2];
    if (c < 32 && p0 + c < a.P) {
        int base, strand;
        rlt_inputs(rlt_x(a, row, p0 + c), a.emb_base, a.emb_strand, a.use_dwells, in[c], base, strand);
    }
    __syncthreads();
    for (int i = 0; i < 32 && p0 + i < a.P; ++i) {
        float acc = bias;
        for (int k = 0; k < nin; ++k) acc = fmaf(w[k], in[i][k], acc);
        acc = fmaxf(acc, 0.f);
        y1[((int64_t)blockIdx.y * a.P + p0 + i) * RL_C + c] = (acc - mu) * is * g + bt;
    }
}

// The k = 17 convolution (zero padding 8) over the scratch rows of one slice, rl_conv17_pool_kernel's tiling: a CTA
// owns 64 positions x 128 output channels, 256 threads with 4 x 8 accumulators.  out[p][co] = sum_t sum_ci
// in[p + t - 8][ci] w_t[t][ci][co].  Modes:
//   FWD    in = y1; r2 = ReLU(out + b17): the masked sum over the window's reads into pooled[b][p] and per-CTA sums of r2
//          and r2^2 (BN2's statistics); grid.y = windows the slice touches
//   BWD    in = y1; dpre2 = [out + b17 > 0] k2 (mask du[b][p] / reads - A2 - xhat2 B2) into out_rows, per-CTA sums of
//          dpre2 (db17); grid.y = rows
//   DGRAD  in = dpre2, w_t = the weights transposed with the taps flipped: dy1 into out_rows; grid.y = rows
enum { CV_FWD = 0, CV_BWD = 1, CV_DGRAD = 2 };
constexpr int CV_PT = 64;
constexpr int CV_ROWS = CV_PT + 2 * RL_PAD;
constexpr int CV_YS = RL_C + 4;
constexpr int CV_KC = 32;
constexpr int CV_SMEM = (CV_ROWS * CV_YS + CV_KC * RL_C) * 4;

struct RltConv {
    const float *in;          // [rows][P][C]
    const float *w_t;         // [17][C in][C out]
    const float *bias;        // [C]
    const uint8_t *mask;      // [B * D]
    int64_t r0, r1, P;
    int D;
    float *pooled;            // FWD: [B][P][C]
    const float *du, *reads;  // BWD: [B][P][C], [B]
    const float *coef;        // BWD: [5][C] k2, A2, B2, mean2, invstd2
    float *out;               // BWD, DGRAD: [rows][P][C]
    double *part;             // FWD: [cta][2][C]; BWD: [cta][C]
};

template <int MODE>
__global__ void __launch_bounds__(256) rlt_conv17_kernel(RltConv a) {
    extern __shared__ __align__(16) float smem_cv[];
    float *ys = smem_cv;
    float *ws = smem_cv + CV_ROWS * CV_YS;
    const int tid = threadIdx.x;
    const int tx = tid % 16, ty = tid / 16;
    const int64_t p0 = (int64_t)blockIdx.x * CV_PT;
    int64_t row_lo, row_hi;
    if (MODE == CV_FWD) {
        const int64_t b = a.r0 / a.D + blockIdx.y;
        row_lo = max(a.r0, b * a.D);
        row_hi = min(a.r1, (b + 1) * a.D);
    } else {
        row_lo = a.r0 + blockIdx.y;
        row_hi = row_lo + 1;
    }
    float bias[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) bias[j] = MODE == CV_DGRAD ? 0.f : a.bias[tx * 8 + j];
    float pooled[4][8];
    double s[8], ss[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        s[j] = ss[j] = 0.0;
#pragma unroll
        for (int i = 0; i < 4; ++i) pooled[i][j] = 0.f;
    }
    for (int64_t row = row_lo; row < row_hi; ++row) {
        const int64_t sr = row - a.r0;
        __syncthreads();
        for (int i = tid; i < CV_ROWS * (RL_C / 4); i += 256) {
            const int r = i / (RL_C / 4), q = i % (RL_C / 4);
            const int64_t p = p0 - RL_PAD + r;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (p >= 0 && p < a.P) v = *reinterpret_cast<const float4 *>(a.in + (sr * a.P + p) * RL_C + q * 4);
            *reinterpret_cast<float4 *>(ys + r * CV_YS + q * 4) = v;
        }
        float acc[4][8];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
        for (int t = 0; t < RL_TAPS; ++t) {
            for (int cc = 0; cc < RL_C / CV_KC; ++cc) {
                __syncthreads();
                const float *wsrc = a.w_t + ((size_t)t * RL_C + cc * CV_KC) * RL_C;
                for (int i = tid; i < CV_KC * RL_C / 4; i += 256)
                    reinterpret_cast<float4 *>(ws)[i] = reinterpret_cast<const float4 *>(wsrc)[i];
                __syncthreads();
#pragma unroll 4
                for (int k = 0; k < CV_KC; ++k) {
                    float av[4];
#pragma unroll
                    for (int i = 0; i < 4; ++i) av[i] = ys[(ty * 4 + i + t) * CV_YS + cc * CV_KC + k];
                    const float4 b0 = *reinterpret_cast<const float4 *>(ws + k * RL_C + tx * 8);
                    const float4 b1 = *reinterpret_cast<const float4 *>(ws + k * RL_C + tx * 8 + 4);
                    const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
                    for (int i = 0; i < 4; ++i)
#pragma unroll
                        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
                }
            }
        }
        const bool keep = a.mask[row] != 0;
        const int64_t b = row / a.D;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int64_t p = p0 + ty * 4 + i;
            if (p >= a.P) continue;
            float o[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int c = tx * 8 + j;
                const float v = acc[i][j] + bias[j];
                if (MODE == CV_FWD) {
                    const float r = fmaxf(v, 0.f);
                    if (keep) pooled[i][j] += r;
                    s[j] += r;
                    ss[j] += (double)r * r;
                } else if (MODE == CV_BWD) {
                    float d = 0.f;
                    if (v > 0.f) {
                        const float dout = keep ? a.du[(b * a.P + p) * RL_C + c] / a.reads[b] : 0.f;
                        const float xh = (v - a.coef[3 * RL_C + c]) * a.coef[4 * RL_C + c];
                        d = a.coef[c] * (dout - a.coef[RL_C + c] - xh * a.coef[2 * RL_C + c]);
                    }
                    o[j] = d;
                    s[j] += d;
                } else {
                    o[j] = v;
                }
            }
            if (MODE != CV_FWD) {
                float *dst = a.out + (sr * a.P + p) * RL_C + tx * 8;
                *reinterpret_cast<float4 *>(dst) = make_float4(o[0], o[1], o[2], o[3]);
                *reinterpret_cast<float4 *>(dst + 4) = make_float4(o[4], o[5], o[6], o[7]);
            }
        }
    }
    if (MODE == CV_DGRAD) return;
    if (MODE == CV_FWD) {
        const int64_t b = a.r0 / a.D + blockIdx.y;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int64_t p = p0 + ty * 4 + i;
            if (p >= a.P) continue;
            float *dst = a.pooled + (b * a.P + p) * RL_C + tx * 8;
#pragma unroll
            for (int j = 0; j < 8; ++j) dst[j] += pooled[i][j];
        }
    }
    // per-CTA channel sums: the 16 position groups in order
    __syncthreads();
    double *red = reinterpret_cast<double *>(smem_cv);       // [2][16][C]
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        red[ty * RL_C + tx * 8 + j] = s[j];
        red[16 * RL_C + ty * RL_C + tx * 8 + j] = ss[j];
    }
    __syncthreads();
    const int64_t cta = (int64_t)blockIdx.y * gridDim.x + blockIdx.x;
    constexpr int NQ = MODE == CV_FWD ? 2 : 1;
    if (tid < NQ * RL_C) {
        const int q = tid / RL_C, c = tid % RL_C;
        double v = 0.0;
        for (int g = 0; g < 16; ++g) v += red[(q * 16 + g) * RL_C + c];
        a.part[(cta * NQ + q) * RL_C + c] = v;
    }
}

// u = BN2(pooled / reads) per (window, position): the pooled mean of BN2's output (BN2 is affine)
__global__ void __launch_bounds__(256) rlt_pool_bn_kernel(const float *__restrict__ pooled, const float *__restrict__ reads,
                                                          const float *__restrict__ mean, const float *__restrict__ invstd,
                                                          const float *__restrict__ gamma, const float *__restrict__ beta,
                                                          int64_t BP, int64_t P, float *__restrict__ u) {
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < BP * RL_C; i += (int64_t)gridDim.x * 256) {
        const int c = (int)(i % RL_C);
        const int64_t b = i / RL_C / P;
        u[i] = (pooled[i] / reads[b] - mean[c]) * invstd[c] * gamma[c] + beta[c];
    }
}

// BN2's backward sums over (window, position): sum du and sum du xhat2(pooled), per-block partials [blk][2][C]
__global__ void __launch_bounds__(RL_C) rlt_bn2_sums_kernel(const float *__restrict__ du, const float *__restrict__ pooled,
                                                            const float *__restrict__ reads, const float *__restrict__ mean,
                                                            const float *__restrict__ invstd, int64_t BP, int64_t P,
                                                            double *__restrict__ part) {
    const int c = threadIdx.x;
    double s = 0.0, sx = 0.0;
    for (int64_t m = blockIdx.x; m < BP; m += gridDim.x) {
        const float g = du[m * RL_C + c];
        const float xh = (pooled[m * RL_C + c] / reads[m / P] - mean[c]) * invstd[c];
        s += g;
        sx += (double)g * xh;
    }
    part[(int64_t)blockIdx.x * 2 * RL_C + c] = s;
    part[(int64_t)blockIdx.x * 2 * RL_C + RL_C + c] = sx;
}

// BatchNorm backward from tot [2][C] = (sum dout, sum dout xhat) over N elements: dbeta, dgamma into the gradient and
// the per-channel coefficients of dx = k (dout - A - xhat B): coef [5][C] = k = gamma invstd, A, B, mean, invstd
__global__ void rlt_bn_coef_kernel(const double *__restrict__ tot, double N, const float *__restrict__ gamma,
                                   const float *__restrict__ mean, const float *__restrict__ invstd,
                                   float *__restrict__ coef, float *__restrict__ dgamma, float *__restrict__ dbeta) {
    const int c = threadIdx.x;
    dbeta[c] = (float)tot[c];
    dgamma[c] = (float)tot[RL_C + c];
    coef[c] = gamma[c] * invstd[c];
    coef[RL_C + c] = (float)(tot[c] / N);
    coef[2 * RL_C + c] = (float)(tot[RL_C + c] / N);
    coef[3 * RL_C + c] = mean[c];
    coef[4 * RL_C + c] = invstd[c];
}

// The sums that make BN1 -> ReLU -> conv1 -> embeddings' backward linear in dout1 = dy1, over the slice's elements:
// per channel [0] sum dout, [1] sum dout xhat1, and with m = [conv1 pre-activation > 0]
//   [2 + k], [11 + k], [20 + k]   sum m dout in_k, sum m in_k, sum m xhat1 in_k  (k < 8 the inputs, k = 8 the bias)
//   [29 + v], [35 + v], [41 + v]  the same three with in = [base == v]
//   [47 + v], [50 + v], [53 + v]  the same three with in = [strand index == v]
// per-block partials [blk][56][C]
__global__ void __launch_bounds__(RL_C) rlt_bn1_sums_kernel(RltIn a, const float *__restrict__ mean,
                                                            const float *__restrict__ invstd, const float *__restrict__ dy1,
                                                            int64_t r0, int64_t n, double *__restrict__ part) {
    const int c = threadIdx.x, nin = RL_EMB + 1 + (a.use_dwells ? 1 : 0);
    __shared__ float in[32][RL_EMB + 2];
    __shared__ int bs[32][2];
    float w[RL_EMB + 2];
    for (int k = 0; k < RL_EMB + 2; ++k) w[k] = k < nin ? a.w1[c * nin + k] : 0.f;
    const float bias = a.b1[c], mu = mean[c], is = invstd[c];
    double acc[RLT_NQ];
#pragma unroll
    for (int q = 0; q < RLT_NQ; ++q) acc[q] = 0.0;
    for (int64_t q0 = blockIdx.x; q0 * 32 < n; q0 += gridDim.x) {
        __syncthreads();
        if (c < 32 && q0 * 32 + c < n) {
            const int64_t e = q0 * 32 + c;
            rlt_inputs(rlt_x(a, r0 + e / a.P, e % a.P), a.emb_base, a.emb_strand, a.use_dwells, in[c], bs[c][0], bs[c][1]);
        }
        __syncthreads();
        const int cnt = (int)min((int64_t)32, n - q0 * 32);
        for (int i = 0; i < cnt; ++i) {
            float pre = bias;
            for (int k = 0; k < nin; ++k) pre = fmaf(w[k], in[i][k], pre);
            const float xh = (fmaxf(pre, 0.f) - mu) * is;
            const double g = dy1[(q0 * 32 + i) * RL_C + c];
            acc[0] += g;
            acc[1] += g * xh;
            if (pre > 0.f) {
#pragma unroll
                for (int k = 0; k < RL_EMB + 2; ++k) {
                    const double v = in[i][k];
                    acc[2 + k] += g * v;
                    acc[11 + k] += v;
                    acc[20 + k] += xh * v;
                }
                acc[10] += g;
                acc[19] += 1.0;
                acc[28] += xh;
                const int base = bs[i][0], strand = bs[i][1];
#pragma unroll
                for (int v = 0; v < 6; ++v)
                    if (base == v) { acc[29 + v] += g; acc[35 + v] += 1.0; acc[41 + v] += xh; }
#pragma unroll
                for (int v = 0; v < 3; ++v)
                    if (strand == v) { acc[47 + v] += g; acc[50 + v] += 1.0; acc[53 + v] += xh; }
            }
        }
    }
#pragma unroll
    for (int q = 0; q < RLT_NQ; ++q) part[((int64_t)blockIdx.x * RLT_NQ + q) * RL_C + c] = acc[q];
}

// BN1's, conv1's and the embeddings' gradients from rlt_bn1_sums_kernel's totals (dx = k (dout - A - xhat B))
struct RltBn1Grads {
    float *dw1, *db1, *dgamma, *dbeta, *demb_base, *demb_strand;
};
__global__ void rlt_bn1_final_kernel(const double *__restrict__ tot, double N, const float *__restrict__ gamma,
                                     const float *__restrict__ invstd, const float *__restrict__ w1, int nin, RltBn1Grads g) {
    __shared__ double qb[9][RL_C];                 // per (base 0-5 | strand 0-2, channel): sum of dpre1
    const int c = threadIdx.x;
    auto T = [&](int q) { return tot[q * RL_C + c]; };
    const double A = T(0) / N, Bc = T(1) / N, k = (double)gamma[c] * invstd[c];
    g.dbeta[c] = (float)T(0);
    g.dgamma[c] = (float)T(1);
    for (int i = 0; i < nin; ++i) g.dw1[c * nin + i] = (float)(k * (T(2 + i) - A * T(11 + i) - Bc * T(20 + i)));
    g.db1[c] = (float)(k * (T(10) - A * T(19) - Bc * T(28)));
    for (int v = 0; v < 6; ++v) qb[v][c] = k * (T(29 + v) - A * T(35 + v) - Bc * T(41 + v));
    for (int v = 0; v < 3; ++v) qb[6 + v][c] = k * (T(47 + v) - A * T(50 + v) - Bc * T(53 + v));
    __syncthreads();
    if (c < 9 * RL_EMB) {
        const int v = c / RL_EMB, i = c % RL_EMB;
        double s = 0.0;
        for (int ch = 0; ch < RL_C; ++ch) s += qb[v][ch] * w1[ch * nin + i];
        if (v < 6) g.demb_base[v * RL_EMB + i] = (float)s;
        else g.demb_strand[(v - 6) * RL_EMB + i] = (float)s;
    }
}

// logits [n][5] = h1 [n][K2] . W^T + b, one warp per position (the loss's logits at lstm_size 384)
__global__ void __launch_bounds__(256) rlt_logits_kernel(const float *__restrict__ h1, const float *__restrict__ w,
                                                         const float *__restrict__ b, int64_t n, int K2,
                                                         float *__restrict__ logits) {
    const int lane = threadIdx.x & 31;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t p = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; p < n; p += nwarps) {
        float s[NCLS];
#pragma unroll
        for (int c = 0; c < NCLS; ++c) s[c] = 0.f;
        for (int k = lane; k < K2; k += 32) {
            const float x = h1[p * K2 + k];
#pragma unroll
            for (int c = 0; c < NCLS; ++c) s[c] = fmaf(x, w[c * K2 + k], s[c]);
        }
#pragma unroll
        for (int c = 0; c < NCLS; ++c)
#pragma unroll
            for (int m = 16; m >= 1; m >>= 1) s[c] += __shfl_xor_sync(0xffffffffu, s[c], m);
        if (lane < NCLS) {
            float v = s[0];
#pragma unroll
            for (int c = 1; c < NCLS; ++c) if (lane == c) v = s[c];
            logits[p * NCLS + lane] = v + b[lane];
        }
    }
}

// LSTM BPTT of one layer, both directions (blockIdx.y), NB windows per CTA, thread j = hidden unit j.  Walks the
// positions in the reverse of the direction's forward order; per step, with dh = dh_out + carry_h:
//   do = dh tanh(c) o (1 - o)      dc = dh o (1 - tanh^2 c) + carry_c
//   di = dc g i (1 - i)            df = dc c_prev f (1 - f)      dg = dc i (1 - g^2)
//   carry_c = dc f                 carry_h = W_hh^T [di, df, dg, do]
// and writes the pre-activation gradients over gi [B*P][2][4H].  W_hh (torch layout [4H][H]: thread j reads column
// j) streams from L2 as in the forward twin; the NB gate-gradient vectors are shared-memory broadcasts.
template <int HS, int NB>
__global__ void __launch_bounds__(HS, 1) rlt_bptt_kernel(const float *__restrict__ save, const float *__restrict__ dh_out,
                                                         const float *__restrict__ w_hh0, const float *__restrict__ w_hh1,
                                                         float *__restrict__ dgi, int64_t B, int64_t P) {
    constexpr int G4 = 4 * HS;
    extern __shared__ __align__(16) float gsm[];        // [2][NB][4 HS]
    const int j = threadIdx.x, dir = blockIdx.y;
    const int64_t b0 = (int64_t)blockIdx.x * NB;
    const int nb = (int)min((int64_t)NB, B - b0);
    const float *w = dir ? w_hh1 : w_hh0;
    float carry_h[NB], carry_c[NB];
#pragma unroll
    for (int n = 0; n < NB; ++n) carry_h[n] = carry_c[n] = 0.f;
    int cur = 0;
    for (int64_t step = 0; step < P; ++step) {
        const int64_t t = dir ? step : P - 1 - step;
        const int64_t tp = dir ? t + 1 : t - 1;          // the previous position in the forward order
        const bool has_prev = tp >= 0 && tp < P;
        float *g = gsm + cur * NB * G4;
#pragma unroll
        for (int n = 0; n < NB; ++n) {
            float di = 0.f, df = 0.f, dg = 0.f, dout = 0.f;
            if (n < nb) {
                const int64_t pos = (b0 + n) * P + t;
                const float *sv = save + (pos * 2 + dir) * (5 * HS) + j;
                const float ig = sv[0], fg = sv[HS], gg = sv[2 * HS], og = sv[3 * HS], c = sv[4 * HS];
                const float cp = has_prev ? save[(((b0 + n) * P + tp) * 2 + dir) * (5 * HS) + 4 * HS + j] : 0.f;
                const float dh = dh_out[pos * (2 * HS) + dir * HS + j] + carry_h[n];
                const float tc = tanhf(c);
                dout = dh * tc * og * (1.f - og);
                const float dc = dh * og * (1.f - tc * tc) + carry_c[n];
                di = dc * gg * ig * (1.f - ig);
                df = dc * cp * fg * (1.f - fg);
                dg = dc * ig * (1.f - gg * gg);
                carry_c[n] = dc * fg;
                float *o = dgi + (pos * 2 + dir) * G4 + j;
                o[0] = di; o[HS] = df; o[2 * HS] = dg; o[3 * HS] = dout;
            }
            g[n * G4 + j] = di;
            g[n * G4 + HS + j] = df;
            g[n * G4 + 2 * HS + j] = dg;
            g[n * G4 + 3 * HS + j] = dout;
        }
        __syncthreads();
        float acc[NB];
#pragma unroll
        for (int n = 0; n < NB; ++n) acc[n] = 0.f;
#pragma unroll 2
        for (int r = 0; r < G4; r += 4) {
            float4 gv[NB];
#pragma unroll
            for (int n = 0; n < NB; ++n) gv[n] = *reinterpret_cast<const float4 *>(g + n * G4 + r);
#pragma unroll
            for (int rr = 0; rr < 4; ++rr) {
                const float wv = __ldg(w + (size_t)(r + rr) * HS + j);
#pragma unroll
                for (int n = 0; n < NB; ++n) {
                    const float gk = rr == 0 ? gv[n].x : rr == 1 ? gv[n].y : rr == 2 ? gv[n].z : gv[n].w;
                    acc[n] = fmaf(wv, gk, acc[n]);
                }
            }
        }
#pragma unroll
        for (int n = 0; n < NB; ++n) carry_h[n] = acc[n];
        cur ^= 1;
    }
}

// torch's conv weight [co][ci][17] -> the convolution's w_t [17][ci][co] and dgrad's [17][co][ci] with the taps flipped
__global__ void __launch_bounds__(256) rlt_w17_pack_kernel(const float *__restrict__ w, float *__restrict__ w_t,
                                                           float *__restrict__ w_dg) {
    const int64_t e = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (e >= (int64_t)RL_C * RL_C * RL_TAPS) return;
    const int t = (int)(e % RL_TAPS), ci = (int)(e / RL_TAPS % RL_C), co = (int)(e / RL_TAPS / RL_C);
    const float v = w[e];
    w_t[((int64_t)t * RL_C + ci) * RL_C + co] = v;
    w_dg[((int64_t)(RL_TAPS - 1 - t) * RL_C + co) * RL_C + ci] = v;
}

// dW17 [co][ci][17] from the per-tap reductions tmp [17][co][ci]
__global__ void __launch_bounds__(256) rlt_w17_grad_kernel(const float *__restrict__ tmp, float *__restrict__ g) {
    const int64_t e = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (e >= (int64_t)RL_C * RL_C * RL_TAPS) return;
    const int t = (int)(e % RL_TAPS), ci = (int)(e / RL_TAPS % RL_C), co = (int)(e / RL_TAPS / RL_C);
    g[e] = tmp[((int64_t)t * RL_C + co) * RL_C + ci];
}

__global__ void __launch_bounds__(256) rlt_add_kernel(const float *__restrict__ a, const float *__restrict__ b,
                                                      float *__restrict__ out, int n) {
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i < n) out[i] = a[i] + b[i];
}

__global__ void __launch_bounds__(256) rlt_to_float_kernel(const double *__restrict__ a, float *__restrict__ out, int n) {
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i < n) out[i] = (float)a[i];
}

// ---------------------------------------------------------------------------------------------------- host side
// The flat parameter array: named_parameters() order of LatentSpaceLSTM
struct RlParams {
    std::vector<std::string> names;
    std::vector<int64_t> off, size;
    int64_t total = 0;
    int64_t at(const std::string &n) const {
        for (size_t i = 0; i < names.size(); ++i)
            if (names[i] == n) return off[i];
        return -1;
    }
    void add(const std::string &n, int64_t k) { names.push_back(n); off.push_back(total); size.push_back(k); total += k; }
    RlParams() = default;
    RlParams(int H, int nin) {
        const int C = RL_C;
        add("base_embedder.weight", 6 * RL_EMB);
        add("strand_embedder.weight", 3 * RL_EMB);
        add("read_level_conv.convs.0.weight", (int64_t)C * nin);
        add("read_level_conv.convs.0.bias", C);
        add("read_level_conv.convs.2.weight", C);
        add("read_level_conv.convs.2.bias", C);
        add("read_level_conv.convs.3.weight", (int64_t)C * C * RL_TAPS);
        add("read_level_conv.convs.3.bias", C);
        add("read_level_conv.convs.5.weight", C);
        add("read_level_conv.convs.5.bias", C);
        add("read_level_conv.expansion_layer.weight", (int64_t)H * C);
        add("read_level_conv.expansion_layer.bias", H);
        add("pre_pool_expansion_layer.weight", (int64_t)H * C);
        add("pre_pool_expansion_layer.bias", H);
        for (int l = 0; l < 2; ++l)
            for (int d = 0; d < 2; ++d) {
                const std::string sfx = "_l" + std::to_string(l) + (d ? "_reverse" : "");
                const int in = l == 0 ? H : 2 * H;
                add("lstm.weight_ih" + sfx, (int64_t)4 * H * in);
                add("lstm.weight_hh" + sfx, (int64_t)4 * H * H);
                add("lstm.bias_ih" + sfx, 4 * H);
                add("lstm.bias_hh" + sfx, 4 * H);
            }
        add("linear.weight", (int64_t)NCLS * 2 * H);
        add("linear.bias", NCLS);
    }
};

// the BatchNorm buffers: running_mean, running_var of convs.2 and convs.5 (device: 4 x C floats in this order)
const char *const RL_BUF_NAMES[4] = {"read_level_conv.convs.2.running_mean", "read_level_conv.convs.2.running_var",
                                     "read_level_conv.convs.5.running_mean", "read_level_conv.convs.5.running_var"};
const char *const RL_NBT_NAMES[2] = {"read_level_conv.convs.2.num_batches_tracked",
                                     "read_level_conv.convs.5.num_batches_tracked"};

// workspace floats per position (B*P): pooled, u (C each), z H, gi 8H, h0, h1 2H each, the saved gates of both layers
// 20H, dh 2H, logits, probs, dlogits, the label
int64_t rlt_floats_per_pos(int H) { return (int64_t)2 * RL_C + 35 * H + 3 * NCLS + 1; }

int64_t rlt_slice_rows(int64_t P, int64_t rows) {
    const int64_t fit = (int64_t)(RLT_SCRATCH / ((size_t)2 * P * RL_C * sizeof(float)));
    return std::max<int64_t>(1, std::min<int64_t>({rows, fit, (int64_t)65535}));      // 65535: the grid's y limit
}

}  // namespace
}  // namespace mdk

using namespace mdk;

enum { RS_STATS, RS_FWD, RS_LSTM, RS_HEAD, RS_BPTT, RS_READ, RS_RED, RS_OPT, RS_N };

struct mdk_rl_trainer {
    int device = 0, sm_count = 132, H = RL_H, use_dwells = 0, nin = 7;
    RlParams lay;
    std::vector<float> host_params, host_buf;
    std::vector<uint8_t> loaded;             // per parameter; then the 4 running-statistics buffers
    int64_t nbt[2] = {0, 0};                 // num_batches_tracked of BN1, BN2
    bool uploaded = false;
    cudaStream_t stream = nullptr;
    float *param = nullptr, *grad = nullptr, *s1 = nullptr, *s2 = nullptr, *run = nullptr;
    // packed weights, rebuilt from param by repack
    float *w17_t = nullptr, *w17_dg = nullptr, *pool_wt = nullptr, *zeros = nullptr;
    float *pool_w = nullptr, *lin_w = nullptr;   // 16-byte aligned copies for the kernels' vector loads
    float *w_ih[2] = {}, *bias[2] = {}, *w_t[2] = {}, *w_ih_t[2] = {};
    float *bn = nullptr;                     // [mean1, invstd1, mean2, invstd2, eval invstd1, eval invstd2, coef 5 C]
    double *red = nullptr;                   // [3][RED_BLOCKS] + [3] loss, correct, sum of squares
    double *tot = nullptr;                   // [RLT_NQ][C] running totals
    // workspace
    int64_t cap_ws = 0, cap_x = 0, cap_scr = 0, cap_dpart = 0, cap_part = 0;
    float *ws = nullptr, *scr = nullptr, *part = nullptr, *w17_acc = nullptr;
    int8_t *x = nullptr;
    double *dpart = nullptr;
    mdk_optim_desc opt{};
    int64_t opt_steps = 0;
    double mu_product = 1.0;
    int bptt_windows = 0;                    // 0: from B
    int64_t slice_rows = 0;                  // 0: rlt_slice_rows
    cudaEvent_t ev[16] = {};
    int ev_kind[16] = {};
    int n_ev = 0;
    float stage_ms[RS_N] = {};
};

namespace {

int alloc_t(void **p, size_t bytes) {
    MDK_CUDA(cudaMalloc(p, std::max<size_t>(bytes, 16)));
    return MDK_OK;
}
int alloc_f(float **p, int64_t n) { return alloc_t(reinterpret_cast<void **>(p), (size_t)n * sizeof(float)); }
template <class T> void free_t(T *&p) { if (p) cudaFree((void *)p); p = nullptr; }

struct RlWs {
    float *pooled, *u, *z, *gi, *h0, *h1, *save[2], *dh, *logits, *probs, *dlogits, *reads;
    int32_t *labels;
    uint8_t *mask;
};

RlWs rlt_view(const mdk_rl_trainer *tr, int64_t B, int64_t P, int64_t D) {
    const int64_t n = B * P, H = tr->H;
    float *o = tr->ws;
    auto take = [&](int64_t k) { float *r = o; o += (k + 63) / 64 * 64; return r; };
    RlWs v;
    v.pooled = take(n * RL_C); v.u = take(n * RL_C); v.z = take(n * H); v.gi = take(n * 8 * H);
    v.h0 = take(n * 2 * H); v.h1 = take(n * 2 * H); v.save[0] = take(n * 10 * H); v.save[1] = take(n * 10 * H);
    v.dh = take(n * 2 * H); v.logits = take(n * NCLS); v.probs = take(n * NCLS); v.dlogits = take(n * NCLS);
    v.labels = reinterpret_cast<int32_t *>(take(n));
    v.reads = take(B);
    v.mask = reinterpret_cast<uint8_t *>(take((B * D + 3) / 4));
    return v;
}
int64_t rlt_ws_floats(int H, int64_t B, int64_t P, int64_t D) {
    return B * P * rlt_floats_per_pos(H) + B + (B * D + 3) / 4 + 16 * 64;
}

// partial-sum sizes of a step: float (split-M wgrad) and double (per-block channel sums)
int64_t rlt_part_floats(int H, int64_t B, int64_t P, int64_t D) {
    auto tiles = [](int64_t n, int64_t k) { return ((n + RT - 1) / RT) * ((k + RT - 1) / RT); };
    const int64_t n = B * P;
    int64_t need = 0;
    auto w = [&](int64_t M, int64_t a, int64_t k) { need = std::max<int64_t>(need, split_for(M, tiles(a, k)).splits * a * k); };
    w(n, 8 * H, 2 * H); w(n, 8 * H, H); w(n, 4 * H, H); w(n, NCLS, 2 * H); w(n, H, RL_C); w(n, 8 * H, 1); w(n, H, 1);
    w(rlt_slice_rows(P, B * D) * P, RL_C, RL_C);
    return need;
}
int64_t rlt_dpart_doubles(int64_t B, int64_t P, int64_t D) {
    const int64_t rows = rlt_slice_rows(P, B * D), ptiles = (P + CV_PT - 1) / CV_PT;
    int64_t need = (int64_t)RED_BLOCKS * RLT_NQ * RL_C;
    need = std::max<int64_t>(need, ptiles * rows * RL_C);                      // BWD
    need = std::max<int64_t>(need, ptiles * (rows / D + 2) * 2 * RL_C);        // FWD
    return need;
}
// y1 and dpre2 of one slice of a training step
int64_t rlt_scratch_floats(int64_t B, int64_t P, int64_t D) { return 2 * rlt_slice_rows(P, B * D) * P * RL_C; }
int64_t rlt_total_bytes(int H, int64_t B, int64_t P, int64_t D, int64_t F) {
    return (rlt_ws_floats(H, B, P, D) + rlt_part_floats(H, B, P, D) + rlt_scratch_floats(B, P, D) +
            (int64_t)RL_TAPS * RL_C * RL_C) * (int64_t)sizeof(float) +
           rlt_dpart_doubles(B, P, D) * (int64_t)sizeof(double) + B * P * D * F;
}

template <class T>
int grow(T **p, int64_t *cap, int64_t need, cudaStream_t s) {
    if (need <= *cap) return MDK_OK;
    MDK_CUDA(cudaStreamSynchronize(s));
    free_t(*p);
    *cap = 0;
    int rc = alloc_t(reinterpret_cast<void **>(p), (size_t)need * sizeof(T));
    if (rc) return rc;
    *cap = need;
    return MDK_OK;
}

int rlt_ensure(mdk_rl_trainer *tr, int64_t B, int64_t P, int64_t D, int64_t F) {
    MDK_REQUIRE(rlt_total_bytes(tr->H, B, P, D, F) <= RLT_WS_BUDGET, MDK_ERR_ARG,
                "rl_trainer: a batch this large exceeds the 64 GiB training workspace budget (see "
                "mdk_rl_trainer_workspace_bytes)");
    int rc;
    if ((rc = grow(&tr->ws, &tr->cap_ws, rlt_ws_floats(tr->H, B, P, D), tr->stream)) ||
        (rc = grow(&tr->x, &tr->cap_x, B * P * D * F, tr->stream)) ||
        (rc = grow(&tr->scr, &tr->cap_scr, rlt_scratch_floats(B, P, D), tr->stream)) ||
        (rc = grow(&tr->dpart, &tr->cap_dpart, rlt_dpart_doubles(B, P, D), tr->stream)) ||
        (rc = grow(&tr->part, &tr->cap_part, rlt_part_floats(tr->H, B, P, D), tr->stream)))
        return rc;
    return MDK_OK;
}

float *P_(mdk_rl_trainer *tr, const char *name) { return tr->param + tr->lay.at(name); }
float *G_(mdk_rl_trainer *tr, const std::string &name) { return tr->grad + tr->lay.at(name); }
float *P_(mdk_rl_trainer *tr, const std::string &name) { return tr->param + tr->lay.at(name); }

// the forward's packed weights from the master weights, on the stream
int repack(mdk_rl_trainer *tr) {
    const int H = tr->H, G4 = 4 * H;
    cudaStream_t s = tr->stream;
    const int n17 = RL_C * RL_C * RL_TAPS;
    rlt_w17_pack_kernel<<<(n17 + 255) / 256, 256, 0, s>>>(P_(tr, "read_level_conv.convs.3.weight"), tr->w17_t, tr->w17_dg);
    MDK_CUDA(cudaMemcpyAsync(tr->pool_w, P_(tr, "pre_pool_expansion_layer.weight"), (size_t)H * RL_C * sizeof(float),
                             cudaMemcpyDeviceToDevice, s));
    MDK_CUDA(cudaMemcpyAsync(tr->lin_w, P_(tr, "linear.weight"), (size_t)NCLS * 2 * H * sizeof(float),
                             cudaMemcpyDeviceToDevice, s));
    transpose_kernel<<<dim3((RL_C + 31) / 32, (H + 31) / 32), 256, 0, s>>>(P_(tr, "pre_pool_expansion_layer.weight"),
                                                                           tr->pool_wt, H, RL_C);
    for (int l = 0; l < 2; ++l) {
        const int in = l == 0 ? H : 2 * H;
        for (int d = 0; d < 2; ++d) {
            const std::string sfx = "_l" + std::to_string(l) + (d ? "_reverse" : "");
            MDK_CUDA(cudaMemcpyAsync(tr->w_ih[l] + (int64_t)d * G4 * in, P_(tr, "lstm.weight_ih" + sfx),
                                     (size_t)G4 * in * sizeof(float), cudaMemcpyDeviceToDevice, s));
            rlt_add_kernel<<<(G4 + 255) / 256, 256, 0, s>>>(P_(tr, "lstm.bias_ih" + sfx), P_(tr, "lstm.bias_hh" + sfx),
                                                            tr->bias[l] + d * G4, G4);
            transpose_kernel<<<dim3((H + 31) / 32, (G4 + 31) / 32), 256, 0, s>>>(P_(tr, "lstm.weight_hh" + sfx),
                                                                                tr->w_t[l] + (int64_t)d * H * G4, G4, H);
        }
        transpose_kernel<<<dim3((in + 31) / 32, (2 * G4 + 31) / 32), 256, 0, s>>>(tr->w_ih[l], tr->w_ih_t[l], 2 * G4, in);
    }
    MDK_CUDA(cudaGetLastError());
    return MDK_OK;
}

int upload(mdk_rl_trainer *tr) {
    if (tr->uploaded) return MDK_OK;
    for (size_t i = 0; i < tr->loaded.size(); ++i)
        MDK_REQUIRE(tr->loaded[i], MDK_ERR_STATE,
                    "rl_trainer: tensor '" + (i < tr->lay.names.size() ? tr->lay.names[i] : std::string(RL_BUF_NAMES[i - tr->lay.names.size()])) +
                        "' was not loaded");
    const int64_t n = tr->lay.total;
    cudaStream_t s = tr->stream;
    MDK_CUDA(cudaMemcpyAsync(tr->param, tr->host_params.data(), n * sizeof(float), cudaMemcpyHostToDevice, s));
    MDK_CUDA(cudaMemcpyAsync(tr->run, tr->host_buf.data(), 4 * RL_C * sizeof(float), cudaMemcpyHostToDevice, s));
    MDK_CUDA(cudaMemsetAsync(tr->s1, 0, n * sizeof(float), s));
    MDK_CUDA(cudaMemsetAsync(tr->s2, 0, n * sizeof(float), s));
    MDK_CUDA(cudaMemsetAsync(tr->grad, 0, n * sizeof(float), s));
    int rc = repack(tr);
    if (rc) return rc;
    MDK_CUDA(cudaStreamSynchronize(s));
    tr->uploaded = true;
    tr->opt_steps = 0;
    tr->mu_product = 1.0;
    return MDK_OK;
}

int sync_host(mdk_rl_trainer *tr) {
    if (!tr->uploaded) return MDK_OK;
    MDK_CUDA(cudaSetDevice(tr->device));
    MDK_CUDA(cudaMemcpyAsync(tr->host_params.data(), tr->param, tr->lay.total * sizeof(float), cudaMemcpyDeviceToHost, tr->stream));
    MDK_CUDA(cudaMemcpyAsync(tr->host_buf.data(), tr->run, 4 * RL_C * sizeof(float), cudaMemcpyDeviceToHost, tr->stream));
    MDK_CUDA(cudaStreamSynchronize(tr->stream));
    return MDK_OK;
}

void mark(mdk_rl_trainer *tr, int kind) {
    if (tr->n_ev < 16) {
        cudaEventRecord(tr->ev[tr->n_ev], tr->stream);
        tr->ev_kind[tr->n_ev] = kind;
        ++tr->n_ev;
    }
}

// dst (+)= sum over M rows of A(m, n) X(m, k); rows n >= rows_split go to dst1.  accumulate: dst0 += (no split)
template <int AMODE, int XMODE>
int wgrad(mdk_rl_trainer *tr, const RedA &A, const RedX &X, int64_t M, int rows_split, float *dst0, float *dst1,
          bool accumulate = false) {
    const int64_t tn = (A.N + RT - 1) / RT, tk = (X.K + RT - 1) / RT;
    const Split sp = split_for(M, tn * tk);
    wgrad_kernel<AMODE, XMODE><<<dim3((unsigned)tn, (unsigned)tk, (unsigned)sp.splits), 256, 0, tr->stream>>>(A, X, M, sp.chunk,
                                                                                                          tr->part);
    const int64_t count = (int64_t)A.N * X.K;
    if (accumulate)
        rlt_accum_partials_kernel<<<(unsigned)((count + 255) / 256), 256, 0, tr->stream>>>(tr->part, sp.splits, count, dst0);
    else
        reduce_partials_kernel<<<(unsigned)((count + 255) / 256), 256, 0, tr->stream>>>(tr->part, sp.splits, count, X.K,
                                                                                       rows_split, dst0, dst1);
    MDK_CUDA(cudaGetLastError());
    return MDK_OK;
}

int colsum(mdk_rl_trainer *tr, const RedA &A, int64_t M, int rows_split, float *dst0, float *dst1) {
    const Split sp = split_for(M, (A.N + 255) / 256);
    colsum_kernel<0><<<dim3((unsigned)((A.N + 255) / 256), (unsigned)sp.splits), 256, 0, tr->stream>>>(A, M, sp.chunk, tr->part);
    reduce_partials_kernel<<<(unsigned)((A.N + 255) / 256), 256, 0, tr->stream>>>(tr->part, sp.splits, A.N, 1, rows_split,
                                                                                 dst0, dst1);
    MDK_CUDA(cudaGetLastError());
    return MDK_OK;
}

void accum(mdk_rl_trainer *tr, int64_t nparts, int n, bool reset) {
    if (reset) cudaMemsetAsync(tr->tot, 0, (size_t)n * sizeof(double), tr->stream);
    rlt_accum_kernel<<<(n + 255) / 256, 256, 0, tr->stream>>>(tr->dpart, nparts, n, tr->tot);
}

int bptt_nb(const mdk_rl_trainer *tr, int64_t B) {
    if (tr->bptt_windows) return tr->bptt_windows;
    for (int nb : {1, 2, 4})
        if (((B + nb - 1) / nb) * 2 <= tr->sm_count) return nb;
    return 8;
}

template <int HS, int NB>
cudaError_t launch_bptt_t(const float *save, const float *dh, const float *w0, const float *w1, float *dgi, int64_t B,
                          int64_t P, cudaStream_t s) {
    const size_t smem = (size_t)2 * NB * 4 * HS * sizeof(float);
    cudaError_t e = cudaFuncSetAttribute(rlt_bptt_kernel<HS, NB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    rlt_bptt_kernel<HS, NB><<<dim3((unsigned)((B + NB - 1) / NB), 2), HS, smem, s>>>(save, dh, w0, w1, dgi, B, P);
    return cudaGetLastError();
}
template <int HS>
cudaError_t launch_bptt_h(int nb, const float *save, const float *dh, const float *w0, const float *w1, float *dgi,
                          int64_t B, int64_t P, cudaStream_t s) {
    switch (nb) {
    case 1: return launch_bptt_t<HS, 1>(save, dh, w0, w1, dgi, B, P, s);
    case 2: return launch_bptt_t<HS, 2>(save, dh, w0, w1, dgi, B, P, s);
    case 4: return launch_bptt_t<HS, 4>(save, dh, w0, w1, dgi, B, P, s);
    default: return launch_bptt_t<HS, 8>(save, dh, w0, w1, dgi, B, P, s);
    }
}

// the rows of one slice of the forward and read backward passes: the automatic length, capped by the setting
int64_t step_slice_rows(const mdk_rl_trainer *tr, int64_t P, int64_t rows) {
    const int64_t sl = rlt_slice_rows(P, rows);
    return tr->slice_rows ? std::min(tr->slice_rows, sl) : sl;
}

RltIn rlt_in(mdk_rl_trainer *tr, int64_t P, int64_t D, int64_t F) {
    return RltIn{tr->x, P_(tr, "base_embedder.weight"), P_(tr, "strand_embedder.weight"),
                 P_(tr, "read_level_conv.convs.0.weight"), P_(tr, "read_level_conv.convs.0.bias"), P, (int)D, (int)F,
                 tr->use_dwells};
}

int check_batch(mdk_rl_trainer *tr, const int8_t *x, const int32_t *labels, int64_t B, int64_t P, int64_t D, int64_t F) {
    MDK_REQUIRE(tr && x, MDK_ERR_ARG, "rl_trainer: NULL argument");
    MDK_REQUIRE(B >= 1 && P >= 1 && D >= 1, MDK_ERR_ARG, "rl_trainer: need B, P, D >= 1");
    MDK_REQUIRE(F == (tr->use_dwells ? 5 : 4) || (!tr->use_dwells && F >= 4), MDK_ERR_ARG,
                "rl_trainer: feature vector length does not match the model (4, or 5 with dwells)");
    MDK_REQUIRE(D <= 65535 && B <= 65535, MDK_ERR_ARG, "rl_trainer: B, D <= 65535");
    if (labels)
        for (int64_t i = 0; i < B * P; ++i)
            MDK_REQUIRE(labels[i] >= 0 && labels[i] < NCLS, MDK_ERR_ARG,
                        "rl_trainer: label out of range [0, 5) (CrossEntropyLoss raises on it)");
    MDK_CUDA(cudaSetDevice(tr->device));
    int rc;
    if ((rc = upload(tr))) return rc;
    return rlt_ensure(tr, B, P, D, F);
}

int stage(mdk_rl_trainer *tr, const RlWs &v, const int8_t *x, const int32_t *labels, int64_t B, int64_t P, int64_t D,
          int64_t F) {
    MDK_CUDA(cudaMemcpyAsync(tr->x, x, (size_t)(B * P * D * F), cudaMemcpyHostToDevice, tr->stream));
    if (labels) MDK_CUDA(cudaMemcpyAsync(v.labels, labels, (size_t)(B * P) * sizeof(int32_t), cudaMemcpyHostToDevice, tr->stream));
    MDK_CUDA(rl_launch_mask(tr->x, B, P, (int)D, (int)F, v.mask, tr->stream));
    rlt_reads_kernel<<<(unsigned)((B + 127) / 128), 128, 0, tr->stream>>>(v.mask, B, (int)D, v.reads);
    MDK_CUDA(cudaGetLastError());
    return MDK_OK;
}

int loss(mdk_rl_trainer *tr, const RlWs &v, int64_t n) {
    loss_kernel<<<RED_BLOCKS, 256, 0, tr->stream>>>(v.logits, v.labels, n, (float)(1.0 / (double)n), v.dlogits, tr->red,
                                                    tr->red + RED_BLOCKS);
    sum_partials_kernel<<<1, 256, 0, tr->stream>>>(tr->red, RED_BLOCKS, tr->red + 3 * RED_BLOCKS);
    sum_partials_kernel<<<1, 256, 0, tr->stream>>>(tr->red + RED_BLOCKS, RED_BLOCKS, tr->red + 3 * RED_BLOCKS + 1);
    MDK_CUDA(cudaGetLastError());
    return MDK_OK;
}

// LSTM layers and head of the training or validation forward from z; save: keep the gates for BPTT
int lstm_head(mdk_rl_trainer *tr, const RlWs &v, int64_t B, int64_t P, bool save, bool engine_probs) {
    const int H = tr->H;
    const int64_t n = B * P;
    cudaStream_t s = tr->stream;
    MDK_CUDA(launch_gemm_fp32(v.z, tr->w_ih[0], tr->bias[0], v.gi, n, H, 8 * H, s));
    MDK_CUDA(rl_launch_lstm_fp32(v.gi, tr->w_t[0], v.h0, B, P, H, s, save ? v.save[0] : nullptr));
    MDK_CUDA(launch_gemm_fp32(v.h0, tr->w_ih[1], tr->bias[1], v.gi, n, 2 * H, 8 * H, s));
    MDK_CUDA(rl_launch_lstm_fp32(v.gi, tr->w_t[1], v.h1, B, P, H, s, save ? v.save[1] : nullptr));
    if (save) mark(tr, RS_LSTM);
    const float *lw = tr->lin_w, *lb = P_(tr, "linear.bias");
    if (engine_probs || H == RL_H) MDK_CUDA(rl_launch_head(v.h1, lw, lb, n, H, v.probs, H == RL_H ? v.logits : nullptr, s));
    if (H != RL_H) {
        rlt_logits_kernel<<<(unsigned)std::min<int64_t>((n + 7) / 8, 132 * 8), 256, 0, s>>>(v.h1, lw, lb, n, 2 * H, v.logits);
        MDK_CUDA(cudaGetLastError());
    }
    return MDK_OK;
}

// the training forward: stats pass, forward pass over the slices, BN2, pooled Linear, LSTM, logits
int forward_train(mdk_rl_trainer *tr, const RlWs &v, int64_t B, int64_t P, int64_t D, int64_t F) {
    cudaStream_t s = tr->stream;
    const int64_t rows = B * D, N = rows * P;
    const RltIn in = rlt_in(tr, P, D, F);
    float *mean1 = tr->bn, *invstd1 = tr->bn + RL_C, *mean2 = tr->bn + 2 * RL_C, *invstd2 = tr->bn + 3 * RL_C;
    rlt_conv1_stats_kernel<<<RED_BLOCKS, RL_C, 0, s>>>(in, N, tr->dpart);
    accum(tr, RED_BLOCKS, 2 * RL_C, true);
    rlt_bn_stats_kernel<<<1, RL_C, 0, s>>>(tr->tot, (double)N, mean1, invstd1, tr->run, tr->run + RL_C);
    MDK_CUDA(cudaGetLastError());
    mark(tr, RS_STATS);
    const int64_t sl = step_slice_rows(tr, P, rows), ptiles = (P + CV_PT - 1) / CV_PT;
    float *y1 = tr->scr;
    MDK_CUDA(cudaMemsetAsync(v.pooled, 0, (size_t)B * P * RL_C * sizeof(float), s));
    MDK_CUDA(cudaMemsetAsync(tr->tot, 0, 2 * RL_C * sizeof(double), s));
    MDK_CUDA(cudaFuncSetAttribute(rlt_conv17_kernel<CV_FWD>, cudaFuncAttributeMaxDynamicSharedMemorySize, CV_SMEM));
    for (int64_t r0 = 0; r0 < rows; r0 += sl) {
        const int64_t r1 = std::min(rows, r0 + sl), nw = (r1 - 1) / D - r0 / D + 1;
        rlt_y1_kernel<<<dim3((unsigned)((P + 31) / 32), (unsigned)(r1 - r0)), RL_C, 0, s>>>(
            in, mean1, invstd1, P_(tr, "read_level_conv.convs.2.weight"), P_(tr, "read_level_conv.convs.2.bias"), r0, y1);
        RltConv a{};
        a.in = y1; a.w_t = tr->w17_t; a.bias = P_(tr, "read_level_conv.convs.3.bias"); a.mask = v.mask;
        a.r0 = r0; a.r1 = r1; a.P = P; a.D = (int)D; a.pooled = v.pooled; a.part = tr->dpart;
        rlt_conv17_kernel<CV_FWD><<<dim3((unsigned)ptiles, (unsigned)nw), 256, CV_SMEM, s>>>(a);
        accum(tr, ptiles * nw, 2 * RL_C, false);
    }
    rlt_bn_stats_kernel<<<1, RL_C, 0, s>>>(tr->tot, (double)N, mean2, invstd2, tr->run + 2 * RL_C, tr->run + 3 * RL_C);
    rlt_pool_bn_kernel<<<(unsigned)std::min<int64_t>((B * P * RL_C + 255) / 256, 132 * 16), 256, 0, s>>>(
        v.pooled, v.reads, mean2, invstd2, P_(tr, "read_level_conv.convs.5.weight"), P_(tr, "read_level_conv.convs.5.bias"),
        B * P, P, v.u);
    MDK_CUDA(launch_gemm_fp32(v.u, tr->pool_w, P_(tr, "pre_pool_expansion_layer.bias"), v.z,
                              B * P, RL_C, tr->H, s));
    tr->nbt[0] += 1;
    tr->nbt[1] += 1;
    mark(tr, RS_FWD);
    return lstm_head(tr, v, B, P, true, false);
}

// gradients of one LSTM layer from its gate gradients in v.gi; X its input rows, hl its output
int layer_grads(mdk_rl_trainer *tr, const RlWs &v, int l, const float *X, int64_t B, int64_t P) {
    const int H = tr->H, in = l == 0 ? H : 2 * H;
    const int64_t n = B * P;
    const std::string s0 = "_l" + std::to_string(l), s1 = s0 + "_reverse";
    const float *hl = l ? v.h1 : v.h0;
    int rc;
    if ((rc = wgrad<0, 0>(tr, RedA{v.gi, 8 * H, 8 * H, nullptr, H}, RedX{X, in, in, P, 0, 0}, n, 4 * H,
                          G_(tr, "lstm.weight_ih" + s0), G_(tr, "lstm.weight_ih" + s1))))
        return rc;
    if ((rc = colsum(tr, RedA{v.gi, 8 * H, 8 * H, nullptr, H}, n, 4 * H, G_(tr, "lstm.bias_ih" + s0),
                     G_(tr, "lstm.bias_ih" + s1))))
        return rc;
    for (int d = 0; d < 2; ++d) {
        const std::string sfx = d ? s1 : s0;
        MDK_CUDA(cudaMemcpyAsync(G_(tr, "lstm.bias_hh" + sfx), G_(tr, "lstm.bias_ih" + sfx), 4 * H * sizeof(float),
                                 cudaMemcpyDeviceToDevice, tr->stream));
        if ((rc = wgrad<0, 1>(tr, RedA{v.gi + d * 4 * H, 8 * H, 4 * H, nullptr, H}, RedX{hl + d * H, 2 * H, H, P, d, 0}, n,
                              4 * H, G_(tr, "lstm.weight_hh" + sfx), nullptr)))
            return rc;
    }
    return MDK_OK;
}

int backward(mdk_rl_trainer *tr, const RlWs &v, int64_t B, int64_t P, int64_t D, int64_t F) {
    const int H = tr->H;
    const int64_t n = B * P, rows = B * D, N = rows * P;
    cudaStream_t s = tr->stream;
    int rc;
    // head
    head_bwd_kernel<<<(unsigned)std::min<int64_t>((n * 2 * H + 255) / 256, 132 * 16), 256, 0, s>>>(
        v.dlogits, tr->lin_w, v.dh, n, 2 * H);
    if ((rc = wgrad<0, 0>(tr, RedA{v.dlogits, NCLS, NCLS, nullptr, H}, RedX{v.h1, 2 * H, 2 * H, P, 0, 0}, n, NCLS,
                          G_(tr, "linear.weight"), nullptr)))
        return rc;
    if ((rc = colsum(tr, RedA{v.dlogits, NCLS, NCLS, nullptr, H}, n, NCLS, G_(tr, "linear.bias"), nullptr))) return rc;
    mark(tr, RS_HEAD);
    // LSTM: layer 1, dh0, layer 0, dz (into dh)
    const int nb = bptt_nb(tr, B);
    for (int l = 1; l >= 0; --l) {
        const std::string sfx = "_l" + std::to_string(l);
        const float *w0 = P_(tr, "lstm.weight_hh" + sfx), *w1 = P_(tr, "lstm.weight_hh" + sfx + "_reverse");
        MDK_CUDA(H == RL_H3 ? launch_bptt_h<RL_H3>(nb, v.save[l], v.dh, w0, w1, v.gi, B, P, s)
                            : launch_bptt_h<RL_H>(nb, v.save[l], v.dh, w0, w1, v.gi, B, P, s));
        mark(tr, RS_BPTT);
        if ((rc = layer_grads(tr, v, l, l ? v.h0 : v.z, B, P))) return rc;
        MDK_CUDA(launch_gemm_fp32(v.gi, tr->w_ih_t[l], tr->zeros, v.dh, n, 8 * H, l ? 2 * H : H, s));
        mark(tr, RS_RED);
    }
    // pre_pool_expansion_layer: dW = dz^T u, db = sum dz, du = dz W (into z)
    const float *dz = v.dh;
    float *du = v.z;
    if ((rc = wgrad<0, 0>(tr, RedA{dz, H, H, nullptr, H}, RedX{v.u, RL_C, RL_C, P, 0, 0}, n, H,
                          G_(tr, "pre_pool_expansion_layer.weight"), nullptr)))
        return rc;
    if ((rc = colsum(tr, RedA{dz, H, H, nullptr, H}, n, H, G_(tr, "pre_pool_expansion_layer.bias"), nullptr))) return rc;
    MDK_CUDA(launch_gemm_fp32(dz, tr->pool_wt, tr->zeros, du, n, H, RL_C, s));
    // BN2's backward sums and coefficients
    float *mean1 = tr->bn, *invstd1 = tr->bn + RL_C, *mean2 = tr->bn + 2 * RL_C, *invstd2 = tr->bn + 3 * RL_C;
    float *coef = tr->bn + 6 * RL_C;
    rlt_bn2_sums_kernel<<<RED_BLOCKS, RL_C, 0, s>>>(du, v.pooled, v.reads, mean2, invstd2, n, P, tr->dpart);
    accum(tr, RED_BLOCKS, 2 * RL_C, true);
    rlt_bn_coef_kernel<<<1, RL_C, 0, s>>>(tr->tot, (double)N, P_(tr, "read_level_conv.convs.5.weight"), mean2, invstd2, coef,
                                          G_(tr, "read_level_conv.convs.5.weight"), G_(tr, "read_level_conv.convs.5.bias"));
    MDK_CUDA(cudaGetLastError());
    // the read pass: totals [0, C) db17, [C, C + 56 C) BN1's sums
    const RltIn in = rlt_in(tr, P, D, F);
    const int64_t sl = step_slice_rows(tr, P, rows), ptiles = (P + CV_PT - 1) / CV_PT;
    float *y1 = tr->scr, *dpre = tr->scr + sl * P * RL_C;
    double *tot17 = tr->tot + RLT_NQ * RL_C;
    MDK_CUDA(cudaMemsetAsync(tr->tot, 0, (RLT_NQ + 1) * RL_C * sizeof(double), s));
    MDK_CUDA(cudaMemsetAsync(tr->w17_acc, 0, (size_t)RL_TAPS * RL_C * RL_C * sizeof(float), s));
    MDK_CUDA(cudaFuncSetAttribute(rlt_conv17_kernel<CV_BWD>, cudaFuncAttributeMaxDynamicSharedMemorySize, CV_SMEM));
    MDK_CUDA(cudaFuncSetAttribute(rlt_conv17_kernel<CV_DGRAD>, cudaFuncAttributeMaxDynamicSharedMemorySize, CV_SMEM));
    for (int64_t r0 = 0; r0 < rows; r0 += sl) {
        const int64_t r1 = std::min(rows, r0 + sl), nr = r1 - r0;
        rlt_y1_kernel<<<dim3((unsigned)((P + 31) / 32), (unsigned)nr), RL_C, 0, s>>>(
            in, mean1, invstd1, P_(tr, "read_level_conv.convs.2.weight"), P_(tr, "read_level_conv.convs.2.bias"), r0, y1);
        RltConv a{};
        a.in = y1; a.w_t = tr->w17_t; a.bias = P_(tr, "read_level_conv.convs.3.bias"); a.mask = v.mask;
        a.r0 = r0; a.r1 = r1; a.P = P; a.D = (int)D; a.du = du; a.reads = v.reads; a.coef = coef; a.out = dpre;
        a.part = tr->dpart;
        rlt_conv17_kernel<CV_BWD><<<dim3((unsigned)ptiles, (unsigned)nr), 256, CV_SMEM, s>>>(a);
        rlt_accum_kernel<<<1, RL_C, 0, s>>>(tr->dpart, ptiles * nr, RL_C, tot17);
        // dW17[t] += dpre2^T y1 shifted by t - 8 within each read
        for (int t = 0; t < RL_TAPS; ++t)
            if ((rc = wgrad<0, 2>(tr, RedA{dpre, RL_C, RL_C, nullptr, H}, RedX{y1, RL_C, RL_C, P, 0, t - RL_PAD}, nr * P,
                                  RL_C, tr->w17_acc + (int64_t)t * RL_C * RL_C, nullptr, true)))
                return rc;
        // dy1 (over y1) = the convolution of dpre2 with the transposed, flipped weights
        a.in = dpre; a.w_t = tr->w17_dg; a.out = y1;
        rlt_conv17_kernel<CV_DGRAD><<<dim3((unsigned)ptiles, (unsigned)nr), 256, CV_SMEM, s>>>(a);
        rlt_bn1_sums_kernel<<<RED_BLOCKS, RL_C, 0, s>>>(in, mean1, invstd1, y1, r0, nr * P, tr->dpart);
        rlt_accum_kernel<<<(RLT_NQ * RL_C + 255) / 256, 256, 0, s>>>(tr->dpart, RED_BLOCKS, RLT_NQ * RL_C, tr->tot);
        MDK_CUDA(cudaGetLastError());
    }
    mark(tr, RS_READ);
    rlt_to_float_kernel<<<1, RL_C, 0, s>>>(tot17, G_(tr, "read_level_conv.convs.3.bias"), RL_C);
    const int n17 = RL_C * RL_C * RL_TAPS;
    rlt_w17_grad_kernel<<<(n17 + 255) / 256, 256, 0, s>>>(tr->w17_acc, G_(tr, "read_level_conv.convs.3.weight"));
    RltBn1Grads g{G_(tr, "read_level_conv.convs.0.weight"), G_(tr, "read_level_conv.convs.0.bias"),
                  G_(tr, "read_level_conv.convs.2.weight"), G_(tr, "read_level_conv.convs.2.bias"),
                  G_(tr, "base_embedder.weight"), G_(tr, "strand_embedder.weight")};
    rlt_bn1_final_kernel<<<1, RL_C, 0, s>>>(tr->tot, (double)N, P_(tr, "read_level_conv.convs.2.weight"), invstd1,
                                            P_(tr, "read_level_conv.convs.0.weight"), tr->nin, g);
    MDK_CUDA(cudaGetLastError());
    mark(tr, RS_RED);
    return MDK_OK;
}

int read_stats(mdk_rl_trainer *tr, int64_t n, bool with_norm, mdk_train_stats *st) {
    double tot[3];
    MDK_CUDA(cudaMemcpyAsync(tot, tr->red + 3 * RED_BLOCKS, sizeof(tot), cudaMemcpyDeviceToHost, tr->stream));
    MDK_CUDA(cudaStreamSynchronize(tr->stream));
    if (st) {
        st->loss = tot[0] / (double)n;
        st->n_correct = (int64_t)tot[1];
        st->n_positions = n;
        st->grad_norm = with_norm ? (float)std::sqrt(tot[2]) : 0.f;
        st->skipped = with_norm && !std::isfinite(st->grad_norm) ? 1 : 0;
    }
    return MDK_OK;
}

}  // namespace

extern "C" {

int mdk_rl_trainer_create(int device, int32_t lstm_size, int32_t cnn_size, int32_t use_dwells, int32_t num_classes,
                          mdk_rl_trainer **out) {
    MDK_REQUIRE(out, MDK_ERR_ARG, "rl_trainer_create: NULL argument");
    MDK_REQUIRE(lstm_size == RL_H || lstm_size == RL_H3, MDK_ERR_UNSUPPORTED, "rl_trainer_create: lstm_size must be 128 or 384");
    MDK_REQUIRE(cnn_size == RL_C, MDK_ERR_UNSUPPORTED, "rl_trainer_create: cnn_size must be 128");
    MDK_REQUIRE(num_classes == NCLS, MDK_ERR_UNSUPPORTED, "rl_trainer_create: the head has 5 classes");
    int ndev = 0;
    MDK_CUDA(cudaGetDeviceCount(&ndev));
    MDK_REQUIRE(device >= 0 && device < ndev, MDK_ERR_ARG, "rl_trainer_create: no such CUDA device");
    cudaDeviceProp prop;
    MDK_CUDA(cudaGetDeviceProperties(&prop, device));
    MDK_REQUIRE(prop.major == 9 && prop.minor == 0, MDK_ERR_UNSUPPORTED,
                "rl_trainer_create: this library is built for sm_90a (Hopper H100) only");
    MDK_CUDA(cudaSetDevice(device));
    mdk_rl_trainer *tr = new (std::nothrow) mdk_rl_trainer();
    MDK_REQUIRE(tr, MDK_ERR_NOMEM, "rl_trainer_create: out of host memory");
    tr->device = device;
    tr->sm_count = prop.multiProcessorCount;
    tr->H = lstm_size;
    tr->use_dwells = use_dwells ? 1 : 0;
    tr->nin = RL_EMB + 1 + tr->use_dwells;
    tr->lay = RlParams(tr->H, tr->nin);
    tr->host_params.assign(tr->lay.total, 0.f);
    tr->host_buf.assign(4 * RL_C, 0.f);
    tr->loaded.assign(tr->lay.names.size() + 4, 0);
    tr->opt.kind = MDK_OPT_RMSPROP;
    tr->opt.alpha = 0.9f; tr->opt.eps = 1e-7f;
    const int H = tr->H, G4 = 4 * H;
    int rc = MDK_OK;
    cudaError_t e = cudaStreamCreateWithFlags(&tr->stream, cudaStreamNonBlocking);
    for (auto &ev : tr->ev)
        if (e == cudaSuccess) e = cudaEventCreate(&ev);
    if (e != cudaSuccess) rc = cuda_fail(e, "rl_trainer_create: stream / events", __FILE__, __LINE__);
    const int64_t n = tr->lay.total;
    if (!rc) rc = alloc_f(&tr->param, n);
    if (!rc) rc = alloc_f(&tr->grad, n);
    if (!rc) rc = alloc_f(&tr->s1, n);
    if (!rc) rc = alloc_f(&tr->s2, n);
    if (!rc) rc = alloc_f(&tr->run, 4 * RL_C);
    if (!rc) rc = alloc_f(&tr->w17_t, (int64_t)RL_TAPS * RL_C * RL_C);
    if (!rc) rc = alloc_f(&tr->w17_dg, (int64_t)RL_TAPS * RL_C * RL_C);
    if (!rc) rc = alloc_f(&tr->w17_acc, (int64_t)RL_TAPS * RL_C * RL_C);
    if (!rc) rc = alloc_f(&tr->pool_wt, (int64_t)RL_C * H);
    if (!rc) rc = alloc_f(&tr->pool_w, (int64_t)RL_C * H);
    if (!rc) rc = alloc_f(&tr->lin_w, (int64_t)NCLS * 2 * H);
    if (!rc) rc = alloc_f(&tr->zeros, 2 * H);
    if (!rc) rc = alloc_f(&tr->bn, 11 * RL_C);
    for (int l = 0; l < 2 && !rc; ++l) {
        const int in = l == 0 ? H : 2 * H;
        rc = alloc_f(&tr->w_ih[l], (int64_t)2 * G4 * in);
        if (!rc) rc = alloc_f(&tr->w_ih_t[l], (int64_t)2 * G4 * in);
        if (!rc) rc = alloc_f(&tr->bias[l], 2 * G4);
        if (!rc) rc = alloc_f(&tr->w_t[l], (int64_t)2 * H * G4);
    }
    if (!rc) rc = alloc_t(reinterpret_cast<void **>(&tr->red), (3 * RED_BLOCKS + 3) * sizeof(double));
    if (!rc) rc = alloc_t(reinterpret_cast<void **>(&tr->tot), (RLT_NQ + 1) * RL_C * sizeof(double));
    if (!rc) {
        e = cudaMemset(tr->zeros, 0, 2 * H * sizeof(float));
        if (e == cudaSuccess) e = cudaMemset(tr->red, 0, (3 * RED_BLOCKS + 3) * sizeof(double));
        if (e != cudaSuccess) rc = cuda_fail(e, "rl_trainer_create", __FILE__, __LINE__);
    }
    if (rc) {
        mdk_rl_trainer_destroy(tr);
        return rc;
    }
    *out = tr;
    return MDK_OK;
}

int mdk_rl_trainer_destroy(mdk_rl_trainer *tr) {
    if (!tr) return MDK_OK;
    cudaSetDevice(tr->device);
    if (tr->stream) cudaStreamSynchronize(tr->stream);
    free_t(tr->param); free_t(tr->grad); free_t(tr->s1); free_t(tr->s2); free_t(tr->run);
    free_t(tr->w17_t); free_t(tr->w17_dg); free_t(tr->w17_acc); free_t(tr->pool_wt); free_t(tr->pool_w); free_t(tr->lin_w); free_t(tr->zeros); free_t(tr->bn);
    for (int l = 0; l < 2; ++l) { free_t(tr->w_ih[l]); free_t(tr->w_ih_t[l]); free_t(tr->bias[l]); free_t(tr->w_t[l]); }
    free_t(tr->red); free_t(tr->tot); free_t(tr->ws); free_t(tr->scr); free_t(tr->part); free_t(tr->x); free_t(tr->dpart);
    for (auto &ev : tr->ev) if (ev) cudaEventDestroy(ev);
    if (tr->stream) cudaStreamDestroy(tr->stream);
    delete tr;
    return MDK_OK;
}

int mdk_rl_trainer_load(mdk_rl_trainer *tr, const char *name, const float *data, int64_t n) {
    MDK_REQUIRE(tr && name && data, MDK_ERR_ARG, "rl_trainer_load: NULL argument");
    const std::string nm(name);
    int rc;
    if ((rc = sync_host(tr))) return rc;
    for (int i = 0; i < 2; ++i)
        if (nm == RL_NBT_NAMES[i]) {
            MDK_REQUIRE(n == 1, MDK_ERR_ARG, "rl_trainer_load: " + nm + " has 1 value");
            tr->nbt[i] = (int64_t)data[0];
            return MDK_OK;
        }
    for (int i = 0; i < 4; ++i)
        if (nm == RL_BUF_NAMES[i]) {
            MDK_REQUIRE(n == RL_C, MDK_ERR_ARG, "rl_trainer_load: " + nm + " has cnn_size values");
            std::memcpy(tr->host_buf.data() + i * RL_C, data, RL_C * sizeof(float));
            tr->loaded[tr->lay.names.size() + i] = 1;
            tr->uploaded = false;
            return MDK_OK;
        }
    for (size_t i = 0; i < tr->lay.names.size(); ++i)
        if (tr->lay.names[i] == nm) {
            MDK_REQUIRE(n == tr->lay.size[i], MDK_ERR_ARG,
                        "rl_trainer_load: " + nm + " has " + std::to_string(tr->lay.size[i]) + " values, got " + std::to_string(n));
            std::memcpy(tr->host_params.data() + tr->lay.off[i], data, (size_t)n * sizeof(float));
            tr->loaded[i] = 1;
            tr->uploaded = false;
            return MDK_OK;
        }
    MDK_REQUIRE(false, MDK_ERR_ARG, "rl_trainer_load: unknown tensor '" + nm + "'");
    return MDK_ERR_ARG;
}

int mdk_rl_trainer_set_optimizer(mdk_rl_trainer *tr, const mdk_optim_desc *opt) {
    MDK_REQUIRE(tr && opt, MDK_ERR_ARG, "rl_trainer_set_optimizer: NULL argument");
    MDK_REQUIRE(opt->kind >= MDK_OPT_RMSPROP && opt->kind <= MDK_OPT_SGD, MDK_ERR_ARG, "rl_trainer_set_optimizer: unknown kind");
    MDK_REQUIRE(!(opt->kind == MDK_OPT_SGD && opt->nesterov && (opt->momentum <= 0.f || opt->dampening != 0.f)), MDK_ERR_ARG,
                "rl_trainer_set_optimizer: Nesterov momentum requires a momentum and zero dampening");
    MDK_CUDA(cudaSetDevice(tr->device));
    tr->opt = *opt;
    tr->opt_steps = 0;
    tr->mu_product = 1.0;
    if (tr->uploaded) {
        const size_t bytes = tr->lay.total * sizeof(float);
        MDK_CUDA(cudaMemsetAsync(tr->s1, 0, bytes, tr->stream));
        MDK_CUDA(cudaMemsetAsync(tr->s2, 0, bytes, tr->stream));
        MDK_CUDA(cudaStreamSynchronize(tr->stream));
    }
    return MDK_OK;
}

int mdk_rl_trainer_step(mdk_rl_trainer *tr, const int8_t *x, const int32_t *labels, int64_t B, int64_t P, int64_t D,
                        int64_t F, float lr, float max_norm, mdk_train_stats *stats) {
    MDK_REQUIRE(labels, MDK_ERR_ARG, "rl_trainer_step: NULL labels");
    int rc;
    if ((rc = check_batch(tr, x, labels, B, P, D, F))) return rc;
    const RlWs v = rlt_view(tr, B, P, D);
    const int64_t n = B * P;
    tr->n_ev = 0;
    mark(tr, -1);
    if ((rc = stage(tr, v, x, labels, B, P, D, F))) return rc;
    if ((rc = forward_train(tr, v, B, P, D, F))) return rc;
    if ((rc = loss(tr, v, n))) return rc;
    if ((rc = backward(tr, v, B, P, D, F))) return rc;
    // the step: norm, skip / clip, the rule (not on expansion_layer, which the forward never uses: torch leaves its
    // gradient None, so no optimizer touches it), the forward's weights
    const int64_t total = tr->lay.total;
    sumsq_kernel<<<RED_BLOCKS, 256, 0, tr->stream>>>(tr->grad, total, tr->red + 2 * RED_BLOCKS);
    sum_partials_kernel<<<1, 256, 0, tr->stream>>>(tr->red + 2 * RED_BLOCKS, RED_BLOCKS, tr->red + 3 * RED_BLOCKS + 2);
    const int64_t t = tr->opt_steps + 1;
    double mu_product = 0.0;
    const OptStep o = opt_step(tr->opt, lr, t, tr->mu_product, &mu_product);
    const int64_t x0 = tr->lay.at("read_level_conv.expansion_layer.weight");
    const int64_t x1 = tr->lay.at("pre_pool_expansion_layer.weight");
    const float mn = max_norm > 0.f ? max_norm : INFINITY;
    const int64_t ranges[2][2] = {{0, x0}, {x1, total}};
    for (const auto &r : ranges) {
        const int64_t len = r[1] - r[0];
        optim_kernel<<<(unsigned)std::min<int64_t>((len + 255) / 256, 132 * 8), 256, 0, tr->stream>>>(
            tr->param + r[0], tr->grad + r[0], tr->s1 + r[0], tr->s2 + r[0], len, tr->red + 3 * RED_BLOCKS + 2, mn, o);
    }
    MDK_CUDA(cudaGetLastError());
    if ((rc = repack(tr))) return rc;
    mark(tr, RS_OPT);
    mdk_train_stats st{};
    if ((rc = read_stats(tr, n, true, &st))) return rc;
    if (!st.skipped) {
        tr->opt_steps = t;
        tr->mu_product = mu_product;
    }
    for (float &ms : tr->stage_ms) ms = 0.f;
    for (int i = 1; i < tr->n_ev; ++i) {
        float ms = 0.f;
        MDK_CUDA(cudaEventElapsedTime(&ms, tr->ev[i - 1], tr->ev[i]));
        tr->stage_ms[tr->ev_kind[i]] += ms;
    }
    if (stats) *stats = st;
    return MDK_OK;
}

int mdk_rl_trainer_eval(mdk_rl_trainer *tr, const int8_t *x, const int32_t *labels, int64_t B, int64_t P, int64_t D,
                        int64_t F, float *probs, float *logits, mdk_train_stats *stats) {
    int rc;
    if ((rc = check_batch(tr, x, labels, B, P, D, F))) return rc;
    const RlWs v = rlt_view(tr, B, P, D);
    const int64_t n = B * P;
    cudaStream_t s = tr->stream;
    if ((rc = stage(tr, v, x, labels, B, P, D, F))) return rc;
    // the engine's fp32 path with the running statistics, one window at a time: its y1 and 4-read partial sums (the
    // engine's fp32 convolution holds a whole window's per-read activations, so validation's scratch grows with D)
    if ((rc = grow(&tr->scr, &tr->cap_scr, (D + (D + 3) / 4) * P * RL_C, s))) return rc;
    float *inv1 = tr->bn + 4 * RL_C, *inv2 = tr->bn + 5 * RL_C;
    rlt_invstd_kernel<<<1, RL_C, 0, s>>>(tr->run + RL_C, inv1);
    rlt_invstd_kernel<<<1, RL_C, 0, s>>>(tr->run + 3 * RL_C, inv2);
    const RlConv1 c1{P_(tr, "base_embedder.weight"), P_(tr, "strand_embedder.weight"), P_(tr, "read_level_conv.convs.0.weight"),
                     P_(tr, "read_level_conv.convs.0.bias"), tr->run, inv1, P_(tr, "read_level_conv.convs.2.weight"),
                     P_(tr, "read_level_conv.convs.2.bias")};
    const RlConv17 c17{tr->w17_t, P_(tr, "read_level_conv.convs.3.bias"), tr->run + 2 * RL_C, inv2,
                       P_(tr, "read_level_conv.convs.5.weight"), P_(tr, "read_level_conv.convs.5.bias")};
    float *y1 = tr->scr, *part = tr->scr + D * P * RL_C;
    for (int64_t b = 0; b < B; ++b)
        MDK_CUDA(rl_launch_conv_fp32(tr->x + b * P * D * F, v.mask + b * D, c1, c17, tr->pool_wt,
                                     P_(tr, "pre_pool_expansion_layer.bias"), 1, P, (int)D, (int)F, tr->use_dwells, tr->H,
                                     y1, part, v.z + b * P * tr->H, s));
    if ((rc = lstm_head(tr, v, B, P, false, true))) return rc;
    if (labels && (rc = loss(tr, v, n))) return rc;
    if (probs) MDK_CUDA(cudaMemcpyAsync(probs, v.probs, n * NCLS * sizeof(float), cudaMemcpyDeviceToHost, s));
    if (logits) MDK_CUDA(cudaMemcpyAsync(logits, v.logits, n * NCLS * sizeof(float), cudaMemcpyDeviceToHost, s));
    if (labels) return read_stats(tr, n, false, stats);
    MDK_CUDA(cudaStreamSynchronize(s));
    if (stats) *stats = mdk_train_stats{};
    return MDK_OK;
}

int mdk_rl_trainer_num_params(mdk_rl_trainer *tr, int64_t *n) {
    MDK_REQUIRE(tr && n, MDK_ERR_ARG, "rl_trainer_num_params: NULL argument");
    *n = tr->lay.total;
    return MDK_OK;
}

int mdk_rl_trainer_read_params(mdk_rl_trainer *tr, float *out, int64_t n) {
    MDK_REQUIRE(tr && out, MDK_ERR_ARG, "rl_trainer_read_params: NULL argument");
    MDK_REQUIRE(n == tr->lay.total, MDK_ERR_ARG, "rl_trainer_read_params: n must be mdk_rl_trainer_num_params");
    int rc;
    if ((rc = sync_host(tr))) return rc;
    std::memcpy(out, tr->host_params.data(), n * sizeof(float));
    return MDK_OK;
}

int mdk_rl_trainer_read_buffers(mdk_rl_trainer *tr, float *out, int64_t n, int64_t *num_batches_tracked) {
    MDK_REQUIRE(tr && out, MDK_ERR_ARG, "rl_trainer_read_buffers: NULL argument");
    MDK_REQUIRE(n == 4 * RL_C, MDK_ERR_ARG, "rl_trainer_read_buffers: n must be 4 cnn_size");
    int rc;
    if ((rc = sync_host(tr))) return rc;
    std::memcpy(out, tr->host_buf.data(), n * sizeof(float));
    if (num_batches_tracked) { num_batches_tracked[0] = tr->nbt[0]; num_batches_tracked[1] = tr->nbt[1]; }
    return MDK_OK;
}

int mdk_rl_trainer_read_grads(mdk_rl_trainer *tr, float *out, int64_t n) {
    MDK_REQUIRE(tr && out, MDK_ERR_ARG, "rl_trainer_read_grads: NULL argument");
    MDK_REQUIRE(n == tr->lay.total, MDK_ERR_ARG, "rl_trainer_read_grads: n must be mdk_rl_trainer_num_params");
    MDK_REQUIRE(tr->uploaded, MDK_ERR_STATE, "rl_trainer_read_grads: no step since the weights were loaded");
    MDK_CUDA(cudaSetDevice(tr->device));
    MDK_CUDA(cudaMemcpyAsync(out, tr->grad, n * sizeof(float), cudaMemcpyDeviceToHost, tr->stream));
    MDK_CUDA(cudaStreamSynchronize(tr->stream));
    return MDK_OK;
}

int mdk_rl_trainer_workspace_bytes(int32_t lstm_size, int64_t B, int64_t P, int64_t D, int64_t F, size_t *bytes,
                                   size_t *budget) {
    MDK_REQUIRE(bytes, MDK_ERR_ARG, "rl_trainer_workspace_bytes: NULL argument");
    MDK_REQUIRE(lstm_size == RL_H || lstm_size == RL_H3, MDK_ERR_UNSUPPORTED, "rl_trainer: lstm_size must be 128 or 384");
    MDK_REQUIRE(B >= 1 && P >= 1 && D >= 1 && F >= 1, MDK_ERR_ARG, "rl_trainer_workspace_bytes: need B, P, D, F >= 1");
    *bytes = (size_t)rlt_total_bytes(lstm_size, B, P, D, F);
    if (budget) *budget = (size_t)RLT_WS_BUDGET;
    return MDK_OK;
}

int mdk_rl_trainer_stage_ms(mdk_rl_trainer *tr, float *ms) {
    MDK_REQUIRE(tr && ms, MDK_ERR_ARG, "rl_trainer_stage_ms: NULL argument");
    for (int i = 0; i < RS_N; ++i) ms[i] = tr->stage_ms[i];
    return MDK_OK;
}

int mdk_rl_trainer_set_bptt_windows(mdk_rl_trainer *tr, int nb) {
    MDK_REQUIRE(tr, MDK_ERR_ARG, "rl_trainer_set_bptt_windows: NULL argument");
    MDK_REQUIRE(nb == 0 || nb == 1 || nb == 2 || nb == 4 || nb == 8, MDK_ERR_ARG,
                "rl_trainer_set_bptt_windows: 0, 1, 2, 4 or 8");
    tr->bptt_windows = nb;
    return MDK_OK;
}

int mdk_rl_trainer_set_slice_rows(mdk_rl_trainer *tr, int64_t rows) {
    MDK_REQUIRE(tr, MDK_ERR_ARG, "rl_trainer_set_slice_rows: NULL argument");
    MDK_REQUIRE(rows >= 0, MDK_ERR_ARG, "rl_trainer_set_slice_rows: rows >= 0 (0: automatic)");
    tr->slice_rows = rows;
    return MDK_OK;
}

int mdk_rl_trainer_bptt_windows(mdk_rl_trainer *tr, int64_t B, int *nb) {
    MDK_REQUIRE(tr && nb, MDK_ERR_ARG, "rl_trainer_bptt_windows: NULL argument");
    MDK_REQUIRE(B >= 1, MDK_ERR_ARG, "rl_trainer_bptt_windows: need B >= 1");
    *nb = bptt_nb(tr, B);
    return MDK_OK;
}

}  // extern "C"
