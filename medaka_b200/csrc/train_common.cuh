// The parts of a training step that the consensus GRU trainer (gru_train.cu) and the read-level trainer (rl_train.cu)
// share: fixed-order reductions, the cross-entropy loss and head backward, the split-M weight-gradient reductions, the
// global norm and the optimizer rules.  No float atomics anywhere: two identical steps give bit-identical results.
#pragma once
#include <cmath>

#include "common.cuh"

namespace mdk {
namespace {     // each trainer's translation unit has its own copy of these kernels

constexpr int RED_BLOCKS = 264;          // blocks of the fixed-shape reductions (2 per SM of an H100 SXM)

// Sum of doubles from a fixed number of per-block partials, by one block, in a fixed order
__device__ __forceinline__ double block_sum(double v, double *sh) {
    const int tid = threadIdx.x;
    sh[tid] = v;
    __syncthreads();
    for (int s = blockDim.x / 2; s > 0; s >>= 1) {
        if (tid < s) sh[tid] += sh[tid + s];
        __syncthreads();
    }
    const double r = sh[0];
    __syncthreads();
    return r;
}

__global__ void __launch_bounds__(256) sum_partials_kernel(const double *__restrict__ part, int n, double *__restrict__ out) {
    __shared__ double sh[256];
    double v = 0.0;
    for (int i = threadIdx.x; i < n; i += 256) v += part[i];
    v = block_sum(v, sh);
    if (threadIdx.x == 0) *out = v;
}

// Cross-entropy of CrossEntropyLoss() over P positions (mean reduction): per position lse(logits) - logits[label];
// dlogits = (softmax - onehot) / P; model_correct: argmax (first maximum, torch.argmax) == label.  Per-block partial
// sums of the loss and the count, RED_BLOCKS blocks.
__global__ void __launch_bounds__(256) loss_kernel(const float *__restrict__ logits, const int32_t *__restrict__ labels,
                                                   int64_t P, float inv_p, float *__restrict__ dlogits,
                                                   double *__restrict__ part_loss, double *__restrict__ part_correct) {
    __shared__ double sh[256];
    double loss = 0.0, correct = 0.0;
    for (int64_t p = (int64_t)blockIdx.x * 256 + threadIdx.x; p < P; p += (int64_t)gridDim.x * 256) {
        float l[NCLS];
#pragma unroll
        for (int c = 0; c < NCLS; ++c) l[c] = logits[p * NCLS + c];
        float mx = l[0];
        int arg = 0;
#pragma unroll
        for (int c = 1; c < NCLS; ++c)
            if (l[c] > mx) { mx = l[c]; arg = c; }
        float e[NCLS], s = 0.f;
#pragma unroll
        for (int c = 0; c < NCLS; ++c) { e[c] = expf(l[c] - mx); s += e[c]; }
        const int y = labels[p];
        loss += (double)(mx + logf(s) - l[y]);
        correct += arg == y ? 1.0 : 0.0;
        const float inv_s = 1.f / s;
#pragma unroll
        for (int c = 0; c < NCLS; ++c) dlogits[p * NCLS + c] = (e[c] * inv_s - (c == y ? 1.f : 0.f)) * inv_p;
    }
    loss = block_sum(loss, sh);
    correct = block_sum(correct, sh);
    if (threadIdx.x == 0) { part_loss[blockIdx.x] = loss; part_correct[blockIdx.x] = correct; }
}

// dh[p][k] = sum_c dlogits[p][c] W_lin[c][k], k < K2 (= 2 H)
__global__ void __launch_bounds__(256) head_bwd_kernel(const float *__restrict__ dlogits, const float *__restrict__ lin_w,
                                                       float *__restrict__ dh, int64_t P, int K2) {
    const int64_t n = P * K2;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (int64_t)gridDim.x * 256) {
        const int64_t p = i / K2;
        const int k = (int)(i - p * K2);
        float a = 0.f;
#pragma unroll
        for (int c = 0; c < NCLS; ++c) a = fmaf(dlogits[p * NCLS + c], lin_w[c * K2 + k], a);
        dh[i] = a;
    }
}

// The operands of the gradient reductions.  A(m, n): row m of a [M][lda] array; AMODE 1 is dG_h, the hidden-side gate
// gradient: A's n third (n >= 2 HS) times r of the same position, unit n - 2 HS (r_save: the save rows of the direction).
// X(m, k): XMODE 0 row m of a [M][ldx] array; XMODE 1 h_{t-1} of direction dir (h of the previous step in that
// direction's order, zero at its first step) for position m = b T + t; XMODE 2 row m + shift when that row lies in the
// same run of T rows as m, else zero.
struct RedA {
    const float *a;
    int64_t lda;
    int N;
    const float *r_save;     // AMODE 1
    int hs;                  // AMODE 1
};
struct RedX {
    const float *x;
    int64_t ldx;
    int K;
    int64_t T;               // XMODE 1, 2
    int dir;                 // XMODE 1
    int shift;               // XMODE 2
};

template <int AMODE>
__device__ __forceinline__ float red_a(const RedA &A, int64_t m, int n) {
    float v = A.a[m * A.lda + n];
    if (AMODE == 1 && n >= 2 * A.hs) v *= A.r_save[m * (NDIR * 4 * A.hs) + (n - 2 * A.hs)];
    return v;
}
template <int XMODE>
__device__ __forceinline__ float red_x(const RedX &X, int64_t m, int k) {
    if (XMODE == 0) return X.x[m * X.ldx + k];
    if (XMODE == 2) {        // row m + shift of the same length-T run of rows (a convolution tap), zero outside it
        const int64_t t = m % X.T + X.shift;
        return t >= 0 && t < X.T ? X.x[(m + X.shift) * X.ldx + k] : 0.f;
    }
    const int64_t t = m % X.T;
    if (X.dir ? t == X.T - 1 : t == 0) return 0.f;
    return X.x[(X.dir ? m + 1 : m - 1) * X.ldx + k];
}

// part[s][n][k] = sum over the s-th chunk of rows m of A(m, n) X(m, k): 128 x 128 output tiles, 16 rows per slice,
// 256 threads with 8 x 8 accumulators (gemm_fp32's register tiling with the reduction along M).
constexpr int RT = 128, RM = 16;

template <int AMODE, int XMODE>
__global__ void __launch_bounds__(256) wgrad_kernel(RedA A, RedX X, int64_t M, int64_t chunk, float *__restrict__ part) {
    __shared__ __align__(16) float As[RM][RT];
    __shared__ __align__(16) float Xs[RM][RT];
    const int tid = threadIdx.x;
    const int n0 = blockIdx.x * RT, k0 = blockIdx.y * RT;
    const int64_t m_begin = (int64_t)blockIdx.z * chunk, m_end = min(M, m_begin + chunk);
    const int tx = tid % 16, ty = tid / 16;
    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) acc[i][jj] = 0.f;
    const int lr = tid / 16, lc = tid % 16;     // loader: row lr of the slice, columns lc + 16 q
    for (int64_t m0 = m_begin; m0 < m_end; m0 += RM) {
        const int64_t m = m0 + lr;
        const bool mok = m < m_end;
#pragma unroll
        for (int q = 0; q < RT / 16; ++q) {
            const int c = lc + 16 * q;
            As[lr][c] = mok && n0 + c < A.N ? red_a<AMODE>(A, m, n0 + c) : 0.f;
            Xs[lr][c] = mok && k0 + c < X.K ? red_x<XMODE>(X, m, k0 + c) : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int mm = 0; mm < RM; ++mm) {
            const float4 a0 = *reinterpret_cast<const float4 *>(&As[mm][ty * 4]);
            const float4 a1 = *reinterpret_cast<const float4 *>(&As[mm][64 + ty * 4]);
            const float4 x0 = *reinterpret_cast<const float4 *>(&Xs[mm][tx * 4]);
            const float4 x1 = *reinterpret_cast<const float4 *>(&Xs[mm][64 + tx * 4]);
            const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            const float xv[8] = {x0.x, x0.y, x0.z, x0.w, x1.x, x1.y, x1.z, x1.w};
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int jj = 0; jj < 8; ++jj) acc[i][jj] = fmaf(av[i], xv[jj], acc[i][jj]);
        }
        __syncthreads();
    }
    float *out = part + (int64_t)blockIdx.z * A.N * X.K;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int n = n0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + i - 4);
        if (n >= A.N) continue;
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
            const int k = k0 + (jj < 4 ? tx * 4 + jj : 64 + tx * 4 + jj - 4);
            if (k < X.K) out[(int64_t)n * X.K + k] = acc[i][jj];
        }
    }
}

// part[s][n] = sum over the s-th chunk of rows m of A(m, n)
template <int AMODE>
__global__ void __launch_bounds__(256) colsum_kernel(RedA A, int64_t M, int64_t chunk, float *__restrict__ part) {
    const int n = blockIdx.x * 256 + threadIdx.x;
    if (n >= A.N) return;
    const int64_t m_begin = (int64_t)blockIdx.y * chunk, m_end = min(M, m_begin + chunk);
    float s = 0.f;
    for (int64_t m = m_begin; m < m_end; ++m) s += red_a<AMODE>(A, m, n);
    part[(int64_t)blockIdx.y * A.N + n] = s;
}

// out = sum_s part[s] in order s = 0, 1, ...: element e = n K + k of the [N][K] result goes to dst0 (n < rows) or dst1
// (row n - rows): a reduction over both directions' gi columns lands in the two directions' tensors
__global__ void __launch_bounds__(256) reduce_partials_kernel(const float *__restrict__ part, int splits, int64_t count,
                                                              int K, int rows, float *__restrict__ dst0,
                                                              float *__restrict__ dst1) {
    const int64_t e = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (e >= count) return;
    float s = 0.f;
    for (int i = 0; i < splits; ++i) s += part[(int64_t)i * count + e];
    const int64_t n = e / K;
    if (n < rows) dst0[e] = s;
    else dst1[e - (int64_t)rows * K] = s;
}

// per-block sums of squares of the gradient (double), RED_BLOCKS blocks
__global__ void __launch_bounds__(256) sumsq_kernel(const float *__restrict__ g, int64_t n, double *__restrict__ part) {
    __shared__ double sh[256];
    double v = 0.0;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (int64_t)gridDim.x * 256) {
        const double x = g[i];
        v += x * x;
    }
    v = block_sum(v, sh);
    if (threadIdx.x == 0) part[blockIdx.x] = v;
}

// Per-step scalars of the optimizer rules, computed on the host in double from the step count (torch's formulas)
struct OptStep {
    int kind;
    float lr, alpha, beta1, beta2, eps, weight_decay, momentum, dampening;
    int nesterov, first;         // SGD: nesterov; the momentum buffer is still empty (torch clones the first gradient)
    float step_size, bc2_sqrt;   // Adam: lr / (1 - beta1^t), sqrt(1 - beta2^t)
    float bc2, coef_g, coef_m;   // NAdam: 1 - beta2^t, -lr (1 - mu_t) / (1 - prod mu), -lr mu_{t+1} / (1 - prod mu mu_{t+1})
};

// One optimizer step on the flat master weights.  The gradient norm comes from the sums of squares: a non-finite norm
// skips the step (GradScaler.step), otherwise the gradient is scaled by max_norm / (norm + 1e-6) when that is < 1
// (clip_grad_norm_).  The stored gradient stays unclipped.
__global__ void __launch_bounds__(256) optim_kernel(float *__restrict__ p, const float *__restrict__ grad,
                                                    float *__restrict__ s1, float *__restrict__ s2, int64_t n,
                                                    const double *__restrict__ sumsq, float max_norm, OptStep o) {
    const float norm = (float)sqrt(*sumsq);
    if (!isfinite(norm)) return;
    const float coef = max_norm / (norm + 1e-6f);
    const bool clip = coef < 1.f;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (int64_t)gridDim.x * 256) {
        float g = grad[i];
        if (clip) g *= coef;
        float w = p[i];
        if (o.weight_decay != 0.f) g = fmaf(o.weight_decay, w, g);
        if (o.kind == MDK_OPT_RMSPROP) {
            const float sa = s1[i] * o.alpha + (1.f - o.alpha) * g * g;
            s1[i] = sa;
            const float avg = sqrtf(sa) + o.eps;
            if (o.momentum > 0.f) {
                const float b = s2[i] * o.momentum + g / avg;
                s2[i] = b;
                w = w - o.lr * b;
            } else {
                w = w - o.lr * (g / avg);
            }
        } else if (o.kind == MDK_OPT_ADAM || o.kind == MDK_OPT_NADAM) {
            const float m = s1[i] + (g - s1[i]) * (1.f - o.beta1);
            const float v = s2[i] * o.beta2 + (1.f - o.beta2) * g * g;
            s1[i] = m;
            s2[i] = v;
            if (o.kind == MDK_OPT_ADAM) {
                const float denom = sqrtf(v) / o.bc2_sqrt + o.eps;
                w = w - o.step_size * (m / denom);
            } else {
                const float denom = sqrtf(v / o.bc2) + o.eps;
                w = w + o.coef_g * (g / denom);
                w = w + o.coef_m * (m / denom);
            }
        } else {   // SGD
            if (o.momentum != 0.f) {
                const float b = o.first ? g : s1[i] * o.momentum + (1.f - o.dampening) * g;
                s1[i] = b;
                g = o.nesterov ? g + o.momentum * b : b;
            }
            w = w - o.lr * g;
        }
        p[i] = w;
    }
}

// dst[c][r] = src[r][c]
__global__ void __launch_bounds__(256) transpose_kernel(const float *__restrict__ src, float *__restrict__ dst, int R, int C) {
    __shared__ float tile[32][33];
    const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
    const int tx = threadIdx.x % 32, ty = threadIdx.x / 32;
    for (int i = ty; i < 32; i += 8)
        if (r0 + i < R && c0 + tx < C) tile[i][tx] = src[(int64_t)(r0 + i) * C + c0 + tx];
    __syncthreads();
    for (int i = ty; i < 32; i += 8)
        if (c0 + i < C && r0 + tx < R) dst[(int64_t)(c0 + i) * R + r0 + tx] = tile[tx][i];
}

// Split-M geometry of one reduction over M rows: about two waves of output tiles x splits, chunks of whole slices and
// of at most CHAIN_ROWS rows.  Each partial is a sequential fp32 sum over its chunk, whose rounding error grows with the
// square root of its length: at 100 x 10 000 positions two waves alone make chunks of up to 166 672 rows, which miss a
// signal-bearing gradient by several times the error of torch's fp32 training.  Chunks of at most 4 096 rows keep every
// chain near the lengths the gradient bars were calibrated on; the partials are still added in a fixed order.
struct Split {
    int splits;
    int64_t chunk;
};
constexpr int64_t CHAIN_ROWS = 4096;
static_assert(CHAIN_ROWS % RM == 0, "chunks of whole slices");
static Split split_for(int64_t M, int64_t tiles) {
    int64_t s = std::max<int64_t>(1, (2 * 132 + tiles - 1) / tiles);
    s = std::min<int64_t>(s, std::max<int64_t>(1, M / 256));
    s = std::max<int64_t>(s, (M + CHAIN_ROWS - 1) / CHAIN_ROWS);
    int64_t chunk = (M + s - 1) / s;
    chunk = (chunk + RM - 1) / RM * RM;
    if (chunk == 0) chunk = RM;
    return {(int)((M + chunk - 1) / chunk), chunk};
}


// The per-step scalars of the optimizer rule at step t (1-based) and learning rate lr; *mu_product_out is NAdam's
// running product after this step
inline OptStep opt_step(const mdk_optim_desc &od, float lr, int64_t t, double mu_product_in, double *mu_product_out) {
    OptStep o{};
    o.kind = od.kind; o.lr = lr; o.alpha = od.alpha; o.beta1 = od.beta1; o.beta2 = od.beta2; o.eps = od.eps;
    o.weight_decay = od.weight_decay; o.momentum = od.momentum; o.dampening = od.dampening; o.nesterov = od.nesterov;
    o.first = t == 1;
    const double b1 = od.beta1, b2 = od.beta2;
    const double bc1 = 1.0 - std::pow(b1, (double)t), bc2 = 1.0 - std::pow(b2, (double)t);
    o.step_size = (float)((double)lr / bc1);
    o.bc2_sqrt = (float)std::sqrt(bc2);
    o.bc2 = (float)bc2;
    const double mu = b1 * (1.0 - 0.5 * std::pow(0.96, (double)t * od.momentum_decay));
    const double mu_next = b1 * (1.0 - 0.5 * std::pow(0.96, (double)(t + 1) * od.momentum_decay));
    const double mu_product = mu_product_in * mu;
    o.coef_g = (float)(-(double)lr * (1.0 - mu) / (1.0 - mu_product));
    o.coef_m = (float)(-(double)lr * mu_next / (1.0 - mu_product * mu_next));
    *mu_product_out = mu_product;
    return o;
}

}  // namespace
}  // namespace mdk
