// Read-level consensus network: LatentSpaceLSTM.forward (medaka/architectures/latent_space_lstm.py:154-207) with
// ReadLevelConv (read_level_modules.py:45-78) and MeanPooler (:81-100), SURVEY.md row f4's network half (the feature
// tensor comes from mdk_read_matrix, pileup.cu).
//
//   x int8 [B][P][D][F]  (base, quality, strand, mapQ [, dwell])                      latent_space_lstm.py:163-183
//   e = base_embedder[base] + strand_embedder[strand + 1]  (6) ++ q / 25 - 1 (++ dwell)          :168-183
//   y1 = BN1(ReLU(Conv1d k=1 (7|8 -> C)))          per read, along positions                       read_level_modules.py:31-40
//   y2 = BN2(ReLU(Conv1d k=17, zero padding 8 (C -> C)))
//   z  = mean over the non-empty reads of Linear(C -> H)(y2)                                        :192-197, MeanPooler
//   two bidirectional LSTM layers (H), Linear(2H -> 5), softmax                                    :198-205
// Sizes: C = cnn_size = 128 with H = lstm_size = 128 (the class defaults) or 384 (every released read-level model);
// other sizes are refused.  BatchNorm runs in inference mode (running statistics), in torch's operation order
// ((x - mean) * invstd * weight + bias).
//
// Kernels (the tensor-core ones run by default; mdk_rl_set_conv selects the fp32 CUDA-core twins for validation, and the
// fp16 mode: rl_conv17_fp16_kernel, rl_proj_fp16_kernel, rl_lstm_fp16_kernel and rl_lstm384_fp16_kernel, the FP16 = true
// forms of the four tensor-core kernels' bodies, one fp16 product hi.hi per contraction):
//   rl_mask_kernel        which (window, read) rows are non-empty (x.sum((1, -1)) != 0, :163-165)
//   rl_conv17_tc_kernel   embedding + k = 1 convolution + ReLU + BN1 built in shared memory, the k = 17 convolution as
//                         a wgmma implicit GEMM, ReLU + BN2 and the masked SUM over a group of reads (99 % of the FLOPs)
//     fp32 twin:          rl_embed_conv1_kernel (-> y1 [B][D][P][C]) + rl_conv17_pool_kernel
//   rl_pool_linear_kernel<H>  sum of the read groups / number of reads, then Linear(C -> H).  (The reference applies the
//                         Linear before the mean; the mean of an affine map is the affine map of the mean.)
//   LSTM input projections gi = X W_ih^T + b_ih + b_hh (both directions in one launch): rl_proj_tc_kernel at H = 384,
//                         the fp32 gemm_fp32_kernel (gru_fp32.cu) at H = 128 and on the fp32 path
//   LSTM recurrences      rl_lstm_tc_kernel (H = 128, one CTA per 16-window tile and direction), rl_lstm384_tc_kernel
//                         (H = 384, one 8-CTA cluster per tile and direction); fp32 twin rl_lstm_fp32<H>
//   head                  Linear(2H -> 5) + softmax + argmax: head_kernel (misc.cu, shared with the counts models) at
//                         H = 128, rl_head768_kernel at H = 384; both also write the decoded outputs of
//                         mdk_rl_submit_decoded / mdk_rl_submit_variant_decoded (HEAD_QUALS / HEAD_VARIANT)
#include <string>
#include <unordered_map>
#include <vector>

#include "common.cuh"
#include "phred.cuh"
#include "ptx.cuh"
#include "rec_common.cuh"
#include "rl_common.cuh"

namespace mdk {

constexpr int RL_G4 = 4 * RL_H;

__device__ __forceinline__ float rl_sigmoid(float x) { return 1.0f / (1.0f + expf(-x)); }

// ---------------------------------------------------------------------------------------------- mask
__global__ void __launch_bounds__(256) rl_mask_kernel(const int8_t *__restrict__ x, int64_t P, int D, int F,
                                                      uint8_t *__restrict__ mask) {
    // one block per (b, d): sum over positions and features != 0  (int sum like torch's int64 reduction of int8 input)
    const int64_t b = blockIdx.x / D;
    const int d = (int)(blockIdx.x % D);
    long long s = 0;
    for (int64_t i = threadIdx.x; i < P * F; i += blockDim.x) {
        const int64_t p = i / F;
        const int f = (int)(i % F);
        s += x[((b * P + p) * D + d) * F + f];
    }
    __shared__ long long red[256];
    red[threadIdx.x] = s;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) mask[blockIdx.x] = red[0] != 0;
}

// ---------------------------------------------------------------------------------------------- embedding + conv k=1
__global__ void __launch_bounds__(RL_C) rl_embed_conv1_kernel(const int8_t *__restrict__ x, const uint8_t *__restrict__ mask,
                                                              RlConv1 a, int64_t P, int D, int F, int use_dwells,
                                                              float *__restrict__ y1) {
    // grid: (position chunks of 32, B * D); thread = output channel
    const int64_t bd = blockIdx.y;
    if (!mask[bd]) return;
    const int64_t b = bd / D;
    const int d = (int)(bd % D);
    const int c = threadIdx.x;
    const int nin = RL_EMB + 1 + (use_dwells ? 1 : 0);
    float w[RL_EMB + 2];
    for (int i = 0; i < nin; ++i) w[i] = a.w[c * nin + i];
    const float bias = a.b[c], mean = a.bn_mean[c], invstd = a.bn_invstd[c], bw = a.bn_w[c], bb = a.bn_b[c];
    __shared__ float in[32][RL_EMB + 2];
    const int64_t p0 = (int64_t)blockIdx.x * 32;
    if (threadIdx.x < 32) {
        const int64_t p = p0 + threadIdx.x;
        if (p < P) {
            const int8_t *v = x + ((b * P + p) * D + d) * F;
            const int base = min(max((int)v[0], 0), 5), strand = min(max((int)v[2] + 1, 0), 2);
            for (int i = 0; i < RL_EMB; ++i) in[threadIdx.x][i] = a.emb_base[base * RL_EMB + i] + a.emb_strand[strand * RL_EMB + i];
            in[threadIdx.x][RL_EMB] = (float)v[1] / 25.0f - 1.0f;
            if (use_dwells) in[threadIdx.x][RL_EMB + 1] = (float)v[4];
        }
    }
    __syncthreads();
    for (int i = 0; i < 32; ++i) {
        const int64_t p = p0 + i;
        if (p >= P) break;
        float acc = bias;
        for (int k = 0; k < nin; ++k) acc = fmaf(w[k], in[i][k], acc);
        acc = fmaxf(acc, 0.f);
        y1[(bd * P + p) * RL_C + c] = (acc - mean) * invstd * bw + bb;
    }
}

// ---------------------------------------------------------------------------------------------- conv k=17 + pooling
constexpr int RL_PT = 64;                        // positions per CTA
constexpr int RL_ROWS = RL_PT + 2 * RL_PAD;      // 80 staged input rows
constexpr int RL_YS = RL_C + 4;                  // padded row stride of the staged input
constexpr int RL_KC = 32;                        // input channels per weight chunk
constexpr int RL_CONV_SMEM = (RL_ROWS * RL_YS + RL_KC * RL_C) * 4;

__global__ void __launch_bounds__(256) rl_conv17_pool_kernel(const float *__restrict__ y1, const uint8_t *__restrict__ mask,
                                                             RlConv17 a, int64_t P, int D, int dgroup,
                                                             float *__restrict__ partial) {
    // grid: (position tiles, read groups, B).  partial [B][n_groups][P][C]
    extern __shared__ __align__(16) float smem_rl[];
    float *ys = smem_rl;                      // [80][132]
    float *ws = smem_rl + RL_ROWS * RL_YS;    // [32][128]
    const int tid = threadIdx.x;
    const int tx = tid % 16, ty = tid / 16;   // 16 channel groups of 8, 16 position groups of 4
    const int64_t b = blockIdx.z;
    const int g = blockIdx.y;
    const int64_t p0 = (int64_t)blockIdx.x * RL_PT;
    float bias[8], mean[8], invstd[8], bw[8], bb[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int c = tx * 8 + j;
        bias[j] = a.b[c]; mean[j] = a.bn_mean[c]; invstd[j] = a.bn_invstd[c]; bw[j] = a.bn_w[c]; bb[j] = a.bn_b[c];
    }
    float pooled[4][8];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) pooled[i][j] = 0.f;
    const int d0 = g * dgroup, d1 = min(D, d0 + dgroup);
    for (int d = d0; d < d1; ++d) {
        const int64_t bd = b * D + d;
        if (!mask[bd]) continue;                                   // (uniform over the CTA)
        __syncthreads();
        // stage rows p0-8 .. p0+71 of this read's y1, zeros outside [0, P)  (Conv1d zero padding)
        for (int i = tid; i < RL_ROWS * (RL_C / 4); i += 256) {
            const int r = i / (RL_C / 4), q = i % (RL_C / 4);
            const int64_t p = p0 - RL_PAD + r;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (p >= 0 && p < P) v = *reinterpret_cast<const float4 *>(y1 + (bd * P + p) * RL_C + q * 4);
            *reinterpret_cast<float4 *>(ys + r * RL_YS + q * 4) = v;
        }
        float acc[4][8];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
        for (int t = 0; t < RL_TAPS; ++t) {
            for (int cc = 0; cc < RL_C / RL_KC; ++cc) {
                __syncthreads();                                   // previous chunk consumed (and ys staged)
                const float *wsrc = a.w_t + ((size_t)t * RL_C + cc * RL_KC) * RL_C;
                for (int i = tid; i < RL_KC * RL_C / 4; i += 256)
                    reinterpret_cast<float4 *>(ws)[i] = reinterpret_cast<const float4 *>(wsrc)[i];
                __syncthreads();
#pragma unroll 4
                for (int k = 0; k < RL_KC; ++k) {
                    float av[4];
#pragma unroll
                    for (int i = 0; i < 4; ++i) av[i] = ys[(ty * 4 + i + t) * RL_YS + cc * RL_KC + k];
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
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float v = fmaxf(acc[i][j] + bias[j], 0.f);
                pooled[i][j] += (v - mean[j]) * invstd[j] * bw[j] + bb[j];
            }
    }
    const int n_groups = gridDim.y;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int64_t p = p0 + ty * 4 + i;
        if (p >= P) continue;
        float *dst = partial + (((b * n_groups + g) * P + p) * RL_C) + tx * 8;
        *reinterpret_cast<float4 *>(dst) = make_float4(pooled[i][0], pooled[i][1], pooled[i][2], pooled[i][3]);
        *reinterpret_cast<float4 *>(dst + 4) = make_float4(pooled[i][4], pooled[i][5], pooled[i][6], pooled[i][7]);
    }
}

// ---------------------------------------------------------------------------------------------- conv k=17 on wgmma
// The same convolution as an implicit GEMM on the tensor cores:  D[co][p] = sum_t sum_ci W[co][ci][t] . y1[p + t - 8][ci].
//   A = one tap's weights [128 co][128 ci]  (K-major fp16 hi | lo planes, pre-tiled in HBM, streamed through a two-stage
//       shared-memory ring with bulk copies: 17 x 64 KiB of weights do not fit shared memory)
//   B = ONE staged activation tile [144 positions][128 ci] (hi | lo) serves all 17 taps: tap t is the same buffer with the
//       descriptor's start address moved down t rows (K-major, no swizzle: a row is 16 bytes inside its k-group block)
//   D = registers, M64 N128 per warpgroup (warpgroup g: output channels 64g .. 64g + 63); three fp16 products per
//       contraction like the GRU kernels (fp32-faithful)
// FP16 (the fp16 mode): one product, W_hi . y1_hi.  The activation tile is one plane, and the ring streams only the 17 hi
// planes of the same pre-tiled weights: 8 MMAs per tap.
// A CTA owns (window b, 128 positions, a group of reads): for each read it builds the activation tile in shared memory
// straight from the int8 features (embedding + k = 1 convolution + ReLU + BN1, never written to HBM), runs 17 x 24 MMAs
// against one pass of the weights, folds the accumulators through ReLU + BN2 into per-thread sums, and writes the
// group's sum once.
constexpr int CT_NPOS = 128;
constexpr int CT_ROWS = CT_NPOS + 2 * RL_PAD;            // 144 staged positions
constexpr int CT_BPLANE = (RL_C / 8) * CT_ROWS * 16;     // 36 864 B
constexpr int CT_BTILE = 2 * CT_BPLANE;                  // hi + lo of one read's activation tile
constexpr int CT_WPLANE = (RL_C / 8) * RL_C * 16;        // 32 768 B: one plane of one tap = one ring stage
constexpr int CT_STAGES = 2;
template <bool FP16> constexpr int CT_OFF_W = FP16 ? CT_BPLANE : CT_BTILE;
template <bool FP16> constexpr int CT_OFF_IN = CT_OFF_W<FP16> + CT_STAGES * CT_WPLANE;
template <bool FP16> constexpr int CT_OFF_BAR = CT_OFF_IN<FP16> + CT_ROWS * 8 * 4;
template <bool FP16> constexpr int CT_SMEM = CT_OFF_BAR<FP16> + 64;

template <bool FP16>
__device__ __forceinline__ void rl_conv17_body(const int8_t *__restrict__ x, const uint8_t *__restrict__ mask, RlConv1 c1,
                                               RlConv17 c17, const uint8_t *__restrict__ w_tc, int64_t P, int D, int F,
                                               int use_dwells, int dgroup, float *__restrict__ partial) {
    extern __shared__ __align__(128) uint8_t smem_ct[];
    uint8_t *sb = smem_ct;                                             // [hi | lo][k-group][144][8 halfs]
    uint8_t *sw = smem_ct + CT_OFF_W<FP16>;                            // [stage][k-group][128][8 halfs]
    float *sin = reinterpret_cast<float *>(smem_ct + CT_OFF_IN<FP16>); // [144][8]
    uint64_t *full = reinterpret_cast<uint64_t *>(smem_ct + CT_OFF_BAR<FP16>);
    constexpr int NPLANES = FP16 ? RL_TAPS : 2 * RL_TAPS;             // weight planes per read
    const int tid = threadIdx.x, wg = tid >> 7, warp = (tid >> 5) & 3, lane = tid & 31;
    const int gq = lane >> 2, cq = lane & 3;
    const int64_t b = blockIdx.z;
    const int g = blockIdx.y;
    const int64_t p0 = (int64_t)blockIdx.x * CT_NPOS;
    const int nin = RL_EMB + 1 + (use_dwells ? 1 : 0);

    if (tid == 0) {
        for (int i = 0; i < CT_STAGES; ++i) mbar_init(&full[i], 1);
        fence_mbar_init();
    }
    __syncthreads();

    // builder constants: this thread's k = 1 convolution channel
    const int bc = tid & 127;
    float w1[RL_EMB + 2];
    for (int i = 0; i < nin; ++i) w1[i] = c1.w[bc * nin + i];
    const float b1 = c1.b[bc], m1 = c1.bn_mean[bc], s1 = c1.bn_invstd[bc], g1 = c1.bn_w[bc], o1 = c1.bn_b[bc];
    // epilogue constants: this thread's output channels co0 and co0 + 8 (accumulator rows)
    const int co0 = wg * 64 + warp * 16 + gq;
    float b2[2], m2[2], s2[2], g2[2], o2[2];
    for (int hb = 0; hb < 2; ++hb) {
        const int co = co0 + 8 * hb;
        b2[hb] = c17.b[co]; m2[hb] = c17.bn_mean[co]; s2[hb] = c17.bn_invstd[co]; g2[hb] = c17.bn_w[co]; o2[hb] = c17.bn_b[co];
    }
    float pooled[64], acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) pooled[i] = 0.f;
    const int d0 = g * dgroup, d1 = min(D, d0 + dgroup);
    uint32_t it = 0;             // weight-plane stages consumed so far
    auto issue = [&](uint32_t k) {   // stage k of the running sequence = plane (k % 34) of the taps (FP16: tap k % 17's hi)
        const uint32_t st = k % CT_STAGES;
        const uint8_t *src = w_tc + (size_t)(FP16 ? k % RL_TAPS * 2 : k % (2 * RL_TAPS)) * CT_WPLANE;   // [tap][hi | lo]
        mbar_arrive_expect_tx(&full[st], CT_WPLANE);
        bulk_g2s(sw + st * CT_WPLANE, src, CT_WPLANE, &full[st]);
    };
    for (int d = d0; d < d1; ++d) {
        if (!mask[b * D + d]) continue;                            // uniform over the CTA
        // ---- build the activation tile (the previous read's MMAs are complete)
        if (tid < CT_ROWS) {
            const int64_t p = p0 - RL_PAD + tid;
            float *row = sin + tid * 8;
            if (p >= 0 && p < P) {
                const int8_t *v = x + ((b * P + p) * D + d) * F;
                const int base = min(max((int)v[0], 0), 5), strand = min(max((int)v[2] + 1, 0), 2);
                for (int i = 0; i < RL_EMB; ++i) row[i] = c1.emb_base[base * RL_EMB + i] + c1.emb_strand[strand * RL_EMB + i];
                row[RL_EMB] = (float)v[1] / 25.0f - 1.0f;
                row[RL_EMB + 1] = use_dwells ? (float)v[4] : 0.f;
            } else {
                row[0] = __int_as_float(0x7fc00000);              // marker: outside the window -> zero row (conv padding)
            }
        }
        if (tid == 0) {                                            // the first two weight planes of this read
            issue(it);
            issue(it + 1);
        }
        __syncthreads();
        for (int r = tid >> 7; r < CT_ROWS; r += 2) {
            const float *row = sin + r * 8;
            float y = 0.f;
            if (!(row[0] != row[0])) {
                float a = b1;
                for (int k = 0; k < nin; ++k) a = fmaf(w1[k], row[k], a);
                a = fmaxf(a, 0.f);
                y = (a - m1) * s1 * g1 + o1;
            }
            __half hi, lo;
            split_f16(y, hi, lo);
            const int off = (bc >> 3) * (CT_ROWS * 16) + r * 16 + (bc & 7) * 2;
            *reinterpret_cast<__half *>(sb + off) = hi;
            if (!FP16) *reinterpret_cast<__half *>(sb + CT_BPLANE + off) = lo;
        }
        fence_proxy_async_smem();
        __syncthreads();
        // ---- 17 taps x (hi plane, lo plane) of the weights.  Each plane starts a fresh wgmma accumulator (16 or 8 MMAs
        // deep) that is added into the fp32 sum on the CUDA cores: one accumulator chained over all 34 planes (400 MMAs,
        // K = 17 x 128 x 3) lost ~10x the fp32 path's accuracy on the pooled output in the tensor core's accumulation.
        // FP16 keeps the per-tap accumulators: 17 hi planes, 8 MMAs each.
        float sum[64];
#pragma unroll
        for (int k = 0; k < 64; ++k) sum[k] = 0.f;
        for (int ps = 0; ps < NPLANES; ++ps, ++it) {
            const uint32_t st = it % CT_STAGES;
            const int t = FP16 ? ps : ps >> 1, lo_plane = FP16 ? 0 : ps & 1;
            mbar_wait(&full[st], (it / CT_STAGES) & 1);
            wg_fence();
            const uint32_t a0 = smem_u32(sw + st * CT_WPLANE) + wg * 64 * 16;
            const uint32_t bb0 = smem_u32(sb) + (uint32_t)t * 16u;
            // hi plane of the weights: x activation hi, then x activation lo;  lo plane: x activation hi
#pragma unroll
            for (int ks = 0; ks < RL_C / 16; ++ks) {
                const uint64_t ad = make_smem_desc(a0 + ks * 2 * (RL_C * 16), RL_C * 16, 128);
                const uint64_t bh = make_smem_desc(bb0 + ks * 2 * (CT_ROWS * 16), CT_ROWS * 16, 128);
                Wgmma<128>::ss(acc, ad, bh, ks ? 1u : 0u);
                if (!FP16 && !lo_plane) Wgmma<128>::ss(acc, ad, make_smem_desc(bb0 + CT_BPLANE + ks * 2 * (CT_ROWS * 16), CT_ROWS * 16, 128), 1u);
            }
            wg_commit();
            wg_wait_all();
            wg_hold(acc);
            __syncthreads();                                       // both warpgroups have read stage st
            if (tid == 0 && ps + 2 < NPLANES) issue(it + 2);
#pragma unroll
            for (int k = 0; k < 64; ++k) sum[k] += acc[k];
        }
#pragma unroll
        for (int k = 0; k < 64; ++k) {
            const int hb = (k >> 1) & 1;
            const float av = fmaxf(sum[k] + b2[hb], 0.f);
            pooled[k] += (av - m2[hb]) * s2[hb] * g2[hb] + o2[hb];
        }
    }
    const int n_groups = gridDim.y;
    float *dst = partial + ((b * n_groups + g) * P + p0) * RL_C + co0;
#pragma unroll
    for (int k = 0; k < 64; ++k) {
        const int n = 8 * (k >> 2) + 2 * cq + (k & 1);
        if (p0 + n < P) dst[(int64_t)n * RL_C + 8 * ((k >> 1) & 1)] = pooled[k];
    }
}

__global__ void __launch_bounds__(256, 1) rl_conv17_tc_kernel(const int8_t *__restrict__ x, const uint8_t *__restrict__ mask,
                                                              RlConv1 c1, RlConv17 c17, const uint8_t *__restrict__ w_tc,
                                                              int64_t P, int D, int F, int use_dwells, int dgroup,
                                                              float *__restrict__ partial) {
    rl_conv17_body<false>(x, mask, c1, c17, w_tc, P, D, F, use_dwells, dgroup, partial);
}
__global__ void __launch_bounds__(256, 1) rl_conv17_fp16_kernel(const int8_t *__restrict__ x, const uint8_t *__restrict__ mask,
                                                                RlConv1 c1, RlConv17 c17, const uint8_t *__restrict__ w_tc,
                                                                int64_t P, int D, int F, int use_dwells, int dgroup,
                                                                float *__restrict__ partial) {
    rl_conv17_body<true>(x, mask, c1, c17, w_tc, P, D, F, use_dwells, dgroup, partial);
}

// ---------------------------------------------------------------------------------------------- mean + Linear(C -> H)
constexpr int RL_PLT = 16;        // positions per CTA of the pooling kernel
template <int HO>                 // output width H: 128 threads, each owns HO / 128 output units
__global__ void __launch_bounds__(RL_C) rl_pool_linear_kernel(const float *__restrict__ partial, const uint8_t *__restrict__ mask,
                                                              const float *__restrict__ w_t, const float *__restrict__ bias,
                                                              int64_t P, int D, int n_groups, float *__restrict__ out) {
    // grid: (position tiles of 16, B); thread = channel while summing, output unit(s) afterwards.  w_t [C k][HO] (transposed)
    constexpr int U = HO / RL_C;
    const int64_t b = blockIdx.y, p0 = (int64_t)blockIdx.x * RL_PLT;
    __shared__ float v[RL_PLT][RL_C];
    __shared__ int n_reads;
    if (threadIdx.x == 0) {
        int n = 0;
        for (int d = 0; d < D; ++d) n += mask[b * D + d];
        n_reads = n;
    }
    __syncthreads();
    for (int i = 0; i < RL_PLT; ++i) {
        const int64_t p = p0 + i;
        float s = 0.f;
        if (p < P)
            for (int g = 0; g < n_groups; ++g) s += partial[((b * n_groups + g) * P + p) * RL_C + threadIdx.x];
        v[i][threadIdx.x] = s / (float)n_reads;            // 0 / 0 = nan when a window has no reads, like the reference
    }
    __syncthreads();
    const int h = threadIdx.x;
    float acc[U][RL_PLT];
#pragma unroll
    for (int u = 0; u < U; ++u)
#pragma unroll
        for (int i = 0; i < RL_PLT; ++i) acc[u][i] = bias[h + u * RL_C];
    for (int k = 0; k < RL_C; ++k) {
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const float w = w_t[k * HO + h + u * RL_C];
#pragma unroll
            for (int i = 0; i < RL_PLT; ++i) acc[u][i] = fmaf(w, v[i][k], acc[u][i]);
        }
    }
#pragma unroll
    for (int u = 0; u < U; ++u)
#pragma unroll
        for (int i = 0; i < RL_PLT; ++i)
            if (p0 + i < P) out[(b * P + p0 + i) * HO + h + u * RL_C] = acc[u][i];
}

// ---------------------------------------------------------------------------------------------- LSTM recurrence, fp32
// gi  [B*P][2 dirs][4H]  (torch gate order i, f, g, o; b_ih + b_hh folded in)
// out [B*P][2H]          (columns dir*H + j)
// w_t [dir][H k][4H]     W_hh^T
// The recurrence on the CUDA cores (validation path, both sizes): one CTA = 8 windows of one direction, thread = hidden
// unit j with all four gates, W_hh^T read from global memory (L2-resident: 0.26 MB per direction at H = 128, 2.36 MB at
// 384), h in shared memory.  SAVE (training) also keeps the gates i, f, g, o and the cell c of every position:
// save [B*P][2 dirs][5H].
constexpr int LF_NB = 8;
template <int H, bool SAVE>
__global__ void __launch_bounds__(H) rl_lstm_fp32(const float *__restrict__ gi, const float *__restrict__ wt,
                                                  float *__restrict__ out, int64_t B, int64_t P,
                                                  float *__restrict__ save) {
    __shared__ __align__(16) float hs[LF_NB][H];
    const int j = threadIdx.x;
    const int dir = blockIdx.y;
    const int64_t b0 = (int64_t)blockIdx.x * LF_NB;
    const int nb = (int)min((int64_t)LF_NB, B - b0);
    const float *w = wt + (size_t)dir * H * (4 * H) + j;
#pragma unroll
    for (int n = 0; n < LF_NB; ++n) hs[n][j] = 0.f;
    float c_state[LF_NB];
#pragma unroll
    for (int n = 0; n < LF_NB; ++n) c_state[n] = 0.f;
    __syncthreads();
    for (int64_t step = 0; step < P; ++step) {
        const int64_t t = dir ? (P - 1 - step) : step;
        float a[4][LF_NB];
#pragma unroll
        for (int n = 0; n < LF_NB; ++n) {
            const bool ok = n < nb;
            const float *row = gi + (((b0 + (ok ? n : 0)) * P + t) * 2 + dir) * (4 * H) + j;
#pragma unroll
            for (int g = 0; g < 4; ++g) a[g][n] = ok ? __ldg(row + g * H) : 0.f;
        }
#pragma unroll 4
        for (int k = 0; k < H; ++k) {
            float wv[4];
#pragma unroll
            for (int g = 0; g < 4; ++g) wv[g] = __ldg(w + (size_t)k * (4 * H) + g * H);
#pragma unroll
            for (int n = 0; n < LF_NB; ++n) {
                const float hk = hs[n][k];
#pragma unroll
                for (int g = 0; g < 4; ++g) a[g][n] = fmaf(wv[g], hk, a[g][n]);
            }
        }
        __syncthreads();                                     // every thread has read h of the previous step
#pragma unroll
        for (int n = 0; n < LF_NB; ++n) {
            const float ig = rl_sigmoid(a[0][n]), fg = rl_sigmoid(a[1][n]), gg = tanhf(a[2][n]), og = rl_sigmoid(a[3][n]);
            const float c = fg * c_state[n] + ig * gg;
            c_state[n] = c;
            const float h = og * tanhf(c);
            hs[n][j] = h;
            if (n < nb) out[((b0 + n) * P + t) * (2 * H) + dir * H + j] = h;
            if (SAVE && n < nb) {
                float *sv = save + (((b0 + n) * P + t) * 2 + dir) * (5 * H) + j;
                sv[0] = ig; sv[H] = fg; sv[2 * H] = gg; sv[3 * H] = og; sv[4 * H] = c;
            }
        }
        __syncthreads();
    }
}

// ---------------------------------------------------------------------------------------------- LSTM on wgmma
// The recurrence with the matvec on the tensor cores:  G^T[4H][16 windows] = W_hh[4H][H] . h^T[H][16]  per time step.
//   A = W_hh: the fp16 hi plane of all four gates stays in REGISTERS (the register form of wgmma; warpgroup g holds
//       hidden units 64g .. 64g + 63 of every gate), the lo plane is a shared-memory operand (pre-tiled per direction)
//   B = the h tile [16 windows][128] (fp16 hi | lo, K-major, double buffered: step t reads buffer t & 1)
//   D = four M64 N16 accumulators per warpgroup, preloaded with the input pre-activations; three products per
//       contraction: W_hi.h_hi, W_hi.h_lo, W_lo.h_hi
// One CTA = 16 windows of one direction, two warpgroups; c and h stay in registers.  FP16 (the fp16 mode): one product,
// W_hi.h_hi; no lo plane in shared memory, and the h tile holds h's hi plane only.
constexpr int LT_N = 16;
constexpr int LT_WLO_GATE = (RL_H / 8) * RL_H * 16;          // 32 768 B: one gate's lo plane as A operand tiles
constexpr int LT_KG = LT_N * 16 + 16;                        // k-group stride of the h tile (+16 B spreads the stores)
constexpr int LT_HPLANE = (RL_H / 8) * LT_KG;
template <bool FP16> constexpr int LT_OFF_H = FP16 ? 0 : 4 * LT_WLO_GATE;
template <bool FP16> constexpr int LT_SMEM = LT_OFF_H<FP16> + 4 * LT_HPLANE;
constexpr int LT_THREADS = 256;
// element (direction d, gate row r, column k) of W_hh's lo plane in the tiles above: [dir][gate][k-group][row][8 halfs]
inline size_t lt_lo_index(int d, int r, int k) {
    return ((((size_t)d * 4 + r / RL_H) * (RL_H / 8) + k / 8) * RL_H + r % RL_H) * 8 + k % 8;
}
// MUFU-based gate functions (ex2.approx / rcp.approx, ~2 ulp)
__device__ __forceinline__ float lt_sigmoid(float x) { return rcp_approx(1.0f + ex2_approx(-1.4426950408889634f * x)); }
__device__ __forceinline__ float lt_tanh(float x) { return fmaf(-2.0f, rcp_approx(1.0f + ex2_approx(2.8853900817779268f * x)), 1.0f); }

template <bool FP16>
__device__ __forceinline__ void rl_lstm_body(const float *__restrict__ gi, const __half *__restrict__ w_hi,
                                             const uint8_t *__restrict__ w_lo_tiles, float *__restrict__ out, int64_t B,
                                             int64_t P) {
    extern __shared__ __align__(128) uint8_t smem_lt[];
    uint8_t *swlo = smem_lt;
    uint8_t *sh = smem_lt + LT_OFF_H<FP16>;                      // [buf 2][hi | lo] LT_HPLANE
    const int tid = threadIdx.x, wg = tid >> 7, warp = (tid >> 5) & 3, lane = tid & 31;
    const int gq = lane >> 2, cq = lane & 3;
    const int dir = blockIdx.y;
    const int64_t b0 = (int64_t)blockIdx.x * LT_N;
    const int nb = (int)min((int64_t)LT_N, B - b0);
    const int j0 = wg * 64 + warp * 16 + gq;                   // hidden units j0 and j0 + 8
    {
        const uint4 *src = reinterpret_cast<const uint4 *>(w_lo_tiles + (size_t)dir * 4 * LT_WLO_GATE);
        if (!FP16)
            for (int i = tid; i < 4 * LT_WLO_GATE / 16; i += LT_THREADS) reinterpret_cast<uint4 *>(swlo)[i] = src[i];
        for (int i = tid; i < 4 * LT_HPLANE / 16; i += LT_THREADS) reinterpret_cast<uint4 *>(sh)[i] = make_uint4(0u, 0u, 0u, 0u);
    }
    uint32_t whi[4][RL_H / 16][4];
#pragma unroll
    for (int g = 0; g < 4; ++g)
#pragma unroll
        for (int ks = 0; ks < RL_H / 16; ++ks) {
            const __half *w = w_hi + (((size_t)dir * 4 + g) * RL_H + j0) * RL_H + ks * 16 + 2 * cq;
            whi[g][ks][0] = *reinterpret_cast<const uint32_t *>(w);
            whi[g][ks][1] = *reinterpret_cast<const uint32_t *>(w + 8 * RL_H);
            whi[g][ks][2] = *reinterpret_cast<const uint32_t *>(w + 8);
            whi[g][ks][3] = *reinterpret_cast<const uint32_t *>(w + 8 * RL_H + 8);
        }
    // accumulator element k = 4i + 2hb + e: hidden unit j0 + 8hb, window 8i + 2cq + e
    float acc[4][8], c_state[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) c_state[k] = 0.f;
    auto fetch = [&](int64_t t) {
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int wdw = 8 * (k >> 2) + 2 * cq + (k & 1);
            const bool ok = wdw < nb;
            const float *row = gi + (((b0 + (ok ? wdw : 0)) * P + t) * 2 + dir) * RL_G4 + j0 + 8 * ((k >> 1) & 1);
#pragma unroll
            for (int g = 0; g < 4; ++g) acc[g][k] = ok ? __ldg(row + g * RL_H) : 0.f;
        }
    };
    fetch(dir ? (P - 1) : 0);
    fence_proxy_async_smem();
    __syncthreads();
    const uint32_t wl = smem_u32(swlo) + wg * 64 * 16;
    for (int64_t step = 0; step < P; ++step) {
        const int64_t t = dir ? (P - 1 - step) : step;
        const int buf = (int)(step & 1);
        const uint32_t h_hi = smem_u32(sh + buf * 2 * LT_HPLANE), h_lo = h_hi + LT_HPLANE;
        wg_fence();
#pragma unroll
        for (int g = 0; g < 4; ++g)
#pragma unroll
            for (int ks = 0; ks < RL_H / 16; ++ks) {
                const uint64_t bh = make_smem_desc(h_hi + ks * 2 * LT_KG, LT_KG, 128);
                Wgmma<16>::rs(acc[g], whi[g][ks], bh, 1u);
                if (FP16) continue;
                Wgmma<16>::rs(acc[g], whi[g][ks], make_smem_desc(h_lo + ks * 2 * LT_KG, LT_KG, 128), 1u);
                Wgmma<16>::ss(acc[g], make_smem_desc(wl + g * LT_WLO_GATE + ks * 2 * (RL_H * 16), RL_H * 16, 128), bh, 1u);
            }
        wg_commit();
        wg_wait_all();
#pragma unroll
        for (int g = 0; g < 4; ++g) wg_hold(acc[g]);
        uint8_t *hw = sh + (buf ^ 1) * 2 * LT_HPLANE;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const float ig = lt_sigmoid(acc[0][k]);
            const float fg = lt_sigmoid(acc[1][k]);
            const float gg = lt_tanh(acc[2][k]);
            const float og = lt_sigmoid(acc[3][k]);
            const float c = fmaf(fg, c_state[k], ig * gg);
            c_state[k] = c;
            const float h = og * lt_tanh(c);
            const int wdw = 8 * (k >> 2) + 2 * cq + (k & 1), j = j0 + 8 * ((k >> 1) & 1);
            if (wdw < nb) out[((b0 + wdw) * P + t) * (2 * RL_H) + dir * RL_H + j] = h;
            __half hi, lo;
            split_f16(h, hi, lo);
            *reinterpret_cast<__half *>(hw + (j >> 3) * LT_KG + wdw * 16 + (j & 7) * 2) = hi;
            if (!FP16) *reinterpret_cast<__half *>(hw + LT_HPLANE + (j >> 3) * LT_KG + wdw * 16 + (j & 7) * 2) = lo;
        }
        if (step + 1 < P) fetch(dir ? (t - 1) : (t + 1));
        fence_proxy_async_smem();
        __syncthreads();
    }
}

__global__ void __launch_bounds__(LT_THREADS, 1) rl_lstm_tc_kernel(const float *__restrict__ gi, const __half *__restrict__ w_hi,
                                                                   const uint8_t *__restrict__ w_lo_tiles,
                                                                   float *__restrict__ out, int64_t B, int64_t P) {
    rl_lstm_body<false>(gi, w_hi, w_lo_tiles, out, B, P);
}
__global__ void __launch_bounds__(LT_THREADS, 1) rl_lstm_fp16_kernel(const float *__restrict__ gi, const __half *__restrict__ w_hi,
                                                                     const uint8_t *__restrict__ w_lo_tiles,
                                                                     float *__restrict__ out, int64_t B, int64_t P) {
    rl_lstm_body<true>(gi, w_hi, w_lo_tiles, out, B, P);
}

// ============================================================================================== lstm_size = 384
// Every released read-level model is `..._rl_lstm384_...`: H = 384 with C = 128.  The convolution and the mask are the
// kernels above; the pooling Linear is rl_pool_linear_kernel<384>.  What changes is the LSTM: W_hh is 4H x H per
// direction (2.25 MiB as fp16 hi + lo, more than one SM holds) and the input projections grow nine-fold (7.1 MFLOP per
// position for both layers and directions), so both get tensor-core kernels of their own.  The fp32 twins
// (rl_lstm_fp32, gemm_fp32_kernel) serve both sizes.
constexpr int RL_G43 = 4 * RL_H3;                  // 1536 gate rows per direction

// ---------------------------------------------------------------------------------------------- projections on wgmma
// gi[M][N] = X[M][K] . W[N][K]^T + bias[N]  (N = 2 dirs x 4H = 3072: both directions in one launch, K = 384 or 768)
// in the transposed formulation: D[128 gate rows][128 positions] per CTA, warpgroup g owns gate rows 64g .. 64g + 63.
//   A = W, pre-tiled per (128-row block, 64-wide K chunk) as [hi | lo][k-group 8][row 128][8 halfs] (32 KiB, one bulk copy)
//   B = X, read as fp32 and split into fp16 hi / lo while it is staged ([hi | lo][k-group 8][position 128][8 halfs])
// K runs in 64-wide chunks through two stages: while the 12 MMAs of chunk c run, the threads stage the activations of
// chunk c + 1 and the bulk copy brings its weights.  Three products per contraction (DESIGN §3); FP16 (the fp16 mode):
// one, W_hi . X_hi: the bulk copy brings the hi half of each weight chunk and X is staged as its hi plane, 4 MMAs per
// chunk.
constexpr int PJ_M = 128;
constexpr int PJ_N = 128;
constexpr int PJ_KC = 64;
constexpr int PJ_WPLANE = (PJ_KC / 8) * PJ_M * 16;          // 16 KiB
constexpr int PJ_XPLANE = (PJ_KC / 8) * PJ_N * 16;          // 16 KiB
constexpr int PJ_WCHUNK = 2 * PJ_WPLANE;                    // hi + lo of one weight chunk (the pre-tiled unit in HBM)
constexpr int PJ_STAGE = PJ_WCHUNK + 2 * PJ_XPLANE;         // 64 KiB
constexpr int PJ_OFF_BAR = 2 * PJ_STAGE;
constexpr int PJ_SMEM = PJ_OFF_BAR + 64;

template <bool FP16>
__device__ __forceinline__ void rl_proj_body(const float *__restrict__ X, const uint8_t *__restrict__ w_tc,
                                             const float *__restrict__ bias, float *__restrict__ C, int64_t M, int K, int N) {
    extern __shared__ __align__(128) uint8_t smem_pj[];
    uint64_t *full = reinterpret_cast<uint64_t *>(smem_pj + PJ_OFF_BAR);
    const int tid = threadIdx.x, wg = tid >> 7, warp = (tid >> 5) & 3, lane = tid & 31;
    const int gq = lane >> 2, cq = lane & 3;
    const int64_t m0 = (int64_t)blockIdx.x * PJ_N;
    const int rb = blockIdx.y;
    const int nchunks = K / PJ_KC;
    if (tid == 0) {
        mbar_init(&full[0], 1);
        mbar_init(&full[1], 1);
        fence_mbar_init();
    }
    __syncthreads();
    auto issue_w = [&](int c) {
        const int st = c & 1;
        constexpr int bytes = FP16 ? PJ_WPLANE : PJ_WCHUNK;
        mbar_arrive_expect_tx(&full[st], bytes);
        bulk_g2s(smem_pj + st * PJ_STAGE, w_tc + ((size_t)rb * nchunks + c) * PJ_WCHUNK, bytes, &full[st]);
    };
    auto stage_x = [&](int c) {
        uint8_t *xs = smem_pj + (c & 1) * PJ_STAGE + PJ_WCHUNK;
        // 128 positions x 64 k: a lane pair reads one 32-byte sector (8 k of one position) and writes one 16-byte row
#pragma unroll 2
        for (int i = tid; i < PJ_N * PJ_KC / 4; i += 256) {
            const int q2 = i & 1, n = (i >> 1) & (PJ_N - 1), kg = i >> 8;
            const int64_t p = m0 + n;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (p < M) v = *reinterpret_cast<const float4 *>(X + p * K + c * PJ_KC + kg * 8 + q2 * 4);
            __half h0, h1, h2, h3, l0, l1, l2, l3;
            split_f16(v.x, h0, l0); split_f16(v.y, h1, l1); split_f16(v.z, h2, l2); split_f16(v.w, h3, l3);
            const int off = kg * (PJ_N * 16) + n * 16 + q2 * 8;
            __half2 hv[2] = {__halves2half2(h0, h1), __halves2half2(h2, h3)};
            __half2 lv[2] = {__halves2half2(l0, l1), __halves2half2(l2, l3)};
            *reinterpret_cast<uint2 *>(xs + off) = *reinterpret_cast<uint2 *>(hv);
            if (!FP16) *reinterpret_cast<uint2 *>(xs + PJ_XPLANE + off) = *reinterpret_cast<uint2 *>(lv);
        }
    };
    // each 64-wide K chunk runs in a fresh accumulator (12 MMAs) that is added into the fp32 sum on the CUDA cores: one
    // chain over all of K (144 MMAs at K = 768) lost accuracy in the tensor core's accumulation
    float acc[64], sum[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) sum[i] = 0.f;
    if (tid == 0) issue_w(0);
    stage_x(0);
    fence_proxy_async_smem();
    for (int c = 0; c < nchunks; ++c) {
        const int st = c & 1;
        __syncthreads();             // activations of chunk c staged and fenced; stage st ^ 1 no longer read (chunk c - 1)
        if (tid == 0 && c + 1 < nchunks) issue_w(c + 1);
        mbar_wait(&full[st], (uint32_t)(c >> 1) & 1u);
        wg_fence();
        const uint32_t wbase = smem_u32(smem_pj + st * PJ_STAGE) + wg * 64 * 16;
        const uint32_t xbase = smem_u32(smem_pj + st * PJ_STAGE + PJ_WCHUNK);
#pragma unroll
        for (int ks = 0; ks < PJ_KC / 16; ++ks) {
            const uint64_t ah = make_smem_desc(wbase + ks * 2 * (PJ_M * 16), PJ_M * 16, 128);
            const uint64_t al = make_smem_desc(wbase + PJ_WPLANE + ks * 2 * (PJ_M * 16), PJ_M * 16, 128);
            const uint64_t bh = make_smem_desc(xbase + ks * 2 * (PJ_N * 16), PJ_N * 16, 128);
            const uint64_t bl = make_smem_desc(xbase + PJ_XPLANE + ks * 2 * (PJ_N * 16), PJ_N * 16, 128);
            Wgmma<128>::ss(acc, ah, bh, ks ? 1u : 0u);
            if (!FP16) {
                Wgmma<128>::ss(acc, ah, bl, 1u);
                Wgmma<128>::ss(acc, al, bh, 1u);
            }
        }
        wg_commit();
        if (c + 1 < nchunks) {
            stage_x(c + 1);
            fence_proxy_async_smem();
        }
        wg_wait_all();
        wg_hold(acc);
#pragma unroll
        for (int i = 0; i < 64; ++i) sum[i] += acc[i];
    }
    // accumulator element k = 4i + 2hb + e: gate row 64wg + 16warp + gq + 8hb, position 8i + 2cq + e
    const int r0 = rb * PJ_M + wg * 64 + warp * 16 + gq;
    const float bias0 = bias[r0], bias1 = bias[r0 + 8];
#pragma unroll
    for (int k = 0; k < 64; ++k) {
        const int64_t p = m0 + 8 * (k >> 2) + 2 * cq + (k & 1);
        const int hb = (k >> 1) & 1;
        if (p < M) C[p * N + r0 + 8 * hb] = sum[k] + (hb ? bias1 : bias0);
    }
}

__global__ void __launch_bounds__(256, 1) rl_proj_tc_kernel(const float *__restrict__ X, const uint8_t *__restrict__ w_tc,
                                                            const float *__restrict__ bias, float *__restrict__ C, int64_t M,
                                                            int K, int N) {
    rl_proj_body<false>(X, w_tc, bias, C, M, K, N);
}
__global__ void __launch_bounds__(256, 1) rl_proj_fp16_kernel(const float *__restrict__ X, const uint8_t *__restrict__ w_tc,
                                                              const float *__restrict__ bias, float *__restrict__ C, int64_t M,
                                                              int K, int N) {
    rl_proj_body<true>(X, w_tc, bias, C, M, K, N);
}

// ---------------------------------------------------------------------------------------------- recurrence on a cluster
// Per time step G^T[4H = 1536][16 windows] = W_hh . h^T with h the 16 windows' previous output, split over a cluster of
// 8 CTAs: CTA rank r owns hidden units 48r .. 48r + 47, i.e. 192 gate rows (4 gates x 48 units), in three warpgroups of
// 64 rows (16 units x 4 gates, warp w = gate w).
//   A = W_hh rows: the fp16 hi plane in registers (24 k-steps x 4 = 96 per thread), the lo plane as shared-memory operand
//       tiles (144 KiB per CTA, pre-tiled per (direction, rank, warpgroup))
//   B = the full h tile [16 windows][384] (fp16 hi | lo, K-major, double buffered): every CTA holds all 384 units
//   D = one M64 N16 accumulator per warpgroup, preloaded with the input pre-activations; 24 k-steps x 3 products
// The four gates of a unit come from four warps: they meet in a 5 KiB exchange buffer per warpgroup (named barrier),
// where each thread takes two (unit, window) pairs; c stays in its registers.  Each thread writes its two new h values
// (hi / lo) into the next h buffer of all 8 CTAs with st.shared::cluster, then fences them to the async proxy at cluster
// scope.  After a CTA barrier, threads 0..7 arrive (release, cluster scope) on the step barrier of CTA 0..7; every
// thread waits (acquire, cluster scope, bounded) on its own CTA's barrier for all 8 arrivals before the next step's MMAs
// read the buffer.  That wait after the last step is also the exit barrier: once a CTA has seen its 8 arrivals, no peer
// writes into its shared memory any more.  The buffer a step writes was last read by the MMAs of the step before, which
// every CTA completed (wgmma.wait_group) before it arrived.  FP16 (the fp16 mode): one product, W_hi.h_hi, 24 MMAs per
// step in the same three chains; no lo plane in shared memory, and only h's hi plane goes to the peers.
constexpr int L3_CL = 8;                                     // CTAs per cluster
constexpr int L3_UNITS = RL_H3 / L3_CL;                      // 48 hidden units per CTA
constexpr int L3_THREADS = 384;                              // 3 warpgroups
constexpr int L3_KS = RL_H3 / 16;                            // 24 k-steps
constexpr int L3_WLO_WG = (RL_H3 / 8) * 64 * 16;             // 48 KiB: one warpgroup's lo plane as A operand tiles
constexpr int L3_KG = LT_N * 16 + 16;                        // k-group stride of the h tile (272 B)
constexpr int L3_HPLANE = (RL_H3 / 8) * L3_KG;               // 13 056 B
constexpr int L3_XS = 20;                                    // window stride of the gate exchange (floats): no bank conflicts
constexpr int L3_XCH_WG = 4 * LT_N * L3_XS * 4;              // 5 KiB
template <bool FP16> constexpr int L3_OFF_H = FP16 ? 0 : 3 * L3_WLO_WG;
template <bool FP16> constexpr int L3_OFF_X = L3_OFF_H<FP16> + 4 * L3_HPLANE;
template <bool FP16> constexpr int L3_OFF_BAR = L3_OFF_X<FP16> + 3 * L3_XCH_WG;
template <bool FP16> constexpr int L3_SMEM = L3_OFF_BAR<FP16> + 16;     // 210 KiB (FP16: 66 KiB)
// element (direction d, gate row r, column k) of W_hh's lo plane in the tiles above: per (direction, cluster rank,
// warpgroup) [k-group][row m = 16 gate + unit within the warpgroup][8 halfs]
inline size_t l3_lo_index(int d, int r, int k) {
    const int gate = r / RL_H3, j = r % RL_H3, rank = j / L3_UNITS, wg = (j % L3_UNITS) / 16, m = gate * 16 + j % 16;
    return (((size_t)(d * L3_CL + rank) * 3 + wg) * (RL_H3 / 8) + k / 8) * (64 * 8) + m * 8 + k % 8;
}

template <bool FP16>
__device__ __forceinline__ void rl_lstm384_body(const float *__restrict__ gi, const __half *__restrict__ w_hi,
                                                const uint8_t *__restrict__ w_lo_tiles, float *__restrict__ out, int64_t B,
                                                int64_t P) {
    extern __shared__ __align__(128) uint8_t smem_l3[];
    uint8_t *swlo = smem_l3;
    uint8_t *sh = smem_l3 + L3_OFF_H<FP16>;                      // [buf 2][hi | lo] L3_HPLANE
    uint64_t *hbar = reinterpret_cast<uint64_t *>(smem_l3 + L3_OFF_BAR<FP16>);
    const int tid = threadIdx.x, wg = tid >> 7, wt = tid & 127, warp = (tid >> 5) & 3, lane = tid & 31;
    const int gq = lane >> 2, cq = lane & 3;
    const uint32_t rank = cluster_ctarank();
    const int dir = blockIdx.y;
    const int64_t b0 = (int64_t)(blockIdx.x / L3_CL) * LT_N;
    const int nb = (int)min((int64_t)LT_N, B - b0);
    const int u0 = (int)rank * L3_UNITS + wg * 16;                 // first hidden unit of this warpgroup
    float *xw = reinterpret_cast<float *>(smem_l3 + L3_OFF_X<FP16> + wg * L3_XCH_WG);  // [gate 4][window 16][L3_XS]
    {
        const uint4 *src = reinterpret_cast<const uint4 *>(w_lo_tiles + ((size_t)dir * L3_CL + rank) * 3 * L3_WLO_WG);
        if (!FP16)
            for (int i = tid; i < 3 * L3_WLO_WG / 16; i += L3_THREADS) reinterpret_cast<uint4 *>(swlo)[i] = src[i];
        for (int i = tid; i < 4 * L3_HPLANE / 16; i += L3_THREADS) reinterpret_cast<uint4 *>(sh)[i] = make_uint4(0u, 0u, 0u, 0u);
    }
    if (tid == 0) {
        mbar_init(&hbar[0], L3_CL);
        mbar_init(&hbar[1], L3_CL);
        fence_mbar_init();
    }
    // hi plane: gate `warp`, units u0 + gq (+8)
    uint32_t whi[L3_KS][4];
#pragma unroll
    for (int ks = 0; ks < L3_KS; ++ks) {
        const __half *w = w_hi + (((size_t)dir * 4 + warp) * RL_H3 + u0 + gq) * RL_H3 + ks * 16 + 2 * cq;
        whi[ks][0] = *reinterpret_cast<const uint32_t *>(w);
        whi[ks][1] = *reinterpret_cast<const uint32_t *>(w + 8 * RL_H3);
        whi[ks][2] = *reinterpret_cast<const uint32_t *>(w + 8);
        whi[ks][3] = *reinterpret_cast<const uint32_t *>(w + 8 * RL_H3 + 8);
    }
    // accumulator element k = 4i + 2hb + e: unit u0 + gq + 8hb of gate `warp`, window 8i + 2cq + e
    float acc[8];
    auto fetch = [&](int64_t t) {
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int wdw = 8 * (k >> 2) + 2 * cq + (k & 1);
            const bool ok = wdw < nb;
            const float *row = gi + (((b0 + (ok ? wdw : 0)) * P + t) * 2 + dir) * RL_G43 + warp * RL_H3 + u0 + gq + 8 * ((k >> 1) & 1);
            acc[k] = ok ? __ldg(row) : 0.f;
        }
    };
    // gate math: this thread's pairs are units u0 + ue, u0 + ue + 1 of window we
    const int ue = 2 * (wt & 7), we = wt >> 3;
    float c_state[2] = {0.f, 0.f};
    const int jg = u0 + ue;                                         // even: the two units share one 32-bit h word
    const uint32_t h_off = (uint32_t)((jg >> 3) * L3_KG + we * 16 + (jg & 7) * 2);
    uint32_t peer_h[L3_CL];
#pragma unroll
    for (int q = 0; q < L3_CL; ++q) peer_h[q] = mapa_shared(smem_u32(sh), (uint32_t)q);
    const uint32_t bar_peer = tid < L3_CL ? mapa_shared(smem_u32(&hbar[0]), (uint32_t)tid) : 0u;
    fetch(dir ? (P - 1) : 0);
    fence_proxy_async_smem();                                     // zeroed h tiles and lo planes -> wgmma
    cluster_sync_all();                                           // every CTA's barriers initialised, h zeroed
    const uint32_t wl = smem_u32(swlo) + wg * L3_WLO_WG;
    for (int64_t step = 0; step < P; ++step) {
        const int64_t t = dir ? (P - 1 - step) : step;
        const int buf = (int)(step & 1);
        const uint32_t h_hi = smem_u32(sh + buf * 2 * L3_HPLANE), h_lo = h_hi + L3_HPLANE;
        wg_fence();
        // three accumulator chains of 24 MMAs (k-steps 0-7 onto the pre-activations, 8-15 and 16-23 from zero), added on
        // the CUDA cores: one chain of 72 lost accuracy in the tensor core's accumulation
        float acc2[8], acc3[8];
#pragma unroll
        for (int ks = 0; ks < L3_KS; ++ks) {
            float (&a)[8] = ks < L3_KS / 3 ? acc : ks < 2 * L3_KS / 3 ? acc2 : acc3;
            const uint64_t bh = make_smem_desc(h_hi + ks * 2 * L3_KG, L3_KG, 128);
            Wgmma<16>::rs(a, whi[ks], bh, (ks == L3_KS / 3 || ks == 2 * L3_KS / 3) ? 0u : 1u);
            if (FP16) continue;
            Wgmma<16>::rs(a, whi[ks], make_smem_desc(h_lo + ks * 2 * L3_KG, L3_KG, 128), 1u);
            Wgmma<16>::ss(a, make_smem_desc(wl + ks * 2 * (64 * 16), 64 * 16, 128), bh, 1u);
        }
        wg_commit();
        wg_wait_all();
        wg_hold(acc);
        wg_hold(acc2);
        wg_hold(acc3);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int wdw = 8 * (k >> 2) + 2 * cq + (k & 1);
            xw[(warp * LT_N + wdw) * L3_XS + gq + 8 * ((k >> 1) & 1)] = acc[k] + (acc2[k] + acc3[k]);
        }
        if (step + 1 < P) fetch(dir ? (t - 1) : (t + 1));           // the next pre-activations load under the gate math
        named_bar_sync(1 + wg, 128);
        float hv[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const float *x = xw + we * L3_XS + ue + e;
            const float ig = lt_sigmoid(x[0]);
            const float fg = lt_sigmoid(x[1 * LT_N * L3_XS]);
            const float gg = lt_tanh(x[2 * LT_N * L3_XS]);
            const float og = lt_sigmoid(x[3 * LT_N * L3_XS]);
            const float c = fmaf(fg, c_state[e], ig * gg);
            c_state[e] = c;
            hv[e] = og * lt_tanh(c);
        }
        if (we < nb)
            *reinterpret_cast<float2 *>(out + ((b0 + we) * P + t) * (2 * RL_H3) + dir * RL_H3 + jg) = make_float2(hv[0], hv[1]);
        __half hi0, lo0, hi1, lo1;
        split_f16(hv[0], hi0, lo0);
        split_f16(hv[1], hi1, lo1);
        __half2 hp = __halves2half2(hi0, hi1), lp = __halves2half2(lo0, lo1);
        const uint32_t hw = *reinterpret_cast<uint32_t *>(&hp), lw = *reinterpret_cast<uint32_t *>(&lp);
        const uint32_t nxt = (uint32_t)((buf ^ 1) * 2 * L3_HPLANE) + h_off;
#pragma unroll
        for (int q = 0; q < L3_CL; ++q) {
            st_cluster_u32(peer_h[q] + nxt, hw);
            if (!FP16) st_cluster_u32(peer_h[q] + nxt + L3_HPLANE, lw);
        }
        fence_proxy_async_cluster();
        __syncthreads();
        if (tid < L3_CL) mbar_arrive_cluster(bar_peer + (uint32_t)((buf ^ 1) * 8));
        mbar_wait_cluster(&hbar[buf ^ 1], (uint32_t)(step >> 1) & 1u);
    }
}

__global__ void __cluster_dims__(L3_CL, 1, 1) __launch_bounds__(L3_THREADS, 1)
    rl_lstm384_tc_kernel(const float *__restrict__ gi, const __half *__restrict__ w_hi, const uint8_t *__restrict__ w_lo_tiles,
                         float *__restrict__ out, int64_t B, int64_t P) {
    rl_lstm384_body<false>(gi, w_hi, w_lo_tiles, out, B, P);
}
__global__ void __cluster_dims__(L3_CL, 1, 1) __launch_bounds__(L3_THREADS, 1)
    rl_lstm384_fp16_kernel(const float *__restrict__ gi, const __half *__restrict__ w_hi, const uint8_t *__restrict__ w_lo_tiles,
                           float *__restrict__ out, int64_t B, int64_t P) {
    rl_lstm384_body<true>(gi, w_hi, w_lo_tiles, out, B, P);
}

// Linear(2H = 768 -> 5) + softmax + argmax: one warp per position, 24 inputs per lane, the weights in shared memory.
// labels (may be NULL for HEAD_PLAIN): argmax of the five probabilities as written, first maximum wins (np.argmax,
// labels.py:1063).  MODE as head_kernel's (misc.cu): HEAD_QUALS also writes the phred byte of the winning probability,
// HEAD_VARIANT the call byte and the phreds of the winning and of the reference class (and the phred byte where quals
// is given), all from the fp32 probabilities the kernel stores (phred.cuh).  HEAD_PLAIN is the ordinary forward's.
template <int MODE>
__global__ void __launch_bounds__(256) rl_head768_kernel(const float *__restrict__ h1, const float *__restrict__ lin_w,
                                                         const float *__restrict__ lin_b, int64_t n_pos,
                                                         float *__restrict__ probs, uint8_t *__restrict__ labels,
                                                         uint8_t *__restrict__ quals, HeadVariant var) {
    constexpr int W2 = 2 * RL_H3;
    __shared__ __align__(16) float ws[NCLS * W2];
    for (int i = threadIdx.x; i < NCLS * W2; i += blockDim.x) ws[i] = lin_w[i];
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t p = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; p < n_pos; p += nwarps) {
        float s[NCLS];
#pragma unroll
        for (int c = 0; c < NCLS; ++c) s[c] = 0.f;
#pragma unroll
        for (int q = 0; q < W2 / 128; ++q) {
            const int k = q * 128 + lane * 4;
            const float4 x = ld_stream4(h1 + p * W2 + k);
#pragma unroll
            for (int c = 0; c < NCLS; ++c) {
                const float4 wv = *reinterpret_cast<const float4 *>(ws + c * W2 + k);
                s[c] = fmaf(x.x, wv.x, fmaf(x.y, wv.y, fmaf(x.z, wv.z, fmaf(x.w, wv.w, s[c]))));
            }
        }
#pragma unroll
        for (int c = 0; c < NCLS; ++c)
#pragma unroll
            for (int m = 16; m >= 1; m >>= 1) s[c] += __shfl_xor_sync(0xffffffffu, s[c], m);
        float mx = -INFINITY;
#pragma unroll
        for (int c = 0; c < NCLS; ++c) { s[c] += lin_b[c]; mx = fmaxf(mx, s[c]); }
        float sum = 0.f;
#pragma unroll
        for (int c = 0; c < NCLS; ++c) { s[c] = expf(s[c] - mx); sum += s[c]; }
        float v = s[0];
#pragma unroll
        for (int c = 1; c < NCLS; ++c) if (lane == c) v = s[c];
        const float pr = v / sum;                  // lane c < 5: probability of class c
        if (lane < NCLS) probs[p * NCLS + lane] = pr;
        if (MODE != HEAD_PLAIN || labels) {        // argmax over lanes 0..4, first maximum wins
            float best = lane < NCLS ? pr : -1.f;
            int arg = lane;
#pragma unroll
            for (int m = 4; m >= 1; m >>= 1) {
                const float ob = __shfl_xor_sync(0xffffffffu, best, m);
                const int oa = __shfl_xor_sync(0xffffffffu, arg, m);
                if (ob > best || (ob == best && oa < arg)) { best = ob; arg = oa; }
            }
            if (MODE == HEAD_PLAIN) {
                if (lane == 0) labels[p] = (uint8_t)arg;
            } else {
                uint8_t ref = 0;
                float p_ref = 0.f;
                if (MODE == HEAD_VARIANT) {        // the reference class's probability from its lane
                    ref = var.ref[p];
                    p_ref = __shfl_sync(0xffffffffu, pr, ref_class(ref));
                }
                if (lane == 0) {
                    if (labels) labels[p] = (uint8_t)arg;
                    if (MODE == HEAD_QUALS || quals) quals[p] = phred_char(best);
                    if (MODE == HEAD_VARIANT) {
                        var.calls[p] = variant_call(arg, ref);
                        var.pred_q[p] = phred_f32(best);
                        var.ref_q[p] = phred_f32(p_ref);
                    }
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------- shared launchers
// (rl_common.cuh): the fp32 kernels above as the trainer (rl_train.cu) runs them
constexpr int RL_DGROUP = 4;      // reads per partial sum of the fp32 convolution

cudaError_t rl_launch_mask(const int8_t *x, int64_t B, int64_t P, int D, int F, uint8_t *mask, cudaStream_t s) {
    rl_mask_kernel<<<(unsigned)(B * D), 256, 0, s>>>(x, P, D, F, mask);
    return cudaGetLastError();
}

cudaError_t rl_launch_conv_fp32(const int8_t *x, const uint8_t *mask, const RlConv1 &c1, const RlConv17 &c17,
                                const float *pool_w_t, const float *pool_b, int64_t B, int64_t P, int D, int F,
                                int use_dwells, int H, float *y1, float *part, float *z, cudaStream_t s) {
    const int n_groups = (D + RL_DGROUP - 1) / RL_DGROUP;
    cudaError_t e = cudaFuncSetAttribute(rl_conv17_pool_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, RL_CONV_SMEM);
    if (e != cudaSuccess) return e;
    rl_embed_conv1_kernel<<<dim3((unsigned)((P + 31) / 32), (unsigned)(B * D)), RL_C, 0, s>>>(x, mask, c1, P, D, F,
                                                                                         use_dwells, y1);
    rl_conv17_pool_kernel<<<dim3((unsigned)((P + RL_PT - 1) / RL_PT), (unsigned)n_groups, (unsigned)B), 256, RL_CONV_SMEM, s>>>(
        y1, mask, c17, P, D, RL_DGROUP, part);
    if (H == RL_H3)
        rl_pool_linear_kernel<RL_H3><<<dim3((unsigned)((P + RL_PLT - 1) / RL_PLT), (unsigned)B), RL_C, 0, s>>>(
            part, mask, pool_w_t, pool_b, P, D, n_groups, z);
    else
        rl_pool_linear_kernel<RL_H><<<dim3((unsigned)((P + RL_PLT - 1) / RL_PLT), (unsigned)B), RL_C, 0, s>>>(
            part, mask, pool_w_t, pool_b, P, D, n_groups, z);
    return cudaGetLastError();
}

cudaError_t rl_launch_lstm_fp32(const float *gi, const float *w_t, float *out, int64_t B, int64_t P, int H,
                                cudaStream_t s, float *save) {
    const dim3 grid((unsigned)((B + LF_NB - 1) / LF_NB), 2);
    if (H == RL_H3) {
        if (save) rl_lstm_fp32<RL_H3, true><<<grid, RL_H3, 0, s>>>(gi, w_t, out, B, P, save);
        else rl_lstm_fp32<RL_H3, false><<<grid, RL_H3, 0, s>>>(gi, w_t, out, B, P, nullptr);
    } else {
        if (save) rl_lstm_fp32<RL_H, true><<<grid, RL_H, 0, s>>>(gi, w_t, out, B, P, save);
        else rl_lstm_fp32<RL_H, false><<<grid, RL_H, 0, s>>>(gi, w_t, out, B, P, nullptr);
    }
    return cudaGetLastError();
}

cudaError_t rl_launch_head(const float *h1, const float *lin_w, const float *lin_b, int64_t n, int H, float *probs,
                           float *logits, cudaStream_t s) {
    if (H != RL_H3) return launch_head(h1, lin_w, lin_b, 1, n, 0, probs, logits, nullptr, s);
    const int64_t blocks = std::min<int64_t>((n + 7) / 8, 132 * 8);
    rl_head768_kernel<HEAD_PLAIN><<<(unsigned)blocks, 256, 0, s>>>(h1, lin_w, lin_b, n, probs, nullptr, nullptr, {});
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------- engine
struct RlLstmLayer {
    float *w_ih = nullptr;      // [2 dirs * 4H][in]   (both directions stacked: one GEMM)
    float *bias = nullptr;      // [2 * 4H]  b_ih + b_hh
    float *w_t = nullptr;       // [2][H k][4H]  W_hh^T (fp32 recurrence)
    __half *w_hi = nullptr;     // [2][4H][H] fp16 hi plane of W_hh, row-major (tensor-core recurrences: -> registers)
    __half *w_lo = nullptr;     // fp16 lo plane of W_hh as the tensor-core recurrence's shared-memory A operand tiles
                                // (lt_lo_index at H = 128, l3_lo_index at 384)
    __half *w_ih_tc = nullptr;  // H = 384: W_ih as rl_proj_tc_kernel's A tiles [row block 24][K chunk][hi | lo][8][128][8]
};

}  // namespace mdk

using namespace mdk;

// Calls are packed into GROUPS (packing.h, DESIGN §4).  Staging a piece is its convolution, in slices of windows bounded
// by RL_CONV_BUDGET, into the open group's z (pooled pre_pool_expansion_layer output) at the piece's window offset; the
// projections, recurrences and head run once per group.  One set of group buffers, one compute stream: the next group's
// convolutions queue behind the group in flight; only copy_in and copy_out run beside the compute.
constexpr size_t RL_CONV_BUDGET = (size_t)2 << 30;     // feature staging + convolution scratch of one slice, bytes
constexpr size_t RL_GROUP_BUDGET = (size_t)24 << 30;   // z, gi, h0, h1, probs, labels of one group, bytes
constexpr int64_t RL_PREFERRED_P = 10000;              // window length mdk_rl_preferred_windows sizes for (chunk_len)

struct mdk_rl_engine {
    int device = 0;
    int use_dwells = 0;
    int H = RL_H;                  // lstm_size: 128 or 384
    int sm_count = 132;
    int wave = 0;                  // windows of one recurrence wave (0: not computed yet)
    int timing = 0;                // record per-stage CUDA events in each group
    cudaEvent_t ev[2][7] = {};     // stage events, by group parity: one group's may be read while the next collects
    std::unordered_map<std::string, std::vector<float>> host;     // state-dict tensors as loaded
    bool prepared = false;
    // device parameters, built from `host` by rl_prepare
    DeviceWeights weights;
    float *emb_base = nullptr, *emb_strand = nullptr;
    float *c1_w = nullptr, *c1_b = nullptr, *bn1[4] = {nullptr, nullptr, nullptr, nullptr};
    float *c17_wt = nullptr, *c17_b = nullptr, *bn2[4] = {nullptr, nullptr, nullptr, nullptr};
    __half *c17_tc = nullptr;      // [17 taps][hi | lo][k-group 16][co 128][8 halfs]: the tensor-core kernel's A operand tiles
    int conv_tc = 1;               // 1: k = 17 convolution on wgmma (default), 0: fp32 CUDA cores
    int lstm_tc = 1;               // 1: LSTM recurrence on wgmma (default), 0: fp32 CUDA cores
    int fp16 = 0;                  // 1: the wgmma stages take one fp16 product per contraction (the fp16 mode)
    float *pool_w = nullptr, *pool_b = nullptr;
    RlLstmLayer lstm[2];
    float *lin_w = nullptr, *lin_b = nullptr;
    cudaStream_t stream = nullptr;                   // compute: convolutions, then each group's LSTM and head
    cudaStream_t copy_in = nullptr;
    CopyOut copy_out;
    // convolution of one slice: features in two staging slots (the copy of the next slice runs under this one's
    // convolution), then mask | y1 (fp32 path only) | partial sums on the compute stream
    int8_t *xbuf[2] = {nullptr, nullptr};
    size_t xcap[2] = {0, 0};
    cudaEvent_t ev_xin[2] = {}, ev_xfree[2] = {};
    int xslot = 0;
    uint8_t *conv = nullptr;
    size_t conv_cap = 0;
    // group buffers, [window][P][...] for up to cap_pos positions
    int64_t cap_pos = 0;
    float *z = nullptr, *gi = nullptr, *h0 = nullptr, *h1 = nullptr, *probs = nullptr;
    uint8_t *labels = nullptr;
    // decoded outputs (mdk_rl_submit_decoded / mdk_rl_submit_variant_decoded), 11 B per position for cap_pos positions:
    // allocated when the first decoded call is staged, freed with the other group buffers when they regrow
    uint8_t *quals = nullptr, *ref = nullptr, *calls = nullptr;
    float *pred_q = nullptr, *ref_q = nullptr;
    Packing pk;
    int64_t last_B = 0, last_P = 0;                  // the last completed mdk_rl_forward (mdk_rl_debug_read), 0 = none
};

namespace {

const std::vector<float> *rl_get(mdk_rl_engine *e, const std::string &name, size_t want) {
    auto it = e->host.find(name);
    if (it == e->host.end()) { set_error("read-level model: tensor '" + name + "' was not loaded"); return nullptr; }
    if (it->second.size() != want) {
        set_error("read-level model: tensor '" + name + "' has " + std::to_string(it->second.size()) + " values, expected " +
                  std::to_string(want));
        return nullptr;
    }
    return &it->second;
}

// LSTM weights of both layers at either size: W_ih of both directions stacked for one projection, b_ih + b_hh, W_hh^T for
// the fp32 recurrence, W_hh as fp16 hi (row-major) and lo (the tensor-core recurrence's operand tiles) planes, and at
// H = 384 W_ih as rl_proj_tc_kernel's operand tiles
int rl_prepare_lstm(mdk_rl_engine *e) {
    const int HH = e->H, G4 = 4 * HH;
    const auto up = [e](auto **dst, const auto &src) { return e->weights.upload(e->stream, dst, src); };
    int rc;
    for (int l = 0; l < 2; ++l) {
        const int in = l == 0 ? HH : 2 * HH;
        std::vector<float> w_ih((size_t)2 * G4 * in), bias((size_t)2 * G4), w_t((size_t)2 * HH * G4);
        std::vector<__half> hi((size_t)2 * G4 * HH), lo((size_t)2 * G4 * HH);
        for (int d = 0; d < 2; ++d) {
            const std::string sfx = "_l" + std::to_string(l) + (d ? "_reverse" : "");
            const std::vector<float> *wih = rl_get(e, "lstm.weight_ih" + sfx, (size_t)G4 * in);
            const std::vector<float> *whh = rl_get(e, "lstm.weight_hh" + sfx, (size_t)G4 * HH);
            const std::vector<float> *bih = rl_get(e, "lstm.bias_ih" + sfx, G4);
            const std::vector<float> *bhh = rl_get(e, "lstm.bias_hh" + sfx, G4);
            if (!wih || !whh || !bih || !bhh) return MDK_ERR_STATE;
            std::copy(wih->begin(), wih->end(), w_ih.begin() + (size_t)d * G4 * in);
            for (int r = 0; r < G4; ++r) bias[(size_t)d * G4 + r] = (*bih)[r] + (*bhh)[r];
            for (int r = 0; r < G4; ++r)
                for (int k = 0; k < HH; ++k) {
                    const float v = (*whh)[(size_t)r * HH + k];
                    w_t[((size_t)d * HH + k) * G4 + r] = v;
                    split_f16(v, hi[((size_t)d * G4 + r) * HH + k], lo[HH == RL_H3 ? l3_lo_index(d, r, k) : lt_lo_index(d, r, k)]);
                }
        }
        RlLstmLayer &L = e->lstm[l];
        if ((rc = up(&L.w_ih, w_ih)) || (rc = up(&L.bias, bias)) || (rc = up(&L.w_t, w_t)) || (rc = up(&L.w_hi, hi)) ||
            (rc = up(&L.w_lo, lo)))
            return rc;
        if (HH != RL_H3) continue;
        // W_ih of both directions as one [3072][in] matrix, tiled per (128-row block, 64-wide K chunk)
        const int nchunks = in / PJ_KC;
        std::vector<__half> ih_t((size_t)2 * G4 * in * 2);
        for (int r = 0; r < 2 * G4; ++r)
            for (int k = 0; k < in; ++k) {
                const size_t chunk = ((size_t)(r / PJ_M) * nchunks + k / PJ_KC) * (PJ_WCHUNK / 2);
                const size_t off = (size_t)((k % PJ_KC) / 8) * (PJ_M * 8) + (r % PJ_M) * 8 + k % 8;
                split_f16(w_ih[(size_t)r * in + k], ih_t[chunk + off], ih_t[chunk + PJ_WPLANE / 2 + off]);
            }
        if ((rc = up(&L.w_ih_tc, ih_t))) return rc;
    }
    return MDK_OK;
}

// Windows of one wave of the tensor-core recurrence: one CTA per (16-window tile, direction) at lstm_size 128, one
// 8-CTA cluster per (tile, direction) at 384, as many clusters as fit the device at once (cudaOccupancyMaxActiveClusters;
// MDK_ERR_UNSUPPORTED when none does).
int rl_wave_windows(mdk_rl_engine *e, int *out) {
    if (e->wave > 0) { *out = e->wave; return MDK_OK; }
    if (e->H == RL_H) {
        e->wave = LT_N * (e->sm_count / 2);
    } else {
        // the three-product kernel: the fp16 one needs less shared memory and fits as many clusters
        MDK_CUDA(cudaFuncSetAttribute(rl_lstm384_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, L3_SMEM<false>));
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(L3_CL, 2);
        cfg.blockDim = dim3(L3_THREADS);
        cfg.dynamicSmemBytes = L3_SMEM<false>;
        cudaLaunchAttribute attr;
        attr.id = cudaLaunchAttributeClusterDimension;
        attr.val.clusterDim.x = L3_CL;
        attr.val.clusterDim.y = 1;
        attr.val.clusterDim.z = 1;
        cfg.attrs = &attr;
        cfg.numAttrs = 1;
        int clusters = 0;
        MDK_CUDA(cudaOccupancyMaxActiveClusters(&clusters, (void *)rl_lstm384_tc_kernel, &cfg));
        MDK_REQUIRE(clusters >= 1, MDK_ERR_UNSUPPORTED,
                    "read-level model: lstm_size = 384 needs a cluster of 8 CTAs with 210 KiB of shared memory each; "
                    "none fits this device");
        e->wave = LT_N * std::max(1, clusters / 2);
    }
    *out = e->wave;
    return MDK_OK;
}

// Most windows of window length P one group holds: one recurrence wave, capped by RL_GROUP_BUDGET (a multiple of the
// 16-window tile when the cap allows one).
int rl_group_limit(mdk_rl_engine *e, int64_t P, int64_t *out) {
    int wave = 0;
    int rc = rl_wave_windows(e, &wave);
    if (rc) return rc;
    const int64_t per_pos = (int64_t)52 * e->H + 4 * NCLS + 1;      // z 4H + gi 32H + h0 8H + h1 8H bytes, probs, label
    int64_t cap = (int64_t)(RL_GROUP_BUDGET / (size_t)(P * per_pos));
    if (cap >= LT_N) cap -= cap % LT_N;
    *out = std::max<int64_t>(1, std::min<int64_t>(wave, cap));
    return MDK_OK;
}

int rl_prepare(mdk_rl_engine *e) {
    if (e->prepared) return MDK_OK;
    const int nin = RL_EMB + 1 + (e->use_dwells ? 1 : 0);
    const int HH = e->H;
    const auto up = [e](auto **dst, const auto &src) { return e->weights.upload(e->stream, dst, src); };
    int rc;
    {   // at 384: one 8-CTA cluster of the recurrence must fit the device
        int wave = 0;
        if ((rc = rl_wave_windows(e, &wave))) return rc;
    }
#define RL_NEED(var, name, n) const std::vector<float> *var = rl_get(e, name, (size_t)(n)); if (!var) return MDK_ERR_STATE;
    RL_NEED(eb, "base_embedder.weight", 6 * RL_EMB)
    RL_NEED(es, "strand_embedder.weight", 3 * RL_EMB)
    RL_NEED(c1w, "read_level_conv.convs.0.weight", RL_C * nin)
    RL_NEED(c1b, "read_level_conv.convs.0.bias", RL_C)
    RL_NEED(c17w, "read_level_conv.convs.3.weight", RL_C * RL_C * RL_TAPS)
    RL_NEED(c17b, "read_level_conv.convs.3.bias", RL_C)
    RL_NEED(pw, "pre_pool_expansion_layer.weight", HH * RL_C)
    RL_NEED(pb, "pre_pool_expansion_layer.bias", HH)
    RL_NEED(lw, "linear.weight", NCLS * 2 * HH)
    RL_NEED(lb, "linear.bias", NCLS)
    if ((rc = up(&e->emb_base, *eb)) || (rc = up(&e->emb_strand, *es)) || (rc = up(&e->c1_w, *c1w)) ||
        (rc = up(&e->c1_b, *c1b)) || (rc = up(&e->c17_b, *c17b)) || (rc = up(&e->pool_b, *pb)) ||
        (rc = up(&e->lin_w, *lw)) || (rc = up(&e->lin_b, *lb)))
        return rc;
    {   // Linear(C -> H) weights transposed to [k][h]: coalesced across the output units
        std::vector<float> wt((size_t)RL_C * HH);
        for (int h = 0; h < HH; ++h)
            for (int k = 0; k < RL_C; ++k) wt[(size_t)k * HH + h] = (*pw)[(size_t)h * RL_C + k];
        if ((rc = up(&e->pool_w, wt))) return rc;
    }
    // conv k = 17 weights: torch [out][in][tap] -> [tap][in][out]
    {
        std::vector<float> wt((size_t)RL_TAPS * RL_C * RL_C);
        for (int o = 0; o < RL_C; ++o)
            for (int i = 0; i < RL_C; ++i)
                for (int t = 0; t < RL_TAPS; ++t) wt[((size_t)t * RL_C + i) * RL_C + o] = (*c17w)[((size_t)o * RL_C + i) * RL_TAPS + t];
        if ((rc = up(&e->c17_wt, wt))) return rc;
        // the same weights as K-major fp16 hi / lo operand tiles, one 64 KiB block per tap
        std::vector<__half> tc((size_t)RL_TAPS * 2 * RL_C * RL_C);
        for (int t = 0; t < RL_TAPS; ++t)
            for (int o = 0; o < RL_C; ++o)
                for (int i = 0; i < RL_C; ++i) {
                    const size_t off = (size_t)(i / 8) * (RL_C * 8) + (size_t)o * 8 + (i % 8);
                    split_f16((*c17w)[((size_t)o * RL_C + i) * RL_TAPS + t], tc[((size_t)t * 2 + 0) * RL_C * RL_C + off],
                              tc[((size_t)t * 2 + 1) * RL_C * RL_C + off]);
                }
        if ((rc = up(&e->c17_tc, tc))) return rc;
    }
    // BatchNorm (inference): mean, 1 / sqrt(var + eps), weight, bias
    for (int l = 0; l < 2; ++l) {
        const std::string base = std::string("read_level_conv.convs.") + (l == 0 ? "2" : "5") + ".";
        RL_NEED(mean, base + "running_mean", RL_C)
        RL_NEED(var, base + "running_var", RL_C)
        RL_NEED(w, base + "weight", RL_C)
        RL_NEED(b, base + "bias", RL_C)
        std::vector<float> invstd(RL_C);
        for (int c = 0; c < RL_C; ++c) invstd[c] = 1.0f / sqrtf((*var)[c] + 1e-5f);
        float **dst = l == 0 ? e->bn1 : e->bn2;
        if ((rc = up(&dst[0], *mean)) || (rc = up(&dst[1], invstd)) || (rc = up(&dst[2], *w)) || (rc = up(&dst[3], *b)))
            return rc;
    }
#undef RL_NEED
    if ((rc = rl_prepare_lstm(e))) return rc;
    e->prepared = true;
    return MDK_OK;
}

size_t rl_round(size_t bytes) { return (bytes + 255) / 256 * 256; }

// Device buffer of at least `need` bytes (grown by 1/8 to spare regrowth); the caller has drained its users
template <class T>
int rl_grow(T **p, size_t *cap, size_t need) {
    if (need <= *cap) return MDK_OK;
    if (*p) cudaFree(*p);
    *p = nullptr;
    *cap = 0;
    void *q = nullptr;
    MDK_CUDA(cudaMalloc(&q, need + need / 8));
    *p = static_cast<T *>(q);
    *cap = need + need / 8;
    return MDK_OK;
}

// Group buffers for `pos` positions.  Only called when no group is open: the compute and copy-out streams are drained
// before the old buffers go.
int rl_ensure_group(mdk_rl_engine *e, int64_t pos) {
    if (pos <= e->cap_pos) return MDK_OK;
    MDK_CUDA(cudaStreamSynchronize(e->stream));
    MDK_CUDA(cudaStreamSynchronize(e->copy_out.stream));
    e->last_B = e->last_P = 0;                       // the last mdk_rl_forward's stages go with the old buffers
    float **fb[5] = {&e->z, &e->gi, &e->h0, &e->h1, &e->probs};
    for (float **p : fb) { if (*p) cudaFree(*p); *p = nullptr; }
    void **db[6] = {(void **)&e->labels, (void **)&e->quals, (void **)&e->ref, (void **)&e->calls, (void **)&e->pred_q,
                    (void **)&e->ref_q};
    for (void **p : db) { if (*p) cudaFree(*p); *p = nullptr; }
    e->cap_pos = 0;
    const size_t n = (size_t)pos, H = (size_t)e->H;
    const size_t floats[5] = {n * H, n * 8 * H, n * 2 * H, n * 2 * H, n * NCLS};
    for (int i = 0; i < 5; ++i) MDK_CUDA(cudaMalloc(fb[i], floats[i] * sizeof(float)));
    MDK_CUDA(cudaMalloc(&e->labels, n));
    e->cap_pos = pos;
    return MDK_OK;
}

// The decoded outputs' group buffers (quals, ref, calls, pred_q, ref_q) for cap_pos positions, allocated when the first
// decoded call is staged.  Nothing frees them while a group collects (rl_ensure_group only runs when one opens, after
// draining the streams), so a group in flight never loses them.
int rl_ensure_decoded(mdk_rl_engine *e) {
    if (e->ref_q) return MDK_OK;                     // allocated last: all five are there
    void **db[5] = {(void **)&e->quals, (void **)&e->ref, (void **)&e->calls, (void **)&e->pred_q, (void **)&e->ref_q};
    const size_t n = (size_t)e->cap_pos, bytes[5] = {n, n, n, n * sizeof(float), n * sizeof(float)};
    for (int i = 0; i < 5; ++i)
        if (!*db[i]) MDK_CUDA(cudaMalloc(db[i], bytes[i]));
    return MDK_OK;
}

void rl_mark(mdk_rl_engine *e, int i) {
    if (e->timing) cudaEventRecord(e->ev[e->pk.serial & 1][i], e->stream);
}

// The convolution of n windows of one call (host features x [n][P][D][F]) into z of the open group at window woff:
// mask, k = 1 and k = 17 convolutions, pooled Linear, in slices whose scratch RL_CONV_BUDGET bounds (one window at
// least).  Each slice's features go to a staging slot on copy_in; a slot is refilled once the convolution that read it
// is done.  Every window is its own grid slice of each kernel, so the slicing does not change any output bit.
int rl_conv(mdk_rl_engine *e, const int8_t *x, int64_t n, int64_t P, int64_t D, int64_t F, int64_t woff) {
    const int dgroup = RL_DGROUP;
    const int n_groups = (int)((D + dgroup - 1) / dgroup);
    const size_t xw = (size_t)P * D * F, yw = e->conv_tc ? 0 : (size_t)D * P * RL_C * 4, pw = (size_t)n_groups * P * RL_C * 4;
    const size_t per_window = 2 * xw + (size_t)D + yw + pw;
    const int64_t slice = std::max<int64_t>(1, std::min<int64_t>(n, (int64_t)(RL_CONV_BUDGET / per_window)));
    const size_t o_y1 = rl_round((size_t)slice * D), o_part = o_y1 + rl_round((size_t)slice * yw);
    int rc;
    if (o_part + (size_t)slice * pw > e->conv_cap) {
        MDK_CUDA(cudaStreamSynchronize(e->stream));
        if ((rc = rl_grow(&e->conv, &e->conv_cap, o_part + (size_t)slice * pw))) return rc;
    }
    cudaStream_t s = e->stream;
    uint8_t *d_mask = e->conv;
    float *d_y1 = (float *)(e->conv + o_y1), *d_part = (float *)(e->conv + o_part);
    RlConv1 c1{e->emb_base, e->emb_strand, e->c1_w, e->c1_b, e->bn1[0], e->bn1[1], e->bn1[2], e->bn1[3]};
    RlConv17 c17{e->c17_wt, e->c17_b, e->bn2[0], e->bn2[1], e->bn2[2], e->bn2[3]};
    if (e->conv_tc && e->fp16)
        MDK_CUDA(cudaFuncSetAttribute(rl_conv17_fp16_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, CT_SMEM<true>));
    else if (e->conv_tc)
        MDK_CUDA(cudaFuncSetAttribute(rl_conv17_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, CT_SMEM<false>));
    else MDK_CUDA(cudaFuncSetAttribute(rl_conv17_pool_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, RL_CONV_SMEM));
    for (int64_t s0 = 0; s0 < n; s0 += slice) {
        const int64_t B = std::min(slice, n - s0);
        const int k = e->xslot;
        e->xslot ^= 1;
        if ((size_t)B * xw > e->xcap[k]) {
            MDK_CUDA(cudaStreamSynchronize(e->stream));
            MDK_CUDA(cudaStreamSynchronize(e->copy_in));
            if ((rc = rl_grow(&e->xbuf[k], &e->xcap[k], (size_t)B * xw))) return rc;
        }
        MDK_CUDA(cudaStreamWaitEvent(e->copy_in, e->ev_xfree[k], 0));
        MDK_CUDA(cudaMemcpyAsync(e->xbuf[k], x + (size_t)s0 * xw, (size_t)B * xw, cudaMemcpyHostToDevice, e->copy_in));
        MDK_CUDA(cudaEventRecord(e->ev_xin[k], e->copy_in));
        MDK_CUDA(cudaStreamWaitEvent(s, e->ev_xin[k], 0));
        if (woff + s0 == 0) rl_mark(e, 0);
        const int8_t *d_x = e->xbuf[k];
        rl_mask_kernel<<<(unsigned)(B * D), 256, 0, s>>>(d_x, P, (int)D, (int)F, d_mask);
        const dim3 grid_tc((unsigned)((P + CT_NPOS - 1) / CT_NPOS), (unsigned)n_groups, (unsigned)B);
        if (e->conv_tc && e->fp16) {
            rl_conv17_fp16_kernel<<<grid_tc, 256, CT_SMEM<true>, s>>>(d_x, d_mask, c1, c17, (const uint8_t *)e->c17_tc, P,
                                                                         (int)D, (int)F, e->use_dwells, dgroup, d_part);
        } else if (e->conv_tc) {
            rl_conv17_tc_kernel<<<grid_tc, 256, CT_SMEM<false>, s>>>(d_x, d_mask, c1, c17, (const uint8_t *)e->c17_tc, P,
                                                                           (int)D, (int)F, e->use_dwells, dgroup, d_part);
        } else {
            rl_embed_conv1_kernel<<<dim3((unsigned)((P + 31) / 32), (unsigned)(B * D)), RL_C, 0, s>>>(d_x, d_mask, c1, P, (int)D, (int)F,
                                                                                                 e->use_dwells, d_y1);
            rl_conv17_pool_kernel<<<dim3((unsigned)((P + RL_PT - 1) / RL_PT), (unsigned)n_groups, (unsigned)B), 256, RL_CONV_SMEM, s>>>(
                d_y1, d_mask, c17, P, (int)D, dgroup, d_part);
        }
        MDK_CUDA(cudaEventRecord(e->ev_xfree[k], s));
        float *z = e->z + (size_t)(woff + s0) * P * e->H;
        if (e->H == RL_H3)
            rl_pool_linear_kernel<RL_H3><<<dim3((unsigned)((P + RL_PLT - 1) / RL_PLT), (unsigned)B), RL_C, 0, s>>>(
                d_part, d_mask, e->pool_w, e->pool_b, P, (int)D, n_groups, z);
        else
            rl_pool_linear_kernel<RL_H><<<dim3((unsigned)((P + RL_PLT - 1) / RL_PLT), (unsigned)B), RL_C, 0, s>>>(
                d_part, d_mask, e->pool_w, e->pool_b, P, (int)D, n_groups, z);
        MDK_CUDA(cudaGetLastError());
    }
    return MDK_OK;
}

// The LSTM input projection at lstm_size 384 and the recurrence of one layer on the tensor cores, in the fp16 mode's
// one-product form (FP16) or the three-product default
template <bool FP16>
cudaError_t rl_proj_tc(const float *in, const RlLstmLayer &L, float *gi, int64_t BP, int K, int N, cudaStream_t s) {
    const auto kernel = FP16 ? rl_proj_fp16_kernel : rl_proj_tc_kernel;
    const cudaError_t err = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, PJ_SMEM);
    if (err != cudaSuccess) return err;
    kernel<<<dim3((unsigned)((BP + PJ_N - 1) / PJ_N), N / PJ_M), 256, PJ_SMEM, s>>>(
        in, (const uint8_t *)L.w_ih_tc, L.bias, gi, BP, K, N);
    return cudaGetLastError();
}

template <bool FP16>
cudaError_t rl_rec_tc(bool h384, const float *gi, const RlLstmLayer &L, float *out, int64_t B, int64_t P, cudaStream_t s) {
    cudaError_t err;
    if (h384) {
        const auto kernel = FP16 ? rl_lstm384_fp16_kernel : rl_lstm384_tc_kernel;
        err = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, L3_SMEM<FP16>);
        if (err != cudaSuccess) return err;
        kernel<<<dim3((unsigned)((B + LT_N - 1) / LT_N * L3_CL), 2), L3_THREADS, L3_SMEM<FP16>, s>>>(
            gi, L.w_hi, (const uint8_t *)L.w_lo, out, B, P);
    } else {
        const auto kernel = FP16 ? rl_lstm_fp16_kernel : rl_lstm_tc_kernel;
        err = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, LT_SMEM<FP16>);
        if (err != cudaSuccess) return err;
        kernel<<<dim3((unsigned)((B + LT_N - 1) / LT_N), 2), LT_THREADS, LT_SMEM<FP16>, s>>>(
            gi, L.w_hi, (const uint8_t *)L.w_lo, out, B, P);
    }
    return cudaGetLastError();
}

// Run the sealed group: the projections, both recurrences and the head over all of its windows on the compute stream,
// then each call's probabilities (and labels) from the group buffers to its own buffers on copy_out.
int rl_run_group(mdk_rl_engine *e) {
    e->last_B = e->last_P = 0;                       // the group buffers are about to be overwritten
    const int64_t B = e->pk.windows, P = e->pk.len, BP = B * P;
    cudaStream_t s = e->stream;
    rl_mark(e, 1);
    const float *layer_in = e->z;
    float *layer_out[2] = {e->h0, e->h1};
    float *d_gi = e->gi;
    const bool h384 = e->H == RL_H3;
    const int G8 = 8 * e->H;                          // gate rows of both directions
    const dim3 grid_fp32((unsigned)((B + LF_NB - 1) / LF_NB), 2);
    for (int l = 0; l < 2; ++l) {
        const RlLstmLayer &L = e->lstm[l];
        const int in = l == 0 ? e->H : 2 * e->H;
        if (h384 && e->lstm_tc) {
            MDK_CUDA(e->fp16 ? rl_proj_tc<true>(layer_in, L, d_gi, BP, in, G8, s) : rl_proj_tc<false>(layer_in, L, d_gi, BP, in, G8, s));
        } else {
            MDK_CUDA(launch_gemm_fp32(layer_in, L.w_ih, L.bias, d_gi, BP, in, G8, s));
        }
        rl_mark(e, 2 + 2 * l);
        if (e->lstm_tc) {
            MDK_CUDA(e->fp16 ? rl_rec_tc<true>(h384, d_gi, L, layer_out[l], B, P, s)
                             : rl_rec_tc<false>(h384, d_gi, L, layer_out[l], B, P, s));
        } else if (h384) {
            rl_lstm_fp32<RL_H3, false><<<grid_fp32, RL_H3, 0, s>>>(d_gi, L.w_t, layer_out[l], B, P, nullptr);
        } else {
            rl_lstm_fp32<RL_H, false><<<grid_fp32, RL_H, 0, s>>>(d_gi, L.w_t, layer_out[l], B, P, nullptr);
        }
        rl_mark(e, 3 + 2 * l);
        layer_in = layer_out[l];
    }
    MDK_CUDA(cudaGetLastError());
    // the previous group's results must have left probs / labels (and the decoded outputs quals, calls, pred_q, ref_q,
    // which copy_back moves on the same stream before recording this event) before the head rewrites them
    if (e->pk.launched >= 0) MDK_CUDA(cudaStreamWaitEvent(s, e->copy_out.ev[e->pk.launched % CopyOut::RING], 0));
    // what the group's pieces want besides probabilities and labels, as GruCall::launch (api.cu)
    bool quals = false, var = false;
    for (const Packing::Piece &p : e->pk.pieces) {
        quals = quals || p.quals;
        var = var || p.ref;
    }
    const HeadVariant hv{e->ref, e->calls, e->pred_q, e->ref_q};
    uint8_t *q = quals ? e->quals : nullptr;
    if (e->H == RL_H3) {
        int64_t blocks = (BP + 7) / 8;
        if (blocks > 132 * 8) blocks = 132 * 8;
        const dim3 g((unsigned)blocks);
        if (var)
            rl_head768_kernel<HEAD_VARIANT><<<g, 256, 0, s>>>(e->h1, e->lin_w, e->lin_b, BP, e->probs, e->labels, q, hv);
        else if (quals)
            rl_head768_kernel<HEAD_QUALS><<<g, 256, 0, s>>>(e->h1, e->lin_w, e->lin_b, BP, e->probs, e->labels, q, {});
        else
            rl_head768_kernel<HEAD_PLAIN><<<g, 256, 0, s>>>(e->h1, e->lin_w, e->lin_b, BP, e->probs, e->labels, nullptr, {});
        MDK_CUDA(cudaGetLastError());
    } else {
        MDK_CUDA(launch_head(e->h1, e->lin_w, e->lin_b, B, P, 0, e->probs, nullptr, e->labels, s, q, var ? &hv : nullptr));
    }
    rl_mark(e, 6);
    return copy_back(e->copy_out, e->pk, s, e->probs, nullptr, e->labels, e->quals, &hv);
}

// The engine's side of the packing core (packing.h) for one call: x_host [B][P][D][F]; for a decoded call (quals or
// variant outputs) `decoded`, and for a variant-decoded one its reference bytes ref [B][P].  Launching alone (flush,
// sync, waits) needs no call.
struct RlCall {
    mdk_rl_engine *e;
    const int8_t *x = nullptr;
    int64_t P = 0, D = 0, F = 0;
    bool decoded = false;
    const uint8_t *ref = nullptr;

    // the group buffers grow, when a group opens, to this call's windows (at most one group of them): without
    // mdk_rl_reserve a group collects calls only as far as the buffers reach
    int open(int64_t windows) {
        e->last_B = e->last_P = 0;                   // this group's convolutions overwrite z of the last mdk_rl_forward
        return rl_ensure_group(e, windows * P);
    }
    int64_t capacity(int64_t len) { return e->cap_pos / len; }
    // The reference bytes go to the group's ref buffer on the COMPUTE stream, like the convolutions that fill z: the
    // group in flight may not have reached its head yet, and a copy on copy_in could overwrite the bytes it reads.
    int stage(int64_t first, int64_t n, int64_t at) {
        int rc;
        if (decoded && (rc = rl_ensure_decoded(e))) return rc;
        if (ref)
            MDK_CUDA(cudaMemcpyAsync(e->ref + (size_t)at * P, ref + (size_t)first * P, (size_t)n * P, cudaMemcpyDefault,
                                     e->stream));
        return rl_conv(e, x + (size_t)first * P * D * F, n, P, D, F, at);
    }
    int launch() { return rl_run_group(e); }
};

int rl_launch(mdk_rl_engine *e) { return e->pk.launch(RlCall{e}); }

// out: the output the call cannot do without (the probabilities, or a decoded call's labels / call bytes)
int rl_check(mdk_rl_engine *e, const int8_t *x, int64_t B, int64_t P, int64_t D, int64_t F, const void *out,
             const char *who) {
    const std::string w(who);
    MDK_REQUIRE(e && x && out, MDK_ERR_ARG, w + ": NULL argument");
    MDK_REQUIRE(B >= 1 && P >= 1 && D >= 1, MDK_ERR_ARG, w + ": need B, P, D >= 1");
    MDK_REQUIRE(F == (e->use_dwells ? 5 : 4) || (!e->use_dwells && F >= 4), MDK_ERR_ARG,
                w + ": feature vector length does not match the model (4, or 5 with dwells)");
    MDK_REQUIRE(D <= 65535 && B <= 65535, MDK_ERR_ARG, w + ": B, D <= 65535");
    return MDK_OK;
}

}  // namespace

extern "C" {

int mdk_rl_create(int device, int32_t lstm_size, int32_t cnn_size, int32_t use_dwells, int32_t num_classes,
                  mdk_rl_engine **out) {
    MDK_REQUIRE(out, MDK_ERR_ARG, "rl_create: out is NULL");
    *out = nullptr;
    MDK_REQUIRE((lstm_size == RL_H || lstm_size == RL_H3) && cnn_size == RL_C, MDK_ERR_UNSUPPORTED,
                "rl_create: supported sizes are lstm_size 128 or 384 with cnn_size 128");
    MDK_REQUIRE(num_classes == NCLS, MDK_ERR_UNSUPPORTED, "rl_create: 5 classes only");
    MDK_CUDA(cudaSetDevice(device));
    int sms = 0;
    MDK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
    mdk_rl_engine *e = new (std::nothrow) mdk_rl_engine();
    MDK_REQUIRE(e, MDK_ERR_NOMEM, "rl_create: out of host memory");
    e->device = device;
    e->use_dwells = use_dwells ? 1 : 0;
    e->H = lstm_size;
    e->sm_count = sms;
    cudaError_t err = cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking);
    if (err == cudaSuccess) err = cudaStreamCreateWithFlags(&e->copy_in, cudaStreamNonBlocking);
    if (err == cudaSuccess) err = create_copy_out(e->copy_out);
    for (int i = 0; i < 2 && err == cudaSuccess; ++i) {
        err = cudaEventCreateWithFlags(&e->ev_xin[i], cudaEventDisableTiming);
        if (err == cudaSuccess) err = cudaEventCreateWithFlags(&e->ev_xfree[i], cudaEventDisableTiming);
    }
    if (err != cudaSuccess) { mdk_rl_destroy(e); return cuda_fail(err, "rl_create: streams / events", __FILE__, __LINE__); }
    *out = e;
    return MDK_OK;
}

int mdk_rl_destroy(mdk_rl_engine *e) {
    if (!e) return MDK_OK;
    cudaSetDevice(e->device);
    for (cudaStream_t s : {e->copy_in, e->stream})
        if (s) { cudaStreamSynchronize(s); cudaStreamDestroy(s); }
    destroy_copy_out(e->copy_out);
    for (auto &set : e->ev)
        for (cudaEvent_t ev : set)
            if (ev) cudaEventDestroy(ev);
    for (cudaEvent_t ev : {e->ev_xin[0], e->ev_xin[1], e->ev_xfree[0], e->ev_xfree[1]})
        if (ev) cudaEventDestroy(ev);
    for (void *p : {(void *)e->xbuf[0], (void *)e->xbuf[1], (void *)e->conv, (void *)e->z, (void *)e->gi, (void *)e->h0,
                    (void *)e->h1, (void *)e->probs, (void *)e->labels, (void *)e->quals, (void *)e->ref,
                    (void *)e->calls, (void *)e->pred_q, (void *)e->ref_q})
        if (p) cudaFree(p);
    delete e;     // and with it the weights (DeviceWeights)
    cudaGetLastError();
    return MDK_OK;
}

int mdk_rl_load(mdk_rl_engine *e, const char *name, const float *data, int64_t n) {
    MDK_REQUIRE(e && name && (data || n == 0) && n >= 0, MDK_ERR_ARG, "rl_load: bad arguments");
    MDK_REQUIRE(!e->prepared, MDK_ERR_STATE, "rl_load: the model has already run; create a new engine to change weights");
    e->host[name] = std::vector<float>(data, data + n);
    return MDK_OK;
}

int mdk_rl_set_conv(mdk_rl_engine *e, int tensor_cores) {
    MDK_REQUIRE(e, MDK_ERR_ARG, "rl_set_conv: engine is NULL");
    const int conv_tc = (tensor_cores & 1) ? 1 : 0, lstm_tc = (tensor_cores & 2) ? 1 : 0, fp16 = (tensor_cores & 4) ? 1 : 0;
    if (conv_tc != e->conv_tc || lstm_tc != e->lstm_tc || fp16 != e->fp16) {
        // the open group's convolutions ran in the old mode: its LSTM and head run in that mode too
        MDK_CUDA(cudaSetDevice(e->device));
        const int rc = rl_launch(e);
        if (rc) return rc;
    }
    e->conv_tc = conv_tc;
    e->lstm_tc = lstm_tc;
    e->fp16 = fp16;
    return MDK_OK;
}

int mdk_rl_set_timing(mdk_rl_engine *e, int on) {
    MDK_REQUIRE(e, MDK_ERR_ARG, "rl_set_timing: engine is NULL");
    if (on && !e->ev[0][0]) {
        MDK_CUDA(cudaSetDevice(e->device));
        for (auto &set : e->ev)
            for (cudaEvent_t &ev : set) MDK_CUDA(cudaEventCreate(&ev));
    }
    e->timing = on ? 1 : 0;
    return MDK_OK;
}

int mdk_rl_stage_ms(mdk_rl_engine *e, float *ms) {
    MDK_REQUIRE(e && ms, MDK_ERR_ARG, "rl_stage_ms: NULL argument");
    for (int i = 0; i < 6; ++i) ms[i] = 0.f;
    if (e->pk.launched < 0 || !e->ev[0][0]) return MDK_OK;
    MDK_CUDA(cudaSetDevice(e->device));
    cudaEvent_t *ev = e->ev[e->pk.launched & 1];
    MDK_CUDA(cudaEventSynchronize(ev[6]));
    for (int i = 0; i < 6; ++i) MDK_CUDA(cudaEventElapsedTime(&ms[i], ev[i], ev[i + 1]));
    return MDK_OK;
}

// A submitted group never holds more than rl_group_limit windows, so the reservation is capped there: asking for a
// 200-window batch at lstm_size 384 and P = 10 000 must not allocate 40 GB of which 22 GB could ever be used.
int mdk_rl_reserve(mdk_rl_engine *e, int64_t windows, int64_t P) {
    MDK_REQUIRE(e && windows >= 1 && P >= 1, MDK_ERR_ARG, "rl_reserve: bad arguments");
    MDK_CUDA(cudaSetDevice(e->device));
    int64_t gmax = 0;
    int rc = rl_group_limit(e, P, &gmax);
    if (rc) return rc;
    if ((rc = rl_launch(e))) return rc;
    return rl_ensure_group(e, std::min(windows, gmax) * P);
}

int64_t mdk_rl_preferred_windows(mdk_rl_engine *e) {
    int64_t n = 0;
    if (!e || cudaSetDevice(e->device) != cudaSuccess || rl_group_limit(e, RL_PREFERRED_P, &n)) return 1;
    return n;
}

int mdk_rl_submit(mdk_rl_engine *e, const int8_t *x_host, int64_t B, int64_t P, int64_t D, int64_t F, float *probs_host,
                  uint8_t *labels_host, int64_t *ticket) {
    int rc = rl_check(e, x_host, B, P, D, F, probs_host, "rl_submit");
    if (rc) return rc;
    MDK_REQUIRE(ticket, MDK_ERR_ARG, "rl_submit: ticket is NULL");
    MDK_CUDA(cudaSetDevice(e->device));
    if ((rc = rl_prepare(e))) return rc;
    int64_t gmax = 0;
    if ((rc = rl_group_limit(e, P, &gmax))) return rc;
    return e->pk.enqueue(RlCall{e, x_host, P, D, F}, B, P, probs_host, nullptr, labels_host, gmax, ticket);
}

int mdk_rl_submit_decoded(mdk_rl_engine *e, const int8_t *x_host, int64_t B, int64_t P, int64_t D, int64_t F,
                          uint8_t *labels_out, uint8_t *quals_out, int64_t *ticket) {
    int rc = rl_check(e, x_host, B, P, D, F, labels_out, "rl_submit_decoded");
    if (rc) return rc;
    MDK_REQUIRE(ticket, MDK_ERR_ARG, "rl_submit_decoded: ticket is NULL");
    MDK_CUDA(cudaSetDevice(e->device));
    if ((rc = rl_prepare(e))) return rc;
    int64_t gmax = 0;
    if ((rc = rl_group_limit(e, P, &gmax))) return rc;
    return e->pk.enqueue(RlCall{e, x_host, P, D, F, quals_out != nullptr}, B, P, nullptr, nullptr, labels_out, gmax,
                         ticket, quals_out);
}

int mdk_rl_submit_variant_decoded(mdk_rl_engine *e, const int8_t *x_host, int64_t B, int64_t P, int64_t D, int64_t F,
                                  const uint8_t *ref_bytes, uint8_t *calls_out, float *pred_q_out, float *ref_q_out,
                                  int64_t *ticket) {
    int rc = rl_check(e, x_host, B, P, D, F, calls_out, "rl_submit_variant_decoded");
    if (rc) return rc;
    MDK_REQUIRE(ref_bytes && pred_q_out && ref_q_out, MDK_ERR_ARG, "rl_submit_variant_decoded: NULL argument");
    MDK_REQUIRE(ticket, MDK_ERR_ARG, "rl_submit_variant_decoded: ticket is NULL");
    MDK_CUDA(cudaSetDevice(e->device));
    if ((rc = rl_prepare(e))) return rc;
    int64_t gmax = 0;
    if ((rc = rl_group_limit(e, P, &gmax))) return rc;
    return e->pk.enqueue(RlCall{e, x_host, P, D, F, true, ref_bytes}, B, P, nullptr, nullptr, calls_out, gmax, ticket,
                         nullptr, ref_bytes, pred_q_out, ref_q_out);
}

int mdk_rl_sync(mdk_rl_engine *e) {
    MDK_REQUIRE(e, MDK_ERR_ARG, "rl_sync: engine is NULL");
    MDK_CUDA(cudaSetDevice(e->device));
    int rc = rl_launch(e);
    if (rc) return rc;
    MDK_CUDA(cudaStreamSynchronize(e->copy_in));
    MDK_CUDA(cudaStreamSynchronize(e->stream));
    MDK_CUDA(cudaStreamSynchronize(e->copy_out.stream));
    return MDK_OK;
}

int mdk_rl_flush(mdk_rl_engine *e) {
    MDK_REQUIRE(e, MDK_ERR_ARG, "rl_flush: engine is NULL");
    MDK_CUDA(cudaSetDevice(e->device));
    return rl_launch(e);
}

int mdk_rl_wait(mdk_rl_engine *e, int64_t ticket) {
    MDK_REQUIRE(e, MDK_ERR_ARG, "rl_wait: engine is NULL");
    MDK_REQUIRE(ticket >= 0 && ticket < e->pk.tickets, MDK_ERR_ARG, "rl_wait: unknown ticket");
    MDK_CUDA(cudaSetDevice(e->device));
    return wait_ticket(e->copy_out, e->pk, RlCall{e}, ticket);
}

// The one-call form: the open group is sealed, then this call runs as one group of its own (however many windows it
// has), so that mdk_rl_debug_read sees all of it.
int mdk_rl_forward(mdk_rl_engine *e, const int8_t *x_host, int64_t B, int64_t P, int64_t D, int64_t F, float *probs_host) {
    int rc = rl_check(e, x_host, B, P, D, F, probs_host, "rl_forward");
    if (rc) return rc;
    MDK_CUDA(cudaSetDevice(e->device));
    if ((rc = rl_prepare(e))) return rc;
    if ((rc = rl_launch(e))) return rc;
    int64_t gmax = 0, ticket = -1;
    if ((rc = rl_group_limit(e, P, &gmax))) return rc;
    if ((rc = e->pk.enqueue(RlCall{e, x_host, P, D, F}, B, P, probs_host, nullptr, nullptr, std::max(B, gmax), &ticket)))
        return rc;
    if ((rc = mdk_rl_wait(e, ticket))) return rc;
    e->last_B = B;
    e->last_P = P;
    return MDK_OK;
}

int mdk_rl_debug_read(mdk_rl_engine *e, int which, float *out_host, int64_t n_floats) {
    MDK_REQUIRE(e && out_host, MDK_ERR_ARG, "rl_debug_read: NULL argument");
    MDK_REQUIRE(which >= 0 && which <= 2, MDK_ERR_ARG, "rl_debug_read: which must be 0 (z), 1 (h0) or 2 (h1)");
    MDK_REQUIRE(e->last_B > 0, MDK_ERR_STATE, "rl_debug_read: no completed forward to read from");
    const int64_t want = e->last_B * e->last_P * (which == 0 ? e->H : 2 * e->H);
    MDK_REQUIRE(n_floats == want, MDK_ERR_ARG,
                "rl_debug_read: n_floats must be " + std::to_string(want) + " (B * P * H for z, B * P * 2H for h0 / h1)");
    MDK_CUDA(cudaSetDevice(e->device));
    MDK_CUDA(cudaStreamSynchronize(e->stream));
    const float *src = which == 0 ? e->z : which == 1 ? e->h0 : e->h1;
    MDK_CUDA(cudaMemcpy(out_host, src, (size_t)n_floats * sizeof(float), cudaMemcpyDeviceToHost));
    return MDK_OK;
}

}  // extern "C"
