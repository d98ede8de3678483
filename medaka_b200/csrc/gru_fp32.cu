// fp32 CUDA-core (FFMA) implementation of the GRU layer: the --full_precision / validation path
// (MDK_PREC_FP32).  Same data flow as the tensor-core path (gru_wg.cu) with fp32 operands:
//   gi  = X . W_ih^T + folded bias           (time-parallel GEMM, gemm_fp32; the read-level LSTM's fp32 projections too)
//   h_t = GRU cell(gi_t, h_{t-1} . W_hh^T)   (persistent recurrent kernel, rec_fp32)
// Reference arithmetic: torch.nn.GRU as used by medaka/architectures/gru.py:46-52,66.
#include "common.cuh"
#include "ptx.cuh"

namespace mdk {

__device__ __forceinline__ float sigmoid_acc(float x) { return 1.0f / (1.0f + expf(-x)); }

// -------------------------------------------------------------------------------------
// Recurrent kernel.  One CTA = NB windows of one direction; HS threads, thread j owns hidden
// unit j: the r/z/n rows of W_hh for unit j stream from shared memory (W_hh^T resident for the
// whole sequence, 192 KiB at HS = 128) or, at HS = 256 where W_hh^T takes 768 KiB, from L2, while
// the NB h vectors are shared-memory broadcasts.
// gi   [B*T][6 HS]  (position p = b*T + t ; columns dir*3HS + gate*HS + j)
// h_out[B*T][2 HS]  (columns dir*HS + j)
// SAVE (training, gru_train.cu): also the activations backpropagation through time reads,
// save[B*T][dir][4][HS] = r, z, n and W_hn.h_{t-1} + b_hn; the inference instantiation compiles as without it.
// -------------------------------------------------------------------------------------
constexpr int REC_NB = 8;

template <int HS, bool SAVE>
__global__ void __launch_bounds__(HS, 1) rec_fp32_kernel(const float *__restrict__ gi,
                                                         const float *__restrict__ w_hh_t,
                                                         const float *__restrict__ b_hn,
                                                         float *__restrict__ h_out, int64_t B, int64_t T,
                                                         float *__restrict__ save) {
    constexpr int G3S = 3 * HS, GIS = NDIR * G3S;
    constexpr bool SMEM_W = HS == H;
    extern __shared__ __align__(16) float smem[];
    float *hs = smem + (SMEM_W ? HS * G3S : 0);     // [2][NB][HS]
    const int j = threadIdx.x;
    const int dir = blockIdx.y;
    const int64_t b0 = (int64_t)blockIdx.x * REC_NB;
    const int nb = (int)min((int64_t)REC_NB, B - b0);

    const float *wsrc = w_hh_t + (int64_t)dir * HS * G3S;
    const float *wt = SMEM_W ? smem : wsrc;     // [HS][3 HS]
    if (SMEM_W)
        for (int i = j; i < HS * G3S / 4; i += HS)
            reinterpret_cast<float4 *>(smem)[i] = reinterpret_cast<const float4 *>(wsrc)[i];
    for (int i = j; i < 2 * REC_NB * HS; i += HS) hs[i] = 0.f;
    const float bhn = b_hn[dir * HS + j];
    float hprev[REC_NB];
#pragma unroll
    for (int n = 0; n < REC_NB; ++n) hprev[n] = 0.f;
    __syncthreads();

    const int64_t col = (int64_t)dir * G3S + j;
    float gnext[3][REC_NB];
    {
        const int64_t t = dir ? (T - 1) : 0;
#pragma unroll
        for (int n = 0; n < REC_NB; ++n) {
            const bool ok = n < nb;
            const float *row = gi + ((b0 + (ok ? n : 0)) * T + t) * GIS + col;
#pragma unroll
            for (int g = 0; g < 3; ++g) gnext[g][n] = ok ? ldg_stream(row + g * HS) : 0.f;
        }
    }
    int cur = 0;
    for (int64_t step = 0; step < T; ++step) {
        const int64_t t = dir ? (T - 1 - step) : step;
        float gcur[3][REC_NB];
#pragma unroll
        for (int g = 0; g < 3; ++g)
#pragma unroll
            for (int n = 0; n < REC_NB; ++n) gcur[g][n] = gnext[g][n];
        if (step + 1 < T) {   // prefetch next step's pre-activations while this step's matvec runs
            const int64_t tn = dir ? (t - 1) : (t + 1);
#pragma unroll
            for (int n = 0; n < REC_NB; ++n) {
                const bool ok = n < nb;
                const float *row = gi + ((b0 + (ok ? n : 0)) * T + tn) * GIS + col;
#pragma unroll
                for (int g = 0; g < 3; ++g) gnext[g][n] = ok ? ldg_stream(row + g * HS) : 0.f;
            }
        }
        float acc[3][REC_NB];
#pragma unroll
        for (int g = 0; g < 3; ++g)
#pragma unroll
            for (int n = 0; n < REC_NB; ++n) acc[g][n] = 0.f;
        const float *hc = hs + cur * REC_NB * HS;
#pragma unroll 2
        for (int k = 0; k < HS; k += 4) {
            float4 hv[REC_NB];
#pragma unroll
            for (int n = 0; n < REC_NB; ++n) hv[n] = *reinterpret_cast<const float4 *>(hc + n * HS + k);
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
                const float wr = wt[(k + kk) * G3S + j];
                const float wz = wt[(k + kk) * G3S + HS + j];
                const float wn = wt[(k + kk) * G3S + 2 * HS + j];
#pragma unroll
                for (int n = 0; n < REC_NB; ++n) {
                    const float hvk = kk == 0 ? hv[n].x : kk == 1 ? hv[n].y : kk == 2 ? hv[n].z : hv[n].w;
                    acc[0][n] = fmaf(wr, hvk, acc[0][n]);
                    acc[1][n] = fmaf(wz, hvk, acc[1][n]);
                    acc[2][n] = fmaf(wn, hvk, acc[2][n]);
                }
            }
        }
        float *hn = hs + (cur ^ 1) * REC_NB * HS;
#pragma unroll
        for (int n = 0; n < REC_NB; ++n) {
            const float r = sigmoid_acc(gcur[0][n] + acc[0][n]);
            const float z = sigmoid_acc(gcur[1][n] + acc[1][n]);
            const float ghn = acc[2][n] + bhn;
            const float nn = tanhf(gcur[2][n] + r * ghn);
            const float h = (1.0f - z) * nn + z * hprev[n];
            hprev[n] = h;
            hn[n * HS + j] = h;
            if (n < nb) h_out[((b0 + n) * T + t) * (NDIR * HS) + dir * HS + j] = h;
            if (SAVE && n < nb) {
                float *sv = save + (((b0 + n) * T + t) * NDIR + dir) * (4 * HS) + j;
                sv[0] = r; sv[HS] = z; sv[2 * HS] = nn; sv[3 * HS] = ghn;
            }
        }
        __syncthreads();
        cur ^= 1;
    }
}

template <int HS, bool SAVE>
static cudaError_t launch_rec_fp32_hs(const float *gi, const float *w_hh_t, const float *b_hn, float *h_out, int64_t B,
                                      int64_t T, cudaStream_t s, float *save) {
    const size_t smem = (size_t)((HS == H ? HS * 3 * HS : 0) + 2 * REC_NB * HS) * sizeof(float);
    // (the attribute is per device: set it on every launch, a process may drive several GPUs from several threads)
    cudaError_t e = cudaFuncSetAttribute(rec_fp32_kernel<HS, SAVE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    dim3 grid((unsigned)((B + REC_NB - 1) / REC_NB), NDIR);
    rec_fp32_kernel<HS, SAVE><<<grid, HS, smem, s>>>(gi, w_hh_t, b_hn, h_out, B, T, save);
    return cudaGetLastError();
}

cudaError_t launch_rec_fp32(const float *gi, const float *w_hh_t, const float *b_hn, float *h_out, int64_t B,
                            int64_t T, cudaStream_t s, int hs, float *save) {
    if (B == 0 || T == 0) return cudaSuccess;
    if (save)
        return hs == H256 ? launch_rec_fp32_hs<H256, true>(gi, w_hh_t, b_hn, h_out, B, T, s, save)
                          : launch_rec_fp32_hs<H, true>(gi, w_hh_t, b_hn, h_out, B, T, s, save);
    return hs == H256 ? launch_rec_fp32_hs<H256, false>(gi, w_hh_t, b_hn, h_out, B, T, s, nullptr)
                      : launch_rec_fp32_hs<H, false>(gi, w_hh_t, b_hn, h_out, B, T, s, nullptr);
}

// -------------------------------------------------------------------------------------
// Input projections, fp32: C[M][N] = A[M][K] . W[N][K]^T + bias[N];  K % 16 == 0, N % 128 == 0.
// The GRU's layer 1 (K = 256, N = 768; K = 512, N = 1536 at gru_size 256) and both layers of the read-level LSTM at either size.
// Classic 128x128x16 shared-memory tiling, 256 threads, 8x8 register tile.
// -------------------------------------------------------------------------------------
constexpr int GM = 128, GN = 128, GK = 16;

__global__ void __launch_bounds__(256) gemm_fp32_kernel(const float *__restrict__ A, const float *__restrict__ W,
                                                        const float *__restrict__ bias, float *__restrict__ C, int64_t M,
                                                        int K, int N) {
    __shared__ float As[GK][GM + 4];
    __shared__ float Ws[GK][GN + 4];
    const int tid = threadIdx.x;
    const int64_t m0 = (int64_t)blockIdx.x * GM;
    const int n0 = blockIdx.y * GN;
    const int tx = tid % 16, ty = tid / 16;   // 16x16 threads, each 8x8 outputs
    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
    // loader mapping: 128 rows x 16 k = 512 float4; thread loads 2 float4 per operand
    const int lrow = tid / 4, lk = (tid % 4) * 4;
    for (int k0 = 0; k0 < K; k0 += GK) {
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            const int r = lrow + half * 64;
            const int64_t gm = m0 + r;
            float4 av = make_float4(0.f, 0.f, 0.f, 0.f);
            if (gm < M) av = *reinterpret_cast<const float4 *>(A + gm * K + k0 + lk);
            As[lk + 0][r] = av.x; As[lk + 1][r] = av.y; As[lk + 2][r] = av.z; As[lk + 3][r] = av.w;
            const float4 wv = *reinterpret_cast<const float4 *>(W + (int64_t)(n0 + r) * K + k0 + lk);
            Ws[lk + 0][r] = wv.x; Ws[lk + 1][r] = wv.y; Ws[lk + 2][r] = wv.z; Ws[lk + 3][r] = wv.w;
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < GK; ++k) {
            // rows {ty*4..+3, 64+ty*4..+3}, cols {tx*4..+3, 64+tx*4..+3}: conflict-free float4 smem reads
            const float4 a0 = *reinterpret_cast<const float4 *>(&As[k][ty * 4]);
            const float4 a1 = *reinterpret_cast<const float4 *>(&As[k][64 + ty * 4]);
            const float4 b0 = *reinterpret_cast<const float4 *>(&Ws[k][tx * 4]);
            const float4 b1 = *reinterpret_cast<const float4 *>(&Ws[k][64 + tx * 4]);
            const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        __syncthreads();
    }
    float bv[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) bv[j] = bias[n0 + (j < 4 ? tx * 4 + j : 64 + tx * 4 + j - 4)];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int64_t gm = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + i - 4);
        if (gm >= M) continue;
        float *dst = C + gm * N + n0;
        *reinterpret_cast<float4 *>(dst + tx * 4) = make_float4(acc[i][0] + bv[0], acc[i][1] + bv[1], acc[i][2] + bv[2], acc[i][3] + bv[3]);
        *reinterpret_cast<float4 *>(dst + 64 + tx * 4) = make_float4(acc[i][4] + bv[4], acc[i][5] + bv[5], acc[i][6] + bv[6], acc[i][7] + bv[7]);
    }
}

cudaError_t launch_gemm_fp32(const float *A, const float *W, const float *bias, float *C, int64_t M, int K, int N,
                             cudaStream_t s) {
    if (M == 0) return cudaSuccess;
    dim3 grid((unsigned)((M + GM - 1) / GM), N / GN);
    gemm_fp32_kernel<<<grid, 256, 0, s>>>(A, W, bias, C, M, K, N);
    return cudaGetLastError();
}

}  // namespace mdk
