// Tensor-core kernels of the consensus GRU at gru_size = 256 (the width `medaka train` builds by default): the layer-1
// input projection and the recurrence of either layer.  Same arithmetic as the H = 128 path (gru_wg.cu): fp16 hi / lo
// operands, three products hi.hi + hi.lo + lo.hi with fp32 accumulation, gate pre-activations pre-scaled for exp2
// (common.cuh gate_scale).  The intermediates are plain fp32 rows in tile-interleaved order (common.cuh tiled_row):
//   gi [rows][1536]  columns dir * 768 + gate * 256 + j
//   h  [rows][512]   columns dir * 256 + j (h0, read by the projection; h1, read by the head)
// The layer-0 input projection and the head are the width-templated kernels of misc.cu.
// MDK_PREC_FP16: rec256_fp16_kernel and gemm256_fp16_kernel, the FP16 = true forms of the same bodies, take one product
// per contraction, hi.hi (operands rounded to the nearest fp16, fp32 accumulation).
#include "common.cuh"
#include "ptx.cuh"

namespace mdk {

namespace {

// D += A . B, m16n8k16, fp16 operands, fp32 accumulators
__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], uint32_t smem_addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
                 : "r"(smem_addr));
}

}  // namespace

// ---------------------------------------------------------------------------------------------- recurrence on a cluster
// Per time step G[768][16 windows] = W_hh . h^T for one (16-window tile, direction), split over a cluster of 4 CTAs:
// CTA rank c owns hidden units 64c .. 64c + 63, i.e. 192 gate rows.  12 warps; warp w computes gate w / 4 of units
// 64c + 16 (w % 4) .. + 15 with mma.sync m16n8k16 over K = 256 (16 k-steps x 2 n-tiles x 3 products = 96 MMAs):
//   A = W_hh rows: the fp16 hi plane in registers (16 k-steps x 4 = 64 per thread), the lo plane in shared memory
//       (192 rows x 256, 96 KiB + padding), both loaded once
//   B = the full h tile [16 windows][256 units] (fp16 hi | lo), double buffered: every CTA holds all 256 units
// The three gates of a unit come from three warps: they meet in an 18 KiB exchange buffer, where threads 0..255 each take
// two units x two windows and keep h in fp32 registers across steps.  Each writes its new h (hi / lo, two units packed)
// into the next h buffer of all 4 CTAs with st.shared::cluster, and as fp32 into the output rows.  One cluster barrier
// (release / acquire) per step then publishes the buffer; it also orders the step's exchange reads before the next
// step's writes, and the one after the last step keeps every CTA alive until no peer writes into its shared memory.
// FP16 (rec256_fp16_kernel): one product, W_hi.h_hi, 32 MMAs per warp-step; no W lo block in shared memory, and only h's
// hi half goes to the peers.  h still leaves the kernel as fp32 rows.
constexpr int R2_CL = 4;                        // CTAs per cluster
constexpr int R2_UNITS = H256 / R2_CL;          // 64 hidden units per CTA
constexpr int R2_ROWS = 3 * R2_UNITS;           // 192 gate rows per CTA
constexpr int R2_THREADS = 384;                 // 12 warps: (gate, 16-unit block)
constexpr int R2_KS = H256 / 16;                // 16 k-steps
constexpr int R2_KP = H256 + 8;                 // row stride of the shared-memory operands (halfs): ldmatrix conflict-free
constexpr int R2_XS = WT + 8;                   // row stride of the gate exchange (floats)
constexpr int R2_WLO_BYTES = R2_ROWS * R2_KP * 2;           // 99 KiB
constexpr int R2_HPLANE = WT * R2_KP;                       // halfs of one h plane (hi or lo)
constexpr int R2_HBUF_BYTES = 2 * 2 * R2_HPLANE * 2;        // [buffer][hi | lo], 33 KiB
template <bool FP16> constexpr int R2_WLO = FP16 ? 0 : R2_WLO_BYTES;
template <bool FP16>
constexpr int R2_SMEM = R2_WLO<FP16> + R2_HBUF_BYTES + R2_ROWS * R2_XS * 4;   // 150 KiB (18 KiB exchange; FP16: 51 KiB)

template <bool FP16>
__device__ __forceinline__ void rec256_body(const float *__restrict__ gi, const __half *__restrict__ w_hh_tm,
                                            const float *__restrict__ b_hn, float *__restrict__ h_out, int64_t T) {
    extern __shared__ __align__(16) uint8_t smem[];
    __half *wlo = reinterpret_cast<__half *>(smem);
    __half *hbuf = reinterpret_cast<__half *>(smem + R2_WLO<FP16>);     // [buf][part][window][R2_KP]
    float *xch = reinterpret_cast<float *>(smem + R2_WLO<FP16> + R2_HBUF_BYTES);   // [gate row][R2_XS]
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t rank = cluster_ctarank();
    const int dir = blockIdx.y;
    const int64_t tile = blockIdx.x / R2_CL;
    const int u0 = (int)rank * R2_UNITS;

    // A operands: hi plane into registers, lo plane into shared memory ([d][part][gate][j][k], gru_pack.cuh)
    const int g_w = warp >> 2, rb = (warp & 3) * 16;
    uint32_t ahi[R2_KS][4];
    {
        const __half *hi = w_hh_tm + ((size_t)(dir * 2 + 0) * 3 + g_w) * H256 * H256;
        const int r0 = u0 + rb + (lane >> 2), k0 = (lane & 3) * 2;
#pragma unroll
        for (int ks = 0; ks < R2_KS; ++ks) {
            const __half *p = hi + (size_t)r0 * H256 + ks * 16 + k0;
            ahi[ks][0] = *reinterpret_cast<const uint32_t *>(p);
            ahi[ks][1] = *reinterpret_cast<const uint32_t *>(p + 8 * H256);
            ahi[ks][2] = *reinterpret_cast<const uint32_t *>(p + 8);
            ahi[ks][3] = *reinterpret_cast<const uint32_t *>(p + 8 * H256 + 8);
        }
    }
    for (int i = tid; i < (FP16 ? 0 : R2_ROWS * (H256 / 8)); i += R2_THREADS) {
        const int r = i / (H256 / 8), kc = (i % (H256 / 8)) * 8, g = r / R2_UNITS, u = r % R2_UNITS;
        const __half *src = w_hh_tm + (((size_t)(dir * 2 + 1) * 3 + g) * H256 + u0 + u) * H256 + kc;
        *reinterpret_cast<uint4 *>(wlo + r * R2_KP + kc) = *reinterpret_cast<const uint4 *>(src);
    }
    for (int i = tid; i < R2_HBUF_BYTES / 16; i += R2_THREADS) reinterpret_cast<uint4 *>(hbuf)[i] = make_uint4(0, 0, 0, 0);

    // gate-math role (threads 0..255): units u0 + 2 up, + 1 and windows wq, wq + 8
    const bool gm = tid < 256;
    const int up = tid & 31, wq = (tid >> 5) & 7;
    const int uc = u0 + 2 * up;                               // first of the thread's two units
    float hprev[2][2] = {{0.f, 0.f}, {0.f, 0.f}};            // [window][unit]
    float2 bhn = make_float2(0.f, 0.f);
    if (gm) bhn = *reinterpret_cast<const float2 *>(b_hn + dir * H256 + uc);
    uint32_t peer[R2_CL];
#pragma unroll
    for (int q = 0; q < R2_CL; ++q) peer[q] = mapa_shared(smem_u32(hbuf), (uint32_t)q);

    const float *gi_col = gi + dir * G3_256 + uc;
    auto gi_row = [&](int64_t t, int w) { return ((tile * T + t) * WT + w) * (int64_t)GI256_COLS; };
    float2 gnext[2][3];
    if (gm) {
        const int64_t t = dir ? T - 1 : 0;
#pragma unroll
        for (int n = 0; n < 2; ++n)
#pragma unroll
            for (int g = 0; g < 3; ++g)
                gnext[n][g] = *reinterpret_cast<const float2 *>(gi_col + gi_row(t, wq + 8 * n) + g * H256);
    }
    // ldmatrix lane addresses: A lo rows rb + (lane % 16) of gate g_w, k half (lane / 16); B windows (lane / 16) * 8 +
    // lane % 8, k half (lane / 8) % 2
    const uint32_t a_lo_addr = smem_u32(wlo + (g_w * R2_UNITS + rb + (lane & 15)) * R2_KP + (lane >> 4) * 8);
    const uint32_t b_off = (uint32_t)((((lane >> 4) * 8 + (lane & 7)) * R2_KP + ((lane >> 3) & 1) * 8) * 2);
    const uint32_t hbuf_addr = smem_u32(hbuf);
    cluster_sync_all();    // every CTA's h buffer zeroed before any peer writes into it

    for (int64_t step = 0; step < T; ++step) {
        const int buf = (int)(step & 1);
        const int64_t t = dir ? T - 1 - step : step;
        float2 gcur[2][3];
#pragma unroll
        for (int n = 0; n < 2; ++n)
#pragma unroll
            for (int g = 0; g < 3; ++g) gcur[n][g] = gnext[n][g];
        if (gm && step + 1 < T) {
            const int64_t tn = dir ? t - 1 : t + 1;
#pragma unroll
            for (int n = 0; n < 2; ++n)
#pragma unroll
                for (int g = 0; g < 3; ++g)
                    gnext[n][g] = *reinterpret_cast<const float2 *>(gi_col + gi_row(tn, wq + 8 * n) + g * H256);
        }
        float acc[2][4] = {};
        const uint32_t hhi = hbuf_addr + (uint32_t)(buf * 2 * R2_HPLANE * 2) + b_off, hlo = hhi + R2_HPLANE * 2;
#pragma unroll
        for (int ks = 0; ks < R2_KS; ++ks) {
            uint32_t bh[4], bl[4], alo[4];
            ldmatrix_x4(bh, hhi + ks * 32);
            if constexpr (FP16) {
#pragma unroll
                for (int nt = 0; nt < 2; ++nt) mma16816(acc[nt], ahi[ks], bh[2 * nt], bh[2 * nt + 1]);
                continue;
            }
            ldmatrix_x4(bl, hlo + ks * 32);
            ldmatrix_x4(alo, a_lo_addr + ks * 32);
#pragma unroll
            for (int nt = 0; nt < 2; ++nt) {
                mma16816(acc[nt], ahi[ks], bh[2 * nt], bh[2 * nt + 1]);
                mma16816(acc[nt], ahi[ks], bl[2 * nt], bl[2 * nt + 1]);
                mma16816(acc[nt], alo, bh[2 * nt], bh[2 * nt + 1]);
            }
        }
#pragma unroll
        for (int nt = 0; nt < 2; ++nt) {
            float *x = xch + (g_w * R2_UNITS + rb + (lane >> 2)) * R2_XS + nt * 8 + (lane & 3) * 2;
            *reinterpret_cast<float2 *>(x) = make_float2(acc[nt][0], acc[nt][1]);
            *reinterpret_cast<float2 *>(x + 8 * R2_XS) = make_float2(acc[nt][2], acc[nt][3]);
        }
        __syncthreads();
        if (gm) {
            const int nxt = buf ^ 1;
#pragma unroll
            for (int n = 0; n < 2; ++n) {
                const int w = wq + 8 * n;
                float hn[2];
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int ul = 2 * up + e;
                    const float pr = xch[ul * R2_XS + w], pz = xch[(R2_UNITS + ul) * R2_XS + w];
                    const float pn = xch[(2 * R2_UNITS + ul) * R2_XS + w];
                    const float gr = e ? gcur[n][0].y : gcur[n][0].x, gz = e ? gcur[n][1].y : gcur[n][1].x;
                    const float gn = e ? gcur[n][2].y : gcur[n][2].x, bn = e ? bhn.y : bhn.x;
                    // pre-scaled: r = 1 / (1 + 2^a), z likewise, n = tanh = 1 - 2 / (2^a + 1)
                    const float r = 1.0f / (1.0f + exp2f(gr + pr));
                    const float z = 1.0f / (1.0f + exp2f(gz + pz));
                    const float nn = 1.0f - 2.0f / (exp2f(gn + r * (pn + bn)) + 1.0f);
                    hn[e] = (1.0f - z) * nn + z * hprev[n][e];
                    hprev[n][e] = hn[e];
                }
                uint32_t vhi, vlo;
                split_f16x2(hn[0], hn[1], vhi, vlo);
                const uint32_t off = (uint32_t)(((nxt * 2) * R2_HPLANE + w * R2_KP + uc) * 2);
#pragma unroll
                for (int q = 0; q < R2_CL; ++q) {
                    st_cluster_u32(peer[q] + off, vhi);
                    if (!FP16) st_cluster_u32(peer[q] + off + R2_HPLANE * 2, vlo);
                }
                *reinterpret_cast<float2 *>(h_out + ((tile * T + t) * WT + w) * H2_256 + dir * H256 + uc) =
                    make_float2(hn[0], hn[1]);
            }
        }
        cluster_sync_all();
    }
}

__global__ void __cluster_dims__(R2_CL, 1, 1) __launch_bounds__(R2_THREADS, 1)
    rec256_tc_kernel(const float *__restrict__ gi, const __half *__restrict__ w_hh_tm, const float *__restrict__ b_hn,
                     float *__restrict__ h_out, int64_t T) {
    rec256_body<false>(gi, w_hh_tm, b_hn, h_out, T);
}
__global__ void __cluster_dims__(R2_CL, 1, 1) __launch_bounds__(R2_THREADS, 1)
    rec256_fp16_kernel(const float *__restrict__ gi, const __half *__restrict__ w_hh_tm, const float *__restrict__ b_hn,
                       float *__restrict__ h_out, int64_t T) {
    rec256_body<true>(gi, w_hh_tm, b_hn, h_out, T);
}

// (the three-product kernel: the fp16 one needs less shared memory and fits at least as many clusters, so one wave, and
// with it the group size, does not depend on the precision)
cudaError_t rec256_max_clusters(int *clusters) {
    cudaError_t e = cudaFuncSetAttribute(rec256_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, R2_SMEM<false>);
    if (e != cudaSuccess) return e;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(R2_CL, NDIR);
    cfg.blockDim = dim3(R2_THREADS);
    cfg.dynamicSmemBytes = R2_SMEM<false>;
    cudaLaunchAttribute attr;
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = R2_CL;
    attr.val.clusterDim.y = 1;
    attr.val.clusterDim.z = 1;
    cfg.attrs = &attr;
    cfg.numAttrs = 1;
    return cudaOccupancyMaxActiveClusters(clusters, (void *)rec256_tc_kernel, &cfg);
}

template <bool FP16>
static cudaError_t launch_rec256(const float *gi, const __half *w_hh_tm, const float *b_hn, float *h_out, int64_t B,
                                 int64_t T, cudaStream_t s) {
    const auto kernel = FP16 ? rec256_fp16_kernel : rec256_tc_kernel;
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, R2_SMEM<FP16>);
    if (e != cudaSuccess) return e;
    const dim3 grid((unsigned)(((B + WT - 1) / WT) * R2_CL), NDIR);
    kernel<<<grid, R2_THREADS, R2_SMEM<FP16>, s>>>(gi, w_hh_tm, b_hn, h_out, T);
    return cudaGetLastError();
}

cudaError_t launch_rec256_tc(const float *gi, const __half *w_hh_tm, const float *b_hn, float *h_out, int64_t B,
                             int64_t T, bool fp16, cudaStream_t s) {
    if (B == 0 || T == 0) return cudaSuccess;
    return fp16 ? launch_rec256<true>(gi, w_hh_tm, b_hn, h_out, B, T, s)
                : launch_rec256<false>(gi, w_hh_tm, b_hn, h_out, B, T, s);
}

// ---------------------------------------------------------------------------------------------- layer-1 projection
// gi[M][1536] = h0[M][512] . W_ih^T + bias (W_ih and bias pre-scaled), three products x_hi.w_hi + x_hi.w_lo + x_lo.w_hi.
// At K = 512, N = 1536 the weights (3 MiB as hi / lo) do not fit the register operands of gemm_tc_kernel: 128 x 128
// output blocks stream 32-wide K slices of both operands through shared memory.  The fp32 activations are split into hi /
// lo as they are staged.  8 warps, 2 (M) x 4 (N), each a 64 x 32 block of 4 x 4 m16n8 tiles.
// FP16 (gemm256_fp16_kernel): one product, x_hi.w_hi: only the hi planes are staged.
constexpr int G2_BM = 128, G2_BN = 128, G2_BK = 32, G2_KP = G2_BK + 8;   // padded row: ldmatrix conflict-free

template <bool FP16>
__device__ __forceinline__ void gemm256_body(const float *__restrict__ x, const __half *__restrict__ w_in_tm,
                                             const float *__restrict__ bias, float *__restrict__ gi, int64_t M) {
    __shared__ __align__(16) __half sa[FP16 ? 1 : 2][G2_BM * G2_KP];    // [hi | lo][row][k]
    __shared__ __align__(16) __half sb[FP16 ? 1 : 2][G2_BN * G2_KP];    // [hi | lo][col][k]
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int wm = warp >> 2, wn = warp & 3;
    const int64_t m0 = (int64_t)blockIdx.x * G2_BM;
    const int n0 = blockIdx.y * G2_BN;
    // weight rows n0 .. n0 + 127 lie in one block blk = n0 / 256 of [blk][part][j][512] (gru_pack.cuh)
    const int blk = n0 / H256, j0 = n0 % H256;
    const __half *whi = w_in_tm + ((size_t)blk * 2 + 0) * H256 * H2_256 + (size_t)j0 * H2_256;
    const __half *wlo = whi + (size_t)H256 * H2_256;
    float acc[4][4][4] = {};
    const uint32_t a_addr = smem_u32(&sa[0][(wm * 64 + (lane & 15)) * G2_KP + (lane >> 4) * 8]);
    const uint32_t b_addr = smem_u32(&sb[0][(wn * 32 + (lane >> 4) * 8 + (lane & 7)) * G2_KP + ((lane >> 3) & 1) * 8]);
    constexpr uint32_t PLANE_A = G2_BM * G2_KP * 2, PLANE_B = G2_BN * G2_KP * 2;
    for (int k0 = 0; k0 < H2_256; k0 += G2_BK) {
        // activations: 128 rows x 32 k = 1024 float4, 4 per thread
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int idx = tid + 256 * i, r = idx >> 3, kc = (idx & 7) * 4;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (m0 + r < M) v = ld_stream4(x + (m0 + r) * H2_256 + k0 + kc);
            uint32_t h01, l01, h23, l23;
            split_f16x2(v.x, v.y, h01, l01);
            split_f16x2(v.z, v.w, h23, l23);
            *reinterpret_cast<uint2 *>(&sa[0][r * G2_KP + kc]) = make_uint2(h01, h23);
            if constexpr (!FP16) *reinterpret_cast<uint2 *>(&sa[1][r * G2_KP + kc]) = make_uint2(l01, l23);
        }
        // weights: 128 rows x 32 k per plane = 512 uint4, 2 per thread per plane
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int idx = tid + 256 * i, r = idx >> 2, kc = (idx & 3) * 8;
            *reinterpret_cast<uint4 *>(&sb[0][r * G2_KP + kc]) =
                *reinterpret_cast<const uint4 *>(whi + (size_t)r * H2_256 + k0 + kc);
            if constexpr (!FP16)
                *reinterpret_cast<uint4 *>(&sb[1][r * G2_KP + kc]) =
                    *reinterpret_cast<const uint4 *>(wlo + (size_t)r * H2_256 + k0 + kc);
        }
        __syncthreads();
#pragma unroll
        for (int ks = 0; ks < G2_BK / 16; ++ks) {
            uint32_t ah[4][4], al[4][4], bh[2][4], bl[2][4];
#pragma unroll
            for (int mt = 0; mt < 4; ++mt) {
                ldmatrix_x4(ah[mt], a_addr + (uint32_t)((mt * 16 * G2_KP + ks * 16) * 2));
                if (!FP16) ldmatrix_x4(al[mt], a_addr + PLANE_A + (uint32_t)((mt * 16 * G2_KP + ks * 16) * 2));
            }
#pragma unroll
            for (int np = 0; np < 2; ++np) {
                ldmatrix_x4(bh[np], b_addr + (uint32_t)((np * 16 * G2_KP + ks * 16) * 2));
                if (!FP16) ldmatrix_x4(bl[np], b_addr + PLANE_B + (uint32_t)((np * 16 * G2_KP + ks * 16) * 2));
            }
#pragma unroll
            for (int mt = 0; mt < 4; ++mt)
#pragma unroll
                for (int nt = 0; nt < 4; ++nt) {
                    const int np = nt >> 1, q = (nt & 1) * 2;
                    mma16816(acc[mt][nt], ah[mt], bh[np][q], bh[np][q + 1]);
                    if (FP16) continue;
                    mma16816(acc[mt][nt], ah[mt], bl[np][q], bl[np][q + 1]);
                    mma16816(acc[mt][nt], al[mt], bh[np][q], bh[np][q + 1]);
                }
        }
        __syncthreads();
    }
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
        const int n = n0 + wn * 32 + nt * 8 + (lane & 3) * 2;
        const float2 b = *reinterpret_cast<const float2 *>(bias + n);
#pragma unroll
        for (int mt = 0; mt < 4; ++mt) {
            const int64_t r = m0 + wm * 64 + mt * 16 + (lane >> 2);
            if (r < M)
                *reinterpret_cast<float2 *>(gi + r * GI256_COLS + n) =
                    make_float2(acc[mt][nt][0] + b.x, acc[mt][nt][1] + b.y);
            if (r + 8 < M)
                *reinterpret_cast<float2 *>(gi + (r + 8) * GI256_COLS + n) =
                    make_float2(acc[mt][nt][2] + b.x, acc[mt][nt][3] + b.y);
        }
    }
}

__global__ void __launch_bounds__(256) gemm256_tc_kernel(const float *__restrict__ x, const __half *__restrict__ w_in_tm,
                                                         const float *__restrict__ bias, float *__restrict__ gi,
                                                         int64_t M) {
    gemm256_body<false>(x, w_in_tm, bias, gi, M);
}
__global__ void __launch_bounds__(256) gemm256_fp16_kernel(const float *__restrict__ x, const __half *__restrict__ w_in_tm,
                                                           const float *__restrict__ bias, float *__restrict__ gi,
                                                           int64_t M) {
    gemm256_body<true>(x, w_in_tm, bias, gi, M);
}

cudaError_t launch_gemm256_tc(const float *h0, const __half *w_in_tm, const float *bias, float *gi, int64_t M, bool fp16,
                              cudaStream_t s) {
    if (M == 0) return cudaSuccess;
    const dim3 grid((unsigned)((M + G2_BM - 1) / G2_BM), GI256_COLS / G2_BN);
    (fp16 ? gemm256_fp16_kernel : gemm256_tc_kernel)<<<grid, 256, 0, s>>>(h0, w_in_tm, bias, gi, M);
    return cudaGetLastError();
}

}  // namespace mdk
