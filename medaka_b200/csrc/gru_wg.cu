// Tensor-core (wgmma) implementation of the GRU gate matmuls for sm_90a  (MDK_PREC_TC).
//
// Reference arithmetic: torch.nn.GRU as used by medaka/architectures/gru.py:46-52,66; parity target is
// the fp32 CPU path (medaka/prediction.py:146-148).  To stay inside 1e-3 (scale-aware) of fp32 through a
// 10 000-step recurrence, every operand is carried as an fp16 pair (hi + lo, ~22 significant bits) and each
// product is three fp16 MMAs, hi*hi + hi*lo + lo*hi, accumulated in fp32.
// MDK_PREC_FP16 (medaka's own GPU arithmetic, the model in half precision): rec_fp16_kernel and gemm_fp16_kernel, the
// FP16 = true forms of the same kernel bodies, take one product per contraction, hi*hi: operands rounded to the nearest
// fp16, fp32 accumulation.  The gate math, biases, h state and head stay fp32 as on the default path.
//
// Both kernels use the TRANSPOSED formulation  G^T[gate rows, N] = W[gate rows, K] . X^T[K, N]:
//   A operand = weights (M = 64 gate rows per warpgroup, K-major = torch's native [out][in] layout)
//   B operand = activations (N windows or positions, K-major = row-major [n][k])
//   D (registers) = hidden unit j x window / position n
// so the thread that holds r_j of a window also holds z_j and n_j of it: the gate math needs no exchange.
//
// Shared-memory operand layout (K-major, no swizzle): [k-group = k/8][row][8 halfs]; a core matrix is 8 rows
// x 16 B = 128 contiguous bytes, LBO = k-group stride, SBO = 128 B (next 8 rows).
#include "common.cuh"
#include "ptx.cuh"
#include "rec_common.cuh"

namespace mdk {

// =====================================================================================================
// Recurrent kernel.  One CTA = NT tiles of 16 windows (N = 16 NT) of one direction, for the whole sequence.
// Two warpgroups; warpgroup g owns hidden units [64g, 64g + 64) of all three gates, so the h tile of a step is
// complete only when both have written their half: one __syncthreads per step, with the tile double buffered
// (step t reads buffer t & 1 and writes the other).
// W_hh hi stays in REGISTERS for the whole sequence (the A operand of the register form of wgmma: 96 registers per
// thread), W_hh lo is a shared-memory A operand, so per step shared memory feeds only one of the three weight planes.
// The pre-activations of the next step are loaded straight into the accumulators (r, z) while the step ends; the
// n gate needs W_in.x and W_hn.h apart, so its input part sits in registers of its own.
// Products per (gate, k-step):
//   NT = 1: the h tile holds hi and lo as ONE operand of 32 rows (rows 0-15 h_hi of the 16 windows, 16-31 their h_lo).
//           One RS m64n32k16 gives W_hi.h_hi in accumulator columns 0-15 and W_hi.h_lo in columns 16-31, one SS
//           m64n16k16 adds W_lo.h_hi (the same descriptor at N = 16 reads rows 0-15) into columns 0-15 (d[0..7]); the
//           pre-activation is d[k] + d[k + 8].  48 MMAs per warpgroup-step instead of 72.
//   NT = 2: hi and lo planes of N = 32 rows each and three m64n32k16 MMAs (no registers left for accumulators twice as
//           wide: 241-253 of 255).
// At both tile counts r and z share one reciprocal (5 MUFU operations per value instead of 6), and the new h goes into
// the tile as fp16 hi / lo pairs by stmatrix (.trans: the accumulator fragment transposed is the K-major tile's layout).
// FP16 (rec_fp16_kernel): one product, W_hi.h_hi (and W_x,hi.x_hi); W_hh lo and W_x lo are not staged.  The h tile keeps
// its hi and lo halves (lo rounded toward zero, split_f16x2_rz, so that h0 read back at ~22 bits rounds to the hi the
// products used), and h0 leaves layer 0 at that precision as on the default path; at NT = 1 the RS MMA runs at N = 16 and
// reads only the hi rows, at NT = 2 only the hi plane.  24 RS MMAs per warpgroup-step at either tile count.
// FUSE_X (layer 0, F <= 16): the input projection W_ih . x_t is the same products per gate on an x tile laid out like
// the h tile (K = 16), so layer 0 needs no gi buffer.  OUT: fp16 hi/lo operand tiles of the projection GEMM (layer 0:
// copied under the next step's MMAs from the h tile buffer, which already holds them in that layout, see store_h0),
// fp32 rows, or (layer 1) partial logits: the 5-row linear head in fp32 on the CUDA cores, from the h values the threads
// already hold, while the next step's MMAs run (see head_partials).
// =====================================================================================================
constexpr int RW_THREADS = 256;
constexpr int RW_ABLK = (H / 8) * 64 * 16;          // W_hh lo of one (gate, warpgroup): [kg 16][row 64][8] = 16 KiB
constexpr int RW_XBLK = 2 * 64 * 16;                // W_ih lo (K = 16) of one (gate, warpgroup): 2 KiB

template <int NT, bool FUSE_X, int OUT, bool FP16 = false>
struct RwCfg {
    static constexpr int N = NT * RT_N;
    static constexpr bool HL = NT == 1;             // hi and lo in one operand of 2N rows (see the kernel's header)
    static constexpr int ROWS = HL ? 2 * N : N;     // rows of an activation operand
    static constexpr int PLANES = HL ? 1 : 2;       // operands per tile buffer
    static constexpr int KG = ROWS * 16 + 16;       // k-group stride of an activation tile (+16 B spreads the 2-byte
                                                    // x stores of one k-group over the banks; 16-B rows for stmatrix)
    static_assert(KG % 16 == 0, "stmatrix rows are 16-byte aligned");
    static constexpr int HPLANE = (H / 8) * KG;
    static constexpr int XPLANE = 2 * KG;
    static constexpr int HLO = HL ? N * 16 : HPLANE;   // bytes from an h value's hi half to its lo half
    static constexpr int XLO = HL ? N * 16 : XPLANE;   // the same in the x tile
    static constexpr int RED = (RW_THREADS / 32) * NCLS * N;                     // head partials of one step (floats)
    static constexpr int wlo_off = 0;                                            // [gate 3][wg 2] RW_ABLK
    static constexpr int wxlo_off = wlo_off + (FP16 ? 0 : 6 * RW_ABLK);          // [gate 3][wg 2] RW_XBLK
    static constexpr int h_off = wxlo_off + (FUSE_X && !FP16 ? 6 * RW_XBLK : 0); // [buf 2][plane PLANES] HPLANE
    static constexpr int x_off = h_off + 2 * PLANES * HPLANE;                    // [buf 2][plane PLANES] XPLANE
    static constexpr int red_off = x_off + (FUSE_X ? 2 * PLANES * XPLANE : 0);   // [buf 2][warp 8][class 5][N] fp32
    static constexpr int total = red_off + (OUT == OUT_LOGITS ? 2 * RED * 4 : 0);
    static_assert(total <= 227 * 1024, "smem budget");
};

__device__ __forceinline__ uint32_t ld_u32(const __half *p) { return *reinterpret_cast<const uint32_t *>(p); }

template <int NT, bool FUSE_X, int OUT, bool FP16>
__device__ __forceinline__ void rec_body(const float *__restrict__ gi, RecX xin, const __half *__restrict__ w_hh,
                                         const float *__restrict__ b_hn, void *__restrict__ h_out, int64_t B, int64_t T,
                                         const float *__restrict__ lin_w, float *__restrict__ plog) {
    using L = RwCfg<NT, FUSE_X, OUT, FP16>;
    constexpr int N = L::N, NA = N / 2;             // values per thread and gate (hidden unit x window)
    constexpr bool HL2 = L::HL && !FP16;            // the accumulators hold the W_hi.h_lo columns too
    constexpr int NACC = HL2 ? L::ROWS / 2 : NA;    // accumulator registers per gate (HL: NA more for the W_hi.h_lo columns)
    constexpr int NX = FUSE_X ? NACC : NA;          // axn: an accumulator only when the x projection is fused
    using MMA = Wgmma<N>;                           // SS: W_lo . h_hi (x_hi); FP16: RS W_hi . h_hi (x_hi)
    using MMA_H = Wgmma<L::ROWS>;                   // RS: W_hi . the whole h (x) operand
    constexpr bool LOGITS = OUT == OUT_LOGITS;
    extern __shared__ __align__(128) uint8_t smem[];
    const int tid = threadIdx.x, wg = tid >> 7, warp = (tid >> 5) & 3, lane = tid & 31;
    const int gq = lane >> 2, cq = lane & 3;
    const int dir = blockIdx.y;
    const int64_t ntiles = (B + RT_N - 1) / RT_N;
    const int64_t wtile0 = (int64_t)blockIdx.x * NT;
    const int j0 = wg * 64 + warp * 16 + gq;        // this thread's hidden units: j0 and j0 + 8
    const uint32_t sbase = smem_u32(smem);

    // ---- prologue: zero the activation tiles, weights into shared memory and registers ----
    for (int i = tid; i < (L::total - L::h_off) / 16; i += RW_THREADS)
        reinterpret_cast<int4 *>(smem + L::h_off)[i] = make_int4(0, 0, 0, 0);
    for (int i = tid; i < (FP16 ? 0 : 3 * H * (H / 8)); i += RW_THREADS) {
        const int kg = i & 15, r = (i >> 4) & (H - 1), gate = i >> 11;
        const uint4 v = *reinterpret_cast<const uint4 *>(w_hh + ((((size_t)dir * 2 + 1) * 3 + gate) * H + r) * H + kg * 8);
        *reinterpret_cast<uint4 *>(smem + L::wlo_off + (gate * 2 + (r >> 6)) * RW_ABLK + kg * 1024 + (r & 63) * 16) = v;
    }
    if (FUSE_X && !FP16) {
        for (int i = tid; i < 3 * H * 2; i += RW_THREADS) {
            const int kg = i & 1, r = (i >> 1) & (H - 1), gate = i >> 8;
            const uint4 v = *reinterpret_cast<const uint4 *>(xin.w_x + ((((size_t)dir * 2 + 1) * 3 + gate) * H + r) * 16 + kg * 8);
            *reinterpret_cast<uint4 *>(smem + L::wxlo_off + (gate * 2 + (r >> 6)) * RW_XBLK + kg * 1024 + (r & 63) * 16) = v;
        }
    }
    float wlin[2][NCLS];                            // LOGITS: W_lin[c][dir * H + j0 + 8 hb], fp32
    if (LOGITS) {
#pragma unroll
        for (int hb = 0; hb < 2; ++hb)
#pragma unroll
            for (int c = 0; c < NCLS; ++c) wlin[hb][c] = lin_w[c * H2 + dir * H + j0 + 8 * hb];
    }
    uint32_t whi[3][H / 16][4];
#pragma unroll
    for (int gate = 0; gate < 3; ++gate)
#pragma unroll
        for (int ks = 0; ks < H / 16; ++ks) {
            const __half *w = w_hh + ((((size_t)dir * 2) * 3 + gate) * H + j0) * H + ks * 16 + 2 * cq;
            whi[gate][ks][0] = ld_u32(w);
            whi[gate][ks][1] = ld_u32(w + 8 * H);
            whi[gate][ks][2] = ld_u32(w + 8);
            whi[gate][ks][3] = ld_u32(w + 8 * H + 8);
        }
    uint32_t wxhi[3][4];
    float bx[3][2] = {};                            // FUSE_X: folded biases of r, z and the input part of n
    if (FUSE_X) {
#pragma unroll
        for (int gate = 0; gate < 3; ++gate) {
            const __half *w = xin.w_x + ((((size_t)dir * 2) * 3 + gate) * H + j0) * 16 + 2 * cq;
            wxhi[gate][0] = ld_u32(w);
            wxhi[gate][1] = ld_u32(w + 8 * 16);
            wxhi[gate][2] = ld_u32(w + 8);
            wxhi[gate][3] = ld_u32(w + 8 * 16 + 8);
            bx[gate][0] = xin.bias[dir * G3 + gate * H + j0];
            bx[gate][1] = xin.bias[dir * G3 + gate * H + j0 + 8];
        }
    }
    const float bhn[2] = {b_hn[dir * H + j0], b_hn[dir * H + j0 + 8]};
    // the h tile row this lane addresses in the step's stmatrix: row c = lane & 7 of matrix m = lane >> 3 (plane m / 2,
    // hidden units of hb = m & 1) of window block 0, in tile buffer 0
    const uint32_t hst_addr = sbase + L::h_off + (lane >> 4) * L::HLO + (wg * 8 + warp * 2 + ((lane >> 3) & 1)) * L::KG +
                              (lane & 7) * 16;

    // Accumulator element k = 4i + 2hb + e: hidden unit j0 + 8hb, window n = 8i + 2cq + e of tile wtile0 + i/2
    // (HL: k >= NA is the lo part of window n - 16, element k - NA).
    float ar[NACC], az[NACC], an[NACC], axn[NX], hp[NA];
#pragma unroll
    for (int k = 0; k < NA; ++k) hp[k] = 0.f;
    // pre-activations of time t into the accumulators (gi in quad layout, common.cuh: the pair e = 0, 1 is contiguous).
    // gi_thr: this thread's first element (tile wtile0, t = 0, its window quad and hidden unit j0); the rest of an address
    // is t and compile-time offsets.
    const float *gi_thr = FUSE_X ? nullptr
                                 : gi + wtile0 * T * GI_TS_FLOATS + ((dir * 3 * 4 + (cq >> 1)) * H + j0) * 4 + 2 * (cq & 1);
    auto load_pre = [&](int64_t t) {
#pragma unroll
        for (int i = 0; i < N / 8; ++i)
#pragma unroll
            for (int hb = 0; hb < 2; ++hb) {
                float2 v[3] = {make_float2(0.f, 0.f), make_float2(0.f, 0.f), make_float2(0.f, 0.f)};
                if (FUSE_X) {
#pragma unroll
                    for (int gate = 0; gate < 3; ++gate) v[gate] = make_float2(bx[gate][hb], bx[gate][hb]);
                } else if (i < 2 || wtile0 + (i >> 1) < ntiles) {     // (the grid has no CTA without a first tile)
                    const float *p = gi_thr + ((i >> 1) * T + t) * GI_TS_FLOATS + (2 * (i & 1) * H + 8 * hb) * 4;
#pragma unroll
                    for (int gate = 0; gate < 3; ++gate) v[gate] = __ldcs(reinterpret_cast<const float2 *>(p + gate * 16 * H));
                }
                const int k = 4 * i + 2 * hb;
                ar[k] = v[0].x; ar[k + 1] = v[0].y;
                az[k] = v[1].x; az[k + 1] = v[1].y;
                axn[k] = v[2].x; axn[k + 1] = v[2].y;
                an[k] = bhn[hb]; an[k + 1] = bhn[hb];
            }
        if constexpr (HL2) {
#pragma unroll
            for (int k = NA; k < NACC; ++k) {
                ar[k] = 0.f; az[k] = 0.f; an[k] = 0.f;
                if constexpr (FUSE_X) axn[k] = 0.f;
            }
        }
    };
    // FUSE_X: x_t staged as the B tile [plane][kg 2][row][8] (hi at row n, lo XLO bytes on); thread entry q = tid + 256 m
    // covers (window q / F, feature q % F)
    const int xF = FUSE_X ? xin.F : 1;
    const float *xsrc[NT];
    int xoff[NT];
    float xreg[NT];
#pragma unroll
    for (int m = 0; m < NT; ++m) {
        const int q = tid + RW_THREADS * m, xn = q / xF, xf = q - xn * xF;
        const bool own = FUSE_X && q < N * xF;
        xoff[m] = own ? (xf >> 3) * L::KG + xn * 16 + (xf & 7) * 2 : -1;
        xsrc[m] = (own && wtile0 * RT_N + xn < B) ? xin.feats + ((wtile0 * RT_N + xn) * T) * xF + xf : nullptr;
        xreg[m] = 0.f;
    }
    auto stage_x = [&](int buf, int m, float v) {
        __half hi, lo;
        split_f16(v, hi, lo);
        *reinterpret_cast<__half *>(smem + L::x_off + buf * L::PLANES * L::XPLANE + xoff[m]) = hi;
        if (!FP16) *reinterpret_cast<__half *>(smem + L::x_off + buf * L::PLANES * L::XPLANE + L::XLO + xoff[m]) = lo;
    };
    const int64_t t_first = dir ? T - 1 : 0;
    if (FUSE_X) {
#pragma unroll
        for (int m = 0; m < NT; ++m) {
            if (xoff[m] < 0) continue;
            stage_x(0, m, xsrc[m] ? xsrc[m][t_first * xF] : 0.f);
        }
    }
    load_pre(t_first);
    fence_proxy_async_smem();   // generic-proxy writes above (weights, zeroed tiles, x_0) -> visible to wgmma reads
    __syncthreads();            // h_{-1} = 0, x_0 and the weights are in shared memory

    // ---- fused linear head (LOGITS), fp32 on the CUDA cores ----
    // head_partials(rb): this direction's logits of the h in hp, summed over the thread's 2 hidden units, then over the 8
    // gq lanes of its cq group (shuffles), into red[rb][warp][class][n].  A thread holds NW = N / 4 windows, wl = 2i + e
    // (window n = 8i + 2cq + e); while more than one is left, each shuffle level hands half of them to the partner lane
    // and keeps the sums of the other half (a reduce-scatter: 5 NW / 2 + 5 NW / 4 + ... shuffles instead of 15 NW);
    // below one window the level is an all-reduce.  Every window's sum runs through the same tree over gq and the same
    // warp order in head_store, whatever its slot in the tile or NT.
    constexpr int NW = N / 4;
    auto head_partials = [&](int rb) {
        float v[NW][NCLS];
#pragma unroll
        for (int wl = 0; wl < NW; ++wl) {
            const int k = 4 * (wl >> 1) + (wl & 1);             // hidden unit j0 at k, j0 + 8 at k + 2
#pragma unroll
            for (int c = 0; c < NCLS; ++c) v[wl][c] = fmaf(wlin[1][c], hp[k + 2], wlin[0][c] * hp[k]);
        }
        int wbase = 0;                                          // window of v[0]
#pragma unroll
        for (int lvl = 0; lvl < 3; ++lvl) {
            const int mask = 16 >> lvl;                         // lane bit of gq bit 2 - lvl
            const int half = (NW >> lvl) / 2;
            if (half > 0) {
                const bool up = lane & mask;
#pragma unroll
                for (int w = 0; w < NW / 2; ++w) {      // (a constant trip count, so that v stays in registers)
                    if (w >= half) continue;
#pragma unroll
                    for (int c = 0; c < NCLS; ++c) {
                        const float send = up ? v[w][c] : v[w + half][c];
                        const float keep = up ? v[w + half][c] : v[w][c];
                        v[w][c] = keep + __shfl_xor_sync(0xffffffffu, send, mask);
                    }
                }
                if (up) wbase += half;
            } else {
#pragma unroll
                for (int c = 0; c < NCLS; ++c) v[0][c] += __shfl_xor_sync(0xffffffffu, v[0][c], mask);
            }
        }
        if (NW >= 8 || !(lane & 4)) {                           // NW = 4: the lanes of a gq pair hold the same sums
            float *red = reinterpret_cast<float *>(smem + L::red_off) + rb * L::RED + (tid >> 5) * NCLS * N;
            const int n = 8 * (wbase >> 1) + 2 * cq + (wbase & 1);
#pragma unroll
            for (int c = 0; c < NCLS; ++c) red[c * N + n] = v[0][c];
        }
    };
    // head_store(rb, t): the 8 warps' partials of red[rb] (published by a __syncthreads), summed in warp order -> plog row t
    auto head_store = [&](int rb, int64_t t) {
        if (tid >= NCLS * N) return;
        const int c = tid / N, n = tid % N;
        const float *red = reinterpret_cast<const float *>(smem + L::red_off) + rb * L::RED + c * N + n;
        float s = red[0];
#pragma unroll
        for (int w = 1; w < RW_THREADS / 32; ++w) s += red[w * NCLS * N];
        const int64_t wt = wtile0 + n / RT_N;
        if (wt < ntiles) plog[((dir * ntiles + wt) * T + t) * PLOG_TS_FLOATS + c * RT_N + (n & 15)] = s;
    };
    // store_h0(b, t) (OUT_TILES): h_t from tile buffer b to the projection GEMM's operand tiles.  The 16 rows of one
    // (window tile m, plane p, k-group kg) are 256 contiguous bytes in the buffer and in the operand tile (rows
    // (wt T + t) 16 .. + 15 of a 128-row tile), so the CTA copies them as they are, one 16-byte row per thread and
    // vector: vector q = tid + 256 r is row q & 15 of piece q >> 4 = (m * 2 + p) * 16 + kg.  Padding windows of a ragged
    // tile go out too (never read back); tiles >= ntiles do not.
    auto store_h0 = [&](int b, int64_t t) {
#pragma unroll
        for (int r = 0; r < NT * 512 / RW_THREADS; ++r) {
            const int q = tid + RW_THREADS * r, row = q & 15, kg = (q >> 4) & 15, p = (q >> 8) & 1, m = q >> 9;
            const int64_t wt = wtile0 + m;
            if (wt >= ntiles) continue;
            const int64_t orow = (wt * T + t) * RT_N + row;
            const int4 v = *reinterpret_cast<const int4 *>(smem + L::h_off + b * L::PLANES * L::HPLANE + p * L::HLO + kg * L::KG +
                                                           (m * RT_N + row) * 16);
            *reinterpret_cast<int4 *>(reinterpret_cast<uint8_t *>(h_out) + (orow >> 7) * (int64_t)XT_TILE_BYTES +
                                      p * XT_PLANE_BYTES + (dir * (H / 8) + kg) * (XT_ROWS * 16) + (orow & (XT_ROWS - 1)) * 16) = v;
        }
    };

#pragma unroll 1
    for (int64_t step = 0; step < T; ++step) {
        const int64_t t = dir ? T - 1 - step : step;
        const int buf = (int)(step & 1);
        const uint32_t hb_addr = sbase + L::h_off + buf * L::PLANES * L::HPLANE;
        wg_fence();
        // k-step outer, gate inner: consecutive MMAs go to different accumulators, so none waits for the one before it
        // (each accumulator still sums its products in the order k-step, then hi.hi, hi.lo, lo.hi)
        if constexpr (FP16) {
#pragma unroll
            for (int ks = 0; ks < H / 16; ++ks) {
                const uint64_t bh = make_smem_desc(hb_addr + ks * 2 * L::KG, L::KG, 128);
#pragma unroll
                for (int gate = 0; gate < 3; ++gate) MMA::rs(gate == 0 ? ar : (gate == 1 ? az : an), whi[gate][ks], bh, 1u);
            }
        } else if constexpr (L::HL) {
#pragma unroll
            for (int ks = 0; ks < H / 16; ++ks) {
                const uint64_t bh = make_smem_desc(hb_addr + ks * 2 * L::KG, L::KG, 128);
#pragma unroll
                for (int gate = 0; gate < 3; ++gate) MMA_H::rs(gate == 0 ? ar : (gate == 1 ? az : an), whi[gate][ks], bh, 1u);
#pragma unroll
                for (int gate = 0; gate < 3; ++gate)
                    MMA::ss(gate == 0 ? ar : (gate == 1 ? az : an),
                            make_smem_desc(sbase + L::wlo_off + (gate * 2 + wg) * RW_ABLK + ks * 2 * 1024, 1024, 128), bh, 1u);
            }
        } else {
#pragma unroll
            for (int ks = 0; ks < H / 16; ++ks) {
                const uint64_t bh = make_smem_desc(hb_addr + ks * 2 * L::KG, L::KG, 128);
                const uint64_t bl = make_smem_desc(hb_addr + L::HPLANE + ks * 2 * L::KG, L::KG, 128);
#pragma unroll
                for (int gate = 0; gate < 3; ++gate) MMA::rs(gate == 0 ? ar : (gate == 1 ? az : an), whi[gate][ks], bh, 1u);
#pragma unroll
                for (int gate = 0; gate < 3; ++gate) MMA::rs(gate == 0 ? ar : (gate == 1 ? az : an), whi[gate][ks], bl, 1u);
#pragma unroll
                for (int gate = 0; gate < 3; ++gate)
                    MMA::ss(gate == 0 ? ar : (gate == 1 ? az : an),
                            make_smem_desc(sbase + L::wlo_off + (gate * 2 + wg) * RW_ABLK + ks * 2 * 1024, 1024, 128), bh, 1u);
            }
        }
        if constexpr (FUSE_X) {
            const uint32_t xa = sbase + L::x_off + buf * L::PLANES * L::XPLANE;
            const uint64_t bh = make_smem_desc(xa, L::KG, 128);
            if constexpr (FP16) {
#pragma unroll
                for (int gate = 0; gate < 3; ++gate) MMA::rs(gate == 0 ? ar : (gate == 1 ? az : axn), wxhi[gate], bh, 1u);
            } else if constexpr (L::HL) {
#pragma unroll
                for (int gate = 0; gate < 3; ++gate) MMA_H::rs(gate == 0 ? ar : (gate == 1 ? az : axn), wxhi[gate], bh, 1u);
#pragma unroll
                for (int gate = 0; gate < 3; ++gate)
                    MMA::ss(gate == 0 ? ar : (gate == 1 ? az : axn),
                            make_smem_desc(sbase + L::wxlo_off + (gate * 2 + wg) * RW_XBLK, 1024, 128), bh, 1u);
            } else {
                const uint64_t bl = make_smem_desc(xa + L::XPLANE, L::KG, 128);
#pragma unroll
                for (int gate = 0; gate < 3; ++gate) MMA::rs(gate == 0 ? ar : (gate == 1 ? az : axn), wxhi[gate], bh, 1u);
#pragma unroll
                for (int gate = 0; gate < 3; ++gate) MMA::rs(gate == 0 ? ar : (gate == 1 ? az : axn), wxhi[gate], bl, 1u);
#pragma unroll
                for (int gate = 0; gate < 3; ++gate)
                    MMA::ss(gate == 0 ? ar : (gate == 1 ? az : axn),
                            make_smem_desc(sbase + L::wxlo_off + (gate * 2 + wg) * RW_XBLK, 1024, 128), bh, 1u);
            }
        }
        wg_commit();
        // FUSE_X: the next step's features load under the MMAs, so that their latency is not paid after the wait (the
        // fence before the barrier waits for outstanding loads)
        if (FUSE_X && step + 1 < T) {
#pragma unroll
            for (int m = 0; m < NT; ++m)
                if (xsrc[m]) xreg[m] = xsrc[m][(dir ? t - 1 : t + 1) * xF];
        }
        // h of the previous step (published by the last barrier, and read by these MMAs) goes out to the h0 tiles; the
        // buffer is rewritten only after the next barrier
        if (OUT == OUT_TILES && step > 0) store_h0(buf, dir ? t + 1 : t - 1);
        // the L2 prefetch of gi three steps ahead runs under the MMAs too
        if (!FUSE_X && tid == 0 && step + GI_PREFETCH_STEPS < T) {
            const int64_t tp = dir ? t - GI_PREFETCH_STEPS : t + GI_PREFETCH_STEPS;
#pragma unroll
            for (int m = 0; m < NT; ++m) {
                if (wtile0 + m >= ntiles) break;
                const float *blk = gi + ((wtile0 + m) * T + tp) * GI_TS_FLOATS + (int64_t)dir * (GI_TS_FLOATS / 2);
#pragma unroll
                for (int i = 0; i < 12; ++i) bulk_prefetch_l2(blk + i * 512, 2048);
            }
        }
        // the head runs under the MMAs too: hp still holds h of the previous step (zeros at step 0: nothing to do); the
        // sums of the step before that, published by the last barrier, go out to plog
        if (LOGITS && step > 0) {
            if (step > 1) head_store((int)((step - 1) & 1), dir ? t + 2 : t - 2);
            head_partials((int)(step & 1));
        }
        wg_wait_all();
        wg_hold(ar); wg_hold(az); wg_hold(an); wg_hold(axn);

        // ---- gate math (weights and biases carry the exp2 scale factors, common.cuh gate_scale) ----
#pragma unroll
        for (int k = 0; k < NA; ++k) {
            float pr = ar[k], pz = az[k], pn = an[k], px = axn[k];
            if constexpr (HL2) {
                pr += ar[k + NA]; pz += az[k + NA]; pn += an[k + NA];
                if constexpr (FUSE_X) px += axn[k + NA];
            }
            // one reciprocal for r and z: r = 1 / a = b / (a b), z = 1 / b = a / (a b); a, b <= 1 + 2^EXP_CLAMP, so the
            // product stays finite
            const float a = 1.f + ex2_approx(fminf(pr, EXP_CLAMP)), b = 1.f + ex2_approx(fminf(pz, EXP_CLAMP));
            const float q = rcp_approx(a * b);
            const float r = b * q, z = a * q;
            const float en = ex2_approx(fminf(fmaf(r, pn, px), EXP_CLAMP));
            const float n = (en - 1.f) * rcp_approx(en + 1.f);
            hp[k] = fmaf(z, hp[k] - n, n);
        }
        // h as fp16 hi / lo into the other tile buffer, one stmatrix per 8 windows: the accumulator block (i, hb) is an
        // 8 x 8 fragment (hidden units j0 - gq + 8 hb + 0..7 x windows 8i + 0..7), and transposed, its row c is the
        // 16-byte row [k-group (j0 + 8 hb) / 8][window 8i + c] of the tile.  Matrices: hi hb 0, hi hb 1, lo hb 0, lo hb 1.
#pragma unroll
        for (int i = 0; i < N / 8; ++i) {
            uint32_t hi[2], lo[2];
#pragma unroll
            for (int hb = 0; hb < 2; ++hb) {
                if constexpr (FP16) split_f16x2_rz(hp[4 * i + 2 * hb], hp[4 * i + 2 * hb + 1], hi[hb], lo[hb]);
                else split_f16x2(hp[4 * i + 2 * hb], hp[4 * i + 2 * hb + 1], hi[hb], lo[hb]);
            }
            stmatrix_x4_trans(hst_addr + (buf ^ 1) * L::PLANES * L::HPLANE + i * 128, hi[0], hi[1], lo[0], lo[1]);
        }
        if (FUSE_X && step + 1 < T) {
#pragma unroll
            for (int m = 0; m < NT; ++m) {
                if (xoff[m] < 0) continue;
                stage_x(buf ^ 1, m, xreg[m]);
            }
        }
        // ---- outputs of this step (OUT_TILES: by store_h0, from the tile buffer) ----
        if (OUT == OUT_ROWS) {
#pragma unroll
            for (int k = 0; k < NA; ++k) {
                const int i = k >> 2, n = 8 * i + 2 * cq + (k & 1);
                const int64_t wt = wtile0 + (i >> 1);
                if (wt >= ntiles) continue;
                const int64_t orow = (wt * T + t) * RT_N + (n & 15);
                reinterpret_cast<float *>(h_out)[orow * H2 + dir * H + j0 + 8 * ((k >> 1) & 1)] = hp[k];
            }
        }
        // (FUSE_X: biases, no loads; unconditional, so that the compiler moves them next to the MMAs that read them)
        if (FUSE_X || step + 1 < T) load_pre(dir ? t - 1 : t + 1);
        fence_proxy_async_smem();     // h / x tile writes -> visible to the next step's wgmma operand reads
        __syncthreads();
    }
    if (OUT == OUT_TILES) store_h0((int)(T & 1), dir ? 0 : T - 1);     // the last step's h
    if (LOGITS) {                     // the last two steps' logits: step T - 2 (partials in red), step T - 1 (in hp)
        if (T > 1) head_store((int)((T - 1) & 1), dir ? 1 : T - 2);
        head_partials((int)(T & 1));
        __syncthreads();
        head_store((int)(T & 1), dir ? 0 : T - 1);
    }
}

template <int NT, bool FUSE_X, int OUT>
__global__ void __launch_bounds__(RW_THREADS, 1)
rec_tc_kernel(const float *__restrict__ gi, RecX xin, const __half *__restrict__ w_hh, const float *__restrict__ b_hn,
              void *__restrict__ h_out, int64_t B, int64_t T, const float *__restrict__ lin_w,
              float *__restrict__ plog) {
    rec_body<NT, FUSE_X, OUT, false>(gi, xin, w_hh, b_hn, h_out, B, T, lin_w, plog);
}
template <int NT, bool FUSE_X, int OUT>
__global__ void __launch_bounds__(RW_THREADS, 1)
rec_fp16_kernel(const float *__restrict__ gi, RecX xin, const __half *__restrict__ w_hh, const float *__restrict__ b_hn,
                void *__restrict__ h_out, int64_t B, int64_t T, const float *__restrict__ lin_w,
                float *__restrict__ plog) {
    rec_body<NT, FUSE_X, OUT, true>(gi, xin, w_hh, b_hn, h_out, B, T, lin_w, plog);
}

template <int NT, bool FX, int OUT, bool FP16>
static cudaError_t launch_rec(const float *gi, const RecX &xin, const __half *w_hh_tm, const float *b_hn, void *out,
                              const float *lin_w, int64_t B, int64_t T, cudaStream_t s) {
    auto kern = FP16 ? rec_fp16_kernel<NT, FX, OUT> : rec_tc_kernel<NT, FX, OUT>;
    constexpr int smem_bytes = RwCfg<NT, FX, OUT, FP16>::total;
    // (the attribute is per device: set it on every launch, a process may drive several GPUs)
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes);
    if (e != cudaSuccess) return e;
    const int64_t tiles = (B + RT_N - 1) / RT_N;
    dim3 grid((unsigned)((tiles + NT - 1) / NT), NDIR);
    constexpr bool LOGITS = OUT == OUT_LOGITS;
    kern<<<grid, RW_THREADS, smem_bytes, s>>>(gi, xin, w_hh_tm, b_hn, LOGITS ? nullptr : out, B, T, lin_w,
                                              LOGITS ? static_cast<float *>(out) : nullptr);
    return cudaGetLastError();
}

template <int NT, bool FP16>
static cudaError_t launch_rec_nt(const float *gi, const RecX *xin, const __half *w_hh_tm, const float *b_hn, int out_kind,
                                 void *out, const float *lin_w, int64_t B, int64_t T, cudaStream_t s) {
    if (xin)    // the fused projection is layer 0, which feeds the GEMM
        return out_kind == OUT_TILES ? launch_rec<NT, true, OUT_TILES, FP16>(gi, *xin, w_hh_tm, b_hn, out, nullptr, B, T, s)
                                     : cudaErrorInvalidValue;
    const RecX none{nullptr, nullptr, nullptr, 0};
    switch (out_kind) {
    case OUT_TILES: return launch_rec<NT, false, OUT_TILES, FP16>(gi, none, w_hh_tm, b_hn, out, nullptr, B, T, s);
    case OUT_ROWS: return launch_rec<NT, false, OUT_ROWS, FP16>(gi, none, w_hh_tm, b_hn, out, nullptr, B, T, s);
    case OUT_LOGITS:
        return lin_w ? launch_rec<NT, false, OUT_LOGITS, FP16>(gi, none, w_hh_tm, b_hn, out, lin_w, B, T, s)
                     : cudaErrorInvalidValue;
    }
    return cudaErrorInvalidValue;
}

cudaError_t launch_rec_tc(const float *gi, const RecX *xin, const __half *w_hh_tm, const float *b_hn, int tiles_per_cta,
                          int out_kind, void *out, const float *lin_w, int64_t B, int64_t T, bool fp16, cudaStream_t s) {
    if (B == 0 || T == 0) return cudaSuccess;
    switch (tiles_per_cta * 2 + (fp16 ? 1 : 0)) {
    case 2: return launch_rec_nt<1, false>(gi, xin, w_hh_tm, b_hn, out_kind, out, lin_w, B, T, s);
    case 3: return launch_rec_nt<1, true>(gi, xin, w_hh_tm, b_hn, out_kind, out, lin_w, B, T, s);
    case 4: return launch_rec_nt<2, false>(gi, xin, w_hh_tm, b_hn, out_kind, out, lin_w, B, T, s);
    case 5: return launch_rec_nt<2, true>(gi, xin, w_hh_tm, b_hn, out_kind, out, lin_w, B, T, s);
    }
    return cudaErrorInvalidValue;
}

// =====================================================================================================
// Layer-1 input projection on tensor cores:  gi[p][blk*128 + j] = sum_k W_ih[blk*128 + j][k] * x[p][k] + bias
// Persistent: grid = 6 weight blocks x CT CTAs; the six CTAs of one tile index walk the same tiles, so an activation
// tile comes from HBM once and from L2 for the other five.  Warpgroup wg owns gate rows [64wg, 64wg + 64) of the CTA's
// block and keeps their W hi and lo A fragments in REGISTERS for the whole kernel (the register form of wgmma: 2 planes
// x 16 k-steps x 4 = 128 registers), so shared memory feeds only the activation operand.
// 128-position activation tiles (written by the layer-0 recurrent kernel directly in operand layout) stream through a
// ring of GW_NQ stages, one 64-wide K slice (hi + lo) each: slice q of every tile goes to stage q.  Thread 0 fills a
// stage with bulk async copies behind its full mbarrier and refills it once all 8 warps have arrived on its empty
// mbarrier.  A warp arrives when wgmma.wait_group 1 shows the group that read the stage complete, so one group of MMAs
// stays in flight across slices and the next tile's slices load under this tile's MMAs.
// At the end of a tile the accumulators (+ bias) go to a staging buffer laid out as gi's quad layout, and warp 0 writes
// it out with one bulk store per lane (one window quad of one tile-step, 2 KiB contiguous in gi) while the next tile's
// MMAs run.
// Per element the sum runs in the order slice q, product (hi.hi, hi.lo, lo.hi), k-step.
// FP16 (gemm_fp16_kernel): one product, W_in,hi . h0_hi: only the W hi fragments go to registers and the ring brings only
// the hi plane of each slice (the h0 tiles keep both planes, read_activation(0) unpacks them).
// =====================================================================================================
constexpr int GW_THREADS = 256;
constexpr int GW_QK = 8;                                        // k-groups per stage (K = 64)
constexpr int GW_STAGE_PLANE = GW_QK * XT_ROWS * 16;            // 16 KiB
constexpr int GW_STAGE = 2 * GW_STAGE_PLANE;                    // hi + lo
constexpr int GW_NQ = XT_K / 8 / GW_QK;                         // slices per tile = stages of the ring
constexpr int GW_KS = XT_K / 16;                                // k-steps per tile
constexpr int GW_TS = XT_ROWS / WT;                             // gi tile-steps per tile
constexpr int GW_QUAD = H * 4;                                  // floats of one (tile-step, block, window quad) piece of gi
// staging: [tile-step 8][window quad 4] pieces, each padded by 16 floats so that the two window quads a warp's float2
// stores reach in one instruction fall in opposite halves of the banks
constexpr int GW_QUAD_PAD = GW_QUAD + 16;
constexpr int GW_OUT_OFF = GW_NQ * GW_STAGE;
constexpr int GW_BAR_OFF = GW_OUT_OFF + GW_TS * 4 * GW_QUAD_PAD * 4;    // full[GW_NQ], empty[GW_NQ]
constexpr int GW_SMEM = GW_BAR_OFF + 2 * GW_NQ * 8;
static_assert(GW_SMEM <= 227 * 1024, "smem budget");
static_assert(GW_TS * 4 == 32, "one bulk store per lane of warp 0");

template <bool FP16>
__device__ __forceinline__ void gemm_body(const uint8_t *__restrict__ x_tiles, const __half *__restrict__ w_in_tm,
                                          const float *__restrict__ bias, float *__restrict__ gi, int64_t P,
                                          int64_t ntiles) {
    constexpr int WPLANES = FP16 ? 1 : 2, NPROD = FP16 ? 1 : 3;
    extern __shared__ __align__(128) uint8_t smem[];
    uint64_t *full = reinterpret_cast<uint64_t *>(smem + GW_BAR_OFF), *empty = full + GW_NQ;
    float *stg = reinterpret_cast<float *>(smem + GW_OUT_OFF);
    const int tid = threadIdx.x, wg = tid >> 7, warp = (tid >> 5) & 3, lane = tid & 31;
    const int gq = lane >> 2, cq = lane & 3;
    const int blk = blockIdx.x;                 // weight block: dir*3 + gate
    const int j0 = wg * 64 + warp * 16 + gq;    // this thread's gate rows: j0 and j0 + 8
    const uint32_t sbase = smem_u32(smem);
    const int64_t my_tiles = blockIdx.y < ntiles ? (ntiles - 1 - blockIdx.y) / gridDim.y + 1 : 0;
    auto issue = [&](int64_t n, int q) {        // slice q of this CTA's n-th tile -> stage q
        const uint8_t *src = x_tiles + (blockIdx.y + n * gridDim.y) * (int64_t)XT_TILE_BYTES + q * GW_STAGE_PLANE;
        mbar_arrive_expect_tx(&full[q], WPLANES * GW_STAGE_PLANE);
        bulk_g2s(smem + q * GW_STAGE, src, GW_STAGE_PLANE, &full[q]);
        if (!FP16) bulk_g2s(smem + q * GW_STAGE + GW_STAGE_PLANE, src + XT_PLANE_BYTES, GW_STAGE_PLANE, &full[q]);
    };
    if (tid == 0) {
        for (int q = 0; q < GW_NQ; ++q) {
            mbar_init(&full[q], 1);
            mbar_init(&empty[q], GW_THREADS / 32);
        }
        fence_mbar_init();
        if (my_tiles > 0)
            for (int q = 0; q < GW_NQ; ++q) issue(0, q);
    }
    // W (row-major fp16 [blk][plane][row j][k 256]) hi and lo A fragments of rows j0, j0 + 8 (layout: ptx.cuh Wgmma)
    uint32_t wa[WPLANES][GW_KS][4];
#pragma unroll
    for (int p = 0; p < WPLANES; ++p)
#pragma unroll
        for (int ks = 0; ks < GW_KS; ++ks) {
            const __half *w = w_in_tm + (((size_t)blk * 2 + p) * H + j0) * H2 + ks * 16 + 2 * cq;
            wa[p][ks][0] = ld_u32(w);
            wa[p][ks][1] = ld_u32(w + 8 * H2);
            wa[p][ks][2] = ld_u32(w + 8);
            wa[p][ks][3] = ld_u32(w + 8 * H2 + 8);
        }
    const float bj[2] = {bias[blk * H + j0], bias[blk * H + j0 + 8]};
    const uint64_t policy = l2_evict_first_policy();
    __syncthreads();                            // the mbarriers are initialised
    // stage q has been read by this warp's MMAs of tile n: release it, and thread 0 refills it with tile n + 1
    auto release = [&](int64_t n, int q) {
        if (lane == 0) mbar_arrive(&empty[q]);
        if (tid == 0 && n + 1 < my_tiles) {
            mbar_wait(&empty[q], (uint32_t)(n & 1));
            issue(n + 1, q);
        }
        __syncwarp();
    };
    float acc[64];
#pragma unroll 1
    for (int64_t n = 0; n < my_tiles; ++n) {
#pragma unroll
        for (int q = 0; q < GW_NQ; ++q) {
            mbar_wait(&full[q], (uint32_t)(n & 1));
            wg_fence();
#pragma unroll
            for (int prod = 0; prod < NPROD; ++prod) {
                const int pa = prod == 2, pb = prod == 1;   // W part hi, hi, lo ; x part hi, lo, hi
#pragma unroll
                for (int kk = 0; kk < GW_QK / 2; ++kk) {
                    const uint64_t b = make_smem_desc(sbase + q * GW_STAGE + pb * GW_STAGE_PLANE + 2 * kk * (XT_ROWS * 16),
                                                      XT_ROWS * 16, 128);
                    Wgmma<128>::rs(acc, wa[pa][q * (GW_QK / 2) + kk], b, (q | prod | kk) ? 1u : 0u);
                }
            }
            wg_commit();
            if (q > 0) {
                wg_wait_1();
                release(n, q - 1);
            }
        }
        wg_wait_all();
        wg_hold(acc);
        release(n, GW_NQ - 1);

        // ---- epilogue: accumulators + bias -> staging (quad layout) -> bulk stores under the next tile's MMAs ----
        const int64_t tile = blockIdx.y + n * gridDim.y;
        const int64_t prem = P - tile * XT_ROWS;    // rows of this tile that exist (a multiple of 16)
        if (tid < 32) bulk_wait_read_all();         // the previous tile's stores have read the staging buffer
        __syncthreads();
#pragma unroll
        for (int k = 0; k < 64; k += 2) {
            // position c = 8i + 2cq + e of the tile: tile-step i / 2, window quad 2 (i & 1) + cq / 2, w4 = 2 (cq & 1) + e
            const int i = k >> 2, hb = (k >> 1) & 1;
            float *o = stg + ((i >> 1) * 4 + 2 * (i & 1) + (cq >> 1)) * GW_QUAD_PAD + (j0 + 8 * hb) * 4 + 2 * (cq & 1);
            *reinterpret_cast<float2 *>(o) = make_float2(acc[k] + bj[hb], acc[k + 1] + bj[hb]);
        }
        fence_proxy_async_smem();                   // staging writes -> visible to the bulk copies
        __syncthreads();
        if (tid < 32) {
            const int ts = lane >> 2, cg = lane & 3;
            if (ts * WT < prem)
                bulk_s2g(gi + (((tile * GW_TS + ts) * 6 + blk) * 4 + cg) * GW_QUAD, stg + lane * GW_QUAD_PAD,
                         GW_QUAD * 4, policy);
            bulk_commit();
        }
    }
    if (tid < 32) bulk_wait_all();
}

__global__ void __launch_bounds__(GW_THREADS, 1)
gemm_tc_kernel(const uint8_t *__restrict__ x_tiles, const __half *__restrict__ w_in_tm, const float *__restrict__ bias,
               float *__restrict__ gi, int64_t P, int64_t ntiles) {
    gemm_body<false>(x_tiles, w_in_tm, bias, gi, P, ntiles);
}
__global__ void __launch_bounds__(GW_THREADS, 1)
gemm_fp16_kernel(const uint8_t *__restrict__ x_tiles, const __half *__restrict__ w_in_tm, const float *__restrict__ bias,
                 float *__restrict__ gi, int64_t P, int64_t ntiles) {
    gemm_body<true>(x_tiles, w_in_tm, bias, gi, P, ntiles);
}

cudaError_t launch_gemm_tc(const void *x_tiles, const __half *w_in_tm, const float *bias, float *gi, int64_t P,
                           int sm_count, bool fp16, cudaStream_t s) {
    if (P == 0) return cudaSuccess;
    const int64_t ntiles = (P + XT_ROWS - 1) / XT_ROWS;
    const auto kernel = fp16 ? gemm_fp16_kernel : gemm_tc_kernel;
    cudaError_t ea = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, GW_SMEM);
    if (ea != cudaSuccess) return ea;
    int64_t ct = sm_count / 6;
    if (ct < 1) ct = 1;
    if (ct > ntiles) ct = ntiles;
    dim3 grid(6, (unsigned)ct);
    kernel<<<grid, GW_THREADS, GW_SMEM, s>>>(reinterpret_cast<const uint8_t *>(x_tiles), w_in_tm, bias, gi, P, ntiles);
    return cudaGetLastError();
}

// =====================================================================================================
// Self test of the wgmma building block: D[128][N] = A[128][K] . B[N][K]^T, fp16 hi/lo split, one CTA of two
// warpgroups (64 rows each), N in 16-column slices, both operands from shared memory in the production layout.
// =====================================================================================================
__global__ void __launch_bounds__(256, 1)
selftest_kernel(const float *__restrict__ A, const float *__restrict__ Bm, float *__restrict__ D, int N, int K) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int a_plane = 128 * K * 2, b_plane = N * K * 2;
    uint8_t *sa = smem, *sb = smem + 2 * a_plane;
    const int tid = threadIdx.x, wg = tid >> 7, warp = (tid >> 5) & 3, lane = tid & 31;
    for (int i = tid; i < 128 * K; i += 256) {
        const int r = i / K, k = i % K;
        __half hi, lo;
        split_f16(A[i], hi, lo);
        const int off = (k / 8) * (128 * 16) + r * 16 + (k % 8) * 2;
        *reinterpret_cast<__half *>(sa + off) = hi;
        *reinterpret_cast<__half *>(sa + a_plane + off) = lo;
    }
    for (int i = tid; i < N * K; i += 256) {
        const int r = i / K, k = i % K;
        __half hi, lo;
        split_f16(Bm[i], hi, lo);
        const int off = (k / 8) * (N * 16) + r * 16 + (k % 8) * 2;
        *reinterpret_cast<__half *>(sb + off) = hi;
        *reinterpret_cast<__half *>(sb + b_plane + off) = lo;
    }
    fence_proxy_async_smem();
    __syncthreads();
    for (int n0 = 0; n0 < N; n0 += 16) {
        float d[8];
        wg_fence();
        uint32_t acc = 0;
        for (int prod = 0; prod < 3; ++prod) {
            const int pa = (prod == 2), pb = (prod == 1);
            for (int ks = 0; ks < K / 16; ++ks) {
                const uint64_t ad = make_smem_desc(smem_u32(sa + pa * a_plane) + ks * 2 * 128 * 16 + wg * 64 * 16, 128 * 16, 128);
                const uint64_t bd = make_smem_desc(smem_u32(sb + pb * b_plane) + ks * 2 * N * 16 + n0 * 16, N * 16, 128);
                Wgmma<16>::ss(d, ad, bd, acc);
                acc = 1;
            }
        }
        wg_commit();
        wg_wait_all();
        wg_hold(d);
        const int row = wg * 64 + warp * 16 + (lane >> 2);
        for (int k = 0; k < 8; ++k)
            D[(row + 8 * ((k >> 1) & 1)) * N + n0 + 8 * (k >> 2) + 2 * (lane & 3) + (k & 1)] = d[k];
    }
}

int selftest_umma(int device, const float *A, const float *B, float *D, int N, int K, int variant) {
    MDK_REQUIRE(N >= 16 && N <= 128 && N % 16 == 0, MDK_ERR_ARG, "selftest_umma: N must be a multiple of 16 in [16,128]");
    MDK_REQUIRE(K >= 16 && K <= 256 && K % 16 == 0, MDK_ERR_ARG, "selftest_umma: K must be a multiple of 16 in [16,256]");
    MDK_REQUIRE(variant == 0, MDK_ERR_ARG, "selftest_umma: variant must be 0");
    MDK_CUDA(cudaSetDevice(device));
    float *dA = nullptr, *dB = nullptr, *dD = nullptr;
    MDK_CUDA(cudaMalloc(&dA, sizeof(float) * 128 * K));
    MDK_CUDA(cudaMalloc(&dB, sizeof(float) * N * K));
    MDK_CUDA(cudaMalloc(&dD, sizeof(float) * 128 * N));
    MDK_CUDA(cudaMemcpy(dA, A, sizeof(float) * 128 * K, cudaMemcpyHostToDevice));
    MDK_CUDA(cudaMemcpy(dB, B, sizeof(float) * N * K, cudaMemcpyHostToDevice));
    const int smem = 2 * 128 * K * 2 + 2 * N * K * 2;
    MDK_REQUIRE(smem <= 227 * 1024, MDK_ERR_ARG, "selftest_umma: N*K too large for shared memory");
    MDK_CUDA(cudaFuncSetAttribute(selftest_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    selftest_kernel<<<1, 256, smem>>>(dA, dB, dD, N, K);
    MDK_CUDA(cudaGetLastError());
    MDK_CUDA(cudaDeviceSynchronize());
    MDK_CUDA(cudaMemcpy(D, dD, sizeof(float) * 128 * N, cudaMemcpyDeviceToHost));
    cudaFree(dA); cudaFree(dB); cudaFree(dD);
    return MDK_OK;
}

}  // namespace mdk
