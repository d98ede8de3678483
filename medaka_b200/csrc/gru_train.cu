// Training of the consensus GRU (medaka train, medaka/training.py + the training half of medaka/torch_ext.py): the
// mdk_trainer object of include/medaka_b200.h, its kernels and its host orchestration.  All arithmetic is fp32, the
// arithmetic of MDK_PREC_FP32.  One step:
//   forward      inproj0 (misc.cu) -> rec_fp32<SAVE> (gru_fp32.cu) -> gemm_fp32 -> rec_fp32<SAVE> -> head (misc.cu): the
//                inference fp32 path's kernels, which also keep r, z, n and W_hn.h_{t-1} + b_hn per position for BPTT
//   loss head    log-softmax cross-entropy (mean over B*T), dlogits, argmax == label count           (loss_kernel)
//   head bwd     dh1 = dlogits . W_lin (head_bwd_kernel); dW_lin, db_lin (wgrad / colsum)
//   BPTT         per layer and direction, time in the reverse of the forward order: dG_i = [dr, dz, dn] into gi
//                (bptt_kernel); dW_ih = dG_i^T X, dW_hh = dG_h^T H_{t-1}, bias sums (wgrad / colsum, split-M partial
//                sums added in a fixed order, no float atomics: two identical steps give bit-identical gradients);
//                layer 1's dX = dG_i . W_ih1 by gemm_fp32 on a transposed copy of W_ih1
//   step         global L2 norm (fixed-order reduction), non-finite skip, clip_grad_norm_ scaling, the optimizer rule
//                (RMSprop, Adam, NAdam, SGD as torch.optim writes them) on the fp32 master weights, then the forward's
//                packed weights rebuilt on the device from them (no host round trip).
// Weights and gradients are one flat array each, in torch state-dict order (ParamLayout).
#include <cmath>
#include <cstring>
#include <new>

#include "common.cuh"
#include "train_common.cuh"

namespace mdk {

// ------------------------------------------------------------------------------------------------------------- kernels
// BPTT of one layer, both directions (blockIdx.y), NB windows per CTA, thread j = hidden unit j.  Walks time in the
// reverse of the direction's forward order; per step, with dh = dh_out (the layer output's gradient) + the carry:
//   dn = dh (1 - z)(1 - n^2)        dz = dh (h_{t-1} - n) z (1 - z)        dr = dn (W_hn h_{t-1} + b_hn) r (1 - r)
//   carry = dh z + W_hr^T dr + W_hz^T dz + W_hn^T (dn r)
// and writes dG_i = [dr, dz, dn] over the layer's gi rows.  W_hh ([3 HS][HS], torch layout: thread j reads column j)
// stays in shared memory at HS = 128 and streams from L2 at HS = 256, as in the forward; the NB gate-gradient vectors
// are shared-memory broadcasts.
template <int HS, int NB>
__global__ void __launch_bounds__(HS, 1) bptt_kernel(const float *__restrict__ save, const float *__restrict__ h,
                                                     const float *__restrict__ dh_out, const float *__restrict__ w_hh0,
                                                     const float *__restrict__ w_hh1, float *__restrict__ dgi,
                                                     int64_t B, int64_t T) {
    constexpr int G3S = 3 * HS;
    constexpr bool SMEM_W = HS == H;
    extern __shared__ __align__(16) float smem[];
    float *gs = smem + (SMEM_W ? G3S * HS : 0);     // [2][NB][3 HS]: dr, dz, dn r
    const int j = threadIdx.x;
    const int dir = blockIdx.y;
    const int64_t b0 = (int64_t)blockIdx.x * NB;
    const int nb = (int)min((int64_t)NB, B - b0);
    const float *wsrc = dir ? w_hh1 : w_hh0;
    const float *w = SMEM_W ? smem : wsrc;
    if (SMEM_W)
        for (int i = j; i < G3S * HS / 4; i += HS)
            reinterpret_cast<float4 *>(smem)[i] = reinterpret_cast<const float4 *>(wsrc)[i];
    float carry[NB];
#pragma unroll
    for (int n = 0; n < NB; ++n) carry[n] = 0.f;
    __syncthreads();

    // per window: dh_out, r, z, n, ghn, h_{t-1} of the step, loaded one step ahead
    auto load = [&](int64_t t, float (&v)[6][NB]) {
        const int64_t tp = dir ? t + 1 : t - 1;
        const bool has_prev = tp >= 0 && tp < T;
#pragma unroll
        for (int n = 0; n < NB; ++n) {
            if (n < nb) {
                const int64_t p = (b0 + n) * T + t;
                const float *sv = save + (p * NDIR + dir) * (4 * HS) + j;
                v[0][n] = dh_out[p * (NDIR * HS) + dir * HS + j];
                v[1][n] = sv[0]; v[2][n] = sv[HS]; v[3][n] = sv[2 * HS]; v[4][n] = sv[3 * HS];
                v[5][n] = has_prev ? h[((b0 + n) * T + tp) * (NDIR * HS) + dir * HS + j] : 0.f;
            } else {
#pragma unroll
                for (int q = 0; q < 6; ++q) v[q][n] = 0.f;
            }
        }
    };
    float nxt[6][NB];
    load(dir ? 0 : T - 1, nxt);
    int cur = 0;
    for (int64_t step = 0; step < T; ++step) {
        const int64_t t = dir ? step : T - 1 - step;
        float v[6][NB];
#pragma unroll
        for (int q = 0; q < 6; ++q)
#pragma unroll
            for (int n = 0; n < NB; ++n) v[q][n] = nxt[q][n];
        if (step + 1 < T) load(dir ? t + 1 : t - 1, nxt);
        float *g = gs + cur * NB * G3S;
        float dhz[NB];
#pragma unroll
        for (int n = 0; n < NB; ++n) {
            const float dh = v[0][n] + carry[n];
            const float r = v[1][n], z = v[2][n], nn = v[3][n], ghn = v[4][n], hp = v[5][n];
            const float dn = dh * (1.f - z) * (1.f - nn * nn);
            const float dz = dh * (hp - nn) * z * (1.f - z);
            const float dr = dn * ghn * r * (1.f - r);
            dhz[n] = dh * z;
            g[n * G3S + j] = dr;
            g[n * G3S + HS + j] = dz;
            g[n * G3S + 2 * HS + j] = dn * r;
            if (n < nb) {
                float *o = dgi + ((b0 + n) * T + t) * (NDIR * G3S) + dir * G3S + j;
                o[0] = dr; o[HS] = dz; o[2 * HS] = dn;
            }
        }
        __syncthreads();
        float acc[NB];
#pragma unroll
        for (int n = 0; n < NB; ++n) acc[n] = 0.f;
#pragma unroll 2
        for (int c = 0; c < HS; c += 4) {
#pragma unroll
            for (int gate = 0; gate < 3; ++gate) {
                float4 gv[NB];
#pragma unroll
                for (int n = 0; n < NB; ++n) gv[n] = *reinterpret_cast<const float4 *>(g + n * G3S + gate * HS + c);
#pragma unroll
                for (int cc = 0; cc < 4; ++cc) {
                    const float wv = w[(gate * HS + c + cc) * HS + j];
#pragma unroll
                    for (int n = 0; n < NB; ++n) {
                        const float gk = cc == 0 ? gv[n].x : cc == 1 ? gv[n].y : cc == 2 ? gv[n].z : gv[n].w;
                        acc[n] = fmaf(wv, gk, acc[n]);
                    }
                }
            }
        }
#pragma unroll
        for (int n = 0; n < NB; ++n) carry[n] = dhz[n] + acc[n];
        cur ^= 1;
    }
}

// The folded biases of one (layer, direction), as gru_pack.cuh builds them: bias_gi = b_ih + b_hh for r, z and b_ih for
// n; b_hn = b_hh's n third
__global__ void __launch_bounds__(256) fold_bias_kernel(const float *__restrict__ b_ih, const float *__restrict__ b_hh,
                                                        float *__restrict__ bias_gi, float *__restrict__ b_hn, int hs) {
    const int r = blockIdx.x * 256 + threadIdx.x;
    if (r >= 3 * hs) return;
    bias_gi[r] = r < 2 * hs ? b_ih[r] + b_hh[r] : b_ih[r];
    if (r >= 2 * hs) b_hn[r - 2 * hs] = b_hh[r];
}

// ---------------------------------------------------------------------------------------------------------- host side
// Offsets of the tensors in the flat weight / gradient arrays, torch state-dict order: for each layer and direction
// weight_ih, weight_hh, bias_ih, bias_hh, then linear.weight, linear.bias
struct ParamLayout {
    int64_t w_ih[2][2], w_hh[2][2], b_ih[2][2], b_hh[2][2], lin_w, lin_b, total;
    ParamLayout() = default;
    ParamLayout(int F, int hs) {
        int64_t o = 0;
        for (int l = 0; l < 2; ++l)
            for (int d = 0; d < NDIR; ++d) {
                const int in = l == 0 ? F : NDIR * hs;
                w_ih[l][d] = o; o += (int64_t)3 * hs * in;
                w_hh[l][d] = o; o += (int64_t)3 * hs * hs;
                b_ih[l][d] = o; o += 3 * hs;
                b_hh[l][d] = o; o += 3 * hs;
            }
        lin_w = o; o += (int64_t)NCLS * NDIR * hs;
        lin_b = o; o += NCLS;
        total = o;
    }
};

// Floats per position of the workspace: the saved activations of both layers (r, z, n, ghn per direction: 16 hs),
// gi (6 hs, then the gate gradients), h0, h1 and the layer-output gradient (2 hs each), logits, probs and dlogits,
// the features and the label
static int64_t train_floats_per_pos(int F, int hs) { return (int64_t)28 * hs + 3 * NCLS + F + 1; }
// Past this the step fails instead of taking the card: 100 windows x 10 000 columns at gru_size 256 (the reference's
// default training shape) need 29.5 GB
constexpr int64_t TRAIN_WS_BUDGET = (int64_t)64 << 30;

}  // namespace mdk

using namespace mdk;

enum { TS_FWD, TS_HEAD, TS_BPTT, TS_RED, TS_OPT, TS_N };

struct mdk_trainer {
    int device = 0;
    int sm_count = 132;
    mdk_model_desc desc{};
    int hs = H;
    ParamLayout lay;
    std::vector<float> host_params;
    std::vector<uint8_t> loaded;      // which (layer, dir) GRU tensors and the linear head were loaded
    bool uploaded = false;
    cudaStream_t stream = nullptr;
    // device state
    float *param = nullptr, *grad = nullptr, *s1 = nullptr, *s2 = nullptr;
    float *w_in[2] = {nullptr, nullptr}, *bias_gi[2] = {nullptr, nullptr}, *b_hn[2] = {nullptr, nullptr};
    float *w_hh_t[2] = {nullptr, nullptr}, *w_ih1_t = nullptr, *zeros = nullptr;
    double *red = nullptr;            // [3][RED_BLOCKS] partials + [3] totals: loss, correct, sum of squares
    // workspace
    int64_t cap_pos = 0;
    float *ws = nullptr;
    float *part = nullptr;
    int64_t cap_part = 0;
    // optimizer
    mdk_optim_desc opt{};
    int64_t opt_steps = 0;            // steps taken (not skipped) since the optimizer was set or the weights loaded
    double mu_product = 1.0;          // NAdam
    int bptt_windows = 0;             // 0: from B
    cudaEvent_t ev[16] = {};
    int ev_kind[16] = {};
    int n_ev = 0;
    float stage_ms[TS_N] = {};
};

namespace {

int alloc_f(float **p, int64_t n) {
    MDK_CUDA(cudaMalloc(reinterpret_cast<void **>(p), (size_t)std::max<int64_t>(n, 1) * sizeof(float)));
    return MDK_OK;
}
void free_p(void *&p) {
    if (p) cudaFree(p);
    p = nullptr;
}
template <class T> void free_t(T *&p) { void *q = p; free_p(q); p = nullptr; }

int in_feat(const mdk_trainer *tr, int layer) { return layer == 0 ? tr->desc.num_features : NDIR * tr->hs; }

// The forward's packed weights of both layers from the master weights (gru_pack.cuh's fp32 arrays), on the stream
int repack(mdk_trainer *tr) {
    const int hs = tr->hs, g3 = 3 * hs;
    cudaStream_t s = tr->stream;
    for (int l = 0; l < 2; ++l) {
        const int in = in_feat(tr, l);
        for (int d = 0; d < NDIR; ++d) {
            const float *w_ih = tr->param + tr->lay.w_ih[l][d], *w_hh = tr->param + tr->lay.w_hh[l][d];
            MDK_CUDA(cudaMemcpyAsync(tr->w_in[l] + (int64_t)d * g3 * in, w_ih, (size_t)g3 * in * sizeof(float),
                                     cudaMemcpyDeviceToDevice, s));
            fold_bias_kernel<<<(g3 + 255) / 256, 256, 0, s>>>(tr->param + tr->lay.b_ih[l][d], tr->param + tr->lay.b_hh[l][d],
                                                            tr->bias_gi[l] + d * g3, tr->b_hn[l] + d * hs, hs);
            transpose_kernel<<<dim3((hs + 31) / 32, (g3 + 31) / 32), 256, 0, s>>>(w_hh, tr->w_hh_t[l] + (int64_t)d * hs * g3,
                                                                                 g3, hs);
        }
    }
    transpose_kernel<<<dim3((NDIR * hs + 31) / 32, (NDIR * g3 + 31) / 32), 256, 0, s>>>(tr->w_in[1], tr->w_ih1_t, NDIR * g3,
                                                                                       NDIR * hs);
    MDK_CUDA(cudaGetLastError());
    return MDK_OK;
}

int upload(mdk_trainer *tr) {
    if (tr->uploaded) return MDK_OK;
    for (uint8_t l : tr->loaded) MDK_REQUIRE(l, MDK_ERR_STATE, "trainer: weights not loaded for every tensor");
    const int64_t n = tr->lay.total;
    MDK_CUDA(cudaMemcpyAsync(tr->param, tr->host_params.data(), n * sizeof(float), cudaMemcpyHostToDevice, tr->stream));
    MDK_CUDA(cudaMemsetAsync(tr->s1, 0, n * sizeof(float), tr->stream));
    MDK_CUDA(cudaMemsetAsync(tr->s2, 0, n * sizeof(float), tr->stream));
    MDK_CUDA(cudaMemsetAsync(tr->grad, 0, n * sizeof(float), tr->stream));
    int rc = repack(tr);
    if (rc) return rc;
    MDK_CUDA(cudaStreamSynchronize(tr->stream));
    tr->uploaded = true;
    tr->opt_steps = 0;
    tr->mu_product = 1.0;
    return MDK_OK;
}

struct WsView {
    float *save[2], *gi, *h0, *h1, *dh, *logits, *probs, *dlogits, *feats;
    int32_t *labels;
};

WsView ws_view(const mdk_trainer *tr, int64_t P) {
    const int64_t hs = tr->hs;
    float *o = tr->ws;
    auto take = [&](int64_t n) { float *r = o; o += (n + 63) / 64 * 64; return r; };
    WsView v;
    v.save[0] = take(P * 8 * hs);
    v.save[1] = take(P * 8 * hs);
    v.gi = take(P * 6 * hs);
    v.h0 = take(P * 2 * hs);
    v.h1 = take(P * 2 * hs);
    v.dh = take(P * 2 * hs);
    v.logits = take(P * NCLS);
    v.probs = take(P * NCLS);
    v.dlogits = take(P * NCLS);
    v.feats = take(P * tr->desc.num_features);
    v.labels = reinterpret_cast<int32_t *>(take(P));
    return v;
}

int64_t ws_floats(const mdk_trainer *tr, int64_t P) {
    return P * train_floats_per_pos(tr->desc.num_features, tr->hs) + 11 * 64;
}

// the largest partial-sum array the reductions of a step over P positions need
int64_t part_floats(const mdk_trainer *tr, int64_t P) {
    const int hs = tr->hs, F = tr->desc.num_features;
    auto tiles = [](int64_t n, int64_t k) { return ((n + RT - 1) / RT) * ((k + RT - 1) / RT); };
    int64_t need = 0;
    auto w = [&](int64_t n, int64_t k) { need = std::max<int64_t>(need, split_for(P, tiles(n, k)).splits * n * k); };
    w(6 * hs, F);
    w(6 * hs, 2 * hs);
    w(3 * hs, hs);
    w(NCLS, 2 * hs);
    w(6 * hs, 1);      // column sums
    return need;
}

int ensure_ws(mdk_trainer *tr, int64_t P) {
    const int64_t need = ws_floats(tr, P);
    // the bytes mdk_trainer_workspace_bytes reports: the workspace and the reductions' partial sums
    MDK_REQUIRE((need + part_floats(tr, P)) * (int64_t)sizeof(float) <= TRAIN_WS_BUDGET, MDK_ERR_ARG,
                "trainer: a batch of this many positions exceeds the 64 GiB training workspace budget (see "
                "mdk_trainer_workspace_bytes)");
    if (need > tr->cap_pos) {
        MDK_CUDA(cudaStreamSynchronize(tr->stream));
        free_t(tr->ws);
        tr->cap_pos = 0;
        int rc;
        if ((rc = alloc_f(&tr->ws, need))) return rc;
        tr->cap_pos = need;
    }
    const int64_t np = part_floats(tr, P);
    if (np > tr->cap_part) {
        MDK_CUDA(cudaStreamSynchronize(tr->stream));
        free_t(tr->part);
        tr->cap_part = 0;
        int rc;
        if ((rc = alloc_f(&tr->part, np))) return rc;
        tr->cap_part = np;
    }
    return MDK_OK;
}

void mark(mdk_trainer *tr, int kind) {
    if (tr->n_ev < 16) {
        cudaEventRecord(tr->ev[tr->n_ev], tr->stream);
        tr->ev_kind[tr->n_ev] = kind;
        ++tr->n_ev;
    }
}

// dst0 / dst1 <- sum over M rows of A(m, n) X(m, k) (rows n < rows_split to dst0)
template <int AMODE, int XMODE>
int wgrad(mdk_trainer *tr, const RedA &A, const RedX &X, int64_t M, int rows_split, float *dst0, float *dst1) {
    const int64_t tn = (A.N + RT - 1) / RT, tk = (X.K + RT - 1) / RT;
    const Split sp = split_for(M, tn * tk);
    wgrad_kernel<AMODE, XMODE><<<dim3((unsigned)tn, (unsigned)tk, (unsigned)sp.splits), 256, 0, tr->stream>>>(A, X, M, sp.chunk,
                                                                                                          tr->part);
    const int64_t count = (int64_t)A.N * X.K;
    reduce_partials_kernel<<<(unsigned)((count + 255) / 256), 256, 0, tr->stream>>>(tr->part, sp.splits, count, X.K,
                                                                                   rows_split, dst0, dst1);
    MDK_CUDA(cudaGetLastError());
    return MDK_OK;
}

template <int AMODE>
int colsum(mdk_trainer *tr, const RedA &A, int64_t M, int rows_split, float *dst0, float *dst1) {
    const Split sp = split_for(M, (A.N + 255) / 256);
    colsum_kernel<AMODE><<<dim3((unsigned)((A.N + 255) / 256), (unsigned)sp.splits), 256, 0, tr->stream>>>(A, M, sp.chunk,
                                                                                                         tr->part);
    reduce_partials_kernel<<<(unsigned)((A.N + 255) / 256), 256, 0, tr->stream>>>(tr->part, sp.splits, A.N, 1, rows_split,
                                                                                 dst0, dst1);
    MDK_CUDA(cudaGetLastError());
    return MDK_OK;
}

int bptt_nb(const mdk_trainer *tr, int64_t B) {
    if (tr->bptt_windows) return tr->bptt_windows;
    // the fewest windows per CTA whose CTAs (both directions) still fit one wave: a training batch (100 windows by
    // default) at 8 per CTA would leave most SMs idle
    for (int nb : {1, 2, 4})
        if (((B + nb - 1) / nb) * NDIR <= tr->sm_count) return nb;
    return 8;
}

template <int HS, int NB>
cudaError_t launch_bptt_t(const float *save, const float *h, const float *dh, const float *w0, const float *w1, float *dgi,
                          int64_t B, int64_t T, cudaStream_t s) {
    const size_t smem = (size_t)((HS == H ? 3 * HS * HS : 0) + 2 * NB * 3 * HS) * sizeof(float);
    cudaError_t e = cudaFuncSetAttribute(bptt_kernel<HS, NB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    bptt_kernel<HS, NB><<<dim3((unsigned)((B + NB - 1) / NB), NDIR), HS, smem, s>>>(save, h, dh, w0, w1, dgi, B, T);
    return cudaGetLastError();
}
template <int HS>
cudaError_t launch_bptt_h(int nb, const float *save, const float *h, const float *dh, const float *w0, const float *w1,
                          float *dgi, int64_t B, int64_t T, cudaStream_t s) {
    switch (nb) {
    case 1: return launch_bptt_t<HS, 1>(save, h, dh, w0, w1, dgi, B, T, s);
    case 2: return launch_bptt_t<HS, 2>(save, h, dh, w0, w1, dgi, B, T, s);
    case 4: return launch_bptt_t<HS, 4>(save, h, dh, w0, w1, dgi, B, T, s);
    default: return launch_bptt_t<HS, 8>(save, h, dh, w0, w1, dgi, B, T, s);
    }
}

// Forward of B windows of T columns from the staged features: logits and probs, the saved activations with save
int forward(mdk_trainer *tr, const WsView &v, int64_t B, int64_t T, bool save) {
    const int64_t P = B * T;
    const int hs = tr->hs;
    cudaStream_t s = tr->stream;
    MDK_CUDA(launch_inproj0(v.feats, tr->w_in[0], tr->bias_gi[0], v.gi, P, tr->desc.num_features, T, 0, s, hs));
    MDK_CUDA(launch_rec_fp32(v.gi, tr->w_hh_t[0], tr->b_hn[0], v.h0, B, T, s, hs, save ? v.save[0] : nullptr));
    MDK_CUDA(launch_gemm_fp32(v.h0, tr->w_in[1], tr->bias_gi[1], v.gi, P, NDIR * hs, 6 * hs, s));
    MDK_CUDA(launch_rec_fp32(v.gi, tr->w_hh_t[1], tr->b_hn[1], v.h1, B, T, s, hs, save ? v.save[1] : nullptr));
    MDK_CUDA(launch_head(v.h1, tr->param + tr->lay.lin_w, tr->param + tr->lay.lin_b, B, T, 0, v.probs, v.logits, nullptr,
                         s, nullptr, nullptr, NDIR * hs));
    return MDK_OK;
}

int loss(mdk_trainer *tr, const WsView &v, int64_t P) {
    loss_kernel<<<RED_BLOCKS, 256, 0, tr->stream>>>(v.logits, v.labels, P, (float)(1.0 / (double)P), v.dlogits, tr->red,
                                                    tr->red + RED_BLOCKS);
    sum_partials_kernel<<<1, 256, 0, tr->stream>>>(tr->red, RED_BLOCKS, tr->red + 3 * RED_BLOCKS);
    sum_partials_kernel<<<1, 256, 0, tr->stream>>>(tr->red + RED_BLOCKS, RED_BLOCKS, tr->red + 3 * RED_BLOCKS + 1);
    MDK_CUDA(cudaGetLastError());
    return MDK_OK;
}

// Gradients of one layer from its gate gradients (in v.gi): dW_ih, dW_hh, the biases; X its input rows
int layer_grads(mdk_trainer *tr, const WsView &v, int l, const float *X, int64_t B, int64_t T) {
    const int64_t P = B * T;
    const int hs = tr->hs, in = in_feat(tr, l);
    float *g = tr->grad;
    const ParamLayout &L = tr->lay;
    int rc;
    const float *hl = l ? v.h1 : v.h0;
    // dW_ih of both directions: dG_i [P][6 hs] against the layer input
    if ((rc = wgrad<0, 0>(tr, RedA{v.gi, 6 * hs, 6 * hs, nullptr, hs}, RedX{X, in, in, T, 0}, P, 3 * hs, g + L.w_ih[l][0],
                          g + L.w_ih[l][1])))
        return rc;
    // db_ih = sum dG_i
    if ((rc = colsum<0>(tr, RedA{v.gi, 6 * hs, 6 * hs, nullptr, hs}, P, 3 * hs, g + L.b_ih[l][0], g + L.b_ih[l][1])))
        return rc;
    for (int d = 0; d < NDIR; ++d) {
        const RedA A{v.gi + d * 3 * hs, 6 * hs, 3 * hs, v.save[l] + d * 4 * hs, hs};
        // dW_hh = dG_h^T H_{t-1};  db_hh = sum dG_h (r, z: as db_ih; n: sum dn r)
        if ((rc = wgrad<1, 1>(tr, A, RedX{hl + d * hs, 2 * hs, hs, T, d}, P, 3 * hs, g + L.w_hh[l][d], nullptr))) return rc;
        if ((rc = colsum<1>(tr, A, P, 3 * hs, g + L.b_hh[l][d], nullptr))) return rc;
    }
    return MDK_OK;
}

int backward(mdk_trainer *tr, const WsView &v, int64_t B, int64_t T) {
    const int64_t P = B * T;
    const int hs = tr->hs, nb = bptt_nb(tr, B);
    cudaStream_t s = tr->stream;
    const ParamLayout &L = tr->lay;
    int rc;
    // head: dh1 = dlogits W_lin; dW_lin = dlogits^T h1; db_lin = sum dlogits
    head_bwd_kernel<<<(unsigned)std::min<int64_t>((P * 2 * hs + 255) / 256, 132 * 16), 256, 0, s>>>(
        v.dlogits, tr->param + L.lin_w, v.dh, P, 2 * hs);
    if ((rc = wgrad<0, 0>(tr, RedA{v.dlogits, NCLS, NCLS, nullptr, hs}, RedX{v.h1, 2 * hs, 2 * hs, T, 0}, P, NCLS,
                          tr->grad + L.lin_w, nullptr)))
        return rc;
    if ((rc = colsum<0>(tr, RedA{v.dlogits, NCLS, NCLS, nullptr, hs}, P, NCLS, tr->grad + L.lin_b, nullptr))) return rc;
    mark(tr, TS_HEAD);
    for (int l = 1; l >= 0; --l) {
        const float *w0 = tr->param + L.w_hh[l][0], *w1 = tr->param + L.w_hh[l][1];
        const float *hl = l ? v.h1 : v.h0;
        MDK_CUDA(hs == H256 ? launch_bptt_h<H256>(nb, v.save[l], hl, v.dh, w0, w1, v.gi, B, T, s)
                            : launch_bptt_h<H>(nb, v.save[l], hl, v.dh, w0, w1, v.gi, B, T, s));
        mark(tr, TS_BPTT);
        if ((rc = layer_grads(tr, v, l, l ? v.h0 : v.feats, B, T))) return rc;
        // dh0 = dG_i1 . W_ih1 (both directions' gates), over dh1, which the layer-1 BPTT has consumed
        if (l == 1) MDK_CUDA(launch_gemm_fp32(v.gi, tr->w_ih1_t, tr->zeros, v.dh, P, 6 * hs, 2 * hs, s));
        mark(tr, TS_RED);
    }
    return MDK_OK;
}

int stage(mdk_trainer *tr, const WsView &v, const float *feats, const int32_t *labels, int64_t B, int64_t T) {
    const int64_t P = B * T;
    MDK_CUDA(cudaMemcpyAsync(v.feats, feats, (size_t)P * tr->desc.num_features * sizeof(float), cudaMemcpyHostToDevice,
                             tr->stream));
    if (labels) MDK_CUDA(cudaMemcpyAsync(v.labels, labels, (size_t)P * sizeof(int32_t), cudaMemcpyHostToDevice, tr->stream));
    return MDK_OK;
}

int check_batch(mdk_trainer *tr, const float *feats, const int32_t *labels, int64_t B, int64_t T) {
    MDK_REQUIRE(tr && feats, MDK_ERR_ARG, "trainer: NULL argument");
    MDK_REQUIRE(B >= 1 && T >= 1, MDK_ERR_ARG, "trainer: empty batch");
    if (labels) {
        const int64_t P = B * T;
        for (int64_t i = 0; i < P; ++i)
            MDK_REQUIRE(labels[i] >= 0 && labels[i] < NCLS, MDK_ERR_ARG,
                        "trainer: label out of range [0, 5) (CrossEntropyLoss raises on it)");
    }
    MDK_CUDA(cudaSetDevice(tr->device));
    int rc;
    if ((rc = upload(tr))) return rc;
    return ensure_ws(tr, B * T);
}

// Before a load changes some of the weights: the host image takes the device's trained weights, so that the tensors
// the load does not name keep their values when the image is uploaded again
int sync_host(mdk_trainer *tr) {
    if (!tr->uploaded) return MDK_OK;
    MDK_CUDA(cudaSetDevice(tr->device));
    MDK_CUDA(cudaMemcpyAsync(tr->host_params.data(), tr->param, tr->lay.total * sizeof(float), cudaMemcpyDeviceToHost,
                             tr->stream));
    MDK_CUDA(cudaStreamSynchronize(tr->stream));
    return MDK_OK;
}

int read_stats(mdk_trainer *tr, int64_t P, bool with_norm, mdk_train_stats *st) {
    double tot[3];
    MDK_CUDA(cudaMemcpyAsync(tot, tr->red + 3 * RED_BLOCKS, sizeof(tot), cudaMemcpyDeviceToHost, tr->stream));
    MDK_CUDA(cudaStreamSynchronize(tr->stream));
    if (st) {
        st->loss = tot[0] / (double)P;
        st->n_correct = (int64_t)tot[1];
        st->n_positions = P;
        st->grad_norm = with_norm ? (float)std::sqrt(tot[2]) : 0.f;
        st->skipped = with_norm && !std::isfinite(st->grad_norm) ? 1 : 0;
    }
    return MDK_OK;
}

}  // namespace

extern "C" {

int mdk_trainer_create(int device, const mdk_model_desc *desc, mdk_trainer **out) {
    MDK_REQUIRE(desc && out, MDK_ERR_ARG, "trainer_create: NULL argument");
    MDK_REQUIRE(desc->gru_size == H || desc->gru_size == H256, MDK_ERR_UNSUPPORTED, "trainer_create: gru_size must be 128 or 256");
    MDK_REQUIRE(desc->n_layers == 2 && desc->bidirectional == 1, MDK_ERR_UNSUPPORTED,
                "trainer_create: only the 2-layer bidirectional GRU is supported");
    MDK_REQUIRE(desc->num_classes == NCLS, MDK_ERR_UNSUPPORTED, "trainer_create: the head has 5 classes");
    MDK_REQUIRE(desc->num_features >= 1 && desc->num_features <= 1024, MDK_ERR_ARG, "trainer_create: bad num_features");
    int ndev = 0;
    MDK_CUDA(cudaGetDeviceCount(&ndev));
    MDK_REQUIRE(device >= 0 && device < ndev, MDK_ERR_ARG, "trainer_create: no such CUDA device");
    cudaDeviceProp prop;
    MDK_CUDA(cudaGetDeviceProperties(&prop, device));
    MDK_REQUIRE(prop.major == 9 && prop.minor == 0, MDK_ERR_UNSUPPORTED,
                "trainer_create: this library is built for sm_90a (Hopper H100) only");
    MDK_CUDA(cudaSetDevice(device));
    mdk_trainer *tr = new (std::nothrow) mdk_trainer();
    MDK_REQUIRE(tr, MDK_ERR_NOMEM, "trainer_create: out of host memory");
    tr->device = device;
    tr->desc = *desc;
    tr->hs = desc->gru_size;
    tr->sm_count = prop.multiProcessorCount;
    tr->lay = ParamLayout(desc->num_features, tr->hs);
    tr->host_params.assign(tr->lay.total, 0.f);
    tr->loaded.assign(5, 0);
    tr->opt.kind = MDK_OPT_RMSPROP;
    tr->opt.alpha = 0.9f; tr->opt.eps = 1e-7f;    // the reference's RMSprop defaults (medaka/training.py)
    const int hs = tr->hs, g3 = 3 * hs;
    int rc = MDK_OK;
    cudaError_t e = cudaStreamCreateWithFlags(&tr->stream, cudaStreamNonBlocking);
    for (auto &ev : tr->ev)
        if (e == cudaSuccess) e = cudaEventCreate(&ev);
    if (e != cudaSuccess) rc = cuda_fail(e, "trainer_create: stream / events", __FILE__, __LINE__);
    const int64_t n = tr->lay.total;
    if (!rc) rc = alloc_f(&tr->param, n);
    if (!rc) rc = alloc_f(&tr->grad, n);
    if (!rc) rc = alloc_f(&tr->s1, n);
    if (!rc) rc = alloc_f(&tr->s2, n);
    for (int l = 0; l < 2 && !rc; ++l) {
        rc = alloc_f(&tr->w_in[l], (int64_t)NDIR * g3 * in_feat(tr, l));
        if (!rc) rc = alloc_f(&tr->bias_gi[l], NDIR * g3);
        if (!rc) rc = alloc_f(&tr->b_hn[l], NDIR * hs);
        if (!rc) rc = alloc_f(&tr->w_hh_t[l], (int64_t)NDIR * hs * g3);
    }
    if (!rc) rc = alloc_f(&tr->w_ih1_t, (int64_t)NDIR * g3 * NDIR * hs);
    if (!rc) rc = alloc_f(&tr->zeros, NDIR * hs);
    if (!rc) {
        e = cudaMalloc(&tr->red, (3 * RED_BLOCKS + 3) * sizeof(double));
        if (e == cudaSuccess) e = cudaMemset(tr->zeros, 0, NDIR * hs * sizeof(float));
        if (e == cudaSuccess) e = cudaMemset(tr->red, 0, (3 * RED_BLOCKS + 3) * sizeof(double));
        if (e != cudaSuccess) rc = cuda_fail(e, "trainer_create", __FILE__, __LINE__);
    }
    if (rc) {
        mdk_trainer_destroy(tr);
        return rc;
    }
    *out = tr;
    return MDK_OK;
}

int mdk_trainer_destroy(mdk_trainer *tr) {
    if (!tr) return MDK_OK;
    cudaSetDevice(tr->device);
    if (tr->stream) cudaStreamSynchronize(tr->stream);
    free_t(tr->param); free_t(tr->grad); free_t(tr->s1); free_t(tr->s2);
    for (int l = 0; l < 2; ++l) { free_t(tr->w_in[l]); free_t(tr->bias_gi[l]); free_t(tr->b_hn[l]); free_t(tr->w_hh_t[l]); }
    free_t(tr->w_ih1_t); free_t(tr->zeros); free_t(tr->red); free_t(tr->ws); free_t(tr->part);
    for (auto &ev : tr->ev) if (ev) cudaEventDestroy(ev);
    if (tr->stream) cudaStreamDestroy(tr->stream);
    delete tr;
    return MDK_OK;
}

int mdk_trainer_load_gru(mdk_trainer *tr, int layer, int direction, const float *w_ih, const float *w_hh, const float *b_ih,
                         const float *b_hh) {
    MDK_REQUIRE(tr, MDK_ERR_ARG, "trainer is NULL");
    MDK_REQUIRE(layer >= 0 && layer < 2 && direction >= 0 && direction < 2, MDK_ERR_ARG, "trainer_load_gru: bad layer/direction");
    MDK_REQUIRE(w_ih && w_hh && b_ih && b_hh, MDK_ERR_ARG, "trainer_load_gru: NULL weight pointer");
    int rc;
    if ((rc = sync_host(tr))) return rc;
    const int hs = tr->hs, g3 = 3 * hs;
    const ParamLayout &L = tr->lay;
    float *hp = tr->host_params.data();
    std::memcpy(hp + L.w_ih[layer][direction], w_ih, (size_t)g3 * in_feat(tr, layer) * sizeof(float));
    std::memcpy(hp + L.w_hh[layer][direction], w_hh, (size_t)g3 * hs * sizeof(float));
    std::memcpy(hp + L.b_ih[layer][direction], b_ih, (size_t)g3 * sizeof(float));
    std::memcpy(hp + L.b_hh[layer][direction], b_hh, (size_t)g3 * sizeof(float));
    tr->loaded[layer * 2 + direction] = 1;
    tr->uploaded = false;
    return MDK_OK;
}

int mdk_trainer_load_linear(mdk_trainer *tr, const float *w, const float *b) {
    MDK_REQUIRE(tr && w && b, MDK_ERR_ARG, "trainer_load_linear: NULL argument");
    int rc;
    if ((rc = sync_host(tr))) return rc;
    float *hp = tr->host_params.data();
    std::memcpy(hp + tr->lay.lin_w, w, (size_t)NCLS * NDIR * tr->hs * sizeof(float));
    std::memcpy(hp + tr->lay.lin_b, b, NCLS * sizeof(float));
    tr->loaded[4] = 1;
    tr->uploaded = false;
    return MDK_OK;
}

int mdk_trainer_set_optimizer(mdk_trainer *tr, const mdk_optim_desc *opt) {
    MDK_REQUIRE(tr && opt, MDK_ERR_ARG, "trainer_set_optimizer: NULL argument");
    MDK_REQUIRE(opt->kind >= MDK_OPT_RMSPROP && opt->kind <= MDK_OPT_SGD, MDK_ERR_ARG, "trainer_set_optimizer: unknown kind");
    MDK_REQUIRE(!(opt->kind == MDK_OPT_SGD && opt->nesterov && (opt->momentum <= 0.f || opt->dampening != 0.f)), MDK_ERR_ARG,
                "trainer_set_optimizer: Nesterov momentum requires a momentum and zero dampening");
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

int mdk_trainer_set_bptt_windows(mdk_trainer *tr, int nb) {
    MDK_REQUIRE(tr, MDK_ERR_ARG, "trainer is NULL");
    MDK_REQUIRE(nb == 0 || nb == 1 || nb == 2 || nb == 4 || nb == 8, MDK_ERR_ARG, "trainer_set_bptt_windows: 0, 1, 2, 4 or 8");
    tr->bptt_windows = nb;
    return MDK_OK;
}

int mdk_trainer_bptt_windows(mdk_trainer *tr, int64_t B, int *nb) {
    MDK_REQUIRE(tr && nb, MDK_ERR_ARG, "trainer_bptt_windows: NULL argument");
    MDK_REQUIRE(B >= 1, MDK_ERR_ARG, "trainer_bptt_windows: need B >= 1");
    *nb = bptt_nb(tr, B);
    return MDK_OK;
}

int mdk_trainer_step(mdk_trainer *tr, const float *feats, const int32_t *labels, int64_t B, int64_t T, float lr,
                     float max_norm, mdk_train_stats *stats) {
    MDK_REQUIRE(labels, MDK_ERR_ARG, "trainer_step: NULL labels");
    int rc;
    if ((rc = check_batch(tr, feats, labels, B, T))) return rc;
    const int64_t P = B * T;
    const WsView v = ws_view(tr, P);
    tr->n_ev = 0;
    mark(tr, -1);
    if ((rc = stage(tr, v, feats, labels, B, T))) return rc;
    if ((rc = forward(tr, v, B, T, true))) return rc;
    mark(tr, TS_FWD);
    if ((rc = loss(tr, v, P))) return rc;
    if ((rc = backward(tr, v, B, T))) return rc;
    // the step: norm, skip / clip, the rule, the forward's weights
    const int64_t n = tr->lay.total;
    sumsq_kernel<<<RED_BLOCKS, 256, 0, tr->stream>>>(tr->grad, n, tr->red + 2 * RED_BLOCKS);
    sum_partials_kernel<<<1, 256, 0, tr->stream>>>(tr->red + 2 * RED_BLOCKS, RED_BLOCKS, tr->red + 3 * RED_BLOCKS + 2);
    const int64_t t = tr->opt_steps + 1;
    double mu_product = 0.0;
    const OptStep o = opt_step(tr->opt, lr, t, tr->mu_product, &mu_product);
    optim_kernel<<<(unsigned)std::min<int64_t>((n + 255) / 256, 132 * 8), 256, 0, tr->stream>>>(
        tr->param, tr->grad, tr->s1, tr->s2, n, tr->red + 3 * RED_BLOCKS + 2, max_norm > 0.f ? max_norm : INFINITY, o);
    MDK_CUDA(cudaGetLastError());
    if ((rc = repack(tr))) return rc;
    mark(tr, TS_OPT);
    mdk_train_stats st{};
    if ((rc = read_stats(tr, P, true, &st))) return rc;
    if (!st.skipped) {
        tr->opt_steps = t;
        tr->mu_product = mu_product;
    }
    for (float &x : tr->stage_ms) x = 0.f;
    for (int i = 1; i < tr->n_ev; ++i) {
        float ms = 0.f;
        MDK_CUDA(cudaEventElapsedTime(&ms, tr->ev[i - 1], tr->ev[i]));
        tr->stage_ms[tr->ev_kind[i]] += ms;
    }
    if (stats) *stats = st;
    return MDK_OK;
}

int mdk_trainer_eval(mdk_trainer *tr, const float *feats, const int32_t *labels, int64_t B, int64_t T, float *probs,
                     float *logits, mdk_train_stats *stats) {
    int rc;
    if ((rc = check_batch(tr, feats, labels, B, T))) return rc;
    const int64_t P = B * T;
    const WsView v = ws_view(tr, P);
    if ((rc = stage(tr, v, feats, labels, B, T))) return rc;
    if ((rc = forward(tr, v, B, T, false))) return rc;
    if (labels && (rc = loss(tr, v, P))) return rc;
    if (probs) MDK_CUDA(cudaMemcpyAsync(probs, v.probs, P * NCLS * sizeof(float), cudaMemcpyDeviceToHost, tr->stream));
    if (logits) MDK_CUDA(cudaMemcpyAsync(logits, v.logits, P * NCLS * sizeof(float), cudaMemcpyDeviceToHost, tr->stream));
    if (labels) return read_stats(tr, P, false, stats);
    MDK_CUDA(cudaStreamSynchronize(tr->stream));
    if (stats) *stats = mdk_train_stats{};
    return MDK_OK;
}

int mdk_trainer_num_params(mdk_trainer *tr, int64_t *n) {
    MDK_REQUIRE(tr && n, MDK_ERR_ARG, "trainer_num_params: NULL argument");
    *n = tr->lay.total;
    return MDK_OK;
}

int mdk_trainer_read_params(mdk_trainer *tr, float *out, int64_t n) {
    MDK_REQUIRE(tr && out, MDK_ERR_ARG, "trainer_read_params: NULL argument");
    MDK_REQUIRE(n == tr->lay.total, MDK_ERR_ARG, "trainer_read_params: n must be mdk_trainer_num_params");
    if (!tr->uploaded) {
        std::memcpy(out, tr->host_params.data(), n * sizeof(float));
        return MDK_OK;
    }
    MDK_CUDA(cudaSetDevice(tr->device));
    MDK_CUDA(cudaMemcpyAsync(out, tr->param, n * sizeof(float), cudaMemcpyDeviceToHost, tr->stream));
    MDK_CUDA(cudaStreamSynchronize(tr->stream));
    return MDK_OK;
}

int mdk_trainer_read_grads(mdk_trainer *tr, float *out, int64_t n) {
    MDK_REQUIRE(tr && out, MDK_ERR_ARG, "trainer_read_grads: NULL argument");
    MDK_REQUIRE(n == tr->lay.total, MDK_ERR_ARG, "trainer_read_grads: n must be mdk_trainer_num_params");
    MDK_REQUIRE(tr->uploaded, MDK_ERR_STATE, "trainer_read_grads: no step since the weights were loaded");
    MDK_CUDA(cudaSetDevice(tr->device));
    MDK_CUDA(cudaMemcpyAsync(out, tr->grad, n * sizeof(float), cudaMemcpyDeviceToHost, tr->stream));
    MDK_CUDA(cudaStreamSynchronize(tr->stream));
    return MDK_OK;
}

int mdk_trainer_workspace_bytes(const mdk_model_desc *desc, int64_t B, int64_t T, size_t *bytes, size_t *budget) {
    MDK_REQUIRE(desc && bytes, MDK_ERR_ARG, "trainer_workspace_bytes: NULL argument");
    MDK_REQUIRE(desc->gru_size == H || desc->gru_size == H256, MDK_ERR_UNSUPPORTED, "trainer: gru_size must be 128 or 256");
    mdk_trainer probe;
    probe.desc = *desc;
    probe.hs = desc->gru_size;
    *bytes = (size_t)(ws_floats(&probe, B * T) + part_floats(&probe, B * T)) * sizeof(float);
    if (budget) *budget = (size_t)TRAIN_WS_BUDGET;
    return MDK_OK;
}

int mdk_trainer_stage_ms(mdk_trainer *tr, float *ms) {
    MDK_REQUIRE(tr && ms, MDK_ERR_ARG, "trainer_stage_ms: NULL argument");
    for (int i = 0; i < TS_N; ++i) ms[i] = tr->stage_ms[i];
    return MDK_OK;
}

}  // extern "C"
