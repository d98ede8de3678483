// What the read-level engine (readlevel.cu) and the read-level trainer (rl_train.cu) share: the network's sizes, the
// convolutions' parameter blocks and launchers of the engine's fp32 kernels, which the trainer's validation forward
// runs unchanged so that its probabilities equal the engine's fp32 path bit for bit.
#pragma once
#include "common.cuh"

namespace mdk {

constexpr int RL_C = 128;        // cnn_size
constexpr int RL_H = 128;        // lstm_size
constexpr int RL_H3 = 384;       // lstm_size of every released read-level model
constexpr int RL_EMB = 6;        // bases_embedding_size
constexpr int RL_TAPS = 17;
constexpr int RL_PAD = 8;

struct RlConv1 {
    const float *emb_base;      // [6][6]
    const float *emb_strand;    // [3][6]
    const float *w;             // [C][in]   in = 7 (+1 dwell)
    const float *b;             // [C]
    const float *bn_mean, *bn_invstd, *bn_w, *bn_b;   // [C]
};

struct RlConv17 {
    const float *w_t;           // [17][C in][C out]  (transposed from torch's [out][in][tap])
    const float *b;             // [C]
    const float *bn_mean, *bn_invstd, *bn_w, *bn_b;
};

// mask [B][D] of the non-empty (window, read) rows of x int8 [B][P][D][F]
cudaError_t rl_launch_mask(const int8_t *x, int64_t B, int64_t P, int D, int F, uint8_t *mask, cudaStream_t s);
// The fp32 convolution path of B windows into z [B][P][H]: embedding + k = 1 convolution + BN1 (y1 [B][D][P][C]),
// k = 17 convolution + BN2 pooled in groups of 4 reads (part [B][groups][P][C]), mean and Linear(C -> H) (pool_w_t
// [C][H]).  Inference BatchNorm; mask from rl_launch_mask.
cudaError_t rl_launch_conv_fp32(const int8_t *x, const uint8_t *mask, const RlConv1 &c1, const RlConv17 &c17,
                                const float *pool_w_t, const float *pool_b, int64_t B, int64_t P, int D, int F,
                                int use_dwells, int H, float *y1, float *part, float *z, cudaStream_t s);
// the fp32 LSTM recurrence of one layer, both directions (gi [B*P][2][4H] with b_ih + b_hh, w_t [2][H][4H] W_hh^T,
// out [B*P][2H]); with save, also the gates i, f, g, o and the cell c per position: save [B*P][2][5H]
cudaError_t rl_launch_lstm_fp32(const float *gi, const float *w_t, float *out, int64_t B, int64_t P, int H,
                                cudaStream_t s, float *save = nullptr);
// the engine's head: probabilities [n][5] of h1 [n][2H] (logits too at H = 128, where the head kernel writes them)
cudaError_t rl_launch_head(const float *h1, const float *lin_w, const float *lin_b, int64_t n, int H, float *probs,
                           float *logits, cudaStream_t s);

}  // namespace mdk
