// Weight packing of the consensus (GRU) engine: the arrays the kernels read (LayerWeights' device arrays), built on the
// host from one layer's weights as loaded.  Host code only, so tests/test_gru_pack.py checks every layout on the CPU.
#pragma once
#include <algorithm>
#include <vector>

#include "common.cuh"
#include "ptx.cuh"

namespace mdk {

// Host images of LayerWeights' device arrays, same names and layouts.  w_x_tm is empty unless layer 0 has in <= 16,
// w_in_tc unless layer 1.
struct PackedLayer {
    std::vector<float> w_in_packed, bias_gi, b_hn, bias_gi_tc, b_hn_tc, w_hh_t;
    std::vector<__half> w_hh_tm, w_x_tm, w_in_tc;
};

// The tensor-core copies are x = w * gate_scale(gate), hi = fp16(x), lo = fp16(x - hi) (split_f16), with separate
// multiplies and adds: built without -march, g++ has no FMA to contract them into.  hs is the GRU width (H or H256); the
// layouts below are written for hs = H and hold with hs in its place (768 -> 6 hs, 128 -> hs, 256 -> 2 hs).  At H256
// the kernels of gru256.cu read w_hh_tm ([d][part][gate][j][k], per cluster rank the rows of its 64 units) and w_in_tc
// ([blk][part][j][k 512], streamed in 128-row slices); w_x_tm is never built.
inline PackedLayer pack_layer(const LayerWeights &lw, int in, int layer, int hs = H) {
    const int g3 = 3 * hs, gi_cols = NDIR * g3, h2 = NDIR * hs;
    PackedLayer p;
    p.w_in_packed.resize((size_t)gi_cols * in);
    p.bias_gi.resize(gi_cols);
    p.bias_gi_tc.resize(gi_cols);
    p.b_hn.resize(NDIR * hs);
    p.b_hn_tc.resize(NDIR * hs);
    p.w_hh_t.resize((size_t)NDIR * hs * g3);
    p.w_hh_tm.resize((size_t)NDIR * 2 * g3 * hs);
    if (layer == 0 && in <= 16 && hs == H) p.w_x_tm.resize((size_t)NDIR * 2 * G3 * 16);
    if (layer == 1) p.w_in_tc.resize((size_t)2 * gi_cols * h2);
    __half hi, lo;
    for (int d = 0; d < NDIR; ++d) {
        const float *w_ih = lw.w_ih[d].data(), *w_hh = lw.w_hh[d].data(), *b_ih = lw.b_ih[d].data(), *b_hh = lw.b_hh[d].data();
        // input weights of both directions stacked: [768][in]
        std::copy(w_ih, w_ih + (size_t)g3 * in, p.w_in_packed.begin() + (size_t)d * g3 * in);
        for (int r = 0; r < g3; ++r) {
            float &b = p.bias_gi[d * g3 + r];
            b = r < 2 * hs ? b_ih[r] + b_hh[r] : b_ih[r];
            p.bias_gi_tc[d * g3 + r] = b * gate_scale(r / hs);
        }
        for (int j = 0; j < hs; ++j) {
            p.b_hn[d * hs + j] = b_hh[2 * hs + j];
            p.b_hn_tc[d * hs + j] = b_hh[2 * hs + j] * GATE_SCALE_N;
        }
        // recurrent weights, transposed fp32 [d][k][384] and fp16 hi/lo blocks [d][part][gate][row j][k]
        for (int c = 0; c < g3; ++c) {
            const int g = c / hs, j = c % hs;
            for (int k = 0; k < hs; ++k) {
                const float v = w_hh[c * hs + k];
                p.w_hh_t[((size_t)d * hs + k) * g3 + c] = v;
                split_f16(v * gate_scale(g), hi, lo);
                p.w_hh_tm[(((size_t)d * 2 + 0) * 3 + g) * hs * hs + j * hs + k] = hi;
                p.w_hh_tm[(((size_t)d * 2 + 1) * 3 + g) * hs * hs + j * hs + k] = lo;
            }
        }
        if (!p.w_x_tm.empty()) {   // [d][part][gate][row j][16], K zero-padded
            for (int c = 0; c < G3; ++c) {
                const int g = c / H, j = c % H;
                for (int k = 0; k < 16; ++k) {
                    const float v = k < in ? w_ih[c * in + k] : 0.f;
                    split_f16(v * gate_scale(g), hi, lo);
                    p.w_x_tm[((((size_t)d * 2 + 0) * 3 + g) * H + j) * 16 + k] = hi;
                    p.w_x_tm[((((size_t)d * 2 + 1) * 3 + g) * H + j) * 16 + k] = lo;
                }
            }
        }
        if (!p.w_in_tc.empty()) {  // [blk = dir*3 + gate][part][row j][k 256]
            for (int r = 0; r < g3; ++r) {
                const int blk = d * 3 + r / hs, j = r % hs;
                for (int k = 0; k < h2; ++k) {
                    split_f16(w_ih[r * h2 + k] * gate_scale(r / hs), hi, lo);
                    p.w_in_tc[((size_t)blk * 2 + 0) * hs * h2 + j * h2 + k] = hi;
                    p.w_in_tc[((size_t)blk * 2 + 1) * hs * h2 + j * h2 + k] = lo;
                }
            }
        }
    }
    return p;
}

}  // namespace mdk
