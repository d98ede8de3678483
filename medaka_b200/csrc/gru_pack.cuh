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
// multiplies and adds: built without -march, g++ has no FMA to contract them into.
inline PackedLayer pack_layer(const LayerWeights &lw, int in, int layer) {
    PackedLayer p;
    p.w_in_packed.resize((size_t)GI_COLS * in);
    p.bias_gi.resize(GI_COLS);
    p.bias_gi_tc.resize(GI_COLS);
    p.b_hn.resize(NDIR * H);
    p.b_hn_tc.resize(NDIR * H);
    p.w_hh_t.resize((size_t)NDIR * H * G3);
    p.w_hh_tm.resize((size_t)NDIR * 2 * G3 * H);
    if (layer == 0 && in <= 16) p.w_x_tm.resize((size_t)NDIR * 2 * G3 * 16);
    if (layer == 1) p.w_in_tc.resize((size_t)2 * GI_COLS * H2);
    __half hi, lo;
    for (int d = 0; d < NDIR; ++d) {
        const float *w_ih = lw.w_ih[d].data(), *w_hh = lw.w_hh[d].data(), *b_ih = lw.b_ih[d].data(), *b_hh = lw.b_hh[d].data();
        // input weights of both directions stacked: [768][in]
        std::copy(w_ih, w_ih + (size_t)G3 * in, p.w_in_packed.begin() + (size_t)d * G3 * in);
        for (int r = 0; r < G3; ++r) {
            float &b = p.bias_gi[d * G3 + r];
            b = r < 2 * H ? b_ih[r] + b_hh[r] : b_ih[r];
            p.bias_gi_tc[d * G3 + r] = b * gate_scale(r / H);
        }
        for (int j = 0; j < H; ++j) {
            p.b_hn[d * H + j] = b_hh[2 * H + j];
            p.b_hn_tc[d * H + j] = b_hh[2 * H + j] * GATE_SCALE_N;
        }
        // recurrent weights, transposed fp32 [d][k][384] and fp16 hi/lo blocks [d][part][gate][row j][k]
        for (int c = 0; c < G3; ++c) {
            const int g = c / H, j = c % H;
            for (int k = 0; k < H; ++k) {
                const float v = w_hh[c * H + k];
                p.w_hh_t[((size_t)d * H + k) * G3 + c] = v;
                split_f16(v * gate_scale(g), hi, lo);
                p.w_hh_tm[(((size_t)d * 2 + 0) * 3 + g) * H * H + j * H + k] = hi;
                p.w_hh_tm[(((size_t)d * 2 + 1) * 3 + g) * H * H + j * H + k] = lo;
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
            for (int r = 0; r < G3; ++r) {
                const int blk = d * 3 + r / H, j = r % H;
                for (int k = 0; k < H2; ++k) {
                    split_f16(w_ih[r * H2 + k] * gate_scale(r / H), hi, lo);
                    p.w_in_tc[((size_t)blk * 2 + 0) * H * H2 + j * H2 + k] = hi;
                    p.w_in_tc[((size_t)blk * 2 + 1) * H * H2 + j * H2 + k] = lo;
                }
            }
        }
    }
    return p;
}

}  // namespace mdk
