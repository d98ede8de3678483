// Host-only driver of the GRU weight packer (medaka_b200/csrc/gru_pack.cuh) at gru_size 256, run by
// tests/test_gru256.py:
//   gru256_pack_check F in.bin out.bin
// in.bin: float32, per layer and direction (state-dict order) w_ih [768][in], w_hh [768][256], b_ih [768], b_hh [768],
// in = F for layer 0 and 512 for layer 1.  out.bin: per layer, the arrays of PackedLayer in declaration order, each as
// an int64 element count and its elements (float32, or fp16 bits).
#include <cstdio>
#include <cstdlib>
#include "../../medaka_b200/csrc/gru_pack.cuh"

using namespace mdk;

template <class T> static void put(FILE *f, const std::vector<T> &v) {
    const int64_t n = (int64_t)v.size();
    fwrite(&n, sizeof(n), 1, f);
    fwrite(v.data(), sizeof(T), v.size(), f);
}

int main(int argc, char **argv) {
    if (argc != 4) return 2;
    const int F = atoi(argv[1]);
    FILE *in = fopen(argv[2], "rb"), *out = fopen(argv[3], "wb");
    if (!in || !out) return 3;
    for (int l = 0; l < 2; ++l) {
        const int nin = l == 0 ? F : H2_256;
        LayerWeights lw;
        for (int d = 0; d < NDIR; ++d) {
            lw.w_ih[d].resize((size_t)G3_256 * nin);
            lw.w_hh[d].resize((size_t)G3_256 * H256);
            lw.b_ih[d].resize(G3_256);
            lw.b_hh[d].resize(G3_256);
            for (std::vector<float> *v : {&lw.w_ih[d], &lw.w_hh[d], &lw.b_ih[d], &lw.b_hh[d]})
                if (fread(v->data(), sizeof(float), v->size(), in) != v->size()) return 4;
        }
        const PackedLayer p = pack_layer(lw, nin, l, H256);
        put(out, p.w_in_packed); put(out, p.bias_gi); put(out, p.b_hn); put(out, p.bias_gi_tc); put(out, p.b_hn_tc);
        put(out, p.w_hh_t); put(out, p.w_hh_tm); put(out, p.w_x_tm); put(out, p.w_in_tc);
    }
    fclose(in);
    return fclose(out) == 0 ? 0 : 5;
}
