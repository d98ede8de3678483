// The consensus quality of one position, shared by the decode entry points (decode.cu) and the engine's heads (misc.cu),
// so that qualities computed inside the forward are bit-identical to those decoded later from its probabilities.
#pragma once
#include <cstdint>

namespace mdk {

// labels.py:387-401 on float32: err = clip(1 - p, 1e-7, 1); q = min(-10 log10(err), 70), with the correctly rounded
// float32 log10
__device__ __forceinline__ float phred_f32(float p_class) {
    const float err = fminf(fmaxf(1.0f - p_class, 1e-7f), 1.0f);
    const float l = __double2float_rn(log10((double)err));
    return fminf(-10.0f * l, 70.0f);
}

// FASTQ byte of the winning class's probability: astype('u1') truncation, +33 (labels.py:1063-1085)
__device__ __forceinline__ uint8_t phred_char(float p_best) { return (uint8_t)((int)phred_f32(p_best) + 33); }

}  // namespace mdk
