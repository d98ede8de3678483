// The consensus quality of one position, shared by the decode entry points (decode.cu) and the engine's heads (misc.cu),
// so that qualities computed inside the forward are bit-identical to those decoded later from its probabilities.
// Likewise the variant call byte of one position (mdk_engine_submit_variant_decoded), which the heads write and the
// device join / decode (mdk_variant_join_cuts, mdk_decode_variants_dev) read.
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

// Reference byte of a column (input of a variant-decoded forward): the draft's label code in the low 3 bits (0..4 =
// '*ACGT', 0 on insertion columns; 5 = 'N'; 6 = any other symbol) and VCALL_INS on insertion columns (minor != 0).
// Call byte (output): the argmax label in the low 3 bits, VCALL_MISM when it differs from the reference code, and the
// reference byte's VCALL_INS.
constexpr uint8_t VCALL_LABEL = 0x07, VCALL_MISM = 0x40, VCALL_INS = 0x80;

__device__ __forceinline__ uint8_t variant_call(int label, uint8_t ref) {
    const int code = ref & VCALL_LABEL;
    return (uint8_t)(label | (label != code ? VCALL_MISM : 0) | (ref & VCALL_INS));
}

// the class whose probability scores the reference (labels.py:949-952): its code, 'N' and other symbols as '*'
__device__ __forceinline__ int ref_class(uint8_t ref) {
    const int code = ref & VCALL_LABEL;
    return code < 5 ? code : 0;
}

}  // namespace mdk
