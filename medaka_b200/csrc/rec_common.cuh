// Device helpers of the recurrent tensor-core kernels (gru_wg.cu; the activations also readlevel.cu): approximate
// activations, tile geometry.
#pragma once
#include "common.cuh"
#include "ptx.cuh"

namespace mdk {

// ---- activations: ex2.approx / rcp.approx only ----
__device__ __forceinline__ float ex2_approx(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float rcp_approx(float x) {
    float y;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
// ---- geometry of the recurrent kernels' shared-memory operand tiles (K-major, SWIZZLE_NONE: [k-group][row][8 halfs]) ----
constexpr int RT_N = 16;                                 // windows per tile
constexpr int GI_PREFETCH_STEPS = 3;
constexpr float EXP_CLAMP = 60.0f;

}  // namespace mdk
