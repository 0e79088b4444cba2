// Constants shared by the network kernels.
#pragma once
#include "common.cuh"

namespace scsfm {
constexpr int PADMODE_ZERO = SCSFM_PADMODE_ZERO;
constexpr int PADMODE_REFLECT = SCSFM_PADMODE_REFLECT;
constexpr int ACT_NONE = SCSFM_ACT_NONE;
constexpr int ACT_RELU = SCSFM_ACT_RELU;
constexpr int ACT_ELU = SCSFM_ACT_ELU;
constexpr int ACT_DISP = SCSFM_ACT_DISP;
constexpr int ROUND_TF32 = SCSFM_ROUND_TF32;

__device__ __forceinline__ float tf32_round(float x) {
    uint32_t u;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
    return __uint_as_float(u);
}
__device__ __forceinline__ float maybe_round(float x, bool on) { return on ? tf32_round(x) : x; }
// what kind::tf32 reads of an fp32 operand: the upper 19 bits (sign, exponent, 10 mantissa bits)
__device__ __forceinline__ float tf32_trunc(float x) { return __uint_as_float(__float_as_uint(x) & 0xFFFFE000u); }
// low part of the split-accumulate operands: x = trunc(x) + (x - trunc(x)) exactly; the remainder has <= 13 significant
// bits and is itself rounded to TF32 (residual <= 2^-21 |x|)
__device__ __forceinline__ float tf32_lo(float x) { return tf32_round(x - tf32_trunc(x)); }
// SCSFM_OPERAND_*: 0 = rounded TF32, 1 = raw bits, 2 = low part
__device__ __forceinline__ float tc_operand(float x, int kind) { return kind == 0 ? tf32_round(x) : (kind == 1 ? x : tf32_lo(x)); }

// SCSFM_ACT_* in the low byte of act
__device__ __forceinline__ float apply_act(float v, int act) {
    switch (act & 0xff) {
        case ACT_RELU: return fmaxf(v, 0.f);
        case ACT_ELU: return v > 0.f ? v : expm1f(v);
        case ACT_DISP: return 10.0f * (1.0f / (1.0f + expf(-v))) + 0.01f;   // alpha*sigmoid+beta, DispResNet.py:98
        default: return v;
    }
}
}  // namespace scsfm
