// NaN-preserving clamp and max, with torch's semantics: torch.clamp(NaN, lo, hi) and NaN.clamp_(min=m) are NaN, whereas
// fminf / fmaxf return the other operand and turn a NaN into a bound.  One FMNMX.NAN instruction each, the cost of the
// plain fminf / fmaxf; for non-NaN operands the results are the same.
#pragma once

namespace mi {

__device__ __forceinline__ float fmax_nan(float a, float b) {
    float r;
    asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
    return r;
}
__device__ __forceinline__ float fmin_nan(float a, float b) {
    float r;
    asm("min.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
    return r;
}
// clamp(v, lo, hi) for lo <= hi: NaN in, NaN out
__device__ __forceinline__ float clamp_nan(float v, float lo, float hi) { return fmin_nan(fmax_nan(v, lo), hi); }

}  // namespace mi
