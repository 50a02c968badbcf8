// nanmax.cuh — the max of torch's relu and max_pool2d: NaN if either operand is NaN (PTX max.NaN).  fmaxf returns the
// other operand instead, so relu(NaN) would come out 0 and a NaN in a pooling window would be dropped.  For non-NaN
// operands max.NaN gives the same bits as fmaxf (it is the same FMNMX instruction, signed zeros included).
#pragma once

namespace mcb {

__device__ __forceinline__ float max_nan(float a, float b) {
  float r;
  asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}

__device__ __forceinline__ float relu_nan(float v) { return max_nan(v, 0.f); }

// torch's relu backward zeroes the gradient where y <= 0, so a NaN y passes it.  hi16 holds a bf16 in its upper half
// (the lower half is ignored): compared as the fp32 value it is, with no conversion
__device__ __forceinline__ bool bf16_le0(uint32_t hi16) { return __uint_as_float(hi16 & 0xFFFF0000u) <= 0.f; }

}  // namespace mcb
