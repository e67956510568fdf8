// Device helpers shared by the attention forward (attention.cu) and backward (attention_bwd.cu) kernels.
#pragma once
#include <cstdint>

namespace b200 {

enum : int { KIND_F16 = 0, KIND_BF16 = 1 };
enum : int { OUT_F16 = 0, OUT_BF16 = 1, OUT_F32 = 2 };

__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// two f32 -> one register of two 16-bit values, lo in the low half (RNE)
template <int KIND>
__device__ __forceinline__ uint32_t pack16(float lo, float hi) {
  uint32_t r;
  if constexpr (KIND == KIND_BF16) asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  else asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}

}  // namespace b200
