// Per-element arithmetic of the fused epilogue (b200_epilogue): out = act(alpha * acc + bias), in f32 with one rounding per
// operation, for the direct grouped convolution (conv_grouped.cu).  It is the expression of the `epilogue` lambda in
// gemm_wgmma.cu, statement for statement, so both routes of a convolution apply alpha, bias, relu and gelu the same way.
// The GEMM keeps its inline copy: calling this function from it moved instructions in a convolution-backward kernel, and the
// GEMM's machine code is held fixed.  A change to one must be made to the other.  bias: f32 [ncols] or nullptr.
#pragma once
#include <cstdint>

__device__ __forceinline__ float epilogue_value(float acc, float alpha, const float* bias, uint32_t col, uint32_t ncols, uint32_t act) {
  float x = acc * alpha;
  if (bias != nullptr && col < ncols) x += __ldg(bias + col);
  if (act == 1) x = fmaxf(x, 0.f);
  else if (act == 2) x = 0.5f * x * (1.f + erff(x * 0.70710678118654752f));
  return x;
}
