// The scale rule and the encode of b200_quantize (quant.cu), shared with the kernels that write quantized outputs themselves
// (norm.cu: b200_norm_quantized_fp8), so a fused store gives the same codes and scales bit for bit.  Device code only;
// include after <cuda_fp16.h> and kernel_params.h.
#pragma once
#include <cstdint>

// ------------------------------------------------------------------------------------------------ value types
__device__ __forceinline__ uint32_t qv_bits(uint32_t v) {
  return (v == B200_QV_Q4F || v == B200_QV_Q4S || v == B200_QV_E2M1) ? 4u : (v == B200_QV_Q2F || v == B200_QV_Q2S) ? 2u : 8u;
}
// QuantValue::range() (scheme.rs:399-411)
__device__ __forceinline__ float qv_lo(uint32_t v) {
  switch (v) {
    case B200_QV_Q8F: return -128.f;
    case B200_QV_Q4F: return -8.f;
    case B200_QV_Q2F: return -2.f;
    case B200_QV_Q8S: return -127.f;
    case B200_QV_Q4S: return -7.f;
    case B200_QV_Q2S: return -1.f;
    case B200_QV_E4M3: return -448.f;
    case B200_QV_E5M2: return -57344.f;
    default: return -6.f;
  }
}
__device__ __forceinline__ float qv_hi(uint32_t v) {
  switch (v) {
    case B200_QV_Q8F: case B200_QV_Q8S: return 127.f;
    case B200_QV_Q4F: case B200_QV_Q4S: return 7.f;
    case B200_QV_Q2F: case B200_QV_Q2S: return 1.f;
    case B200_QV_E4M3: return 448.f;
    case B200_QV_E5M2: return 57344.f;
    default: return 6.f;
  }
}

// ------------------------------------------------------------------------------------------------ scale storage policy
// ScaleDtype::max_representable (scheme.rs:208-218)
__device__ __forceinline__ float scale_max(uint32_t dt) {
  switch (dt) {
    case B200_F16: return 65504.f;
    case B200_BF16: return __uint_as_float(0x7F7F0000u);
    case B200_UE8M0: return __uint_as_float(0x7F000000u);   // 2^127
    case B200_F8E4M3: return 448.f;
    default: return __uint_as_float(0x7F7FFFFFu);
  }
}

// UE8M0: the smallest power of two not below s, clamped to codes 0..254 (2^-127 .. 2^127).
__device__ __forceinline__ uint32_t ue8m0_code(float s) {
  const uint32_t b = __float_as_uint(s);
  const uint32_t e = b >> 23, m = b & 0x7FFFFFu;
  if (e == 0) return m > 0x400000u ? 1u : 0u;   // zero and f32 subnormals: 2^-127 is m = 0x400000
  const uint32_t c = e + (m != 0);
  return c > 254u ? 254u : c;
}
__device__ __forceinline__ float ue8m0_value(uint32_t c) {
  return c == 255u ? __uint_as_float(0x7FC00000u) : c == 0u ? __uint_as_float(0x00400000u) : __uint_as_float(c << 23);
}

// ScaleDtype::round_up (scheme.rs:235-270) / round_up_to_dtype (cubecl-std/src/quant/round.rs), bit for bit; UE8M0 above.
__device__ __forceinline__ float round_up_scale(float s, uint32_t dt) {
  if (dt == B200_F32) return s;
  if (dt == B200_UE8M0) return ue8m0_value(ue8m0_code(s));
  if (s != s) return s;
  const float mx = scale_max(dt);
  if (s >= mx) return mx;
  if (dt == B200_F16 && s < 6.103515625e-05f) return ceilf(s / 5.9604644775390625e-08f) * 5.9604644775390625e-08f;
  if (dt == B200_F8E4M3 && s < 0.015625f) return ceilf(s / 0.001953125f) * 0.001953125f;
  const uint32_t step = dt == B200_F16 ? (1u << 13) : dt == B200_BF16 ? (1u << 16) : (1u << 20);
  return __uint_as_float((__float_as_uint(s) + (step - 1)) & ~(step - 1));
}

__device__ __forceinline__ uint32_t f32_to_e4m3(float f) {
  unsigned short r;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(0.f), "f"(f));
  return r & 0xFFu;
}
__device__ __forceinline__ uint32_t f32_to_e5m2(float f) {
  unsigned short r;
  asm("cvt.rn.satfinite.e5m2x2.f32 %0, %1, %2;" : "=h"(r) : "f"(0.f), "f"(f));
  return r & 0xFFu;
}

// The stored bits of a scale already on the dtype's grid (round_up_scale's result): every conversion here is exact.
__device__ __forceinline__ uint32_t scale_bits(float s, uint32_t dt) {
  switch (dt) {
    case B200_F16: return __half_as_ushort(__float2half_rn(s));
    case B200_BF16: return __float_as_uint(s) >> 16;
    case B200_F8E4M3: return f32_to_e4m3(s) & 0x7Fu;
    case B200_UE8M0: return ue8m0_code(s);
    default: return __float_as_uint(s);
  }
}

// q = x / eff, then: integers RNE and clamp to range(); fp8 RNE with satfinite; e2m1 RNE (ties to the even code) saturating
// at +-6.  A zero scale gives code 0; NaN gives 0 (integers, e2m1) or 0x7F (fp8); +-inf saturates to the range end.
// `rcp` is 1 / eff when eff is a power of two whose reciprocal is an f32 (pow2): x * rcp is then the same correctly rounded
// value as x / eff, bit for bit, at a fraction of the cost.  Any other scale divides.
__device__ __forceinline__ uint32_t encode_one(float x, float eff, float rcp, bool pow2, uint32_t v, float lo, float hi) {
  if (eff == 0.f) return 0u;
  const float q = pow2 ? x * rcp : x / eff;
  if (v == B200_QV_E4M3 || v == B200_QV_E5M2) {
    if (q != q) return 0x7Fu;
    return v == B200_QV_E4M3 ? f32_to_e4m3(q) : f32_to_e5m2(q);
  }
  if (v == B200_QV_E2M1) {
    if (q != q) return 0u;
    const float a = fabsf(q);
    const uint32_t c = a <= 0.25f ? 0u : a < 0.75f ? 1u : a <= 1.25f ? 2u : a < 1.75f ? 3u
                     : a <= 2.5f ? 4u : a < 3.5f ? 5u : a <= 5.f ? 6u : 7u;
    return c | ((__float_as_uint(q) >> 28) & 8u);
  }
  if (q != q) return 0u;
  const float r = fminf(fmaxf(rintf(q), lo), hi);
  return static_cast<uint32_t>(static_cast<int32_t>(r));
}

// |f| as bits for a finite f, 0 for NaN and inf (the block absmax only sees finite values)
__device__ __forceinline__ uint32_t finite_abs_bits(float f) {
  const float a = fabsf(f);
  return a < INFINITY ? __float_as_uint(a) : 0u;   // NaN and inf excluded
}
