// The fp8 KV-cache encoder shared by attention_kv.cu (attn_kv_write_fp8, b200_kvcache_write_fp8) and rope.cu
// (b200_rope_kvcache_write), so both write the same cache bytes for the same 16-bit values.
// include after <cuda_bf16.h> and <cuda_fp16.h>.
#pragma once
#include <cstdint>

// One 16-bit value -> f32, exactly.
__device__ __forceinline__ float kv_in_f32(uint32_t h, bool bf16) {
  return bf16 ? __uint_as_float(h << 16) : __half2float(__ushort_as_half(static_cast<unsigned short>(h)));
}

// Eight 16-bit values (16 bytes) -> eight fp8 bytes: sat_rn(x / s) per value (f32 division rounded to nearest, then RNE to
// the cache format with satfinite: +-448 (e4m3) or +-57344 (e5m2) for larger magnitudes, NaN stays NaN).
__device__ __forceinline__ uint2 kv_quant8(uint4 x, float s, bool bf16, bool e5m2) {
  const uint32_t w[4] = {x.x, x.y, x.z, x.w};
  uint32_t q[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float lo = __fdiv_rn(kv_in_f32(w[i] & 0xFFFFu, bf16), s), hi = __fdiv_rn(kv_in_f32(w[i] >> 16, bf16), s);
    unsigned short r;
    if (e5m2) asm("cvt.rn.satfinite.e5m2x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
    else asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
    q[i] = r;
  }
  return make_uint2(q[0] | (q[1] << 16), q[2] | (q[3] << 16));
}
