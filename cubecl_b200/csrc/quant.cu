// Hand-written sm_90a quantize / dequantize along the innermost axis under CubeCL's quantization schemes
// (crates/cubecl-common/src/quant/scheme.rs: QuantValue, per-tensor / per-block / two-level scales, ScaleDtype).
// HBM-bound: 128-bit loads of the input (or of the codes), one pass per level of scales.
//
//   quant_absmax_<in>   finite-only |x| max of the whole tensor (schemes with a tensor level), one u32 atomicMax per block
//                       on the bit pattern of a non-negative float into a pooled word: exact and order-independent.
//   quant_encode_<in>   a block of B values is owned by G = B / VEC lanes, each holding one 128-bit vector; the block absmax
//                       is a shfl_xor max inside the group, every lane encodes its slice and stores its codes in one store,
//                       the group leader stores the block scale.  A per-tensor scheme runs the same kernel on fixed chunks.
//   quant_decode_<out>  16 bytes of codes per thread, outputs leave as 128-bit stores.
//
// The value type and the scale dtype are uniform runtime parameters.  All arithmetic is IEEE f32 (no fast-math, denormals
// kept).  q = x / eff divides with `/`, except where eff is a power of two whose reciprocal is an f32: there the encode
// multiplies by that exact reciprocal, which rounds the same real value x * 2^-e once and so gives the quotient's bits
// (encode_one).  The numpy oracle in tests/quant_oracle.py, which always divides, reproduces every code and scale bit for bit.
//
// Codes are one compact row-major bit stream: field i of a row sits at bit offset i * bits, from the low bits upward (two
// e2m1 per byte with element 2i in the low nibble).  Read as little-endian u32 words this is the reference's PackedU32(0)
// stream; it is also its Native / PackedNative(0) stream.
// Compiled to a cubin: nvcc -cubin -gencode arch=compute_90a,code=sm_90a
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cstdint>

#include "kernel_params.h"

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
__device__ __forceinline__ float e4m3_to_f32(uint32_t b) {
  uint32_t h;
  asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(h) : "h"(static_cast<unsigned short>(b & 0xFFu)));
  return __half2float(__ushort_as_half(static_cast<unsigned short>(h & 0xFFFFu)));
}
__device__ __forceinline__ float e5m2_to_f32(uint32_t b) {
  uint32_t h;
  asm("cvt.rn.f16x2.e5m2x2 %0, %1;" : "=r"(h) : "h"(static_cast<unsigned short>(b & 0xFFu)));
  return __half2float(__ushort_as_half(static_cast<unsigned short>(h & 0xFFFFu)));
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
// A stored block scale read back as f32; e4m3 scales are read with the sign ignored, as b200_matmul_scaled reads them.
__device__ __forceinline__ float load_scale(uint64_t base, uint64_t i, uint32_t dt) {
  switch (dt) {
    case B200_F16: return __half2float(__ushort_as_half(__ldg(reinterpret_cast<const unsigned short*>(base) + i)));
    case B200_BF16: return __uint_as_float(static_cast<uint32_t>(__ldg(reinterpret_cast<const unsigned short*>(base) + i)) << 16);
    case B200_F8E4M3: return e4m3_to_f32(__ldg(reinterpret_cast<const unsigned char*>(base) + i) & 0x7Fu);
    case B200_UE8M0: return ue8m0_value(__ldg(reinterpret_cast<const unsigned char*>(base) + i));
    default: return __ldg(reinterpret_cast<const float*>(base) + i);
  }
}

// ------------------------------------------------------------------------------------------------ codes
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

__device__ __forceinline__ float decode_one(uint32_t field, uint32_t v, uint32_t bits) {
  switch (v) {
    case B200_QV_E4M3: return e4m3_to_f32(field);
    case B200_QV_E5M2: return e5m2_to_f32(field);
    case B200_QV_E2M1: {
      const float m = (field & 4u) ? ((field & 2u) ? ((field & 1u) ? 6.f : 4.f) : ((field & 1u) ? 3.f : 2.f))
                                   : ((field & 2u) ? ((field & 1u) ? 1.5f : 1.f) : ((field & 1u) ? 0.5f : 0.f));
      return (field & 8u) ? -m : m;
    }
    default: {   // sign extension of an n-bit field, cast_masked_plain (dequantize.rs:177-202)
      const uint32_t sb = 1u << (bits - 1);
      return static_cast<float>(static_cast<int32_t>(field ^ sb) - static_cast<int32_t>(sb));
    }
  }
}

// ------------------------------------------------------------------------------------------------ input chunks
template <int DT>
struct In;
template <>
struct In<B200_F32> {
  static constexpr int VEC = 4;
  static __device__ __forceinline__ float get(uint64_t base, uint64_t i) { return __ldg(reinterpret_cast<const float*>(base) + i); }
  static __device__ __forceinline__ void unpack(uint4 r, float (&f)[VEC]) {
    f[0] = __uint_as_float(r.x); f[1] = __uint_as_float(r.y); f[2] = __uint_as_float(r.z); f[3] = __uint_as_float(r.w);
  }
};
template <>
struct In<B200_F16> {
  static constexpr int VEC = 8;
  static __device__ __forceinline__ float get(uint64_t base, uint64_t i) {
    return __half2float(__ushort_as_half(__ldg(reinterpret_cast<const unsigned short*>(base) + i)));
  }
  static __device__ __forceinline__ void unpack(uint4 r, float (&f)[VEC]) {
    const uint32_t w[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      f[2 * j] = __half2float(__ushort_as_half(static_cast<unsigned short>(w[j] & 0xFFFFu)));
      f[2 * j + 1] = __half2float(__ushort_as_half(static_cast<unsigned short>(w[j] >> 16)));
    }
  }
};
template <>
struct In<B200_BF16> {
  static constexpr int VEC = 8;
  static __device__ __forceinline__ float get(uint64_t base, uint64_t i) {
    return __uint_as_float(static_cast<uint32_t>(__ldg(reinterpret_cast<const unsigned short*>(base) + i)) << 16);
  }
  static __device__ __forceinline__ void unpack(uint4 r, float (&f)[VEC]) {
    const uint32_t w[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      f[2 * j] = __uint_as_float(w[j] << 16);
      f[2 * j + 1] = __uint_as_float(w[j] & 0xFFFF0000u);
    }
  }
};

__device__ __forceinline__ uint4 ldg_stream_u4(uint64_t p) {
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
  return v;
}

// Chunk `idx` of the [rows, K] view: VEC consecutive elements of one row (fewer at a row end; the rest read as 0).  `f` is
// the chunk's position in the compact row-major order.  Compact rows (pitch == K: one row, or K a multiple of VEC) need
// no division.
template <int DT>
__device__ __forceinline__ uint32_t load_chunk(const QuantParams& p, uint64_t cpr, uint64_t idx, uint64_t& f,
                                               float (&x)[In<DT>::VEC]) {
  constexpr int VEC = In<DT>::VEC;
  uint64_t e, left;
  if (p.pitch == p.K) {
    f = e = idx * VEC;
    left = p.rows * p.K - f;
  } else {
    const uint64_t r = idx / cpr, k0 = (idx - r * cpr) * VEC;
    e = r * p.pitch + k0;
    f = r * p.K + k0;
    left = p.K - k0;
  }
  const uint32_t n = static_cast<uint32_t>(left < VEC ? left : VEC);
  if (n == VEC) {
    In<DT>::unpack(ldg_stream_u4(p.in + e * (DT == B200_F32 ? 4 : 2)), x);
  } else {
#pragma unroll
    for (int j = 0; j < VEC; ++j) x[j] = j < static_cast<int>(n) ? In<DT>::get(p.in, e + j) : 0.f;
  }
  return n;
}

__device__ __forceinline__ uint32_t finite_abs_bits(float f) {
  const float a = fabsf(f);
  return a < INFINITY ? __float_as_uint(a) : 0u;   // NaN and inf excluded
}

// ------------------------------------------------------------------------------------------------ absmax pass
template <int DT>
__device__ __forceinline__ void absmax_body(const QuantParams& p) {
  constexpr int VEC = In<DT>::VEC;
  constexpr int U = 4;   // chunks in flight per thread
  const uint64_t cpr = (p.K + VEC - 1) / VEC, chunks = p.rows * cpr;
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  uint32_t m = 0;
  for (uint64_t base = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; base < chunks; base += U * stride) {
    float x[U][VEC];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const uint64_t idx = base + u * stride;
      uint64_t f;
      if (idx < chunks) {
        load_chunk<DT>(p, cpr, idx, f, x[u]);
      } else {
#pragma unroll
        for (int j = 0; j < VEC; ++j) x[u][j] = 0.f;
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u)
#pragma unroll
      for (int j = 0; j < VEC; ++j) m = max(m, finite_abs_bits(x[u][j]));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xFFFFFFFFu, m, o));
  __shared__ uint32_t s_m[32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) s_m[warp] = m;
  __syncthreads();
  if (warp == 0) {
    m = lane < static_cast<int>(blockDim.x >> 5) ? s_m[lane] : 0u;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xFFFFFFFFu, m, o));
    if (lane == 0 && m) atomicMax(reinterpret_cast<unsigned int*>(p.amax), m);
  }
}

// ------------------------------------------------------------------------------------------------ encode pass
__device__ __forceinline__ void store_codes(uint64_t addr, uint64_t packed, uint32_t bytes, uint32_t full_bytes) {
  if (bytes == full_bytes && (addr & (full_bytes - 1)) == 0) {
    switch (full_bytes) {
      case 8: *reinterpret_cast<uint64_t*>(addr) = packed; return;
      case 4: *reinterpret_cast<uint32_t*>(addr) = static_cast<uint32_t>(packed); return;
      case 2: *reinterpret_cast<unsigned short*>(addr) = static_cast<unsigned short>(packed); return;
      default: *reinterpret_cast<unsigned char*>(addr) = static_cast<unsigned char>(packed); return;
    }
  }
  for (uint32_t b = 0; b < bytes; ++b) reinterpret_cast<unsigned char*>(addr)[b] = static_cast<unsigned char>(packed >> (8 * b));
}

// Encode one loaded chunk: block scale (group max), codes, stores.
template <int DT>
__device__ __forceinline__ void encode_chunk(const QuantParams& p, const float (&x)[In<DT>::VEC], uint64_t f, uint32_t n,
                                             float tensor, uint32_t v, uint32_t bits, float lo, float hi) {
  constexpr int VEC = In<DT>::VEC;
  float eff = tensor;
  if (p.block) {
    uint32_t m = 0;
#pragma unroll
    for (int j = 0; j < VEC; ++j) m = max(m, finite_abs_bits(x[j]));
    const uint32_t G = p.block / VEC, lane = threadIdx.x & 31;
    const uint32_t gmask = G >= 32 ? 0xFFFFFFFFu : (((1u << G) - 1u) << (lane & ~(G - 1)));
    for (uint32_t o = 1; o < G; o <<= 1) m = max(m, __shfl_xor_sync(gmask, m, o));
    const float amax_b = __uint_as_float(m);
    float s = 0.f;
    if (amax_b != 0.f) s = round_up_scale(p.amax ? (amax_b / hi) / tensor : amax_b / hi, p.scale_dt);
    eff = p.amax ? tensor * s : s;
    if ((f & (p.block - 1)) == 0) {
      const uint64_t si = f >> p.block_log2;
      const uint32_t sbits = scale_bits(s, p.scale_dt);
      switch (p.scale_dt) {
        case B200_F32: reinterpret_cast<uint32_t*>(p.block_scales)[si] = sbits; break;
        case B200_F16: case B200_BF16: reinterpret_cast<unsigned short*>(p.block_scales)[si] = static_cast<unsigned short>(sbits); break;
        default: reinterpret_cast<unsigned char*>(p.block_scales)[si] = static_cast<unsigned char>(sbits); break;
      }
    }
  }
  const uint32_t eb = __float_as_uint(eff);
  const bool pow2 = ((eb & 0x7FFFFFu) == 0 && eb >= 0x00800000u && eb < 0x7F800000u) || eb == 0x00400000u;
  const float rcp = pow2 ? 1.f / eff : 0.f;
  const uint32_t mask = (1u << bits) - 1u;
  uint64_t packed = 0;
#pragma unroll
  for (int j = 0; j < VEC; ++j) packed |= static_cast<uint64_t>(encode_one(x[j], eff, rcp, pow2, v, lo, hi) & mask) << (j * bits);
  const uint64_t bit0 = f * bits;   // a multiple of 8: VEC * bits and K * bits are
  store_codes(p.values + (bit0 >> 3), packed, n * bits / 8, VEC * bits / 8);
}

template <int DT>
__device__ __forceinline__ void encode_body(const QuantParams& p) {
  constexpr int VEC = In<DT>::VEC;
  const uint32_t v = p.value, bits = qv_bits(v);
  const float lo = qv_lo(v), hi = qv_hi(v);
  // tensor level: one f32 per tensor (the only level), or the global scale over the blocks
  float tensor = 0.f;
  if (p.amax) {
    const float amax_t = __uint_as_float(*reinterpret_cast<const volatile uint32_t*>(p.amax));
    tensor = amax_t / hi;
    if (p.block) tensor = tensor / scale_max(p.scale_dt);
    if (blockIdx.x == 0 && threadIdx.x == 0) *reinterpret_cast<float*>(p.tensor_scale) = tensor;
  }
  const uint64_t cpr = (p.K + VEC - 1) / VEC, chunks = p.rows * cpr;
  const uint64_t idx = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  // block schemes: chunks is a multiple of the group size, so a group is either wholly in range or wholly out
  if (idx >= chunks) return;
  float x[VEC];
  uint64_t f;
  const uint32_t n = load_chunk<DT>(p, cpr, idx, f, x);
  encode_chunk<DT>(p, x, f, n, tensor, v, bits, lo, hi);
}

// ------------------------------------------------------------------------------------------------ decode pass
template <int ODT>
__device__ __forceinline__ void store8(uint64_t out, uint64_t i, const float (&y)[8], uint32_t valid, bool vec) {
  if (ODT == B200_F32) {
    float* o = reinterpret_cast<float*>(out) + i;
    if (vec && valid == 8) {
      reinterpret_cast<float4*>(o)[0] = make_float4(y[0], y[1], y[2], y[3]);
      reinterpret_cast<float4*>(o)[1] = make_float4(y[4], y[5], y[6], y[7]);
    } else {
      for (uint32_t j = 0; j < valid; ++j) o[j] = y[j];
    }
  } else {
    unsigned short h[8];
#pragma unroll
    for (int j = 0; j < 8; ++j)
      h[j] = ODT == B200_F16 ? __half_as_ushort(__float2half_rn(y[j])) : __bfloat16_as_ushort(__float2bfloat16_rn(y[j]));
    unsigned short* o = reinterpret_cast<unsigned short*>(out) + i;
    if (vec && valid == 8) {
      uint4 w;
      w.x = h[0] | (static_cast<uint32_t>(h[1]) << 16); w.y = h[2] | (static_cast<uint32_t>(h[3]) << 16);
      w.z = h[4] | (static_cast<uint32_t>(h[5]) << 16); w.w = h[6] | (static_cast<uint32_t>(h[7]) << 16);
      *reinterpret_cast<uint4*>(o) = w;
    } else {
      for (uint32_t j = 0; j < valid; ++j) o[j] = h[j];
    }
  }
}

// One thread: 16 bytes of codes = 128 / BITS elements, in groups of 8 (a block holds a whole number of groups).
template <int ODT, int BITS>
__device__ __forceinline__ void decode_body(const QuantDecodeParams& p) {
  constexpr uint32_t EPT = 128 / BITS, GROUPS = EPT / 8;
  const uint64_t t = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const uint64_t nbytes = p.n * BITS / 8;
  if (t * 16 >= nbytes) return;
  const bool vec = (p.flags & 1u) != 0;
  uint32_t w[4];
  if (vec && t * 16 + 16 <= nbytes) {
    const uint4 u = ldg_stream_u4(p.values + t * 16);
    w[0] = u.x; w[1] = u.y; w[2] = u.z; w[3] = u.w;
  } else {
    const unsigned char* src = reinterpret_cast<const unsigned char*>(p.values);
#pragma unroll
    for (int b = 0; b < 16; ++b) {
      const uint32_t byte = t * 16 + b < nbytes ? __ldg(src + t * 16 + b) : 0u;
      if (b % 4 == 0) w[b / 4] = 0;
      w[b / 4] |= byte << (8 * (b % 4));
    }
  }
  const float g = p.tensor_scale ? __ldg(reinterpret_cast<const float*>(p.tensor_scale)) : 0.f;
  const uint64_t i0 = t * EPT;
#pragma unroll
  for (uint32_t gi = 0; gi < GROUPS; ++gi) {
    const uint64_t i = i0 + gi * 8;
    if (i >= p.n) break;
    float eff = g;
    if (p.block) {
      const float s = load_scale(p.block_scales, i >> p.block_log2, p.scale_dt);
      eff = p.tensor_scale ? g * s : s;   // multiply_global_scale (dequantize.rs:62-65), rounded once in f32
    }
    // group gi holds 8 * BITS bits starting at bit gi * 8 * BITS of the 128
    const uint32_t bit = gi * 8 * BITS;
    const uint64_t word = BITS == 8 ? (static_cast<uint64_t>(w[bit / 32]) | (static_cast<uint64_t>(w[bit / 32 + 1]) << 32))
                                    : static_cast<uint64_t>(w[bit / 32] >> (bit % 32));
    float y[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const uint32_t field = static_cast<uint32_t>(word >> (j * BITS)) & ((1u << BITS) - 1u);
      y[j] = decode_one(field, p.value, BITS) * eff;
    }
    const uint32_t valid = p.n - i < 8 ? static_cast<uint32_t>(p.n - i) : 8u;
    store8<ODT>(p.out, i, y, valid, vec);
  }
}

template <int ODT>
__device__ __forceinline__ void decode_dispatch(const QuantDecodeParams& p) {
  const uint32_t bits = qv_bits(p.value);
  if (bits == 8) decode_body<ODT, 8>(p);
  else if (bits == 4) decode_body<ODT, 4>(p);
  else decode_body<ODT, 2>(p);
}

// Two cubins come from this source (cubecl_b200/build.py): QUANT_PART 0 ("quant") quantize / dequantize, QUANT_PART 1
// ("quant_mm") the operand preparation of the quantized matmul.
#ifndef QUANT_PART
#define QUANT_PART 0
#endif

#if QUANT_PART == 1
// ------------------------------------------------------------------------------------------------ quantized-matmul operands
// (capi.cpp: b200_matmul_quantized, gemm_wgmma.cu: QM_BLOCK)
// The effective scale of GEMM block j of row r, as b200_dequantize defines it: f32(s), rn(g * f32(s)) with a tensor level,
// or g for a per-tensor side.  A coarser block repeats its scale `rep` times; rows [rows, rows_pad) are written as 0.
template <int DT>   // block-scale dtype, or -1 for a per-tensor side
__device__ __forceinline__ void scales_body(const QuantScalesParams& p) {
  const uint64_t total = p.batch * p.nblk * p.rows_pad;
  const float g = p.tensor_scale ? __ldg(reinterpret_cast<const float*>(p.tensor_scale)) : 0.f;
  for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += static_cast<uint64_t>(gridDim.x) * blockDim.x) {
    const uint64_t r = i % p.rows_pad, t = i / p.rows_pad;
    const uint64_t j = t % p.nblk, b = t / p.nblk;
    float eff = 0.f;
    if (r < p.rows) {
      if constexpr (DT < 0) {
        eff = g;
      } else {
        const uint64_t per_row = p.nblk / p.rep;
        const float s = load_scale(p.block_scales, (b * p.rows + r) * per_row + j / p.rep, DT);
        eff = p.tensor_scale ? __fmul_rn(g, s) : s;
      }
    }
    reinterpret_cast<float*>(p.out)[i] = eff;
  }
}

// 4- and 2-bit code streams widened exactly to one s8 per element (sign extension, as b200_dequantize reads a field);
// one thread writes 16 output bytes, the pitch padding as 0.
__device__ __forceinline__ void widen_body(const QuantWidenParams& p) {
  const uint64_t vpr = p.pitch / 16, total = p.rows * vpr;
  const uint32_t bits = p.bits, sb = 1u << (bits - 1), mask = (1u << bits) - 1u;
  const uint64_t row_bytes = p.K * bits / 8;
  for (uint64_t t = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; t < total; t += static_cast<uint64_t>(gridDim.x) * blockDim.x) {
    const uint64_t r = t / vpr, c0 = (t - r * vpr) * 16;
    const uint64_t src = p.in + r * row_bytes + c0 * bits / 8;
    const uint32_t nbytes = 2u * bits;   // 16 fields
    uint64_t word = 0;
    if (c0 + 16 <= p.K && (src & (nbytes - 1)) == 0) {
      word = bits == 4 ? __ldg(reinterpret_cast<const unsigned long long*>(src)) : __ldg(reinterpret_cast<const unsigned int*>(src));
    } else {
      const uint64_t left = c0 < p.K ? (p.K - c0) * bits / 8 : 0;
      for (uint32_t b = 0; b < nbytes; ++b)
        if (b < left) word |= static_cast<uint64_t>(__ldg(reinterpret_cast<const unsigned char*>(src) + b)) << (8 * b);
    }
    uint32_t w[4] = {0u, 0u, 0u, 0u};
#pragma unroll
    for (int e = 0; e < 16; ++e) {
      const uint32_t f = static_cast<uint32_t>(word >> (e * bits)) & mask;
      const uint32_t s8 = c0 + e < p.K ? ((f ^ sb) - sb) & 0xFFu : 0u;
      w[e / 4] |= s8 << (8 * (e % 4));
    }
    *reinterpret_cast<uint4*>(p.out + r * p.pitch + c0) = make_uint4(w[0], w[1], w[2], w[3]);
  }
}

extern "C" __global__ void __launch_bounds__(256) quant_scales_f32_f32(const QuantScalesParams p) { scales_body<B200_F32>(p); }
extern "C" __global__ void __launch_bounds__(256) quant_scales_f32_f16(const QuantScalesParams p) { scales_body<B200_F16>(p); }
extern "C" __global__ void __launch_bounds__(256) quant_scales_f32_bf16(const QuantScalesParams p) { scales_body<B200_BF16>(p); }
extern "C" __global__ void __launch_bounds__(256) quant_scales_f32_ue8m0(const QuantScalesParams p) { scales_body<B200_UE8M0>(p); }
extern "C" __global__ void __launch_bounds__(256) quant_scales_f32_ue4m3(const QuantScalesParams p) { scales_body<B200_F8E4M3>(p); }
extern "C" __global__ void __launch_bounds__(256) quant_scales_f32_tensor(const QuantScalesParams p) { scales_body<-1>(p); }
extern "C" __global__ void __launch_bounds__(256) quant_widen_s8(const QuantWidenParams p) { widen_body(p); }
#endif  // QUANT_PART == 1

#if QUANT_PART == 0
#define QUANT_KERNELS(tag, DT)                                                                                     \
  extern "C" __global__ void __launch_bounds__(256) quant_absmax_##tag(const QuantParams p) { absmax_body<DT>(p); }  \
  extern "C" __global__ void __launch_bounds__(256) quant_encode_##tag(const QuantParams p) { encode_body<DT>(p); }  \
  extern "C" __global__ void __launch_bounds__(256) quant_decode_##tag(const QuantDecodeParams p) { decode_dispatch<DT>(p); }
QUANT_KERNELS(f32, B200_F32)
QUANT_KERNELS(f16, B200_F16)
QUANT_KERNELS(bf16, B200_BF16)
#endif  // QUANT_PART == 0
