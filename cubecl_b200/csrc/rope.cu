// Rotary position embeddings (capi.cpp: b200_rope, b200_rope_kvcache_write, b200_rope_cos_sin; contracts in
// include/cubecl_b200.h, thread layout in kernel_params.h: RopeParams).
//
// HBM-bound: every q / k element is read once and written once.  A thread owns up to 8 pair-columns of a token, reads their
// 8 cos and 8 sin once, and loops over every head of that token, so the table costs rot * 4 bytes per token against
// (Hq + Hk) * D * 2 * esize of q / k traffic.  Copies move raw element bits (NaN payloads and -0 survive); rotated values are
// widened exactly to f32 and every product and sum is an explicit _rn intrinsic: nothing is contracted into an fma, and the
// 16-byte and the element-wise path fill the same registers, so an element's bits depend on (a, b, c, s) alone.  No shared
// memory, no atomics.
//
// rope_<dt>_<neox|gptj>             b200_rope
// rope_kv_<dt>_<neox|gptj>          b200_rope_kvcache_write into 16-bit caches: rotated k and v go to their cache slots
// rope_kv_fp8_<dt>_<neox|gptj>      the same into fp8 caches, through the encoder attn_kv_write_fp8 uses (kv_quant.cuh)
// rope_cos_sin                      b200_rope_cos_sin, in f64
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cstdint>
#include <type_traits>

#include "kernel_params.h"
#include "kv_quant.cuh"

namespace {

__device__ __forceinline__ float rope_f32(float v) { return v; }
__device__ __forceinline__ float rope_f32(__nv_bfloat16 v) { return __bfloat162float(v); }
__device__ __forceinline__ float rope_f32(__half v) { return __half2float(v); }
template <typename T>
__device__ __forceinline__ T rope_to(float v) {
  if constexpr (sizeof(T) == 4) return v;
  else if constexpr (std::is_same_v<T, __nv_bfloat16>) return __float2bfloat16_rn(v);
  else return __float2half_rn(v);
}

// m <= 8 consecutive raw elements; one 16-byte load (two for f32) when vec and the chunk is whole
template <typename T>
__device__ __forceinline__ void rope_ld8(const T* p, bool vec, uint32_t m, T (&v)[8]) {
  if (vec && m == 8) {
    if constexpr (sizeof(T) == 4) {
      const float4 a = reinterpret_cast<const float4*>(p)[0], b = reinterpret_cast<const float4*>(p)[1];
      v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    } else {
      const uint4 a = *reinterpret_cast<const uint4*>(p);
      memcpy(v, &a, 16);
    }
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i)
      if ((uint32_t)i < m) v[i] = p[i];
  }
}
template <typename T>
__device__ __forceinline__ void rope_st8(T* p, bool vec, uint32_t m, const T (&v)[8]) {
  if (vec && m == 8) {
    if constexpr (sizeof(T) == 4) {
      reinterpret_cast<float4*>(p)[0] = make_float4(v[0], v[1], v[2], v[3]);
      reinterpret_cast<float4*>(p)[1] = make_float4(v[4], v[5], v[6], v[7]);
    } else {
      uint4 a;
      memcpy(&a, v, 16);
      *reinterpret_cast<uint4*>(p) = a;
    }
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i)
      if ((uint32_t)i < m) p[i] = v[i];
  }
}
// m <= 8 consecutive f32 table entries
__device__ __forceinline__ void rope_ld8f(const float* p, bool vec, uint32_t m, float (&v)[8]) {
  if (vec && m == 8) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(p)), b = __ldg(reinterpret_cast<const float4*>(p) + 1);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = (uint32_t)i < m ? __ldg(p + i) : 0.0f;
  }
}

// (a, b) <- (rn(rn(a c) - rn(b s)), rn(rn(b c) + rn(a s))), rounded to T
template <typename T>
__device__ __forceinline__ void rope_pair(T& a, T& b, float c, float s) {
  const float x = rope_f32(a), y = rope_f32(b);
  a = rope_to<T>(__fsub_rn(__fmul_rn(x, c), __fmul_rn(y, s)));
  b = rope_to<T>(__fadd_rn(__fmul_rn(y, c), __fmul_rn(x, s)));
}

// Where a k (or v) row of the cache kernels goes: a 16-bit cache stores the raw elements, an fp8 cache their codes.
template <typename T, bool FP8>
__device__ __forceinline__ void rope_cache_st8(uint64_t base, uint64_t off, bool vec, uint32_t m, const T (&v)[8], float scale,
                                               bool bf16, bool e5m2) {
  if constexpr (!FP8) {
    rope_st8(reinterpret_cast<T*>(base) + off, vec, m, v);
  } else {
    uint32_t w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const uint32_t lo = (uint32_t)(2 * i) < m ? __bfloat16_as_ushort(reinterpret_cast<const __nv_bfloat16&>(v[2 * i])) : 0u;
      const uint32_t hi = (uint32_t)(2 * i + 1) < m ? __bfloat16_as_ushort(reinterpret_cast<const __nv_bfloat16&>(v[2 * i + 1])) : 0u;
      w[i] = lo | (hi << 16);
    }
    const uint4 x = make_uint4(w[0], w[1], w[2], w[3]);
    const uint2 q = kv_quant8(x, scale, bf16, e5m2);
    uint8_t* o = reinterpret_cast<uint8_t*>(base) + off;
    if (vec && m == 8) {
      *reinterpret_cast<uint2*>(o) = q;
    } else {
      const uint8_t* b = reinterpret_cast<const uint8_t*>(&q);
#pragma unroll
      for (int i = 0; i < 8; ++i)
        if ((uint32_t)i < m) o[i] = b[i];
    }
  }
}

// MODE 0: b200_rope.  MODE 1 / 2: b200_rope_kvcache_write into a 16-bit / fp8 cache.
template <typename T, bool GPTJ, int MODE>
__device__ __forceinline__ void rope_body(const RopeParams& p) {
  constexpr bool KV = MODE != 0, FP8 = MODE == 2;
  const bool vec = p.vec != 0;
  const bool bf16 = p.in_bf16 != 0, e5m2 = p.e5m2 != 0;
  for (uint64_t u = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; u < p.units;
       u += static_cast<uint64_t>(gridDim.x) * blockDim.x) {
    const uint64_t n = u / p.groups;
    const uint32_t g = static_cast<uint32_t>(u % p.groups);
    const uint64_t b = n / p.S, s = n % p.S;
    const int64_t pos = p.positions ? reinterpret_cast<const int*>(p.positions)[n] : static_cast<int64_t>(s);
    const bool in_range = pos >= 0 && pos < static_cast<int64_t>(p.P);
    // the cache kernels: this token's slot, or none (its k and v are then not written)
    int64_t slot = -1;
    if constexpr (KV) {
      slot = reinterpret_cast<const int*>(p.slots)[n];
      if (static_cast<uint64_t>(slot) >= p.slot_end) slot = -1;
    }
    const uint64_t pg = static_cast<uint64_t>(slot) / p.page, prow = static_cast<uint64_t>(slot) % p.page;
    // f(h, src, dst) over the q heads (into qo), then the k heads (into ko, or the k cache: dst = its element offset)
    auto each_head = [&](auto&& f, bool pass_only) {
      if (!pass_only || p.pass_q) {
        const T* q = reinterpret_cast<const T*>(p.q) + b * p.q_sb + s * p.q_ss;
        T* qo = reinterpret_cast<T*>(p.qo) + b * p.qo_sb + s * p.qo_ss;
        for (uint32_t h = 0; h < p.Hq; ++h) f(false, h, q + h * p.q_sh, qo + h * p.qo_sh, 0ull);
      }
      if (KV ? slot >= 0 : (!pass_only || p.pass_k)) {
        const T* k = reinterpret_cast<const T*>(p.k) + b * p.k_sb + s * p.k_ss;
        T* ko = reinterpret_cast<T*>(p.ko) + b * p.ko_sb + s * p.ko_ss;
        const uint64_t kc = pg * p.kc_sp + prow * p.kc_sr;
        for (uint32_t h = 0; h < p.Hk; ++h) f(true, h, k + h * p.k_sh, ko + h * p.ko_sh, kc + h * p.kc_sh);
      }
    };
    // store x (m elements at column col) to dst, or for a k head of the cache kernels to the k cache
    auto put = [&](bool isk, uint32_t h, T* dst, uint64_t kc, uint32_t col, uint32_t m, const T (&x)[8]) {
      if (KV && isk) {
        const float ks = FP8 ? reinterpret_cast<const float*>(p.k_scale)[h] : 1.0f;
        rope_cache_st8<T, FP8>(p.kc, kc + col, vec, m, x, ks, bf16, e5m2);
      } else {
        rope_st8(dst + col, vec, m, x);
      }
    };
    if (g < p.gr) {
      // ---- rotary: pairs [i0, i0 + m)
      const uint32_t i0 = g * 8u, m = min(8u, p.half - i0);
      float c[8], sn[8];
      if (in_range) {
        const float* row = reinterpret_cast<const float*>(p.cos_sin) + static_cast<uint64_t>(pos) * p.rot;
        rope_ld8f(row + i0, vec, m, c);
        rope_ld8f(row + p.half + i0, vec, m, sn);
        if (p.inverse) {
#pragma unroll
          for (int i = 0; i < 8; ++i) sn[i] = -sn[i];
        }
      }
      // columns of the two 8-element halves: NeoX a at i0, b at half + i0; GPT-J pairs interleaved from 2 i0
      const uint32_t c0 = GPTJ ? 2u * i0 : i0, c1 = GPTJ ? 2u * i0 + 8u : p.half + i0;
      const uint32_t m0 = GPTJ ? min(8u, 2u * m) : m, m1 = GPTJ ? (2u * m > 8u ? 2u * m - 8u : 0u) : m;
      each_head([&](bool isk, uint32_t h, const T* src, T* dst, uint64_t kc) {
        if (!in_range && !(isk ? p.pass_k : p.pass_q)) return;   // in place: the row stays as it is
        T x0[8], x1[8];
        rope_ld8(src + c0, vec, m0, x0);
        if (m1) rope_ld8(src + c1, vec, m1, x1);
        if (in_range) {
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            if constexpr (GPTJ) {
              if (i < 4) rope_pair(x0[2 * i], x0[2 * i + 1], c[i], sn[i]);
              else rope_pair(x1[2 * i - 8], x1[2 * i - 7], c[i], sn[i]);
            } else {
              rope_pair(x0[i], x1[i], c[i], sn[i]);
            }
          }
        }
        put(isk, h, dst, kc, c0, m0, x0);
        if (m1) put(isk, h, dst, kc, c1, m1, x1);
      }, false);
    } else if (g < p.gr + p.gp) {
      // ---- pass-through columns [j0, j0 + m) of the outputs that are out of place
      const uint32_t j0 = p.rot + (g - p.gr) * 8u, m = min(8u, p.D - j0);
      each_head([&](bool isk, uint32_t h, const T* src, T* dst, uint64_t kc) {
        T x[8];
        rope_ld8(src + j0, vec, m, x);
        put(isk, h, dst, kc, j0, m, x);
      }, true);
    } else if (KV && slot >= 0) {
      // ---- v columns [j0, j0 + 8) of every kv head into the v cache
      const uint32_t j0 = (g - p.gr - p.gp) * 8u;
      const bool vvec = p.vvec != 0;
      const T* v = reinterpret_cast<const T*>(p.vn) + b * p.vn_sb + s * p.vn_ss + j0;
      const uint64_t vc = pg * p.vc_sp + prow * p.vc_sr + j0;
      for (uint32_t h = 0; h < p.Hk; ++h) {
        T x[8];
        rope_ld8(v + h * p.vn_sh, vvec, 8u, x);
        const float vs = FP8 ? reinterpret_cast<const float*>(p.v_scale)[h] : 1.0f;
        rope_cache_st8<T, FP8>(p.vc, vc + h * p.vc_sh, true, 8u, x, vs, bf16, e5m2);
      }
    }
  }
}

}  // namespace

#define ROPE_KERNEL(NAME, T, GPTJ, MODE)                                                                       \
  extern "C" __global__ void __launch_bounds__(kRopeThreads, MODE ? kRopeKvCtasPerSm : kRopeCtasPerSm)          \
      NAME(const __grid_constant__ RopeParams p) {                                                            \
    rope_body<T, GPTJ, MODE>(p);                                                                              \
  }
ROPE_KERNEL(rope_f32_neox, float, false, 0)
ROPE_KERNEL(rope_f32_gptj, float, true, 0)
ROPE_KERNEL(rope_bf16_neox, __nv_bfloat16, false, 0)
ROPE_KERNEL(rope_bf16_gptj, __nv_bfloat16, true, 0)
ROPE_KERNEL(rope_f16_neox, __half, false, 0)
ROPE_KERNEL(rope_f16_gptj, __half, true, 0)
ROPE_KERNEL(rope_kv_bf16_neox, __nv_bfloat16, false, 1)
ROPE_KERNEL(rope_kv_bf16_gptj, __nv_bfloat16, true, 1)
ROPE_KERNEL(rope_kv_f16_neox, __half, false, 1)
ROPE_KERNEL(rope_kv_f16_gptj, __half, true, 1)
ROPE_KERNEL(rope_kv_fp8_bf16_neox, __nv_bfloat16, false, 2)
ROPE_KERNEL(rope_kv_fp8_bf16_gptj, __nv_bfloat16, true, 2)
ROPE_KERNEL(rope_kv_fp8_f16_neox, __half, false, 2)
ROPE_KERNEL(rope_kv_fp8_f16_gptj, __half, true, 2)

// The table, in f64: inv_freq_i by the kind's rule, then af * cos / sin of p * inv_freq_i, each rounded once to f32.
extern "C" __global__ void __launch_bounds__(kRopeThreads) rope_cos_sin(const __grid_constant__ RopeTableParams p) {
  constexpr double kPi = 3.14159265358979323846264338327950, kTwoPi = 2.0 * kPi;
  for (uint64_t u = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; u < p.n;
       u += static_cast<uint64_t>(gridDim.x) * blockDim.x) {
    const uint64_t pos = u / p.half;
    const uint32_t i = static_cast<uint32_t>(u % p.half);
    double inv;
    if (p.kind == B200_ROPE_INV_FREQ) {
      inv = static_cast<double>(reinterpret_cast<const float*>(p.inv_freq)[i]);
    } else {
      inv = 1.0 / pow(p.base, static_cast<double>(2u * i) / static_cast<double>(2u * p.half));
      if (p.kind == B200_ROPE_LINEAR) {
        inv = inv / p.factor;
      } else if (p.kind == B200_ROPE_LLAMA3) {
        const double w = kTwoPi / inv;
        if (w > p.orig / p.low_ff) {
          inv = inv / p.factor;
        } else if (!(w < p.orig / p.high_ff)) {
          const double m = (p.orig / w - p.low_ff) / (p.high_ff - p.low_ff);
          inv = (1.0 - m) * inv / p.factor + m * inv;
        }
      } else if (p.kind == B200_ROPE_YARN) {
        const double r = fmin(fmax((static_cast<double>(i) - p.ramp_lo) / (p.ramp_hi - p.ramp_lo), 0.0), 1.0);
        const double ext = 1.0 - r;   // HF's inv_freq_extrapolation_factor
        inv = inv / p.factor * (1.0 - ext) + inv * ext;
      }
    }
    // sincospi of angle / pi: an exact range reduction, so no slow path for large angles (the division costs one f64
    // rounding, far below an f32 ulp)
    double sv, cv;
    sincospi(static_cast<double>(pos) * inv / kPi, &sv, &cv);
    float* row = reinterpret_cast<float*>(p.out) + pos * (2u * p.half);
    row[i] = static_cast<float>(p.af * cv);
    row[p.half + i] = static_cast<float>(p.af * sv);
  }
}
