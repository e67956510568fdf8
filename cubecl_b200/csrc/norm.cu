// RMSNorm and LayerNorm over the innermost axis, with an optional fused residual add, an optional fp8 block-quantized
// output, and the backward (capi.cpp: b200_norm, b200_norm_quantized_fp8, b200_norm_backward; contracts in
// include/cubecl_b200.h, geometry in kernel_params.h: NormParams).
//
// HBM-bound: a row is read once into registers (32 values per thread), reduced, and written once.  Every sum runs in one
// order fixed by n: a thread's chunks in increasing order and the 8 values of a chunk in order, an xor butterfly over the
// warp, the row group's warps in order, then the CTAs of a cluster in rank order.  The 128-bit and the element-wise path fill
// the same registers, so a row's bits depend neither on its position, the batch, the alignment nor the SM count.  Every
// operation is an explicit _rn intrinsic: nothing is contracted into an fma.  No atomics.
#include <cooperative_groups.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cstdint>
#include <type_traits>

#include "kernel_params.h"
#include "quant_common.cuh"

namespace cg = cooperative_groups;

extern __shared__ __align__(16) float norm_smem[];

struct NormFp8 {};   // the output type of the quantizing forward

__device__ __forceinline__ float norm_f32(float v) { return v; }
__device__ __forceinline__ float norm_f32(__nv_bfloat16 v) { return __bfloat162float(v); }
__device__ __forceinline__ float norm_f32(__half v) { return __half2float(v); }
__device__ __forceinline__ void norm_put(float* o, float v) { *o = v; }
__device__ __forceinline__ void norm_put(__nv_bfloat16* o, float v) { *o = __float2bfloat16_rn(v); }
__device__ __forceinline__ void norm_put(__half* o, float v) { *o = __float2half_rn(v); }
// v rounded to nearest-even in T and read back
template <typename T>
__device__ __forceinline__ float norm_round(float v) {
  if constexpr (sizeof(T) == 4) return v;
  else { T h; norm_put(&h, v); return norm_f32(h); }
}

// m <= 8 consecutive elements as f32 (the rest 0): one or two 128-bit loads when `vec` and the chunk is whole
template <typename T>
__device__ __forceinline__ void norm_ld8(const T* p, bool vec, uint32_t m, float (&v)[8]) {
  if (vec && m == 8) {
    if constexpr (sizeof(T) == 4) {
      const float4 a = __ldg(reinterpret_cast<const float4*>(p)), b = __ldg(reinterpret_cast<const float4*>(p) + 1);
      v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    } else {
      const uint4 a = __ldg(reinterpret_cast<const uint4*>(p));
      const T* h = reinterpret_cast<const T*>(&a);
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] = norm_f32(h[i]);
    }
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = (uint32_t)i < m ? norm_f32(p[i]) : 0.0f;
  }
}
template <typename T>
__device__ __forceinline__ void norm_st8(T* p, bool vec, uint32_t m, const float (&v)[8]) {
  if (vec && m == 8) {
    if constexpr (sizeof(T) == 4) {
      reinterpret_cast<float4*>(p)[0] = make_float4(v[0], v[1], v[2], v[3]);
      reinterpret_cast<float4*>(p)[1] = make_float4(v[4], v[5], v[6], v[7]);
    } else {
      uint4 a;
      T* h = reinterpret_cast<T*>(&a);
#pragma unroll
      for (int i = 0; i < 8; ++i) norm_put(h + i, v[i]);
      *reinterpret_cast<uint4*>(p) = a;
    }
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i)
      if ((uint32_t)i < m) norm_put(p + i, v[i]);
  }
}

// weight (1 when absent) or bias (+0 when absent) of columns [j0, j0 + m): f32 or the x dtype
template <typename TX>
__device__ __forceinline__ void norm_affine(uint64_t base, bool f32, uint32_t j0, bool vec, uint32_t m, float dflt, float (&v)[8]) {
  if (!base) {
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = dflt;
  } else if (f32) {
    norm_ld8(reinterpret_cast<const float*>(base) + j0, vec, m, v);
  } else {
    norm_ld8(reinterpret_cast<const TX*>(base) + j0, vec, m, v);
  }
}

// The calling thread's row group: nt threads of one CTA (nt = 32 in the warp class, p.nt in the CTA class), or of each CTA of
// a cluster of `ranks`; a CTA holds kNormThreads / nt groups, each on its own row (or backward unit).
struct NormGroup {
  uint32_t nt, tid, group, groups, ranks, rank;
  // the first column of chunk c of this thread and how many of its 8 columns are in the row (0 when inactive)
  __device__ __forceinline__ uint32_t col(int c) const { return ((c * ranks + rank) * nt + tid) * 8u; }
  __device__ __forceinline__ uint32_t cnt(uint32_t j0, uint32_t n, bool active) const { return active && j0 < n ? min(8u, n - j0) : 0u; }
};
template <bool WARP>
__device__ __forceinline__ NormGroup norm_group(const NormParams& p) {
  NormGroup g;
  g.nt = WARP ? 32u : p.nt;
  g.tid = threadIdx.x & (g.nt - 1u);
  g.group = threadIdx.x / g.nt;
  g.groups = kNormThreads / g.nt;
  g.ranks = WARP ? 1u : p.ranks;
  g.rank = (!WARP && g.ranks > 1) ? cg::this_cluster().block_rank() : 0u;
  return g;
}

// The row-group sum of NV per-thread partials, returned to every thread of the group: xor butterfly, the group's warps in
// order, ranks in order.  Every thread of the CTA calls it (inactive groups too: it holds CTA barriers).
template <int NV, bool WARP>
__device__ __forceinline__ void norm_reduce(const NormGroup& g, float (&s)[NV]) {
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1)
#pragma unroll
    for (int k = 0; k < NV; ++k) s[k] = __fadd_rn(s[k], __shfl_xor_sync(0xFFFFFFFFu, s[k], m));
  if constexpr (!WARP) {
    __shared__ float red[kNormThreads / 32][NV];
    __shared__ float ctot[NV];
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5, w0 = g.group * (g.nt >> 5), w1 = w0 + (g.nt >> 5);
    if (lane == 0)
#pragma unroll
      for (int k = 0; k < NV; ++k) red[warp][k] = s[k];
    __syncthreads();
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      float a = red[w0][k];
      for (uint32_t w = w0 + 1; w < w1; ++w) a = __fadd_rn(a, red[w][k]);
      s[k] = a;
    }
    if (g.ranks > 1) {
      cg::cluster_group cl = cg::this_cluster();
      if (threadIdx.x == 0)
#pragma unroll
        for (int k = 0; k < NV; ++k) ctot[k] = s[k];
      cl.sync();
#pragma unroll
      for (int k = 0; k < NV; ++k) {
        float a = *cl.map_shared_rank(&ctot[k], 0);
        for (uint32_t r = 1; r < g.ranks; ++r) a = __fadd_rn(a, *cl.map_shared_rank(&ctot[k], r));
        s[k] = a;
      }
      cl.sync();   // no CTA rewrites ctot (or exits) while a peer still reads it
    } else {
      __syncthreads();
    }
  }
}

__device__ __forceinline__ float norm_rstd(float var, float eps) { return __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn(var, eps))); }

// The y of one chunk as fp8 codes and block scales, exactly as quant_encode_f32 writes b200_quantize's block-only schemes:
// the block's G = block / 8 chunks sit on G consecutive lanes.  Every lane of the warp calls it (m = 0 past the row's end).
__device__ __forceinline__ void norm_store_fp8(const NormParams& p, uint64_t r, uint32_t j0, uint32_t m, bool vec, const float (&y)[8]) {
  uint32_t am = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i)
    if ((uint32_t)i < m) am = max(am, finite_abs_bits(y[i]));
  for (uint32_t o = 1; o < (p.block >> 3); o <<= 1) am = max(am, __shfl_xor_sync(0xFFFFFFFFu, am, o));
  if (!m) return;
  const float lo = qv_lo(p.value), hi = qv_hi(p.value), amax = __uint_as_float(am);
  const float s = amax != 0.f ? round_up_scale(amax / hi, p.scale_dt) : 0.f;
  const uint32_t eb = __float_as_uint(s);
  const bool pow2 = ((eb & 0x7FFFFFu) == 0 && eb >= 0x00800000u && eb < 0x7F800000u) || eb == 0x00400000u;
  const float rcp = pow2 ? 1.f / s : 0.f;
  const uint64_t f = r * p.n + j0;
  uint64_t packed = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) packed |= (uint64_t)(encode_one(y[i], s, rcp, pow2, p.value, lo, hi) & 0xFFu) << (8 * i);
  unsigned char* codes = reinterpret_cast<unsigned char*>(p.y) + f;
  if (vec) *reinterpret_cast<uint64_t*>(codes) = packed;
  else
    for (int i = 0; i < 8; ++i) codes[i] = (unsigned char)(packed >> (8 * i));
  if ((j0 & (p.block - 1)) == 0) {
    const uint64_t si = f >> p.block_log2;
    const uint32_t sb = scale_bits(s, p.scale_dt);
    if (p.scale_dt == B200_F32) reinterpret_cast<uint32_t*>(p.block_scales)[si] = sb;
    else reinterpret_cast<unsigned char*>(p.block_scales)[si] = (unsigned char)sb;
  }
}

// ------------------------------------------------------------------------------------------------ forward
// Every load of a row's x (and residual) is issued before the first use, so a thread has all its chunks in flight; weight
// and bias, the same for every row, come from L1 / L2 where they are used.
template <typename TX, typename TY, bool WARP>
__device__ __forceinline__ void norm_fwd(const NormParams& p) {
  const NormGroup g = norm_group<WARP>(p);
  const uint32_t n = p.n;
  const bool vec = p.vec != 0, layer = p.kind == B200_NORM_LAYER, w_f32 = p.w_f32 != 0;
  const uint64_t step = (uint64_t)(gridDim.x / g.ranks) * g.groups;
  for (uint64_t base = (uint64_t)(blockIdx.x / g.ranks) * g.groups; base < p.t; base += step) {
    const uint64_t r = base + g.group;
    const bool active = r < p.t;
    float v[kNormChunks][8];
#pragma unroll
    for (int c = 0; c < kNormChunks; ++c) {
      const uint32_t j0 = g.col(c), m = g.cnt(j0, n, active);
      if (m) norm_ld8(reinterpret_cast<const TX*>(p.x) + r * p.x_stride + j0, vec, m, v[c]);
    }
    if (p.residual) {
      float e[kNormChunks][8];
#pragma unroll
      for (int c = 0; c < kNormChunks; ++c) {
        const uint32_t j0 = g.col(c), m = g.cnt(j0, n, active);
        if (m) norm_ld8(reinterpret_cast<const TX*>(p.residual) + r * p.residual_stride + j0, vec, m, e[c]);
      }
#pragma unroll
      for (int c = 0; c < kNormChunks; ++c) {
        const uint32_t j0 = g.col(c), m = g.cnt(j0, n, active);
        if (!m) continue;
#pragma unroll
        for (int i = 0; i < 8; ++i) v[c][i] = norm_round<TX>(__fadd_rn(v[c][i], e[c][i]));
        norm_st8(reinterpret_cast<TX*>(p.h_out) + r * p.h_stride + j0, vec, m, v[c]);
      }
    }
    float s[1] = {0.0f};
#pragma unroll
    for (int c = 0; c < kNormChunks; ++c) {
      const uint32_t m = g.cnt(g.col(c), n, active);
#pragma unroll
      for (int i = 0; i < 8; ++i)
        if ((uint32_t)i < m) s[0] = __fadd_rn(s[0], layer ? v[c][i] : __fmul_rn(v[c][i], v[c][i]));
    }
    norm_reduce<1, WARP>(g, s);
    float mu = 0.0f, var = __fdiv_rn(s[0], (float)n);
    if (layer) {
      mu = var;
      s[0] = 0.0f;
#pragma unroll
      for (int c = 0; c < kNormChunks; ++c) {
        const uint32_t m = g.cnt(g.col(c), n, active);
#pragma unroll
        for (int i = 0; i < 8; ++i)
          if ((uint32_t)i < m) { const float d = __fsub_rn(v[c][i], mu); s[0] = __fadd_rn(s[0], __fmul_rn(d, d)); }
      }
      norm_reduce<1, WARP>(g, s);
      var = __fdiv_rn(s[0], (float)n);
    }
    const float rstd = norm_rstd(var, p.eps);
    if (active && g.tid == 0 && g.rank == 0) {
      if (p.mean) reinterpret_cast<float*>(p.mean)[r] = mu;
      if (p.rstd) reinterpret_cast<float*>(p.rstd)[r] = rstd;
    }
#pragma unroll
    for (int c = 0; c < kNormChunks; ++c) {
      const uint32_t j0 = g.col(c), m = g.cnt(j0, n, active);
      float y[8];
      if (m) {
        float w[8], b[8];
        norm_affine<TX>(p.weight, w_f32, j0, vec, m, 1.0f, w);
        norm_affine<TX>(p.bias, w_f32, j0, vec, m, 0.0f, b);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float xh = __fmul_rn(layer ? __fsub_rn(v[c][i], mu) : v[c][i], rstd);
          y[i] = __fadd_rn(__fmul_rn(xh, w[i]), b[i]);
        }
      }
      if constexpr (std::is_same<TY, NormFp8>::value) {
        norm_store_fp8(p, r, j0, m, vec, y);
      } else if (m) {
        norm_st8(reinterpret_cast<TY*>(p.y) + r * p.y_stride + j0, vec, m, y);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ backward
// Unit u owns rows [u * rows_per_unit, min(t, (u + 1) * rows_per_unit)).  Per row: x^ and g = rn(f32(dy) * w) are kept in
// registers, c1 = rn(sum rn(g * x^) / n) and c2 = rn(sum g / n) are reduced together, and dweight / dbias collect
// rn(f32(dy) * x^) / f32(dy) in the unit's shared-memory accumulators (cell (c * 8 + i) * nt + tid: a thread's own).
template <typename TX, typename TG, bool WARP>
__device__ __forceinline__ void norm_bwd(const NormParams& p) {
  const NormGroup g = norm_group<WARP>(p);
  const uint64_t u = (uint64_t)(blockIdx.x / g.ranks) * g.groups + g.group;
  const bool unit = u < p.units;
  const uint32_t n = p.n, nt = g.nt, tid = g.tid;
  const bool vec = p.vec != 0, layer = p.kind == B200_NORM_LAYER, w_f32 = p.w_f32 != 0;
  const bool want_w = p.dweight != 0, want_b = p.dbias != 0;
  float* acc_w = norm_smem + g.group * 2u * kNormChunks * 8u * nt;
  float* acc_b = acc_w + kNormChunks * 8u * nt;
#pragma unroll
  for (int k = 0; k < kNormChunks * 8; ++k) { acc_w[k * nt + tid] = 0.0f; acc_b[k * nt + tid] = 0.0f; }
  const uint64_t r0 = u * p.rows_per_unit, r1 = min(p.t, r0 + p.rows_per_unit);
  for (uint32_t i_row = 0; i_row < p.rows_per_unit; ++i_row) {   // the same trip count in every group of the CTA
    const uint64_t r = r0 + i_row;
    const bool active = unit && r < r1;
    const float rstd = active ? __ldg(reinterpret_cast<const float*>(p.rstd) + r) : 0.0f;
    const float mu = active && layer ? __ldg(reinterpret_cast<const float*>(p.mean) + r) : 0.0f;
    float xh[kNormChunks][8], gg[kNormChunks][8];
#pragma unroll
    for (int c = 0; c < kNormChunks; ++c) {
      const uint32_t j0 = g.col(c), m = g.cnt(j0, n, active);
      if (!m) continue;
      norm_ld8(reinterpret_cast<const TX*>(p.x) + r * p.h_stride + j0, vec, m, xh[c]);
      norm_ld8(reinterpret_cast<const TG*>(p.dy) + r * p.dy_stride + j0, vec, m, gg[c]);
    }
    float s[2] = {0.0f, 0.0f};
#pragma unroll
    for (int c = 0; c < kNormChunks; ++c) {
      const uint32_t j0 = g.col(c), m = g.cnt(j0, n, active);
      if (!m) continue;
      float w[8];
      norm_affine<TX>(p.weight, w_f32, j0, vec, m, 1.0f, w);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        if ((uint32_t)i >= m) continue;
        const float d = gg[c][i];
        xh[c][i] = __fmul_rn(layer ? __fsub_rn(xh[c][i], mu) : xh[c][i], rstd);
        gg[c][i] = __fmul_rn(d, w[i]);
        s[0] = __fadd_rn(s[0], __fmul_rn(gg[c][i], xh[c][i]));
        s[1] = __fadd_rn(s[1], gg[c][i]);
        const uint32_t cell = (c * 8 + i) * nt + tid;
        if (want_w) acc_w[cell] = __fadd_rn(acc_w[cell], __fmul_rn(d, xh[c][i]));
        if (want_b) acc_b[cell] = __fadd_rn(acc_b[cell], d);
      }
    }
    norm_reduce<2, WARP>(g, s);
    const float c1 = __fdiv_rn(s[0], (float)n), c2 = __fdiv_rn(s[1], (float)n);
#pragma unroll
    for (int c = 0; c < kNormChunks; ++c) {
      const uint32_t j0 = g.col(c), m = g.cnt(j0, n, active);
      if (!m) continue;
      float dx[8], dh[8];
      if (p.d_h) norm_ld8(reinterpret_cast<const TG*>(p.d_h) + r * p.d_h_stride + j0, vec, m, dh);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float e = __fsub_rn(gg[c][i], __fmul_rn(xh[c][i], c1));
        if (layer) e = __fsub_rn(e, c2);
        dx[i] = __fmul_rn(rstd, e);
        if (p.d_h) dx[i] = __fadd_rn(dx[i], dh[i]);
      }
      norm_st8(reinterpret_cast<TG*>(p.dx) + r * p.dx_stride + j0, vec, m, dx);
    }
  }
  if (!unit || (!want_w && !want_b)) return;
  float* part_w = reinterpret_cast<float*>(p.part) + u * n;
  float* part_b = reinterpret_cast<float*>(p.part) + ((uint64_t)p.units + u) * n;
#pragma unroll
  for (int c = 0; c < kNormChunks; ++c) {
    const uint32_t j0 = g.col(c), m = g.cnt(j0, n, true);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if ((uint32_t)i >= m) continue;
      const uint32_t cell = (c * 8 + i) * nt + tid;
      if (want_w) part_w[j0 + i] = acc_w[cell];
      if (want_b) part_b[j0 + i] = acc_b[cell];
    }
  }
}

// dweight[j] = part_w[0][j] + part_w[1][j] + ... in unit order (likewise dbias); grid (ceil(n / 256), 2)
extern "C" __global__ void __launch_bounds__(kNormThreads) norm_bwd_reduce(const __grid_constant__ NormParams p) {
  const uint32_t j = blockIdx.x * kNormThreads + threadIdx.x;
  const uint64_t out = blockIdx.y ? p.dbias : p.dweight;
  if (j >= p.n || !out) return;
  const float* part = reinterpret_cast<const float*>(p.part) + (uint64_t)blockIdx.y * p.units * p.n + j;
  float a = part[0];
  for (uint32_t u = 1; u < p.units; ++u) a = __fadd_rn(a, part[(uint64_t)u * p.n]);
  reinterpret_cast<float*>(out)[j] = a;
}

#define NORM_FWD(tx, TX, ty, TY)                                                                                             \
  extern "C" __global__ void __launch_bounds__(kNormThreads, 2) norm_fwd_##tx##_##ty##_warp(const __grid_constant__ NormParams p) { \
    norm_fwd<TX, TY, true>(p);                                                                                               \
  }                                                                                                                          \
  extern "C" __global__ void __launch_bounds__(kNormThreads, 2) norm_fwd_##tx##_##ty##_cta(const __grid_constant__ NormParams p) { \
    norm_fwd<TX, TY, false>(p);                                                                                              \
  }
#define NORM_BWD(tx, TX, tg, TG)                                                                                             \
  extern "C" __global__ void __launch_bounds__(kNormThreads, 2) norm_bwd_##tx##_##tg##_warp(const __grid_constant__ NormParams p) { \
    norm_bwd<TX, TG, true>(p);                                                                                               \
  }                                                                                                                          \
  extern "C" __global__ void __launch_bounds__(kNormThreads, 2) norm_bwd_##tx##_##tg##_cta(const __grid_constant__ NormParams p) { \
    norm_bwd<TX, TG, false>(p);                                                                                              \
  }
#define NORM_ROW(tx, TX)                                                                                                     \
  NORM_FWD(tx, TX, f32, float) NORM_FWD(tx, TX, bf16, __nv_bfloat16) NORM_FWD(tx, TX, f16, __half) NORM_FWD(tx, TX, fp8, NormFp8) \
  NORM_BWD(tx, TX, f32, float) NORM_BWD(tx, TX, bf16, __nv_bfloat16) NORM_BWD(tx, TX, f16, __half)
NORM_ROW(f32, float)
NORM_ROW(bf16, __nv_bfloat16)
NORM_ROW(f16, __half)
