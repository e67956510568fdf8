// Softmax cross-entropy over the vocabulary: per-row loss and lse, the logits gradient, and the forward that writes the
// gradient in the same launch (capi.cpp: b200_cross_entropy, b200_cross_entropy_backward; contracts in
// include/cubecl_b200.h, geometry in kernel_params.h: XentParams).
//
// HBM-bound.  A row is streamed once: each thread keeps a running (max m, sum s, sum of logits sx) over its 8-element chunks,
// rescaling s once per chunk when the chunk raises m, then the states are merged in an order fixed by v: an xor butterfly
// over the warp, the group's warps in order, the cluster's CTAs in rank order through distributed shared memory.  The
// gradient pass re-reads the thread's own chunks (from L2 in the fused launch) and writes each gradient once.  The 128-bit
// and the element-wise path fill the same registers, so a row's bits depend neither on its position, the batch, the
// alignment nor the SM count.  Every operation is an explicit _rn intrinsic; exponentials are ex2.approx.ftz and
// lg2.approx.  No atomics.
#include <cooperative_groups.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cstdint>

#include "attention.cuh"
#include "kernel_params.h"

namespace cg = cooperative_groups;
using b200::ex2;

constexpr float kXentLog2e = 1.4426950408889634f;
constexpr float kXentLn2 = 0.6931471805599453f;
constexpr int kXentUnroll = 4;   // chunks a thread has in flight

__device__ __forceinline__ float lg2(float x) {
  float y;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__device__ __forceinline__ float xent_f32(float v) { return v; }
__device__ __forceinline__ float xent_f32(__nv_bfloat16 v) { return __bfloat162float(v); }
__device__ __forceinline__ float xent_f32(__half v) { return __half2float(v); }
__device__ __forceinline__ void xent_put(float* o, float v) { *o = v; }
__device__ __forceinline__ void xent_put(__nv_bfloat16* o, float v) { *o = __float2bfloat16_rn(v); }
__device__ __forceinline__ void xent_put(__half* o, float v) { *o = __float2half_rn(v); }

// m <= 8 consecutive elements as f32: one or two 128-bit loads when `vec` and the chunk is whole.  Plain (coherent) loads:
// in place, the gradient overwrites the logits this kernel reads.
template <typename T>
__device__ __forceinline__ void xent_ld8(const T* p, bool vec, uint32_t m, float (&v)[8]) {
  if (vec && m == 8) {
    if constexpr (sizeof(T) == 4) {
      const float4 a = reinterpret_cast<const float4*>(p)[0], b = reinterpret_cast<const float4*>(p)[1];
      v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    } else {
      const uint4 a = *reinterpret_cast<const uint4*>(p);
      const T* h = reinterpret_cast<const T*>(&a);
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] = xent_f32(h[i]);
    }
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = (uint32_t)i < m ? xent_f32(p[i]) : 0.0f;
  }
}
template <typename T>
__device__ __forceinline__ void xent_st8(T* p, bool vec, uint32_t m, const float (&v)[8]) {
  if (vec && m == 8) {
    if constexpr (sizeof(T) == 4) {
      reinterpret_cast<float4*>(p)[0] = make_float4(v[0], v[1], v[2], v[3]);
      reinterpret_cast<float4*>(p)[1] = make_float4(v[4], v[5], v[6], v[7]);
    } else {
      uint4 a;
      T* h = reinterpret_cast<T*>(&a);
#pragma unroll
      for (int i = 0; i < 8; ++i) xent_put(h + i, v[i]);
      *reinterpret_cast<uint4*>(p) = a;
    }
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i)
      if ((uint32_t)i < m) xent_put(p + i, v[i]);
  }
}

// A row's running state: max, sum of ex2 relative to the max (shifted by 0 while the max is -inf), sum of the logits.
struct XentStat {
  float m, s, sx;
};

// One chunk of m >= 1 values, in column order.
__device__ __forceinline__ void xent_chunk(XentStat& st, const float (&a)[8], uint32_t m) {
  float cm = a[0];
#pragma unroll
  for (int i = 1; i < 8; ++i)
    if ((uint32_t)i < m) cm = fmaxf(cm, a[i]);
  const float mn = fmaxf(st.m, cm);
  if (mn != st.m) st.s = __fmul_rn(st.s, ex2(__fmul_rn(__fsub_rn(st.m, mn), kXentLog2e)));
  st.m = mn;
  const float sh = mn == -INFINITY ? 0.0f : mn;
#pragma unroll
  for (int i = 0; i < 8; ++i)
    if ((uint32_t)i < m) {
      st.s = __fadd_rn(st.s, ex2(__fmul_rn(__fsub_rn(a[i], sh), kXentLog2e)));
      st.sx = __fadd_rn(st.sx, a[i]);
    }
}

// Symmetric in its operands, so both lanes of a butterfly pair hold the same state.
__device__ __forceinline__ XentStat xent_merge(const XentStat& a, const XentStat& b) {
  const float M = fmaxf(a.m, b.m);
  const float sa = a.m == M ? a.s : __fmul_rn(a.s, ex2(__fmul_rn(__fsub_rn(a.m, M), kXentLog2e)));
  const float sb = b.m == M ? b.s : __fmul_rn(b.s, ex2(__fmul_rn(__fsub_rn(b.m, M), kXentLog2e)));
  return {M, __fadd_rn(sa, sb), __fadd_rn(a.sx, b.sx)};
}

// The calling thread's row group: nt threads of one CTA in each of `ranks` CTAs (rank = blockIdx.x % ranks: a 1-D cluster's
// block rank in the forward, plain CTAs in the backward, which merges nothing).
struct XentGroup {
  uint32_t nt, tid, group, groups, ranks, rank;
};
template <bool WARP>
__device__ __forceinline__ XentGroup xent_group(const XentParams& p) {
  XentGroup g;
  g.nt = WARP ? 32u : p.nt;
  g.tid = threadIdx.x & (g.nt - 1u);
  g.group = threadIdx.x / g.nt;
  g.groups = kXentThreads / g.nt;
  g.ranks = WARP ? 1u : p.ranks;
  g.rank = blockIdx.x % g.ranks;
  return g;
}

// The row-group merge, returned to every thread of the group.  Every thread of the CTA calls it (it holds CTA barriers).
template <bool WARP>
__device__ __forceinline__ XentStat xent_reduce(const XentGroup& g, XentStat st) {
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) {
    const XentStat q{__shfl_xor_sync(0xFFFFFFFFu, st.m, o), __shfl_xor_sync(0xFFFFFFFFu, st.s, o),
                     __shfl_xor_sync(0xFFFFFFFFu, st.sx, o)};
    st = xent_merge(st, q);
  }
  if constexpr (!WARP) {
    __shared__ XentStat red[kXentThreads / 32];
    __shared__ XentStat ctot;
    const uint32_t warp = threadIdx.x >> 5, w0 = g.group * (g.nt >> 5), w1 = w0 + (g.nt >> 5);
    if ((threadIdx.x & 31u) == 0) red[warp] = st;
    __syncthreads();
    st = red[w0];
    for (uint32_t w = w0 + 1; w < w1; ++w) st = xent_merge(st, red[w]);
    if (g.ranks > 1) {   // then nt = kXentThreads: one group per CTA
      cg::cluster_group cl = cg::this_cluster();
      if (threadIdx.x == 0) ctot = st;
      cl.sync();
      st = *cl.map_shared_rank(&ctot, 0);
      for (uint32_t r = 1; r < g.ranks; ++r) st = xent_merge(st, *cl.map_shared_rank(&ctot, r));
      cl.sync();   // no CTA rewrites ctot (or exits) while a peer still reads it
    } else {
      __syncthreads();
    }
  }
  return st;
}

__device__ __forceinline__ int64_t xent_target(const XentParams& p, uint64_t r) {
  return p.t64 ? reinterpret_cast<const int64_t*>(p.targets)[r] : (int64_t)reinterpret_cast<const int32_t*>(p.targets)[r];
}

enum { XENT_FWD = 0, XENT_FUSED = 1, XENT_BWD = 2 };

// Rows base + group, base stepping over the grid.  FWD: loss and lse; FUSED: those and the gradient; BWD: the gradient from
// the given lse.
template <typename TX, typename TG, int MODE, bool WARP>
__device__ __forceinline__ void xent_rows(const XentParams& p) {
  const XentGroup g = xent_group<WARP>(p);
  const uint32_t v = p.v, nch = (v + 7) / 8, cstep = g.ranks * g.nt, q0 = g.rank * g.nt + g.tid;
  const bool vec = p.vec != 0, smooth = p.eps_v != 0.0f, zl = p.z != 0.0f;
  const uint64_t step = (uint64_t)(gridDim.x / g.ranks) * g.groups;
  for (uint64_t base = (uint64_t)(blockIdx.x / g.ranks) * g.groups; base < p.t; base += step) {
    const uint64_t r = base + g.group;
    const bool active = r < p.t;
    const TX* x = reinterpret_cast<const TX*>(p.logits) + r * p.ls;
    const int64_t y = active ? xent_target(p, r) : 0;
    const bool counted = y != (int64_t)p.ignore_index, bad = counted && (y < 0 || y >= (int64_t)v);
    const bool writer = active && g.tid == 0 && g.rank == 0;
    float lse = 0.0f;
    if constexpr (MODE != XENT_BWD) {
      const float xy = writer && counted && !bad ? xent_f32(x[y]) : 0.0f;
      XentStat st{-INFINITY, 0.0f, 0.0f};
      if (active)
        for (uint32_t q = q0; q < nch; q += kXentUnroll * cstep) {
          float a[kXentUnroll][8];
#pragma unroll
          for (int u = 0; u < kXentUnroll; ++u) {
            const uint32_t qu = q + u * cstep;
            if (qu < nch) xent_ld8(x + qu * 8u, vec, min(8u, v - qu * 8u), a[u]);
          }
#pragma unroll
          for (int u = 0; u < kXentUnroll; ++u) {
            const uint32_t qu = q + u * cstep;
            if (qu < nch) xent_chunk(st, a[u], min(8u, v - qu * 8u));
          }
        }
      st = xent_reduce<WARP>(g, st);
      lse = __fadd_rn(st.m, __fmul_rn(lg2(st.s), kXentLn2));
      if (writer) {
        float loss = 0.0f;
        if (bad) {
          loss = __int_as_float(0x7FC00000);
        } else if (counted) {
          loss = __fsub_rn(lse, __fmul_rn(p.omega, xy));
          if (smooth) loss = __fsub_rn(loss, __fmul_rn(p.eps_v, st.sx));
          if (zl) loss = __fadd_rn(loss, __fmul_rn(p.z, __fmul_rn(lse, lse)));
        }
        reinterpret_cast<float*>(p.loss)[r] = loss;
        if (p.lse) reinterpret_cast<float*>(p.lse)[r] = lse;
      }
    } else {
      if (active && counted && !bad) lse = reinterpret_cast<const float*>(p.lse)[r];
    }
    if constexpr (MODE != XENT_FWD) {
      if (!active) continue;
      TG* dx = reinterpret_cast<TG*>(p.dlogits) + r * p.gs;
      if (!counted || bad) {   // +0 for an ignored row, NaN for a target outside [0, v)
        float f[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) f[i] = bad ? __int_as_float(0x7FC00000) : 0.0f;
        for (uint32_t q = q0; q < nch; q += cstep) xent_st8(dx + q * 8u, vec, min(8u, v - q * 8u), f);
        continue;
      }
      const float* dl = reinterpret_cast<const float*>(p.dloss);
      float gr = p.reduction == 0 ? dl[r] : dl[0];
      if (p.reduction == 2) gr = __fdiv_rn(gr, __uint2float_rn(*reinterpret_cast<const uint32_t*>(p.count)));
      const float zf = zl ? __fadd_rn(1.0f, __fmul_rn(p.z2, lse)) : 1.0f;
      const uint32_t yc = (uint32_t)y;
      for (uint32_t q = q0; q < nch; q += kXentUnroll * cstep) {
        float a[kXentUnroll][8];
#pragma unroll
        for (int u = 0; u < kXentUnroll; ++u) {
          const uint32_t qu = q + u * cstep;
          if (qu < nch) xent_ld8(x + qu * 8u, vec, min(8u, v - qu * 8u), a[u]);
        }
#pragma unroll
        for (int u = 0; u < kXentUnroll; ++u) {
          const uint32_t qu = q + u * cstep;
          if (qu >= nch) continue;
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            float d = ex2(__fmul_rn(__fsub_rn(a[u][i], lse), kXentLog2e));
            if (zl) d = __fmul_rn(d, zf);
            if (qu * 8u + i == yc) d = __fsub_rn(d, p.omega);
            if (smooth) d = __fsub_rn(d, p.eps_v);
            a[u][i] = __fmul_rn(gr, d);
          }
          xent_st8(dx + qu * 8u, vec, min(8u, v - qu * 8u), a[u]);
        }
      }
    }
  }
}

// count[0] = the rows whose target is not ignore_index: one CTA of kXentTotalThreads; integer sums are exact in any order.
extern "C" __global__ void __launch_bounds__(kXentTotalThreads) xent_count(const __grid_constant__ XentParams p) {
  __shared__ uint32_t part[kXentTotalThreads / 32];
  uint32_t n = 0;
  for (uint64_t r = threadIdx.x; r < p.t; r += kXentTotalThreads) n += xent_target(p, r) != (int64_t)p.ignore_index ? 1u : 0u;
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) n += __shfl_xor_sync(0xFFFFFFFFu, n, o);
  if ((threadIdx.x & 31u) == 0) part[threadIdx.x >> 5] = n;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < kXentTotalThreads / 32; ++w) n += part[w];
    *reinterpret_cast<uint32_t*>(p.count) = n;
  }
}

// loss[0] = the sum of the row losses p.partials[0, t) (MEAN: divided once by count[0]): thread i adds rows i, i + 1024, ...
// in order from +0, then an xor butterfly over each warp, then the warps in order.  The order depends on t alone.
extern "C" __global__ void __launch_bounds__(kXentTotalThreads) xent_total(const __grid_constant__ XentParams p) {
  __shared__ float part[kXentTotalThreads / 32];
  const float* l = reinterpret_cast<const float*>(p.partials);
  float a = 0.0f;
  for (uint64_t r = threadIdx.x; r < p.t; r += kXentTotalThreads) a = __fadd_rn(a, l[r]);
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) a = __fadd_rn(a, __shfl_xor_sync(0xFFFFFFFFu, a, o));
  if ((threadIdx.x & 31u) == 0) part[threadIdx.x >> 5] = a;
  __syncthreads();
  if (threadIdx.x == 0) {
    a = part[0];
    for (int w = 1; w < kXentTotalThreads / 32; ++w) a = __fadd_rn(a, part[w]);
    if (p.reduction == 2) a = __fdiv_rn(a, __uint2float_rn(*reinterpret_cast<const uint32_t*>(p.count)));
    *reinterpret_cast<float*>(p.loss) = a;
  }
}

#define XENT_KERNEL(name, TX, TG, MODE)                                                                                     \
  extern "C" __global__ void __launch_bounds__(kXentThreads, MODE == XENT_FUSED ? kXentFusedCtasPerSm : kXentCtasPerSm)      \
      name##_warp(const __grid_constant__ XentParams p) {                                                                  \
    xent_rows<TX, TG, MODE, true>(p);                                                                                     \
  }                                                                                                                        \
  extern "C" __global__ void __launch_bounds__(kXentThreads, MODE == XENT_FUSED ? kXentFusedCtasPerSm : kXentCtasPerSm)      \
      name##_cta(const __grid_constant__ XentParams p) {                                                                   \
    xent_rows<TX, TG, MODE, false>(p);                                                                                    \
  }
#define XENT_GRAD(tx, TX, tg, TG) XENT_KERNEL(xent_fused_##tx##_##tg, TX, TG, XENT_FUSED) XENT_KERNEL(xent_bwd_##tx##_##tg, TX, TG, XENT_BWD)
#define XENT_ROW(tx, TX)                                                                                                   \
  XENT_KERNEL(xent_fwd_##tx, TX, float, XENT_FWD)                                                                          \
  XENT_GRAD(tx, TX, f32, float) XENT_GRAD(tx, TX, bf16, __nv_bfloat16) XENT_GRAD(tx, TX, f16, __half)
XENT_ROW(f32, float)
XENT_ROW(bf16, __nv_bfloat16)
XENT_ROW(f16, __half)
