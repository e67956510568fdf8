// Direct NHWC grouped and depthwise 2-D convolution for narrow groups (group width Cg = C / groups < 64), forward and both
// gradients (capi.cpp: b200_conv2d_grouped*).  Layers this narrow would leave most of a 64-channel k-block and a 128-wide
// wgmma tile empty; they are bound by memory or by CUDA-core FMAs, so every output element is one f32 FMA chain on the CUDA
// cores.  Lanes run over consecutive channels, so a warp's loads and stores of one pixel are contiguous.
//
// Order contract (the numpy oracle in tests/conv_grouped_oracle.py restates it):
//   forward  acc = +0; for ky, kx, ci ascending: acc = fma(x, w, acc); then the fused epilogue (epilogue.cuh)
//   dgrad    acc = +0; for ky, kx ascending, taps with (h + ph - ky dh) % sh == 0 (likewise w) only; for co in the group
//            ascending: acc = fma(dy, w, acc), dy read as +0 outside [0, OH) x [0, OW)
//   wgrad    per segment of seg_len pixels: acc = +0; for pixels ascending: acc = fma(dy, x, acc); the segments' partials
//            are then added in segment order, dw = ((p0 + p1) + p2) + ...
// Input outside x reads as +0 and is multiplied like any other element.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cstdint>

#include "epilogue.cuh"
#include "kernel_params.h"

extern __shared__ __align__(16) uint16_t grp_halo[];

template <bool BF16>
__device__ __forceinline__ float grp_f32(uint16_t b) {
  if constexpr (BF16) return __uint_as_float(static_cast<uint32_t>(b) << 16);
  else return __half2float(__ushort_as_half(b));
}
__device__ __forceinline__ void grp_put(float* o, float v) { *o = v; }
__device__ __forceinline__ void grp_put(__nv_bfloat16* o, float v) { *o = __float2bfloat16_rn(v); }
__device__ __forceinline__ void grp_put(__half* o, float v) { *o = __float2half_rn(v); }

// ------------------------------------------------------------------------------------------------ forward
// CTA: kGrpTileH x kGrpTileW output pixels of image n x kGrpChunk output channels.  Warp r owns output row oh0 + r, lane l
// output channel co0 + l, and each thread the kGrpTileW pixels of its row.  STAGED: the input halo of the chunk's input
// channels [cin_lo, cin_hi) is first copied to shared memory ([hy][hx][staged_ci], zeros outside x); otherwise x is read
// from global memory.
template <bool BF16, typename TO, bool STAGED>
__device__ __forceinline__ void grp_forward(const ConvGroupedParams& p) {
  const uint32_t lane = threadIdx.x & 31u, row = threadIdx.x >> 5;
  uint32_t b = blockIdx.x;
  const uint32_t tw = b % p.tiles_w;
  b /= p.tiles_w;
  const uint32_t th = b % p.tiles_h, n = b / p.tiles_h;
  const uint32_t co0 = blockIdx.y * kGrpChunk, co_end = min(co0 + kGrpChunk, p.Cout);
  const uint32_t cin_lo = (co0 / p.Coutg) * p.Cg;
  const int32_t oh0 = (int32_t)(th * kGrpTileH), ow0 = (int32_t)(tw * kGrpTileW);
  const int32_t iy0 = oh0 * p.sh - p.ph, ix0 = ow0 * p.sw - p.pw;
  const uint32_t hw = (kGrpTileW - 1) * p.sw + (p.KW - 1) * p.dw + 1;
  const uint16_t* x = reinterpret_cast<const uint16_t*>(p.x) + (uint64_t)n * p.x_sn;
  if constexpr (STAGED) {
    const uint32_t cin_hi = min(p.C, ((co_end - 1) / p.Coutg + 1) * p.Cg), span = cin_hi - cin_lo;
    const uint32_t hh = (kGrpTileH - 1) * p.sh + (p.KH - 1) * p.dh + 1, pitch = p.staged_ci;
    if (p.vec_x && cin_lo % 8 == 0 && span % 8 == 0) {
      const uint32_t vpp = span / 8, total = hh * hw * vpp;
      for (uint32_t i = threadIdx.x; i < total; i += blockDim.x) {
        const uint32_t v = i % vpp, px = i / vpp, hx = px % hw, hy = px / hw;
        const int32_t iy = iy0 + (int32_t)hy, ix = ix0 + (int32_t)hx;
        uint4 val = make_uint4(0u, 0u, 0u, 0u);
        if (iy >= 0 && iy < (int32_t)p.H && ix >= 0 && ix < (int32_t)p.W)
          val = __ldg(reinterpret_cast<const uint4*>(x + (uint64_t)iy * p.x_sh + (uint64_t)ix * p.x_sw + cin_lo + 8u * v));
        *reinterpret_cast<uint4*>(grp_halo + px * pitch + 8u * v) = val;
      }
    } else {
      const uint32_t total = hh * hw * span;
      for (uint32_t i = threadIdx.x; i < total; i += blockDim.x) {
        const uint32_t c = i % span, px = i / span, hx = px % hw, hy = px / hw;
        const int32_t iy = iy0 + (int32_t)hy, ix = ix0 + (int32_t)hx;
        uint16_t val = 0;
        if (iy >= 0 && iy < (int32_t)p.H && ix >= 0 && ix < (int32_t)p.W)
          val = __ldg(x + (uint64_t)iy * p.x_sh + (uint64_t)ix * p.x_sw + cin_lo + c);
        grp_halo[px * pitch + c] = val;
      }
    }
    __syncthreads();
  }
  const uint32_t co = co0 + lane;
  const int32_t oh = oh0 + (int32_t)row;
  if (co >= p.Cout || oh >= (int32_t)p.OH) return;
  const uint32_t cg = (co / p.Coutg) * p.Cg;   // the group's first input channel
  const uint16_t* w = reinterpret_cast<const uint16_t*>(p.w) + (uint64_t)co * p.w_sco;
  float acc[kGrpTileW];
#pragma unroll
  for (int j = 0; j < kGrpTileW; ++j) acc[j] = 0.f;
  for (uint32_t ky = 0; ky < p.KH; ++ky) {
    const int32_t iy = oh * p.sh - p.ph + (int32_t)(ky * p.dh);
    const bool row_in = iy >= 0 && iy < (int32_t)p.H;
    for (uint32_t kx = 0; kx < p.KW; ++kx) {
      const uint16_t* wk = w + ky * p.w_sky + kx * p.w_skx;
      for (uint32_t ci = 0; ci < p.Cg; ++ci) {
        const float wv = grp_f32<BF16>(__ldg(wk + ci));
#pragma unroll
        for (int j = 0; j < kGrpTileW; ++j) {
          float xv;
          if constexpr (STAGED) {
            const uint32_t hy = row * p.sh + ky * p.dh, hx = (uint32_t)j * p.sw + kx * p.dw;
            xv = grp_f32<BF16>(grp_halo[(hy * hw + hx) * p.staged_ci + (cg - cin_lo) + ci]);
          } else {
            const int32_t ix = (ow0 + j) * p.sw - p.pw + (int32_t)(kx * p.dw);
            xv = (row_in && ix >= 0 && ix < (int32_t)p.W) ? grp_f32<BF16>(__ldg(x + (uint64_t)iy * p.x_sh + (uint64_t)ix * p.x_sw + cg + ci)) : 0.f;
          }
          acc[j] = __fmaf_rn(xv, wv, acc[j]);
        }
      }
    }
  }
  const float* bias = reinterpret_cast<const float*>(p.bias);
  TO* out = reinterpret_cast<TO*>(p.out) + (uint64_t)n * p.o_sn + (uint64_t)oh * p.o_sh + co;
#pragma unroll
  for (int j = 0; j < kGrpTileW; ++j) {
    const int32_t ow = ow0 + j;
    if (ow >= (int32_t)p.OW) break;
    const float v = p.epi_on ? epilogue_value(acc[j], p.alpha, bias, co, p.Cout, p.epi_act) : acc[j];
    grp_put(out + (uint64_t)ow * p.o_sw, v);
  }
}

// ------------------------------------------------------------------------------------------------ data gradient
// Thread: one dx pixel (blockIdx.x * 8 + warp, over N * H * W) x one channel (blockIdx.y * kGrpChunk + lane).
template <bool BF16, typename TO>
__device__ __forceinline__ void grp_dgrad(const ConvGroupedParams& p) {
  // 32-bit index arithmetic throughout (N * H * W < 2^31, |h + ph - ky dh| < 2^31): a 64-bit division per tap costs more
  // than the tap's loads
  const uint32_t c = blockIdx.y * kGrpChunk + (threadIdx.x & 31u);
  const uint32_t pix = blockIdx.x * 8u + (threadIdx.x >> 5);
  if (c >= p.C || pix >= p.N * p.H * p.W) return;
  const uint32_t wx = pix % p.W, hy = (pix / p.W) % p.H, n = pix / (p.W * p.H);
  const uint32_t g = c / p.Cg, ci = c - g * p.Cg, co_lo = g * p.Coutg;
  const uint16_t* dy = reinterpret_cast<const uint16_t*>(p.x) + (uint64_t)n * p.x_sn;
  const uint16_t* w = reinterpret_cast<const uint16_t*>(p.w) + ci;
  float acc = 0.f;
  for (uint32_t ky = 0; ky < p.KH; ++ky) {
    const int32_t nh = (int32_t)hy + p.ph - (int32_t)ky * p.dh;
    if (nh % p.sh != 0) continue;
    const int32_t oh = nh / p.sh;
    const bool oh_in = oh >= 0 && oh < (int32_t)p.OH;
    for (uint32_t kx = 0; kx < p.KW; ++kx) {
      const int32_t nw = (int32_t)wx + p.pw - (int32_t)kx * p.dw;
      if (nw % p.sw != 0) continue;
      const int32_t ow = nw / p.sw;
      const bool in = oh_in && ow >= 0 && ow < (int32_t)p.OW;
      const uint16_t* dyp = in ? dy + (uint64_t)oh * p.x_sh + (uint64_t)ow * p.x_sw : nullptr;
      const uint16_t* wk = w + ky * p.w_sky + kx * p.w_skx;
      for (uint32_t j = 0; j < p.Coutg; ++j) {
        const uint32_t co = co_lo + j;
        const float dv = in ? grp_f32<BF16>(__ldg(dyp + co)) : 0.f;
        acc = __fmaf_rn(dv, grp_f32<BF16>(__ldg(wk + (uint64_t)co * p.w_sco)), acc);
      }
    }
  }
  grp_put(reinterpret_cast<TO*>(p.out) + (uint64_t)n * p.o_sn + (uint64_t)hy * p.o_sh + (uint64_t)wx * p.o_sw + c, acc);
}

// ------------------------------------------------------------------------------------------------ weight gradient
// Thread: dw element t = (kpos * Cout + co) * Cg + ci (lanes over ci, then co), segment blockIdx.y of seg_len pixels.
template <bool BF16, typename TO>
__device__ __forceinline__ void grp_wgrad(const ConvGroupedParams& p) {
  const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= p.elems) return;
  const uint32_t ci = (uint32_t)(t % p.Cg);
  const uint64_t r = t / p.Cg;
  const uint32_t co = (uint32_t)(r % p.Cout), kpos = (uint32_t)(r / p.Cout), kx = kpos % p.KW, ky = kpos / p.KW;
  const uint32_t c = (co / p.Coutg) * p.Cg + ci;
  const uint64_t ohw = (uint64_t)p.OH * p.OW, P = (uint64_t)p.N * ohw;
  const uint64_t p0 = (uint64_t)blockIdx.y * p.seg_len, p1 = min(p0 + p.seg_len, P);
  uint32_t n = (uint32_t)(p0 / ohw), oh = (uint32_t)((p0 % ohw) / p.OW), ow = (uint32_t)(p0 % p.OW);
  const uint16_t* x = reinterpret_cast<const uint16_t*>(p.x) + c;
  const uint16_t* dy = reinterpret_cast<const uint16_t*>(p.w) + co;
  const int32_t ky_off = (int32_t)(ky * p.dh) - p.ph, kx_off = (int32_t)(kx * p.dw) - p.pw;
  float acc = 0.f;
  for (uint64_t q = p0; q < p1; ++q) {
    const int32_t iy = (int32_t)oh * p.sh + ky_off, ix = (int32_t)ow * p.sw + kx_off;
    const float xv = (iy >= 0 && iy < (int32_t)p.H && ix >= 0 && ix < (int32_t)p.W)
                         ? grp_f32<BF16>(__ldg(x + (uint64_t)n * p.x_sn + (uint64_t)iy * p.x_sh + (uint64_t)ix * p.x_sw)) : 0.f;
    const float dv = grp_f32<BF16>(__ldg(dy + (uint64_t)n * p.y_sn + (uint64_t)oh * p.y_sh + (uint64_t)ow * p.y_sw));
    acc = __fmaf_rn(dv, xv, acc);
    if (++ow == p.OW) {
      ow = 0;
      if (++oh == p.OH) { oh = 0; ++n; }
    }
  }
  if (p.nseg > 1) reinterpret_cast<float*>(p.part)[(uint64_t)blockIdx.y * p.elems + t] = acc;
  else grp_put(reinterpret_cast<TO*>(p.out) + (uint64_t)co * p.o_sn + (uint64_t)kpos * p.o_sw + ci, acc);
}

// dw = the partials of segments 0, 1, ... added in that order.
template <typename TO>
__device__ __forceinline__ void grp_wgrad_combine(const ConvGroupedParams& p) {
  const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= p.elems) return;
  const float* part = reinterpret_cast<const float*>(p.part) + t;
  float acc = part[0];
  for (uint32_t s = 1; s < p.nseg; ++s) acc = __fadd_rn(acc, part[(uint64_t)s * p.elems]);
  const uint32_t ci = (uint32_t)(t % p.Cg);
  const uint64_t r = t / p.Cg;
  const uint32_t co = (uint32_t)(r % p.Cout), kpos = (uint32_t)(r / p.Cout);
  grp_put(reinterpret_cast<TO*>(p.out) + (uint64_t)co * p.o_sn + (uint64_t)kpos * p.o_sw + ci, acc);
}

#define GRP_KERNELS(IN, OUT, BF, TO)                                                                                       \
  extern "C" __global__ void __launch_bounds__(256) conv2d_grp_##IN##_##OUT(const __grid_constant__ ConvGroupedParams p) { \
    if (p.staged_ci) grp_forward<BF, TO, true>(p);                                                                          \
    else grp_forward<BF, TO, false>(p);                                                                                     \
  }                                                                                                                         \
  extern "C" __global__ void __launch_bounds__(256) conv2d_grp_dgrad_##IN##_##OUT(const __grid_constant__ ConvGroupedParams p) { \
    grp_dgrad<BF, TO>(p);                                                                                                   \
  }                                                                                                                         \
  extern "C" __global__ void __launch_bounds__(256) conv2d_grp_wgrad_##IN##_##OUT(const __grid_constant__ ConvGroupedParams p) { \
    grp_wgrad<BF, TO>(p);                                                                                                   \
  }

GRP_KERNELS(bf16, bf16, true, __nv_bfloat16)
GRP_KERNELS(bf16, f32, true, float)
GRP_KERNELS(f16, f16, false, __half)
GRP_KERNELS(f16, f32, false, float)

extern "C" __global__ void __launch_bounds__(256) conv2d_grp_wgrad_combine_bf16(const __grid_constant__ ConvGroupedParams p) {
  grp_wgrad_combine<__nv_bfloat16>(p);
}
extern "C" __global__ void __launch_bounds__(256) conv2d_grp_wgrad_combine_f16(const __grid_constant__ ConvGroupedParams p) {
  grp_wgrad_combine<__half>(p);
}
extern "C" __global__ void __launch_bounds__(256) conv2d_grp_wgrad_combine_f32(const __grid_constant__ ConvGroupedParams p) {
  grp_wgrad_combine<float>(p);
}
