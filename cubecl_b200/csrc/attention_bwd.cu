// Fused scaled-dot-product attention, backward (capi.cpp: b200_attention_backward): dq, dk and dv from q, k, v, the forward's
// out and lse, and dout.  P is recomputed from lse, so the [Sq, Sk] matrices never leave the SM.  Three launches:
//   attn_bwd_delta_*  CUDA cores: delta_i = sum_d dout_id * out_id (f32) and L_i = lse_i * log2 e, into the padded workspace
//                     (kernel_params.h: AttnBwdParams).  Memory-bound.
//   attn_bwd_dq_*     one CTA per (b, h, 128-query block), three warpgroups as the forward: the producer loads Q and dO once,
//                     then streams blocks of 64 keys of K and V through a two-stage ring.  Each consumer (64 query rows) forms
//                     S = Q K^T and dP = dO V^T (wgmma, both operands K-major), P and dS in registers, and dQ += dS K
//                     (register-A wgmma, K an MN-major B operand).  Causal CTAs stop at the diagonal, longest first; each
//                     consumer stops at its own diagonal block and masks only its last block.
//   attn_bwd_dkdv_*   one CTA per (b, hkv, 128-key block): K and V stay resident; the producer streams Q, dO (64 query rows)
//                     and the block's L and delta slices for every query block of every one of the G query heads of the kv
//                     head.  Each consumer (64 keys) forms S^T = K Q^T and dP^T = V dO^T, then dV += P^T dO and dK += dS^T Q
//                     (register-A wgmma, dO and Q MN-major B operands).  L and delta index columns of S^T: they are staged in
//                     shared memory with each Q and dO stage.  Causal CTAs start at the diagonal query block.
// The m64nN accumulator layout is the A-fragment layout of the k16 register operand, so P and dS need no shuffles.
// Numerics: t = s * scale_log2 with the forward's f32 scale_log2 (an explicit f32 product, never contracted, so t is the
// forward's t bit for bit); p = ex2.approx.ftz(t - L) with L = lse * log2 e formed once per row in f32; dS = p * (dP - delta)
// in f32 from the f32 p; P and dS are rounded (RNE) to the input dtype for the register-A products.  dQ, dK and dV are f32
// sums; the epilogue multiplies dQ and dK by scale in f32 and rounds once (RNE) to the grad dtype.  Masked keys (j >= Sk,
// and j > i when causal) get p = +0; query rows past Sq read L = +inf and give p = +0.  Every dq row is summed by one CTA in
// increasing key order, every dk / dv row by one CTA in (group head, query block) order: no atomics, bitwise reproducible.
//
// Compiled to a cubin (no host code here): nvcc -cubin -gencode arch=compute_90a,code=sm_90a
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "attention.cuh"
#include "kernel_params.h"
#include "ptx.cuh"

using namespace b200;

namespace {

constexpr float kLog2e = 1.44269504088896340736f;

__device__ __forceinline__ uint64_t l2_policy_evict_last() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}

__device__ __forceinline__ float2 lds_f2(uint32_t addr) {
  float2 v;
  asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr));
  return v;
}

template <int KIND>
__device__ __forceinline__ float2 unpack16(uint32_t x) {
  if constexpr (KIND == KIND_BF16) return make_float2(__uint_as_float(x << 16), __uint_as_float(x & 0xFFFF0000u));
  else return __half22float2(*reinterpret_cast<const __half2*>(&x));
}

// ------------------------------------------------------------------------------------------------ delta and L
template <int KIND, int OUT>
__device__ __forceinline__ void delta_body(const AttnBwdParams& p) {
  const uint64_t rows = static_cast<uint64_t>(p.B) * p.Hq * p.Sqp;
  const uint64_t row = static_cast<uint64_t>(blockIdx.x) * 16u + (threadIdx.x >> 4);
  const uint32_t c = threadIdx.x & 15u;                      // 8 columns of the row
  const unsigned mask = 0xFFFFu << (threadIdx.x & 16u);      // the row's half warp
  if (row >= rows) return;                                   // whole half warps leave
  float* L = reinterpret_cast<float*>(p.ws) + row;
  float* dl = L + rows;
  const uint64_t bh = row / p.Sqp;
  const uint32_t i = static_cast<uint32_t>(row - bh * p.Sqp);
  if (i >= p.Sq) {
    if (c == 0) { *L = INFINITY; *dl = 0.f; }
    return;
  }
  const uint64_t b = bh / p.Hq, h = bh - b * p.Hq;
  float acc = 0.f;
  if (c * 8u < p.D) {
    const uint4 dv = *reinterpret_cast<const uint4*>(p.dout + 2u * (b * p.d_sb + h * p.d_sh + i * p.d_ss + c * 8u));
    const uint32_t dw[4] = {dv.x, dv.y, dv.z, dv.w};
    float o[8];
    const uint64_t oe = b * p.o_sb + h * p.o_sh + i * p.o_ss + c * 8u;
    if constexpr (OUT == OUT_F32) {
      const float4 a = *reinterpret_cast<const float4*>(p.out + 4u * oe), z = *reinterpret_cast<const float4*>(p.out + 4u * oe + 16u);
      o[0] = a.x; o[1] = a.y; o[2] = a.z; o[3] = a.w; o[4] = z.x; o[5] = z.y; o[6] = z.z; o[7] = z.w;
    } else {
      const uint4 ov = *reinterpret_cast<const uint4*>(p.out + 2u * oe);
      const uint32_t ow[4] = {ov.x, ov.y, ov.z, ov.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = unpack16<KIND>(ow[e]);
        o[2 * e] = f.x;
        o[2 * e + 1] = f.y;
      }
    }
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 f = unpack16<KIND>(dw[e]);
      acc = fmaf(f.x, o[2 * e], acc);
      acc = fmaf(f.y, o[2 * e + 1], acc);
    }
  }
#pragma unroll
  for (int off = 8; off > 0; off >>= 1) acc += __shfl_xor_sync(mask, acc, off);
  if (c == 0) {
    *dl = acc;
    *L = reinterpret_cast<const float*>(p.lse)[bh * p.Sq + i] * kLog2e;
  }
}

// the first workspace row of varlen sequence b (kernel_params.h: AttnVarlenParams)
__device__ __forceinline__ uint64_t varlen_ws_start(int qs, uint32_t b) {
  return (static_cast<uint64_t>(qs) + static_cast<uint64_t>(kAttnBlock) * b) / kAttnBlock * kAttnBlock;
}

// varlen: blocks of 16 rows over (b, h, row group), nqb * 8 groups per (b, h); rows past the sequence's padded blocks leave
// at once, padded rows get L = +inf and delta = 0, and so do rows whose lse is -inf (no visible key: exp2(t - L) would be +inf)
template <int KIND, int OUT>
__device__ __forceinline__ void delta_varlen_body(const AttnVarlenParams& p) {
  const uint32_t groups = p.nqb * (kAttnBlock / 16u);
  const uint32_t bh = blockIdx.x / groups, b = bh / p.Hq, h = bh - b * p.Hq;
  const int i = static_cast<int>((blockIdx.x - bh * groups) * 16u + (threadIdx.x >> 4));
  const uint32_t c = threadIdx.x & 15u;
  const unsigned mask = 0xFFFFu << (threadIdx.x & 16u);
  int qs, Lq;
  varlen_seq(p.cu_q, b, p.Tq, p.max_q, qs, Lq);
  if (i >= (Lq + kAttnBlock - 1) / kAttnBlock * kAttnBlock) return;   // whole half warps leave
  const uint64_t start = varlen_ws_start(qs, b);
  float* L = reinterpret_cast<float*>(p.ws) + static_cast<uint64_t>(h) * p.Tqp + start + i;
  float* dl = L + static_cast<uint64_t>(p.Hq) * p.Tqp;
  if (i >= Lq) {
    if (c == 0) { *L = INFINITY; *dl = 0.f; }
    return;
  }
  const uint64_t tok = static_cast<uint64_t>(qs) + i;
  float acc = 0.f;
  if (c * 8u < p.D) {
    const uint4 dv = *reinterpret_cast<const uint4*>(p.dout + 2u * (tok * p.d_st + h * p.d_sh + c * 8u));
    const uint32_t dw[4] = {dv.x, dv.y, dv.z, dv.w};
    float o[8];
    const uint64_t oe = tok * p.o_st + h * p.o_sh + c * 8u;
    if constexpr (OUT == OUT_F32) {
      const float4 a = *reinterpret_cast<const float4*>(p.out + 4u * oe), z = *reinterpret_cast<const float4*>(p.out + 4u * oe + 16u);
      o[0] = a.x; o[1] = a.y; o[2] = a.z; o[3] = a.w; o[4] = z.x; o[5] = z.y; o[6] = z.z; o[7] = z.w;
    } else {
      const uint4 ov = *reinterpret_cast<const uint4*>(p.out + 2u * oe);
      const uint32_t ow[4] = {ov.x, ov.y, ov.z, ov.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = unpack16<KIND>(ow[e]);
        o[2 * e] = f.x;
        o[2 * e + 1] = f.y;
      }
    }
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 f = unpack16<KIND>(dw[e]);
      acc = fmaf(f.x, o[2 * e], acc);
      acc = fmaf(f.y, o[2 * e + 1], acc);
    }
  }
#pragma unroll
  for (int off = 8; off > 0; off >>= 1) acc += __shfl_xor_sync(mask, acc, off);
  if (c == 0) {
    const float lse = reinterpret_cast<const float*>(p.lse)[static_cast<uint64_t>(h) * p.Tq + tok];
    *dl = lse == -INFINITY ? 0.f : acc;
    *L = lse == -INFINITY ? INFINITY : lse * kLog2e;
  }
}

// ------------------------------------------------------------------------------------------------ shared epilogue
// acc (one consumer's m64 x DB f32 fragment) times mul, rounded to the grad dtype, staged in the consumer's 64 rows of a
// SWIZZLE_128B tile (chunks of `chunk` bytes, the consumer's rows `rows_off` bytes in) and stored through 4-D TMA stores
// that the unit clips at the tensor's S and D.  The staging rows are read by no other warpgroup.
// VL with rows_left < 64 (a varlen block the sequence ends inside; a TMA box would write the next sequence's rows): the
// staged rows < rows_left are copied out with 16-byte stores to gbase + row * gst (bytes) instead.
template <int DB, int OUT, bool VL = false>
__device__ __forceinline__ void store_rows(const float (&acc)[DB / 2], float mul, uint32_t tile, uint32_t chunk, uint32_t rows_off,
                                           const CUtensorMap* tm, int row0, uint32_t rows, int h, int b, uint32_t D, uint32_t cw,
                                           int rows_left = 64, uint64_t gbase = 0, uint64_t gst = 0) {
  constexpr int NCH = DB / 64;
  constexpr uint32_t OSZ = (OUT == OUT_F32) ? 4u : 2u;
  constexpr int CW = 128 / OSZ;        // output columns per 128-byte staging row
  constexpr int NST = DB / CW;         // TMA stores
  const uint32_t t = threadIdx.x & 127u, lane = t & 31u;
  const uint32_t r = (t >> 5) * 16u + (lane >> 2), col = 2u * (lane & 3u);
#pragma unroll
  for (int c = 0; c < NST; ++c) {
    const uint32_t buf = tile + (c % NCH) * chunk + rows_off;
    if (c >= NCH) {   // the buffer is reused: the store that read it has finished reading
      if (t == 0) tma_store_wait_read<0>();
      asm volatile("bar.sync %0, 128;" ::"r"(1u + cw) : "memory");
    }
#pragma unroll
    for (int jj = 0; jj < CW / 8; ++jj) {
      const int j = c * (CW / 8) + jj;
      const uint32_t cb = (8u * jj + col) * OSZ;
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const uint32_t rr = r + 8u * hh;
        const uint32_t addr = buf + rr * 128u + ((((cb >> 4) ^ (rr & 7u)) << 4) | (cb & 15u));
        const float x0 = acc[4 * j + 2 * hh] * mul, x1 = acc[4 * j + 2 * hh + 1] * mul;
        if constexpr (OUT == OUT_F32) {
          asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(x0), "f"(x1) : "memory");
        } else {
          asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(pack16<OUT == OUT_BF16 ? KIND_BF16 : KIND_F16>(x0, x1)) : "memory");
        }
      }
    }
    fence_proxy_async_smem();   // generic-proxy writes -> visible to the TMA unit
    asm volatile("bar.sync %0, 128;" ::"r"(1u + cw) : "memory");
    if constexpr (VL) {
      if (rows_left < 64) {
        for (int u = static_cast<int>(t); u < rows_left * 8; u += 128) {
          const uint32_t rr = static_cast<uint32_t>(u) >> 3, k = static_cast<uint32_t>(u) & 7u;
          const uint32_t cc = c * CW + k * (16u / OSZ);
          if (cc >= D) continue;
          uint4 x;
          asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(x.x), "=r"(x.y), "=r"(x.z), "=r"(x.w)
                       : "r"(buf + rr * 128u + ((k ^ (rr & 7u)) << 4)));
          *reinterpret_cast<uint4*>(gbase + rr * gst + cc * OSZ) = x;
        }
        continue;
      }
    }
    if (t == 0 && row0 < static_cast<int>(rows) && c * CW < static_cast<int>(D)) {
      tma_store_4d(tm, buf, c * CW, row0, h, b);
      tma_store_commit();
    }
  }
}

// ------------------------------------------------------------------------------------------------ dq
// VL: the varlen kernels (P = AttnVarlenParams); the dense kernels have VL = false and P = AttnBwdParams
template <int KIND, int DB, int OUT, bool VL, class P>
__device__ __forceinline__ void dq_body(const CUtensorMap* tq, const CUtensorMap* tk, const CUtensorMap* tv, const CUtensorMap* tdo,
                                        const CUtensorMap* tdq, const P& p) {
  constexpr int NCH = DB / 64;
  constexpr int KB = kAttnBwdDqKeys;
  static_assert(KB == 64 && kAttnBlock == 128, "two consumers of 64 query rows, 64-key blocks");
  constexpr uint32_t QCHUNK = kAttnBlock * 128u, QTILE = NCH * QCHUNK;
  constexpr uint32_t KCHUNK = KB * 128u, KTILE = NCH * KCHUNK;
  constexpr int NA = DB / 2;   // dQ accumulators per thread (m64 x DB)
  constexpr int NS = KB / 2;   // S and dP accumulators per thread (m64 x KB)
  constexpr uint32_t ST = kAttnBwdStages;

  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sq = base, sdo = base + QTILE;
  auto sk = [&](uint32_t s) { return base + 2u * QTILE + KTILE * (2u * s); };
  auto sv = [&](uint32_t s) { return base + 2u * QTILE + KTILE * (2u * s + 1u); };
  const uint32_t bars = base + 2u * QTILE + 2u * ST * KTILE;
  const uint32_t q_bar = bars;
  auto full_k = [&](uint32_t s) { return bars + 8u * (1u + s); };
  auto full_v = [&](uint32_t s) { return bars + 8u * (1u + ST + s); };
  auto empty = [&](uint32_t s) { return bars + 8u * (1u + 2u * ST + s); };

  // work: query block (last first), head, batch -- the forward's order
  const uint32_t per = p.Hq * p.B;
  const uint32_t qb = p.nqb - 1u - blockIdx.x / per;
  const uint32_t rem = blockIdx.x % per;
  const uint32_t b = rem / p.Hq, h = rem - b * p.Hq, hk = h / p.group;
  const int q0 = static_cast<int>(qb * kAttnBlock);
  // key blocks [kb_lo, nkb); rows and keys are addressed at (qrow, krow) + block offsets in head h / hk of batch bb
  uint32_t kb_lo = 0, nkb, nkb_all = 0;
  int qrow = q0, krow = 0, bb = static_cast<int>(b), qs = 0;
  int Lq = 0, Lk = 0, off = 0;   // varlen: the sequence's lengths, off = Lk - Lq
  if constexpr (VL) {
    int ks;
    varlen_seq(p.cu_q, b, p.Tq, p.max_q, qs, Lq);
    varlen_seq(p.cu_k, b, p.Tk, p.max_k, ks, Lk);
    if (q0 >= Lq) return;   // past the sequence: no load, no store
    off = Lk - Lq;
    int lo, hi;
    band_blocks(q0, min(q0 + kAttnBlock, Lq) - 1, off, p.left, p.right, Lk, KB, lo, hi);
    kb_lo = static_cast<uint32_t>(lo);
    nkb = static_cast<uint32_t>(hi);
    qrow = qs + q0;
    krow = ks;
    bb = 0;
  } else {
    nkb_all = (p.Sk + KB - 1) / KB;
    nkb = p.causal ? min(nkb_all, 2u * qb + 2u) : nkb_all;
  }

  const uint32_t wg = threadIdx.x >> 7;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(tq);
    tma_prefetch_desc(tk);
    tma_prefetch_desc(tv);
    tma_prefetch_desc(tdo);
    tma_prefetch_desc(tdq);
    mbar_init(q_bar, 1);
    for (uint32_t s = 0; s < ST; ++s) {
      mbar_init(full_k(s), 1);
      mbar_init(full_v(s), 1);
      mbar_init(empty(s), 2);   // one arrive per consumer warpgroup
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ===================================================================== TMA producer (one thread)
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      mbar_arrive_expect_tx(q_bar, 2u * QTILE);
#pragma unroll
      for (int c = 0; c < NCH; ++c) {
        tma_load_4d(sq + c * QCHUNK, tq, q_bar, c * 64, qrow, static_cast<int>(h), bb);
        tma_load_4d(sdo + c * QCHUNK, tdo, q_bar, c * 64, qrow, static_cast<int>(h), bb);
      }
      uint32_t s = 0, ph = 0;
      for (uint32_t kb = kb_lo; kb < nkb; ++kb) {
        mbar_wait(empty(s), ph ^ 1u);
        const int k0 = krow + static_cast<int>(kb * KB);
        mbar_arrive_expect_tx(full_k(s), KTILE);
#pragma unroll
        for (int c = 0; c < NCH; ++c) tma_load_4d(sk(s) + c * KCHUNK, tk, full_k(s), c * 64, k0, static_cast<int>(hk), bb);
        mbar_arrive_expect_tx(full_v(s), KTILE);
#pragma unroll
        for (int c = 0; c < NCH; ++c) tma_load_4d(sv(s) + c * KCHUNK, tv, full_v(s), c * 64, k0, static_cast<int>(hk), bb);
        if (++s == ST) { s = 0; ph ^= 1u; }
      }
    }
    return;
  }

  // ======================================================================= consumers: 64 query rows each
  setmaxnreg_inc<232>();
  const uint32_t cw = wg - 1u;
  const uint32_t t = threadIdx.x & 127u;
  const uint32_t lane = t & 31u, wq = t >> 5;
  const uint32_t r = wq * 16u + (lane >> 2);
  const uint32_t i0 = qb * kAttnBlock + cw * 64u + r, i1 = i0 + 8u;
  const uint32_t col = 2u * (lane & 3u);
  const float c2 = p.scale_log2;
  // a causal consumer stops at its own diagonal block: keys < q0 + 64 (cw + 1).  varlen: the consumer's rows reach key
  // blocks [kbc_lo, kbc_hi); blocks inside keys [lo of its last row, hi of its first] need no mask
  uint32_t nkb_c = 0;
  int kbc_lo = 0, kbc_hi = 0, lo_c = 0, hi_c = 0;
  uint64_t plane, rb;
  if constexpr (VL) {
    const int c0 = q0 + static_cast<int>(cw * 64u);
    if (c0 < Lq) band_blocks(c0, min(c0 + 64, Lq) - 1, off, p.left, p.right, Lk, KB, kbc_lo, kbc_hi);
    lo_c = band_lo(c0 + 63, off, p.left, Lk);
    hi_c = band_hi(c0, off, p.right, Lk);
    plane = static_cast<uint64_t>(p.Hq) * p.Tqp;
    rb = static_cast<uint64_t>(h) * p.Tqp + varlen_ws_start(qs, b);
  } else {
    nkb_c = p.causal ? min(nkb_all, 2u * qb + cw + 1u) : nkb_all;
    plane = static_cast<uint64_t>(p.B) * p.Hq * p.Sqp;
    rb = (static_cast<uint64_t>(b) * p.Hq + h) * p.Sqp;
  }
  const float* ws = reinterpret_cast<const float*>(p.ws);
  const float L0 = ws[rb + i0], L1 = ws[rb + i1];
  const float dl0 = ws[plane + rb + i0], dl1 = ws[plane + rb + i1];

  float dq[NA];
#pragma unroll
  for (int i = 0; i < NA; ++i) dq[i] = 0.f;

  mbar_wait(q_bar, 0);
  uint32_t s = 0, ph = 0;
  for (uint32_t kb = kb_lo; kb < nkb; ++kb) {
    bool skip;
    if constexpr (VL) skip = static_cast<int>(kb) < kbc_lo || static_cast<int>(kb) >= kbc_hi;
    else skip = kb >= nkb_c;
    if (skip) {   // past this consumer's diagonal (varlen: outside its rows' band): release the stage once it has landed
      mbar_wait(full_k(s), ph);
      mbar_wait(full_v(s), ph);
      if (t == 0) mbar_arrive(empty(s));
      if (++s == ST) { s = 0; ph ^= 1u; }
      continue;
    }
    // ---- S = Q K^T and dP = dO V^T
    float sc[NS], dp[NS];
    mbar_wait(full_k(s), ph);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < DB / 16; ++kk) {
      const uint32_t ch = kk / 4, off = 2u * (kk % 4);
      const uint64_t da = make_smem_desc_sw128(sq + ch * QCHUNK + cw * 64u * 128u, 16, 1024) + off;
      const uint64_t db = make_smem_desc_sw128(sk(s) + ch * KCHUNK, 16, 1024) + off;
      wgmma_ss<KB, KIND, KIND, 0, 0>(sc, da, db, kk != 0 ? 1u : 0u);
    }
    wgmma_commit();
    mbar_wait(full_v(s), ph);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < DB / 16; ++kk) {
      const uint32_t ch = kk / 4, off = 2u * (kk % 4);
      const uint64_t da = make_smem_desc_sw128(sdo + ch * QCHUNK + cw * 64u * 128u, 16, 1024) + off;
      const uint64_t db = make_smem_desc_sw128(sv(s) + ch * KCHUNK, 16, 1024) + off;
      wgmma_ss<KB, KIND, KIND, 0, 0>(dp, da, db, kk != 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_operands(sc);
    wgmma_fence_operands(dp);

    // ---- p = exp2(t - L) (masked on the consumer's last block; varlen: on every block the band or Lk cuts, with dS a select
    // too, since dP of keys past Lk reads the next sequence's V), dS = p (dP - delta), both to 16 bits in the A layout
    bool last;
    if constexpr (VL) last = static_cast<int>(kb * KB) < lo_c || static_cast<int>(kb * KB) + KB - 1 > hi_c;
    else last = kb + 1u == nkb_c;
    const uint32_t key0 = kb * KB + col;
    int lo0 = 0, hi0 = 0, lo1 = 0, hi1 = 0;   // varlen: this thread's rows see keys [lo, hi]
    if constexpr (VL) {
      if (last) {
        lo0 = band_lo(static_cast<int>(i0), off, p.left, Lk);
        hi0 = band_hi(static_cast<int>(i0), off, p.right, Lk);
        lo1 = band_lo(static_cast<int>(i1), off, p.left, Lk);
        hi1 = band_hi(static_cast<int>(i1), off, p.right, Lk);
      }
    }
    uint32_t ds[NS / 2];
#pragma unroll
    for (int j = 0; j < KB / 8; ++j) {
      float v[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float pv = ex2(__fmul_rn(sc[4 * j + e], c2) - (e < 2 ? L0 : L1));
        if constexpr (VL) {
          const int kk = static_cast<int>(key0 + 8u * j + (e & 1));
          const bool hide = last && ((e < 2) ? (kk < lo0 || kk > hi0) : (kk < lo1 || kk > hi1));
          if (hide) pv = 0.f;
          v[e] = hide ? 0.f : pv * (dp[4 * j + e] - (e < 2 ? dl0 : dl1));
        } else {
          if (last) {
            const uint32_t key = key0 + 8u * j + (e & 1);
            const uint32_t row = (e < 2) ? i0 : i1;
            if (key >= p.Sk || (p.causal && key > row)) pv = 0.f;
          }
          v[e] = pv * (dp[4 * j + e] - (e < 2 ? dl0 : dl1));
        }
      }
      ds[2 * j] = pack16<KIND>(v[0], v[1]);
      ds[2 * j + 1] = pack16<KIND>(v[2], v[3]);
    }

    // ---- dQ += dS K: K [keys, D] is an MN-major B operand, 16 keys (2048 bytes of rows) per instruction
    if constexpr (VL) {   // K rows past Lk are the next sequence's (0 * NaN = NaN in the product): zero them
      const int valid = Lk - static_cast<int>(kb * KB);
      if (valid < KB) zero_rows(sk(s), NCH, KCHUNK, valid, KB, 1u + cw);
    }
    wgmma_fence_operands(dq);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < KB / 16; ++kk) {
      const uint64_t db = make_smem_desc_sw128(sk(s) + kk * 2048u, KCHUNK, 1024);
      const uint32_t a[4] = {ds[4 * kk], ds[4 * kk + 1], ds[4 * kk + 2], ds[4 * kk + 3]};
      wgmma_rs<DB, KIND, 1>(dq, a, db, 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_operands(dq);
    if (t == 0) mbar_arrive(empty(s));
    if (++s == ST) { s = 0; ph ^= 1u; }
  }

  // ---- epilogue: scale * dQ through the consumer's rows of the Q tile
  if constexpr (VL) {
    const int row0 = q0 + static_cast<int>(cw * 64u);
    constexpr uint32_t GSZ = OUT == OUT_F32 ? 4u : 2u;
    // rows past Lq belong to the next sequence: a block the sequence ends inside is copied out row by row (none when the
    // consumer's rows all lie past Lq)
    store_rows<DB, OUT, true>(dq, p.scale, sq, QCHUNK, cw * 64u * 128u, tdq, qrow + static_cast<int>(cw * 64u), p.Tq, static_cast<int>(h),
                              0, p.D, cw, min(Lq - row0, 64), p.dq + GSZ * ((qrow + cw * 64u) * p.dq_st + h * p.dq_sh), GSZ * p.dq_st);
  } else {
    store_rows<DB, OUT>(dq, p.scale, sq, QCHUNK, cw * 64u * 128u, tdq, q0 + static_cast<int>(cw * 64u), p.Sq, static_cast<int>(h),
                        static_cast<int>(b), p.D, cw);
  }
  if (t == 0) tma_store_wait<0>();   // outstanding stores read this CTA's shared memory: finish before exit
}

// ------------------------------------------------------------------------------------------------ dk, dv
// the dk / dv kernel's block order: key-block major when causal (varlen: never)
[[maybe_unused]] __device__ __forceinline__ uint32_t causal_order(const AttnBwdParams& p) { return p.causal; }
[[maybe_unused]] __device__ __forceinline__ uint32_t causal_order(const AttnVarlenParams&) { return 0u; }

template <int KIND, int DB, int OUT, bool VL, class P>
__device__ __forceinline__ void dkdv_body(const CUtensorMap* tq, const CUtensorMap* tk, const CUtensorMap* tv, const CUtensorMap* tdo,
                                          const CUtensorMap* tdk, const CUtensorMap* tdv, const P& p) {
  constexpr int NCH = DB / 64;
  constexpr int QB = kAttnBwdDkdvQueries;
  static_assert(QB == 64 && kAttnBlock == 128, "two consumers of 64 keys, 64-query blocks");
  constexpr uint32_t KCHUNK = kAttnBlock * 128u, KTILE = NCH * KCHUNK;
  constexpr uint32_t QCHUNK = QB * 128u, QTILE = NCH * QCHUNK;
  constexpr int NA = DB / 2;   // dK and dV accumulators per thread (m64 x DB each)
  constexpr int NS = QB / 2;   // S^T and dP^T accumulators per thread (m64 x QB)
  constexpr uint32_t ST = kAttnBwdStages;

  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sk = base, sv = base + KTILE;
  auto sq = [&](uint32_t s) { return base + 2u * KTILE + QTILE * (2u * s); };
  auto sdo = [&](uint32_t s) { return base + 2u * KTILE + QTILE * (2u * s + 1u); };
  const uint32_t vecs = base + 2u * KTILE + 2u * ST * QTILE;
  auto sl = [&](uint32_t s) { return vecs + s * 2u * QB * 4u; };            // L of the stage's query rows
  auto sd = [&](uint32_t s) { return vecs + s * 2u * QB * 4u + QB * 4u; };  // delta
  const uint32_t bars = vecs + ST * 2u * QB * 4u;
  const uint32_t kv_bar = bars;
  auto full_q = [&](uint32_t s) { return bars + 8u * (1u + s); };
  auto full_do = [&](uint32_t s) { return bars + 8u * (1u + ST + s); };
  auto empty = [&](uint32_t s) { return bars + 8u * (1u + 2u * ST + s); };

  // work: see AttnBwdParams (varlen: the non-causal order)
  const uint32_t Hkv = p.Hkv;
  const uint32_t per = p.B * Hkv;
  const uint32_t kb = causal_order(p) ? blockIdx.x / per : blockIdx.x % p.nkb;
  const uint32_t rem = causal_order(p) ? blockIdx.x % per : blockIdx.x / p.nkb;
  const uint32_t b = rem / Hkv, hk = rem - b * Hkv;
  const uint32_t k0 = kb * kAttnBlock;
  // query blocks [qb0, qb0 + per_head) of every group head; rows and keys at (qrow, krow) + block offsets in batch bb
  uint32_t qb0, per_head;
  int qrow = 0, krow = 0, bb = static_cast<int>(b), qs = 0;
  int Lq = 0, Lk = 0, off = 0;   // varlen: the sequence's lengths, off = Lk - Lq
  if constexpr (VL) {
    int ks;
    varlen_seq(p.cu_q, b, p.Tq, p.max_q, qs, Lq);
    varlen_seq(p.cu_k, b, p.Tk, p.max_k, ks, Lk);
    if (static_cast<int>(k0) >= Lk) return;   // past the sequence: no load, no store
    off = Lk - Lq;
    int lo, hi;
    band_blocks(static_cast<int>(k0), min(static_cast<int>(k0) + kAttnBlock, Lk) - 1, -off, p.right, p.left, Lq, QB, lo, hi);
    qb0 = static_cast<uint32_t>(lo);
    per_head = static_cast<uint32_t>(hi - lo);
    qrow = qs;
    krow = ks;
    bb = 0;
  } else {
    qb0 = p.causal ? k0 / QB : 0u;                                    // the diagonal query block
    per_head = p.nqd > qb0 ? p.nqd - qb0 : 0u;
  }
  const uint32_t steps = p.group * per_head;                          // group == 0 when Hq == 0

  const uint32_t wg = threadIdx.x >> 7;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(tq);
    tma_prefetch_desc(tk);
    tma_prefetch_desc(tv);
    tma_prefetch_desc(tdo);
    tma_prefetch_desc(tdk);
    tma_prefetch_desc(tdv);
    mbar_init(kv_bar, 1);
    for (uint32_t s = 0; s < ST; ++s) {
      mbar_init(full_q(s), 1);
      mbar_init(full_do(s), 1);
      mbar_init(empty(s), 2);
    }
    fence_mbar_init();
  }
  __syncthreads();

  uint64_t plane, wsb;   // the workspace's delta plane; the sequence's first row (dense: the batch's, per head Sqp rows)
  if constexpr (VL) {
    plane = static_cast<uint64_t>(p.Hq) * p.Tqp;
    wsb = varlen_ws_start(qs, b);
  } else {
    plane = static_cast<uint64_t>(p.B) * p.Hq * p.Sqp;
    wsb = 0;
  }
  if (wg == 0) {
    // ===================================================================== TMA producer (one thread)
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      mbar_arrive_expect_tx(kv_bar, 2u * KTILE);
#pragma unroll
      for (int c = 0; c < NCH; ++c) {
        tma_load_4d(sk + c * KCHUNK, tk, kv_bar, c * 64, krow + static_cast<int>(k0), static_cast<int>(hk), bb);
        tma_load_4d(sv + c * KCHUNK, tv, kv_bar, c * 64, krow + static_cast<int>(k0), static_cast<int>(hk), bb);
      }
      const uint64_t pol = l2_policy_evict_last();   // every key block of the head reads these slices
      const uint8_t* ws = reinterpret_cast<const uint8_t*>(p.ws);
      uint32_t s = 0, ph = 0;
      for (uint32_t step = 0; step < steps; ++step) {
        const uint32_t g = step / per_head, qb = qb0 + step % per_head;
        const uint32_t h = hk * p.group + g;
        const int q0 = static_cast<int>(qb * QB);
        uint64_t row;
        if constexpr (VL) row = static_cast<uint64_t>(h) * p.Tqp + wsb + static_cast<uint64_t>(q0);
        else row = (static_cast<uint64_t>(b) * p.Hq + h) * p.Sqp + static_cast<uint64_t>(q0);
        mbar_wait(empty(s), ph ^ 1u);
        mbar_arrive_expect_tx(full_q(s), QTILE + QB * 4u);
#pragma unroll
        for (int c = 0; c < NCH; ++c) tma_load_4d(sq(s) + c * QCHUNK, tq, full_q(s), c * 64, qrow + q0, static_cast<int>(h), bb);
        bulk_load_1d(sl(s), ws + 4u * row, QB * 4u, full_q(s), pol);
        mbar_arrive_expect_tx(full_do(s), QTILE + QB * 4u);
#pragma unroll
        for (int c = 0; c < NCH; ++c) tma_load_4d(sdo(s) + c * QCHUNK, tdo, full_do(s), c * 64, qrow + q0, static_cast<int>(h), bb);
        bulk_load_1d(sd(s), ws + 4u * (plane + row), QB * 4u, full_do(s), pol);
        if (++s == ST) { s = 0; ph ^= 1u; }
      }
    }
    return;
  }

  // ======================================================================= consumers: 64 keys each
  setmaxnreg_inc<232>();
  const uint32_t cw = wg - 1u;
  const uint32_t t = threadIdx.x & 127u;
  const uint32_t lane = t & 31u, wq = t >> 5;
  const uint32_t r = wq * 16u + (lane >> 2);
  const uint32_t j0 = k0 + cw * 64u + r, j1 = j0 + 8u;   // this thread's two key rows
  const uint32_t col = 2u * (lane & 3u);
  const float c2 = p.scale_log2;
  // this consumer's diagonal query block (varlen: every block of the CTA's range runs, masked where the band or Lq cuts it)
  uint32_t qb_c = 0;
  if constexpr (!VL) qb_c = p.causal ? (k0 + cw * 64u) / QB : 0u;

  float dk[NA], dv[NA];
#pragma unroll
  for (int i = 0; i < NA; ++i) dk[i] = dv[i] = 0.f;

  mbar_wait(kv_bar, 0);
  uint32_t s = 0, ph = 0;
  for (uint32_t step = 0; step < steps; ++step) {
    const uint32_t qb = qb0 + step % per_head;
    bool skip = false;
    if constexpr (!VL) skip = qb < qb_c;
    if (skip) {   // every query of the block is above this consumer's keys: release the stage once it has landed
      mbar_wait(full_q(s), ph);
      mbar_wait(full_do(s), ph);
      if (t == 0) mbar_arrive(empty(s));
      if (++s == ST) { s = 0; ph ^= 1u; }
      continue;
    }
    // ---- S^T = K Q^T and dP^T = V dO^T
    float st[NS], dpt[NS];
    mbar_wait(full_q(s), ph);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < DB / 16; ++kk) {
      const uint32_t ch = kk / 4, off = 2u * (kk % 4);
      const uint64_t da = make_smem_desc_sw128(sk + ch * KCHUNK + cw * 64u * 128u, 16, 1024) + off;
      const uint64_t db = make_smem_desc_sw128(sq(s) + ch * QCHUNK, 16, 1024) + off;
      wgmma_ss<QB, KIND, KIND, 0, 0>(st, da, db, kk != 0 ? 1u : 0u);
    }
    wgmma_commit();
    mbar_wait(full_do(s), ph);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < DB / 16; ++kk) {
      const uint32_t ch = kk / 4, off = 2u * (kk % 4);
      const uint64_t da = make_smem_desc_sw128(sv + ch * KCHUNK + cw * 64u * 128u, 16, 1024) + off;
      const uint64_t db = make_smem_desc_sw128(sdo(s) + ch * QCHUNK, 16, 1024) + off;
      wgmma_ss<QB, KIND, KIND, 0, 0>(dpt, da, db, kk != 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_operands(st);
    wgmma_fence_operands(dpt);

    // ---- P^T and dS^T (columns are queries: L and delta from the stage), the causal mask on the diagonal block only (varlen:
    // on every block the band or Lq cuts, dS^T a select too)
    bool diag;
    if constexpr (VL) {   // some (key, query) pair of the consumer's 64 keys and this block is hidden
      const int c0 = static_cast<int>(k0 + cw * 64u), i0 = static_cast<int>(qb * QB);
      diag = i0 < band_lo(c0 + 63, -off, p.right, Lq) || i0 + QB - 1 > band_hi(c0, -off, p.left, Lq);
    } else {
      diag = p.causal && qb == qb_c;
    }
    const uint32_t qcol0 = qb * QB + col;
    // varlen: query i sees key j iff i < Lq and -right <= i - j + off <= left (host: |i - j + off| < 2^31); d0 is that
    // difference for this thread's first key and column pair
    const int d0 = static_cast<int>(qcol0) - static_cast<int>(j0) + off;
    uint32_t pa[NS / 2], da[NS / 2];
#pragma unroll
    for (int j = 0; j < QB / 8; ++j) {
      const float2 lv = lds_f2(sl(s) + (8u * j + col) * 4u);
      const float2 dl = lds_f2(sd(s) + (8u * j + col) * 4u);
      float pv[4], v[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float x = ex2(__fmul_rn(st[4 * j + e], c2) - ((e & 1) ? lv.y : lv.x));
        if constexpr (VL) {
          const int qi = static_cast<int>(qcol0 + 8u * j + (e & 1)), d = d0 + 8 * j + (e & 1) - ((e < 2) ? 0 : 8);
          const bool hide = diag && (qi >= Lq || (p.right >= 0 && d < -p.right) || (p.left >= 0 && d > p.left));
          pv[e] = hide ? 0.f : x;
          v[e] = hide ? 0.f : x * (dpt[4 * j + e] - ((e & 1) ? dl.y : dl.x));
        } else {
          if (diag && ((e < 2) ? j0 : j1) > qcol0 + 8u * j + (e & 1)) x = 0.f;
          pv[e] = x;
          v[e] = x * (dpt[4 * j + e] - ((e & 1) ? dl.y : dl.x));
        }
      }
      pa[2 * j] = pack16<KIND>(pv[0], pv[1]);
      pa[2 * j + 1] = pack16<KIND>(pv[2], pv[3]);
      da[2 * j] = pack16<KIND>(v[0], v[1]);
      da[2 * j + 1] = pack16<KIND>(v[2], v[3]);
    }

    // ---- dV += P^T dO and dK += dS^T Q: dO and Q [queries, D] are MN-major B operands
    if constexpr (VL) {   // Q and dO rows past Lq are the next sequence's (0 * NaN = NaN in the products): zero them
      const int valid = Lq - static_cast<int>(qb * QB);
      if (valid < QB) {
        zero_rows(sq(s), NCH, QCHUNK, valid, QB, 1u + cw);
        zero_rows(sdo(s), NCH, QCHUNK, valid, QB, 1u + cw);
      }
    }
    wgmma_fence_operands(dv);
    wgmma_fence_operands(dk);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < QB / 16; ++kk) {
      const uint64_t db = make_smem_desc_sw128(sdo(s) + kk * 2048u, QCHUNK, 1024);
      const uint32_t a[4] = {pa[4 * kk], pa[4 * kk + 1], pa[4 * kk + 2], pa[4 * kk + 3]};
      wgmma_rs<DB, KIND, 1>(dv, a, db, 1u);
    }
#pragma unroll
    for (int kk = 0; kk < QB / 16; ++kk) {
      const uint64_t db = make_smem_desc_sw128(sq(s) + kk * 2048u, QCHUNK, 1024);
      const uint32_t a[4] = {da[4 * kk], da[4 * kk + 1], da[4 * kk + 2], da[4 * kk + 3]};
      wgmma_rs<DB, KIND, 1>(dk, a, db, 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_operands(dv);
    wgmma_fence_operands(dk);
    if (t == 0) mbar_arrive(empty(s));
    if (++s == ST) { s = 0; ph ^= 1u; }
  }

  // ---- epilogue: scale * dK through the consumer's rows of the K tile, dV through its rows of the V tile
  const int row0 = static_cast<int>(k0 + cw * 64u);
  if constexpr (VL) {
    constexpr uint32_t GSZ = OUT == OUT_F32 ? 4u : 2u;
    // rows past Lk belong to the next sequence: a block the sequence ends inside is copied out row by row (none when the
    // consumer's rows all lie past Lk)
    const int left = min(Lk - row0, 64);
    const uint64_t r = static_cast<uint64_t>(krow + row0);
    store_rows<DB, OUT, true>(dk, p.scale, sk, KCHUNK, cw * 64u * 128u, tdk, krow + row0, p.Tk, static_cast<int>(hk), 0, p.D, cw, left,
                              p.dk + GSZ * (r * p.dk_st + hk * p.dk_sh), GSZ * p.dk_st);
    store_rows<DB, OUT, true>(dv, 1.0f, sv, KCHUNK, cw * 64u * 128u, tdv, krow + row0, p.Tk, static_cast<int>(hk), 0, p.D, cw, left,
                              p.dv + GSZ * (r * p.dv_st + hk * p.dv_sh), GSZ * p.dv_st);
  } else {
    store_rows<DB, OUT>(dk, p.scale, sk, KCHUNK, cw * 64u * 128u, tdk, row0, p.Sk, static_cast<int>(hk), static_cast<int>(b), p.D, cw);
    store_rows<DB, OUT>(dv, 1.0f, sv, KCHUNK, cw * 64u * 128u, tdv, row0, p.Sk, static_cast<int>(hk), static_cast<int>(b), p.D, cw);
  }
  if (t == 0) tma_store_wait<0>();
}

}  // namespace

// attn_bwd_delta_<in>_<out>: out in the input dtype or f32; varlen (compiled with -DATTN_VARLEN into its own cubin):
// attn_bwd_varlen_{delta,dq,dkdv}_...
#ifdef ATTN_VARLEN
#define BWD_VL true
#define BWD_P AttnVarlenParams
#define BWD_NAME(K, REST) attn_bwd_varlen_##K##_##REST
#define DELTA_KERNEL(NAME, KIND, OUT) \
  extern "C" __global__ void __launch_bounds__(256) NAME(const __grid_constant__ AttnVarlenParams p) { delta_varlen_body<KIND, OUT>(p); }
#else
#define BWD_VL false
#define BWD_P AttnBwdParams
#define BWD_NAME(K, REST) attn_bwd_##K##_##REST
#define DELTA_KERNEL(NAME, KIND, OUT) \
  extern "C" __global__ void __launch_bounds__(256) NAME(const __grid_constant__ AttnBwdParams p) { delta_body<KIND, OUT>(p); }
#endif
DELTA_KERNEL(BWD_NAME(delta, f16_f16), KIND_F16, OUT_F16)
DELTA_KERNEL(BWD_NAME(delta, f16_f32), KIND_F16, OUT_F32)
DELTA_KERNEL(BWD_NAME(delta, bf16_bf16), KIND_BF16, OUT_BF16)
DELTA_KERNEL(BWD_NAME(delta, bf16_f32), KIND_BF16, OUT_F32)

// attn_bwd_dq_<in>_d<64|128>_<grad> and attn_bwd_dkdv_<in>_d<64|128>_<grad>; D <= 64 runs the d64 kernels
#define DQ_KERNEL(NAME, KIND, DB, OUT)                                                                               \
  extern "C" __global__ void __launch_bounds__(384, 1)                                                               \
      NAME(const __grid_constant__ CUtensorMap tq, const __grid_constant__ CUtensorMap tk,                         \
           const __grid_constant__ CUtensorMap tv, const __grid_constant__ CUtensorMap tdo,                        \
           const __grid_constant__ CUtensorMap tdq, const __grid_constant__ BWD_P p) {                              \
    dq_body<KIND, DB, OUT, BWD_VL>(&tq, &tk, &tv, &tdo, &tdq, p);                                                   \
  }
#define DKDV_KERNEL(NAME, KIND, DB, OUT)                                                                             \
  extern "C" __global__ void __launch_bounds__(384, 1)                                                               \
      NAME(const __grid_constant__ CUtensorMap tq, const __grid_constant__ CUtensorMap tk,                         \
           const __grid_constant__ CUtensorMap tv, const __grid_constant__ CUtensorMap tdo,                        \
           const __grid_constant__ CUtensorMap tdk, const __grid_constant__ CUtensorMap tdv,                       \
           const __grid_constant__ BWD_P p) {                                                                       \
    dkdv_body<KIND, DB, OUT, BWD_VL>(&tq, &tk, &tv, &tdo, &tdk, &tdv, p);                                           \
  }
#define BWD_D(IN, KIND, OUT16)                                         \
  DQ_KERNEL(BWD_NAME(dq, IN##_d64_##IN), KIND, 64, OUT16)              \
  DQ_KERNEL(BWD_NAME(dq, IN##_d64_f32), KIND, 64, OUT_F32)             \
  DQ_KERNEL(BWD_NAME(dq, IN##_d128_##IN), KIND, 128, OUT16)            \
  DQ_KERNEL(BWD_NAME(dq, IN##_d128_f32), KIND, 128, OUT_F32)           \
  DKDV_KERNEL(BWD_NAME(dkdv, IN##_d64_##IN), KIND, 64, OUT16)          \
  DKDV_KERNEL(BWD_NAME(dkdv, IN##_d64_f32), KIND, 64, OUT_F32)         \
  DKDV_KERNEL(BWD_NAME(dkdv, IN##_d128_##IN), KIND, 128, OUT16)        \
  DKDV_KERNEL(BWD_NAME(dkdv, IN##_d128_f32), KIND, 128, OUT_F32)
BWD_D(f16, KIND_F16, OUT_F16)
BWD_D(bf16, KIND_BF16, OUT_BF16)
