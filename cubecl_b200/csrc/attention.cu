// Fused scaled-dot-product attention, forward (capi.cpp: b200_attention): out = softmax(scale * Q K^T) V per (batch, head),
// with the log-sum-exp of every row.  The [Sq, Sk] score matrix never leaves the SM.
//
// One CTA per (b, h, 128-query block), three warpgroups:
//   warpgroup 0    producer: one thread loads the Q tile once, then streams K and V blocks of 128 keys through a two-stage
//                  ring (a full barrier for K and one for V per stage, so S = Q K^T can start before V lands; one empty
//                  barrier per stage).  Every load is a 4-D tiled TMA load over (D, S, H, B): the view's strides are in the
//                  tensor map, and GQA is the kv head index h / group in the load coordinates.
//   warpgroups 1-2 consumers, 64 query rows each.  Per key block: S = Q K^T (wgmma, both operands K-major, f32 sums of exact
//                  16-bit products), the masks (keys >= Sk, and keys above the diagonal when causal) to -inf, the online
//                  softmax in base 2, P rounded to the input dtype in registers, O += P V (register-A wgmma, V an MN-major B
//                  operand).  The m64nN accumulator layout of S is the A-fragment layout of the k16 register operand, so P
//                  needs no shuffles.
// Numerics: t = s * (scale * log2 e) is formed once per score and the running row maximum m is a maximum of those t, so
// the row's maximal score contributes exp2(0) = 1 exactly; p = exp2(t - m) (ex2.approx.ftz: an argument <= -126 gives +0).
// The row sum l adds the f32 p values; P V reads p rounded (RNE) to the input dtype.  out = O / l (f32 division) rounded
// once (RNE) to the output dtype; lse = (m + log2 l) * ln 2.  Every row is produced by one CTA in increasing key order: no
// atomics, bitwise reproducible.
// Causal CTAs stop at the diagonal block (top-left alignment: key j is visible to query i iff j <= i).  The grid is 1-D,
// query blocks from the last (longest causal rows) to the first.
// The epilogue stages O / l in the consumer's own rows of the Q tile (SWIZZLE_128B, 128-byte column groups) and leaves
// through 4-D TMA stores that the unit clips at Sq and D; lse is written for rows < Sq.
//
// Compiled to a cubin (no host code here): nvcc -cubin -gencode arch=compute_90a,code=sm_90a
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "attention.cuh"
#include "kernel_params.h"
#include "ptx.cuh"

using namespace b200;

namespace {

// VL: the varlen kernels (P = AttnVarlenParams; kernel_params.h); the dense kernels have VL = false and P = AttnParams
template <int KIND, int DB, int OUT, bool VL, class P>
__device__ __forceinline__ void attn_body(const CUtensorMap* tq, const CUtensorMap* tk, const CUtensorMap* tv, const CUtensorMap* to,
                                          const P& p) {
  constexpr int NCH = DB / 64;                                // 128-byte (64-element) column chunks of a head
  constexpr uint32_t CHUNK = kAttnBlock * 128u;               // one chunk of a 128-row tile
  constexpr uint32_t TILE = NCH * CHUNK;                      // a 128-row tile of Q, K or V
  constexpr int NO = DB / 2;                                  // O accumulators per thread (m64 x DB)
  constexpr uint32_t OSZ = (OUT == OUT_F32) ? 4u : 2u;
  constexpr int CW = 128 / OSZ;                               // output columns per 128-byte staging row
  constexpr int NST = DB / CW;                                // TMA stores per consumer

  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sq = base;
  auto sk = [&](uint32_t s) { return base + TILE * (1u + 2u * s); };
  auto sv = [&](uint32_t s) { return base + TILE * (2u + 2u * s); };
  const uint32_t bars = base + TILE * (1u + 2u * kAttnStages);
  const uint32_t q_bar = bars;
  auto full_k = [&](uint32_t s) { return bars + 8u * (1u + s); };
  auto full_v = [&](uint32_t s) { return bars + 8u * (1u + kAttnStages + s); };
  auto empty = [&](uint32_t s) { return bars + 8u * (1u + 2u * kAttnStages + s); };

  // work: query block (last first), head, batch
  const uint32_t per = p.Hq * p.B;
  const uint32_t qb = p.nqb - 1u - blockIdx.x / per;
  const uint32_t rem = blockIdx.x % per;
  const uint32_t b = rem / p.Hq, h = rem - b * p.Hq, hk = h / p.group;
  const int q0 = static_cast<int>(qb * kAttnBlock);
  // key blocks [kb_lo, nkb); rows and keys are addressed at (qrow, krow) + block offsets in head h / hk of batch bb
  uint32_t kb_lo = 0, nkb;
  int qrow = q0, krow = 0, bb = static_cast<int>(b);
  int Lq = 0, Lk = 0, off = 0;   // varlen: the sequence's lengths, off = Lk - Lq
  if constexpr (VL) {
    int qs, ks;
    varlen_seq(p.cu_q, b, p.Tq, p.max_q, qs, Lq);
    varlen_seq(p.cu_k, b, p.Tk, p.max_k, ks, Lk);
    if (q0 >= Lq) return;   // past the sequence: no load, no store
    off = Lk - Lq;
    int lo, hi;
    band_blocks(q0, min(q0 + kAttnBlock, Lq) - 1, off, p.left, p.right, Lk, kAttnBlock, lo, hi);
    kb_lo = static_cast<uint32_t>(lo);
    nkb = static_cast<uint32_t>(hi);
    qrow = qs + q0;
    krow = ks;
    bb = 0;
  } else {
    const uint32_t nkb_all = (p.Sk + kAttnBlock - 1) / kAttnBlock;
    nkb = p.causal ? min(nkb_all, qb + 1u) : nkb_all;
  }

  const uint32_t wg = threadIdx.x >> 7;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(tq);
    tma_prefetch_desc(tk);
    tma_prefetch_desc(tv);
    tma_prefetch_desc(to);
    mbar_init(q_bar, 1);
    for (uint32_t s = 0; s < kAttnStages; ++s) {
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
      mbar_arrive_expect_tx(q_bar, TILE);
#pragma unroll
      for (int c = 0; c < NCH; ++c) tma_load_4d(sq + c * CHUNK, tq, q_bar, c * 64, qrow, static_cast<int>(h), bb);
      uint32_t s = 0, ph = 0;
      for (uint32_t kb = kb_lo; kb < nkb; ++kb) {
        mbar_wait(empty(s), ph ^ 1u);
        const int k0 = krow + static_cast<int>(kb * kAttnBlock);
        mbar_arrive_expect_tx(full_k(s), TILE);
#pragma unroll
        for (int c = 0; c < NCH; ++c) tma_load_4d(sk(s) + c * CHUNK, tk, full_k(s), c * 64, k0, static_cast<int>(hk), bb);
        mbar_arrive_expect_tx(full_v(s), TILE);
#pragma unroll
        for (int c = 0; c < NCH; ++c) tma_load_4d(sv(s) + c * CHUNK, tv, full_v(s), c * 64, k0, static_cast<int>(hk), bb);
        if (++s == kAttnStages) { s = 0; ph ^= 1u; }
      }
    }
    return;
  }

  // ======================================================================= consumers: 64 query rows each
  setmaxnreg_inc<232>();
  const uint32_t cw = wg - 1u;
  const uint32_t t = threadIdx.x & 127u;
  const uint32_t lane = t & 31u, wq = t >> 5;
  // fragment of m64nN: this thread holds rows r and r + 8 (of the consumer's 64), column pairs 8 j + 2 (lane % 4)
  const uint32_t r = wq * 16u + (lane >> 2);
  const uint32_t i0 = qb * kAttnBlock + cw * 64u + r, i1 = i0 + 8u;
  const uint32_t col = 2u * (lane & 3u);
  const float c2 = p.scale_log2;

  float o[NO];
#pragma unroll
  for (int i = 0; i < NO; ++i) o[i] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;   // running maxima (base-2 scaled) and this thread's row-sum parts
  // varlen: blocks inside [lo of the consumer's last row, hi of its first] need no mask
  int lo_c = 0, hi_c = 0;
  if constexpr (VL) {
    const int c0 = q0 + static_cast<int>(cw * 64u);
    lo_c = band_lo(c0 + 63, off, p.left, Lk);
    hi_c = band_hi(c0, off, p.right, Lk);
  }

  mbar_wait(q_bar, 0);
  uint32_t s = 0, ph = 0;
  for (uint32_t kb = kb_lo; kb < nkb; ++kb) {
    // ---- S = Q K^T
    float sc[64];
    mbar_wait(full_k(s), ph);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < DB / 16; ++kk) {
      const uint32_t ch = kk / 4, off = 2u * (kk % 4);
      const uint64_t da = make_smem_desc_sw128(sq + ch * CHUNK + cw * 64u * 128u, 16, 1024) + off;
      const uint64_t db = make_smem_desc_sw128(sk(s) + ch * CHUNK, 16, 1024) + off;
      wgmma_ss<128, KIND, KIND, 0, 0>(sc, da, db, kk != 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_operands(sc);

    // ---- scale, mask (the last block holds the diagonal of a causal CTA and the keys past Sk; varlen: every block the band
    // or Lk cuts), row maxima
    bool last;
    if constexpr (VL) last = static_cast<int>(kb * kAttnBlock) < lo_c || static_cast<int>(kb * kAttnBlock) + kAttnBlock - 1 > hi_c;
    else last = kb + 1u == nkb;
    const uint32_t key0 = kb * kAttnBlock + col;
    int lo0 = 0, hi0 = 0, lo1 = 0, hi1 = 0;   // varlen: this thread's rows see keys [lo, hi]
    if constexpr (VL) {
      if (last) {
        lo0 = band_lo(static_cast<int>(i0), off, p.left, Lk);
        hi0 = band_hi(static_cast<int>(i0), off, p.right, Lk);
        lo1 = band_lo(static_cast<int>(i1), off, p.left, Lk);
        hi1 = band_hi(static_cast<int>(i1), off, p.right, Lk);
      }
    }
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float v = sc[4 * j + e] * c2;
        if (last) {
          const uint32_t key = key0 + 8u * j + (e & 1);
          if constexpr (VL) {
            const int kk = static_cast<int>(key);
            if ((e < 2) ? (kk < lo0 || kk > hi0) : (kk < lo1 || kk > hi1)) v = -INFINITY;
          } else {
            const uint32_t row = (e < 2) ? i0 : i1;
            if (key >= p.Sk || (p.causal && key > row)) v = -INFINITY;
          }
        }
        sc[4 * j + e] = v;
        if (e < 2) mx0 = fmaxf(mx0, v); else mx1 = fmaxf(mx1, v);
      }
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xFFFFFFFFu, mx0, 1));
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xFFFFFFFFu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xFFFFFFFFu, mx1, 1));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xFFFFFFFFu, mx1, 2));
    // dense: every row sees key 0 in block 0, so the maxima are finite from the first block on.  varlen: a row may have seen
    // no key yet; its maximum -inf subtracts 0, so p = exp2(-inf) = 0 and l and O stay 0
    const float n0 = fmaxf(m0, mx0), n1 = fmaxf(m1, mx1);
    float z0 = n0, z1 = n1;   // the maxima subtracted
    if constexpr (VL) {
      if (n0 == -INFINITY) z0 = 0.f;
      if (n1 == -INFINITY) z1 = 0.f;
    }
    const float a0 = ex2(m0 - z0), a1 = ex2(m1 - z1);   // block 0: exp2(-inf) = 0 rescales the zero O and l
    m0 = n0;
    m1 = n1;

    // ---- p = exp2(t - m), row sums from the f32 p, P to 16 bits in the A-fragment layout
    uint32_t pa[32];
    float s0 = 0.f, s1 = 0.f;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const float p0 = ex2(sc[4 * j] - z0), p1 = ex2(sc[4 * j + 1] - z0);
      const float p2 = ex2(sc[4 * j + 2] - z1), p3 = ex2(sc[4 * j + 3] - z1);
      s0 += p0 + p1;
      s1 += p2 + p3;
      pa[2 * j] = pack16<KIND>(p0, p1);
      pa[2 * j + 1] = pack16<KIND>(p2, p3);
    }
    l0 = l0 * a0 + s0;
    l1 = l1 * a1 + s1;
#pragma unroll
    for (int j = 0; j < NO / 4; ++j) {
      o[4 * j] *= a0;
      o[4 * j + 1] *= a0;
      o[4 * j + 2] *= a1;
      o[4 * j + 3] *= a1;
    }

    // ---- O += P V: V [keys, D] is an MN-major B operand, 16 keys (2048 bytes of rows) per instruction
    mbar_wait(full_v(s), ph);
    if constexpr (VL) {   // V rows past Lk are the next sequence's (maybe NaN or inf; 0 * NaN = NaN in the product): zero them
      const int valid = Lk - static_cast<int>(kb * kAttnBlock);
      if (valid < kAttnBlock) zero_rows(sv(s), NCH, CHUNK, valid, kAttnBlock, 1u + cw);
    }
    wgmma_fence_operands(o);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
      const uint64_t db = make_smem_desc_sw128(sv(s) + kk * 2048u, CHUNK, 1024);
      const uint32_t a[4] = {pa[4 * kk], pa[4 * kk + 1], pa[4 * kk + 2], pa[4 * kk + 3]};
      wgmma_rs<DB, KIND, 1>(o, a, db, 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_operands(o);
    if (t == 0) mbar_arrive(empty(s));
    if (++s == kAttnStages) { s = 0; ph ^= 1u; }
  }

  // ---- epilogue: l over the quad, O / l through the consumer's rows of the Q tile, TMA stores clipped at Sq and D
  l0 += __shfl_xor_sync(0xFFFFFFFFu, l0, 1);
  l0 += __shfl_xor_sync(0xFFFFFFFFu, l0, 2);
  l1 += __shfl_xor_sync(0xFFFFFFFFu, l1, 1);
  l1 += __shfl_xor_sync(0xFFFFFFFFu, l1, 2);
  const int row0 = q0 + static_cast<int>(cw * 64u);
  if constexpr (VL) {
    if (row0 + 64 > Lq) {   // the sequence ends inside these rows: direct stores of rows < Lq (a TMA box would write past it)
      if (row0 < Lq)
        store_frag_direct<DB, OUT>(o, l0, l1, p.out + OSZ * ((qrow + cw * 64u) * p.o_st + h * p.o_sh), OSZ * p.o_st, Lq - row0, p.D);
      if (p.lse != 0 && (lane & 3u) == 0) {
        float* lse = reinterpret_cast<float*>(p.lse) + static_cast<uint64_t>(h) * p.Tq + (qrow - q0);
        constexpr float kLn2 = 0.693147180559945309f;
        if (static_cast<int>(i0) < Lq) lse[i0] = (m0 + log2f(l0)) * kLn2;
        if (static_cast<int>(i1) < Lq) lse[i1] = (m1 + log2f(l1)) * kLn2;
      }
      return;
    }
  }
#pragma unroll
  for (int c = 0; c < NST; ++c) {
    const uint32_t buf = sq + (c % NCH) * CHUNK + cw * 64u * 128u;
    if (c >= NCH) {   // the buffer is reused: the store that read it has finished reading
      if (t == 0) tma_store_wait_read<0>();
      asm volatile("bar.sync %0, 128;" ::"r"(1u + cw) : "memory");
    }
#pragma unroll
    for (int jj = 0; jj < CW / 8; ++jj) {
      const int j = c * (CW / 8) + jj;
      float v0 = __fdiv_rn(o[4 * j], l0), v1 = __fdiv_rn(o[4 * j + 1], l0);
      float v2 = __fdiv_rn(o[4 * j + 2], l1), v3 = __fdiv_rn(o[4 * j + 3], l1);
      if constexpr (VL) {   // a row without keys: l = 0, out = +0
        if (!(l0 > 0.f)) v0 = v1 = 0.f;
        if (!(l1 > 0.f)) v2 = v3 = 0.f;
      }
      const uint32_t cb = (8u * jj + col) * OSZ;   // byte of the pair inside the 128-byte row
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const uint32_t rr = r + 8u * hh;
        const uint32_t addr = buf + rr * 128u + ((((cb >> 4) ^ (rr & 7u)) << 4) | (cb & 15u));
        const float x0 = hh ? v2 : v0, x1 = hh ? v3 : v1;
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
      if (t == 0 && c * CW < static_cast<int>(p.D)) {
        tma_store_4d(to, buf, c * CW, qrow + static_cast<int>(cw * 64u), static_cast<int>(h), 0);
        tma_store_commit();
      }
    } else if (t == 0 && row0 < static_cast<int>(p.Sq) && c * CW < static_cast<int>(p.D)) {
      tma_store_4d(to, buf, c * CW, row0, static_cast<int>(h), static_cast<int>(b));
      tma_store_commit();
    }
  }
  if (p.lse != 0 && (lane & 3u) == 0) {
    constexpr float kLn2 = 0.693147180559945309f;
    if constexpr (VL) {   // a full block: every row is the sequence's
      float* lse = reinterpret_cast<float*>(p.lse) + static_cast<uint64_t>(h) * p.Tq + (qrow - q0);
      lse[i0] = (m0 + log2f(l0)) * kLn2;
      lse[i1] = (m1 + log2f(l1)) * kLn2;
    } else {
      float* lse = reinterpret_cast<float*>(p.lse) + (static_cast<uint64_t>(b) * p.Hq + h) * p.Sq;
      if (i0 < p.Sq) lse[i0] = (m0 + log2f(l0)) * kLn2;
      if (i1 < p.Sq) lse[i1] = (m1 + log2f(l1)) * kLn2;
    }
  }
  if (t == 0) tma_store_wait<0>();   // outstanding stores read this CTA's shared memory: finish before exit
}

}  // namespace

// name: attn_fwd_<in>_d<64|128>_<out>; D <= 64 runs the d64 kernel, 64 < D <= 128 the d128 kernel
// varlen (compiled with -DATTN_VARLEN into its own cubin): attn_fwd_varlen_<in>_d<64|128>_<out>
#ifdef ATTN_VARLEN
#define ATTN_VL true
#define ATTN_P AttnVarlenParams
#define ATTN_NAME(IN, D, OUT) attn_fwd_varlen_##IN##_d##D##_##OUT
#else
#define ATTN_VL false
#define ATTN_P AttnParams
#define ATTN_NAME(IN, D, OUT) attn_fwd_##IN##_d##D##_##OUT
#endif
#define ATTN_KERNEL(NAME, KIND, DB, OUT)                                                                             \
  extern "C" __global__ void __launch_bounds__(384, 1)                                                               \
      NAME(const __grid_constant__ CUtensorMap tq, const __grid_constant__ CUtensorMap tk,                         \
           const __grid_constant__ CUtensorMap tv, const __grid_constant__ CUtensorMap to,                         \
           const __grid_constant__ ATTN_P p) {                                                                      \
    attn_body<KIND, DB, OUT, ATTN_VL>(&tq, &tk, &tv, &to, p);                                                       \
  }
#define ATTN_D(IN, KIND, OUT16)                                  \
  ATTN_KERNEL(ATTN_NAME(IN, 64, IN), KIND, 64, OUT16)            \
  ATTN_KERNEL(ATTN_NAME(IN, 64, f32), KIND, 64, OUT_F32)         \
  ATTN_KERNEL(ATTN_NAME(IN, 128, IN), KIND, 128, OUT16)          \
  ATTN_KERNEL(ATTN_NAME(IN, 128, f32), KIND, 128, OUT_F32)
ATTN_D(f16, KIND_F16, OUT_F16)
ATTN_D(bf16, KIND_BF16, OUT_BF16)
