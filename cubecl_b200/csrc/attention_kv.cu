// Attention against a KV cache (capi.cpp: b200_attention_kvcache): decoding, speculative decoding and chunked prefill.  The
// queries of sequence b attend to its first L_b = cache_seqlens[b] cached keys, stored in pages reached through a block table.
//
// attn_kv_<in>_d<64|128>_<out>: one CTA per (b, hk, m-tile, split), 160 threads.
//   warp 4        producer: loads the m-tile's Q rows once with one 4-D TMA box (64, st, gt, 1) per 64-column chunk over q's
//                 (D, Sq, Hq, B) map, then streams K and V blocks of kAttnKvBlock keys through kAttnKvStages stages.  The warp
//                 reads the block table 32 chunks at a time, one batch ahead, and lane 0 issues one TMA load per page chunk
//                 over the cache's (D, page, Hkv, P) map.  Chunks at or past L_b are neither looked up nor loaded.
//   warps 0-3     one m64 consumer warpgroup.  An m-tile packs the G = Hq / Hkv query heads of kv head hk with the Sq queries
//                 (row r = g * st + i), so every K / V byte is read once per kv head, not once per query head.  Per block:
//                 S = Q K^T (wgmma, f32), masks as selects on the blocks that straddle L_b or the causal diagonal, the online
//                 softmax in base 2 with the forward's numerics, P rounded to the input dtype, O += P V (register-A wgmma).
//                 The V rows of keys >= L_b in the last block are zeroed in shared memory first: stale cache slots may hold
//                 NaN or inf, and 0 * NaN = NaN inside the MMA.
// Visibility: key j is visible to query i iff j < L_b and, when causal, j <= L_b - Sq + i (bottom-right).  A row with no
// visible key has m = -inf; the softmax then subtracts 0 instead of m, so p = +0 and O and l stay 0.
// nsplit == 1 (ws == 0): out = O / l rounded once, lse = (m + log2 l) ln 2; an empty row gives +0 and -inf.
// nsplit > 1: every split writes un-normalised f32 O and (m, l) to the workspace (kernel_params.h), and attn_kv_combine_<out>
// merges the splits in index order.  No atomics anywhere: bitwise reproducible for fixed shapes and SM count.
// attn_kv_write: the scatter of new tokens into the cache (b200_kvcache_write).
// -DATTN_KV_FP8 (cubin attention_kv_fp8) builds the fp8-cache kernels instead (b200_attention_kvcache_fp8): the same body with
// cache format CF_E4M3 / CF_E5M2.  The producer loads 128-byte fp8 rows through kAttnKvF8Stages stages; the consumer widens K
// before Q K^T and V while Q K^T runs into 16-bit swizzled buffers (V rows of keys >= L_b become zeros there), so the wgmma
// code is unchanged; t = s * scale_log2 * k_scale[hk], out = (v_scale[hk] O) / l.  attn_kv_combine_fp8_<out> applies v_scale
// to the merged sum, and attn_kv_write_fp8 quantizes new tokens (b200_kvcache_write_fp8).
//
// Compiled to a cubin (no host code here): nvcc -cubin -gencode arch=compute_90a,code=sm_90a
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "attention.cuh"
#include "kernel_params.h"
#include "ptx.cuh"

using namespace b200;

namespace {

constexpr float kLn2 = 0.693147180559945309f;

template <int OUT>
__device__ __forceinline__ void store_pair(uint64_t addr, float x0, float x1) {
  if constexpr (OUT == OUT_F32) {
    asm volatile("st.global.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(x0), "f"(x1) : "memory");
  } else {
    asm volatile("st.global.b32 [%0], %1;" ::"l"(addr), "r"(pack16<OUT == OUT_BF16 ? KIND_BF16 : KIND_F16>(x0, x1)) : "memory");
  }
}

// Cache formats: the 16-bit input dtype itself, or fp8 widened on chip.
enum : int { CF_16 = 0, CF_E4M3 = 1, CF_E5M2 = 2 };

// Four fp8 values (memory order) -> two pairs of the 16-bit KIND, exactly: every e4m3 and e5m2 value is an f16 and a bf16
// value.  bf16 goes through f32 (f16 -> f32 -> bf16, each step exact).
template <int KIND, int CF>
__device__ __forceinline__ void widen4(uint32_t w, uint32_t& lo, uint32_t& hi) {
  const unsigned short w0 = static_cast<unsigned short>(w), w1 = static_cast<unsigned short>(w >> 16);
  if constexpr (CF == CF_E4M3) {
    asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(lo) : "h"(w0));
    asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(hi) : "h"(w1));
  } else {
    asm("cvt.rn.f16x2.e5m2x2 %0, %1;" : "=r"(lo) : "h"(w0));
    asm("cvt.rn.f16x2.e5m2x2 %0, %1;" : "=r"(hi) : "h"(w1));
  }
  if constexpr (KIND == KIND_BF16) {
    asm("{.reg .b16 a, b; .reg .f32 x, y;\n\t"
        "mov.b32 {a, b}, %0; cvt.f32.f16 x, a; cvt.f32.f16 y, b; cvt.rn.bf16x2.f32 %0, y, x;}" : "+r"(lo));
    asm("{.reg .b16 a, b; .reg .f32 x, y;\n\t"
        "mov.b32 {a, b}, %0; cvt.f32.f16 x, a; cvt.f32.f16 y, b; cvt.rn.bf16x2.f32 %0, y, x;}" : "+r"(hi));
  }
}

// Widen one fp8 block (kAttnKvBlock rows of 128 swizzled bytes at src, as the 128-byte TMA box wrote it) into the 16-bit
// 128-byte-swizzled layout at dst that the 16-bit kernels' TMA loads produce (DB / 64 chunks of kAttnKvBlock rows x 128
// bytes).  Rows >= z are written as zeros (the V rows of keys past L: stale bytes may be NaN or inf).  One 16-byte unit of 16
// values per thread and step; the two 16-byte stores of a unit go out in an order that keeps a quarter warp on distinct banks.
template <int KIND, int CF, int DB>
__device__ __forceinline__ void widen_block(uint32_t src, uint32_t dst, uint32_t z, uint32_t t) {
  constexpr uint32_t UPR = DB / 16;   // 16-byte fp8 units per row
#pragma unroll
  for (uint32_t i = 0; i < kAttnKvBlock * UPR / 128u; ++i) {
    const uint32_t u = t + 128u * i, j = u / UPR, g = u % UPR, sw = j & 7u;
    uint32_t w0, w1, w2, w3;
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(w0), "=r"(w1), "=r"(w2), "=r"(w3) : "r"(src + j * 128u + ((g ^ sw) << 4)));
    uint32_t h[8] = {0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u};
    if (j < z) {
      widen4<KIND, CF>(w0, h[0], h[1]);
      widen4<KIND, CF>(w1, h[2], h[3]);
      widen4<KIND, CF>(w2, h[4], h[5]);
      widen4<KIND, CF>(w3, h[6], h[7]);
    }
    const uint32_t row = dst + (g >> 2) * (kAttnKvBlock * 128u) + j * 128u;
    const uint32_t c0 = 2u * (g & 3u), f = (g >> 2) & 1u;   // 16-byte groups c0, c0 + 1; f: store c0 + 1 first
    const uint32_t a0 = row + (((c0 + f) ^ sw) << 4), a1 = row + (((c0 + 1u - f) ^ sw) << 4);
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(a0), "r"(f ? h[4] : h[0]), "r"(f ? h[5] : h[1]), "r"(f ? h[6] : h[2]),
                 "r"(f ? h[7] : h[3]) : "memory");
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(a1), "r"(f ? h[0] : h[4]), "r"(f ? h[1] : h[5]), "r"(f ? h[2] : h[6]),
                 "r"(f ? h[3] : h[7]) : "memory");
  }
}

template <int KIND, int DB, int OUT, int CF = CF_16>
__device__ __forceinline__ void kv_body(const CUtensorMap* tq, const CUtensorMap* tk, const CUtensorMap* tv, const AttnKvParams& p) {
  constexpr int NCH = DB / 64;                          // 128-byte (64-element) column chunks of a head
  constexpr int KB = kAttnKvBlock;
  constexpr uint32_t QCH = kAttnKvRows * 128u;          // one chunk of the Q tile
  constexpr uint32_t KCH = KB * 128u;                   // one chunk of a K or V block
  constexpr uint32_t KT = NCH * KCH;
  constexpr int NO = DB / 2;                            // O accumulators per thread (m64 x DB)
  constexpr uint32_t OSZ = (OUT == OUT_F32) ? 4u : 2u;
  constexpr uint32_t NST = CF == CF_16 ? kAttnKvStages : kAttnKvF8Stages;
  constexpr uint32_t ST = CF == CF_16 ? KT : KB * 128u;   // bytes of a K or V stage (fp8: one 128-byte row per key)

  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sq = base;
  auto sk = [&](uint32_t s) { return base + NCH * QCH + 2u * ST * s; };
  auto sv = [&](uint32_t s) { return base + NCH * QCH + 2u * ST * s + ST; };
  // fp8: the widened K of even and odd blocks, then the widened V
  const uint32_t kw = base + NCH * QCH + 2u * ST * NST, vw = kw + 2u * KT;
  const uint32_t bars = kw + (CF == CF_16 ? 0u : 3u * KT);
  const uint32_t q_bar = bars;
  auto full_k = [&](uint32_t s) { return bars + 8u * (1u + s); };
  auto full_v = [&](uint32_t s) { return bars + 8u * (1u + NST + s); };
  auto empty = [&](uint32_t s) { return bars + 8u * (1u + 2u * NST + s); };

  // ---- work unit and its key blocks
  const uint32_t mtiles = p.mtg * p.mts;
  uint32_t x = blockIdx.x;
  const uint32_t mt = x % mtiles;
  x /= mtiles;
  const uint32_t split = x % p.nsplit;
  x /= p.nsplit;
  const uint32_t hk = x % p.Hkv, b = x / p.Hkv;
  const uint32_t g0 = (mt / p.mts) * p.gt, q0 = (mt % p.mts) * p.st;   // first group head, first query of the tile
  const int L = min(max(reinterpret_cast<const int*>(p.seqlens)[b], 0), static_cast<int>(p.cap));
  const int Sq = static_cast<int>(p.Sq);
  // keys some row of the tile sees: j < L, and j <= L - Sq + i_last when causal
  const int i_last = min(Sq, static_cast<int>(q0 + p.st)) - 1;
  const int kend = p.causal ? min(L, L - Sq + i_last + 1) : L;
  const uint32_t kb0 = split * p.bps;
  const uint32_t kb1 = min(min(kb0 + p.bps, p.nkb), kend > 0 ? static_cast<uint32_t>(kend + KB - 1) / KB : 0u);
  const uint32_t nkb = kb1 > kb0 ? kb1 - kb0 : 0u;

  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
  if (threadIdx.x == 128) {
    tma_prefetch_desc(tq);
    tma_prefetch_desc(tk);
    tma_prefetch_desc(tv);
    mbar_init(q_bar, 1);
    for (uint32_t s = 0; s < NST; ++s) {
      mbar_init(full_k(s), 1);
      mbar_init(full_v(s), 1);
      mbar_init(empty(s), 1);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == 4) {
    // ===================================================================== TMA producer warp (lane 0 issues)
    if (nkb == 0) return;
    const uint32_t h0 = hk * p.group + g0;
    if (lane == 0) {
      mbar_arrive_expect_tx(q_bar, NCH * p.gt * p.st * 128u);
#pragma unroll
      for (int c = 0; c < NCH; ++c)
        tma_load_4d(sq + c * QCH, tq, q_bar, c * 64, static_cast<int>(q0), static_cast<int>(h0), static_cast<int>(b));
    }
    const uint32_t R = p.rows, per = KB / R;   // keys per load, loads per block (1, 2 or 4)
    const int* tbl = reinterpret_cast<const int*>(p.table);
    // page id of chunk c (keys c R .. c R + R - 1); never reads a table entry at or past ceil(L / page)
    auto page_of = [&](uint32_t c) -> int {
      const uint32_t j0 = c * R;
      if (j0 >= static_cast<uint32_t>(L)) return 0;
      return tbl ? tbl[b * p.t_sb + (j0 / p.page) * p.t_sp] : static_cast<int>(b);
    };
    uint32_t cbase = kb0 * per;
    int cur = page_of(cbase + lane), nxt = page_of(cbase + 32u + lane);
    uint32_t s = 0, ph = 0;
    for (uint32_t kb = kb0; kb < kb1; ++kb) {
      const uint32_t c = kb * per;
      if (c - cbase == 32u) {   // 32 % per == 0: batches start on block boundaries
        cbase += 32u;
        cur = nxt;
        nxt = page_of(cbase + 32u + lane);
      }
      int pg[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) pg[i] = __shfl_sync(0xFFFFFFFFu, cur, (c - cbase + i) & 31u);
      const int k0 = static_cast<int>(kb) * KB;
      const uint32_t nload = min(per, static_cast<uint32_t>(L - k0 + R - 1) / R);   // chunks that start below L
      mbar_wait(empty(s), ph ^ 1u);
      if constexpr (CF != CF_16) {
        // fp8: one 128-byte box per page chunk covers the whole head (columns >= D read as zeros)
        if (lane == 0) {
          mbar_arrive_expect_tx(full_k(s), nload * R * 128u);
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            if (i >= static_cast<int>(nload)) break;
            const int row = static_cast<int>((static_cast<uint32_t>(k0) + i * R) % p.page);
            tma_load_4d(sk(s) + i * R * 128u, tk, full_k(s), 0, row, static_cast<int>(hk), pg[i]);
          }
          mbar_arrive_expect_tx(full_v(s), nload * R * 128u);
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            if (i >= static_cast<int>(nload)) break;
            const int row = static_cast<int>((static_cast<uint32_t>(k0) + i * R) % p.page);
            tma_load_4d(sv(s) + i * R * 128u, tv, full_v(s), 0, row, static_cast<int>(hk), pg[i]);
          }
        }
      } else if (lane == 0) {
        mbar_arrive_expect_tx(full_k(s), nload * NCH * R * 128u);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          if (i >= static_cast<int>(nload)) break;
          const int row = static_cast<int>((static_cast<uint32_t>(k0) + i * R) % p.page);
#pragma unroll
          for (int cc = 0; cc < NCH; ++cc)
            tma_load_4d(sk(s) + cc * KCH + i * R * 128u, tk, full_k(s), cc * 64, row, static_cast<int>(hk), pg[i]);
        }
        mbar_arrive_expect_tx(full_v(s), nload * NCH * R * 128u);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          if (i >= static_cast<int>(nload)) break;
          const int row = static_cast<int>((static_cast<uint32_t>(k0) + i * R) % p.page);
#pragma unroll
          for (int cc = 0; cc < NCH; ++cc)
            tma_load_4d(sv(s) + cc * KCH + i * R * 128u, tv, full_v(s), cc * 64, row, static_cast<int>(hk), pg[i]);
        }
      }
      __syncwarp();
      if (++s == NST) { s = 0; ph ^= 1u; }
    }
    return;
  }

  // ======================================================================= consumer warpgroup: 64 rows
  const uint32_t t = threadIdx.x;
  // fragment of m64nN: this thread holds rows r and r + 8, column pairs 8 j + col
  const uint32_t r = warp * 16u + (lane >> 2);
  const uint32_t col = 2u * (lane & 3u);
  // fp8: c = scale_log2 * k_scale[hk], one f32 product per CTA
  const float c2 = CF == CF_16 ? p.scale_log2 : p.scale_log2 * reinterpret_cast<const float*>(p.k_scale)[hk];
  int lim[2];            // keys below lim are visible to the row
  bool valid[2];          // the row is a real (head, query) of this tile
  uint32_t hrow[2], irow[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const uint32_t rr = r + 8u * hh, g = rr / p.st, i = q0 + rr % p.st;
    valid[hh] = rr < p.gt * p.st && i < p.Sq && g0 + g < p.group;
    hrow[hh] = hk * p.group + g0 + g;
    irow[hh] = i;
    lim[hh] = p.causal ? min(L, L - Sq + static_cast<int>(i) + 1) : L;
  }
  const int lim_min = min(lim[0], lim[1]);

  float o[NO];
#pragma unroll
  for (int i = 0; i < NO; ++i) o[i] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;

  if (nkb) mbar_wait(q_bar, 0);
  uint32_t s = 0, ph = 0;
  for (uint32_t kb = kb0; kb < kb1; ++kb) {
    // ---- S = Q K^T (64 keys)
    float sc[32];
    mbar_wait(full_k(s), ph);
    // fp8: widen K into the buffer of this block's parity (the other one may still be read by the previous block's
    // wgmma in a slower warp; every warp has passed that wgmma's wait before the barrier after this block's V widening)
    const uint32_t kbuf = kw + (kb & 1u) * KT;
    if constexpr (CF != CF_16) {
      widen_block<KIND, CF, DB>(sk(s), kbuf, KB, t);
      fence_proxy_async_smem();   // generic-proxy writes -> visible to wgmma
      asm volatile("bar.sync 1, 128;" ::: "memory");
    }
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < DB / 16; ++kk) {
      const uint32_t ch = kk / 4, off = 2u * (kk % 4);
      const uint64_t da = make_smem_desc_sw128(sq + ch * QCH, 16, 1024) + off;
      const uint64_t db = make_smem_desc_sw128((CF == CF_16 ? sk(s) : kbuf) + ch * KCH, 16, 1024) + off;
      wgmma_ss<64, KIND, KIND, 0, 0>(sc, da, db, kk != 0 ? 1u : 0u);
    }
    wgmma_commit();
    if constexpr (CF != CF_16) {
      // widen V while S = Q K^T runs; the V rows of keys >= L become zeros here (stale slots, or chunks never loaded)
      mbar_wait(full_v(s), ph);
      widen_block<KIND, CF, DB>(sv(s), vw, static_cast<uint32_t>(min(max(L - static_cast<int>(kb) * KB, 0), KB)), t);
      fence_proxy_async_smem();
      asm volatile("bar.sync 1, 128;" ::: "memory");
      if (t == 0) mbar_arrive(empty(s));   // every consumer thread is done with the fp8 stage
    }
    wgmma_wait<0>();
    wgmma_fence_operands(sc);

    // ---- scale, mask (a select: stale keys may score NaN), row maxima
    const int k0 = static_cast<int>(kb) * KB;
    const bool edge = k0 + KB > lim_min;
    const int key0 = k0 + static_cast<int>(col);
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float v = sc[4 * j + e] * c2;
        if (edge) v = key0 + 8 * j + (e & 1) < lim[e >> 1] ? v : -INFINITY;
        sc[4 * j + e] = v;
        if (e < 2) mx0 = fmaxf(mx0, v); else mx1 = fmaxf(mx1, v);
      }
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xFFFFFFFFu, mx0, 1));
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xFFFFFFFFu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xFFFFFFFFu, mx1, 1));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xFFFFFFFFu, mx1, 2));
    const float n0 = fmaxf(m0, mx0), n1 = fmaxf(m1, mx1);
    // a row that has seen no visible key yet subtracts 0: its p are exp2(-inf) = +0
    const float z0 = n0 == -INFINITY ? 0.f : n0, z1 = n1 == -INFINITY ? 0.f : n1;
    const float a0 = ex2(m0 - z0), a1 = ex2(m1 - z1);
    m0 = n0;
    m1 = n1;

    // ---- p = exp2(t - m), row sums from the f32 p, P to 16 bits in the A-fragment layout
    uint32_t pa[16];
    float s0 = 0.f, s1 = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
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

    // ---- the last block: zero the V rows of keys >= L (stale slots, or chunks never loaded)
    if constexpr (CF == CF_16) {
      mbar_wait(full_v(s), ph);
      if (k0 + KB > L) {
        const uint32_t z = static_cast<uint32_t>(L - k0);
        for (uint32_t u = t; u < NCH * KB * 8u; u += 128u) {
          const uint32_t row = (u >> 3) % KB;
          if (row >= z) asm volatile("st.shared.v4.b32 [%0], {%1, %1, %1, %1};" ::"r"(sv(s) + u * 16u), "r"(0u) : "memory");
        }
        fence_proxy_async_smem();   // generic-proxy writes -> visible to wgmma
        asm volatile("bar.sync 1, 128;" ::: "memory");
      }
    }

    // ---- O += P V: V [keys, D] is an MN-major B operand, 16 keys (2048 bytes of rows) per instruction
    wgmma_fence_operands(o);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < KB / 16; ++kk) {
      const uint64_t db = make_smem_desc_sw128((CF == CF_16 ? sv(s) : vw) + kk * 2048u, KCH, 1024);
      const uint32_t a[4] = {pa[4 * kk], pa[4 * kk + 1], pa[4 * kk + 2], pa[4 * kk + 3]};
      wgmma_rs<DB, KIND, 1>(o, a, db, 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_operands(o);
    if constexpr (CF == CF_16) {
      if (t == 0) mbar_arrive(empty(s));
    }
    if (++s == NST) { s = 0; ph ^= 1u; }
  }

  // ---- epilogue: l over the quad; out and lse directly, or the split's partial O and (m, l)
  l0 += __shfl_xor_sync(0xFFFFFFFFu, l0, 1);
  l0 += __shfl_xor_sync(0xFFFFFFFFu, l0, 2);
  l1 += __shfl_xor_sync(0xFFFFFFFFu, l1, 1);
  l1 += __shfl_xor_sync(0xFFFFFFFFu, l1, 2);
  const uint64_t rows = static_cast<uint64_t>(p.B) * p.Hq * p.Sq;
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    if (!valid[hh]) continue;
    const float m = hh ? m1 : m0, l = hh ? l1 : l0;
    const uint64_t row = (static_cast<uint64_t>(b) * p.Hq + hrow[hh]) * p.Sq + irow[hh];
    if (p.ws == 0) {
      const uint64_t dst = p.out + (b * p.o_sb + hrow[hh] * p.o_sh + irow[hh] * p.o_ss) * OSZ;
#pragma unroll
      for (int j = 0; j < DB / 8; ++j) {
        const uint32_t c = 8u * j + col;
        if (c >= p.D) continue;
        if constexpr (CF != CF_16) {
          // out = (v_scale O) / l, rounded once
          const float vs = reinterpret_cast<const float*>(p.v_scale)[hk];
          const float v0 = l > 0.f ? __fdiv_rn(__fmul_rn(vs, o[4 * j + 2 * hh]), l) : 0.f;
          const float v1 = l > 0.f ? __fdiv_rn(__fmul_rn(vs, o[4 * j + 2 * hh + 1]), l) : 0.f;
          store_pair<OUT>(dst + c * OSZ, v0, v1);
          continue;
        }
        const float v0 = l > 0.f ? __fdiv_rn(o[4 * j + 2 * hh], l) : 0.f;
        const float v1 = l > 0.f ? __fdiv_rn(o[4 * j + 2 * hh + 1], l) : 0.f;
        store_pair<OUT>(dst + c * OSZ, v0, v1);
      }
      if (p.lse != 0 && (lane & 3u) == 0)
        reinterpret_cast<float*>(p.lse)[row] = l > 0.f ? (m + log2f(l)) * kLn2 : -INFINITY;
    } else {
      float* ws = reinterpret_cast<float*>(p.ws);
      const uint64_t prow = split * rows + row;
#pragma unroll
      for (int j = 0; j < DB / 8; ++j) {
        const uint32_t c = 8u * j + col;
        if (c >= p.D) continue;
        store_pair<OUT_F32>(reinterpret_cast<uint64_t>(ws + prow * p.D + c), o[4 * j + 2 * hh], o[4 * j + 2 * hh + 1]);
      }
      if ((lane & 3u) == 0) store_pair<OUT_F32>(reinterpret_cast<uint64_t>(ws + p.nsplit * rows * p.D + 2 * prow), m, l);
    }
  }
}

// Merge of the splits of one row, 4 columns per thread, in split order: m = max m_s, w_s = exp2(m_s - m),
// out = sum w_s O_s / sum w_s l_s (f32, rounded once), lse = (m + log2 l) ln 2; every split empty: +0 and -inf.
// F8 (fp8 caches): out = (v_scale[h / G] * sum w_s O_s) / sum w_s l_s.
template <int OUT, bool F8 = false>
__device__ __forceinline__ void kv_combine(const AttnKvParams& p) {
  constexpr uint32_t OSZ = (OUT == OUT_F32) ? 4u : 2u;
  const uint32_t cpr = p.D / 4;
  const uint64_t rows = static_cast<uint64_t>(p.B) * p.Hq * p.Sq;
  const uint64_t idx = static_cast<uint64_t>(blockIdx.x) * kAttnKvCombineThreads + threadIdx.x;
  const uint64_t row = idx / cpr;
  if (row >= rows) return;
  const uint32_t c = 4u * static_cast<uint32_t>(idx % cpr);
  const float* O = reinterpret_cast<const float*>(p.ws);
  const float2* ml = reinterpret_cast<const float2*>(O + p.nsplit * rows * p.D);
  float m = -INFINITY;
  for (uint32_t s = 0; s < p.nsplit; ++s) m = fmaxf(m, ml[s * rows + row].x);
  const float z = m == -INFINITY ? 0.f : m;
  float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f, l = 0.f;
  for (uint32_t s = 0; s < p.nsplit; ++s) {
    const float2 e = ml[s * rows + row];
    const float w = ex2(e.x - z);
    const float4 v = *reinterpret_cast<const float4*>(O + (s * rows + row) * p.D + c);
    l += w * e.y;
    a0 += w * v.x;
    a1 += w * v.y;
    a2 += w * v.z;
    a3 += w * v.w;
  }
  const uint64_t i = row % p.Sq, bh = row / p.Sq, h = bh % p.Hq, b = bh / p.Hq;
  const uint64_t dst = p.out + (b * p.o_sb + h * p.o_sh + i * p.o_ss + c) * OSZ;
  const bool any = l > 0.f;
  if constexpr (F8) {
    const float vs = reinterpret_cast<const float*>(p.v_scale)[h / p.group];
    a0 = __fmul_rn(vs, a0);
    a1 = __fmul_rn(vs, a1);
    a2 = __fmul_rn(vs, a2);
    a3 = __fmul_rn(vs, a3);
  }
  store_pair<OUT>(dst, any ? __fdiv_rn(a0, l) : 0.f, any ? __fdiv_rn(a1, l) : 0.f);
  store_pair<OUT>(dst + 2 * OSZ, any ? __fdiv_rn(a2, l) : 0.f, any ? __fdiv_rn(a3, l) : 0.f);
  if (p.lse != 0 && c == 0) reinterpret_cast<float*>(p.lse)[row] = any ? (m + log2f(l)) * kLn2 : -INFINITY;
}

}  // namespace

#ifndef ATTN_KV_FP8
// name: attn_kv_<in>_d<64|128>_<out>; D <= 64 runs the d64 kernel, 64 < D <= 128 the d128 kernel
#define ATTN_KV_KERNEL(NAME, KIND, DB, OUT)                                                                     \
  extern "C" __global__ void __launch_bounds__(kAttnKvThreads, 1)                                              \
      NAME(const __grid_constant__ CUtensorMap tq, const __grid_constant__ CUtensorMap tk,                    \
           const __grid_constant__ CUtensorMap tv, const __grid_constant__ AttnKvParams p) {                  \
    kv_body<KIND, DB, OUT>(&tq, &tk, &tv, p);                                                                  \
  }
#define ATTN_KV_D(IN, KIND, OUT16)                                  \
  ATTN_KV_KERNEL(attn_kv_##IN##_d64_##IN, KIND, 64, OUT16)          \
  ATTN_KV_KERNEL(attn_kv_##IN##_d64_f32, KIND, 64, OUT_F32)         \
  ATTN_KV_KERNEL(attn_kv_##IN##_d128_##IN, KIND, 128, OUT16)        \
  ATTN_KV_KERNEL(attn_kv_##IN##_d128_f32, KIND, 128, OUT_F32)
ATTN_KV_D(f16, KIND_F16, OUT_F16)
ATTN_KV_D(bf16, KIND_BF16, OUT_BF16)

#define ATTN_KV_COMBINE(NAME, OUT)                                                                                      \
  extern "C" __global__ void __launch_bounds__(kAttnKvCombineThreads) NAME(const __grid_constant__ AttnKvParams p) { \
    kv_combine<OUT>(p);                                                                                                 \
  }
ATTN_KV_COMBINE(attn_kv_combine_f16, OUT_F16)
ATTN_KV_COMBINE(attn_kv_combine_bf16, OUT_BF16)
ATTN_KV_COMBINE(attn_kv_combine_f32, OUT_F32)

// Scatter of new tokens into the cache: 16-byte loads and stores of 16-bit elements, grid-stride.
extern "C" __global__ void __launch_bounds__(256) attn_kv_write(const __grid_constant__ AttnKvWriteParams p) {
  const uint32_t dc = p.D / 8;
  for (uint64_t u = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; u < p.units;
       u += static_cast<uint64_t>(gridDim.x) * blockDim.x) {
    const uint64_t d = (u % dc) * 8, rest = u / dc;
    const uint64_t hk = rest % p.Hkv, n = rest / p.Hkv;
    const int64_t slot = reinterpret_cast<const int*>(p.slots)[n];
    if (slot < 0 || static_cast<uint64_t>(slot) >= p.slot_end) continue;
    const uint64_t pg = static_cast<uint64_t>(slot) / p.page, row = static_cast<uint64_t>(slot) % p.page;
    const uint64_t b = n / p.Snew, t = n % p.Snew;
    const uint4 kx = *reinterpret_cast<const uint4*>(p.kn + (b * p.kn_sb + t * p.kn_st + hk * p.kn_sh + d) * 2);
    const uint4 vx = *reinterpret_cast<const uint4*>(p.vn + (b * p.vn_sb + t * p.vn_st + hk * p.vn_sh + d) * 2);
    *reinterpret_cast<uint4*>(p.kc + (pg * p.kc_sp + row * p.kc_sr + hk * p.kc_sh + d) * 2) = kx;
    *reinterpret_cast<uint4*>(p.vc + (pg * p.vc_sp + row * p.vc_sr + hk * p.vc_sh + d) * 2) = vx;
  }
}
#else
// -DATTN_KV_FP8 (cubin attention_kv_fp8): the fp8-cache kernels.
// name: attn_kv_<in>_<e4m3|e5m2>_d<64|128>_<out>
#define ATTN_KV_F8_KERNEL(NAME, KIND, DB, OUT, CF)                                                              \
  extern "C" __global__ void __launch_bounds__(kAttnKvThreads, 1)                                              \
      NAME(const __grid_constant__ CUtensorMap tq, const __grid_constant__ CUtensorMap tk,                    \
           const __grid_constant__ CUtensorMap tv, const __grid_constant__ AttnKvParams p) {                  \
    kv_body<KIND, DB, OUT, CF>(&tq, &tk, &tv, p);                                                              \
  }
#define ATTN_KV_F8_D(IN, KIND, OUT16, F, CF)                                      \
  ATTN_KV_F8_KERNEL(attn_kv_##IN##_##F##_d64_##IN, KIND, 64, OUT16, CF)           \
  ATTN_KV_F8_KERNEL(attn_kv_##IN##_##F##_d64_f32, KIND, 64, OUT_F32, CF)          \
  ATTN_KV_F8_KERNEL(attn_kv_##IN##_##F##_d128_##IN, KIND, 128, OUT16, CF)         \
  ATTN_KV_F8_KERNEL(attn_kv_##IN##_##F##_d128_f32, KIND, 128, OUT_F32, CF)
ATTN_KV_F8_D(f16, KIND_F16, OUT_F16, e4m3, CF_E4M3)
ATTN_KV_F8_D(f16, KIND_F16, OUT_F16, e5m2, CF_E5M2)
ATTN_KV_F8_D(bf16, KIND_BF16, OUT_BF16, e4m3, CF_E4M3)
ATTN_KV_F8_D(bf16, KIND_BF16, OUT_BF16, e5m2, CF_E5M2)

#define ATTN_KV_F8_COMBINE(NAME, OUT)                                                                                   \
  extern "C" __global__ void __launch_bounds__(kAttnKvCombineThreads) NAME(const __grid_constant__ AttnKvParams p) { \
    kv_combine<OUT, true>(p);                                                                                           \
  }
ATTN_KV_F8_COMBINE(attn_kv_combine_fp8_f16, OUT_F16)
ATTN_KV_F8_COMBINE(attn_kv_combine_fp8_bf16, OUT_BF16)
ATTN_KV_F8_COMBINE(attn_kv_combine_fp8_f32, OUT_F32)

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

// Scatter of new tokens into an fp8 cache, quantized with per-head scales: 16-byte loads and 8-byte stores, grid-stride.
extern "C" __global__ void __launch_bounds__(256) attn_kv_write_fp8(const __grid_constant__ AttnKvWriteParams p) {
  const uint32_t dc = p.D / 8;
  const bool bf16 = p.in_bf16 != 0, e5m2 = p.e5m2 != 0;
  for (uint64_t u = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; u < p.units;
       u += static_cast<uint64_t>(gridDim.x) * blockDim.x) {
    const uint64_t d = (u % dc) * 8, rest = u / dc;
    const uint64_t hk = rest % p.Hkv, n = rest / p.Hkv;
    const int64_t slot = reinterpret_cast<const int*>(p.slots)[n];
    if (slot < 0 || static_cast<uint64_t>(slot) >= p.slot_end) continue;
    const uint64_t pg = static_cast<uint64_t>(slot) / p.page, row = static_cast<uint64_t>(slot) % p.page;
    const uint64_t b = n / p.Snew, t = n % p.Snew;
    const uint4 kx = *reinterpret_cast<const uint4*>(p.kn + (b * p.kn_sb + t * p.kn_st + hk * p.kn_sh + d) * 2);
    const uint4 vx = *reinterpret_cast<const uint4*>(p.vn + (b * p.vn_sb + t * p.vn_st + hk * p.vn_sh + d) * 2);
    const float ks = reinterpret_cast<const float*>(p.k_scale)[hk], vs = reinterpret_cast<const float*>(p.v_scale)[hk];
    *reinterpret_cast<uint2*>(p.kc + pg * p.kc_sp + row * p.kc_sr + hk * p.kc_sh + d) = kv_quant8(kx, ks, bf16, e5m2);
    *reinterpret_cast<uint2*>(p.vc + pg * p.vc_sp + row * p.vc_sr + hk * p.vc_sh + d) = kv_quant8(vx, vs, bf16, e5m2);
  }
}
#endif
