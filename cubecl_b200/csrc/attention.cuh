// Device helpers shared by the attention forward (attention.cu) and backward (attention_bwd.cu) kernels.
#pragma once
#include <cstdint>

namespace b200 {

enum : int { KIND_F16 = 0, KIND_BF16 = 1 };
enum : int { OUT_F16 = 0, OUT_BF16 = 1, OUT_F32 = 2 };

__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// two f32 -> one register of two 16-bit values, lo in the low half (RNE)
template <int KIND>
__device__ __forceinline__ uint32_t pack16(float lo, float hi) {
  uint32_t r;
  if constexpr (KIND == KIND_BF16) asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  else asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}

// Varlen (kernel_params.h: AttnVarlenParams): sequence b's first row and length, each cu value clamped to [0, T] and the
// length to [0, maxlen], so malformed offsets give unspecified values but never an access outside the tensor.
__device__ __forceinline__ void varlen_seq(uint64_t cu, uint32_t b, uint32_t T, uint32_t maxlen, int& start, int& len) {
  const int32_t* c = reinterpret_cast<const int32_t*>(cu);
  const int lo = min(max(__ldg(c + b), 0), static_cast<int>(T)), hi = min(max(__ldg(c + b + 1), 0), static_cast<int>(T));
  start = lo;
  len = min(max(hi - lo, 0), static_cast<int>(maxlen));
}

// The band of keys row i sees: [band_lo, band_hi], clamped to [0, L] and [-1, L - 1] (empty when lo > hi).  With (off, left,
// right, L) = (Lk - Lq, left, right, Lk) it is the keys of query i; with (Lq - Lk, right, left, Lq) the queries of key i.
__device__ __forceinline__ int band_lo(int i, int off, int left, int L) {
  if (left < 0) return 0;
  return static_cast<int>(min(max(static_cast<long long>(i) + off - left, 0ll), static_cast<long long>(L)));
}
__device__ __forceinline__ int band_hi(int i, int off, int right, int L) {
  if (right < 0) return L - 1;
  return static_cast<int>(min(max(static_cast<long long>(i) + off + right, -1ll), static_cast<long long>(L) - 1));
}

// The blocks of `blk` columns that rows [ra, rb] of a band reach: [*lo, *hi), empty when nothing is visible.
__device__ __forceinline__ void band_blocks(int ra, int rb, int off, int left, int right, int L, int blk, int& lo, int& hi) {
  const int a = band_lo(ra, off, left, L), z = band_hi(rb, off, right, L);
  lo = a / blk;
  hi = z >= a ? z / blk + 1 : lo;
}

// Zeroes rows [from, rows) of a SWIZZLE_128B tile of `nch` chunks (128-byte rows, chunk stride `chunk` bytes) with the 128
// threads of one warpgroup, then makes the zeros visible to wgmma (the async proxy) and syncs the warpgroup on named barrier
// `bar`.  The swizzle permutes 16-byte units inside a row, so a row stays a row.
__device__ __forceinline__ void zero_rows(uint32_t tile, int nch, uint32_t chunk, int from, int rows, uint32_t bar) {
  const uint32_t t = threadIdx.x & 127u;
  const int units = (rows - from) * 8;
  for (int c = 0; c < nch; ++c)
    for (int u = static_cast<int>(t); u < units; u += 128) {
      const uint32_t addr = tile + c * chunk + static_cast<uint32_t>(from) * 128u + static_cast<uint32_t>(u) * 16u;
      asm volatile("st.shared.v4.b32 [%0], {%1, %1, %1, %1};" ::"r"(addr), "r"(0u) : "memory");
    }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  asm volatile("bar.sync %0, 128;" ::"r"(bar) : "memory");
}

// Direct stores of one forward consumer's m64 x DB f32 fragment O divided by the row sums l0, l1 (+0 for a row without keys,
// l = 0), rounded once to the output dtype, for rows < rows_left of a [T, H, D] view: partial blocks at a sequence's end,
// where a TMA store would write the next sequence's rows.  base is the byte address of the consumer's first row, st the row
// stride in bytes.
template <int DB, int OUT>
__device__ __forceinline__ void store_frag_direct(const float (&acc)[DB / 2], float l0, float l1, uint64_t base, uint64_t st,
                                                  int rows_left, uint32_t D) {
  constexpr uint32_t OSZ = (OUT == OUT_F32) ? 4u : 2u;
  const uint32_t t = threadIdx.x & 127u, lane = t & 31u;
  const int r = static_cast<int>((t >> 5) * 16u + (lane >> 2));
  const uint32_t col = 2u * (lane & 3u);
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int rr = r + 8 * hh;
    if (rr >= rows_left) continue;
    const float l = hh ? l1 : l0;
    const uint64_t row = base + static_cast<uint64_t>(rr) * st + col * OSZ;
#pragma unroll
    for (int j = 0; j < DB / 8; ++j) {
      if (8u * j + col >= D) continue;
      const float x0 = l > 0.f ? __fdiv_rn(acc[4 * j + 2 * hh], l) : 0.f, x1 = l > 0.f ? __fdiv_rn(acc[4 * j + 2 * hh + 1], l) : 0.f;
      const uint64_t a = row + 8u * j * OSZ;
      if constexpr (OUT == OUT_F32) {
        asm volatile("st.global.v2.f32 [%0], {%1, %2};" ::"l"(a), "f"(x0), "f"(x1) : "memory");
      } else {
        asm volatile("st.global.b32 [%0], %1;" ::"l"(a), "r"(pack16<OUT == OUT_BF16 ? KIND_BF16 : KIND_F16>(x0, x1)) : "memory");
      }
    }
  }
}

}  // namespace b200
