// Hand-written sm_90a GEMM: TMA -> 128B-swizzled smem ring -> wgmma (accumulators in registers) -> direct stores.
// Persistent, warp-specialised: warpgroup 0 is the producer (one thread issues the TMA loads), warpgroups 1 and 2 each
// run wgmma on 64 rows of the CTA's 128-row tile.  Optional 2-CTA cluster (CG = 2, "2sm" tiles of 256 x BLOCK_N): each
// CTA computes its own 128 rows and loads half of the B tile, multicast into both CTAs, so a pair reads B from L2 once.
//
// Replaces: the (out-of-tree, cubek) `matmul::launch` kernel bodies that CubeCL lowers to nvcuda::wmma / mma.sync
// through crates/cubecl-cpp/src/shared/mma.rs:48-174 and crates/cubecl-cpp/src/cuda/ptx/mma.rs:30-61.
// Semantics follow the reference's CPU expectation `test_simple_cube_expected`
// (crates/cubecl-core/src/runtime_tests/cmma.rs:695-721): inputs widened to f32, f32 accumulate over increasing k.
// Shape / batch-broadcast rule: crates/cubecl-zspace/src/shape.rs:489-517 (resolved on the host, see capi.cpp).
//
// Compiled to a cubin (no host code here): nvcc -cubin -gencode arch=compute_90a,code=sm_90a
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "kernel_params.h"
#include "ptx.cuh"

using namespace b200;

enum : int { KIND_F16 = 0, KIND_BF16 = 1, KIND_TF32 = 2, KIND_E4M3 = 3, KIND_E5M2 = 4, KIND_U8 = 5, KIND_S8 = 6 };
enum : int { OUT_F16 = 0, OUT_BF16 = 1, OUT_F32 = 2 };  // OUT_F32 is a raw 32-bit store: it also carries the s32 accumulators of the int kinds

constexpr int kNumThreads = 384;  // warpgroup 0: TMA producer, warpgroups 1-2: wgmma + epilogue (64 rows each)

#include <type_traits>
struct TileCoord {
  uint32_t b, m_blk, n_blk;
};

__device__ __forceinline__ TileCoord tile_coord(uint32_t t, const GemmParams& p) {
  const uint32_t per_batch = p.tiles_m * p.tiles_n;
  TileCoord c;
  c.b = t / per_batch;
  uint32_t r = t - c.b * per_batch;
  const uint32_t strip = p.group_m * p.tiles_n;
  const uint32_t g = r / strip;
  const uint32_t first_m = g * p.group_m;
  const uint32_t gsize = min(p.group_m, p.tiles_m - first_m);
  const uint32_t in = r - g * strip;
  c.m_blk = first_m + in % gsize;
  c.n_blk = in / gsize;
  return c;
}

struct WorkUnit {
  uint32_t tile, kb0, kb1;
  uint32_t slab;   // partial units: slab index (range * sk_umax + unit within the range)
  bool partial;
};

// The sequence of work units of one CTA pair: stream-K ranges first, whole tiles after (see GemmParams).  Every role of the
// CTA (TMA producers, MMA issuer, epilogue warps) walks the same sequence with its own copy of this iterator.
struct UnitIter {
  uint32_t c, C, num_kb;
  uint32_t r;          // current stream-K range (c, c + C, ...), >= sk_ranges once the head is done
  uint32_t u;          // unit index inside the current range
  uint64_t pos, hi;    // unconsumed part [pos, hi) of the current range, in linear k-blocks
  uint32_t next_tile;  // next whole tile
  bool open;           // [pos, hi) of range r has been set up
};

__device__ __forceinline__ UnitIter unit_iter(uint32_t cluster, uint32_t n_clusters, uint32_t num_kb) {
  UnitIter it;
  it.c = cluster; it.C = n_clusters; it.num_kb = num_kb;
  it.r = cluster; it.u = 0; it.pos = 0; it.hi = 0; it.next_tile = cluster; it.open = false;
  return it;
}

__device__ __forceinline__ uint64_t sk_range_lo(uint32_t r, const GemmParams& p, uint32_t num_kb) {
  return (static_cast<uint64_t>(r) * p.sk_tiles * num_kb) / p.sk_ranges;
}
// range that owns linear k-block x: the largest r with sk_range_lo(r) <= x (ranges are non-empty: sk_ranges <= sk_tiles * num_kb)
__device__ __forceinline__ uint32_t sk_owner(uint64_t x, const GemmParams& p, uint32_t num_kb) {
  return static_cast<uint32_t>(((x + 1) * p.sk_ranges - 1) / (static_cast<uint64_t>(p.sk_tiles) * num_kb));
}

__device__ __forceinline__ bool next_unit(UnitIter& it, const GemmParams& p, WorkUnit& w) {
  while (p.sk_tiles != 0 && it.r < p.sk_ranges) {
    if (!it.open) {
      it.pos = sk_range_lo(it.r, p, it.num_kb);
      it.hi = sk_range_lo(it.r + 1, p, it.num_kb);
      it.u = 0;
      it.open = true;
    }
    if (it.pos < it.hi) {
      const uint32_t tau = static_cast<uint32_t>(it.pos / it.num_kb);
      const uint64_t t0 = static_cast<uint64_t>(tau) * it.num_kb;
      const uint64_t end = (it.hi < t0 + it.num_kb) ? it.hi : t0 + it.num_kb;
      w.tile = p.full_tiles + tau;
      w.kb0 = static_cast<uint32_t>(it.pos - t0);
      w.kb1 = static_cast<uint32_t>(end - t0);
      w.partial = !(w.kb0 == 0 && w.kb1 == it.num_kb);
      w.slab = it.r * p.sk_umax + it.u;
      it.pos = end;
      ++it.u;
      return true;
    }
    it.r += it.C;
    it.open = false;
  }
  if (it.next_tile < p.full_tiles) {
    w.tile = it.next_tile; w.kb0 = 0; w.kb1 = it.num_kb; w.slab = 0; w.partial = false;
    it.next_tile += it.C;
    return true;
  }
  return false;
}


// Stores of one accumulator fragment pair: columns n, n + 1 of one output row.
template <int OUT>
__device__ __forceinline__ void store_pair(uint64_t row_ptr, uint32_t n, uint32_t N, bool vec, uint32_t v0, uint32_t v1) {
  if constexpr (OUT == OUT_F32) {
    uint32_t* dst = reinterpret_cast<uint32_t*>(row_ptr) + n;
    if (vec && n + 1 < N) *reinterpret_cast<uint2*>(dst) = make_uint2(v0, v1);
    else { if (n < N) dst[0] = v0; if (n + 1 < N) dst[1] = v1; }
  } else {
    uint16_t* dst = reinterpret_cast<uint16_t*>(row_ptr) + n;
    uint32_t packed;   // cvt packs (hi, lo): lo lands in the low half, the lower address
    if constexpr (OUT == OUT_BF16) asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(packed) : "r"(v1), "r"(v0));
    else asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(packed) : "r"(v1), "r"(v0));
    if (vec && n + 1 < N) *reinterpret_cast<uint32_t*>(dst) = packed;
    else { if (n < N) dst[0] = static_cast<uint16_t>(packed & 0xFFFFu); if (n + 1 < N) dst[1] = static_cast<uint16_t>(packed >> 16); }
  }
}

__device__ __forceinline__ uint32_t acc_bits(float x) { return __float_as_uint(x); }
__device__ __forceinline__ uint32_t acc_bits(uint32_t x) { return x; }

// PROMOTE (the block-scaled kernels): every k-block is summed by wgmma into a fresh register partial (one 128- or 112-column
// part of the tile at a time), which is then added to the f32 accumulators with round-to-nearest adds.  wgmma truncates as it
// accumulates; promoting per 64 elements of K keeps that error to one k-block instead of letting it build up over K.
// MT: 128-row sub-tiles of M per CTA.  MT = 2 (the 2sm_m512 pair tile, 512 x BLOCK_N per CTA pair) gives each consumer
// warpgroup two m64 row blocks that share every B stage: per FLOP the pair reads a third less operand data from L2 than the
// 256 x 256 tile at the same accumulator count per thread.
// QM (integer-quantized operands, s8 codes, K-major; capi.cpp: b200_matmul_quantized):
//   QM_BLOCK   per-block scales.  Each Bk-element block j of K is summed exactly by wgmma into a fresh s32 partial, which is
//              folded into f32 accumulators as acc = fma(f32(D_j), rn(eff_a[m, j] * eff_b[n, j]), acc) in increasing j.  The
//              producer also loads the stage's f32 effective-scale tiles ([128/Bk][rows] boxes of a block-major buffer) through
//              tma_a_lo / tma_b_lo into a region after the operand ring.
//   QM_TENSOR  one f32 scale per side: the s8 mainloop into s32 accumulators; the epilogue stores rn(f32(D) * rn(g_a * g_b)).
//   QM_FP8     fp8 codes (capi.cpp: b200_matmul_quantized_fp8; KIND the lhs format, the rhs format chosen at run time as for
//              the mixed fp8 kernels): the QM_BLOCK producer and fold, each block summed by fp8 wgmma into a fresh f32 partial
//              P_j and folded as acc = fma(P_j, rn(eff_a * eff_b), acc) -- no integer conversion.
enum : int { QM_NONE = 0, QM_BLOCK = 1, QM_TENSOR = 2, QM_FP8 = 3 };
// CONV (2-D convolution as an implicit GEMM; capi.cpp: b200_conv2d): the A tile of k-block kb is one im2col load -- 128
// consecutive output pixels x 64 channels of kernel position kb / cv_cblk, channel block kb % cv_cblk -- which TMA writes in
// exactly the 128B-swizzled [128 rows x 128 B] layout of a K-major A tile; B is the weights' [n_local x 64 channels] box of
// that (kernel position, channel block).  Channels past C read as zero on both sides.  Everything after the load is the GEMM.
// CB (convolution backward; capi.cpp: b200_conv2d_backward_data / _weight):
//   CB_DGRAD  the CONV producer; the epilogue stores GEMM row (n, i, j) of one output phase at its dx pixel (GemmParams dx_*),
//             with row addresses computed once per tile.  Direct stores only: a TMA store cannot describe that row mapping.
//   CB_WGRAD  MN-major A (dy: 64 output channels x 64 pixels per chunk, tiled) and B: each 64-column chunk of the B tile is one
//             im2col load of 64 pixels x 64 channels of x at one (kernel position, channel block), which TMA writes as
//             [64 pixel rows x 128 B], exactly an MN-major B chunk.  Pixels past N * OH * OW read as zero on both sides (tiled
//             out-of-bounds fill for dy; the im2col walk runs into image N for x).  The epilogue maps virtual column
//             (kpos, ch) to dw's column and drops ch >= C, in the direct stores and in the TMA-store coordinate.
// CONV_DIMS (capi.cpp: b200_conv3d*): 3 runs the CONV producer, CB_DGRAD epilogue and CB_WGRAD producer over a 3-D convolution
// -- 5-D im2col loads (C, W, H, D, N) with offsets (kx dw, ky dh, kz dd), pixels and kernel positions decoded with the depth
// term (GemmParams cv_odhw, cv_khw, dx_sd).  2 is the 2-D convolution; every other stage of the kernel is the same.
//   CB_TCONV  transposed convolution, every stride phase of a layer in one launch (TconvParams, kernel_params.h): per tile
//             the producer finds the tile's phase and loads through that phase's im2col and weight maps; the consumers run
//             the phase's own k-block count from zeroed accumulators (a phase no tap reaches runs none and stores
//             act(bias)), then store as CB_DGRAD at the phase's rows.
//   CB_GRP_M  grouped matmul, ragged M (GroupedParams, kernel_params.h): each CTA reads the group offsets once into a table
//             in shared memory and maps every tile to (group, m-block, n-block) from it; A rows start at the group's first
//             row, B is the group's batch of the 3-D rhs map.  A tile that the group's end cuts leaves through direct
//             stores of the group's rows only.
//   CB_GRP_K  grouped matmul, ragged K (the weight gradient; MN-major operands as CB_WGRAD): tile t belongs to group
//             t / (tiles_m * tiles_n) and runs that group's k-blocks from its first position; in the last one the rows of
//             positions past the group are zeroed in shared memory before the MMAs.  A group without k-blocks stores +0.
enum : int { CB_NONE = 0, CB_DGRAD = 1, CB_WGRAD = 2, CB_TCONV = 3, CB_GRP_M = 4, CB_GRP_K = 5 };

// phase of tile t in a transposed-convolution launch (phases in table order, tiles in one list)
__device__ __forceinline__ uint32_t tconv_phase(uint32_t t, const TconvParams& tp) {
  uint32_t q = 0;
  while (q + 1 < tp.phases && t >= tp.ph[q + 1].tile0) ++q;
  return q;
}
// tile_coord inside one phase's grid of tiles_m x p.tiles_n tiles
__device__ __forceinline__ TileCoord tconv_coord(uint32_t loc, uint32_t tiles_m, const GemmParams& p) {
  const uint32_t strip = p.group_m * p.tiles_n, g = loc / strip, first_m = g * p.group_m;
  const uint32_t gsize = min(p.group_m, tiles_m - first_m), in = loc - g * strip;
  TileCoord c;
  c.b = 0;
  c.m_blk = first_m + in % gsize;
  c.n_blk = in / gsize;
  return c;
}
// tile t's coordinate: in phase q's grid for a transposed convolution, tile_coord otherwise
template <int CB>
__device__ __forceinline__ TileCoord unit_coord(uint32_t t, const GemmParams& p, const TconvParams* tcp, uint32_t q) {
  if constexpr (CB == CB_TCONV) return tconv_coord(t - tcp->ph[q].tile0, tcp->ph[q].tiles_m, p);
  else return tile_coord(t, p);
}

// Grouped matmul: the shared-memory table of one CTA (GroupedParams), built by one warp.  Lane l takes groups
// [l S, (l + 1) S), S = ceil(G / 32): a running maximum of offs (o_{-1} = 0) clamped to T gives the ends o[g], and a
// prefix sum of the groups' tile-rows of `rows` rows gives pre[g] (pre[G] = all of them).  A non-empty group's tile-rows
// start at its first row rounded down to a multiple of mask + 1.
__device__ __forceinline__ void grp_tables(const GroupedParams& gp, uint32_t* o, uint32_t* pre, uint32_t rows, uint32_t mask,
                                           uint32_t lane) {
  const uint32_t G = gp.groups, S = (G + 31u) / 32u, b = min(lane * S, G), e = min(b + S, G);
  const int32_t* offs = reinterpret_cast<const int32_t*>(gp.offs);
  int32_t mx = 0;
  for (uint32_t i = b; i < e; ++i) {
    const int32_t v = __ldg(offs + i);
    o[i] = static_cast<uint32_t>(v);
    mx = max(mx, v);
  }
  int32_t run = mx;   // inclusive running maximum over the lanes
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int32_t y = __shfl_up_sync(0xFFFFFFFFu, run, d);
    if (static_cast<int>(lane) >= d) run = max(run, y);
  }
  int32_t m = __shfl_up_sync(0xFFFFFFFFu, run, 1);
  if (lane == 0) m = 0;
  uint32_t prev = min(static_cast<uint32_t>(m), gp.T), cnt = 0;
  for (uint32_t i = b; i < e; ++i) {
    m = max(m, static_cast<int32_t>(o[i]));
    const uint32_t end = min(static_cast<uint32_t>(m), gp.T), tr = end > prev ? (end - (prev & ~mask) + rows - 1u) / rows : 0u;
    o[i] = end;
    pre[i] = tr;
    cnt += tr;
    prev = end;
  }
  uint32_t sum = cnt;   // inclusive prefix sum over the lanes
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, sum, d);
    if (static_cast<int>(lane) >= d) sum += y;
  }
  uint32_t acc = sum - cnt;
  for (uint32_t i = b; i < e; ++i) {
    const uint32_t tr = pre[i];
    pre[i] = acc;
    acc += tr;
  }
  if (lane == 31) pre[G] = sum;
}

struct GrpUnit {
  TileCoord tc;       // b = the group
  uint32_t g;
  uint32_t lo, hi;    // the group's rows (ragged M) or positions (ragged K): [o_{g-1}, o_g)
  uint32_t row0;      // ragged M: first row of the group's tile-rows (lo rounded down to a multiple of MASK + 1)
  uint32_t nkb;       // k-blocks of the tile
};
// tile t of a grouped launch: its group (ragged M: the last g with pre[g] <= t / tiles_n, by bisection), and its coordinate
// inside the group's grid of tile-rows x tiles_n in group_m strips; ragged M runs ceil(K / BLOCK_K) k-blocks per tile
template <int CB, uint32_t MASK, uint32_t BLOCK_K>
__device__ __forceinline__ GrpUnit grp_unit(uint32_t t, const GemmParams& p, const GroupedParams& gp, const uint32_t* o, const uint32_t* pre) {
  uint32_t g, loc, tiles_m;
  if constexpr (CB == CB_GRP_M) {
    const uint32_t q = t / p.tiles_n;
    uint32_t lo = 0, hi = gp.groups;
    while (hi - lo > 1u) {
      const uint32_t mid = (lo + hi) >> 1;
      if (pre[mid] <= q) lo = mid; else hi = mid;
    }
    g = lo;
    loc = t - pre[g] * p.tiles_n;
    tiles_m = pre[g + 1] - pre[g];
  } else {
    const uint32_t per = p.tiles_m * p.tiles_n;
    g = t / per;
    loc = t - g * per;
    tiles_m = p.tiles_m;
  }
  GrpUnit u;
  u.tc = tconv_coord(loc, tiles_m, p);
  u.tc.b = g;
  u.g = g;
  u.lo = g ? o[g - 1] : 0u;
  u.hi = o[g];
  u.row0 = u.lo & ~MASK;
  u.nkb = (CB == CB_GRP_M) ? (p.K + BLOCK_K - 1u) / BLOCK_K : (u.hi - u.lo + 63u) / 64u;
  return u;
}

// Ragged K, the last k-block of a group: rows of positions >= o_g (the next group's, or zeros past T) are cleared in the four
// [64 positions x 128 B] MN-major chunks of the stage (A's two, then B's two) -- 0 * NaN is NaN inside an MMA.  A position is
// one whole 128-byte row of a chunk whatever the swizzle.  Both consumer warpgroups (thread ct of 256), then one barrier.
__device__ __forceinline__ void grp_zero_rows(uint32_t stage, uint32_t keep, uint32_t ct) {
  const uint32_t per = (64u - keep) * 8u;   // 16-byte units per chunk
  for (uint32_t u = ct; u < 4u * per; u += 256u) {
    const uint32_t c = u / per, r = u - c * per;
    asm volatile("st.shared.v4.b32 [%0], {%1, %1, %1, %1};" ::"r"(stage + c * 8192u + keep * 128u + r * 16u), "r"(0u) : "memory");
  }
  fence_proxy_async_smem();   // generic-proxy writes -> visible to wgmma's async-proxy reads
  asm volatile("bar.sync 1, 256;" ::: "memory");
}

template <int CG, int BLOCK_N, bool A_MN, bool B_MN, int KIND, int OUT, int STAGES, bool PROMOTE = false, int MT = 1, int QM = QM_NONE,
          bool CONV = false, int CB = CB_NONE, int CONV_DIMS = 2>
__device__ __forceinline__ void gemm_body(const CUtensorMap* tma_a_hi, const CUtensorMap* tma_b_hi, const CUtensorMap* tma_a_lo,
                                          const CUtensorMap* tma_b_lo, const CUtensorMap* tma_out, const GemmParams& p,
                                          const TconvParams* tcp = nullptr, const GroupedParams* gpp = nullptr) {
  constexpr bool INT_ACC = (KIND == KIND_U8 || KIND == KIND_S8) && QM != QM_BLOCK;
  constexpr bool GRP = (CB == CB_GRP_M || CB == CB_GRP_K);
  // ragged M also takes fp8-quantized K-major operands (gemm_grouped_qf8_*): the QM_FP8 producer loads the lhs scale tile at
  // the group's rows (m0) and the rhs one from the group's batch (bb)
  static_assert(!GRP || (!CONV && !PROMOTE && MT == 1 && CONV_DIMS == 2 &&
                         (((KIND == KIND_BF16 || KIND == KIND_F16) && QM == QM_NONE) ||
                          (CB == CB_GRP_M && QM == QM_FP8 && !A_MN && !B_MN))),
                "grouped matmul: 16-bit kinds (fp8-quantized K-major operands for ragged M), one M sub-tile");
  static_assert(CB != CB_GRP_K || (A_MN && B_MN), "ragged K: MN-major operands");
  static_assert(QM == QM_NONE || ((QM == QM_FP8 ? (KIND == KIND_E4M3 || KIND == KIND_E5M2) : KIND == KIND_S8) && !A_MN && !B_MN &&
                                  !PROMOTE && MT == 1), "quantized operands: s8 (fp8 for QM_FP8), K-major");
  constexpr bool QBLK = (QM == QM_BLOCK || QM == QM_FP8);   // per-block scale tiles in every stage
  // ragged M with an M-contiguous lhs: the group's first row is the innermost coordinate of the A loads, and such loads at
  // coordinates that are not a multiple of 16 bytes faulted (illegal instruction) on an H100 -- the group's tile-rows start
  // at a multiple of 64 rows instead, and the rows before the group are not stored.  With per-block scale tiles the row is
  // the innermost coordinate of the f32 A scale load ([blocks][rows]): tile-rows start at a multiple of 4 rows.
  constexpr uint32_t GRP_MASK = (CB == CB_GRP_M && A_MN) ? 63u : (CB == CB_GRP_M && QBLK) ? 3u : 0u;
  static_assert(!CONV || ((KIND == KIND_BF16 || KIND == KIND_F16) && !A_MN && !B_MN && !PROMOTE && MT == 1 && QM == QM_NONE),
                "convolution: 16-bit kinds, K-major operands");
  static_assert(CB != CB_DGRAD || CONV, "data gradient: the convolution producer");
  static_assert(CB != CB_TCONV || CONV, "transposed convolution: the convolution producer");
  static_assert(CONV_DIMS == 2 || (CONV_DIMS == 3 && (CONV || CB == CB_WGRAD)), "3-D: the convolution kernels");
  static_assert(CB != CB_WGRAD || (!CONV && A_MN && B_MN && (KIND == KIND_BF16 || KIND == KIND_F16) && !PROMOTE && MT == 1 && QM == QM_NONE),
                "weight gradient: 16-bit kinds, MN-major operands");
  // per-block scale tiles of one stage, sized for the finest block (Bk = 32: four blocks per 128-element stage)
  constexpr uint32_t SC_A_BYTES = QBLK ? 128u * 4u * 4u : 0u;
  constexpr uint32_t SC_STAGE_BYTES = QBLK ? SC_A_BYTES + BLOCK_N * 4u * 4u : 0u;
  constexpr int ESZ = (KIND == KIND_TF32) ? 4 : (KIND >= KIND_E4M3) ? 1 : 2;
  static_assert(ESZ == 2 || (!A_MN && !B_MN), "wgmma reads MN-major operands for 16-bit kinds only");
  constexpr int BLOCK_K = 128 / ESZ;  // one 128-byte swizzle row of K per stage
  constexpr int MMA_K = 32 / ESZ;     // K per wgmma instruction: 32 bytes
  constexpr int N_LOCAL = BLOCK_N / CG;  // rows of the B tile this CTA loads (multicast to the pair)
  constexpr uint32_t A_SUB_BYTES = 128 * 128;       // one 128-row sub-tile of A: 128 rows x 128 B
  constexpr uint32_t A_BYTES = MT * A_SUB_BYTES;
  constexpr uint32_t B_BYTES = BLOCK_N * 128;
  constexpr uint32_t STAGE_BYTES = A_BYTES + B_BYTES;
  constexpr int CHUNK_N = 64;                        // MN-major operand (16-bit): M/N elements per 128-byte row
  constexpr uint32_t CHUNK_BYTES = BLOCK_K * 128;    // MN-major operand: one [BLOCK_K x 128 B] chunk
  constexpr int NUM_CHUNKS = N_LOCAL / CHUNK_N;      // B chunks this CTA loads
  constexpr int NACC = BLOCK_N / 2;                  // accumulator registers per thread (m64 x BLOCK_N per warpgroup)
  static_assert(STAGE_BYTES % 1024 == 0, "stages must keep 1024-byte alignment for SWIZZLE_128B");
  using Acc = typename std::conditional<INT_ACC, uint32_t, float>::type;
  static_assert(!PROMOTE || (KIND == KIND_BF16 && !A_MN && !B_MN && MT == 1), "promoted accumulation: bf16, K-major operands");
  static_assert(MT == 1 || (MT == 2 && ESZ == 2), "two M sub-tiles per CTA: 16-bit kinds");
  constexpr int PH = (BLOCK_N % 128 == 0) ? 128 : 112;   // promoted partial: columns per wgmma (N = 224 -> two of 112)
  static_assert(!PROMOTE || BLOCK_N % PH == 0, "promoted partials tile BLOCK_N");
  constexpr int CW = (OUT == OUT_F32) ? 32 : 64;         // TMA-store staging: columns per 128-byte staging row

  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sc_base = smem_base + STAGES * STAGE_BYTES;   // QM_BLOCK: per-stage [A scales | B scales]
  const uint32_t bar_base = sc_base + STAGES * SC_STAGE_BYTES;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (STAGES + s); };
  const uint32_t split_flag = bar_base + 16u * STAGES;  // "this CTA reduces the slabs" broadcast among the consumer threads
  const uint32_t epi_base = bar_base + 1024u;            // TMA-store staging: one [64 rows x 128 B] tile per consumer warpgroup

  const uint32_t wg = threadIdx.x >> 7;
  const uint32_t rank = (CG == 2) ? cluster_ctarank() : 0u;
  const uint32_t cluster_id = (CG == 2) ? cluster_id_x() : blockIdx.x;
  const uint32_t n_clusters = (CG == 2) ? num_clusters_x() : gridDim.x;

  // grouped matmul: the offset table after the TMA-store staging (GroupedParams)
  uint32_t* const grp_o = reinterpret_cast<uint32_t*>(smem_raw + (epi_base + 16384u - smem_u32(smem_raw)));
  uint32_t* const grp_pre = grp_o + kGroupedMaxGroups;
  if (threadIdx.x == 0) {
    // a transposed-convolution phase without taps has no maps, nor has a grouped launch without k-blocks
    if ((CB != CB_TCONV || tcp->ph[0].num_kb != 0) && (!GRP || p.K != 0)) {
      tma_prefetch_desc(tma_a_hi);
      tma_prefetch_desc(tma_b_hi);
    }
    if (p.k_segments > 1) { tma_prefetch_desc(tma_a_lo); tma_prefetch_desc(tma_b_lo); }
    if constexpr (QBLK) { tma_prefetch_desc(tma_a_lo); tma_prefetch_desc(tma_b_lo); }
    if (p.tma_store) tma_prefetch_desc(tma_out);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full_bar(s), 1);        // one arrive.expect_tx by this CTA's producer; the peer's multicast bytes counted too
      mbar_init(empty_bar(s), 2 * CG);  // one arrive per consumer warpgroup of every CTA that writes into this stage
    }
    fence_mbar_init();
  }
  if constexpr (GRP) {
    if (threadIdx.x < 32) grp_tables(*gpp, grp_o, grp_pre, 128u * CG, GRP_MASK, threadIdx.x);
  }
  if constexpr (CG == 2) cluster_sync_all(); else __syncthreads();
  // grouped matmul: units past the device's tile count are skipped by every role alike
  uint32_t grp_total = 0;
  if constexpr (CB == CB_GRP_M) grp_total = grp_pre[gpp->groups] * p.tiles_n;
  else if constexpr (CB == CB_GRP_K) grp_total = p.full_tiles;

  // 3xTF32: x = hi + lo with hi = the top 19 bits of x (exactly what the tf32 datapath reads from an f32 operand, so the
  // ORIGINAL tensors serve as "hi") and lo = x - hi materialised once.  A*B ~= hi*hi + hi*lo + lo*hi is accumulated by
  // running the K loop over three segments with the operand tensor maps swapped per segment.
  const uint32_t seg_kb = (p.K + BLOCK_K - 1) / BLOCK_K;
  // hybrid schedule: the two bf16 segments cover K in 64-element stages (half as many k-blocks as the tf32 segment)
  const bool hyb = (KIND == KIND_TF32) && p.hyb != 0 && p.k_segments == 3;
  const uint32_t seg_kb1 = hyb ? (p.K + 63u) / 64u : seg_kb;
  const uint32_t num_kb = (p.k_segments == 3) ? seg_kb + 2u * seg_kb1 : seg_kb * p.k_segments;
  // (segment, k-block within it) of linear k-block kb
  auto seg_of = [&](uint32_t kb, uint32_t& seg, uint32_t& kk) {
    seg = 0; kk = kb;
    if (kk >= seg_kb) { kk -= seg_kb; seg = 1u + kk / seg_kb1; kk -= (seg - 1u) * seg_kb1; }
  };

  if (wg == 0) {
    // ===================================================================== TMA producer (one thread)
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      uint32_t s = 0, ph = 0;
      UnitIter it = unit_iter(cluster_id, n_clusters, num_kb);
      WorkUnit wu;
      while (next_unit(it, p, wu)) {
        if constexpr (CB == CB_TCONV) {
          // transposed convolution: the tile's phase, and its first pixel decoded with the phase's extents, once per tile;
          // per k-block the phase's im2col load at offsets (tap * dilation) and its weight load, as the data gradient
          const uint32_t q = tconv_phase(wu.tile, *tcp);
          const TconvPhase& P = tcp->ph[q];
          const TileCoord tc = tconv_coord(wu.tile - P.tile0, P.tiles_m, p);
          const uint32_t mu = (tc.m_blk * CG + rank) * 128u;
          const int n_row = static_cast<int>(tc.n_blk * BLOCK_N + rank * N_LOCAL);
          const CUtensorMap* am = reinterpret_cast<const CUtensorMap*>(&tcp->a[q]);
          const CUtensorMap* bm = reinterpret_cast<const CUtensorMap*>(&tcp->b[q]);
          int cv_w, cv_h, cv_d = 0, cv_n;
          if constexpr (CONV_DIMS == 3) {
            const uint32_t n = mu / P.e_dhw, r0 = mu - n * P.e_dhw, a = r0 / P.e_hw, r = r0 - a * P.e_hw, i = r / P.e_w;
            cv_n = static_cast<int>(n);
            cv_d = static_cast<int>(a) + P.lo_d;
            cv_h = static_cast<int>(i) + P.lo_h;
            cv_w = static_cast<int>(r - i * P.e_w) + P.lo_w;
          } else {
            const uint32_t n = mu / P.e_hw, r = mu - n * P.e_hw, i = r / P.e_w;
            cv_n = static_cast<int>(n);
            cv_h = static_cast<int>(i) + P.lo_h;
            cv_w = static_cast<int>(r - i * P.e_w) + P.lo_w;
          }
          for (uint32_t kb = 0; kb < P.num_kb; ++kb) {
            mbar_wait(empty_bar(s), ph ^ 1);
            const uint32_t sa = smem_base + s * STAGE_BYTES;
            const uint32_t sb = sa + A_BYTES;
            const uint32_t fb = full_bar(s);
            mbar_arrive_expect_tx(fb, STAGE_BYTES);
            const uint32_t kpos = kb / p.cv_cblk, cb = kb - kpos * p.cv_cblk;
            const int c0 = static_cast<int>(cb * 64u);
            if constexpr (CONV_DIMS == 3) {
              const uint32_t tz = kpos / P.t_hw, tr = kpos - tz * P.t_hw, ty = tr / P.t_w, tx = tr - ty * P.t_w;
              tma_load_im2col_5d(sa, am, fb, c0, cv_w, cv_h, cv_d, cv_n, static_cast<uint16_t>(tx * P.dil_w),
                                 static_cast<uint16_t>(ty * P.dil_h), static_cast<uint16_t>(tz * P.dil_d));
            } else {
              const uint32_t ty = kpos / P.t_w, tx = kpos - ty * P.t_w;
              tma_load_im2col_4d(sa, am, fb, c0, cv_w, cv_h, cv_n, static_cast<uint16_t>(tx * P.dil_w), static_cast<uint16_t>(ty * P.dil_h));
            }
            if constexpr (CG == 2) tma_load_3d_mc(sb + rank * N_LOCAL * 128u, bm, fb, static_cast<uint16_t>(3), c0, static_cast<int>(kpos), n_row);
            else tma_load_3d(sb, bm, fb, c0, static_cast<int>(kpos), n_row);
            if (++s == STAGES) { s = 0; ph ^= 1; }
          }
          continue;
        }
        GrpUnit gu;
        if constexpr (GRP) {
          if (wu.tile >= grp_total) break;
          gu = grp_unit<CB, GRP_MASK, BLOCK_K>(wu.tile, p, *gpp, grp_o, grp_pre);
          wu.kb0 = 0;
          wu.kb1 = gu.nkb;
        }
        TileCoord tc = tile_coord(wu.tile, p);
        if constexpr (GRP) tc = gu.tc;
        int m0 = static_cast<int>((tc.m_blk * CG + rank) * (128 * MT));
        if constexpr (CB == CB_GRP_M) m0 += static_cast<int>(gu.row0);   // the group's first tile-row
        const int nb0 = static_cast<int>(tc.n_blk * BLOCK_N);
        const int ba = static_cast<int>(tc.b * p.a_bmul), bb = static_cast<int>(tc.b * p.b_bmul);
        uint32_t seg, kk;  // segment (0 unless k_segments == 3), k-block within it
        seg_of(wu.kb0, seg, kk);
        // convolution: input pixel of the tile's first row (output pixel (n, oh, ow) at kernel position (0, 0)), once per tile
        int cv_w = 0, cv_h = 0, cv_d = 0, cv_n = 0;
        if constexpr (CONV && CONV_DIMS == 3) {
          const uint32_t mu = static_cast<uint32_t>(m0), n = mu / p.cv_odhw, r0 = mu - n * p.cv_odhw, od = r0 / p.cv_ohw;
          const uint32_t r = r0 - od * p.cv_ohw, oh = r / p.cv_ow;
          cv_n = static_cast<int>(n);
          cv_d = static_cast<int>(od) * p.cv_stride_d - p.cv_pad_d;
          cv_h = static_cast<int>(oh) * p.cv_stride_h - p.cv_pad_h;
          cv_w = static_cast<int>(r - oh * p.cv_ow) * p.cv_stride_w - p.cv_pad_w;
        } else if constexpr (CONV) {
          const uint32_t mu = static_cast<uint32_t>(m0), n = mu / p.cv_ohw, r = mu - n * p.cv_ohw, oh = r / p.cv_ow;
          cv_n = static_cast<int>(n);
          cv_h = static_cast<int>(oh) * p.cv_stride_h - p.cv_pad_h;
          cv_w = static_cast<int>(r - oh * p.cv_ow) * p.cv_stride_w - p.cv_pad_w;
        }
        // 3-D weight gradient: each B chunk's (channel block, kernel position) is fixed for the tile, decoded here once to its
        // first channel and its im2col offsets (kx dw, ky dh, kz dd; each <= 31, packed 5 bits apart) -- decoding it per k-block
        // needs more than the producer's 40 registers
        int wg3_c0[NUM_CHUNKS > 0 ? NUM_CHUNKS : 1];
        uint32_t wg3_off[NUM_CHUNKS > 0 ? NUM_CHUNKS : 1];
        if constexpr (CB == CB_WGRAD && CONV_DIMS == 3) {
#pragma unroll
          for (int c = 0; c < NUM_CHUNKS; ++c) {
            const int ci = static_cast<int>(rank) * NUM_CHUNKS + c;
            // a chunk past N (odd chunk count) loads the last chunk again: its columns are never stored
            const uint32_t col = min(static_cast<uint32_t>(nb0 + ci * CHUNK_N), p.N - CHUNK_N) / CHUNK_N;
            const uint32_t kpos = col / p.cv_cblk, cb = col - kpos * p.cv_cblk;
            const uint32_t kz = kpos / p.cv_khw, kr = kpos - kz * p.cv_khw, ky = kr / p.cv_kw, kx = kr - ky * p.cv_kw;
            wg3_c0[c] = static_cast<int>(cb * 64u);
            wg3_off[c] = kx * p.cv_dil_w | (ky * p.cv_dil_h) << 5 | (kz * p.cv_dil_d) << 10;
          }
        }
        for (uint32_t kb = wu.kb0; kb < wu.kb1; ++kb) {
          mbar_wait(empty_bar(s), ph ^ 1);   // every consumer of the pair has released the stage
          const uint32_t sa = smem_base + s * STAGE_BYTES;
          const uint32_t sb = sa + A_BYTES;
          const uint32_t fb = full_bar(s);
          if constexpr (CONV) {
            mbar_arrive_expect_tx(fb, STAGE_BYTES);
            const uint32_t kpos = kb / p.cv_cblk, cb = kb - kpos * p.cv_cblk;
            const int c0 = static_cast<int>(cb * 64u);
            if constexpr (CONV_DIMS == 3) {
              const uint32_t kz = kpos / p.cv_khw, kr = kpos - kz * p.cv_khw, ky = kr / p.cv_kw, kx = kr - ky * p.cv_kw;
              tma_load_im2col_5d(sa, tma_a_hi, fb, c0, cv_w, cv_h, cv_d, cv_n, static_cast<uint16_t>(kx * p.cv_dil_w),
                                 static_cast<uint16_t>(ky * p.cv_dil_h), static_cast<uint16_t>(kz * p.cv_dil_d));
            } else {
              const uint32_t ky = kpos / p.cv_kw, kx = kpos - ky * p.cv_kw;
              tma_load_im2col_4d(sa, tma_a_hi, fb, c0, cv_w, cv_h, cv_n, static_cast<uint16_t>(kx * p.cv_dil_w),
                                 static_cast<uint16_t>(ky * p.cv_dil_h));
            }
            const int n_row = nb0 + static_cast<int>(rank * N_LOCAL);
            if constexpr (CG == 2) tma_load_3d_mc(sb + rank * N_LOCAL * 128u, tma_b_hi, fb, static_cast<uint16_t>(3), c0, static_cast<int>(kpos), n_row);
            else tma_load_3d(sb, tma_b_hi, fb, c0, static_cast<int>(kpos), n_row);
            if (++s == STAGES) { s = 0; ph ^= 1; }
            continue;
          }
          if constexpr (QBLK) {
            // the scale tiles of this stage: A rows of this CTA, and every column of the B tile (each CTA of a pair loads
            // its own copy, no multicast)
            mbar_arrive_expect_tx(fb, STAGE_BYTES + (128u + BLOCK_N) * 4u * p.q_nsub);
            const uint32_t sc = sc_base + s * SC_STAGE_BYTES;
            const int j0 = static_cast<int>(kk * p.q_nsub);
            tma_load_3d(sc, tma_a_lo, fb, m0, j0, ba);
            tma_load_3d(sc + SC_A_BYTES, tma_b_lo, fb, nb0, j0, bb);
          } else {
            mbar_arrive_expect_tx(fb, STAGE_BYTES);
          }
          // B rows [rank * N_LOCAL, (rank + 1) * N_LOCAL) of the tile land at the same offset in both CTAs of a pair
          auto load_b = [&](uint32_t dst, const CUtensorMap* m, int c0, int c1, int c2) {
            if constexpr (CG == 2) tma_load_3d_mc(dst, m, fb, static_cast<uint16_t>(3), c0, c1, c2);
            else tma_load_3d(dst, m, fb, c0, c1, c2);
          };
          bool h16 = false;
          if constexpr (KIND == KIND_TF32) h16 = hyb && seg != 0;
          if (h16) {
            // bf16 stage of the hybrid schedule (K-major operands): the same bytes per stage, 64 elements of K
            const int k0 = static_cast<int>(kk * 64u);
            const int ea = ba + static_cast<int>(seg == 2 ? p.hyb_nba : 0u), eb = bb + static_cast<int>(seg == 1 ? p.hyb_nbb : 0u);
            tma_load_3d(sa, tma_a_lo, fb, k0, m0, ea);
            load_b(sb + rank * N_LOCAL * 128u, tma_b_lo, k0, nb0 + static_cast<int>(rank * N_LOCAL), eb);
          } else {
            int k0 = static_cast<int>(kk * BLOCK_K);
            if constexpr (CB == CB_GRP_K) k0 += static_cast<int>(gu.lo);   // the group's first position
            const CUtensorMap* tma_a = (seg == 2) ? tma_a_lo : tma_a_hi;
            const CUtensorMap* tma_b = (seg == 1) ? tma_b_lo : tma_b_hi;
            if constexpr (A_MN) {
#pragma unroll
              for (int c = 0; c < MT * 128 / CHUNK_N; ++c) tma_load_3d(sa + c * CHUNK_BYTES, tma_a, fb, m0 + c * CHUNK_N, k0, ba);
            } else {
#pragma unroll
              for (int mt = 0; mt < MT; ++mt) tma_load_3d(sa + mt * A_SUB_BYTES, tma_a, fb, k0, m0 + mt * 128, ba);
            }
            if constexpr (CB == CB_WGRAD && CONV_DIMS == 3) {
              // input pixel of output pixel k0 = (n, od, oh, ow) at kernel position (0, 0, 0)
              const uint32_t px = static_cast<uint32_t>(k0), n = px / p.cv_odhw, r0 = px - n * p.cv_odhw, od = r0 / p.cv_ohw;
              const uint32_t r = r0 - od * p.cv_ohw, oh = r / p.cv_ow;
              const int d = static_cast<int>(od) * p.cv_stride_d - p.cv_pad_d;
              const int h = static_cast<int>(oh) * p.cv_stride_h - p.cv_pad_h;
              const int w = static_cast<int>(r - oh * p.cv_ow) * p.cv_stride_w - p.cv_pad_w;
#pragma unroll
              for (int c = 0; c < NUM_CHUNKS; ++c) {
                const int ci = static_cast<int>(rank) * NUM_CHUNKS + c;
                const uint32_t o = wg3_off[c];
                const uint16_t ow_ = static_cast<uint16_t>(o & 31u), oh_ = static_cast<uint16_t>((o >> 5) & 31u), od_ = static_cast<uint16_t>(o >> 10);
                if constexpr (CG == 2)
                  tma_load_im2col_5d_mc(sb + ci * CHUNK_BYTES, tma_b, fb, static_cast<uint16_t>(3), wg3_c0[c], w, h, d,
                                        static_cast<int>(n), ow_, oh_, od_);
                else
                  tma_load_im2col_5d(sb + ci * CHUNK_BYTES, tma_b, fb, wg3_c0[c], w, h, d, static_cast<int>(n), ow_, oh_, od_);
              }
            } else if constexpr (CB == CB_WGRAD) {
              // input pixel of output pixel k0 = (n, oh, ow) at kernel position (0, 0)
              const uint32_t px = static_cast<uint32_t>(k0), n = px / p.cv_ohw, r = px - n * p.cv_ohw, oh = r / p.cv_ow;
              const int h = static_cast<int>(oh) * p.cv_stride_h - p.cv_pad_h;
              const int w = static_cast<int>(r - oh * p.cv_ow) * p.cv_stride_w - p.cv_pad_w;
#pragma unroll
              for (int c = 0; c < NUM_CHUNKS; ++c) {
                const int ci = static_cast<int>(rank) * NUM_CHUNKS + c;
                // a chunk past N (odd chunk count) loads the last chunk again: its columns are never stored
                const uint32_t col = min(static_cast<uint32_t>(nb0 + ci * CHUNK_N), p.N - CHUNK_N) / CHUNK_N;
                const uint32_t kpos = col / p.cv_cblk, cb = col - kpos * p.cv_cblk;
                const uint32_t ky = kpos / p.cv_kw, kx = kpos - ky * p.cv_kw;
                const uint16_t ow_ = static_cast<uint16_t>(kx * p.cv_dil_w), oh_ = static_cast<uint16_t>(ky * p.cv_dil_h);
                if constexpr (CG == 2)
                  tma_load_im2col_4d_mc(sb + ci * CHUNK_BYTES, tma_b, fb, static_cast<uint16_t>(3), static_cast<int>(cb * 64u), w, h,
                                        static_cast<int>(n), ow_, oh_);
                else
                  tma_load_im2col_4d(sb + ci * CHUNK_BYTES, tma_b, fb, static_cast<int>(cb * 64u), w, h, static_cast<int>(n), ow_, oh_);
              }
            } else if constexpr (B_MN) {
#pragma unroll
              for (int c = 0; c < NUM_CHUNKS; ++c) {
                const int ci = static_cast<int>(rank) * NUM_CHUNKS + c;
                load_b(sb + ci * CHUNK_BYTES, tma_b, nb0 + ci * CHUNK_N, k0, bb);
              }
            } else {
              load_b(sb + rank * N_LOCAL * 128u, tma_b, k0, nb0 + static_cast<int>(rank * N_LOCAL), bb);
            }
          }
          if (++kk == (seg == 0 ? seg_kb : seg_kb1)) { kk = 0; ++seg; }
          if (++s == STAGES) { s = 0; ph ^= 1; }
        }
      }
    }
  } else {
    // ===================================================================== wgmma consumers (64 rows of each sub-tile) + epilogue
    setmaxnreg_inc<232>();
    const uint32_t cw = wg - 1;                    // 64-row half of each 128-row sub-tile
    const uint32_t ct = threadIdx.x - 128;         // consumer thread 0..255
    const uint32_t t = threadIdx.x & 127;          // thread in the warpgroup
    const uint32_t lane = t & 31, wq = t >> 5;
    const uint32_t peer_empty0 = (CG == 2) ? mapa_shared(empty_bar(0), rank ^ 1u) : 0u;
    const bool elected = (t == 0);
    auto release = [&](uint32_t st) {
      if (elected) {
        mbar_arrive(empty_bar(st));
        if constexpr (CG == 2) mbar_arrive_cluster(peer_empty0 + 8u * st);
      }
    };
    // 8-bit kinds: the rhs format of a mixed pair is chosen at run time (same smem layout, another instruction)
    const bool mixed = (ESZ == 1) && p.fmt_mixed != 0 && p.fmt_b != ((KIND == KIND_E5M2 || KIND == KIND_S8) ? 1u : 0u);
    constexpr int KIND_OTHER = (KIND == KIND_E4M3) ? KIND_E5M2 : (KIND == KIND_E5M2) ? KIND_E4M3 : (KIND == KIND_U8) ? KIND_S8
                               : (KIND == KIND_S8) ? KIND_U8 : KIND;
    const uint32_t osz = (OUT == OUT_F32) ? 4 : 2;
    float gab = 0.f;   // QM_TENSOR: rn(g_a * g_b), read once per CTA from the device
    if constexpr (QM == QM_TENSOR) gab = __fmul_rn(__ldg(reinterpret_cast<const float*>(p.q_ga)), __ldg(reinterpret_cast<const float*>(p.q_gb)));
    Acc acc[MT][NACC];
    uint32_t s = 0, ph = 0;
    UnitIter it = unit_iter(cluster_id, n_clusters, num_kb);
    WorkUnit wu;
    while (next_unit(it, p, wu)) {
      // transposed convolution: the tile's phase, its k-blocks and its pixel count; tq_keep masks the accumulators of a tile
      // without k-blocks to +0
      uint32_t tq = 0, tq_m = 0, tq_keep = 0;
      if constexpr (CB == CB_TCONV) {
        tq = tconv_phase(wu.tile, *tcp);
        wu.kb0 = 0;
        wu.kb1 = tcp->ph[tq].num_kb;
        tq_m = tcp->ph[tq].M;
        tq_keep = wu.kb1 != 0 ? 0xFFFFFFFFu : 0u;
      }
      // grouped matmul: the tile's group and k-blocks; a tile without k-blocks reads its accumulators as +0 (tq_keep)
      GrpUnit gu;
      if constexpr (GRP) {
        if (wu.tile >= grp_total) break;
        gu = grp_unit<CB, GRP_MASK, BLOCK_K>(wu.tile, p, *gpp, grp_o, grp_pre);
        wu.kb0 = 0;
        wu.kb1 = gu.nkb;
        tq_keep = gu.nkb != 0 ? 0xFFFFFFFFu : 0u;
        if constexpr (CB == CB_GRP_M) gu.tc.b = 0;   // out is 2-D: the group picks rows, not a batch
      }
      TileCoord tc = unit_coord<CB>(wu.tile, p, tcp, tq);
      if constexpr (GRP) tc = gu.tc;
      uint32_t seg = 0, kk = 0;
      if constexpr (KIND == KIND_TF32) seg_of(wu.kb0, seg, kk);
      uint32_t prev = 0;
      if constexpr (PROMOTE || QBLK) {
#pragma unroll
        for (int i = 0; i < NACC; ++i) acc[0][i] = 0.f;
      }
      for (uint32_t kb = wu.kb0; kb < wu.kb1; ++kb) {
        mbar_wait(full_bar(s), ph);
        const uint32_t sa = smem_base + s * STAGE_BYTES;
        const uint32_t sb = sa + A_BYTES;
        if constexpr (CB == CB_GRP_K) {
          const uint32_t keep = (gu.hi - gu.lo) & 63u;
          if (kb + 1u == wu.kb1 && keep != 0) grp_zero_rows(sa, keep, ct);
        }
        // A rows of (sub-tile mt, half cw): K-major 128-byte rows, or the (2 mt + cw)-th 64-element MN-major chunk
        auto a_desc_of = [&](int mt) {
          return A_MN ? make_smem_desc_sw128(sa + (2u * mt + cw) * CHUNK_BYTES, CHUNK_BYTES, 1024)
                      : make_smem_desc_sw128(sa + mt * A_SUB_BYTES + cw * 64u * 128u, 16, 1024);
        };
        const uint64_t a_desc = a_desc_of(0);
        const uint64_t b_desc = B_MN ? make_smem_desc_sw128(sb, CHUNK_BYTES, 1024) : make_smem_desc_sw128(sb, 16, 1024);
        if constexpr (PROMOTE) {
          float part[PH / 2];
#pragma unroll
          for (int h = 0; h < BLOCK_N / PH; ++h) {
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 4; ++k)
              wgmma_ss<PH, KIND_BF16, KIND_BF16, 0, 0>(part, a_desc + 2 * k, b_desc + ((h * PH * 128u) >> 4) + 2 * k, k != 0 ? 1u : 0u);
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_fence_operands(part);
#pragma unroll
            for (int i = 0; i < PH / 2; ++i) acc[0][PH / 2 * h + i] += part[i];
          }
          release(s);
        } else if constexpr (QM == QM_BLOCK) {
          // per scale block j of the stage (K = 128 / nsub elements, 4 / nsub wgmma of K = 32), per 64-column part h:
          // exact s32 partial, then the fold.  Rows r, r + 8 of the fragment and column pairs n, n + 1 read their scales
          // from the stage's tiles ([nsub][128] row scales, [nsub][BLOCK_N] column scales).
          const uint32_t sc = sc_base + s * SC_STAGE_BYTES;
          const uint32_t row = cw * 64u + wq * 16u + (lane >> 2);
          // straight-line code per block size (a run-time trip count around wgmma costs registers and spills)
          auto fold_stage = [&](auto ns) {
            constexpr uint32_t NSUB = decltype(ns)::value, KPER = 4u / NSUB;
#pragma unroll
            for (uint32_t j = 0; j < NSUB; ++j) {
              float ra0, ra1;
              asm volatile("ld.shared.f32 %0, [%1];" : "=f"(ra0) : "r"(sc + (j * 128u + row) * 4u) : "memory");
              asm volatile("ld.shared.f32 %0, [%1];" : "=f"(ra1) : "r"(sc + (j * 128u + row + 8u) * 4u) : "memory");
              const uint32_t scb = sc + SC_A_BYTES + (j * BLOCK_N + 2u * (lane & 3u)) * 4u;
#pragma unroll
              for (int h = 0; h < BLOCK_N / 64; ++h) {
                uint32_t part[32];   // 64-column partials: 64 accumulators + 32 partials stay within the register budget
                wgmma_fence();
#pragma unroll
                for (uint32_t k = 0; k < KPER; ++k) {
                  const uint32_t kk2 = 2u * (j * KPER + k);
                  wgmma_ss<64, KIND_S8, KIND_S8, 0, 0>(part, a_desc + kk2, b_desc + ((h * 64u * 128u) >> 4) + kk2, k != 0 ? 1u : 0u);
                }
                wgmma_commit();
                wgmma_wait<0>();
                wgmma_fence_operands(part);
#pragma unroll
                for (int g = 0; g < 8; ++g) {
                  float cb0, cb1;
                  asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(cb0), "=f"(cb1) : "r"(scb + (h * 64u + 8u * g) * 4u) : "memory");
                  const float sc4[4] = {__fmul_rn(ra0, cb0), __fmul_rn(ra0, cb1), __fmul_rn(ra1, cb0), __fmul_rn(ra1, cb1)};
#pragma unroll
                  for (int e = 0; e < 4; ++e) {
                    // |D_j| < 2^22: the magic-number conversion is exact (s32 -> f32 in an integer add and an f32 subtract)
                    const float d = __fsub_rn(__int_as_float(static_cast<int>(part[4 * g + e]) + 0x4B400000), 12582912.f);
                    acc[0][32 * h + 4 * g + e] = __fmaf_rn(d, sc4[e], acc[0][32 * h + 4 * g + e]);
                  }
                }
              }
            }
          };
          if (p.q_nsub == 4) fold_stage(std::integral_constant<uint32_t, 4>{});
          else if (p.q_nsub == 2) fold_stage(std::integral_constant<uint32_t, 2>{});
          else fold_stage(std::integral_constant<uint32_t, 1>{});
          release(s);
        } else if constexpr (QM == QM_FP8) {
          // the QM_BLOCK fold on f32 partials: per scale block j of the stage and 64-column part h (unit u = j * HP + h), 4 / nsub
          // fp8 wgmma k32 into a fresh partial, then acc = fma(P_j, rn(eff_a * eff_b), acc).  Two partial buffers: unit u + 1's
          // wgmma is issued before unit u is folded, so the tensor cores run under the fold.
          const uint32_t sc = sc_base + s * SC_STAGE_BYTES;
          const uint32_t row = cw * 64u + wq * 16u + (lane >> 2);
          auto fold_stage = [&](auto ns, auto kb_) {
            constexpr uint32_t NSUB = decltype(ns)::value, KPER = 4u / NSUB, HP = BLOCK_N / 64, U = NSUB * HP;
            constexpr int KB = decltype(kb_)::value;
            float part[2][32];
            auto issue = [&](uint32_t u) {
              const uint32_t j = u / HP, h = u % HP;
              wgmma_fence();
#pragma unroll
              for (uint32_t k = 0; k < KPER; ++k) {
                const uint32_t kk2 = 2u * (j * KPER + k);
                wgmma_ss<64, KIND, KB, 0, 0>(part[u & 1u], a_desc + kk2, b_desc + ((h * 64u * 128u) >> 4) + kk2, k != 0 ? 1u : 0u);
              }
              wgmma_commit();
            };
            issue(0);
#pragma unroll
            for (uint32_t u = 0; u < U; ++u) {
              const uint32_t j = u / HP, h = u % HP;
              if (u + 1 < U) {
                issue(u + 1);
                wgmma_wait<1>();
              } else {
                wgmma_wait<0>();
              }
              wgmma_fence_operands(part[u & 1u]);
              float ra0, ra1;
              asm volatile("ld.shared.f32 %0, [%1];" : "=f"(ra0) : "r"(sc + (j * 128u + row) * 4u) : "memory");
              asm volatile("ld.shared.f32 %0, [%1];" : "=f"(ra1) : "r"(sc + (j * 128u + row + 8u) * 4u) : "memory");
              const uint32_t scb = sc + SC_A_BYTES + (j * BLOCK_N + 2u * (lane & 3u)) * 4u;
#pragma unroll
              for (int g = 0; g < 8; ++g) {
                float cb0, cb1;
                asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(cb0), "=f"(cb1) : "r"(scb + (h * 64u + 8u * g) * 4u) : "memory");
                const float sc4[4] = {__fmul_rn(ra0, cb0), __fmul_rn(ra0, cb1), __fmul_rn(ra1, cb0), __fmul_rn(ra1, cb1)};
#pragma unroll
                for (int e = 0; e < 4; ++e)
                  acc[0][32 * h + 4 * g + e] = __fmaf_rn(part[u & 1u][4 * g + e], sc4[e], acc[0][32 * h + 4 * g + e]);
              }
            }
          };
          // straight-line code per (block size, rhs format)
          auto by_nsub = [&](auto kb_) {
            if (p.q_nsub == 4) fold_stage(std::integral_constant<uint32_t, 4>{}, kb_);
            else if (p.q_nsub == 2) fold_stage(std::integral_constant<uint32_t, 2>{}, kb_);
            else fold_stage(std::integral_constant<uint32_t, 1>{}, kb_);
          };
          if (mixed) by_nsub(std::integral_constant<int, KIND_OTHER>{});
          else by_nsub(std::integral_constant<int, KIND>{});
          release(s);
        } else {
  #pragma unroll
          for (int mt = 0; mt < MT; ++mt) wgmma_fence_operands(acc[mt]);
          wgmma_fence();
          bool h16 = false;
          if constexpr (KIND == KIND_TF32) {
            h16 = hyb && seg != 0;
            if (++kk == (seg == 0 ? seg_kb : seg_kb1)) { kk = 0; ++seg; }
          }
          if (h16) {
            // bf16 stage of the hybrid schedule: 16 elements of K (32 bytes) per instruction, K-major operands
            if constexpr (KIND == KIND_TF32) {
  #pragma unroll
              for (int k = 0; k < 4; ++k)
                wgmma_ss<BLOCK_N, KIND_BF16, KIND_BF16, 0, 0>(acc[0], a_desc + 2 * k, b_desc + 2 * k, (kb != wu.kb0 || k != 0) ? 1u : 0u);
            }
          } else if (mixed) {
            if constexpr (ESZ == 1) {
  #pragma unroll
              for (int k = 0; k < BLOCK_K / MMA_K; ++k)
                wgmma_ss<BLOCK_N, KIND, KIND_OTHER, 0, 0>(acc[0], a_desc + 2 * k, b_desc + 2 * k, (kb != wu.kb0 || k != 0) ? 1u : 0u);
            }
          } else {
  #pragma unroll
            for (int k = 0; k < BLOCK_K / MMA_K; ++k) {
              const uint64_t b_k = b_desc + static_cast<uint64_t>(B_MN ? ((k * MMA_K * 128) >> 4) : 2 * k);
  #pragma unroll
              for (int mt = 0; mt < MT; ++mt) {
                const uint64_t a_k = a_desc_of(mt) + static_cast<uint64_t>(A_MN ? ((k * MMA_K * 128) >> 4) : 2 * k);
                wgmma_ss<BLOCK_N, KIND, KIND, A_MN ? 1 : 0, B_MN ? 1 : 0>(acc[mt], a_k, b_k, (kb != wu.kb0 || k != 0) ? 1u : 0u);
              }
            }
          }
          wgmma_commit();
          if (kb != wu.kb0) {
            wgmma_wait<1>();   // the previous k-block's MMAs have retired: its stage may be refilled
            release(prev);
          }
  #pragma unroll
          for (int mt = 0; mt < MT; ++mt) wgmma_fence_operands(acc[mt]);   // after the wait: fencing the accumulators of the group still in flight would retire it first
          prev = s;
        }
        if (++s == STAGES) { s = 0; ph ^= 1; }
      }
      if constexpr (!PROMOTE && !QBLK) {
        wgmma_wait<0>();
#pragma unroll
        for (int mt = 0; mt < MT; ++mt) wgmma_fence_operands(acc[mt]);
        if constexpr (GRP) {
          if (wu.kb1 != wu.kb0) release(prev);
        } else if (CB != CB_TCONV || wu.kb1 != wu.kb0) {
          release(prev);   // a tile without k-blocks holds no stage
        }
      }

      // fragment of m64nNk*: thread (warp wq, lane) holds rows 16 wq + lane / 4 (+8) and column pairs 8 j + 2 (lane % 4)
      uint32_t m_cta = (tc.m_blk * CG + rank) * (128u * MT);
      if constexpr (CB == CB_GRP_M) m_cta += gu.row0;
      const uint32_t c0 = tc.n_blk * BLOCK_N + 2u * (lane & 3u);
      // fused epilogue of fragment group j: v = {(r, n), (r, n + 1), (r + 8, n), (r + 8, n + 1)}
      auto epilogue = [&](uint32_t n, uint32_t (&v)[4]) {
        if (!INT_ACC && QM == QM_NONE && p.epi_on) {
          const float* bias = reinterpret_cast<const float*>(p.bias);
          if constexpr (CB == CB_GRP_M) {
            if (bias != nullptr) bias += gu.g * gpp->bias_stride;   // the group's row of the [G, N] bias
          }
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const uint32_t col = n + (e & 1);
            float x = __uint_as_float(v[e]) * p.alpha;
            if (bias != nullptr && col < p.N) x += __ldg(bias + col);
            if (p.epi_act == 1) x = fmaxf(x, 0.f);
            else if (p.epi_act == 2) x = 0.5f * x * (1.f + erff(x * 0.70710678118654752f));
            v[e] = __float_as_uint(x);
          }
        }
      };
      // data gradient: the dx addresses of this thread's two fragment rows, once per tile
      uint64_t dg_row[2] = {0, 0};
      if constexpr (CB == CB_DGRAD && CONV_DIMS == 3) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const uint32_t r = m_cta + cw * 64u + wq * 16u + (lane >> 2) + 8u * h;
          const uint32_t n = r / p.cv_odhw, r0 = r - n * p.cv_odhw, a = r0 / p.cv_ohw, rr = r0 - a * p.cv_ohw, i = rr / p.cv_ow, j = rr - i * p.cv_ow;
          dg_row[h] = p.out + (n * p.dx_sn + a * p.dx_sd + i * p.dx_si + j * p.dx_sj) * osz;
        }
      } else if constexpr (CB == CB_DGRAD) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const uint32_t r = m_cta + cw * 64u + wq * 16u + (lane >> 2) + 8u * h;
          const uint32_t n = r / p.cv_ohw, rr = r - n * p.cv_ohw, i = rr / p.cv_ow, j = rr - i * p.cv_ow;
          dg_row[h] = p.out + (n * p.dx_sn + i * p.dx_si + j * p.dx_sj) * osz;
        }
      } else if constexpr (CB == CB_TCONV) {
        const TconvPhase& P = tcp->ph[tq];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const uint32_t r = m_cta + cw * 64u + wq * 16u + (lane >> 2) + 8u * h;
          if constexpr (CONV_DIMS == 3) {
            const uint32_t n = r / P.e_dhw, r0 = r - n * P.e_dhw, a = r0 / P.e_hw, rr = r0 - a * P.e_hw, i = rr / P.e_w, j = rr - i * P.e_w;
            dg_row[h] = P.out + (n * p.dx_sn + a * p.dx_sd + i * p.dx_si + j * p.dx_sj) * osz;
          } else {
            const uint32_t n = r / P.e_hw, rr = r - n * P.e_hw, i = rr / P.e_w, j = rr - i * P.e_w;
            dg_row[h] = P.out + (n * p.dx_sn + i * p.dx_si + j * p.dx_sj) * osz;
          }
        }
      }
      // direct stores of fragment group j of sub-tile mt
      auto store_group = [&](int mt, int j, uint32_t (&v)[4]) {
        const uint32_t n = c0 + 8u * j;
        if (n >= p.N) return;
        epilogue(n, v);
        const uint32_t r0 = m_cta + mt * 128u + cw * 64u + wq * 16u + (lane >> 2);
        if constexpr (CB == CB_DGRAD) {
          if (r0 < p.M) store_pair<OUT>(dg_row[0], n, p.N, p.vec_store != 0, v[0], v[1]);
          if (r0 + 8 < p.M) store_pair<OUT>(dg_row[1], n, p.N, p.vec_store != 0, v[2], v[3]);
        } else if constexpr (CB == CB_TCONV) {
          if (r0 < tq_m) store_pair<OUT>(dg_row[0], n, p.N, p.vec_store != 0, v[0], v[1]);
          if (r0 + 8 < tq_m) store_pair<OUT>(dg_row[1], n, p.N, p.vec_store != 0, v[2], v[3]);
        } else if constexpr (CB == CB_WGRAD) {
          // virtual column n = (kpos, ch): dw row r0, element kpos * dw_sp + ch; channels ch >= C are dropped (a pair never
          // straddles two kernel positions)
          const uint32_t kpos = n / (p.cv_cblk * 64u), ch = n - kpos * p.cv_cblk * 64u;
          const uint64_t row0 = p.out + (static_cast<uint64_t>(r0) * p.out_row_stride + kpos * p.dw_sp) * osz;
          if (r0 < p.M) store_pair<OUT>(row0, ch, p.dw_c, p.vec_store != 0, v[0], v[1]);
          if (r0 + 8 < p.M) store_pair<OUT>(row0 + static_cast<uint64_t>(8) * p.out_row_stride * osz, ch, p.dw_c, p.vec_store != 0, v[2], v[3]);
        } else if constexpr (CB == CB_GRP_M) {
          // rows of the group only: the rows around it belong to other groups (or to none)
          const uint64_t row0 = p.out + static_cast<uint64_t>(r0) * p.out_row_stride * osz;
          if (r0 >= gu.lo && r0 < gu.hi) store_pair<OUT>(row0, n, p.N, p.vec_store != 0, v[0], v[1]);
          if (r0 + 8 >= gu.lo && r0 + 8 < gu.hi) store_pair<OUT>(row0 + static_cast<uint64_t>(8) * p.out_row_stride * osz, n, p.N, p.vec_store != 0, v[2], v[3]);
        } else {
          const uint64_t row0 = p.out + (static_cast<uint64_t>(tc.b) * p.out_batch_stride + static_cast<uint64_t>(r0) * p.out_row_stride) * osz;
          if (r0 < p.M) store_pair<OUT>(row0, n, p.N, p.vec_store != 0, v[0], v[1]);
          if (r0 + 8 < p.M) store_pair<OUT>(row0 + static_cast<uint64_t>(8) * p.out_row_stride * osz, n, p.N, p.vec_store != 0, v[2], v[3]);
        }
      };
      auto frag = [&](int mt, int j, uint32_t (&v)[4]) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          if constexpr (QM == QM_TENSOR) v[e] = __float_as_uint(__fmul_rn(__int2float_rn(static_cast<int>(acc[mt][4 * j + e])), gab));
          // transposed convolution: a tile without k-blocks (a phase no tap reaches) sums to +0 -- read as such through a
          // mask, as no wgmma has cleared the accumulators (writing them on this data-dependent path would serialise every
          // wgmma; a select here is hoisted out of the store loop, which then no longer unrolls)
          else if constexpr (CB == CB_TCONV || GRP) v[e] = acc_bits(acc[mt][4 * j + e]) & tq_keep;
          else v[e] = acc_bits(acc[mt][4 * j + e]);
        }
      };
      // the host plans no stream-K head for these (nor for CB_TCONV, whose units are all whole tiles: the path stays compiled
      // there all the same, as without it the direct-store loop below is not unrolled and the accumulators move to local memory)
      const bool partial = (MT == 1) && !INT_ACC && QM == QM_NONE && wu.partial;

      // grouped, ragged M: only a CTA tile that lies inside its group leaves through the TMA store (it cannot clip at o_g)
      bool grp_full = true;
      if constexpr (CB == CB_GRP_M) grp_full = m_cta >= gu.lo && m_cta + 128u <= gu.hi;
      if (CB != CB_DGRAD && CB != CB_TCONV && !partial && (CB == CB_GRP_M ? (p.tma_store && grp_full) : p.tma_store != 0)) {
        // fragments -> (epilogue, convert) -> 128B-swizzled [64 rows x 128 B] staging tile -> one TMA store per 128-byte column
        // group; the TMA unit clips ragged edges.  A direct store writes 16 bytes per row per instruction, 8 rows apart.
        const uint32_t stage_smem = epi_base + cw * 8192u;
        const uint32_t rl = wq * 16u + (lane >> 2);   // row of the first fragment value inside the staging tile
#pragma unroll
        for (int mt = 0; mt < MT; ++mt) {
          const int m_row0 = static_cast<int>(m_cta + mt * 128u + cw * 64u);
#pragma unroll   // fully: a run-time chunk index would index the accumulators dynamically and move them to local memory
          for (int c = 0; c < BLOCK_N / CW; ++c) {
            const uint32_t n0 = tc.n_blk * BLOCK_N + c * CW;
            if (t == 0) tma_store_wait_read<0>();   // the previous store has finished reading the staging tile
            asm volatile("bar.sync %0, 128;" ::"r"(2u + cw) : "memory");
#pragma unroll
            for (int jj = 0; jj < CW / 8; ++jj) {
              const int j = c * (CW / 8) + jj;
              uint32_t v[4];
              frag(mt, j, v);
              epilogue(c0 + 8u * j, v);
              const uint32_t cb = (8u * jj + 2u * (lane & 3u)) * osz;   // byte of the pair inside the 128-byte row
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const uint32_t r = rl + 8u * h;
                const uint32_t addr = stage_smem + r * 128u + ((((cb >> 4) ^ (r & 7u)) << 4) | (cb & 15u));
                if constexpr (OUT == OUT_F32) {
                  asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(addr), "r"(v[2 * h]), "r"(v[2 * h + 1]) : "memory");
                } else {
                  uint32_t packed;
                  if constexpr (OUT == OUT_BF16) asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(packed) : "r"(v[2 * h + 1]), "r"(v[2 * h]));
                  else asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(packed) : "r"(v[2 * h + 1]), "r"(v[2 * h]));
                  asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(packed) : "memory");
                }
              }
            }
            fence_proxy_async_smem();   // generic-proxy writes -> visible to the TMA unit
            asm volatile("bar.sync %0, 128;" ::"r"(2u + cw) : "memory");
            if (t == 0 && m_row0 < static_cast<int>(p.M) && n0 < p.N) {
              if constexpr (CB == CB_WGRAD) {
                // tma_out describes dw as (C, Cout, KH * KW): the store clips channels past C
                const uint32_t kpos = n0 / (p.cv_cblk * 64u);
                tma_store_3d(tma_out, stage_smem, static_cast<int>(n0 - kpos * p.cv_cblk * 64u), m_row0, static_cast<int>(kpos));
              } else {
                tma_store_3d(tma_out, stage_smem, static_cast<int>(n0), m_row0, static_cast<int>(tc.b));
              }
              tma_store_commit();
            }
          }
          // 224-wide tiles with 16-bit outputs: the last 32 columns are half a staging row; a 64-wide box would spill into the
          // neighbouring tile, so they leave through direct stores
#pragma unroll
          for (int j = BLOCK_N / CW * CW / 8; j < NACC / 4; ++j) {
            uint32_t v[4];
            frag(mt, j, v);
            store_group(mt, j, v);
          }
        }
      } else if (!partial) {
#pragma unroll
        for (int mt = 0; mt < MT; ++mt) {
#pragma unroll
          for (int j = 0; j < NACC / 4; ++j) {
            uint32_t v[4];
            frag(mt, j, v);
            store_group(mt, j, v);
          }
        }
      } else {
        // part of a stream-K tile's K range: raw f32 accumulators -> this unit's slab, [j][consumer thread] x 16 B (one warp
        // store covers 512 contiguous bytes); the reduction reads them back in the same fragment order
        const uint64_t cta_slab_bytes = static_cast<uint64_t>(128) * BLOCK_N * 4;
        uint4* dst = reinterpret_cast<uint4*>(p.split_ws + (static_cast<uint64_t>(wu.slab) * CG + rank) * cta_slab_bytes) + ct;
#pragma unroll
        for (int j = 0; j < NACC / 4; ++j)
          __stcg(dst + j * 256, make_uint4(acc_bits(acc[0][4 * j]), acc_bits(acc[0][4 * j + 1]), acc_bits(acc[0][4 * j + 2]), acc_bits(acc[0][4 * j + 3])));
        // publish the slab, take a ticket for (tile, CTA rank); whoever completes the tile's set of parts reduces them in k order
        const uint32_t tau = wu.tile - p.full_tiles;
        const uint32_t first = sk_owner(static_cast<uint64_t>(tau) * num_kb, p, num_kb);               // range holding the tile's k-block 0
        const uint32_t parts = sk_owner(static_cast<uint64_t>(tau + 1) * num_kb - 1, p, num_kb) - first + 1;
        __threadfence();
        asm volatile("bar.sync 1, 256;" ::: "memory");
        if (ct == 0) {
          unsigned int* ticket = reinterpret_cast<unsigned int*>(p.split_tickets) + tau * CG + rank;
          const unsigned int old = atomicAdd(ticket, 1u);
          const uint32_t last = (old == parts - 1) ? 1u : 0u;
          if (last) *ticket = 0;  // every part has arrived: leave the ticket ready for the next launch
          asm volatile("st.shared.u32 [%0], %1;" ::"r"(split_flag), "r"(last) : "memory");
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");
        uint32_t last;
        asm volatile("ld.shared.u32 %0, [%1];" : "=r"(last) : "r"(split_flag) : "memory");
        if (last) {
          __threadfence();
          // slab of part j of this tile: range first + j; the tile is that range's (tau - first tile of the range)-th unit
          auto part_slab = [&](uint32_t j) {
            const uint32_t r = first + j;
            const uint32_t u = tau - static_cast<uint32_t>(sk_range_lo(r, p, num_kb) / num_kb);
            return reinterpret_cast<const float4*>(p.split_ws + ((static_cast<uint64_t>(r) * p.sk_umax + u) * CG + rank) * cta_slab_bytes) + ct;
          };
          // parts are ADDED in k order (bit-reproducible whoever arrived last), one fragment group at a time: the accumulators
          // are not written here (writing them on this data-dependent path makes ptxas serialise every wgmma of the kernel)
#pragma unroll 1
          for (int j = 0; j < NACC / 4; ++j) {
            float4 sum = make_float4(0.f, 0.f, 0.f, 0.f);
            for (uint32_t sl = 0; sl < parts; ++sl) {
              const float4 x = __ldcg(part_slab(sl) + j * 256);
              sum.x += x.x; sum.y += x.y; sum.z += x.z; sum.w += x.w;
            }
            uint32_t v[4] = {__float_as_uint(sum.x), __float_as_uint(sum.y), __float_as_uint(sum.z), __float_as_uint(sum.w)};
            store_group(0, j, v);
          }
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");  // the flag word is reused by the next partial unit
      }
    }
    if (t == 0) tma_store_wait<0>();   // outstanding TMA stores read this CTA's shared memory: finish before teardown
  }

  // a CTA of a pair must not exit while its peer may still multicast into its shared memory or arrive on its barriers
  if constexpr (CG == 2) cluster_sync_all(); else __syncthreads();
}

// Dynamic shared memory a variant needs (host mirrors this in capi.cpp: gemm_smem_bytes()).
//   1024 (alignment slack) + STAGES * (MT * 16384 + BLOCK_N * 128) + 1024 (barriers) + 16384 (TMA-store staging)

#define GEMM_KERNEL_PM(NAME, CG, BN, AMN, BMN, KIND, OUT, STAGES, PROMOTE, MT)                                     \
  extern "C" __global__ void __launch_bounds__(kNumThreads, 1)                                                     \
      NAME(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b,                  \
           const __grid_constant__ CUtensorMap tma_a_lo, const __grid_constant__ CUtensorMap tma_b_lo,            \
           const __grid_constant__ CUtensorMap tma_out, const __grid_constant__ GemmParams p) {                    \
    gemm_body<CG, BN, AMN, BMN, KIND, OUT, STAGES, PROMOTE, MT>(&tma_a, &tma_b, &tma_a_lo, &tma_b_lo, &tma_out, p); \
  }
#define GEMM_KERNEL_P(NAME, CG, BN, AMN, BMN, KIND, OUT, STAGES, PROMOTE) GEMM_KERNEL_PM(NAME, CG, BN, AMN, BMN, KIND, OUT, STAGES, PROMOTE, 1)
#define GEMM_KERNEL(NAME, CG, BN, AMN, BMN, KIND, OUT, STAGES) GEMM_KERNEL_P(NAME, CG, BN, AMN, BMN, KIND, OUT, STAGES, false)

// name: gemm_<in>_<out>_<cg>sm_n<BLOCK_N>_<a><b>
//   a: k = lhs stored [M,K] row-major (K-major), m = lhs stored [K,M] (transposed view, M contiguous)
//   b: n = rhs stored [K,N] row-major (N contiguous), k = rhs stored [N,K] (transposed view, K contiguous)
// wgmma reads MN-major shared-memory operands for 16-bit kinds only: tf32 and 8-bit kinds have the `kk` layout alone (the
// host stages other layouts K-major first).
#define GEMM_LAYOUTS(PFX, CG, BN, KIND, OUT, STAGES)           \
  GEMM_KERNEL(PFX##_kn, CG, BN, false, true, KIND, OUT, STAGES)  \
  GEMM_KERNEL(PFX##_kk, CG, BN, false, false, KIND, OUT, STAGES) \
  GEMM_KERNEL(PFX##_mn, CG, BN, true, true, KIND, OUT, STAGES)   \
  GEMM_KERNEL(PFX##_mk, CG, BN, true, false, KIND, OUT, STAGES)
#define GEMM_DTYPES(TILE, CG, BN, STAGES)                                                  \
  GEMM_LAYOUTS(gemm_bf16_bf16_##TILE, CG, BN, KIND_BF16, OUT_BF16, STAGES)                  \
  GEMM_LAYOUTS(gemm_bf16_f32_##TILE, CG, BN, KIND_BF16, OUT_F32, STAGES)                    \
  GEMM_LAYOUTS(gemm_f16_f16_##TILE, CG, BN, KIND_F16, OUT_F16, STAGES)                      \
  GEMM_LAYOUTS(gemm_f16_f32_##TILE, CG, BN, KIND_F16, OUT_F32, STAGES)                      \
  GEMM_LAYOUTS(gemm_f16_bf16_##TILE, CG, BN, KIND_F16, OUT_BF16, STAGES)                    \
  GEMM_KERNEL(gemm_tf32_f32_##TILE##_kk, CG, BN, false, false, KIND_TF32, OUT_F32, STAGES)
// 8-bit integer inputs: u8 / s8 (s32 accumulate, exact): 128 elements of K per 128-byte row.  fp8 inputs run on the f16
// kernels after an exact widening pass (capi.cpp: run_gemm_fp8_as_f16): wgmma accumulates fp8 products with less than f32
// precision.
#define GEMM_INT8(TILE, CG, BN, STAGES)                                                      \
  GEMM_KERNEL(gemm_u8_i32_##TILE##_kk, CG, BN, false, false, KIND_U8, OUT_F32, STAGES)        \
  GEMM_KERNEL(gemm_s8_i32_##TILE##_kk, CG, BN, false, false, KIND_S8, OUT_F32, STAGES)
// block-scaled kinds: operands expanded to bf16 x * scale (capi.cpp: b200_matmul_scaled), promoted accumulation
#define GEMM_MX(TILE, CG, BN, STAGES)                                                                     \
  GEMM_KERNEL_P(gemm_mx_bf16_##TILE##_kk, CG, BN, false, false, KIND_BF16, OUT_BF16, STAGES, true)         \
  GEMM_KERNEL_P(gemm_mx_f16_##TILE##_kk, CG, BN, false, false, KIND_BF16, OUT_F16, STAGES, true)           \
  GEMM_KERNEL_P(gemm_mx_f32_##TILE##_kk, CG, BN, false, false, KIND_BF16, OUT_F32, STAGES, true)

// integer-quantized operands (s8 codes, capi.cpp: b200_matmul_quantized): gemm_q8_* fold per-block scales (QSTAGES stages
// hold the scale tiles too), gemm_q8t_* apply two per-tensor scales in the epilogue
#define GEMM_KERNEL_Q(NAME, CG, BN, OUT, STAGES, QM)                                                                  \
  extern "C" __global__ void __launch_bounds__(kNumThreads, 1)                                                     \
      NAME(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b,                  \
           const __grid_constant__ CUtensorMap tma_a_sc, const __grid_constant__ CUtensorMap tma_b_sc,            \
           const __grid_constant__ CUtensorMap tma_out, const __grid_constant__ GemmParams p) {                    \
    gemm_body<CG, BN, false, false, KIND_S8, OUT, STAGES, false, 1, QM>(&tma_a, &tma_b, &tma_a_sc, &tma_b_sc, &tma_out, p); \
  }
#define GEMM_Q8T(TILE, CG, BN, STAGES)                                                     \
  GEMM_KERNEL_Q(gemm_q8t_bf16_##TILE##_kk, CG, BN, OUT_BF16, STAGES, QM_TENSOR)            \
  GEMM_KERNEL_Q(gemm_q8t_f16_##TILE##_kk, CG, BN, OUT_F16, STAGES, QM_TENSOR)              \
  GEMM_KERNEL_Q(gemm_q8t_f32_##TILE##_kk, CG, BN, OUT_F32, STAGES, QM_TENSOR)
#define GEMM_Q(TILE, CG, BN, STAGES, QSTAGES)                                              \
  GEMM_KERNEL_Q(gemm_q8_bf16_##TILE##_kk, CG, BN, OUT_BF16, QSTAGES, QM_BLOCK)             \
  GEMM_KERNEL_Q(gemm_q8_f16_##TILE##_kk, CG, BN, OUT_F16, QSTAGES, QM_BLOCK)               \
  GEMM_KERNEL_Q(gemm_q8_f32_##TILE##_kk, CG, BN, OUT_F32, QSTAGES, QM_BLOCK)               \
  GEMM_Q8T(TILE, CG, BN, STAGES)

// fp8-quantized operands (capi.cpp: b200_matmul_quantized_fp8): gemm_qf8_<lhs format>_<out>_<tile>_kk, the QM_BLOCK stages
#define GEMM_KERNEL_QF8(NAME, CG, BN, KIND, OUT)                                                                  \
  extern "C" __global__ void __launch_bounds__(kNumThreads, 1)                                                     \
      NAME(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b,                  \
           const __grid_constant__ CUtensorMap tma_a_sc, const __grid_constant__ CUtensorMap tma_b_sc,            \
           const __grid_constant__ CUtensorMap tma_out, const __grid_constant__ GemmParams p) {                    \
    gemm_body<CG, BN, false, false, KIND, OUT, 5, false, 1, QM_FP8>(&tma_a, &tma_b, &tma_a_sc, &tma_b_sc, &tma_out, p); \
  }
#define GEMM_QF8(TILE, CG, BN)                                                    \
  GEMM_KERNEL_QF8(gemm_qf8_e4m3_bf16_##TILE##_kk, CG, BN, KIND_E4M3, OUT_BF16)     \
  GEMM_KERNEL_QF8(gemm_qf8_e4m3_f16_##TILE##_kk, CG, BN, KIND_E4M3, OUT_F16)       \
  GEMM_KERNEL_QF8(gemm_qf8_e4m3_f32_##TILE##_kk, CG, BN, KIND_E4M3, OUT_F32)       \
  GEMM_KERNEL_QF8(gemm_qf8_e5m2_bf16_##TILE##_kk, CG, BN, KIND_E5M2, OUT_BF16)     \
  GEMM_KERNEL_QF8(gemm_qf8_e5m2_f16_##TILE##_kk, CG, BN, KIND_E5M2, OUT_F16)       \
  GEMM_KERNEL_QF8(gemm_qf8_e5m2_f32_##TILE##_kk, CG, BN, KIND_E5M2, OUT_F32)

// 2-D convolution (implicit GEMM, CONV): tma_a = im2col map of x, tma_b = 3-D weight map; tma_a_lo / tma_b_lo are unused
// name: conv2d_<in>_<out>_<tile>
#define CONV_KERNEL(NAME, CG, BN, KIND, OUT, STAGES)                                                                \
  extern "C" __global__ void __launch_bounds__(kNumThreads, 1)                                                     \
      NAME(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b,                  \
           const __grid_constant__ CUtensorMap tma_a_lo, const __grid_constant__ CUtensorMap tma_b_lo,            \
           const __grid_constant__ CUtensorMap tma_out, const __grid_constant__ GemmParams p) {                    \
    gemm_body<CG, BN, false, false, KIND, OUT, STAGES, false, 1, QM_NONE, true>(&tma_a, &tma_b, &tma_a_lo, &tma_b_lo, &tma_out, p); \
  }
// 3-D convolution (CONV_DIMS = 3): 5-D im2col maps of x (forward, weight gradient) or dy (data gradient); names conv3d_*
#define CONV3D_KERNEL(NAME, CG, BN, AMN, KIND, OUT, STAGES, CONV, CB)                                               \
  extern "C" __global__ void __launch_bounds__(kNumThreads, 1)                                                     \
      NAME(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b,                  \
           const __grid_constant__ CUtensorMap tma_a_lo, const __grid_constant__ CUtensorMap tma_b_lo,            \
           const __grid_constant__ CUtensorMap tma_out, const __grid_constant__ GemmParams p) {                    \
    gemm_body<CG, BN, AMN, AMN, KIND, OUT, STAGES, false, 1, QM_NONE, CONV, CB, 3>(&tma_a, &tma_b, &tma_a_lo, &tma_b_lo, &tma_out, p); \
  }
#define CONV3D_ONE(TILE, CG, BN, STAGES, IN, OUTT, KIND, OUT)                                                   \
  CONV3D_KERNEL(conv3d_##IN##_##OUTT##_##TILE, CG, BN, false, KIND, OUT, STAGES, true, CB_NONE)                 \
  CONV3D_KERNEL(conv3d_dgrad_##IN##_##OUTT##_##TILE, CG, BN, false, KIND, OUT, STAGES, true, CB_DGRAD)          \
  CONV3D_KERNEL(conv3d_wgrad_##IN##_##OUTT##_##TILE, CG, BN, true, KIND, OUT, STAGES, false, CB_WGRAD)
#define CONV3D_DTYPES(TILE, CG, BN, STAGES)                                 \
  CONV3D_ONE(TILE, CG, BN, STAGES, bf16, bf16, KIND_BF16, OUT_BF16)          \
  CONV3D_ONE(TILE, CG, BN, STAGES, bf16, f32, KIND_BF16, OUT_F32)            \
  CONV3D_ONE(TILE, CG, BN, STAGES, f16, f16, KIND_F16, OUT_F16)              \
  CONV3D_ONE(TILE, CG, BN, STAGES, f16, f32, KIND_F16, OUT_F32)

#define CONV_DTYPES(TILE, CG, BN, STAGES)                                  \
  CONV_KERNEL(conv2d_bf16_bf16_##TILE, CG, BN, KIND_BF16, OUT_BF16, STAGES) \
  CONV_KERNEL(conv2d_bf16_f32_##TILE, CG, BN, KIND_BF16, OUT_F32, STAGES)   \
  CONV_KERNEL(conv2d_f16_f16_##TILE, CG, BN, KIND_F16, OUT_F16, STAGES)     \
  CONV_KERNEL(conv2d_f16_f32_##TILE, CG, BN, KIND_F16, OUT_F32, STAGES)

// Convolution backward: conv2d_dgrad_* (tma_a = im2col map of dy, tma_b = 3-D map of one phase's flipped weights) and
// conv2d_wgrad_* (tma_a = 3-D map of dy as (Cout, pixels), tma_b = im2col map of x, tma_out = (C, Cout, KH * KW) map of dw)
#define CONV_BWD_KERNEL(NAME, CG, BN, AMN, KIND, OUT, STAGES, CONV, CB)                                            \
  extern "C" __global__ void __launch_bounds__(kNumThreads, 1)                                                     \
      NAME(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b,                  \
           const __grid_constant__ CUtensorMap tma_a_lo, const __grid_constant__ CUtensorMap tma_b_lo,            \
           const __grid_constant__ CUtensorMap tma_out, const __grid_constant__ GemmParams p) {                    \
    gemm_body<CG, BN, AMN, AMN, KIND, OUT, STAGES, false, 1, QM_NONE, CONV, CB>(&tma_a, &tma_b, &tma_a_lo, &tma_b_lo, &tma_out, p); \
  }
#define CONV_BWD_DTYPES(TILE, CG, BN, STAGES)                                                                  \
  CONV_BWD_KERNEL(conv2d_dgrad_bf16_bf16_##TILE, CG, BN, false, KIND_BF16, OUT_BF16, STAGES, true, CB_DGRAD)   \
  CONV_BWD_KERNEL(conv2d_dgrad_bf16_f32_##TILE, CG, BN, false, KIND_BF16, OUT_F32, STAGES, true, CB_DGRAD)     \
  CONV_BWD_KERNEL(conv2d_dgrad_f16_f16_##TILE, CG, BN, false, KIND_F16, OUT_F16, STAGES, true, CB_DGRAD)       \
  CONV_BWD_KERNEL(conv2d_dgrad_f16_f32_##TILE, CG, BN, false, KIND_F16, OUT_F32, STAGES, true, CB_DGRAD)       \
  CONV_BWD_KERNEL(conv2d_wgrad_bf16_bf16_##TILE, CG, BN, true, KIND_BF16, OUT_BF16, STAGES, false, CB_WGRAD)   \
  CONV_BWD_KERNEL(conv2d_wgrad_bf16_f32_##TILE, CG, BN, true, KIND_BF16, OUT_F32, STAGES, false, CB_WGRAD)     \
  CONV_BWD_KERNEL(conv2d_wgrad_f16_f16_##TILE, CG, BN, true, KIND_F16, OUT_F16, STAGES, false, CB_WGRAD)       \
  CONV_BWD_KERNEL(conv2d_wgrad_f16_f32_##TILE, CG, BN, true, KIND_F16, OUT_F32, STAGES, false, CB_WGRAD)

// Transposed convolution, stride > 1: every phase of a layer in one launch.  The im2col and weight maps of each phase are
// in the TconvParams parameter; names conv2d_tconv_<in>_<out>_<tile> (4-D im2col) and conv3d_tconv_* (5-D)
#define TCONV_KERNEL(NAME, CG, BN, KIND, OUT, STAGES, DIMS)                                                        \
  extern "C" __global__ void __launch_bounds__(kNumThreads, 1)                                                     \
      NAME(const __grid_constant__ TconvParams tp, const __grid_constant__ GemmParams p) {                         \
    const CUtensorMap* a0 = reinterpret_cast<const CUtensorMap*>(&tp.a[0]);                                        \
    const CUtensorMap* b0 = reinterpret_cast<const CUtensorMap*>(&tp.b[0]);                                        \
    gemm_body<CG, BN, false, false, KIND, OUT, STAGES, false, 1, QM_NONE, true, CB_TCONV, DIMS>(a0, b0, a0, b0, a0, p, &tp); \
  }
#define TCONV_DTYPES(TILE, CG, BN, STAGES, DIMS, PFX)                                        \
  TCONV_KERNEL(PFX##_tconv_bf16_bf16_##TILE, CG, BN, KIND_BF16, OUT_BF16, STAGES, DIMS)      \
  TCONV_KERNEL(PFX##_tconv_bf16_f32_##TILE, CG, BN, KIND_BF16, OUT_F32, STAGES, DIMS)        \
  TCONV_KERNEL(PFX##_tconv_f16_f16_##TILE, CG, BN, KIND_F16, OUT_F16, STAGES, DIMS)          \
  TCONV_KERNEL(PFX##_tconv_f16_f32_##TILE, CG, BN, KIND_F16, OUT_F32, STAGES, DIMS)

// Grouped matmul (GroupedParams; capi.cpp: b200_matmul_grouped): tma_a = lhs, tma_b = rhs (ragged M: 3-D with the group as
// batch), tma_out = out for the TMA-store path.  Names gemm_grouped_m_<in>_<out>_<tile>_<a><b> (ragged M, the four operand
// layouts of gemm_*) and gemm_grouped_k_<in>_<out>_<tile> (ragged K: M-contiguous lhs, N-contiguous rhs)
#define GRP_KERNEL(NAME, CG, BN, AMN, BMN, KIND, OUT, CB)                                                         \
  extern "C" __global__ void __launch_bounds__(kNumThreads, 1)                                                     \
      NAME(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b,                  \
           const __grid_constant__ CUtensorMap tma_out, const __grid_constant__ GroupedParams gp,                 \
           const __grid_constant__ GemmParams p) {                                                                \
    gemm_body<CG, BN, AMN, BMN, KIND, OUT, 6, false, 1, QM_NONE, false, CB>(&tma_a, &tma_b, &tma_a, &tma_b, &tma_out, p, nullptr, &gp); \
  }
#define GRP_ONE(TILE, CG, BN, IN, OUTT, KIND, OUT)                                                     \
  GRP_KERNEL(gemm_grouped_m_##IN##_##OUTT##_##TILE##_kn, CG, BN, false, true, KIND, OUT, CB_GRP_M)   \
  GRP_KERNEL(gemm_grouped_m_##IN##_##OUTT##_##TILE##_kk, CG, BN, false, false, KIND, OUT, CB_GRP_M)  \
  GRP_KERNEL(gemm_grouped_m_##IN##_##OUTT##_##TILE##_mn, CG, BN, true, true, KIND, OUT, CB_GRP_M)    \
  GRP_KERNEL(gemm_grouped_m_##IN##_##OUTT##_##TILE##_mk, CG, BN, true, false, KIND, OUT, CB_GRP_M)   \
  GRP_KERNEL(gemm_grouped_k_##IN##_##OUTT##_##TILE, CG, BN, true, true, KIND, OUT, CB_GRP_K)
#define GRP_DTYPES(TILE, CG, BN)                                 \
  GRP_ONE(TILE, CG, BN, bf16, bf16, KIND_BF16, OUT_BF16)          \
  GRP_ONE(TILE, CG, BN, bf16, f32, KIND_BF16, OUT_F32)            \
  GRP_ONE(TILE, CG, BN, f16, f16, KIND_F16, OUT_F16)              \
  GRP_ONE(TILE, CG, BN, f16, f32, KIND_F16, OUT_F32)

// Grouped matmul of fp8-quantized operands, ragged M (capi.cpp: b200_matmul_grouped_quantized_fp8): the maps of
// gemm_qf8_* (lhs codes [T, K], rhs codes with the group as batch, and their effective-scale tiles), tma_out, GroupedParams.
// Names gemm_grouped_qf8_<lhs format>_<out>_<tile>_kk; the rhs format is chosen at run time
#define GRP_QF8_KERNEL(NAME, CG, BN, KIND, OUT)                                                                   \
  extern "C" __global__ void __launch_bounds__(kNumThreads, 1)                                                     \
      NAME(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b,                  \
           const __grid_constant__ CUtensorMap tma_a_sc, const __grid_constant__ CUtensorMap tma_b_sc,            \
           const __grid_constant__ CUtensorMap tma_out, const __grid_constant__ GroupedParams gp,                 \
           const __grid_constant__ GemmParams p) {                                                                \
    gemm_body<CG, BN, false, false, KIND, OUT, 5, false, 1, QM_FP8, false, CB_GRP_M>(&tma_a, &tma_b, &tma_a_sc, &tma_b_sc, &tma_out, p, \
                                                                                     nullptr, &gp);               \
  }
#define GRP_QF8(TILE, CG, BN)                                                          \
  GRP_QF8_KERNEL(gemm_grouped_qf8_e4m3_bf16_##TILE##_kk, CG, BN, KIND_E4M3, OUT_BF16)   \
  GRP_QF8_KERNEL(gemm_grouped_qf8_e4m3_f16_##TILE##_kk, CG, BN, KIND_E4M3, OUT_F16)     \
  GRP_QF8_KERNEL(gemm_grouped_qf8_e4m3_f32_##TILE##_kk, CG, BN, KIND_E4M3, OUT_F32)     \
  GRP_QF8_KERNEL(gemm_grouped_qf8_e5m2_bf16_##TILE##_kk, CG, BN, KIND_E5M2, OUT_BF16)   \
  GRP_QF8_KERNEL(gemm_grouped_qf8_e5m2_f16_##TILE##_kk, CG, BN, KIND_E5M2, OUT_F16)     \
  GRP_QF8_KERNEL(gemm_grouped_qf8_e5m2_f32_##TILE##_kk, CG, BN, KIND_E5M2, OUT_F32)

// The kernels are built as eleven cubins from this one source (cubecl_b200/build.py compiles them in parallel):
//   GEMM_PART 0 ("gemm")       256 x 256 pair tiles (2-CTA cluster, 128 x 256 per CTA) and the bf16 peak probe
//   GEMM_PART 1 ("gemm_b")     256 x 128 pair tiles, 256 x 224 block-scaled pair tiles
//   GEMM_PART 2 ("gemm_c")     128 x 128 single-CTA tiles, 512 x 128 pair tiles
//   GEMM_PART 3 ("gemm_q")     the quantized-operand kernels of every tile
//   GEMM_PART 4 ("gemm_conv")  the 2-D convolution kernels of the 2sm_n128 and 1sm_n128 tiles
//   GEMM_PART 5 ("gemm_convbwd")  the convolution backward kernels (data and weight gradients) of the same two tiles
//   GEMM_PART 6 ("gemm_conv3d")   the 3-D convolution kernels (forward, data and weight gradients) of the same two tiles
//   GEMM_PART 7 ("gemm_convt")    the phase-batched transposed-convolution kernels, 2-D and 3-D, of the same two tiles
//   GEMM_PART 8 ("gemm_grouped")  the grouped-matmul kernels (ragged M and ragged K) of the same two tiles
//   GEMM_PART 9 ("gemm_qf8")      the fp8-quantized kernels (QM_FP8) of the same two tiles
//   GEMM_PART 10 ("gemm_grouped_qf8")  the fp8-quantized grouped-matmul kernels (QM_FP8, ragged M) of the same two tiles
#ifndef GEMM_PART
#define GEMM_PART 0
#endif

#if GEMM_PART == 0
// 128 x 256 per CTA: 48 KB/stage -> 4 stages = 192 KB
GEMM_DTYPES(2sm_n256, 2, 256, 4)
GEMM_INT8(2sm_n256, 2, 256, 4)
GEMM_MX(2sm_n256, 2, 256, 4)
#endif
#if GEMM_PART == 1
// 128 x 128 per CTA: 32 KB/stage -> 6 stages = 192 KB
GEMM_DTYPES(2sm_n128, 2, 128, 6)
GEMM_INT8(2sm_n128, 2, 128, 6)
GEMM_MX(2sm_n128, 2, 128, 6)
// block-scaled kinds: 224 columns per tile (two promoted partials of 112), 4 x 44 KB stages
GEMM_MX(2sm_n224, 2, 224, 4)
#endif
#if GEMM_PART == 2
// single CTA, 128 x 128 tiles (small problems; also the bring-up path)
GEMM_DTYPES(1sm_n128, 1, 128, 6)
GEMM_INT8(1sm_n128, 1, 128, 6)
GEMM_MX(1sm_n128, 1, 128, 6)
// 512 x 128 pair tiles (MT = 2: 256 rows per CTA, two m64 blocks per consumer warpgroup), 16-bit kinds: 4 x 48 KB stages
#define GEMM_M512(PFX, KIND, OUT)                                                     \
  GEMM_KERNEL_PM(PFX##_2sm_m512_kn, 2, 128, false, true, KIND, OUT, 4, false, 2)       \
  GEMM_KERNEL_PM(PFX##_2sm_m512_kk, 2, 128, false, false, KIND, OUT, 4, false, 2)      \
  GEMM_KERNEL_PM(PFX##_2sm_m512_mn, 2, 128, true, true, KIND, OUT, 4, false, 2)        \
  GEMM_KERNEL_PM(PFX##_2sm_m512_mk, 2, 128, true, false, KIND, OUT, 4, false, 2)
GEMM_M512(gemm_bf16_bf16, KIND_BF16, OUT_BF16)
GEMM_M512(gemm_bf16_f32, KIND_BF16, OUT_F32)
GEMM_M512(gemm_f16_f16, KIND_F16, OUT_F16)
GEMM_M512(gemm_f16_f32, KIND_F16, OUT_F32)
GEMM_M512(gemm_f16_bf16, KIND_F16, OUT_BF16)
#endif
#if GEMM_PART == 3
// per-block stages carry (128 + BLOCK_N) x 16 B of scales: the largest count that fits 227 KB (capi.cpp: gemm_smem_bytes)
// 2sm_n256 has the per-tensor kernels only: its 128 f32 accumulators and a partial exceed the 168 registers a thread of a
// 384-thread CTA gets, and the per-block fold would spill
GEMM_Q8T(2sm_n256, 2, 256, 4)
GEMM_Q(2sm_n128, 2, 128, 6, 5)
GEMM_Q(1sm_n128, 1, 128, 6, 5)
#endif
#if GEMM_PART == 4
// the stage counts of the GEMM tiles of the same shape.  No 256 x 256 tile: with 128 accumulators per thread its consumer
// spills at the 168 registers a thread of a 384-thread CTA gets (as gemm_*_2sm_n256_kk does), and these kernels do not spill
CONV_DTYPES(2sm_n128, 2, 128, 6)
CONV_DTYPES(1sm_n128, 1, 128, 6)
#endif
#if GEMM_PART == 5
CONV_BWD_DTYPES(2sm_n128, 2, 128, 6)
CONV_BWD_DTYPES(1sm_n128, 1, 128, 6)
#endif
#if GEMM_PART == 6
CONV3D_DTYPES(2sm_n128, 2, 128, 6)
CONV3D_DTYPES(1sm_n128, 1, 128, 6)
#endif
#if GEMM_PART == 7
TCONV_DTYPES(2sm_n128, 2, 128, 6, 2, conv2d)
TCONV_DTYPES(1sm_n128, 1, 128, 6, 2, conv2d)
TCONV_DTYPES(2sm_n128, 2, 128, 6, 3, conv3d)
TCONV_DTYPES(1sm_n128, 1, 128, 6, 3, conv3d)
#endif
#if GEMM_PART == 8
GRP_DTYPES(2sm_n128, 2, 128)
GRP_DTYPES(1sm_n128, 1, 128)
#endif
#if GEMM_PART == 9
// the per-block stage count of gemm_q8_* (capi.cpp: gemm_q8_stages)
GEMM_QF8(2sm_n128, 2, 128)
GEMM_QF8(1sm_n128, 1, 128)
#endif
#if GEMM_PART == 10
GRP_QF8(2sm_n128, 2, 128)
GRP_QF8(1sm_n128, 1, 128)
#endif

#if GEMM_PART == 0
// ---------------------------------------------------------------------------------------------------------------------
// wgmma peak probe: the accounting of compute_cmma_throughput (crates/cubecl-std/src/throughput/runners/
// compute_cmma.rs:16,41-42: ops = cubes * planes * 2mnk * n_iter) moved to Hopper's tensor cores -- each of the two
// consumer warpgroups of every CTA issues n_iter x 4 back-to-back wgmma m64n256k(32 bytes) on operands resident in shared
// memory (all ones), so it measures the MMA pipe with no TMA / HBM in the loop.  PK 0 = bf16 (K = 16 per instruction),
// 1 = e4m3 (K = 32).  out[cta] = acc[0] = 64 * n_iter (bf16) or 128 * n_iter (e4m3).
template <int PK>
__device__ __forceinline__ void wgmma_probe_body(float* out, uint32_t n_iter) {
  extern __shared__ uint8_t smem_probe_raw[];
  const uint32_t smem_base = (smem_u32(smem_probe_raw) + 1023u) & ~1023u;
  const uint32_t sa = smem_base, sb = smem_base + 16384;   // A: 128 x 128 B, B: 256 x 128 B
  const uint32_t ones = PK == 0 ? 0x3F803F80u : 0x38383838u;  // bf16 1.0 pairs / e4m3 1.0 bytes
  for (uint32_t i = threadIdx.x; i < (16384 + 32768) / 4; i += blockDim.x)
    asm volatile("st.shared.u32 [%0], %1;" ::"r"(smem_base + 4 * i), "r"(ones) : "memory");
  fence_proxy_async_smem();  // generic-proxy stores -> visible to the tensor core's async-proxy reads
  __syncthreads();
  const uint32_t wg = threadIdx.x >> 7;
  if (wg == 0) return;
  float acc[128];
  const uint64_t a_desc = make_smem_desc_sw128(sa + (wg - 1) * 8192u, 16, 1024), b_desc = make_smem_desc_sw128(sb, 16, 1024);
  for (uint32_t i = 0; i < n_iter; ++i) {
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if constexpr (PK == 0) wgmma_ss<256, KIND_BF16, KIND_BF16, 0, 0>(acc, a_desc + 2 * k, b_desc + 2 * k, (i | k) != 0 ? 1u : 0u);
      else wgmma_ss<256, KIND_E4M3, KIND_E4M3, 0, 0>(acc, a_desc + 2 * k, b_desc + 2 * k, (i | k) != 0 ? 1u : 0u);
    }
    wgmma_commit();
  }
  wgmma_wait<0>();
  wgmma_fence_operands(acc);
  if (threadIdx.x == 128) out[blockIdx.x] = acc[0];
}
extern "C" __global__ void __launch_bounds__(384, 1) wgmma_probe_bf16(float* out, uint32_t n_iter) { wgmma_probe_body<0>(out, n_iter); }
extern "C" __global__ void __launch_bounds__(384, 1) wgmma_probe_e4m3(float* out, uint32_t n_iter) { wgmma_probe_body<1>(out, n_iter); }
#endif  // GEMM_PART == 0
