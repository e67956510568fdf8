// The host-kernel interface: every parameter block the kernels take as a __grid_constant__ argument, and the layout
// constants both sides rely on.  capi.cpp (g++) fills these structs and hands their address to cuLaunchKernel; the .cu
// files (nvcc) read them.  One definition serves both, so a field added here moves on both sides at once.  Plain C++17,
// no CUDA types.  Dtype and quant-value fields carry the public codes of include/cubecl_b200.h (b200_dtype,
// b200_quant_value).
#pragma once
#include <cstdint>

#include "../../include/cubecl_b200.h"

// ================================================================================================ gemm_wgmma.cu
struct GemmParams {
  uint64_t out;               // device pointer of out[batch, M, N]
  uint64_t out_row_stride;    // in elements
  uint64_t out_batch_stride;  // in elements
  uint32_t M, N, K, batch;
  uint32_t tiles_m, tiles_n;  // tile grid per batch; a tile is (128*CG) x BLOCK_N
  uint32_t group_m;           // rasterisation: tiles are walked in column strips of `group_m` tile-rows (L2 reuse)
  uint32_t a_bmul, b_bmul;    // 0 = operand broadcast over batch (tensor map has batch extent 1), 1 = batched
  uint32_t vec_store;         // 1 when every output row start is 16-byte aligned
  uint32_t k_segments;        // 1, or 3 for the 3xTF32 schedule: the K loop runs three times over (A,B), (A,B_lo), (A_lo,B)
  uint32_t epi_act;           // fused epilogue (float accumulators only): 0 = none, 1 = relu, 2 = gelu (erf form)
  uint64_t bias;              // f32[N] added per output column, or 0
  float alpha;                // out = act(alpha * acc + bias[n]); the epilogue is skipped when alpha == 1, bias == 0, act == 0
  uint32_t epi_on;
  // Stream-K head (deterministic, replaces a mostly empty LAST wave): tiles [0, full_tiles) are whole "data-parallel" tiles;
  // the k-blocks of the remaining `sk_tiles` tiles form one linear space of sk_tiles * num_kb k-blocks that is cut into
  // `sk_ranges` equal ranges; cluster c works through ranges c, c + C, ... FIRST (a range may cover the end of one tile and
  // the start of the next: one work unit per tile it touches), then through its whole tiles c, c + C, ....  A unit that
  // covers only part of a tile's K stores its f32 accumulators to its own slab and takes a ticket for the tile; whoever
  // completes the tile adds the slabs in k order (so the result does not depend on who came last) and writes the output --
  // under the MMAs of the following whole tiles, which is why the partial tiles go first.  sk_tiles == 0 disables it.
  uint32_t full_tiles, sk_tiles, sk_ranges, sk_umax;  // sk_umax: slabs reserved per range (max tiles a range can touch)
  uint64_t split_ws;          // slabs: [sk_ranges][sk_umax][CG] x (128 x BLOCK_N f32, in accumulator-fragment order)
  uint64_t split_tickets;     // u32 [sk_tiles][CG] in the reduce workspace (kWsGemmTicketOffset), zero on entry and on exit
  // 8-bit kinds: a MIXED pair (e4m3 x e5m2, u8 x s8 ..., the reference's manual-MMA cartesian products,
  // crates/cubecl-cpp/src/cuda/mma/manual.rs:151-186) when fmt_mixed != 0; fmt_b is then the rhs format (0 = e4m3 / u8,
  // 1 = e5m2 / s8).  The lhs format is the kernel's own.
  uint32_t fmt_b, fmt_mixed;
  // Hybrid f32 schedule (tf32 kernels, k_segments == 3): segment 0 is the tf32 product of the ORIGINAL operands (their top
  // 19 bits); segments 1 and 2 are the cross terms A*B_lo and A_lo*B on bf16 copies at twice the tensor rate -- bf16
  // wgmma into the same f32 accumulators, 64 elements of K per stage instead of 32.  tma_a_lo / tma_b_lo then describe
  // bf16 PAIR buffers [2 * entries][rows][pitch]: entries [0, hyb_nba) hold bf16(x), entries [hyb_nba, 2 hyb_nba) hold
  // bf16(x - trunc_tf32(x)).  Two tensor passes' worth of time instead of 3xTF32's three.
  uint32_t hyb, hyb_nba, hyb_nbb;
  // 1: whole tiles leave through swizzled shared-memory staging and TMA stores (tma_out describes `out` as (N, M, batch),
  // [128 B x 64 rows] boxes); needs a 16-byte aligned base and row / batch pitches.  0: each thread stores its own fragment.
  uint32_t tma_store;
  // Quantized operands (QM != 0, see gemm_body): q_nsub = 128 / Bk scale blocks per 128-element stage of K (per-block
  // kernels); q_ga / q_gb = device pointers of the two f32 tensor scales (per-tensor kernels).
  uint32_t q_nsub, q_pad;
  uint64_t q_ga, q_gb;
  // 2-D convolution as an implicit GEMM (conv2d_* kernels; capi.cpp: b200_conv2d): GEMM row m is output pixel
  // (n, oh, ow) = (m / cv_ohw, (m % cv_ohw) / cv_ow, m % cv_ow), and K runs over (kernel position, 64-channel block) with
  // cv_cblk channel blocks per position.  tma_a_hi is a 4-D im2col map of x (C, W, H, N); tma_b_hi a 3-D map of the weights
  // (C, KH * KW, Cout).  K = KH * KW * cv_cblk * 64.
  uint32_t cv_ohw, cv_ow, cv_cblk, cv_kw;
  int32_t cv_stride_h, cv_stride_w, cv_pad_h, cv_pad_w;
  uint32_t cv_dil_h, cv_dil_w;
  // Convolution backward (capi.cpp: b200_conv2d_backward_data / _weight).
  // Data gradient, stride > 1 (conv2d_dgrad_*): one output phase (h = rh + sh * i, w = rw + sw * j) run as a stride-1
  // convolution of dy.  GEMM row m = (n, i, j) of the phase grid (the cv_ohw / cv_ow geometry above) is stored at
  // out + n * dx_sn + i * dx_si + j * dx_sj elements; `out` already points at pixel (0, rh, rw).
  uint64_t dx_sn, dx_si, dx_sj;
  // Weight gradient (conv2d_wgrad_*): A = dy as [K = pixels, M = Cout] (MN-major), B = the im2col of x, 64 pixels x 64
  // channels of one (kernel position, channel block) per load, K = N * OH * OW pixels.  Virtual column n = (kpos, ch) with
  // kpos = n / (cv_cblk * 64) is dw's element kpos * dw_sp + ch of row co; columns with ch >= dw_c are dropped.
  uint64_t dw_sp;
  uint32_t dw_c, dw_pad;
  // 3-D convolution (conv3d_* kernels; capi.cpp: b200_conv3d*): GEMM row / wgrad pixel m is output pixel (n, od, oh, ow)
  // with n = m / cv_odhw, od = (m % cv_odhw) / cv_ohw and (oh, ow) from the remainder as above; kernel position kpos is
  // (kz, ky, kx) = (kpos / cv_khw, (kpos % cv_khw) / cv_kw, kpos % cv_kw).  The im2col maps are 5-D (C, W, H, D, N).  The
  // data gradient's phase row (n, a, i, j) is stored at out + n * dx_sn + a * dx_sd + i * dx_si + j * dx_sj elements.
  uint32_t cv_odhw, cv_khw;
  int32_t cv_stride_d, cv_pad_d;
  uint32_t cv_dil_d, cv_pad2;
  uint64_t dx_sd;
};

// ================================================================================================ aux_kernels.cu
struct FillParams {
  uint64_t out, n, seed;
  float lo, scale;     // value = lo + u * scale
  uint32_t dtype;      // b200_dtype: F32, F16, BF16, F8E4M3, F8E5M2
  uint32_t mode;       // 0 uniform hash, 1 (i % modulus) as a number
  uint32_t modulus, pad;
};

struct SimtGemmParams {
  uint64_t a, b, out;
  uint64_t a_sb, a_sm, a_sk;  // strides in elements: batch, m, k
  uint64_t b_sb, b_sk, b_sn;
  uint64_t o_sb, o_sm, o_sn;
  uint32_t M, N, K, batch;
  uint32_t in_dtype, out_dtype;  // b200_dtype: F32, F16, BF16; inputs also F8E4M3, F8E5M2, U8, I8
  uint64_t bias;                 // fused epilogue, same meaning as GemmParams
  float alpha;
  uint32_t epi_act, epi_on;
  uint32_t b_dtype_p1;           // rhs dtype + 1 when it differs from in_dtype (mixed fp8 / int8 pairs), 0 = same as lhs
};

struct ScaledSimtParams {
  uint64_t a, b, sa, sb, out;
  uint32_t batch, M, N, K;       // K in elements
  uint32_t a_dtype, b_dtype, out_dtype, scale_block;
  uint32_t a_bmul, b_bmul, scale_ue4m3, pad1;   // scale_ue4m3: scales are |e4m3| (NVFP4: the sign bit is ignored) instead of ue8m0
};

// Scales are the reference's row-major [rows, K / scale_block] layout, or (packed) the 128-row chunk layout
// b200_matmul_scaled takes with scales_packed = 1.
struct DequantParams {
  uint64_t in, scales, out;
  uint32_t rows_per_batch, batch, K, dtype;     // K in elements; dtype F8E4M3, F8E5M2 or F4E2M1X2
  uint32_t scale_block, scale_ue4m3, packed, atoms;
};

struct SplitParams {
  uint64_t in, out;
  uint64_t batch, rows, cols;   // logical [batch, rows, cols], cols innermost (stride 1)
  uint64_t in_bs, in_rs;        // input strides in elements
  uint64_t out_rs;              // output row pitch in elements (>= cols, multiple of 4 so rows stay 16-byte aligned for TMA)
};

struct GatherParams {
  uint64_t in, out, n;
  uint64_t shape[8], strides[8];
  uint32_t rank, esz;
};

struct ConvertF16Params {
  uint64_t in, out;
  uint64_t batch, rows, cols;        // logical [batch, rows, cols], cols innermost in the OUTPUT
  uint64_t in_sb, in_sr, in_sc;      // input strides in elements
  uint64_t out_pitch;                // output row pitch in elements (multiple of 8)
  uint32_t dtype, pad;               // F8E4M3 or F8E5M2
};

struct RepitchParams {
  uint64_t in, out;
  uint64_t batch, rows, cols;        // logical [batch, rows, cols] of the copy, cols innermost in the OUTPUT
  uint64_t in_sb, in_sr, in_sc;      // input strides in elements
  uint64_t out_pitch;                // output row pitch in elements (16-byte multiple)
  uint32_t esz, pad;
};

// Convolution data gradient (conv_dgrad_weights): every output phase's flipped, channel-transposed weights in one pooled
// buffer.  Phase (rh, rw) owns taps ky with (ky * dh - ph - rh) % sh == 0 (likewise kx); its block starts at element
// off[rh * sw + rw] and is [C][Th][Tw][cp] with tap th = (kmax_h[rh] - ky) / qh (ascending dy offset), co innermost and
// channels [Cout, cp) zero.  The phases partition the taps, so the blocks fill KH * KW * C * cp elements.
constexpr int kDgradMaxStride = 8;
struct ConvDgradWeightsParams {
  uint64_t w, out;
  uint64_t s_co, s_ky, s_kx, s_c;      // w [Cout, KH, KW, C] strides in elements
  uint64_t C, Cout, cp;                // cp: output channel pitch (Cout padded to 8)
  uint64_t off[kDgradMaxStride * kDgradMaxStride];
  uint32_t KH, KW, sh, sw, dh, dw, ph, pw, qh, qw;
  uint32_t kmax_h[kDgradMaxStride], kmax_w[kDgradMaxStride], taps_h[kDgradMaxStride], taps_w[kDgradMaxStride];
};

// 3-D convolution data gradient (conv3d_dgrad_weights): as ConvDgradWeightsParams with a depth dimension.  Arrays are
// indexed by dimension (0 = D, 1 = H, 2 = W) and phase.  Phase (rd, rh, rw) owns taps (kz, ky, kx) of its per-dimension
// progressions and its block is [C][Td][Th][Tw][cp].  Blocks are laid out in (rd, rh, rw) order; as the phases of each
// dimension partition its taps, block (rd, rh, rw) starts at element
//   C * cp * (pre[0][rd] * KH * KW + taps[0][rd] * (pre[1][rh] * KW + taps[1][rh] * pre[2][rw])),
// pre[i][r] = taps[i][0] + ... + taps[i][r - 1] (no per-phase offset table: up to 8^3 phases).
struct Conv3dDgradWeightsParams {
  uint64_t w, out;
  uint64_t s_co, s_kz, s_ky, s_kx, s_c;   // w [Cout, KD, KH, KW, C] strides in elements
  uint64_t C, Cout, cp;
  uint32_t k[3], s[3], d[3], p[3], q[3], pad;
  uint32_t kmax[3][kDgradMaxStride], taps[3][kDgradMaxStride];
};

// Transposed convolution with stride > 1 (conv2d_tconv_* / conv3d_tconv_*; capi.cpp: b200_conv_transpose2d / 3d): up to
// kTconvMaxPhases output phases of one layer in one launch.  Each phase is the stride-1 convolution a data-gradient phase
// runs (x in dy's role, the conv_dgrad_weights / conv3d_dgrad_weights block of the phase as its weights).  The tiles of all
// phases form one list, phase after phase in table order (most k-blocks first, so the longest tiles start first); a tile
// of phase q has local index t - tile0 inside the phase's (tiles_m x GemmParams::tiles_n) grid and runs num_kb k-blocks
// (0: no tap reaches the phase, the tile stores act(bias)).  GEMM row m of a phase is pixel (n, a, i, j) of its
// (e_d, e_h, e_w) grid, stored at out + n * dx_sn + a * dx_sd + i * dx_si + j * dx_sj elements (GemmParams strides).
// The maps live in the launch's parameter space beside GemmParams: 16 maps (2 KB) and the table fit its 4 KB, and a
// parameter needs no pooled buffer written ahead of the launch.
constexpr int kTconvMaxPhases = 8;
struct alignas(64) TmapBytes {   // one CUtensorMap (cuda.h: 128 bytes, 64-byte aligned), filled on the host
  uint64_t opaque[16];
};
struct TconvPhase {
  uint64_t out;                  // device address of the phase's first pixel (0, rd, rh, rw)
  uint32_t tile0, tiles_m;       // first tile in the launch's list, tile rows of 128 * CG pixels
  uint32_t M, num_kb;            // pixels N * e_d * e_h * e_w; k-blocks = taps * GemmParams::cv_cblk
  uint32_t e_dhw, e_hw, e_w;     // pixel grid: e_d * e_h * e_w, e_h * e_w, e_w
  uint32_t t_hw, t_w;            // taps: t_h * t_w, t_w (tap index = (tz * t_h + ty) * t_w + tx)
  int32_t lo_d, lo_h, lo_w;      // x offset of the first tap: the im2col map's lower corner
  uint32_t dil_d, dil_h, dil_w;  // x offset between consecutive taps
  uint32_t pad;
};
struct TconvParams {
  TmapBytes a[kTconvMaxPhases];  // im2col map of x per phase (4-D or 5-D)
  TmapBytes b[kTconvMaxPhases];  // the phase's weights (cp, taps, Cout), [n_local x 64 channels] boxes
  TconvPhase ph[kTconvMaxPhases];
  uint32_t phases, pad[3];
};

// Grouped matmul for mixture-of-experts layers (gemm_grouped_m_* / gemm_grouped_k_*, cubin gemm_grouped; capi.cpp:
// b200_matmul_grouped).  offs: i32 [groups] cumulative ends on the device, read only by the kernel; on read
// o_g = min(max(offs[g], o_{g-1}), T) with o_{-1} = 0, so group g owns positions [o_{g-1}, o_g) and a malformed table only makes
// groups empty or short.  Every CTA reads offs once into a table at the end of its shared memory (after the TMA-store staging):
// u32 o[kGroupedMaxGroups] (the clamped ends), then u32 pre[kGroupedMaxGroups + 1] (pre[g] = tile-rows of the groups before g,
// a tile-row being 128 * CG rows of a group; pre[groups] = every group's).
//   mode 0, ragged M (gemm_grouped_m_*): lhs [T, K] x rhs [G, K, N] -> out [T, N].  Tiles are listed group after group, each
//        group's pre[g + 1] - pre[g] tile-rows x GemmParams::tiles_n in GemmParams::group_m strips; units past pre[groups] *
//        tiles_n are skipped.  A rows come from r_g + m_blk * 128 * CG of the 2-D lhs map, B from the 3-D rhs map at batch g;
//        r_g = o_{g-1}, or with an M-contiguous lhs o_{g-1} rounded down to a multiple of 64 (the group's first row is then the
//        innermost coordinate of the A loads; loads there at a coordinate that is not a multiple of 16 bytes faulted).  A CTA tile inside its group leaves through
//        the TMA store, any other through direct stores of rows in [o_{g-1}, o_g); rows >= o_{G-1} are never written.  bias (GemmParams::bias) is f32 [G, N], row g at bias + g * bias_stride.
//   mode 1, ragged K (gemm_grouped_k_*, the weight gradient): lhs [M, T] (M-contiguous) x rhs [T, N] (N-contiguous) ->
//        out [G, M, N], out[g] = lhs[:, o_{g-1}:o_g] @ rhs[o_{g-1}:o_g, :].  Tile t is group t / (tiles_m * tiles_n); it runs
//        ceil(n_g / 64) k-blocks from position o_{g-1}, and zeroes the rows of positions >= o_g in both operands of its last
//        k-block before the MMAs read them.  A group without positions stores +0.
// The host sizes the grid from an upper bound on the tiles (GemmParams::full_tiles): (ceil(T / (128 CG)) + G) * tiles_n in
// mode 0 (ceil((T + 63 G) / (128 CG)) + G tile-rows with an M-contiguous lhs), G * tiles_m * tiles_n in mode 1.  Shared memory: gemm_smem_bytes(variant) + kGroupedTableBytes.
constexpr int kGroupedMaxGroups = 1024;
constexpr uint32_t kGroupedTableBytes = (2 * kGroupedMaxGroups + 4) * 4;
struct GroupedParams {
  uint64_t offs;          // i32 [groups] cumulative ends, 4-byte aligned
  uint64_t bias_stride;   // mode 0: elements between the bias rows of consecutive groups
  uint32_t groups, T;     // G (1 .. kGroupedMaxGroups); T = the ragged extent (lhs rows, or positions)
  uint32_t mode, pad;     // 0 ragged M, 1 ragged K
};

// ================================================================================================ attention.cu
// Fused attention forward (attn_fwd_*; capi.cpp: b200_attention).  One CTA per (b, h, kAttnBlock-query block), grid
// nqb * Hq * B with block x = ((nqb - 1 - qb) * B + b) * Hq + h; K and V stream in blocks of kAttnBlock keys through
// kAttnStages stages.  Shared memory: 1024 (alignment slack) + (1 + 2 * kAttnStages) tiles of kAttnBlock rows x DB 16-bit
// elements (DB = 64 or 128: Q, then K and V per stage) + 1024 (barriers).  The tensor maps are 4-D (D, S, H, B).
constexpr int kAttnBlock = 128;
constexpr int kAttnStages = 2;
struct AttnParams {
  uint64_t lse;          // f32 [B, Hq, Sq] compact, or 0
  uint32_t B, Hq, Sq, Sk;
  uint32_t group;        // Hq / Hkv: query head h reads kv head h / group
  uint32_t nqb;          // query blocks: ceil(Sq / kAttnBlock)
  uint32_t causal;       // 1: key j visible to query i iff j <= i
  uint32_t D;            // head dim (the store clips columns >= D)
  float scale_log2;      // scale * log2(e)
  uint32_t pad;
};

// Fused attention backward (attn_bwd_*; capi.cpp: b200_attention_backward), three launches on one stream:
//   attn_bwd_delta_<in>_<out>  16 threads per workspace row, 16 rows per 256-thread block, grid ceil(B * Hq * Sqp / 16).
//   attn_bwd_dq_*              one CTA per (b, h, kAttnBlock-query block), grid nqb * Hq * B ordered as the forward's; K and V
//                              stream in blocks of kAttnBwdDqKeys keys.  Shared memory: 1024 + 2 tiles of kAttnBlock rows (Q,
//                              dO) + 2 * kAttnBwdStages tiles of kAttnBwdDqKeys rows (K, V) + 1024, tiles of DB 16-bit columns.
//   attn_bwd_dkdv_*            one CTA per (b, hkv, kAttnBlock-key block), grid nkb * Hkv * B: block x = (kb * B + b) * Hkv + hk
//                              when causal (key blocks with the most visible queries first), x = (b * Hkv + hk) * nkb + kb
//                              otherwise (the CTAs of one kv head run together and share Q and dO in L2).  K and V stay
//                              resident; Q, dO and the workspace slices stream per (group head, query block of
//                              kAttnBwdDkdvQueries).  Shared memory: 1024 + 2 tiles of kAttnBlock rows + 2 * kAttnBwdStages
//                              tiles of kAttnBwdDkdvQueries rows + kAttnBwdStages * 2 * kAttnBwdDkdvQueries f32 + 1024.
// The score tiles are 64 wide in both kernels: at DB = 128 the dq consumer holds dQ (64 registers) plus S and dP (32 each),
// the dkdv consumer dK and dV (64 each) plus S^T and dP^T (32 each); 128-wide score tiles would not fit setmaxnreg's 232.
// Workspace ws: f32 [2][B * Hq][Sqp], Sqp = nqb * kAttnBlock.  Plane 0 holds L = lse * log2 e for rows < Sq and +inf past Sq
// (so p = exp2(t - L) is +0 for the zero-filled query rows past Sq), plane 1 delta = rowsum(dout * out) and 0 past Sq.  Rows
// are padded so every query block's slice is a 16-byte aligned bulk copy.
constexpr int kAttnBwdDqKeys = 64;
constexpr int kAttnBwdDkdvQueries = 64;
constexpr int kAttnBwdStages = 2;
struct AttnBwdParams {
  uint64_t ws;                    // workspace (above)
  uint64_t lse;                   // delta kernel: the forward's compact f32 [B, Hq, Sq] log-sum-exp
  uint64_t out, dout;             // delta kernel: views with a unit D stride, 16-byte aligned base and strides
  uint64_t o_sb, o_sh, o_ss;      // out strides in elements (B, H, S)
  uint64_t d_sb, d_sh, d_ss;      // dout strides in elements
  uint32_t B, Hq, Sq, Sk;
  uint32_t group;                 // Hq / Hkv
  uint32_t nqb;                   // ceil(Sq / kAttnBlock)
  uint32_t nkb;                   // ceil(Sk / kAttnBlock)
  uint32_t nqd;                   // ceil(Sq / kAttnBwdDkdvQueries)
  uint32_t Sqp;                   // nqb * kAttnBlock
  uint32_t causal;                // 1: key j visible to query i iff j <= i
  uint32_t D;
  float scale_log2;               // scale * log2(e), the forward's value
  float scale;                    // multiplies dQ and dK in the epilogue
  uint32_t Hkv;
};

// Variable-length (packed) attention: attention.cu and attention_bwd.cu compiled with -DATTN_VARLEN (attn_fwd_varlen_*,
// attn_bwd_varlen_*; capi.cpp: b200_attention_varlen, b200_attention_varlen_backward).  The dense bodies with per-sequence
// addressing: q, out, dout, dq are [Tq, Hq, D] and k, v, dk, dv [Tk, Hkv, D], read through 4-D maps (D, T, H, 1).  Sequence b
// owns rows [cu_q[b], cu_q[b + 1]) and [cu_k[b], cu_k[b + 1]); on read each cu value is clamped to [0, T] and each length to
// [0, max_seqlen], so no access leaves the tensors.  With positions i, j inside the sequence and off = Lk - Lq, key j is
// visible to query i iff j < Lk, (left < 0 or j >= i + off - left) and (right < 0 or j <= i + off + right).
// Grids from host extents only: forward and dq nqb * Hq * B, dkdv nkb * Hkv * B (nqb = ceil(max_q / kAttnBlock), nkb =
// ceil(max_k / kAttnBlock)) in the dense kernels' orders, with the delta kernel's nqb * 8 * Hq * B blocks of 16 rows; a CTA
// whose block starts at or past its sequence's length exits at once.
// Workspace ws (backward): f32 [2][Hq][Tqp], Tqp = (ceil(Tq / kAttnBlock) + B) * kAttnBlock.  Sequence b's rows start at
// floor((cu_q[b] + kAttnBlock * b) / kAttnBlock) * kAttnBlock (a 16-byte aligned start that never reaches the previous
// sequence's padded rows) and span ceil(Lq / kAttnBlock) whole blocks: L = +inf and delta = 0 past Lq and for rows whose lse is
// -inf (no visible key).
struct AttnVarlenParams {
  uint64_t lse;                   // f32 [Hq, Tq] compact (forward: 0 = not written)
  uint64_t cu_q, cu_k;            // i32 [B + 1]
  uint64_t ws;                    // backward workspace (above)
  uint64_t out, dout;             // forward: out (direct stores of partial blocks); delta kernel: out and dout views
  uint64_t o_st, o_sh, d_st, d_sh;  // out / dout strides in elements (T, H)
  uint64_t dq, dk, dv;            // backward: direct stores of partial blocks
  uint64_t dq_st, dq_sh, dk_st, dk_sh, dv_st, dv_sh;
  uint32_t B, Hq, Hkv, Tq, Tk;
  uint32_t group;                 // Hq / Hkv
  uint32_t max_q, max_k;          // max_seqlen_q, max_seqlen_k
  uint32_t nqb, nkb;              // ceil(max_q / kAttnBlock), ceil(max_k / kAttnBlock)
  uint32_t Tqp;                   // workspace rows per head
  uint32_t D;
  int32_t left, right;            // window; -1: unbounded
  float scale_log2;               // scale * log2(e)
  float scale;                    // backward: multiplies dQ and dK in the epilogue
};

// Paged varlen attention: attention.cu compiled with -DATTN_VARLEN -DATTN_PAGED (attn_fwd_paged_*; capi.cpp:
// b200_attention_varlen_paged).  The varlen forward with its queries (cu_q, Tq, max_q, window, out, lse) and K / V read from a
// paged cache [P, page, Hkv, D] through 4-D maps (D, page, Hkv, P): sequence b has Lk = clamp(seqlens[b], 0, min(max_k, cap))
// keys, key j at row j % page of page table[b * t_sb + (j / page) * t_sp] (table 0: page b).  A 128-key block arrives as
// kAttnBlock / rows loads of `rows` keys (rows divides the page, or rows = kAttnBlock with one page per sequence); loads of
// chunks at or past Lk are not issued.  The cu_k, Tk and backward fields of the base are unused.
struct AttnVarlenPagedParams : AttnVarlenParams {
  uint64_t table;                 // i32 block table, or 0
  uint64_t t_sb, t_sp;            // its strides in elements
  uint64_t seqlens;               // i32 [B] cache lengths
  uint32_t page, rows;            // keys per page, keys per TMA load
  uint32_t cap;                   // capacity max_pages * page
  uint32_t pad;
};

// Paged varlen attention against fp8 caches: attention.cu compiled with -DATTN_VARLEN -DATTN_PAGED -DATTN_PAGED_FP8
// (attn_fwd_paged_<in>_<e4m3|e5m2>_d<64|128>_<out>, cubin attention_paged_fp8; capi.cpp: b200_attention_varlen_paged_fp8).
// The paged varlen kernel with e4m3 / e5m2 caches read through UINT8 maps: a chunk of `rows` keys arrives as one box of
// 128 bytes x rows (the whole head, columns >= D zero-filled) in an fp8 stage of kAttnBlock 128-byte rows, and the
// kAttnF8WidenWarps idle warps of the producer warpgroup widen it into the 16-bit ring of the 16-bit kernel (K and V rows of
// keys >= Lk as zeros).  Their full barriers count one arrive per widening warp instead of TMA bytes.
// Shared memory: 1024 (alignment slack) + (1 + 2 * kAttnStages) tiles of kAttnBlock rows x DB 16-bit (Q and the 16-bit
// ring) + kAttnStages x 2 fp8 stages of kAttnBlock x 128 bytes + 1024 (13 barriers: q, full K / V and empty of the ring,
// full K / V and empty of the fp8 stages).  At DB = 128: 1024 + 5 x 32768 + 65536 + 1024 = 231424 bytes, under the 232448-byte
// opt-in limit; at DB = 64: 148480.  Both fp8 stages fit, so there is no one-stage variant.  Registers: the producer
// warpgroup runs at 64 (the widening spills at 40 and 56), the consumers at 216.  k_scale and v_scale are f32 [Hkv]:
// t = s * (scale_log2 * k_scale[hk]) and out = (v_scale[hk] O) / l.
constexpr int kAttnF8WidenWarps = 3;
struct AttnVarlenPagedFp8Params : AttnVarlenPagedParams {
  uint64_t k_scale, v_scale;      // f32 [Hkv] per-head scales
};

// ================================================================================================ attention_kv.cu
// Attention against a KV cache (attn_kv_*; capi.cpp: b200_attention_kvcache).  One CTA per (b, hk, m-tile, split), grid
// B * Hkv * nsplit * mtiles with block x = ((b * Hkv + hk) * nsplit + split) * mtiles + mt (the m-tiles that share a key range
// run side by side).  kAttnKvThreads threads: warps 0-3 are the consumer warpgroup, warp 4 the producer.  An m-tile packs gt
// heads of one kv head's group with st queries, gt * st <= kAttnKvRows, row r = g * st + i; m-tile mt covers group heads
// [(mt / mts) * gt, +gt) and queries [(mt % mts) * st, +st).  Keys stream in blocks of kAttnKvBlock through kAttnKvStages
// stages; a block arrives as kAttnKvBlock / rows TMA loads of `rows` keys (one page, or one block inside a larger page).
// Split s covers key blocks [s * bps, min((s + 1) * bps, nkb)) of the capacity; nkb = ceil(cap / kAttnKvBlock).
// Shared memory: 1024 (alignment slack) + DB / 64 chunks x (kAttnKvRows Q rows + 2 * kAttnKvStages * kAttnKvBlock K / V rows)
// of 128 bytes + kAttnKvBarBytes.
// Workspace (nsplit > 1, ws != 0): f32 O [nsplit][rows][D], then f32 (m, l) [nsplit][rows][2], rows = B * Hq * Sq in
// (b, h, i) order.  O is un-normalised, m is the split's row maximum of t = s * scale_log2 (-inf when the split saw no key) and
// l its row sum of exp2(t - m).  attn_kv_combine_<out> (kAttnKvCombineThreads threads, one per 4 columns of a row) reads it.
// fp8 caches (attn_kv_<in>_<e4m3|e5m2>_d<64|128>_<out>, cubin attention_kv_fp8): a K or V block arrives as 128-byte rows (one
// box of 128 bytes x rows keys per load, columns >= D zero-filled) through kAttnKvF8Stages stages, and the consumer widens
// it into 16-bit swizzled buffers: two K buffers (alternating blocks) and one V buffer.  Shared memory: 1024 + DB / 64 x
// kAttnKvRows Q rows of 128 bytes + kAttnKvF8Stages x 2 x kAttnKvBlock x 128 + 3 x DB / 64 x kAttnKvBlock x 128 +
// kAttnKvF8BarBytes.  k_scale and v_scale are f32 [Hkv]: t = s * (scale_log2 * k_scale[hk]), and v_scale[hk] multiplies the
// un-normalised O (or, with splits, the combined sum) just before the division by l.  The workspace holds the unscaled O.
constexpr int kAttnKvBlock = 64;
constexpr int kAttnKvStages = 4;
constexpr int kAttnKvRows = 64;
constexpr int kAttnKvThreads = 160;
constexpr int kAttnKvBarBytes = 128;
constexpr int kAttnKvMaxSplits = 128;
constexpr int kAttnKvSplitCost = 2;   // the split plan's fixed cost of one CTA, in key blocks (prologue and epilogue)
constexpr int kAttnKvCombineThreads = 256;
constexpr int kAttnKvF8Stages = 8;
constexpr int kAttnKvF8BarBytes = 256;
struct AttnKvParams {
  uint64_t out;               // [B, Hq, Sq, D] view, unit D stride (direct path and combine)
  uint64_t o_sb, o_sh, o_ss;  // out strides in elements
  uint64_t lse;               // f32 [B, Hq, Sq] compact, or 0
  uint64_t ws;                // 0: the attention kernel writes out and lse itself (nsplit == 1); else the workspace above
  uint64_t table;             // i32 block table, element (b, p) at table + b * t_sb + p * t_sp; 0: page b is sequence b
  uint64_t t_sb, t_sp;
  uint64_t seqlens;           // i32 [B] cache lengths, clamped to [0, cap] on read
  uint32_t B, Hq, Hkv, Sq, D;
  uint32_t group;             // G = Hq / Hkv
  uint32_t gt, st, mtg, mts;  // tile: gt heads x st queries; m-tiles mtg * mts
  uint32_t page, rows;        // keys per page, keys per TMA load
  uint32_t cap, nkb;          // capacity max_pages * page, its key blocks
  uint32_t nsplit, bps;       // splits, key blocks per split
  uint32_t causal;            // 1: query i also needs j <= L - Sq + i (bottom-right)
  float scale_log2;           // scale * log2(e)
  uint64_t k_scale, v_scale;  // fp8 caches: f32 [Hkv] scales (the 16-bit kernels do not read them)
};

// b200_kvcache_write (attn_kv_write): one thread per 16-byte unit of a (token, kv head) row, for k and v.  Token n = b * Snew + t
// goes to flat slot slots[n] (page slot / page, row slot % page); a slot < 0 or >= P * page is skipped.  Strides in elements.
struct AttnKvWriteParams {
  uint64_t kn, vn, kc, vc, slots;
  uint64_t kn_sb, kn_st, kn_sh, vn_sb, vn_st, vn_sh;   // new tokens [B, Snew, Hkv, D]
  uint64_t kc_sp, kc_sr, kc_sh, vc_sp, vc_sr, vc_sh;   // caches [P, page, Hkv, D]
  uint64_t units;                                      // B * Snew * Hkv * D / 8
  uint32_t Snew, Hkv, D, page;
  uint64_t slot_end;                                   // P * page
  // b200_kvcache_write_fp8 (attn_kv_write_fp8): one thread per 8 elements; element x of kv head hk is stored as
  // sat_rn(x / scale[hk]) in the cache format.  The 16-bit attn_kv_write does not read these.
  uint64_t k_scale, v_scale;                           // f32 [Hkv]
  uint32_t in_bf16, e5m2;                              // new tokens bf16 (else f16); cache e5m2 (else e4m3)
};

// ================================================================================================ conv_grouped.cu
// Direct NHWC grouped convolution (b200_conv2d_grouped*, group width Cg = C / groups < 64).  Group g owns input channels
// [g Cg, (g+1) Cg) and output channels [g Coutg, (g+1) Coutg).  Every strided operand has a unit channel stride; strides
// are in elements.
//   conv2d_grp_*        x [N, H, W, C], w [Cout, KH, KW, Cg] -> out [N, OH, OW, Cout] (fused epilogue as GemmParams)
//   conv2d_grp_dgrad_*  dy [N, OH, OW, Cout], w -> dx [N, H, W, C]
//   conv2d_grp_wgrad_*  x, dy -> f32 partials [nseg][elems] (nseg > 1) or dw (nseg == 1); conv2d_grp_wgrad_combine_* adds the
//                       partials in segment order into dw.  Element t = (kpos * Cout + co) * Cg + ci, kpos = ky * KW + kx.
// Forward tile: kGrpTileH x kGrpTileW output pixels of one image x kGrpChunk output channels (one per lane); the input halo
// of those channels is staged in shared memory when it fits (staged_ci != 0: that many channels per halo pixel).
constexpr int kGrpChunk = 32;
constexpr int kGrpTileH = 8;
constexpr int kGrpTileW = 8;
constexpr int kGrpSmemMax = 48 * 1024;
struct ConvGroupedParams {
  uint64_t x, w, out, bias;          // x: x, or dy (dgrad); w: w, or dy (wgrad); bias: f32[Cout] or 0 (forward only)
  uint64_t x_sn, x_sh, x_sw;         // x (forward, wgrad) or dy (dgrad): the strided NHWC input
  uint64_t w_sco, w_sky, w_skx;      // w (forward, dgrad)
  uint64_t y_sn, y_sh, y_sw;         // dy (wgrad)
  uint64_t o_sn, o_sh, o_sw;         // out / dx: one pixel pitch; dw: o_sn = Cout stride, o_sw = kernel-position stride
  uint64_t part;                     // wgrad: f32 partials [nseg][elems]
  uint64_t seg_len, elems;           // wgrad: pixels per segment (the last may be shorter), Cout * KH * KW * Cg
  uint32_t N, H, W, C, OH, OW, Cout, KH, KW, Cg, Coutg, nseg;
  int32_t sh, sw, ph, pw, dh, dw;
  uint32_t tiles_w, tiles_h, staged_ci, vec_x;   // forward: tile grid, halo channels per pixel (0 = not staged), 16-byte loads
  float alpha;
  uint32_t epi_act, epi_on, pad;
};

// ================================================================================================ reduce.cu
struct ReduceParams {
  uint64_t in;        // input view, element (o, l, i) at in + (o * s_outer + l * s_len + inner_off(i)) elements
  uint64_t out;       // output [outer (* segments), inner]: f32 values, u32 indices (arg ops), or u32 keys (arg ops, split pass)
  uint64_t out2;      // arg ops, split pass: u32 indices along the reduced axis; 0 otherwise
  uint64_t final_out; // column kernels, split pass with a fused finish (flags bit 2): the real output [outer, inner]; the block
                      // that completes a column tile's last segment (ticket) combines the partials in `out` / `out2` itself
  uint64_t ws;        // the per-stream reduce workspace (layout below)
  uint64_t outer, len, inner;
  uint64_t s_outer, s_len;      // element strides of the outer and the reduced axis
  uint64_t row_len, row_pitch;  // inner_off(i) = (i / row_len) * row_pitch + i % row_len; row_len == inner (or len, for
                                // reductions over all elements, where i is the flat index): no pitch
  uint64_t seg_len;   // the reduced axis is cut into nseg = ceil(len / seg_len) segments reduced independently (first pass of
  uint32_t nseg;      // a two-pass reduction); nseg == 1: whole axis
  uint32_t ctu;       // column kernels: column units (one 128-bit vector, or one element) per block tile; bulk-copy kernels:
                      // ring depth in stages
  float scale;        // applied to the final value (mean = 1/len, sum = 1)
  uint32_t flags;     // bit 0: record stage timings in the workspace debug words; bit 1: column kernels use vector units;
                      // bit 2: fused finish of a split column reduction (see final_out)
};

// Reduce workspace, one per stream, zeroed once at allocation (every ticket is left at zero by the kernel that used it).
constexpr uint32_t kWsMaxBlocks = 4096;                                    // grid cap of the all-elements reduction
constexpr uint32_t kWsIdxOffset = kWsMaxBlocks * 4;                        // after f32 partials[kWsMaxBlocks]: u64 packed pairs
constexpr uint32_t kWsTicketOffset = kWsIdxOffset + kWsMaxBlocks * 8;      // u32 last-block ticket of the grid stage
constexpr uint32_t kWsDebugOffset = kWsTicketOffset + 64;                  // four u64 words: stage timings (ReduceParams::flags bit 0)
constexpr uint32_t kWsGemmTicketOffset = kWsTicketOffset + 256;            // u32 per (stream-K head tile, CTA rank) of a GEMM
static_assert(kWsDebugOffset + 4 * 8 <= kWsGemmTicketOffset, "debug words overlap the GEMM tickets");
constexpr uint32_t kWsGemmTickets = 1024;
constexpr uint32_t kWsColTicketOffset = kWsGemmTicketOffset + kWsGemmTickets * 4;  // u32 per (outer, column tile) of a fused
constexpr uint32_t kWsColTickets = 1024;                                            // split column reduction
constexpr uint32_t kWsBytes = kWsColTicketOffset + kWsColTickets * 4;

// Cross-GPU exchange fused into the grid stage (one kernel = local reduce + all-reduce of the scalar over NVLink peer
// memory).  Every rank owns a mailbox its peers can write; an entry is (epoch << 32) | 32 payload bits, stored with ONE
// 64-bit system-scope store so value and flag arrive together.
struct XgpuParams {
  uint64_t mailbox[8];   // device pointers of every rank's slot set (own included), indexed by rank
  uint32_t rank, nranks, epoch, pad;
  uint64_t index_offset; // arg ops: global index of this rank's element 0 (outer-axis shard offset)
};
// A slot set is value slots u64[2][8] (epoch parity x source rank), then index slots u64[2][8] (arg ops: the second word,
// same epoch tag).  The mailbox holds one set per DEVICE SET, addressed by the set's device bitmask: overlapping sets
// ({0,1} and {0,1,2,3}) never share slots, and every rank derives the same offset.
constexpr uint32_t kMailboxIndexOffset = 2 * 8 * 8;
constexpr uint32_t kMailboxSetBytes = 2 * kMailboxIndexOffset;
constexpr uint32_t kMailboxBytes = 256 * kMailboxSetBytes;

// Bulk-copy all-elements kernels (_tma): kBulkConsumers consumer threads plus one producer warp, kBulkStageBytes per ring stage.
constexpr uint32_t kBulkStageBytes = 16384;
constexpr int kBulkConsumers = 256;
// Column kernels: threads per block (row lanes x column units).
constexpr int kColsThreads = 256;

struct ArgCombineParams {
  uint64_t keys, idx, out;      // u32 keys and u32 indices [outer, nseg, inner] -> u32 indices [outer, inner]
  uint64_t outer, nseg, inner;
};

struct ScanParams {
  uint64_t in;        // input view, element (o, l, i) at in + (o * s_outer + l * s_len + inner_off(i)) elements
  uint64_t out;       // compact [outer, len, inner] output
  uint64_t carry;     // f32 [outer, nseg, inner]: the value every segment starts from (0: the identity)
  uint64_t outer, len, inner;
  uint64_t s_outer, s_len;
  uint64_t row_len, row_pitch;  // as ReduceParams
  uint64_t seg_len;
  uint32_t nseg;
  uint32_t flags;     // bit 0: exclusive; bit 1: column kernel uses vector units
};
// Scans: a row-kernel thread owns kScanElems consecutive elements per tile; a column-kernel block owns at most kScanColUnits
// column units (one per thread).
constexpr int kScanElems = 16;
constexpr int kScanColUnits = 256;

// ================================================================================================ quant.cu
struct QuantParams {
  uint64_t in;            // input rows: element (r, k) at in + (r * pitch + k) elements; 16-byte aligned base and rows
  uint64_t values;        // codes, compact [rows, K * bits / 8] bytes
  uint64_t block_scales;  // compact [rows, K / block] in scale_dt; 0 without a block level
  uint64_t tensor_scale;  // f32 [1]; 0 without a tensor level
  uint64_t amax;          // u32 [1]: bits of the finite |x| max of the tensor (quant_absmax); 0 without a tensor level
  uint64_t rows, K, pitch;
  uint32_t value;         // b200_quant_value
  uint32_t block;         // values per block scale; 0 = per-tensor only
  uint32_t scale_dt;      // block-scale dtype (b200_dtype)
  uint32_t block_log2;    // log2(block) (blocks are powers of two)
};

struct QuantDecodeParams {
  uint64_t values, block_scales, tensor_scale, out;
  uint64_t n;             // elements
  uint32_t value, block, scale_dt;
  uint32_t flags;         // bit 0: values and out are 16-byte aligned (vector loads and stores)
  uint32_t block_log2, pad;
};

// Quantized-matmul operands (b200_matmul_quantized)
struct QuantScalesParams {
  uint64_t block_scales;  // [batch, rows, nblk / rep] in the block-scale dtype; unused by the per-tensor kernel
  uint64_t tensor_scale;  // f32 [1] on the device, or 0
  uint64_t out;           // f32 [batch][nblk][rows_pad], block-major: one TMA box per GEMM stage
  uint64_t batch, rows, rows_pad, nblk;
  uint32_t rep;           // GEMM blocks per stored block (this side's block / the GEMM's Bk)
  uint32_t pad;
};

struct QuantWidenParams {
  uint64_t in, out;       // in: compact code rows of K * bits / 8 bytes; out: s8 rows `pitch` bytes apart (16-byte multiple)
  uint64_t rows, K, pitch;
  uint32_t bits, pad;
};

// ================================================================================================ moe.cu
// Mixture-of-experts routing (capi.cpp: b200_moe_*).  Index arrays are compact i32: ids / row_of [T, k], slot_of [T * k].
struct MoeRouteParams {
  uint64_t logits;        // [T, E] in the logits dtype, element (t, e) at logits + t * stride + e
  uint64_t bias;          // f32 [E] selection bias, or 0
  uint64_t ids, weights;  // i32 / f32 [T, k]
  uint64_t T, stride;
  uint32_t E, k, score, renorm;  // score: b200_moe_score
  uint32_t n_group, topk_group;  // n_group <= 1: no group limit
  float scale;
  uint32_t pad;
};

struct MoePlanParams {
  uint64_t ids, offs, row_of, slot_of;
  uint64_t hist;          // i32 [E][ctas]: each CTA's count per expert, then (moe_plan_scan) the first row of its run
  uint32_t n;             // T * k slots
  uint32_t E, ctas;
  uint32_t warp_slots;    // consecutive slots per warp (a multiple of kMoePlanWarpSlots); a CTA owns 8 warps' worth
};

struct MoePermuteParams {
  uint64_t src, dst, slot_of;
  uint64_t src_pitch, dst_pitch, row_bytes;  // bytes
  uint64_t rows;          // T * k
  uint32_t k, pad;
};

// b200_moe_combine (ys -> y) and b200_moe_combine_backward (dy, ys -> d_ys, d_w); strides in elements
struct MoeCombineParams {
  uint64_t ys, weights, row_of, y;
  uint64_t d_ys, d_w;
  uint64_t ys_stride, y_stride, d_ys_stride;  // y / y_stride are dy and its stride in the backward
  uint64_t rows;          // rows of ys (and d_ys); row_of entries outside [0, rows) are dropped slots
  uint32_t T, k, N;
  uint32_t vec;           // 1: every row start is 16-byte aligned and N % 8 == 0 (8-element vector access)
};

constexpr int kMoeMaxExperts = 1024;
constexpr int kMoeMaxK = 32;
constexpr int kMoeRouteWarps = 4;      // tokens per route CTA, one warp each
constexpr int kMoePlanWarps = 8;       // a plan CTA: 8 warps, each owning warp_slots consecutive slots
constexpr int kMoePlanWarpSlots = 256; // the least warp_slots; more once T * k needs over kMoePlanMaxCtas CTAs
constexpr int kMoePlanMaxCtas = 1024;  // bounds the [E][CTAs] table: at most 4 MiB, 1024 entries per scan thread
constexpr int kMoeScanThreads = 1024;
constexpr int kMoePermuteWarps = 8;    // rows per permute CTA, one warp each
constexpr int kMoeThreads = 256;       // combine / combine-backward CTA; a thread owns 8 consecutive columns per step
constexpr int kMoeBwdMaxN = 32768;     // the backward stages dy[t] as f32 in shared memory
