// Mixture-of-experts routing (capi.cpp: b200_moe_*; contracts in include/cubecl_b200.h): top-k gating, the expert-sorted
// dispatch plan the grouped matmul takes (offs, row_of, slot_of), the row gather into expert order, and the weighted
// combine with its backward.
//
// Determinism: no floating-point atomics and no atomics at all -- every position is a function of the input alone.  The plan
// is a counting sort whose counts come from __match_any_sync groups (a leader lane adds its group's size), and whose ranks
// are taken in slot order: warp by warp within a CTA, CTA by CTA within an expert (moe_plan_scan's fixed-order scan).
// Every float reduction runs in a fixed order (a lane's elements in index order, then an xor butterfly, then warps in
// order), so results are bitwise reproducible from run to run.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cstdint>
#include <type_traits>

#include "kernel_params.h"

extern __shared__ __align__(16) uint32_t moe_smem[];

__device__ __forceinline__ float moe_f32(float v) { return v; }
__device__ __forceinline__ float moe_f32(__nv_bfloat16 v) { return __bfloat162float(v); }
__device__ __forceinline__ float moe_f32(__half v) { return __half2float(v); }
__device__ __forceinline__ void moe_put(float* o, float v) { *o = v; }
__device__ __forceinline__ void moe_put(__nv_bfloat16* o, float v) { *o = __float2bfloat16_rn(v); }
__device__ __forceinline__ void moe_put(__half* o, float v) { *o = __float2half_rn(v); }

// 8 consecutive elements as f32: 16-byte vector access when `vec`, else element by element up to `n` (the row's end).
template <typename T>
__device__ __forceinline__ void moe_ld8(const T* p, bool vec, uint32_t n, float (&v)[8]) {
  if (vec) {
    if constexpr (sizeof(T) == 4) {
      const float4 a = __ldg(reinterpret_cast<const float4*>(p)), b = __ldg(reinterpret_cast<const float4*>(p) + 1);
      v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    } else {
      const uint4 a = __ldg(reinterpret_cast<const uint4*>(p));
      const T* h = reinterpret_cast<const T*>(&a);
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] = moe_f32(h[i]);
    }
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = (uint32_t)i < n ? moe_f32(p[i]) : 0.0f;
  }
}
template <typename T>
__device__ __forceinline__ void moe_st8(T* p, bool vec, uint32_t n, const float (&v)[8]) {
  if (vec) {
    if constexpr (sizeof(T) == 4) {
      reinterpret_cast<float4*>(p)[0] = make_float4(v[0], v[1], v[2], v[3]);
      reinterpret_cast<float4*>(p)[1] = make_float4(v[4], v[5], v[6], v[7]);
    } else {
      uint4 a;
      T* h = reinterpret_cast<T*>(&a);
#pragma unroll
      for (int i = 0; i < 8; ++i) moe_put(h + i, v[i]);
      *reinterpret_cast<uint4*>(p) = a;
    }
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i)
      if ((uint32_t)i < n) moe_put(p + i, v[i]);
  }
}

// ------------------------------------------------------------------------------------------------ route
// A selection key as an unsigned order: larger is better, -0 ties +0, NaN ranks below -inf (1) and 0 marks an expert that is
// taken or not eligible.  A candidate is (order << 32) | ~e, so equal keys go to the lower index.
__device__ __forceinline__ uint32_t moe_ord(float f) {
  if (f != f) return 1u;
  if (f == 0.0f) f = 0.0f;
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float moe_unord(uint32_t o) {
  if (o <= 1u) return __uint_as_float(0x7FC00000u);
  return __uint_as_float((o & 0x80000000u) ? (o & 0x7FFFFFFFu) : ~o);
}
__device__ __forceinline__ uint64_t moe_cand(uint32_t ord, uint32_t e) { return ((uint64_t)ord << 32) | (0xFFFFFFFFu - e); }
__device__ __forceinline__ uint64_t moe_warp_max(uint64_t v) {
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) {
    const uint64_t o = __shfl_xor_sync(0xFFFFFFFFu, v, m);
    v = o > v ? o : v;
  }
  return v;
}
__device__ __forceinline__ float moe_sigmoid(float l) { return 1.0f / (1.0f + expf(-l)); }

// One warp per token.  Shared memory per warp: E selection orders, then n_group group orders.
template <typename T>
__device__ __forceinline__ void moe_route(const MoeRouteParams& p) {
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  const uint64_t t = (uint64_t)blockIdx.x * kMoeRouteWarps + warp;
  if (t >= p.T) return;
  const uint32_t E = p.E, G = p.n_group > 1 ? p.n_group : 0u;
  uint32_t* ord = moe_smem + warp * (E + (E >> 1));
  uint32_t* gord = ord + E;
  const T* row = reinterpret_cast<const T*>(p.logits) + t * p.stride;
  const float* bias = reinterpret_cast<const float*>(p.bias);
  const bool sig = p.score == B200_MOE_SIGMOID;
  // softmax: max (NaN ignored), then the sum of expf(l - max): a lane's experts in order, then the butterfly
  float mx = -INFINITY, sum = 0.0f;
  if (!sig) {
    for (uint32_t e = lane; e < E; e += 32) mx = fmaxf(mx, moe_f32(row[e]));
#pragma unroll
    for (int m = 16; m >= 1; m >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xFFFFFFFFu, mx, m));
    for (uint32_t e = lane; e < E; e += 32) sum += expf(moe_f32(row[e]) - mx);
#pragma unroll
    for (int m = 16; m >= 1; m >>= 1) sum += __shfl_xor_sync(0xFFFFFFFFu, sum, m);
  }
  // keys: the logit without a bias (both scores are monotone in it), else rn(s_e + b_e)
  for (uint32_t e = lane; e < E; e += 32) {
    const float l = moe_f32(row[e]);
    float key = l;
    if (bias) key = (sig ? moe_sigmoid(l) : expf(l - mx) / sum) + bias[e];
    ord[e] = moe_ord(key);
  }
  __syncwarp();
  if (G) {
    // group-limited: a group's score is the sum of its two best keys; only the topk_group best groups stay eligible
    const uint32_t gs = E / G;
    for (uint32_t g = lane; g < G; g += 32) {
      uint64_t b1 = 0, b2 = 0;
      for (uint32_t i = 0; i < gs; ++i) {
        const uint64_t c = moe_cand(ord[g * gs + i], g * gs + i);
        if (c > b1) { b2 = b1; b1 = c; } else if (c > b2) b2 = c;
      }
      gord[g] = moe_ord(moe_unord((uint32_t)(b1 >> 32)) + moe_unord((uint32_t)(b2 >> 32)));
    }
    __syncwarp();
    for (uint32_t j = 0; j < p.topk_group; ++j) {
      uint64_t best = 0;
      for (uint32_t g = lane; g < G; g += 32)
        if (gord[g] != 0xFFFFFFFFu) { const uint64_t c = moe_cand(gord[g], g); best = c > best ? c : best; }
      best = moe_warp_max(best);
      __syncwarp();
      if (lane == 0) gord[0xFFFFFFFFu - (uint32_t)best] = 0xFFFFFFFFu;   // chosen
      __syncwarp();
    }
    for (uint32_t e = lane; e < E; e += 32)
      if (gord[e / gs] != 0xFFFFFFFFu) ord[e] = 0u;
    __syncwarp();
  }
  // top-k: each lane keeps its best candidate; the winner of a round marks its expert taken and rescans its own experts
  auto local_best = [&]() {
    uint64_t b = 0;
    for (uint32_t e = lane; e < E; e += 32) { const uint64_t c = moe_cand(ord[e], e); b = c > b ? c : b; }
    return b;
  };
  uint64_t mine = local_best();
  uint32_t sel = 0;
  for (uint32_t j = 0; j < p.k; ++j) {
    const uint64_t w = moe_warp_max(mine);
    const uint32_t e = 0xFFFFFFFFu - (uint32_t)w;
    if (lane == j) sel = e;
    if ((e & 31u) == lane) { ord[e] = 0u; mine = local_best(); }
  }
  // weights: w_j = s_{e_j}; renormalised by their sum in j order; then rn(w_j * scale)
  float w = 0.0f;
  if (lane < p.k) {
    const float l = moe_f32(row[sel]);
    w = sig ? moe_sigmoid(l) : expf(l - mx) / sum;
  }
  if (p.renorm) {
    float tot = 0.0f;
    for (uint32_t j = 0; j < p.k; ++j) tot += __shfl_sync(0xFFFFFFFFu, w, j);
    w = w / tot;
  }
  if (lane < p.k) {
    reinterpret_cast<int32_t*>(p.ids)[t * p.k + lane] = (int32_t)sel;
    reinterpret_cast<float*>(p.weights)[t * p.k + lane] = w * p.scale;
  }
}

extern "C" __global__ void __launch_bounds__(kMoeRouteWarps * 32) moe_route_f32(const __grid_constant__ MoeRouteParams p) { moe_route<float>(p); }
extern "C" __global__ void __launch_bounds__(kMoeRouteWarps * 32) moe_route_bf16(const __grid_constant__ MoeRouteParams p) { moe_route<__nv_bfloat16>(p); }
extern "C" __global__ void __launch_bounds__(kMoeRouteWarps * 32) moe_route_f16(const __grid_constant__ MoeRouteParams p) { moe_route<__half>(p); }

// ------------------------------------------------------------------------------------------------ plan
// Counting sort of the T * k slots by expert.  With S = warp_slots (256, or a larger multiple of 256 once T * k needs more
// than 1024 CTAs), CTA c owns slots [c * 8S, (c + 1) * 8S) and warp w of it the S slots from c * 8S + w * S.  cnt[w][e]: how many of warp w's slots go to expert e (ids outside [0, E) are dropped).
__device__ __forceinline__ int32_t moe_plan_id(const MoePlanParams& p, uint32_t slot) {
  const int32_t e = slot < p.n ? __ldg(reinterpret_cast<const int32_t*>(p.ids) + slot) : -1;
  return (e >= 0 && (uint32_t)e < p.E) ? e : -1;
}
__device__ __forceinline__ void moe_plan_count(const MoePlanParams& p, uint32_t* cnt) {
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  for (uint32_t i = threadIdx.x; i < kMoePlanWarps * p.E; i += blockDim.x) cnt[i] = 0u;
  __syncthreads();
  const uint32_t base = (blockIdx.x * kMoePlanWarps + warp) * p.warp_slots;
  for (uint32_t i = 0; i < p.warp_slots; i += 32) {
    const int32_t e = moe_plan_id(p, base + i + lane);
    const uint32_t grp = __match_any_sync(0xFFFFFFFFu, e);
    if (e >= 0 && lane == (uint32_t)(__ffs(grp) - 1)) cnt[warp * p.E + e] += __popc(grp);
    __syncwarp();
  }
  __syncthreads();
}

extern "C" __global__ void __launch_bounds__(kMoePlanWarps * 32) moe_plan_histogram(const __grid_constant__ MoePlanParams p) {
  moe_plan_count(p, moe_smem);
  int32_t* hist = reinterpret_cast<int32_t*>(p.hist);
  for (uint32_t e = threadIdx.x; e < p.E; e += blockDim.x) {
    uint32_t s = 0;
    for (int w = 0; w < kMoePlanWarps; ++w) s += moe_smem[w * p.E + e];
    hist[(uint64_t)e * p.ctas + blockIdx.x] = (int32_t)s;
  }
}

// One CTA: the exclusive scan of hist in its [E][ctas] order (expert-major, CTAs in order), in place: each entry becomes the
// first sorted row of that CTA's run of that expert.  offs[e] = the end of expert e's rows.
extern "C" __global__ void __launch_bounds__(kMoeScanThreads) moe_plan_scan(const __grid_constant__ MoePlanParams p) {
  __shared__ uint32_t warp_tot[kMoeScanThreads / 32];
  int32_t* hist = reinterpret_cast<int32_t*>(p.hist);
  int32_t* offs = reinterpret_cast<int32_t*>(p.offs);
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  const uint64_t total = (uint64_t)p.E * p.ctas, per = (total + kMoeScanThreads - 1) / kMoeScanThreads;
  const uint64_t lo = min(total, threadIdx.x * per), hi = min(total, lo + per);
  if (p.ctas == 0) {
    for (uint32_t e = threadIdx.x; e < p.E; e += blockDim.x) offs[e] = 0;
    return;
  }
  uint32_t own = 0;
  for (uint64_t i = lo; i < hi; ++i) own += (uint32_t)hist[i];
  uint32_t inc = own;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t o = __shfl_up_sync(0xFFFFFFFFu, inc, d);
    if (lane >= (uint32_t)d) inc += o;
  }
  if (lane == 31) warp_tot[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    uint32_t v = warp_tot[lane], s = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t o = __shfl_up_sync(0xFFFFFFFFu, s, d);
      if (lane >= (uint32_t)d) s += o;
    }
    warp_tot[lane] = s - v;
  }
  __syncthreads();
  uint32_t run = warp_tot[warp] + inc - own;
  uint32_t e = (uint32_t)(lo / p.ctas), c = (uint32_t)(lo % p.ctas);
  for (uint64_t i = lo; i < hi; ++i) {
    const uint32_t v = (uint32_t)hist[i];
    hist[i] = (int32_t)run;
    run += v;
    if (++c == p.ctas) { offs[e++] = (int32_t)run; c = 0; }
  }
}

// Stable re-rank: each warp's runs start where the warps before it in the CTA end (from the CTA's scanned run starts); a
// slot's row is its run's next row plus its rank among the lanes of its __match_any_sync group.  row_of[slot] = row (-1 when
// dropped), slot_of[row] = slot; slot_of past the kept count (offs[E-1]) is -1.
extern "C" __global__ void __launch_bounds__(kMoePlanWarps * 32) moe_plan_scatter(const __grid_constant__ MoePlanParams p) {
  uint32_t* cnt = moe_smem;
  moe_plan_count(p, cnt);
  const int32_t* hist = reinterpret_cast<const int32_t*>(p.hist);
  for (uint32_t e = threadIdx.x; e < p.E; e += blockDim.x) {
    uint32_t run = (uint32_t)hist[(uint64_t)e * p.ctas + blockIdx.x];
    for (int w = 0; w < kMoePlanWarps; ++w) {
      const uint32_t c = cnt[w * p.E + e];
      cnt[w * p.E + e] = run;
      run += c;
    }
  }
  __syncthreads();
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  const uint32_t base = (blockIdx.x * kMoePlanWarps + warp) * p.warp_slots;
  const uint32_t kept = (uint32_t)reinterpret_cast<const int32_t*>(p.offs)[p.E - 1];
  int32_t* row_of = reinterpret_cast<int32_t*>(p.row_of);
  int32_t* slot_of = reinterpret_cast<int32_t*>(p.slot_of);
  for (uint32_t i = 0; i < p.warp_slots; i += 32) {
    const uint32_t slot = base + i + lane;
    const int32_t e = moe_plan_id(p, slot);
    const uint32_t grp = __match_any_sync(0xFFFFFFFFu, e);
    int32_t row = -1;
    if (e >= 0) row = (int32_t)(cnt[warp * p.E + e] + __popc(grp & ((1u << lane) - 1u)));
    __syncwarp();
    if (e >= 0 && lane == (uint32_t)(__ffs(grp) - 1)) cnt[warp * p.E + e] += __popc(grp);
    __syncwarp();
    if (slot < p.n) {
      row_of[slot] = row;
      if (row >= 0) slot_of[row] = (int32_t)slot;
      if (slot >= kept) slot_of[slot] = -1;
    }
  }
}

// ------------------------------------------------------------------------------------------------ permute
// dst[r] = src[slot_of[r] / k] for r with 0 <= slot_of[r] < T * k: one warp per row, V-byte units (16 when every row start
// and row_bytes allow it).
template <int V>
__device__ __forceinline__ void moe_permute(const MoePermuteParams& p) {
  typedef typename std::conditional<V == 16, uint4, typename std::conditional<V == 4, uint32_t, uint8_t>::type>::type U;
  const uint32_t lane = threadIdx.x & 31u;
  const uint64_t r = (uint64_t)blockIdx.x * kMoePermuteWarps + (threadIdx.x >> 5);
  if (r >= p.rows) return;
  const int32_t slot = __ldg(reinterpret_cast<const int32_t*>(p.slot_of) + r);
  if (slot < 0 || (uint64_t)slot >= p.rows) return;
  const U* __restrict__ s = reinterpret_cast<const U*>(p.src + (uint64_t)(slot / p.k) * p.src_pitch);
  U* __restrict__ d = reinterpret_cast<U*>(p.dst + r * p.dst_pitch);
  const uint32_t n = (uint32_t)(p.row_bytes / V);
  uint32_t i = lane;
  for (; i + 96 < n; i += 128) {
    const U a = __ldg(s + i), b = __ldg(s + i + 32), c = __ldg(s + i + 64), e = __ldg(s + i + 96);
    __stcg(d + i, a); __stcg(d + i + 32, b); __stcg(d + i + 64, c); __stcg(d + i + 96, e);
  }
  for (; i < n; i += 32) __stcg(d + i, __ldg(s + i));
}
extern "C" __global__ void __launch_bounds__(kMoePermuteWarps * 32) moe_permute_v16(const __grid_constant__ MoePermuteParams p) { moe_permute<16>(p); }
extern "C" __global__ void __launch_bounds__(kMoePermuteWarps * 32) moe_permute_v4(const __grid_constant__ MoePermuteParams p) { moe_permute<4>(p); }
extern "C" __global__ void __launch_bounds__(kMoePermuteWarps * 32) moe_permute_v1(const __grid_constant__ MoePermuteParams p) { moe_permute<1>(p); }

// ------------------------------------------------------------------------------------------------ combine
// y[t, n] = RNE(acc_k): acc_0 = +0, acc_{j+1} = fma(w[t, j], f32(ys[row_of[t, j], n]), acc_j) over increasing j, dropped slots
// skipped; without weights acc_{j+1} = acc_j + f32(ys[...]).  Grid (T, column chunks of 256 x 8).
template <typename TS, typename TY>
__device__ __forceinline__ void moe_combine(const MoeCombineParams& p) {
  const uint32_t t = blockIdx.x, c0 = (blockIdx.y * kMoeThreads + threadIdx.x) * 8u;
  if (c0 >= p.N) return;
  const bool vec = p.vec != 0;
  const uint32_t n = p.N - c0;
  const int32_t* row_of = reinterpret_cast<const int32_t*>(p.row_of) + (uint64_t)t * p.k;
  const float* wt = p.weights ? reinterpret_cast<const float*>(p.weights) + (uint64_t)t * p.k : nullptr;
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.0f;
  for (uint32_t j = 0; j < p.k; ++j) {
    const int32_t r = __ldg(row_of + j);
    if (r < 0 || (uint64_t)r >= p.rows) continue;
    float v[8];
    moe_ld8(reinterpret_cast<const TS*>(p.ys) + (uint64_t)r * p.ys_stride + c0, vec, n, v);
    if (wt) {
      const float w = __ldg(wt + j);
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = fmaf(w, v[i], acc[i]);
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = acc[i] + v[i];
    }
  }
  moe_st8(reinterpret_cast<TY*>(p.y) + (uint64_t)t * p.y_stride + c0, vec, n, acc);
}

// Backward, one CTA per token: dy[t] is read once into shared memory as f32.  For each j: d_ys[r] = RNE(rn(w * dy)) and
// d_w[t, j] = the dot product of dy[t] and ys[r] -- a thread's fma chain over its columns in increasing order, an xor
// butterfly over the warp, then the warps' sums in warp order; +0 for a dropped slot.
template <typename TG, typename TS>
__device__ __forceinline__ void moe_combine_bwd(const MoeCombineParams& p) {
  __shared__ float red[kMoeThreads / 32];
  float* dy = reinterpret_cast<float*>(moe_smem);
  const uint32_t t = blockIdx.x, lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  const bool vec = p.vec != 0;
  const TG* dyg = reinterpret_cast<const TG*>(p.y) + (uint64_t)t * p.y_stride;
  for (uint32_t c0 = threadIdx.x * 8u; c0 < p.N; c0 += kMoeThreads * 8u) {
    float v[8];
    moe_ld8(dyg + c0, vec, p.N - c0, v);
#pragma unroll
    for (int i = 0; i < 8; ++i)
      if (c0 + i < p.N) dy[c0 + i] = v[i];
  }
  __syncthreads();
  const int32_t* row_of = reinterpret_cast<const int32_t*>(p.row_of) + (uint64_t)t * p.k;
  const float* wt = reinterpret_cast<const float*>(p.weights) + (uint64_t)t * p.k;
  for (uint32_t j = 0; j < p.k; ++j) {
    const int32_t r = __ldg(row_of + j);
    const bool live = r >= 0 && (uint64_t)r < p.rows;
    float part = 0.0f;
    if (live) {
      const float w = __ldg(wt + j);
      const TS* ys = reinterpret_cast<const TS*>(p.ys) + (uint64_t)r * p.ys_stride;
      TG* dys = reinterpret_cast<TG*>(p.d_ys) + (uint64_t)r * p.d_ys_stride;
      for (uint32_t c0 = threadIdx.x * 8u; c0 < p.N; c0 += kMoeThreads * 8u) {
        const uint32_t n = p.N - c0;
        float v[8], g[8];
        moe_ld8(ys + c0, vec, n, v);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float d = (uint32_t)i < n ? dy[c0 + i] : 0.0f;
          part = fmaf(d, v[i], part);
          g[i] = w * d;
        }
        moe_st8(dys + c0, vec, n, g);
      }
    }
#pragma unroll
    for (int m = 16; m >= 1; m >>= 1) part += __shfl_xor_sync(0xFFFFFFFFu, part, m);
    if (lane == 0) red[warp] = part;
    __syncthreads();
    if (threadIdx.x == 0) {
      float s = 0.0f;
      if (live)
        for (int w = 0; w < kMoeThreads / 32; ++w) s += red[w];
      reinterpret_cast<float*>(p.d_w)[(uint64_t)t * p.k + j] = s;
    }
    __syncthreads();
  }
}

#define MOE_COMBINE(ta, TA, tb, TB)                                                                                          \
  extern "C" __global__ void __launch_bounds__(kMoeThreads) moe_combine_##ta##_##tb(const __grid_constant__ MoeCombineParams p) { \
    moe_combine<TA, TB>(p);                                                                                                  \
  }                                                                                                                          \
  extern "C" __global__ void __launch_bounds__(kMoeThreads) moe_combine_bwd_##ta##_##tb(const __grid_constant__ MoeCombineParams p) { \
    moe_combine_bwd<TA, TB>(p);                                                                                              \
  }
#define MOE_COMBINE_ROW(ta, TA) MOE_COMBINE(ta, TA, f32, float) MOE_COMBINE(ta, TA, bf16, __nv_bfloat16) MOE_COMBINE(ta, TA, f16, __half)
MOE_COMBINE_ROW(f32, float)
MOE_COMBINE_ROW(bf16, __nv_bfloat16)
MOE_COMBINE_ROW(f16, __half)
