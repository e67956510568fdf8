// Token sampling from logits: temperature, top-k, min-p, top-p and a Philox draw per row in one launch (capi.cpp: b200_sample;
// contract in include/cubecl_b200.h, geometry in kernel_params.h: SampleParams).
//
// A row is read from HBM once into shared memory, split over the CTAs of a cluster (rank r holds a contiguous slice, so rank
// order is column order).  Every later step reads shared memory only:
//   load     z = rn(x / T) per element into the slice, with the row's max and its NaN / +inf flag (greedy rows: the argmax
//            of x instead, nothing stored);
//   top-k    a radix select of the k-th largest order-preserving u32 key of z, three passes of 11 / 11 / 10 bits;
//   masses   w = ex2(rn(rn(z - m) * log2e)) kept by top-k and min-p, stored over z; the mass is q = floor(w * 2^40);
//   top-p    a radix select of the threshold tau over the masses, four passes of 11 / 11 / 11 / 8 bits, each bin holding the
//            u64 sum of its masses;
//   draw     per-32-column chunk sums of the nucleus, the ranks' totals in rank order through distributed shared memory, then
//            the CTA holding t finds its chunk and one warp scans it.
// Histograms are 32-bit shared-memory integer atomics (native ATOMS.ADD; a 64-bit one is a compare-and-swap loop): counts
// aggregated per warp with match.any, and each mass added as three parts of 14 / 14 / 13 bits whose per-CTA sums stay below
// 2^29.  Every sum is an integer sum, so no result depends on the order anything is added in.  The histograms of the cluster's CTAs are summed
// through distributed shared memory; there are no global atomics.
#include <cooperative_groups.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cstdint>

#include "attention.cuh"
#include "kernel_params.h"

namespace cg = cooperative_groups;
using b200::ex2;

constexpr float kSampleLog2e = 1.4426950408889634f;
constexpr float kSampleMassScale = 1099511627776.0f;   // 2^40
constexpr int kSampleWarps = kSampleThreads / 32;
constexpr int kSampleChunks = kSampleMaxSlice / 32;     // nucleus mass per 32 columns of the slice
constexpr int kSampleUnroll = 4;                        // 16-byte loads a thread has in flight

__device__ __forceinline__ float smp_f32(float v) { return v; }
__device__ __forceinline__ float smp_f32(__nv_bfloat16 v) { return __bfloat162float(v); }
__device__ __forceinline__ float smp_f32(__half v) { return __half2float(v); }

// m <= 8 consecutive elements as f32: one or two 128-bit loads when `vec` and the chunk is whole.
template <typename T>
__device__ __forceinline__ void smp_ld8(const T* p, bool vec, uint32_t m, float (&v)[8]) {
  if (vec && m == 8) {
    if constexpr (sizeof(T) == 4) {
      const float4 a = __ldg(reinterpret_cast<const float4*>(p)), b = __ldg(reinterpret_cast<const float4*>(p) + 1);
      v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    } else {
      const uint4 a = __ldg(reinterpret_cast<const uint4*>(p));
      const T* h = reinterpret_cast<const T*>(&a);
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] = smp_f32(h[i]);
    }
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = (uint32_t)i < m ? smp_f32(p[i]) : 0.0f;
  }
}

// Philox4x32-10 (Salmon et al., Random123) at key (lo, hi of seed) and counter (lo, hi of offset, 0, 0): r0 + 2^32 r1.
__device__ __forceinline__ uint64_t smp_philox(uint64_t seed, uint64_t offset) {
  uint32_t c0 = (uint32_t)offset, c1 = (uint32_t)(offset >> 32), c2 = 0, c3 = 0;
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    c0 = hi1 ^ c1 ^ k0; c1 = lo1; c2 = hi0 ^ c3 ^ k1; c3 = lo0;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return (uint64_t)c0 | ((uint64_t)c1 << 32);
}

// Order-preserving u32 key of a non-NaN f32, -0 and +0 the same key.
__device__ __forceinline__ uint32_t smp_key(float z) {
  const uint32_t b = z == 0.0f ? 0u : __float_as_uint(z);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

// q = floor(w * 2^40): the product is exact (w <= 1), the conversion truncates.
__device__ __forceinline__ uint64_t smp_mass(float w) { return __float2ull_rz(__fmul_rn(w, kSampleMassScale)); }

// ceil(p * S) for an f32 p in (0, 1], exactly: p = M * 2^-sh with a 24-bit M, so the product needs 88 bits.
__device__ __forceinline__ uint64_t smp_ceil_mul(float p, uint64_t S) {
  const uint32_t b = __float_as_uint(p), ex = (b >> 23) & 0xFFu;
  const uint64_t M = ex ? ((b & 0x7FFFFFu) | 0x800000u) : (b & 0x7FFFFFu);
  const uint32_t sh = ex ? 150u - ex : 149u;   // >= 23 for p <= 1
  const uint64_t lo = M * S, hi = __umul64hi(M, S);
  if (sh >= 128) return (lo | hi) ? 1 : 0;
  if (sh >= 64) {
    const uint32_t s = sh - 64;
    const uint64_t rem = lo | (s ? hi & ((1ull << s) - 1) : 0);
    return (s ? hi >> s : hi) + (rem ? 1 : 0);
  }
  return ((lo >> sh) | (hi << (64 - sh))) + ((lo & ((1ull << sh) - 1)) ? 1 : 0);
}

// A row's parameters: the per-row arrays where given, else the scalars; `bad` is the contract's invalid-parameter rule.
struct SmpRow {
  float temp, top_p, min_p;
  int32_t top_k;
  uint64_t seed, offset;
  bool bad;
};
__device__ __forceinline__ SmpRow smp_row(const SampleParams& p, uint64_t r) {
  SmpRow s;
  s.temp = p.temperatures ? reinterpret_cast<const float*>(p.temperatures)[r] : p.temperature;
  s.top_k = p.top_ks ? reinterpret_cast<const int32_t*>(p.top_ks)[r] : p.top_k;
  s.top_p = p.top_ps ? reinterpret_cast<const float*>(p.top_ps)[r] : p.top_p;
  s.min_p = p.min_ps ? reinterpret_cast<const float*>(p.min_ps)[r] : p.min_p;
  s.seed = p.seeds ? reinterpret_cast<const uint64_t*>(p.seeds)[r] : p.seed;
  s.offset = p.offsets ? reinterpret_cast<const uint64_t*>(p.offsets)[r] : p.offset;
  s.bad = !(s.temp >= 0.0f) || s.temp == INFINITY || !(s.top_p > 0.0f && s.top_p <= 1.0f) || !(s.min_p >= 0.0f && s.min_p <= 1.0f);
  return s;
}

// The load pass's state: max (first index of it), and whether a NaN or +inf was seen.  The merge is exact and symmetric.
struct SmpStat {
  float m;
  uint32_t idx, bad;
};
__device__ __forceinline__ void smp_take(SmpStat& a, float x, uint32_t i) {
  if (x != x || x == INFINITY) a.bad = 1u;
  else if (x > a.m || (x == a.m && i < a.idx)) { a.m = x; a.idx = i; }
}
__device__ __forceinline__ SmpStat smp_merge(const SmpStat& a, const SmpStat& b) {
  const bool tb = b.m > a.m || (b.m == a.m && b.idx < a.idx);
  return {tb ? b.m : a.m, tb ? b.idx : a.idx, a.bad | b.bad};
}

__device__ __forceinline__ void smp_sync(uint32_t ranks) {
  if (ranks > 1) cg::this_cluster().sync();
  else __syncthreads();
}
template <typename T>
__device__ __forceinline__ T* smp_peer(T* p, uint32_t r, uint32_t ranks) {
  return ranks > 1 ? cg::this_cluster().map_shared_rank(p, r) : p;
}

__device__ __forceinline__ uint64_t smp_warp_sum(uint64_t v) {
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, o);
  return v;
}

// Shared state of the row kernel (static; the slice and the histograms are dynamic: kSampleHistWords after the slice).
struct SmpShared {
  uint64_t tot[kSampleBins];                 // a radix pass's histogram summed over the cluster
  uint64_t chunk[kSampleChunks];             // nucleus mass of each 32 columns of the slice
  uint64_t wsum[kSampleWarps];
  uint64_t ssum, lsum;                       // this CTA's kept mass and nucleus mass, read by the cluster's peers
  uint64_t need;
  uint32_t digit, pick;
};
__device__ __forceinline__ SmpShared& smp_shared() {
  __shared__ SmpShared s;
  return s;
}

// One radix pass after every CTA of the cluster added its elements into h (its own buffer; PARTS = 3: a bin's weight is
// h[b] + 2^14 h[b + kSampleBins] + 2^28 h[b + 2 kSampleBins]): the bins of all ranks are summed, and the bin d is found,
// scanning from the top, where the weight above d is < need <= the weight at or above d.  Returns d and sets need to
// need - (weight above d), the same in every thread of the cluster.  The ranks' histograms are read 16 bytes per thread in
// bin order, so a warp's reads of a peer coalesce.
template <int BINS, int PARTS>
__device__ __forceinline__ uint32_t smp_find(SmpShared& sh, uint32_t* h, uint32_t ranks, uint32_t rank, uint64_t& need) {
  constexpr int PER = BINS / kSampleThreads;
  static_assert(PER >= 1 && PER * kSampleThreads == BINS, "bins per thread");
  constexpr int V4 = BINS / 4;
  smp_sync(ranks);
  for (uint32_t i = threadIdx.x; i < (uint32_t)V4; i += kSampleThreads) {
    uint64_t a0 = 0, a1 = 0, a2 = 0, a3 = 0;
    for (uint32_t r = 0; r < ranks; ++r) {
      const uint4* ph = reinterpret_cast<const uint4*>(smp_peer(h, (rank + r) % ranks, ranks));
#pragma unroll
      for (int part = 0; part < PARTS; ++part) {
        const uint4 u = ph[part * (kSampleBins / 4) + i];
        a0 += (uint64_t)u.x << (14 * part); a1 += (uint64_t)u.y << (14 * part);
        a2 += (uint64_t)u.z << (14 * part); a3 += (uint64_t)u.w << (14 * part);
      }
    }
    sh.tot[4 * i] = a0; sh.tot[4 * i + 1] = a1; sh.tot[4 * i + 2] = a2; sh.tot[4 * i + 3] = a3;
  }
  __syncthreads();
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5, b0 = threadIdx.x * PER;
  uint64_t c[PER], tot = 0;
#pragma unroll
  for (int j = 0; j < PER; ++j) c[j] = sh.tot[b0 + j];
#pragma unroll
  for (int j = 0; j < PER; ++j) tot += c[j];
  uint64_t inc = tot;   // suffix sum over the warp's lanes >= lane
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint64_t t = __shfl_down_sync(0xFFFFFFFFu, inc, o);
    if (lane + o < 32) inc += t;
  }
  if (lane == 0) sh.wsum[warp] = inc;
  __syncthreads();
  uint64_t above = inc - tot;
  for (uint32_t w = warp + 1; w < kSampleWarps; ++w) above += sh.wsum[w];
  if (above < need && need <= above + tot) {
    uint64_t acc = above;
    bool found = false;
#pragma unroll
    for (int j = PER - 1; j >= 0; --j) {
      if (!found && acc + c[j] >= need) {
        sh.digit = b0 + j;
        sh.need = need - acc;
        found = true;
      }
      acc += c[j];
    }
  }
  __syncthreads();
  need = sh.need;
  return sh.digit;
}

template <typename TX, bool GREEDY_ONLY>
__device__ __forceinline__ void smp_rows(const SampleParams& p) {
  extern __shared__ __align__(16) float zs[];
  __shared__ SmpStat wstat[kSampleWarps], cstat;
  const uint32_t ranks = p.ranks, rank = blockIdx.x % ranks, tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
  const uint32_t s0 = rank * p.slice, n = min(p.slice, p.v - s0), nch = (n + 7) / 8;
  const bool vec = p.vec != 0;
  uint32_t* const hist = reinterpret_cast<uint32_t*>(zs + p.slice);   // [2][3][kSampleBins]
  const uint64_t step = gridDim.x / ranks;
  uint32_t par = 0;
  for (uint64_t r = blockIdx.x / ranks; r < p.b; r += step) {
    const SmpRow row = smp_row(p, r);
    const bool greedy = GREEDY_ONLY || row.temp == 0.0f;
    int64_t id = -1;
    bool writer = rank == 0 && tid == 0;   // the thread that writes ids[r]
    if (!row.bad) {
      // ---- load: z into the slice (greedy: the argmax of x), max and the NaN / +inf flag
      const TX* x = reinterpret_cast<const TX*>(p.logits) + r * p.ls + s0;
      SmpStat st{-INFINITY, 0xFFFFFFFFu, 0u};
      for (uint32_t c = tid; c < nch; c += kSampleUnroll * kSampleThreads) {
        float a[kSampleUnroll][8];
#pragma unroll
        for (int u = 0; u < kSampleUnroll; ++u) {
          const uint32_t cu = c + u * kSampleThreads;
          if (cu < nch) smp_ld8(x + cu * 8u, vec, min(8u, n - cu * 8u), a[u]);
        }
#pragma unroll
        for (int u = 0; u < kSampleUnroll; ++u) {
          const uint32_t cu = c + u * kSampleThreads, m = cu < nch ? min(8u, n - cu * 8u) : 0u;
          if (!GREEDY_ONLY && !greedy) {
#pragma unroll
            for (int i = 0; i < 8; ++i) a[u][i] = __fdiv_rn(a[u][i], row.temp);
            if (m == 8) {
              reinterpret_cast<float4*>(zs + cu * 8u)[0] = make_float4(a[u][0], a[u][1], a[u][2], a[u][3]);
              reinterpret_cast<float4*>(zs + cu * 8u)[1] = make_float4(a[u][4], a[u][5], a[u][6], a[u][7]);
            } else {
#pragma unroll
              for (int i = 0; i < 8; ++i)
                if ((uint32_t)i < m) zs[cu * 8u + i] = a[u][i];
            }
          }
#pragma unroll
          for (int i = 0; i < 8; ++i)
            if ((uint32_t)i < m) smp_take(st, a[u][i], s0 + cu * 8u + i);
        }
      }
#pragma unroll
      for (int o = 16; o >= 1; o >>= 1) {
        const SmpStat q{__shfl_xor_sync(0xFFFFFFFFu, st.m, o), __shfl_xor_sync(0xFFFFFFFFu, st.idx, o),
                        __shfl_xor_sync(0xFFFFFFFFu, st.bad, o)};
        st = smp_merge(st, q);
      }
      if (lane == 0) wstat[warp] = st;
      __syncthreads();
      st = wstat[0];
      for (int w = 1; w < kSampleWarps; ++w) st = smp_merge(st, wstat[w]);
      if (ranks > 1) {
        if (tid == 0) cstat = st;
        cg::this_cluster().sync();
        for (uint32_t q = 0; q < ranks; ++q)
          if (q != rank) st = smp_merge(st, *smp_peer(&cstat, q, ranks));
      }
      const bool ok = !st.bad && st.m != -INFINITY;
      if (greedy) {
        if (ok) id = st.idx;
      } else if constexpr (!GREEDY_ONLY) {
        if (ok) {
          SmpShared& sh = smp_shared();
          const float zmax = st.m;
          // ---- top-k: the key K of the k-th largest z (with multiplicity)
          const bool topk = row.top_k >= 1 && (uint32_t)row.top_k < p.v;
          uint32_t K = 0;
          if (topk) {
            uint64_t need = (uint64_t)row.top_k;
            uint32_t pmask = 0;
#pragma unroll 1
            for (int pass = 0; pass < 3; ++pass) {
              const uint32_t shift = pass == 0 ? 21u : pass == 1 ? 10u : 0u, dmask = pass == 2 ? 0x3FFu : 0x7FFu;
              uint32_t* h = hist + par * kSampleHistWords;
              par ^= 1u;
              for (uint32_t i = tid; i < kSampleBins; i += kSampleThreads) h[i] = 0u;
              __syncthreads();
              for (uint32_t base = 0; base < n; base += kSampleThreads) {
                const uint32_t i = base + tid;
                const uint32_t key = i < n ? smp_key(zs[i]) : 0u;
                const bool in = i < n && (key & pmask) == K;
                const uint32_t d = in ? (key >> shift) & dmask : 0xFFFFFFFFu;
                const uint32_t same = __match_any_sync(0xFFFFFFFFu, d);
                if (in && lane == (uint32_t)(__ffs(same) - 1)) atomicAdd(&h[d], (uint32_t)__popc(same));
              }
              const uint32_t d = pass == 2 ? smp_find<1024, 1>(sh, h, ranks, rank, need)
                                           : smp_find<kSampleBins, 1>(sh, h, ranks, rank, need);
              K |= d << shift;
              pmask |= dmask << shift;
            }
          }
          // ---- masses: w kept by top-k and min-p, stored over z; S = the kept mass
          uint64_t S = 0;
          for (uint32_t i = tid; i < n; i += kSampleThreads) {
            const float z = zs[i];
            float w = ex2(__fmul_rn(__fsub_rn(z, zmax), kSampleLog2e));
            if ((topk && smp_key(z) < K) || !(w >= row.min_p)) w = 0.0f;
            zs[i] = w;
            S += smp_mass(w);
          }
          // ---- top-p: tau, the largest kept mass with (kept mass at or above it) >= ceil(top_p * S); 1 keeps every q > 0
          uint64_t tau = 1;
          if (row.top_p < 1.0f) {
            S = smp_warp_sum(S);
            if (lane == 0) sh.wsum[warp] = S;
            __syncthreads();
            S = 0;
            for (int w = 0; w < kSampleWarps; ++w) S += sh.wsum[w];
            if (ranks > 1) {
              if (tid == 0) sh.ssum = S;
              cg::this_cluster().sync();
              for (uint32_t q = 0; q < ranks; ++q)
                if (q != rank) S += *smp_peer(&sh.ssum, q, ranks);
            }
            uint64_t need = smp_ceil_mul(row.top_p, S), pre = 0, pmask = 0;
#pragma unroll 1
            for (int pass = 0; pass < 4; ++pass) {
              const uint32_t shift = pass == 0 ? 30u : pass == 1 ? 19u : pass == 2 ? 8u : 0u;
              const uint64_t dmask = pass == 3 ? 0xFFull : 0x7FFull;
              uint32_t* h = hist + par * kSampleHistWords;
              par ^= 1u;
              for (uint32_t i = tid; i < kSampleHistWords; i += kSampleThreads) h[i] = 0u;
              __syncthreads();
              for (uint32_t i = tid; i < n; i += kSampleThreads) {
                const uint64_t q = smp_mass(zs[i]);
                if (q && (q & pmask) == pre) {
                  const uint32_t d = (uint32_t)((q >> shift) & dmask);
                  atomicAdd(&h[d], (uint32_t)q & 0x3FFFu);
                  atomicAdd(&h[kSampleBins + d], (uint32_t)(q >> 14) & 0x3FFFu);
                  atomicAdd(&h[2 * kSampleBins + d], (uint32_t)(q >> 28));
                }
              }
              const uint64_t d = pass == 3 ? smp_find<256, 3>(sh, h, ranks, rank, need)
                                           : smp_find<kSampleBins, 3>(sh, h, ranks, rank, need);
              pre |= d << shift;
              pmask |= dmask << shift;
            }
            tau = pre;
          }
          // ---- the nucleus (q >= tau): mass per 32 columns, this CTA's total, the ranks before it
          uint64_t L = 0;
          for (uint32_t base = 0; base < n; base += kSampleThreads) {
            const uint32_t i = base + tid;
            uint64_t q = i < n ? smp_mass(zs[i]) : 0;
            q = smp_warp_sum(q >= tau ? q : 0);
            if (lane == 0) sh.chunk[(base >> 5) + warp] = q;
            L += q;
          }
          if (lane == 0) sh.wsum[warp] = L;
          __syncthreads();
          L = 0;
          for (int w = 0; w < kSampleWarps; ++w) L += sh.wsum[w];
          uint64_t pre = 0, tot = L;
          if (ranks > 1) {
            if (tid == 0) sh.lsum = L;
            cg::this_cluster().sync();
            for (uint32_t q = 0; q < ranks; ++q) {
              if (q == rank) continue;
              const uint64_t lq = *smp_peer(&sh.lsum, q, ranks);
              tot += lq;
              if (q < rank) pre += lq;
            }
          }
          // ---- draw: t = floor(r * S' / 2^64); the CTA whose slice holds t finds the column
          const uint64_t t = __umul64hi(smp_philox(row.seed, row.offset), tot);
          writer = false;
          if (t >= pre && t - pre < L) {
            const uint64_t tl = t - pre;
            constexpr int CPT = kSampleChunks / kSampleThreads;   // chunks per thread
            const uint32_t c0 = tid * CPT;
            uint64_t cs[CPT], own = 0;
            const uint32_t nchunks = ((n + kSampleThreads - 1) / kSampleThreads) * kSampleWarps;
#pragma unroll
            for (int j = 0; j < CPT; ++j) {
              cs[j] = c0 + j < nchunks ? sh.chunk[c0 + j] : 0;
              own += cs[j];
            }
            uint64_t inc = own;   // prefix over the warp's lanes <= lane
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
              const uint64_t v = __shfl_up_sync(0xFFFFFFFFu, inc, o);
              if (lane >= (uint32_t)o) inc += v;
            }
            __syncthreads();   // every thread has read wsum above
            if (lane == 31) sh.wsum[warp] = inc;
            __syncthreads();
            uint64_t below = inc - own;
            for (uint32_t w = 0; w < warp; ++w) below += sh.wsum[w];
            if (below <= tl && tl < below + own) {
              uint64_t acc = below;
              bool found = false;
#pragma unroll
              for (int j = 0; j < CPT; ++j) {
                if (!found && tl < acc + cs[j]) {
                  sh.pick = c0 + j;
                  sh.need = tl - acc;
                  found = true;
                }
                acc += cs[j];
              }
            }
            __syncthreads();
            if (warp == 0) {
              const uint32_t i = sh.pick * 32u + lane;
              const uint64_t tc = sh.need;
              uint64_t q = i < n ? smp_mass(zs[i]) : 0;
              q = q >= tau ? q : 0;
              uint64_t inc2 = q;
#pragma unroll
              for (int o = 1; o < 32; o <<= 1) {
                const uint64_t v = __shfl_up_sync(0xFFFFFFFFu, inc2, o);
                if (lane >= (uint32_t)o) inc2 += v;
              }
              if (q && inc2 - q <= tc && tc < inc2) {
                id = s0 + i;
                writer = true;
              }
            }
          }
        }
      }
    }
    if (writer) {
      if (p.ids64) reinterpret_cast<int64_t*>(p.ids)[r] = id;
      else reinterpret_cast<int32_t*>(p.ids)[r] = (int32_t)id;
    }
    smp_sync(ranks);   // every rank has read this row's parameters and is done with the shared state
    if (p.advance && rank == 0 && tid == 0) reinterpret_cast<uint64_t*>(p.offsets)[r] = row.offset + 1;
  }
}

#define SAMPLE_KERNELS(tx, TX)                                                                                             \
  extern "C" __global__ void __launch_bounds__(kSampleThreads, 2) sample_##tx(const __grid_constant__ SampleParams p) {     \
    smp_rows<TX, false>(p);                                                                                                \
  }                                                                                                                        \
  extern "C" __global__ void __launch_bounds__(kSampleThreads, 4) sample_greedy_##tx(const __grid_constant__ SampleParams p) { \
    smp_rows<TX, true>(p);                                                                                                 \
  }
SAMPLE_KERNELS(f32, float)
SAMPLE_KERNELS(bf16, __nv_bfloat16)
SAMPLE_KERNELS(f16, __half)
