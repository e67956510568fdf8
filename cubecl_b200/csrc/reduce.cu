// Hand-written sm_90a reductions: sum / mean / prod / max / min / argmax / argmin over all elements, over the
// innermost axis ("rows") or over an outer/middle axis ("columns").  HBM-bound: coalesced 128-bit (optionally 256-bit)
// streaming loads -- or 16 KB bulk copies (cp.async.bulk, UBLKCP) into a shared-memory ring for the `_tma` variants --
// many independent accumulators per thread, __shfl_down warp stage, smem block stage, and a last-block-done grid stage
// inside the same launch (no second kernel, no host sync).
//
// Replaces: the (out-of-tree, cubek) `reduce::launch` kernel bodies and the in-tree reduction-shaped kernels
//   examples/sum_things/src/lib.rs:6-33            (sum_basic / sum_subgroup -> plane_sum)
//   crates/cubecl-std/src/throughput/runners/memory_read.rs:68-154   (vec4 streaming read-accumulate)
//   cubecl-book/src/getting-started/src/bin/v5-gpu.rs:50-57          (row-sum, one unit per row)
// plane_sum in the reference is an xor butterfly (crates/cubecl-cpp/src/shared/plane.rs:61-70); a shfl_down tree
// produces the same value in lane 0 for commutative ops and needs no broadcast.
//
// Inputs are VIEWS: every kernel takes element strides for the outer and the reduced axis plus an optional row pitch, so
// pitched `TensorHandle::empty` tensors (crates/cubecl-runtime/src/allocator.rs:21-72) and transposed views are read in
// place -- 1x the logical bytes, no `into_contiguous` pass.  Any base alignment is accepted (scalar head / tail peel).
//
// Arg-reductions: ties -> lowest index; NaN compares as the extreme value (first NaN wins), i.e. numpy semantics.  They run
// on a monotone integer key of the value packed with the complemented index, (key << 32) | ~index, so "better" is a plain
// unsigned 64-bit max -- associative and commutative, hence independent of the reduction tree.
// Compiled to a cubin: nvcc -cubin -gencode arch=compute_90a,code=sm_90a
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cstdint>

#include "kernel_params.h"
#include "ptx.cuh"

enum : int { OP_SUM = 0, OP_PROD = 1, OP_MAX = 2, OP_MIN = 3, OP_ARGMAX = 4, OP_ARGMIN = 5 };

constexpr int kMaxWarps = 32;

// ------------------------------------------------------------------------------------------------ value ops
template <int OP>
struct ValOp;
template <>
struct ValOp<OP_SUM> {
  static __device__ __forceinline__ float identity() { return 0.f; }
  static __device__ __forceinline__ float apply(float a, float b) { return a + b; }
};
template <>
struct ValOp<OP_PROD> {
  static __device__ __forceinline__ float identity() { return 1.f; }
  static __device__ __forceinline__ float apply(float a, float b) { return a * b; }
};
// max/min propagate NaN (like the reference's `max`/`min` on floats lowered to fmaxf would NOT; we choose the
// numpy/IEEE-754-2019 "maximum" semantics and the oracle states the same rule).
template <>
struct ValOp<OP_MAX> {
  static __device__ __forceinline__ float identity() { return -INFINITY; }
  static __device__ __forceinline__ float apply(float a, float b) {
    float d;
    asm("max.NaN.f32 %0, %1, %2;" : "=f"(d) : "f"(a), "f"(b));  // one FMNMX.NAN: NaN if either input is NaN
    return d;
  }
};
template <>
struct ValOp<OP_MIN> {
  static __device__ __forceinline__ float identity() { return INFINITY; }
  static __device__ __forceinline__ float apply(float a, float b) {
    float d;
    asm("min.NaN.f32 %0, %1, %2;" : "=f"(d) : "f"(a), "f"(b));
    return d;
  }
};
// arg ops never use the float algebra; the specialisations exist so shared code instantiates
template <>
struct ValOp<OP_ARGMAX> : ValOp<OP_MAX> {};
template <>
struct ValOp<OP_ARGMIN> : ValOp<OP_MIN> {};

// ------------------------------------------------------------------------------------------------ arg ops: keys and pairs
// Monotone key of a float: larger key <=> "better" candidate.  -0.0 is folded onto +0.0 first (the two zeros tie, as they
// do under IEEE comparison).  Non-NaN keys lie in [0x007FFFFF, 0xFF800000]; NaN gets the top key (the extreme for both
// argmax and argmin: first NaN wins); 0 is below every key and serves as the identity.
template <int OP>
__device__ __forceinline__ uint32_t arg_key(float f) {
  f = __fadd_rn(f, 0.0f);
  const uint32_t u = __float_as_uint(f);
  uint32_t k = u ^ (static_cast<uint32_t>(static_cast<int32_t>(u) >> 31) | 0x80000000u);
  if (OP == OP_ARGMIN) k = ~k;
  return (f != f) ? 0xFFFFFFFFu : k;
}
__device__ __forceinline__ uint64_t arg_pack(uint32_t key, uint32_t idx) { return (static_cast<uint64_t>(key) << 32) | static_cast<uint32_t>(~idx); }
__device__ __forceinline__ uint32_t arg_index(uint64_t packed) { return ~static_cast<uint32_t>(packed); }
__device__ __forceinline__ uint64_t umax64(uint64_t a, uint64_t b) { return a > b ? a : b; }

// Per-thread running candidate, fed in INCREASING index order (so a strict compare keeps the lowest index on ties).
struct ArgAcc {
  uint32_t k = 0, i = 0xFFFFFFFFu;
  template <int OP>
  __device__ __forceinline__ void feed(float f, uint32_t idx) {
    const uint32_t key = arg_key<OP>(f);
    if (key > k) { k = key; i = idx; }
  }
  __device__ __forceinline__ uint64_t packed() const { return arg_pack(k, i); }
};

// ------------------------------------------------------------------------------------------------ loads
struct float8 {
  float4 lo, hi;
};
// sm_90 has no 256-bit loads: two adjacent 128-bit streaming loads
__device__ __forceinline__ float8 ldg_stream_v8(const float* p) {
  float8 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%8];\n\t"
               "ld.global.nc.L1::no_allocate.v4.f32 {%4,%5,%6,%7}, [%8+16];"
               : "=f"(v.lo.x), "=f"(v.lo.y), "=f"(v.lo.z), "=f"(v.lo.w), "=f"(v.hi.x), "=f"(v.hi.y), "=f"(v.hi.z),
                 "=f"(v.hi.w)
               : "l"(p));
  return v;
}

__device__ __forceinline__ uint4 ldg_stream_u4(const void* p) {
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p));
  return v;
}

template <int DT>
struct Elem;
template <>
struct Elem<B200_F32> {
  using T = float;
  static constexpr int VEC = 4;  // elements per 128-bit load
  static __device__ __forceinline__ float get(const void* base, uint64_t i) { return reinterpret_cast<const float*>(base)[i]; }
  static __device__ __forceinline__ void unpack(uint4 r, float (&f)[4]) {
    f[0] = __uint_as_float(r.x); f[1] = __uint_as_float(r.y); f[2] = __uint_as_float(r.z); f[3] = __uint_as_float(r.w);
  }
};
template <>
struct Elem<B200_F16> {
  using T = __half;
  static constexpr int VEC = 8;
  static __device__ __forceinline__ float get(const void* base, uint64_t i) { return __half2float(reinterpret_cast<const __half*>(base)[i]); }
  static __device__ __forceinline__ void unpack(uint4 r, float (&f)[8]) {
    const uint32_t w[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float2 t = __half22float2(*reinterpret_cast<const __half2*>(&w[j]));
      f[2 * j] = t.x; f[2 * j + 1] = t.y;
    }
  }
};
template <>
struct Elem<B200_BF16> {
  using T = __nv_bfloat16;
  static constexpr int VEC = 8;
  static __device__ __forceinline__ float get(const void* base, uint64_t i) { return __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(base)[i]); }
  static __device__ __forceinline__ void unpack(uint4 r, float (&f)[8]) {
    const uint32_t w[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      f[2 * j] = __uint_as_float(w[j] << 16);
      f[2 * j + 1] = __uint_as_float(w[j] & 0xFFFF0000u);
    }
  }
};

// ------------------------------------------------------------------------------------------------ block stages
template <int OP>
__device__ __forceinline__ float warp_reduce(float v) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v = ValOp<OP>::apply(v, __shfl_down_sync(0xffffffffu, v, off));
  return v;
}

// Result valid in thread 0.
template <int OP>
__device__ __forceinline__ float block_reduce(float v, float* smem /* kMaxWarps */) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = (blockDim.x + 31) >> 5;
  v = warp_reduce<OP>(v);
  if (lane == 0) smem[warp] = v;
  __syncthreads();
  if (warp == 0) {
    v = (lane < nwarps) ? smem[lane] : ValOp<OP>::identity();
    v = warp_reduce<OP>(v);
  }
  __syncthreads();
  return v;
}

__device__ __forceinline__ uint64_t warp_max64(uint64_t v) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v = umax64(v, __shfl_down_sync(0xffffffffu, v, off));
  return v;
}

// Result valid in thread 0.
__device__ __forceinline__ uint64_t block_max64(uint64_t v, uint64_t* smem /* kMaxWarps */) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = (blockDim.x + 31) >> 5;
  v = warp_max64(v);
  if (lane == 0) smem[warp] = v;
  __syncthreads();
  if (warp == 0) {
    v = (lane < nwarps) ? smem[lane] : 0ull;
    v = warp_max64(v);
  }
  __syncthreads();
  return v;
}

__device__ __forceinline__ void st_sys_u64(uint64_t addr, uint64_t v) {
  asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(addr), "l"(v) : "memory");
}
__device__ __forceinline__ uint64_t ld_sys_u64(uint64_t addr) {
  uint64_t v;
  asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(addr) : "memory");
  return v;
}

// Programmatic dependent launch (PDL): a reduction over all elements touches only its input until its grid stage, so the
// NEXT such launch on the stream may start streaming while this one's last block is still finishing.  `pdl_trigger` (after
// the streaming loop) lets a dependent launch begin; `pdl_wait` (before the first access to the shared workspace) holds this
// launch until its predecessor has completed and flushed.  Both are no-ops unless the host asked for the overlap.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ================================================================================================ grid stage
// Per-block partial -> workspace; the last block to finish (ticket) reduces the partials in block order (deterministic for a
// fixed grid) and writes out[0] * scale -- or, in the XGPU form, exchanges the rank's scalar with its peers first.
template <int OP, bool XGPU>
__device__ __forceinline__ void grid_stage_value(const ReduceParams& p, float block_val, float* s_red, const XgpuParams* xg) {
  __shared__ bool s_last;
  float* partials = reinterpret_cast<float*>(p.ws);
  unsigned int* ticket = reinterpret_cast<unsigned int*>(p.ws + kWsTicketOffset);
  pdl_wait();
  if (threadIdx.x == 0) {
    partials[blockIdx.x] = block_val;
    __threadfence();
    const unsigned int t = atomicAdd(ticket, 1u);
    s_last = (t == gridDim.x - 1);
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  const uint64_t t_stage = (p.flags & 1u) ? b200::globaltimer_ns() : 0;
  if constexpr (OP == OP_SUM) {
    // grid stage of a sum in f64: <= 4096 partials, so the only f32 roundings are inside the blocks and the last one
    __shared__ double s_dred[kMaxWarps];
    double d = 0.0;
    for (uint32_t i = threadIdx.x; i < gridDim.x; i += blockDim.x) d += static_cast<double>(__ldcg(partials + i));
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) d += __shfl_down_sync(0xffffffffu, d, off);
    if ((threadIdx.x & 31) == 0) s_dred[threadIdx.x >> 5] = d;
    __syncthreads();
    if (threadIdx.x < 32) {
      const int nwarps = (blockDim.x + 31) >> 5;
      d = (static_cast<int>(threadIdx.x) < nwarps) ? s_dred[threadIdx.x] : 0.0;
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) d += __shfl_down_sync(0xffffffffu, d, off);
      if constexpr (!XGPU) {
        if (threadIdx.x == 0) {
          reinterpret_cast<float*>(p.out)[0] = static_cast<float>(d * static_cast<double>(p.scale));
          *ticket = 0;  // ready for the next launch on this stream
        }
      } else {
        // ---- fused all-reduce: publish this rank's scalar into every peer's mailbox, gather the others, sum in rank order
        __shared__ float s_peer[8];
        d = __shfl_sync(0xffffffffu, d, 0);
        const float mine = static_cast<float>(d * static_cast<double>(p.scale));
        const uint32_t slot_base = (xg->epoch & 1u) * 8u;
        const uint64_t t_x0 = (p.flags & 1u) ? b200::globaltimer_ns() : 0;
        if (threadIdx.x < xg->nranks) {
          const uint32_t peer = threadIdx.x;
          st_sys_u64(xg->mailbox[peer] + (slot_base + xg->rank) * 8ull,
                     (static_cast<uint64_t>(xg->epoch) << 32) | __float_as_uint(mine));
          const uint64_t src = xg->mailbox[xg->rank] + (slot_base + peer) * 8ull;
          const uint64_t t0 = b200::globaltimer_ns();
          uint64_t w = ld_sys_u64(src);
          while (static_cast<uint32_t>(w >> 32) != xg->epoch) {
            if (b200::globaltimer_ns() - t0 > 4000000000ull) asm volatile("trap;");  // a peer never arrived: fail loudly
            w = ld_sys_u64(src);
          }
          s_peer[peer] = __uint_as_float(static_cast<uint32_t>(w));
        }
        __syncwarp();
        if (threadIdx.x == 0) {
          double total = 0.0;
          for (uint32_t r = 0; r < xg->nranks; ++r) total += static_cast<double>(s_peer[r]);  // same order on every rank
          reinterpret_cast<float*>(p.out)[0] = static_cast<float>(total);
          *ticket = 0;
          if (p.flags & 1u) {
            uint64_t* dbg = reinterpret_cast<uint64_t*>(p.ws + kWsDebugOffset);
            const uint64_t now = b200::globaltimer_ns();
            dbg[0] = now - t_x0;     // exchange: publish -> every peer's value seen
            dbg[1] = t_x0 - t_stage; // reading the partials + f64 tree
          }
        }
      }
    }
  } else {
    float f = ValOp<OP>::identity();
    for (uint32_t i = threadIdx.x; i < gridDim.x; i += blockDim.x) f = ValOp<OP>::apply(f, __ldcg(partials + i));
    f = block_reduce<OP>(f, s_red);
    if (threadIdx.x == 0) {
      reinterpret_cast<float*>(p.out)[0] = f * p.scale;
      *ticket = 0;
    }
  }
}

template <bool XGPU>
__device__ __forceinline__ void grid_stage_arg(const ReduceParams& p, uint64_t block_pair, uint64_t* s_red64, const XgpuParams* xg) {
  __shared__ bool s_last;
  uint64_t* partials = reinterpret_cast<uint64_t*>(p.ws + kWsIdxOffset);
  unsigned int* ticket = reinterpret_cast<unsigned int*>(p.ws + kWsTicketOffset);
  pdl_wait();
  if (threadIdx.x == 0) {
    partials[blockIdx.x] = block_pair;
    __threadfence();
    s_last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  uint64_t v = 0;
  for (uint32_t k = threadIdx.x; k < gridDim.x; k += blockDim.x) v = umax64(v, __ldcg(partials + k));
  v = block_max64(v, s_red64);
  if constexpr (!XGPU) {
    if (threadIdx.x == 0) {
      reinterpret_cast<uint32_t*>(p.out)[0] = arg_index(v);
      *ticket = 0;
    }
  } else if (threadIdx.x < 32) {
    // ---- fused (key, index) exchange: NCCL has no arg-reduce; every rank publishes its pair, then takes the max of the
    // packed pairs with GLOBAL indices (same tie rule: lowest global index), so all ranks agree.  Indices must fit 32 bits.
    __shared__ uint64_t s_pp[8];
    v = __shfl_sync(0xffffffffu, v, 0);
    const uint32_t key = static_cast<uint32_t>(v >> 32);
    const uint32_t gi = arg_index(v) + static_cast<uint32_t>(xg->index_offset);
    const uint32_t slot_base = (xg->epoch & 1u) * 8u;
    const uint64_t tag = static_cast<uint64_t>(xg->epoch) << 32;
    if (threadIdx.x < xg->nranks) {
      const uint32_t peer = threadIdx.x;
      st_sys_u64(xg->mailbox[peer] + (slot_base + xg->rank) * 8ull, tag | key);
      st_sys_u64(xg->mailbox[peer] + kMailboxIndexOffset + (slot_base + xg->rank) * 8ull, tag | gi);
      const uint64_t src = xg->mailbox[xg->rank] + (slot_base + peer) * 8ull;
      const uint64_t t0 = b200::globaltimer_ns();
      uint64_t w0 = ld_sys_u64(src), w1 = ld_sys_u64(src + kMailboxIndexOffset);
      while (static_cast<uint32_t>(w0 >> 32) != xg->epoch || static_cast<uint32_t>(w1 >> 32) != xg->epoch) {
        if (b200::globaltimer_ns() - t0 > 4000000000ull) asm volatile("trap;");
        w0 = ld_sys_u64(src);
        w1 = ld_sys_u64(src + kMailboxIndexOffset);
      }
      s_pp[peer] = arg_pack(static_cast<uint32_t>(w0), static_cast<uint32_t>(w1));
    }
    __syncwarp();
    if (threadIdx.x == 0) {
      uint64_t best = 0;
      for (uint32_t r = 0; r < xg->nranks; ++r) best = umax64(best, s_pp[r]);
      reinterpret_cast<uint32_t*>(p.out)[0] = arg_index(best);
      *ticket = 0;
    }
  }
}

// ================================================================================================ reduce over ALL elements (contiguous)
// Grid-stride over 128-bit (VEC elements) vectors, UNROLL independent loads in flight per thread, one accumulator per
// load slot and vector lane (value ops) or one running (key, index) candidate fed in increasing index order (arg ops).
// A base that is not 16-byte (WIDE: 32-byte) aligned -- a sub-slice view, Handle::offset -- is handled by peeling a scalar
// head up to the next boundary, never by issuing a misaligned vector load.
template <int OP, int DT, int UNROLL, bool WIDE /* 256-bit loads, f32 only */, bool XGPU = false, bool BLOCKED = false>
__device__ __forceinline__ void reduce_all_body(const ReduceParams& p, const XgpuParams* xg = nullptr) {
  using E = Elem<DT>;
  using T = typename E::T;
  constexpr bool ARG = (OP >= OP_ARGMAX);
  constexpr int VEC = WIDE ? 8 : E::VEC;
  constexpr uint32_t ALIGN = WIDE ? 32u : 16u;
  __shared__ float s_red[kMaxWarps];
  __shared__ uint64_t s_red64[kMaxWarps];
  // Let a dependent launch begin right away: it only streams its own input until its griddepcontrol.wait, so its blocks take
  // over SM slots as this grid's blocks retire and the two kernels' ramp / tail overlap completely (every block of this grid
  // is resident or done by the time the dependent may launch, so the dependent can never starve it).
  pdl_trigger();

  const uint64_t n = p.len;
  const uint32_t mis = static_cast<uint32_t>(p.in) & (ALIGN - 1u);
  uint64_t head = mis ? (ALIGN - mis) / sizeof(T) : 0;
  if (head > n) head = n;
  const uint64_t nb = n - head, nvec = nb / VEC;
  const uint64_t tid = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const uint64_t nthreads = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  const char* base0 = reinterpret_cast<const char*>(p.in);
  const char* base = base0 + head * sizeof(T);

  float acc[UNROLL][VEC];
#pragma unroll
  for (int u = 0; u < UNROLL; ++u)
#pragma unroll
    for (int j = 0; j < VEC; ++j) acc[u][j] = ValOp<OP>::identity();
  ArgAcc cand;
  float local = ValOp<OP>::identity();
  auto feed = [&](int u, int j, float f, uint64_t idx) {
    if constexpr (ARG) cand.feed<OP>(f, static_cast<uint32_t>(idx));
    else acc[u][j] = ValOp<OP>::apply(acc[u][j], f);
  };

  // head: the elements in front of the first aligned vector (lowest indices, so they are fed first)
  if (tid < head) {
    const float f = E::get(base0, tid);
    if constexpr (ARG) cand.feed<OP>(f, static_cast<uint32_t>(tid));
    else local = ValOp<OP>::apply(local, f);
  }

  uint64_t v = tid;
  if constexpr (BLOCKED) {
    // tile = blockDim * UNROLL consecutive vectors (64 KB for 512 threads x 8 x 16 B), tiles dealt round-robin to blocks:
    // at any instant the whole grid reads ONE contiguous window instead of UNROLL windows nthreads apart
    const uint64_t tile = static_cast<uint64_t>(blockDim.x) * UNROLL;
    const uint64_t ntiles = nvec / tile;
    for (uint64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
      const uint64_t base_v = t * tile + threadIdx.x;
      uint4 r[UNROLL];
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) r[u] = ldg_stream_u4(base + (base_v + static_cast<uint64_t>(u) * blockDim.x) * 16);
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        float f[E::VEC];
        E::unpack(r[u], f);
#pragma unroll
        for (int j = 0; j < E::VEC; ++j) feed(u, j, f[j], head + (base_v + static_cast<uint64_t>(u) * blockDim.x) * VEC + j);
      }
    }
    v = ntiles * tile + tid;  // leftover vectors: grid-stride below
  } else {
    // main: UNROLL vectors per thread per trip, all loads issued before any use.  Addresses come from ONE running pointer
    // advanced by the grid stride (two live registers instead of UNROLL precomputed 64-bit offsets -- those spilled).
    const uint64_t cnt = (nvec > tid) ? (nvec - 1 - tid) / nthreads + 1 : 0;  // vectors this thread owns
    const uint64_t stride = nthreads * (VEC * sizeof(T));
    const char* ptr = base + tid * (VEC * sizeof(T));
    uint32_t idx32 = static_cast<uint32_t>(head + tid * VEC);   // arg ops only (n < 2^32 there)
    const uint32_t istep = static_cast<uint32_t>(nthreads * VEC);
    for (uint64_t trip = cnt / UNROLL; trip > 0; --trip) {
      if constexpr (WIDE) {
        float8 r[UNROLL];
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) { r[u] = ldg_stream_v8(reinterpret_cast<const float*>(ptr)); ptr += stride; }
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
          acc[u][0] = ValOp<OP>::apply(acc[u][0], r[u].lo.x); acc[u][1] = ValOp<OP>::apply(acc[u][1], r[u].lo.y);
          acc[u][2] = ValOp<OP>::apply(acc[u][2], r[u].lo.z); acc[u][3] = ValOp<OP>::apply(acc[u][3], r[u].lo.w);
          acc[u][4] = ValOp<OP>::apply(acc[u][4], r[u].hi.x); acc[u][5] = ValOp<OP>::apply(acc[u][5], r[u].hi.y);
          acc[u][6] = ValOp<OP>::apply(acc[u][6], r[u].hi.z); acc[u][7] = ValOp<OP>::apply(acc[u][7], r[u].hi.w);
        }
      } else {
        uint4 r[UNROLL];
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) { r[u] = ldg_stream_u4(ptr); ptr += stride; }
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
          float f[E::VEC];
          E::unpack(r[u], f);
#pragma unroll
          for (int j = 0; j < E::VEC; ++j) feed(u, j, f[j], idx32 + j);
          idx32 += istep;
        }
      }
    }
    // remaining whole vectors (fewer than UNROLL)
    for (uint32_t k = static_cast<uint32_t>(cnt % UNROLL); k > 0; --k) {
      if constexpr (WIDE) {
        float8 r = ldg_stream_v8(reinterpret_cast<const float*>(ptr));
        acc[0][0] = ValOp<OP>::apply(acc[0][0], r.lo.x); acc[0][1] = ValOp<OP>::apply(acc[0][1], r.lo.y);
        acc[0][2] = ValOp<OP>::apply(acc[0][2], r.lo.z); acc[0][3] = ValOp<OP>::apply(acc[0][3], r.lo.w);
        acc[0][4] = ValOp<OP>::apply(acc[0][4], r.hi.x); acc[0][5] = ValOp<OP>::apply(acc[0][5], r.hi.y);
        acc[0][6] = ValOp<OP>::apply(acc[0][6], r.hi.z); acc[0][7] = ValOp<OP>::apply(acc[0][7], r.hi.w);
      } else {
        float f[E::VEC];
        E::unpack(ldg_stream_u4(ptr), f);
#pragma unroll
        for (int j = 0; j < E::VEC; ++j) feed(0, j, f[j], idx32 + j);
        idx32 += istep;
      }
      ptr += stride;
    }
    v = nvec;  // nothing left for the shared leftover loop below
  }
  // leftover whole vectors of the BLOCKED form
  for (; v < nvec; v += nthreads) {
    float f[E::VEC];
    E::unpack(ldg_stream_u4(base + v * 16), f);
#pragma unroll
    for (int j = 0; j < E::VEC; ++j) feed(0, j, f[j], head + v * VEC + j);
  }
  // scalar tail (nb % VEC elements)
  for (uint64_t i = nvec * VEC + tid; i < nb; i += nthreads) {
    const float f = E::get(base, i);
    if constexpr (ARG) cand.feed<OP>(f, static_cast<uint32_t>(head + i));
    else local = ValOp<OP>::apply(local, f);
  }

  if constexpr (ARG) {
    const uint64_t block_pair = block_max64(cand.packed(), s_red64);
    grid_stage_arg<XGPU>(p, block_pair, s_red64, xg);
  } else {
#pragma unroll
    for (int u = 0; u < UNROLL; ++u)
#pragma unroll
      for (int j = 0; j < VEC; ++j) local = ValOp<OP>::apply(local, acc[u][j]);
    const float block_val = block_reduce<OP>(local, s_red);
    grid_stage_value<OP, XGPU>(p, block_val, s_red, xg);
  }
}

// ================================================================================================ reduce over ALL elements: bulk-copy staged
// The same reduction with the HBM stream moved by the TMA unit: one producer thread issues 16 KB cp.async.bulk copies
// (evict_first) into a ring of shared-memory stages, eight consumer warps read their 128-bit slices back from shared memory
// and accumulate.  One CTA per SM, tiles dealt round-robin over the grid, so at any instant the grid reads ONE contiguous
// window of gridDim x 16 KB x (stages in flight); no register is spent on loads in flight and no address arithmetic per
// 16 bytes.  Head (unaligned base) and tail (< one tile) elements go through plain loads.
constexpr int kBulkStages = 8;       // at most; the launch picks the ring depth (ReduceParams::ctu): 8 = one CTA per SM,
                                     // <= 6 lets two CTAs share an SM (the next launch's CTA can start under PDL)

template <int OP, int DT>
__device__ __forceinline__ void reduce_all_bulk_body(const ReduceParams& p) {
  using E = Elem<DT>;
  using T = typename E::T;
  constexpr int VEC = E::VEC;
  constexpr int PER = kBulkStageBytes / 16 / kBulkConsumers;  // 128-bit slices per consumer per stage (4)
  extern __shared__ uint8_t bulk_smem_raw[];
  __shared__ float s_red[kMaxWarps];
  __shared__ uint64_t s_bars[2 * kBulkStages];
  const uint32_t ring = (b200::smem_u32(bulk_smem_raw) + 127u) & ~127u;
  const uint32_t full0 = b200::smem_u32(s_bars), empty0 = full0 + 8u * kBulkStages;
  const uint32_t stages = (p.ctu >= 2 && p.ctu <= static_cast<uint32_t>(kBulkStages)) ? p.ctu : static_cast<uint32_t>(kBulkStages);

  const uint64_t n = p.len;
  const uint32_t mis = static_cast<uint32_t>(p.in) & 15u;
  uint64_t head = mis ? (16u - mis) / sizeof(T) : 0;
  if (head > n) head = n;
  const char* base0 = reinterpret_cast<const char*>(p.in);
  const char* base = base0 + head * sizeof(T);
  const uint64_t nb = n - head;
  constexpr uint64_t TILE_ELEMS = kBulkStageBytes / sizeof(T);
  const uint64_t ntiles = nb / TILE_ELEMS;

  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (uint32_t s = 0; s < stages; ++s) {
      b200::mbar_init(full0 + 8u * s, 1);
      b200::mbar_init(empty0 + 8u * s, kBulkConsumers / 32);
    }
    b200::fence_mbar_init();
  }
  __syncthreads();
  pdl_trigger();   // see reduce_all_body: a dependent launch may start streaming beside this one

  float local = ValOp<OP>::identity();
  if (warp == kBulkConsumers / 32) {
    // ------------------------------------------------------------------ producer (one lane)
    if (lane == 0) {
      const uint64_t pol = b200::l2_policy_evict_first();
      uint32_t s = 0, ph = 0;
      for (uint64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        b200::mbar_wait(empty0 + 8u * s, ph ^ 1u);
        b200::mbar_arrive_expect_tx(full0 + 8u * s, kBulkStageBytes);
        b200::bulk_load_1d(ring + s * kBulkStageBytes, base + t * kBulkStageBytes, kBulkStageBytes, full0 + 8u * s, pol);
        if (++s == stages) { s = 0; ph ^= 1u; }
      }
    }
    __syncwarp();
  } else {
    // ------------------------------------------------------------------ consumers
    float acc[PER][VEC];
#pragma unroll
    for (int u = 0; u < PER; ++u)
#pragma unroll
      for (int j = 0; j < VEC; ++j) acc[u][j] = ValOp<OP>::identity();
    uint32_t s = 0, ph = 0;
    for (uint64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
      b200::mbar_wait(full0 + 8u * s, ph);
      const uint32_t src = ring + s * kBulkStageBytes + threadIdx.x * 16u;
      uint4 r[PER];
#pragma unroll
      for (int u = 0; u < PER; ++u)
        asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r[u].x), "=r"(r[u].y), "=r"(r[u].z), "=r"(r[u].w) : "r"(src + u * (kBulkConsumers * 16u)));
#pragma unroll
      for (int u = 0; u < PER; ++u) {
        float f[VEC];
        E::unpack(r[u], f);
#pragma unroll
        for (int j = 0; j < VEC; ++j) acc[u][j] = ValOp<OP>::apply(acc[u][j], f[j]);
      }
      __syncwarp();
      if (lane == 0) b200::mbar_arrive(empty0 + 8u * s);  // every lane has consumed its slices: the stage may be refilled
      if (++s == stages) { s = 0; ph ^= 1u; }
    }
    // head + tail through plain loads, spread over the consumers of the whole grid
    const uint64_t ctid = static_cast<uint64_t>(blockIdx.x) * kBulkConsumers + threadIdx.x;
    const uint64_t cthreads = static_cast<uint64_t>(gridDim.x) * kBulkConsumers;
    if (ctid < head) local = ValOp<OP>::apply(local, E::get(base0, ctid));
    for (uint64_t i = ntiles * TILE_ELEMS + ctid; i < nb; i += cthreads) local = ValOp<OP>::apply(local, E::get(base, i));
#pragma unroll
    for (int u = 0; u < PER; ++u)
#pragma unroll
      for (int j = 0; j < VEC; ++j) local = ValOp<OP>::apply(local, acc[u][j]);
  }
  const float block_val = block_reduce<OP>(local, s_red);
  grid_stage_value<OP, false>(p, block_val, s_red, nullptr);
}

// ================================================================================================ reduce over ALL elements of a pitched view
// Logical rows of `row_len` elements, `row_pitch` elements apart (PitchedMemoryLayoutPolicy: the padding is never read).
// A thread walks units (one 128-bit vector when row length, pitch and base allow it, one element otherwise) w = tid,
// tid + nthreads, ...; the (row, column) position is advanced incrementally, four loads in flight.
template <int OP, int DT, bool VECTOR>
__device__ __forceinline__ void all_pitched_walk(const ReduceParams& p, float& local, ArgAcc& cand) {
  using E = Elem<DT>;
  using T = typename E::T;
  constexpr bool ARG = (OP >= OP_ARGMAX);
  constexpr int UV = VECTOR ? E::VEC : 1;
  const uint64_t upr = p.row_len / UV;                 // units per row
  const uint64_t total = (p.len / p.row_len) * upr;    // len = rows * row_len
  const uint64_t tid = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const uint64_t nthreads = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  const uint64_t dr = nthreads / upr, dc = nthreads - dr * upr;
  uint64_t w = tid, r = tid / upr, c = tid - r * upr;
  const char* base = reinterpret_cast<const char*>(p.in);
  float a[4] = {ValOp<OP>::identity(), ValOp<OP>::identity(), ValOp<OP>::identity(), ValOp<OP>::identity()};
  while (w < total) {
    uint4 q[4];
    float sc[4];
    uint64_t wi[4];
    bool ok[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      ok[u] = w < total;
      wi[u] = w;
      if (ok[u]) {
        const uint64_t off = r * p.row_pitch + c * UV;
        if constexpr (VECTOR) q[u] = ldg_stream_u4(base + off * sizeof(T));
        else sc[u] = E::get(base, off);
      }
      w += nthreads; c += dc; r += dr;
      if (c >= upr) { c -= upr; ++r; }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (!ok[u]) continue;
      if constexpr (VECTOR) {
        float f[E::VEC];
        E::unpack(q[u], f);
#pragma unroll
        for (int j = 0; j < E::VEC; ++j) {
          if constexpr (ARG) cand.feed<OP>(f[j], static_cast<uint32_t>(wi[u] * UV + j));
          else a[u] = ValOp<OP>::apply(a[u], f[j]);
        }
      } else {
        if constexpr (ARG) cand.feed<OP>(sc[u], static_cast<uint32_t>(wi[u]));
        else a[u] = ValOp<OP>::apply(a[u], sc[u]);
      }
    }
  }
  if constexpr (!ARG) local = ValOp<OP>::apply(ValOp<OP>::apply(a[0], a[1]), ValOp<OP>::apply(a[2], a[3]));
}

template <int OP, int DT>
__device__ __forceinline__ void reduce_all_pitched_body(const ReduceParams& p) {
  using E = Elem<DT>;
  using T = typename E::T;
  constexpr bool ARG = (OP >= OP_ARGMAX);
  __shared__ float s_red[kMaxWarps];
  __shared__ uint64_t s_red64[kMaxWarps];
  float local = ValOp<OP>::identity();
  ArgAcc cand;
  const bool vec_ok = (p.row_len % E::VEC) == 0 && ((p.row_pitch * sizeof(T)) % 16) == 0 && (p.in % 16) == 0;
  if (vec_ok) all_pitched_walk<OP, DT, true>(p, local, cand);
  else all_pitched_walk<OP, DT, false>(p, local, cand);
  if constexpr (ARG) {
    const uint64_t block_pair = block_max64(cand.packed(), s_red64);
    grid_stage_arg<false>(p, block_pair, s_red64, nullptr);
  } else {
    const float block_val = block_reduce<OP>(local, s_red);
    grid_stage_value<OP, false>(p, block_val, s_red, nullptr);
  }
}

// ================================================================================================ rows: reduce the innermost axis
// Work items q in [0, outer * nseg): row o = q / nseg, segment s = q % nseg of the axis ([s * seg_len, min(len, ..+seg_len))),
// element l of the item at in + o * s_outer + s * seg_len + l.  gridDim.x blocks walk the items; `blockDim.x / TPR` items per
// block pass, TPR threads per item (TPR <= 32: a sub-warp per item, TPR = blockDim: a block per item).  128-bit loads on
// the 16-byte aligned body of every item, scalar head / tail around it (any base, pitch or segment alignment).
template <int OP, int DT>
__device__ __forceinline__ void rows_store(const ReduceParams& p, uint64_t q, uint64_t l0, float value, uint64_t pair) {
  constexpr bool ARG = (OP >= OP_ARGMAX);
  if constexpr (!ARG) {
    reinterpret_cast<float*>(p.out)[q] = value * p.scale;
  } else if (p.out2 == 0) {
    reinterpret_cast<uint32_t*>(p.out)[q] = arg_index(pair);
  } else {  // split pass: key and index along the WHOLE axis, combined by argcombine
    reinterpret_cast<uint32_t*>(p.out)[q] = static_cast<uint32_t>(pair >> 32);
    reinterpret_cast<uint32_t*>(p.out2)[q] = arg_index(pair) + static_cast<uint32_t>(l0);
  }
}

template <int OP, int DT>
__device__ __forceinline__ void reduce_rows_body(const ReduceParams& p, int tpr_log2) {
  using E = Elem<DT>;
  using T = typename E::T;
  constexpr bool ARG = (OP >= OP_ARGMAX);
  constexpr int VEC = E::VEC;
  __shared__ float s_red[kMaxWarps];
  __shared__ uint64_t s_red64[kMaxWarps];
  pdl_wait();   // second pass of a split reduction: wait for the first pass's partials (no-op otherwise)
  const uint32_t tpr = 1u << tpr_log2;
  const uint32_t rows_per_block = blockDim.x >> tpr_log2;
  const uint32_t sub = threadIdx.x >> tpr_log2;  // which item of this block pass
  const uint32_t t = threadIdx.x & (tpr - 1);
  const char* base = reinterpret_cast<const char*>(p.in);
  const uint64_t items = p.outer * p.nseg;
  const uint64_t rstride = static_cast<uint64_t>(gridDim.x) * rows_per_block;

  // every item starts on a 16-byte boundary and is a whole number of vectors (the common, unpitched or well-pitched case)
  const bool uniform = (p.in % 16) == 0 && ((p.s_outer * sizeof(T)) % 16) == 0 && (p.len % VEC) == 0 &&
                       (p.nseg == 1 || (p.seg_len % VEC) == 0);
  if (tpr <= 32 && uniform && p.nseg == 1 && p.len / VEC <= tpr) {
    // short rows (at most one 128-bit vector per thread): 4 independent rows in flight per thread group, so the loads of
    // consecutive rows overlap instead of serialising behind each row's shuffle tree
    const uint64_t nvec = p.len / VEC;
    for (uint64_t row0 = static_cast<uint64_t>(blockIdx.x) * rows_per_block; row0 < items; row0 += 4 * rstride) {
      uint4 q[4];
      bool ok[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint64_t row = row0 + j * rstride + sub;
        ok[j] = row < items && t < nvec;
        if (ok[j]) q[j] = ldg_stream_u4(base + (row * p.s_outer + static_cast<uint64_t>(t) * VEC) * sizeof(T));
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float r = ValOp<OP>::identity();
        ArgAcc cand;
        if (ok[j]) {
          float f[VEC];
          E::unpack(q[j], f);
#pragma unroll
          for (int e = 0; e < VEC; ++e) {
            if constexpr (ARG) cand.feed<OP>(f[e], t * VEC + e);
            else r = ValOp<OP>::apply(r, f[e]);
          }
        }
        uint64_t pr = cand.packed();
        for (uint32_t o = tpr >> 1; o > 0; o >>= 1) {
          if constexpr (ARG) pr = umax64(pr, __shfl_down_sync(0xffffffffu, pr, o));
          else r = ValOp<OP>::apply(r, __shfl_down_sync(0xffffffffu, r, o));
        }
        const uint64_t row = row0 + j * rstride + sub;
        if (t == 0 && row < items) rows_store<OP, DT>(p, row, 0, r, pr);
      }
    }
    return;
  }

  for (uint64_t row0 = static_cast<uint64_t>(blockIdx.x) * rows_per_block; row0 < items; row0 += rstride) {
    const uint64_t q = row0 + sub;
    float a0 = ValOp<OP>::identity(), a1 = a0, a2 = a0, a3 = a0;
    ArgAcc cand;
    uint64_t l0 = 0;
    if (q < items) {
      const uint64_t o = q / p.nseg, s = q - o * p.nseg;
      l0 = s * p.seg_len;
      const uint64_t L = (p.len - l0 < p.seg_len) ? p.len - l0 : p.seg_len;
      const char* rb = base + (o * p.s_outer + l0) * sizeof(T);
      // scalar head up to the next 16-byte boundary, vector body, scalar tail
      const uint32_t mis = static_cast<uint32_t>(reinterpret_cast<uint64_t>(rb)) & 15u;
      uint64_t head = mis ? (16u - mis) / sizeof(T) : 0;
      if (head > L) head = L;
      const uint64_t nvec = (L - head) / VEC;
      const char* vb = rb + head * sizeof(T);
      for (uint64_t i = t; i < head; i += tpr) {   // up to VEC - 1 head elements, possibly more than the item has threads
        const float f = E::get(rb, i);
        if constexpr (ARG) cand.feed<OP>(f, static_cast<uint32_t>(i));
        else a1 = ValOp<OP>::apply(a1, f);
      }
      uint64_t v = t;
      for (; v + 3ull * tpr < nvec; v += 4ull * tpr) {
        uint4 r0 = ldg_stream_u4(vb + (v)*16);
        uint4 r1 = ldg_stream_u4(vb + (v + tpr) * 16);
        uint4 r2 = ldg_stream_u4(vb + (v + 2ull * tpr) * 16);
        uint4 r3 = ldg_stream_u4(vb + (v + 3ull * tpr) * 16);
        float f0[VEC], f1[VEC], f2[VEC], f3[VEC];
        E::unpack(r0, f0); E::unpack(r1, f1); E::unpack(r2, f2); E::unpack(r3, f3);
        if constexpr (ARG) {
          const uint32_t i0 = static_cast<uint32_t>(head + v * VEC), st = tpr * VEC;
#pragma unroll
          for (int j = 0; j < VEC; ++j) cand.feed<OP>(f0[j], i0 + j);
#pragma unroll
          for (int j = 0; j < VEC; ++j) cand.feed<OP>(f1[j], i0 + st + j);
#pragma unroll
          for (int j = 0; j < VEC; ++j) cand.feed<OP>(f2[j], i0 + 2 * st + j);
#pragma unroll
          for (int j = 0; j < VEC; ++j) cand.feed<OP>(f3[j], i0 + 3 * st + j);
        } else {
#pragma unroll
          for (int j = 0; j < VEC; ++j) {
            a0 = ValOp<OP>::apply(a0, f0[j]); a1 = ValOp<OP>::apply(a1, f1[j]);
            a2 = ValOp<OP>::apply(a2, f2[j]); a3 = ValOp<OP>::apply(a3, f3[j]);
          }
        }
      }
      for (; v < nvec; v += tpr) {
        float f[VEC];
        E::unpack(ldg_stream_u4(vb + v * 16), f);
#pragma unroll
        for (int j = 0; j < VEC; ++j) {
          if constexpr (ARG) cand.feed<OP>(f[j], static_cast<uint32_t>(head + v * VEC + j));
          else a0 = ValOp<OP>::apply(a0, f[j]);
        }
      }
      for (uint64_t i = head + nvec * VEC + t; i < L; i += tpr) {
        const float f = E::get(rb, i);
        if constexpr (ARG) cand.feed<OP>(f, static_cast<uint32_t>(i));
        else a1 = ValOp<OP>::apply(a1, f);
      }
    }
    float r = ValOp<OP>::apply(ValOp<OP>::apply(a0, a1), ValOp<OP>::apply(a2, a3));
    uint64_t pr = cand.packed();
    if (tpr <= 32) {
      // sub-warp tree: items never straddle a warp because tpr divides 32
      for (uint32_t o = tpr >> 1; o > 0; o >>= 1) {
        if constexpr (ARG) pr = umax64(pr, __shfl_down_sync(0xffffffffu, pr, o));
        else r = ValOp<OP>::apply(r, __shfl_down_sync(0xffffffffu, r, o));
      }
      if (t == 0 && q < items) rows_store<OP, DT>(p, q, l0, r, pr);
    } else {
      // tpr / 32 whole warps per item (tpr == blockDim.x: one item per block): warp trees, then the item's first thread adds
      // its warps' partials in warp order
      const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wpr = tpr >> 5;
      if constexpr (ARG) { pr = warp_max64(pr); if (lane == 0) s_red64[warp] = pr; }
      else { r = warp_reduce<OP>(r); if (lane == 0) s_red[warp] = r; }
      __syncthreads();
      if (t == 0 && q < items) {
        for (uint32_t w = 1; w < wpr; ++w) {
          if constexpr (ARG) pr = umax64(pr, s_red64[warp + w]);
          else r = ValOp<OP>::apply(r, s_red[warp + w]);
        }
        rows_store<OP, DT>(p, q, l0, r, pr);
      }
      __syncthreads();  // the partial slots are reused by the next pass
    }
  }
}

// ================================================================================================ columns: reduce an outer / middle axis
// View [outer, len, inner], inner > 1.  A block tile is `ctu` column UNITS (a unit = one 128-bit vector of consecutive inner
// elements when the layout allows it, else one element) x RL = blockDim / ctu row lanes: thread (rl, cu) walks rows
// l = rl, rl + RL, ... of its unit, four loads in flight, consecutive threads on consecutive units (coalesced); the RL
// partial results per unit are combined through shared memory.  Work items = (outer x segment) x tiles over the grid.
// Few columns with a long axis: small ctu -> many row lanes.  Many columns with a short axis: ctu = blockDim, one row lane.
template <int OP, int DT, bool VECTOR, int NL /* loads in flight per thread */>
__device__ __forceinline__ void reduce_cols_tiles(const ReduceParams& p, uint64_t* s_raw) {
  using E = Elem<DT>;
  using T = typename E::T;
  constexpr bool ARG = (OP >= OP_ARGMAX);
  constexpr int UV = VECTOR ? E::VEC : 1;
  float* s_val = reinterpret_cast<float*>(s_raw);
  const uint64_t units = p.inner / UV;
  const uint32_t ctu = p.ctu;
  const uint32_t RL = kColsThreads / ctu;
  const uint32_t rl = threadIdx.x / ctu, cu = threadIdx.x - rl * ctu;
  const bool active = rl < RL;
  const uint64_t tiles = (units + ctu - 1) / ctu;
  const uint64_t items = p.outer * p.nseg * tiles;
  const char* base = reinterpret_cast<const char*>(p.in);
  uint32_t tree0 = 1;
  while (tree0 < RL) tree0 <<= 1;
  tree0 >>= 1;

  for (uint64_t item = blockIdx.x; item < items; item += gridDim.x) {
    const uint64_t q = item / tiles, tile = item - q * tiles;
    const uint64_t o = q / p.nseg, s = q - o * p.nseg;
    const uint64_t l0 = s * p.seg_len;
    const uint64_t L = (p.len - l0 < p.seg_len) ? p.len - l0 : p.seg_len;
    const uint64_t unit = tile * ctu + cu;
    const bool valid = active && unit < units;
    const uint64_t i0 = unit * UV;
    uint64_t ioff = i0;
    if (p.row_len != p.inner) { const uint64_t rr = i0 / p.row_len; ioff = rr * p.row_pitch + (i0 - rr * p.row_len); }
    const char* cb = base + (o * p.s_outer + l0 * p.s_len + ioff) * sizeof(T);
    const uint64_t lstep = p.s_len * sizeof(T);

    // NL loads in flight per thread, folded into four accumulator sets
    float a[4][UV];
    ArgAcc cand[UV];
#pragma unroll
    for (int u = 0; u < 4; ++u)
#pragma unroll
      for (int j = 0; j < UV; ++j) a[u][j] = ValOp<OP>::identity();
    if (valid) {
      uint64_t l = rl;
      for (; l + static_cast<uint64_t>(NL - 1) * RL < L; l += static_cast<uint64_t>(NL) * RL) {
        float f[NL][UV];
        if constexpr (VECTOR) {
          uint4 r[NL];
#pragma unroll
          for (int u = 0; u < NL; ++u) r[u] = ldg_stream_u4(cb + (l + static_cast<uint64_t>(u) * RL) * lstep);
#pragma unroll
          for (int u = 0; u < NL; ++u) E::unpack(r[u], f[u]);
        } else {
#pragma unroll
          for (int u = 0; u < NL; ++u) f[u][0] = E::get(cb + (l + static_cast<uint64_t>(u) * RL) * lstep, 0);
        }
#pragma unroll
        for (int u = 0; u < NL; ++u)
#pragma unroll
          for (int j = 0; j < UV; ++j) {
            if constexpr (ARG) cand[j].feed<OP>(f[u][j], static_cast<uint32_t>(l0 + l + static_cast<uint64_t>(u) * RL));
            else a[u & 3][j] = ValOp<OP>::apply(a[u & 3][j], f[u][j]);
          }
      }
      for (; l < L; l += RL) {
        float f[UV];
        if constexpr (VECTOR) E::unpack(ldg_stream_u4(cb + l * lstep), f);
        else f[0] = E::get(cb + l * lstep, 0);
#pragma unroll
        for (int j = 0; j < UV; ++j) {
          if constexpr (ARG) cand[j].feed<OP>(f[j], static_cast<uint32_t>(l0 + l));
          else a[0][j] = ValOp<OP>::apply(a[0][j], f[j]);
        }
      }
    }
    float res[UV];
    uint64_t resp[UV];
#pragma unroll
    for (int j = 0; j < UV; ++j) {
      res[j] = ValOp<OP>::apply(ValOp<OP>::apply(a[0][j], a[1][j]), ValOp<OP>::apply(a[2][j], a[3][j]));
      resp[j] = cand[j].packed();
    }
    // combine the row lanes of each unit through shared memory: slot (rl, cu) at [threadIdx.x * UV + j]; lanes that found
    // nothing hold the identity.  The result is valid in the lanes with rl == 0.  (block-uniform control flow)
    auto combine_lanes = [&]() {
      if (RL <= 1) return;
#pragma unroll
      for (int j = 0; j < UV; ++j) {
        if constexpr (ARG) s_raw[threadIdx.x * UV + j] = resp[j];
        else s_val[threadIdx.x * UV + j] = res[j];
      }
      for (uint32_t st = tree0; st >= 1; st >>= 1) {
        __syncthreads();
        if (active && rl < st && rl + st < RL) {
          const uint32_t other = (threadIdx.x + st * ctu) * UV;
#pragma unroll
          for (int j = 0; j < UV; ++j) {
            if constexpr (ARG) s_raw[threadIdx.x * UV + j] = umax64(s_raw[threadIdx.x * UV + j], s_raw[other + j]);
            else s_val[threadIdx.x * UV + j] = ValOp<OP>::apply(s_val[threadIdx.x * UV + j], s_val[other + j]);
          }
        }
      }
      if (rl == 0) {
#pragma unroll
        for (int j = 0; j < UV; ++j) {
          if constexpr (ARG) resp[j] = s_raw[threadIdx.x * UV + j];
          else res[j] = s_val[threadIdx.x * UV + j];
        }
      }
      __syncthreads();  // the slots are reused (next combine / next item)
    };
    combine_lanes();
    const bool fused = (p.flags & 4u) != 0;
    if (valid && rl == 0) {
      const uint64_t ob = q * p.inner + i0;
#pragma unroll
      for (int j = 0; j < UV; ++j) {
        if constexpr (!ARG) {
          reinterpret_cast<float*>(p.out)[ob + j] = fused ? res[j] : res[j] * p.scale;
        } else if (p.out2 == 0) {
          reinterpret_cast<uint32_t*>(p.out)[ob + j] = arg_index(resp[j]);
        } else {
          reinterpret_cast<uint32_t*>(p.out)[ob + j] = static_cast<uint32_t>(resp[j] >> 32);
          reinterpret_cast<uint32_t*>(p.out2)[ob + j] = arg_index(resp[j]);  // already global along the axis (l0 + l was fed)
        }
      }
    }
    if (fused) {
      // Fused finish of a split reduction: every block publishes its segment's partials, takes a ticket for its (outer,
      // column tile); whoever completes the set re-reads all nseg partial rows of the tile -- each row lane a fixed subset of
      // the segments, then the same lane tree -- so the result does not depend on which block came last.  No second launch.
      __shared__ uint32_t s_last;
      __syncthreads();            // the row-lane-0 threads have stored the partials ...
      if (threadIdx.x == 0) {
        __threadfence();          // ... and this (cumulative) fence publishes them before the ticket
        unsigned int* ticket = reinterpret_cast<unsigned int*>(p.ws + kWsColTicketOffset) + (o * tiles + tile);
        const unsigned int old = atomicAdd(ticket, 1u);
        s_last = (old == p.nseg - 1) ? 1u : 0u;
        if (s_last) *ticket = 0;  // left ready for the next launch on this stream
      }
      __syncthreads();
      if (s_last) {
        __threadfence();
#pragma unroll
        for (int j = 0; j < UV; ++j) { res[j] = ValOp<OP>::identity(); resp[j] = 0; }
        if (valid) {
          for (uint64_t sg = rl; sg < p.nseg; sg += RL) {
            const uint64_t at = (o * p.nseg + sg) * p.inner + i0;
#pragma unroll
            for (int j = 0; j < UV; ++j) {
              if constexpr (ARG) resp[j] = umax64(resp[j], arg_pack(__ldcg(reinterpret_cast<const uint32_t*>(p.out) + at + j),
                                                                    __ldcg(reinterpret_cast<const uint32_t*>(p.out2) + at + j)));
              else res[j] = ValOp<OP>::apply(res[j], __ldcg(reinterpret_cast<const float*>(p.out) + at + j));
            }
          }
        }
        combine_lanes();
        if (valid && rl == 0) {
#pragma unroll
          for (int j = 0; j < UV; ++j) {
            if constexpr (ARG) reinterpret_cast<uint32_t*>(p.final_out)[o * p.inner + i0 + j] = arg_index(resp[j]);
            else reinterpret_cast<float*>(p.final_out)[o * p.inner + i0 + j] = res[j] * p.scale;
          }
        }
      }
    }
  }
}

template <int OP, int DT, int NL>
__device__ __forceinline__ void reduce_cols_body(const ReduceParams& p) {
  using E = Elem<DT>;
  using T = typename E::T;
  __shared__ uint64_t s_raw[kColsThreads * E::VEC];
  pdl_wait();   // second pass of a split reduction launched with programmatic serialization: the partials must be complete
  const uint64_t esz = sizeof(T);
  const bool vec_ok = (p.flags & 2u) != 0 &&  // the host sized ctu for vector units
                      (p.inner % E::VEC) == 0 && (p.row_len % E::VEC) == 0 && (p.in % 16) == 0 && ((p.s_len * esz) % 16) == 0 &&
                      ((p.s_outer * esz) % 16) == 0 && ((p.row_pitch * esz) % 16) == 0;
  if (vec_ok) reduce_cols_tiles<OP, DT, true, NL>(p, s_raw);
  else reduce_cols_tiles<OP, DT, false, NL>(p, s_raw);
}

// ================================================================================================ second pass of a split arg-reduction
// keys / indices [outer, nseg, inner] (u32, u32) -> indices [outer, inner]: max of the packed pairs over the segments.
extern "C" __global__ void __launch_bounds__(256) reduce_argcombine(const __grid_constant__ ArgCombineParams p) {
  const uint64_t total = p.outer * p.inner;
  const uint32_t* keys = reinterpret_cast<const uint32_t*>(p.keys);
  const uint32_t* idx = reinterpret_cast<const uint32_t*>(p.idx);
  if (p.nseg >= 8) {
    // many segments, (usually) few outputs: a warp per output, lanes over the segments (a serial walk of thousands of
    // dependent-latency loads by one thread took longer than the first pass)
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t warp = (static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const uint64_t nwarps = (static_cast<uint64_t>(gridDim.x) * blockDim.x) >> 5;
    for (uint64_t e = warp; e < total; e += nwarps) {
      const uint64_t o = e / p.inner, i = e - o * p.inner;
      uint64_t best = 0;
      for (uint64_t s = lane; s < p.nseg; s += 32) {
        const uint64_t at = (o * p.nseg + s) * p.inner + i;
        best = umax64(best, arg_pack(keys[at], idx[at]));
      }
      best = warp_max64(best);
      if (lane == 0) reinterpret_cast<uint32_t*>(p.out)[e] = arg_index(best);
    }
    return;
  }
  for (uint64_t e = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; e < total;
       e += static_cast<uint64_t>(gridDim.x) * blockDim.x) {
    const uint64_t o = e / p.inner, i = e - o * p.inner;
    uint64_t best = 0;
    for (uint64_t s = 0; s < p.nseg; ++s) {
      const uint64_t at = (o * p.nseg + s) * p.inner + i;
      best = umax64(best, arg_pack(keys[at], idx[at]));
    }
    reinterpret_cast<uint32_t*>(p.out)[e] = arg_index(best);
  }
}

// ================================================================================================ entry points
// two 512-thread blocks per SM (<= 64 registers) unless the variant keeps more than 8 loads in flight per thread
#define REDUCE_ALL(NAME, OP, DT, UNROLL, WIDE)                                                                            \
  extern "C" __global__ void __launch_bounds__(512, ((UNROLL) * ((WIDE) ? 2 : 1) <= 8) ? 2 : 1) NAME(const __grid_constant__ ReduceParams p) { \
    reduce_all_body<OP, DT, UNROLL, WIDE>(p);                                                                             \
  }
#define REDUCE_ALL_BULK(NAME, OP, DT)                                                                               \
  extern "C" __global__ void __launch_bounds__(kBulkConsumers + 32, 2) NAME(const __grid_constant__ ReduceParams p) { \
    reduce_all_bulk_body<OP, DT>(p);                                                                                \
  }
#define REDUCE_ALL_PITCHED(NAME, OP, DT)                                                           \
  extern "C" __global__ void __launch_bounds__(512) NAME(const __grid_constant__ ReduceParams p) {  \
    reduce_all_pitched_body<OP, DT>(p);                                                            \
  }
#define REDUCE_ROWS(NAME, OP, DT)                                                                                   \
  extern "C" __global__ void __launch_bounds__(512) NAME(const __grid_constant__ ReduceParams p, int tpr_log2) {    \
    reduce_rows_body<OP, DT>(p, tpr_log2);                                                                          \
  }
#define REDUCE_COLS(NAME, OP, DT)                                                                                 \
  extern "C" __global__ void __launch_bounds__(kColsThreads) NAME(const __grid_constant__ ReduceParams p) {        \
    reduce_cols_body<OP, DT, 4>(p);                                                                               \
  }                                                                                                               \
  extern "C" __global__ void __launch_bounds__(kColsThreads) NAME##_n8(const __grid_constant__ ReduceParams p) {   \
    reduce_cols_body<OP, DT, 8>(p);                                                                               \
  }

#define ALL_SHAPES(OPN, OP, DTN, DT)                                                \
  REDUCE_ALL(reduce_all_##OPN##_##DTN, OP, DT, (DT == B200_F32 ? 8 : 4), false)     \
  REDUCE_ALL_BULK(reduce_all_##OPN##_##DTN##_tma, OP, DT)                           \
  REDUCE_ALL_PITCHED(reduce_allp_##OPN##_##DTN, OP, DT)                             \
  REDUCE_ROWS(reduce_rows_##OPN##_##DTN, OP, DT)                                    \
  REDUCE_COLS(reduce_cols_##OPN##_##DTN, OP, DT)
#define ALL_ARG_SHAPES(OPN, OP, DTN, DT)                                            \
  REDUCE_ALL(reduce_all_##OPN##_##DTN, OP, DT, 4, false)                            \
  REDUCE_ALL_PITCHED(reduce_allp_##OPN##_##DTN, OP, DT)                             \
  REDUCE_ROWS(reduce_rows_##OPN##_##DTN, OP, DT)                                    \
  REDUCE_COLS(reduce_cols_##OPN##_##DTN, OP, DT)
#define ALL_DTYPES(M, OPN, OP) M(OPN, OP, f32, B200_F32) M(OPN, OP, f16, B200_F16) M(OPN, OP, bf16, B200_BF16)

ALL_DTYPES(ALL_SHAPES, sum, OP_SUM)
ALL_DTYPES(ALL_SHAPES, prod, OP_PROD)
ALL_DTYPES(ALL_SHAPES, max, OP_MAX)
ALL_DTYPES(ALL_SHAPES, min, OP_MIN)
ALL_DTYPES(ALL_ARG_SHAPES, argmax, OP_ARGMAX)
ALL_DTYPES(ALL_ARG_SHAPES, argmin, OP_ARGMIN)

// local sum + cross-GPU all-reduce of the scalar in one launch (see XgpuParams)
extern "C" __global__ void __launch_bounds__(512, 2) reduce_all_sum_f32_xgpu(const __grid_constant__ ReduceParams p,
                                                                          const __grid_constant__ XgpuParams xg) {
  reduce_all_body<OP_SUM, B200_F32, 8, false, true>(p, &xg);
}
extern "C" __global__ void __launch_bounds__(512) reduce_all_argmax_f32_xgpu(const __grid_constant__ ReduceParams p,
                                                                             const __grid_constant__ XgpuParams xg) {
  reduce_all_body<OP_ARGMAX, B200_F32, 4, false, true>(p, &xg);
}
extern "C" __global__ void __launch_bounds__(512) reduce_all_argmin_f32_xgpu(const __grid_constant__ ReduceParams p,
                                                                             const __grid_constant__ XgpuParams xg) {
  reduce_all_body<OP_ARGMIN, B200_F32, 4, false, true>(p, &xg);
}

// tuning variants of the headline kernel (f32 sum over all elements); the host picks one by name.
#define REDUCE_ALL_BLOCKED(NAME, UNROLL)                                                           \
  extern "C" __global__ void __launch_bounds__(512) NAME(const __grid_constant__ ReduceParams p) {  \
    reduce_all_body<OP_SUM, B200_F32, UNROLL, false, false, true>(p);                              \
  }
REDUCE_ALL_BLOCKED(reduce_all_sum_f32_b4, 4)
REDUCE_ALL_BLOCKED(reduce_all_sum_f32_b8, 8)
REDUCE_ALL(reduce_all_sum_f32_u2, OP_SUM, B200_F32, 2, false)
REDUCE_ALL(reduce_all_sum_f32_u4, OP_SUM, B200_F32, 4, false)
REDUCE_ALL(reduce_all_sum_f32_u16, OP_SUM, B200_F32, 16, false)
REDUCE_ALL(reduce_all_sum_f32_w2, OP_SUM, B200_F32, 2, true)
REDUCE_ALL(reduce_all_sum_f32_w4, OP_SUM, B200_F32, 4, true)
// the arg-reduction with more loads in flight (tuning variant)
REDUCE_ALL(reduce_all_argmax_f32_u8, OP_ARGMAX, B200_F32, 8, false)

// ================================================================================================ scans along an axis
// cumsum / cumprod / cummax / cummin of the view [outer, len, inner] into a COMPACT row-major output of the same shape:
// inclusive out[l] = x[0] (+) ... (+) x[l], exclusive out[0] = identity, out[l] = x[0] (+) ... (+) x[l-1].  The device-wide
// form of the reference's plane scans (crates/cubecl-core/src/runtime_tests/plane.rs:191-405).  f32 running values; a
// 16-bit output is the running value rounded to nearest-even once, at the store.
//
// A long axis with few items is cut into nseg segments: the reduce first pass writes one partial per segment, an exclusive
// scan of the partials (f32 -> f32, these kernels) turns them into per-segment carries, and the final scan starts every
// segment from its carry (`carry` != 0).  Every combination order is fixed by the launch geometry: results are bitwise
// reproducible for a given shape and SM count.
template <int ODT>
struct OutElem;
template <>
struct OutElem<B200_F32> {
  using T = float;
  static constexpr int VEC = 4;
  static __device__ __forceinline__ void put(void* base, uint64_t i, float v) { reinterpret_cast<float*>(base)[i] = v; }
  static __device__ __forceinline__ uint4 pack(const float* f) {
    return make_uint4(__float_as_uint(f[0]), __float_as_uint(f[1]), __float_as_uint(f[2]), __float_as_uint(f[3]));
  }
};
template <>
struct OutElem<B200_F16> {
  using T = __half;
  static constexpr int VEC = 8;
  static __device__ __forceinline__ void put(void* base, uint64_t i, float v) { reinterpret_cast<__half*>(base)[i] = __float2half_rn(v); }
  static __device__ __forceinline__ uint4 pack(const float* f) {
    uint32_t w[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const __half2 h = __floats2half2_rn(f[2 * j], f[2 * j + 1]);
      w[j] = *reinterpret_cast<const uint32_t*>(&h);
    }
    return make_uint4(w[0], w[1], w[2], w[3]);
  }
};
template <>
struct OutElem<B200_BF16> {
  using T = __nv_bfloat16;
  static constexpr int VEC = 8;
  static __device__ __forceinline__ void put(void* base, uint64_t i, float v) {
    reinterpret_cast<__nv_bfloat16*>(base)[i] = __float2bfloat16_rn(v);
  }
  static __device__ __forceinline__ uint4 pack(const float* f) {
    uint32_t w[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const __nv_bfloat162 h = __floats2bfloat162_rn(f[2 * j], f[2 * j + 1]);
      w[j] = *reinterpret_cast<const uint32_t*>(&h);
    }
    return make_uint4(w[0], w[1], w[2], w[3]);
  }
};

__device__ __forceinline__ void stg_stream_u4(void* p, uint4 v) {
  asm volatile("st.global.cs.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// ------------------------------------------------------------------------------------------------ rows: the axis is innermost
// Work items q in [0, outer * nseg) as in reduce_rows_body, TPR threads per item (TPR <= 32: a sub-warp group, TPR > 32: the
// whole block, blockDim == TPR).  An item is walked in tiles of TPR x kScanElems elements: each thread loads its
// kScanElems consecutive elements (128-bit loads), scans them serially in registers, the group scans the thread totals
// (shfl_up, width min(TPR, 32), then a shared-memory stage across warps), and the running carry of the item joins in front.
// A base that is not 16-byte aligned costs one scalar head tile; outputs leave as 128-bit stores when their address allows.
template <int OP, int DT, int ODT>
__device__ __forceinline__ void scan_rows_body(const ScanParams& p, int tpr_log2) {
  using E = Elem<DT>;
  using T = typename E::T;
  using O = OutElem<ODT>;
  using OT = typename O::T;
  using V = ValOp<OP>;
  constexpr int VEC = E::VEC, OVEC = O::VEC, NE = kScanElems;
  static_assert(NE % VEC == 0 && NE % OVEC == 0, "tile chunk must be whole vectors");
  __shared__ float s_warp[kMaxWarps];
  pdl_wait();   // launches 2 and 3 of a segmented scan read what the previous launch wrote
  const uint32_t tpr = 1u << tpr_log2;
  const uint32_t per_block = blockDim.x >> tpr_log2;
  const uint32_t sub = threadIdx.x >> tpr_log2, t = threadIdx.x & (tpr - 1);
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t gw = tpr < 32 ? tpr : 32;                     // shuffle width
  const uint32_t gl = lane & (gw - 1);                          // lane within the shuffle segment
  const uint32_t gmask = tpr >= 32 ? 0xffffffffu : (((1u << tpr) - 1u) << (lane & ~(tpr - 1)));
  const bool excl = (p.flags & 1u) != 0;
  const uint64_t items = p.outer * p.nseg;
  const uint64_t qstride = static_cast<uint64_t>(gridDim.x) * per_block;

  for (uint64_t q = static_cast<uint64_t>(blockIdx.x) * per_block + sub; q < items; q += qstride) {
    const uint64_t o = q / p.nseg, s = q - o * p.nseg;
    const uint64_t l0 = s * p.seg_len;
    const uint64_t L = (p.len - l0 < p.seg_len) ? p.len - l0 : p.seg_len;
    const char* ib = reinterpret_cast<const char*>(p.in) + (o * p.s_outer + l0) * sizeof(T);
    char* ob = reinterpret_cast<char*>(p.out) + (o * p.len + l0) * sizeof(OT);
    float carry = p.carry ? reinterpret_cast<const float*>(p.carry)[q] : V::identity();
    const uint32_t mis = static_cast<uint32_t>(reinterpret_cast<uint64_t>(ib)) & 15u;
    uint64_t head = mis ? (16u - mis) / sizeof(T) : 0;
    if (head > L) head = L;
    const bool ovec = ((reinterpret_cast<uint64_t>(ob) + head * sizeof(OT)) & 15u) == 0;

    for (uint64_t pos = 0; pos < L;) {
      const bool head_tile = (pos == 0 && head != 0);
      const uint64_t cnt = head_tile ? head : ((L - pos < static_cast<uint64_t>(tpr) * NE) ? L - pos : static_cast<uint64_t>(tpr) * NE);
      const uint64_t c0 = static_cast<uint64_t>(t) * NE;   // this thread's chunk within the tile
      float v[NE];
#pragma unroll
      for (int u = 0; u < NE / VEC; ++u) {
        const uint64_t e = c0 + u * VEC;
        if (!head_tile && e + VEC <= cnt) {
          float f[VEC];
          E::unpack(ldg_stream_u4(ib + (pos + e) * sizeof(T)), f);
#pragma unroll
          for (int j = 0; j < VEC; ++j) v[u * VEC + j] = f[j];
        } else {
#pragma unroll
          for (int j = 0; j < VEC; ++j) v[u * VEC + j] = (e + j < cnt) ? E::get(ib, pos + e + j) : V::identity();
        }
      }
      // serial inclusive scan of the chunk
#pragma unroll
      for (int j = 1; j < NE; ++j) v[j] = V::apply(v[j - 1], v[j]);
      // scan of the chunk totals over the item's threads
      float incl = v[NE - 1];
#pragma unroll
      for (uint32_t off = 1; off < 32; off <<= 1) {
        if (off < gw) {
          const float y = __shfl_up_sync(gmask, incl, off, gw);
          if (gl >= off) incl = V::apply(y, incl);
        }
      }
      float before = __shfl_up_sync(gmask, incl, 1, gw);
      if (gl == 0) before = V::identity();
      float tile_total;
      if (tpr > 32) {   // one item per block: combine the warps through shared memory, in warp order
        if (lane == 31) s_warp[warp] = incl;
        __syncthreads();
        float pre = V::identity();
        tile_total = V::identity();
        const uint32_t nw = tpr >> 5;
        for (uint32_t w = 0; w < nw; ++w) {
          const float x = s_warp[w];
          if (w < warp) pre = V::apply(pre, x);
          tile_total = V::apply(tile_total, x);
        }
        __syncthreads();   // the slots are reused by the next tile
        before = V::apply(pre, before);
      } else {
        tile_total = __shfl_sync(gmask, incl, gw - 1, gw);
      }
      const float prefix = V::apply(carry, before);
      carry = V::apply(carry, tile_total);
      float r[NE];
      r[0] = excl ? prefix : V::apply(prefix, v[0]);
#pragma unroll
      for (int j = 1; j < NE; ++j) r[j] = V::apply(prefix, excl ? v[j - 1] : v[j]);
#pragma unroll
      for (int u = 0; u < NE / OVEC; ++u) {
        const uint64_t e = c0 + u * OVEC;
        if (!head_tile && ovec && e + OVEC <= cnt) {
          stg_stream_u4(ob + (pos + e) * sizeof(OT), O::pack(&r[u * OVEC]));
        } else {
#pragma unroll
          for (int j = 0; j < OVEC; ++j)
            if (e + j < cnt) O::put(ob, pos + e + j, r[u * OVEC + j]);
        }
      }
      pos += cnt;
    }
  }
}

// ------------------------------------------------------------------------------------------------ columns: any other axis
// Each thread owns one column UNIT (a 128-bit vector of consecutive inner elements when the layout allows it, else one
// element) and walks the item's segment of the axis serially with the running value in registers, kScanColLoads rows of
// loads in flight; consecutive threads own consecutive units, so loads and stores are coalesced.  Work items = (outer x
// segment) x tiles of blockDim units.  Per column this is the serial f32 order exactly.
constexpr int kScanColLoads = 8;

template <int OP, int DT, int ODT, bool VECTOR>
__device__ __forceinline__ void scan_cols_tiles(const ScanParams& p) {
  using E = Elem<DT>;
  using T = typename E::T;
  using O = OutElem<ODT>;
  using OT = typename O::T;
  using V = ValOp<OP>;
  constexpr int UV = VECTOR ? E::VEC : 1;
  constexpr int NL = kScanColLoads;
  static_assert(!VECTOR || UV % O::VEC == 0, "a vector unit stores whole 128-bit output vectors");
  const uint64_t units = p.inner / UV;
  const uint32_t ctu = blockDim.x;
  const uint64_t tiles = (units + ctu - 1) / ctu;
  const uint64_t items = p.outer * p.nseg * tiles;
  const bool excl = (p.flags & 1u) != 0;
  const bool ovec = VECTOR && (p.out % 16) == 0;
  const char* base = reinterpret_cast<const char*>(p.in);

  for (uint64_t item = blockIdx.x; item < items; item += gridDim.x) {
    const uint64_t q = item / tiles, tile = item - q * tiles;
    const uint64_t o = q / p.nseg, s = q - o * p.nseg;
    const uint64_t unit = tile * ctu + threadIdx.x;
    if (unit >= units) continue;
    const uint64_t l0 = s * p.seg_len;
    const uint64_t L = (p.len - l0 < p.seg_len) ? p.len - l0 : p.seg_len;
    const uint64_t i0 = unit * UV;
    uint64_t ioff = i0;
    if (p.row_len != p.inner) { const uint64_t rr = i0 / p.row_len; ioff = rr * p.row_pitch + (i0 - rr * p.row_len); }
    const char* cb = base + (o * p.s_outer + l0 * p.s_len + ioff) * sizeof(T);
    const uint64_t lstep = p.s_len * sizeof(T);
    char* ob = reinterpret_cast<char*>(p.out) + ((o * p.len + l0) * p.inner + i0) * sizeof(OT);
    const uint64_t ostep = p.inner * sizeof(OT);
    float run[UV];
#pragma unroll
    for (int j = 0; j < UV; ++j) run[j] = p.carry ? reinterpret_cast<const float*>(p.carry)[q * p.inner + i0 + j] : V::identity();

    auto emit = [&](const float (&f)[UV], uint64_t l) {
      float r[UV];
#pragma unroll
      for (int j = 0; j < UV; ++j) {
        const float nxt = V::apply(run[j], f[j]);
        r[j] = excl ? run[j] : nxt;
        run[j] = nxt;
      }
      char* dst = ob + l * ostep;
      if (ovec) {
#pragma unroll
        for (int k = 0; k < UV / O::VEC; ++k) stg_stream_u4(dst + k * 16, O::pack(&r[k * O::VEC]));
      } else {
#pragma unroll
        for (int j = 0; j < UV; ++j) O::put(dst, j, r[j]);
      }
    };

    uint64_t l = 0;
    for (; l + NL <= L; l += NL) {
      float f[NL][UV];
      if constexpr (VECTOR) {
        uint4 r[NL];
#pragma unroll
        for (int u = 0; u < NL; ++u) r[u] = ldg_stream_u4(cb + (l + u) * lstep);
#pragma unroll
        for (int u = 0; u < NL; ++u) E::unpack(r[u], f[u]);
      } else {
#pragma unroll
        for (int u = 0; u < NL; ++u) f[u][0] = E::get(cb + (l + u) * lstep, 0);
      }
#pragma unroll
      for (int u = 0; u < NL; ++u) emit(f[u], l + u);
    }
    for (; l < L; ++l) {
      float f[UV];
      if constexpr (VECTOR) E::unpack(ldg_stream_u4(cb + l * lstep), f);
      else f[0] = E::get(cb + l * lstep, 0);
      emit(f, l);
    }
  }
}

template <int OP, int DT, int ODT>
__device__ __forceinline__ void scan_cols_body(const ScanParams& p) {
  using E = Elem<DT>;
  using T = typename E::T;
  pdl_wait();
  const uint64_t esz = sizeof(T);
  const bool vec_ok = (p.flags & 2u) != 0 &&  // the host counted vector units
                      (p.inner % E::VEC) == 0 && (p.row_len % E::VEC) == 0 && (p.in % 16) == 0 && ((p.s_len * esz) % 16) == 0 &&
                      ((p.s_outer * esz) % 16) == 0 && ((p.row_pitch * esz) % 16) == 0;
  if (vec_ok) scan_cols_tiles<OP, DT, ODT, true>(p);
  else scan_cols_tiles<OP, DT, ODT, false>(p);
}

#define SCAN_KERNELS(NAME_SFX, OP, DT, ODT)                                                                              \
  extern "C" __global__ void __launch_bounds__(512) scan_rows_##NAME_SFX(const __grid_constant__ ScanParams p, int tpr_log2) { \
    scan_rows_body<OP, DT, ODT>(p, tpr_log2);                                                                          \
  }                                                                                                                    \
  extern "C" __global__ void __launch_bounds__(kScanColUnits) scan_cols_##NAME_SFX(const __grid_constant__ ScanParams p) { \
    scan_cols_body<OP, DT, ODT>(p);                                                                                    \
  }
// output f32 for every input dtype; a 16-bit input may also keep its own dtype (suffix _<out dtype>)
#define SCAN_DTYPES(OPN, OP)                                 \
  SCAN_KERNELS(OPN##_f32, OP, B200_F32, B200_F32)            \
  SCAN_KERNELS(OPN##_f16, OP, B200_F16, B200_F32)            \
  SCAN_KERNELS(OPN##_f16_f16, OP, B200_F16, B200_F16)        \
  SCAN_KERNELS(OPN##_bf16, OP, B200_BF16, B200_F32)          \
  SCAN_KERNELS(OPN##_bf16_bf16, OP, B200_BF16, B200_BF16)

SCAN_DTYPES(sum, OP_SUM)
SCAN_DTYPES(prod, OP_PROD)
SCAN_DTYPES(max, OP_MAX)
SCAN_DTYPES(min, OP_MIN)
