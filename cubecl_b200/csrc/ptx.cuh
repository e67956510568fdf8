// Inline-PTX wrappers for sm_90a: mbarrier, TMA (cp.async.bulk.tensor), wgmma (warpgroup MMA from shared memory),
// cluster primitives.  Everything here is device-only and header-only; compiled into the prebuilt cubins.
//
// These replace what the reference would have obtained from NVRTC-compiled generated C++:
//   mbarrier  -> crates/cubecl-cpp/src/cuda/barrier.rs (reference emits cuda::barrier / mbarrier PTX)
//   TMA       -> crates/cubecl-cpp/src/cuda/tma.rs:11-45
//   MMA       -> crates/cubecl-cpp/src/shared/mma.rs:48-174 (wmma) -- here wgmma, which the reference lacks
#pragma once
#include <cstdint>
#include <cuda.h>

namespace b200 {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ uint64_t globaltimer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}

__device__ __forceinline__ uint32_t cluster_id_x() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%clusterid.x;" : "=r"(r));
  return r;
}

__device__ __forceinline__ uint32_t num_clusters_x() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%nclusterid.x;" : "=r"(r));
  return r;
}

__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// Map a shared::cta address of *this* CTA to the shared::cluster address of the same offset in CTA `rank`.
__device__ __forceinline__ uint32_t mapa_shared(uint32_t addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank));
  return r;
}

// ---------------------------------------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}

__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}

// Arrive on a barrier that lives in another CTA of the cluster (address from mapa_shared).  Releases at CTA scope: the
// arrive only says "this stage's shared memory may be overwritten", and the wgmma wait before it already ordered the reads
// (a cluster-scope release costs a GPU-wide memory barrier per call).
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t cluster_bar) {
  asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(cluster_bar) : "memory");
}

__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}

__device__ __forceinline__ uint32_t mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t done;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(done)
      : "r"(bar), "r"(parity)
      : "memory");
  return done;
}

#ifndef B200_MBAR_TIMEOUT_NS
#define B200_MBAR_TIMEOUT_NS 4000000000ull  // a pipeline wait longer than 4 s is a deadlock: trap loudly, never hang the GPU
#endif

// try_wait with a suspend-time hint: the thread may be parked by the hardware for up to `ns` before the instruction
// returns false, instead of re-issuing the poll (fewer executed instructions per waiting warp, less issue-slot and power
// pressure next to the MMA / TMA warps).
__device__ __forceinline__ uint32_t mbar_try_wait_hint(uint32_t bar, uint32_t parity, uint32_t ns) {
  uint32_t done;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(done)
      : "r"(bar), "r"(parity), "r"(ns)
      : "memory");
  return done;
}

#ifndef B200_MBAR_SUSPEND_NS
#define B200_MBAR_SUSPEND_NS 20000u
#endif

__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  // slow path: parked polls; the deadline is only looked at every 64 polls (the clock read is not free either)
  uint64_t t0 = 0;
  uint32_t polls = 0;
  while (!mbar_try_wait_hint(bar, parity, B200_MBAR_SUSPEND_NS)) {
    if ((++polls & 63u) == 0) {
      const uint64_t now = globaltimer_ns();
      if (t0 == 0) t0 = now;
      else if (now - t0 > B200_MBAR_TIMEOUT_NS) asm volatile("trap;");
    }
  }
}

// ---------------------------------------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}

// 3-D tiled load, signalling an mbarrier in this CTA.
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      :
      : "r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

// 4-D im2col load of an NHWC tensor: `pixelsPerColumn` pixels x `channelsPerPixel` channels, starting at pixel (n, h, w)
// and walking the map's pixel bounding box in W, then H, then N order (with the map's element strides); every pixel is
// read at (h + off_h, w + off_w), channels from c.  Out-of-bounds elements are zero-filled.
__device__ __forceinline__ void tma_load_im2col_4d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c, int w, int h, int n,
                                                   uint16_t off_w, uint16_t off_h) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2], {%7, %8};"
      :
      : "r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c), "r"(w), "r"(h), "r"(n), "h"(off_w), "h"(off_h)
      : "memory");
}

// Multicast 4-D im2col load: as tma_load_im2col_4d, the box landing at the same smem offset in every CTA of `mask`, each
// CTA's own barrier (same offset) receiving the complete_tx.
__device__ __forceinline__ void tma_load_im2col_4d_mc(uint32_t dst, const CUtensorMap* m, uint32_t bar, uint16_t mask, int c, int w,
                                                      int h, int n, uint16_t off_w, uint16_t off_h) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes.multicast::cluster"
      " [%0], [%1, {%4, %5, %6, %7}], [%2], {%8, %9}, %3;"
      :
      : "r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "h"(mask), "r"(c), "r"(w), "r"(h), "r"(n), "h"(off_w), "h"(off_h)
      : "memory");
}

// 5-D im2col load of an NDHWC tensor: as tma_load_im2col_4d with one more spatial dimension, walking W, then H, then D,
// then N; every pixel is read at (d + off_d, h + off_h, w + off_w).  The PTX ISA gives rank-5 offsets 5 bits ([0, 31]).
__device__ __forceinline__ void tma_load_im2col_5d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c, int w, int h, int d, int n,
                                                   uint16_t off_w, uint16_t off_h, uint16_t off_d) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6, %7}], [%2], {%8, %9, %10};"
      :
      : "r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c), "r"(w), "r"(h), "r"(d), "r"(n), "h"(off_w), "h"(off_h),
        "h"(off_d)
      : "memory");
}

// Multicast 5-D im2col load (see tma_load_im2col_4d_mc).
__device__ __forceinline__ void tma_load_im2col_5d_mc(uint32_t dst, const CUtensorMap* m, uint32_t bar, uint16_t mask, int c, int w,
                                                      int h, int d, int n, uint16_t off_w, uint16_t off_h, uint16_t off_d) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes.multicast::cluster"
      " [%0], [%1, {%4, %5, %6, %7, %8}], [%2], {%9, %10, %11}, %3;"
      :
      : "r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "h"(mask), "r"(c), "r"(w), "r"(h), "r"(d), "r"(n), "h"(off_w),
        "h"(off_h), "h"(off_d)
      : "memory");
}

// Multicast 3-D load: the box lands at the same smem offset in every CTA of `mask`, each CTA's own barrier
// (same offset) receives the complete_tx.
__device__ __forceinline__ void tma_load_3d_mc(uint32_t dst, const CUtensorMap* m, uint32_t bar, uint16_t mask, int c0,
                                               int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
      " [%0], [%1, {%4, %5, %6}], [%2], %3;"
      :
      : "r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "h"(mask), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

// 3-D tiled store smem -> global (bulk async-group completion); the box is clipped at the tensor's edges.
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* m, uint32_t src, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
               :
               : "l"(reinterpret_cast<uint64_t>(m)), "r"(src), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}

// 4-D tiled load, signalling an mbarrier in this CTA (coordinates innermost first).
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      :
      : "r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// 4-D tiled store smem -> global (bulk async-group completion); the box is clipped at the tensor's edges.
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* m, uint32_t src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
               :
               : "l"(reinterpret_cast<uint64_t>(m)), "r"(src), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}

__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }

template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}

template <int N>
__device__ __forceinline__ void tma_store_wait() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// 1-D bulk copy global -> shared (UBLKCP in SASS): `bytes` and both addresses multiples of 16; completes on `bar`.
// `policy` is an L2 cache policy (createpolicy): streaming reads use evict_first so they do not displace resident data.
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ void bulk_load_1d(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
      :
      : "r"(dst), "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(bar), "l"(policy)
      : "memory");
}

// ---------------------------------------------------------------------------------------------- wgmma
// Shared-memory matrix descriptor (sm_90), SWIZZLE_128B.  Offsets are byte values, multiples of 16.
//   bits [0,14)  start address >> 4        bits [16,30) leading-dim byte offset >> 4
//   bits [32,46) stride-dim byte offset >> 4   bits [62,64) layout type (1 = SWIZZLE_128B)
// K-major operand: rows of 128 B along K, 8-row swizzle atoms SBO = 1024 B apart (LBO unused).
// MN-major operand (16-bit types only): 128-byte rows run along M/N, 8 k-rows per atom (SBO = 1024), the next 64-element
// M/N chunk LBO bytes further.
__device__ __forceinline__ uint64_t make_smem_desc_sw128(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((saddr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// The accumulator registers are live across wgmma_commit / wgmma_wait: keep the compiler from moving their uses.
template <int R>
__device__ __forceinline__ void wgmma_fence_operands(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
template <int R>
__device__ __forceinline__ void wgmma_fence_operands(uint32_t (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+r"(d[i])::"memory");
}

// Register budget per warpgroup (producer warpgroups give registers to the wgmma warpgroups).
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }

// Register / operand lists of the m64nNk* accumulator fragments (N / 2 registers per thread).
#define B200_WG_REGS_64 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}"
#define B200_WG_OPS_R64 "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31])
#define B200_WG_DA_64 "%32"
#define B200_WG_DB_64 "%33"
#define B200_WG_SC_64 "%34"
#define B200_WG_REGS_112 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55}"
#define B200_WG_OPS_F112 "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55])
#define B200_WG_OPS_R112 "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55])
#define B200_WG_DA_112 "%56"
#define B200_WG_DB_112 "%57"
#define B200_WG_SC_112 "%58"
#define B200_WG_REGS_128 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}"
#define B200_WG_OPS_F128 "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
#define B200_WG_OPS_R128 "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
#define B200_WG_DA_128 "%64"
#define B200_WG_DB_128 "%65"
#define B200_WG_SC_128 "%66"
#define B200_WG_REGS_256 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}"
#define B200_WG_OPS_F256 "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
#define B200_WG_OPS_R256 "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63]), "+r"(d[64]), "+r"(d[65]), "+r"(d[66]), "+r"(d[67]), "+r"(d[68]), "+r"(d[69]), "+r"(d[70]), "+r"(d[71]), "+r"(d[72]), "+r"(d[73]), "+r"(d[74]), "+r"(d[75]), "+r"(d[76]), "+r"(d[77]), "+r"(d[78]), "+r"(d[79]), "+r"(d[80]), "+r"(d[81]), "+r"(d[82]), "+r"(d[83]), "+r"(d[84]), "+r"(d[85]), "+r"(d[86]), "+r"(d[87]), "+r"(d[88]), "+r"(d[89]), "+r"(d[90]), "+r"(d[91]), "+r"(d[92]), "+r"(d[93]), "+r"(d[94]), "+r"(d[95]), "+r"(d[96]), "+r"(d[97]), "+r"(d[98]), "+r"(d[99]), "+r"(d[100]), "+r"(d[101]), "+r"(d[102]), "+r"(d[103]), "+r"(d[104]), "+r"(d[105]), "+r"(d[106]), "+r"(d[107]), "+r"(d[108]), "+r"(d[109]), "+r"(d[110]), "+r"(d[111]), "+r"(d[112]), "+r"(d[113]), "+r"(d[114]), "+r"(d[115]), "+r"(d[116]), "+r"(d[117]), "+r"(d[118]), "+r"(d[119]), "+r"(d[120]), "+r"(d[121]), "+r"(d[122]), "+r"(d[123]), "+r"(d[124]), "+r"(d[125]), "+r"(d[126]), "+r"(d[127])
#define B200_WG_DA_256 "%128"
#define B200_WG_DB_256 "%129"
#define B200_WG_SC_256 "%130"

// D (+)= A[smem] * B[smem] for one warpgroup, m64 x N, f32 (F) or s32 (R) accumulators.  scale_d == 0: D = A * B.
#define B200_WGMMA(N, C, KS, TYPES, TAIL)                                                                              \
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, " B200_WG_SC_##N ", 0;\n\t"                                   \
               "wgmma.mma_async.sync.aligned.m64n" #N "k" #KS "." TYPES " " B200_WG_REGS_##N ", " B200_WG_DA_##N ", "  \
               B200_WG_DB_##N ", p" TAIL ";\n\t}"                                                                      \
               : B200_WG_OPS_##C##N                                                                                    \
               : "l"(da), "l"(db), "r"(scale_d))

// Operand kinds (the GEMM's KIND values): 0 f16, 1 bf16, 2 tf32, 3 e4m3, 4 e5m2, 5 u8, 6 s8.  TA / TB: 1 = MN-major
// operand (16-bit kinds only).  8-bit kinds may pair different formats (KA != KB).
#define B200_WGMMA_16(N, T)                                                       \
  if constexpr (TA == 0 && TB == 0) B200_WGMMA(N, F, 16, "f32." T "." T, ", 1, 1, 0, 0"); \
  else if constexpr (TA == 0) B200_WGMMA(N, F, 16, "f32." T "." T, ", 1, 1, 0, 1");        \
  else if constexpr (TB == 0) B200_WGMMA(N, F, 16, "f32." T "." T, ", 1, 1, 1, 0");        \
  else B200_WGMMA(N, F, 16, "f32." T "." T, ", 1, 1, 1, 1");
#define B200_WGMMA_ALL(N)                                                                                     \
  if constexpr (KA == 0) { B200_WGMMA_16(N, "f16") }                                                          \
  else if constexpr (KA == 1) { B200_WGMMA_16(N, "bf16") }                                                    \
  else if constexpr (KA == 2) B200_WGMMA(N, F, 8, "f32.tf32.tf32", ", 1, 1");                                 \
  else if constexpr (KA == 3 && KB == 3) B200_WGMMA(N, F, 32, "f32.e4m3.e4m3", ", 1, 1");                     \
  else if constexpr (KA == 3 && KB == 4) B200_WGMMA(N, F, 32, "f32.e4m3.e5m2", ", 1, 1");                     \
  else if constexpr (KA == 4 && KB == 3) B200_WGMMA(N, F, 32, "f32.e5m2.e4m3", ", 1, 1");                     \
  else if constexpr (KA == 4 && KB == 4) B200_WGMMA(N, F, 32, "f32.e5m2.e5m2", ", 1, 1");                     \
  else if constexpr (KA == 5 && KB == 5) B200_WGMMA(N, R, 32, "s32.u8.u8", "");                               \
  else if constexpr (KA == 5 && KB == 6) B200_WGMMA(N, R, 32, "s32.u8.s8", "");                               \
  else if constexpr (KA == 6 && KB == 5) B200_WGMMA(N, R, 32, "s32.s8.u8", "");                               \
  else B200_WGMMA(N, R, 32, "s32.s8.s8", "");

// m64n64 f32 accumulators (the register list is B200_WG_REGS_64)
#define B200_WG_OPS_F64 "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])

// m64n64: s8 x s8 into s32, fp8 (e4m3 / e5m2, any pair) into f32, or f16 / bf16 with both operands K-major into f32 (the
// attention backward's 64-wide score tiles).
template <int N, int KA, int KB, int TA, int TB, typename Acc>
__device__ __forceinline__ void wgmma_ss(Acc (&d)[N / 2], uint64_t da, uint64_t db, uint32_t scale_d) {
  static_assert(N == 112 || N == 128 || N == 256 || (N == 64 && KA == 6 && KB == 6) ||
                    (N == 64 && (KA == 3 || KA == 4) && (KB == 3 || KB == 4)) ||
                    (N == 64 && KA == KB && KA <= 1 && TA == 0 && TB == 0),
                "m64n112 / m64n128 / m64n256; m64n64 s8, fp8, or f16 / bf16 K-major");
  if constexpr (N == 64 && KA == 6) B200_WGMMA(64, R, 32, "s32.s8.s8", "");
  else if constexpr (N == 64 && KA == 3 && KB == 3) B200_WGMMA(64, F, 32, "f32.e4m3.e4m3", ", 1, 1");
  else if constexpr (N == 64 && KA == 3 && KB == 4) B200_WGMMA(64, F, 32, "f32.e4m3.e5m2", ", 1, 1");
  else if constexpr (N == 64 && KA == 4 && KB == 3) B200_WGMMA(64, F, 32, "f32.e5m2.e4m3", ", 1, 1");
  else if constexpr (N == 64 && KA == 4 && KB == 4) B200_WGMMA(64, F, 32, "f32.e5m2.e5m2", ", 1, 1");
  else if constexpr (N == 64 && KA == 0) B200_WGMMA(64, F, 16, "f32.f16.f16", ", 1, 1, 0, 0");
  else if constexpr (N == 64) B200_WGMMA(64, F, 16, "f32.bf16.bf16", ", 1, 1, 0, 0");
  else if constexpr (N == 112) { B200_WGMMA_ALL(112) } else if constexpr (N == 128) { B200_WGMMA_ALL(128) } else { B200_WGMMA_ALL(256) }
}

// Register-A operand of m64nNk16 (16-bit kinds): four registers of two values each, after the N / 2 accumulators.  Thread
// (warp w, lane) holds rows 16 w + lane / 4 (+8) and k = 2 (lane % 4) (+1, +8, +9): a0 (r, k), a1 (r + 8, k), a2 (r, k + 8),
// a3 (r + 8, k + 8) -- the layout of columns 16 kk .. 16 kk + 15 of an m64nN f32 accumulator fragment, packed in pairs.
#define B200_WG_A_64 "{%32, %33, %34, %35}"
#define B200_WG_DB_RS_64 "%36"
#define B200_WG_SC_RS_64 "%37"
#define B200_WG_A_128 "{%64, %65, %66, %67}"
#define B200_WG_DB_RS_128 "%68"
#define B200_WG_SC_RS_128 "%69"
#define B200_WGMMA_RS(N, T, TB)                                                                                         \
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, " B200_WG_SC_RS_##N ", 0;\n\t"                                    \
               "wgmma.mma_async.sync.aligned.m64n" #N "k16.f32." T "." T " " B200_WG_REGS_##N ", " B200_WG_A_##N ", "    \
               B200_WG_DB_RS_##N ", p, 1, 1, " #TB ";\n\t}"                                                             \
               : B200_WG_OPS_F##N                                                                                       \
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d))

// D (+)= A[registers] * B[smem] for one warpgroup, m64 x N x k16, f32 accumulators, f16 (KIND 0) or bf16 (KIND 1).  TB: 1 = B
// is an MN-major operand.  scale_d == 0: D = A * B.
template <int N, int KIND, int TB>
__device__ __forceinline__ void wgmma_rs(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
  static_assert((N == 64 || N == 128) && (KIND == 0 || KIND == 1) && (TB == 0 || TB == 1), "m64n64 / m64n128, f16 / bf16");
  if constexpr (N == 64 && KIND == 0 && TB == 0) B200_WGMMA_RS(64, "f16", 0);
  else if constexpr (N == 64 && KIND == 0) B200_WGMMA_RS(64, "f16", 1);
  else if constexpr (N == 64 && TB == 0) B200_WGMMA_RS(64, "bf16", 0);
  else if constexpr (N == 64) B200_WGMMA_RS(64, "bf16", 1);
  else if constexpr (KIND == 0 && TB == 0) B200_WGMMA_RS(128, "f16", 0);
  else if constexpr (KIND == 0) B200_WGMMA_RS(128, "f16", 1);
  else if constexpr (TB == 0) B200_WGMMA_RS(128, "bf16", 0);
  else B200_WGMMA_RS(128, "bf16", 1);
}

}  // namespace b200
