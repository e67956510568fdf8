// Auxiliary sm_90a kernels (cubin):
//  * counter-hash generators so host (numpy) and device produce bit-identical synthetic operands without PCIe traffic
//  * a strided SIMT matmul for operands whose strides/alignment TMA cannot describe (still a CUDA path, never a CPU one);
//    it accumulates in f32 over increasing k with separate mul/add roundings, i.e. exactly the reference's CPU order
//    (crates/cubecl-core/src/runtime_tests/cmma.rs:695-721), so it is bit-comparable with the oracle
//  * the two "what the reference would run on this GPU" probes, written by hand from CubeCL's emit rules:
//      wmma_probe_f16            <- crates/cubecl-std/src/throughput/runners/compute_cmma.rs:47-91 lowered through
//                                   crates/cubecl-cpp/src/shared/mma.rs:67-155 (nvcuda::wmma 16x16x16, f16 -> f16)
//      memread_probe_vec4        <- crates/cubecl-std/src/throughput/runners/memory_read.rs:68-154 (float_4 loads)
//  * the 3xTF32 low-part split (f32 matmul at near-f32 accuracy on the tf32 tensor pipe)
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>
#include <mma.h>
#include <cstdint>

#include "kernel_params.h"

// ------------------------------------------------------------------------------------------------ generators
// splitmix64 finaliser over (seed, index); the numpy mirror lives in cubecl_b200/synth.py.
__device__ __forceinline__ uint32_t hash_u32(uint64_t seed, uint64_t i) {
  uint64_t z = seed * 0x9E3779B97F4A7C15ull + i + 0x632BE59BD9B4E019ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z = z ^ (z >> 31);
  return static_cast<uint32_t>(z >> 32);
}
__device__ __forceinline__ float hash_uniform(uint64_t seed, uint64_t i, float lo, float scale) {
  // 24 random bits -> [0,1) exactly representable, then one multiply and one add, both rounded to nearest
  const float u = static_cast<float>(hash_u32(seed, i) >> 8) * (1.0f / 16777216.0f);
  return __fadd_rn(lo, __fmul_rn(u, scale));
}

extern "C" __global__ void __launch_bounds__(256) fill_kernel(const __grid_constant__ FillParams p) {
  for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < p.n;
       i += static_cast<uint64_t>(gridDim.x) * blockDim.x) {
    const float v = (p.mode == 0) ? hash_uniform(p.seed, i, p.lo, p.scale) : static_cast<float>(i % p.modulus);
    if (p.dtype == B200_F32) reinterpret_cast<float*>(p.out)[i] = v;
    else if (p.dtype == B200_F16) reinterpret_cast<__half*>(p.out)[i] = __float2half_rn(v);
    else if (p.dtype == B200_BF16) reinterpret_cast<__nv_bfloat16*>(p.out)[i] = __float2bfloat16_rn(v);
    else reinterpret_cast<uint8_t*>(p.out)[i] = __nv_cvt_float_to_fp8(v, __NV_SATFINITE, p.dtype == B200_F8E4M3 ? __NV_E4M3 : __NV_E5M2);
  }
}

// ------------------------------------------------------------------------------------------------ strided SIMT matmul
__device__ __forceinline__ float load_as_f32(uint64_t base, uint64_t idx, uint32_t dt) {
  if (dt == B200_F32) return reinterpret_cast<const float*>(base)[idx];
  if (dt == B200_F16) return __half2float(reinterpret_cast<const __half*>(base)[idx]);
  if (dt == B200_BF16) return __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(base)[idx]);
  const __half_raw h = __nv_cvt_fp8_to_halfraw(reinterpret_cast<const uint8_t*>(base)[idx], dt == B200_F8E4M3 ? __NV_E4M3 : __NV_E5M2);
  return __half2float(__half(h));
}
__device__ __forceinline__ void store_from_f32(uint64_t base, uint64_t idx, uint32_t dt, float v) {
  if (dt == B200_F32) reinterpret_cast<float*>(base)[idx] = v;
  else if (dt == B200_F16) reinterpret_cast<__half*>(base)[idx] = __float2half_rn(v);
  else reinterpret_cast<__nv_bfloat16*>(base)[idx] = __float2bfloat16_rn(v);
}

__device__ __forceinline__ int load_as_i32(uint64_t base, uint64_t idx, uint32_t dt) {
  return dt == B200_U8 ? static_cast<int>(reinterpret_cast<const uint8_t*>(base)[idx]) : static_cast<int>(reinterpret_cast<const int8_t*>(base)[idx]);
}

extern "C" __global__ void __launch_bounds__(256) gemm_simt_strided(const __grid_constant__ SimtGemmParams p) {
  __shared__ float sa[16][17];
  __shared__ float sb[16][17];
  const uint32_t tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const uint32_t n = blockIdx.x * 16 + tx, bz = blockIdx.z;
  const bool integer = (p.in_dtype == B200_U8 || p.in_dtype == B200_I8);  // exact s32 accumulation
  // 16-row tiles of M are walked with a stride of gridDim.y (the y extent of a grid stops at 65535)
  for (uint64_t mt = blockIdx.y; mt * 16 < p.M; mt += gridDim.y) {
  const uint32_t m = static_cast<uint32_t>(mt * 16) + ty;
  float acc = 0.f;
  int iacc = 0;
  for (uint32_t k0 = 0; k0 < p.K; k0 += 16) {
    const uint32_t ka = k0 + tx, kb = k0 + ty;
    const bool va = (m < p.M && ka < p.K), vb = (kb < p.K && n < p.N);
    const uint64_t ia = bz * p.a_sb + static_cast<uint64_t>(m) * p.a_sm + static_cast<uint64_t>(ka) * p.a_sk;
    const uint64_t ib = bz * p.b_sb + static_cast<uint64_t>(kb) * p.b_sk + static_cast<uint64_t>(n) * p.b_sn;
    const uint32_t b_dt = p.b_dtype_p1 ? p.b_dtype_p1 - 1 : p.in_dtype;
    if (integer) {  // 8-bit integers are exact in f32, so the staging tiles stay float
      sa[ty][tx] = va ? static_cast<float>(load_as_i32(p.a, ia, p.in_dtype)) : 0.f;
      sb[ty][tx] = vb ? static_cast<float>(load_as_i32(p.b, ib, b_dt)) : 0.f;
    } else {
      sa[ty][tx] = va ? load_as_f32(p.a, ia, p.in_dtype) : 0.f;
      sb[ty][tx] = vb ? load_as_f32(p.b, ib, b_dt) : 0.f;
    }
    __syncthreads();
    const uint32_t kmax = min(16u, p.K - k0);
    if (integer) {
      for (uint32_t k = 0; k < kmax; ++k) iacc += static_cast<int>(sa[ty][k]) * static_cast<int>(sb[k][tx]);
    } else {
      for (uint32_t k = 0; k < kmax; ++k) acc = __fadd_rn(acc, __fmul_rn(sa[ty][k], sb[k][tx]));  // no FMA: reference order
    }
    __syncthreads();
  }
  if (m < p.M && n < p.N) {
    const uint64_t io = bz * p.o_sb + static_cast<uint64_t>(m) * p.o_sm + static_cast<uint64_t>(n) * p.o_sn;
    if (integer) {
      reinterpret_cast<int*>(p.out)[io] = iacc;
    } else {
      if (p.epi_on) {
        acc *= p.alpha;
        if (p.bias) acc += reinterpret_cast<const float*>(p.bias)[n];
        if (p.epi_act == 1) acc = fmaxf(acc, 0.f);
        else if (p.epi_act == 2) acc = 0.5f * acc * (1.f + erff(acc * 0.70710678118654752f));
      }
      store_from_f32(p.out, io, p.out_dtype, acc);
    }
  }
  }  // m tiles
}

// ---------------------------------------------------------------------------------------------------------------------
// Block-scaled (MX) support.
__device__ __forceinline__ float ue8m0_to_f32(uint32_t bits) {
  if (bits == 255u) return __uint_as_float(0x7FC00000u);      // NaN
  if (bits == 0u) return __uint_as_float(0x00400000u);        // 2^-127 (an f32 subnormal)
  return __uint_as_float(bits << 23);
}
__device__ __forceinline__ float mx_elem_to_f32(uint64_t base, uint64_t idx, uint32_t dt) {
  if (dt == B200_F4E2M1X2) {  // packed e2m1: element 2i in the low nibble of byte i (e2m1x2::from_f32_slice, cubecl-common/src/float/fp4.rs:204-216)
    const uint32_t byte = reinterpret_cast<const uint8_t*>(base)[idx >> 1];
    const uint32_t nib = (idx & 1) ? (byte >> 4) : (byte & 0xFu);
    const float mag[8] = {0.f, 0.5f, 1.f, 1.5f, 2.f, 3.f, 4.f, 6.f};
    const float v = mag[nib & 7u];
    return (nib & 8u) ? -v : v;
  }
  return load_as_f32(base, idx, dt);
}

// Reference-order block-scaled matmul (the expected-value loop of test_cmma_scaled, cmma.rs:1572-1590):
//   out[m,n] = sum over l, increasing, in f32 with separately rounded operations, of ((a[m,l] * sa[m,l/32]) * b[n,l]) * sb[n,l/32]
// One thread per output element; the path for shapes TMA cannot describe, and the on-device cross-check of the wgmma path.
extern "C" __global__ void __launch_bounds__(256) gemm_scaled_simt(const __grid_constant__ ScaledSimtParams p) {
  const uint64_t total = static_cast<uint64_t>(p.batch) * p.M * p.N;
  const uint32_t n_scales = (p.K + p.scale_block - 1) / p.scale_block;
  for (uint64_t i = blockIdx.x * static_cast<uint64_t>(blockDim.x) + threadIdx.x; i < total; i += static_cast<uint64_t>(gridDim.x) * blockDim.x) {
    const uint32_t n = static_cast<uint32_t>(i % p.N);
    const uint32_t m = static_cast<uint32_t>((i / p.N) % p.M);
    const uint32_t b = static_cast<uint32_t>(i / (static_cast<uint64_t>(p.N) * p.M));
    const uint64_t arow = (static_cast<uint64_t>(b) * p.a_bmul * p.M + m), brow = (static_cast<uint64_t>(b) * p.b_bmul * p.N + n);
    const uint8_t* sa = reinterpret_cast<const uint8_t*>(p.sa) + arow * n_scales;
    const uint8_t* sb = reinterpret_cast<const uint8_t*>(p.sb) + brow * n_scales;
    float acc = 0.f;
    for (uint32_t l = 0; l < p.K; ++l) {
      const float av = mx_elem_to_f32(p.a, arow * p.K + l, p.a_dtype), bv = mx_elem_to_f32(p.b, brow * p.K + l, p.b_dtype);
      const float as = p.scale_ue4m3 ? fabsf(load_as_f32(reinterpret_cast<uint64_t>(sa), l / p.scale_block, B200_F8E4M3)) : ue8m0_to_f32(sa[l / p.scale_block]);
      const float bs = p.scale_ue4m3 ? fabsf(load_as_f32(reinterpret_cast<uint64_t>(sb), l / p.scale_block, B200_F8E4M3)) : ue8m0_to_f32(sb[l / p.scale_block]);
      acc = __fadd_rn(acc, __fmul_rn(__fmul_rn(__fmul_rn(av, as), bv), bs));
    }
    store_from_f32(p.out, i, p.out_dtype, acc);
  }
}

// Block-scaled operand -> bf16 [rows, K]: x * scale per element, for the wgmma GEMM (Hopper's tensor cores take no scale
// factors).  Exact: an e2m1 / e4m3 / e5m2 value times a ue8m0 power of two, or e2m1 times a ue4m3 scale (at most 6
// significant bits), fits bf16's 8-bit significand; bf16 products are exact in the f32 accumulators.  Scales are the
// reference's row-major [rows, K / scale_block] layout, or the packed 128-row chunk layout when `packed`.
extern "C" __global__ void __launch_bounds__(256) dequant_scaled_bf16(const __grid_constant__ DequantParams p) {
  const uint32_t n_scales = p.K / p.scale_block;
  const uint64_t groups = static_cast<uint64_t>(p.batch) * p.rows_per_batch * (p.K / 8);   // 8 outputs (16 B) per thread
  const uint8_t* sc = reinterpret_cast<const uint8_t*>(p.scales);
  for (uint64_t g = blockIdx.x * static_cast<uint64_t>(blockDim.x) + threadIdx.x; g < groups; g += static_cast<uint64_t>(gridDim.x) * blockDim.x) {
    const uint64_t row = g / (p.K / 8);
    const uint32_t k0 = static_cast<uint32_t>(g % (p.K / 8)) * 8u;
    const uint32_t si = k0 / p.scale_block;   // scale_block is 16 or 32: one scale per group of 8
    uint64_t sidx;
    if (p.packed) {
      const uint64_t b = row / p.rows_per_batch;
      const uint32_t r = static_cast<uint32_t>(row % p.rows_per_batch);
      const uint64_t tiles = (p.rows_per_batch + 127) / 128;
      const uint32_t lr = r % 128;
      sidx = ((b * tiles + r / 128) * p.atoms + si / 4) * 512 + (lr % 32) * 16 + (lr / 32) * 4 + si % 4;
    } else {
      sidx = row * n_scales + si;
    }
    const float s = p.scale_ue4m3 ? fabsf(load_as_f32(p.scales, sidx, B200_F8E4M3)) : ue8m0_to_f32(sc[sidx]);
    uint32_t w[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float lo = mx_elem_to_f32(p.in, row * p.K + k0 + 2 * j, p.dtype) * s;
      const float hi = mx_elem_to_f32(p.in, row * p.K + k0 + 2 * j + 1, p.dtype) * s;
      __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi);
      w[j] = *reinterpret_cast<uint32_t*>(&h);
    }
    reinterpret_cast<uint4*>(p.out)[g] = make_uint4(w[0], w[1], w[2], w[3]);
  }
}

// ------------------------------------------------------------------------------------------------ 3xTF32 split
// lo = x - hi, hi = x with the low 13 mantissa bits cleared: the tf32 datapath ignores those bits of an f32 operand, so
// the ORIGINAL tensor already acts as "hi" and only `lo` (exact in f32) is materialised, with the input's own strides
// compacted to a [batch, rows, out_rs] copy (rows padded to 16 bytes).  The GEMM then accumulates hi*hi + hi*lo + lo*hi in one launch
// (GemmParams::k_segments == 3).
// (a non-finite x has no low part: inf - inf would turn an infinite product into NaN)
__device__ __forceinline__ float tf32_lo(float x) {
  const float lo = x - __uint_as_float(__float_as_uint(x) & 0xFFFFE000u);
  return (fabsf(x) < __int_as_float(0x7F800000)) ? lo : 0.f;
}

extern "C" __global__ void __launch_bounds__(256) split_tf32_lo(const __grid_constant__ SplitParams p) {
  const uint64_t tid = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const uint64_t nthreads = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  const bool vec = (p.cols % 4 == 0) && (p.in_rs % 4 == 0) && (p.in_bs % 4 == 0) && (p.in % 16 == 0) && (p.out % 16 == 0);
  if (vec && p.in_rs == p.cols && p.out_rs == p.cols && (p.batch == 1 || p.in_bs == p.rows * p.cols)) {
    // compact input and output (the common case): one flat stream of 128-bit vectors, no index arithmetic -- this pass runs in
    // front of every 3xTF32 GEMM, where a scalar, divide-per-element form costs several times its traffic time
    const uint64_t nv = p.batch * p.rows * p.cols / 4;
    const float4* in = reinterpret_cast<const float4*>(p.in);
    float4* out = reinterpret_cast<float4*>(p.out);
    for (uint64_t i = tid; i < nv; i += nthreads) {
      const float4 x = in[i];
      out[i] = make_float4(tf32_lo(x.x), tf32_lo(x.y), tf32_lo(x.z), tf32_lo(x.w));
    }
    return;
  }
  if (vec) {
    // strided rows, vector columns: one division per 128-bit vector
    const uint64_t vpr = p.cols / 4, per = p.rows * vpr, nv = p.batch * per;
    for (uint64_t i = tid; i < nv; i += nthreads) {
      const uint64_t b = i / per, rem = i - b * per;
      const uint64_t r = rem / vpr, c = (rem - r * vpr) * 4;
      const float4 x = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(p.in) + b * p.in_bs + r * p.in_rs + c);
      *reinterpret_cast<float4*>(reinterpret_cast<float*>(p.out) + (b * p.rows + r) * p.out_rs + c) =
          make_float4(tf32_lo(x.x), tf32_lo(x.y), tf32_lo(x.z), tf32_lo(x.w));
    }
    return;
  }
  const uint64_t per = p.rows * p.cols, total = p.batch * per;
  for (uint64_t i = tid; i < total; i += nthreads) {
    const uint64_t b = i / per, rem = i - b * per;
    const uint64_t r = rem / p.cols, c = rem - r * p.cols;
    reinterpret_cast<float*>(p.out)[(b * p.rows + r) * p.out_rs + c] = tf32_lo(reinterpret_cast<const float*>(p.in)[b * p.in_bs + r * p.in_rs + c]);
  }
}

// Hybrid f32 schedule (GemmParams::hyb): the cross terms A*B_lo + A_lo*B run on bf16 copies.  One pass writes both planes of
// the operand's pair buffer: plane 0 = bf16(x) (round to nearest even), plane 1 = bf16(x - trunc_tf32(x)); planes are
// batch * rows * out_rs elements apart, rows pitched to out_rs (a multiple of 8 elements = 16 bytes, for TMA).
__device__ __forceinline__ uint32_t bf16x2_bits(float lo, float hi) {
  const __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<const uint32_t*>(&h);
}
// plane 0 only multiplies low parts: a non-finite x contributes through the tf32 segment alone (inf * lo with lo == 0 would be
// NaN), and a finite x that rounds up to the bf16 infinity is kept at the largest finite bf16
__device__ __forceinline__ uint32_t bf16_main_bits(float x) {
  if (!(fabsf(x) < __int_as_float(0x7F800000))) return 0u;
  const __nv_bfloat16 h = __float2bfloat16_rn(x);
  uint32_t b = *reinterpret_cast<const uint16_t*>(&h);
  if ((b & 0x7FFFu) == 0x7F80u) b -= 1u;
  return b;
}
__device__ __forceinline__ uint32_t bf16x2_main(float lo, float hi) { return bf16_main_bits(lo) | (bf16_main_bits(hi) << 16); }
extern "C" __global__ void __launch_bounds__(256) split_f32_bf16_pair(const __grid_constant__ SplitParams p) {
  const uint64_t tid = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const uint64_t nthreads = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  const uint64_t plane = p.batch * p.rows * p.out_rs;
  uint16_t* out = reinterpret_cast<uint16_t*>(p.out);
  const float* in = reinterpret_cast<const float*>(p.in);
  const bool al = (p.in % 16 == 0) && (p.out % 16 == 0) && (p.in_rs % 4 == 0) && (p.in_bs % 4 == 0);
  if (al && p.cols % 8 == 0 && p.in_rs == p.cols && p.out_rs == p.cols && (p.batch == 1 || p.in_bs == p.rows * p.cols)) {
    // compact input and output: a flat stream, 32 bytes in and 2 x 16 bytes out per thread and trip
    const uint64_t nv = plane / 8;
    const float4* in4 = reinterpret_cast<const float4*>(in);
    uint4* o0 = reinterpret_cast<uint4*>(out);
    uint4* o1 = reinterpret_cast<uint4*>(out + plane);
    for (uint64_t i = tid; i < nv; i += nthreads) {
      const float4 x = in4[2 * i], y = in4[2 * i + 1];
      o0[i] = make_uint4(bf16x2_main(x.x, x.y), bf16x2_main(x.z, x.w), bf16x2_main(y.x, y.y), bf16x2_main(y.z, y.w));
      o1[i] = make_uint4(bf16x2_bits(tf32_lo(x.x), tf32_lo(x.y)), bf16x2_bits(tf32_lo(x.z), tf32_lo(x.w)),
                         bf16x2_bits(tf32_lo(y.x), tf32_lo(y.y)), bf16x2_bits(tf32_lo(y.z), tf32_lo(y.w)));
    }
    return;
  }
  if (al && p.cols % 4 == 0) {
    // strided rows, vector columns: one division per 4-element vector (8-byte stores; out_rs is a multiple of 8 elements)
    const uint64_t vpr = p.cols / 4, per = p.rows * vpr, nv = p.batch * per;
    for (uint64_t i = tid; i < nv; i += nthreads) {
      const uint64_t b = i / per, rem = i - b * per;
      const uint64_t r = rem / vpr, c4 = (rem - r * vpr) * 4;
      const float4 x = *reinterpret_cast<const float4*>(in + b * p.in_bs + r * p.in_rs + c4);
      uint16_t* o = out + (b * p.rows + r) * p.out_rs + c4;
      *reinterpret_cast<uint2*>(o) = make_uint2(bf16x2_main(x.x, x.y), bf16x2_main(x.z, x.w));
      *reinterpret_cast<uint2*>(o + plane) = make_uint2(bf16x2_bits(tf32_lo(x.x), tf32_lo(x.y)), bf16x2_bits(tf32_lo(x.z), tf32_lo(x.w)));
    }
    return;
  }
  const uint64_t per = p.rows * p.cols, total = p.batch * per;
  for (uint64_t i = tid; i < total; i += nthreads) {
    const uint64_t b = i / per, rem = i - b * per;
    const uint64_t r = rem / p.cols, cc = rem - r * p.cols;
    const float x = in[b * p.in_bs + r * p.in_rs + cc];
    uint16_t* o = out + (b * p.rows + r) * p.out_rs + cc;
    o[0] = static_cast<uint16_t>(bf16_main_bits(x));
    o[plane] = static_cast<uint16_t>(bf16x2_bits(tf32_lo(x), 0.f) & 0xFFFFu);
  }
}

// ------------------------------------------------------------------------------------------------ reference probes
// compute_cmma_throughput: A,B = fill(1), acc = 0, n_iter x mma_sync(acc, a, b, acc), unit 0 of each plane-0 stores.
// Launch exactly like compute_cmma.rs:20-42: grid = SMs*32, block = 256 (8 planes).
extern "C" __global__ void __launch_bounds__(256) wmma_probe_f16(__half* out, uint32_t n_iter) {
  using namespace nvcuda;
  wmma::fragment<wmma::matrix_a, 16, 16, 16, __half, wmma::row_major> a;
  wmma::fragment<wmma::matrix_b, 16, 16, 16, __half, wmma::col_major> b;
  wmma::fragment<wmma::accumulator, 16, 16, 16, __half> acc;
  wmma::fill_fragment(a, __float2half(1.0f));
  wmma::fill_fragment(b, __float2half(1.0f));
  wmma::fill_fragment(acc, __float2half(0.0f));
  for (uint32_t i = 0; i < n_iter; ++i) wmma::mma_sync(acc, a, b, acc);
  if (threadIdx.x < 32 && blockIdx.x == 0) wmma::store_matrix_sync(out, acc, 16, wmma::mem_row_major);
}
// bf16 -> f32 variant (what a cubek bf16 matmul would accumulate with: cuda_compiler.rs:27-31)
extern "C" __global__ void __launch_bounds__(256) wmma_probe_bf16(float* out, uint32_t n_iter) {
  using namespace nvcuda;
  wmma::fragment<wmma::matrix_a, 16, 16, 16, __nv_bfloat16, wmma::row_major> a;
  wmma::fragment<wmma::matrix_b, 16, 16, 16, __nv_bfloat16, wmma::col_major> b;
  wmma::fragment<wmma::accumulator, 16, 16, 16, float> acc;
  wmma::fill_fragment(a, __float2bfloat16(1.0f));
  wmma::fill_fragment(b, __float2bfloat16(1.0f));
  wmma::fill_fragment(acc, 0.0f);
  for (uint32_t i = 0; i < n_iter; ++i) wmma::mma_sync(acc, a, b, acc);
  if (threadIdx.x < 32 && blockIdx.x == 0) wmma::store_matrix_sync(out, acc, 16, wmma::mem_row_major);
}

// memory_read_throughput: acc += input[ABSOLUTE_POS + step * stride] over `steps` coalesced float_4 lines,
// one accumulator per unit (memory_read.rs:95-99), unit 0 writes one line.
extern "C" __global__ void __launch_bounds__(256) memread_probe_vec4(const float4* __restrict__ in, float4* out,
                                                                      uint64_t lines, uint32_t steps) {
  const uint64_t pos = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (uint32_t s = 0; s < steps; ++s) {
    const uint64_t idx = pos + s * stride;
    if (idx < lines) {
      const float4 v = in[idx];
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
  }
  if (pos == 0 || acc.x == -1.2345e33f) out[0] = acc;  // the data-dependent arm keeps every unit's loads alive
}

// memory_write_throughput (crates/cubecl-std/src/throughput/runners/memory_write.rs): the copy kernel with the load
// removed -- every unit writes one constant float_4 line per step, coalesced, `steps` passes over `lines`.
extern "C" __global__ void __launch_bounds__(256) memwrite_probe_vec4(float4* out, uint64_t lines, uint32_t steps) {
  const uint64_t pos = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  const float4 v = make_float4(1.f, 2.f, 3.f, 4.f);
  for (uint32_t s = 0; s < steps; ++s) {
    const uint64_t idx = pos + s * stride;
    if (idx < lines) out[idx] = v;
  }
}

// memory_direct (runners/memory_direct.rs): a line in and a line back out; ops_count counts BOTH directions, which is
// the convention of the copy roofline (and of MEASURED_PEAKS.json's hbm_gbs).
extern "C" __global__ void __launch_bounds__(256) memcopy_probe_vec4(const float4* __restrict__ in, float4* out,
                                                                      uint64_t lines, uint32_t steps) {
  const uint64_t pos = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  for (uint32_t s = 0; s < steps; ++s) {
    const uint64_t idx = pos + s * stride;
    if (idx < lines) out[idx] = in[idx];
  }
}

// ------------------------------------------------------------------------------------------------ into_contiguous
// Gather a strided rank<=8 tensor into a compact row-major buffer (crates/cubecl-std/src/tensor/contiguous.rs is the
// reference's generic version).  Only used in front of kernels that need contiguous input (reduce) when the caller
// hands in a pitched / permuted TensorHandle; element size 1, 2, 4 or 8 bytes.
extern "C" __global__ void __launch_bounds__(256) gather_strided(const __grid_constant__ GatherParams p) {
  for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < p.n;
       i += static_cast<uint64_t>(gridDim.x) * blockDim.x) {
    uint64_t rem = i, off = 0;
#pragma unroll 1
    for (int d = static_cast<int>(p.rank) - 1; d >= 0; --d) {
      const uint64_t q = rem / p.shape[d];
      off += (rem - q * p.shape[d]) * p.strides[d];
      rem = q;
    }
    if (p.esz == 4) reinterpret_cast<uint32_t*>(p.out)[i] = reinterpret_cast<const uint32_t*>(p.in)[off];
    else if (p.esz == 2) reinterpret_cast<uint16_t*>(p.out)[i] = reinterpret_cast<const uint16_t*>(p.in)[off];
    else if (p.esz == 8) reinterpret_cast<uint64_t*>(p.out)[i] = reinterpret_cast<const uint64_t*>(p.in)[off];
    else reinterpret_cast<uint8_t*>(p.out)[i] = reinterpret_cast<const uint8_t*>(p.in)[off];
  }
}


// ------------------------------------------------------------------------------------------------ operand staging
// Copy a strided [batch, rows, cols] operand into a pitched buffer TMA can describe (pitch a multiple of 16 bytes): one
// 16-byte output vector per thread, gathered element by element from the (possibly misaligned) input rows.  Only in front
// of the tensor-core GEMM for operands whose own pitch / base is not 16-byte aligned (bf16 with K = 4097, odd sub-views).
// fp8 (e4m3 / e5m2) operand -> f16, exactly (f16 holds every e4m3 and e5m2 value), with the operand's own strides compacted to
// [batch, rows, out_pitch].  wgmma accumulates fp8 products with less than f32 precision, so fp8 matmuls run on the f16 kernels.
extern "C" __global__ void __launch_bounds__(256) convert_fp8_f16(const __grid_constant__ ConvertF16Params p) {
  const uint64_t vpr = p.out_pitch / 8;                  // 16-byte output vectors per row
  const uint64_t total = p.batch * p.rows * vpr;
  const uint8_t* in = reinterpret_cast<const uint8_t*>(p.in);
  for (uint64_t v = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; v < total;
       v += static_cast<uint64_t>(gridDim.x) * blockDim.x) {
    const uint64_t row = v / vpr, cv = v - row * vpr;
    const uint64_t b = row / p.rows, r = row - b * p.rows;
    const uint64_t c0 = cv * 8;
    const uint64_t src = b * p.in_sb + r * p.in_sr;
    uint32_t w[4] = {0u, 0u, 0u, 0u};                    // padding columns are written as zeros
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (c0 + j < p.cols) {
        const __nv_fp8_storage_t x = in[src + (c0 + j) * p.in_sc];
        const __half_raw h = __nv_cvt_fp8_to_halfraw(x, p.dtype == B200_F8E5M2 ? __NV_E5M2 : __NV_E4M3);
        w[j >> 1] |= static_cast<uint32_t>(h.x) << (16 * (j & 1));
      }
    }
    reinterpret_cast<uint4*>(p.out)[row * vpr + cv] = make_uint4(w[0], w[1], w[2], w[3]);
  }
}

extern "C" __global__ void __launch_bounds__(256) repitch_rows(const __grid_constant__ RepitchParams p) {
  const uint32_t per = 16 / p.esz;                       // elements per output vector
  const uint64_t vpr = p.out_pitch / per;                // vectors per output row
  const uint64_t total = p.batch * p.rows * vpr;
  for (uint64_t v = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; v < total;
       v += static_cast<uint64_t>(gridDim.x) * blockDim.x) {
    const uint64_t row = v / vpr, cv = v - row * vpr;
    const uint64_t b = row / p.rows, r = row - b * p.rows;
    const uint64_t c0 = cv * per;
    const uint64_t src = b * p.in_sb + r * p.in_sr;
    uint32_t w[4] = {0u, 0u, 0u, 0u};                    // padding columns are written as zeros (TMA never reads them anyway)
    if (p.esz == 4) {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (c0 + j < p.cols) w[j] = reinterpret_cast<const uint32_t*>(p.in)[src + (c0 + j) * p.in_sc];
    } else if (p.esz == 2) {
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (c0 + j < p.cols) w[j >> 1] |= static_cast<uint32_t>(reinterpret_cast<const uint16_t*>(p.in)[src + (c0 + j) * p.in_sc]) << (16 * (j & 1));
    } else {
#pragma unroll
      for (int j = 0; j < 16; ++j)
        if (c0 + j < p.cols) w[j >> 2] |= static_cast<uint32_t>(reinterpret_cast<const uint8_t*>(p.in)[src + (c0 + j) * p.in_sc]) << (8 * (j & 3));
    }
    reinterpret_cast<uint4*>(p.out)[row * vpr + cv] = make_uint4(w[0], w[1], w[2], w[3]);
  }
}

// ------------------------------------------------------------------------------------------------ convolution backward
// Weights of every data-gradient phase (see ConvDgradWeightsParams): w'[c, th, tw, co] = w[co, ky, kx, c] with the taps of
// each phase in ascending dy-offset order.  A block transposes one 32 (co) x 32 (c) tile of one kernel position through
// shared memory, so both the reads (along c) and the writes (along co) are coalesced.  grid = (c tiles * co tiles, KH * KW).
extern "C" __global__ void __launch_bounds__(256) conv_dgrad_weights(const __grid_constant__ ConvDgradWeightsParams p) {
  __shared__ uint16_t tile[32][33];
  const uint32_t kpos = blockIdx.y, ky = kpos / p.KW, kx = kpos - ky * p.KW;
  const uint64_t c_tiles = (p.C + 31) / 32;
  const uint64_t c0 = (blockIdx.x % c_tiles) * 32, co0 = (blockIdx.x / c_tiles) * 32;
  const uint32_t tx = threadIdx.x & 31u, ty = threadIdx.x >> 5;
  const uint16_t* w = reinterpret_cast<const uint16_t*>(p.w);
  for (uint32_t r = ty; r < 32; r += 8) {
    const uint64_t co = co0 + r, c = c0 + tx;
    tile[r][tx] = (co < p.Cout && c < p.C) ? w[co * p.s_co + ky * p.s_ky + kx * p.s_kx + c * p.s_c] : static_cast<uint16_t>(0);
  }
  __syncthreads();
  // phase of this kernel position and its tap index inside the phase
  const uint32_t rh = (ky * p.dh + p.sh * p.ph - p.ph) % p.sh, rw = (kx * p.dw + p.sw * p.pw - p.pw) % p.sw;
  const uint32_t th = (p.kmax_h[rh] - ky) / p.qh, tw = (p.kmax_w[rw] - kx) / p.qw;
  const uint64_t base = p.off[rh * p.sw + rw] + (static_cast<uint64_t>(th) * p.taps_w[rw] + tw) * p.cp;
  const uint64_t c_pitch = static_cast<uint64_t>(p.taps_h[rh]) * p.taps_w[rw] * p.cp;
  uint16_t* out = reinterpret_cast<uint16_t*>(p.out);
  for (uint32_t r = ty; r < 32; r += 8) {
    const uint64_t c = c0 + r, co = co0 + tx;
    if (c < p.C && co < p.cp) out[base + c * c_pitch + co] = tile[tx][r];
  }
}

// Conv3dDgradWeightsParams: one block per (32 input channels x 32 output channels, kernel position (kz, ky, kx)).
extern "C" __global__ void __launch_bounds__(256) conv3d_dgrad_weights(const __grid_constant__ Conv3dDgradWeightsParams p) {
  __shared__ uint16_t tile[32][33];
  const uint32_t khw = p.k[1] * p.k[2], kpos = blockIdx.y;
  const uint32_t kk[3] = {kpos / khw, (kpos % khw) / p.k[2], kpos % p.k[2]};
  const uint64_t c_tiles = (p.C + 31) / 32;
  const uint64_t c0 = (blockIdx.x % c_tiles) * 32, co0 = (blockIdx.x / c_tiles) * 32;
  const uint32_t tx = threadIdx.x & 31u, ty = threadIdx.x >> 5;
  const uint16_t* w = reinterpret_cast<const uint16_t*>(p.w);
  for (uint32_t r = ty; r < 32; r += 8) {
    const uint64_t co = co0 + r, c = c0 + tx;
    tile[r][tx] = (co < p.Cout && c < p.C) ? w[co * p.s_co + kk[0] * p.s_kz + kk[1] * p.s_ky + kk[2] * p.s_kx + c * p.s_c]
                                           : static_cast<uint16_t>(0);
  }
  __syncthreads();
  // per dimension: this position's phase, its tap index inside the phase, the phase's tap count and the taps before it
  uint32_t t[3], n[3], pre[3];
  for (int i = 0; i < 3; ++i) {
    const uint32_t r = (kk[i] * p.d[i] + p.s[i] * p.p[i] - p.p[i]) % p.s[i];
    t[i] = (p.kmax[i][r] - kk[i]) / p.q[i];
    n[i] = p.taps[i][r];
    pre[i] = 0;
    for (uint32_t j = 0; j < r; ++j) pre[i] += p.taps[i][j];
  }
  const uint64_t blk = p.C * p.cp *
      (static_cast<uint64_t>(pre[0]) * khw + static_cast<uint64_t>(n[0]) * (static_cast<uint64_t>(pre[1]) * p.k[2] + static_cast<uint64_t>(n[1]) * pre[2]));
  const uint64_t base = blk + ((static_cast<uint64_t>(t[0]) * n[1] + t[1]) * n[2] + t[2]) * p.cp;
  const uint64_t c_pitch = static_cast<uint64_t>(n[0]) * n[1] * n[2] * p.cp;
  uint16_t* out = reinterpret_cast<uint16_t*>(p.out);
  for (uint32_t r = ty; r < 32; r += 8) {
    const uint64_t c = c0 + r, co = co0 + tx;
    if (c < p.C && co < p.cp) out[base + c * c_pitch + co] = tile[tx][r];
  }
}
