/* cubecl_b200.h -- C ABI of the H100-native dense linear-algebra hot path (wgmma matmul + HBM-bound reduction).
 *
 * This is the drop-in boundary a CubeCL maintainer binds from Rust (see INTEGRATION.md for the `extern "C"` block and the
 * `CudaServer` hook).  Plain pointers and sizes only; no torch / C++ types.  All device pointers are CUdeviceptr values
 * carried as uint64_t, all streams are CUstream carried as void* (NULL = the context's own compute stream).
 *
 * Citations are into the reference tree (tracel-ai/cubecl @ 4057f39e), i.e. the interface each entry point replaces.
 *
 * Threading (crates/cubecl-common/src/device/handle/mod.rs:18-24): one thread per device at a time; distinct contexts
 * are independent.  The only process-global state is the dlopen'ed driver/NCCL symbol tables and the last-error string,
 * which is thread-local.
 *
 * Errors (crates/cubecl-runtime/src/server/base.rs:177-272): every call returns a b200_status; the message is available
 * from b200_last_error() on the calling thread.  Asynchronous device faults surface at the next b200_sync()/b200_read(),
 * like ServerError::ServerUnhealthy does at sync/read (crates/cubecl-cuda/src/compute/server.rs:981-1022).
 *
 * There is no CPU fallback anywhere behind this header: without a CUDA driver and an sm_90 device b200_init() fails.
 */
#ifndef CUBECL_B200_H
#define CUBECL_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200_ABI_VERSION 1

typedef struct b200_ctx b200_ctx;
typedef uint64_t b200_dptr;   /* CUdeviceptr */
typedef void* b200_stream;    /* CUstream; NULL = context compute stream */
typedef void* b200_event;     /* CUevent */

/* Mirrors LaunchError / ServerError variants (server/base.rs:177-272) so a Rust shim can map 1:1. */
typedef enum b200_status {
  B200_OK = 0,
  B200_ERR_COMPILATION = 1,        /* LaunchError::CompilationError  -- here: cubin image failed to load */
  B200_ERR_OUT_OF_MEMORY = 2,      /* LaunchError::OutOfMemory */
  B200_ERR_TOO_MANY_RESOURCES = 3, /* LaunchError::TooManyResources (smem / units / cube dim) */
  B200_ERR_UNKNOWN = 4,            /* LaunchError::Unknown */
  B200_ERR_IO = 5,                 /* LaunchError::IoError / IoError::* */
  B200_ERR_INVALID_ARG = 6,        /* shape/stride/dtype validation failed before launch */
  B200_ERR_UNSUPPORTED = 7,        /* feature absent (dtype/layout not implemented) -- callers self-skip like runtime_tests do */
  B200_ERR_NO_DEVICE = 8,          /* no driver / no sm_90 device: fail loudly, never fall back */
  B200_ERR_COMM = 9,               /* NCCL failure -> ServerError::Generic (server.rs:773-776) */
  B200_ERR_UNHEALTHY = 10          /* deferred device fault surfaced at sync -> ServerError::ServerUnhealthy */
} b200_status;

/* Element types.  Values double as the NCCL dtype selector of communication.rs:34-108 for all_reduce. */
typedef enum b200_dtype {
  B200_F32 = 0, B200_F16 = 1, B200_BF16 = 2, B200_U32 = 3, B200_I32 = 4, B200_F64 = 5, B200_I64 = 6, B200_U64 = 7,
  B200_U8 = 8, B200_I8 = 9,
  B200_F8E4M3 = 10, B200_F8E5M2 = 11,  /* fp8 matmul inputs (FloatKind::E4M3 / E5M2; manual-MMA dtypes of cuda/mma/manual.rs:108-186) */
  B200_F4E2M1X2 = 12,                  /* two e2m1 per byte, element 2i in the low nibble (e2m1x2, cubecl-common/src/float/fp4.rs:28,204-216) */
  B200_UE8M0 = 13                      /* block scale 2^(bits-127) (FloatKind::UE8M0; scales_type of ScaledMmaConfig) */
} b200_dtype;

/* Reduction instructions of the `reduce::launch` surface (cubek); in-tree semantics: examples/sum_things/src/lib.rs:6-33,
 * cubecl-book/.../v1-cpu.rs:7-15.  Arg ops: ties -> lowest index, NaN is the extreme and the first NaN wins. */
typedef enum b200_reduce_op {
  B200_REDUCE_SUM = 0, B200_REDUCE_PROD = 1, B200_REDUCE_MAX = 2, B200_REDUCE_MIN = 3,
  B200_REDUCE_ARGMAX = 4, B200_REDUCE_ARGMIN = 5, B200_REDUCE_MEAN = 6
} b200_reduce_op;

/* ReduceOperation{Sum,Mean} -- crates/cubecl-runtime/src/server/base.rs:623-628 */
typedef enum b200_comm_op { B200_COMM_SUM = 0, B200_COMM_MEAN = 1 } b200_comm_op;

/* HardwareProperties subset -- crates/cubecl-ir/src/properties.rs:26-58, probed like cubecl-cuda/src/runtime.rs:52-350 */
typedef struct b200_props {
  int32_t device;
  int32_t cc_major, cc_minor;
  int32_t num_sms;                 /* num_streaming_multiprocessors */
  int32_t max_shared_per_block;    /* opt-in maximum (max_shared_memory_size) */
  int32_t clock_khz, mem_clock_khz;
  int32_t plane_size;              /* 32 */
  uint64_t total_mem;
  char name[128];
} b200_props;

/* ---- lifecycle: R::client(device) -> DeviceService::init (cubecl-cuda/src/runtime.rs:52-350) ------------------------ */
int b200_abi_version(void);
int b200_device_count(int* count);
/* The embedded prebuilt sm_90a images ("gemm" | "gemm_b" | "gemm_c" | "reduce" | "aux" | "quant" | "gemm_q" | "quant_mm" | "gemm_conv"), for a host that prefers to cuModuleLoadData them into
 * its own module cache (CudaContext::modules, crates/cubecl-cuda/src/compute/context.rs:38-62,293). No GPU needed. */
int b200_get_cubin(const char* name, const void** image, size_t* size);
int b200_init(int device, b200_ctx** out);   /* cuInit, primary ctx retain, load the embedded sm_90a cubins (context.rs:293) */
int b200_destroy(b200_ctx* ctx);
int b200_get_props(b200_ctx* ctx, b200_props* out);
/* Dry-run planning context (DryRun, crates/cubecl-runtime/src/dry_run.rs:45,88,121): needs no driver and no device.  Ops
 * called on it (b200_matmul, b200_reduce*, b200_alloc, ...) validate and plan exactly like a real context but RECORD each
 * pooled allocation, TMA descriptor and kernel launch as one text line instead of executing it.  b200_plan_text copies the
 * log (and clears it when it fit); *needed = bytes required.  Device pointers passed to ops may be any non-zero values. */
int b200_plan_begin(int num_sms, b200_ctx** out);
int b200_plan_text(b200_ctx* ctx, char* buf, size_t capacity, size_t* needed);
/* Runtime knobs, string-typed like cubecl.toml keys (config/base.rs:18-120).  Keys: "gemm.variant"
 * (auto|2sm_n256|2sm_n128|1sm_n128|simt; opt-in: 2sm_m512 = 512 x 128 pair tile for 16-bit kinds, 2sm_n224 = 256 x 224 pair tile
 * for block-scaled kinds), "gemm.f32" (hybrid|3xtf32|tf32: f32 inputs as one
 * tf32 pass + two bf16 cross-term passes in ONE launch (default, ~2^-20 of the product), three tf32 passes, or one), "gemm.group_m",
 * "gemm.l2_promotion" (256|128|64|0: TMA L2 promotion bytes of the operand tensor maps), "gemm.split_k" (auto|off|on|1..8:
 * deterministic stream-K head -- the tiles of a partial last wave are cut along K into equal ranges that run FIRST, slabs
 * added in k order; N = ranges per tile), "gemm.epilogue" (tma|direct: whole tiles leave through shared-memory staging and
 * TMA stores, or each thread stores its own fragment), "gemm.stage" (on|off: operands TMA cannot describe --
 * unaligned row pitch / base -- are first copied into an aligned pooled buffer and run on the tensor cores; off = strided SIMT kernel), "reduce.variant"
 * (auto|u2|u4|u8|u16|b4|b8|w2|w4: load-unroll / blocked / 2 x 128-bit forms of the all-elements kernel; tma: 16 KB bulk copies
 * into a shared-memory ring), "reduce.threads", "reduce.blocks_per_sm" (all-elements kernel), "reduce.rows_vpt" (128-bit
 * vectors per thread that size the threads-per-row of the row kernel), "reduce.rows_blocks_per_sm" /
 * "reduce.cols_blocks_per_sm" (below this many blocks per SM a long reduced axis is cut into segments: two passes),
 * "reduce.debug" (1: the fused reduce + exchange records its stage timings, see b200_reduce_debug), "reduce.pdl" (on|off:
 * back-to-back all-element reductions on the context's own stream overlap through programmatic dependent launch -- the next
 * launch streams its input while the previous one's last block finishes; results are unchanged). */
int b200_set_option(b200_ctx* ctx, const char* key, const char* value);
/* Number of device kernels this context has launched so far (bench.py reports it as gpu_launches). */
int b200_launch_count(b200_ctx* ctx, uint64_t* count);
/* Name of the kernel (cubin entry point) the context launched most recently, NUL-terminated, truncated to `capacity`:
 * what a measurement harness reports as the kernel it timed (bench.py: roofline.kernel). */
int b200_last_kernel(b200_ctx* ctx, char* buf, size_t capacity);

/* ---- memory: ComputeClient::{empty,create_from_slice,read_one} (cubecl-runtime/src/client.rs:654,452,256) ----------- */
/* Pooled device allocation, 512-byte aligned (mem_alignment, cubecl-cuda/src/runtime.rs:81). */
int b200_alloc(b200_ctx* ctx, size_t bytes, b200_dptr* out);
/* b200_free returns the page to the pool as of the CONTEXT's stream: a buffer that work queued on another stream (the
 * `s` argument of the compute / copy entry points) may still touch must be freed with b200_free_async naming that stream --
 * the pool then re-issues the page only after an event recorded there has completed (the reference binds pool memory to
 * its stream and waits on cross-stream events, crates/cubecl-runtime/src/stream/event.rs:50-57). */
int b200_free(b200_ctx* ctx, b200_dptr ptr);
int b200_free_async(b200_ctx* ctx, b200_dptr ptr, b200_stream last_use);
int b200_memory_usage(b200_ctx* ctx, uint64_t* bytes_in_use, uint64_t* bytes_reserved);  /* MemoryUsage, memory_management/base.rs:7-28 */
int b200_memory_cleanup(b200_ctx* ctx);                                                  /* client.memory_cleanup */
/* Pinned host staging (compute/stream.rs:138-178 pinned pool). */
int b200_host_alloc(b200_ctx* ctx, size_t bytes, void** out);
int b200_host_free(b200_ctx* ctx, void* ptr);
/* Stream-ordered copies.  b200_write/read are asynchronous when `host` is pinned; call b200_sync before reusing `host`. */
int b200_write(b200_ctx* ctx, b200_stream s, b200_dptr dst, const void* host_src, size_t bytes);
int b200_read(b200_ctx* ctx, b200_stream s, void* host_dst, b200_dptr src, size_t bytes);
int b200_copy(b200_ctx* ctx, b200_stream s, b200_dptr dst, b200_dptr src, size_t bytes);
int b200_memset32(b200_ctx* ctx, b200_stream s, b200_dptr dst, uint32_t value, size_t words);

/* ---- streams / sync / timing: ComputeClient::sync (client.rs:1013), Fence = CUevent (compute/sync/fence.rs) ---------- */
int b200_stream_create(b200_ctx* ctx, b200_stream* out);
int b200_stream_destroy(b200_ctx* ctx, b200_stream s);
int b200_sync(b200_ctx* ctx, b200_stream s);
int b200_event_create(b200_ctx* ctx, b200_event* out);
int b200_event_record(b200_ctx* ctx, b200_event e, b200_stream s);
int b200_stream_wait_event(b200_ctx* ctx, b200_stream s, b200_event e);   /* cross-stream dependency (MultiStream::resolve, stream/event.rs:220) */
int b200_event_elapsed_ms(b200_ctx* ctx, b200_event start, b200_event end, float* ms);
int b200_event_destroy(b200_ctx* ctx, b200_event e);

/* ---- matmul::launch (cubek; shape rule crates/cubecl-zspace/src/shape.rs:489-517) ----------------------------------
 * out[..,m,n] = sum_k lhs[..,m,k] * rhs[..,k,n]; equal rank >= 2, leading dims broadcast (1 vs d); shapes/strides in
 * ELEMENTS (TensorHandle, cubecl-std/src/tensor/handle.rs:13-23).  f32 accumulation over k.  Inputs f16/bf16/f32 with
 * `out_dtype` = the input dtype or F32; fp8 inputs (F8E4M3 / F8E5M2, both operands the same format, kind::f8f6f4) with
 * `out_dtype` BF16, F16 or F32; U8 / I8 inputs (kind::i8) with exact I32 accumulation and `out_dtype` I32.  Row strides may be pitched (allocator.rs:21-72); rhs may be given transposed
 * (stride_k == 1, MatrixBatchLayout::MildlyPermuted{transposed}, matrix_batch_layout.rs:8-19).  f32 inputs run on the tf32
 * tensor pipe, by default with the hybrid split (tf32 main product + bf16 cross terms, f32-grade accuracy; see "gemm.f32").
 * Returns B200_ERR_INVALID_ARG on shape mismatch -- the MatmulShapeError of shape.rs:489-517. */
int b200_matmul(b200_ctx* ctx, b200_stream s, b200_dtype in_dtype, b200_dtype out_dtype,
                b200_dptr lhs, b200_dptr rhs, b200_dptr out, int rank,
                const uint64_t* shape_lhs, const uint64_t* strides_lhs,
                const uint64_t* shape_rhs, const uint64_t* strides_rhs,
                const uint64_t* shape_out, const uint64_t* strides_out);
/* The same product with DIFFERENT 8-bit formats for the two operands -- the pairs the reference instantiates for its manual
 * MMA: i8 x u8 / u8 x i8 -> i32 (crates/cubecl-cpp/src/cuda/mma/manual.rs:151-166) and fp8 e4m3 x e5m2 / e5m2 x e4m3
 * (:170-186).  Same wgmma kernels (the instruction names the type of each operand); equal formats behave exactly like
 * b200_matmul.  Other combinations: B200_ERR_UNSUPPORTED. */
int b200_matmul_mixed(b200_ctx* ctx, b200_stream s, b200_dtype lhs_dtype, b200_dtype rhs_dtype, b200_dtype out_dtype,
                      b200_dptr lhs, b200_dptr rhs, b200_dptr out, int rank,
                      const uint64_t* shape_lhs, const uint64_t* strides_lhs,
                      const uint64_t* shape_rhs, const uint64_t* strides_rhs,
                      const uint64_t* shape_out, const uint64_t* strides_out);

/* Fused epilogue (SURVEY 8f-4): out = act(alpha * (lhs @ rhs) + bias[n]) applied to the f32 accumulators inside the GEMM
 * epilogue (accumulator registers -> here -> staging / store), no extra pass over the output.  bias: f32[N] device pointer or 0.
 * activation: 0 none, 1 relu, 2 gelu (erf form).  Float inputs only. */
typedef struct b200_epilogue {
  float alpha;
  int32_t activation;
  b200_dptr bias;
} b200_epilogue;
int b200_matmul_fused(b200_ctx* ctx, b200_stream s, b200_dtype in_dtype, b200_dtype out_dtype,
                      b200_dptr lhs, b200_dptr rhs, b200_dptr out, int rank,
                      const uint64_t* shape_lhs, const uint64_t* strides_lhs,
                      const uint64_t* shape_rhs, const uint64_t* strides_rhs,
                      const uint64_t* shape_out, const uint64_t* strides_out, const b200_epilogue* epilogue);

/* Block-scaled (MX) matmul: out[b,m,n] = sum_k (lhs[b,m,k] * lhs_scales[b,m,k/32]) * (rhs[b,n,k] * rhs_scales[b,n,k/32]),
 * f32 accumulation.  Replaces MmaDefinition::new_scaled / execute_scaled (crates/cubecl-core/src/frontend/cmma.rs:438-460,
 * 798-840), the ScaledMmaConfig feature rows (crates/cubecl-ir/src/features.rs:190-211; on CUDA the reference offers them
 * for sm_120 only, cubecl-cpp/src/cuda/mma/manual.rs:201-255 -- sm_90 tensor cores take no scales: each operand is expanded
 * once to bf16 x * scale, exactly, and multiplied by the bf16 wgmma GEMM) and is
 * pinned by test_cmma_scaled / test_cmma_scaled_fp4 (crates/cubecl-core/src/runtime_tests/cmma.rs:1476-1700).
 * Layouts follow those tests: lhs [batch, m, k] and rhs [batch, n, k] K-contiguous ("col-major" rhs), dtypes B200_F8E4M3 /
 * B200_F8E5M2 (mixable) or both B200_F4E2M1X2 (k / 2 bytes per row); scales are B200_UE8M0 bytes [batch, rows, k / 32]
 * row-major (scales_packed = 0) or in the packed 128-row chunk form [batch * ceil(rows/128)][ceil(k/128)][512 B],
 * byte (r % 32) * 16 + (r / 32) * 4 + s (scales_packed = 1).  out [batch, m, n] contiguous, f32 / bf16 / f16.
 * scale_block = 32: ue8m0 scales (MXFP8 / MXFP4).  scale_block = 16: NVFP4 -- packed e2m1 operands with e4m3 scale bytes
 * [batch, rows, k / 16] whose sign is ignored (the third ScaledMmaConfig row of manual.rs:241-250).
 * k must be a multiple of 32.  Operands that TMA cannot describe take the reference-order SIMT path. */
int b200_matmul_scaled(b200_ctx* ctx, b200_stream stream, b200_dtype lhs_dtype, b200_dtype rhs_dtype, b200_dtype out_dtype,
                       b200_dptr lhs, b200_dptr rhs, b200_dptr lhs_scales, b200_dptr rhs_scales, b200_dptr out,
                       uint64_t batch, uint64_t m, uint64_t n, uint64_t k, int scale_block, int scales_packed);

/* ---- reduce::launch (cubek) -----------------------------------------------------------------------------------------
 * Reduces `axis` (0..rank-1) of a CONTIGUOUS row-major input, or every element when axis == -1.  Output is contiguous
 * with the reduced axis removed (one element for axis == -1): F32 values, or U32 indices along the axis for arg ops.
 * Input dtype F32 / F16 / BF16, f32 accumulation; `in` needs element alignment only (a sub-slice view is fine: the kernels
 * peel scalar head / tail elements around the 128-bit body).  One launch, no host sync -- two launches when few outputs
 * meet a long axis (segments first, then the partials; deterministic); uses a per-stream workspace owned by ctx. */
int b200_reduce(b200_ctx* ctx, b200_stream s, b200_reduce_op op, b200_dtype in_dtype,
                b200_dptr in, b200_dptr out, int rank, const uint64_t* shape, int axis);

/* Same, for an input described by strides in elements.  Pitched rows (TensorHandle::empty -> PitchedMemoryLayoutPolicy,
 * crates/cubecl-runtime/src/allocator.rs:21-72) and axis permutations that keep the kept axes in order (a transposed view)
 * are reduced IN PLACE -- the kernels take the outer / axis strides and the row pitch, so the traffic is 1x the logical
 * bytes and the padding is never read.  Only views no such description fits (broadcast strides, gaps between outer
 * dimensions, permuted outputs) are first gathered into a pooled compact temporary (into_contiguous,
 * crates/cubecl-std/src/tensor/contiguous.rs).  strides == NULL means contiguous. */
int b200_reduce_strided(b200_ctx* ctx, b200_stream s, b200_reduce_op op, b200_dtype in_dtype,
                        b200_dptr in, b200_dptr out, int rank, const uint64_t* shape, const uint64_t* strides, int axis);
/* Stage timings of the most recent fused reduce + exchange launched on `s` with option "reduce.debug" = 1, in ns:
 * words4[0] = exchange (publish to the peers' mailboxes -> every peer's value seen), words4[1] = partials + f64 tree of the
 * last block; words4[2..3] reserved.  Synchronises the stream. */
int b200_reduce_debug(b200_ctx* ctx, b200_stream s, uint64_t* words4);
/* out (compact row-major) = gather of the strided rank<=8 tensor `in`. */
int b200_into_contiguous(b200_ctx* ctx, b200_stream s, b200_dtype dtype, b200_dptr in, b200_dptr out, int rank,
                         const uint64_t* shape, const uint64_t* strides);

/* ---- scans along an axis: the device-wide form of the plane scans plane_inclusive_sum / plane_exclusive_sum /
 * plane_inclusive_prod / plane_exclusive_prod (crates/cubecl-core/src/runtime_tests/plane.rs:191-405) ---------------------
 * cumsum / cumprod / cummax / cummin of `axis` (0..rank-1): inclusive out[.., l, ..] = x[0] op ... op x[l]; exclusive
 * (exclusive != 0) out[.., 0, ..] = identity (0, 1, -inf, +inf) and out[.., l, ..] = x[0] op ... op x[l-1].  op is SUM, PROD,
 * MAX or MIN (ARGMAX / ARGMIN / MEAN: B200_ERR_UNSUPPORTED); max / min follow b200_reduce's rule (a NaN makes every later
 * output NaN).  Input F32 / F16 / BF16, f32 running values; out_dtype F32 or the input dtype (a 16-bit output is the running
 * value rounded to nearest-even once), anything else B200_ERR_INVALID_ARG.  out is compact row-major with the input's
 * shape.  Contiguous inputs and pitched rows are read in place (any element-aligned base); other views (strides != NULL)
 * are first gathered with b200_into_contiguous.  An extent of 0 is a no-op.  One launch when whole rows / column tiles fill
 * the GPU, else three (segment partials, their exclusive scan, the segments from their carries): bitwise reproducible for
 * the same shape, dtypes and SM count.  Stream-ordered, no host sync, temporaries from the pool. */
int b200_scan(b200_ctx* ctx, b200_stream s, b200_reduce_op op, int exclusive, b200_dtype in_dtype, b200_dtype out_dtype,
              b200_dptr in, b200_dptr out, int rank, const uint64_t* shape, const uint64_t* strides /* NULL = contiguous */,
              int axis);

/* ---- quantize / dequantize along the innermost axis: CubeCL's QuantScheme (crates/cubecl-common/src/quant/scheme.rs) -----
 * Layout.  x is [..., K] (rank >= 1).  Codes are one compact row-major byte stream [..., K * bits / 8]: field i of a row sits
 * at bit offset i * bits, from the low bits upward (8-bit values are bytes; two e2m1 per byte, element 2i in the low nibble,
 * as B200_F4E2M1X2).  Read as little-endian u32 words this stream is the reference's PackedU32(0) store, and it is also its
 * Native / PackedNative(0) store, so the scheme has no store field: K * bits must be a multiple of 8.  Block scales are compact
 * [..., K / block] in the block-scale dtype (for MXFP8 / MXFP4 the row-major scales of b200_matmul_scaled, scales_packed = 0;
 * for E2M1 / 16 / F8E4M3 its scale_block = 16 layout); the tensor scale is one f32.
 * Schemes.  block in {0, 8, 16, 32, 64, 128} (other sizes: B200_ERR_UNSUPPORTED) with K % block == 0; block == 0 is per-tensor
 * f32 only and needs tensor_scale = 1 (a level-less scheme resolves to it, scheme.rs:94-104).  block > 0 with tensor_scale = 1
 * is two-level: b200_quantize takes F16 or F8E4M3 (ue4m3) block scales only (F32 / UE8M0 gain nothing and BF16 drives the
 * global scale subnormal, scheme.rs:200-207: B200_ERR_UNSUPPORTED); b200_dequantize takes every block-scale dtype.
 * Scale rule.  range_max = the positive end of QuantValue::range() (127, 7, 1, 448, 57344, 6); amax = max |x| over FINITE x.
 * One level: s = round_up(amax / range_max) in the scale dtype.  Two levels: g = (amax_tensor / range_max) /
 * max_representable(block dtype), s_b = round_up((amax_b / range_max) / g) (0 for a block whose amax is 0), effective scale
 * g * f32(s_b) rounded once in f32.  round_up is ScaleDtype::round_up bit for bit for F32 / F16 / BF16 / UE4M3; UE8M0, which the
 * reference leaves unimplemented, takes the smallest power of two >= s, clamped to codes 0..254 (unlike the OCP MX recipe
 * floor(log2 amax) - emax, it never clips the block maximum).  IEEE f32 throughout, division by `/`.
 * Encoding.  q = x / eff; integers: round half to even, clamp to range(); e4m3 / e5m2: round to nearest even, satfinite;
 * e2m1: round to nearest, ties to the even code, saturating at +-6.  A zero scale gives code 0; +-inf saturates to the range
 * end; NaN gives code 0 (integers, e2m1) or 0x7F (fp8).
 * Dequantize.  out = RNE(f32(q) * eff) in F32 / F16 / BF16, compact.  Integer fields are sign-extended; ue8m0 scales are
 * 2^(b-127) (255 = NaN); e4m3 scales are read with the sign ignored.
 * Malformed input is B200_ERR_INVALID_ARG: K not divisible, a sub-byte row, a null pointer for a present level or a non-null
 * one for an absent level, a dtype or value outside the lists (block_scale is only read when block > 0).  An extent of 0 is a no-op.  Stream-ordered, no host sync,
 * temporaries from the pool.  Inputs F32 / F16 / BF16: contiguous tensors and pitched rows with 16-byte aligned base and rows
 * are read in place, any other view is first gathered with b200_into_contiguous.  A scheme with a tensor level runs a
 * memset, an absmax pass and the encode pass; a block-only scheme is one launch; dequantize is one launch. */
typedef enum b200_quant_value {            /* QuantValue, scheme.rs:358-377, in its order */
  B200_QV_Q8F = 0, B200_QV_E5M2 = 1, B200_QV_E4M3 = 2, B200_QV_Q4F = 3, B200_QV_E2M1 = 4,
  B200_QV_Q2F = 5, B200_QV_Q8S = 6, B200_QV_Q4S = 7, B200_QV_Q2S = 8
} b200_quant_value;
typedef struct b200_quant_scheme {
  int32_t value;         /* b200_quant_value */
  int32_t block;         /* values per block scale along the innermost axis; 0 = no block level */
  int32_t block_scale;   /* b200_dtype: F32, F16, BF16, UE8M0, F8E4M3 (= ue4m3: written with the sign clear); ignored when block == 0 */
  int32_t tensor_scale;  /* 1 = one f32 per-tensor scale (the only level, or the global level over the blocks) */
} b200_quant_scheme;
int b200_quantize(b200_ctx* ctx, b200_stream s, const b200_quant_scheme* scheme, b200_dtype in_dtype, b200_dptr in,
                  b200_dptr values, b200_dptr block_scales, b200_dptr tensor_scale,
                  int rank, const uint64_t* shape, const uint64_t* strides /* NULL = contiguous */);
int b200_dequantize(b200_ctx* ctx, b200_stream s, const b200_quant_scheme* scheme, b200_dtype out_dtype,
                    b200_dptr values, b200_dptr block_scales, b200_dptr tensor_scale, b200_dptr out,
                    int rank, const uint64_t* shape);

/* ---- matmul of integer-quantized operands on the s8 tensor cores, scales applied inside the GEMM ----------------------------
 * out[b, m, n] = sum_k deq(lhs)[b, m, k] * deq(rhs)[b, n, k]; lhs holds codes [batch, M, K], rhs [batch, N, K], both quantized
 * along K exactly as b200_quantize writes them (values, block_scales, tensor_scale as there); out is [batch, M, N] contiguous
 * in F32 / BF16 / F16.  Values Q8F / Q8S / Q4F / Q4S / Q2F / Q2S, independently per side (Q8 bytes feed the tensor cores, Q4 / Q2
 * codes are first widened exactly to one s8 per element); per-tensor, per-block (32, 64, 128) or two-level on either side, every
 * block-scale dtype b200_dequantize reads.  Tensor scales are read on the device: no host sync, b200_quantize and this call
 * may be enqueued back to back.
 * Arithmetic (bit-exact; integer fields sign-extended as b200_dequantize reads them).  eff_x[b, r, j] is the effective scale of
 * block j of row r as b200_dequantize defines it: f32(s), rn(g * f32(s)) with two levels, g for a per-tensor side.
 *   Per-block (either side has a block level): Bk = the smaller present block; a coarser block repeats its scale and a
 *   per-tensor side uses g for every block.  D_j = the exact integer dot product over block j (|D_j| <= 2^21).  Blocks fold in
 *   increasing j: acc_0 = 0, acc_{j+1} = fma(f32(D_j), rn(eff_a[m, j] * eff_b[n, j]), acc_j); out = RNE(acc_J).
 *   Per-tensor x per-tensor: D = the exact s32 dot product over K (needs K < 131072); out = RNE(rn(rn(f32(D)) * rn(g_a * g_b))).
 *   NaN and inf scales propagate as IEEE says.  No stream-K head runs: every output is one serial fold, reproducible bit for bit.
 * Errors: B200_ERR_INVALID_ARG for K not divisible by a block, a null pointer for a present level or a non-null one for an absent
 * level, an unknown value or dtype, K == 0 with a non-empty output; B200_ERR_UNSUPPORTED for minifloat values (use
 * b200_matmul_scaled), blocks of 8 or 16, and per-tensor x per-tensor with K >= 131072.  batch, M or N of 0 is a no-op.
 * Launches: per-tensor x per-tensor 1; per-block 2 scale passes + 1 GEMM; +1 per Q4 / Q2 operand (widening) and per Q8 operand
 * TMA cannot read in place (base not 16-byte aligned or K % 16 != 0: staging).  Temporaries come from the pool, stream-ordered. */
typedef struct b200_quant_operand {
  b200_quant_scheme scheme;   /* as passed to b200_quantize */
  b200_dptr values;           /* codes [batch, rows, K * bits / 8], the compact bit stream b200_quantize writes */
  b200_dptr block_scales;     /* [batch, rows, K / block] in scheme.block_scale, or 0 when block == 0 */
  b200_dptr tensor_scale;     /* f32[1] ON THE DEVICE, or 0 when the scheme has no tensor level */
} b200_quant_operand;
int b200_matmul_quantized(b200_ctx* ctx, b200_stream s, const b200_quant_operand* lhs, const b200_quant_operand* rhs,
                          b200_dtype out_dtype, b200_dptr out, uint64_t batch, uint64_t m, uint64_t n, uint64_t k);

/* ---- 2-D convolution (cubek's convolution kernels), an implicit GEMM on the wgmma kernel --------------------------------
 * out[n, oh, ow, co] = act(alpha * sum_{ky, kx, c} x[n, oh*sh - ph + ky*dh, ow*sw - pw + kx*dw, c] * w[co, ky, kx, c] + bias[co]).
 * Input outside x reads as zero; f32 accumulation; the epilogue is b200_epilogue (NULL = none).  x is [N, H, W, C] (NHWC), w is
 * [Cout, KH, KW, C], out is [N, OH, OW, Cout] with OH = floor((H + 2*ph - dh*(KH-1) - 1) / sh) + 1 and OW likewise (PyTorch's
 * rule).  Shapes and strides in elements; NULL strides = compact.
 * Dtypes: F16 or BF16 inputs; out_dtype the input dtype or F32 (the rule of b200_matmul); anything else B200_ERR_UNSUPPORTED.
 * Views: x with unit channel stride and 16-byte aligned base and strides, and w whose (KH, KW) flatten into one stride with
 * the same alignment, are read in place (compact NHWC x and compact [Cout, KH, KW, C] w are); any other view (NCHW x, PyTorch's
 * OIHW weights passed as a stride-permuted view) is first gathered with b200_into_contiguous.  out needs a unit channel
 * stride and outer strides that flatten to one pixel pitch >= Cout (a channel slice of a wider NHWC tensor is fine).  When
 * C * 2 bytes is not a multiple of 16 (e.g. an RGB stem, C = 3) both operands are copied with C padded to a multiple of 8
 * zero channels.
 * Errors: B200_ERR_INVALID_ARG for a channel mismatch, a wrong out_shape, OH or OW < 1, stride / dilation < 1, negative padding,
 * an unknown activation or a null pointer; B200_ERR_UNSUPPORTED for shapes outside the 4-D im2col limits: pixel-box corners
 * -p and p - d*(K-1) in [-128, 127], conv strides <= 8, N*OH*OW < 2^31.  An extent of 0 in x or w is a no-op.
 * Launches: 1 (the GEMM) for in-place operands; +1 per gathered operand; when C * 2 % 16 != 0, +1 per operand (the channel
 * padding copy) and +1 more for an operand whose spatial dimensions do not flatten into one stride.  Stream-ordered, no host
 * sync, temporaries from the pool; bitwise reproducible for a fixed shape, dtypes and SM count.  The tile is chosen like
 * b200_matmul's ("gemm.variant" 2sm_n128 | 1sm_n128, "gemm.split_k", "gemm.epilogue" apply). */
typedef struct b200_conv2d_args {
  int32_t stride_h, stride_w, pad_h, pad_w, dilation_h, dilation_w;
} b200_conv2d_args;
int b200_conv2d(b200_ctx* ctx, b200_stream s, b200_dtype in_dtype, b200_dtype out_dtype,
                b200_dptr x, const uint64_t* x_shape, const uint64_t* x_strides,
                b200_dptr w, const uint64_t* w_shape, const uint64_t* w_strides,
                b200_dptr out, const uint64_t* out_shape, const uint64_t* out_strides,
                const b200_conv2d_args* args, const b200_epilogue* epilogue);

/* Gradients of b200_conv2d (same args, same NHWC / [Cout, KH, KW, C] layouts, f32 accumulation, no epilogue).
 *   dx[n, h, w, c]    = sum over (oh, ow, ky, kx) with oh*sh - ph + ky*dh = h, ow*sw - pw + kx*dw = w of dy[n, oh, ow, co] * w[co, ky, kx, c]
 *   dw[co, ky, kx, c] = sum over (n, oh, ow) of dy[n, oh, ow, co] * x[n, oh*sh - ph + ky*dh, ow*sw - pw + kx*dw, c]
 * dy must have the shape b200_conv2d gives for (dx or x, w or dw, args): [N, OH, OW, Cout]; that admits every H and W that
 * PyTorch's output_padding admits.  The bias gradient needs no entry point: it is b200_reduce (sum) over axis 0 of dy viewed as
 * [N * OH * OW, Cout].
 * Dtypes: F16 or BF16 dy / w / x; out_dtype the input dtype or F32.
 * Views: dy and x follow b200_conv2d's input rules (gathered when not readable in place; C or Cout with C * 2 % 16 != 0 copied
 * with the channels padded to 8 zeros); b200_conv2d_backward_weight also gathers a dy whose pixels do not share one pitch.
 * backward_data reads w through any strides.  dx follows b200_conv2d's out rule (unit channel stride, one pixel pitch >= C).
 * dw needs a unit channel stride, (KH, KW) flattening into one stride and any Cout stride; other dw views get
 * B200_ERR_UNSUPPORTED.
 * Errors: B200_ERR_INVALID_ARG for a channel mismatch, a dy shape that is not the output rule's, stride / dilation < 1, negative
 * padding or a null pointer; B200_ERR_UNSUPPORTED for strides > 8, pixel-box corners outside [-128, 127] (backward_weight: the
 * forward's corners; backward_data: per output phase, below), N*H*W or N*OH*OW >= 2^31.  An empty dx / dw is a no-op; when dy
 * has no pixels (N = 0) dw is written as zeros, and when Cout = 0 dx is.
 *
 * backward_data: with stride 1, dx is a stride-1 convolution of dy with the flipped, channel-transposed weights
 * w'[c, ky', kx', co] = w[co, KH-1-ky', KW-1-kx', c]: launches = 1 weight-prep kernel + 1 conv2d GEMM.  With stride > 1, dx
 * splits into sh * sw phases (h = rh + sh*i, w = rw + sw*j); each phase is a stride-1 convolution of dy over the taps
 * ky with (rh + ph - ky*dh) % sh == 0 (dilation dh / gcd(sh, dh)), one conv2d_dgrad GEMM per phase with taps and pixels, whose
 * epilogue stores its rows straight into dx.  Its pixel-box corners are the first tap's dy offset and that offset + the
 * phase extent - OH (likewise for w).  Phases no tap reaches (a 1x1 stride-2 layer has three) are exact zeros: one memset of
 * dx, only when such a phase exists.  Temporaries: the prepared weights (|w| elements, Cout padded to 8) plus dy's copies.
 * backward_weight: one conv2d_wgrad GEMM with M = Cout, N = KH * KW * pad64(C), K = N * OH * OW; dy is read as an MN-major
 * [pixels, Cout] operand, x through a 64-pixel im2col load per (kernel position, 64-channel block).  K is long and the tiles are
 * few, so the stream-K head ("gemm.split_k" auto) may cut a tile into more than 8 k-ranges (each >= 8 k-blocks of 64 pixels),
 * reduced in k order.
 * Both: stream-ordered, no host sync, temporaries from the pool, bitwise reproducible for a fixed shape, dtypes and SM count;
 * "gemm.variant" (2sm_n128 | 1sm_n128), "gemm.split_k" and "gemm.epilogue" apply (backward_data's stride > 1 phases always
 * store directly). */
int b200_conv2d_backward_data(b200_ctx* ctx, b200_stream s, b200_dtype in_dtype, b200_dtype out_dtype,
                              b200_dptr dy, const uint64_t* dy_shape, const uint64_t* dy_strides,
                              b200_dptr w, const uint64_t* w_shape, const uint64_t* w_strides,
                              b200_dptr dx, const uint64_t* dx_shape, const uint64_t* dx_strides,
                              const b200_conv2d_args* args);
int b200_conv2d_backward_weight(b200_ctx* ctx, b200_stream s, b200_dtype in_dtype, b200_dtype out_dtype,
                                b200_dptr x, const uint64_t* x_shape, const uint64_t* x_strides,
                                b200_dptr dy, const uint64_t* dy_shape, const uint64_t* dy_strides,
                                b200_dptr dw, const uint64_t* dw_shape, const uint64_t* dw_strides,
                                const b200_conv2d_args* args);

/* ---- grouped and depthwise 2-D convolution, forward and both gradients ------------------------------------------------
 * As b200_conv2d / _backward_data / _backward_weight with `groups` > 1 groups: x is [N, H, W, C], w and dw are
 * [Cout, KH, KW, Cg] with Cg = C / groups (PyTorch's grouped weight [Cout, C / groups, KH, KW] permuted as for b200_conv2d),
 * out and dy are [N, OH, OW, Cout].  Group g owns input channels [g Cg, (g+1) Cg) and output channels [g Coutg, (g+1) Coutg),
 * Coutg = Cout / groups; any channel multiplier Coutg / Cg is allowed (groups = C is depthwise).
 *   out[n, oh, ow, co] = act(alpha * sum_{ky, kx, ci < Cg} x[n, oh*sh - ph + ky*dh, ow*sw - pw + kx*dw, g*Cg + ci] * w[co, ky, kx, ci]
 *                            + bias[co]),  g = co / Coutg
 * and the gradients of that sum (f32 accumulation, no epilogue; the bias gradient is b200_reduce over axis 0 of dy).  Input
 * outside x reads as +0 and is multiplied like any other element (an inf weight gives NaN at a padded window).  A NaN or inf
 * in group g's input or dy channels reaches only group g's outputs.  Dtypes, stride / padding / dilation limits, the
 * output-shape rule, the out / dx / dw view rules and the zero-extent rules are those of the groups == 1 functions.
 * Errors: B200_ERR_INVALID_ARG for groups == 0, C or Cout not divisible by groups, or a weight channel extent != C / groups,
 * plus the groups == 1 functions' errors; B200_ERR_UNSUPPORTED for their limits.
 * Routing (from the shape alone):
 *   groups == 1: the groups == 1 function itself (same plan, same bits).
 *   Cg >= 64: one groups == 1 call per group on channel slices (x, dy, out, dx in place through their pixel pitch; w and dw
 *     as row blocks); a slice whose base is not 16-byte aligned takes that function's gather or padding copy.
 *   Cg < 64: direct NHWC kernels on the CUDA cores, one launch each (+1 per x / dy / w view without a unit channel stride,
 *     which is gathered first), in a fixed order of f32 FMAs, bitwise reproducible:
 *     forward (conv2d_grp_*): acc = +0; for ky, kx, ci ascending: acc = fma(x, w, acc); then the epilogue.
 *     backward_data (conv2d_grp_dgrad_*): acc = +0; for ky, kx ascending over the taps with (h + ph - ky*dh) % sh == 0 and
 *       (w + pw - kx*dw) % sw == 0, then co in the group ascending: acc = fma(dy, w, acc); dy reads as +0 outside
 *       [0, OH) x [0, OW).
 *     backward_weight (conv2d_grp_wgrad_*): the P = N*OH*OW pixels are cut into segments of L pixels, with
 *       E = Cout*KH*KW*Cg, S' = min(4096, max(1, ceil(2^18 / E))), L = max(64, ceil(P / S')), S = ceil(P / L) (1 when P = 0).
 *       Per segment, acc = +0; for pixels ascending (n, oh, ow order): acc = fma(dy, x, acc).  S == 1 writes dw directly;
 *       otherwise the f32 partials go to a pooled S * E * 4-byte buffer and conv2d_grp_wgrad_combine_* writes
 *       dw = ((p_0 + p_1) + p_2) + ....  The dry-run plan records "conv grouped wgrad pixels= elements= segments= length=". */
int b200_conv2d_grouped(b200_ctx* ctx, b200_stream s, b200_dtype in_dtype, b200_dtype out_dtype,
                        b200_dptr x, const uint64_t* x_shape, const uint64_t* x_strides,
                        b200_dptr w, const uint64_t* w_shape, const uint64_t* w_strides,
                        b200_dptr out, const uint64_t* out_shape, const uint64_t* out_strides,
                        const b200_conv2d_args* args, uint32_t groups, const b200_epilogue* epilogue);
int b200_conv2d_grouped_backward_data(b200_ctx* ctx, b200_stream s, b200_dtype in_dtype, b200_dtype out_dtype,
                                      b200_dptr dy, const uint64_t* dy_shape, const uint64_t* dy_strides,
                                      b200_dptr w, const uint64_t* w_shape, const uint64_t* w_strides,
                                      b200_dptr dx, const uint64_t* dx_shape, const uint64_t* dx_strides,
                                      const b200_conv2d_args* args, uint32_t groups);
int b200_conv2d_grouped_backward_weight(b200_ctx* ctx, b200_stream s, b200_dtype in_dtype, b200_dtype out_dtype,
                                        b200_dptr x, const uint64_t* x_shape, const uint64_t* x_strides,
                                        b200_dptr dy, const uint64_t* dy_shape, const uint64_t* dy_strides,
                                        b200_dptr dw, const uint64_t* dw_shape, const uint64_t* dw_strides,
                                        const b200_conv2d_args* args, uint32_t groups);

/* ---- 3-D convolution, forward and both gradients, an implicit GEMM on the wgmma kernel -----------------------------------
 * out[n, od, oh, ow, co] = act(alpha * sum_{kz, ky, kx, c} x[n, od*sd - pd + kz*dd, oh*sh - ph + ky*dh, ow*sw - pw + kx*dw, c]
 *                              * w[co, kz, ky, kx, c] + bias[co])
 * x is [N, D, H, W, C] (NDHWC), w is [Cout, KD, KH, KW, C] (PyTorch's OIDHW weight permuted as for b200_conv2d), out and dy
 * are [N, OD, OH, OW, Cout] with PyTorch's output rule in each dimension.  The gradients are b200_conv2d's with the depth term
 * added; the bias gradient is b200_reduce (sum) over axis 0 of dy viewed as [N * OD * OH * OW, Cout].  No groups argument.
 * Every rule that is not specific to 3-D is b200_conv2d's (and its gradients'): F16 / BF16 in, out the input dtype or F32,
 * anything else B200_ERR_UNSUPPORTED; zero extents are no-ops (the gradients' zero-fill rules apply); INVALID_ARG versus
 * UNSUPPORTED as for 2-D; bitwise reproducible for a fixed shape, dtypes and SM count; "gemm.variant" (2sm_n128 | 1sm_n128),
 * "gemm.split_k" and "gemm.epilogue" apply.  Inputs with unit channel stride and 16-byte aligned base and strides are read in
 * place (w and dw need (KD, KH, KW) to flatten into one stride); any other view is gathered at rank 5, and C * 2 % 16 != 0
 * is copied with the channels padded to 8.  out and dx need a unit channel stride and one pixel pitch >= their channels
 * across N, D, H and W.
 * Limits of the 5-D im2col map, B200_ERR_UNSUPPORTED, each named in the message:
 *   corners: pixel-box corners in [-16, 15] (cuTensorMapEncodeIm2col, rank 5): -p and p - d*(K-1) per dimension for the
 *     forward and backward_weight, each phase's lower and upper corner for backward_data;
 *   offsets: the load's im2col offsets kx*dw, ky*dh, kz*dd are 5-bit for rank 5 (PTX ISA), so d*(K-1) <= 31 per dimension
 *     (backward_data: the phase's (taps - 1) * dilation);
 *   stride: <= 8 per dimension;
 *   size: N*OD*OH*OW < 2^31 (backward_data also N*D*H*W), KD*KH*KW*pad64(C) < 2^31.
 * backward_data: dx splits into sd*sh*sw phases (d = rd + sd*a, h = rh + sh*i, w = rw + sw*j); one conv3d_dgrad_weights launch
 * writes every phase's flipped, channel-transposed weights into one buffer of |w| elements, then stride 1 runs one conv3d GEMM
 * and stride > 1 one conv3d_dgrad GEMM per phase with taps and pixels, plus one memset of dx when some phase receives no tap.
 * The dry-run plan records each phase as "conv3d dgrad phase r=(rd,rh,rw) taps_d= taps_h= taps_w= dil= lower= upper= extent=".
 * backward_weight: one conv3d_wgrad GEMM with M = Cout, N = KD*KH*KW*pad64(C), K = N*OD*OH*OW (stream-K head as 2-D). */
typedef struct b200_conv3d_args {
  int32_t stride_d, stride_h, stride_w, pad_d, pad_h, pad_w, dilation_d, dilation_h, dilation_w;
} b200_conv3d_args;
int b200_conv3d(b200_ctx* ctx, b200_stream s, b200_dtype in_dtype, b200_dtype out_dtype,
                b200_dptr x, const uint64_t* x_shape, const uint64_t* x_strides,
                b200_dptr w, const uint64_t* w_shape, const uint64_t* w_strides,
                b200_dptr out, const uint64_t* out_shape, const uint64_t* out_strides,
                const b200_conv3d_args* args, const b200_epilogue* epilogue);
int b200_conv3d_backward_data(b200_ctx* ctx, b200_stream s, b200_dtype in_dtype, b200_dtype out_dtype,
                              b200_dptr dy, const uint64_t* dy_shape, const uint64_t* dy_strides,
                              b200_dptr w, const uint64_t* w_shape, const uint64_t* w_strides,
                              b200_dptr dx, const uint64_t* dx_shape, const uint64_t* dx_strides,
                              const b200_conv3d_args* args);
int b200_conv3d_backward_weight(b200_ctx* ctx, b200_stream s, b200_dtype in_dtype, b200_dtype out_dtype,
                                b200_dptr x, const uint64_t* x_shape, const uint64_t* x_strides,
                                b200_dptr dy, const uint64_t* dy_shape, const uint64_t* dy_strides,
                                b200_dptr dw, const uint64_t* dw_shape, const uint64_t* dw_strides,
                                const b200_conv3d_args* args);

/* ---- transposed convolution, 2-D and 3-D (PyTorch's ConvTranspose2d / 3d), with the fused epilogue -----------------------
 * out[n, oh, ow, co] = act(alpha * sum_{ih, iw, ky, kx, ci : oh = ih*sh - ph + ky*dh, ow = iw*sw - pw + kx*dw}
 *                                  x[n, ih, iw, ci] * w[ci, ky, kx, co] + bias[co])
 * x is [N, H, W, Cin] (NHWC), w is [Cin, KH, KW, Cout] (PyTorch's [Cin, Cout, KH, KW] permuted), out is [N, OH, OW, Cout]
 * with OH = (H-1)*sh - 2*ph + dh*(KH-1) + oph + 1, 0 <= oph < sh (likewise OW; 3-D adds D / KD / sd / pd / dd / opd with
 * the NDHWC layouts of b200_conv3d).  output_padding is no argument: out_shape implies it, and exactly the output extents
 * that b200_conv2d's output rule maps back to x's extents are accepted (PyTorch's stride <= oph < dilation is refused with
 * B200_ERR_UNSUPPORTED).  A position the sum does not reach is act(bias[co]) (act(0) without a bias).  No groups argument.
 * This is b200_conv2d_backward_data / b200_conv3d_backward_data with x in dy's role (w has exactly their w layout:
 * [Cin, KH, KW, Cout] is [Cout_conv, KH, KW, C_conv]) plus the epilogue, and every rule is theirs: dtypes, views, channel
 * padding, the out pixel-pitch rule, the corner / offset / stride <= 8 / pixel-count limits (each phase's corners), the
 * error codes; zero extents of out are no-ops.  Unlike there, the stride <= 8 limit holds for every kernel shape, and an
 * empty kernel (some kernel extent 0, Cin = 0 alike: out is act(bias)) needs x's batch, Cin = w's first extent, C = w's
 * last, and per dimension the output rule above with 0 <= op < s (B200_ERR_INVALID_ARG otherwise).
 * Launches: stride 1 in every dimension is one phase: the weight prep (conv_dgrad_weights / conv3d_dgrad_weights) and one
 *   conv2d_* / conv3d_* forward GEMM with the epilogue.  Stride > 1: the prep and then every phase with pixels, those no tap
 *   reaches included, in conv2d_tconv_* / conv3d_tconv_* launches of up to 8 phases each (one launch for any stride-2
 *   layer), phases with the most k-blocks first; no memset.
 * The dry-run plan records each phase, in walk order, as "conv tconv phase r=(rh,rw) taps_h= taps_w= dil= lower= upper=
 * extent= kblocks=" (3-D: "conv3d tconv phase r=(rd,rh,rw) taps_d= ...").
 * Gradients are existing entry points with roles swapped (same args):
 *   dx    = b200_conv2d(dy, w) -- w read as conv weights with Cout := Cin, no flip;
 *   dw    = b200_conv2d_backward_weight(x := dy, dy := x);
 *   dbias = b200_reduce (sum) over axis 0 of dy viewed as [N * OH * OW, Cout].
 * (3-D: b200_conv3d, b200_conv3d_backward_weight.) */
int b200_conv_transpose2d(b200_ctx* ctx, b200_stream s, b200_dtype in_dtype, b200_dtype out_dtype,
                          b200_dptr x, const uint64_t* x_shape, const uint64_t* x_strides,
                          b200_dptr w, const uint64_t* w_shape, const uint64_t* w_strides,
                          b200_dptr out, const uint64_t* out_shape, const uint64_t* out_strides,
                          const b200_conv2d_args* args, const b200_epilogue* epilogue);
int b200_conv_transpose3d(b200_ctx* ctx, b200_stream s, b200_dtype in_dtype, b200_dtype out_dtype,
                          b200_dptr x, const uint64_t* x_shape, const uint64_t* x_strides,
                          b200_dptr w, const uint64_t* w_shape, const uint64_t* w_strides,
                          b200_dptr out, const uint64_t* out_shape, const uint64_t* out_strides,
                          const b200_conv3d_args* args, const b200_epilogue* epilogue);

/* ---- fused scaled-dot-product attention, forward (PyTorch's scaled_dot_product_attention) ---------------------------------
 * out[b, h, i, :] = sum_j softmax_j(scale * q[b, h, i, :] . k[b, h / G, j, :]) * v[b, h / G, j, :]      G = Hq / Hkv
 * lse[b, h, i]    = log sum_j exp(scale * q[b, h, i, :] . k[b, h / G, j, :])                         (natural log, f32)
 * q is [B, Hq, Sq, D], k and v are [B, Hkv, Sk, D], out is [B, Hq, Sq, D]: shapes and strides in elements, so [B, S, H, D]
 * tensors and the q / k / v slices of a fused [B, S, 3, H, D] projection are stride-permuted views read with no copy.
 * Hq % Hkv == 0 (GQA / MQA, torch's enable_gqa=True).  causal != 0: key j is visible to query i only when j <= i (top-left
 * alignment, torch's is_causal=True); every row then sees key 0, so no row is empty.  scale: any finite float.
 * Dtypes: in_dtype B200_F16 or B200_BF16 for q, k and v; out_dtype the input dtype or B200_F32.  D <= 128, D % 8 == 0, v's
 * head dim equal to D.  A D that is not a multiple of 64 is read with the tensor-map box past D zero-filled (exact for both
 * products) and the store is clipped to D.
 * Numerics: scores are f32 sums of exact 16-bit products.  The softmax runs in base 2 with a running row maximum: t = s *
 * (scale * log2 e) is formed once per score and p = exp2(t - m), so the row's maximal score contributes exp2(0) = 1 exactly
 * (an argument below -126 gives +0).  P is rounded (RNE) to the input dtype before the P.V product; the row sum l adds the
 * f32 p values.  out = O / l (f32 division) rounded once (RNE) to out_dtype; lse = (m + log2 l) * ln 2.  Bitwise
 * reproducible for fixed shapes, dtypes and views: every output row is produced by one CTA in increasing key order (no
 * atomics, no split over keys).
 * Views: q, k and v are read in place when their D stride is 1 and the base and the S, H and B strides are 16-byte aligned;
 * any other view is first gathered into a compact [B, H, S, D] pooled temporary with b200_into_contiguous (one extra launch
 * per operand).  out needs a unit D stride and a 16-byte aligned base and strides, else B200_ERR_UNSUPPORTED naming out.
 * lse: 0 (not written) or an f32 [B, Hq, Sq] compact buffer, 4-byte aligned.
 * Errors: B200_ERR_INVALID_ARG for mismatched B or D, Hkv == 0 or Hq % Hkv != 0, a k / v shape mismatch, a wrong out shape,
 * Sk == 0 with Sq > 0, a non-finite scale, or a null pointer (rank 4 is implied by the shape arrays; the wrappers refuse
 * other ranks with B200_ERR_INVALID_ARG); B200_ERR_UNSUPPORTED for the dtypes, D > 128, D % 8 != 0, Dv != D, extents >= 2^31
 * or more than 2^31 - 1 CTAs.  Zero extents: B, Hq or Sq = 0 is a no-op with no launch.
 * Launches: the gathers, then one attn_fwd_<in>_d<64|128>_<out> launch (D <= 64: the d64 kernel) of ceil(Sq / 128) * Hq * B
 * CTAs, queued on `s` with no host synchronisation; temporaries come from the pool in stream order (as the convolution
 * entries).  The dry-run plan records each 4-D tensor map as "tmap4d esz= dims=(D,S,H,B) strides=(S,H,B bytes) box=(..)
 * swizzle=" in the order q, k, v, out.  b200_last_kernel names the kernel. */
typedef struct b200_attention_args {
  float scale;       /* multiplies q.k before the softmax */
  int32_t causal;    /* 1: key j visible to query i iff j <= i (top-left) */
} b200_attention_args;
int b200_attention(b200_ctx* ctx, b200_stream s, b200_dtype in_dtype, b200_dtype out_dtype,
                   b200_dptr q, const uint64_t* q_shape, const uint64_t* q_strides,
                   b200_dptr k, const uint64_t* k_shape, const uint64_t* k_strides,
                   b200_dptr v, const uint64_t* v_shape, const uint64_t* v_strides,
                   b200_dptr out, const uint64_t* out_shape, const uint64_t* out_strides,
                   b200_dptr lse, const b200_attention_args* args);

/* ---- fused scaled-dot-product attention, backward (PyTorch's SDPA backward, given the forward's out and lse) --------------
 * With P_ij = exp(scale * q_i . k_j - lse_i) (0 for keys hidden by causal), delta_i = sum_d dout_id * out_id and
 * dS_ij = P_ij * (dout_i . v_j - delta_i):
 *   dq_i = scale * sum_j dS_ij k_j      dk_j = scale * sum_{h in group, i} dS_ij q_i      dv_j = sum_{h in group, i} P_ij dout_i
 * (with GQA / MQA, dk and dv of kv head hk sum over the G = Hq / Hkv query heads that read it).  q, out, dout and dq are
 * [B, Hq, Sq, D]; k, v, dk and dv are [B, Hkv, Sk, D]; lse is the forward's compact f32 [B, Hq, Sq] (b200_attention's lse
 * output, natural log).  args, dtypes of q / k / v, views, causal rule and D limits are b200_attention's; out is in the input
 * dtype or f32 (out_dtype), dout in the input dtype, dq, dk and dv all in grad_dtype (the input dtype or B200_F32).
 * Numerics: t = s * (scale * log2 e) with the forward's f32 factor, so the recomputed scores are the forward's bit for bit;
 * L_i = lse_i * log2 e is formed once per row in f32 and p = exp2(t - L) (ex2.approx.ftz).  dS is formed in f32 from the f32
 * p; P and dS are rounded (RNE) to the input dtype for the products dV += P^T dO, dK += dS^T Q and dQ += dS K.  delta is an
 * f32 sum.  dq, dk and dv are f32 sums, multiplied by scale (dq, dk) in f32 and rounded once (RNE) to grad_dtype.  Bitwise
 * reproducible for fixed shapes, dtypes and views: every dq row comes from one CTA in increasing key order, every dk / dv row
 * from one CTA in (group head, query block) order; no atomics.  Q.K^T and dO.V^T are computed by both the dq and the dk / dv
 * kernel (7 GEMM-sized products where an atomic dq needs 5).
 * Views: q, k, v, out and dout are read in place under b200_attention's rule for its inputs, else gathered into a compact
 * pooled copy (one b200_into_contiguous launch each).  dq, dk and dv need a unit D stride and a 16-byte aligned base and
 * strides (so they can be the slices of one fused [B, S, 3, H, D] gradient buffer), else B200_ERR_UNSUPPORTED naming the
 * tensor.  lse must be non-null and 4-byte aligned.
 * dk and dv are always written in full: a key no query sees gets +0 (causal with j >= Sq, and every key when Sq = 0 or
 * Hq = 0).  Only B = 0, or Sk = 0 together with Sq = 0, launches nothing.
 * Errors: as b200_attention, plus B200_ERR_INVALID_ARG when out, dout or dq differ from q's shape or dk or dv from k's, a
 * null or misaligned lse; B200_ERR_UNSUPPORTED for an out_dtype or grad_dtype other than the input dtype or f32.
 * Launches, all on `s` with no host synchronisation: the gathers; a pooled f32 workspace of 2 * B * Hq * ceil(Sq / 128) * 128
 * values ("alloc"); attn_bwd_delta_<in>_<out> (ceil(rows / 16) blocks of 256 threads); attn_bwd_dq_<in>_d<64|128>_<grad>
 * (ceil(Sq / 128) * Hq * B CTAs) after its maps q, k, v, dout, dq; attn_bwd_dkdv_<in>_d<64|128>_<grad> (ceil(Sk / 128) *
 * Hkv * B CTAs) after its maps q, k, v, dout, dk, dv.  With Sq = 0 or Hq = 0 only the dk / dv kernel runs (its q and dout
 * maps then describe k and are never read).  The maps are "tmap4d" plan lines as b200_attention's. */
int b200_attention_backward(b200_ctx* ctx, b200_stream s, b200_dtype in_dtype, b200_dtype out_dtype, b200_dtype grad_dtype,
                            b200_dptr q, const uint64_t* q_shape, const uint64_t* q_strides,
                            b200_dptr k, const uint64_t* k_shape, const uint64_t* k_strides,
                            b200_dptr v, const uint64_t* v_shape, const uint64_t* v_strides,
                            b200_dptr out, const uint64_t* out_shape, const uint64_t* out_strides,
                            b200_dptr dout, const uint64_t* dout_shape, const uint64_t* dout_strides,
                            b200_dptr lse,
                            b200_dptr dq, const uint64_t* dq_shape, const uint64_t* dq_strides,
                            b200_dptr dk, const uint64_t* dk_shape, const uint64_t* dk_strides,
                            b200_dptr dv, const uint64_t* dv_shape, const uint64_t* dv_strides,
                            const b200_attention_args* args);

/* ---- variable-length (packed) attention, forward (flash_attn_varlen_func, torch.nn.attention.varlen.varlen_attn) -----------
 * B sequences packed along one token axis.  q and out are [Tq, Hq, D], k and v [Tk, Hkv, D] (shapes and strides in elements,
 * so the q / k / v slices of a fused [T, 3, H, D] projection are views read with no copy); Hq % Hkv == 0 (GQA / MQA, hk = h /
 * (Hq / Hkv)).  Sequence b owns query rows [cu_q[b], cu_q[b + 1]) and key rows [cu_k[b], cu_k[b + 1]), lengths Lq_b and Lk_b:
 *   out[cu_q[b] + i, h, :] = sum_{j visible} softmax_j(scale * q_i . k_j) * v_j          (k_j, v_j: row cu_k[b] + j, head hk)
 *   lse[h, cu_q[b] + i]    = log sum_{j visible} exp(scale * q_i . k_j)                   (natural log, f32)
 * Offsets: cu_seqlens_q and cu_seqlens_k are compact i32 [batch + 1] device arrays, read by the kernels only: the host never
 * reads them, so the call does not synchronise and can be captured in a CUDA graph.  args->max_seqlen_q / max_seqlen_k are
 * host bounds on the lengths (torch's max_q / max_k), and size the grid.  On the device each cu value is clamped to [0, T] and
 * each length to [0, max_seqlen]: malformed offsets give unspecified values, but no access leaves q, k, v, out or lse.
 * Visibility (torch's window_size, flash-attn >= 2.1): with off = Lk_b - Lq_b, key j is visible to query i iff j < Lk_b,
 * (window_left < 0 or j >= i + off - window_left) and (window_right < 0 or j <= i + off + window_right).  (-1, -1) is full
 * attention; (-1, 0) is causal aligned bottom-right (b200_attention_kvcache's rule; with Lq == Lk it is b200_attention's
 * top-left causal); (W, 0) a causal sliding window.  A row with no visible key gets out = +0 and lse = -inf.
 * Rows outside every sequence (at or past cu_q[batch], and any row no sequence owns) are not written, in out or lse.
 * Numerics: b200_attention's (f32 scores, base-2 online softmax with t = s * (scale * log2 e), ex2.approx.ftz, P rounded RNE
 * to the input dtype, out = O / l rounded once).  A sequence with Lq == Lk and window (-1, -1) or (-1, 0) gives the bits of a
 * b200_attention call on that sequence alone (causal = 0 or 1).  Every row comes from one CTA in increasing key order: no
 * atomics, bitwise reproducible.  Neighbouring sequences never meet: scores of keys past Lk_b are masked with a select and
 * their V rows are zeroed on chip before the P.V product, and a block the sequence ends inside is stored row by row.
 * Dtypes and limits: b200_attention's (f16 / bf16 in, out in the input dtype or f32, D <= 128, D % 8 == 0, v's head dim equal
 * to D); max_seqlen_q and max_seqlen_k below 2^30.  Views: q, k and v are read in place under b200_attention's rule (unit D
 * stride, 16-byte aligned base and T, H strides), else gathered into a compact [T, H, D] pooled copy.  out needs a unit D
 * stride and a 16-byte aligned base and strides.  lse: 0 (not written) or a compact f32 [Hq, Tq] buffer, 4-byte aligned.
 * Errors: B200_ERR_INVALID_ARG for a k head dim other than D, a v shape mismatch, Hkv == 0 or Hq % Hkv != 0, a wrong out shape,
 * a window side below -1, a negative max_seqlen, a non-finite scale, a null pointer or a misaligned lse / cu array (the
 * wrappers also refuse cu arrays that are not compact i32 [batch + 1]); B200_ERR_UNSUPPORTED for the dtypes, D, Dv != D, out a
 * tensor map cannot write, extents >= 2^31, max_seqlen >= 2^30 or more than 2^31 - 1 CTAs.  batch, Tq, Hq or max_seqlen_q = 0:
 * no launch.
 * Launches: the gathers, then one attn_fwd_varlen_<in>_d<64|128>_<out> launch of ceil(max_seqlen_q / 128) * Hq * batch CTAs
 * (a CTA whose block starts at or past its sequence's Lq exits at once; key blocks that no row of the CTA sees are skipped, not
 * loaded), on `s` with no host synchronisation.  The dry-run plan records "tmap4d" lines in the order q, k, v, out with dims
 * (D, T, H, 1). */
typedef struct b200_attention_varlen_args {
  float scale;            /* multiplies q.k before the softmax */
  int32_t window_left;    /* keys before the aligned diagonal a query sees; -1: unbounded */
  int32_t window_right;   /* keys after the aligned diagonal a query sees; -1: unbounded (0: causal) */
  int32_t max_seqlen_q;   /* >= every Lq_b */
  int32_t max_seqlen_k;   /* >= every Lk_b */
} b200_attention_varlen_args;
int b200_attention_varlen(b200_ctx* ctx, b200_stream s, b200_dtype in_dtype, b200_dtype out_dtype,
                          b200_dptr q, const uint64_t* q_shape, const uint64_t* q_strides,
                          b200_dptr k, const uint64_t* k_shape, const uint64_t* k_strides,
                          b200_dptr v, const uint64_t* v_shape, const uint64_t* v_strides,
                          b200_dptr cu_seqlens_q, b200_dptr cu_seqlens_k, uint64_t batch,
                          b200_dptr out, const uint64_t* out_shape, const uint64_t* out_strides,
                          b200_dptr lse, const b200_attention_varlen_args* args);

/* ---- variable-length (packed) attention, backward --------------------------------------------------------------------------
 * b200_attention_backward's formulas per sequence of b200_attention_varlen (its layout, offsets, args and visibility): dq
 * [Tq, Hq, D], dk and dv [Tk, Hkv, D] from q, k, v, the forward's out and lse (compact f32 [Hq, Tq], non-null) and dout; dk
 * and dv of kv head hk sum over its G query heads.  A row without visible keys (lse = -inf) gives dq = +0 and adds nothing to
 * dk or dv; a key no query sees gets dk = dv = +0.  Rows outside every sequence are not written, in dq, dk or dv.
 * Numerics: b200_attention_backward's (the forward's scores bit for bit, p = exp2(t - lse * log2 e), P and dS rounded RNE,
 * f32 sums, dq and dk multiplied by scale and rounded once).  A sequence with Lq == Lk and window (-1, -1) or (-1, 0) gives the
 * bits of a b200_attention_backward call on that sequence alone.  Every dq row comes from one CTA in key order and every dk /
 * dv row from one CTA in (group head, query block) order: no atomics, bitwise reproducible.  Q and dO rows past Lq_b (and K
 * rows past Lk_b in the dq kernel) are zeroed on chip before they enter a product.
 * Dtypes, views and limits: b200_attention_varlen's; out in the input dtype or f32 (out_dtype), dout in the input dtype; dq, dk
 * and dv in grad_dtype (the input dtype or B200_F32) with a unit D stride and a 16-byte aligned base and strides (so they can
 * be slices of one fused [T, 3, H, D] gradient buffer), else B200_ERR_UNSUPPORTED naming the tensor.  out and dout are read in
 * place under the input rule, else gathered.
 * Errors: b200_attention_varlen's, plus B200_ERR_INVALID_ARG when out, dout or dq differ from q's shape or dk or dv from k's,
 * and B200_ERR_UNSUPPORTED for an out_dtype or grad_dtype other than the input dtype or f32.  batch = 0, or no query rows (Tq,
 * Hq or max_seqlen_q = 0) together with no key rows (Tk or max_seqlen_k = 0), launches nothing.
 * Launches, on `s` with no host synchronisation: the gathers; with query rows, a pooled f32 workspace of 2 * Hq * Tqp values,
 * Tqp = (ceil(Tq / 128) + batch) * 128 ("alloc"; each sequence gets its own 128-row aligned slices), then
 * attn_bwd_varlen_delta_<in>_<out> (ceil(max_seqlen_q / 128) * 8 * Hq * batch blocks of 256 threads) and
 * attn_bwd_varlen_dq_<in>_d<64|128>_<grad> (ceil(max_seqlen_q / 128) * Hq * batch CTAs) after its maps q, k, v, dout, dq; with
 * key rows, attn_bwd_varlen_dkdv_<in>_d<64|128>_<grad> (ceil(max_seqlen_k / 128) * Hkv * batch CTAs) after its maps q, k, v,
 * dout, dk, dv.  The maps are "tmap4d" plan lines with dims (D, T, H, 1). */
int b200_attention_varlen_backward(b200_ctx* ctx, b200_stream s, b200_dtype in_dtype, b200_dtype out_dtype, b200_dtype grad_dtype,
                                   b200_dptr q, const uint64_t* q_shape, const uint64_t* q_strides,
                                   b200_dptr k, const uint64_t* k_shape, const uint64_t* k_strides,
                                   b200_dptr v, const uint64_t* v_shape, const uint64_t* v_strides,
                                   b200_dptr out, const uint64_t* out_shape, const uint64_t* out_strides,
                                   b200_dptr dout, const uint64_t* dout_shape, const uint64_t* dout_strides,
                                   b200_dptr lse, b200_dptr cu_seqlens_q, b200_dptr cu_seqlens_k, uint64_t batch,
                                   b200_dptr dq, const uint64_t* dq_shape, const uint64_t* dq_strides,
                                   b200_dptr dk, const uint64_t* dk_shape, const uint64_t* dk_strides,
                                   b200_dptr dv, const uint64_t* dv_shape, const uint64_t* dv_strides,
                                   const b200_attention_varlen_args* args);

/* ---- attention against a KV cache (decoding, speculative decoding, chunked prefill; forward only) ------------------------
 * Sequence b of the batch has L_b = cache_seqlens[b] keys in the cache.  With G = Hq / Hkv and hk = h / G:
 *   out[b, h, i, :] = sum_{j visible} softmax_j(scale * q[b, h, i, :] . K_b[j, hk, :]) * V_b[j, hk, :]
 *   lse[b, h, i]    = log sum_{j visible} exp(scale * q[b, h, i, :] . K_b[j, hk, :])                      (natural log, f32)
 * q and out are [B, Hq, Sq, D] (the Sq new queries of each sequence, usually 1); k_cache and v_cache are [P, page, Hkv, D]:
 * P pages of `page` keys.  Shapes and strides in elements, so a [P, Hkv, page, D] (head-major) cache is the same call with
 * permuted strides, and a [B, Sq, Hq, D] q is a stride-permuted view.
 * Lengths: cache_seqlens is a compact i32 [B] device array, read by the kernels only (the host never reads it, so the call
 * does not synchronise).  Each value is clamped to [0, max_pages * page].
 * Visibility: query i of sequence b sees key j iff j < L_b and, when args->causal != 0, j <= L_b - Sq + i (bottom-right
 * alignment: flash_attn_with_kvcache's rule, torch's causal_lower_right; the new queries are the last Sq keys).  This is the
 * only difference from b200_attention's args.  A row with no visible key (L_b = 0, or causal with L_b < Sq - i) gets out = +0
 * and lse = -inf.
 * Paging: key j of sequence b is row j % page of page block_table[b, j / page], kv head hk.  block_table is an i32 [B, max_pages]
 * array with any strides (4-byte aligned).  Entries at or past ceil(L_b / page) are never read; an out-of-range page id
 * reads zeros and cannot fault.  block_table = 0: sequence b is page b (P must equal B, max_pages = 1), the plain contiguous
 * [B, Smax, Hkv, D] cache.  With one page per sequence (no table, or max_pages == 1) the page may have any size; otherwise
 * page must be a multiple of 16 that divides 64 (the kernel's key block) or is a multiple of 64.
 * Stale slots: cache slots at or past L_b may hold anything, NaN and inf included (serving caches reuse freed pages); they
 * never reach out.  Scores are masked with a select, and the V rows of keys >= L_b are zeroed on chip before the P.V product.
 * Dtypes and limits: as b200_attention (f16 / bf16 in, out in the input dtype or f32, D <= 128, D % 8 == 0, the caches' head
 * dim equal to D).  out and both caches need a unit D stride and a 16-byte aligned base and strides, else
 * B200_ERR_UNSUPPORTED: a cache is read in place through a 4-D tensor map over (D, page, Hkv, P), never gathered (a copy of the
 * whole cache per step would cost more than the attention).  q is read in place or gathered like b200_attention's inputs.
 * lse: 0 or a compact f32 [B, Hq, Sq] buffer.
 * Work: one CTA per (b, hk, m-tile, split).  An m-tile holds gt heads of one kv head's group times st queries (gt * st <= 64),
 * so each K / V byte is read once per kv head; gt and st minimise the m-tile count ceil(G / gt) * ceil(Sq / st) (ties: the
 * larger st).  The split count depends on shapes only (B, Hkv, the m-tiles, the capacity max_pages * page and the SM count),
 * never on the lengths: split s takes an equal range of the capacity's 64-key blocks; a split past L_b writes an empty partial.
 * Numerics: b200_attention's (f32 scores, base-2 online softmax with t = s * (scale * log2 e), ex2.approx.ftz, P rounded RNE to
 * the input dtype).  One split: out = O / l rounded once.  Several: each split keeps un-normalised f32 O_s with its maximum
 * m_s and sum l_s, and the combine forms m = max m_s, w_s = exp2(m_s - m), out = sum_s w_s O_s / sum_s w_s l_s in f32 in split
 * order, rounded once; lse = (m + log2 l) * ln 2.  No atomics: bitwise reproducible for fixed shapes and SM count, and equal
 * bits for the same keys in any page layout of equal capacity.
 * Errors: B200_ERR_INVALID_ARG for a k_cache head dim other than D, a v_cache shape mismatch, Hkv == 0 or Hq % Hkv != 0, a wrong
 * out shape, an empty cache (P or page 0), a block table that is not [B, >= 1] (or no table with P != B), a non-finite scale,
 * a null pointer or a misaligned lse / cache_seqlens / block_table; B200_ERR_UNSUPPORTED for the dtypes, D, Dv != D, the page
 * rule above, caches or out a tensor map cannot read, extents or capacity >= 2^31.  B, Hq or Sq = 0: no launch.
 * Launches, on `s` with no host synchronisation: the gather of q if needed; one split: one attn_kv_<in>_d<64|128>_<out> launch of
 * B * Hkv * m-tiles CTAs that writes out and lse.  Several: a pooled f32 workspace of nsplit * B * Hq * Sq * (D + 2) values
 * ("alloc"), the attn_kv launch of B * Hkv * m-tiles * nsplit CTAs, then attn_kv_combine_<out>.  The dry-run plan records the
 * maps as "tmap4d" lines in the order q (box (64, st, gt, 1)), k_cache, v_cache (box (64, rows, 1, 1), rows = 64 or the page). */
int b200_attention_kvcache(b200_ctx* ctx, b200_stream s, b200_dtype in_dtype, b200_dtype out_dtype,
                           b200_dptr q, const uint64_t* q_shape, const uint64_t* q_strides,
                           b200_dptr k_cache, const uint64_t* kc_shape, const uint64_t* kc_strides,
                           b200_dptr v_cache, const uint64_t* vc_shape, const uint64_t* vc_strides,
                           b200_dptr block_table, const uint64_t* bt_shape, const uint64_t* bt_strides,
                           b200_dptr cache_seqlens,
                           b200_dptr out, const uint64_t* out_shape, const uint64_t* out_strides,
                           b200_dptr lse, const b200_attention_args* args);

/* Scatter of new keys and values into a paged KV cache (vLLM's reshape_and_cache).  k_new and v_new are [B, Snew, Hkv, D] views,
 * k_cache and v_cache [P, page, Hkv, D] as in b200_attention_kvcache; slot_mapping is a compact i32 [B * Snew] device array.
 * Token t of sequence b goes to flat slot s = slot_mapping[b * Snew + t], that is row s % page of page s / page, for every kv
 * head.  A negative slot, or one >= P * page, is skipped.  No length is updated on the device: the caller keeps the lengths
 * (cache_seqlens) itself, as a serving scheduler already does, and uploads them for the attention call.  Two tokens mapped to
 * one slot leave one of them there, unspecified which.
 * dtype: B200_F16 or B200_BF16; D % 8 == 0.  The caches need a unit D stride and a 16-byte aligned base and strides (else
 * B200_ERR_UNSUPPORTED); k_new / v_new views that do not are gathered first.  Errors: B200_ERR_INVALID_ARG for shape
 * mismatches, a null pointer or a misaligned slot_mapping.  One attn_kv_write launch (16-byte loads and stores) on `s`. */
int b200_kvcache_write(b200_ctx* ctx, b200_stream s, b200_dtype dtype,
                       b200_dptr k_new, const uint64_t* kn_shape, const uint64_t* kn_strides,
                       b200_dptr v_new, const uint64_t* vn_shape, const uint64_t* vn_strides,
                       b200_dptr k_cache, const uint64_t* kc_shape, const uint64_t* kc_strides,
                       b200_dptr v_cache, const uint64_t* vc_shape, const uint64_t* vc_strides,
                       b200_dptr slot_mapping);

/* ---- fp8 KV caches (vLLM's kv_cache_dtype="fp8", FlashAttention-3's k_descale / v_descale) ------------------------------
 * b200_attention_kvcache with the caches in B200_F8E4M3 or B200_F8E5M2 (cache_dtype, both caches) and two compact f32 [Hkv]
 * device arrays k_scale and v_scale (read by the kernels only: no synchronisation, graph-capturable; a per-tensor scale is the
 * same value in every entry).  The cache holds K = k_scale[hk] * k8 and V = v_scale[hk] * v8.  q is f16 or bf16, out q's dtype
 * or f32; shapes, paging, block_table, cache_seqlens, bottom-right causal, stale slots, lse and the errors are those of
 * b200_attention_kvcache.
 * Numerics: K and V are widened on chip to q's dtype (exact: every e4m3 and e5m2 value is an f16 and a bf16 value); t = s * c
 * with s the f32 score of q against the widened K and c = (scale * log2 e) * k_scale[hk], one f32 product per CTA; the online
 * softmax and P rounding of b200_attention_kvcache; v_scale is applied once to the un-normalised f32 sum just before the
 * division: out = (v_scale * O) / l rounded once, and with several splits out = (v_scale * sum_s w_s O_s) / sum_s w_s l_s.
 * lse does not depend on v_scale.  So power-of-two scales (and scales of 1) give bit for bit the output of
 * b200_attention_kvcache on the dequantized 16-bit cache.
 * Views: a cache is read in place with a unit D stride and a 16-byte aligned base and strides, in bytes: a compact fp8 cache
 * needs D % 16 == 0.  Errors beyond b200_attention_kvcache's: B200_ERR_UNSUPPORTED for a cache dtype that is not fp8;
 * B200_ERR_INVALID_ARG for a null or not 4-byte aligned k_scale or v_scale.
 * Launches: one attn_kv_<in>_<e4m3|e5m2>_d<64|128>_<out> launch (split count and m-tile as b200_attention_kvcache), plus
 * attn_kv_combine_fp8_<out> when the keys are split.  The plan's k_cache and v_cache maps have esz=1 and box (128, rows, 1, 1). */
int b200_attention_kvcache_fp8(b200_ctx* ctx, b200_stream s, b200_dtype in_dtype, b200_dtype cache_dtype, b200_dtype out_dtype,
                               b200_dptr q, const uint64_t* q_shape, const uint64_t* q_strides,
                               b200_dptr k_cache, const uint64_t* kc_shape, const uint64_t* kc_strides,
                               b200_dptr v_cache, const uint64_t* vc_shape, const uint64_t* vc_strides,
                               b200_dptr block_table, const uint64_t* bt_shape, const uint64_t* bt_strides,
                               b200_dptr cache_seqlens, b200_dptr k_scale, b200_dptr v_scale,
                               b200_dptr out, const uint64_t* out_shape, const uint64_t* out_strides,
                               b200_dptr lse, const b200_attention_args* args);

/* b200_kvcache_write into fp8 caches (vLLM's reshape_and_cache with an fp8 cache): k_new and v_new are f16 or bf16 (dtype),
 * the caches cache_dtype (B200_F8E4M3 or B200_F8E5M2), k_scale and v_scale compact f32 [Hkv] device arrays.  Each stored value
 * is sat_rn(x / scale[hk]): an f32 division rounded to nearest, then RNE to the cache format with saturation to +-448 (e4m3)
 * or +-57344 (e5m2); NaN stays NaN.  In torch: (x.float() / s).clamp(-max, max).to(float8).  Slots, views and errors as
 * b200_kvcache_write, plus b200_attention_kvcache_fp8's cache-dtype and scale errors.  One attn_kv_write_fp8 launch (16-byte
 * loads, 8-byte stores). */
int b200_kvcache_write_fp8(b200_ctx* ctx, b200_stream s, b200_dtype dtype, b200_dtype cache_dtype,
                           b200_dptr k_new, const uint64_t* kn_shape, const uint64_t* kn_strides,
                           b200_dptr v_new, const uint64_t* vn_shape, const uint64_t* vn_strides,
                           b200_dptr k_cache, const uint64_t* kc_shape, const uint64_t* kc_strides,
                           b200_dptr v_cache, const uint64_t* vc_shape, const uint64_t* vc_strides,
                           b200_dptr slot_mapping, b200_dptr k_scale, b200_dptr v_scale);

/* ---- collectives: ServerCommunication (server/base.rs:632-739), CUDA impl cubecl-cuda/src/compute/server.rs:666-926 -- */
#define B200_UNIQUE_ID_BYTES 128
int b200_comm_get_unique_id(b200_ctx* ctx, void* id128);            /* ncclGetUniqueId (communication.rs:11-25 holds it per device set) */
/* Communicator for the device set `device_ids` (keyed by the sorted set, CommunicationId server/base.rs:605-620);
 * this context's rank is the position of its device in the sorted list (server.rs:669-703). */
int b200_comm_init(b200_ctx* ctx, const int* device_ids, int n, const void* id128);
/* src -> dst (may alias) of bytes/elem_size elements on the communicator's comm stream, after an event wait on
 * `compute` (server.rs:705-780). */
int b200_all_reduce(b200_ctx* ctx, b200_stream compute, b200_dptr src, b200_dptr dst, size_t bytes, b200_dtype dtype,
                    b200_comm_op op, const int* device_ids, int n);
/* Make `compute` wait for everything issued on the comm stream (server.rs:782-798). */
int b200_sync_collective(b200_ctx* ctx, b200_stream compute);

/* ---- fused reduce + all-reduce over NVLink peer memory (no NCCL on the data path) -----------------------------------
 * The reduce path's exchange step is one f32 per rank.  Instead of reduce kernel -> event -> ncclAllReduce -> event
 * (client.rs:790 + server.rs:705-798), the LAST block of the reduce kernel stores this rank's scalar (value+epoch in one
 * 64-bit system-scope store) into every peer's mailbox and gathers theirs, so local reduce + exchange are ONE launch.
 * Setup: every rank exports its mailbox, the handles are exchanged out of band, every rank connects.  Ranks = position in
 * the sorted device set (as for b200_comm_init).  Works across processes (CUDA IPC) and inside one process (peer access). */
#define B200_IPC_HANDLE_BYTES 64
int b200_p2p_export(b200_ctx* ctx, void* ipc_handle64, uint64_t* local_ptr, int64_t* pid);
/* arrays are indexed like device_ids: n x 64-byte handles, n pointers, n pids (as returned by b200_p2p_export on each rank) */
int b200_p2p_connect(b200_ctx* ctx, const int* device_ids, int n, const void* ipc_handles, const uint64_t* local_ptrs,
                     const int64_t* pids);
/* out[0] (on every rank) = sum over ranks of sum(in[0..n)).  Collective: every rank of the set must call it, in the same
 * order; a missing peer trips the kernel's 4 s deadline (device trap -> B200_ERR_UNHEALTHY at sync).  SUM of F32 only. */
int b200_reduce_all_reduce(b200_ctx* ctx, b200_stream s, b200_reduce_op op, b200_dtype in_dtype, b200_dptr in, b200_dptr out,
                           uint64_t n, const int* device_ids, int ndev);

/* Arg-reduce across ranks (NCCL has no arg-reduce: SURVEY 8e "all-gather 8 pairs + local select", here inside the kernel):
 * out[0] (u32, on every rank) = GLOBAL index of the extremum of the concatenation of all ranks' inputs, where this rank's
 * element 0 has global index `index_offset`.  Same tie / NaN rule as b200_reduce.  Global indices must fit 32 bits. */
int b200_argreduce_all_reduce(b200_ctx* ctx, b200_stream s, b200_reduce_op op, b200_dtype in_dtype, b200_dptr in, b200_dptr out,
                              uint64_t n, uint64_t index_offset, const int* device_ids, int ndev);

/* ---- synthetic operands + reference-equivalent probes (examples/throughput) ----------------------------------------- */
/* out[i] = lo + u(seed,i) * (hi - lo), u in [0,1) from a counter hash the host can reproduce (cubecl_b200/synth.py);
 * mode 1: out[i] = i % modulus. */
int b200_fill_uniform(b200_ctx* ctx, b200_stream s, b200_dtype dtype, b200_dptr out, uint64_t n, uint64_t seed, float lo, float hi);
int b200_fill_modulo(b200_ctx* ctx, b200_stream s, b200_dtype dtype, b200_dptr out, uint64_t n, uint32_t modulus);
/* compute_cmma_throughput as CubeCL would JIT it today (wmma 16x16x16): launches grid = SMs*32, block = 256, `n_iter`
 * dependent mma_sync per plane; *ops = cubes * planes * 2*m*n*k * n_iter (compute_cmma.rs:16,41-42). dtype F16 or BF16. */
int b200_probe_wmma(b200_ctx* ctx, b200_stream s, b200_dtype dtype, uint32_t n_iter, b200_dptr scratch_1k, double* ops);
/* The same accounting on the Hopper tensor cores: one CTA per SM, whose two warpgroups each issue n_iter x 4 dependent wgmma
 * m64n256k16 (bf16->f32, register accumulators) on smem-resident operands; *ops = SMs * 2 * n_iter * 4 * 2*64*256*16.
 * scratch: >= 4 * num_sms bytes; scratch[cta] = 64 * n_iter afterwards. */
int b200_probe_umma(b200_ctx* ctx, b200_stream s, uint32_t n_iter, b200_dptr scratch, double* ops);
/* The same probe for the other operand kinds: dtype B200_BF16 (as above) or B200_F8E4M3 (wgmma m64n256k32); block_scaled != 0
 * is B200_ERR_UNSUPPORTED (sm_90 has no block-scaled MMA).  *ops = SMs * 2 * n_iter * 4 * 2*64*256*K with K = 16 / 32;
 * scratch[cta] = 4 * K * n_iter afterwards. */
int b200_probe_umma_kind(b200_ctx* ctx, b200_stream s, b200_dtype dtype, int block_scaled, uint32_t n_iter, b200_dptr scratch,
                         double* ops);
/* memory_read_throughput with float_4 lines over `bytes` of `buf` (memory_read.rs:68-154): grid = SMs*32, block = 256. */
int b200_probe_memread(b200_ctx* ctx, b200_stream s, b200_dptr buf, uint64_t bytes, b200_dptr scratch_16);
/* memory_write_throughput (memory_write.rs: writes only) and memory_direct (memory_direct.rs: copy, both directions counted). */
int b200_probe_memwrite(b200_ctx* ctx, b200_stream s, b200_dptr dst, uint64_t bytes);
int b200_probe_memcopy(b200_ctx* ctx, b200_stream s, b200_dptr dst, b200_dptr src, uint64_t bytes);

/* Thread-local message of the last failing call on this thread ("" if none). */
const char* b200_last_error(void);

#ifdef __cplusplus
}
#endif
#endif /* CUBECL_B200_H */
