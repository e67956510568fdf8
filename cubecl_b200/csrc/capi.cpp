// Host side of the C ABI declared in include/cubecl_b200.h.
//
// What this file is: the H100-native stand-in for the pieces of cubecl-cuda that sit between `ComputeClient::launch` and
// `cuLaunchKernel` on the dense-LA hot path -- minus NVRTC.  It loads libcuda (and, lazily, libnccl) with dlopen exactly
// like cudarc's dynamic loading does (reference Cargo.toml:179-187), retains the device's primary context, loads the
// PREBUILT sm_90a cubins embedded in this library with cuModuleLoadData (the call the reference makes with NVRTC's PTX at
// crates/cubecl-cuda/src/compute/context.rs:293), keeps a small exclusive-page memory pool + pinned staging
// (semantics of crates/cubecl-runtime/src/memory_management, crates/cubecl-cuda/src/compute/storage/gpu.rs:174-207),
// encodes TMA descriptors (same cuTensorMapEncodeTiled call as crates/cubecl-cuda/src/compute/server.rs:1210-1224) and
// launches.  No kernels are generated, compiled or autotuned at run time and nothing here can run without a GPU.
#include "../../include/cubecl_b200.h"
#include "kernel_params.h"

#include <cuda.h>
#include <dlfcn.h>
#include <unistd.h>

#include <algorithm>
#include <memory>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>

// ================================================================================================ embedded cubins
extern "C" {
extern const unsigned char b200_cubin_gemm[];
extern const unsigned char b200_cubin_gemm_end[];
extern const unsigned char b200_cubin_gemm_b[];
extern const unsigned char b200_cubin_gemm_b_end[];
extern const unsigned char b200_cubin_gemm_c[];
extern const unsigned char b200_cubin_gemm_c_end[];
extern const unsigned char b200_cubin_reduce[];
extern const unsigned char b200_cubin_reduce_end[];
extern const unsigned char b200_cubin_aux[];
extern const unsigned char b200_cubin_aux_end[];
extern const unsigned char b200_cubin_quant[];
extern const unsigned char b200_cubin_quant_end[];
extern const unsigned char b200_cubin_gemm_q[];
extern const unsigned char b200_cubin_gemm_q_end[];
extern const unsigned char b200_cubin_quant_mm[];
extern const unsigned char b200_cubin_quant_mm_end[];
extern const unsigned char b200_cubin_gemm_conv[];
extern const unsigned char b200_cubin_gemm_conv_end[];
extern const unsigned char b200_cubin_gemm_convbwd[];
extern const unsigned char b200_cubin_gemm_convbwd_end[];
extern const unsigned char b200_cubin_conv_grouped[];
extern const unsigned char b200_cubin_conv_grouped_end[];
extern const unsigned char b200_cubin_gemm_conv3d[];
extern const unsigned char b200_cubin_gemm_conv3d_end[];
extern const unsigned char b200_cubin_gemm_convt[];
extern const unsigned char b200_cubin_gemm_convt_end[];
extern const unsigned char b200_cubin_attention[];
extern const unsigned char b200_cubin_attention_end[];
extern const unsigned char b200_cubin_attention_bwd[];
extern const unsigned char b200_cubin_attention_bwd_end[];
extern const unsigned char b200_cubin_attention_kv[];
extern const unsigned char b200_cubin_attention_kv_end[];
extern const unsigned char b200_cubin_attention_varlen[];
extern const unsigned char b200_cubin_attention_varlen_end[];
extern const unsigned char b200_cubin_attention_varlen_bwd[];
extern const unsigned char b200_cubin_attention_varlen_bwd_end[];
extern const unsigned char b200_cubin_attention_kv_fp8[];
extern const unsigned char b200_cubin_attention_kv_fp8_end[];
}

// ================================================================================================ errors
static thread_local std::string g_last_error;

static int fail(int status, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_last_error = buf;
  return status;
}

extern "C" const char* b200_last_error(void) { return g_last_error.c_str(); }
extern "C" int b200_abi_version(void) { return B200_ABI_VERSION; }

// ================================================================================================ driver loading
#define DRV_FUNCTIONS(X)                                                                                              \
  X(cuInit) X(cuDeviceGetCount) X(cuDeviceGet) X(cuDeviceGetName) X(cuDeviceGetAttribute) X(cuDeviceTotalMem)        \
  X(cuDevicePrimaryCtxRetain) X(cuDevicePrimaryCtxRelease) X(cuCtxSetCurrent) X(cuCtxSynchronize)                    \
  X(cuModuleLoadData) X(cuModuleUnload) X(cuModuleGetFunction) X(cuFuncSetAttribute) X(cuFuncGetAttribute)           \
  X(cuLaunchKernelEx) X(cuLaunchKernel) X(cuOccupancyMaxActiveClusters)                                              \
  X(cuMemAlloc) X(cuMemFree) X(cuMemAllocHost) X(cuMemFreeHost) X(cuMemcpyHtoDAsync) X(cuMemcpyDtoHAsync)            \
  X(cuMemcpyDtoDAsync) X(cuMemsetD32Async) X(cuMemsetD2D16Async) X(cuMemsetD2D32Async) X(cuMemGetInfo)                 \
  X(cuStreamCreate) X(cuStreamDestroy) X(cuStreamSynchronize) X(cuStreamWaitEvent)                                   \
  X(cuEventCreate) X(cuEventRecord) X(cuEventElapsedTime) X(cuEventDestroy) X(cuEventSynchronize) X(cuEventQuery)                    \
  X(cuTensorMapEncodeTiled) X(cuTensorMapEncodeIm2col) X(cuGetErrorString) X(cuGetErrorName)                                                    \
  X(cuIpcGetMemHandle) X(cuIpcOpenMemHandle) X(cuIpcCloseMemHandle) X(cuCtxEnablePeerAccess) X(cuDeviceCanAccessPeer)

struct Driver {
  void* lib = nullptr;
  bool ok = false;
  std::string why;
#define X(n) decltype(&n) n##_p = nullptr;
  DRV_FUNCTIONS(X)
#undef X
};
static Driver g_drv;
static std::once_flag g_drv_once;

static void load_driver() {
  const char* names[] = {"libcuda.so.1", "libcuda.so"};
  for (const char* n : names) {
    g_drv.lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
    if (g_drv.lib) break;
  }
  if (!g_drv.lib) {
    g_drv.why = "cannot dlopen libcuda.so.1 (no NVIDIA driver): this library has no CPU fallback";
    return;
  }
  using GetProc = CUresult (*)(const char*, void**, int, cuuint64_t, CUdriverProcAddressQueryResult*);
  GetProc get_proc = reinterpret_cast<GetProc>(dlsym(g_drv.lib, "cuGetProcAddress_v2"));
  if (!get_proc) {
    g_drv.why = "libcuda has no cuGetProcAddress_v2 (driver older than CUDA 12)";
    return;
  }
#define X(n)                                                                                              \
  {                                                                                                       \
    void* fp = nullptr;                                                                                   \
    CUdriverProcAddressQueryResult q;                                                                     \
    CUresult r = get_proc(#n, &fp, 12080, CU_GET_PROC_ADDRESS_DEFAULT, &q);                               \
    if (r != CUDA_SUCCESS || !fp) {                                                                       \
      g_drv.why = std::string("driver symbol missing: ") + #n;                                            \
      return;                                                                                             \
    }                                                                                                     \
    g_drv.n##_p = reinterpret_cast<decltype(&n)>(fp);                                                     \
  }
  DRV_FUNCTIONS(X)
#undef X
  CUresult r = g_drv.cuInit_p(0);
  if (r != CUDA_SUCCESS) {
    g_drv.why = "cuInit failed (" + std::to_string(static_cast<int>(r)) + "): no usable GPU";
    return;
  }
  g_drv.ok = true;
}

static int ensure_driver() {
  std::call_once(g_drv_once, load_driver);
  if (!g_drv.ok) return fail(B200_ERR_NO_DEVICE, "%s", g_drv.why.c_str());
  return B200_OK;
}

static const char* cu_err(CUresult r) {
  const char* s = nullptr;
  if (g_drv.cuGetErrorString_p && g_drv.cuGetErrorString_p(r, &s) == CUDA_SUCCESS && s) return s;
  return "unknown CUDA error";
}

static int map_cu(CUresult r) {
  switch (r) {
    case CUDA_ERROR_OUT_OF_MEMORY: return B200_ERR_OUT_OF_MEMORY;
    case CUDA_ERROR_LAUNCH_OUT_OF_RESOURCES: return B200_ERR_TOO_MANY_RESOURCES;
    case CUDA_ERROR_INVALID_IMAGE:
    case CUDA_ERROR_NO_BINARY_FOR_GPU:
    case CUDA_ERROR_INVALID_SOURCE: return B200_ERR_COMPILATION;
    case CUDA_ERROR_ILLEGAL_ADDRESS:
    case CUDA_ERROR_LAUNCH_FAILED:
    case CUDA_ERROR_ILLEGAL_INSTRUCTION:
    case CUDA_ERROR_MISALIGNED_ADDRESS:
    case CUDA_ERROR_HARDWARE_STACK_ERROR:
    case CUDA_ERROR_LAUNCH_TIMEOUT: return B200_ERR_UNHEALTHY;
    default: return B200_ERR_UNKNOWN;
  }
}

#define CU_CHECK(call)                                                                               \
  do {                                                                                               \
    CUresult _r = (call);                                                                            \
    if (_r != CUDA_SUCCESS) return fail(map_cu(_r), "%s failed: %s (%d)", #call, cu_err(_r), (int)_r); \
  } while (0)

// ================================================================================================ NCCL loading (lazy)
typedef struct ncclComm* ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
enum { ncclSuccess = 0 };
// ncclDataType_t / ncclRedOp_t numeric values are ABI-stable across NCCL 2.x
enum { ncclInt8 = 0, ncclUint8 = 1, ncclInt32 = 2, ncclUint32 = 3, ncclInt64 = 4, ncclUint64 = 5, ncclFloat16 = 6,
       ncclFloat32 = 7, ncclFloat64 = 8, ncclBfloat16 = 9 };
enum { ncclSum = 0, ncclProd = 1, ncclMax = 2, ncclMin = 3, ncclAvg = 4 };

struct Nccl {
  void* lib = nullptr;
  bool ok = false;
  std::string why;
  int (*GetUniqueId)(ncclUniqueId*) = nullptr;
  int (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  int (*CommDestroy)(ncclComm_t) = nullptr;
  int (*AllReduce)(const void*, void*, size_t, int, int, ncclComm_t, CUstream) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
};
static Nccl g_nccl;
static std::once_flag g_nccl_once;

static void load_nccl() {
  // If torch already mapped its bundled libnccl.so.2 the soname lookup returns that copy; otherwise the system one.
  g_nccl.lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!g_nccl.lib) {
    g_nccl.why = std::string("cannot dlopen libnccl.so.2: ") + (dlerror() ? dlerror() : "?");
    return;
  }
#define L(field, sym)                                                        \
  g_nccl.field = reinterpret_cast<decltype(g_nccl.field)>(dlsym(g_nccl.lib, sym)); \
  if (!g_nccl.field) { g_nccl.why = std::string("nccl symbol missing: ") + sym; return; }
  L(GetUniqueId, "ncclGetUniqueId")
  L(CommInitRank, "ncclCommInitRank")
  L(CommDestroy, "ncclCommDestroy")
  L(AllReduce, "ncclAllReduce")
  L(GetErrorString, "ncclGetErrorString")
#undef L
  g_nccl.ok = true;
}

static int ensure_nccl() {
  std::call_once(g_nccl_once, load_nccl);
  if (!g_nccl.ok) return fail(B200_ERR_COMM, "%s", g_nccl.why.c_str());
  return B200_OK;
}

#define NCCL_CHECK(call)                                                                                      \
  do {                                                                                                        \
    int _r = (call);                                                                                          \
    if (_r != ncclSuccess) return fail(B200_ERR_COMM, "%s failed: %s", #call, g_nccl.GetErrorString(_r));     \
  } while (0)

// ================================================================================================ context
struct PoolBlock {
  size_t size;
  bool in_use;
  // Stream-ordered reuse (the reference's pools are per-stream and cross-stream hand-offs wait on events,
  // cubecl-runtime/src/stream/event.rs:50-57): a freed page remembers the stream that last used it and an event recorded
  // there; the same stream may take it back at once, any other requester only once the event has completed.
  CUstream last_stream = nullptr;
  CUevent done = nullptr;
  bool pending = false;
};

struct CommState {
  ncclComm_t comm = nullptr;
  int rank = -1, n = 0;
};

// Peer-memory exchange state for one device set (fused reduce + all-reduce over NVLink).
struct P2PState {
  uint64_t mailbox[8] = {0};
  int rank = -1, n = 0;
  uint32_t epoch = 0;
  std::vector<CUdeviceptr> opened;  // IPC mappings to close
};

struct b200_ctx {
  int device = -1;
  CUdevice dev{};
  CUcontext cuctx = nullptr;
  b200_props props{};
  CUstream stream = nullptr;       // default compute stream
  CUstream comm_stream = nullptr;  // dedicated NCCL stream (server.rs:944)
  CUevent comm_event = nullptr;
  std::vector<CUmodule> modules;
  std::unordered_map<std::string, CUfunction> funcs;
  // exclusive-page pool: exact-size free lists
  std::map<size_t, std::vector<CUdeviceptr>> free_lists;
  std::unordered_map<CUdeviceptr, PoolBlock> blocks;
  uint64_t bytes_in_use = 0, bytes_reserved = 0;
  std::unordered_map<void*, size_t> pinned;
  std::unordered_map<CUstream, CUdeviceptr> reduce_ws;
  std::vector<CUstream> dead_streams;   // streams destroyed through b200_stream_destroy (drained there): never record on them again
  std::map<std::string, CUtensorMap> tmap_cache;
  std::map<std::vector<int>, CommState> comms;
  std::map<std::vector<int>, P2PState> p2p;
  CUdeviceptr mailbox = 0;
  std::unordered_map<std::string, std::string> options;
  std::unordered_map<std::string, std::string> env_cache;   // B200_<KEY> environment defaults, read once
  uint64_t launches = 0;
  // Dry-run planning context (no driver, no device): every launch / descriptor / pool request is RECORDED instead of
  // executed, so the host logic (validation, batch collapse, variant choice, split plans) is testable on a CPU box.
  // Mirrors the reference's DryRun mode (crates/cubecl-runtime/src/dry_run.rs:45,88,121).
  bool dry = false;
  std::string plan;
  std::string pending_kernel;
  std::string last_kernel;         // name of the most recently launched kernel (b200_last_kernel)
  // Programmatic dependent launch of back-to-back all-element reductions on the context's own stream (every kernel there
  // is launched by this library, so the predecessor is known): output pointer of the reduce_all launch that is the LAST
  // kernel queued on c->stream, 0 if the last kernel was anything else.
  uint64_t pdl_prev_out = 0;
  uint64_t fake_next = 0x7000000000ull;
};

static inline CUstream resolve_stream(b200_ctx* c, b200_stream s) { return s ? static_cast<CUstream>(s) : c->stream; }

#define CTX_ENTER(c)                                                  \
  if (!(c)) return fail(B200_ERR_INVALID_ARG, "null context");        \
  if (!(c)->dry) CU_CHECK(g_drv.cuCtxSetCurrent_p((c)->cuctx));
// entry points that talk to the driver directly (copies, streams, events, collectives) do not exist on a planning context
#define CTX_ENTER_DEVICE(c)                                           \
  CTX_ENTER(c);                                                       \
  if ((c)->dry) return fail(B200_ERR_UNSUPPORTED, "%s is not available on a dry-run planning context", __func__);

static std::string opt(b200_ctx* c, const char* key, const char* dflt) {
  auto it = c->options.find(key);
  if (it != c->options.end()) return it->second;
  // environment fallback B200_<KEY>, looked up once per key (getenv on every launch is measurable next to a 20 us kernel)
  auto ev = c->env_cache.find(key);
  if (ev == c->env_cache.end()) {
    std::string env = std::string("B200_") + key;
    for (auto& ch : env) ch = (ch == '.') ? '_' : static_cast<char>(toupper(ch));
    const char* e = getenv(env.c_str());
    ev = c->env_cache.emplace(key, e ? std::string(e) : std::string("\x01unset")).first;
  }
  if (ev->second != "\x01unset") return ev->second;
  return dflt;
}

static int load_module(b200_ctx* c, const unsigned char* begin, const unsigned char* end, const char* what) {
  if (end <= begin) return fail(B200_ERR_COMPILATION, "embedded cubin '%s' is empty (library was built without kernels)", what);
  CUmodule m;
  CUresult r = g_drv.cuModuleLoadData_p(&m, begin);
  if (r != CUDA_SUCCESS)
    return fail(B200_ERR_COMPILATION, "cuModuleLoadData(%s) failed: %s -- the cubins are sm_90a only", what, cu_err(r));
  c->modules.push_back(m);
  return B200_OK;
}

static int get_func(b200_ctx* c, const std::string& name, CUfunction* out) {
  c->last_kernel = name;
  if (c->dry) { c->pending_kernel = name; *out = nullptr; return B200_OK; }
  auto it = c->funcs.find(name);
  if (it != c->funcs.end()) { *out = it->second; return B200_OK; }
  // modules are loaded in the order gemm, reduce, aux, gemm_b, gemm_c, quant, gemm_q, quant_mm, gemm_conv, gemm_convbwd,
  // conv_grouped, gemm_conv3d, gemm_convt, attention, attention_bwd, attention_kv, attention_varlen, attention_varlen_bwd,
  // attention_kv_fp8; the kernel name says where a
  // kernel lives (no failing lookups, which API-level tools such as compute-sanitizer would report)
  auto starts = [&](const char* pfx) { return name.rfind(pfx, 0) == 0; };
  auto has = [&](const char* part) { return name.find(part) != std::string::npos; };
  const bool tc_gemm = starts("gemm_") && name != "gemm_simt_strided" && name != "gemm_scaled_simt";
  const size_t home = name == "conv3d_dgrad_weights" ? 2
                      : starts("attn_kv_") && (has("_e4m3_") || has("_e5m2_") || has("_fp8")) ? 18
                      : starts("attn_bwd_varlen_") ? 17
                      : starts("attn_fwd_varlen_") ? 16
                      : starts("attn_kv_") ? 15
                      : starts("attn_bwd_") ? 14
                      : starts("attn_") ? 13
                      : starts("conv2d_tconv_") || starts("conv3d_tconv_") ? 12
                      : starts("conv3d_") ? 11
                      : starts("conv2d_grp_") ? 10
                      : starts("conv2d_dgrad_") || starts("conv2d_wgrad_") ? 9
                      : starts("conv2d_") ? 8
                      : starts("gemm_q8") ? 6
                      : starts("quant_scales_") || starts("quant_widen_") ? 7
                      : starts("quant_") ? 5
                      : tc_gemm && (has("_2sm_n128_") || has("_2sm_n224_")) ? 3
                      : tc_gemm && (has("_1sm_n128_") || has("_2sm_m512_")) ? 4
                      : tc_gemm || starts("wgmma_probe_") ? 0
                      : starts("reduce_") || starts("scan_") ? 1 : 2;
  if (home < c->modules.size()) {
    CUfunction f;
    if (g_drv.cuModuleGetFunction_p(&f, c->modules[home], name.c_str()) == CUDA_SUCCESS) {
      c->funcs[name] = f;
      *out = f;
      return B200_OK;
    }
  }
  return fail(B200_ERR_COMPILATION, "kernel '%s' not found in the prebuilt cubins", name.c_str());
}

extern "C" int b200_get_cubin(const char* name, const void** image, size_t* size) {
  if (!name || !image || !size) return fail(B200_ERR_INVALID_ARG, "get_cubin: null argument");
  const unsigned char *b = nullptr, *e = nullptr;
  if (!strcmp(name, "gemm")) { b = b200_cubin_gemm; e = b200_cubin_gemm_end; }
  else if (!strcmp(name, "reduce")) { b = b200_cubin_reduce; e = b200_cubin_reduce_end; }
  else if (!strcmp(name, "aux")) { b = b200_cubin_aux; e = b200_cubin_aux_end; }
  else if (!strcmp(name, "gemm_b")) { b = b200_cubin_gemm_b; e = b200_cubin_gemm_b_end; }
  else if (!strcmp(name, "gemm_c")) { b = b200_cubin_gemm_c; e = b200_cubin_gemm_c_end; }
  else if (!strcmp(name, "quant")) { b = b200_cubin_quant; e = b200_cubin_quant_end; }
  else if (!strcmp(name, "gemm_q")) { b = b200_cubin_gemm_q; e = b200_cubin_gemm_q_end; }
  else if (!strcmp(name, "quant_mm")) { b = b200_cubin_quant_mm; e = b200_cubin_quant_mm_end; }
  else if (!strcmp(name, "gemm_conv")) { b = b200_cubin_gemm_conv; e = b200_cubin_gemm_conv_end; }
  else if (!strcmp(name, "gemm_convbwd")) { b = b200_cubin_gemm_convbwd; e = b200_cubin_gemm_convbwd_end; }
  else if (!strcmp(name, "conv_grouped")) { b = b200_cubin_conv_grouped; e = b200_cubin_conv_grouped_end; }
  else if (!strcmp(name, "gemm_conv3d")) { b = b200_cubin_gemm_conv3d; e = b200_cubin_gemm_conv3d_end; }
  else if (!strcmp(name, "gemm_convt")) { b = b200_cubin_gemm_convt; e = b200_cubin_gemm_convt_end; }
  else if (!strcmp(name, "attention")) { b = b200_cubin_attention; e = b200_cubin_attention_end; }
  else if (!strcmp(name, "attention_bwd")) { b = b200_cubin_attention_bwd; e = b200_cubin_attention_bwd_end; }
  else if (!strcmp(name, "attention_kv")) { b = b200_cubin_attention_kv; e = b200_cubin_attention_kv_end; }
  else if (!strcmp(name, "attention_varlen")) { b = b200_cubin_attention_varlen; e = b200_cubin_attention_varlen_end; }
  else if (!strcmp(name, "attention_varlen_bwd")) { b = b200_cubin_attention_varlen_bwd; e = b200_cubin_attention_varlen_bwd_end; }
  else if (!strcmp(name, "attention_kv_fp8")) { b = b200_cubin_attention_kv_fp8; e = b200_cubin_attention_kv_fp8_end; }
  else return fail(B200_ERR_INVALID_ARG, "get_cubin: unknown image '%s' (gemm|gemm_b|gemm_c|reduce|aux|quant|gemm_q|quant_mm|gemm_conv|gemm_convbwd|conv_grouped|gemm_conv3d|gemm_convt|attention|attention_bwd|attention_kv|attention_varlen|attention_varlen_bwd|attention_kv_fp8)", name);
  *image = b;
  *size = static_cast<size_t>(e - b);
  return B200_OK;
}

extern "C" int b200_device_count(int* count) {
  if (!count) return fail(B200_ERR_INVALID_ARG, "null count");
  int rc = ensure_driver();
  if (rc) return rc;
  CU_CHECK(g_drv.cuDeviceGetCount_p(count));
  return B200_OK;
}

extern "C" int b200_init(int device, b200_ctx** out) {
  if (!out) return fail(B200_ERR_INVALID_ARG, "null out");
  *out = nullptr;
  int rc = ensure_driver();
  if (rc) return rc;
  int n = 0;
  CU_CHECK(g_drv.cuDeviceGetCount_p(&n));
  if (device < 0 || device >= n) return fail(B200_ERR_NO_DEVICE, "device %d out of range (%d devices)", device, n);
  b200_ctx* c = new b200_ctx();
  c->device = device;
  auto bail = [&](int code) { delete c; return code; };
  CUresult r;
  if ((r = g_drv.cuDeviceGet_p(&c->dev, device)) != CUDA_SUCCESS) return bail(fail(map_cu(r), "cuDeviceGet: %s", cu_err(r)));
  if ((r = g_drv.cuDevicePrimaryCtxRetain_p(&c->cuctx, c->dev)) != CUDA_SUCCESS)
    return bail(fail(map_cu(r), "cuDevicePrimaryCtxRetain: %s", cu_err(r)));
  if ((r = g_drv.cuCtxSetCurrent_p(c->cuctx)) != CUDA_SUCCESS) return bail(fail(map_cu(r), "cuCtxSetCurrent: %s", cu_err(r)));
  auto attr = [&](CUdevice_attribute a) { int v = 0; g_drv.cuDeviceGetAttribute_p(&v, a, c->dev); return v; };
  c->props.device = device;
  c->props.cc_major = attr(CU_DEVICE_ATTRIBUTE_COMPUTE_CAPABILITY_MAJOR);
  c->props.cc_minor = attr(CU_DEVICE_ATTRIBUTE_COMPUTE_CAPABILITY_MINOR);
  c->props.num_sms = attr(CU_DEVICE_ATTRIBUTE_MULTIPROCESSOR_COUNT);
  c->props.max_shared_per_block = attr(CU_DEVICE_ATTRIBUTE_MAX_SHARED_MEMORY_PER_BLOCK_OPTIN);
  c->props.clock_khz = attr(CU_DEVICE_ATTRIBUTE_CLOCK_RATE);
  c->props.mem_clock_khz = attr(CU_DEVICE_ATTRIBUTE_MEMORY_CLOCK_RATE);
  c->props.plane_size = 32;
  size_t total = 0;
  g_drv.cuDeviceTotalMem_p(&total, c->dev);
  c->props.total_mem = total;
  g_drv.cuDeviceGetName_p(c->props.name, sizeof(c->props.name), c->dev);
  if (c->props.cc_major != 9 || c->props.cc_minor != 0) {
    g_drv.cuDevicePrimaryCtxRelease_p(c->dev);
    return bail(fail(B200_ERR_NO_DEVICE, "device %d is sm_%d%d; this library ships sm_90a cubins only (H100)", device,
                     c->props.cc_major, c->props.cc_minor));
  }
  if ((rc = load_module(c, b200_cubin_gemm, b200_cubin_gemm_end, "gemm")) ||
      (rc = load_module(c, b200_cubin_reduce, b200_cubin_reduce_end, "reduce")) ||
      (rc = load_module(c, b200_cubin_aux, b200_cubin_aux_end, "aux")) ||
      (rc = load_module(c, b200_cubin_gemm_b, b200_cubin_gemm_b_end, "gemm_b")) ||
      (rc = load_module(c, b200_cubin_gemm_c, b200_cubin_gemm_c_end, "gemm_c")) ||
      (rc = load_module(c, b200_cubin_quant, b200_cubin_quant_end, "quant")) ||
      (rc = load_module(c, b200_cubin_gemm_q, b200_cubin_gemm_q_end, "gemm_q")) ||
      (rc = load_module(c, b200_cubin_quant_mm, b200_cubin_quant_mm_end, "quant_mm")) ||
      (rc = load_module(c, b200_cubin_gemm_conv, b200_cubin_gemm_conv_end, "gemm_conv")) ||
      (rc = load_module(c, b200_cubin_gemm_convbwd, b200_cubin_gemm_convbwd_end, "gemm_convbwd")) ||
      (rc = load_module(c, b200_cubin_conv_grouped, b200_cubin_conv_grouped_end, "conv_grouped")) ||
      (rc = load_module(c, b200_cubin_gemm_conv3d, b200_cubin_gemm_conv3d_end, "gemm_conv3d")) ||
      (rc = load_module(c, b200_cubin_gemm_convt, b200_cubin_gemm_convt_end, "gemm_convt")) ||
      (rc = load_module(c, b200_cubin_attention, b200_cubin_attention_end, "attention")) ||
      (rc = load_module(c, b200_cubin_attention_bwd, b200_cubin_attention_bwd_end, "attention_bwd")) ||
      (rc = load_module(c, b200_cubin_attention_kv, b200_cubin_attention_kv_end, "attention_kv")) ||
      (rc = load_module(c, b200_cubin_attention_varlen, b200_cubin_attention_varlen_end, "attention_varlen")) ||
      (rc = load_module(c, b200_cubin_attention_varlen_bwd, b200_cubin_attention_varlen_bwd_end, "attention_varlen_bwd")) ||
      (rc = load_module(c, b200_cubin_attention_kv_fp8, b200_cubin_attention_kv_fp8_end, "attention_kv_fp8"))) {
    for (CUmodule m : c->modules) g_drv.cuModuleUnload_p(m);
    g_drv.cuDevicePrimaryCtxRelease_p(c->dev);
    return bail(rc);
  }
  if ((r = g_drv.cuStreamCreate_p(&c->stream, CU_STREAM_NON_BLOCKING)) != CUDA_SUCCESS ||
      (r = g_drv.cuStreamCreate_p(&c->comm_stream, CU_STREAM_NON_BLOCKING)) != CUDA_SUCCESS ||
      (r = g_drv.cuEventCreate_p(&c->comm_event, CU_EVENT_DISABLE_TIMING)) != CUDA_SUCCESS) {
    // release what exists: streams created so far, the loaded modules, the retained primary context
    if (c->comm_stream) g_drv.cuStreamDestroy_p(c->comm_stream);
    if (c->stream) g_drv.cuStreamDestroy_p(c->stream);
    for (CUmodule m : c->modules) g_drv.cuModuleUnload_p(m);
    g_drv.cuDevicePrimaryCtxRelease_p(c->dev);
    return bail(fail(map_cu(r), "stream/event creation failed: %s", cu_err(r)));
  }
  *out = c;
  return B200_OK;
}

extern "C" int b200_destroy(b200_ctx* c) {
  if (!c) return B200_OK;
  if (c->dry) { delete c; return B200_OK; }
  if (g_drv.ok && g_drv.cuCtxSetCurrent_p(c->cuctx) == CUDA_SUCCESS) {
    g_drv.cuCtxSynchronize_p();
    for (auto& kv : c->comms)
      if (kv.second.comm && g_nccl.ok) g_nccl.CommDestroy(kv.second.comm);
    for (auto& kv : c->p2p)
      for (CUdeviceptr q : kv.second.opened) g_drv.cuIpcCloseMemHandle_p(q);
    if (c->mailbox) g_drv.cuMemFree_p(c->mailbox);
    for (auto& kv : c->blocks) {
      if (kv.second.done) g_drv.cuEventDestroy_p(kv.second.done);
      g_drv.cuMemFree_p(kv.first);
    }
    for (auto& kv : c->reduce_ws) g_drv.cuMemFree_p(kv.second);
    for (auto& kv : c->pinned) g_drv.cuMemFreeHost_p(kv.first);
    if (c->comm_event) g_drv.cuEventDestroy_p(c->comm_event);
    if (c->comm_stream) g_drv.cuStreamDestroy_p(c->comm_stream);
    if (c->stream) g_drv.cuStreamDestroy_p(c->stream);
    for (CUmodule m : c->modules) g_drv.cuModuleUnload_p(m);
    g_drv.cuDevicePrimaryCtxRelease_p(c->dev);
  }
  delete c;
  return B200_OK;
}

extern "C" int b200_plan_begin(int num_sms, b200_ctx** out) {
  if (!out || num_sms < 1) return fail(B200_ERR_INVALID_ARG, "plan_begin: bad arguments");
  b200_ctx* c = new b200_ctx();
  c->dry = true;
  c->device = 0;
  c->props.num_sms = num_sms;
  c->props.cc_major = 9;
  c->props.plane_size = 32;
  snprintf(c->props.name, sizeof(c->props.name), "dry-run (%d SMs)", num_sms);
  *out = c;
  return B200_OK;
}

extern "C" int b200_plan_text(b200_ctx* c, char* buf, size_t capacity, size_t* needed) {
  if (!c || !c->dry) return fail(B200_ERR_INVALID_ARG, "plan_text: not a planning context");
  if (needed) *needed = c->plan.size() + 1;
  if (buf && capacity) {
    const size_t n = std::min(capacity - 1, c->plan.size());
    memcpy(buf, c->plan.data(), n);
    buf[n] = 0;
    if (capacity > c->plan.size()) c->plan.clear();
  }
  return B200_OK;
}

extern "C" int b200_get_props(b200_ctx* c, b200_props* out) {
  if (!c || !out) return fail(B200_ERR_INVALID_ARG, "null argument");
  *out = c->props;
  return B200_OK;
}

extern "C" int b200_set_option(b200_ctx* c, const char* key, const char* value) {
  if (!c || !key || !value) return fail(B200_ERR_INVALID_ARG, "null argument");
  static const char* known[] = {"gemm.variant", "gemm.f32", "gemm.group_m", "gemm.split_k", "gemm.epilogue", "gemm.l2_promotion", "gemm.stage", "reduce.variant", "reduce.threads",
                                "reduce.blocks_per_sm", "reduce.rows_vpt", "reduce.rows_blocks_per_sm", "reduce.cols_blocks_per_sm",
                                "reduce.debug", "reduce.pdl", "reduce.tma_stages", "reduce.tma_ctas_per_sm", "reduce.cols_split_target", "reduce.cols_loads", "reduce.cols_fused"};
  for (const char* k : known)
    if (!strcmp(k, key)) { c->options[key] = value; return B200_OK; }
  return fail(B200_ERR_INVALID_ARG, "unknown option '%s'", key);
}

extern "C" int b200_last_kernel(b200_ctx* c, char* buf, size_t capacity) {
  if (!c || !buf || capacity == 0) return fail(B200_ERR_INVALID_ARG, "last_kernel: bad arguments");
  snprintf(buf, capacity, "%s", c->last_kernel.c_str());
  return B200_OK;
}

extern "C" int b200_launch_count(b200_ctx* c, uint64_t* count) {
  if (!c || !count) return fail(B200_ERR_INVALID_ARG, "null argument");
  *count = c->launches;
  return B200_OK;
}

// ================================================================================================ memory
static size_t pool_round(size_t bytes) {
  if (bytes == 0) bytes = 1;
  const size_t align = bytes >= (64u << 20) ? (2u << 20) : bytes >= (1u << 20) ? (64u << 10) : 512;
  return (bytes + align - 1) / align * align;
}

static int pool_alloc(b200_ctx* c, size_t bytes, CUdeviceptr* out, CUstream for_stream = nullptr) {
  const size_t sz = pool_round(bytes);
  if (c->dry) {
    *out = c->fake_next;
    c->fake_next += (sz + 511) / 512 * 512;
    char line[96];
    snprintf(line, sizeof(line), "alloc %zu\n", sz);
    c->plan += line;
    return B200_OK;
  }
  auto it = c->free_lists.find(sz);
  if (it != c->free_lists.end()) {
    std::vector<CUdeviceptr>& fl = it->second;
    for (size_t i = fl.size(); i-- > 0;) {
      PoolBlock& b = c->blocks[fl[i]];
      bool usable = !b.pending || (for_stream != nullptr && b.last_stream == for_stream);
      if (!usable && b.done && g_drv.cuEventQuery_p(b.done) == CUDA_SUCCESS) { b.pending = false; usable = true; }
      if (!usable) continue;  // still in flight on another stream: leave it for later
      *out = fl[i];
      fl.erase(fl.begin() + static_cast<long>(i));
      b.in_use = true;
      c->bytes_in_use += sz;
      return B200_OK;
    }
  }
  CUdeviceptr p = 0;
  CUresult r = g_drv.cuMemAlloc_p(&p, sz);
  if (r == CUDA_ERROR_OUT_OF_MEMORY) {
    // release cached pages and retry once (memory_cleanup semantics); cuMemFree synchronises, so pending pages are safe
    for (auto& fl : c->free_lists) {
      for (CUdeviceptr q : fl.second) {
        PoolBlock& b = c->blocks[q];
        if (b.done) g_drv.cuEventDestroy_p(b.done);
        g_drv.cuMemFree_p(q);
        c->bytes_reserved -= fl.first;
        c->blocks.erase(q);
      }
      fl.second.clear();
    }
    r = g_drv.cuMemAlloc_p(&p, sz);
  }
  if (r != CUDA_SUCCESS) return fail(map_cu(r), "cuMemAlloc(%zu bytes) failed: %s", sz, cu_err(r));
  PoolBlock nb;
  nb.size = sz;
  nb.in_use = true;
  c->blocks[p] = nb;
  c->bytes_reserved += sz;
  c->bytes_in_use += sz;
  *out = p;
  return B200_OK;
}

// `used_on`: the stream whose queued work may still touch the page (nullptr = the context's compute stream).
static int pool_free(b200_ctx* c, CUdeviceptr p, CUstream used_on = nullptr) {
  if (c->dry) return B200_OK;
  auto it = c->blocks.find(p);
  if (it == c->blocks.end() || !it->second.in_use) return fail(B200_ERR_INVALID_ARG, "b200_free: pointer not owned by this context");
  PoolBlock& b = it->second;
  b.in_use = false;
  // a stream this context already destroyed was synchronised at that point: the page is idle as far as it is concerned
  if (used_on && std::find(c->dead_streams.begin(), c->dead_streams.end(), used_on) != c->dead_streams.end()) used_on = nullptr;
  b.last_stream = used_on ? used_on : c->stream;
  if (!b.done && g_drv.cuEventCreate_p(&b.done, CU_EVENT_DISABLE_TIMING) != CUDA_SUCCESS) b.done = nullptr;
  b.pending = (b.done != nullptr) && g_drv.cuEventRecord_p(b.done, b.last_stream) == CUDA_SUCCESS;
  c->bytes_in_use -= b.size;
  c->free_lists[b.size].push_back(p);
  return B200_OK;
}

extern "C" int b200_alloc(b200_ctx* c, size_t bytes, b200_dptr* out) {
  CTX_ENTER(c);
  if (!out) return fail(B200_ERR_INVALID_ARG, "null out");
  CUdeviceptr p;
  int rc = pool_alloc(c, bytes, &p);
  if (rc) return rc;
  *out = static_cast<b200_dptr>(p);
  return B200_OK;
}

extern "C" int b200_free(b200_ctx* c, b200_dptr ptr) {
  CTX_ENTER(c);
  return pool_free(c, static_cast<CUdeviceptr>(ptr));
}

// The stream-ordered form: `last_use` is the stream whose queued work may still touch the buffer (NULL = the context's
// stream).  The page is handed out again only once an event recorded there has completed (or to that same stream).
extern "C" int b200_free_async(b200_ctx* c, b200_dptr ptr, b200_stream last_use) {
  CTX_ENTER(c);
  return pool_free(c, static_cast<CUdeviceptr>(ptr), resolve_stream(c, last_use));
}

extern "C" int b200_memory_usage(b200_ctx* c, uint64_t* in_use, uint64_t* reserved) {
  if (!c) return fail(B200_ERR_INVALID_ARG, "null context");
  if (in_use) *in_use = c->bytes_in_use;
  if (reserved) *reserved = c->bytes_reserved;
  return B200_OK;
}

extern "C" int b200_memory_cleanup(b200_ctx* c) {
  CTX_ENTER_DEVICE(c);
  CU_CHECK(g_drv.cuCtxSynchronize_p());
  for (auto& fl : c->free_lists) {
    for (CUdeviceptr q : fl.second) {
      PoolBlock& b = c->blocks[q];
      if (b.done) g_drv.cuEventDestroy_p(b.done);
      g_drv.cuMemFree_p(q);
      c->bytes_reserved -= fl.first;
      c->blocks.erase(q);
    }
    fl.second.clear();
  }
  return B200_OK;
}

extern "C" int b200_host_alloc(b200_ctx* c, size_t bytes, void** out) {
  CTX_ENTER_DEVICE(c);
  if (!out) return fail(B200_ERR_INVALID_ARG, "null out");
  void* p = nullptr;
  CU_CHECK(g_drv.cuMemAllocHost_p(&p, bytes ? bytes : 1));
  c->pinned[p] = bytes;
  *out = p;
  return B200_OK;
}

extern "C" int b200_host_free(b200_ctx* c, void* ptr) {
  CTX_ENTER_DEVICE(c);
  auto it = c->pinned.find(ptr);
  if (it == c->pinned.end()) return fail(B200_ERR_INVALID_ARG, "b200_host_free: pointer not owned by this context");
  CU_CHECK(g_drv.cuMemFreeHost_p(ptr));
  c->pinned.erase(it);
  return B200_OK;
}

extern "C" int b200_write(b200_ctx* c, b200_stream s, b200_dptr dst, const void* src, size_t bytes) {
  CTX_ENTER_DEVICE(c);
  if (bytes == 0) return B200_OK;
  CU_CHECK(g_drv.cuMemcpyHtoDAsync_p(static_cast<CUdeviceptr>(dst), src, bytes, resolve_stream(c, s)));
  return B200_OK;
}

extern "C" int b200_read(b200_ctx* c, b200_stream s, void* dst, b200_dptr src, size_t bytes) {
  CTX_ENTER_DEVICE(c);
  if (bytes == 0) return B200_OK;
  CU_CHECK(g_drv.cuMemcpyDtoHAsync_p(dst, static_cast<CUdeviceptr>(src), bytes, resolve_stream(c, s)));
  return B200_OK;
}

extern "C" int b200_copy(b200_ctx* c, b200_stream s, b200_dptr dst, b200_dptr src, size_t bytes) {
  CTX_ENTER_DEVICE(c);
  if (bytes == 0) return B200_OK;
  CU_CHECK(g_drv.cuMemcpyDtoDAsync_p(static_cast<CUdeviceptr>(dst), static_cast<CUdeviceptr>(src), bytes, resolve_stream(c, s)));
  return B200_OK;
}

extern "C" int b200_memset32(b200_ctx* c, b200_stream s, b200_dptr dst, uint32_t value, size_t words) {
  CTX_ENTER_DEVICE(c);
  if (words == 0) return B200_OK;
  CU_CHECK(g_drv.cuMemsetD32Async_p(static_cast<CUdeviceptr>(dst), value, words, resolve_stream(c, s)));
  return B200_OK;
}

// ================================================================================================ streams / events
extern "C" int b200_stream_create(b200_ctx* c, b200_stream* out) {
  CTX_ENTER_DEVICE(c);
  if (!out) return fail(B200_ERR_INVALID_ARG, "null out");
  CUstream s;
  CU_CHECK(g_drv.cuStreamCreate_p(&s, CU_STREAM_NON_BLOCKING));
  c->dead_streams.erase(std::remove(c->dead_streams.begin(), c->dead_streams.end(), s), c->dead_streams.end());  // the handle value may be recycled
  *out = s;
  return B200_OK;
}

extern "C" int b200_stream_destroy(b200_ctx* c, b200_stream s) {
  CTX_ENTER_DEVICE(c);
  if (!s) return B200_OK;
  CU_CHECK(g_drv.cuStreamSynchronize_p(static_cast<CUstream>(s)));   // pages freed on this stream are idle from here on
  for (auto& kv : c->blocks)
    if (kv.second.last_stream == static_cast<CUstream>(s)) { kv.second.last_stream = nullptr; kv.second.pending = false; }
  auto it = c->reduce_ws.find(static_cast<CUstream>(s));
  if (it != c->reduce_ws.end()) { g_drv.cuMemFree_p(it->second); c->reduce_ws.erase(it); }
  CU_CHECK(g_drv.cuStreamDestroy_p(static_cast<CUstream>(s)));
  c->dead_streams.push_back(static_cast<CUstream>(s));
  return B200_OK;
}

extern "C" int b200_sync(b200_ctx* c, b200_stream s) {
  CTX_ENTER(c);
  if (c->dry) return B200_OK;
  CUresult r = g_drv.cuStreamSynchronize_p(resolve_stream(c, s));
  if (r != CUDA_SUCCESS) return fail(B200_ERR_UNHEALTHY, "stream sync surfaced a device fault: %s (%d)", cu_err(r), (int)r);
  return B200_OK;
}

extern "C" int b200_event_create(b200_ctx* c, b200_event* out) {
  CTX_ENTER_DEVICE(c);
  if (!out) return fail(B200_ERR_INVALID_ARG, "null out");
  CUevent e;
  CU_CHECK(g_drv.cuEventCreate_p(&e, CU_EVENT_DEFAULT));
  *out = e;
  return B200_OK;
}

extern "C" int b200_event_record(b200_ctx* c, b200_event e, b200_stream s) {
  CTX_ENTER_DEVICE(c);
  CU_CHECK(g_drv.cuEventRecord_p(static_cast<CUevent>(e), resolve_stream(c, s)));
  return B200_OK;
}

extern "C" int b200_stream_wait_event(b200_ctx* c, b200_stream s, b200_event e) {
  CTX_ENTER_DEVICE(c);
  CU_CHECK(g_drv.cuStreamWaitEvent_p(resolve_stream(c, s), static_cast<CUevent>(e), 0));
  return B200_OK;
}

extern "C" int b200_event_elapsed_ms(b200_ctx* c, b200_event a, b200_event b, float* ms) {
  CTX_ENTER_DEVICE(c);
  if (!ms) return fail(B200_ERR_INVALID_ARG, "null ms");
  CU_CHECK(g_drv.cuEventSynchronize_p(static_cast<CUevent>(b)));
  CU_CHECK(g_drv.cuEventElapsedTime_p(ms, static_cast<CUevent>(a), static_cast<CUevent>(b)));
  return B200_OK;
}

extern "C" int b200_event_destroy(b200_ctx* c, b200_event e) {
  CTX_ENTER_DEVICE(c);
  if (e) CU_CHECK(g_drv.cuEventDestroy_p(static_cast<CUevent>(e)));
  return B200_OK;
}

// ================================================================================================ launch helper
static int launch(b200_ctx* c, CUfunction f, unsigned grid_x, unsigned grid_y, unsigned grid_z, unsigned block,
                  unsigned smem, unsigned cluster_x, CUstream st, void** args, bool pdl = false) {
  CUlaunchConfig cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDimX = grid_x; cfg.gridDimY = grid_y; cfg.gridDimZ = grid_z;
  cfg.blockDimX = block; cfg.blockDimY = 1; cfg.blockDimZ = 1;
  cfg.sharedMemBytes = smem;
  cfg.hStream = st;
  CUlaunchAttribute at[2];
  unsigned nat = 0;
  if (cluster_x > 1) {
    at[nat].id = CU_LAUNCH_ATTRIBUTE_CLUSTER_DIMENSION;
    at[nat].value.clusterDim.x = cluster_x; at[nat].value.clusterDim.y = 1; at[nat].value.clusterDim.z = 1;
    ++nat;
  }
  if (pdl) {  // this kernel may begin once every block of the preceding kernel has triggered (griddepcontrol) or exited
    at[nat].id = CU_LAUNCH_ATTRIBUTE_PROGRAMMATIC_STREAM_SERIALIZATION;
    at[nat].value.programmaticStreamSerializationAllowed = 1;
    ++nat;
  }
  if (nat) { cfg.attrs = at; cfg.numAttrs = nat; }
  if (st == c->stream) c->pdl_prev_out = 0;   // whoever launches a reduce_all sets it again after this call
  if (c->dry) {
    char line[256];
    snprintf(line, sizeof(line), "launch %s grid=(%u,%u,%u) block=%u smem=%u cluster=%u%s\n", c->pending_kernel.c_str(), grid_x,
             grid_y, grid_z, block, smem, cluster_x, pdl ? " pdl" : "");
    c->plan += line;
    c->launches++;
    return B200_OK;
  }
  CUresult r = g_drv.cuLaunchKernelEx_p(&cfg, f, args, nullptr);
  if (r != CUDA_SUCCESS) return fail(map_cu(r), "cuLaunchKernelEx failed: %s (%d)", cu_err(r), (int)r);
  c->launches++;
  return B200_OK;
}

static size_t dtype_size(int dt) {
  switch (dt) {
    case B200_F32: case B200_U32: case B200_I32: return 4;
    case B200_F16: case B200_BF16: return 2;
    case B200_F64: case B200_I64: case B200_U64: return 8;
    case B200_U8: case B200_I8: case B200_F8E4M3: case B200_F8E5M2: return 1;
    default: return 0;
  }
}

// ================================================================================================ matmul
struct GemmVariant {
  const char* tag;  // suffix in the kernel name
  int cg, block_n, stages;
  double eff;       // MMA-pipe efficiency assumed relative to 2sm_n256 (not measured on H100): the 128-wide tiles issue
                    // m64n128 wgmma, which moves twice the shared-memory operand bytes per FLOP of m64n256.
                    // 0 = never chosen automatically (gemm.variant=<tag> only)
  int mt;           // 128-row sub-tiles of M per CTA: the tile is (128 * cg * mt) x block_n
};
static const GemmVariant kVariants[] = {{"2sm_n256", 2, 256, 4, 1.0, 1}, {"2sm_n128", 2, 128, 6, 0.9, 1}, {"1sm_n128", 1, 128, 6, 0.85, 1},
                                        // 512 x 128 pair tile (256 rows per CTA), 16-bit kinds; opt-in until measured
                                        {"2sm_m512", 2, 128, 4, 0.0, 2},
                                        // block-scaled kinds only: 256 x 224 pair tile; opt-in until measured
                                        {"2sm_n224", 2, 224, 4, 0.0, 1}};
// alignment slack + operand ring (A: 128 * mt rows, B: block_n rows, 128 B of K each) + barrier block + TMA-store staging
static unsigned gemm_smem_bytes(const GemmVariant& v) { return 1024 + v.stages * (16384 * v.mt + v.block_n * 128) + 1024 + 16384; }
// The per-block quantized kernels (gemm_q8_*) add f32 scale tiles for (128 + block_n) rows x 4 blocks to every stage and run
// the largest stage count that fits 227 KB (gemm_wgmma.cu: GEMM_Q).
static int gemm_q8_stages(const GemmVariant& v) { return v.block_n == 256 ? 3 : 5; }
static unsigned gemm_q8_smem_bytes(const GemmVariant& v) {
  return 1024 + gemm_q8_stages(v) * (16384 + v.block_n * 128 + (128 + v.block_n) * 16) + 1024 + 16384;
}

static int encode_tmap(b200_ctx* c, CUtensorMap* out, CUtensorMapDataType dt, size_t esz, uint64_t base, uint64_t d0,
                       uint64_t d1, uint64_t d2, uint64_t s1_elems, uint64_t s2_elems, uint32_t b0, uint32_t b1,
                       CUtensorMapSwizzle swz = CU_TENSOR_MAP_SWIZZLE_128B, uint32_t b2 = 1) {
  // L2 promotion: how much of a line's neighbourhood a TMA load pulls into L2 (tuning knob; 256 B measured best so far)
  const int promo_bytes = atoi(opt(c, "gemm.l2_promotion", "256").c_str());
  const CUtensorMapL2promotion promo = promo_bytes >= 256 ? CU_TENSOR_MAP_L2_PROMOTION_L2_256B
                                       : promo_bytes >= 128 ? CU_TENSOR_MAP_L2_PROMOTION_L2_128B
                                       : promo_bytes >= 64 ? CU_TENSOR_MAP_L2_PROMOTION_L2_64B : CU_TENSOR_MAP_L2_PROMOTION_NONE;
  char key[256];
  snprintf(key, sizeof(key), "%d|%d|%llx|%llu|%llu|%llu|%llu|%llu|%u|%u|%u|%d", (int)dt, (int)swz, (unsigned long long)base,
           (unsigned long long)d0, (unsigned long long)d1, (unsigned long long)d2, (unsigned long long)s1_elems,
           (unsigned long long)s2_elems, b0, b1, b2, (int)promo);
  if (c->dry) {
    char line[256];
    if (b2 == 1)
      snprintf(line, sizeof(line), "tmap esz=%zu dims=(%llu,%llu,%llu) strides=(%llu,%llu) box=(%u,%u) swizzle=%d\n", esz,
               (unsigned long long)d0, (unsigned long long)d1, (unsigned long long)d2, (unsigned long long)(s1_elems * esz),
               (unsigned long long)(s2_elems * esz), b0, b1, (int)swz);
    else
      snprintf(line, sizeof(line), "tmap esz=%zu dims=(%llu,%llu,%llu) strides=(%llu,%llu) box=(%u,%u,%u) swizzle=%d\n", esz,
               (unsigned long long)d0, (unsigned long long)d1, (unsigned long long)d2, (unsigned long long)(s1_elems * esz),
               (unsigned long long)(s2_elems * esz), b0, b1, b2, (int)swz);
    c->plan += line;
    memset(out, 0, sizeof(*out));
    return B200_OK;
  }
  auto it = c->tmap_cache.find(key);
  if (it != c->tmap_cache.end()) { *out = it->second; return B200_OK; }
  cuuint64_t dims[3] = {d0, d1, d2};
  cuuint64_t strides[2] = {s1_elems * esz, s2_elems * esz};
  cuuint32_t box[3] = {b0, b1, b2};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = g_drv.cuTensorMapEncodeTiled_p(out, dt, 3, reinterpret_cast<void*>(base), dims, strides, box, estr,
                                              CU_TENSOR_MAP_INTERLEAVE_NONE, swz, promo, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return fail(B200_ERR_INVALID_ARG, "cuTensorMapEncodeTiled failed: %s (dims %llu,%llu,%llu strides %llu,%llu box %u,%u)",
                cu_err(r), (unsigned long long)d0, (unsigned long long)d1, (unsigned long long)d2,
                (unsigned long long)strides[0], (unsigned long long)strides[1], b0, b1);
  if (c->tmap_cache.size() > 512) c->tmap_cache.clear();
  c->tmap_cache[key] = *out;
  return B200_OK;
}

// 4-D im2col map of an NHWC tensor (dims innermost first: C, W, H, N; strides of W, H, N in elements), SWIZZLE_128B, zero
// out-of-bounds fill.  Corners (w, h) bound the pixels a load walks; estr_w / estr_h are the conv strides.  Same cache as
// encode_tmap.
static int encode_im2col(b200_ctx* c, CUtensorMap* out, CUtensorMapDataType dt, size_t esz, uint64_t base, const uint64_t dims[4],
                         const uint64_t strides[3], const int lower[2], const int upper[2], uint32_t channels, uint32_t pixels,
                         uint32_t estr_w, uint32_t estr_h) {
  const int promo_bytes = atoi(opt(c, "gemm.l2_promotion", "256").c_str());
  const CUtensorMapL2promotion promo = promo_bytes >= 256 ? CU_TENSOR_MAP_L2_PROMOTION_L2_256B
                                       : promo_bytes >= 128 ? CU_TENSOR_MAP_L2_PROMOTION_L2_128B
                                       : promo_bytes >= 64 ? CU_TENSOR_MAP_L2_PROMOTION_L2_64B : CU_TENSOR_MAP_L2_PROMOTION_NONE;
  char key[320];
  snprintf(key, sizeof(key), "im2col|%d|%llx|%llu|%llu|%llu|%llu|%llu|%llu|%llu|%d|%d|%d|%d|%u|%u|%u|%u|%d", (int)dt,
           (unsigned long long)base, (unsigned long long)dims[0], (unsigned long long)dims[1], (unsigned long long)dims[2],
           (unsigned long long)dims[3], (unsigned long long)strides[0], (unsigned long long)strides[1], (unsigned long long)strides[2],
           lower[0], lower[1], upper[0], upper[1], channels, pixels, estr_w, estr_h, (int)promo);
  if (c->dry) {
    char line[320];
    snprintf(line, sizeof(line),
             "tmap im2col esz=%zu dims=(%llu,%llu,%llu,%llu) strides=(%llu,%llu,%llu) lower=(%d,%d) upper=(%d,%d) channels=%u pixels=%u "
             "estrides=(1,%u,%u,1) swizzle=%d\n",
             esz, (unsigned long long)dims[0], (unsigned long long)dims[1], (unsigned long long)dims[2], (unsigned long long)dims[3],
             (unsigned long long)(strides[0] * esz), (unsigned long long)(strides[1] * esz), (unsigned long long)(strides[2] * esz),
             lower[0], lower[1], upper[0], upper[1], channels, pixels, estr_w, estr_h, (int)CU_TENSOR_MAP_SWIZZLE_128B);
    c->plan += line;
    memset(out, 0, sizeof(*out));
    return B200_OK;
  }
  auto it = c->tmap_cache.find(key);
  if (it != c->tmap_cache.end()) { *out = it->second; return B200_OK; }
  cuuint64_t gdim[4] = {dims[0], dims[1], dims[2], dims[3]};
  cuuint64_t gstr[3] = {strides[0] * esz, strides[1] * esz, strides[2] * esz};
  cuuint32_t estr[4] = {1, estr_w, estr_h, 1};
  CUresult r = g_drv.cuTensorMapEncodeIm2col_p(out, dt, 4, reinterpret_cast<void*>(base), gdim, gstr, lower, upper, channels, pixels, estr,
                                               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, promo,
                                               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return fail(B200_ERR_INVALID_ARG, "cuTensorMapEncodeIm2col failed: %s (dims %llu,%llu,%llu,%llu corners (%d,%d)..(%d,%d))", cu_err(r),
                (unsigned long long)dims[0], (unsigned long long)dims[1], (unsigned long long)dims[2], (unsigned long long)dims[3],
                lower[0], lower[1], upper[0], upper[1]);
  if (c->tmap_cache.size() > 512) c->tmap_cache.clear();
  c->tmap_cache[key] = *out;
  return B200_OK;
}

// 5-D im2col map of an NDHWC tensor (dims innermost first: C, W, H, D, N; strides of W, H, D, N in elements): as
// encode_im2col with a depth dimension.  Corners (w, h, d) must lie in [-16, 15] (cuda.h, rank 5); estr_* are the conv strides.
static int encode_im2col5(b200_ctx* c, CUtensorMap* out, CUtensorMapDataType dt, size_t esz, uint64_t base, const uint64_t dims[5],
                          const uint64_t strides[4], const int lower[3], const int upper[3], uint32_t channels, uint32_t pixels,
                          const uint32_t estr_whd[3]) {
  const int promo_bytes = atoi(opt(c, "gemm.l2_promotion", "256").c_str());
  const CUtensorMapL2promotion promo = promo_bytes >= 256 ? CU_TENSOR_MAP_L2_PROMOTION_L2_256B
                                       : promo_bytes >= 128 ? CU_TENSOR_MAP_L2_PROMOTION_L2_128B
                                       : promo_bytes >= 64 ? CU_TENSOR_MAP_L2_PROMOTION_L2_64B : CU_TENSOR_MAP_L2_PROMOTION_NONE;
  std::string key = "im2col5d|" + std::to_string((int)dt) + "|" + std::to_string(base);
  for (int i = 0; i < 5; ++i) key += "|" + std::to_string(dims[i]);
  for (int i = 0; i < 4; ++i) key += "|" + std::to_string(strides[i]);
  for (int i = 0; i < 3; ++i) key += "|" + std::to_string(lower[i]) + "|" + std::to_string(upper[i]) + "|" + std::to_string(estr_whd[i]);
  key += "|" + std::to_string(channels) + "|" + std::to_string(pixels) + "|" + std::to_string((int)promo);
  if (c->dry) {
    char line[400];
    snprintf(line, sizeof(line),
             "tmap im2col5d esz=%zu dims=(%llu,%llu,%llu,%llu,%llu) strides=(%llu,%llu,%llu,%llu) lower=(%d,%d,%d) upper=(%d,%d,%d) "
             "channels=%u pixels=%u estrides=(1,%u,%u,%u,1) swizzle=%d\n",
             esz, (unsigned long long)dims[0], (unsigned long long)dims[1], (unsigned long long)dims[2], (unsigned long long)dims[3],
             (unsigned long long)dims[4], (unsigned long long)(strides[0] * esz), (unsigned long long)(strides[1] * esz),
             (unsigned long long)(strides[2] * esz), (unsigned long long)(strides[3] * esz), lower[0], lower[1], lower[2], upper[0],
             upper[1], upper[2], channels, pixels, estr_whd[0], estr_whd[1], estr_whd[2], (int)CU_TENSOR_MAP_SWIZZLE_128B);
    c->plan += line;
    memset(out, 0, sizeof(*out));
    return B200_OK;
  }
  auto it = c->tmap_cache.find(key);
  if (it != c->tmap_cache.end()) { *out = it->second; return B200_OK; }
  cuuint64_t gdim[5] = {dims[0], dims[1], dims[2], dims[3], dims[4]};
  cuuint64_t gstr[4] = {strides[0] * esz, strides[1] * esz, strides[2] * esz, strides[3] * esz};
  cuuint32_t estr[5] = {1, estr_whd[0], estr_whd[1], estr_whd[2], 1};
  CUresult r = g_drv.cuTensorMapEncodeIm2col_p(out, dt, 5, reinterpret_cast<void*>(base), gdim, gstr, lower, upper, channels, pixels, estr,
                                               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, promo,
                                               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return fail(B200_ERR_INVALID_ARG, "cuTensorMapEncodeIm2col (rank 5) failed: %s (dims %llu,%llu,%llu,%llu,%llu corners (%d,%d,%d)..(%d,%d,%d))",
                cu_err(r), (unsigned long long)dims[0], (unsigned long long)dims[1], (unsigned long long)dims[2], (unsigned long long)dims[3],
                (unsigned long long)dims[4], lower[0], lower[1], lower[2], upper[0], upper[1], upper[2]);
  if (c->tmap_cache.size() > 512) c->tmap_cache.clear();
  c->tmap_cache[key] = *out;
  return B200_OK;
}

// Geometry of a 2-D convolution run as an implicit GEMM (b200_conv2d): x is NHWC with unit channel stride, w is
// [Cout, KH * KW, C] with unit channel stride; strides in elements.
struct ConvGeom {
  uint64_t N, H, W, C, KH, KW, OH, OW, Cout;
  int32_t sh, sw, ph, pw, dh, dw;
  uint64_t x_sw, x_sh, x_sn;   // x: pixel (w), row (h) and image (n) strides
  uint64_t w_sp, w_sco;        // w: kernel-position and output-channel strides
  // An explicit, asymmetric pixel box (stride 1 only): the im2col walk covers OW x OH pixels from the lower corner
  // (lo_w, lo_h) instead of the forward's (-pw, -ph) .. (pw - dw (KW - 1), ph - dh (KH - 1)).  A data-gradient phase.
  bool box = false;
  int32_t lo_h = 0, lo_w = 0;
  // 0: the forward (conv2d_*); 1: a data-gradient phase with the phase-addressed epilogue (conv2d_dgrad_*, dx_* strides);
  // 2: the weight gradient (conv2d_wgrad_*): A = dy [Cout x pixels], B = x through im2col, out = dw (dw_sp, dw_c)
  int mode = 0;
  uint64_t dx_sn = 0, dx_si = 0, dx_sj = 0;
  uint64_t dw_sp = 0, dw_c = 0;
  // 3-D convolution (b200_conv3d*): dims = 3 adds a depth dimension to everything above (x strides x_sd, a pixel box corner
  // lo_d, dx stride dx_sd per phase row).  The defaults leave every 2-D path as it is.
  int dims = 2;
  uint64_t D = 1, KD = 1, OD = 1;
  int32_t sd = 1, pd = 0, dd = 1, lo_d = 0;
  uint64_t x_sd = 0, dx_sd = 0;
};

// One batched problem with LINEAR batch strides (0 = broadcast).  Strides in elements.
struct GemmProblem {
  int in_dtype, out_dtype;
  int rhs_dtype = -1;           // >= 0: a mixed 8-bit pair (fp8 e4m3 x e5m2, u8 x i8); in_dtype is then the lhs format
  uint64_t a, b, out;
  uint64_t a_lo = 0, b_lo = 0;  // 3xTF32: compact low parts (same logical layout class as a / b), 0 otherwise
  bool mx = false;              // block-scaled operands expanded to bf16: the gemm_mx_* kernels (promoted accumulation)
  bool hybrid = false;          // a_lo / b_lo are bf16 PAIR buffers [2][entries][rows][pitch]: bf16(x) planes, then bf16(x - trunc_tf32(x))
  uint64_t bias = 0;            // fused epilogue: out = act(alpha * acc + bias[n])
  float alpha = 1.0f;
  uint32_t act = 0;
  uint64_t M, N, K, batch;
  uint64_t a_sm, a_sk, a_sb;
  uint64_t b_sk, b_sn, b_sb;
  uint64_t o_sm, o_sn, o_sb;
  // integer-quantized operands (b200_matmul_quantized): s8 codes, K-major.  q = 1: per-block scales folded per Bk block of K
  // from the f32 effective-scale buffers sa_q / sb_q ([batch][K / Bk][rows padded to 4]); q = 2: per-tensor scales g_a, g_b
  // read from the device in the epilogue
  int q = 0;
  uint32_t q_bk = 0;
  uint64_t q_sa = 0, q_sb = 0, q_ga = 0, q_gb = 0;
  // 2-D convolution (b200_conv2d): a = x, b = w, M = N * OH * OW, N = Cout, K = KH * KW * (C padded to 64), batch 1
  const ConvGeom* conv = nullptr;
  uint64_t sk_max_parts = 8;    // stream-K head: at most this many ranges per tile (sk_plan)
};

static bool variant_has(const GemmVariant& v, const GemmProblem& g) {
  if (g.conv) return !strcmp(v.tag, "2sm_n128") || !strcmp(v.tag, "1sm_n128");   // gemm_wgmma.cu: GEMM_PART 4
  if (g.q == 1 && v.block_n == 256) return false;   // the per-block fold has 128-wide tiles only (gemm_wgmma.cu: GEMM_Q)
  if (!strcmp(v.tag, "2sm_n224")) return g.mx;
  if (!strcmp(v.tag, "2sm_m512")) return !g.mx && (g.in_dtype == B200_BF16 || g.in_dtype == B200_F16);
  return true;
}

static int launch_simt(b200_ctx* c, CUstream st, const GemmProblem& g) {
  CUfunction f;
  int rc = get_func(c, "gemm_simt_strided", &f);
  if (rc) return rc;
  if (g.batch > 65535) return fail(B200_ERR_UNSUPPORTED, "simt matmul: batch %llu > 65535", (unsigned long long)g.batch);
  if (g.M >= (1ull << 32) || g.N >= (1ull << 32) || g.K >= (1ull << 32))
    return fail(B200_ERR_UNSUPPORTED, "simt matmul: extents must fit 32 bits (M=%llu N=%llu K=%llu)", (unsigned long long)g.M,
                (unsigned long long)g.N, (unsigned long long)g.K);
  const uint32_t epi_on = (g.alpha != 1.0f || g.bias != 0 || g.act != 0) ? 1u : 0u;
  SimtGemmParams p{g.a, g.b, g.out, g.a_sb, g.a_sm, g.a_sk, g.b_sb, g.b_sk, g.b_sn, g.o_sb, g.o_sm, g.o_sn,
                   (uint32_t)g.M, (uint32_t)g.N, (uint32_t)g.K, (uint32_t)g.batch, (uint32_t)g.in_dtype, (uint32_t)g.out_dtype,
                   g.bias, g.alpha, g.act, epi_on, g.rhs_dtype >= 0 ? (uint32_t)g.rhs_dtype + 1u : 0u};
  void* args[] = {&p};
  // gridDim.y is limited to 65535: taller problems (M > 1,048,560) walk their 16-row tiles with a stride of gridDim.y
  const uint64_t tiles_m = (g.M + 15) / 16;
  return launch(c, f, (unsigned)((g.N + 15) / 16), (unsigned)std::min<uint64_t>(tiles_m, 65535), (unsigned)g.batch, 256, 0, 1, st, args);
}

// Can TMA describe one operand in place?  `mn` x K elements, strides in elements.  K-major (rows of K) or MN-major (rows of
// the M / N extent): unit inner stride, 16-byte aligned base, row pitch and batch stride, pitch >= row, strides < 2^40 bytes.
static bool operand_tma_ok(uint64_t ptr, size_t esz, uint64_t mn, uint64_t K, uint64_t s_mn, uint64_t s_k, uint64_t s_b, bool* mn_major) {
  auto al16 = [&](uint64_t elems) { return (elems * esz) % 16 == 0; };
  const uint64_t lim = 1ull << 40;
  if (ptr % 16 || !al16(s_b)) return false;
  if (s_mn * esz >= lim || s_k * esz >= lim || s_b * esz >= lim) return false;
  if ((s_k == 1 || K == 1) && (mn == 1 || (al16(s_mn) && s_mn >= K))) { *mn_major = false; return true; }
  if ((s_mn == 1 || mn == 1) && (K == 1 || (al16(s_k) && s_k >= mn))) { *mn_major = true; return true; }
  return false;
}
static bool extents_tma_ok(const GemmProblem& g) {
  return g.M < (1ull << 31) && g.N < (1ull << 31) && g.K < (1ull << 31) && g.batch < (1ull << 31) && (g.o_sn == 1 || g.N == 1);
}
static bool tma_ok(const GemmProblem& g, bool* a_mn, bool* b_mn) {
  const size_t esz = dtype_size(g.in_dtype);
  return extents_tma_ok(g) && operand_tma_ok(g.a, esz, g.M, g.K, g.a_sm, g.a_sk, g.a_sb, a_mn) &&
         operand_tma_ok(g.b, esz, g.N, g.K, g.b_sn, g.b_sk, g.b_sb, b_mn);
}

static int reduce_workspace(b200_ctx* c, CUstream st, CUdeviceptr* out);

// Stream-K head plan for `tiles` tiles on `clusters` clusters (gemm_wgmma.cu, GemmParams): the rem = tiles % clusters
// tiles that would form a partial last wave are instead cut along K into `ranges` equal ranges processed FIRST, so all
// clusters stay busy and the slab exchange runs under the whole tiles that follow.
//   time (in tile-times) without: full_waves + 1.
//   with: full_waves + 1.4 * head + overhead / num_kb, head = ceil(ranges / clusters) * share / num_kb.
// While the head runs, S clusters stream the operands of ONE tile, so the phase needs S times the operand bandwidth of a
// normal wave with less panel sharing in L2; the model charges it 1.4x its MMA time.  Equal parts (ranges = rem * S) are
// preferred to an even cut over all clusters whenever they fit, so S = floor(clusters / rem) when that is >= 2.  The
// exchange is modelled as hidden when whole tiles follow (~4 k-block times) and exposed, (14 + 8 parts) k-block times, when
// the head is the whole problem.  These constants are not measured on H100.
// gemm.split_k: auto (only when the model gains >= 4 %), off, on (whenever rem != 0), or N = 1..8 (N ranges per tile).
struct SkPlan {
  double time = 0;           // modelled time in tile-times
  uint64_t sk_tiles = 0, ranges = 0, umax = 0;
  bool bad_option = false;
};
// max_parts caps the ranges per tile of the automatic plan (8 for every GEMM but the convolution weight gradient, whose few
// tiles have a very long K).
static SkPlan sk_plan(uint64_t tiles, uint64_t clusters, uint64_t num_kb, const std::string& option, bool eligible,
                      uint64_t max_parts = 8) {
  SkPlan pl;
  const uint64_t full_waves = tiles / clusters, rem = tiles % clusters;
  pl.time = static_cast<double>(full_waves + (rem ? 1 : 0));
  if (option == "off" || !eligible || rem == 0 || num_kb < 2) return pl;
  const uint64_t total_kb = rem * num_kb;
  auto model = [&](uint64_t ranges, bool even_parts) {
    const uint64_t share = (total_kb + ranges - 1) / ranges;
    const double parts = std::max(1.0, static_cast<double>(ranges) / static_cast<double>(rem));
    const double head = static_cast<double>((ranges + clusters - 1) / clusters) * static_cast<double>(share) / static_cast<double>(num_kb);
    const double overhead = (full_waves >= 1 ? 4.0 : 14.0 + 8.0 * parts) / static_cast<double>(num_kb);
    return static_cast<double>(full_waves) + (even_parts ? 1.4 : 1.6) * head + overhead;
  };
  uint64_t ranges = 0;
  bool force = false, even = true;
  if (option == "auto" || option == "on") {
    force = (option == "on");
    const uint64_t s_fit = std::min<uint64_t>(clusters / rem, max_parts);
    if (s_fit >= 2) {
      // equal parts; when whole tiles follow, as many as fit; when the head is everything, the S the model likes best
      uint64_t best_s = s_fit;
      if (full_waves == 0)
        for (uint64_t s2 = 2; s2 <= s_fit; ++s2)
          if (num_kb / s2 >= 8 && model(rem * s2, true) < model(rem * best_s, true) - 1e-12) best_s = s2;
      ranges = rem * best_s;
    } else {
      ranges = clusters;       // more than half a wave of tiles: an even cut over all pairs, tiles in 1-2 uneven parts
      even = false;
    }
  } else {
    const int want = atoi(option.c_str());
    if (want < 1 || want > 8) { pl.bad_option = true; return pl; }
    if (want == 1) return pl;
    ranges = rem * static_cast<uint64_t>(want);
    force = true;
  }
  ranges = std::min(ranges, total_kb);                                    // every range owns at least one k-block
  if (ranges <= rem && !force) return pl;                                 // no tile would be cut
  const uint64_t share = (total_kb + ranges - 1) / ranges;
  const double t_sk = model(ranges, even);
  if (!force) {
    if (share < 8) return pl;                                             // slices too thin to amortise an exchange
    if (t_sk > 0.96 * pl.time) return pl;
  }
  pl.time = t_sk;
  pl.sk_tiles = rem;
  pl.ranges = ranges;
  pl.umax = (share + num_kb - 1) / num_kb + 1;                            // tiles one range can touch
  return pl;
}

// k-blocks (pipeline stages) one tile's K loop runs: 3xTF32 walks K three times; the hybrid f32 schedule once in tf32 stages
// (32 elements) and twice in bf16 stages (64 elements)
static uint64_t gemm_num_kb(const GemmProblem& g, uint32_t block_k) {
  const uint64_t seg = (g.K + block_k - 1) / block_k;
  if (!(g.a_lo != 0 && g.b_lo != 0)) return seg;
  return g.hybrid ? seg + 2 * ((g.K + 63) / 64) : 3 * seg;
}

// Tile variant by modelled time (ties -> larger tile, less L2 traffic): waves of tiles, with the last partial wave replaced by a
// stream-K head where that pays (sk_plan).  nullptr: gemm.variant names no variant this dtype / kind has.
// stream_k = false: a launch that plans no stream-K head (whole tiles only) is costed by its waves alone.
static const GemmVariant* pick_variant(b200_ctx* c, const GemmProblem& g, SkPlan* sk_out, bool stream_k = true) {
  const size_t esz = dtype_size(g.in_dtype);
  const uint32_t block_k = static_cast<uint32_t>(128 / esz);
  const std::string forced = opt(c, "gemm.variant", "auto");
  const std::string split_opt = opt(c, "gemm.split_k", "auto");
  const bool float_acc = !(g.in_dtype == B200_U8 || g.in_dtype == B200_I8);
  const uint64_t num_kb = gemm_num_kb(g, block_k);
  const GemmVariant* best = nullptr;
  double best_cost = 0;
  for (const GemmVariant& v : kVariants) {
    if (forced != "auto" && forced != v.tag) continue;
    if (forced == "auto" && v.eff <= 0.0) continue;
    if (!variant_has(v, g)) continue;
    if (forced == "auto" && v.cg == 2 && g.M <= 128) continue;  // a CTA pair would idle its second half: one CTA per tile
    const uint64_t tile_m = 128ull * v.cg * v.mt;
    const uint64_t tm = (g.M + tile_m - 1) / tile_m, tn = (g.N + v.block_n - 1) / v.block_n;
    const uint64_t tiles = tm * tn * g.batch;
    const uint64_t clusters = std::max(1, c->props.num_sms / v.cg);
    // the slab exchange is a per-128-row-CTA-tile protocol with f32 accumulators: not for the 512-row tile, not for integers
    const SkPlan sk = sk_plan(tiles, clusters, num_kb, split_opt, float_acc && v.mt == 1 && stream_k, g.sk_max_parts);
    const double eff = v.eff > 0 ? v.eff : 1.0;
    const double cost = sk.time * (128.0 * v.mt * v.block_n) / eff;  // per-SM MMA time
    if (!best || cost < best_cost * 0.999) { best = &v; best_cost = cost; *sk_out = sk; }
  }
  return best;
}

static int launch_wgmma(b200_ctx* c, CUstream st, const GemmProblem& g, bool a_mn, bool b_mn) {
  const size_t esz = dtype_size(g.in_dtype), osz = dtype_size(g.out_dtype);
  const char* in_tag = g.q == 1 ? "q8" : g.q == 2 ? "q8t" : g.mx ? "mx" : g.in_dtype == B200_BF16 ? "bf16" : g.in_dtype == B200_F16 ? "f16" : g.in_dtype == B200_F8E4M3 ? "e4m3"
                       : g.in_dtype == B200_F8E5M2 ? "e5m2" : g.in_dtype == B200_U8 ? "u8" : g.in_dtype == B200_I8 ? "s8" : "tf32";
  const char* out_tag = g.out_dtype == B200_BF16 ? "bf16" : g.out_dtype == B200_F16 ? "f16" : g.out_dtype == B200_I32 ? "i32" : "f32";
  const uint32_t block_k = static_cast<uint32_t>(128 / esz);
  const std::string forced = opt(c, "gemm.variant", "auto");
  const uint64_t k_segments = (g.a_lo != 0 && g.b_lo != 0) ? 3 : 1;
  SkPlan best_sk;
  const GemmVariant* best = pick_variant(c, g, &best_sk);
  if (!best) return fail(B200_ERR_INVALID_ARG, "gemm.variant '%s' is not a wgmma variant", forced.c_str());
  if (best_sk.bad_option) return fail(B200_ERR_INVALID_ARG, "gemm.split_k must be auto, off, on or 1..8");
  const GemmVariant& v = *best;

  const int cmode = g.conv ? g.conv->mode : 0;
  const bool cv3 = g.conv && g.conv->dims == 3;
  const std::string cpfx = cv3 ? "conv3d_" : "conv2d_";
  const std::string name = g.conv ? cpfx + (cmode == 1 ? "dgrad_" : cmode == 2 ? "wgrad_" : "") + in_tag + "_" + out_tag + "_" + v.tag
                                  : std::string("gemm_") + in_tag + "_" + out_tag + "_" + v.tag + (a_mn ? "_m" : "_k") + (b_mn ? "n" : "k");
  CUfunction f;
  int rc = get_func(c, name, &f);
  if (rc) return rc;
  const unsigned smem = g.q == 1 ? gemm_q8_smem_bytes(v) : gemm_smem_bytes(v);
  if (!c->dry) CU_CHECK(g_drv.cuFuncSetAttribute_p(f, CU_FUNC_ATTRIBUTE_MAX_DYNAMIC_SHARED_SIZE_BYTES, (int)smem));

  const CUtensorMapDataType dt = g.in_dtype == B200_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                                 : g.in_dtype == B200_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16
                                 : esz == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8
                                            : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
  const bool a_bcast = (g.a_sb == 0 || g.batch == 1), b_bcast = (g.b_sb == 0 || g.batch == 1);
  CUtensorMap ta, tb;
  auto pad16 = [&](uint64_t elems) { const uint64_t q = 16 / esz; return (elems + q - 1) / q * q; };
  const uint32_t chunk = static_cast<uint32_t>(128 / esz);  // MN-major operands (16-bit): elements per 128-byte row
  const uint32_t n_local = v.block_n / v.cg;   // B rows each CTA of a pair loads (multicast to both)
  // im2col map of the convolution input: `pixels` output pixels x 64 channels per load, walking the input pixels the output
  // grid reads at kernel position (0, 0)
  auto conv_im2col = [&](CUtensorMap* m, uint64_t base, uint32_t pixels) {
    const ConvGeom& cv = *g.conv;
    if (cv.dims == 3) {
      const uint64_t dims5[5] = {cv.C, cv.W, cv.H, cv.D, cv.N}, strides4[4] = {cv.x_sw, cv.x_sh, cv.x_sd, cv.x_sn};
      int lo[3] = {-cv.pw, -cv.ph, -cv.pd};
      int up[3] = {cv.pw - cv.dw * (int)(cv.KW - 1), cv.ph - cv.dh * (int)(cv.KH - 1), cv.pd - cv.dd * (int)(cv.KD - 1)};
      if (cv.box) {
        lo[0] = cv.lo_w; lo[1] = cv.lo_h; lo[2] = cv.lo_d;
        up[0] = cv.lo_w + (int)cv.OW - (int)cv.W; up[1] = cv.lo_h + (int)cv.OH - (int)cv.H; up[2] = cv.lo_d + (int)cv.OD - (int)cv.D;
      }
      const uint32_t estr[3] = {(uint32_t)cv.sw, (uint32_t)cv.sh, (uint32_t)cv.sd};
      return encode_im2col5(c, m, dt, esz, base, dims5, strides4, lo, up, 64, pixels, estr);
    }
    const uint64_t dims[4] = {cv.C, cv.W, cv.H, cv.N}, strides[3] = {cv.x_sw, cv.x_sh, cv.x_sn};
    int lower[2] = {-cv.pw, -cv.ph};
    int upper[2] = {cv.pw - cv.dw * (int)(cv.KW - 1), cv.ph - cv.dh * (int)(cv.KH - 1)};
    if (cv.box) {
      lower[0] = cv.lo_w; lower[1] = cv.lo_h;
      upper[0] = cv.lo_w + (int)cv.OW - (int)cv.W; upper[1] = cv.lo_h + (int)cv.OH - (int)cv.H;
    }
    return encode_im2col(c, m, dt, esz, base, dims, strides, lower, upper, 64, pixels, (uint32_t)cv.sw, (uint32_t)cv.sh);
  };
  if (g.conv && cmode != 2) {
    rc = conv_im2col(&ta, g.a, 128);
  } else if (!a_mn) {
    const uint64_t a_sm = g.M > 1 ? g.a_sm : pad16(g.K);
    rc = encode_tmap(c, &ta, dt, esz, g.a, g.K, g.M, a_bcast ? 1 : g.batch, a_sm, a_bcast ? a_sm * g.M : g.a_sb, block_k, 128);
  } else {
    const uint64_t a_sk = g.K > 1 ? g.a_sk : pad16(g.M);
    rc = encode_tmap(c, &ta, dt, esz, g.a, g.M, g.K, a_bcast ? 1 : g.batch, a_sk, a_bcast ? a_sk * g.K : g.a_sb, chunk, block_k);
  }
  if (rc) return rc;
  if (cmode == 2) {
    // weight gradient: 64 pixels x 64 channels of x per MN-major B chunk
    rc = conv_im2col(&tb, g.b, 64);
  } else if (g.conv) {
    // [n_local output channels x 64 channels] of one kernel position
    const ConvGeom& cv = *g.conv;
    rc = encode_tmap(c, &tb, dt, esz, g.b, cv.C, cv.KD * cv.KH * cv.KW, cv.Cout, cv.w_sp, cv.w_sco, 64, 1, CU_TENSOR_MAP_SWIZZLE_128B, n_local);
  } else if (!b_mn) {
    const uint64_t b_sn = g.N > 1 ? g.b_sn : pad16(g.K);
    rc = encode_tmap(c, &tb, dt, esz, g.b, g.K, g.N, b_bcast ? 1 : g.batch, b_sn, b_bcast ? b_sn * g.N : g.b_sb, block_k, n_local);
  } else {
    const uint64_t b_sk = g.K > 1 ? g.b_sk : pad16(g.N);
    rc = encode_tmap(c, &tb, dt, esz, g.b, g.N, g.K, b_bcast ? 1 : g.batch, b_sk, b_bcast ? b_sk * g.K : g.b_sb, chunk, block_k);
  }
  if (rc) return rc;
  // 3xTF32: compact low parts (K-major: [rows, K]); hybrid: bf16 pair buffers
  CUtensorMap ta_lo = ta, tb_lo = tb;
  const bool split = (g.a_lo != 0 && g.b_lo != 0);
  if (split && g.hybrid) {
    // bf16 pair buffers: planes [0, entries) = bf16(x), [entries, 2 entries) = bf16(lo); 64 elements of K per stage
    const uint64_t ab = a_bcast ? 1 : g.batch, bb = b_bcast ? 1 : g.batch;
    auto pad8 = [](uint64_t e) { return (e + 7) / 8 * 8; };
    const CUtensorMapDataType d16 = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
    rc = encode_tmap(c, &ta_lo, d16, 2, g.a_lo, g.K, g.M, 2 * ab, pad8(g.K), pad8(g.K) * g.M, 64, 128);
    if (rc) return rc;
    rc = encode_tmap(c, &tb_lo, d16, 2, g.b_lo, g.K, g.N, 2 * bb, pad8(g.K), pad8(g.K) * g.N, 64, n_local);
    if (rc) return rc;
  } else if (split) {
    const uint64_t ab = a_bcast ? 1 : g.batch, bb = b_bcast ? 1 : g.batch;
    rc = encode_tmap(c, &ta_lo, dt, esz, g.a_lo, g.K, g.M, ab, pad16(g.K), pad16(g.K) * g.M, block_k, 128);
    if (rc) return rc;
    rc = encode_tmap(c, &tb_lo, dt, esz, g.b_lo, g.K, g.N, bb, pad16(g.K), pad16(g.K) * g.N, block_k, n_local);
    if (rc) return rc;
  } else if (g.q == 1) {
    // effective-scale tiles of one stage: [128 / Bk blocks][128 rows] of A, [128 / Bk][block_n] of B (no swizzle)
    const uint64_t nblk = g.K / g.q_bk, ra = (g.M + 3) / 4 * 4, rb = (g.N + 3) / 4 * 4;
    const uint32_t nsub = 128u / g.q_bk;
    rc = encode_tmap(c, &ta_lo, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, g.q_sa, ra, nblk, a_bcast ? 1 : g.batch, ra, ra * nblk, 128, nsub,
                     CU_TENSOR_MAP_SWIZZLE_NONE);
    if (rc) return rc;
    rc = encode_tmap(c, &tb_lo, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, g.q_sb, rb, nblk, b_bcast ? 1 : g.batch, rb, rb * nblk,
                     (uint32_t)v.block_n, nsub, CU_TENSOR_MAP_SWIZZLE_NONE);
    if (rc) return rc;
  }

  GemmParams p;
  memset(&p, 0, sizeof(p));
  if (g.rhs_dtype >= 0 && g.rhs_dtype != g.in_dtype) {
    p.fmt_b = (g.rhs_dtype == B200_F8E5M2 || g.rhs_dtype == B200_I8) ? 1u : 0u;   // 0 = e4m3 / u8, 1 = e5m2 / s8
    p.fmt_mixed = 1;
  }
  p.k_segments = (uint32_t)k_segments;
  if (split && g.hybrid) {
    p.hyb = 1;
    p.hyb_nba = a_bcast ? 1u : (uint32_t)g.batch;
    p.hyb_nbb = b_bcast ? 1u : (uint32_t)g.batch;
  }
  if (g.q == 1) p.q_nsub = 128u / g.q_bk;
  if (g.conv) {
    const ConvGeom& cv = *g.conv;
    p.cv_ohw = (uint32_t)(cv.OH * cv.OW); p.cv_ow = (uint32_t)cv.OW;
    p.cv_cblk = (uint32_t)((cv.C + 63) / 64); p.cv_kw = (uint32_t)cv.KW;
    p.cv_stride_h = cv.sh; p.cv_stride_w = cv.sw; p.cv_pad_h = cv.ph; p.cv_pad_w = cv.pw;
    p.cv_dil_h = (uint32_t)cv.dh; p.cv_dil_w = (uint32_t)cv.dw;
    p.dx_sn = cv.dx_sn; p.dx_si = cv.dx_si; p.dx_sj = cv.dx_sj;
    p.dw_sp = cv.dw_sp; p.dw_c = (uint32_t)cv.dw_c;
    if (cv.dims == 3) {
      p.cv_odhw = (uint32_t)(cv.OD * cv.OH * cv.OW); p.cv_khw = (uint32_t)(cv.KH * cv.KW);
      p.cv_stride_d = cv.sd; p.cv_pad_d = cv.pd; p.cv_dil_d = (uint32_t)cv.dd;
      p.dx_sd = cv.dx_sd;
    }
  }
  p.q_ga = g.q_ga; p.q_gb = g.q_gb;
  p.alpha = g.alpha; p.bias = g.bias; p.epi_act = g.act;
  p.epi_on = (g.alpha != 1.0f || g.bias != 0 || g.act != 0) ? 1u : 0u;
  p.out = g.out;
  p.out_row_stride = g.o_sm;
  p.out_batch_stride = g.o_sb;
  p.M = (uint32_t)g.M; p.N = (uint32_t)g.N; p.K = (uint32_t)g.K; p.batch = (uint32_t)g.batch;
  p.tiles_m = (uint32_t)((g.M + 128 * v.cg * v.mt - 1) / (128 * v.cg * v.mt));
  p.tiles_n = (uint32_t)((g.N + v.block_n - 1) / v.block_n);
  p.group_m = (uint32_t)std::max(1, atoi(opt(c, "gemm.group_m", "8").c_str()));
  p.a_bmul = a_bcast ? 0 : 1;
  p.b_bmul = b_bcast ? 0 : 1;
  p.vec_store = (g.out % 16 == 0 && (g.o_sm * osz) % 16 == 0 && (g.o_sb * osz) % 16 == 0) ? 1 : 0;
  if (cmode == 1 && ((p.dx_sn * osz) % 16 || (p.dx_si * osz) % 16 || (p.dx_sj * osz) % 16 || (p.dx_sd * osz) % 16)) p.vec_store = 0;
  if (cmode == 2 && (p.dw_sp * osz) % 16) p.vec_store = 0;
  // whole tiles leave through swizzled staging tiles and TMA stores when `out` is describable: (N, M, batch), [128 B x 64 rows] boxes
  const std::string epi = opt(c, "gemm.epilogue", "tma");
  if (epi != "tma" && epi != "direct") return fail(B200_ERR_INVALID_ARG, "gemm.epilogue must be tma or direct");
  CUtensorMap tout;
  memset(&tout, 0, sizeof(tout));
  const uint64_t lim40 = 1ull << 40;
  if (cmode == 2 && p.vec_store && epi == "tma" && g.o_sm * osz < lim40 && p.dw_sp * osz < lim40) {
    // dw as (C, Cout, KD * KH * KW): a staging tile of 64-column chunk (kpos, ch0) lands at (ch0, co, kpos), clipped at C
    const ConvGeom& cv = *g.conv;
    rc = encode_tmap(c, &tout, osz == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_UINT16, osz, g.out, cv.dw_c, g.M,
                     cv.KD * cv.KH * cv.KW, g.o_sm, cv.dw_sp, static_cast<uint32_t>(128 / osz), 64);
    if (rc) return rc;
    p.tma_store = 1;
  } else if (cmode == 0 && p.vec_store && epi == "tma" && g.o_sm * osz < lim40 && g.o_sb * osz < lim40 && (g.M == 1 || g.o_sm >= g.N)) {
    const uint64_t o_sm = g.M > 1 ? g.o_sm : (g.N + 15) / 16 * 16;
    const uint64_t o_sb = g.batch > 1 ? g.o_sb : o_sm * g.M;
    rc = encode_tmap(c, &tout, osz == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_UINT16, osz, g.out, g.N, g.M, g.batch,
                     o_sm, o_sb, static_cast<uint32_t>(128 / osz), 64);
    if (rc) return rc;
    p.tma_store = 1;
  }

  const uint64_t total_tiles = static_cast<uint64_t>(p.tiles_m) * p.tiles_n * p.batch;
  if (total_tiles >= (1ull << 32)) return fail(B200_ERR_UNSUPPORTED, "too many tiles");
  const unsigned max_clusters = (unsigned)std::max(1, c->props.num_sms / v.cg);
  unsigned clusters = (unsigned)std::min<uint64_t>(total_tiles, max_clusters);

  // Stream-K head (plan chosen with the variant above)
  CUdeviceptr slabs = 0;
  p.full_tiles = (uint32_t)total_tiles;
  if (best_sk.sk_tiles) {
    if (best_sk.sk_tiles * v.cg > kWsGemmTickets) return fail(B200_ERR_UNSUPPORTED, "stream-K head: %llu tiles exceed the ticket area", (unsigned long long)best_sk.sk_tiles);
    CUdeviceptr ws = 0;
    rc = reduce_workspace(c, st, &ws);
    if (rc) return rc;
    const uint64_t slab_bytes = 128ull * v.cg * v.block_n * 4;
    rc = pool_alloc(c, best_sk.ranges * best_sk.umax * slab_bytes, &slabs, st);
    if (rc) return rc;
    p.full_tiles = (uint32_t)(total_tiles - best_sk.sk_tiles);
    p.sk_tiles = (uint32_t)best_sk.sk_tiles;
    p.sk_ranges = (uint32_t)best_sk.ranges;
    p.sk_umax = (uint32_t)best_sk.umax;
    p.split_ws = slabs;
    p.split_tickets = ws + kWsGemmTicketOffset;
    // the head's ranges are dealt to clusters 0 .. ranges-1 (mod the grid); whole tiles to every cluster
    clusters = (unsigned)std::min<uint64_t>(std::max<uint64_t>(p.full_tiles, best_sk.ranges), max_clusters);
    if (c->dry) {
      char line[200];
      snprintf(line, sizeof(line), "gemm stream-k head: %u whole tiles + %u tiles in %u k-ranges (<= %u slabs per range)\n", p.full_tiles, p.sk_tiles,
               p.sk_ranges, p.sk_umax);
      c->plan += line;
    }
  }
  void* args[] = {&ta, &tb, &ta_lo, &tb_lo, &tout, &p};
  rc = launch(c, f, clusters * v.cg, 1, 1, 384, smem, v.cg, st, args);
  if (slabs) pool_free(c, slabs, st);  // stream-ordered: reusable by later work once this launch has drained
  return rc;
}

static inline uint64_t pad4(uint64_t elems) { return (elems + 3) / 4 * 4; }

// lo = x - trunc_tf32(x) of a logical [batch, rows, cols] view (cols innermost), written with row pitch pad4(cols)
static int launch_split(b200_ctx* c, CUstream st, uint64_t in, uint64_t out, uint64_t batch, uint64_t rows, uint64_t cols,
                        uint64_t in_bs, uint64_t in_rs) {
  CUfunction f;
  int rc = get_func(c, "split_tf32_lo", &f);
  if (rc) return rc;
  SplitParams p{in, out, batch, rows, cols, in_bs, in_rs, pad4(cols)};
  const uint64_t total = batch * rows * cols;
  const unsigned grid = (unsigned)std::min<uint64_t>((total / 4 + 255) / 256 + 1, (uint64_t)c->props.num_sms * 16);
  void* args[] = {&p};
  return launch(c, f, std::max(1u, grid), 1, 1, 256, 0, 1, st, args);
}

// bf16 pair of a logical [batch, rows, cols] f32 view: plane 0 = bf16(x), plane 1 = bf16(x - trunc_tf32(x)), rows pitched to 8 elements
static inline uint64_t pad8e(uint64_t elems) { return (elems + 7) / 8 * 8; }
static int launch_split_pair(b200_ctx* c, CUstream st, uint64_t in, uint64_t out, uint64_t batch, uint64_t rows, uint64_t cols,
                             uint64_t in_bs, uint64_t in_rs) {
  CUfunction f;
  int rc = get_func(c, "split_f32_bf16_pair", &f);
  if (rc) return rc;
  SplitParams p{in, out, batch, rows, cols, in_bs, in_rs, pad8e(cols)};
  const uint64_t total = batch * rows * cols;
  const unsigned grid = (unsigned)std::min<uint64_t>((total / 8 + 255) / 256 + 1, (uint64_t)c->props.num_sms * 16);
  void* args[] = {&p};
  return launch(c, f, std::max(1u, grid), 1, 1, 256, 0, 1, st, args);
}

// One pass that copies an operand TMA cannot describe (row pitch or base not 16-byte aligned, no unit stride) into a pooled
// buffer it can: [batch, rows, pitch] with the operand's own contiguous dimension innermost when it has one.
static int stage_operand(b200_ctx* c, CUstream st, size_t esz, uint64_t ptr, uint64_t batch, uint64_t mn, uint64_t K, uint64_t s_mn, uint64_t s_k,
                         uint64_t s_b, CUdeviceptr* out, uint64_t* o_smn, uint64_t* o_sk, uint64_t* o_sb) {
  // rows of the M / N extent are kept (coalesced both ways) where wgmma reads them: 16-bit operands
  const bool keep_mn_major = (s_mn == 1 && s_k != 1) && esz == 2;
  const uint64_t rows = keep_mn_major ? K : mn, cols = keep_mn_major ? mn : K;
  const uint64_t q = 16 / esz, pitch = (cols + q - 1) / q * q;
  const uint64_t nb = (s_b == 0) ? 1 : batch;                  // a broadcast operand is staged once
  CUdeviceptr buf;
  int rc = pool_alloc(c, nb * rows * pitch * esz, &buf, st);
  if (rc) return rc;
  CUfunction f;
  rc = get_func(c, "repitch_rows", &f);
  if (rc) { pool_free(c, buf, st); return rc; }
  RepitchParams p{ptr, buf, nb, rows, cols, s_b, keep_mn_major ? s_k : s_mn, keep_mn_major ? s_mn : s_k, pitch, (uint32_t)esz, 0};
  const uint64_t vecs = nb * rows * (pitch / q);               // one 16-byte output vector per thread
  const unsigned grid = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>((vecs + 255) / 256, 0x7FFFFFFFull));
  void* args[] = {&p};
  rc = launch(c, f, grid, 1, 1, 256, 0, 1, st, args);
  if (rc) { pool_free(c, buf, st); return rc; }
  *out = buf;
  *o_smn = keep_mn_major ? 1 : pitch;
  *o_sk = keep_mn_major ? pitch : 1;
  *o_sb = (s_b == 0) ? 0 : rows * pitch;
  return B200_OK;
}

static int run_gemm_staged(b200_ctx* c, CUstream st, const GemmProblem& g);
static int run_gemm(b200_ctx* c, CUstream st, const GemmProblem& g);

// An fp8 operand widened to f16 (exact) in a pooled [batch, rows, pitch] buffer that keeps the operand's own contiguous
// dimension innermost when it has one (wgmma reads 16-bit operands in either major).
static int widen_fp8_operand(b200_ctx* c, CUstream st, int dtype, uint64_t ptr, uint64_t batch, uint64_t mn, uint64_t K, uint64_t s_mn,
                             uint64_t s_k, uint64_t s_b, CUdeviceptr* out, uint64_t* o_smn, uint64_t* o_sk, uint64_t* o_sb) {
  const bool keep_mn_major = (s_mn == 1 && s_k != 1);
  const uint64_t rows = keep_mn_major ? K : mn, cols = keep_mn_major ? mn : K;
  const uint64_t pitch = (cols + 7) / 8 * 8;
  const uint64_t nb = (s_b == 0) ? 1 : batch;
  CUdeviceptr buf;
  int rc = pool_alloc(c, nb * rows * pitch * 2, &buf, st);
  if (rc) return rc;
  CUfunction f;
  rc = get_func(c, "convert_fp8_f16", &f);
  if (rc) { pool_free(c, buf, st); return rc; }
  ConvertF16Params p{ptr, buf, nb, rows, cols, s_b, keep_mn_major ? s_k : s_mn, keep_mn_major ? s_mn : s_k, pitch, (uint32_t)dtype, 0};
  const uint64_t vecs = nb * rows * (pitch / 8);
  const unsigned grid = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>((vecs + 255) / 256, (uint64_t)c->props.num_sms * 16));
  void* args[] = {&p};
  rc = launch(c, f, grid, 1, 1, 256, 0, 1, st, args);
  if (rc) { pool_free(c, buf, st); return rc; }
  *out = buf;
  *o_smn = keep_mn_major ? 1 : pitch;
  *o_sk = keep_mn_major ? pitch : 1;
  *o_sb = (s_b == 0) ? 0 : rows * pitch;
  return B200_OK;
}

// fp8 products accumulate with less than f32 precision in wgmma; the reference's expectation is an f32 sum of exact products.
// Both operands are widened to f16 (exact for e4m3 and e5m2, mixed pairs included) and the f16 kernels accumulate in f32.
static int run_gemm_fp8_as_f16(b200_ctx* c, CUstream st, const GemmProblem& g) {
  const int rdt = g.rhs_dtype >= 0 ? g.rhs_dtype : g.in_dtype;
  GemmProblem h = g;
  h.in_dtype = B200_F16;
  h.rhs_dtype = -1;
  CUdeviceptr wa = 0, wb = 0;
  int rc = widen_fp8_operand(c, st, g.in_dtype, g.a, g.batch, g.M, g.K, g.a_sm, g.a_sk, g.a_sb, &wa, &h.a_sm, &h.a_sk, &h.a_sb);
  if (!rc) rc = widen_fp8_operand(c, st, rdt, g.b, g.batch, g.N, g.K, g.b_sn, g.b_sk, g.b_sb, &wb, &h.b_sn, &h.b_sk, &h.b_sb);
  if (!rc) {
    h.a = wa;
    h.b = wb;
    rc = run_gemm(c, st, h);
  }
  if (wa) pool_free(c, wa, st);
  if (wb) pool_free(c, wb, st);
  return rc;
}

static int run_gemm(b200_ctx* c, CUstream st, const GemmProblem& g) {
  if (g.M == 0 || g.N == 0 || g.batch == 0) return B200_OK;
  const std::string forced = opt(c, "gemm.variant", "auto");
  bool a_mn = false, b_mn = false;
  const bool tma = g.K > 0 && tma_ok(g, &a_mn, &b_mn);
  const bool big = g.M * g.N * g.K * g.batch >= (1ull << 21);
  const bool fp8 = (g.in_dtype == B200_F8E4M3 || g.in_dtype == B200_F8E5M2);
  if (fp8 && forced != "simt" && g.K > 0 && extents_tma_ok(g) && (tma || (forced == "auto" && big && opt(c, "gemm.stage", "on") == "on")))
    return run_gemm_fp8_as_f16(c, st, g);
  // wgmma reads MN-major operands for 16-bit types only: tf32 / 8-bit operands in that layout are staged K-major first
  if (tma && forced != "simt" && dtype_size(g.in_dtype) != 2 && (a_mn || b_mn)) return run_gemm_staged(c, st, g);
  if (forced == "simt" || !tma) {
    if (forced != "simt" && forced != "auto")
      return fail(B200_ERR_UNSUPPORTED, "gemm.variant=%s forced but operands are not TMA-describable", forced.c_str());
    // Operands whose pitch / base TMA cannot describe (bf16 with K = 4097, an odd sub-view): one staging pass into an
    // aligned pooled copy, then the tensor-core kernel -- the strided SIMT kernel is kept for tiny problems and for
    // outputs without a unit inner stride.  gemm.stage=off keeps the SIMT path (reference-order arithmetic) for everything.
    if (forced == "auto" && g.K > 0 && big && extents_tma_ok(g) && opt(c, "gemm.stage", "on") == "on") return run_gemm_staged(c, st, g);
    return launch_simt(c, st, g);
  }
  const std::string f32_mode = g.in_dtype == B200_F32 ? opt(c, "gemm.f32", "hybrid") : std::string();
  if (g.in_dtype == B200_F32 && f32_mode != "hybrid" && f32_mode != "3xtf32" && f32_mode != "tf32")
    return fail(B200_ERR_INVALID_ARG, "gemm.f32 must be hybrid, 3xtf32 or tf32");
  if (f32_mode == "hybrid") {
    // f32-grade product in TWO tensor passes' worth of time, one launch: x = hi + lo with hi = the top 19 bits (what the tf32
    // datapath reads from the original tensor).  hi*hi runs as kind::tf32 on the originals; the cross terms A*B_lo + A_lo*B run
    // as kind::f16 on bf16 copies (bf16(A), bf16(B_lo), bf16(A_lo), bf16(B)) at twice the tf32 rate, into the same f32
    // accumulators.  The cross terms are ~2^-11 of the product, so their bf16 rounding (2^-9) lands at ~2^-20 of it.
    const uint64_t ab = (g.a_sb == 0) ? 1 : g.batch, bb = (g.b_sb == 0) ? 1 : g.batch;
    const uint64_t a_elems = !a_mn ? g.M * pad8e(g.K) : g.K * pad8e(g.M), b_elems = !b_mn ? g.N * pad8e(g.K) : g.K * pad8e(g.N);
    CUdeviceptr a_p = 0, b_p = 0;
    int rc = pool_alloc(c, 2 * ab * a_elems * 2, &a_p, st);
    if (rc) return rc;
    rc = pool_alloc(c, 2 * bb * b_elems * 2, &b_p, st);
    if (rc) { pool_free(c, a_p, st); return rc; }
    rc = !a_mn ? launch_split_pair(c, st, g.a, a_p, ab, g.M, g.K, g.a_sb, g.a_sm) : launch_split_pair(c, st, g.a, a_p, ab, g.K, g.M, g.a_sb, g.a_sk);
    if (!rc) rc = !b_mn ? launch_split_pair(c, st, g.b, b_p, bb, g.N, g.K, g.b_sb, g.b_sn) : launch_split_pair(c, st, g.b, b_p, bb, g.K, g.N, g.b_sb, g.b_sk);
    if (!rc) {
      GemmProblem h = g;
      h.a_lo = a_p;
      h.b_lo = b_p;
      h.hybrid = true;
      rc = launch_wgmma(c, st, h, a_mn, b_mn);
    }
    pool_free(c, a_p, st);
    pool_free(c, b_p, st);
    return rc;
  }
  if (f32_mode == "3xtf32") {
    // 3xTF32 in ONE GEMM launch: the tf32 datapath reads only the top 19 bits of an f32 operand, so the original tensors
    // are the "hi" parts; only lo = x - hi is materialised (compact), and the kernel runs K three times:
    // (A,B) + (A,B_lo) + (A_lo,B), f32 accumulation throughout.
    const uint64_t ab = (g.a_sb == 0) ? 1 : g.batch, bb = (g.b_sb == 0) ? 1 : g.batch;
    const uint64_t a_elems = !a_mn ? g.M * pad4(g.K) : g.K * pad4(g.M), b_elems = !b_mn ? g.N * pad4(g.K) : g.K * pad4(g.N);
    CUdeviceptr a_lo = 0, b_lo = 0;
    int rc = pool_alloc(c, ab * a_elems * 4, &a_lo, st);
    if (rc) return rc;
    rc = pool_alloc(c, bb * b_elems * 4, &b_lo, st);
    if (rc) { pool_free(c, a_lo, st); return rc; }
    rc = !a_mn ? launch_split(c, st, g.a, a_lo, ab, g.M, g.K, g.a_sb, g.a_sm) : launch_split(c, st, g.a, a_lo, ab, g.K, g.M, g.a_sb, g.a_sk);
    if (!rc) rc = !b_mn ? launch_split(c, st, g.b, b_lo, bb, g.N, g.K, g.b_sb, g.b_sn) : launch_split(c, st, g.b, b_lo, bb, g.K, g.N, g.b_sb, g.b_sk);
    if (!rc) {
      GemmProblem h = g;
      h.a_lo = a_lo;
      h.b_lo = b_lo;
      rc = launch_wgmma(c, st, h, a_mn, b_mn);
    }
    // stream-ordered reuse: the pool hands these pages out again only to later work on this context
    pool_free(c, a_lo, st);
    pool_free(c, b_lo, st);
    return rc;
  }
  return launch_wgmma(c, st, g, a_mn, b_mn);
}

static int run_gemm_staged(b200_ctx* c, CUstream st, const GemmProblem& g) {
  const size_t esz = dtype_size(g.in_dtype);
  GemmProblem h = g;
  CUdeviceptr sa = 0, sb = 0;
  bool mn = false;
  int rc = B200_OK;
  if (!operand_tma_ok(g.a, esz, g.M, g.K, g.a_sm, g.a_sk, g.a_sb, &mn) || (mn && esz != 2)) {
    rc = stage_operand(c, st, esz, g.a, g.batch, g.M, g.K, g.a_sm, g.a_sk, g.a_sb, &sa, &h.a_sm, &h.a_sk, &h.a_sb);
    if (!rc) h.a = sa;
  }
  if (!rc && (!operand_tma_ok(g.b, esz, g.N, g.K, g.b_sn, g.b_sk, g.b_sb, &mn) || (mn && esz != 2))) {
    rc = stage_operand(c, st, esz, g.b, g.batch, g.N, g.K, g.b_sn, g.b_sk, g.b_sb, &sb, &h.b_sn, &h.b_sk, &h.b_sb);
    if (!rc) h.b = sb;
  }
  if (!rc) {
    bool a_mn = false, b_mn = false;
    rc = tma_ok(h, &a_mn, &b_mn) ? run_gemm(c, st, h) : launch_simt(c, st, g);
  }
  if (sa) pool_free(c, sa, st);
  if (sb) pool_free(c, sb, st);
  return rc;
}

// Collapse batch dims [0, nb) of one operand into a linear stride; false if the offsets are not linear in the flat index.
static bool linear_batch(int nb, const uint64_t* out_shape, const uint64_t* shape, const uint64_t* strides, uint64_t* flat) {
  uint64_t inner_stride = 0, inner_extent = 1;
  bool have = false;
  for (int i = nb - 1; i >= 0; --i) {
    if (out_shape[i] == 1) continue;
    const uint64_t st = (shape[i] == 1) ? 0 : strides[i];
    if (!have) { inner_stride = st; inner_extent = out_shape[i]; have = true; *flat = st; continue; }
    if (st != inner_stride * inner_extent) return false;
    inner_extent *= out_shape[i];
  }
  if (!have) *flat = 0;
  return true;
}

static int matmul_rec(b200_ctx* c, CUstream st, GemmProblem g, int nb, const uint64_t* ob, const uint64_t* ls,
                      const uint64_t* lst, const uint64_t* rs, const uint64_t* rst, const uint64_t* ost) {
  uint64_t fa = 0, fb = 0, fo = 0;
  if (linear_batch(nb, ob, ls, lst, &fa) && linear_batch(nb, ob, rs, rst, &fb) && linear_batch(nb, ob, ob, ost, &fo)) {
    uint64_t batch = 1;
    for (int i = 0; i < nb; ++i) batch *= ob[i];
    g.batch = batch; g.a_sb = fa; g.b_sb = fb; g.o_sb = fo;
    if (batch == 1) { g.a_sb = g.b_sb = 0; g.o_sb = 0; }
    return run_gemm(c, st, g);
  }
  // peel the outermost non-unit batch dim and recurse
  int d = 0;
  while (d < nb && ob[d] == 1) ++d;
  const size_t esz = dtype_size(g.in_dtype), osz = dtype_size(g.out_dtype);
  for (uint64_t i = 0; i < ob[d]; ++i) {
    GemmProblem h = g;
    h.a += (ls[d] == 1 ? 0 : i * lst[d]) * esz;
    h.b += (rs[d] == 1 ? 0 : i * rst[d]) * esz;
    h.out += i * ost[d] * osz;
    int rc = matmul_rec(c, st, h, nb - d - 1, ob + d + 1, ls + d + 1, lst + d + 1, rs + d + 1, rst + d + 1, ost + d + 1);
    if (rc) return rc;
  }
  return B200_OK;
}

static int matmul_impl(b200_ctx* c, b200_stream s, b200_dtype in_dtype, b200_dtype out_dtype, b200_dptr lhs,
                       b200_dptr rhs, b200_dptr out, int rank, const uint64_t* shape_lhs, const uint64_t* strides_lhs,
                       const uint64_t* shape_rhs, const uint64_t* strides_rhs, const uint64_t* shape_out,
                       const uint64_t* strides_out, const b200_epilogue* ep, int rhs_dtype = -1);

extern "C" int b200_matmul(b200_ctx* c, b200_stream s, b200_dtype in_dtype, b200_dtype out_dtype, b200_dptr lhs,
                           b200_dptr rhs, b200_dptr out, int rank, const uint64_t* shape_lhs, const uint64_t* strides_lhs,
                           const uint64_t* shape_rhs, const uint64_t* strides_rhs, const uint64_t* shape_out,
                           const uint64_t* strides_out) {
  return matmul_impl(c, s, in_dtype, out_dtype, lhs, rhs, out, rank, shape_lhs, strides_lhs, shape_rhs, strides_rhs, shape_out,
                     strides_out, nullptr);
}

extern "C" int b200_matmul_fused(b200_ctx* c, b200_stream s, b200_dtype in_dtype, b200_dtype out_dtype, b200_dptr lhs,
                                 b200_dptr rhs, b200_dptr out, int rank, const uint64_t* shape_lhs, const uint64_t* strides_lhs,
                                 const uint64_t* shape_rhs, const uint64_t* strides_rhs, const uint64_t* shape_out,
                                 const uint64_t* strides_out, const b200_epilogue* ep) {
  if (!ep) return fail(B200_ERR_INVALID_ARG, "matmul_fused: null epilogue");
  if (ep->activation < 0 || ep->activation > 2) return fail(B200_ERR_INVALID_ARG, "matmul_fused: unknown activation %d", ep->activation);
  if (in_dtype == B200_U8 || in_dtype == B200_I8) return fail(B200_ERR_UNSUPPORTED, "matmul_fused: integer accumulators have no float epilogue");
  return matmul_impl(c, s, in_dtype, out_dtype, lhs, rhs, out, rank, shape_lhs, strides_lhs, shape_rhs, strides_rhs, shape_out,
                     strides_out, ep);
}

// ------------------------------------------------------------------------------------------------ block-scaled matmul
extern "C" int b200_matmul_scaled(b200_ctx* c, b200_stream s, b200_dtype lhs_dtype, b200_dtype rhs_dtype, b200_dtype out_dtype,
                                  b200_dptr lhs, b200_dptr rhs, b200_dptr lhs_scales, b200_dptr rhs_scales, b200_dptr out,
                                  uint64_t batch, uint64_t M, uint64_t N, uint64_t K, int scale_block, int scales_packed) {
  CTX_ENTER(c);
  const bool fp4 = (lhs_dtype == B200_F4E2M1X2);
  auto is_fp8 = [](int d) { return d == B200_F8E4M3 || d == B200_F8E5M2; };
  if (!(fp4 ? rhs_dtype == B200_F4E2M1X2 : (is_fp8(lhs_dtype) && is_fp8(rhs_dtype))))
    return fail(B200_ERR_UNSUPPORTED, "matmul_scaled: operands must be fp8 (e4m3/e5m2, mixable) or both packed e2m1");
  if (out_dtype != B200_F32 && out_dtype != B200_BF16 && out_dtype != B200_F16)
    return fail(B200_ERR_UNSUPPORTED, "matmul_scaled: output must be f32, bf16 or f16");
  // scale_block 32: ue8m0 scales (MXFP8 / MXFP4); scale_block 16: ue4m3 scales, packed e2m1 operands only (NVFP4)
  const bool nvf4 = (scale_block == 16);
  if (scale_block != 32 && !(nvf4 && fp4))
    return fail(B200_ERR_UNSUPPORTED, "matmul_scaled: scale block %d (32 = ue8m0 scales; 16 = ue4m3 scales, packed e2m1 operands only)", scale_block);
  if (K == 0 || K % 32) return fail(B200_ERR_INVALID_ARG, "matmul_scaled: K = %llu must be a positive multiple of 32", (unsigned long long)K);
  if (batch == 0 || M == 0 || N == 0) return B200_OK;
  if (!lhs || !rhs || !lhs_scales || !rhs_scales || !out) return fail(B200_ERR_INVALID_ARG, "matmul_scaled: null device pointer");
  if (M >= (1ull << 31) || N >= (1ull << 31) || K >= (1ull << 31) || batch >= (1ull << 20)) return fail(B200_ERR_UNSUPPORTED, "matmul_scaled: extent too large");
  CUstream st = resolve_stream(c, s);
  const uint64_t n_scales = K / scale_block, atoms = (n_scales + 3) / 4;
  const uint64_t k_bytes = fp4 ? K / 2 : K;
  const std::string forced = opt(c, "gemm.variant", "auto");
  const bool tma = (lhs % 16 == 0 && rhs % 16 == 0 && k_bytes % 16 == 0 && (!scales_packed || (lhs_scales % 16 == 0 && rhs_scales % 16 == 0)));
  if (forced == "simt" || !tma) {
    if (scales_packed) return fail(B200_ERR_UNSUPPORTED, "matmul_scaled: packed scales need 16-byte aligned operands and K rows");
    if (forced != "simt" && forced != "auto")
      return fail(B200_ERR_UNSUPPORTED, "gemm.variant=%s forced but operands are not TMA-describable", forced.c_str());
    CUfunction f;
    int rc = get_func(c, "gemm_scaled_simt", &f);
    if (rc) return rc;
    ScaledSimtParams p{lhs, rhs, lhs_scales, rhs_scales, out, (uint32_t)batch, (uint32_t)M, (uint32_t)N, (uint32_t)K,
                       (uint32_t)lhs_dtype, (uint32_t)rhs_dtype, (uint32_t)out_dtype, (uint32_t)scale_block, 1u, 1u, nvf4 ? 1u : 0u, 0u};
    const uint64_t total = batch * M * N;
    const unsigned grid = (unsigned)std::min<uint64_t>((total + 255) / 256, (uint64_t)c->props.num_sms * 16);
    void* args[] = {&p};
    return launch(c, f, std::max(1u, grid), 1, 1, 256, 0, 1, st, args);
  }
  // Hopper's tensor cores take no scale factors: each operand is expanded once to bf16 x * scale (exact, see
  // dequant_scaled_bf16) and the bf16 wgmma GEMM accumulates the products in f32
  const uint64_t ab = batch * M, bb = batch * N;
  CUdeviceptr da = 0, db = 0;
  int rc = pool_alloc(c, ab * K * 2, &da, st);
  if (rc) return rc;
  rc = pool_alloc(c, bb * K * 2, &db, st);
  if (rc) { pool_free(c, da, st); return rc; }
  auto dequant = [&](uint64_t in, uint64_t scales, CUdeviceptr out_bf16, uint64_t rows, int dtype) {
    CUfunction f;
    int r = get_func(c, "dequant_scaled_bf16", &f);
    if (r) return r;
    DequantParams p{in, scales, out_bf16, (uint32_t)rows, (uint32_t)batch, (uint32_t)K, fp4 ? (uint32_t)B200_F4E2M1X2 : (uint32_t)dtype,
                    (uint32_t)scale_block, nvf4 ? 1u : 0u, scales_packed ? 1u : 0u, (uint32_t)atoms};
    const uint64_t groups = batch * rows * (K / 8);
    const unsigned grid = (unsigned)std::min<uint64_t>((groups + 255) / 256, (uint64_t)c->props.num_sms * 16);
    void* args[] = {&p};
    return launch(c, f, std::max(1u, grid), 1, 1, 256, 0, 1, st, args);
  };
  rc = dequant(lhs, lhs_scales, da, M, lhs_dtype);
  if (!rc) rc = dequant(rhs, rhs_scales, db, N, rhs_dtype);
  if (!rc) {
    GemmProblem g{};
    g.in_dtype = B200_BF16;
    g.out_dtype = out_dtype;
    g.a = da; g.b = db; g.out = out;
    g.M = M; g.N = N; g.K = K; g.batch = batch;
    g.a_sm = K; g.a_sk = 1; g.a_sb = batch > 1 ? M * K : 0;
    g.b_sn = K; g.b_sk = 1; g.b_sb = batch > 1 ? N * K : 0;
    g.o_sm = N; g.o_sn = 1; g.o_sb = batch > 1 ? M * N : 0;
    g.mx = true;
    rc = launch_wgmma(c, st, g, false, false);
  }
  pool_free(c, da, st);
  pool_free(c, db, st);
  return rc;
}

// Mixed 8-bit operand formats (the cartesian products the reference instantiates for its manual MMA,
// crates/cubecl-cpp/src/cuda/mma/manual.rs:151-166 i8 x u8 / u8 x i8 and :170-186 fp8 pairs): same kernels, the two format
// operand types of the wgmma instruction differ.
extern "C" int b200_matmul_mixed(b200_ctx* c, b200_stream s, b200_dtype lhs_dtype, b200_dtype rhs_dtype, b200_dtype out_dtype, b200_dptr lhs,
                                 b200_dptr rhs, b200_dptr out, int rank, const uint64_t* shape_lhs, const uint64_t* strides_lhs,
                                 const uint64_t* shape_rhs, const uint64_t* strides_rhs, const uint64_t* shape_out,
                                 const uint64_t* strides_out) {
  auto fp8 = [](int d) { return d == B200_F8E4M3 || d == B200_F8E5M2; };
  auto int8 = [](int d) { return d == B200_U8 || d == B200_I8; };
  if (lhs_dtype != rhs_dtype && !((fp8(lhs_dtype) && fp8(rhs_dtype)) || (int8(lhs_dtype) && int8(rhs_dtype))))
    return fail(B200_ERR_UNSUPPORTED, "matmul_mixed: operand formats %d x %d cannot be mixed (fp8 e4m3/e5m2 pairs, u8/i8 pairs)", (int)lhs_dtype, (int)rhs_dtype);
  return matmul_impl(c, s, lhs_dtype, out_dtype, lhs, rhs, out, rank, shape_lhs, strides_lhs, shape_rhs, strides_rhs, shape_out,
                     strides_out, nullptr, lhs_dtype == rhs_dtype ? -1 : (int)rhs_dtype);
}

static int matmul_impl(b200_ctx* c, b200_stream s, b200_dtype in_dtype, b200_dtype out_dtype, b200_dptr lhs,
                       b200_dptr rhs, b200_dptr out, int rank, const uint64_t* shape_lhs, const uint64_t* strides_lhs,
                       const uint64_t* shape_rhs, const uint64_t* strides_rhs, const uint64_t* shape_out,
                       const uint64_t* strides_out, const b200_epilogue* ep, int rhs_dtype) {
  CTX_ENTER(c);
  if (rank < 2 || rank > 8) return fail(B200_ERR_INVALID_ARG, "matmul: rank %d unsupported (need 2..8)", rank);
  if (!shape_lhs || !strides_lhs || !shape_rhs || !strides_rhs || !shape_out || !strides_out)
    return fail(B200_ERR_INVALID_ARG, "matmul: null shape/stride array");
  const bool fp8 = (in_dtype == B200_F8E4M3 || in_dtype == B200_F8E5M2);
  const bool int8 = (in_dtype == B200_U8 || in_dtype == B200_I8);
  if (in_dtype != B200_F32 && in_dtype != B200_F16 && in_dtype != B200_BF16 && !fp8 && !int8)
    return fail(B200_ERR_UNSUPPORTED, "matmul: input dtype %d unsupported (f32, f16, bf16, f8e4m3, f8e5m2, u8, i8)", (int)in_dtype);
  if (int8 ? (out_dtype != B200_I32)
      : fp8 ? (out_dtype != B200_F32 && out_dtype != B200_BF16 && out_dtype != B200_F16)
            : (out_dtype != in_dtype && out_dtype != B200_F32))
    return fail(B200_ERR_UNSUPPORTED, "matmul: output dtype must equal the input dtype or be f32 (fp8 inputs: bf16/f16/f32; u8/i8 inputs: i32)");
  const int nb = rank - 2;
  const uint64_t M = shape_lhs[rank - 2], K = shape_lhs[rank - 1], K2 = shape_rhs[rank - 2], N = shape_rhs[rank - 1];
  // shape.rs:489-517: inner dims must agree, batch dims broadcast 1 vs d
  if (K != K2) return fail(B200_ERR_INVALID_ARG, "matmul: inner dimensions differ (lhs k=%llu, rhs k=%llu)", (unsigned long long)K, (unsigned long long)K2);
  if (shape_out[rank - 2] != M || shape_out[rank - 1] != N)
    return fail(B200_ERR_INVALID_ARG, "matmul: output is [%llu,%llu], expected [%llu,%llu]", (unsigned long long)shape_out[rank - 2],
                (unsigned long long)shape_out[rank - 1], (unsigned long long)M, (unsigned long long)N);
  for (int i = 0; i < nb; ++i) {
    const uint64_t l = shape_lhs[i], r = shape_rhs[i], o = shape_out[i];
    const uint64_t expect = l == r ? l : (l == 1 ? r : (r == 1 ? l : 0));
    if (expect == 0 && !(l == 0 && r == 0)) return fail(B200_ERR_INVALID_ARG, "matmul: batch dim %d cannot broadcast (%llu vs %llu)", i, (unsigned long long)l, (unsigned long long)r);
    if (o != expect) return fail(B200_ERR_INVALID_ARG, "matmul: output batch dim %d is %llu, expected %llu", i, (unsigned long long)o, (unsigned long long)expect);
  }
  if (!lhs || !rhs || !out) {
    uint64_t n = M * N;
    for (int i = 0; i < nb; ++i) n *= shape_out[i];
    if (n == 0) return B200_OK;
    return fail(B200_ERR_INVALID_ARG, "matmul: null device pointer");
  }
  CUstream st = resolve_stream(c, s);
  GemmProblem g{};
  g.in_dtype = in_dtype; g.out_dtype = out_dtype; g.rhs_dtype = rhs_dtype;
  g.a = lhs; g.b = rhs; g.out = out;
  g.M = M; g.N = N; g.K = K; g.batch = 1;
  g.a_sm = strides_lhs[rank - 2]; g.a_sk = strides_lhs[rank - 1];
  g.b_sk = strides_rhs[rank - 2]; g.b_sn = strides_rhs[rank - 1];
  g.o_sm = strides_out[rank - 2]; g.o_sn = strides_out[rank - 1];
  if (ep) { g.alpha = ep->alpha; g.bias = ep->bias; g.act = (uint32_t)ep->activation; }
  for (int i = 0; i < nb; ++i)
    if (shape_out[i] == 0) return B200_OK;
  return matmul_rec(c, st, g, nb, shape_out, shape_lhs, strides_lhs, shape_rhs, strides_rhs, strides_out);
}

// ================================================================================================ reduce
static int reduce_workspace(b200_ctx* c, CUstream st, CUdeviceptr* out) {
  if (c->dry) { *out = 0x6000000000ull; return B200_OK; }
  auto it = c->reduce_ws.find(st);
  if (it != c->reduce_ws.end()) { *out = it->second; return B200_OK; }
  CUdeviceptr p;
  CUresult r = g_drv.cuMemAlloc_p(&p, kWsBytes);
  if (r != CUDA_SUCCESS) return fail(map_cu(r), "reduce workspace allocation failed: %s", cu_err(r));
  r = g_drv.cuMemsetD32Async_p(p, 0, kWsBytes / 4, st);  // ticket starts at 0; kernels reset it themselves
  if (r != CUDA_SUCCESS) { g_drv.cuMemFree_p(p); return fail(map_cu(r), "reduce workspace memset failed: %s", cu_err(r)); }
  c->reduce_ws[st] = p;
  *out = p;
  return B200_OK;
}

static const char* op_tag(int op) {
  switch (op) {
    case B200_REDUCE_SUM: case B200_REDUCE_MEAN: return "sum";
    case B200_REDUCE_PROD: return "prod";
    case B200_REDUCE_MAX: return "max";
    case B200_REDUCE_MIN: return "min";
    case B200_REDUCE_ARGMAX: return "argmax";
    case B200_REDUCE_ARGMIN: return "argmin";
    default: return nullptr;
  }
}
static const char* dt_tag(int dt) { return dt == B200_F32 ? "f32" : dt == B200_F16 ? "f16" : dt == B200_BF16 ? "bf16" : nullptr; }
static bool fill_dtype_ok(int dt) { return dt_tag(dt) || dt == B200_F8E4M3 || dt == B200_F8E5M2; }

extern "C" int b200_into_contiguous(b200_ctx* c, b200_stream s, b200_dtype dtype, b200_dptr in, b200_dptr out, int rank,
                                    const uint64_t* shape, const uint64_t* strides);

// A reducible VIEW of the input: logical [outer, len, inner] with explicit element strides and an optional row pitch.
struct RView {
  uint64_t in = 0;
  uint64_t outer = 1, len = 1, inner = 1;
  uint64_t s_outer = 0, s_len = 1;
  uint64_t row_len = 1, row_pitch = 1;
};

static unsigned opt_uint(b200_ctx* c, const char* key, unsigned dflt, unsigned lo, unsigned hi) {
  const std::string v = opt(c, key, "");
  if (v.empty()) return dflt;
  const long x = atol(v.c_str());
  return (unsigned)std::min<long>(hi, std::max<long>(lo, x));
}
static uint64_t pow2_ceil(uint64_t x) { uint64_t p = 1; while (p < x) p <<= 1; return p; }
static uint64_t pow2_floor(uint64_t x) { uint64_t p = 1; while (p * 2 <= x) p <<= 1; return p; }
static uint64_t ceil_div(uint64_t a, uint64_t b) { return (a + b - 1) / b; }

// Reduce every element of the view `v` (v.len elements in logical rows of v.row_len, v.row_pitch apart) to out[0].
static int launch_reduce_all(b200_ctx* c, CUstream st, int op, int dt, const RView& v, uint64_t out, float scale) {
  const bool arg = (op == B200_REDUCE_ARGMAX || op == B200_REDUCE_ARGMIN);
  const bool pitched = v.row_len != v.len;
  const uint64_t n = v.len;
  const size_t esz = dtype_size(dt);
  std::string name = std::string(pitched ? "reduce_allp_" : "reduce_all_") + op_tag(op) + "_" + dt_tag(dt);
  unsigned threads = opt_uint(c, "reduce.threads", 512, 32, 512) / 32 * 32;
  unsigned bps = opt_uint(c, "reduce.blocks_per_sm", 4, 1, 64);
  unsigned smem = 0, stages = 0;
  bool bulk = false;
  if (!pitched && !arg) {
    // variants: the plain 128-bit streaming kernel, its tuning forms (f32 sum only) and the bulk-copy staged kernel
    // auto = the bulk-copy staged kernel once the input is big enough to fill a ring on every SM; plain loads below that
    const std::string var = opt(c, "reduce.variant", "auto");
    if (var == "tma" || var == "auto") {
      bulk = n * esz >= (var == "tma" ? 64ull * kBulkStageBytes : (uint64_t)c->props.num_sms * 8 * kBulkStageBytes);
    } else if (var != "u8") {
      if (std::string(op_tag(op)) == "sum" && dt == B200_F32) name += "_" + var;
    }
  }
  const uint64_t vec = 16 / esz;
  unsigned grid;
  if (bulk) {
    name += "_tma";
    threads = kBulkConsumers + 32;            // consumer warps + one producer warp
    stages = opt_uint(c, "reduce.tma_stages", 6, 2, 8);   // 6 x 16 KB ring stages (1 GiB f32)
    smem = stages * kBulkStageBytes + 128;
    const uint64_t tiles = n * esz / kBulkStageBytes;
    const unsigned per_sm = stages <= 6 ? opt_uint(c, "reduce.tma_ctas_per_sm", 1, 1, 2) : 1;
    grid = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>(tiles, (uint64_t)c->props.num_sms * per_sm));
  } else {
    const uint64_t want = (n / vec + threads - 1) / threads;  // blocks that still get >= 1 vector per thread
    grid = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>(want, std::min<uint64_t>((uint64_t)c->props.num_sms * bps, kWsMaxBlocks)));
  }
  CUfunction f;
  int rc = get_func(c, name, &f);
  if (rc) return rc;
  if (smem && !c->dry) CU_CHECK(g_drv.cuFuncSetAttribute_p(f, CU_FUNC_ATTRIBUTE_MAX_DYNAMIC_SHARED_SIZE_BYTES, (int)smem));
  CUdeviceptr ws;
  rc = reduce_workspace(c, st, &ws);
  if (rc) return rc;
  ReduceParams p{};
  p.in = v.in; p.out = out; p.ws = ws;
  p.outer = 1; p.len = n; p.inner = 1;
  p.row_len = v.row_len; p.row_pitch = v.row_pitch;
  p.seg_len = n; p.nseg = 1; p.scale = scale;
  p.ctu = stages;                             // bulk-copy kernels: ring depth
  void* args[] = {&p};
  // Overlap with the preceding all-element reduction on the context's stream: safe because that kernel writes only its
  // 4-byte result and the workspace, this one reads neither before its own griddepcontrol.wait -- unless its input is the
  // predecessor's output.
  const uint64_t in_end = v.in + (pitched ? (n / v.row_len) * v.row_pitch : n) * esz;
  const bool pdl = st == c->stream && c->pdl_prev_out != 0 && opt(c, "reduce.pdl", "on") == "on" &&
                   !(c->pdl_prev_out + 4 > v.in && c->pdl_prev_out < in_end);
  rc = launch(c, f, grid, 1, 1, threads, smem, 1, st, args, pdl);
  if (!rc && st == c->stream) c->pdl_prev_out = out;
  return rc;
}

// One launch of the rows kernel: items = outer x nseg, item (o, s) covers elements [s * seg_len, ..) of row o.
static int launch_rows_kernel(b200_ctx* c, CUstream st, int op, int dt, const RView& v, uint64_t seg_len, uint64_t out, uint64_t out2, float scale,
                              bool pdl = false) {
  const std::string name = std::string("reduce_rows_") + op_tag(op) + "_" + dt_tag(dt);
  CUfunction f;
  int rc = get_func(c, name, &f);
  if (rc) return rc;
  const size_t esz = dtype_size(dt);
  const uint64_t vec = 16 / esz;
  const uint64_t nseg = ceil_div(v.len, seg_len), items = v.outer * nseg;
  // Threads per item (power of two): about `vpt` 128-bit vectors per thread, so a 32 KB row is one 256-thread block and the
  // grid has many more blocks than resident slots (the hardware scheduler balances the tail block by block; a warp per
  // 32 KB row would leave a last, nearly empty wave).
  // 16 vectors per thread for inputs that stream from HBM for a while, 8 for small launch-bound inputs
  const bool big = v.outer * v.len * esz >= (128ull << 20);
  const unsigned vpt = opt_uint(c, "reduce.rows_vpt", big ? 16 : 8, 1, 64);
  const uint64_t nv = ceil_div(std::min(seg_len, v.len), vec);
  uint64_t tpr = std::min<uint64_t>(512, pow2_ceil(ceil_div(nv, vpt)));
  int tpr_log2 = 0;
  while ((1ull << tpr_log2) < tpr) ++tpr_log2;
  const unsigned threads = tpr > 256 ? (unsigned)tpr : 256;
  const uint64_t items_per_block = threads >> tpr_log2;
  uint64_t blocks = ceil_div(items, items_per_block);
  const bool uniform = (v.in % 16) == 0 && ((v.s_outer * esz) % 16) == 0 && (v.len % vec) == 0;
  if (tpr <= 32 && uniform && nseg == 1 && v.len / vec <= tpr) blocks = ceil_div(blocks, 4);  // short rows: four rows in flight per thread group
  const unsigned grid = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>(blocks, 0x7FFFFFFFull));
  ReduceParams p{};
  p.in = v.in; p.out = out; p.out2 = out2;
  p.outer = v.outer; p.len = v.len; p.inner = 1;
  p.s_outer = v.s_outer; p.s_len = 1;
  p.row_len = 1; p.row_pitch = 1;
  p.seg_len = seg_len; p.nseg = (uint32_t)nseg; p.scale = scale;
  void* args[] = {&p, &tpr_log2};
  return launch(c, f, grid, 1, 1, threads, 0, 1, st, args, pdl);
}

// One launch of the column kernel over the view (items = outer x nseg x column tiles).
// `final_out` != 0 with a segmented axis: finish in the same launch when the (outer, column tile) tickets fit the workspace
// (*fused = true), else the caller runs the second pass.
static int launch_cols_kernel(b200_ctx* c, CUstream st, int op, int dt, const RView& v, uint64_t seg_len, uint64_t out, uint64_t out2, float scale,
                              uint64_t final_out = 0, bool* fused = nullptr, bool pdl = false) {
  const bool arg_op = (op == B200_REDUCE_ARGMAX || op == B200_REDUCE_ARGMIN);
  const std::string name = std::string("reduce_cols_") + op_tag(op) + "_" + dt_tag(dt) + (opt(c, "reduce.cols_loads", arg_op ? "4" : "8") == "8" ? "_n8" : "");
  CUfunction f;
  int rc = get_func(c, name, &f);
  if (rc) return rc;
  const size_t esz = dtype_size(dt);
  const uint64_t vec = 16 / esz;
  const bool vector = v.inner % vec == 0 && v.row_len % vec == 0 && v.in % 16 == 0 && (v.s_len * esz) % 16 == 0 &&
                      (v.s_outer * esz) % 16 == 0 && (v.row_pitch * esz) % 16 == 0;
  const uint64_t units = vector ? v.inner / vec : v.inner;
  const uint64_t nseg = ceil_div(v.len, seg_len);
  const uint64_t seg = std::min(seg_len, v.len);
  // tile shape: RL row lanes x ctu column units per kColsThreads-thread block.  A warp's worth of units (512 contiguous bytes per row
  // in vector mode) keeps the loads coalesced; the rest of the block goes to row lanes as long as every lane still has ~4 rows
  const uint64_t ctu_min = std::min<uint64_t>(units, 32);
  const uint64_t rl_max = kColsThreads / ctu_min;
  const uint64_t rl = std::min<uint64_t>(rl_max, std::max<uint64_t>(1, pow2_floor(std::max<uint64_t>(1, seg / 4))));
  const uint64_t ctu = std::min<uint64_t>(units, kColsThreads / rl);
  const uint64_t tiles = ceil_div(units, ctu);
  const uint64_t items = v.outer * nseg * tiles;
  const unsigned bps = 8;
  // short axis: a block's item is small, so blocks walk several items (persistent grid); long axis: one item per block
  const uint64_t cap = seg * ctu * (vector ? 16 : esz) >= (64u << 10) ? 0x7FFFFFFFull : (uint64_t)c->props.num_sms * bps;
  const unsigned grid = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>(items, cap));
  ReduceParams p{};
  p.in = v.in; p.out = out; p.out2 = out2;
  p.outer = v.outer; p.len = v.len; p.inner = v.inner;
  p.s_outer = v.s_outer; p.s_len = v.s_len;
  p.row_len = v.row_len; p.row_pitch = v.row_pitch;
  p.seg_len = seg_len; p.nseg = (uint32_t)nseg; p.ctu = (uint32_t)ctu; p.scale = scale;
  p.flags = vector ? 2u : 0u;
  if (fused) *fused = false;
  if (final_out && nseg > 1 && v.outer * tiles <= kWsColTickets && opt(c, "reduce.cols_fused", "off") == "on") {
    CUdeviceptr ws;
    rc = reduce_workspace(c, st, &ws);
    if (rc) return rc;
    p.ws = ws; p.final_out = final_out; p.flags |= 4u;
    if (fused) *fused = true;
  }
  if (nseg > 1 && !(p.flags & 4u)) p.scale = 1.0f;   // first pass of a two-launch reduction: the scale (mean) belongs to the second
  void* args[] = {&p};
  return launch(c, f, grid, 1, 1, kColsThreads, 0, 1, st, args, pdl);
}

static int launch_argcombine(b200_ctx* c, CUstream st, uint64_t keys, uint64_t idx, uint64_t out, uint64_t outer, uint64_t nseg, uint64_t inner) {
  CUfunction f;
  int rc = get_func(c, "reduce_argcombine", &f);
  if (rc) return rc;
  ArgCombineParams p{keys, idx, out, outer, nseg, inner};
  const uint64_t threads = nseg >= 8 ? outer * inner * 32 : outer * inner;   // a warp per output when there are many segments
  const unsigned grid = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>(ceil_div(threads, 256), (uint64_t)c->props.num_sms * 8));
  void* args[] = {&p};
  return launch(c, f, grid, 1, 1, 256, 0, 1, st, args);
}

// Reduce the `len` axis of the view.  Few outputs with a long axis are reduced in two passes (segments of the axis first,
// then the per-segment partials), both deterministic; everything else is one launch.
static int reduce_axis_view(b200_ctx* c, CUstream st, int op, int dt, const RView& v, uint64_t out, float scale) {
  const bool arg = (op == B200_REDUCE_ARGMAX || op == B200_REDUCE_ARGMIN);
  const uint64_t sms = c->props.num_sms;
  const size_t esz = dtype_size(dt);
  const uint64_t vec = 16 / esz;
  // Segment the axis when whole rows / columns cannot fill the machine: aim at ~16 blocks per SM (several waves of small
  // blocks, so the block scheduler evens out the tail) while every segment keeps a useful amount of work.
  uint64_t seg_len = v.len;
  if (v.inner == 1) {
    const unsigned bps = opt_uint(c, "reduce.rows_blocks_per_sm", 4, 1, 64);
    if (v.outer < sms * bps && v.len >= 16384 && v.outer * v.len * esz >= (32ull << 20)) {   // below ~32 MB one launch wins (launch-bound)
      const uint64_t nseg = std::min<uint64_t>(ceil_div(sms * 16, v.outer), v.len / 4096);
      if (nseg > 1) seg_len = ceil_div(ceil_div(v.len, nseg), 512) * 512;   // 512 elements: segments stay vector-aligned
    }
  } else {
    const uint64_t units = (v.inner % vec == 0) ? v.inner / vec : v.inner;
    const uint64_t tiles = ceil_div(units, std::min<uint64_t>(units, 32));
    const unsigned bps = opt_uint(c, "reduce.cols_blocks_per_sm", 4, 1, 64);
    if (v.outer * tiles < sms * bps && v.len >= 256) {
      // ~8 blocks per SM (two resident waves of big blocks) for value ops (eight loads in flight per thread) and arg ops (four)
      // alike.  Target 0: exactly one resident wave (4 blocks per SM).
      const unsigned tgt = opt_uint(c, "reduce.cols_split_target", 8, 0, 256);
      uint64_t nseg;
      if (tgt == 0) nseg = std::max<uint64_t>(1, (sms * 4) / (v.outer * tiles));
      else nseg = ceil_div(sms * tgt, v.outer * tiles);
      nseg = std::min<uint64_t>(nseg, v.len / 64);
      if (nseg > 1) seg_len = ceil_div(v.len, nseg);
    }
  }
  const uint64_t nseg = ceil_div(v.len, seg_len);
  if (arg && nseg > 1 && !c->dry && v.len >= (1ull << 32)) return fail(B200_ERR_UNSUPPORTED, "arg-reduce: axis extent does not fit u32 indices");
  if (nseg == 1) {
    return v.inner == 1 ? launch_rows_kernel(c, st, op, dt, v, v.len, out, 0, scale) : launch_cols_kernel(c, st, op, dt, v, v.len, out, 0, scale);
  }
  // two passes: partials [outer, nseg, inner] (f32 values, or u32 keys + u32 indices), then the partials
  const uint64_t count = v.outer * nseg * v.inner;
  CUdeviceptr tmp = 0, tmp2 = 0;
  int rc = pool_alloc(c, count * 4, &tmp, st);
  if (rc) return rc;
  if (arg) {
    rc = pool_alloc(c, count * 4, &tmp2, st);
    if (rc) { pool_free(c, tmp, st); return rc; }
  }
  bool fused = false;
  rc = v.inner == 1 ? launch_rows_kernel(c, st, op, dt, v, seg_len, tmp, tmp2, 1.0f)
                    : launch_cols_kernel(c, st, op, dt, v, seg_len, tmp, tmp2, scale, out, &fused);
  if (!rc && !fused) {
    if (arg) {
      rc = launch_argcombine(c, st, tmp, tmp2, out, v.outer, nseg, v.inner);
    } else {
      RView t;
      t.in = tmp; t.outer = v.outer; t.len = nseg; t.inner = v.inner;
      t.s_outer = nseg * v.inner; t.s_len = v.inner; t.row_len = v.inner; t.row_pitch = v.inner;
      // the second pass only depends on the first: launched with programmatic serialization, its blocks are resident (and
      // past their prologue) when the first pass drains; they wait in griddepcontrol.wait
      const bool pdl = opt(c, "reduce.pdl", "on") == "on";
      rc = v.inner == 1 ? launch_rows_kernel(c, st, op, B200_F32, t, nseg, out, 0, scale, pdl)
                        : launch_cols_kernel(c, st, op, B200_F32, t, nseg, out, 0, scale, 0, nullptr, pdl);
    }
  }
  pool_free(c, tmp, st);
  if (tmp2) pool_free(c, tmp2, st);
  return rc;
}

// Can the strided tensor be reduced IN PLACE?  Yes when, in memory order, it is a dense tensor whose innermost rows may be
// pitched (what PitchedMemoryLayoutPolicy produces, crates/cubecl-runtime/src/allocator.rs:21-72) -- in any axis
// permutation that keeps the kept axes in their logical order (a transposed view reduces the other physical axis).
// Anything else (broadcast strides, gaps elsewhere, permuted outputs) goes through into_contiguous.
static bool plan_view(int rank, const uint64_t* shape, const uint64_t* strides, int axis, bool arg, uint64_t in, RView* v) {
  struct Dim { uint64_t ext, st; int pos; bool ax; };
  std::vector<Dim> d;
  bool unit_axis = false;
  uint64_t expect = 1;
  std::vector<uint64_t> cst(rank);
  for (int i = rank - 1; i >= 0; --i) { cst[i] = expect; expect *= shape[i]; }
  for (int i = 0; i < rank; ++i) {
    if (shape[i] == 1) { if (i == axis) unit_axis = true; continue; }
    d.push_back(Dim{shape[i], strides ? strides[i] : cst[i], i, i == axis});
  }
  std::stable_sort(d.begin(), d.end(), [](const Dim& a, const Dim& b) { return a.st > b.st; });
  const int k = (int)d.size();
  bool pitched = false;
  if (k > 0) {
    if (d[k - 1].st != 1) return false;
    for (int j = k - 2; j >= 0; --j) {
      const uint64_t e = d[j + 1].st * d[j + 1].ext;
      if (d[j].st == e) continue;
      if (j == k - 2 && d[j].st > e) { pitched = true; continue; }
      return false;
    }
  }
  // kept axes must appear in memory order exactly as in logical order (otherwise the output would need a permuted store)
  int last = -1;
  for (int j = 0; j < k; ++j) {
    if (d[j].ax && !(axis < 0)) continue;
    if (axis < 0 && !arg) continue;     // a value reduction over everything is order-independent
    if (d[j].pos < last) return false;
    last = d[j].pos;
  }
  v->in = in;
  uint64_t total = 1;
  for (int j = 0; j < k; ++j) total *= d[j].ext;
  const uint64_t row = k > 0 ? d[k - 1].ext : 1, pitch = pitched ? d[k - 2].st : row;
  if (axis < 0) {
    v->outer = 1; v->len = total; v->inner = 1;
    v->row_len = pitched ? row : total; v->row_pitch = pitched ? pitch : total;
    return true;
  }
  if (unit_axis) {  // reducing an axis of extent 1: a (converting) copy of everything else
    v->outer = 1; v->len = 1; v->s_len = 0; v->inner = total;
    v->row_len = pitched ? row : total; v->row_pitch = pitched ? pitch : total;
    return true;
  }
  int pa = -1;
  for (int j = 0; j < k; ++j) if (d[j].ax) pa = j;
  if (pa < 0) return false;
  v->outer = 1; v->inner = 1;
  for (int j = 0; j < pa; ++j) v->outer *= d[j].ext;
  for (int j = pa + 1; j < k; ++j) v->inner *= d[j].ext;
  v->len = d[pa].ext;
  v->s_len = d[pa].st;
  v->s_outer = pa > 0 ? d[pa - 1].st : 0;
  if (pitched && pa <= k - 3) { v->row_len = row; v->row_pitch = pitch; }
  else { v->row_len = v->inner; v->row_pitch = v->inner; }
  return true;
}

static int reduce_impl(b200_ctx* c, b200_stream s, b200_reduce_op op, b200_dtype in_dtype, b200_dptr in, b200_dptr out,
                       int rank, const uint64_t* shape, const uint64_t* strides, int axis) {
  if (!op_tag(op)) return fail(B200_ERR_INVALID_ARG, "reduce: unknown op %d", (int)op);
  if (!dt_tag(in_dtype)) return fail(B200_ERR_UNSUPPORTED, "reduce: input dtype %d unsupported (f32, f16, bf16)", (int)in_dtype);
  if (rank < 1 || rank > 8 || !shape) return fail(B200_ERR_INVALID_ARG, "reduce: bad rank/shape");
  if (axis < -1 || axis >= rank) return fail(B200_ERR_INVALID_ARG, "reduce: axis %d out of range for rank %d", axis, rank);
  uint64_t n = 1, len = 1;
  for (int i = 0; i < rank; ++i) n *= shape[i];
  len = axis < 0 ? n : shape[axis];
  uint64_t outputs = 1;
  for (int i = 0; i < rank; ++i) if (axis >= 0 && i != axis) outputs *= shape[i];
  if (outputs == 0) return B200_OK;  // empty output
  if (len == 0) return fail(B200_ERR_INVALID_ARG, "reduce: reduced extent is 0 (identity-filled outputs are not defined by the reference)");
  if (!in || !out) return fail(B200_ERR_INVALID_ARG, "reduce: null device pointer");
  const bool arg = (op == B200_REDUCE_ARGMAX || op == B200_REDUCE_ARGMIN);
  if (arg && len >= (1ull << 32)) return fail(B200_ERR_UNSUPPORTED, "arg-reduce: axis extent %llu does not fit u32 indices", (unsigned long long)len);
  if (in % dtype_size(in_dtype)) return fail(B200_ERR_INVALID_ARG, "reduce: input pointer is not aligned to its element size");
  const float scale = (op == B200_REDUCE_MEAN) ? static_cast<float>(1.0 / static_cast<double>(len)) : 1.0f;
  CUstream st = resolve_stream(c, s);
  RView v;
  if (plan_view(rank, shape, strides, axis, arg, in, &v)) {
    if (axis < 0) return launch_reduce_all(c, st, op, in_dtype, v, out, scale);
    return reduce_axis_view(c, st, op, in_dtype, v, out, scale);
  }
  // not reducible in place: gather into a compact temporary first (into_contiguous), then reduce that
  CUdeviceptr tmp;
  int rc = pool_alloc(c, n * dtype_size(in_dtype), &tmp, st);
  if (rc) return rc;
  rc = b200_into_contiguous(c, s, in_dtype, in, tmp, rank, shape, strides);
  if (!rc) {
    RView w;
    const bool ok = plan_view(rank, shape, nullptr, axis, arg, tmp, &w);
    rc = !ok ? fail(B200_ERR_UNKNOWN, "reduce: contiguous plan failed")
             : axis < 0 ? launch_reduce_all(c, st, op, in_dtype, w, out, scale) : reduce_axis_view(c, st, op, in_dtype, w, out, scale);
  }
  pool_free(c, tmp, st);
  return rc;
}

extern "C" int b200_reduce(b200_ctx* c, b200_stream s, b200_reduce_op op, b200_dtype in_dtype, b200_dptr in, b200_dptr out,
                           int rank, const uint64_t* shape, int axis) {
  CTX_ENTER(c);
  return reduce_impl(c, s, op, in_dtype, in, out, rank, shape, nullptr, axis);
}

extern "C" int b200_reduce_strided(b200_ctx* c, b200_stream s, b200_reduce_op op, b200_dtype in_dtype, b200_dptr in, b200_dptr out,
                                   int rank, const uint64_t* shape, const uint64_t* strides, int axis) {
  CTX_ENTER(c);
  return reduce_impl(c, s, op, in_dtype, in, out, rank, shape, strides, axis);
}

// ================================================================================================ scan
static std::string scan_name(const char* family, int op, int dt, int odt) {
  std::string n = std::string(family) + op_tag(op) + "_" + dt_tag(dt);
  if (odt != B200_F32) n += std::string("_") + dt_tag(odt);
  return n;
}

// Column units of the view: 128-bit vectors of consecutive inner elements when the layout allows it, else elements.
static bool scan_cols_vector(const RView& v, size_t esz) {
  const uint64_t vec = 16 / esz;
  return v.inner % vec == 0 && v.row_len % vec == 0 && v.in % 16 == 0 && (v.s_len * esz) % 16 == 0 && (v.s_outer * esz) % 16 == 0 &&
         (v.row_pitch * esz) % 16 == 0;
}
static uint64_t scan_cols_ctu(uint64_t units) { return std::min<uint64_t>(kScanColUnits, std::max<uint64_t>(32, pow2_ceil(units))); }

// One launch of scan_rows over items (row, segment): TPR threads per item sized so every thread walks about four tiles.
static int launch_scan_rows(b200_ctx* c, CUstream st, int op, int dt, int odt, const RView& v, uint64_t seg_len, uint64_t out,
                            uint64_t carry, bool exclusive, bool pdl) {
  CUfunction f;
  int rc = get_func(c, scan_name("scan_rows_", op, dt, odt), &f);
  if (rc) return rc;
  const uint64_t nseg = ceil_div(v.len, seg_len), items = v.outer * nseg;
  const uint64_t chunks = ceil_div(std::min(seg_len, v.len), kScanElems);
  const uint64_t tpr = std::min<uint64_t>(512, pow2_ceil(ceil_div(chunks, 4)));
  int tpr_log2 = 0;
  while ((1ull << tpr_log2) < tpr) ++tpr_log2;
  const unsigned threads = tpr > 32 ? (unsigned)tpr : 256;   // a multi-warp item owns its block
  const unsigned grid = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>(ceil_div(items, threads / tpr), 0x7FFFFFFFull));
  ScanParams p{};
  p.in = v.in; p.out = out; p.carry = carry;
  p.outer = v.outer; p.len = v.len; p.inner = 1;
  p.s_outer = v.s_outer; p.s_len = 1;
  p.row_len = 1; p.row_pitch = 1;
  p.seg_len = seg_len; p.nseg = (uint32_t)nseg;
  p.flags = exclusive ? 1u : 0u;
  void* args[] = {&p, &tpr_log2};
  return launch(c, f, grid, 1, 1, threads, 0, 1, st, args, pdl);
}

// One launch of scan_cols over items (outer, segment, tile of column units).
static int launch_scan_cols(b200_ctx* c, CUstream st, int op, int dt, int odt, const RView& v, uint64_t seg_len, uint64_t out,
                            uint64_t carry, bool exclusive, bool pdl) {
  CUfunction f;
  int rc = get_func(c, scan_name("scan_cols_", op, dt, odt), &f);
  if (rc) return rc;
  const size_t esz = dtype_size(dt);
  const bool vector = scan_cols_vector(v, esz);
  const uint64_t units = vector ? v.inner / (16 / esz) : v.inner;
  const uint64_t ctu = scan_cols_ctu(units);
  const uint64_t nseg = ceil_div(v.len, seg_len);
  const uint64_t items = v.outer * nseg * ceil_div(units, ctu);
  const unsigned grid = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>(items, 0x7FFFFFFFull));
  ScanParams p{};
  p.in = v.in; p.out = out; p.carry = carry;
  p.outer = v.outer; p.len = v.len; p.inner = v.inner;
  p.s_outer = v.s_outer; p.s_len = v.s_len;
  p.row_len = v.row_len; p.row_pitch = v.row_pitch;
  p.seg_len = seg_len; p.nseg = (uint32_t)nseg;
  p.flags = (exclusive ? 1u : 0u) | (vector ? 2u : 0u);
  void* args[] = {&p};
  return launch(c, f, grid, 1, 1, (unsigned)ctu, 0, 1, st, args, pdl);
}

static int launch_scan(b200_ctx* c, CUstream st, int op, int dt, int odt, const RView& v, uint64_t seg_len, uint64_t out, uint64_t carry,
                       bool exclusive, bool pdl) {
  return v.inner == 1 ? launch_scan_rows(c, st, op, dt, odt, v, seg_len, out, carry, exclusive, pdl)
                      : launch_scan_cols(c, st, op, dt, odt, v, seg_len, out, carry, exclusive, pdl);
}

// Scan the `len` axis of the view into the compact output.  Whole items (rows, or tiles of columns) are scanned in one
// launch; when they cannot fill the machine, the axis is cut into segments and scanned in three stream-ordered launches:
// the reduce first pass (one partial per segment), an exclusive scan of the partials (the carries), and the scan of every
// segment from its carry.  That path reads the input twice.  The segmentation follows reduce_axis_view's policy.
static int scan_axis_view(b200_ctx* c, CUstream st, int op, int dt, int odt, const RView& v, uint64_t out, bool exclusive) {
  const uint64_t sms = c->props.num_sms;
  const size_t esz = dtype_size(dt);
  uint64_t seg_len = v.len;
  if (v.inner == 1) {
    // fewer than 4 rows per SM, a long axis and >= 32 MB: ~16 segments per SM, each >= 4096 elements, 512-element aligned
    if (v.outer < sms * 4 && v.len >= 16384 && v.outer * v.len * esz >= (32ull << 20)) {
      const uint64_t nseg = std::min<uint64_t>(ceil_div(sms * 16, v.outer), v.len / 4096);
      if (nseg > 1) seg_len = ceil_div(ceil_div(v.len, nseg), 512) * 512;
    }
  } else {
    // fewer than 4 column blocks per SM on an axis of >= 256 rows: ~8 blocks per SM, every segment >= 64 rows
    const uint64_t units = scan_cols_vector(v, esz) ? v.inner / (16 / esz) : v.inner;
    const uint64_t blocks = v.outer * ceil_div(units, scan_cols_ctu(units));
    if (blocks < sms * 4 && v.len >= 256) {
      const uint64_t nseg = std::min<uint64_t>(ceil_div(sms * 8, blocks), v.len / 64);
      if (nseg > 1) seg_len = ceil_div(v.len, nseg);
    }
  }
  const uint64_t nseg = ceil_div(v.len, seg_len);
  if (nseg == 1) return launch_scan(c, st, op, dt, odt, v, v.len, out, 0, exclusive, false);
  const uint64_t count = v.outer * nseg * v.inner;
  CUdeviceptr partials = 0, carries = 0;
  int rc = pool_alloc(c, count * 4, &partials, st);
  if (rc) return rc;
  rc = pool_alloc(c, count * 4, &carries, st);
  if (rc) { pool_free(c, partials, st); return rc; }
  rc = v.inner == 1 ? launch_rows_kernel(c, st, op, dt, v, seg_len, partials, 0, 1.0f)
                    : launch_cols_kernel(c, st, op, dt, v, seg_len, partials, 0, 1.0f);
  if (!rc) {
    RView t;
    t.in = partials; t.outer = v.outer; t.len = nseg; t.inner = v.inner;
    t.s_outer = nseg * v.inner; t.s_len = v.inner; t.row_len = v.inner; t.row_pitch = v.inner;
    rc = launch_scan(c, st, op, B200_F32, B200_F32, t, nseg, carries, 0, true, true);
  }
  if (!rc) rc = launch_scan(c, st, op, dt, odt, v, seg_len, out, carries, exclusive, true);
  pool_free(c, partials, st);
  pool_free(c, carries, st);
  return rc;
}

static int scan_impl(b200_ctx* c, b200_stream s, b200_reduce_op op, int exclusive, b200_dtype in_dtype, b200_dtype out_dtype,
                     b200_dptr in, b200_dptr out, int rank, const uint64_t* shape, const uint64_t* strides, int axis) {
  if (op == B200_REDUCE_ARGMAX || op == B200_REDUCE_ARGMIN || op == B200_REDUCE_MEAN)
    return fail(B200_ERR_UNSUPPORTED, "scan: op %d has no scan (sum, prod, max, min)", (int)op);
  if (!op_tag(op)) return fail(B200_ERR_INVALID_ARG, "scan: unknown op %d", (int)op);
  if (!dt_tag(in_dtype)) return fail(B200_ERR_UNSUPPORTED, "scan: input dtype %d unsupported (f32, f16, bf16)", (int)in_dtype);
  if (out_dtype != B200_F32 && out_dtype != in_dtype)
    return fail(B200_ERR_INVALID_ARG, "scan: output dtype %d must be f32 or the input dtype", (int)out_dtype);
  if (rank < 1 || rank > 8 || !shape) return fail(B200_ERR_INVALID_ARG, "scan: bad rank/shape");
  if (axis < 0 || axis >= rank) return fail(B200_ERR_INVALID_ARG, "scan: axis %d out of range for rank %d", axis, rank);
  uint64_t n = 1;
  for (int i = 0; i < rank; ++i) n *= shape[i];
  if (n == 0) return B200_OK;
  if (!in || !out) return fail(B200_ERR_INVALID_ARG, "scan: null device pointer");
  if (in % dtype_size(in_dtype) || out % dtype_size(out_dtype))
    return fail(B200_ERR_INVALID_ARG, "scan: a pointer is not aligned to its element size");
  CUstream st = resolve_stream(c, s);
  // The output is logical row-major, so the input is read in place only when its dimensions lie in memory in their logical
  // order (contiguous, or pitched rows): then the view keeps the scanned axis at its logical position.
  bool in_order = true;
  if (strides) {
    int prev = -1;
    for (int i = 0; i < rank; ++i) {
      if (shape[i] == 1) continue;
      if (prev >= 0 && strides[prev] <= strides[i]) in_order = false;
      prev = i;
    }
  }
  RView v;
  if (in_order && plan_view(rank, shape, strides, axis, false, in, &v)) return scan_axis_view(c, st, op, in_dtype, out_dtype, v, out, exclusive != 0);
  // any other view: gather into a compact temporary first (into_contiguous), then scan that
  CUdeviceptr tmp;
  int rc = pool_alloc(c, n * dtype_size(in_dtype), &tmp, st);
  if (rc) return rc;
  rc = b200_into_contiguous(c, s, in_dtype, in, tmp, rank, shape, strides);
  if (!rc) {
    RView w;
    rc = !plan_view(rank, shape, nullptr, axis, false, tmp, &w) ? fail(B200_ERR_UNKNOWN, "scan: contiguous plan failed")
                                                                : scan_axis_view(c, st, op, in_dtype, out_dtype, w, out, exclusive != 0);
  }
  pool_free(c, tmp, st);
  return rc;
}

extern "C" int b200_scan(b200_ctx* c, b200_stream s, b200_reduce_op op, int exclusive, b200_dtype in_dtype, b200_dtype out_dtype,
                         b200_dptr in, b200_dptr out, int rank, const uint64_t* shape, const uint64_t* strides, int axis) {
  CTX_ENTER(c);
  return scan_impl(c, s, op, exclusive, in_dtype, out_dtype, in, out, rank, shape, strides, axis);
}

// ================================================================================================ quantize / dequantize
// Kernels in csrc/quant.cu.
static uint32_t log2_u32(uint32_t v) {
  uint32_t l = 0;
  while (v > 1) { v >>= 1; ++l; }
  return l;
}

static constexpr unsigned kQuantThreads = 256;

// Bits of a b200_quant_value (QuantValue::size_bits, scheme.rs:381-387); 0 for a value outside the enum.
static uint32_t quant_bits(int32_t v) {
  switch (v) {
    case B200_QV_Q8F: case B200_QV_E5M2: case B200_QV_E4M3: case B200_QV_Q8S: return 8;
    case B200_QV_Q4F: case B200_QV_E2M1: case B200_QV_Q4S: return 4;
    case B200_QV_Q2F: case B200_QV_Q2S: return 2;
    default: return 0;
  }
}
static size_t scale_dtype_size(int32_t dt) {
  switch (dt) {
    case B200_F32: return 4;
    case B200_F16: case B200_BF16: return 2;
    case B200_UE8M0: case B200_F8E4M3: return 1;
    default: return 0;
  }
}

// A device-side memset that a dry-run planning context records as one line.
static int memset32_async(b200_ctx* c, CUstream st, CUdeviceptr dst, uint32_t value, size_t words) {
  if (c->dry) {
    char line[64];
    snprintf(line, sizeof(line), "memset32 %zu\n", words);
    c->plan += line;
    return B200_OK;
  }
  CU_CHECK(g_drv.cuMemsetD32Async_p(dst, value, words, st));
  return B200_OK;
}

// The checks both directions share: the scheme's fields, the shape, and which pointers its levels need.  block_scale is
// read only when the scheme has a block level (block > 0); with block == 0 it is ignored, whatever it holds.  `what` names the
// call in messages.  On success *n is the element count and *K the innermost extent.
static int quant_check(const char* what, const b200_quant_scheme* q, int rank, const uint64_t* shape, b200_dptr block_scales,
                       b200_dptr tensor_scale, uint64_t* n, uint64_t* K) {
  if (!q) return fail(B200_ERR_INVALID_ARG, "%s: null scheme", what);
  const uint32_t bits = quant_bits(q->value);
  if (!bits) return fail(B200_ERR_INVALID_ARG, "%s: unknown quant value %d", what, (int)q->value);
  if (q->tensor_scale != 0 && q->tensor_scale != 1) return fail(B200_ERR_INVALID_ARG, "%s: tensor_scale must be 0 or 1", what);
  if (q->block < 0) return fail(B200_ERR_INVALID_ARG, "%s: negative block %d", what, (int)q->block);
  if (q->block == 0 && !q->tensor_scale)
    return fail(B200_ERR_INVALID_ARG, "%s: a scheme without a block level needs the tensor level (per-tensor f32)", what);
  if (q->block > 0 && !scale_dtype_size(q->block_scale))
    return fail(B200_ERR_INVALID_ARG, "%s: block-scale dtype %d is not F32, F16, BF16, UE8M0 or F8E4M3", what, (int)q->block_scale);
  if (q->block != 0 && q->block != 8 && q->block != 16 && q->block != 32 && q->block != 64 && q->block != 128)
    return fail(B200_ERR_UNSUPPORTED, "%s: block %d (0, 8, 16, 32, 64, 128)", what, (int)q->block);
  if (rank < 1 || rank > 8 || !shape) return fail(B200_ERR_INVALID_ARG, "%s: bad rank/shape", what);
  *n = 1;
  for (int i = 0; i < rank; ++i) *n *= shape[i];
  *K = shape[rank - 1];
  if (q->block > 0 && *K % (uint64_t)q->block)
    return fail(B200_ERR_INVALID_ARG, "%s: innermost extent %llu is not a multiple of the block %d", what, (unsigned long long)*K,
                (int)q->block);
  if (*K * bits % 8) return fail(B200_ERR_INVALID_ARG, "%s: a row of %llu %u-bit values is not a whole number of bytes", what,
                                 (unsigned long long)*K, bits);
  if (*n == 0) return B200_OK;
  if ((q->block > 0) != (block_scales != 0))
    return fail(B200_ERR_INVALID_ARG, "%s: block_scales must be non-null exactly when the scheme has a block level", what);
  if ((q->tensor_scale != 0) != (tensor_scale != 0))
    return fail(B200_ERR_INVALID_ARG, "%s: tensor_scale must be non-null exactly when the scheme has a tensor level", what);
  if ((q->block > 0 && block_scales % scale_dtype_size(q->block_scale)) || tensor_scale % 4)
    return fail(B200_ERR_INVALID_ARG, "%s: a scale pointer is not aligned to its element size", what);
  return B200_OK;
}

// The input as rows of K elements `pitch` apart, read in place when base and rows are 16-byte aligned.  A per-tensor scheme
// on a contiguous input runs as one row (scales do not care about rows there).
static bool quant_rows_view(int rank, const uint64_t* shape, const uint64_t* strides, uint64_t n, size_t esz, bool per_tensor,
                            uint64_t in, uint64_t* rows, uint64_t* K, uint64_t* pitch) {
  *K = shape[rank - 1];
  *rows = n / *K;
  *pitch = *K;
  if (strides) {
    // innermost unit-stride (or extent 1); every other non-unit dimension nests at its successor's extent; the first
    // non-unit leading dimension sets the row pitch
    uint64_t expect = 0;
    bool first = true;
    if (*K > 1 && strides[rank - 1] != 1) return false;
    for (int i = rank - 2; i >= 0; --i) {
      if (shape[i] == 1) continue;
      if (first) {
        if (strides[i] < *K) return false;
        *pitch = strides[i];
        first = false;
      } else if (strides[i] != expect) {
        return false;
      }
      expect = strides[i] * shape[i];
    }
  }
  if (per_tensor && *pitch == *K) { *rows = 1; *K = n; *pitch = n; }
  return in % 16 == 0 && (*rows == 1 || (*pitch * esz) % 16 == 0);
}

static int quant_impl(b200_ctx* c, b200_stream s, const b200_quant_scheme* q, b200_dtype in_dtype, b200_dptr in, b200_dptr values,
                      b200_dptr block_scales, b200_dptr tensor_scale, int rank, const uint64_t* shape, const uint64_t* strides) {
  uint64_t n = 0, K = 0;
  int rc = quant_check("quantize", q, rank, shape, block_scales, tensor_scale, &n, &K);
  if (rc) return rc;
  if (q->block > 0 && q->tensor_scale && q->block_scale != B200_F16 && q->block_scale != B200_F8E4M3)
    return fail(B200_ERR_UNSUPPORTED, "quantize: two-level schemes take F16 or F8E4M3 (ue4m3) block scales, not dtype %d",
                (int)q->block_scale);
  if (!dt_tag(in_dtype)) return fail(B200_ERR_INVALID_ARG, "quantize: input dtype %d is not F32, F16 or BF16", (int)in_dtype);
  if (n == 0) return B200_OK;
  if (!in || !values) return fail(B200_ERR_INVALID_ARG, "quantize: null device pointer");
  const size_t esz = dtype_size(in_dtype);
  if (in % esz) return fail(B200_ERR_INVALID_ARG, "quantize: input pointer is not aligned to its element size");
  CUstream st = resolve_stream(c, s);
  QuantParams p{};
  p.values = values; p.block_scales = block_scales; p.tensor_scale = tensor_scale;
  p.value = (uint32_t)q->value; p.block = (uint32_t)q->block; p.scale_dt = q->block > 0 ? (uint32_t)q->block_scale : B200_F32;
  p.block_log2 = log2_u32(p.block);
  CUdeviceptr tmp = 0, amax = 0;
  uint64_t rows, pitch;
  if (quant_rows_view(rank, shape, strides, n, esz, q->block == 0, in, &rows, &K, &pitch)) {
    p.in = in;
  } else {
    // any other view (or an unaligned base / row): gather into a compact pooled temporary first
    rc = pool_alloc(c, n * esz, &tmp, st);
    if (rc) return rc;
    std::vector<uint64_t> cs(rank);
    uint64_t acc = 1;
    for (int i = rank - 1; i >= 0; --i) { cs[i] = acc; acc *= shape[i]; }
    rc = b200_into_contiguous(c, s, in_dtype, in, tmp, rank, shape, strides ? strides : cs.data());
    quant_rows_view(rank, shape, nullptr, n, esz, q->block == 0, tmp, &rows, &K, &pitch);
    p.in = tmp;
  }
  p.rows = rows; p.K = K; p.pitch = pitch;
  const uint64_t vec = 16 / esz, chunks = rows * ((K + vec - 1) / vec);
  if (!rc && q->tensor_scale) {
    // the tensor level first: the finite |x| max of the whole tensor, atomicMax'ed as u32 bits into a pooled word
    rc = pool_alloc(c, 4, &amax, st);
    if (!rc) rc = memset32_async(c, st, amax, 0, 1);
    CUfunction f;
    if (!rc) rc = get_func(c, std::string("quant_absmax_") + dt_tag(in_dtype), &f);
    if (!rc) {
      p.amax = amax;
      const uint64_t want = ceil_div(chunks, (uint64_t)kQuantThreads * 4);
      const unsigned grid = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>(want, (uint64_t)c->props.num_sms * 8));
      void* args[] = {&p};
      rc = launch(c, f, grid, 1, 1, kQuantThreads, 0, 1, st, args);
    }
  }
  if (!rc) {
    CUfunction f;
    rc = get_func(c, std::string("quant_encode_") + dt_tag(in_dtype), &f);
    if (!rc) {
      const uint64_t grid = std::max<uint64_t>(1, ceil_div(chunks, (uint64_t)kQuantThreads));
      if (grid > 0x7FFFFFFFull) rc = fail(B200_ERR_TOO_MANY_RESOURCES, "quantize: %llu chunks exceed one launch", (unsigned long long)chunks);
      void* args[] = {&p};
      if (!rc) rc = launch(c, f, (unsigned)grid, 1, 1, kQuantThreads, 0, 1, st, args);
    }
  }
  if (amax) pool_free(c, amax, st);
  if (tmp) pool_free(c, tmp, st);
  return rc;
}

extern "C" int b200_quantize(b200_ctx* c, b200_stream s, const b200_quant_scheme* scheme, b200_dtype in_dtype, b200_dptr in,
                             b200_dptr values, b200_dptr block_scales, b200_dptr tensor_scale, int rank, const uint64_t* shape,
                             const uint64_t* strides) {
  CTX_ENTER(c);
  return quant_impl(c, s, scheme, in_dtype, in, values, block_scales, tensor_scale, rank, shape, strides);
}

extern "C" int b200_dequantize(b200_ctx* c, b200_stream s, const b200_quant_scheme* scheme, b200_dtype out_dtype, b200_dptr values,
                               b200_dptr block_scales, b200_dptr tensor_scale, b200_dptr out, int rank, const uint64_t* shape) {
  CTX_ENTER(c);
  uint64_t n = 0, K = 0;
  int rc = quant_check("dequantize", scheme, rank, shape, block_scales, tensor_scale, &n, &K);
  if (rc) return rc;
  if (!dt_tag(out_dtype)) return fail(B200_ERR_INVALID_ARG, "dequantize: output dtype %d is not F32, F16 or BF16", (int)out_dtype);
  if (n == 0) return B200_OK;
  if (!values || !out) return fail(B200_ERR_INVALID_ARG, "dequantize: null device pointer");
  if (out % dtype_size(out_dtype)) return fail(B200_ERR_INVALID_ARG, "dequantize: output pointer is not aligned to its element size");
  CUfunction f;
  rc = get_func(c, std::string("quant_decode_") + dt_tag(out_dtype), &f);
  if (rc) return rc;
  QuantDecodeParams p{};
  p.values = values; p.block_scales = block_scales; p.tensor_scale = tensor_scale; p.out = out; p.n = n;
  p.value = (uint32_t)scheme->value; p.block = (uint32_t)scheme->block;
  p.scale_dt = scheme->block > 0 ? (uint32_t)scheme->block_scale : B200_F32;
  p.flags = (values % 16 == 0 && out % 16 == 0) ? 1u : 0u;
  p.block_log2 = log2_u32(p.block);
  const uint64_t threads = ceil_div(n * quant_bits(scheme->value) / 8, (uint64_t)16);
  const uint64_t grid = std::max<uint64_t>(1, ceil_div(threads, (uint64_t)kQuantThreads));
  if (grid > 0x7FFFFFFFull) return fail(B200_ERR_TOO_MANY_RESOURCES, "dequantize: %llu elements exceed one launch", (unsigned long long)n);
  void* args[] = {&p};
  return launch(c, f, (unsigned)grid, 1, 1, kQuantThreads, 0, 1, resolve_stream(c, s), args);
}

// ------------------------------------------------------------------------------------------------ quantized matmul
// Kernels: csrc/quant.cu (QUANT_PART 1) and csrc/gemm_wgmma.cu (gemm_q8_*, gemm_q8t_*).
static const char* quant_scale_tag(int32_t dt) {
  switch (dt) {
    case B200_F32: return "f32";
    case B200_F16: return "f16";
    case B200_BF16: return "bf16";
    case B200_UE8M0: return "ue8m0";
    default: return "ue4m3";
  }
}

// The codes of one operand as s8 rows TMA can read: Q8 codes in place (16-byte aligned base, K % 16 == 0) or through the
// staging pass; Q4 / Q2 codes widened exactly to one s8 per element.  *tmp is the pooled buffer, if any.
static int qmm_codes(b200_ctx* c, CUstream st, const b200_quant_operand* o, uint64_t batch, uint64_t rows, uint64_t K,
                     CUdeviceptr* tmp, uint64_t* ptr, uint64_t* pitch) {
  const uint32_t bits = quant_bits(o->scheme.value);
  if (bits == 8) {
    if (o->values % 16 == 0 && K % 16 == 0) { *ptr = o->values; *pitch = K; return B200_OK; }
    uint64_t s_mn, s_k, s_b;
    int rc = stage_operand(c, st, 1, o->values, batch, rows, K, K, 1, rows * K, tmp, &s_mn, &s_k, &s_b);
    *ptr = *tmp; *pitch = s_mn;
    return rc;
  }
  const uint64_t total_rows = batch * rows, pch = (K + 15) / 16 * 16;
  int rc = pool_alloc(c, total_rows * pch, tmp, st);
  if (rc) return rc;
  CUfunction f;
  rc = get_func(c, "quant_widen_s8", &f);
  if (rc) return rc;
  QuantWidenParams p{o->values, *tmp, total_rows, K, pch, bits, 0};
  const uint64_t vecs = total_rows * (pch / 16);
  const unsigned grid = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>(ceil_div(vecs, (uint64_t)kQuantThreads), (uint64_t)c->props.num_sms * 16));
  void* args[] = {&p};
  *ptr = *tmp; *pitch = pch;
  return launch(c, f, grid, 1, 1, kQuantThreads, 0, 1, st, args);
}

// The f32 effective scales of one operand per GEMM block of bk elements, block-major [batch][K / bk][rows padded to 4].
static int qmm_scales(b200_ctx* c, CUstream st, const b200_quant_operand* o, uint64_t batch, uint64_t rows, uint64_t K, uint32_t bk,
                      CUdeviceptr* out) {
  const uint64_t rows_pad = (rows + 3) / 4 * 4, nblk = K / bk, total = batch * nblk * rows_pad;
  int rc = pool_alloc(c, total * 4, out, st);
  if (rc) return rc;
  const int32_t block = o->scheme.block;
  CUfunction f;
  rc = get_func(c, std::string("quant_scales_f32_") + (block ? quant_scale_tag(o->scheme.block_scale) : "tensor"), &f);
  if (rc) return rc;
  QuantScalesParams p{block ? o->block_scales : 0, o->tensor_scale, *out, batch, rows, rows_pad, nblk, block ? (uint32_t)block / bk : 1u, 0};
  const unsigned grid = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>(ceil_div(total, (uint64_t)kQuantThreads), (uint64_t)c->props.num_sms * 16));
  void* args[] = {&p};
  return launch(c, f, grid, 1, 1, kQuantThreads, 0, 1, st, args);
}

extern "C" int b200_matmul_quantized(b200_ctx* c, b200_stream s, const b200_quant_operand* lhs, const b200_quant_operand* rhs,
                                     b200_dtype out_dtype, b200_dptr out, uint64_t batch, uint64_t m, uint64_t n, uint64_t k) {
  CTX_ENTER(c);
  if (!lhs || !rhs) return fail(B200_ERR_INVALID_ARG, "matmul_quantized: null operand");
  const bool empty = (batch == 0 || m == 0 || n == 0);
  const b200_quant_operand* ops[2] = {lhs, rhs};
  const uint64_t rows[2] = {m, n};
  for (int i = 0; i < 2; ++i) {
    const char* what = i == 0 ? "matmul_quantized (lhs)" : "matmul_quantized (rhs)";
    const uint64_t shape[2] = {empty ? 0 : batch * rows[i], k};
    uint64_t nel = 0, K = 0;
    int rc = quant_check(what, &ops[i]->scheme, 2, shape, ops[i]->block_scales, ops[i]->tensor_scale, &nel, &K);
    if (rc) return rc;
    const int32_t v = ops[i]->scheme.value;
    if (v == B200_QV_E4M3 || v == B200_QV_E5M2 || v == B200_QV_E2M1)
      return fail(B200_ERR_UNSUPPORTED, "%s: minifloat values (e4m3 / e5m2 / e2m1) with block scales run through b200_matmul_scaled", what);
    if (ops[i]->scheme.block == 8 || ops[i]->scheme.block == 16)
      return fail(B200_ERR_UNSUPPORTED, "%s: block %d (32, 64 or 128: s8 wgmma consumes K in steps of 32)", what, (int)ops[i]->scheme.block);
  }
  if (out_dtype != B200_F32 && out_dtype != B200_BF16 && out_dtype != B200_F16)
    return fail(B200_ERR_INVALID_ARG, "matmul_quantized: output dtype %d is not F32, BF16 or F16", (int)out_dtype);
  if (empty) return B200_OK;
  if (k == 0) return fail(B200_ERR_INVALID_ARG, "matmul_quantized: K must be positive");
  const bool per_tensor = lhs->scheme.block == 0 && rhs->scheme.block == 0;
  // |q| <= 128 on either side: one product is at most 2^14, so the exact s32 dot product over K needs K * 2^14 < 2^31
  if (per_tensor && k >= (1ull << 17))
    return fail(B200_ERR_UNSUPPORTED, "matmul_quantized: per-tensor x per-tensor needs K < 131072 (exact s32 dot products), K = %llu",
                (unsigned long long)k);
  if (!out || !lhs->values || !rhs->values) return fail(B200_ERR_INVALID_ARG, "matmul_quantized: null device pointer");
  const size_t osz = dtype_size(out_dtype);
  if (out % osz) return fail(B200_ERR_INVALID_ARG, "matmul_quantized: output pointer is not aligned to its element size");
  if (m >= (1ull << 31) || n >= (1ull << 31) || k >= (1ull << 31) || batch >= (1ull << 20))
    return fail(B200_ERR_UNSUPPORTED, "matmul_quantized: extent too large");
  CUstream st = resolve_stream(c, s);
  CUdeviceptr tmp[4] = {0, 0, 0, 0};   // lhs codes, rhs codes, lhs scales, rhs scales
  uint64_t pa = 0, pb = 0, pitch_a = 0, pitch_b = 0;
  int rc = qmm_codes(c, st, lhs, batch, m, k, &tmp[0], &pa, &pitch_a);
  if (!rc) rc = qmm_codes(c, st, rhs, batch, n, k, &tmp[1], &pb, &pitch_b);
  GemmProblem g{};
  g.in_dtype = B200_I8; g.out_dtype = out_dtype;
  g.a = pa; g.b = pb; g.out = out;
  g.M = m; g.N = n; g.K = k; g.batch = batch;
  g.a_sm = pitch_a; g.a_sk = 1; g.a_sb = batch > 1 ? m * pitch_a : 0;
  g.b_sn = pitch_b; g.b_sk = 1; g.b_sb = batch > 1 ? n * pitch_b : 0;
  g.o_sm = n; g.o_sn = 1; g.o_sb = batch > 1 ? m * n : 0;
  if (per_tensor) {
    g.q = 2;
    g.q_ga = lhs->tensor_scale; g.q_gb = rhs->tensor_scale;
  } else {
    // kernel block: the finer of the present block levels; a coarser block repeats its scale, a per-tensor side uses g
    const int32_t ba = lhs->scheme.block, bb = rhs->scheme.block;
    g.q = 1;
    g.q_bk = (uint32_t)(ba == 0 ? bb : bb == 0 ? ba : std::min(ba, bb));
    if (!rc) rc = qmm_scales(c, st, lhs, batch, m, k, g.q_bk, &tmp[2]);
    if (!rc) rc = qmm_scales(c, st, rhs, batch, n, k, g.q_bk, &tmp[3]);
    g.q_sa = tmp[2]; g.q_sb = tmp[3];
  }
  if (!rc) rc = launch_wgmma(c, st, g, false, false);
  for (CUdeviceptr t : tmp)
    if (t) pool_free(c, t, st);   // stream-ordered: reusable by later work once the GEMM has drained
  return rc;
}

// ------------------------------------------------------------------------------------------------ 2-D convolution
// Strides of a rank-4 view with every extent-1 dimension given the stride a compact tensor would have there (the address of
// its only index is unchanged), so layout tests do not trip over strides that are never used.
static void conv_norm_strides(const uint64_t* shape, const uint64_t* strides, uint64_t* out) {
  uint64_t inner = 1;
  for (int d = 3; d >= 0; --d) {
    out[d] = strides ? strides[d] : inner;
    if (shape[d] == 1) out[d] = inner;
    inner = out[d] * shape[d];
  }
}

// A stride of `e` 16-bit elements that a tensor map can take: a 16-byte multiple below 2^40 bytes.
static bool conv_al16(uint64_t e) { return e % 8 == 0 && e * 2 < (1ull << 40); }

// Two adjacent dimensions [outer, inner] of a view as one strided dimension: its stride, or 0 when they do not flatten.
static uint64_t conv_flat_stride(uint64_t outer, uint64_t inner, uint64_t s_outer, uint64_t s_inner) {
  return inner == 1 ? s_outer : (outer == 1 || s_outer == inner * s_inner) ? s_inner : 0;
}

// Checks every convolution entry point shares; what: the entry point, for messages.  The dtypes, the epilogue's activation,
// the args, and the weights' channels w_c against the input channels of one group, in_c.
static int conv_check_args(const char* what, b200_dtype in_dtype, b200_dtype out_dtype, const b200_conv2d_args& a, const b200_epilogue* ep,
                           uint64_t in_c, uint64_t w_c) {
  if (in_dtype != B200_F16 && in_dtype != B200_BF16)
    return fail(B200_ERR_UNSUPPORTED, "%s: input dtype %d unsupported (f16, bf16)", what, (int)in_dtype);
  if (out_dtype != in_dtype && out_dtype != B200_F32)
    return fail(B200_ERR_UNSUPPORTED, "%s: output dtype must equal the input dtype or be f32", what);
  if (ep && (ep->activation < 0 || ep->activation > 2)) return fail(B200_ERR_INVALID_ARG, "%s: unknown activation %d", what, ep->activation);
  if (a.stride_h < 1 || a.stride_w < 1 || a.dilation_h < 1 || a.dilation_w < 1 || a.pad_h < 0 || a.pad_w < 0)
    return fail(B200_ERR_INVALID_ARG, "%s: strides and dilations must be >= 1 and padding >= 0", what);
  if (w_c != in_c)
    return fail(B200_ERR_INVALID_ARG, "%s: weights have %llu channels, the input has %llu", what, (unsigned long long)w_c, (unsigned long long)in_c);
  return B200_OK;
}

// Extents < 2^31, then PyTorch's output rule for the input [N, H, W, C] and weights [Cout, KH, KW, *]: y (the forward's out
// or a gradient's dy, y_name in messages) must be [N, OH, OW, Cout].  An empty kernel has no output extent to check.
static int conv_check_shape(const char* what, const b200_conv2d_args& a, const uint64_t* in, const uint64_t* w, const uint64_t* y,
                            const char* y_name, uint64_t* OH, uint64_t* OW) {
  const uint64_t lim = 1ull << 31;
  for (int d = 0; d < 4; ++d)
    if (in[d] >= lim || w[d] >= lim || y[d] >= lim) return fail(B200_ERR_UNSUPPORTED, "%s: extents must be < 2^31", what);
  const int64_t KH = (int64_t)w[1], KW = (int64_t)w[2];
  if (KH == 0 || KW == 0) return B200_OK;
  const int64_t nh = (int64_t)in[1] + 2 * (int64_t)a.pad_h - (int64_t)a.dilation_h * (KH - 1) - 1;
  const int64_t nw = (int64_t)in[2] + 2 * (int64_t)a.pad_w - (int64_t)a.dilation_w * (KW - 1) - 1;
  if (nh < 0 || nw < 0)
    return fail(B200_ERR_INVALID_ARG, "%s: the dilated kernel is larger than the padded input (output extent < 1)", what);
  *OH = (uint64_t)(nh / a.stride_h) + 1;
  *OW = (uint64_t)(nw / a.stride_w) + 1;
  if (y[0] != in[0] || y[1] != *OH || y[2] != *OW || y[3] != w[0])
    return fail(B200_ERR_INVALID_ARG, "%s: %s is [%llu,%llu,%llu,%llu], expected [%llu,%llu,%llu,%llu]", what, y_name, (unsigned long long)y[0],
                (unsigned long long)y[1], (unsigned long long)y[2], (unsigned long long)y[3], (unsigned long long)in[0],
                (unsigned long long)*OH, (unsigned long long)*OW, (unsigned long long)w[0]);
  return B200_OK;
}

// The 4-D im2col limits of the tensor map (cuda.h: cuTensorMapEncodeIm2col): pixel-box corners in [-128, 127] ...
static int conv_check_corners(const char* what, const int64_t corners[4]) {
  for (int i = 0; i < 4; ++i)
    if (corners[i] < -128 || corners[i] > 127)
      return fail(B200_ERR_UNSUPPORTED, "%s: im2col pixel-box corner %lld outside [-128, 127]", what, (long long)corners[i]);
  return B200_OK;
}

// ... with the forward's corners -pad and pad - dilation * (kernel - 1) ...
static int conv_check_fwd_corners(const char* what, const b200_conv2d_args& a, uint64_t KH, uint64_t KW) {
  const int64_t corners[4] = {-(int64_t)a.pad_h, -(int64_t)a.pad_w, (int64_t)a.pad_h - (int64_t)a.dilation_h * ((int64_t)KH - 1),
                              (int64_t)a.pad_w - (int64_t)a.dilation_w * ((int64_t)KW - 1)};
  return conv_check_corners(what, corners);
}

// ... and an element stride (the conv stride) <= 8, which also bounds the data gradient's phases per dimension.
static int conv_check_stride(const char* what, const b200_conv2d_args& a) {
  if (a.stride_h > kDgradMaxStride || a.stride_w > kDgradMaxStride)
    return fail(B200_ERR_UNSUPPORTED, "%s: the conv stride must be <= %d", what, kDgradMaxStride);
  return B200_OK;
}

// Device pointers present, and the output's (out_name in messages) aligned to its element size.
static int conv_check_ptrs(const char* what, uint64_t a, uint64_t b, uint64_t out, const char* out_name, b200_dtype out_dtype) {
  if (!a || !b || !out) return fail(B200_ERR_INVALID_ARG, "%s: null device pointer", what);
  if (out % dtype_size(out_dtype)) return fail(B200_ERR_INVALID_ARG, "%s: %s pointer is not aligned to its element size", what, out_name);
  return B200_OK;
}

// An NHWC output (out or dx; normalised strides ns): unit channel stride, and one pixel pitch >= its channels for N, H, W.
static int conv_check_pixels(const char* what, const char* name, const uint64_t* shape, const uint64_t* ns) {
  if (ns[3] != 1 || ns[2] < shape[3] || ns[1] != shape[2] * ns[2] || ns[0] != shape[1] * ns[1])
    return fail(B200_ERR_UNSUPPORTED, "%s: %s must have unit channel stride and one pixel pitch >= its channels for N, H, W", what, name);
  return B200_OK;
}

// dw [Cout, KH, KW, C'] (normalised strides ds): unit channel stride, (KH, KW) flattening into one kernel-position stride
// (*dw_sp), and an output-channel stride.
static int conv_check_dw(const char* what, const uint64_t* shape, const uint64_t* ds, size_t osz, uint64_t* dw_sp) {
  *dw_sp = conv_flat_stride(shape[1], shape[2], ds[1], ds[2]);
  if (ds[3] != 1 || *dw_sp == 0 || ds[0] * osz >= (1ull << 40) || *dw_sp * osz >= (1ull << 40))
    return fail(B200_ERR_UNSUPPORTED, "%s: dw must have unit channel stride and (KH, KW) flattening into one stride", what);
  return B200_OK;
}

// Pooled copy of an operand seen as [batch, rows, C] (strides in elements) with C padded to `cp` zero channels (repitch_rows
// writes the padding columns as zeros).
static int conv_pad_channels(b200_ctx* c, CUstream st, uint64_t in, uint64_t batch, uint64_t rows, uint64_t C, uint64_t s_b,
                             uint64_t s_r, uint64_t s_c, uint64_t cp, CUdeviceptr* out) {
  CUdeviceptr buf;
  int rc = pool_alloc(c, batch * rows * cp * 2, &buf, st);
  if (rc) return rc;
  CUfunction f;
  rc = get_func(c, "repitch_rows", &f);
  if (rc) { pool_free(c, buf, st); return rc; }
  RepitchParams p{in, buf, batch, rows, C, s_b, s_r, s_c, cp, 2u, 0u};
  const uint64_t vecs = batch * rows * (cp / 8);
  const unsigned grid = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>((vecs + 255) / 256, 0x7FFFFFFFull));
  void* args[] = {&p};
  rc = launch(c, f, grid, 1, 1, 256, 0, 1, st, args);
  if (rc) { pool_free(c, buf, st); return rc; }
  *out = buf;
  return B200_OK;
}

// A compact pooled copy of a rank-4 view (b200_into_contiguous).
static int conv_gather(b200_ctx* c, CUstream st, b200_dtype dt, uint64_t in, const uint64_t* shape, const uint64_t* strides,
                       CUdeviceptr* out) {
  CUdeviceptr buf;
  int rc = pool_alloc(c, shape[0] * shape[1] * shape[2] * shape[3] * 2, &buf, st);
  if (rc) return rc;
  rc = b200_into_contiguous(c, static_cast<b200_stream>(st), dt, in, buf, 4, shape, strides);
  if (rc) { pool_free(c, buf, st); return rc; }
  *out = buf;
  return B200_OK;
}

// An operand [N, H, W, C] (normalised strides `ns`) as the convolution maps read it: unit channel stride, 16-byte aligned base
// and strides, channels a multiple of 8.  A view that does not qualify is gathered into a compact pooled copy; channel counts
// that are not multiples of 8 are copied with the channels padded to 8 zeros.  flat: the leading dimensions the map reads
// as one strided dimension -- none (x, and dy in the data gradient), (H, W) (the forward's weights: one kernel-position
// dimension, returned as s_w) or (N, H, W) (dy in the weight gradient: [pixels, Cout]).  tmp[0] / tmp[1] receive the pooled
// copies (the caller frees them).
struct NhwcOperand {
  uint64_t ptr, C, s_w, s_h, s_n;
};
enum ConvFlat { kFlatNone, kFlatHW, kFlatNHW };
static int conv_prep_nhwc(b200_ctx* c, CUstream st, b200_dtype dt, uint64_t ptr, const uint64_t* shape, const uint64_t* ns, ConvFlat flat,
                          CUdeviceptr tmp[2], NhwcOperand* o) {
  const uint64_t N = shape[0], H = shape[1], W = shape[2], C = shape[3];
  const uint64_t spx = conv_flat_stride(H, W, ns[1], ns[2]);   // (H, W) as one pixel dimension
  int rc = B200_OK;
  if (C % 8 == 0) {
    bool in_place = ptr % 16 == 0 && ns[3] == 1 && conv_al16(ns[0]);
    if (flat == kFlatHW) in_place = in_place && spx != 0 && conv_al16(spx);
    else in_place = in_place && conv_al16(ns[1]) && conv_al16(ns[2]) && (flat == kFlatNone || (ns[1] == W * ns[2] && ns[0] == H * ns[1]));
    if (in_place) {
      *o = {ptr, C, flat == kFlatHW ? spx : ns[2], ns[1], ns[0]};
      return B200_OK;
    }
    rc = conv_gather(c, st, dt, ptr, shape, ns, &tmp[0]);
    *o = {tmp[0], C, C, W * C, H * W * C};
    return rc;
  }
  const uint64_t cp = (C + 7) / 8 * 8;
  uint64_t in = ptr, sb = ns[0], sp = spx, sc = ns[3];
  if (spx == 0) {
    rc = conv_gather(c, st, dt, ptr, shape, ns, &tmp[0]);
    in = tmp[0]; sb = H * W * C; sp = C; sc = 1;
  }
  if (!rc) rc = conv_pad_channels(c, st, in, N, H * W, C, sb, sp, sc, cp, &tmp[1]);
  *o = {tmp[1], cp, cp, W * cp, H * W * cp};
  return rc;
}

// The implicit GEMM of a convolution map: M pixel rows of A and N rows of B, each K elements with unit k stride (the weight
// gradient, which reads both MN-major, sets its own operand strides); out rows o_sm apart with unit column stride.
static GemmProblem conv_problem(b200_dtype in_dtype, b200_dtype out_dtype, uint64_t a, uint64_t b, uint64_t out, uint64_t M, uint64_t N,
                                uint64_t K, uint64_t o_sm, ConvGeom* g) {
  GemmProblem gp{};
  gp.in_dtype = in_dtype; gp.out_dtype = out_dtype;
  gp.a = a; gp.b = b; gp.out = out;
  gp.M = M; gp.N = N; gp.K = K; gp.batch = 1;
  gp.a_sm = K; gp.a_sk = 1; gp.b_sn = K; gp.b_sk = 1;
  gp.o_sm = o_sm; gp.o_sn = 1; gp.o_sb = 0;
  gp.conv = g;
  return gp;
}

extern "C" int b200_conv2d(b200_ctx* c, b200_stream s, b200_dtype in_dtype, b200_dtype out_dtype, b200_dptr x, const uint64_t* x_shape,
                           const uint64_t* x_strides, b200_dptr w, const uint64_t* w_shape, const uint64_t* w_strides, b200_dptr out,
                           const uint64_t* out_shape, const uint64_t* out_strides, const b200_conv2d_args* args, const b200_epilogue* ep) {
  CTX_ENTER(c);
  const char* what = "conv2d";
  if (!x_shape || !w_shape || !out_shape || !args) return fail(B200_ERR_INVALID_ARG, "%s: null shape or args", what);
  const b200_conv2d_args& a = *args;
  const uint64_t N = x_shape[0], H = x_shape[1], W = x_shape[2], C = x_shape[3];
  const uint64_t Cout = w_shape[0], KH = w_shape[1], KW = w_shape[2];
  int rc = conv_check_args(what, in_dtype, out_dtype, a, ep, C, w_shape[3]);
  if (rc) return rc;
  if (N == 0 || H == 0 || W == 0 || C == 0 || Cout == 0 || KH == 0 || KW == 0) return B200_OK;
  uint64_t OH = 0, OW = 0;
  if ((rc = conv_check_shape(what, a, x_shape, w_shape, out_shape, "out", &OH, &OW))) return rc;
  if ((rc = conv_check_fwd_corners(what, a, KH, KW)) || (rc = conv_check_stride(what, a))) return rc;
  const uint64_t M = N * OH * OW, lim = 1ull << 31;
  if (M >= lim) return fail(B200_ERR_UNSUPPORTED, "%s: N * OH * OW = %llu must be < 2^31", what, (unsigned long long)M);
  if ((rc = conv_check_ptrs(what, x, w, out, "output", out_dtype))) return rc;
  uint64_t os[4], xs[4], ws[4];
  conv_norm_strides(out_shape, out_strides, os);
  if ((rc = conv_check_pixels(what, "out", out_shape, os))) return rc;
  if (KH * KW * ((C + 63) / 64 * 64) >= lim) return fail(B200_ERR_UNSUPPORTED, "%s: KH * KW * C (C padded to 64) must be < 2^31", what);
  CUstream st = resolve_stream(c, s);
  conv_norm_strides(x_shape, x_strides, xs);
  conv_norm_strides(w_shape, w_strides, ws);
  CUdeviceptr tmp[4] = {0, 0, 0, 0};
  NhwcOperand xo{}, wo{};
  rc = conv_prep_nhwc(c, st, in_dtype, x, x_shape, xs, kFlatNone, &tmp[0], &xo);
  if (!rc) rc = conv_prep_nhwc(c, st, in_dtype, w, w_shape, ws, kFlatHW, &tmp[2], &wo);
  if (!rc) {
    ConvGeom g{};
    g.N = N; g.H = H; g.W = W; g.C = xo.C; g.KH = KH; g.KW = KW; g.OH = OH; g.OW = OW; g.Cout = Cout;
    g.sh = a.stride_h; g.sw = a.stride_w; g.ph = a.pad_h; g.pw = a.pad_w; g.dh = a.dilation_h; g.dw = a.dilation_w;
    g.x_sw = xo.s_w; g.x_sh = xo.s_h; g.x_sn = xo.s_n;
    g.w_sp = wo.s_w; g.w_sco = wo.s_n;
    GemmProblem gp = conv_problem(in_dtype, out_dtype, xo.ptr, wo.ptr, out, M, Cout, KH * KW * ((g.C + 63) / 64 * 64), os[2], &g);
    if (ep) { gp.alpha = ep->alpha; gp.bias = ep->bias; gp.act = (uint32_t)ep->activation; }
    rc = launch_wgmma(c, st, gp, false, false);
  }
  for (CUdeviceptr t : tmp)
    if (t) pool_free(c, t, st);   // stream-ordered: reusable by later work once the GEMM has drained
  return rc;
}

// ------------------------------------------------------------------------------------------------ convolution backward
// Zeros written to `rows` rows of `cols` elements, `pitch` elements apart (a 2-D device memset; recorded as one plan line).
static int memset2d_zero(b200_ctx* c, CUstream st, CUdeviceptr dst, size_t esz, uint64_t pitch, uint64_t cols, uint64_t rows) {
  if (c->dry) {
    char line[96];
    snprintf(line, sizeof(line), "memset2d esz=%zu cols=%llu rows=%llu\n", esz, (unsigned long long)cols, (unsigned long long)rows);
    c->plan += line;
    return B200_OK;
  }
  if (esz == 4) CU_CHECK(g_drv.cuMemsetD2D32Async_p(dst, pitch * 4, 0u, cols, rows, st));
  else CU_CHECK(g_drv.cuMemsetD2D16Async_p(dst, pitch * 2, 0, cols, rows, st));
  return B200_OK;
}

// One dimension of the data gradient's phase decomposition.  Output index h = r + s * i (phase r, 0 <= r < s) receives
// dy[i + e] * w[k] for the taps k with (r + p - k * d) % s == 0, e = (r + p - k * d) / s.  Sorted by e ascending (k
// descending) the taps are an arithmetic progression: e_t = e0 + t * d', d' = d / gcd(s, d).
struct DgradPhase1D {
  uint32_t r, taps, kmax;   // kmax: the tap with the smallest e (t = 0); taps == 0: the phase receives nothing
  int64_t e0;
  uint32_t dil, step;       // tap t is k = kmax - t * step (step = s / gcd(s, d)) and reads dy offset e0 + t * dil
  uint64_t extent;          // ceil((H - r) / s), 0 when r >= H
};
static DgradPhase1D dgrad_phase(uint64_t H, uint64_t K, int64_t s, int64_t p, int64_t d, uint32_t r) {
  DgradPhase1D ph{};
  ph.r = r;
  int64_t g = s, b = d;
  while (b) { const int64_t t = g % b; g = b; b = t; }
  ph.dil = (uint32_t)(d / g);
  ph.step = (uint32_t)(s / g);
  ph.extent = r < H ? (H - r + s - 1) / s : 0;
  for (int64_t k = (int64_t)K - 1; k >= 0; --k) {
    const int64_t num = (int64_t)r + p - k * d;
    if (((num % s) + s) % s != 0) continue;
    if (ph.taps == 0) { ph.kmax = (uint32_t)k; ph.e0 = num / s; }
    ++ph.taps;
  }
  return ph;
}

// The taps of a phase in walk order (ascending dy offset), comma-separated, for the plan lines.
static std::string dgrad_taps(const DgradPhase1D& q) {
  std::string s;
  for (uint32_t t = 0; t < q.taps; ++t) s += (t ? "," : "") + std::to_string(q.kmax - t * q.step);
  return s;
}

// The 2-D data gradient's phases (also b200_conv_transpose2d's, x in dy's role): per dimension, and the im2col corner
// limits of every phase that runs.  dx is [N, H, W, *] from dy [N, OH, OW, Cout]; *zero_phase: a phase with pixels receives
// no tap (or Cout == 0).
static int dgrad2_plan(const char* what, const b200_conv2d_args& a, uint64_t H, uint64_t W, uint64_t KH, uint64_t KW, uint64_t OH,
                       uint64_t OW, uint64_t Cout, std::vector<DgradPhase1D>* phs, std::vector<DgradPhase1D>* pws, bool* zero_phase) {
  for (int r = 0; r < a.stride_h; ++r) phs->push_back(dgrad_phase(H, KH, a.stride_h, a.pad_h, a.dilation_h, (uint32_t)r));
  for (int r = 0; r < a.stride_w; ++r) pws->push_back(dgrad_phase(W, KW, a.stride_w, a.pad_w, a.dilation_w, (uint32_t)r));
  *zero_phase = false;
  for (const DgradPhase1D& ph : *phs)
    for (const DgradPhase1D& pw : *pws) {
      if (!ph.extent || !pw.extent) continue;
      if (!ph.taps || !pw.taps || Cout == 0) { *zero_phase = true; continue; }
      const int64_t corners[4] = {ph.e0, pw.e0, ph.e0 + (int64_t)ph.extent - (int64_t)OH, pw.e0 + (int64_t)pw.extent - (int64_t)OW};
      int rc = conv_check_corners(what, corners);
      if (rc) return rc;
    }
  return B200_OK;
}

// Every phase's flipped, channel-transposed weights [C][Th][Tw][cp] in one pooled buffer (*buf) of KH * KW * C * cp
// elements, written by conv_dgrad_weights from w [Cout, KH, KW, C] (strides ws); wp->off holds each phase's block.
static int dgrad2_prep(b200_ctx* c, CUstream st, uint64_t w, const uint64_t ws[4], const b200_conv2d_args& a, uint64_t C, uint64_t Cout,
                       uint64_t cp, uint64_t KH, uint64_t KW, const std::vector<DgradPhase1D>& phs, const std::vector<DgradPhase1D>& pws,
                       CUdeviceptr* buf, ConvDgradWeightsParams* wp_out) {
  ConvDgradWeightsParams& wp = *wp_out;
  memset(&wp, 0, sizeof(wp));
  int rc = pool_alloc(c, KH * KW * C * cp * 2, buf, st);
  if (rc) return rc;
  wp.w = w; wp.out = *buf;
  wp.s_co = ws[0]; wp.s_ky = ws[1]; wp.s_kx = ws[2]; wp.s_c = ws[3];
  wp.C = C; wp.Cout = Cout; wp.cp = cp;
  wp.KH = (uint32_t)KH; wp.KW = (uint32_t)KW; wp.sh = (uint32_t)a.stride_h; wp.sw = (uint32_t)a.stride_w;
  wp.dh = (uint32_t)a.dilation_h; wp.dw = (uint32_t)a.dilation_w; wp.ph = (uint32_t)a.pad_h; wp.pw = (uint32_t)a.pad_w;
  wp.qh = phs[0].step; wp.qw = pws[0].step;
  uint64_t off = 0;
  for (const DgradPhase1D& ph : phs)
    for (const DgradPhase1D& pw : pws) {
      wp.off[ph.r * a.stride_w + pw.r] = off;
      off += (uint64_t)ph.taps * pw.taps * C * cp;
    }
  for (const DgradPhase1D& ph : phs) { wp.kmax_h[ph.r] = ph.kmax; wp.taps_h[ph.r] = ph.taps; }
  for (const DgradPhase1D& pw : pws) { wp.kmax_w[pw.r] = pw.kmax; wp.taps_w[pw.r] = pw.taps; }
  CUfunction f;
  rc = get_func(c, "conv_dgrad_weights", &f);
  void* kargs[] = {&wp};
  if (!rc) rc = launch(c, f, (unsigned)(((C + 31) / 32) * ((cp + 31) / 32)), (unsigned)(KH * KW), 1, 256, 0, 1, st, kargs);
  return rc;
}

// One phase (ph, pw) as a stride-1 convolution of dy (read through y) into C channels: its geometry, with the phase-addressed
// epilogue of dx (normalised strides os) unless the conv stride is 1.
static ConvGeom dgrad2_geom(uint64_t N, uint64_t OH, uint64_t OW, uint64_t cp, uint64_t C, const DgradPhase1D& ph, const DgradPhase1D& pw,
                            const NhwcOperand& y, const uint64_t os[4], const b200_conv2d_args& a) {
  ConvGeom g{};
  g.N = N; g.H = OH; g.W = OW; g.C = cp; g.KH = ph.taps; g.KW = pw.taps; g.OH = ph.extent; g.OW = pw.extent; g.Cout = C;
  g.sh = 1; g.sw = 1; g.ph = (int32_t)-ph.e0; g.pw = (int32_t)-pw.e0; g.dh = (int32_t)ph.dil; g.dw = (int32_t)pw.dil;
  g.x_sw = y.s_w; g.x_sh = y.s_h; g.x_sn = y.s_n;
  g.w_sp = cp; g.w_sco = (uint64_t)ph.taps * pw.taps * cp;
  g.box = true; g.lo_h = (int32_t)ph.e0; g.lo_w = (int32_t)pw.e0;
  g.mode = a.stride_h == 1 && a.stride_w == 1 ? 0 : 1;
  g.dx_sn = os[0]; g.dx_si = (uint64_t)a.stride_h * os[1]; g.dx_sj = (uint64_t)a.stride_w * os[2];
  return g;
}

// The plan line of phase (ph, pw): `head` r=(rh,rw) taps_h= taps_w= dil= lower= upper= extent=, no newline.
static std::string dgrad2_phase_line(const char* head, const DgradPhase1D& ph, const DgradPhase1D& pw, uint64_t OH, uint64_t OW) {
  return std::string(head) + " r=(" + std::to_string(ph.r) + "," + std::to_string(pw.r) + ") taps_h=" + dgrad_taps(ph) +
         " taps_w=" + dgrad_taps(pw) + " dil=(" + std::to_string(ph.dil) + "," + std::to_string(pw.dil) + ") lower=(" +
         std::to_string(ph.e0) + "," + std::to_string(pw.e0) + ") upper=(" + std::to_string(ph.e0 + (int64_t)ph.extent - (int64_t)OH) +
         "," + std::to_string(pw.e0 + (int64_t)pw.extent - (int64_t)OW) + ") extent=(" + std::to_string(ph.extent) + "," +
         std::to_string(pw.extent) + ")";
}

extern "C" int b200_conv2d_backward_data(b200_ctx* c, b200_stream s, b200_dtype in_dtype, b200_dtype out_dtype, b200_dptr dy,
                                         const uint64_t* dy_shape, const uint64_t* dy_strides, b200_dptr w, const uint64_t* w_shape,
                                         const uint64_t* w_strides, b200_dptr dx, const uint64_t* dx_shape, const uint64_t* dx_strides,
                                         const b200_conv2d_args* args) {
  CTX_ENTER(c);
  const char* what = "conv2d_backward_data";
  if (!dy_shape || !w_shape || !dx_shape || !args) return fail(B200_ERR_INVALID_ARG, "%s: null shape or args", what);
  const b200_conv2d_args& a = *args;
  const uint64_t N = dx_shape[0], H = dx_shape[1], W = dx_shape[2], C = dx_shape[3];
  const uint64_t Cout = w_shape[0], KH = w_shape[1], KW = w_shape[2];
  uint64_t OH = 0, OW = 0;
  int rc = conv_check_args(what, in_dtype, out_dtype, a, nullptr, C, w_shape[3]);
  if (!rc) rc = conv_check_shape(what, a, dx_shape, w_shape, dy_shape, "dy", &OH, &OW);
  if (!rc && KH && KW) rc = conv_check_stride(what, a);
  if (rc) return rc;
  if (N == 0 || H == 0 || W == 0 || C == 0) return B200_OK;   // no dx
  const uint64_t lim = 1ull << 31;
  if (N * H * W >= lim) return fail(B200_ERR_UNSUPPORTED, "%s: N * H * W = %llu must be < 2^31", what, (unsigned long long)(N * H * W));
  if (KH * KW * ((Cout + 63) / 64 * 64) >= lim) return fail(B200_ERR_UNSUPPORTED, "%s: KH * KW * Cout (Cout padded to 64) must be < 2^31", what);
  // phases of each dimension, and the im2col limits of every phase that runs
  std::vector<DgradPhase1D> phs, pws;
  bool zero_phase = false;
  if ((rc = dgrad2_plan(what, a, H, W, KH, KW, OH, OW, Cout, &phs, &pws, &zero_phase))) return rc;
  if ((rc = conv_check_ptrs(what, dy, w, dx, "dx", out_dtype))) return rc;
  const size_t osz = dtype_size(out_dtype);
  uint64_t os[4], ys[4], ws[4];
  conv_norm_strides(dx_shape, dx_strides, os);
  if ((rc = conv_check_pixels(what, "dx", dx_shape, os))) return rc;
  CUstream st = resolve_stream(c, s);
  // dx pixels that no tap reaches are exact zeros: one memset of dx, before the phases that overwrite the rest
  if (zero_phase) {
    rc = memset2d_zero(c, st, dx, osz, os[2], C, N * H * W);
    if (rc) return rc;
  }
  if (Cout == 0 || KH == 0 || KW == 0) return B200_OK;
  conv_norm_strides(dy_shape, dy_strides, ys);
  conv_norm_strides(w_shape, w_strides, ws);
  CUdeviceptr tmp[3] = {0, 0, 0};
  NhwcOperand y{};
  rc = conv_prep_nhwc(c, st, in_dtype, dy, dy_shape, ys, kFlatNone, tmp, &y);
  // every phase's flipped, channel-transposed weights [C][Th][Tw][cp] in one pooled buffer of KH * KW * C * cp elements
  const uint64_t cp = y.C;
  ConvDgradWeightsParams wp;
  memset(&wp, 0, sizeof(wp));
  if (!rc) rc = dgrad2_prep(c, st, w, ws, a, C, Cout, cp, KH, KW, phs, pws, &tmp[2], &wp);
  // one stride-1 convolution of dy per phase that has taps and pixels
  for (const DgradPhase1D& ph : phs)
    for (const DgradPhase1D& pw : pws) {
      if (rc) break;
      if (!ph.extent || !pw.extent || !ph.taps || !pw.taps) continue;
      ConvGeom g = dgrad2_geom(N, OH, OW, cp, C, ph, pw, y, os, a);
      if (c->dry) c->plan += dgrad2_phase_line("conv dgrad phase", ph, pw, OH, OW) + "\n";
      const GemmProblem gp = conv_problem(in_dtype, out_dtype, y.ptr, tmp[2] + wp.off[ph.r * a.stride_w + pw.r] * 2,
                                          dx + ((uint64_t)ph.r * os[1] + (uint64_t)pw.r * os[2]) * osz, N * ph.extent * pw.extent, C,
                                          (uint64_t)ph.taps * pw.taps * ((cp + 63) / 64 * 64), os[2], &g);
      rc = launch_wgmma(c, st, gp, false, false);
    }
  for (CUdeviceptr t : tmp)
    if (t) pool_free(c, t, st);   // stream-ordered: reusable by later work once the GEMMs have drained
  return rc;
}

extern "C" int b200_conv2d_backward_weight(b200_ctx* c, b200_stream s, b200_dtype in_dtype, b200_dtype out_dtype, b200_dptr x,
                                           const uint64_t* x_shape, const uint64_t* x_strides, b200_dptr dy, const uint64_t* dy_shape,
                                           const uint64_t* dy_strides, b200_dptr dw, const uint64_t* dw_shape, const uint64_t* dw_strides,
                                           const b200_conv2d_args* args) {
  CTX_ENTER(c);
  const char* what = "conv2d_backward_weight";
  if (!x_shape || !dy_shape || !dw_shape || !args) return fail(B200_ERR_INVALID_ARG, "%s: null shape or args", what);
  const b200_conv2d_args& a = *args;
  const uint64_t N = x_shape[0], H = x_shape[1], W = x_shape[2], C = x_shape[3];
  const uint64_t Cout = dw_shape[0], KH = dw_shape[1], KW = dw_shape[2];
  uint64_t OH = 0, OW = 0;
  int rc = conv_check_args(what, in_dtype, out_dtype, a, nullptr, C, dw_shape[3]);
  if (!rc) rc = conv_check_shape(what, a, x_shape, dw_shape, dy_shape, "dy", &OH, &OW);
  if (!rc && KH && KW) rc = conv_check_stride(what, a);
  if (rc) return rc;
  if (Cout == 0 || C == 0 || KH == 0 || KW == 0) return B200_OK;   // no dw
  if ((rc = conv_check_fwd_corners(what, a, KH, KW))) return rc;   // x is read through the forward's map
  const uint64_t P = N * OH * OW, lim = 1ull << 31;
  if (P >= lim) return fail(B200_ERR_UNSUPPORTED, "%s: N * OH * OW = %llu must be < 2^31", what, (unsigned long long)P);
  const uint64_t cx = (C + 7) / 8 * 8;
  if (KH * KW * ((cx + 63) / 64 * 64) >= lim) return fail(B200_ERR_UNSUPPORTED, "%s: KH * KW * C (C padded to 64) must be < 2^31", what);
  if ((rc = conv_check_ptrs(what, x, dy, dw, "dw", out_dtype))) return rc;
  const size_t osz = dtype_size(out_dtype);
  uint64_t ds[4], xs[4], ys[4], dw_sp = 0;
  conv_norm_strides(dw_shape, dw_strides, ds);
  if ((rc = conv_check_dw(what, dw_shape, ds, osz, &dw_sp))) return rc;
  CUstream st = resolve_stream(c, s);
  if (P == 0) {
    // no pixels: dw is exactly zero
    if (ds[0] == KH * KW * dw_sp) return memset2d_zero(c, st, dw, osz, dw_sp, C, Cout * KH * KW);
    for (uint64_t co = 0; co < Cout && !rc; ++co) rc = memset2d_zero(c, st, dw + co * ds[0] * osz, osz, dw_sp, C, KH * KW);
    return rc;
  }
  conv_norm_strides(x_shape, x_strides, xs);
  conv_norm_strides(dy_shape, dy_strides, ys);
  CUdeviceptr tmp[4] = {0, 0, 0, 0};
  NhwcOperand xo{}, yo{};
  rc = conv_prep_nhwc(c, st, in_dtype, x, x_shape, xs, kFlatNone, &tmp[0], &xo);
  if (!rc) rc = conv_prep_nhwc(c, st, in_dtype, dy, dy_shape, ys, kFlatNHW, &tmp[2], &yo);
  if (!rc) {
    ConvGeom g{};
    g.N = N; g.H = H; g.W = W; g.C = xo.C; g.KH = KH; g.KW = KW; g.OH = OH; g.OW = OW; g.Cout = Cout;
    g.sh = a.stride_h; g.sw = a.stride_w; g.ph = a.pad_h; g.pw = a.pad_w; g.dh = a.dilation_h; g.dw = a.dilation_w;
    g.x_sw = xo.s_w; g.x_sh = xo.s_h; g.x_sn = xo.s_n;
    g.mode = 2; g.dw_sp = dw_sp; g.dw_c = C;
    GemmProblem gp = conv_problem(in_dtype, out_dtype, yo.ptr, xo.ptr, dw, Cout, KH * KW * ((xo.C + 63) / 64 * 64), P, ds[0], &g);
    gp.a_sm = 1; gp.a_sk = yo.s_w; gp.b_sn = 1; gp.b_sk = xo.s_w;   // both operands MN-major
    // few tiles, a long K: the stream-K head may cut a tile into as many ranges as fill the SMs, each >= 8 k-blocks
    gp.sk_max_parts = std::max<uint64_t>(8, (P + 63) / 64 / 8);
    rc = launch_wgmma(c, st, gp, true, true);
  }
  for (CUdeviceptr t : tmp)
    if (t) pool_free(c, t, st);   // stream-ordered: reusable by later work once the GEMM has drained
  return rc;
}

// ------------------------------------------------------------------------------------------------ 3-D convolution
// b200_conv3d*: the 2-D machinery with a depth dimension.  Arrays over the spatial dimensions are ordered (D, H, W).
// Rank-5 tensor maps take pixel-box corners in [-16, 15] (cuda.h: cuTensorMapEncodeIm2col) and the load's im2col offsets
// in [0, 31] (5 bits each; PTX ISA, cp.async.bulk.tensor im2col mode).
static constexpr int64_t kIm2col5Lo = -16, kIm2col5Hi = 15, kIm2col5MaxOffset = 31;

// Strides of a rank-5 view with extent-1 dimensions normalised (see conv_norm_strides).
static void conv3_norm_strides(const uint64_t* shape, const uint64_t* strides, uint64_t* out) {
  uint64_t inner = 1;
  for (int d = 4; d >= 0; --d) {
    out[d] = strides ? strides[d] : inner;
    if (shape[d] == 1) out[d] = inner;
    inner = out[d] * shape[d];
  }
}

// (D, H, W) = dimensions 1..3 of a rank-5 view as one strided dimension: its stride, or 0.
static uint64_t conv3_flat_dhw(const uint64_t* shape, const uint64_t* ns) {
  const uint64_t s_hw = conv_flat_stride(shape[2], shape[3], ns[2], ns[3]);
  return s_hw == 0 ? 0 : conv_flat_stride(shape[1], shape[2] * shape[3], ns[1], s_hw);
}

// conv_check_args for the 3-D args: dtypes, activation, strides / dilations >= 1, padding >= 0, channels.
static int conv3_check_args(const char* what, b200_dtype in_dtype, b200_dtype out_dtype, const b200_conv3d_args& a, const b200_epilogue* ep,
                            uint64_t in_c, uint64_t w_c) {
  const b200_conv2d_args hw{a.stride_h, a.stride_w, a.pad_h, a.pad_w, a.dilation_h, a.dilation_w};
  if (a.stride_d < 1 || a.dilation_d < 1 || a.pad_d < 0)
    return fail(B200_ERR_INVALID_ARG, "%s: strides and dilations must be >= 1 and padding >= 0", what);
  return conv_check_args(what, in_dtype, out_dtype, hw, ep, in_c, w_c);
}

// Extents < 2^31, then PyTorch's output rule per dimension: y must be [N, OD, OH, OW, Cout] for in [N, D, H, W, C] and
// w [Cout, KD, KH, KW, *].  O receives (OD, OH, OW).
static int conv3_check_shape(const char* what, const b200_conv3d_args& a, const uint64_t* in, const uint64_t* w, const uint64_t* y,
                             const char* y_name, uint64_t O[3]) {
  const uint64_t lim = 1ull << 31;
  for (int d = 0; d < 5; ++d)
    if (in[d] >= lim || w[d] >= lim || y[d] >= lim) return fail(B200_ERR_UNSUPPORTED, "%s: extents must be < 2^31", what);
  if (w[1] == 0 || w[2] == 0 || w[3] == 0) return B200_OK;
  const int64_t s[3] = {a.stride_d, a.stride_h, a.stride_w}, p[3] = {a.pad_d, a.pad_h, a.pad_w};
  const int64_t dl[3] = {a.dilation_d, a.dilation_h, a.dilation_w};
  for (int i = 0; i < 3; ++i) {
    const int64_t n = (int64_t)in[1 + i] + 2 * p[i] - dl[i] * ((int64_t)w[1 + i] - 1) - 1;
    if (n < 0) return fail(B200_ERR_INVALID_ARG, "%s: the dilated kernel is larger than the padded input (output extent < 1)", what);
    O[i] = (uint64_t)(n / s[i]) + 1;
  }
  if (y[0] != in[0] || y[1] != O[0] || y[2] != O[1] || y[3] != O[2] || y[4] != w[0])
    return fail(B200_ERR_INVALID_ARG, "%s: %s is [%llu,%llu,%llu,%llu,%llu], expected [%llu,%llu,%llu,%llu,%llu]", what, y_name,
                (unsigned long long)y[0], (unsigned long long)y[1], (unsigned long long)y[2], (unsigned long long)y[3],
                (unsigned long long)y[4], (unsigned long long)in[0], (unsigned long long)O[0], (unsigned long long)O[1],
                (unsigned long long)O[2], (unsigned long long)w[0]);
  return B200_OK;
}

// The rank-5 im2col limits: pixel-box corners in [-16, 15], and the largest im2col offset (dilation * (taps - 1)) of each
// dimension in [0, 31].
static int conv3_check_corners(const char* what, const int64_t* corners, int n) {
  for (int i = 0; i < n; ++i)
    if (corners[i] < kIm2col5Lo || corners[i] > kIm2col5Hi)
      return fail(B200_ERR_UNSUPPORTED, "%s: im2col pixel-box corner %lld outside [-16, 15] (rank-5 tensor map)", what, (long long)corners[i]);
  return B200_OK;
}
static int conv3_check_offsets(const char* what, const int64_t max_off[3]) {
  for (int i = 0; i < 3; ++i)
    if (max_off[i] > kIm2col5MaxOffset)
      return fail(B200_ERR_UNSUPPORTED, "%s: im2col offset dilation * (kernel - 1) = %lld exceeds 31 (5-bit rank-5 offsets)", what,
                  (long long)max_off[i]);
  return B200_OK;
}
// The forward's map (also backward_weight's x): corners -p and p - d*(K-1), offsets d*(K-1), and conv strides <= 8.
static int conv3_check_fwd(const char* what, const b200_conv3d_args& a, const uint64_t* w) {
  const int64_t p[3] = {a.pad_d, a.pad_h, a.pad_w}, dl[3] = {a.dilation_d, a.dilation_h, a.dilation_w};
  int64_t corners[6], off[3];
  for (int i = 0; i < 3; ++i) {
    off[i] = dl[i] * ((int64_t)w[1 + i] - 1);
    corners[2 * i] = -p[i];
    corners[2 * i + 1] = p[i] - off[i];
  }
  int rc = conv3_check_corners(what, corners, 6);
  if (!rc) rc = conv3_check_offsets(what, off);
  return rc;
}
static int conv3_check_stride(const char* what, const b200_conv3d_args& a) {
  if (a.stride_d > kDgradMaxStride || a.stride_h > kDgradMaxStride || a.stride_w > kDgradMaxStride)
    return fail(B200_ERR_UNSUPPORTED, "%s: the conv stride must be <= %d", what, kDgradMaxStride);
  return B200_OK;
}

// An NDHWC output (out or dx): unit channel stride, one pixel pitch >= its channels across N, D, H, W.
static int conv3_check_pixels(const char* what, const char* name, const uint64_t* shape, const uint64_t* ns) {
  if (ns[4] != 1 || ns[3] < shape[4] || ns[2] != shape[3] * ns[3] || ns[1] != shape[2] * ns[2] || ns[0] != shape[1] * ns[1])
    return fail(B200_ERR_UNSUPPORTED, "%s: %s must have unit channel stride and one pixel pitch >= its channels for N, D, H, W", what, name);
  return B200_OK;
}

// An operand [N, D, H, W, C] (normalised strides ns) as the convolution maps read it; conv_prep_nhwc with a depth dimension.
// flat: none (x, dy in the data gradient), (D, H, W) (the weights: one kernel-position stride, returned as s_w) or
// (N, D, H, W) (dy in the weight gradient: [pixels, Cout]).
struct NdhwcOperand {
  uint64_t ptr, C, s_w, s_h, s_d, s_n;
};
static int conv3_prep(b200_ctx* c, CUstream st, b200_dtype dt, uint64_t ptr, const uint64_t* shape, const uint64_t* ns, ConvFlat flat,
                      CUdeviceptr tmp[2], NdhwcOperand* o) {
  const uint64_t N = shape[0], D = shape[1], H = shape[2], W = shape[3], C = shape[4];
  const uint64_t spx = conv3_flat_dhw(shape, ns);   // (D, H, W) as one pixel dimension
  int rc = B200_OK;
  auto gather = [&]() -> int {
    CUdeviceptr buf;
    int r = pool_alloc(c, N * D * H * W * C * 2, &buf, st);
    if (r) return r;
    r = b200_into_contiguous(c, static_cast<b200_stream>(st), dt, ptr, buf, 5, shape, ns);
    if (r) { pool_free(c, buf, st); return r; }
    tmp[0] = buf;
    return B200_OK;
  };
  if (C % 8 == 0) {
    bool in_place = ptr % 16 == 0 && ns[4] == 1 && conv_al16(ns[0]);
    if (flat == kFlatHW) in_place = in_place && spx != 0 && conv_al16(spx);
    else in_place = in_place && conv_al16(ns[1]) && conv_al16(ns[2]) && conv_al16(ns[3]) &&
                    (flat == kFlatNone || (ns[2] == W * ns[3] && ns[1] == H * ns[2] && ns[0] == D * ns[1]));
    if (in_place) {
      *o = {ptr, C, flat == kFlatHW ? spx : ns[3], ns[2], ns[1], ns[0]};
      return B200_OK;
    }
    rc = gather();
    *o = {tmp[0], C, C, W * C, H * W * C, D * H * W * C};
    return rc;
  }
  const uint64_t cp = (C + 7) / 8 * 8;
  uint64_t in = ptr, sb = ns[0], sp = spx, sc = ns[4];
  if (spx == 0) {
    rc = gather();
    in = tmp[0]; sb = D * H * W * C; sp = C; sc = 1;
  }
  if (!rc) rc = conv_pad_channels(c, st, in, N, D * H * W, C, sb, sp, sc, cp, &tmp[1]);
  *o = {tmp[1], cp, cp, W * cp, H * W * cp, D * H * W * cp};
  return rc;
}

// ConvGeom of a 3-D map: input extents I = (D, H, W), kernel K, output O, per-dimension stride / pad / dilation.
static ConvGeom conv3_geom(uint64_t N, const uint64_t I[3], uint64_t C, const uint64_t K[3], const uint64_t O[3], uint64_t Cout,
                           const int32_t s[3], const int32_t p[3], const int32_t d[3]) {
  ConvGeom g{};
  g.dims = 3;
  g.N = N; g.D = I[0]; g.H = I[1]; g.W = I[2]; g.C = C; g.KD = K[0]; g.KH = K[1]; g.KW = K[2];
  g.OD = O[0]; g.OH = O[1]; g.OW = O[2]; g.Cout = Cout;
  g.sd = s[0]; g.sh = s[1]; g.sw = s[2]; g.pd = p[0]; g.ph = p[1]; g.pw = p[2]; g.dd = d[0]; g.dh = d[1]; g.dw = d[2];
  return g;
}

extern "C" int b200_conv3d(b200_ctx* c, b200_stream s, b200_dtype in_dtype, b200_dtype out_dtype, b200_dptr x, const uint64_t* x_shape,
                           const uint64_t* x_strides, b200_dptr w, const uint64_t* w_shape, const uint64_t* w_strides, b200_dptr out,
                           const uint64_t* out_shape, const uint64_t* out_strides, const b200_conv3d_args* args, const b200_epilogue* ep) {
  CTX_ENTER(c);
  const char* what = "conv3d";
  if (!x_shape || !w_shape || !out_shape || !args) return fail(B200_ERR_INVALID_ARG, "%s: null shape or args", what);
  const b200_conv3d_args& a = *args;
  const uint64_t N = x_shape[0], C = x_shape[4], Cout = w_shape[0];
  const uint64_t I[3] = {x_shape[1], x_shape[2], x_shape[3]}, K[3] = {w_shape[1], w_shape[2], w_shape[3]};
  int rc = conv3_check_args(what, in_dtype, out_dtype, a, ep, C, w_shape[4]);
  if (rc) return rc;
  if (N == 0 || I[0] == 0 || I[1] == 0 || I[2] == 0 || C == 0 || Cout == 0 || K[0] == 0 || K[1] == 0 || K[2] == 0) return B200_OK;
  uint64_t O[3] = {0, 0, 0};
  if ((rc = conv3_check_shape(what, a, x_shape, w_shape, out_shape, "out", O))) return rc;
  if ((rc = conv3_check_fwd(what, a, w_shape)) || (rc = conv3_check_stride(what, a))) return rc;
  const uint64_t M = N * O[0] * O[1] * O[2], lim = 1ull << 31, KK = K[0] * K[1] * K[2];
  if (M >= lim) return fail(B200_ERR_UNSUPPORTED, "%s: N * OD * OH * OW = %llu must be < 2^31", what, (unsigned long long)M);
  if ((rc = conv_check_ptrs(what, x, w, out, "output", out_dtype))) return rc;
  uint64_t os[5], xs[5], ws[5];
  conv3_norm_strides(out_shape, out_strides, os);
  if ((rc = conv3_check_pixels(what, "out", out_shape, os))) return rc;
  if (KK * ((C + 63) / 64 * 64) >= lim) return fail(B200_ERR_UNSUPPORTED, "%s: KD * KH * KW * C (C padded to 64) must be < 2^31", what);
  CUstream st = resolve_stream(c, s);
  conv3_norm_strides(x_shape, x_strides, xs);
  conv3_norm_strides(w_shape, w_strides, ws);
  CUdeviceptr tmp[4] = {0, 0, 0, 0};
  NdhwcOperand xo{}, wo{};
  rc = conv3_prep(c, st, in_dtype, x, x_shape, xs, kFlatNone, &tmp[0], &xo);
  if (!rc) rc = conv3_prep(c, st, in_dtype, w, w_shape, ws, kFlatHW, &tmp[2], &wo);
  if (!rc) {
    const int32_t sv[3] = {a.stride_d, a.stride_h, a.stride_w}, pv[3] = {a.pad_d, a.pad_h, a.pad_w};
    const int32_t dv[3] = {a.dilation_d, a.dilation_h, a.dilation_w};
    ConvGeom g = conv3_geom(N, I, xo.C, K, O, Cout, sv, pv, dv);
    g.x_sw = xo.s_w; g.x_sh = xo.s_h; g.x_sd = xo.s_d; g.x_sn = xo.s_n;
    g.w_sp = wo.s_w; g.w_sco = wo.s_n;
    GemmProblem gp = conv_problem(in_dtype, out_dtype, xo.ptr, wo.ptr, out, M, Cout, KK * ((g.C + 63) / 64 * 64), os[3], &g);
    if (ep) { gp.alpha = ep->alpha; gp.bias = ep->bias; gp.act = (uint32_t)ep->activation; }
    rc = launch_wgmma(c, st, gp, false, false);
  }
  for (CUdeviceptr t : tmp)
    if (t) pool_free(c, t, st);   // stream-ordered: reusable by later work once the GEMM has drained
  return rc;
}

// The 3-D data gradient's phases (also b200_conv_transpose3d's): per dimension (D, H, W) of dx extents I from dy extents
// O, and the rank-5 im2col limits (corners, offsets) of every phase that runs.  *zero_phase as dgrad2_plan.
static int dgrad3_plan(const char* what, const int64_t sv[3], const int64_t pv[3], const int64_t dv[3], const uint64_t I[3],
                       const uint64_t K[3], const uint64_t O[3], uint64_t Cout, std::vector<DgradPhase1D> ph[3], bool* zero_phase) {
  for (int i = 0; i < 3; ++i)
    for (int64_t r = 0; r < sv[i]; ++r) ph[i].push_back(dgrad_phase(I[i], K[i], sv[i], pv[i], dv[i], (uint32_t)r));
  *zero_phase = false;
  for (const DgradPhase1D& pd : ph[0])
    for (const DgradPhase1D& phh : ph[1])
      for (const DgradPhase1D& pw : ph[2]) {
        const DgradPhase1D* q[3] = {&pd, &phh, &pw};
        if (!pd.extent || !phh.extent || !pw.extent) continue;
        if (!pd.taps || !phh.taps || !pw.taps || Cout == 0) { *zero_phase = true; continue; }
        int64_t corners[6], off[3];
        for (int i = 0; i < 3; ++i) {
          corners[2 * i] = q[i]->e0;
          corners[2 * i + 1] = q[i]->e0 + (int64_t)q[i]->extent - (int64_t)O[i];
          off[i] = (int64_t)(q[i]->taps - 1) * q[i]->dil;
        }
        int rc = conv3_check_corners(what, corners, 6);
        if (!rc) rc = conv3_check_offsets(what, off);
        if (rc) return rc;
      }
  return B200_OK;
}

// conv3d_dgrad_weights' parameters for the phases ph of w [Cout, KD, KH, KW, C], and where each phase's block starts.
struct Dgrad3Prep {
  Conv3dDgradWeightsParams wp;
  uint64_t pre[3][kDgradMaxStride];
  uint64_t k1, k2, ccp;
  Dgrad3Prep(const std::vector<DgradPhase1D> ph[3], const uint64_t K[3], const int64_t sv[3], const int64_t pv[3], const int64_t dv[3],
             uint64_t C, uint64_t cp) : k1(K[1]), k2(K[2]), ccp(C * cp) {
    memset(&wp, 0, sizeof(wp));
    for (int i = 0; i < 3; ++i) {
      uint64_t acc = 0;
      for (const DgradPhase1D& q : ph[i]) { pre[i][q.r] = acc; acc += q.taps; wp.kmax[i][q.r] = q.kmax; wp.taps[i][q.r] = q.taps; }
      wp.k[i] = (uint32_t)K[i]; wp.s[i] = (uint32_t)sv[i]; wp.d[i] = (uint32_t)dv[i]; wp.p[i] = (uint32_t)pv[i]; wp.q[i] = ph[i][0].step;
    }
    wp.C = C; wp.cp = cp;
  }
  // first element of phase (rd, rh, rw)'s block
  uint64_t off(uint32_t rd, uint32_t rh, uint32_t rw) const {
    return ccp * (pre[0][rd] * k1 * k2 + (uint64_t)wp.taps[0][rd] * (pre[1][rh] * k2 + (uint64_t)wp.taps[1][rh] * pre[2][rw]));
  }
};

// Every phase's flipped, channel-transposed weights in one pooled buffer (*buf) of KK * C * cp elements (conv3d_dgrad_weights).
static int dgrad3_prep(b200_ctx* c, CUstream st, uint64_t w, const uint64_t ws[5], uint64_t Cout, uint64_t KK, Dgrad3Prep* pr, CUdeviceptr* buf) {
  Conv3dDgradWeightsParams& wp = pr->wp;
  int rc = pool_alloc(c, KK * wp.C * wp.cp * 2, buf, st);
  if (rc) return rc;
  wp.w = w; wp.out = *buf;
  wp.s_co = ws[0]; wp.s_kz = ws[1]; wp.s_ky = ws[2]; wp.s_kx = ws[3]; wp.s_c = ws[4];
  wp.Cout = Cout;
  CUfunction f;
  rc = get_func(c, "conv3d_dgrad_weights", &f);
  void* kargs[] = {&wp};
  if (!rc) rc = launch(c, f, (unsigned)(((wp.C + 31) / 32) * ((wp.cp + 31) / 32)), (unsigned)KK, 1, 256, 0, 1, st, kargs);
  return rc;
}

// Phase q = (D, H, W) phases as a stride-1 3-D convolution of dy (y, extents O) into C channels; dgrad2_geom with depth.
static ConvGeom dgrad3_geom(uint64_t N, const uint64_t O[3], uint64_t cp, uint64_t C, const DgradPhase1D* const q[3], const NdhwcOperand& y,
                            const uint64_t os[5], const int64_t sv[3]) {
  const uint64_t T[3] = {q[0]->taps, q[1]->taps, q[2]->taps}, E[3] = {q[0]->extent, q[1]->extent, q[2]->extent};
  const int32_t one[3] = {1, 1, 1}, pp[3] = {(int32_t)-q[0]->e0, (int32_t)-q[1]->e0, (int32_t)-q[2]->e0};
  const int32_t dil[3] = {(int32_t)q[0]->dil, (int32_t)q[1]->dil, (int32_t)q[2]->dil};
  ConvGeom g = conv3_geom(N, O, cp, T, E, C, one, pp, dil);
  g.x_sw = y.s_w; g.x_sh = y.s_h; g.x_sd = y.s_d; g.x_sn = y.s_n;
  g.w_sp = cp; g.w_sco = T[0] * T[1] * T[2] * cp;
  g.box = true; g.lo_d = (int32_t)q[0]->e0; g.lo_h = (int32_t)q[1]->e0; g.lo_w = (int32_t)q[2]->e0;
  g.mode = sv[0] == 1 && sv[1] == 1 && sv[2] == 1 ? 0 : 1;
  g.dx_sn = os[0]; g.dx_sd = (uint64_t)sv[0] * os[1]; g.dx_si = (uint64_t)sv[1] * os[2]; g.dx_sj = (uint64_t)sv[2] * os[3];
  return g;
}

// The plan line of phase q: `head` r=(rd,rh,rw) taps_d= taps_h= taps_w= dil= lower= upper= extent=, no newline.
static std::string dgrad3_phase_line(const char* head, const DgradPhase1D* const q[3], const uint64_t O[3]) {
  std::string line = std::string(head) + " r=(" + std::to_string(q[0]->r) + "," + std::to_string(q[1]->r) + "," + std::to_string(q[2]->r) + ")";
  const char* tn[3] = {" taps_d=", " taps_h=", " taps_w="};
  for (int i = 0; i < 3; ++i) line += tn[i] + dgrad_taps(*q[i]);
  auto triple = [&](auto f) { return "(" + std::to_string(f(0)) + "," + std::to_string(f(1)) + "," + std::to_string(f(2)) + ")"; };
  line += " dil=" + triple([&](int i) { return (int64_t)q[i]->dil; });
  line += " lower=" + triple([&](int i) { return q[i]->e0; });
  line += " upper=" + triple([&](int i) { return q[i]->e0 + (int64_t)q[i]->extent - (int64_t)O[i]; });
  line += " extent=" + triple([&](int i) { return (int64_t)q[i]->extent; });
  return line;
}

extern "C" int b200_conv3d_backward_data(b200_ctx* c, b200_stream s, b200_dtype in_dtype, b200_dtype out_dtype, b200_dptr dy,
                                         const uint64_t* dy_shape, const uint64_t* dy_strides, b200_dptr w, const uint64_t* w_shape,
                                         const uint64_t* w_strides, b200_dptr dx, const uint64_t* dx_shape, const uint64_t* dx_strides,
                                         const b200_conv3d_args* args) {
  CTX_ENTER(c);
  const char* what = "conv3d_backward_data";
  if (!dy_shape || !w_shape || !dx_shape || !args) return fail(B200_ERR_INVALID_ARG, "%s: null shape or args", what);
  const b200_conv3d_args& a = *args;
  const uint64_t N = dx_shape[0], C = dx_shape[4], Cout = w_shape[0];
  const uint64_t I[3] = {dx_shape[1], dx_shape[2], dx_shape[3]}, K[3] = {w_shape[1], w_shape[2], w_shape[3]};
  const int64_t sv[3] = {a.stride_d, a.stride_h, a.stride_w}, pv[3] = {a.pad_d, a.pad_h, a.pad_w};
  const int64_t dv[3] = {a.dilation_d, a.dilation_h, a.dilation_w};
  uint64_t O[3] = {0, 0, 0};
  int rc = conv3_check_args(what, in_dtype, out_dtype, a, nullptr, C, w_shape[4]);
  if (!rc) rc = conv3_check_shape(what, a, dx_shape, w_shape, dy_shape, "dy", O);
  if (!rc && K[0] && K[1] && K[2]) rc = conv3_check_stride(what, a);
  if (rc) return rc;
  if (N == 0 || I[0] == 0 || I[1] == 0 || I[2] == 0 || C == 0) return B200_OK;   // no dx
  const uint64_t lim = 1ull << 31, P = N * I[0] * I[1] * I[2], KK = K[0] * K[1] * K[2];
  if (P >= lim) return fail(B200_ERR_UNSUPPORTED, "%s: N * D * H * W = %llu must be < 2^31", what, (unsigned long long)P);
  if (KK * ((Cout + 63) / 64 * 64) >= lim)
    return fail(B200_ERR_UNSUPPORTED, "%s: KD * KH * KW * Cout (Cout padded to 64) must be < 2^31", what);
  // phases of each dimension, and the im2col limits of every phase that runs
  std::vector<DgradPhase1D> ph[3];
  bool zero_phase = false;
  if ((rc = dgrad3_plan(what, sv, pv, dv, I, K, O, Cout, ph, &zero_phase))) return rc;
  if ((rc = conv_check_ptrs(what, dy, w, dx, "dx", out_dtype))) return rc;
  const size_t osz = dtype_size(out_dtype);
  uint64_t os[5], ys[5], ws[5];
  conv3_norm_strides(dx_shape, dx_strides, os);
  if ((rc = conv3_check_pixels(what, "dx", dx_shape, os))) return rc;
  CUstream st = resolve_stream(c, s);
  // dx pixels that no tap reaches are exact zeros: one memset of dx, before the phases that overwrite the rest
  if (zero_phase) {
    rc = memset2d_zero(c, st, dx, osz, os[3], C, P);
    if (rc) return rc;
  }
  if (Cout == 0 || KK == 0) return B200_OK;
  conv3_norm_strides(dy_shape, dy_strides, ys);
  conv3_norm_strides(w_shape, w_strides, ws);
  CUdeviceptr tmp[3] = {0, 0, 0};
  NdhwcOperand y{};
  rc = conv3_prep(c, st, in_dtype, dy, dy_shape, ys, kFlatNone, tmp, &y);
  // every phase's flipped, channel-transposed weights [C][Td][Th][Tw][cp] in one pooled buffer of |w| * cp / Cout elements, in
  // (rd, rh, rw) order (Conv3dDgradWeightsParams)
  const uint64_t cp = y.C;
  Dgrad3Prep prep(ph, K, sv, pv, dv, C, cp);
  if (!rc) rc = dgrad3_prep(c, st, w, ws, Cout, KK, &prep, &tmp[2]);
  // one stride-1 convolution of dy per phase that has taps and pixels
  for (const DgradPhase1D& pd : ph[0])
    for (const DgradPhase1D& phh : ph[1])
      for (const DgradPhase1D& pw : ph[2]) {
        if (rc) break;
        const DgradPhase1D* q[3] = {&pd, &phh, &pw};
        if (!pd.extent || !phh.extent || !pw.extent || !pd.taps || !phh.taps || !pw.taps) continue;
        ConvGeom g = dgrad3_geom(N, O, cp, C, q, y, os, sv);
        if (c->dry) c->plan += dgrad3_phase_line("conv3d dgrad phase", q, O) + "\n";
        const GemmProblem gp = conv_problem(in_dtype, out_dtype, y.ptr, tmp[2] + prep.off(pd.r, phh.r, pw.r) * 2,
                                            dx + ((uint64_t)pd.r * os[1] + (uint64_t)phh.r * os[2] + (uint64_t)pw.r * os[3]) * osz,
                                            N * g.OD * g.OH * g.OW, C, g.KD * g.KH * g.KW * ((cp + 63) / 64 * 64), os[3], &g);
        rc = launch_wgmma(c, st, gp, false, false);
      }
  for (CUdeviceptr t : tmp)
    if (t) pool_free(c, t, st);   // stream-ordered: reusable by later work once the GEMMs have drained
  return rc;
}

extern "C" int b200_conv3d_backward_weight(b200_ctx* c, b200_stream s, b200_dtype in_dtype, b200_dtype out_dtype, b200_dptr x,
                                           const uint64_t* x_shape, const uint64_t* x_strides, b200_dptr dy, const uint64_t* dy_shape,
                                           const uint64_t* dy_strides, b200_dptr dw, const uint64_t* dw_shape, const uint64_t* dw_strides,
                                           const b200_conv3d_args* args) {
  CTX_ENTER(c);
  const char* what = "conv3d_backward_weight";
  if (!x_shape || !dy_shape || !dw_shape || !args) return fail(B200_ERR_INVALID_ARG, "%s: null shape or args", what);
  const b200_conv3d_args& a = *args;
  const uint64_t N = x_shape[0], C = x_shape[4], Cout = dw_shape[0];
  const uint64_t I[3] = {x_shape[1], x_shape[2], x_shape[3]}, K[3] = {dw_shape[1], dw_shape[2], dw_shape[3]};
  uint64_t O[3] = {0, 0, 0};
  int rc = conv3_check_args(what, in_dtype, out_dtype, a, nullptr, C, dw_shape[4]);
  if (!rc) rc = conv3_check_shape(what, a, x_shape, dw_shape, dy_shape, "dy", O);
  if (!rc && K[0] && K[1] && K[2]) rc = conv3_check_stride(what, a);
  if (rc) return rc;
  const uint64_t KK = K[0] * K[1] * K[2];
  if (Cout == 0 || C == 0 || KK == 0) return B200_OK;   // no dw
  if ((rc = conv3_check_fwd(what, a, dw_shape))) return rc;   // x is read through the forward's map
  const uint64_t P = N * O[0] * O[1] * O[2], lim = 1ull << 31;
  if (P >= lim) return fail(B200_ERR_UNSUPPORTED, "%s: N * OD * OH * OW = %llu must be < 2^31", what, (unsigned long long)P);
  const uint64_t cx = (C + 7) / 8 * 8;
  if (KK * ((cx + 63) / 64 * 64) >= lim) return fail(B200_ERR_UNSUPPORTED, "%s: KD * KH * KW * C (C padded to 64) must be < 2^31", what);
  if ((rc = conv_check_ptrs(what, x, dy, dw, "dw", out_dtype))) return rc;
  const size_t osz = dtype_size(out_dtype);
  uint64_t ds[5], xs[5], ys[5];
  conv3_norm_strides(dw_shape, dw_strides, ds);
  const uint64_t dw_sp = conv3_flat_dhw(dw_shape, ds);
  if (ds[4] != 1 || dw_sp == 0 || ds[0] * osz >= (1ull << 40) || dw_sp * osz >= (1ull << 40))
    return fail(B200_ERR_UNSUPPORTED, "%s: dw must have unit channel stride and (KD, KH, KW) flattening into one stride", what);
  CUstream st = resolve_stream(c, s);
  if (P == 0) {
    // no pixels: dw is exactly zero
    if (ds[0] == KK * dw_sp) return memset2d_zero(c, st, dw, osz, dw_sp, C, Cout * KK);
    for (uint64_t co = 0; co < Cout && !rc; ++co) rc = memset2d_zero(c, st, dw + co * ds[0] * osz, osz, dw_sp, C, KK);
    return rc;
  }
  conv3_norm_strides(x_shape, x_strides, xs);
  conv3_norm_strides(dy_shape, dy_strides, ys);
  CUdeviceptr tmp[4] = {0, 0, 0, 0};
  NdhwcOperand xo{}, yo{};
  rc = conv3_prep(c, st, in_dtype, x, x_shape, xs, kFlatNone, &tmp[0], &xo);
  if (!rc) rc = conv3_prep(c, st, in_dtype, dy, dy_shape, ys, kFlatNHW, &tmp[2], &yo);
  if (!rc) {
    const int32_t sv[3] = {a.stride_d, a.stride_h, a.stride_w}, pv[3] = {a.pad_d, a.pad_h, a.pad_w};
    const int32_t dv[3] = {a.dilation_d, a.dilation_h, a.dilation_w};
    ConvGeom g = conv3_geom(N, I, xo.C, K, O, Cout, sv, pv, dv);
    g.x_sw = xo.s_w; g.x_sh = xo.s_h; g.x_sd = xo.s_d; g.x_sn = xo.s_n;
    g.mode = 2; g.dw_sp = dw_sp; g.dw_c = C;
    GemmProblem gp = conv_problem(in_dtype, out_dtype, yo.ptr, xo.ptr, dw, Cout, KK * ((xo.C + 63) / 64 * 64), P, ds[0], &g);
    gp.a_sm = 1; gp.a_sk = yo.s_w; gp.b_sn = 1; gp.b_sk = xo.s_w;   // both operands MN-major
    gp.sk_max_parts = std::max<uint64_t>(8, (P + 63) / 64 / 8);      // as b200_conv2d_backward_weight
    rc = launch_wgmma(c, st, gp, true, true);
  }
  for (CUdeviceptr t : tmp)
    if (t) pool_free(c, t, st);   // stream-ordered: reusable by later work once the GEMM has drained
  return rc;
}

// ------------------------------------------------------------------------------------------------ transposed convolution
// b200_conv_transpose2d / 3d: the transpose of b200_conv2d / 3d, which is the data gradient's computation with x in dy's
// role and the output in dx's.  The data gradient's phase plan, limits and weight prep are reused as they are; what differs
// is the fused epilogue, that a phase no tap reaches stores act(bias) instead of a memset's zeros, and the strided launch:
// every phase of the layer in one conv2d_tconv_* / conv3d_tconv_* launch (gemm_wgmma.cu: CB_TCONV).

// One output phase: its per-dimension phases (D, H, W; a 2-D layer has a unit depth phase), pixels, k-blocks, the element
// offset of its weight block and the address of its first output pixel.
struct TconvRun {
  const DgradPhase1D* q[3];
  uint64_t M, num_kb, woff, out;
};

// The phase-batched launches of a strided transposed convolution: the runs sorted by k-blocks (most first, ties in phase
// order), kTconvMaxPhases per launch.  x is read through xo (extents X = (D, H, W), 2-D: D = 1), the weight blocks from wbuf
// ([Cout][taps][cp] per phase); dx_s = output strides (n, d, h, w) of one phase's pixel grid, pitch = the output pixel pitch.
static int launch_tconv(b200_ctx* c, CUstream st, int dims, b200_dtype in_dtype, b200_dtype out_dtype, const NdhwcOperand& xo, uint64_t N,
                        const uint64_t X[3], uint64_t Cout, CUdeviceptr wbuf, std::vector<TconvRun> runs, const uint64_t dx_s[4], uint64_t pitch,
                        const b200_epilogue* ep) {
  const size_t osz = dtype_size(out_dtype);
  const uint64_t cp = xo.C, cblk = (cp + 63) / 64;
  std::stable_sort(runs.begin(), runs.end(), [](const TconvRun& a, const TconvRun& b) { return a.num_kb > b.num_kb; });
  // the tile: the GEMM's wave model (whole tiles, no stream-K head) over the layer's pixels and its longest phase
  ConvGeom cg_probe{};
  GemmProblem gp = conv_problem(in_dtype, out_dtype, 0, 0, 0, 0, Cout, std::max<uint64_t>(1, runs[0].num_kb) * 64, pitch, &cg_probe);
  for (const TconvRun& r : runs) gp.M += r.M;
  // gemm.split_k is validated as for every GEMM, though these launches plan no stream-K head (their tiles differ in k-blocks)
  const std::string split_opt = opt(c, "gemm.split_k", "auto");
  const int split_n = atoi(split_opt.c_str());
  if (split_opt != "auto" && split_opt != "off" && split_opt != "on" && (split_n < 1 || split_n > 8))
    return fail(B200_ERR_INVALID_ARG, "gemm.split_k must be auto, off, on or 1..8");
  SkPlan no_sk;
  const GemmVariant* vp = pick_variant(c, gp, &no_sk, false);
  if (!vp) return fail(B200_ERR_INVALID_ARG, "gemm.variant '%s' is not a wgmma variant", opt(c, "gemm.variant", "auto").c_str());
  const GemmVariant& v = *vp;
  const char* io = in_dtype == B200_BF16 ? (out_dtype == B200_F32 ? "bf16_f32_" : "bf16_bf16_") : (out_dtype == B200_F32 ? "f16_f32_" : "f16_f16_");
  CUfunction f;
  int rc = get_func(c, std::string(dims == 3 ? "conv3d_tconv_" : "conv2d_tconv_") + io + v.tag, &f);
  if (rc) return rc;
  const unsigned smem = gemm_smem_bytes(v);
  if (!c->dry) CU_CHECK(g_drv.cuFuncSetAttribute_p(f, CU_FUNC_ATTRIBUTE_MAX_DYNAMIC_SHARED_SIZE_BYTES, (int)smem));
  const CUtensorMapDataType dt = in_dtype == B200_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  const uint64_t tiles_n = (Cout + v.block_n - 1) / v.block_n, rows = 128ull * v.cg;
  static_assert(sizeof(CUtensorMap) == sizeof(TmapBytes), "TmapBytes holds one CUtensorMap");
  for (size_t g0 = 0; g0 < runs.size() && !rc; g0 += kTconvMaxPhases) {
    const size_t nq = std::min<size_t>(kTconvMaxPhases, runs.size() - g0);
    TconvParams tp;
    memset(&tp, 0, sizeof(tp));
    GemmParams p;
    memset(&p, 0, sizeof(p));
    bool vec = (pitch * osz) % 16 == 0;
    for (int i = 0; i < 4; ++i) vec = vec && (dx_s[i] * osz) % 16 == 0;
    uint64_t tiles = 0, pixels = 0;
    for (size_t k = 0; k < nq && !rc; ++k) {
      const TconvRun& r = runs[g0 + k];
      const DgradPhase1D* const* q = r.q;
      TconvPhase& P = tp.ph[k];
      P.out = r.out;
      vec = vec && r.out % 16 == 0;
      P.tile0 = (uint32_t)tiles;
      P.tiles_m = (uint32_t)((r.M + rows - 1) / rows);
      tiles += P.tiles_m * tiles_n;
      pixels += r.M;
      P.M = (uint32_t)r.M; P.num_kb = (uint32_t)r.num_kb;
      P.e_dhw = (uint32_t)(q[0]->extent * q[1]->extent * q[2]->extent); P.e_hw = (uint32_t)(q[1]->extent * q[2]->extent); P.e_w = (uint32_t)q[2]->extent;
      P.t_hw = q[1]->taps * q[2]->taps; P.t_w = q[2]->taps;
      P.lo_d = (int32_t)q[0]->e0; P.lo_h = (int32_t)q[1]->e0; P.lo_w = (int32_t)q[2]->e0;
      P.dil_d = q[0]->dil; P.dil_h = q[1]->dil; P.dil_w = q[2]->dil;
      if (c->dry) {
        const std::string head = dims == 3 ? dgrad3_phase_line("conv3d tconv phase", q, X) : dgrad2_phase_line("conv tconv phase", *q[1], *q[2], X[1], X[2]);
        c->plan += head + " kblocks=" + std::to_string(r.num_kb) + "\n";
      }
      if (!r.num_kb) continue;   // no loads: the maps stay empty
      // x through im2col over the phase's pixel box; the phase's weights as (cp, taps, Cout) in [n_local x 64 channel] boxes
      CUtensorMap am, bm;
      int lo[3], up[3];
      for (int i = 0; i < 3; ++i) {
        lo[2 - i] = (int)q[i]->e0;
        up[2 - i] = (int)(q[i]->e0 + (int64_t)q[i]->extent - (int64_t)X[i]);
      }
      if (dims == 3) {
        const uint64_t d5[5] = {cp, X[2], X[1], X[0], N}, s4[4] = {xo.s_w, xo.s_h, xo.s_d, xo.s_n};
        const uint32_t one[3] = {1, 1, 1};
        rc = encode_im2col5(c, &am, dt, 2, xo.ptr, d5, s4, lo, up, 64, 128, one);
      } else {
        const uint64_t d4[4] = {cp, X[2], X[1], N}, s3[3] = {xo.s_w, xo.s_h, xo.s_n};
        rc = encode_im2col(c, &am, dt, 2, xo.ptr, d4, s3, lo, up, 64, 128, 1, 1);
      }
      const uint64_t taps = (uint64_t)q[0]->taps * q[1]->taps * q[2]->taps;
      if (!rc) rc = encode_tmap(c, &bm, dt, 2, wbuf + r.woff * 2, cp, taps, Cout, cp, taps * cp, 64, 1, CU_TENSOR_MAP_SWIZZLE_128B, (uint32_t)(v.block_n / v.cg));
      memcpy(&tp.a[k], &am, sizeof(am));
      memcpy(&tp.b[k], &bm, sizeof(bm));
    }
    if (rc) break;
    if (tiles >= (1ull << 32)) return fail(B200_ERR_UNSUPPORTED, "too many tiles");
    tp.phases = (uint32_t)nq;
    p.out = runs[g0].out;
    p.out_row_stride = pitch;
    p.M = (uint32_t)pixels; p.N = (uint32_t)Cout; p.K = 0; p.batch = 1;
    p.tiles_n = (uint32_t)tiles_n;
    p.group_m = (uint32_t)std::max(1, atoi(opt(c, "gemm.group_m", "8").c_str()));
    p.k_segments = 1;
    p.vec_store = vec ? 1 : 0;
    p.cv_cblk = (uint32_t)cblk;
    p.dx_sn = dx_s[0]; p.dx_sd = dx_s[1]; p.dx_si = dx_s[2]; p.dx_sj = dx_s[3];
    if (ep) { p.alpha = ep->alpha; p.bias = ep->bias; p.epi_act = (uint32_t)ep->activation; }
    else p.alpha = 1.0f;
    p.epi_on = (p.alpha != 1.0f || p.bias != 0 || p.epi_act != 0) ? 1u : 0u;
    p.full_tiles = (uint32_t)tiles;   // whole tiles only: no stream-K head
    const unsigned clusters = (unsigned)std::min<uint64_t>(tiles, (uint64_t)std::max(1, c->props.num_sms / v.cg));
    void* args[] = {&tp, &p};
    rc = launch(c, f, clusters * v.cg, 1, 1, 384, smem, v.cg, st, args);
  }
  return rc;
}

// output_padding = the output extent past the one the conv rule maps back to x's extent; PyTorch also accepts
// stride <= op < dilation, which this entry point refuses (the conv rule cannot map such an output back to x).
static int tconv_check_output_padding(const char* what, uint64_t xi, uint64_t oi, int64_t s, int64_t p, int64_t d, uint64_t k) {
  if (k == 0 || xi == 0) return B200_OK;
  const int64_t op = (int64_t)oi - (((int64_t)xi - 1) * s - 2 * p + d * ((int64_t)k - 1) + 1);
  if (op >= s && op < std::max(s, d))
    return fail(B200_ERR_UNSUPPORTED, "%s: output_padding %lld >= stride %lld is not supported", what, (long long)op, (long long)s);
  return B200_OK;
}

// An empty kernel (some extent 0), which the convolution's output rule does not cover: x [N, *X, Cin] and out [N, *O, C] with
// w [Cin, *K, C], and per dimension O = (X - 1) * s - 2 * p + d * (K - 1) + op + 1 with 0 <= op < s.  The sum is empty, so
// out is act(bias).  rank 4 or 5.
static int tconv_check_empty_kernel(const char* what, int rank, const uint64_t* x, const uint64_t* w, const uint64_t* out,
                                    const int64_t* s, const int64_t* p, const int64_t* d) {
  const int n = rank - 2;
  bool ok = x[0] == out[0] && x[rank - 1] == w[0] && w[rank - 1] == out[rank - 1];
  for (int i = 0; i < n && ok; ++i) {
    const int64_t op = (int64_t)out[1 + i] - (((int64_t)x[1 + i] - 1) * s[i] - 2 * p[i] + d[i] * ((int64_t)w[1 + i] - 1) + 1);
    ok = op >= 0 && op < s[i];
  }
  if (!ok) return fail(B200_ERR_INVALID_ARG, "%s: with an empty kernel, out must be x's batch and the transposed output rule's extents", what);
  return B200_OK;
}

extern "C" int b200_conv_transpose2d(b200_ctx* c, b200_stream s, b200_dtype in_dtype, b200_dtype out_dtype, b200_dptr x,
                                     const uint64_t* x_shape, const uint64_t* x_strides, b200_dptr w, const uint64_t* w_shape,
                                     const uint64_t* w_strides, b200_dptr out, const uint64_t* out_shape, const uint64_t* out_strides,
                                     const b200_conv2d_args* args, const b200_epilogue* ep) {
  CTX_ENTER(c);
  const char* what = "conv_transpose2d";
  if (!x_shape || !w_shape || !out_shape || !args) return fail(B200_ERR_INVALID_ARG, "%s: null shape or args", what);
  const b200_conv2d_args& a = *args;
  // the data gradient's names: dy = x [N, OH, OW, Cin], w [Cin, KH, KW, C], dx = out [N, H, W, C]
  const uint64_t N = out_shape[0], H = out_shape[1], W = out_shape[2], C = out_shape[3];
  const uint64_t Cin = w_shape[0], KH = w_shape[1], KW = w_shape[2];
  uint64_t OH = 0, OW = 0;
  int rc = conv_check_args(what, in_dtype, out_dtype, a, ep, C, w_shape[3]);
  if (!rc) rc = tconv_check_output_padding(what, x_shape[1], H, a.stride_h, a.pad_h, a.dilation_h, KH);
  if (!rc) rc = tconv_check_output_padding(what, x_shape[2], W, a.stride_w, a.pad_w, a.dilation_w, KW);
  if (!rc) rc = conv_check_shape(what, a, out_shape, w_shape, x_shape, "x", &OH, &OW);
  if (!rc && (KH == 0 || KW == 0)) {
    const int64_t sv[2] = {a.stride_h, a.stride_w}, pv[2] = {a.pad_h, a.pad_w}, dv[2] = {a.dilation_h, a.dilation_w};
    rc = tconv_check_empty_kernel(what, 4, x_shape, w_shape, out_shape, sv, pv, dv);
    OH = x_shape[1]; OW = x_shape[2];
  }
  if (!rc) rc = conv_check_stride(what, a);   // whatever the kernel: it also bounds the phases per dimension
  if (rc) return rc;
  if (N == 0 || H == 0 || W == 0 || C == 0) return B200_OK;   // no output
  const uint64_t lim = 1ull << 31;
  if (N * H * W >= lim) return fail(B200_ERR_UNSUPPORTED, "%s: N * OH * OW = %llu must be < 2^31", what, (unsigned long long)(N * H * W));
  if (KH * KW * ((Cin + 63) / 64 * 64) >= lim) return fail(B200_ERR_UNSUPPORTED, "%s: KH * KW * Cin (Cin padded to 64) must be < 2^31", what);
  std::vector<DgradPhase1D> phs, pws;
  bool zero_phase = false;
  if ((rc = dgrad2_plan(what, a, H, W, KH, KW, OH, OW, Cin, &phs, &pws, &zero_phase))) return rc;
  if ((rc = conv_check_ptrs(what, x, w, out, "output", out_dtype))) return rc;
  const size_t osz = dtype_size(out_dtype);
  uint64_t os[4], xs[4], ws[4];
  conv_norm_strides(out_shape, out_strides, os);
  if ((rc = conv_check_pixels(what, "out", out_shape, os))) return rc;
  CUstream st = resolve_stream(c, s);
  const bool taps = Cin != 0 && KH != 0 && KW != 0;
  conv_norm_strides(x_shape, x_strides, xs);
  conv_norm_strides(w_shape, w_strides, ws);
  CUdeviceptr tmp[3] = {0, 0, 0};
  NhwcOperand y{};
  ConvDgradWeightsParams wp;
  memset(&wp, 0, sizeof(wp));
  if (taps) {
    rc = conv_prep_nhwc(c, st, in_dtype, x, x_shape, xs, kFlatNone, tmp, &y);
    if (!rc) rc = dgrad2_prep(c, st, w, ws, a, C, Cin, y.C, KH, KW, phs, pws, &tmp[2], &wp);
  }
  if (!rc && taps && a.stride_h == 1 && a.stride_w == 1) {
    // one phase with every tap: the forward convolution kernel with the epilogue
    const DgradPhase1D &ph = phs[0], &pw = pws[0];
    ConvGeom g = dgrad2_geom(N, OH, OW, y.C, C, ph, pw, y, os, a);
    if (c->dry) c->plan += dgrad2_phase_line("conv tconv phase", ph, pw, OH, OW) + " kblocks=" +
                           std::to_string((uint64_t)ph.taps * pw.taps * ((y.C + 63) / 64)) + "\n";
    GemmProblem gp = conv_problem(in_dtype, out_dtype, y.ptr, tmp[2], out, N * H * W, C, KH * KW * ((y.C + 63) / 64 * 64), os[2], &g);
    if (ep) { gp.alpha = ep->alpha; gp.bias = ep->bias; gp.act = (uint32_t)ep->activation; }
    rc = launch_wgmma(c, st, gp, false, false);
  } else if (!rc) {
    // every phase with pixels, those no tap reaches included, in phase-batched launches
    static const DgradPhase1D unit = {0, 1, 0, 0, 1, 1, 1};
    std::vector<TconvRun> runs;
    const uint64_t cblk = taps ? (y.C + 63) / 64 : 0;
    for (const DgradPhase1D& ph : phs)
      for (const DgradPhase1D& pw : pws) {
        if (!ph.extent || !pw.extent) continue;
        TconvRun r{{&unit, &ph, &pw}, N * ph.extent * pw.extent, (uint64_t)ph.taps * pw.taps * cblk,
                   taps ? wp.off[ph.r * a.stride_w + pw.r] : 0, out + ((uint64_t)ph.r * os[1] + (uint64_t)pw.r * os[2]) * osz};
        runs.push_back(r);
      }
    if (!taps) y = NhwcOperand{0, 8, 8, 8, 8};
    const uint64_t X[3] = {1, OH, OW};
    const uint64_t dx_s[4] = {os[0], 0, (uint64_t)a.stride_h * os[1], (uint64_t)a.stride_w * os[2]};
    const NdhwcOperand xo{y.ptr, y.C, y.s_w, y.s_h, 0, y.s_n};
    rc = launch_tconv(c, st, 2, in_dtype, out_dtype, xo, N, X, C, tmp[2], runs, dx_s, os[2], ep);
  }
  for (CUdeviceptr t : tmp)
    if (t) pool_free(c, t, st);   // stream-ordered: reusable by later work once the GEMMs have drained
  return rc;
}

extern "C" int b200_conv_transpose3d(b200_ctx* c, b200_stream s, b200_dtype in_dtype, b200_dtype out_dtype, b200_dptr x,
                                     const uint64_t* x_shape, const uint64_t* x_strides, b200_dptr w, const uint64_t* w_shape,
                                     const uint64_t* w_strides, b200_dptr out, const uint64_t* out_shape, const uint64_t* out_strides,
                                     const b200_conv3d_args* args, const b200_epilogue* ep) {
  CTX_ENTER(c);
  const char* what = "conv_transpose3d";
  if (!x_shape || !w_shape || !out_shape || !args) return fail(B200_ERR_INVALID_ARG, "%s: null shape or args", what);
  const b200_conv3d_args& a = *args;
  // the data gradient's names: dy = x [N, OD, OH, OW, Cin], w [Cin, KD, KH, KW, C], dx = out [N, D, H, W, C]
  const uint64_t N = out_shape[0], C = out_shape[4], Cin = w_shape[0];
  const uint64_t I[3] = {out_shape[1], out_shape[2], out_shape[3]}, K[3] = {w_shape[1], w_shape[2], w_shape[3]};
  const int64_t sv[3] = {a.stride_d, a.stride_h, a.stride_w}, pv[3] = {a.pad_d, a.pad_h, a.pad_w};
  const int64_t dv[3] = {a.dilation_d, a.dilation_h, a.dilation_w};
  uint64_t O[3] = {0, 0, 0};
  int rc = conv3_check_args(what, in_dtype, out_dtype, a, ep, C, w_shape[4]);
  for (int i = 0; i < 3 && !rc; ++i) rc = tconv_check_output_padding(what, x_shape[1 + i], I[i], sv[i], pv[i], dv[i], K[i]);
  if (!rc) rc = conv3_check_shape(what, a, out_shape, w_shape, x_shape, "x", O);
  if (!rc && (K[0] == 0 || K[1] == 0 || K[2] == 0)) {
    rc = tconv_check_empty_kernel(what, 5, x_shape, w_shape, out_shape, sv, pv, dv);
    for (int i = 0; i < 3; ++i) O[i] = x_shape[1 + i];
  }
  if (!rc) rc = conv3_check_stride(what, a);   // whatever the kernel: it also bounds the phases per dimension (Dgrad3Prep)
  if (rc) return rc;
  if (N == 0 || I[0] == 0 || I[1] == 0 || I[2] == 0 || C == 0) return B200_OK;   // no output
  const uint64_t lim = 1ull << 31, P = N * I[0] * I[1] * I[2], KK = K[0] * K[1] * K[2];
  if (P >= lim) return fail(B200_ERR_UNSUPPORTED, "%s: N * OD * OH * OW = %llu must be < 2^31", what, (unsigned long long)P);
  if (KK * ((Cin + 63) / 64 * 64) >= lim)
    return fail(B200_ERR_UNSUPPORTED, "%s: KD * KH * KW * Cin (Cin padded to 64) must be < 2^31", what);
  std::vector<DgradPhase1D> ph[3];
  bool zero_phase = false;
  if ((rc = dgrad3_plan(what, sv, pv, dv, I, K, O, Cin, ph, &zero_phase))) return rc;
  if ((rc = conv_check_ptrs(what, x, w, out, "output", out_dtype))) return rc;
  const size_t osz = dtype_size(out_dtype);
  uint64_t os[5], xs[5], ws[5];
  conv3_norm_strides(out_shape, out_strides, os);
  if ((rc = conv3_check_pixels(what, "out", out_shape, os))) return rc;
  CUstream st = resolve_stream(c, s);
  const bool taps = Cin != 0 && KK != 0;
  conv3_norm_strides(x_shape, x_strides, xs);
  conv3_norm_strides(w_shape, w_strides, ws);
  CUdeviceptr tmp[3] = {0, 0, 0};
  NdhwcOperand y{};
  // the weight prep (and its per-phase offsets) only when some phase has taps
  std::unique_ptr<Dgrad3Prep> prep;
  if (taps) {
    rc = conv3_prep(c, st, in_dtype, x, x_shape, xs, kFlatNone, tmp, &y);
    prep.reset(new Dgrad3Prep(ph, K, sv, pv, dv, C, y.C));
    if (!rc) rc = dgrad3_prep(c, st, w, ws, Cin, KK, prep.get(), &tmp[2]);
  }
  if (!rc && taps && sv[0] == 1 && sv[1] == 1 && sv[2] == 1) {
    const DgradPhase1D* q[3] = {&ph[0][0], &ph[1][0], &ph[2][0]};
    ConvGeom g = dgrad3_geom(N, O, y.C, C, q, y, os, sv);
    if (c->dry) c->plan += dgrad3_phase_line("conv3d tconv phase", q, O) + " kblocks=" + std::to_string(KK * ((y.C + 63) / 64)) + "\n";
    GemmProblem gp = conv_problem(in_dtype, out_dtype, y.ptr, tmp[2], out, P, C, KK * ((y.C + 63) / 64 * 64), os[3], &g);
    if (ep) { gp.alpha = ep->alpha; gp.bias = ep->bias; gp.act = (uint32_t)ep->activation; }
    rc = launch_wgmma(c, st, gp, false, false);
  } else if (!rc) {
    std::vector<TconvRun> runs;
    const uint64_t cblk = taps ? (y.C + 63) / 64 : 0;
    for (const DgradPhase1D& pd : ph[0])
      for (const DgradPhase1D& phh : ph[1])
        for (const DgradPhase1D& pw : ph[2]) {
          if (!pd.extent || !phh.extent || !pw.extent) continue;
          TconvRun r{{&pd, &phh, &pw}, N * pd.extent * phh.extent * pw.extent, (uint64_t)pd.taps * phh.taps * pw.taps * cblk,
                     taps ? prep->off(pd.r, phh.r, pw.r) : 0,
                     out + ((uint64_t)pd.r * os[1] + (uint64_t)phh.r * os[2] + (uint64_t)pw.r * os[3]) * osz};
          runs.push_back(r);
        }
    if (!taps) y = NdhwcOperand{0, 8, 8, 8, 8, 8};
    const uint64_t dx_s[4] = {os[0], (uint64_t)sv[0] * os[1], (uint64_t)sv[1] * os[2], (uint64_t)sv[2] * os[3]};
    rc = launch_tconv(c, st, 3, in_dtype, out_dtype, y, N, O, C, tmp[2], runs, dx_s, os[3], ep);
  }
  for (CUdeviceptr t : tmp)
    if (t) pool_free(c, t, st);   // stream-ordered: reusable by later work once the GEMMs have drained
  return rc;
}

// ------------------------------------------------------------------------------------------------ grouped convolution
// Routing, from the shape alone: groups == 1 is the plain entry point; a group width Cg = C / groups of at least one
// k-block (64 channels) runs one implicit GEMM per group on channel slices; narrower groups run the direct kernels of
// conv_grouped.cu, for which the GEMM route would multiply mostly zero-padded k-blocks.  The direct route applies the same
// checks as the GEMM route, so both accept the same shapes.
constexpr uint64_t kGrpGemmMinCg = 64;

static int grp_check(const char* what, uint32_t groups, uint64_t C, uint64_t Cout, uint64_t w_c) {
  if (groups == 0) return fail(B200_ERR_INVALID_ARG, "%s: groups must be >= 1", what);
  if (C % groups || Cout % groups)
    return fail(B200_ERR_INVALID_ARG, "%s: groups = %u must divide C = %llu and Cout = %llu", what, groups, (unsigned long long)C,
                (unsigned long long)Cout);
  if (w_c != C / groups)
    return fail(B200_ERR_INVALID_ARG, "%s: weights have %llu channels, C / groups = %llu", what, (unsigned long long)w_c,
                (unsigned long long)(C / groups));
  return B200_OK;
}

// The parameter fields every direct kernel reads: the input [N, H, W, C], the output extents, the weights [Cout, KH, KW, *],
// groups and args; the rest is zero.
static ConvGroupedParams grp_params(const uint64_t* in, uint64_t OH, uint64_t OW, const uint64_t* w, uint32_t groups, const b200_conv2d_args& a) {
  ConvGroupedParams p;
  memset(&p, 0, sizeof(p));
  p.N = (uint32_t)in[0]; p.H = (uint32_t)in[1]; p.W = (uint32_t)in[2]; p.C = (uint32_t)in[3]; p.OH = (uint32_t)OH; p.OW = (uint32_t)OW;
  p.Cout = (uint32_t)w[0]; p.KH = (uint32_t)w[1]; p.KW = (uint32_t)w[2]; p.Cg = (uint32_t)(in[3] / groups); p.Coutg = (uint32_t)(w[0] / groups);
  p.sh = a.stride_h; p.sw = a.stride_w; p.ph = a.pad_h; p.pw = a.pad_w; p.dh = a.dilation_h; p.dw = a.dilation_w;
  return p;
}

// A rank-4 operand the direct kernels read through its strides: kept in place with a unit channel stride, else gathered
// into a compact pooled copy (*tmp, freed by the caller).  s: the strides to read it with.
static int grp_operand(b200_ctx* c, CUstream st, b200_dtype dt, uint64_t ptr, const uint64_t* shape, const uint64_t* ns,
                       CUdeviceptr* tmp, uint64_t* out, uint64_t s[4]) {
  if (ns[3] == 1) {
    *out = ptr;
    for (int d = 0; d < 4; ++d) s[d] = ns[d];
    return B200_OK;
  }
  int rc = conv_gather(c, st, dt, ptr, shape, ns, tmp);
  *out = *tmp;
  s[3] = 1; s[2] = shape[3]; s[1] = shape[2] * shape[3]; s[0] = shape[1] * shape[2] * shape[3];
  return rc;
}

static const char* grp_tag(b200_dtype dt) { return dt == B200_BF16 ? "bf16" : dt == B200_F16 ? "f16" : "f32"; }

extern "C" int b200_conv2d_grouped(b200_ctx* c, b200_stream s, b200_dtype in_dtype, b200_dtype out_dtype, b200_dptr x,
                                   const uint64_t* x_shape, const uint64_t* x_strides, b200_dptr w, const uint64_t* w_shape,
                                   const uint64_t* w_strides, b200_dptr out, const uint64_t* out_shape, const uint64_t* out_strides,
                                   const b200_conv2d_args* args, uint32_t groups, const b200_epilogue* ep) {
  CTX_ENTER(c);
  const char* what = "conv2d_grouped";
  if (!x_shape || !w_shape || !out_shape || !args) return fail(B200_ERR_INVALID_ARG, "%s: null shape or args", what);
  if (groups == 1)
    return b200_conv2d(c, s, in_dtype, out_dtype, x, x_shape, x_strides, w, w_shape, w_strides, out, out_shape, out_strides, args, ep);
  const b200_conv2d_args& a = *args;
  const uint64_t N = x_shape[0], H = x_shape[1], W = x_shape[2], C = x_shape[3];
  const uint64_t Cout = w_shape[0], KH = w_shape[1], KW = w_shape[2];
  int rc = grp_check(what, groups, C, Cout, w_shape[3]);
  if (!rc) rc = conv_check_args(what, in_dtype, out_dtype, a, ep, C / groups, w_shape[3]);
  if (rc) return rc;
  if (N == 0 || H == 0 || W == 0 || C == 0 || Cout == 0 || KH == 0 || KW == 0) return B200_OK;
  uint64_t OH = 0, OW = 0;
  if ((rc = conv_check_shape(what, a, x_shape, w_shape, out_shape, "out", &OH, &OW))) return rc;
  if ((rc = conv_check_ptrs(what, x, w, out, "output", out_dtype))) return rc;
  const size_t osz = dtype_size(out_dtype);
  const uint64_t Cg = C / groups, Coutg = Cout / groups;
  uint64_t xs[4], ws[4], os[4];
  conv_norm_strides(x_shape, x_strides, xs);
  conv_norm_strides(w_shape, w_strides, ws);
  conv_norm_strides(out_shape, out_strides, os);
  if (Cg >= kGrpGemmMinCg) {
    // one b200_conv2d per group: x, w and out are read and written in place through channel slices
    const uint64_t sx[4] = {N, H, W, Cg}, sw[4] = {Coutg, KH, KW, Cg}, so[4] = {N, OH, OW, Coutg};
    for (uint64_t g = 0; g < groups && !rc; ++g) {
      b200_epilogue eg{};
      if (ep) {
        eg = *ep;
        if (eg.bias) eg.bias += g * Coutg * 4;
      }
      rc = b200_conv2d(c, s, in_dtype, out_dtype, x + g * Cg * xs[3] * 2, sx, xs, w + g * Coutg * ws[0] * 2, sw, ws,
                       out + g * Coutg * os[3] * osz, so, os, args, ep ? &eg : nullptr);
    }
    return rc;
  }
  if ((rc = conv_check_fwd_corners(what, a, KH, KW)) || (rc = conv_check_stride(what, a))) return rc;
  const uint64_t lim = 1ull << 31;
  if (N * OH * OW >= lim) return fail(B200_ERR_UNSUPPORTED, "%s: N * OH * OW = %llu must be < 2^31", what, (unsigned long long)(N * OH * OW));
  if ((rc = conv_check_pixels(what, "out", out_shape, os))) return rc;
  const uint64_t tiles_h = (OH + kGrpTileH - 1) / kGrpTileH, tiles_w = (OW + kGrpTileW - 1) / kGrpTileW;
  const uint64_t chunks = (Cout + kGrpChunk - 1) / kGrpChunk;
  if (N * tiles_h * tiles_w >= lim || chunks > 65535)
    return fail(B200_ERR_UNSUPPORTED, "%s: too many output tiles (N * ceil(OH / 8) * ceil(OW / 8) < 2^31, Cout <= 2^21)", what);
  CUstream st = resolve_stream(c, s);
  CUdeviceptr tmp[2] = {0, 0};
  ConvGroupedParams p = grp_params(x_shape, OH, OW, w_shape, groups, a);
  uint64_t xsr[4], wsr[4];
  rc = grp_operand(c, st, in_dtype, x, x_shape, xs, &tmp[0], &p.x, xsr);
  if (!rc) rc = grp_operand(c, st, in_dtype, w, w_shape, ws, &tmp[1], &p.w, wsr);
  if (!rc) {
    p.out = out;
    p.x_sn = xsr[0]; p.x_sh = xsr[1]; p.x_sw = xsr[2];
    p.w_sco = wsr[0]; p.w_sky = wsr[1]; p.w_skx = wsr[2];
    p.o_sn = os[0]; p.o_sh = os[1]; p.o_sw = os[2];
    p.tiles_h = (uint32_t)tiles_h; p.tiles_w = (uint32_t)tiles_w;
    p.vec_x = (p.x % 16 == 0 && xsr[0] % 8 == 0 && xsr[1] % 8 == 0 && xsr[2] % 8 == 0) ? 1u : 0u;
    if (ep) {
      p.alpha = ep->alpha; p.bias = ep->bias; p.epi_act = (uint32_t)ep->activation;
    } else {
      p.alpha = 1.0f;
    }
    p.epi_on = (p.alpha != 1.0f || p.bias != 0 || p.epi_act != 0) ? 1u : 0u;
    // the input channels one chunk of kGrpChunk output channels reads, at most; the halo is staged when it fits
    uint64_t span = 0;
    for (uint64_t co0 = 0; co0 < Cout; co0 += kGrpChunk) {
      const uint64_t co_end = std::min<uint64_t>(co0 + kGrpChunk, Cout);
      span = std::max(span, std::min(C, ((co_end - 1) / Coutg + 1) * Cg) - (co0 / Coutg) * Cg);
    }
    const uint64_t pitch = (span + 7) / 8 * 8;
    const uint64_t hh = (kGrpTileH - 1) * (uint64_t)a.stride_h + (KH - 1) * (uint64_t)a.dilation_h + 1;
    const uint64_t hw = (kGrpTileW - 1) * (uint64_t)a.stride_w + (KW - 1) * (uint64_t)a.dilation_w + 1;
    const uint64_t smem = hh * hw * pitch * 2;
    p.staged_ci = smem <= (uint64_t)kGrpSmemMax ? (uint32_t)pitch : 0u;
    CUfunction f;
    rc = get_func(c, std::string("conv2d_grp_") + grp_tag(in_dtype) + "_" + grp_tag(out_dtype), &f);
    void* kargs[] = {&p};
    if (!rc) rc = launch(c, f, (unsigned)(N * tiles_h * tiles_w), (unsigned)chunks, 1, 256, p.staged_ci ? (unsigned)smem : 0u, 1, st, kargs);
  }
  for (CUdeviceptr t : tmp)
    if (t) pool_free(c, t, st);
  return rc;
}

extern "C" int b200_conv2d_grouped_backward_data(b200_ctx* c, b200_stream s, b200_dtype in_dtype, b200_dtype out_dtype, b200_dptr dy,
                                                 const uint64_t* dy_shape, const uint64_t* dy_strides, b200_dptr w,
                                                 const uint64_t* w_shape, const uint64_t* w_strides, b200_dptr dx,
                                                 const uint64_t* dx_shape, const uint64_t* dx_strides, const b200_conv2d_args* args,
                                                 uint32_t groups) {
  CTX_ENTER(c);
  const char* what = "conv2d_grouped_backward_data";
  if (!dy_shape || !w_shape || !dx_shape || !args) return fail(B200_ERR_INVALID_ARG, "%s: null shape or args", what);
  if (groups == 1)
    return b200_conv2d_backward_data(c, s, in_dtype, out_dtype, dy, dy_shape, dy_strides, w, w_shape, w_strides, dx, dx_shape, dx_strides, args);
  const b200_conv2d_args& a = *args;
  const uint64_t N = dx_shape[0], H = dx_shape[1], W = dx_shape[2], C = dx_shape[3];
  const uint64_t Cout = w_shape[0], KH = w_shape[1], KW = w_shape[2];
  uint64_t OH = 0, OW = 0;
  int rc = grp_check(what, groups, C, Cout, w_shape[3]);
  if (!rc) rc = conv_check_args(what, in_dtype, out_dtype, a, nullptr, C / groups, w_shape[3]);
  if (!rc) rc = conv_check_shape(what, a, dx_shape, w_shape, dy_shape, "dy", &OH, &OW);
  if (!rc && KH && KW) rc = conv_check_stride(what, a);
  if (rc) return rc;
  if (N == 0 || H == 0 || W == 0 || C == 0) return B200_OK;   // no dx
  if ((rc = conv_check_ptrs(what, dy, w, dx, "dx", out_dtype))) return rc;
  const size_t osz = dtype_size(out_dtype);
  const uint64_t Cg = C / groups, Coutg = Cout / groups;
  uint64_t ys[4], ws[4], os[4];
  conv_norm_strides(dy_shape, dy_strides, ys);
  conv_norm_strides(w_shape, w_strides, ws);
  conv_norm_strides(dx_shape, dx_strides, os);
  if (Cg >= kGrpGemmMinCg) {
    const uint64_t sy[4] = {N, OH, OW, Coutg}, sw[4] = {Coutg, KH, KW, Cg}, sx[4] = {N, H, W, Cg};
    for (uint64_t g = 0; g < groups && !rc; ++g)
      rc = b200_conv2d_backward_data(c, s, in_dtype, out_dtype, dy + g * Coutg * ys[3] * 2, sy, ys, w + g * Coutg * ws[0] * 2, sw, ws,
                                     dx + g * Cg * os[3] * osz, sx, os, args);
    return rc;
  }
  if (KH && KW && (rc = conv_check_fwd_corners(what, a, KH, KW))) return rc;
  const uint64_t lim = 1ull << 31;
  if (N * H * W >= lim) return fail(B200_ERR_UNSUPPORTED, "%s: N * H * W = %llu must be < 2^31", what, (unsigned long long)(N * H * W));
  if ((rc = conv_check_pixels(what, "dx", dx_shape, os))) return rc;
  const uint64_t chunks = (C + kGrpChunk - 1) / kGrpChunk;
  if (chunks > 65535) return fail(B200_ERR_UNSUPPORTED, "%s: C must be <= 2^21", what);
  CUstream st = resolve_stream(c, s);
  CUdeviceptr tmp[2] = {0, 0};
  ConvGroupedParams p = grp_params(dx_shape, OH, OW, w_shape, groups, a);
  uint64_t ysr[4] = {0, 0, 0, 1}, wsr[4] = {0, 0, 0, 1};
  // an empty dy or kernel reads nothing: dx comes out as +0 from the same launch
  if (Cout && KH && KW) {
    rc = grp_operand(c, st, in_dtype, dy, dy_shape, ys, &tmp[0], &p.x, ysr);
    if (!rc) rc = grp_operand(c, st, in_dtype, w, w_shape, ws, &tmp[1], &p.w, wsr);
  }
  if (!rc) {
    p.out = dx;
    p.x_sn = ysr[0]; p.x_sh = ysr[1]; p.x_sw = ysr[2];
    p.w_sco = wsr[0]; p.w_sky = wsr[1]; p.w_skx = wsr[2];
    p.o_sn = os[0]; p.o_sh = os[1]; p.o_sw = os[2];
    CUfunction f;
    rc = get_func(c, std::string("conv2d_grp_dgrad_") + grp_tag(in_dtype) + "_" + grp_tag(out_dtype), &f);
    void* kargs[] = {&p};
    if (!rc) rc = launch(c, f, (unsigned)((N * H * W + 7) / 8), (unsigned)chunks, 1, 256, 0, 1, st, kargs);
  }
  for (CUdeviceptr t : tmp)
    if (t) pool_free(c, t, st);
  return rc;
}

// Segments of the weight gradient's pixel sum, a function of the shape only: enough (elements x segments) threads to fill
// the GPU (2^18, at most 4096 segments), each segment at least 64 pixels.
static void grp_wgrad_segments(uint64_t P, uint64_t elems, uint64_t* seg_len, uint64_t* nseg) {
  const uint64_t want = std::min<uint64_t>(4096, std::max<uint64_t>(1, ((1ull << 18) + elems - 1) / elems));
  *seg_len = std::max<uint64_t>(64, (P + want - 1) / want);
  *nseg = P ? (P + *seg_len - 1) / *seg_len : 1;
}

extern "C" int b200_conv2d_grouped_backward_weight(b200_ctx* c, b200_stream s, b200_dtype in_dtype, b200_dtype out_dtype, b200_dptr x,
                                                   const uint64_t* x_shape, const uint64_t* x_strides, b200_dptr dy,
                                                   const uint64_t* dy_shape, const uint64_t* dy_strides, b200_dptr dw,
                                                   const uint64_t* dw_shape, const uint64_t* dw_strides, const b200_conv2d_args* args,
                                                   uint32_t groups) {
  CTX_ENTER(c);
  const char* what = "conv2d_grouped_backward_weight";
  if (!x_shape || !dy_shape || !dw_shape || !args) return fail(B200_ERR_INVALID_ARG, "%s: null shape or args", what);
  if (groups == 1)
    return b200_conv2d_backward_weight(c, s, in_dtype, out_dtype, x, x_shape, x_strides, dy, dy_shape, dy_strides, dw, dw_shape, dw_strides,
                                       args);
  const b200_conv2d_args& a = *args;
  const uint64_t N = x_shape[0], H = x_shape[1], W = x_shape[2], C = x_shape[3];
  const uint64_t Cout = dw_shape[0], KH = dw_shape[1], KW = dw_shape[2];
  uint64_t OH = 0, OW = 0;
  int rc = grp_check(what, groups, C, Cout, dw_shape[3]);
  if (!rc) rc = conv_check_args(what, in_dtype, out_dtype, a, nullptr, C / groups, dw_shape[3]);
  if (!rc) rc = conv_check_shape(what, a, x_shape, dw_shape, dy_shape, "dy", &OH, &OW);
  if (!rc && KH && KW) rc = conv_check_stride(what, a);
  if (rc) return rc;
  if (Cout == 0 || C == 0 || KH == 0 || KW == 0) return B200_OK;   // no dw
  if ((rc = conv_check_fwd_corners(what, a, KH, KW))) return rc;
  const uint64_t P = N * OH * OW, lim = 1ull << 31;
  if (P >= lim) return fail(B200_ERR_UNSUPPORTED, "%s: N * OH * OW = %llu must be < 2^31", what, (unsigned long long)P);
  if ((rc = conv_check_ptrs(what, x, dy, dw, "dw", out_dtype))) return rc;
  const size_t osz = dtype_size(out_dtype);
  const uint64_t Cg = C / groups, Coutg = Cout / groups;
  uint64_t xs[4], ys[4], ds[4];
  conv_norm_strides(x_shape, x_strides, xs);
  conv_norm_strides(dy_shape, dy_strides, ys);
  conv_norm_strides(dw_shape, dw_strides, ds);
  if (Cg >= kGrpGemmMinCg) {
    const uint64_t sx[4] = {N, H, W, Cg}, sy[4] = {N, OH, OW, Coutg}, sw[4] = {Coutg, KH, KW, Cg};
    for (uint64_t g = 0; g < groups && !rc; ++g)
      rc = b200_conv2d_backward_weight(c, s, in_dtype, out_dtype, x + g * Cg * xs[3] * 2, sx, xs, dy + g * Coutg * ys[3] * 2, sy, ys,
                                       dw + g * Coutg * ds[0] * osz, sw, ds, args);
    return rc;
  }
  uint64_t dw_sp = 0;
  if ((rc = conv_check_dw(what, dw_shape, ds, osz, &dw_sp))) return rc;
  const uint64_t elems = Cout * KH * KW * Cg;
  if (elems >= lim) return fail(B200_ERR_UNSUPPORTED, "%s: Cout * KH * KW * C / groups = %llu must be < 2^31", what, (unsigned long long)elems);
  uint64_t seg_len = 0, nseg = 0;
  grp_wgrad_segments(P, elems, &seg_len, &nseg);
  if (c->dry) {
    char line[160];
    snprintf(line, sizeof(line), "conv grouped wgrad pixels=%llu elements=%llu segments=%llu length=%llu\n", (unsigned long long)P,
             (unsigned long long)elems, (unsigned long long)nseg, (unsigned long long)seg_len);
    c->plan += line;
  }
  CUstream st = resolve_stream(c, s);
  CUdeviceptr tmp[3] = {0, 0, 0};
  ConvGroupedParams p = grp_params(x_shape, OH, OW, dw_shape, groups, a);
  uint64_t xsr[4], ysr[4];
  rc = grp_operand(c, st, in_dtype, x, x_shape, xs, &tmp[0], &p.x, xsr);
  if (!rc) rc = grp_operand(c, st, in_dtype, dy, dy_shape, ys, &tmp[1], &p.w, ysr);
  if (!rc && nseg > 1) rc = pool_alloc(c, nseg * elems * 4, &tmp[2], st);
  if (!rc) {
    p.out = dw; p.part = tmp[2];
    p.x_sn = xsr[0]; p.x_sh = xsr[1]; p.x_sw = xsr[2];
    p.y_sn = ysr[0]; p.y_sh = ysr[1]; p.y_sw = ysr[2];
    p.o_sn = ds[0]; p.o_sw = dw_sp;
    p.seg_len = seg_len; p.elems = elems; p.nseg = (uint32_t)nseg;
    const unsigned blocks = (unsigned)((elems + 255) / 256);
    void* kargs[] = {&p};
    CUfunction f;
    rc = get_func(c, std::string("conv2d_grp_wgrad_") + grp_tag(in_dtype) + "_" + grp_tag(out_dtype), &f);
    if (!rc) rc = launch(c, f, blocks, (unsigned)nseg, 1, 256, 0, 1, st, kargs);
    if (!rc && nseg > 1) rc = get_func(c, std::string("conv2d_grp_wgrad_combine_") + grp_tag(out_dtype), &f);
    if (!rc && nseg > 1) rc = launch(c, f, blocks, 1, 1, 256, 0, 1, st, kargs);
  }
  for (CUdeviceptr t : tmp)
    if (t) pool_free(c, t, st);
  return rc;
}

// Stage timings (ns) of the most recent fused reduce + exchange launched with option reduce.debug=1 on stream `s`:
// words[0] = exchange (publish -> all peers seen), words[1] = partials + f64 tree of the last block.  Synchronises the stream.
// ================================================================================================ attention
// 4-D tiled map (dims innermost first; strides of dims 1..3 in elements), zero out-of-bounds fill.  Its own plan line and
// cache key; encode_tmap's are unchanged.
static int encode_tmap4(b200_ctx* c, CUtensorMap* out, CUtensorMapDataType dt, size_t esz, uint64_t base, const uint64_t dims[4],
                        const uint64_t strides[3], const uint32_t box[4], CUtensorMapSwizzle swz) {
  const int promo_bytes = atoi(opt(c, "gemm.l2_promotion", "256").c_str());
  const CUtensorMapL2promotion promo = promo_bytes >= 256 ? CU_TENSOR_MAP_L2_PROMOTION_L2_256B
                                       : promo_bytes >= 128 ? CU_TENSOR_MAP_L2_PROMOTION_L2_128B
                                       : promo_bytes >= 64 ? CU_TENSOR_MAP_L2_PROMOTION_L2_64B : CU_TENSOR_MAP_L2_PROMOTION_NONE;
  std::string key = "tiled4d|" + std::to_string((int)dt) + "|" + std::to_string((int)swz) + "|" + std::to_string(base);
  for (int i = 0; i < 4; ++i) key += "|" + std::to_string(dims[i]) + "|" + std::to_string(box[i]);
  for (int i = 0; i < 3; ++i) key += "|" + std::to_string(strides[i]);
  key += "|" + std::to_string((int)promo);
  if (c->dry) {
    char line[320];
    snprintf(line, sizeof(line), "tmap4d esz=%zu dims=(%llu,%llu,%llu,%llu) strides=(%llu,%llu,%llu) box=(%u,%u,%u,%u) swizzle=%d\n", esz,
             (unsigned long long)dims[0], (unsigned long long)dims[1], (unsigned long long)dims[2], (unsigned long long)dims[3],
             (unsigned long long)(strides[0] * esz), (unsigned long long)(strides[1] * esz), (unsigned long long)(strides[2] * esz), box[0],
             box[1], box[2], box[3], (int)swz);
    c->plan += line;
    memset(out, 0, sizeof(*out));
    return B200_OK;
  }
  auto it = c->tmap_cache.find(key);
  if (it != c->tmap_cache.end()) { *out = it->second; return B200_OK; }
  cuuint64_t gdim[4] = {dims[0], dims[1], dims[2], dims[3]};
  cuuint64_t gstr[3] = {strides[0] * esz, strides[1] * esz, strides[2] * esz};
  cuuint32_t bx[4] = {box[0], box[1], box[2], box[3]};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = g_drv.cuTensorMapEncodeTiled_p(out, dt, 4, reinterpret_cast<void*>(base), gdim, gstr, bx, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                              swz, promo, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return fail(B200_ERR_INVALID_ARG, "cuTensorMapEncodeTiled (rank 4) failed: %s (dims %llu,%llu,%llu,%llu strides %llu,%llu,%llu)", cu_err(r),
                (unsigned long long)dims[0], (unsigned long long)dims[1], (unsigned long long)dims[2], (unsigned long long)dims[3],
                (unsigned long long)gstr[0], (unsigned long long)gstr[1], (unsigned long long)gstr[2]);
  if (c->tmap_cache.size() > 512) c->tmap_cache.clear();
  c->tmap_cache[key] = *out;
  return B200_OK;
}

// An attention operand: the device pointer and dtype, the 4-D shape and normalised strides (elements) as the caller passed
// them, and which axes a tensor map reads as rows (S, T or a page's keys) and as heads.  Axis 3 is D, the map's innermost
// dimension, and axis 0 (B, a varlen tensor's unit batch, or the page) its outermost.
struct AttnView {
  uint64_t ptr;
  b200_dtype dt;
  size_t esz;
  uint64_t shape[4], ns[4];
  int row, head;
  uint64_t rows() const { return shape[row]; }
  uint64_t heads() const { return shape[head]; }
  uint64_t s_row() const { return ns[row]; }
  uint64_t s_head() const { return ns[head]; }
  uint64_t s_batch() const { return ns[0]; }
};

// [B, H, S, D] (dense q, k, v, out and grads); [B or P, S or page, H, D] (KV caches and new tokens); a varlen [T, H, D] (strides
// null: compact), seen as [1, T, H, D].
enum AttnLayout { kAttnBHSD, kAttnBSHD, kAttnTHD };

static AttnView attn_view(uint64_t ptr, b200_dtype dt, const uint64_t* shape, const uint64_t* strides, AttnLayout layout) {
  AttnView v{};
  v.ptr = ptr; v.dt = dt; v.esz = dtype_size(dt);
  const bool thd = layout == kAttnTHD;
  uint64_t st3[4] = {0, 0, 0, 0};
  if (thd && strides) memcpy(st3 + 1, strides, 3 * sizeof(uint64_t));
  for (int d = 0; d < 4; ++d) v.shape[d] = !thd ? shape[d] : d ? shape[d - 1] : 1;
  conv_norm_strides(v.shape, thd && strides ? st3 : strides, v.ns);
  v.row = layout == kAttnBHSD ? 2 : 1;
  v.head = layout == kAttnBHSD ? 1 : 2;
  return v;
}

// A view a tensor map (or the 16-byte loads of the delta and cache-write kernels) reads in place: unit D stride, 16-byte
// aligned base, and the other strides 16-byte multiples below 2^40 bytes.
static bool attn_view_ok(const AttnView& v) {
  if (v.ptr % 16 || v.ns[3] != 1) return false;
  for (int d = 0; d < 3; ++d)
    if ((v.ns[d] * v.esz) % 16 || v.ns[d] * v.esz >= (1ull << 40)) return false;
  return true;
}

// v in place when attn_view_ok, else gathered into a compact pooled copy *tmp (the caller frees it) that v then describes.
static int attn_stage(b200_ctx* c, CUstream st, AttnView* v, CUdeviceptr* tmp) {
  if (attn_view_ok(*v)) return B200_OK;
  const uint64_t* sh = v->shape;
  int rc = pool_alloc(c, sh[0] * sh[1] * sh[2] * sh[3] * v->esz, tmp, st);
  if (rc) return rc;
  rc = b200_into_contiguous(c, static_cast<b200_stream>(st), v->dt, v->ptr, *tmp, 4, sh, v->ns);
  v->ptr = *tmp;
  v->ns[3] = 1; v->ns[2] = sh[3]; v->ns[1] = sh[2] * sh[3]; v->ns[0] = sh[1] * sh[2] * sh[3];
  return rc;
}

// The 128-byte swizzled map of v with dims (D, rows, heads, axis 0).  A load (box 64 x rows x heads) reads the input dtype; a
// store (out and the grads: 128-byte x 64-row boxes) moves raw 16- or 32-bit words.  An fp8 cache moves raw bytes, 128 (a
// whole head, D <= 128) per box row.
static int attn_map(b200_ctx* c, CUtensorMap* m, const AttnView& v, bool store, uint32_t rows = 64, uint32_t heads = 1) {
  const CUtensorMapDataType dt = v.esz == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                                 : v.esz == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8
                                 : store    ? CU_TENSOR_MAP_DATA_TYPE_UINT16
                                 : v.dt == B200_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  const uint32_t box[4] = {store || v.esz == 1 ? (uint32_t)(128 / v.esz) : 64u, rows, heads, 1};
  const uint64_t dims[4] = {v.shape[3], v.rows(), v.heads(), v.shape[0]}, strides[3] = {v.s_row(), v.s_head(), v.s_batch()};
  return encode_tmap4(c, m, dt, v.esz, v.ptr, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
}

static int attn_set_smem(b200_ctx* c, CUfunction f, unsigned smem) {
  if (c->dry) return B200_OK;
  CUresult r = g_drv.cuFuncSetAttribute_p(f, CU_FUNC_ATTRIBUTE_MAX_DYNAMIC_SHARED_SIZE_BYTES, (int)smem);
  return r != CUDA_SUCCESS ? fail(map_cu(r), "cuFuncSetAttribute: %s", cu_err(r)) : B200_OK;
}

// The head-dim bucket the kernels are instantiated for, and the kernels' f32 scale * log2(e).
static uint32_t attn_db(uint64_t D) { return D <= 64 ? 64 : 128; }
static float attn_scale_log2(float scale) { return (float)((double)scale * 1.4426950408889634074); }

static std::string attn_dims(const uint64_t* s, int rank) {
  std::string r = "[";
  for (int d = 0; d < rank; ++d) r += (d ? "," : "") + std::to_string(s[d]);
  return r + "]";
}

// ---- checks the attention entry points share; what: the entry point, for messages
static int attn_check_in_dtype(const char* what, b200_dtype in) {
  if (in != B200_F16 && in != B200_BF16) return fail(B200_ERR_UNSUPPORTED, "%s: input dtype %d unsupported (f16, bf16)", what, (int)in);
  return B200_OK;
}

// out ("output") or the grads ("grad"): the input dtype or f32.
static int attn_check_out_dtype(const char* what, const char* name, b200_dtype in, b200_dtype dt) {
  if (dt != in && dt != B200_F32) return fail(B200_ERR_UNSUPPORTED, "%s: %s dtype must equal the input dtype or be f32", what, name);
  return B200_OK;
}

// v equals k but for the head dim, which must be k's.
static int attn_check_v(const char* what, const char* k_name, const char* v_name, const uint64_t* k, const uint64_t* v, int rank) {
  if (memcmp(v, k, (rank - 1) * sizeof(uint64_t)))
    return fail(B200_ERR_INVALID_ARG, "%s: %s %s does not match %s %s", what, v_name, attn_dims(v, rank).c_str(), k_name,
                attn_dims(k, rank).c_str());
  if (v[rank - 1] != k[rank - 1])
    return fail(B200_ERR_UNSUPPORTED, "%s: %s's head dim %llu differs from D = %llu", what, v_name, (unsigned long long)v[rank - 1],
                (unsigned long long)k[rank - 1]);
  return B200_OK;
}

static int attn_check_gqa(const char* what, uint64_t Hq, uint64_t Hkv) {
  if (Hkv == 0 || Hq % Hkv)
    return fail(B200_ERR_INVALID_ARG, "%s: Hq = %llu must be a multiple of Hkv = %llu", what, (unsigned long long)Hq, (unsigned long long)Hkv);
  return B200_OK;
}

// Each named shape must equal its `want`.
struct AttnSame {
  const char* name;
  const uint64_t *shape, *want;
};
static int attn_check_same(const char* what, int rank, std::initializer_list<AttnSame> same) {
  for (const AttnSame& t : same)
    if (memcmp(t.shape, t.want, rank * sizeof(uint64_t)))
      return fail(B200_ERR_INVALID_ARG, "%s: %s is %s, expected %s", what, t.name, attn_dims(t.shape, rank).c_str(), attn_dims(t.want, rank).c_str());
  return B200_OK;
}

static int attn_check_scale_d(const char* what, float scale, uint64_t D) {
  if (!std::isfinite(scale)) return fail(B200_ERR_INVALID_ARG, "%s: scale must be finite", what);
  if (D == 0 || D > 128 || D % 8)
    return fail(B200_ERR_UNSUPPORTED, "%s: head dim D = %llu unsupported (a multiple of 8 in [8, 128])", what, (unsigned long long)D);
  return B200_OK;
}

static int attn_check_extents(const char* what, std::initializer_list<uint64_t> extents) {
  for (uint64_t e : extents)
    if (e >= (1ull << 31)) return fail(B200_ERR_UNSUPPORTED, "%s: extents must be < 2^31", what);
  return B200_OK;
}

// out or a grad (name), written in place.
static int attn_check_out_view(const char* what, const char* name, const AttnView& v) {
  if (attn_view_ok(v)) return B200_OK;
  return fail(B200_ERR_UNSUPPORTED, "%s: %s needs a unit D stride and a 16-byte aligned base and %s strides", what, name,
              v.row == 2 ? "S, H, B" : "T, H");
}

static int attn_check_caches(const char* what, const AttnView& kc, const AttnView& vc) {
  if (attn_view_ok(kc) && attn_view_ok(vc)) return B200_OK;
  return fail(B200_ERR_UNSUPPORTED, "%s: a cache needs a unit D stride and a 16-byte aligned base and page, row and head strides "
              "(it is read in place, never gathered)", what);
}

// ---- launch sequences the dense and varlen entry points share
// Stages q, k and v, maps them (loads of kAttnBlock rows) and out, then launches `<prefix><in>_d<DB>_<out>` on `ctas` CTAs
// with the filled parameter block p.
static int attn_fwd_launch(b200_ctx* c, CUstream st, const std::string& prefix, AttnView q, AttnView k, AttnView v, const AttnView& o,
                           uint64_t ctas, void* p) {
  CUdeviceptr tmp[3] = {0, 0, 0};
  int rc = attn_stage(c, st, &q, &tmp[0]);
  if (!rc) rc = attn_stage(c, st, &k, &tmp[1]);
  if (!rc) rc = attn_stage(c, st, &v, &tmp[2]);
  CUtensorMap mq, mk, mv, mo;
  if (!rc) rc = attn_map(c, &mq, q, false, kAttnBlock);
  if (!rc) rc = attn_map(c, &mk, k, false, kAttnBlock);
  if (!rc) rc = attn_map(c, &mv, v, false, kAttnBlock);
  if (!rc) rc = attn_map(c, &mo, o, true);
  const uint32_t DB = attn_db(q.shape[3]);
  CUfunction f = nullptr;
  if (!rc) rc = get_func(c, prefix + dt_tag(q.dt) + "_d" + std::to_string(DB) + "_" + dt_tag(o.dt), &f);
  const unsigned smem = 1024 + (1 + 2 * kAttnStages) * kAttnBlock * DB * 2 + 1024;
  if (!rc) rc = attn_set_smem(c, f, smem);
  void* kargs[] = {&mq, &mk, &mv, &mo, p};
  if (!rc) rc = launch(c, f, (unsigned)ctas, 1, 1, 384, smem, 1, st, kargs);
  for (CUdeviceptr t : tmp)
    if (t) pool_free(c, t, st);   // stream-ordered: reusable once the kernel has drained
  return rc;
}

struct AttnBwdOps {
  AttnView q, k, v, out, dout, dq, dk, dv;
};

// Stages what the present sides read: q, out and dout with query rows (has_q), k and v with keys (has_k); tmp[0..4] receive
// the copies (the caller frees them).
static int attn_bwd_stage(b200_ctx* c, CUstream st, AttnBwdOps* o, bool has_q, bool has_k, CUdeviceptr tmp[5]) {
  int rc = has_q ? attn_stage(c, st, &o->q, &tmp[0]) : B200_OK;
  if (!rc && has_k) rc = attn_stage(c, st, &o->k, &tmp[1]);
  if (!rc && has_k) rc = attn_stage(c, st, &o->v, &tmp[2]);
  if (!rc && has_q) rc = attn_stage(c, st, &o->out, &tmp[3]);
  if (!rc && has_q) rc = attn_stage(c, st, &o->dout, &tmp[4]);
  return rc;
}

// With query rows: `<prefix>delta_*` (delta and L into the workspace) and `<prefix>dq_*` on q_ctas CTAs; with keys:
// `<prefix>dkdv_*` on k_ctas CTAs.  A side that is absent is never read, so its maps take the other side's views.  p: the
// kernels' filled parameter block, workspace included.
static int attn_bwd_launch(b200_ctx* c, CUstream st, const std::string& prefix, AttnBwdOps o, bool has_q, bool has_k, uint64_t q_ctas,
                           uint64_t k_ctas, void* p) {
  if (!has_k) o.k = o.v = o.q;
  if (!has_q) o.q = o.dout = o.k;
  const uint32_t DB = attn_db(o.q.shape[3]);
  const std::string in = dt_tag(o.q.dt), tail = "_d" + std::to_string(DB) + "_" + dt_tag(o.dq.dt);
  CUfunction f = nullptr;
  int rc = B200_OK;
  if (has_q) {   // one 256-thread block per 16 workspace rows
    rc = get_func(c, prefix + "delta_" + in + "_" + dt_tag(o.out.dt), &f);
    void* kargs[] = {p};
    if (!rc) rc = launch(c, f, (unsigned)(q_ctas * (kAttnBlock / 16)), 1, 1, 256, 0, 1, st, kargs);
  }
  if (!rc && has_q) {   // dq: query tiles of kAttnBlock rows, key tiles of kAttnBwdDqKeys
    CUtensorMap mq, mk, mv, mdo, mdq;
    rc = attn_map(c, &mq, o.q, false, kAttnBlock);
    if (!rc) rc = attn_map(c, &mk, o.k, false, kAttnBwdDqKeys);
    if (!rc) rc = attn_map(c, &mv, o.v, false, kAttnBwdDqKeys);
    if (!rc) rc = attn_map(c, &mdo, o.dout, false, kAttnBlock);
    if (!rc) rc = attn_map(c, &mdq, o.dq, true);
    if (!rc) rc = get_func(c, prefix + "dq_" + in + tail, &f);
    const unsigned smem = 1024 + 2 * kAttnBlock * DB * 2 + 2 * kAttnBwdStages * kAttnBwdDqKeys * DB * 2 + 1024;
    if (!rc) rc = attn_set_smem(c, f, smem);
    void* kargs[] = {&mq, &mk, &mv, &mdo, &mdq, p};
    if (!rc) rc = launch(c, f, (unsigned)q_ctas, 1, 1, 384, smem, 1, st, kargs);
  }
  if (!rc && has_k) {   // dk and dv: query tiles of kAttnBwdDkdvQueries rows, key tiles of kAttnBlock
    CUtensorMap mq, mk, mv, mdo, mdk, mdv;
    rc = attn_map(c, &mq, o.q, false, kAttnBwdDkdvQueries);
    if (!rc) rc = attn_map(c, &mk, o.k, false, kAttnBlock);
    if (!rc) rc = attn_map(c, &mv, o.v, false, kAttnBlock);
    if (!rc) rc = attn_map(c, &mdo, o.dout, false, kAttnBwdDkdvQueries);
    if (!rc) rc = attn_map(c, &mdk, o.dk, true);
    if (!rc) rc = attn_map(c, &mdv, o.dv, true);
    if (!rc) rc = get_func(c, prefix + "dkdv_" + in + tail, &f);
    const unsigned smem = 1024 + 2 * kAttnBlock * DB * 2 + 2 * kAttnBwdStages * kAttnBwdDkdvQueries * DB * 2 +
                          kAttnBwdStages * 2 * kAttnBwdDkdvQueries * 4 + 1024;
    if (!rc) rc = attn_set_smem(c, f, smem);
    void* kargs[] = {&mq, &mk, &mv, &mdo, &mdk, &mdv, p};
    if (!rc) rc = launch(c, f, (unsigned)k_ctas, 1, 1, 384, smem, 1, st, kargs);
  }
  return rc;
}

// ------------------------------------------------------------------------------------------------ dense attention
extern "C" int b200_attention(b200_ctx* c, b200_stream s, b200_dtype in_dtype, b200_dtype out_dtype, b200_dptr q, const uint64_t* q_shape,
                              const uint64_t* q_strides, b200_dptr k, const uint64_t* k_shape, const uint64_t* k_strides, b200_dptr v,
                              const uint64_t* v_shape, const uint64_t* v_strides, b200_dptr out, const uint64_t* out_shape,
                              const uint64_t* out_strides, b200_dptr lse, const b200_attention_args* args) {
  CTX_ENTER(c);
  const char* what = "attention";
  if (!q_shape || !k_shape || !v_shape || !out_shape || !args) return fail(B200_ERR_INVALID_ARG, "%s: null shape or args", what);
  int rc = attn_check_in_dtype(what, in_dtype);
  if (!rc) rc = attn_check_out_dtype(what, "output", in_dtype, out_dtype);
  if (rc) return rc;
  const uint64_t B = q_shape[0], Hq = q_shape[1], Sq = q_shape[2], D = q_shape[3];
  const uint64_t Hkv = k_shape[1], Sk = k_shape[2];
  if (k_shape[0] != B || k_shape[3] != D)
    return fail(B200_ERR_INVALID_ARG, "%s: k %s differs from q %s in batch or head dim", what, attn_dims(k_shape, 4).c_str(),
                attn_dims(q_shape, 4).c_str());
  rc = attn_check_v(what, "k", "v", k_shape, v_shape, 4);
  if (!rc) rc = attn_check_gqa(what, Hq, Hkv);
  if (!rc) rc = attn_check_same(what, 4, {{"out", out_shape, q_shape}});
  if (!rc && Sk == 0 && Sq > 0) rc = fail(B200_ERR_INVALID_ARG, "%s: Sk = 0 leaves every query row without keys", what);
  if (!rc) rc = attn_check_scale_d(what, args->scale, D);
  if (!rc) rc = attn_check_extents(what, {B, Hq, Sq, Hkv, Sk});
  if (rc) return rc;
  if (B == 0 || Hq == 0 || Sq == 0) return B200_OK;
  const uint64_t nqb = (Sq + kAttnBlock - 1) / kAttnBlock, ctas = nqb * Hq * B;
  if (ctas >= (1ull << 31))
    return fail(B200_ERR_UNSUPPORTED, "%s: ceil(Sq / %d) * Hq * B = %llu CTAs must be < 2^31", what, kAttnBlock, (unsigned long long)ctas);
  if (!q || !k || !v || !out) return fail(B200_ERR_INVALID_ARG, "%s: null device pointer", what);
  if (lse % 4) return fail(B200_ERR_INVALID_ARG, "%s: lse pointer is not 4-byte aligned", what);
  const AttnView ov = attn_view(out, out_dtype, out_shape, out_strides, kAttnBHSD);
  if ((rc = attn_check_out_view(what, "out", ov))) return rc;

  AttnParams p{};
  p.lse = lse;
  p.B = (uint32_t)B; p.Hq = (uint32_t)Hq; p.Sq = (uint32_t)Sq; p.Sk = (uint32_t)Sk;
  p.group = (uint32_t)(Hq / Hkv);
  p.nqb = (uint32_t)nqb;
  p.causal = args->causal != 0 ? 1u : 0u;
  p.D = (uint32_t)D;
  p.scale_log2 = attn_scale_log2(args->scale);
  return attn_fwd_launch(c, resolve_stream(c, s), "attn_fwd_", attn_view(q, in_dtype, q_shape, q_strides, kAttnBHSD),
                         attn_view(k, in_dtype, k_shape, k_strides, kAttnBHSD), attn_view(v, in_dtype, v_shape, v_strides, kAttnBHSD), ov,
                         ctas, &p);
}

// Backward of b200_attention (see cubecl_b200.h): the delta / L pass, then the dq and the dk / dv kernels.
extern "C" int b200_attention_backward(b200_ctx* c, b200_stream s, b200_dtype in_dtype, b200_dtype out_dtype, b200_dtype grad_dtype,
                                       b200_dptr q, const uint64_t* q_shape, const uint64_t* q_strides, b200_dptr k,
                                       const uint64_t* k_shape, const uint64_t* k_strides, b200_dptr v, const uint64_t* v_shape,
                                       const uint64_t* v_strides, b200_dptr out, const uint64_t* out_shape, const uint64_t* out_strides,
                                       b200_dptr dout, const uint64_t* dout_shape, const uint64_t* dout_strides, b200_dptr lse,
                                       b200_dptr dq, const uint64_t* dq_shape, const uint64_t* dq_strides, b200_dptr dk,
                                       const uint64_t* dk_shape, const uint64_t* dk_strides, b200_dptr dv, const uint64_t* dv_shape,
                                       const uint64_t* dv_strides, const b200_attention_args* args) {
  CTX_ENTER(c);
  const char* what = "attention_backward";
  if (!q_shape || !k_shape || !v_shape || !out_shape || !dout_shape || !dq_shape || !dk_shape || !dv_shape || !args)
    return fail(B200_ERR_INVALID_ARG, "%s: null shape or args", what);
  int rc = attn_check_in_dtype(what, in_dtype);
  if (!rc) rc = attn_check_out_dtype(what, "output", in_dtype, out_dtype);
  if (!rc) rc = attn_check_out_dtype(what, "grad", in_dtype, grad_dtype);
  if (rc) return rc;
  const uint64_t B = q_shape[0], Hq = q_shape[1], Sq = q_shape[2], D = q_shape[3];
  const uint64_t Hkv = k_shape[1], Sk = k_shape[2];
  if (k_shape[0] != B || k_shape[3] != D)
    return fail(B200_ERR_INVALID_ARG, "%s: k %s differs from q %s in batch or head dim", what, attn_dims(k_shape, 4).c_str(),
                attn_dims(q_shape, 4).c_str());
  rc = attn_check_v(what, "k", "v", k_shape, v_shape, 4);
  if (!rc) rc = attn_check_gqa(what, Hq, Hkv);
  if (!rc)
    rc = attn_check_same(what, 4, {{"out", out_shape, q_shape}, {"dout", dout_shape, q_shape}, {"dq", dq_shape, q_shape},
                                   {"dk", dk_shape, k_shape}, {"dv", dv_shape, k_shape}});
  if (!rc && Sk == 0 && Sq > 0) rc = fail(B200_ERR_INVALID_ARG, "%s: Sk = 0 leaves every query row without keys", what);
  if (!rc) rc = attn_check_scale_d(what, args->scale, D);
  if (!rc) rc = attn_check_extents(what, {B, Hq, Sq, Hkv, Sk});
  if (rc) return rc;
  // B = 0, or no queries and no keys: nothing to write.  Sq = 0 or Hq = 0 with keys still writes zero dk and dv.
  if (B == 0 || (Sk == 0 && Sq == 0)) return B200_OK;
  const uint64_t nqb = (Sq + kAttnBlock - 1) / kAttnBlock, nkb = (Sk + kAttnBlock - 1) / kAttnBlock;
  const uint64_t rows = B * Hq * nqb * kAttnBlock;   // workspace rows, padded per (b, h) to whole query blocks
  const bool has_q = rows > 0;
  const uint64_t lim = 1ull << 31;
  if (nqb * Hq * B >= lim || nkb * Hkv * B >= lim || rows / 16 >= lim) return fail(B200_ERR_UNSUPPORTED, "%s: more than 2^31 - 1 CTAs", what);
  if (!k || !v || !dk || !dv || (has_q && (!q || !out || !dout || !dq || !lse))) return fail(B200_ERR_INVALID_ARG, "%s: null device pointer", what);
  if (lse % 4) return fail(B200_ERR_INVALID_ARG, "%s: lse pointer is not 4-byte aligned", what);
  AttnBwdOps o{attn_view(q, in_dtype, q_shape, q_strides, kAttnBHSD),          attn_view(k, in_dtype, k_shape, k_strides, kAttnBHSD),
               attn_view(v, in_dtype, v_shape, v_strides, kAttnBHSD),          attn_view(out, out_dtype, out_shape, out_strides, kAttnBHSD),
               attn_view(dout, in_dtype, dout_shape, dout_strides, kAttnBHSD), attn_view(dq, grad_dtype, dq_shape, dq_strides, kAttnBHSD),
               attn_view(dk, grad_dtype, dk_shape, dk_strides, kAttnBHSD),     attn_view(dv, grad_dtype, dv_shape, dv_strides, kAttnBHSD)};
  if (has_q) rc = attn_check_out_view(what, "dq", o.dq);
  if (!rc) rc = attn_check_out_view(what, "dk", o.dk);
  if (!rc) rc = attn_check_out_view(what, "dv", o.dv);
  if (rc) return rc;

  CUstream st = resolve_stream(c, s);
  CUdeviceptr tmp[6] = {0, 0, 0, 0, 0, 0};   // gathers of q, k, v, out, dout; the workspace
  rc = attn_bwd_stage(c, st, &o, has_q, true, tmp);
  if (!rc && has_q) rc = pool_alloc(c, 2 * rows * 4, &tmp[5], st);
  AttnBwdParams p{};
  p.ws = tmp[5];
  p.lse = lse;
  p.out = o.out.ptr; p.dout = o.dout.ptr;
  p.o_sb = o.out.s_batch(); p.o_sh = o.out.s_head(); p.o_ss = o.out.s_row();
  p.d_sb = o.dout.s_batch(); p.d_sh = o.dout.s_head(); p.d_ss = o.dout.s_row();
  p.B = (uint32_t)B; p.Hq = (uint32_t)Hq; p.Sq = (uint32_t)Sq; p.Sk = (uint32_t)Sk; p.Hkv = (uint32_t)Hkv;
  p.group = (uint32_t)(Hq / Hkv);
  p.nqb = (uint32_t)nqb; p.nkb = (uint32_t)nkb;
  p.nqd = (uint32_t)((Sq + kAttnBwdDkdvQueries - 1) / kAttnBwdDkdvQueries);
  p.Sqp = (uint32_t)(nqb * kAttnBlock);
  p.causal = args->causal != 0 ? 1u : 0u;
  p.D = (uint32_t)D;
  p.scale_log2 = attn_scale_log2(args->scale);
  p.scale = args->scale;
  if (!rc) rc = attn_bwd_launch(c, st, "attn_bwd_", o, has_q, true, nqb * Hq * B, nkb * Hkv * B, &p);
  for (CUdeviceptr t : tmp)
    if (t) pool_free(c, t, st);   // stream-ordered: reusable once the kernels have drained
  return rc;
}

// ------------------------------------------------------------------------------------------------ varlen attention
// The checks both varlen entries share (see cubecl_b200.h); 0 or the failure status.
static int vl_check(const char* what, b200_dtype in_dtype, const uint64_t* q_shape, const uint64_t* k_shape, const uint64_t* v_shape,
                    uint64_t batch, const b200_attention_varlen_args* args) {
  int rc = attn_check_in_dtype(what, in_dtype);
  if (rc) return rc;
  const uint64_t Tq = q_shape[0], Hq = q_shape[1], D = q_shape[2], Tk = k_shape[0], Hkv = k_shape[1];
  if (k_shape[2] != D)
    return fail(B200_ERR_INVALID_ARG, "%s: k's head dim %llu differs from q's D = %llu", what, (unsigned long long)k_shape[2], (unsigned long long)D);
  rc = attn_check_v(what, "k", "v", k_shape, v_shape, 3);
  if (!rc) rc = attn_check_gqa(what, Hq, Hkv);
  if (!rc && (args->window_left < -1 || args->window_right < -1))
    rc = fail(B200_ERR_INVALID_ARG, "%s: window (%d, %d): each side must be >= 0, or -1 for unbounded", what, args->window_left,
              args->window_right);
  if (!rc && (args->max_seqlen_q < 0 || args->max_seqlen_k < 0))
    rc = fail(B200_ERR_INVALID_ARG, "%s: max_seqlen_q = %d and max_seqlen_k = %d must be >= 0", what, args->max_seqlen_q, args->max_seqlen_k);
  if (!rc) rc = attn_check_scale_d(what, args->scale, D);
  if (!rc) rc = attn_check_extents(what, {batch, Tq, Hq, Tk, Hkv});
  if (!rc && (args->max_seqlen_q >= (1 << 30) || args->max_seqlen_k >= (1 << 30)))
    rc = fail(B200_ERR_UNSUPPORTED, "%s: max_seqlen_q and max_seqlen_k must be < 2^30", what);
  return rc;
}

// Variable-length attention, forward (see cubecl_b200.h): one attn_fwd_varlen_* launch.
extern "C" int b200_attention_varlen(b200_ctx* c, b200_stream s, b200_dtype in_dtype, b200_dtype out_dtype, b200_dptr q,
                                     const uint64_t* q_shape, const uint64_t* q_strides, b200_dptr k, const uint64_t* k_shape,
                                     const uint64_t* k_strides, b200_dptr v, const uint64_t* v_shape, const uint64_t* v_strides,
                                     b200_dptr cu_seqlens_q, b200_dptr cu_seqlens_k, uint64_t batch, b200_dptr out,
                                     const uint64_t* out_shape, const uint64_t* out_strides, b200_dptr lse,
                                     const b200_attention_varlen_args* args) {
  CTX_ENTER(c);
  const char* what = "attention_varlen";
  if (!q_shape || !k_shape || !v_shape || !out_shape || !args) return fail(B200_ERR_INVALID_ARG, "%s: null shape or args", what);
  int rc = vl_check(what, in_dtype, q_shape, k_shape, v_shape, batch, args);
  if (!rc) rc = attn_check_out_dtype(what, "output", in_dtype, out_dtype);
  if (!rc) rc = attn_check_same(what, 3, {{"out", out_shape, q_shape}});
  if (rc) return rc;
  const uint64_t Tq = q_shape[0], Hq = q_shape[1], D = q_shape[2], Tk = k_shape[0], Hkv = k_shape[1], B = batch;
  const uint64_t max_q = (uint64_t)args->max_seqlen_q, max_k = (uint64_t)args->max_seqlen_k;
  if (B == 0 || Tq == 0 || Hq == 0 || max_q == 0) return B200_OK;   // no query row
  const uint64_t nqb = (max_q + kAttnBlock - 1) / kAttnBlock, ctas = nqb * Hq * B;
  if (ctas >= (1ull << 31))
    return fail(B200_ERR_UNSUPPORTED, "%s: ceil(max_seqlen_q / %d) * Hq * B = %llu CTAs must be < 2^31", what, kAttnBlock,
                (unsigned long long)ctas);
  if (!q || !k || !v || !out || !cu_seqlens_q || !cu_seqlens_k) return fail(B200_ERR_INVALID_ARG, "%s: null device pointer", what);
  if (lse % 4 || cu_seqlens_q % 4 || cu_seqlens_k % 4)
    return fail(B200_ERR_INVALID_ARG, "%s: lse, cu_seqlens_q and cu_seqlens_k must be 4-byte aligned", what);
  const AttnView ov = attn_view(out, out_dtype, out_shape, out_strides, kAttnTHD);
  if ((rc = attn_check_out_view(what, "out", ov))) return rc;

  AttnVarlenParams p{};
  p.lse = lse;
  p.cu_q = cu_seqlens_q; p.cu_k = cu_seqlens_k;
  p.out = out; p.o_st = ov.s_row(); p.o_sh = ov.s_head();
  p.B = (uint32_t)B; p.Hq = (uint32_t)Hq; p.Hkv = (uint32_t)Hkv; p.Tq = (uint32_t)Tq; p.Tk = (uint32_t)Tk;
  p.group = (uint32_t)(Hq / Hkv);
  p.max_q = (uint32_t)max_q; p.max_k = (uint32_t)max_k;
  p.nqb = (uint32_t)nqb; p.nkb = (uint32_t)((max_k + kAttnBlock - 1) / kAttnBlock);
  p.D = (uint32_t)D;
  p.left = args->window_left; p.right = args->window_right;
  p.scale_log2 = attn_scale_log2(args->scale);
  p.scale = args->scale;
  return attn_fwd_launch(c, resolve_stream(c, s), "attn_fwd_varlen_", attn_view(q, in_dtype, q_shape, q_strides, kAttnTHD),
                         attn_view(k, in_dtype, k_shape, k_strides, kAttnTHD), attn_view(v, in_dtype, v_shape, v_strides, kAttnTHD), ov,
                         ctas, &p);
}

// Backward of b200_attention_varlen (see cubecl_b200.h): the delta / L pass, then the dq and the dk / dv kernels.
extern "C" int b200_attention_varlen_backward(b200_ctx* c, b200_stream s, b200_dtype in_dtype, b200_dtype out_dtype, b200_dtype grad_dtype,
                                              b200_dptr q, const uint64_t* q_shape, const uint64_t* q_strides, b200_dptr k,
                                              const uint64_t* k_shape, const uint64_t* k_strides, b200_dptr v, const uint64_t* v_shape,
                                              const uint64_t* v_strides, b200_dptr out, const uint64_t* out_shape,
                                              const uint64_t* out_strides, b200_dptr dout, const uint64_t* dout_shape,
                                              const uint64_t* dout_strides, b200_dptr lse, b200_dptr cu_seqlens_q,
                                              b200_dptr cu_seqlens_k, uint64_t batch, b200_dptr dq, const uint64_t* dq_shape,
                                              const uint64_t* dq_strides, b200_dptr dk, const uint64_t* dk_shape,
                                              const uint64_t* dk_strides, b200_dptr dv, const uint64_t* dv_shape,
                                              const uint64_t* dv_strides, const b200_attention_varlen_args* args) {
  CTX_ENTER(c);
  const char* what = "attention_varlen_backward";
  if (!q_shape || !k_shape || !v_shape || !out_shape || !dout_shape || !dq_shape || !dk_shape || !dv_shape || !args)
    return fail(B200_ERR_INVALID_ARG, "%s: null shape or args", what);
  int rc = vl_check(what, in_dtype, q_shape, k_shape, v_shape, batch, args);
  if (!rc) rc = attn_check_out_dtype(what, "output", in_dtype, out_dtype);
  if (!rc) rc = attn_check_out_dtype(what, "grad", in_dtype, grad_dtype);
  if (!rc)
    rc = attn_check_same(what, 3, {{"out", out_shape, q_shape}, {"dout", dout_shape, q_shape}, {"dq", dq_shape, q_shape},
                                   {"dk", dk_shape, k_shape}, {"dv", dv_shape, k_shape}});
  if (rc) return rc;
  const uint64_t Tq = q_shape[0], Hq = q_shape[1], D = q_shape[2], Tk = k_shape[0], Hkv = k_shape[1], B = batch;
  const uint64_t max_q = (uint64_t)args->max_seqlen_q, max_k = (uint64_t)args->max_seqlen_k;
  // query rows to differentiate (delta and dq); key rows to differentiate (dk and dv: +0 where no query sees them)
  const bool has_q = B > 0 && Tq > 0 && Hq > 0 && max_q > 0, has_k = B > 0 && Tk > 0 && max_k > 0;
  if (!has_q && !has_k) return B200_OK;
  const uint64_t nqb = (max_q + kAttnBlock - 1) / kAttnBlock, nkb = (max_k + kAttnBlock - 1) / kAttnBlock;
  const uint64_t Tqp = ((Tq + kAttnBlock - 1) / kAttnBlock + B) * kAttnBlock;   // workspace rows per head
  if (nqb * Hq * B >= (1ull << 31) || nkb * Hkv * B >= (1ull << 31) || nqb * 8 * Hq * B >= (1ull << 31))
    return fail(B200_ERR_UNSUPPORTED, "%s: more than 2^31 - 1 CTAs", what);
  if (!cu_seqlens_q || !cu_seqlens_k || !k || !v || !dk || !dv || (has_q && (!q || !out || !dout || !dq || !lse)))
    return fail(B200_ERR_INVALID_ARG, "%s: null device pointer", what);
  if (lse % 4 || cu_seqlens_q % 4 || cu_seqlens_k % 4)
    return fail(B200_ERR_INVALID_ARG, "%s: lse, cu_seqlens_q and cu_seqlens_k must be 4-byte aligned", what);
  AttnBwdOps o{attn_view(q, in_dtype, q_shape, q_strides, kAttnTHD),          attn_view(k, in_dtype, k_shape, k_strides, kAttnTHD),
               attn_view(v, in_dtype, v_shape, v_strides, kAttnTHD),          attn_view(out, out_dtype, out_shape, out_strides, kAttnTHD),
               attn_view(dout, in_dtype, dout_shape, dout_strides, kAttnTHD), attn_view(dq, grad_dtype, dq_shape, dq_strides, kAttnTHD),
               attn_view(dk, grad_dtype, dk_shape, dk_strides, kAttnTHD),     attn_view(dv, grad_dtype, dv_shape, dv_strides, kAttnTHD)};
  if (has_q) rc = attn_check_out_view(what, "dq", o.dq);
  if (!rc && has_k) rc = attn_check_out_view(what, "dk", o.dk);
  if (!rc && has_k) rc = attn_check_out_view(what, "dv", o.dv);
  if (rc) return rc;

  CUstream st = resolve_stream(c, s);
  CUdeviceptr tmp[6] = {0, 0, 0, 0, 0, 0};   // gathers of q, k, v, out, dout; the workspace
  // out and dout are read by the delta kernel with 16-byte loads, so they follow the maps' rule
  rc = attn_bwd_stage(c, st, &o, has_q, has_k, tmp);
  if (!rc && has_q) rc = pool_alloc(c, 2 * Hq * Tqp * 4, &tmp[5], st);
  AttnVarlenParams p{};
  p.lse = lse;
  p.cu_q = cu_seqlens_q; p.cu_k = cu_seqlens_k;
  p.ws = tmp[5];
  p.out = o.out.ptr; p.dout = o.dout.ptr;
  p.o_st = o.out.s_row(); p.o_sh = o.out.s_head(); p.d_st = o.dout.s_row(); p.d_sh = o.dout.s_head();
  p.dq = dq; p.dk = dk; p.dv = dv;
  p.dq_st = o.dq.s_row(); p.dq_sh = o.dq.s_head(); p.dk_st = o.dk.s_row(); p.dk_sh = o.dk.s_head(); p.dv_st = o.dv.s_row(); p.dv_sh = o.dv.s_head();
  p.B = (uint32_t)B; p.Hq = (uint32_t)Hq; p.Hkv = (uint32_t)Hkv; p.Tq = (uint32_t)Tq; p.Tk = (uint32_t)Tk;
  p.group = (uint32_t)(Hq / Hkv);
  p.max_q = (uint32_t)max_q; p.max_k = (uint32_t)max_k;
  p.nqb = (uint32_t)nqb; p.nkb = (uint32_t)nkb;
  p.Tqp = (uint32_t)Tqp;
  p.D = (uint32_t)D;
  p.left = args->window_left; p.right = args->window_right;
  p.scale_log2 = attn_scale_log2(args->scale);
  p.scale = args->scale;
  if (!rc) rc = attn_bwd_launch(c, st, "attn_bwd_varlen_", o, has_q, has_k, nqb * Hq * B, nkb * Hkv * B, &p);
  for (CUdeviceptr t : tmp)
    if (t) pool_free(c, t, st);   // stream-ordered: reusable once the kernels have drained
  return rc;
}

// ------------------------------------------------------------------------------------------------ KV-cache attention
// The m-tile of b200_attention_kvcache: st queries of gt heads of one kv head's G (gt * st <= kAttnKvRows), the pair with the
// fewest m-tiles ceil(G / gt) * ceil(Sq / st); among equals the largest st.
static void kv_tile(uint64_t G, uint64_t Sq, uint32_t* gt, uint32_t* st) {
  uint64_t best = UINT64_MAX;
  for (uint64_t s = std::min<uint64_t>(Sq, kAttnKvRows); s >= 1; --s) {
    const uint64_t g = std::min<uint64_t>(G, kAttnKvRows / s);
    const uint64_t n = ((G + g - 1) / g) * ((Sq + s - 1) / s);
    if (n < best) { best = n; *gt = (uint32_t)g; *st = (uint32_t)s; }
  }
}

// The split count of b200_attention_kvcache from shapes only: `units` = B * Hkv * m-tiles CTAs per split, nkb key blocks of
// capacity, one CTA per SM.  The count n minimising ceil(units * n / sms) * (ceil(nkb / n) + kAttnKvSplitCost), over the n
// whose equal ranges of ceil(nkb / n) blocks are all non-empty; ties keep the smaller n.
static uint32_t kv_splits(uint64_t units, uint64_t nkb, int sms) {
  uint64_t best_n = 1, best = UINT64_MAX;
  for (uint64_t n = 1; n <= std::min<uint64_t>(nkb, kAttnKvMaxSplits); ++n) {
    const uint64_t bps = (nkb + n - 1) / n;
    if ((nkb + bps - 1) / bps != n) continue;
    const uint64_t cost = (units * n + sms - 1) / sms * (bps + kAttnKvSplitCost);
    if (cost < best) { best = cost; best_n = n; }
  }
  return (uint32_t)best_n;
}

// An fp8 KV cache: its format and the f32 [Hkv] per-head scales (device pointers, read by the kernels only).
struct KvFp8 {
  b200_dtype cache;
  b200_dptr k_scale, v_scale;
};

static int kv_check_fp8(const char* what, const KvFp8* f8) {
  if (f8 && f8->cache != B200_F8E4M3 && f8->cache != B200_F8E5M2)
    return fail(B200_ERR_UNSUPPORTED, "%s: cache dtype %d unsupported (f8e4m3, f8e5m2)", what, (int)f8->cache);
  return B200_OK;
}

static int kv_check_scales(const char* what, const KvFp8* f8) {
  if (!f8) return B200_OK;
  if (!f8->k_scale || !f8->v_scale) return fail(B200_ERR_INVALID_ARG, "%s: null k_scale or v_scale", what);
  if (f8->k_scale % 4 || f8->v_scale % 4) return fail(B200_ERR_INVALID_ARG, "%s: k_scale and v_scale must be 4-byte aligned", what);
  return B200_OK;
}

// Attention of q against a paged KV cache (see cubecl_b200.h): one attn_kv_* launch, plus attn_kv_combine_* when the keys
// are split.  f8: an fp8 cache (b200_attention_kvcache_fp8), else the caches hold the input dtype.
static int kv_attend(b200_ctx* c, b200_stream s, const char* what, b200_dtype in_dtype, const KvFp8* f8, b200_dtype out_dtype, b200_dptr q,
                     const uint64_t* q_shape, const uint64_t* q_strides, b200_dptr k_cache, const uint64_t* kc_shape,
                     const uint64_t* kc_strides, b200_dptr v_cache, const uint64_t* vc_shape, const uint64_t* vc_strides,
                     b200_dptr block_table, const uint64_t* bt_shape, const uint64_t* bt_strides, b200_dptr cache_seqlens,
                     b200_dptr out, const uint64_t* out_shape, const uint64_t* out_strides, b200_dptr lse,
                     const b200_attention_args* args) {
  auto ull = [](uint64_t x) { return (unsigned long long)x; };
  if (!q_shape || !kc_shape || !vc_shape || !out_shape || !args) return fail(B200_ERR_INVALID_ARG, "%s: null shape or args", what);
  if (block_table && !bt_shape) return fail(B200_ERR_INVALID_ARG, "%s: null block-table shape", what);
  int rc = attn_check_in_dtype(what, in_dtype);
  if (!rc) rc = attn_check_out_dtype(what, "output", in_dtype, out_dtype);
  if (!rc) rc = kv_check_fp8(what, f8);
  if (rc) return rc;
  const b200_dtype cache_dtype = f8 ? f8->cache : in_dtype;
  const uint64_t B = q_shape[0], Hq = q_shape[1], Sq = q_shape[2], D = q_shape[3];
  const uint64_t P = kc_shape[0], page = kc_shape[1], Hkv = kc_shape[2];
  if (kc_shape[3] != D)
    return fail(B200_ERR_INVALID_ARG, "%s: k_cache head dim %llu differs from q's D = %llu", what, ull(kc_shape[3]), ull(D));
  rc = attn_check_v(what, "k_cache", "v_cache", kc_shape, vc_shape, 4);
  if (!rc) rc = attn_check_gqa(what, Hq, Hkv);
  if (!rc) rc = attn_check_same(what, 4, {{"out", out_shape, q_shape}});
  if (rc) return rc;
  if (page == 0 || P == 0) return fail(B200_ERR_INVALID_ARG, "%s: empty cache (P = %llu pages of %llu keys)", what, ull(P), ull(page));
  const uint64_t max_pages = block_table ? bt_shape[1] : 1;
  if (block_table && (bt_shape[0] != B || max_pages == 0))
    return fail(B200_ERR_INVALID_ARG, "%s: block_table is [%llu,%llu], expected [%llu, max_pages >= 1]", what, ull(bt_shape[0]),
                ull(bt_shape[1]), ull(B));
  if (!block_table && P != B)
    return fail(B200_ERR_INVALID_ARG, "%s: without a block table the cache holds one page per sequence (P = %llu, B = %llu)", what, ull(P), ull(B));
  if (max_pages > 1 && (page % 16 || (kAttnKvBlock % page && page % kAttnKvBlock)))
    return fail(B200_ERR_UNSUPPORTED, "%s: a page of %llu keys must be a multiple of 16 that divides %d or is a multiple of it", what,
                ull(page), kAttnKvBlock);
  if ((rc = attn_check_scale_d(what, args->scale, D))) return rc;
  const uint64_t lim = 1ull << 31, cap = max_pages * page;
  if (B >= lim || Hq >= lim || Sq >= lim || P >= lim || page >= lim || max_pages >= lim || cap >= lim)
    return fail(B200_ERR_UNSUPPORTED, "%s: extents and the capacity max_pages * page must be < 2^31", what);
  if (B == 0 || Hq == 0 || Sq == 0) return B200_OK;
  if (!q || !k_cache || !v_cache || !cache_seqlens || !out) return fail(B200_ERR_INVALID_ARG, "%s: null device pointer", what);
  if (lse % 4 || cache_seqlens % 4 || block_table % 4)
    return fail(B200_ERR_INVALID_ARG, "%s: lse, cache_seqlens and block_table must be 4-byte aligned", what);
  if ((rc = kv_check_scales(what, f8))) return rc;
  AttnView qv = attn_view(q, in_dtype, q_shape, q_strides, kAttnBHSD), ov = attn_view(out, out_dtype, out_shape, out_strides, kAttnBHSD);
  const AttnView kv = attn_view(k_cache, cache_dtype, kc_shape, kc_strides, kAttnBSHD), vv = attn_view(v_cache, cache_dtype, vc_shape, vc_strides, kAttnBSHD);
  if ((rc = attn_check_out_view(what, "out", ov)) || (rc = attn_check_caches(what, kv, vv))) return rc;

  const uint64_t G = Hq / Hkv;
  uint32_t gt = 1, stq = 1;
  kv_tile(G, Sq, &gt, &stq);
  const uint64_t mtg = (G + gt - 1) / gt, mts = (Sq + stq - 1) / stq;
  const uint64_t nkb = (cap + kAttnKvBlock - 1) / kAttnKvBlock;
  const uint64_t units = B * Hkv * mtg * mts;
  const uint32_t nsplit = kv_splits(units, nkb, c->props.num_sms);
  const uint64_t bps = (nkb + nsplit - 1) / nsplit, ctas = units * nsplit, rows = B * Hq * Sq;
  if (ctas >= lim || rows * (D / 4) / kAttnKvCombineThreads >= lim)
    return fail(B200_ERR_UNSUPPORTED, "%s: more than 2^31 - 1 CTAs", what);

  CUstream st = resolve_stream(c, s);
  CUdeviceptr tmp[2] = {0, 0};   // the gather of q; the split workspace
  rc = attn_stage(c, st, &qv, &tmp[0]);
  if (!rc && nsplit > 1) rc = pool_alloc(c, (size_t)nsplit * rows * (D + 2) * 4, &tmp[1], st);
  if (!rc) {
    const uint32_t DB = attn_db(D);
    const uint32_t R = max_pages == 1 ? kAttnKvBlock : (uint32_t)std::min<uint64_t>(page, kAttnKvBlock);
    CUtensorMap mq, mk, mv;
    rc = attn_map(c, &mq, qv, false, stq, gt);
    if (!rc) rc = attn_map(c, &mk, kv, false, R);
    if (!rc) rc = attn_map(c, &mv, vv, false, R);
    AttnKvParams p{};
    p.out = out; p.o_sb = ov.s_batch(); p.o_sh = ov.s_head(); p.o_ss = ov.s_row();
    p.lse = lse;
    p.ws = tmp[1];
    p.table = block_table;
    if (block_table) {
      p.t_sb = bt_strides ? bt_strides[0] : max_pages;
      p.t_sp = bt_strides ? bt_strides[1] : 1;
    }
    p.seqlens = cache_seqlens;
    p.B = (uint32_t)B; p.Hq = (uint32_t)Hq; p.Hkv = (uint32_t)Hkv; p.Sq = (uint32_t)Sq; p.D = (uint32_t)D;
    p.group = (uint32_t)G;
    p.gt = gt; p.st = stq; p.mtg = (uint32_t)mtg; p.mts = (uint32_t)mts;
    p.page = (uint32_t)page; p.rows = R;
    p.cap = (uint32_t)cap; p.nkb = (uint32_t)nkb;
    p.nsplit = nsplit; p.bps = (uint32_t)bps;
    p.causal = args->causal != 0 ? 1u : 0u;
    p.scale_log2 = attn_scale_log2(args->scale);
    if (f8) { p.k_scale = f8->k_scale; p.v_scale = f8->v_scale; }
    CUfunction f = nullptr;
    const std::string in_tag = dt_tag(in_dtype), out_tag = dt_tag(out_dtype);
    const std::string fmt = !f8 ? "" : f8->cache == B200_F8E5M2 ? "_e5m2" : "_e4m3";
    if (!rc) rc = get_func(c, "attn_kv_" + in_tag + fmt + "_d" + std::to_string(DB) + "_" + out_tag, &f);
    const unsigned smem = !f8 ? 1024 + (DB / 64) * (kAttnKvRows + 2 * kAttnKvStages * kAttnKvBlock) * 128 + kAttnKvBarBytes
                              : 1024 + (DB / 64) * (kAttnKvRows + 3 * kAttnKvBlock) * 128 + kAttnKvF8Stages * 2 * kAttnKvBlock * 128 +
                                    kAttnKvF8BarBytes;
    if (!rc) rc = attn_set_smem(c, f, smem);
    void* kargs[] = {&mq, &mk, &mv, &p};
    if (!rc) rc = launch(c, f, (unsigned)ctas, 1, 1, kAttnKvThreads, smem, 1, st, kargs);
    if (!rc && nsplit > 1) {
      rc = get_func(c, std::string(f8 ? "attn_kv_combine_fp8_" : "attn_kv_combine_") + out_tag, &f);
      void* cargs[] = {&p};
      if (!rc) rc = launch(c, f, (unsigned)((rows * (D / 4) + kAttnKvCombineThreads - 1) / kAttnKvCombineThreads), 1, 1,
                           kAttnKvCombineThreads, 0, 1, st, cargs);
    }
  }
  for (CUdeviceptr t : tmp)
    if (t) pool_free(c, t, st);   // stream-ordered: reusable once the kernels have drained
  return rc;
}

extern "C" int b200_attention_kvcache(b200_ctx* c, b200_stream s, b200_dtype in_dtype, b200_dtype out_dtype, b200_dptr q,
                                      const uint64_t* q_shape, const uint64_t* q_strides, b200_dptr k_cache, const uint64_t* kc_shape,
                                      const uint64_t* kc_strides, b200_dptr v_cache, const uint64_t* vc_shape, const uint64_t* vc_strides,
                                      b200_dptr block_table, const uint64_t* bt_shape, const uint64_t* bt_strides, b200_dptr cache_seqlens,
                                      b200_dptr out, const uint64_t* out_shape, const uint64_t* out_strides, b200_dptr lse,
                                      const b200_attention_args* args) {
  CTX_ENTER(c);
  return kv_attend(c, s, "attention_kvcache", in_dtype, nullptr, out_dtype, q, q_shape, q_strides, k_cache, kc_shape, kc_strides, v_cache,
                   vc_shape, vc_strides, block_table, bt_shape, bt_strides, cache_seqlens, out, out_shape, out_strides, lse, args);
}

extern "C" int b200_attention_kvcache_fp8(b200_ctx* c, b200_stream s, b200_dtype in_dtype, b200_dtype cache_dtype, b200_dtype out_dtype,
                                          b200_dptr q, const uint64_t* q_shape, const uint64_t* q_strides, b200_dptr k_cache,
                                          const uint64_t* kc_shape, const uint64_t* kc_strides, b200_dptr v_cache, const uint64_t* vc_shape,
                                          const uint64_t* vc_strides, b200_dptr block_table, const uint64_t* bt_shape,
                                          const uint64_t* bt_strides, b200_dptr cache_seqlens, b200_dptr k_scale, b200_dptr v_scale,
                                          b200_dptr out, const uint64_t* out_shape, const uint64_t* out_strides, b200_dptr lse,
                                          const b200_attention_args* args) {
  CTX_ENTER(c);
  const KvFp8 f8{cache_dtype, k_scale, v_scale};
  return kv_attend(c, s, "attention_kvcache_fp8", in_dtype, &f8, out_dtype, q, q_shape, q_strides, k_cache, kc_shape, kc_strides, v_cache,
                   vc_shape, vc_strides, block_table, bt_shape, bt_strides, cache_seqlens, out, out_shape, out_strides, lse, args);
}

// Scatter of new tokens into a paged KV cache (see cubecl_b200.h): one attn_kv_write launch, or attn_kv_write_fp8 (f8: an
// fp8 cache, quantized with its per-head scales).
static int kv_write(b200_ctx* c, b200_stream s, const char* what, b200_dtype dtype, const KvFp8* f8, b200_dptr k_new, const uint64_t* kn_shape,
                    const uint64_t* kn_strides, b200_dptr v_new, const uint64_t* vn_shape, const uint64_t* vn_strides,
                    b200_dptr k_cache, const uint64_t* kc_shape, const uint64_t* kc_strides, b200_dptr v_cache,
                    const uint64_t* vc_shape, const uint64_t* vc_strides, b200_dptr slot_mapping) {
  if (!kn_shape || !vn_shape || !kc_shape || !vc_shape) return fail(B200_ERR_INVALID_ARG, "%s: null shape", what);
  if (dtype != B200_F16 && dtype != B200_BF16) return fail(B200_ERR_UNSUPPORTED, "%s: dtype %d unsupported (f16, bf16)", what, (int)dtype);
  if (int rc0 = kv_check_fp8(what, f8)) return rc0;
  const b200_dtype cache_dtype = f8 ? f8->cache : dtype;
  const uint64_t B = kn_shape[0], Snew = kn_shape[1], Hkv = kn_shape[2], D = kn_shape[3];
  const uint64_t P = kc_shape[0], page = kc_shape[1];
  if (memcmp(vn_shape, kn_shape, 4 * sizeof(uint64_t)))
    return fail(B200_ERR_INVALID_ARG, "%s: v_new %s does not match k_new %s", what, attn_dims(vn_shape, 4).c_str(), attn_dims(kn_shape, 4).c_str());
  if (memcmp(vc_shape, kc_shape, 4 * sizeof(uint64_t))) return fail(B200_ERR_INVALID_ARG, "%s: v_cache does not match k_cache", what);
  if (kc_shape[2] != Hkv || kc_shape[3] != D)
    return fail(B200_ERR_INVALID_ARG, "%s: k_cache %s differs from k_new %s in heads or head dim", what, attn_dims(kc_shape, 4).c_str(),
                attn_dims(kn_shape, 4).c_str());
  if (D % 8) return fail(B200_ERR_UNSUPPORTED, "%s: head dim D = %llu must be a multiple of 8", what, (unsigned long long)D);
  const uint64_t units = B * Snew * Hkv * (D / 8);
  if (units == 0) return B200_OK;
  if (!k_new || !v_new || !k_cache || !v_cache || !slot_mapping) return fail(B200_ERR_INVALID_ARG, "%s: null device pointer", what);
  if (slot_mapping % 4) return fail(B200_ERR_INVALID_ARG, "%s: slot_mapping must be 4-byte aligned", what);
  if (int rc0 = kv_check_scales(what, f8)) return rc0;
  const AttnView kc = attn_view(k_cache, cache_dtype, kc_shape, kc_strides, kAttnBSHD), vc = attn_view(v_cache, cache_dtype, vc_shape, vc_strides, kAttnBSHD);
  int rc = attn_check_caches(what, kc, vc);
  if (rc) return rc;
  // the kernel moves 16-byte units: other views of the new tokens are gathered into a compact copy first
  AttnView kn = attn_view(k_new, dtype, kn_shape, kn_strides, kAttnBSHD), vn = attn_view(v_new, dtype, vn_shape, vn_strides, kAttnBSHD);
  CUstream st = resolve_stream(c, s);
  CUdeviceptr tmp[2] = {0, 0};
  rc = attn_stage(c, st, &kn, &tmp[0]);
  if (!rc) rc = attn_stage(c, st, &vn, &tmp[1]);
  if (!rc) {
    AttnKvWriteParams p{};
    p.kn = kn.ptr; p.vn = vn.ptr; p.kc = k_cache; p.vc = v_cache; p.slots = slot_mapping;
    p.kn_sb = kn.s_batch(); p.kn_st = kn.s_row(); p.kn_sh = kn.s_head();
    p.vn_sb = vn.s_batch(); p.vn_st = vn.s_row(); p.vn_sh = vn.s_head();
    p.kc_sp = kc.s_batch(); p.kc_sr = kc.s_row(); p.kc_sh = kc.s_head();
    p.vc_sp = vc.s_batch(); p.vc_sr = vc.s_row(); p.vc_sh = vc.s_head();
    p.units = units;
    p.Snew = (uint32_t)Snew; p.Hkv = (uint32_t)Hkv; p.D = (uint32_t)D; p.page = (uint32_t)page;
    p.slot_end = P * page;
    if (f8) {
      p.k_scale = f8->k_scale; p.v_scale = f8->v_scale;
      p.in_bf16 = dtype == B200_BF16 ? 1u : 0u;
      p.e5m2 = f8->cache == B200_F8E5M2 ? 1u : 0u;
    }
    CUfunction f = nullptr;
    rc = get_func(c, f8 ? "attn_kv_write_fp8" : "attn_kv_write", &f);
    void* kargs[] = {&p};
    const unsigned grid = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>((units + 255) / 256, (uint64_t)c->props.num_sms * 32));
    if (!rc) rc = launch(c, f, grid, 1, 1, 256, 0, 1, st, kargs);
  }
  for (CUdeviceptr t : tmp)
    if (t) pool_free(c, t, st);
  return rc;
}

extern "C" int b200_kvcache_write(b200_ctx* c, b200_stream s, b200_dtype dtype, b200_dptr k_new, const uint64_t* kn_shape,
                                  const uint64_t* kn_strides, b200_dptr v_new, const uint64_t* vn_shape, const uint64_t* vn_strides,
                                  b200_dptr k_cache, const uint64_t* kc_shape, const uint64_t* kc_strides, b200_dptr v_cache,
                                  const uint64_t* vc_shape, const uint64_t* vc_strides, b200_dptr slot_mapping) {
  CTX_ENTER(c);
  return kv_write(c, s, "kvcache_write", dtype, nullptr, k_new, kn_shape, kn_strides, v_new, vn_shape, vn_strides, k_cache, kc_shape,
                  kc_strides, v_cache, vc_shape, vc_strides, slot_mapping);
}

extern "C" int b200_kvcache_write_fp8(b200_ctx* c, b200_stream s, b200_dtype dtype, b200_dtype cache_dtype, b200_dptr k_new,
                                      const uint64_t* kn_shape, const uint64_t* kn_strides, b200_dptr v_new, const uint64_t* vn_shape,
                                      const uint64_t* vn_strides, b200_dptr k_cache, const uint64_t* kc_shape, const uint64_t* kc_strides,
                                      b200_dptr v_cache, const uint64_t* vc_shape, const uint64_t* vc_strides, b200_dptr slot_mapping,
                                      b200_dptr k_scale, b200_dptr v_scale) {
  CTX_ENTER(c);
  const KvFp8 f8{cache_dtype, k_scale, v_scale};
  return kv_write(c, s, "kvcache_write_fp8", dtype, &f8, k_new, kn_shape, kn_strides, v_new, vn_shape, vn_strides, k_cache, kc_shape,
                  kc_strides, v_cache, vc_shape, vc_strides, slot_mapping);
}

extern "C" int b200_reduce_debug(b200_ctx* c, b200_stream s, uint64_t* words4) {
  CTX_ENTER_DEVICE(c);
  if (!words4) return fail(B200_ERR_INVALID_ARG, "reduce_debug: null output");
  CUstream st = resolve_stream(c, s);
  CUdeviceptr ws;
  int rc = reduce_workspace(c, st, &ws);
  if (rc) return rc;
  CU_CHECK(g_drv.cuMemcpyDtoHAsync_p(words4, ws + kWsDebugOffset, 32, st));
  CU_CHECK(g_drv.cuStreamSynchronize_p(st));
  return B200_OK;
}

extern "C" int b200_into_contiguous(b200_ctx* c, b200_stream s, b200_dtype dtype, b200_dptr in, b200_dptr out, int rank,
                                    const uint64_t* shape, const uint64_t* strides) {
  CTX_ENTER(c);
  const size_t esz = dtype_size(dtype);
  if (!esz) return fail(B200_ERR_INVALID_ARG, "into_contiguous: unknown dtype %d", (int)dtype);
  if (rank < 1 || rank > 8 || !shape || !strides) return fail(B200_ERR_INVALID_ARG, "into_contiguous: bad rank/shape/strides");
  GatherParams p;
  memset(&p, 0, sizeof(p));
  p.in = in; p.out = out; p.rank = (uint32_t)rank; p.esz = (uint32_t)esz; p.n = 1;
  for (int i = 0; i < rank; ++i) { p.shape[i] = shape[i]; p.strides[i] = strides[i]; p.n *= shape[i]; }
  if (p.n == 0) return B200_OK;
  if (!in || !out) return fail(B200_ERR_INVALID_ARG, "into_contiguous: null device pointer");
  CUfunction f;
  int rc = get_func(c, "gather_strided", &f);
  if (rc) return rc;
  const unsigned grid = (unsigned)std::min<uint64_t>((p.n + 255) / 256, (uint64_t)c->props.num_sms * 32);
  void* args[] = {&p};
  return launch(c, f, std::max(1u, grid), 1, 1, 256, 0, 1, resolve_stream(c, s), args);
}

// ================================================================================================ collectives
extern "C" int b200_comm_get_unique_id(b200_ctx* c, void* id128) {
  CTX_ENTER_DEVICE(c);
  if (!id128) return fail(B200_ERR_INVALID_ARG, "null id");
  int rc = ensure_nccl();
  if (rc) return rc;
  ncclUniqueId id;
  NCCL_CHECK(g_nccl.GetUniqueId(&id));
  memcpy(id128, &id, sizeof(id));
  return B200_OK;
}

static std::vector<int> sorted_ids(const int* ids, int n) {
  std::vector<int> v(ids, ids + n);
  std::sort(v.begin(), v.end());
  return v;
}

extern "C" int b200_comm_init(b200_ctx* c, const int* device_ids, int n, const void* id128) {
  CTX_ENTER_DEVICE(c);
  if (!device_ids || n < 1 || !id128) return fail(B200_ERR_INVALID_ARG, "comm_init: bad arguments");
  int rc = ensure_nccl();
  if (rc) return rc;
  std::vector<int> key = sorted_ids(device_ids, n);
  if (c->comms.count(key)) return B200_OK;  // idempotent, like ensure_init_collective (client.rs:755-767)
  auto it = std::find(key.begin(), key.end(), c->device);
  if (it == key.end()) return fail(B200_ERR_INVALID_ARG, "comm_init: device %d is not in the device set", c->device);
  CommState cs;
  cs.rank = static_cast<int>(it - key.begin());
  cs.n = n;
  ncclUniqueId id;
  memcpy(&id, id128, sizeof(id));
  NCCL_CHECK(g_nccl.CommInitRank(&cs.comm, n, id, cs.rank));
  c->comms[key] = cs;
  return B200_OK;
}

extern "C" int b200_all_reduce(b200_ctx* c, b200_stream compute, b200_dptr src, b200_dptr dst, size_t bytes, b200_dtype dtype,
                               b200_comm_op op, const int* device_ids, int n) {
  CTX_ENTER_DEVICE(c);
  if (!device_ids || n < 1) return fail(B200_ERR_INVALID_ARG, "all_reduce: bad device set");
  int rc = ensure_nccl();
  if (rc) return rc;
  auto it = c->comms.find(sorted_ids(device_ids, n));
  if (it == c->comms.end()) return fail(B200_ERR_COMM, "all_reduce: no communicator for this device set (call b200_comm_init)");
  int nt;
  switch (dtype) {  // communication.rs:34-108
    case B200_F32: nt = ncclFloat32; break;
    case B200_F16: nt = ncclFloat16; break;
    case B200_BF16: nt = ncclBfloat16; break;
    case B200_F64: nt = ncclFloat64; break;
    case B200_I32: nt = ncclInt32; break;
    case B200_U32: nt = ncclUint32; break;
    case B200_I64: nt = ncclInt64; break;
    case B200_U64: nt = ncclUint64; break;
    case B200_I8: nt = ncclInt8; break;
    case B200_U8: nt = ncclUint8; break;
    default: return fail(B200_ERR_UNSUPPORTED, "all_reduce: dtype %d", (int)dtype);
  }
  const size_t esz = dtype_size(dtype);
  if (bytes % esz) return fail(B200_ERR_INVALID_ARG, "all_reduce: %zu bytes is not a multiple of the element size", bytes);
  CUstream cs = resolve_stream(c, compute);
  // compute -> comm dependency, then the collective on the comm stream (server.rs:749)
  CU_CHECK(g_drv.cuEventRecord_p(c->comm_event, cs));
  CU_CHECK(g_drv.cuStreamWaitEvent_p(c->comm_stream, c->comm_event, 0));
  NCCL_CHECK(g_nccl.AllReduce(reinterpret_cast<const void*>(src), reinterpret_cast<void*>(dst), bytes / esz, nt,
                              op == B200_COMM_MEAN ? ncclAvg : ncclSum, it->second.comm, c->comm_stream));
  return B200_OK;
}

extern "C" int b200_sync_collective(b200_ctx* c, b200_stream compute) {
  CTX_ENTER_DEVICE(c);
  CU_CHECK(g_drv.cuEventRecord_p(c->comm_event, c->comm_stream));
  CU_CHECK(g_drv.cuStreamWaitEvent_p(resolve_stream(c, compute), c->comm_event, 0));
  return B200_OK;
}

// ------------------------------------------------------------------------------------------------ peer-memory exchange

static int ensure_mailbox(b200_ctx* c) {
  if (c->mailbox) return B200_OK;
  CU_CHECK(g_drv.cuMemAlloc_p(&c->mailbox, kMailboxBytes));
  CU_CHECK(g_drv.cuMemsetD32Async_p(c->mailbox, 0, kMailboxBytes / 4, c->stream));
  CU_CHECK(g_drv.cuStreamSynchronize_p(c->stream));
  return B200_OK;
}

extern "C" int b200_p2p_export(b200_ctx* c, void* ipc_handle64, uint64_t* local_ptr, int64_t* pid) {
  CTX_ENTER_DEVICE(c);
  if (!ipc_handle64 || !local_ptr || !pid) return fail(B200_ERR_INVALID_ARG, "p2p_export: null argument");
  int rc = ensure_mailbox(c);
  if (rc) return rc;
  CUipcMemHandle h;
  static_assert(sizeof(CUipcMemHandle) == B200_IPC_HANDLE_BYTES, "IPC handle size");
  CU_CHECK(g_drv.cuIpcGetMemHandle_p(&h, c->mailbox));
  memcpy(ipc_handle64, &h, sizeof(h));
  *local_ptr = c->mailbox;
  *pid = static_cast<int64_t>(getpid());
  return B200_OK;
}

extern "C" int b200_p2p_connect(b200_ctx* c, const int* device_ids, int n, const void* ipc_handles, const uint64_t* local_ptrs,
                                const int64_t* pids) {
  CTX_ENTER_DEVICE(c);
  if (!device_ids || n < 1 || n > 8 || !ipc_handles || !local_ptrs || !pids)
    return fail(B200_ERR_INVALID_ARG, "p2p_connect: bad arguments (1..8 devices)");
  int rc = ensure_mailbox(c);
  if (rc) return rc;
  // the arrays are indexed like device_ids; ranks follow the SORTED device set (same keying as b200_comm_init)
  std::vector<int> key = sorted_ids(device_ids, n);
  if (c->p2p.count(key)) return B200_OK;
  P2PState st;
  st.n = n;
  unsigned mask = 0;
  for (int id : key) mask |= 1u << (static_cast<unsigned>(id) & 7u);
  const uint64_t set_off = static_cast<uint64_t>(mask & 0xFFu) * kMailboxSetBytes;
  for (int r = 0; r < n; ++r) {
    int src = -1;
    for (int j = 0; j < n; ++j)
      if (device_ids[j] == key[r]) src = j;
    if (key[r] == c->device) {
      st.rank = r;
      st.mailbox[r] = c->mailbox + set_off;
      continue;
    }
    if (pids[src] == static_cast<int64_t>(getpid())) {
      // same process (the reference's one-process model): enable peer access to that device's primary context
      CUdevice pd;
      CUcontext pctx;
      CU_CHECK(g_drv.cuDeviceGet_p(&pd, key[r]));
      int can = 0;
      CU_CHECK(g_drv.cuDeviceCanAccessPeer_p(&can, c->dev, pd));
      if (!can) return fail(B200_ERR_UNSUPPORTED, "p2p_connect: device %d cannot access device %d", c->device, key[r]);
      CU_CHECK(g_drv.cuDevicePrimaryCtxRetain_p(&pctx, pd));
      CUresult r2 = g_drv.cuCtxEnablePeerAccess_p(pctx, 0);
      g_drv.cuDevicePrimaryCtxRelease_p(pd);
      if (r2 != CUDA_SUCCESS && r2 != CUDA_ERROR_PEER_ACCESS_ALREADY_ENABLED)
        return fail(map_cu(r2), "cuCtxEnablePeerAccess(%d) failed: %s", key[r], cu_err(r2));
      st.mailbox[r] = local_ptrs[src] + set_off;
    } else {
      CUipcMemHandle h;
      memcpy(&h, static_cast<const char*>(ipc_handles) + static_cast<size_t>(src) * B200_IPC_HANDLE_BYTES, sizeof(h));
      CUdeviceptr mapped = 0;
      CUresult r2 = g_drv.cuIpcOpenMemHandle_p(&mapped, h, CU_IPC_MEM_LAZY_ENABLE_PEER_ACCESS);
      if (r2 != CUDA_SUCCESS) return fail(map_cu(r2), "cuIpcOpenMemHandle(device %d) failed: %s", key[r], cu_err(r2));
      st.opened.push_back(mapped);
      st.mailbox[r] = mapped + set_off;
    }
  }
  if (st.rank < 0) return fail(B200_ERR_INVALID_ARG, "p2p_connect: device %d is not in the device set", c->device);
  c->p2p[key] = st;
  return B200_OK;
}

static int reduce_all_reduce_impl(b200_ctx* c, b200_stream s, b200_reduce_op op, b200_dtype in_dtype, b200_dptr in, b200_dptr out,
                                  uint64_t n, uint64_t index_offset, const int* device_ids, int ndev) {
  const bool arg = (op == B200_REDUCE_ARGMAX || op == B200_REDUCE_ARGMIN);
  if (op != B200_REDUCE_SUM && !arg) return fail(B200_ERR_UNSUPPORTED, "reduce_all_reduce: SUM, ARGMAX and ARGMIN are fused");
  if (in_dtype != B200_F32) return fail(B200_ERR_UNSUPPORTED, "reduce_all_reduce: only f32 input is fused");
  if (!device_ids || ndev < 1) return fail(B200_ERR_INVALID_ARG, "reduce_all_reduce: bad device set");
  if (!in || !out || n == 0) return fail(B200_ERR_INVALID_ARG, "reduce_all_reduce: null pointer or empty input");
  if (arg && index_offset + n > (1ull << 32)) return fail(B200_ERR_UNSUPPORTED, "reduce_all_reduce: global indices must fit 32 bits");
  auto it = c->p2p.find(sorted_ids(device_ids, ndev));
  if (it == c->p2p.end()) return fail(B200_ERR_COMM, "reduce_all_reduce: device set not connected (call b200_p2p_connect)");
  P2PState& st = it->second;
  CUstream cs = resolve_stream(c, s);
  CUfunction f;
  int rc = get_func(c, op == B200_REDUCE_SUM ? "reduce_all_sum_f32_xgpu" : op == B200_REDUCE_ARGMAX ? "reduce_all_argmax_f32_xgpu" : "reduce_all_argmin_f32_xgpu", &f);
  if (rc) return rc;
  CUdeviceptr ws;
  rc = reduce_workspace(c, cs, &ws);
  if (rc) return rc;
  unsigned threads = (unsigned)std::min(512, std::max(32, atoi(opt(c, "reduce.threads", "512").c_str()))) / 32 * 32;
  unsigned bps = (unsigned)std::max(1, atoi(opt(c, "reduce.blocks_per_sm", "4").c_str()));
  const uint64_t want = (n / 4 + threads - 1) / threads;
  unsigned grid = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>(want, std::min<uint64_t>((uint64_t)c->props.num_sms * bps, kWsMaxBlocks)));
  ReduceParams p{};
  p.in = in; p.out = out; p.ws = ws;
  p.outer = 1; p.len = n; p.inner = 1;
  p.row_len = n; p.row_pitch = n; p.seg_len = n; p.nseg = 1; p.scale = 1.0f;
  p.flags = opt(c, "reduce.debug", "0") == "1" ? 1u : 0u;
  XgpuParams xg;
  memset(&xg, 0, sizeof(xg));
  for (int r = 0; r < st.n; ++r) xg.mailbox[r] = st.mailbox[r];
  xg.rank = (uint32_t)st.rank;
  xg.nranks = (uint32_t)st.n;
  xg.index_offset = index_offset;
  xg.epoch = st.epoch + 1;  // every rank calls in the same order (collective semantics), so epochs agree
  void* args[] = {&p, &xg};
  const bool pdl = cs == c->stream && c->pdl_prev_out != 0 && opt(c, "reduce.pdl", "on") == "on" &&
                   !(c->pdl_prev_out + 4 > in && c->pdl_prev_out < in + n * 4);
  rc = launch(c, f, grid, 1, 1, threads, 0, 1, cs, args, pdl);
  if (!rc && cs == c->stream) c->pdl_prev_out = out;
  if (!rc) st.epoch += 1;   // only a launch that really went out consumes the epoch (a failed call must not desynchronise the ranks)
  return rc;
}

extern "C" int b200_reduce_all_reduce(b200_ctx* c, b200_stream s, b200_reduce_op op, b200_dtype in_dtype, b200_dptr in,
                                      b200_dptr out, uint64_t n, const int* device_ids, int ndev) {
  CTX_ENTER(c);
  if (op != B200_REDUCE_SUM) return fail(B200_ERR_UNSUPPORTED, "reduce_all_reduce: SUM only (use b200_argreduce_all_reduce for arg ops)");
  return reduce_all_reduce_impl(c, s, op, in_dtype, in, out, n, 0, device_ids, ndev);
}

extern "C" int b200_argreduce_all_reduce(b200_ctx* c, b200_stream s, b200_reduce_op op, b200_dtype in_dtype, b200_dptr in,
                                         b200_dptr out, uint64_t n, uint64_t index_offset, const int* device_ids, int ndev) {
  CTX_ENTER(c);
  if (op != B200_REDUCE_ARGMAX && op != B200_REDUCE_ARGMIN) return fail(B200_ERR_INVALID_ARG, "argreduce_all_reduce: ARGMAX or ARGMIN");
  return reduce_all_reduce_impl(c, s, op, in_dtype, in, out, n, index_offset, device_ids, ndev);
}

// ================================================================================================ generators / probes
static int launch_fill(b200_ctx* c, b200_stream s, int dtype, uint64_t out, uint64_t n, FillParams p) {
  if (!fill_dtype_ok(dtype)) return fail(B200_ERR_UNSUPPORTED, "fill: dtype %d unsupported", dtype);
  if (n == 0) return B200_OK;
  CUfunction f;
  int rc = get_func(c, "fill_kernel", &f);
  if (rc) return rc;
  p.out = out; p.n = n; p.dtype = (uint32_t)dtype;
  const unsigned grid = (unsigned)std::min<uint64_t>((n + 255) / 256, (uint64_t)c->props.num_sms * 32);
  void* args[] = {&p};
  return launch(c, f, grid, 1, 1, 256, 0, 1, resolve_stream(c, s), args);
}

extern "C" int b200_fill_uniform(b200_ctx* c, b200_stream s, b200_dtype dtype, b200_dptr out, uint64_t n, uint64_t seed, float lo, float hi) {
  CTX_ENTER(c);
  FillParams p{};
  p.seed = seed; p.lo = lo; p.scale = hi - lo; p.mode = 0; p.modulus = 1;
  return launch_fill(c, s, dtype, out, n, p);
}

extern "C" int b200_fill_modulo(b200_ctx* c, b200_stream s, b200_dtype dtype, b200_dptr out, uint64_t n, uint32_t modulus) {
  CTX_ENTER(c);
  if (modulus == 0) return fail(B200_ERR_INVALID_ARG, "fill_modulo: modulus 0");
  FillParams p{};
  p.mode = 1; p.modulus = modulus;
  return launch_fill(c, s, dtype, out, n, p);
}

extern "C" int b200_probe_wmma(b200_ctx* c, b200_stream s, b200_dtype dtype, uint32_t n_iter, b200_dptr scratch, double* ops) {
  CTX_ENTER(c);
  CUfunction f;
  int rc = get_func(c, dtype == B200_BF16 ? "wmma_probe_bf16" : "wmma_probe_f16", &f);
  if (rc) return rc;
  const unsigned grid = (unsigned)c->props.num_sms * 32, block = 256;
  uint64_t sp = scratch;
  void* args[] = {&sp, &n_iter};
  rc = launch(c, f, grid, 1, 1, block, 0, 1, resolve_stream(c, s), args);
  if (!rc && ops) *ops = static_cast<double>(grid) * (block / 32) * 2.0 * 16 * 16 * 16 * n_iter;
  return rc;
}

// Tensor-core peak probe (wgmma_probe_* in gemm_wgmma.cu): one CTA per SM, two warpgroups each issuing 4 m64n256 wgmma per
// iteration on shared-memory operands.  K per instruction: 16 (bf16), 32 (e4m3).
static int probe_wgmma(b200_ctx* c, b200_stream s, const char* name, double k_per_instr, uint32_t n_iter, b200_dptr scratch, double* ops) {
  CUfunction f;
  int rc = get_func(c, name, &f);
  if (rc) return rc;
  const unsigned smem = 16384 + 32768 + 1024;
  CU_CHECK(g_drv.cuFuncSetAttribute_p(f, CU_FUNC_ATTRIBUTE_MAX_DYNAMIC_SHARED_SIZE_BYTES, (int)smem));
  const unsigned grid = (unsigned)std::max(1, c->props.num_sms);
  uint64_t sp = scratch;
  void* args[] = {&sp, &n_iter};
  rc = launch(c, f, grid, 1, 1, 384, smem, 1, resolve_stream(c, s), args);
  if (!rc && ops) *ops = static_cast<double>(grid) * 2 * n_iter * 4.0 * 2.0 * 64 * 256 * k_per_instr;
  return rc;
}

extern "C" int b200_probe_umma(b200_ctx* c, b200_stream s, uint32_t n_iter, b200_dptr scratch, double* ops) {
  CTX_ENTER_DEVICE(c);
  return probe_wgmma(c, s, "wgmma_probe_bf16", 16.0, n_iter, scratch, ops);
}

extern "C" int b200_probe_umma_kind(b200_ctx* c, b200_stream s, b200_dtype dtype, int block_scaled, uint32_t n_iter, b200_dptr scratch,
                                    double* ops) {
  CTX_ENTER_DEVICE(c);
  if (block_scaled) return fail(B200_ERR_UNSUPPORTED, "probe_umma_kind: sm_90 tensor cores have no block-scaled MMA");
  if (dtype == B200_BF16) return probe_wgmma(c, s, "wgmma_probe_bf16", 16.0, n_iter, scratch, ops);
  if (dtype == B200_F8E4M3) return probe_wgmma(c, s, "wgmma_probe_e4m3", 32.0, n_iter, scratch, ops);
  return fail(B200_ERR_UNSUPPORTED, "probe_umma_kind: bf16 or f8e4m3");
}

extern "C" int b200_probe_memread(b200_ctx* c, b200_stream s, b200_dptr buf, uint64_t bytes, b200_dptr scratch) {
  CTX_ENTER(c);
  CUfunction f;
  int rc = get_func(c, "memread_probe_vec4", &f);
  if (rc) return rc;
  const unsigned grid = (unsigned)c->props.num_sms * 32, block = 256;
  uint64_t lines = bytes / 16;
  const uint64_t per_pass = static_cast<uint64_t>(grid) * block;
  uint32_t steps = (uint32_t)((lines + per_pass - 1) / per_pass);
  uint64_t in = buf, out = scratch;
  void* args[] = {&in, &out, &lines, &steps};
  return launch(c, f, grid, 1, 1, block, 0, 1, resolve_stream(c, s), args);
}

// mode 0: write-only (memory_write.rs), mode 1: copy (memory_direct.rs); `bytes` per buffer
extern "C" int b200_probe_memwrite(b200_ctx* c, b200_stream s, b200_dptr dst, uint64_t bytes) {
  CTX_ENTER(c);
  CUfunction f;
  int rc = get_func(c, "memwrite_probe_vec4", &f);
  if (rc) return rc;
  const unsigned grid = (unsigned)c->props.num_sms * 32, block = 256;
  uint64_t lines = bytes / 16, out = dst;
  const uint64_t per_pass = static_cast<uint64_t>(grid) * block;
  uint32_t steps = (uint32_t)((lines + per_pass - 1) / per_pass);
  void* args[] = {&out, &lines, &steps};
  return launch(c, f, grid, 1, 1, block, 0, 1, resolve_stream(c, s), args);
}

extern "C" int b200_probe_memcopy(b200_ctx* c, b200_stream s, b200_dptr dst, b200_dptr src, uint64_t bytes) {
  CTX_ENTER(c);
  CUfunction f;
  int rc = get_func(c, "memcopy_probe_vec4", &f);
  if (rc) return rc;
  const unsigned grid = (unsigned)c->props.num_sms * 32, block = 256;
  uint64_t lines = bytes / 16, in = src, out = dst;
  const uint64_t per_pass = static_cast<uint64_t>(grid) * block;
  uint32_t steps = (uint32_t)((lines + per_pass - 1) / per_pass);
  void* args[] = {&in, &out, &lines, &steps};
  return launch(c, f, grid, 1, 1, block, 0, 1, resolve_stream(c, s), args);
}
