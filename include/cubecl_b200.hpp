// cubecl_b200.hpp -- header-only C++ host layer above the C ABI (include/cubecl_b200.h).
//
// The reference's host side is Rust; this image has no Rust toolchain, so this is the compiled-language mirror of the
// reference's launch surface for the dense-LA path (the Python mirror in cubecl_b200/ serves the tests and the bench):
//
//   cubecl::ComputeClient   crates/cubecl-runtime/src/client.rs:44-48  (create_from_slice:452, empty:654, read_one:256,
//                           sync:1013, memory_usage:1048); one client per device (R::client(device))
//   cubecl::Handle          crates/cubecl-runtime/src/server/handle.rs:10-21  (ref-counted pool slice)
//   cubecl::TensorHandle    crates/cubecl-std/src/tensor/handle.rs:13-150     (handle + shape + strides in elements + dtype)
//   cubecl::matmul::launch  cubek matmul::launch; shape rule crates/cubecl-zspace/src/shape.rs:489-517
//   cubecl::reduce::launch  cubek reduce::launch; semantics examples/sum_things/src/lib.rs:6-33
//
// Error behaviour mirrors the reference: launch never throws; failures are queued on the client and surface as
// ServerError at the next sync()/read_one() (crates/cubecl-cuda/src/compute/server.rs:269-284,981-1002).
#pragma once
#include <cstdint>
#include <cstring>
#include <memory>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "cubecl_b200.h"

namespace cubecl {

struct ServerError : std::runtime_error {
  using std::runtime_error::runtime_error;
};
struct MatmulShapeError : std::invalid_argument {
  using std::invalid_argument::invalid_argument;
};

enum class DType : int { F32 = B200_F32, F16 = B200_F16, BF16 = B200_BF16, U32 = B200_U32, U8 = B200_U8, I8 = B200_I8,
                         F8E4M3 = B200_F8E4M3, F8E5M2 = B200_F8E5M2,
                         F4E2M1X2 = B200_F4E2M1X2,  // one element = one byte holding two e2m1 values
                         UE8M0 = B200_UE8M0 };
inline size_t dtype_size(DType d) {
  switch (d) {
    case DType::F16: case DType::BF16: return 2;
    case DType::F32: case DType::U32: return 4;
    default: return 1;
  }
}

using Shape = std::vector<uint64_t>;
using Strides = std::vector<uint64_t>;

inline Strides contiguous_strides(const Shape& shape) {
  Strides s(shape.size());
  uint64_t acc = 1;
  for (size_t i = shape.size(); i-- > 0;) { s[i] = acc; acc *= shape[i]; }
  return s;
}

/// calculate_matmul_output (crates/cubecl-zspace/src/shape.rs:489-517)
inline Shape calculate_matmul_output(const Shape& lhs, const Shape& rhs) {
  const size_t rank = lhs.size();
  if (rank != rhs.size()) throw MatmulShapeError("RankMismatch");
  if (rank < 2) throw MatmulShapeError("matmul needs rank >= 2");
  if (lhs[rank - 1] != rhs[rank - 2]) throw MatmulShapeError("IncompatibleShapes");
  Shape out;
  for (size_t i = 0; i + 2 < rank; ++i) {
    if (lhs[i] == rhs[i] || rhs[i] == 1) out.push_back(lhs[i]);
    else if (lhs[i] == 1) out.push_back(rhs[i]);
    else throw MatmulShapeError("IncompatibleDims");
  }
  out.push_back(lhs[rank - 2]);
  out.push_back(rhs[rank - 1]);
  return out;
}

class ComputeClient;

/// Pooled device buffer; the last copy returns it to the pool.
class Handle {
 public:
  Handle() = default;
  uint64_t ptr() const { return rec_ ? rec_->ptr : 0; }
  size_t size() const { return rec_ ? rec_->size : 0; }

 private:
  friend class ComputeClient;
  struct Rec {
    b200_ctx* ctx;
    uint64_t ptr;
    size_t size;
    Rec(b200_ctx* c, uint64_t p, size_t s) : ctx(c), ptr(p), size(s) {}
    Rec(const Rec&) = delete;
    Rec& operator=(const Rec&) = delete;
    ~Rec() { if (ctx && ptr) b200_free(ctx, ptr); }
  };
  std::shared_ptr<Rec> rec_;
};

class ComputeClient {
 public:
  explicit ComputeClient(int device = 0) : device_(device) {
    if (b200_init(device, &ctx_) != B200_OK) throw ServerError(std::string("b200_init: ") + b200_last_error());
  }
  ~ComputeClient() { if (ctx_) b200_destroy(ctx_); }
  ComputeClient(const ComputeClient&) = delete;
  ComputeClient& operator=(const ComputeClient&) = delete;

  b200_ctx* raw() const { return ctx_; }
  int device() const { return device_; }

  Handle empty(size_t size) {
    uint64_t p = 0;
    check(b200_alloc(ctx_, size, &p));
    Handle h;
    h.rec_ = std::shared_ptr<Handle::Rec>(new Handle::Rec{ctx_, p, size});  // in place: a temporary Rec would free the block
    return h;
  }
  Handle create_from_slice(const void* data, size_t bytes) {
    Handle h = empty(bytes);
    if (bytes) { check(b200_write(ctx_, nullptr, h.ptr(), data, bytes)); check(b200_sync(ctx_, nullptr)); }
    return h;
  }
  /// Blocking read of the whole buffer; surfaces deferred errors first (Result<Bytes, ServerError>).
  std::vector<uint8_t> read_one(const Handle& h) {
    std::vector<uint8_t> out(h.size());
    if (h.size()) check(b200_read(ctx_, nullptr, out.data(), h.ptr(), h.size()));
    sync();
    return out;
  }
  void sync() {
    if (b200_sync(ctx_, nullptr) != B200_OK) errors_.push_back(b200_last_error());
    flush();
  }
  void flush() {
    if (errors_.empty()) return;
    std::string msg = "ServerUnhealthy:";
    for (auto& e : errors_) msg += " " + e + ";";
    errors_.clear();
    throw ServerError(msg);
  }
  void defer(std::string e) { errors_.push_back(std::move(e)); }
  std::pair<uint64_t, uint64_t> memory_usage() {
    uint64_t a = 0, b = 0;
    check(b200_memory_usage(ctx_, &a, &b));
    return {a, b};
  }
  void set_option(const char* key, const char* value) { check(b200_set_option(ctx_, key, value)); }

 private:
  void check(int rc) {
    if (rc != B200_OK) throw ServerError(b200_last_error());
  }
  b200_ctx* ctx_ = nullptr;
  int device_;
  std::vector<std::string> errors_;
};

struct TensorHandle {
  Handle handle;
  Shape shape;
  Strides strides;  // elements
  DType dtype;

  static TensorHandle new_contiguous(Shape shape, Handle handle, DType dtype) {
    Strides st = contiguous_strides(shape);
    return TensorHandle{std::move(handle), std::move(shape), std::move(st), dtype};
  }
  static TensorHandle empty(ComputeClient& client, Shape shape, DType dtype) {
    uint64_t n = 1;
    for (auto s : shape) n *= s;
    return new_contiguous(std::move(shape), client.empty(n ? n * dtype_size(dtype) : 1), dtype);
  }
  /// Swap the last two dims without moving data (MatrixBatchLayout::MildlyPermuted{transposed}).
  TensorHandle transposed() const {
    TensorHandle t = *this;
    const size_t r = shape.size();
    std::swap(t.shape[r - 1], t.shape[r - 2]);
    std::swap(t.strides[r - 1], t.strides[r - 2]);
    return t;
  }
};

namespace matmul {
/// out = lhs @ rhs, f32 accumulation, batch dims broadcast.  Errors are deferred to client.sync().
inline void launch(ComputeClient& client, const TensorHandle& lhs, const TensorHandle& rhs, const TensorHandle& out) {
  const int rank = static_cast<int>(lhs.shape.size());
  if (rhs.shape.size() != lhs.shape.size() || out.shape.size() != lhs.shape.size() || lhs.dtype != rhs.dtype) {
    client.defer("InvalidArgument: matmul operands must have equal rank and dtype");
    return;
  }
  const int rc = b200_matmul(client.raw(), nullptr, static_cast<b200_dtype>(lhs.dtype), static_cast<b200_dtype>(out.dtype),
                             lhs.handle.ptr(), rhs.handle.ptr(), out.handle.ptr(), rank, lhs.shape.data(), lhs.strides.data(),
                             rhs.shape.data(), rhs.strides.data(), out.shape.data(), out.strides.data());
  if (rc != B200_OK) client.defer(b200_last_error());
}
/// Block-scaled (MX) matmul, the GEMM-level form of MmaDefinition::new_scaled / execute_scaled
/// (crates/cubecl-core/src/frontend/cmma.rs:438-460, 798-840): lhs [.., M, K] and rhs [.., N, K] K-contiguous (fp8, or both
/// F4E2M1X2 with K/2 bytes per row), scales [.., rows, K/scale_block] (UE8M0 for block 32; e4m3 bytes for NVFP4, block 16).
inline void launch_scaled(ComputeClient& client, const TensorHandle& lhs, const TensorHandle& rhs, const TensorHandle& lhs_scales,
                          const TensorHandle& rhs_scales, const TensorHandle& out, int scale_block = 32, bool scales_packed = false) {
  const size_t r = lhs.shape.size();
  if (r < 2 || rhs.shape.size() != r || out.shape.size() != r || lhs.shape[r - 1] != rhs.shape[r - 1]) {
    client.defer("InvalidArgument: matmul_scaled needs lhs [..,M,K] and rhs [..,N,K] of equal rank and K");
    return;
  }
  uint64_t batch = 1;
  for (size_t i = 0; i + 2 < r; ++i) batch *= lhs.shape[i];
  const uint64_t k = lhs.shape[r - 1] * (lhs.dtype == DType::F4E2M1X2 ? 2 : 1);
  const int rc = b200_matmul_scaled(client.raw(), nullptr, static_cast<b200_dtype>(lhs.dtype), static_cast<b200_dtype>(rhs.dtype),
                                    static_cast<b200_dtype>(out.dtype), lhs.handle.ptr(), rhs.handle.ptr(), lhs_scales.handle.ptr(),
                                    rhs_scales.handle.ptr(), out.handle.ptr(), batch, lhs.shape[r - 2], rhs.shape[r - 2], k, scale_block,
                                    scales_packed ? 1 : 0);
  if (rc != B200_OK) client.defer(b200_last_error());
}
/// out (contiguous [batch, m, n], F32 / BF16 / F16) = deq(lhs) x deq(rhs)^T of two integer-quantized operands on the s8 tensor
/// cores, scales applied inside the GEMM; see b200_matmul_quantized in cubecl_b200.h for the contract. Errors deferred.
inline void launch_quantized(ComputeClient& client, const b200_quant_operand& lhs, const b200_quant_operand& rhs, const TensorHandle& out,
                             uint64_t batch, uint64_t m, uint64_t n, uint64_t k) {
  const int rc = b200_matmul_quantized(client.raw(), nullptr, &lhs, &rhs, static_cast<b200_dtype>(out.dtype), out.handle.ptr(),
                                       batch, m, n, k);
  if (rc != B200_OK) client.defer(b200_last_error());
}
}  // namespace matmul

namespace conv {
/// 2-D convolution: x [N, H, W, C] (NHWC), w [Cout, KH, KW, C], out [N, OH, OW, Cout]; f32 accumulation, optional fused epilogue
/// (nullptr = none).  See b200_conv2d in cubecl_b200.h for the contract.  Errors are deferred to client.sync().
inline void launch(ComputeClient& client, const TensorHandle& x, const TensorHandle& w, const TensorHandle& out,
                   const b200_conv2d_args& args, const b200_epilogue* epilogue = nullptr) {
  if (x.shape.size() != 4 || w.shape.size() != 4 || out.shape.size() != 4 || x.dtype != w.dtype) {
    client.defer("InvalidArgument: conv2d needs rank-4 x, w and out, and x and w of one dtype");
    return;
  }
  const int rc = b200_conv2d(client.raw(), nullptr, static_cast<b200_dtype>(x.dtype), static_cast<b200_dtype>(out.dtype),
                             x.handle.ptr(), x.shape.data(), x.strides.data(), w.handle.ptr(), w.shape.data(), w.strides.data(),
                             out.handle.ptr(), out.shape.data(), out.strides.data(), &args, epilogue);
  if (rc != B200_OK) client.defer(b200_last_error());
}

/// Input gradient: dy [N, OH, OW, Cout], w [Cout, KH, KW, C] -> dx [N, H, W, C].  See b200_conv2d_backward_data.  Errors are
/// deferred to client.sync().
inline void backward_data(ComputeClient& client, const TensorHandle& dy, const TensorHandle& w, const TensorHandle& dx,
                          const b200_conv2d_args& args) {
  if (dy.shape.size() != 4 || w.shape.size() != 4 || dx.shape.size() != 4 || dy.dtype != w.dtype) {
    client.defer("InvalidArgument: conv2d_backward_data needs rank-4 dy, w and dx, and dy and w of one dtype");
    return;
  }
  const int rc = b200_conv2d_backward_data(client.raw(), nullptr, static_cast<b200_dtype>(dy.dtype), static_cast<b200_dtype>(dx.dtype),
                                           dy.handle.ptr(), dy.shape.data(), dy.strides.data(), w.handle.ptr(), w.shape.data(),
                                           w.strides.data(), dx.handle.ptr(), dx.shape.data(), dx.strides.data(), &args);
  if (rc != B200_OK) client.defer(b200_last_error());
}

/// Weight gradient: x [N, H, W, C], dy [N, OH, OW, Cout] -> dw [Cout, KH, KW, C].  The bias gradient is reduce (sum) over
/// axis 0 of dy viewed as [N * OH * OW, Cout].  See b200_conv2d_backward_weight.  Errors are deferred to client.sync().
inline void backward_weight(ComputeClient& client, const TensorHandle& x, const TensorHandle& dy, const TensorHandle& dw,
                            const b200_conv2d_args& args) {
  if (x.shape.size() != 4 || dy.shape.size() != 4 || dw.shape.size() != 4 || x.dtype != dy.dtype) {
    client.defer("InvalidArgument: conv2d_backward_weight needs rank-4 x, dy and dw, and x and dy of one dtype");
    return;
  }
  const int rc = b200_conv2d_backward_weight(client.raw(), nullptr, static_cast<b200_dtype>(x.dtype), static_cast<b200_dtype>(dw.dtype),
                                             x.handle.ptr(), x.shape.data(), x.strides.data(), dy.handle.ptr(), dy.shape.data(),
                                             dy.strides.data(), dw.handle.ptr(), dw.shape.data(), dw.strides.data(), &args);
  if (rc != B200_OK) client.defer(b200_last_error());
}

/// Grouped / depthwise convolution: w [Cout, KH, KW, C / groups].  See b200_conv2d_grouped.  Errors are deferred to client.sync().
inline void launch_grouped(ComputeClient& client, const TensorHandle& x, const TensorHandle& w, const TensorHandle& out,
                           const b200_conv2d_args& args, uint32_t groups, const b200_epilogue* epilogue = nullptr) {
  if (x.shape.size() != 4 || w.shape.size() != 4 || out.shape.size() != 4 || x.dtype != w.dtype) {
    client.defer("InvalidArgument: conv2d_grouped needs rank-4 x, w and out, and x and w of one dtype");
    return;
  }
  const int rc = b200_conv2d_grouped(client.raw(), nullptr, static_cast<b200_dtype>(x.dtype), static_cast<b200_dtype>(out.dtype),
                                     x.handle.ptr(), x.shape.data(), x.strides.data(), w.handle.ptr(), w.shape.data(), w.strides.data(),
                                     out.handle.ptr(), out.shape.data(), out.strides.data(), &args, groups, epilogue);
  if (rc != B200_OK) client.defer(b200_last_error());
}

/// Input gradient of launch_grouped.  See b200_conv2d_grouped_backward_data.  Errors are deferred to client.sync().
inline void backward_data_grouped(ComputeClient& client, const TensorHandle& dy, const TensorHandle& w, const TensorHandle& dx,
                                  const b200_conv2d_args& args, uint32_t groups) {
  if (dy.shape.size() != 4 || w.shape.size() != 4 || dx.shape.size() != 4 || dy.dtype != w.dtype) {
    client.defer("InvalidArgument: conv2d_grouped_backward_data needs rank-4 dy, w and dx, and dy and w of one dtype");
    return;
  }
  const int rc = b200_conv2d_grouped_backward_data(client.raw(), nullptr, static_cast<b200_dtype>(dy.dtype),
                                                   static_cast<b200_dtype>(dx.dtype), dy.handle.ptr(), dy.shape.data(),
                                                   dy.strides.data(), w.handle.ptr(), w.shape.data(), w.strides.data(), dx.handle.ptr(),
                                                   dx.shape.data(), dx.strides.data(), &args, groups);
  if (rc != B200_OK) client.defer(b200_last_error());
}

/// Weight gradient of launch_grouped: dw [Cout, KH, KW, C / groups].  See b200_conv2d_grouped_backward_weight.
inline void backward_weight_grouped(ComputeClient& client, const TensorHandle& x, const TensorHandle& dy, const TensorHandle& dw,
                                    const b200_conv2d_args& args, uint32_t groups) {
  if (x.shape.size() != 4 || dy.shape.size() != 4 || dw.shape.size() != 4 || x.dtype != dy.dtype) {
    client.defer("InvalidArgument: conv2d_grouped_backward_weight needs rank-4 x, dy and dw, and x and dy of one dtype");
    return;
  }
  const int rc = b200_conv2d_grouped_backward_weight(client.raw(), nullptr, static_cast<b200_dtype>(x.dtype),
                                                     static_cast<b200_dtype>(dw.dtype), x.handle.ptr(), x.shape.data(),
                                                     x.strides.data(), dy.handle.ptr(), dy.shape.data(), dy.strides.data(),
                                                     dw.handle.ptr(), dw.shape.data(), dw.strides.data(), &args, groups);
  if (rc != B200_OK) client.defer(b200_last_error());
}
}  // namespace conv

namespace conv3d {
/// 3-D convolution: x [N, D, H, W, C] (NDHWC), w [Cout, KD, KH, KW, C], out [N, OD, OH, OW, Cout]; f32 accumulation, optional
/// fused epilogue (nullptr = none).  See b200_conv3d in cubecl_b200.h.  Errors are deferred to client.sync().
inline void launch(ComputeClient& client, const TensorHandle& x, const TensorHandle& w, const TensorHandle& out,
                   const b200_conv3d_args& args, const b200_epilogue* epilogue = nullptr) {
  if (x.shape.size() != 5 || w.shape.size() != 5 || out.shape.size() != 5 || x.dtype != w.dtype) {
    client.defer("InvalidArgument: conv3d needs rank-5 x, w and out, and x and w of one dtype");
    return;
  }
  const int rc = b200_conv3d(client.raw(), nullptr, static_cast<b200_dtype>(x.dtype), static_cast<b200_dtype>(out.dtype),
                             x.handle.ptr(), x.shape.data(), x.strides.data(), w.handle.ptr(), w.shape.data(), w.strides.data(),
                             out.handle.ptr(), out.shape.data(), out.strides.data(), &args, epilogue);
  if (rc != B200_OK) client.defer(b200_last_error());
}

/// Input gradient: dy [N, OD, OH, OW, Cout], w [Cout, KD, KH, KW, C] -> dx [N, D, H, W, C].  See b200_conv3d_backward_data.
/// Errors are deferred to client.sync().
inline void backward_data(ComputeClient& client, const TensorHandle& dy, const TensorHandle& w, const TensorHandle& dx,
                          const b200_conv3d_args& args) {
  if (dy.shape.size() != 5 || w.shape.size() != 5 || dx.shape.size() != 5 || dy.dtype != w.dtype) {
    client.defer("InvalidArgument: conv3d_backward_data needs rank-5 dy, w and dx, and dy and w of one dtype");
    return;
  }
  const int rc = b200_conv3d_backward_data(client.raw(), nullptr, static_cast<b200_dtype>(dy.dtype), static_cast<b200_dtype>(dx.dtype),
                                           dy.handle.ptr(), dy.shape.data(), dy.strides.data(), w.handle.ptr(), w.shape.data(),
                                           w.strides.data(), dx.handle.ptr(), dx.shape.data(), dx.strides.data(), &args);
  if (rc != B200_OK) client.defer(b200_last_error());
}

/// Weight gradient: x [N, D, H, W, C], dy [N, OD, OH, OW, Cout] -> dw [Cout, KD, KH, KW, C].  The bias gradient is reduce (sum)
/// over axis 0 of dy viewed as [N * OD * OH * OW, Cout].  See b200_conv3d_backward_weight.  Errors are deferred to client.sync().
inline void backward_weight(ComputeClient& client, const TensorHandle& x, const TensorHandle& dy, const TensorHandle& dw,
                            const b200_conv3d_args& args) {
  if (x.shape.size() != 5 || dy.shape.size() != 5 || dw.shape.size() != 5 || x.dtype != dy.dtype) {
    client.defer("InvalidArgument: conv3d_backward_weight needs rank-5 x, dy and dw, and x and dy of one dtype");
    return;
  }
  const int rc = b200_conv3d_backward_weight(client.raw(), nullptr, static_cast<b200_dtype>(x.dtype), static_cast<b200_dtype>(dw.dtype),
                                             x.handle.ptr(), x.shape.data(), x.strides.data(), dy.handle.ptr(), dy.shape.data(),
                                             dy.strides.data(), dw.handle.ptr(), dw.shape.data(), dw.strides.data(), &args);
  if (rc != B200_OK) client.defer(b200_last_error());
}
}  // namespace conv3d

namespace conv_transpose {
/// Transposed convolution, 2-D or 3-D by rank: x [N, (D,) H, W, Cin], w [Cin, (KD,) KH, KW, Cout], out [N, (OD,) OH, OW, Cout]
/// (out's shape gives the output padding); f32 accumulation, optional fused epilogue.  args: b200_conv2d_args (rank 4) or
/// b200_conv3d_args (rank 5).  See b200_conv_transpose2d in cubecl_b200.h.  Errors are deferred to client.sync().
inline void launch(ComputeClient& client, const TensorHandle& x, const TensorHandle& w, const TensorHandle& out,
                   const b200_conv2d_args& args, const b200_epilogue* epilogue = nullptr) {
  if (x.shape.size() != 4 || w.shape.size() != 4 || out.shape.size() != 4 || x.dtype != w.dtype) {
    client.defer("InvalidArgument: conv_transpose2d needs rank-4 x, w and out, and x and w of one dtype");
    return;
  }
  const int rc = b200_conv_transpose2d(client.raw(), nullptr, static_cast<b200_dtype>(x.dtype), static_cast<b200_dtype>(out.dtype),
                                       x.handle.ptr(), x.shape.data(), x.strides.data(), w.handle.ptr(), w.shape.data(),
                                       w.strides.data(), out.handle.ptr(), out.shape.data(), out.strides.data(), &args, epilogue);
  if (rc != B200_OK) client.defer(b200_last_error());
}
inline void launch(ComputeClient& client, const TensorHandle& x, const TensorHandle& w, const TensorHandle& out,
                   const b200_conv3d_args& args, const b200_epilogue* epilogue = nullptr) {
  if (x.shape.size() != 5 || w.shape.size() != 5 || out.shape.size() != 5 || x.dtype != w.dtype) {
    client.defer("InvalidArgument: conv_transpose3d needs rank-5 x, w and out, and x and w of one dtype");
    return;
  }
  const int rc = b200_conv_transpose3d(client.raw(), nullptr, static_cast<b200_dtype>(x.dtype), static_cast<b200_dtype>(out.dtype),
                                       x.handle.ptr(), x.shape.data(), x.strides.data(), w.handle.ptr(), w.shape.data(),
                                       w.strides.data(), out.handle.ptr(), out.shape.data(), out.strides.data(), &args, epilogue);
  if (rc != B200_OK) client.defer(b200_last_error());
}
}  // namespace conv_transpose

namespace attention {
/// Fused scaled-dot-product attention, forward: q [B, Hq, Sq, D], k and v [B, Hkv, Sk, D], out [B, Hq, Sq, D] (views by
/// strides); lse: nullptr or a compact f32 [B, Hq, Sq] tensor receiving the row log-sum-exp.  See b200_attention in
/// cubecl_b200.h.  Errors are deferred to client.sync().
inline void launch(ComputeClient& client, const TensorHandle& q, const TensorHandle& k, const TensorHandle& v, const TensorHandle& out,
                   float scale, bool causal = false, const TensorHandle* lse = nullptr) {
  if (q.shape.size() != 4 || k.shape.size() != 4 || v.shape.size() != 4 || out.shape.size() != 4 || q.dtype != k.dtype || q.dtype != v.dtype) {
    client.defer("InvalidArgument: attention needs rank-4 q, k, v and out, and q, k and v of one dtype");
    return;
  }
  const b200_attention_args args{scale, causal ? 1 : 0};
  const int rc = b200_attention(client.raw(), nullptr, static_cast<b200_dtype>(q.dtype), static_cast<b200_dtype>(out.dtype), q.handle.ptr(),
                                q.shape.data(), q.strides.data(), k.handle.ptr(), k.shape.data(), k.strides.data(), v.handle.ptr(),
                                v.shape.data(), v.strides.data(), out.handle.ptr(), out.shape.data(), out.strides.data(),
                                lse ? lse->handle.ptr() : 0, &args);
  if (rc != B200_OK) client.defer(b200_last_error());
}

/// Fused scaled-dot-product attention, backward: dq [B, Hq, Sq, D], dk and dv [B, Hkv, Sk, D] (one grad dtype) from q, k, v,
/// the forward's out and lse (compact f32 [B, Hq, Sq]) and dout.  See b200_attention_backward in cubecl_b200.h.  Errors are
/// deferred to client.sync().
inline void launch_backward(ComputeClient& client, const TensorHandle& q, const TensorHandle& k, const TensorHandle& v, const TensorHandle& out,
                            const TensorHandle& dout, const TensorHandle& lse, const TensorHandle& dq, const TensorHandle& dk,
                            const TensorHandle& dv, float scale, bool causal = false) {
  for (const TensorHandle* t : {&q, &k, &v, &out, &dout, &dq, &dk, &dv}) {
    if (t->shape.size() != 4) {
      client.defer("InvalidArgument: attention backward needs rank-4 q, k, v, out, dout, dq, dk and dv");
      return;
    }
  }
  if (q.dtype != k.dtype || q.dtype != v.dtype || q.dtype != dout.dtype || dq.dtype != dk.dtype || dq.dtype != dv.dtype) {
    client.defer("InvalidArgument: attention backward needs q, k, v and dout of one dtype and dq, dk and dv of one dtype");
    return;
  }
  const b200_attention_args args{scale, causal ? 1 : 0};
  const int rc = b200_attention_backward(
      client.raw(), nullptr, static_cast<b200_dtype>(q.dtype), static_cast<b200_dtype>(out.dtype), static_cast<b200_dtype>(dq.dtype),
      q.handle.ptr(), q.shape.data(), q.strides.data(), k.handle.ptr(), k.shape.data(), k.strides.data(), v.handle.ptr(), v.shape.data(),
      v.strides.data(), out.handle.ptr(), out.shape.data(), out.strides.data(), dout.handle.ptr(), dout.shape.data(), dout.strides.data(),
      lse.handle.ptr(), dq.handle.ptr(), dq.shape.data(), dq.strides.data(), dk.handle.ptr(), dk.shape.data(), dk.strides.data(),
      dv.handle.ptr(), dv.shape.data(), dv.strides.data(), &args);
  if (rc != B200_OK) client.defer(b200_last_error());
}

/// Variable-length (packed) attention, forward: q [Tq, Hq, D], k and v [Tk, Hkv, D], out [Tq, Hq, D] (views by strides);
/// sequence b owns rows [cu_q[b], cu_q[b + 1]) of q and [cu_k[b], cu_k[b + 1]) of k and v (compact i32 [B + 1] tensors read on
/// the device); window (left, right), -1 unbounded, (-1, 0) bottom-right causal.  lse: nullptr or a compact f32 [Hq, Tq]
/// tensor.  See b200_attention_varlen in cubecl_b200.h.  Errors are deferred to client.sync().
inline void launch_varlen(ComputeClient& client, const TensorHandle& q, const TensorHandle& k, const TensorHandle& v,
                          const TensorHandle& cu_seqlens_q, const TensorHandle& cu_seqlens_k, int32_t max_seqlen_q, int32_t max_seqlen_k,
                          const TensorHandle& out, float scale, int32_t window_left = -1, int32_t window_right = -1,
                          const TensorHandle* lse = nullptr) {
  if (q.shape.size() != 3 || k.shape.size() != 3 || v.shape.size() != 3 || out.shape.size() != 3 || q.dtype != k.dtype ||
      q.dtype != v.dtype || cu_seqlens_q.shape.size() != 1 || cu_seqlens_q.shape != cu_seqlens_k.shape || cu_seqlens_q.shape[0] < 1) {
    client.defer("InvalidArgument: attention_varlen needs rank-3 q, k, v and out of one input dtype and cu arrays [B + 1] of one length");
    return;
  }
  const b200_attention_varlen_args args{scale, window_left, window_right, max_seqlen_q, max_seqlen_k};
  const int rc = b200_attention_varlen(
      client.raw(), nullptr, static_cast<b200_dtype>(q.dtype), static_cast<b200_dtype>(out.dtype), q.handle.ptr(), q.shape.data(),
      q.strides.data(), k.handle.ptr(), k.shape.data(), k.strides.data(), v.handle.ptr(), v.shape.data(), v.strides.data(),
      cu_seqlens_q.handle.ptr(), cu_seqlens_k.handle.ptr(), cu_seqlens_q.shape[0] - 1, out.handle.ptr(), out.shape.data(),
      out.strides.data(), lse ? lse->handle.ptr() : 0, &args);
  if (rc != B200_OK) client.defer(b200_last_error());
}

/// Variable-length (packed) attention, backward: dq [Tq, Hq, D], dk and dv [Tk, Hkv, D] (one grad dtype) from q, k, v, the
/// forward's out and lse (compact f32 [Hq, Tq]) and dout, with the forward's offsets, window and scale.  See
/// b200_attention_varlen_backward in cubecl_b200.h.  Errors are deferred to client.sync().
inline void launch_varlen_backward(ComputeClient& client, const TensorHandle& q, const TensorHandle& k, const TensorHandle& v,
                                   const TensorHandle& out, const TensorHandle& dout, const TensorHandle& lse,
                                   const TensorHandle& cu_seqlens_q, const TensorHandle& cu_seqlens_k, int32_t max_seqlen_q,
                                   int32_t max_seqlen_k, const TensorHandle& dq, const TensorHandle& dk, const TensorHandle& dv, float scale,
                                   int32_t window_left = -1, int32_t window_right = -1) {
  for (const TensorHandle* t : {&q, &k, &v, &out, &dout, &dq, &dk, &dv}) {
    if (t->shape.size() != 3) {
      client.defer("InvalidArgument: attention_varlen backward needs rank-3 q, k, v, out, dout, dq, dk and dv");
      return;
    }
  }
  if (q.dtype != k.dtype || q.dtype != v.dtype || q.dtype != dout.dtype || dq.dtype != dk.dtype || dq.dtype != dv.dtype ||
      cu_seqlens_q.shape.size() != 1 || cu_seqlens_q.shape != cu_seqlens_k.shape || cu_seqlens_q.shape[0] < 1) {
    client.defer("InvalidArgument: attention_varlen backward needs q, k, v and dout of one dtype, dq, dk and dv of one dtype and cu "
                 "arrays [B + 1] of one length");
    return;
  }
  const b200_attention_varlen_args args{scale, window_left, window_right, max_seqlen_q, max_seqlen_k};
  const int rc = b200_attention_varlen_backward(
      client.raw(), nullptr, static_cast<b200_dtype>(q.dtype), static_cast<b200_dtype>(out.dtype), static_cast<b200_dtype>(dq.dtype),
      q.handle.ptr(), q.shape.data(), q.strides.data(), k.handle.ptr(), k.shape.data(), k.strides.data(), v.handle.ptr(), v.shape.data(),
      v.strides.data(), out.handle.ptr(), out.shape.data(), out.strides.data(), dout.handle.ptr(), dout.shape.data(), dout.strides.data(),
      lse.handle.ptr(), cu_seqlens_q.handle.ptr(), cu_seqlens_k.handle.ptr(), cu_seqlens_q.shape[0] - 1, dq.handle.ptr(), dq.shape.data(),
      dq.strides.data(), dk.handle.ptr(), dk.shape.data(), dk.strides.data(), dv.handle.ptr(), dv.shape.data(), dv.strides.data(), &args);
  if (rc != B200_OK) client.defer(b200_last_error());
}

/// Attention against a KV cache: q [B, Hq, Sq, D] against k_cache, v_cache [P, page, Hkv, D] (views by strides); sequence b
/// sees its first cache_seqlens[b] keys (compact i32 [B] on the device), key j in page block_table[b, j / page] (i32
/// [B, max_pages]; nullptr: page b); causal is bottom-right.  lse: nullptr or a compact f32 [B, Hq, Sq] tensor.  See
/// b200_attention_kvcache in cubecl_b200.h.  Errors are deferred to client.sync().
inline void launch_kvcache(ComputeClient& client, const TensorHandle& q, const TensorHandle& k_cache, const TensorHandle& v_cache,
                           const TensorHandle& cache_seqlens, const TensorHandle& out, const TensorHandle* block_table, float scale,
                           bool causal = false, const TensorHandle* lse = nullptr) {
  if (q.shape.size() != 4 || k_cache.shape.size() != 4 || v_cache.shape.size() != 4 || out.shape.size() != 4 ||
      (block_table && block_table->shape.size() != 2) || q.dtype != k_cache.dtype || q.dtype != v_cache.dtype) {
    client.defer("InvalidArgument: attention_kvcache needs rank-4 q, caches and out of one input dtype and a rank-2 block table");
    return;
  }
  const b200_attention_args args{scale, causal ? 1 : 0};
  const int rc = b200_attention_kvcache(
      client.raw(), nullptr, static_cast<b200_dtype>(q.dtype), static_cast<b200_dtype>(out.dtype), q.handle.ptr(), q.shape.data(),
      q.strides.data(), k_cache.handle.ptr(), k_cache.shape.data(), k_cache.strides.data(), v_cache.handle.ptr(), v_cache.shape.data(),
      v_cache.strides.data(), block_table ? block_table->handle.ptr() : 0, block_table ? block_table->shape.data() : nullptr,
      block_table ? block_table->strides.data() : nullptr, cache_seqlens.handle.ptr(), out.handle.ptr(), out.shape.data(),
      out.strides.data(), lse ? lse->handle.ptr() : 0, &args);
  if (rc != B200_OK) client.defer(b200_last_error());
}

/// Scatter of k_new, v_new [B, Snew, Hkv, D] into k_cache, v_cache [P, page, Hkv, D]: token n = b * Snew + t goes to flat slot
/// slot_mapping[n] (compact i32; negative slots are skipped).  See b200_kvcache_write in cubecl_b200.h.  Errors are deferred to
/// client.sync().
inline void kvcache_write(ComputeClient& client, const TensorHandle& k_new, const TensorHandle& v_new, const TensorHandle& k_cache,
                          const TensorHandle& v_cache, const TensorHandle& slot_mapping) {
  if (k_new.shape.size() != 4 || v_new.shape.size() != 4 || k_cache.shape.size() != 4 || v_cache.shape.size() != 4) {
    client.defer("InvalidArgument: kvcache_write needs rank-4 new tokens and caches");
    return;
  }
  const int rc = b200_kvcache_write(client.raw(), nullptr, static_cast<b200_dtype>(k_cache.dtype), k_new.handle.ptr(), k_new.shape.data(),
                                    k_new.strides.data(), v_new.handle.ptr(), v_new.shape.data(), v_new.strides.data(), k_cache.handle.ptr(),
                                    k_cache.shape.data(), k_cache.strides.data(), v_cache.handle.ptr(), v_cache.shape.data(),
                                    v_cache.strides.data(), slot_mapping.handle.ptr());
  if (rc != B200_OK) client.defer(b200_last_error());
}

/// launch_kvcache against an fp8 cache: k_cache, v_cache F8E4M3 or F8E5M2 (one dtype) hold K = k_scale[hk] * k8 and
/// V = v_scale[hk] * v8, with k_scale, v_scale compact f32 [Hkv] tensors.  See b200_attention_kvcache_fp8 in cubecl_b200.h.
/// Errors are deferred to client.sync().
inline void launch_kvcache_fp8(ComputeClient& client, const TensorHandle& q, const TensorHandle& k_cache, const TensorHandle& v_cache,
                               const TensorHandle& cache_seqlens, const TensorHandle& k_scale, const TensorHandle& v_scale,
                               const TensorHandle& out, const TensorHandle* block_table, float scale, bool causal = false,
                               const TensorHandle* lse = nullptr) {
  if (q.shape.size() != 4 || k_cache.shape.size() != 4 || v_cache.shape.size() != 4 || out.shape.size() != 4 ||
      (block_table && block_table->shape.size() != 2) || k_cache.dtype != v_cache.dtype) {
    client.defer("InvalidArgument: attention_kvcache_fp8 needs rank-4 q, caches and out, caches of one dtype and a rank-2 block table");
    return;
  }
  const b200_attention_args args{scale, causal ? 1 : 0};
  const int rc = b200_attention_kvcache_fp8(
      client.raw(), nullptr, static_cast<b200_dtype>(q.dtype), static_cast<b200_dtype>(k_cache.dtype), static_cast<b200_dtype>(out.dtype),
      q.handle.ptr(), q.shape.data(), q.strides.data(), k_cache.handle.ptr(), k_cache.shape.data(), k_cache.strides.data(),
      v_cache.handle.ptr(), v_cache.shape.data(), v_cache.strides.data(), block_table ? block_table->handle.ptr() : 0,
      block_table ? block_table->shape.data() : nullptr, block_table ? block_table->strides.data() : nullptr, cache_seqlens.handle.ptr(),
      k_scale.handle.ptr(), v_scale.handle.ptr(), out.handle.ptr(), out.shape.data(), out.strides.data(), lse ? lse->handle.ptr() : 0,
      &args);
  if (rc != B200_OK) client.defer(b200_last_error());
}

/// kvcache_write into fp8 caches: each value x of kv head hk is stored as sat_rn(x / scale[hk]).  See b200_kvcache_write_fp8 in
/// cubecl_b200.h.  Errors are deferred to client.sync().
inline void kvcache_write_fp8(ComputeClient& client, const TensorHandle& k_new, const TensorHandle& v_new, const TensorHandle& k_cache,
                              const TensorHandle& v_cache, const TensorHandle& slot_mapping, const TensorHandle& k_scale,
                              const TensorHandle& v_scale) {
  if (k_new.shape.size() != 4 || v_new.shape.size() != 4 || k_cache.shape.size() != 4 || v_cache.shape.size() != 4 ||
      k_cache.dtype != v_cache.dtype) {
    client.defer("InvalidArgument: kvcache_write_fp8 needs rank-4 new tokens and caches of one dtype");
    return;
  }
  const int rc = b200_kvcache_write_fp8(client.raw(), nullptr, static_cast<b200_dtype>(k_new.dtype), static_cast<b200_dtype>(k_cache.dtype),
                                        k_new.handle.ptr(), k_new.shape.data(), k_new.strides.data(), v_new.handle.ptr(), v_new.shape.data(),
                                        v_new.strides.data(), k_cache.handle.ptr(), k_cache.shape.data(), k_cache.strides.data(),
                                        v_cache.handle.ptr(), v_cache.shape.data(), v_cache.strides.data(), slot_mapping.handle.ptr(),
                                        k_scale.handle.ptr(), v_scale.handle.ptr());
  if (rc != B200_OK) client.defer(b200_last_error());
}
}  // namespace attention

namespace reduce {
enum class Op : int { Sum = B200_REDUCE_SUM, Prod = B200_REDUCE_PROD, Max = B200_REDUCE_MAX, Min = B200_REDUCE_MIN,
                      ArgMax = B200_REDUCE_ARGMAX, ArgMin = B200_REDUCE_ARGMIN, Mean = B200_REDUCE_MEAN };
/// Reduce `axis` of a contiguous input (-1 = every element); output f32 (u32 indices for arg ops). Errors deferred.
inline void launch(ComputeClient& client, const TensorHandle& input, const TensorHandle& output, int axis, Op op) {
  const int rc = b200_reduce(client.raw(), nullptr, static_cast<b200_reduce_op>(op), static_cast<b200_dtype>(input.dtype),
                             input.handle.ptr(), output.handle.ptr(), static_cast<int>(input.shape.size()), input.shape.data(), axis);
  if (rc != B200_OK) client.defer(b200_last_error());
}
}  // namespace reduce

namespace scan {
/// Inclusive (or exclusive) cumulative sum / prod / max / min along `axis` into a compact output of the input's shape;
/// output dtype F32 or the input's. Errors deferred.
inline void launch(ComputeClient& client, const TensorHandle& input, const TensorHandle& output, int axis, reduce::Op op,
                   bool exclusive = false) {
  const int rc = b200_scan(client.raw(), nullptr, static_cast<b200_reduce_op>(op), exclusive ? 1 : 0,
                           static_cast<b200_dtype>(input.dtype), static_cast<b200_dtype>(output.dtype), input.handle.ptr(),
                           output.handle.ptr(), static_cast<int>(input.shape.size()), input.shape.data(), input.strides.data(),
                           axis);
  if (rc != B200_OK) client.defer(b200_last_error());
}
}  // namespace scan

namespace quant {
/// QuantScheme (value, block level, per-tensor level); see b200_quantize in cubecl_b200.h for the contract.
using Scheme = b200_quant_scheme;
/// Codes [..., K * bits / 8], block scales [..., K / block] and the f32 tensor scale of `input` (any strides) along its
/// innermost axis; pass 0 for an absent level. Errors deferred.
inline void quantize(ComputeClient& client, const TensorHandle& input, const Scheme& scheme, b200_dptr values,
                     b200_dptr block_scales, b200_dptr tensor_scale) {
  const int rc = b200_quantize(client.raw(), nullptr, &scheme, static_cast<b200_dtype>(input.dtype), input.handle.ptr(), values,
                               block_scales, tensor_scale, static_cast<int>(input.shape.size()), input.shape.data(),
                               input.strides.data());
  if (rc != B200_OK) client.defer(b200_last_error());
}
/// output (contiguous F32 / F16 / BF16, the quantized tensor's shape) = the dequantized values. Errors deferred.
inline void dequantize(ComputeClient& client, const Scheme& scheme, b200_dptr values, b200_dptr block_scales, b200_dptr tensor_scale,
                       const TensorHandle& output) {
  const int rc = b200_dequantize(client.raw(), nullptr, &scheme, static_cast<b200_dtype>(output.dtype), values, block_scales,
                                 tensor_scale, output.handle.ptr(), static_cast<int>(output.shape.size()), output.shape.data());
  if (rc != B200_OK) client.defer(b200_last_error());
}
}  // namespace quant

}  // namespace cubecl
