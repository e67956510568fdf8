//! `cubecl-b200-sys`: raw bindings (`sys`, generated from `include/cubecl_b200.h`, ABI version 1) plus a thin safe layer.
//!
//! SOURCE ONLY -- never compiled in the authoring image (no Rust toolchain).  `sys.rs` is GENERATED from the header by
//! `tools/gen_rust_sys.py` and the CPU test `tests/test_rust_bindings.py` fails when header and bindings drift apart; the
//! safe layer below is hand-written against those signatures and the same test checks that every `sys::` function it
//! calls exists with the argument count used here.
//!
//! Intended use inside cubecl-cuda: `CudaServer` resolves `BufferBinding`s to `CUdeviceptr`s on the runner thread and
//! passes them here together with the `CUstream` of the current `StreamId` (crates/cubecl-cuda/src/compute/server.rs:
//! 1024-1144); errors are queued on the stream like any launch error (server.rs:269-284).  See INTEGRATION.md.

pub mod launch;
pub mod sys;

use core::ffi::{c_int, c_void, CStr};
use std::ffi::CString;

pub use sys::{b200_dptr, b200_event, b200_stream};

/// `b200_status`, mirroring LaunchError / ServerError (crates/cubecl-runtime/src/server/base.rs:177-272).
#[repr(i32)]
#[derive(Clone, Copy, Debug, PartialEq, Eq)]
pub enum Status {
    Ok = 0,
    Compilation = 1,
    OutOfMemory = 2,
    TooManyResources = 3,
    Unknown = 4,
    Io = 5,
    InvalidArg = 6,
    Unsupported = 7,
    NoDevice = 8,
    Comm = 9,
    Unhealthy = 10,
}

/// `b200_dtype`.
#[repr(i32)]
#[derive(Clone, Copy, Debug, PartialEq, Eq)]
pub enum DType {
    F32 = 0,
    F16 = 1,
    BF16 = 2,
    U32 = 3,
    I32 = 4,
    F64 = 5,
    I64 = 6,
    U64 = 7,
    U8 = 8,
    I8 = 9,
    F8E4M3 = 10,
    F8E5M2 = 11,
    F4E2M1x2 = 12,
    UE8M0 = 13,
}

/// `b200_reduce_op`.
#[repr(i32)]
#[derive(Clone, Copy, Debug, PartialEq, Eq)]
pub enum ReduceOp {
    Sum = 0,
    Prod = 1,
    Max = 2,
    Min = 3,
    ArgMax = 4,
    ArgMin = 5,
    Mean = 6,
}

/// `b200_comm_op` = ReduceOperation{Sum,Mean} (server/base.rs:623-628).
#[repr(i32)]
#[derive(Clone, Copy, Debug, PartialEq, Eq)]
pub enum CommOp {
    Sum = 0,
    Mean = 1,
}

/// `b200_quant_value` = QuantValue (crates/cubecl-common/src/quant/scheme.rs:358-377), in its order.
#[repr(i32)]
#[derive(Clone, Copy, Debug, PartialEq, Eq)]
pub enum QuantValue {
    Q8F = 0,
    E5M2 = 1,
    E4M3 = 2,
    Q4F = 3,
    E2M1 = 4,
    Q2F = 5,
    Q8S = 6,
    Q4S = 7,
    Q2S = 8,
}

/// `b200_quant_scheme`: the value type, an optional block level (`block` values per scale stored as `block_scale`, one of
/// F32 / F16 / BF16 / UE8M0 / F8E4M3 = ue4m3) and an optional per-tensor f32 level.
#[derive(Clone, Copy, Debug, PartialEq, Eq)]
pub struct QuantScheme {
    pub value: QuantValue,
    pub block: u32,
    pub block_scale: DType,
    pub tensor_scale: bool,
}

impl QuantScheme {
    fn raw(&self) -> sys::b200_quant_scheme {
        sys::b200_quant_scheme {
            value: self.value as i32,
            block: self.block as i32,
            block_scale: self.block_scale as i32,
            tensor_scale: self.tensor_scale as i32,
        }
    }
}

/// `b200_quant_operand`: one operand of [`Context::matmul_quantized`], its codes and scales as `b200_quantize` wrote them
/// (0 for an absent level; the tensor scale stays on the device).
#[derive(Clone, Copy, Debug)]
pub struct QuantOperand {
    pub scheme: QuantScheme,
    pub values: b200_dptr,
    pub block_scales: b200_dptr,
    pub tensor_scale: b200_dptr,
}

impl QuantOperand {
    fn raw(&self) -> sys::b200_quant_operand {
        sys::b200_quant_operand {
            scheme: self.scheme.raw(),
            values: self.values,
            block_scales: self.block_scales,
            tensor_scale: self.tensor_scale,
        }
    }
}

/// Activation of the fused GEMM epilogue (`b200_epilogue.activation`).
#[repr(i32)]
#[derive(Clone, Copy, Debug, PartialEq, Eq)]
pub enum Activation {
    None = 0,
    Relu = 1,
    Gelu = 2,
}

/// Error carrying the status and the thread-local message of the failing call.
#[derive(Debug)]
pub struct Error {
    pub status: i32,
    pub message: String,
}

/// b200_conv3d_args from (stride_d, stride_h, stride_w, pad_d, pad_h, pad_w, dilation_d, dilation_h, dilation_w).
fn conv3d_args(a: [i32; 9]) -> sys::b200_conv3d_args {
    sys::b200_conv3d_args {
        stride_d: a[0], stride_h: a[1], stride_w: a[2], pad_d: a[3], pad_h: a[4], pad_w: a[5], dilation_d: a[6], dilation_h: a[7],
        dilation_w: a[8],
    }
}

fn check(rc: c_int) -> Result<(), Error> {
    if rc == 0 {
        return Ok(());
    }
    let message = unsafe { CStr::from_ptr(sys::b200_last_error()) }.to_string_lossy().into_owned();
    Err(Error { status: rc, message })
}

/// One context per device; `Send` but not `Sync`, like `CudaServer` (one runner thread per device).
pub struct Context(*mut sys::b200_ctx);
unsafe impl Send for Context {}

/// Strided tensor view: device pointer + shape + strides in ELEMENTS (TensorHandle, cubecl-std/src/tensor/handle.rs:13-23).
pub struct TensorView<'a> {
    pub ptr: b200_dptr,
    pub shape: &'a [u64],
    pub strides: &'a [u64],
}

/// out = act(alpha * acc + bias[n]) inside the GEMM epilogue; `bias` is an f32[N] device pointer or 0.
pub struct Epilogue {
    pub alpha: f32,
    pub activation: Activation,
    pub bias: b200_dptr,
}

impl Context {
    pub fn new(device: i32) -> Result<Self, Error> {
        let mut p = core::ptr::null_mut();
        check(unsafe { sys::b200_init(device, &mut p) })?;
        Ok(Self(p))
    }

    pub fn raw(&self) -> *mut sys::b200_ctx {
        self.0
    }

    pub fn properties(&self) -> Result<sys::b200_props, Error> {
        let mut props = core::mem::MaybeUninit::<sys::b200_props>::zeroed();
        check(unsafe { sys::b200_get_props(self.0, props.as_mut_ptr()) })?;
        Ok(unsafe { props.assume_init() })
    }

    /// String-typed runtime knob ("gemm.variant", "gemm.f32", "reduce.variant", ...; see the header).
    pub fn set_option(&mut self, key: &str, value: &str) -> Result<(), Error> {
        let k = CString::new(key).map_err(|_| Error { status: Status::InvalidArg as i32, message: "NUL in key".into() })?;
        let v = CString::new(value).map_err(|_| Error { status: Status::InvalidArg as i32, message: "NUL in value".into() })?;
        check(unsafe { sys::b200_set_option(self.0, k.as_ptr(), v.as_ptr()) })
    }

    /// Entry-point name of the kernel this context launched most recently (what a harness reports as the kernel it timed).
    pub fn last_kernel(&self) -> Result<String, Error> {
        let mut buf = [0u8; 256];
        check(unsafe { sys::b200_last_kernel(self.0, buf.as_mut_ptr() as *mut core::ffi::c_char, buf.len()) })?;
        let end = buf.iter().position(|&b| b == 0).unwrap_or(buf.len());
        Ok(String::from_utf8_lossy(&buf[..end]).into_owned())
    }

    pub fn launch_count(&self) -> Result<u64, Error> {
        let mut n = 0u64;
        check(unsafe { sys::b200_launch_count(self.0, &mut n) })?;
        Ok(n)
    }

    // ---- memory (standalone use; inside CubeCL the retained pool owns the buffers) --------------------------------
    pub fn alloc(&mut self, bytes: usize) -> Result<b200_dptr, Error> {
        let mut p: b200_dptr = 0;
        check(unsafe { sys::b200_alloc(self.0, bytes, &mut p) })?;
        Ok(p)
    }

    /// # Safety
    /// `ptr` must come from [`Context::alloc`] on this context and must not be used by work enqueued after this call.
    pub unsafe fn free(&mut self, ptr: b200_dptr) -> Result<(), Error> {
        check(sys::b200_free(self.0, ptr))
    }

    /// Frees in the order of `last_use`, the stream whose queued work may still touch the buffer (null = the context's
    /// stream): the pool re-issues the page only once an event recorded there has completed.
    ///
    /// # Safety
    /// Same contract as [`Context::free`].
    pub unsafe fn free_async(&mut self, ptr: b200_dptr, last_use: b200_stream) -> Result<(), Error> {
        check(sys::b200_free_async(self.0, ptr, last_use))
    }

    /// Stream-ordered host -> device copy; asynchronous when `src` is pinned (sync before reusing it).
    ///
    /// # Safety
    /// `dst` must be a live device allocation of at least `src.len()` bytes.
    pub unsafe fn write(&mut self, stream: b200_stream, dst: b200_dptr, src: &[u8]) -> Result<(), Error> {
        check(sys::b200_write(self.0, stream, dst, src.as_ptr() as *const c_void, src.len()))
    }

    /// Stream-ordered device -> host copy; call [`Context::sync`] before reading `dst`.
    ///
    /// # Safety
    /// `src` must be a live device allocation of at least `dst.len()` bytes.
    pub unsafe fn read(&mut self, stream: b200_stream, dst: &mut [u8], src: b200_dptr) -> Result<(), Error> {
        check(sys::b200_read(self.0, stream, dst.as_mut_ptr() as *mut c_void, src, dst.len()))
    }

    // ---- streams / events ------------------------------------------------------------------------------------------
    pub fn stream_create(&mut self) -> Result<b200_stream, Error> {
        let mut s: b200_stream = core::ptr::null_mut();
        check(unsafe { sys::b200_stream_create(self.0, &mut s) })?;
        Ok(s)
    }

    /// # Safety
    /// `stream` must come from [`Context::stream_create`] and must not be used afterwards.
    pub unsafe fn stream_destroy(&mut self, stream: b200_stream) -> Result<(), Error> {
        check(sys::b200_stream_destroy(self.0, stream))
    }

    /// Waits for `stream` (null = the context's compute stream); deferred device faults surface here as `Unhealthy`.
    pub fn sync(&mut self, stream: b200_stream) -> Result<(), Error> {
        check(unsafe { sys::b200_sync(self.0, stream) })
    }

    pub fn event_create(&mut self) -> Result<b200_event, Error> {
        let mut e: b200_event = core::ptr::null_mut();
        check(unsafe { sys::b200_event_create(self.0, &mut e) })?;
        Ok(e)
    }

    /// # Safety
    /// `event` / `stream` must be live handles of this context.
    pub unsafe fn event_record(&mut self, event: b200_event, stream: b200_stream) -> Result<(), Error> {
        check(sys::b200_event_record(self.0, event, stream))
    }

    /// # Safety
    /// `event` / `stream` must be live handles of this context.
    pub unsafe fn stream_wait_event(&mut self, stream: b200_stream, event: b200_event) -> Result<(), Error> {
        check(sys::b200_stream_wait_event(self.0, stream, event))
    }

    /// # Safety
    /// Both events must be live, recorded handles of this context.
    pub unsafe fn event_elapsed_ms(&mut self, start: b200_event, end: b200_event) -> Result<f32, Error> {
        let mut ms = 0f32;
        check(sys::b200_event_elapsed_ms(self.0, start, end, &mut ms))?;
        Ok(ms)
    }

    /// # Safety
    /// `event` must be a live handle of this context and must not be used afterwards.
    pub unsafe fn event_destroy(&mut self, event: b200_event) -> Result<(), Error> {
        check(sys::b200_event_destroy(self.0, event))
    }

    // ---- matmul::launch ---------------------------------------------------------------------------------------------
    /// out = lhs @ rhs, f32 accumulate, batch broadcast (shape.rs:489-517), enqueued on `stream`.
    ///
    /// # Safety
    /// The pointers must be live device allocations of this device large enough for the described views, and must stay
    /// alive until the stream has passed this launch (the pool's handle ref-count guarantees that inside CubeCL).
    pub unsafe fn matmul(
        &mut self, stream: b200_stream, in_dtype: DType, out_dtype: DType,
        lhs: &TensorView, rhs: &TensorView, out: &TensorView,
    ) -> Result<(), Error> {
        let rank = lhs.shape.len();
        assert!(rhs.shape.len() == rank && out.shape.len() == rank);
        assert!(lhs.strides.len() == rank && rhs.strides.len() == rank && out.strides.len() == rank);
        check(sys::b200_matmul(
            self.0, stream, in_dtype as c_int, out_dtype as c_int, lhs.ptr, rhs.ptr, out.ptr, rank as c_int,
            lhs.shape.as_ptr(), lhs.strides.as_ptr(), rhs.shape.as_ptr(), rhs.strides.as_ptr(),
            out.shape.as_ptr(), out.strides.as_ptr(),
        ))
    }

    /// The same product with different 8-bit formats per operand (i8 x u8, e4m3 x e5m2 ...: the reference's manual-MMA
    /// pairs, crates/cubecl-cpp/src/cuda/mma/manual.rs:151-186).
    ///
    /// # Safety
    /// Same contract as [`Context::matmul`].
    pub unsafe fn matmul_mixed(
        &mut self, stream: b200_stream, lhs_dtype: DType, rhs_dtype: DType, out_dtype: DType,
        lhs: &TensorView, rhs: &TensorView, out: &TensorView,
    ) -> Result<(), Error> {
        let rank = lhs.shape.len();
        assert!(rhs.shape.len() == rank && out.shape.len() == rank);
        assert!(lhs.strides.len() == rank && rhs.strides.len() == rank && out.strides.len() == rank);
        check(sys::b200_matmul_mixed(
            self.0, stream, lhs_dtype as c_int, rhs_dtype as c_int, out_dtype as c_int, lhs.ptr, rhs.ptr, out.ptr,
            rank as c_int, lhs.shape.as_ptr(), lhs.strides.as_ptr(), rhs.shape.as_ptr(), rhs.strides.as_ptr(),
            out.shape.as_ptr(), out.strides.as_ptr(),
        ))
    }

    /// out = act(alpha * (lhs @ rhs) + bias[n]) in one launch.
    ///
    /// # Safety
    /// Same contract as [`Context::matmul`]; `epilogue.bias` must be 0 or an f32[N] device allocation.
    pub unsafe fn matmul_fused(
        &mut self, stream: b200_stream, in_dtype: DType, out_dtype: DType,
        lhs: &TensorView, rhs: &TensorView, out: &TensorView, epilogue: &Epilogue,
    ) -> Result<(), Error> {
        let rank = lhs.shape.len();
        assert!(rhs.shape.len() == rank && out.shape.len() == rank);
        assert!(lhs.strides.len() == rank && rhs.strides.len() == rank && out.strides.len() == rank);
        let e = sys::b200_epilogue { alpha: epilogue.alpha, activation: epilogue.activation as i32, bias: epilogue.bias };
        check(sys::b200_matmul_fused(
            self.0, stream, in_dtype as c_int, out_dtype as c_int, lhs.ptr, rhs.ptr, out.ptr, rank as c_int,
            lhs.shape.as_ptr(), lhs.strides.as_ptr(), rhs.shape.as_ptr(), rhs.strides.as_ptr(),
            out.shape.as_ptr(), out.strides.as_ptr(), &e,
        ))
    }

    /// 2-D convolution: x [N, H, W, C] (NHWC), w [Cout, KH, KW, C], out [N, OH, OW, Cout], f32 accumulation, optional fused
    /// epilogue; `args` = (stride_h, stride_w, pad_h, pad_w, dilation_h, dilation_w).  See b200_conv2d in cubecl_b200.h.
    ///
    /// # Safety
    /// Same contract as [`Context::matmul`]; `epilogue.bias` must be 0 or an f32[Cout] device allocation.
    pub unsafe fn conv2d(
        &mut self, stream: b200_stream, in_dtype: DType, out_dtype: DType, x: &TensorView, w: &TensorView, out: &TensorView,
        args: [i32; 6], epilogue: Option<&Epilogue>,
    ) -> Result<(), Error> {
        assert!(x.shape.len() == 4 && w.shape.len() == 4 && out.shape.len() == 4);
        assert!(x.strides.len() == 4 && w.strides.len() == 4 && out.strides.len() == 4);
        let a = sys::b200_conv2d_args {
            stride_h: args[0], stride_w: args[1], pad_h: args[2], pad_w: args[3], dilation_h: args[4], dilation_w: args[5],
        };
        let e = epilogue.map(|e| sys::b200_epilogue { alpha: e.alpha, activation: e.activation as i32, bias: e.bias });
        check(sys::b200_conv2d(
            self.0, stream, in_dtype as c_int, out_dtype as c_int, x.ptr, x.shape.as_ptr(), x.strides.as_ptr(), w.ptr,
            w.shape.as_ptr(), w.strides.as_ptr(), out.ptr, out.shape.as_ptr(), out.strides.as_ptr(), &a,
            e.as_ref().map_or(std::ptr::null(), |e| e as *const sys::b200_epilogue),
        ))
    }

    /// Input gradient of [`Context::conv2d`]: dy [N, OH, OW, Cout], w [Cout, KH, KW, C] -> dx [N, H, W, C], f32 accumulation.
    /// See b200_conv2d_backward_data in cubecl_b200.h.
    ///
    /// # Safety
    /// Same contract as [`Context::matmul`] for the three pointers.
    pub unsafe fn conv2d_backward_data(
        &mut self, stream: b200_stream, in_dtype: DType, out_dtype: DType, dy: &TensorView, w: &TensorView, dx: &TensorView,
        args: [i32; 6],
    ) -> Result<(), Error> {
        assert!(dy.shape.len() == 4 && w.shape.len() == 4 && dx.shape.len() == 4);
        assert!(dy.strides.len() == 4 && w.strides.len() == 4 && dx.strides.len() == 4);
        let a = sys::b200_conv2d_args {
            stride_h: args[0], stride_w: args[1], pad_h: args[2], pad_w: args[3], dilation_h: args[4], dilation_w: args[5],
        };
        check(sys::b200_conv2d_backward_data(
            self.0, stream, in_dtype as c_int, out_dtype as c_int, dy.ptr, dy.shape.as_ptr(), dy.strides.as_ptr(), w.ptr,
            w.shape.as_ptr(), w.strides.as_ptr(), dx.ptr, dx.shape.as_ptr(), dx.strides.as_ptr(), &a,
        ))
    }

    /// Weight gradient of [`Context::conv2d`]: x [N, H, W, C], dy [N, OH, OW, Cout] -> dw [Cout, KH, KW, C], f32 accumulation.
    /// The bias gradient is [`Context::reduce`] (sum) over axis 0 of dy viewed as [N * OH * OW, Cout].  See
    /// b200_conv2d_backward_weight in cubecl_b200.h.
    ///
    /// # Safety
    /// Same contract as [`Context::matmul`] for the three pointers.
    pub unsafe fn conv2d_backward_weight(
        &mut self, stream: b200_stream, in_dtype: DType, out_dtype: DType, x: &TensorView, dy: &TensorView, dw: &TensorView,
        args: [i32; 6],
    ) -> Result<(), Error> {
        assert!(x.shape.len() == 4 && dy.shape.len() == 4 && dw.shape.len() == 4);
        assert!(x.strides.len() == 4 && dy.strides.len() == 4 && dw.strides.len() == 4);
        let a = sys::b200_conv2d_args {
            stride_h: args[0], stride_w: args[1], pad_h: args[2], pad_w: args[3], dilation_h: args[4], dilation_w: args[5],
        };
        check(sys::b200_conv2d_backward_weight(
            self.0, stream, in_dtype as c_int, out_dtype as c_int, x.ptr, x.shape.as_ptr(), x.strides.as_ptr(), dy.ptr,
            dy.shape.as_ptr(), dy.strides.as_ptr(), dw.ptr, dw.shape.as_ptr(), dw.strides.as_ptr(), &a,
        ))
    }

    /// 3-D convolution: x [N, D, H, W, C] (NDHWC), w [Cout, KD, KH, KW, C], out [N, OD, OH, OW, Cout], f32 accumulation,
    /// optional fused epilogue; `args` = (stride_d, stride_h, stride_w, pad_d, pad_h, pad_w, dilation_d, dilation_h,
    /// dilation_w).  See b200_conv3d in cubecl_b200.h.
    ///
    /// # Safety
    /// Same contract as [`Context::conv2d`].
    pub unsafe fn conv3d(
        &mut self, stream: b200_stream, in_dtype: DType, out_dtype: DType, x: &TensorView, w: &TensorView, out: &TensorView,
        args: [i32; 9], epilogue: Option<&Epilogue>,
    ) -> Result<(), Error> {
        assert!(x.shape.len() == 5 && w.shape.len() == 5 && out.shape.len() == 5);
        assert!(x.strides.len() == 5 && w.strides.len() == 5 && out.strides.len() == 5);
        let a = conv3d_args(args);
        let e = epilogue.map(|e| sys::b200_epilogue { alpha: e.alpha, activation: e.activation as i32, bias: e.bias });
        check(sys::b200_conv3d(
            self.0, stream, in_dtype as c_int, out_dtype as c_int, x.ptr, x.shape.as_ptr(), x.strides.as_ptr(), w.ptr,
            w.shape.as_ptr(), w.strides.as_ptr(), out.ptr, out.shape.as_ptr(), out.strides.as_ptr(), &a,
            e.as_ref().map_or(std::ptr::null(), |e| e as *const sys::b200_epilogue),
        ))
    }

    /// Input gradient of [`Context::conv3d`]: dy [N, OD, OH, OW, Cout], w [Cout, KD, KH, KW, C] -> dx [N, D, H, W, C].  See
    /// b200_conv3d_backward_data in cubecl_b200.h.
    ///
    /// # Safety
    /// Same contract as [`Context::matmul`] for the three pointers.
    pub unsafe fn conv3d_backward_data(
        &mut self, stream: b200_stream, in_dtype: DType, out_dtype: DType, dy: &TensorView, w: &TensorView, dx: &TensorView,
        args: [i32; 9],
    ) -> Result<(), Error> {
        assert!(dy.shape.len() == 5 && w.shape.len() == 5 && dx.shape.len() == 5);
        assert!(dy.strides.len() == 5 && w.strides.len() == 5 && dx.strides.len() == 5);
        let a = conv3d_args(args);
        check(sys::b200_conv3d_backward_data(
            self.0, stream, in_dtype as c_int, out_dtype as c_int, dy.ptr, dy.shape.as_ptr(), dy.strides.as_ptr(), w.ptr,
            w.shape.as_ptr(), w.strides.as_ptr(), dx.ptr, dx.shape.as_ptr(), dx.strides.as_ptr(), &a,
        ))
    }

    /// Weight gradient of [`Context::conv3d`]: x [N, D, H, W, C], dy [N, OD, OH, OW, Cout] -> dw [Cout, KD, KH, KW, C].  The
    /// bias gradient is [`Context::reduce`] (sum) over axis 0 of dy viewed as [N * OD * OH * OW, Cout].  See
    /// b200_conv3d_backward_weight in cubecl_b200.h.
    ///
    /// # Safety
    /// Same contract as [`Context::matmul`] for the three pointers.
    pub unsafe fn conv3d_backward_weight(
        &mut self, stream: b200_stream, in_dtype: DType, out_dtype: DType, x: &TensorView, dy: &TensorView, dw: &TensorView,
        args: [i32; 9],
    ) -> Result<(), Error> {
        assert!(x.shape.len() == 5 && dy.shape.len() == 5 && dw.shape.len() == 5);
        assert!(x.strides.len() == 5 && dy.strides.len() == 5 && dw.strides.len() == 5);
        let a = conv3d_args(args);
        check(sys::b200_conv3d_backward_weight(
            self.0, stream, in_dtype as c_int, out_dtype as c_int, x.ptr, x.shape.as_ptr(), x.strides.as_ptr(), dy.ptr,
            dy.shape.as_ptr(), dy.strides.as_ptr(), dw.ptr, dw.shape.as_ptr(), dw.strides.as_ptr(), &a,
        ))
    }

    /// Transposed convolution: x [N, H, W, Cin], w [Cin, KH, KW, Cout] -> out [N, OH, OW, Cout] (out's shape gives the output
    /// padding), f32 accumulation, optional fused epilogue; `args` as [`Context::conv2d`].  Gradients: dx =
    /// [`Context::conv2d`] (dy, w), dw = [`Context::conv2d_backward_weight`] (x := dy, dy := x).  See b200_conv_transpose2d
    /// in cubecl_b200.h.
    ///
    /// # Safety
    /// Same contract as [`Context::conv2d`].
    pub unsafe fn conv_transpose2d(
        &mut self, stream: b200_stream, in_dtype: DType, out_dtype: DType, x: &TensorView, w: &TensorView, out: &TensorView,
        args: [i32; 6], epilogue: Option<&Epilogue>,
    ) -> Result<(), Error> {
        assert!(x.shape.len() == 4 && w.shape.len() == 4 && out.shape.len() == 4);
        assert!(x.strides.len() == 4 && w.strides.len() == 4 && out.strides.len() == 4);
        let a = sys::b200_conv2d_args {
            stride_h: args[0], stride_w: args[1], pad_h: args[2], pad_w: args[3], dilation_h: args[4], dilation_w: args[5],
        };
        let e = epilogue.map(|e| sys::b200_epilogue { alpha: e.alpha, activation: e.activation as i32, bias: e.bias });
        check(sys::b200_conv_transpose2d(
            self.0, stream, in_dtype as c_int, out_dtype as c_int, x.ptr, x.shape.as_ptr(), x.strides.as_ptr(), w.ptr,
            w.shape.as_ptr(), w.strides.as_ptr(), out.ptr, out.shape.as_ptr(), out.strides.as_ptr(), &a,
            e.as_ref().map_or(std::ptr::null(), |e| e as *const sys::b200_epilogue),
        ))
    }

    /// 3-D [`Context::conv_transpose2d`]: x [N, D, H, W, Cin], w [Cin, KD, KH, KW, Cout] -> out [N, OD, OH, OW, Cout]; `args`
    /// as [`Context::conv3d`].  See b200_conv_transpose3d in cubecl_b200.h.
    ///
    /// # Safety
    /// Same contract as [`Context::conv2d`].
    pub unsafe fn conv_transpose3d(
        &mut self, stream: b200_stream, in_dtype: DType, out_dtype: DType, x: &TensorView, w: &TensorView, out: &TensorView,
        args: [i32; 9], epilogue: Option<&Epilogue>,
    ) -> Result<(), Error> {
        assert!(x.shape.len() == 5 && w.shape.len() == 5 && out.shape.len() == 5);
        assert!(x.strides.len() == 5 && w.strides.len() == 5 && out.strides.len() == 5);
        let a = conv3d_args(args);
        let e = epilogue.map(|e| sys::b200_epilogue { alpha: e.alpha, activation: e.activation as i32, bias: e.bias });
        check(sys::b200_conv_transpose3d(
            self.0, stream, in_dtype as c_int, out_dtype as c_int, x.ptr, x.shape.as_ptr(), x.strides.as_ptr(), w.ptr,
            w.shape.as_ptr(), w.strides.as_ptr(), out.ptr, out.shape.as_ptr(), out.strides.as_ptr(), &a,
            e.as_ref().map_or(std::ptr::null(), |e| e as *const sys::b200_epilogue),
        ))
    }

    /// Fused scaled-dot-product attention, forward: q [B, Hq, Sq, D], k and v [B, Hkv, Sk, D] -> out [B, Hq, Sq, D] (views by
    /// strides), f16 / bf16 in, out in the input dtype or f32; `lse`: 0 or an f32 [B, Hq, Sq] compact buffer for the row
    /// log-sum-exp; `causal`: key j visible to query i iff j <= i.  See b200_attention in cubecl_b200.h.
    ///
    /// # Safety
    /// Same contract as [`Context::conv2d`]; `lse`, when non-zero, must hold B * Hq * Sq f32 values.
    pub unsafe fn attention(
        &mut self, stream: b200_stream, in_dtype: DType, out_dtype: DType, q: &TensorView, k: &TensorView, v: &TensorView,
        out: &TensorView, lse: b200_dptr, scale: f32, causal: bool,
    ) -> Result<(), Error> {
        for t in [q, k, v, out] {
            assert!(t.shape.len() == 4 && t.strides.len() == 4);
        }
        let a = sys::b200_attention_args { scale, causal: causal as i32 };
        check(sys::b200_attention(
            self.0, stream, in_dtype as c_int, out_dtype as c_int, q.ptr, q.shape.as_ptr(), q.strides.as_ptr(), k.ptr,
            k.shape.as_ptr(), k.strides.as_ptr(), v.ptr, v.shape.as_ptr(), v.strides.as_ptr(), out.ptr, out.shape.as_ptr(),
            out.strides.as_ptr(), lse, &a,
        ))
    }

    /// Fused scaled-dot-product attention, backward: dq [B, Hq, Sq, D], dk and dv [B, Hkv, Sk, D] in `grad_dtype` (the input
    /// dtype or f32) from q, k, v, the forward's `out` (in `out_dtype`) and `lse` (its compact f32 [B, Hq, Sq] buffer) and
    /// `dout` (in the input dtype).  See b200_attention_backward in cubecl_b200.h.
    ///
    /// # Safety
    /// Same contract as [`Context::conv2d`]; `lse` must hold B * Hq * Sq f32 values.
    pub unsafe fn attention_backward(
        &mut self, stream: b200_stream, in_dtype: DType, out_dtype: DType, grad_dtype: DType, q: &TensorView, k: &TensorView,
        v: &TensorView, out: &TensorView, dout: &TensorView, lse: b200_dptr, dq: &TensorView, dk: &TensorView, dv: &TensorView,
        scale: f32, causal: bool,
    ) -> Result<(), Error> {
        for t in [q, k, v, out, dout, dq, dk, dv] {
            assert!(t.shape.len() == 4 && t.strides.len() == 4);
        }
        let a = sys::b200_attention_args { scale, causal: causal as i32 };
        check(sys::b200_attention_backward(
            self.0, stream, in_dtype as c_int, out_dtype as c_int, grad_dtype as c_int, q.ptr, q.shape.as_ptr(), q.strides.as_ptr(),
            k.ptr, k.shape.as_ptr(), k.strides.as_ptr(), v.ptr, v.shape.as_ptr(), v.strides.as_ptr(), out.ptr, out.shape.as_ptr(),
            out.strides.as_ptr(), dout.ptr, dout.shape.as_ptr(), dout.strides.as_ptr(), lse, dq.ptr, dq.shape.as_ptr(),
            dq.strides.as_ptr(), dk.ptr, dk.shape.as_ptr(), dk.strides.as_ptr(), dv.ptr, dv.shape.as_ptr(), dv.strides.as_ptr(), &a,
        ))
    }

    /// Variable-length (packed) attention, forward: q [Tq, Hq, D], k and v [Tk, Hkv, D] -> out [Tq, Hq, D] (views by strides);
    /// sequence b owns rows [cu_q[b], cu_q[b + 1]) of q and [cu_k[b], cu_k[b + 1]) of k and v (compact i32 [batch + 1] device
    /// buffers); `window` (left, right), -1 unbounded, (-1, 0) bottom-right causal; `lse`: 0 or a compact f32 [Hq, Tq] buffer.
    /// See b200_attention_varlen in cubecl_b200.h.
    ///
    /// # Safety
    /// Same contract as [`Context::conv2d`]; the cu buffers must hold batch + 1 i32 values, `lse`, when non-zero, Hq * Tq f32.
    pub unsafe fn attention_varlen(
        &mut self, stream: b200_stream, in_dtype: DType, out_dtype: DType, q: &TensorView, k: &TensorView, v: &TensorView,
        cu_seqlens_q: b200_dptr, cu_seqlens_k: b200_dptr, batch: u64, max_seqlen: (i32, i32), out: &TensorView, lse: b200_dptr,
        scale: f32, window: (i32, i32),
    ) -> Result<(), Error> {
        for t in [q, k, v, out] {
            assert!(t.shape.len() == 3 && t.strides.len() == 3);
        }
        let a = sys::b200_attention_varlen_args {
            scale, window_left: window.0, window_right: window.1, max_seqlen_q: max_seqlen.0, max_seqlen_k: max_seqlen.1,
        };
        check(sys::b200_attention_varlen(
            self.0, stream, in_dtype as c_int, out_dtype as c_int, q.ptr, q.shape.as_ptr(), q.strides.as_ptr(), k.ptr,
            k.shape.as_ptr(), k.strides.as_ptr(), v.ptr, v.shape.as_ptr(), v.strides.as_ptr(), cu_seqlens_q, cu_seqlens_k, batch,
            out.ptr, out.shape.as_ptr(), out.strides.as_ptr(), lse, &a,
        ))
    }

    /// Variable-length (packed) attention, backward: dq [Tq, Hq, D], dk and dv [Tk, Hkv, D] in `grad_dtype` from q, k, v, the
    /// forward's `out` and `lse` (compact f32 [Hq, Tq]) and `dout`, with the forward's offsets, window and scale.  See
    /// b200_attention_varlen_backward in cubecl_b200.h.
    ///
    /// # Safety
    /// Same contract as [`Context::attention_varlen`]; `lse` must hold Hq * Tq f32 values.
    pub unsafe fn attention_varlen_backward(
        &mut self, stream: b200_stream, in_dtype: DType, out_dtype: DType, grad_dtype: DType, q: &TensorView, k: &TensorView,
        v: &TensorView, out: &TensorView, dout: &TensorView, lse: b200_dptr, cu_seqlens_q: b200_dptr, cu_seqlens_k: b200_dptr,
        batch: u64, max_seqlen: (i32, i32), dq: &TensorView, dk: &TensorView, dv: &TensorView, scale: f32, window: (i32, i32),
    ) -> Result<(), Error> {
        for t in [q, k, v, out, dout, dq, dk, dv] {
            assert!(t.shape.len() == 3 && t.strides.len() == 3);
        }
        let a = sys::b200_attention_varlen_args {
            scale, window_left: window.0, window_right: window.1, max_seqlen_q: max_seqlen.0, max_seqlen_k: max_seqlen.1,
        };
        check(sys::b200_attention_varlen_backward(
            self.0, stream, in_dtype as c_int, out_dtype as c_int, grad_dtype as c_int, q.ptr, q.shape.as_ptr(), q.strides.as_ptr(),
            k.ptr, k.shape.as_ptr(), k.strides.as_ptr(), v.ptr, v.shape.as_ptr(), v.strides.as_ptr(), out.ptr, out.shape.as_ptr(),
            out.strides.as_ptr(), dout.ptr, dout.shape.as_ptr(), dout.strides.as_ptr(), lse, cu_seqlens_q, cu_seqlens_k, batch,
            dq.ptr, dq.shape.as_ptr(), dq.strides.as_ptr(), dk.ptr, dk.shape.as_ptr(), dk.strides.as_ptr(), dv.ptr, dv.shape.as_ptr(),
            dv.strides.as_ptr(), &a,
        ))
    }

    /// Attention of q [B, Hq, Sq, D] against a KV cache `k_cache`, `v_cache` [P, page, Hkv, D] (views by strides): sequence b
    /// sees its first `cache_seqlens`[b] keys (a compact i32 [B] device buffer), key j in page `block_table`[b, j / page] (an
    /// i32 [B, max_pages] view; `None`: page b); `causal` is bottom-right.  See b200_attention_kvcache in cubecl_b200.h.
    ///
    /// # Safety
    /// Same contract as [`Context::conv2d`]; `cache_seqlens` must hold B i32 values and `lse`, when non-zero, B * Hq * Sq f32
    /// values.
    pub unsafe fn attention_kvcache(
        &mut self, stream: b200_stream, in_dtype: DType, out_dtype: DType, q: &TensorView, k_cache: &TensorView, v_cache: &TensorView,
        block_table: Option<&TensorView>, cache_seqlens: b200_dptr, out: &TensorView, lse: b200_dptr, scale: f32, causal: bool,
    ) -> Result<(), Error> {
        for t in [q, k_cache, v_cache, out] {
            assert!(t.shape.len() == 4 && t.strides.len() == 4);
        }
        if let Some(t) = block_table {
            assert!(t.shape.len() == 2 && t.strides.len() == 2);
        }
        let a = sys::b200_attention_args { scale, causal: causal as i32 };
        let (bt, bt_shape, bt_strides) = match block_table {
            Some(t) => (t.ptr, t.shape.as_ptr(), t.strides.as_ptr()),
            None => (0, std::ptr::null(), std::ptr::null()),
        };
        check(sys::b200_attention_kvcache(
            self.0, stream, in_dtype as c_int, out_dtype as c_int, q.ptr, q.shape.as_ptr(), q.strides.as_ptr(), k_cache.ptr,
            k_cache.shape.as_ptr(), k_cache.strides.as_ptr(), v_cache.ptr, v_cache.shape.as_ptr(), v_cache.strides.as_ptr(), bt,
            bt_shape, bt_strides, cache_seqlens, out.ptr, out.shape.as_ptr(), out.strides.as_ptr(), lse, &a,
        ))
    }

    /// Paged variable-length attention: packed q [Tq, Hq, D] -> out [Tq, Hq, D] (sequence b owns rows [cu_q[b], cu_q[b + 1]),
    /// a compact i32 [batch + 1] device buffer) against `k_cache`, `v_cache` [P, page, Hkv, D] in q's dtype: sequence b sees its
    /// first `cache_seqlens`[b] keys (a compact i32 [batch] device buffer), key j in page `block_table`[b, j / page] (an i32
    /// [batch, max_pages] view; `None`: page b); `window` as [`Context::attention_varlen`]'s with the queries aligned to the last
    /// keys.  See b200_attention_varlen_paged in cubecl_b200.h.
    ///
    /// # Safety
    /// Same contract as [`Context::conv2d`]; `cu_seqlens_q` must hold batch + 1 i32 values, `cache_seqlens` batch, and `lse`,
    /// when non-zero, Hq * Tq f32 values.
    pub unsafe fn attention_varlen_paged(
        &mut self, stream: b200_stream, in_dtype: DType, out_dtype: DType, q: &TensorView, k_cache: &TensorView, v_cache: &TensorView,
        block_table: Option<&TensorView>, cu_seqlens_q: b200_dptr, cache_seqlens: b200_dptr, batch: u64, max_seqlen: (i32, i32),
        out: &TensorView, lse: b200_dptr, scale: f32, window: (i32, i32),
    ) -> Result<(), Error> {
        for t in [q, out] {
            assert!(t.shape.len() == 3 && t.strides.len() == 3);
        }
        for t in [k_cache, v_cache] {
            assert!(t.shape.len() == 4 && t.strides.len() == 4);
        }
        if let Some(t) = block_table {
            assert!(t.shape.len() == 2 && t.strides.len() == 2);
        }
        let a = sys::b200_attention_varlen_args {
            scale, window_left: window.0, window_right: window.1, max_seqlen_q: max_seqlen.0, max_seqlen_k: max_seqlen.1,
        };
        let (bt, bt_shape, bt_strides) = match block_table {
            Some(t) => (t.ptr, t.shape.as_ptr(), t.strides.as_ptr()),
            None => (0, std::ptr::null(), std::ptr::null()),
        };
        check(sys::b200_attention_varlen_paged(
            self.0, stream, in_dtype as c_int, out_dtype as c_int, q.ptr, q.shape.as_ptr(), q.strides.as_ptr(), k_cache.ptr,
            k_cache.shape.as_ptr(), k_cache.strides.as_ptr(), v_cache.ptr, v_cache.shape.as_ptr(), v_cache.strides.as_ptr(), bt,
            bt_shape, bt_strides, cu_seqlens_q, cache_seqlens, batch, out.ptr, out.shape.as_ptr(), out.strides.as_ptr(), lse, &a,
        ))
    }

    /// Scatter of `k_new`, `v_new` [B, Snew, Hkv, D] into `k_cache`, `v_cache` [P, page, Hkv, D]: token b * Snew + t goes to flat
    /// slot `slot_mapping`[b * Snew + t] (a compact i32 device buffer; negative slots are skipped).  See b200_kvcache_write.
    ///
    /// # Safety
    /// Same contract as [`Context::conv2d`]; `slot_mapping` must hold B * Snew i32 values.
    pub unsafe fn kvcache_write(
        &mut self, stream: b200_stream, dtype: DType, k_new: &TensorView, v_new: &TensorView, k_cache: &TensorView, v_cache: &TensorView,
        slot_mapping: b200_dptr,
    ) -> Result<(), Error> {
        for t in [k_new, v_new, k_cache, v_cache] {
            assert!(t.shape.len() == 4 && t.strides.len() == 4);
        }
        check(sys::b200_kvcache_write(
            self.0, stream, dtype as c_int, k_new.ptr, k_new.shape.as_ptr(), k_new.strides.as_ptr(), v_new.ptr, v_new.shape.as_ptr(),
            v_new.strides.as_ptr(), k_cache.ptr, k_cache.shape.as_ptr(), k_cache.strides.as_ptr(), v_cache.ptr, v_cache.shape.as_ptr(),
            v_cache.strides.as_ptr(), slot_mapping,
        ))
    }

    /// [`Context::attention_kvcache`] against an fp8 cache: `k_cache`, `v_cache` in `cache_dtype` (F8E4M3 or F8E5M2) hold
    /// K = k_scale[hk] * k8 and V = v_scale[hk] * v8, with `k_scale`, `v_scale` compact f32 [Hkv] device buffers.  See
    /// b200_attention_kvcache_fp8 in cubecl_b200.h.
    ///
    /// # Safety
    /// Same contract as [`Context::attention_kvcache`]; `k_scale` and `v_scale` must hold Hkv f32 values.
    pub unsafe fn attention_kvcache_fp8(
        &mut self, stream: b200_stream, in_dtype: DType, cache_dtype: DType, out_dtype: DType, q: &TensorView, k_cache: &TensorView,
        v_cache: &TensorView, block_table: Option<&TensorView>, cache_seqlens: b200_dptr, k_scale: b200_dptr, v_scale: b200_dptr,
        out: &TensorView, lse: b200_dptr, scale: f32, causal: bool,
    ) -> Result<(), Error> {
        for t in [q, k_cache, v_cache, out] {
            assert!(t.shape.len() == 4 && t.strides.len() == 4);
        }
        if let Some(t) = block_table {
            assert!(t.shape.len() == 2 && t.strides.len() == 2);
        }
        let a = sys::b200_attention_args { scale, causal: causal as i32 };
        let (bt, bt_shape, bt_strides) = match block_table {
            Some(t) => (t.ptr, t.shape.as_ptr(), t.strides.as_ptr()),
            None => (0, std::ptr::null(), std::ptr::null()),
        };
        check(sys::b200_attention_kvcache_fp8(
            self.0, stream, in_dtype as c_int, cache_dtype as c_int, out_dtype as c_int, q.ptr, q.shape.as_ptr(), q.strides.as_ptr(),
            k_cache.ptr, k_cache.shape.as_ptr(), k_cache.strides.as_ptr(), v_cache.ptr, v_cache.shape.as_ptr(), v_cache.strides.as_ptr(),
            bt, bt_shape, bt_strides, cache_seqlens, k_scale, v_scale, out.ptr, out.shape.as_ptr(), out.strides.as_ptr(), lse, &a,
        ))
    }

    /// [`Context::kvcache_write`] into fp8 caches (`cache_dtype` F8E4M3 or F8E5M2): each value x of kv head hk is stored as
    /// sat_rn(x / scale[hk]).  See b200_kvcache_write_fp8.
    ///
    /// # Safety
    /// Same contract as [`Context::kvcache_write`]; `k_scale` and `v_scale` must hold Hkv f32 values.
    pub unsafe fn kvcache_write_fp8(
        &mut self, stream: b200_stream, dtype: DType, cache_dtype: DType, k_new: &TensorView, v_new: &TensorView, k_cache: &TensorView,
        v_cache: &TensorView, slot_mapping: b200_dptr, k_scale: b200_dptr, v_scale: b200_dptr,
    ) -> Result<(), Error> {
        for t in [k_new, v_new, k_cache, v_cache] {
            assert!(t.shape.len() == 4 && t.strides.len() == 4);
        }
        check(sys::b200_kvcache_write_fp8(
            self.0, stream, dtype as c_int, cache_dtype as c_int, k_new.ptr, k_new.shape.as_ptr(), k_new.strides.as_ptr(), v_new.ptr,
            v_new.shape.as_ptr(), v_new.strides.as_ptr(), k_cache.ptr, k_cache.shape.as_ptr(), k_cache.strides.as_ptr(), v_cache.ptr,
            v_cache.shape.as_ptr(), v_cache.strides.as_ptr(), slot_mapping, k_scale, v_scale,
        ))
    }

    /// [`Context::attention_varlen_paged`] against an fp8 cache: `k_cache`, `v_cache` in `cache_dtype` (F8E4M3 or F8E5M2) hold
    /// K = k_scale[hk] * k8 and V = v_scale[hk] * v8, with `k_scale`, `v_scale` compact f32 [Hkv] device buffers.  See
    /// b200_attention_varlen_paged_fp8 in cubecl_b200.h.
    ///
    /// # Safety
    /// Same contract as [`Context::attention_varlen_paged`]; `k_scale` and `v_scale` must hold Hkv f32 values.
    pub unsafe fn attention_varlen_paged_fp8(
        &mut self, stream: b200_stream, in_dtype: DType, cache_dtype: DType, out_dtype: DType, q: &TensorView, k_cache: &TensorView,
        v_cache: &TensorView, block_table: Option<&TensorView>, cu_seqlens_q: b200_dptr, cache_seqlens: b200_dptr, batch: u64,
        k_scale: b200_dptr, v_scale: b200_dptr, max_seqlen: (i32, i32), out: &TensorView, lse: b200_dptr, scale: f32, window: (i32, i32),
    ) -> Result<(), Error> {
        for t in [q, out] {
            assert!(t.shape.len() == 3 && t.strides.len() == 3);
        }
        for t in [k_cache, v_cache] {
            assert!(t.shape.len() == 4 && t.strides.len() == 4);
        }
        if let Some(t) = block_table {
            assert!(t.shape.len() == 2 && t.strides.len() == 2);
        }
        let a = sys::b200_attention_varlen_args {
            scale, window_left: window.0, window_right: window.1, max_seqlen_q: max_seqlen.0, max_seqlen_k: max_seqlen.1,
        };
        let (bt, bt_shape, bt_strides) = match block_table {
            Some(t) => (t.ptr, t.shape.as_ptr(), t.strides.as_ptr()),
            None => (0, std::ptr::null(), std::ptr::null()),
        };
        check(sys::b200_attention_varlen_paged_fp8(
            self.0, stream, in_dtype as c_int, cache_dtype as c_int, out_dtype as c_int, q.ptr, q.shape.as_ptr(), q.strides.as_ptr(),
            k_cache.ptr, k_cache.shape.as_ptr(), k_cache.strides.as_ptr(), v_cache.ptr, v_cache.shape.as_ptr(), v_cache.strides.as_ptr(),
            bt, bt_shape, bt_strides, cu_seqlens_q, cache_seqlens, batch, k_scale, v_scale, out.ptr, out.shape.as_ptr(),
            out.strides.as_ptr(), lse, &a,
        ))
    }

    /// Grouped / depthwise [`Context::conv2d`]: w [Cout, KH, KW, C / groups].  See b200_conv2d_grouped in cubecl_b200.h.
    ///
    /// # Safety
    /// Same contract as [`Context::conv2d`].
    pub unsafe fn conv2d_grouped(
        &mut self, stream: b200_stream, in_dtype: DType, out_dtype: DType, x: &TensorView, w: &TensorView, out: &TensorView,
        args: [i32; 6], groups: u32, epilogue: Option<&Epilogue>,
    ) -> Result<(), Error> {
        assert!(x.shape.len() == 4 && w.shape.len() == 4 && out.shape.len() == 4);
        assert!(x.strides.len() == 4 && w.strides.len() == 4 && out.strides.len() == 4);
        let a = sys::b200_conv2d_args {
            stride_h: args[0], stride_w: args[1], pad_h: args[2], pad_w: args[3], dilation_h: args[4], dilation_w: args[5],
        };
        let e = epilogue.map(|e| sys::b200_epilogue { alpha: e.alpha, activation: e.activation as i32, bias: e.bias });
        check(sys::b200_conv2d_grouped(
            self.0, stream, in_dtype as c_int, out_dtype as c_int, x.ptr, x.shape.as_ptr(), x.strides.as_ptr(), w.ptr,
            w.shape.as_ptr(), w.strides.as_ptr(), out.ptr, out.shape.as_ptr(), out.strides.as_ptr(), &a, groups,
            e.as_ref().map_or(std::ptr::null(), |e| e as *const sys::b200_epilogue),
        ))
    }

    /// Input gradient of [`Context::conv2d_grouped`].  See b200_conv2d_grouped_backward_data in cubecl_b200.h.
    ///
    /// # Safety
    /// Same contract as [`Context::matmul`] for the three pointers.
    pub unsafe fn conv2d_grouped_backward_data(
        &mut self, stream: b200_stream, in_dtype: DType, out_dtype: DType, dy: &TensorView, w: &TensorView, dx: &TensorView,
        args: [i32; 6], groups: u32,
    ) -> Result<(), Error> {
        assert!(dy.shape.len() == 4 && w.shape.len() == 4 && dx.shape.len() == 4);
        assert!(dy.strides.len() == 4 && w.strides.len() == 4 && dx.strides.len() == 4);
        let a = sys::b200_conv2d_args {
            stride_h: args[0], stride_w: args[1], pad_h: args[2], pad_w: args[3], dilation_h: args[4], dilation_w: args[5],
        };
        check(sys::b200_conv2d_grouped_backward_data(
            self.0, stream, in_dtype as c_int, out_dtype as c_int, dy.ptr, dy.shape.as_ptr(), dy.strides.as_ptr(), w.ptr,
            w.shape.as_ptr(), w.strides.as_ptr(), dx.ptr, dx.shape.as_ptr(), dx.strides.as_ptr(), &a, groups,
        ))
    }

    /// Weight gradient of [`Context::conv2d_grouped`]: dw [Cout, KH, KW, C / groups].  See
    /// b200_conv2d_grouped_backward_weight in cubecl_b200.h.
    ///
    /// # Safety
    /// Same contract as [`Context::matmul`] for the three pointers.
    pub unsafe fn conv2d_grouped_backward_weight(
        &mut self, stream: b200_stream, in_dtype: DType, out_dtype: DType, x: &TensorView, dy: &TensorView, dw: &TensorView,
        args: [i32; 6], groups: u32,
    ) -> Result<(), Error> {
        assert!(x.shape.len() == 4 && dy.shape.len() == 4 && dw.shape.len() == 4);
        assert!(x.strides.len() == 4 && dy.strides.len() == 4 && dw.strides.len() == 4);
        let a = sys::b200_conv2d_args {
            stride_h: args[0], stride_w: args[1], pad_h: args[2], pad_w: args[3], dilation_h: args[4], dilation_w: args[5],
        };
        check(sys::b200_conv2d_grouped_backward_weight(
            self.0, stream, in_dtype as c_int, out_dtype as c_int, x.ptr, x.shape.as_ptr(), x.strides.as_ptr(), dy.ptr,
            dy.shape.as_ptr(), dy.strides.as_ptr(), dw.ptr, dw.shape.as_ptr(), dw.strides.as_ptr(), &a, groups,
        ))
    }

    /// Block-scaled (MX / NVFP4) matmul: lhs [batch, m, k], rhs [batch, n, k] K-contiguous, scales per `scale_block`
    /// (32: ue8m0, 16: e4m3) elements of K; replaces `MmaDefinition::new_scaled` / `execute_scaled` tiles
    /// (crates/cubecl-core/src/frontend/cmma.rs:438-460, 798-840) at GEMM level.
    ///
    /// # Safety
    /// Same contract as [`Context::matmul`] for all five pointers.
    #[allow(clippy::too_many_arguments)]
    pub unsafe fn matmul_scaled(
        &mut self, stream: b200_stream, lhs_dtype: DType, rhs_dtype: DType, out_dtype: DType,
        lhs: b200_dptr, rhs: b200_dptr, lhs_scales: b200_dptr, rhs_scales: b200_dptr, out: b200_dptr,
        batch: u64, m: u64, n: u64, k: u64, scale_block: i32, scales_packed: bool,
    ) -> Result<(), Error> {
        check(sys::b200_matmul_scaled(
            self.0, stream, lhs_dtype as c_int, rhs_dtype as c_int, out_dtype as c_int, lhs, rhs, lhs_scales, rhs_scales,
            out, batch, m, n, k, scale_block as c_int, scales_packed as c_int,
        ))
    }

    // ---- reduce::launch ---------------------------------------------------------------------------------------------
    /// Reduce `axis` (None = every element); output contiguous f32 (u32 indices for arg ops).
    ///
    /// # Safety
    /// Same contract as [`Context::matmul`].
    pub unsafe fn reduce(
        &mut self, stream: b200_stream, op: ReduceOp, in_dtype: DType, input: &TensorView, out: b200_dptr,
        axis: Option<usize>,
    ) -> Result<(), Error> {
        assert!(input.strides.len() == input.shape.len());
        check(sys::b200_reduce_strided(
            self.0, stream, op as c_int, in_dtype as c_int, input.ptr, out, input.shape.len() as c_int,
            input.shape.as_ptr(), input.strides.as_ptr(), axis.map(|a| a as c_int).unwrap_or(-1),
        ))
    }

    /// Inclusive (or exclusive) cumulative sum / prod / max / min of `axis` into the compact row-major `out` of the input's
    /// shape; `out_dtype` F32 or the input's (the device-wide form of the plane scans, runtime_tests/plane.rs:191-405).
    ///
    /// # Safety
    /// Same contract as [`Context::matmul`].
    #[allow(clippy::too_many_arguments)]
    pub unsafe fn scan(
        &mut self, stream: b200_stream, op: ReduceOp, exclusive: bool, in_dtype: DType, out_dtype: DType, input: &TensorView,
        out: b200_dptr, axis: usize,
    ) -> Result<(), Error> {
        assert!(input.strides.len() == input.shape.len());
        check(sys::b200_scan(
            self.0, stream, op as c_int, exclusive as c_int, in_dtype as c_int, out_dtype as c_int, input.ptr, out,
            input.shape.len() as c_int, input.shape.as_ptr(), input.strides.as_ptr(), axis as c_int,
        ))
    }

    /// Mixture-of-experts top-k gating: `logits` [t, e] (F32 / BF16 / F16, row stride `logits_stride`) -> `ids` i32 [t, k] and
    /// `weights` f32 [t, k]; `bias` is an f32 [e] selection bias or 0.  The contract is `b200_moe_route`'s in
    /// include/cubecl_b200.h.
    ///
    /// # Safety
    /// Every pointer must be a live device allocation of this context large enough for its extents.
    #[allow(clippy::too_many_arguments)]
    pub unsafe fn moe_route(
        &mut self, stream: b200_stream, logits_dtype: DType, logits: b200_dptr, t: u64, e: u64, logits_stride: u64, bias: b200_dptr,
        args: &sys::b200_moe_route_args, ids: b200_dptr, weights: b200_dptr,
    ) -> Result<(), Error> {
        check(sys::b200_moe_route(self.0, stream, logits_dtype as c_int, logits, t, e, logits_stride, bias, args, ids, weights))
    }

    /// The expert-sorted dispatch plan of `ids` i32 [t, k] over `e` experts: `offs` i32 [e] (what the grouped matmuls take),
    /// `row_of` i32 [t, k] and `slot_of` i32 [t * k].  See `b200_moe_plan`.
    ///
    /// # Safety
    /// Same contract as [`Context::moe_route`].
    #[allow(clippy::too_many_arguments)]
    pub unsafe fn moe_plan(
        &mut self, stream: b200_stream, ids: b200_dptr, t: u64, k: u64, e: u64, offs: b200_dptr, row_of: b200_dptr, slot_of: b200_dptr,
    ) -> Result<(), Error> {
        check(sys::b200_moe_plan(self.0, stream, ids, t, k, e, offs, row_of, slot_of))
    }

    /// Gather rows into expert order: dst[r] = src[slot_of[r] / k], rows of `row_bytes` bytes at byte pitches.  See
    /// `b200_moe_permute`.
    ///
    /// # Safety
    /// Same contract as [`Context::moe_route`].
    #[allow(clippy::too_many_arguments)]
    pub unsafe fn moe_permute(
        &mut self, stream: b200_stream, src: b200_dptr, src_pitch: u64, slot_of: b200_dptr, t: u64, k: u64, dst: b200_dptr,
        dst_pitch: u64, row_bytes: u64,
    ) -> Result<(), Error> {
        check(sys::b200_moe_permute(self.0, stream, src, src_pitch, slot_of, t, k, dst, dst_pitch, row_bytes))
    }

    /// Weighted un-permute: y [t, n] = sum_j weights[t, j] * ys[row_of[t, j]] (`weights` 0: the plain sum).  See
    /// `b200_moe_combine`.
    ///
    /// # Safety
    /// Same contract as [`Context::moe_route`].
    #[allow(clippy::too_many_arguments)]
    pub unsafe fn moe_combine(
        &mut self, stream: b200_stream, ys_dtype: DType, y_dtype: DType, ys: b200_dptr, rows: u64, ys_stride: u64, weights: b200_dptr,
        row_of: b200_dptr, t: u64, k: u64, n: u64, y: b200_dptr, y_stride: u64,
    ) -> Result<(), Error> {
        check(sys::b200_moe_combine(
            self.0, stream, ys_dtype as c_int, y_dtype as c_int, ys, rows, ys_stride, weights, row_of, t, k, n, y, y_stride,
        ))
    }

    /// Gradients of [`Context::moe_combine`]: d_ys [rows, n] in `grad_dtype` and d_w f32 [t, k].  See
    /// `b200_moe_combine_backward`.
    ///
    /// # Safety
    /// Same contract as [`Context::moe_route`].
    #[allow(clippy::too_many_arguments)]
    pub unsafe fn moe_combine_backward(
        &mut self, stream: b200_stream, grad_dtype: DType, ys_dtype: DType, dy: b200_dptr, dy_stride: u64, ys: b200_dptr, rows: u64,
        ys_stride: u64, weights: b200_dptr, row_of: b200_dptr, t: u64, k: u64, n: u64, d_ys: b200_dptr, d_ys_stride: u64,
        d_w: b200_dptr,
    ) -> Result<(), Error> {
        check(sys::b200_moe_combine_backward(
            self.0, stream, grad_dtype as c_int, ys_dtype as c_int, dy, dy_stride, ys, rows, ys_stride, weights, row_of, t, k, n, d_ys,
            d_ys_stride, d_w,
        ))
    }

    /// RMSNorm / LayerNorm of rows `x` [t, n] (x_stride elements apart) into `y` (`y_dtype`), with an optional fused residual
    /// (`residual` and `h_out` both non-zero: h = x + residual rounded to x's dtype, written to `h_out`); `weight`, `bias`,
    /// `mean` and `rstd` may be 0.  The contract is `b200_norm`'s in include/cubecl_b200.h.
    ///
    /// # Safety
    /// Every pointer must be 0 where the contract allows it, or a live device allocation of this context large enough for
    /// its extents and strides.
    #[allow(clippy::too_many_arguments)]
    pub unsafe fn norm(
        &mut self, stream: b200_stream, args: &sys::b200_norm_args, y_dtype: DType, t: u64, n: u64, x: b200_dptr, x_stride: u64,
        residual: b200_dptr, residual_stride: u64, h_out: b200_dptr, h_stride: u64, weight: b200_dptr, bias: b200_dptr,
        y: b200_dptr, y_stride: u64, mean: b200_dptr, rstd: b200_dptr,
    ) -> Result<(), Error> {
        check(sys::b200_norm(
            self.0, stream, args, y_dtype as c_int, t, n, x, x_stride, residual, residual_stride, h_out, h_stride, weight, bias, y,
            y_stride, mean, rstd,
        ))
    }

    /// [`Context::norm`] with y stored as fp8 codes `values` [t, n] and `block_scales` [t, n / block], bit for bit what
    /// `b200_quantize(scheme)` writes for the f32 output.  See `b200_norm_quantized_fp8`.
    ///
    /// # Safety
    /// Same contract as [`Context::norm`].
    #[allow(clippy::too_many_arguments)]
    pub unsafe fn norm_quantized_fp8(
        &mut self, stream: b200_stream, args: &sys::b200_norm_args, scheme: &QuantScheme, t: u64, n: u64, x: b200_dptr,
        x_stride: u64, residual: b200_dptr, residual_stride: u64, h_out: b200_dptr, h_stride: u64, weight: b200_dptr,
        bias: b200_dptr, values: b200_dptr, block_scales: b200_dptr, mean: b200_dptr, rstd: b200_dptr,
    ) -> Result<(), Error> {
        let raw = scheme.raw();
        check(sys::b200_norm_quantized_fp8(
            self.0, stream, args, &raw, t, n, x, x_stride, residual, residual_stride, h_out, h_stride, weight, bias, values,
            block_scales, mean, rstd,
        ))
    }

    /// Gradients of [`Context::norm`]: `dx` [t, n] in `grad_dtype` (plus `d_h`, the residual stream's gradient, when
    /// non-zero), `dweight` and `dbias` f32 [n] (0 = not computed), from `dy`, the forward's `h`, `weight`, `rstd` and, for
    /// LayerNorm, `mean`.  See `b200_norm_backward`.
    ///
    /// # Safety
    /// Same contract as [`Context::norm`].
    #[allow(clippy::too_many_arguments)]
    pub unsafe fn norm_backward(
        &mut self, stream: b200_stream, args: &sys::b200_norm_args, grad_dtype: DType, t: u64, n: u64, dy: b200_dptr,
        dy_stride: u64, h: b200_dptr, h_stride: u64, weight: b200_dptr, mean: b200_dptr, rstd: b200_dptr, d_h: b200_dptr,
        d_h_stride: u64, dx: b200_dptr, dx_stride: u64, dweight: b200_dptr, dbias: b200_dptr,
    ) -> Result<(), Error> {
        check(sys::b200_norm_backward(
            self.0, stream, args, grad_dtype as c_int, t, n, dy, dy_stride, h, h_stride, weight, mean, rstd, d_h, d_h_stride, dx,
            dx_stride, dweight, dbias,
        ))
    }

    /// Rotate `q` [B, S, Hq, D] and / or `k` [B, S, Hk, D] (0 = absent; shapes and strides in elements, null strides =
    /// compact) by the rows of the f32 table `cos_sin` [p, rot_dim] at `positions` (i32 [B, S], 0 = s), in place or into
    /// `q_out` / `k_out`.  The contract is `b200_rope`'s in include/cubecl_b200.h.
    ///
    /// # Safety
    /// Every pointer must be 0 where the contract allows it, or a live device allocation of this context large enough for
    /// its extents and strides; every shape and stride pointer must point at 4 values (or be null where allowed).
    #[allow(clippy::too_many_arguments)]
    pub unsafe fn rope(
        &mut self, stream: b200_stream, args: &sys::b200_rope_args, dtype: DType, q: b200_dptr, q_shape: *const u64,
        q_strides: *const u64, k: b200_dptr, k_shape: *const u64, k_strides: *const u64, q_out: b200_dptr, qo_shape: *const u64,
        qo_strides: *const u64, k_out: b200_dptr, ko_shape: *const u64, ko_strides: *const u64, positions: b200_dptr,
        cos_sin: b200_dptr, p: u64,
    ) -> Result<(), Error> {
        check(sys::b200_rope(
            self.0, stream, args, dtype as c_int, q, q_shape, q_strides, k, k_shape, k_strides, q_out, qo_shape, qo_strides, k_out,
            ko_shape, ko_strides, positions, cos_sin, p,
        ))
    }

    /// The decode / prefill step in one launch: [`Context::rope`] of `q` and `k_new`, with the rotated k and `v_new` written to
    /// their cache slots, bit for bit `b200_rope` then `b200_kvcache_write(_fp8)`.  See `b200_rope_kvcache_write`.
    ///
    /// # Safety
    /// Same contract as [`Context::rope`].
    #[allow(clippy::too_many_arguments)]
    pub unsafe fn rope_kvcache_write(
        &mut self, stream: b200_stream, args: &sys::b200_rope_args, dtype: DType, cache_dtype: DType, q: b200_dptr,
        q_shape: *const u64, q_strides: *const u64, q_out: b200_dptr, qo_shape: *const u64, qo_strides: *const u64, k_new: b200_dptr,
        kn_shape: *const u64, kn_strides: *const u64, v_new: b200_dptr, vn_shape: *const u64, vn_strides: *const u64,
        k_cache: b200_dptr, kc_shape: *const u64, kc_strides: *const u64, v_cache: b200_dptr, vc_shape: *const u64,
        vc_strides: *const u64, slot_mapping: b200_dptr, positions: b200_dptr, cos_sin: b200_dptr, p: u64, k_scale: b200_dptr,
        v_scale: b200_dptr,
    ) -> Result<(), Error> {
        check(sys::b200_rope_kvcache_write(
            self.0, stream, args, dtype as c_int, cache_dtype as c_int, q, q_shape, q_strides, q_out, qo_shape, qo_strides, k_new,
            kn_shape, kn_strides, v_new, vn_shape, vn_strides, k_cache, kc_shape, kc_strides, v_cache, vc_shape, vc_strides,
            slot_mapping, positions, cos_sin, p, k_scale, v_scale,
        ))
    }

    /// Fill `cos_sin` (compact f32 [p, rot_dim]) with the table of `args`' rule, computed in f64.  See `b200_rope_cos_sin`.
    ///
    /// # Safety
    /// `cos_sin` (and `args.inv_freq` when used) must be live device allocations of this context of the stated sizes.
    pub unsafe fn rope_cos_sin(
        &mut self, stream: b200_stream, args: &sys::b200_rope_table_args, p: u64, cos_sin: b200_dptr,
    ) -> Result<(), Error> {
        check(sys::b200_rope_cos_sin(self.0, stream, args, p, cos_sin))
    }

    /// Softmax cross-entropy of `logits` [t, v] (unit column stride, row stride `logits_stride` in elements) against
    /// `targets` (i32 / i64 [t]): `loss` (f32 [t] for NONE, one f32 otherwise) and `lse` (f32 [t], 0 = absent); with `dloss`
    /// and `dlogits` (0 = absent; may be `logits` itself) also the gradient in the same launch.  The contract is
    /// `b200_cross_entropy`'s in include/cubecl_b200.h.
    ///
    /// # Safety
    /// Every pointer must be 0 where the contract allows it, or a live device allocation of this context large enough for its
    /// extents and strides.
    #[allow(clippy::too_many_arguments)]
    pub unsafe fn cross_entropy(
        &mut self, stream: b200_stream, args: &sys::b200_xent_args, logits_dtype: DType, target_dtype: DType, t: u64, v: u64,
        logits: b200_dptr, logits_stride: u64, targets: b200_dptr, loss: b200_dptr, lse: b200_dptr, dloss: b200_dptr,
        grad_dtype: DType, dlogits: b200_dptr, dlogits_stride: u64,
    ) -> Result<(), Error> {
        check(sys::b200_cross_entropy(
            self.0, stream, args, logits_dtype as c_int, target_dtype as c_int, t, v, logits, logits_stride, targets, loss, lse,
            dloss, grad_dtype as c_int, dlogits, dlogits_stride,
        ))
    }

    /// The logits' gradient from the forward's `lse` and `dloss`; see `b200_cross_entropy_backward`.
    ///
    /// # Safety
    /// Same contract as [`Context::cross_entropy`].
    #[allow(clippy::too_many_arguments)]
    pub unsafe fn cross_entropy_backward(
        &mut self, stream: b200_stream, args: &sys::b200_xent_args, logits_dtype: DType, target_dtype: DType, grad_dtype: DType,
        t: u64, v: u64, logits: b200_dptr, logits_stride: u64, targets: b200_dptr, lse: b200_dptr, dloss: b200_dptr,
        dlogits: b200_dptr, dlogits_stride: u64,
    ) -> Result<(), Error> {
        check(sys::b200_cross_entropy_backward(
            self.0, stream, args, logits_dtype as c_int, target_dtype as c_int, grad_dtype as c_int, t, v, logits, logits_stride,
            targets, lse, dloss, dlogits, dlogits_stride,
        ))
    }

    /// Token sampling: `ids` (i32 / i64 [b]) drawn from `logits` [b, v] (unit column stride, row stride `logits_stride` in
    /// elements) under temperature, top-k, min-p and top-p, from per-row Philox seeds and offsets; -1 for an invalid row.  The
    /// contract is `b200_sample`'s in include/cubecl_b200.h.
    ///
    /// # Safety
    /// `logits`, `ids` and every non-zero per-row array of `args` must be live device allocations of this context large
    /// enough for `b` rows.
    #[allow(clippy::too_many_arguments)]
    pub unsafe fn sample(
        &mut self, stream: b200_stream, args: &sys::b200_sample_args, logits_dtype: DType, ids_dtype: DType, b: u64, v: u64,
        logits: b200_dptr, logits_stride: u64, ids: b200_dptr,
    ) -> Result<(), Error> {
        check(sys::b200_sample(self.0, stream, args, logits_dtype as c_int, ids_dtype as c_int, b, v, logits, logits_stride, ids))
    }

    /// Quantize `input` ([..., K], F32 / F16 / BF16, any strides) along its innermost axis under `scheme` into compact
    /// codes [..., K * bits / 8], block scales [..., K / block] and the f32 tensor scale (0 for an absent level); the
    /// contract is `b200_quantize`'s in include/cubecl_b200.h.
    ///
    /// # Safety
    /// Same contract as [`Context::matmul`].
    #[allow(clippy::too_many_arguments)]
    pub unsafe fn quantize(
        &mut self, stream: b200_stream, scheme: &QuantScheme, in_dtype: DType, input: &TensorView, values: b200_dptr,
        block_scales: b200_dptr, tensor_scale: b200_dptr,
    ) -> Result<(), Error> {
        assert!(input.strides.len() == input.shape.len());
        let raw = scheme.raw();
        check(sys::b200_quantize(
            self.0, stream, &raw, in_dtype as c_int, input.ptr, values, block_scales, tensor_scale, input.shape.len() as c_int,
            input.shape.as_ptr(), input.strides.as_ptr(),
        ))
    }

    /// out (compact, F32 / F16 / BF16) = the values of quantized codes of `shape` under `scheme` (`b200_dequantize`).
    ///
    /// # Safety
    /// Same contract as [`Context::matmul`].
    #[allow(clippy::too_many_arguments)]
    pub unsafe fn dequantize(
        &mut self, stream: b200_stream, scheme: &QuantScheme, out_dtype: DType, values: b200_dptr, block_scales: b200_dptr,
        tensor_scale: b200_dptr, out: b200_dptr, shape: &[u64],
    ) -> Result<(), Error> {
        let raw = scheme.raw();
        check(sys::b200_dequantize(
            self.0, stream, &raw, out_dtype as c_int, values, block_scales, tensor_scale, out, shape.len() as c_int,
            shape.as_ptr(),
        ))
    }

    /// out [batch, m, n] (contiguous, F32 / BF16 / F16) = deq(lhs) x deq(rhs)^T of two integer-quantized operands, codes
    /// [batch, m | n, k] quantized along k, on the s8 tensor cores with the scales applied inside the GEMM; the bit-exact
    /// contract is `b200_matmul_quantized`'s in include/cubecl_b200.h.
    ///
    /// # Safety
    /// Same contract as [`Context::matmul`].
    #[allow(clippy::too_many_arguments)]
    pub unsafe fn matmul_quantized(
        &mut self, stream: b200_stream, lhs: &QuantOperand, rhs: &QuantOperand, out_dtype: DType, out: b200_dptr, batch: u64,
        m: u64, n: u64, k: u64,
    ) -> Result<(), Error> {
        let (a, b) = (lhs.raw(), rhs.raw());
        check(sys::b200_matmul_quantized(self.0, stream, &a, &b, out_dtype as c_int, out, batch, m, n, k))
    }

    /// out [batch, m, n] (contiguous, F32 / BF16 / F16) = deq(lhs) x deq(rhs)^T of two fp8-quantized operands (E4M3 / E5M2 on
    /// either side), codes [batch, m | n, k] quantized along k, on the fp8 tensor cores with the block scales folded in f32
    /// inside the GEMM; the contract is `b200_matmul_quantized_fp8`'s in include/cubecl_b200.h.
    ///
    /// # Safety
    /// Same contract as [`Context::matmul`].
    #[allow(clippy::too_many_arguments)]
    pub unsafe fn matmul_quantized_fp8(
        &mut self, stream: b200_stream, lhs: &QuantOperand, rhs: &QuantOperand, out_dtype: DType, out: b200_dptr, batch: u64,
        m: u64, n: u64, k: u64,
    ) -> Result<(), Error> {
        let (a, b) = (lhs.raw(), rhs.raw());
        check(sys::b200_matmul_quantized_fp8(self.0, stream, &a, &b, out_dtype as c_int, out, batch, m, n, k))
    }

    /// out [t, n] (contiguous, F32 / BF16 / F16): grouped matmul of fp8-quantized operands for mixture-of-experts layers, lhs
    /// codes [t, k] (tokens sorted by expert) against rhs codes [groups, n, k] (the experts' weights), both quantized along k;
    /// `offs` is a compact i32 [groups] device array of cumulative ends read on the device only, and rows past the last group
    /// are not written.  The contract is `b200_matmul_grouped_quantized_fp8`'s in include/cubecl_b200.h.
    ///
    /// # Safety
    /// Same contract as [`Context::matmul`]; `offs` must hold `groups` i32 values on this context's device.
    #[allow(clippy::too_many_arguments)]
    pub unsafe fn matmul_grouped_quantized_fp8(
        &mut self, stream: b200_stream, lhs: &QuantOperand, rhs: &QuantOperand, offs: b200_dptr, groups: u64, out_dtype: DType,
        out: b200_dptr, t: u64, n: u64, k: u64,
    ) -> Result<(), Error> {
        let (a, b) = (lhs.raw(), rhs.raw());
        check(sys::b200_matmul_grouped_quantized_fp8(self.0, stream, &a, &b, offs, groups, out_dtype as c_int, out, t, n, k))
    }

    /// out (compact row-major) = gather of the strided tensor `input` (into_contiguous, cubecl-std/src/tensor/contiguous.rs).
    ///
    /// # Safety
    /// Same contract as [`Context::matmul`].
    pub unsafe fn into_contiguous(
        &mut self, stream: b200_stream, dtype: DType, input: &TensorView, out: b200_dptr,
    ) -> Result<(), Error> {
        assert!(input.strides.len() == input.shape.len());
        check(sys::b200_into_contiguous(
            self.0, stream, dtype as c_int, input.ptr, out, input.shape.len() as c_int, input.shape.as_ptr(),
            input.strides.as_ptr(),
        ))
    }

    // ---- collectives (ServerCommunication, server/base.rs:632-739) ---------------------------------------------------
    pub fn comm_unique_id(&mut self) -> Result<[u8; sys::B200_UNIQUE_ID_BYTES], Error> {
        let mut id = [0u8; sys::B200_UNIQUE_ID_BYTES];
        check(unsafe { sys::b200_comm_get_unique_id(self.0, id.as_mut_ptr() as *mut c_void) })?;
        Ok(id)
    }

    pub fn comm_init(&mut self, device_ids: &[i32], id: &[u8; sys::B200_UNIQUE_ID_BYTES]) -> Result<(), Error> {
        check(unsafe {
            sys::b200_comm_init(self.0, device_ids.as_ptr(), device_ids.len() as c_int, id.as_ptr() as *const c_void)
        })
    }

    /// In-place or out-of-place all-reduce of a whole buffer on the comm stream, ordered after `compute`.
    ///
    /// # Safety
    /// `src` / `dst` must be live device allocations of at least `bytes` bytes.
    pub unsafe fn all_reduce(
        &mut self, compute: b200_stream, src: b200_dptr, dst: b200_dptr, bytes: usize, dtype: DType, op: CommOp,
        device_ids: &[i32],
    ) -> Result<(), Error> {
        check(sys::b200_all_reduce(
            self.0, compute, src, dst, bytes, dtype as c_int, op as c_int, device_ids.as_ptr(), device_ids.len() as c_int,
        ))
    }

    /// Make `compute` wait for everything issued on the comm stream (server.rs:782-798).
    pub fn sync_collective(&mut self, compute: b200_stream) -> Result<(), Error> {
        check(unsafe { sys::b200_sync_collective(self.0, compute) })
    }

    /// Local f32 sum + exchange of the scalar through NVLink peer mailboxes in ONE kernel (after `b200_p2p_connect`).
    ///
    /// # Safety
    /// Same contract as [`Context::matmul`]; every rank of `device_ids` must make the same call.
    pub unsafe fn reduce_all_reduce(
        &mut self, stream: b200_stream, input: b200_dptr, out: b200_dptr, n: u64, device_ids: &[i32],
    ) -> Result<(), Error> {
        check(sys::b200_reduce_all_reduce(
            self.0, stream, ReduceOp::Sum as c_int, DType::F32 as c_int, input, out, n, device_ids.as_ptr(),
            device_ids.len() as c_int,
        ))
    }
}

impl Drop for Context {
    fn drop(&mut self) {
        unsafe { sys::b200_destroy(self.0) };
    }
}

/// The embedded prebuilt sm_90a image `name` ("gemm" | "gemm_b" | "gemm_c" | "reduce" | "aux") for a host that prefers to
/// `cuModuleLoadData` it into its own module cache (CudaContext::modules, cubecl-cuda/src/compute/context.rs:38-62,293).
pub fn cubin(name: &str) -> Result<&'static [u8], Error> {
    let n = CString::new(name).map_err(|_| Error { status: Status::InvalidArg as i32, message: "NUL in name".into() })?;
    let mut image: *const c_void = core::ptr::null();
    let mut size = 0usize;
    check(unsafe { sys::b200_get_cubin(n.as_ptr(), &mut image, &mut size) })?;
    Ok(unsafe { core::slice::from_raw_parts(image as *const u8, size) })
}
