//! cubek-shaped launch surface over the safe layer: `matmul::launch` / `reduce::launch` taking tensor handles, the
//! std-lib op convention of the reference (`op::launch(client, &TensorHandle...)`, crates/cubecl-std/src/tensor/
//! identity.rs:39-83).  SOURCE ONLY (no Rust toolchain in the authoring image); the Python mirror of exactly this logic
//! (cubecl_b200/matmul.py, reduce.py) is what the GPU parity tests drive.
//!
//! Inside cubecl-cuda the `Context` is owned by `CudaServer` and `TensorHandle::ptr` is what `BufferBinding` resolves to
//! on the runner thread (INTEGRATION.md section 3); standalone, it is a pointer from `Context::alloc`.

use crate::{b200_dptr, b200_stream, Context, DType, Error, Epilogue, QuantOperand, QuantScheme, ReduceOp, Status, TensorView};

/// Buffer + shape + strides (in ELEMENTS) + dtype: `TensorHandle<R>` of crates/cubecl-std/src/tensor/handle.rs:13-23
/// with the `Handle` already resolved to a device pointer.
#[derive(Clone, Debug)]
pub struct TensorHandle {
    pub ptr: b200_dptr,
    pub shape: Vec<u64>,
    pub strides: Vec<u64>,
    pub dtype: DType,
}

impl TensorHandle {
    /// Row-major contiguous strides for `shape` (`TensorHandle::new_contiguous`, handle.rs:62-75).
    pub fn new_contiguous(ptr: b200_dptr, shape: &[u64], dtype: DType) -> Self {
        let mut strides = vec![1u64; shape.len()];
        for i in (0..shape.len().saturating_sub(1)).rev() {
            strides[i] = strides[i + 1] * shape[i + 1];
        }
        Self { ptr, shape: shape.to_vec(), strides, dtype }
    }

    /// Swap the last two dims without moving data (`MatrixBatchLayout::MildlyPermuted { transposed: true, .. }`,
    /// crates/cubecl-std/src/tensor/matrix_batch_layout.rs:8-19): goes straight into a TMA descriptor, no copy.
    pub fn transposed(&self) -> Self {
        let r = self.shape.len();
        assert!(r >= 2);
        let mut t = self.clone();
        t.shape.swap(r - 2, r - 1);
        t.strides.swap(r - 2, r - 1);
        t
    }

    fn view(&self) -> TensorView<'_> {
        TensorView { ptr: self.ptr, shape: &self.shape, strides: &self.strides }
    }
}

fn invalid(message: String) -> Error {
    Error { status: Status::InvalidArg as i32, message }
}

pub mod matmul {
    use super::*;

    /// Batch-broadcast matmul shape rule, restated from crates/cubecl-zspace/src/shape.rs:489-517: equal rank >= 2;
    /// leading dims equal or one of them 1; inner dims agree.
    pub fn calculate_matmul_output(lhs: &[u64], rhs: &[u64]) -> Result<Vec<u64>, Error> {
        let rank = lhs.len();
        if rank != rhs.len() {
            return Err(invalid(format!("rank mismatch: lhs {}, rhs {}", rank, rhs.len())));
        }
        if rank < 2 {
            return Err(invalid("matmul needs rank >= 2".to_string()));
        }
        let mut out = Vec::with_capacity(rank);
        for i in 0..rank - 2 {
            let (l, r) = (lhs[i], rhs[i]);
            if l == r || r == 1 {
                out.push(l);
            } else if l == 1 {
                out.push(r);
            } else {
                return Err(invalid(format!("batch dims {} and {} cannot broadcast", l, r)));
            }
        }
        if lhs[rank - 1] != rhs[rank - 2] {
            return Err(invalid(format!("inner dims differ: lhs k={}, rhs k={}", lhs[rank - 1], rhs[rank - 2])));
        }
        out.push(lhs[rank - 2]);
        out.push(rhs[rank - 1]);
        Ok(out)
    }

    /// `matmul::launch(client, lhs, rhs, out)`: out[.., m, n] = sum_k lhs[.., m, k] * rhs[.., k, n], f32 accumulation.
    /// Shape errors are returned here; device faults surface at the next `Context::sync` like the reference's launches.
    ///
    /// # Safety
    /// The handles must describe live device allocations of `ctx`'s device that outlive the enqueued launch.
    pub unsafe fn launch(
        ctx: &mut Context, stream: b200_stream, lhs: &TensorHandle, rhs: &TensorHandle, out: &TensorHandle,
    ) -> Result<(), Error> {
        if lhs.dtype != rhs.dtype {
            return Err(invalid("lhs and rhs dtypes differ".to_string()));
        }
        let expect = calculate_matmul_output(&lhs.shape, &rhs.shape)?;
        if expect != out.shape {
            return Err(invalid(format!("out shape {:?} != {:?}", out.shape, expect)));
        }
        ctx.matmul(stream, lhs.dtype, out.dtype, &lhs.view(), &rhs.view(), &out.view())
    }

    /// out = act(alpha * (lhs @ rhs) + bias[n]) inside the GEMM epilogue.
    ///
    /// # Safety
    /// As [`launch`]; `epilogue.bias` must be 0 or an f32[N] device allocation.
    pub unsafe fn launch_fused(
        ctx: &mut Context, stream: b200_stream, lhs: &TensorHandle, rhs: &TensorHandle, out: &TensorHandle,
        epilogue: &Epilogue,
    ) -> Result<(), Error> {
        if lhs.dtype != rhs.dtype {
            return Err(invalid("lhs and rhs dtypes differ".to_string()));
        }
        let expect = calculate_matmul_output(&lhs.shape, &rhs.shape)?;
        if expect != out.shape {
            return Err(invalid(format!("out shape {:?} != {:?}", out.shape, expect)));
        }
        ctx.matmul_fused(stream, lhs.dtype, out.dtype, &lhs.view(), &rhs.view(), &out.view(), epilogue)
    }

    /// One integer-quantized matmul operand: codes [.., rows, K * bits / 8] and its scales (`None` for an absent level).
    pub struct QuantizedTensor<'a> {
        pub scheme: &'a QuantScheme,
        pub values: &'a TensorHandle,
        pub block_scales: Option<&'a TensorHandle>,
        pub tensor_scale: Option<&'a TensorHandle>,
    }

    /// `matmul::launch_quantized(client, lhs, rhs, out)`: lhs [.., M, K] and rhs [.., N, K] quantized along K (K elements:
    /// `k`), equal leading dims flattened into one batch; out [.., M, N] contiguous F32 / BF16 / F16.
    ///
    /// # Safety
    /// As [`launch`].
    pub unsafe fn launch_quantized(
        ctx: &mut Context, stream: b200_stream, lhs: &QuantizedTensor, rhs: &QuantizedTensor, out: &TensorHandle, k: u64,
    ) -> Result<(), Error> {
        let (a, b, batch, m, n) = quantized_args(lhs, rhs, out)?;
        ctx.matmul_quantized(stream, &a, &b, out.dtype, out.ptr, batch, m, n, k)
    }

    /// `matmul::launch_quantized_fp8(client, lhs, rhs, out)`: as [`launch_quantized`] for E4M3 / E5M2 codes, on the fp8 tensor
    /// cores (`b200_matmul_quantized_fp8`).
    ///
    /// # Safety
    /// As [`launch`].
    pub unsafe fn launch_quantized_fp8(
        ctx: &mut Context, stream: b200_stream, lhs: &QuantizedTensor, rhs: &QuantizedTensor, out: &TensorHandle, k: u64,
    ) -> Result<(), Error> {
        let (a, b, batch, m, n) = quantized_args(lhs, rhs, out)?;
        ctx.matmul_quantized_fp8(stream, &a, &b, out.dtype, out.ptr, batch, m, n, k)
    }

    // the two operands, the batch and (M, N) of a quantized matmul into `out`
    fn quantized_args(
        lhs: &QuantizedTensor, rhs: &QuantizedTensor, out: &TensorHandle,
    ) -> Result<(QuantOperand, QuantOperand, u64, u64, u64), Error> {
        let r = out.shape.len();
        if r < 2 || lhs.values.shape.len() != r || rhs.values.shape.len() != r || lhs.values.shape[..r - 2] != rhs.values.shape[..r - 2] {
            return Err(invalid("lhs [.., M, K] and rhs [.., N, K] need the rank of out and equal leading dims".to_string()));
        }
        let (m, n) = (lhs.values.shape[r - 2], rhs.values.shape[r - 2]);
        let batch: u64 = out.shape[..r - 2].iter().product();
        let op = |q: &QuantizedTensor| QuantOperand {
            scheme: *q.scheme,
            values: q.values.ptr,
            block_scales: q.block_scales.map_or(0, |t| t.ptr),
            tensor_scale: q.tensor_scale.map_or(0, |t| t.ptr),
        };
        Ok((op(lhs), op(rhs), batch, m, n))
    }
}

pub mod reduce {
    use super::*;

    /// Shape of the result: the reduced axis removed, `[1]` for `axis == None` or a rank-1 input.
    pub fn output_shape(shape: &[u64], axis: Option<usize>) -> Result<Vec<u64>, Error> {
        match axis {
            None => Ok(vec![1]),
            Some(a) if a >= shape.len() => Err(invalid(format!("axis {} out of range for rank {}", a, shape.len()))),
            Some(a) => {
                let mut out: Vec<u64> = shape.iter().enumerate().filter(|(i, _)| *i != a).map(|(_, d)| *d).collect();
                if out.is_empty() {
                    out.push(1);
                }
                Ok(out)
            }
        }
    }

    /// U32 indices for the arg ops, F32 values otherwise.
    pub fn output_dtype(op: ReduceOp) -> DType {
        match op {
            ReduceOp::ArgMax | ReduceOp::ArgMin => DType::U32,
            _ => DType::F32,
        }
    }

    /// `reduce::launch(client, input, output, axis, op)`; `output` must be contiguous with [`output_shape`] and
    /// [`output_dtype`].  Arg ops: ties -> lowest index, the first NaN wins.
    ///
    /// # Safety
    /// As [`super::matmul::launch`].
    pub unsafe fn launch(
        ctx: &mut Context, stream: b200_stream, input: &TensorHandle, output: &TensorHandle, axis: Option<usize>,
        op: ReduceOp,
    ) -> Result<(), Error> {
        if output.dtype != output_dtype(op) {
            return Err(invalid("reduce: wrong output dtype for this op".to_string()));
        }
        if output.shape != output_shape(&input.shape, axis)? {
            return Err(invalid("reduce: wrong output shape".to_string()));
        }
        ctx.reduce(stream, op, input.dtype, &input.view(), output.ptr, axis)
    }
}

pub mod scan {
    use super::*;

    /// `scan::launch(client, input, output, axis, op, exclusive)`: cumulative sum / prod / max / min along `axis`;
    /// `output` is contiguous with the input's shape, F32 or the input's dtype.
    ///
    /// # Safety
    /// As [`super::matmul::launch`].
    pub unsafe fn launch(
        ctx: &mut Context, stream: b200_stream, input: &TensorHandle, output: &TensorHandle, axis: usize, op: ReduceOp,
        exclusive: bool,
    ) -> Result<(), Error> {
        if output.shape != input.shape {
            return Err(invalid("scan: output shape differs from the input's".to_string()));
        }
        if axis >= input.shape.len() {
            return Err(invalid(format!("axis {} out of range for rank {}", axis, input.shape.len())));
        }
        ctx.scan(stream, op, exclusive, input.dtype, output.dtype, &input.view(), output.ptr, axis)
    }
}

pub mod quant {
    use super::*;

    /// `quant::quantize(client, input, scheme, values, block_scales, tensor_scale)`: codes, block scales and tensor scale
    /// of `input` along its innermost axis (`block_scales` / `tensor_scale` are `None` for an absent level).
    ///
    /// # Safety
    /// As [`super::matmul::launch`].
    pub unsafe fn quantize(
        ctx: &mut Context, stream: b200_stream, input: &TensorHandle, scheme: &QuantScheme, values: &TensorHandle,
        block_scales: Option<&TensorHandle>, tensor_scale: Option<&TensorHandle>,
    ) -> Result<(), Error> {
        ctx.quantize(
            stream, scheme, input.dtype, &input.view(), values.ptr, block_scales.map_or(0, |t| t.ptr),
            tensor_scale.map_or(0, |t| t.ptr),
        )
    }

    /// `quant::dequantize(client, values, block_scales, tensor_scale, scheme, output)`: `output` is contiguous, F32 / F16 /
    /// BF16, with the logical shape of the quantized tensor.
    ///
    /// # Safety
    /// As [`super::matmul::launch`].
    pub unsafe fn dequantize(
        ctx: &mut Context, stream: b200_stream, values: &TensorHandle, block_scales: Option<&TensorHandle>,
        tensor_scale: Option<&TensorHandle>, scheme: &QuantScheme, output: &TensorHandle,
    ) -> Result<(), Error> {
        ctx.dequantize(
            stream, scheme, output.dtype, values.ptr, block_scales.map_or(0, |t| t.ptr), tensor_scale.map_or(0, |t| t.ptr),
            output.ptr, &output.shape,
        )
    }
}

pub mod conv {
    use super::*;

    /// [N, OH, OW, Cout] of x [N, H, W, C] and w [Cout, KH, KW, C]; PyTorch's rule
    /// OH = (H + 2 pad_h - dilation_h (KH - 1) - 1) / stride_h + 1, OW likewise.  `args` as [`Context::conv2d`].
    pub fn calculate_conv2d_output(x: &[u64], w: &[u64], args: [i32; 6]) -> Result<Vec<u64>, Error> {
        if x.len() != 4 || w.len() != 4 {
            return Err(invalid("conv2d needs rank-4 x [N, H, W, C] and w [Cout, KH, KW, C]".to_string()));
        }
        if x[3] != w[3] {
            return Err(invalid(format!("channels differ: x has {}, w has {}", x[3], w[3])));
        }
        let [sh, sw, ph, pw, dh, dw] = args.map(i64::from);
        if sh < 1 || sw < 1 || dh < 1 || dw < 1 || ph < 0 || pw < 0 {
            return Err(invalid("strides and dilations must be >= 1 and padding >= 0".to_string()));
        }
        let nh = x[1] as i64 + 2 * ph - dh * (w[1] as i64 - 1) - 1;
        let nw = x[2] as i64 + 2 * pw - dw * (w[2] as i64 - 1) - 1;
        if nh < 0 || nw < 0 {
            return Err(invalid("the dilated kernel is larger than the padded input".to_string()));
        }
        Ok(vec![x[0], (nh / sh + 1) as u64, (nw / sw + 1) as u64, w[0]])
    }

    /// `conv::launch(client, x, w, out, ...)`: NHWC 2-D convolution on the wgmma GEMM with the input loaded through TMA im2col.
    ///
    /// # Safety
    /// As [`super::matmul::launch`]; `epilogue.bias` must be 0 or an f32[Cout] device allocation.
    pub unsafe fn launch(
        ctx: &mut Context, stream: b200_stream, x: &TensorHandle, w: &TensorHandle, out: &TensorHandle, args: [i32; 6],
        epilogue: Option<&Epilogue>,
    ) -> Result<(), Error> {
        if x.dtype != w.dtype {
            return Err(invalid("x and w dtypes differ".to_string()));
        }
        let expect = calculate_conv2d_output(&x.shape, &w.shape, args)?;
        if expect != out.shape {
            return Err(invalid(format!("out shape {:?} != {:?}", out.shape, expect)));
        }
        ctx.conv2d(stream, x.dtype, out.dtype, &x.view(), &w.view(), &out.view(), args, epilogue)
    }
}
