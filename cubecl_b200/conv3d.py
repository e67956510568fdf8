"""3-D convolution surface, forward and both gradients, with the names of conv.py.

out[n, od, oh, ow, co] = act(alpha * sum_{kz, ky, kx, c} x[n, od*sd - pd + kz*dd, oh*sh - ph + ky*dh, ow*sw - pw + kx*dw, c]
                             * w[co, kz, ky, kx, c] + bias[co])

x is NDHWC [N, D, H, W, C], w is [Cout, KD, KH, KW, C] (PyTorch's OIDHW weight permuted), out and dy are NDHWC
[N, OD, OH, OW, Cout]; input outside x reads as zero, f32 accumulation.  The kernels are the wgmma GEMM's with the input
loaded through a 5-D TMA im2col map, see include/cubecl_b200.h (b200_conv3d).  The bias gradient is
reduce.launch(client, "sum", dy viewed as [N * OD * OH * OW, Cout], axis=0).  There is no groups argument.
"""
from __future__ import annotations

from .client import ComputeClient, TensorHandle
from .conv import ConvShapeError, _enqueue, _epilogue_check, _pair


def calculate_conv3d_output(x_shape, w_shape, stride=1, padding=0, dilation=1) -> list[int]:
    """[N, OD, OH, OW, Cout] of an NDHWC input [N, D, H, W, C] and weights [Cout, KD, KH, KW, C]; PyTorch's rule in each
    dimension: O = floor((I + 2*p - d*(K-1) - 1) / s) + 1."""
    x_shape, w_shape = [int(s) for s in x_shape], [int(s) for s in w_shape]
    if len(x_shape) != 5 or len(w_shape) != 5:
        raise ConvShapeError(f"conv3d needs rank-5 x [N,D,H,W,C] and w [Cout,KD,KH,KW,C], got {x_shape} and {w_shape}")
    s, p, d = _pair(stride, "stride", 3), _pair(padding, "padding", 3), _pair(dilation, "dilation", 3)
    if x_shape[4] != w_shape[4]:
        raise ConvShapeError(f"channels differ: x has {x_shape[4]}, w has {w_shape[4]}")
    if min(s) < 1 or min(d) < 1 or min(p) < 0:
        raise ConvShapeError("strides and dilations must be >= 1 and padding >= 0")
    out = [x_shape[0]]
    for i in range(3):
        n = x_shape[1 + i] + 2 * p[i] - d[i] * (w_shape[1 + i] - 1) - 1
        if n < 0:
            raise ConvShapeError(f"the dilated kernel {w_shape[1:4]} is larger than the padded input {x_shape[1:4]}")
        out.append(n // s[i] + 1)
    return out + [w_shape[0]]


def launch(client: ComputeClient, x: TensorHandle, w: TensorHandle, out: TensorHandle, stride=1, padding=0, dilation=1,
           alpha: float = 1.0, bias: TensorHandle | None = None, activation: str | None = None, stream=None) -> None:
    """Enqueue the 3-D convolution on the client's stream.  stride / padding / dilation are ints or (d, h, w) triples.
    Optional fused epilogue: out = activation(alpha * conv + bias[co]) with `bias` an f32 [Cout] tensor.  Errors are deferred
    to client.sync() / read_one() like conv.launch."""
    _enqueue(client, "conv3d", x, w, out, stride, padding, dilation, stream, 1, _epilogue_check("conv3d", w, alpha, bias, activation),
             spatial=3)


def launch_alloc(client: ComputeClient, x: TensorHandle, w: TensorHandle, out_dtype: str | None = None, **kwargs) -> TensorHandle:
    """Convenience: allocate a compact NDHWC `out` with the output rule, then launch (keyword arguments as launch)."""
    shape = calculate_conv3d_output(x.shape, w.shape, kwargs.get("stride", 1), kwargs.get("padding", 0), kwargs.get("dilation", 1))
    out = TensorHandle.empty_contiguous(client, shape, out_dtype or x.dtype)
    launch(client, x, w, out, **kwargs)
    return out


def backward_data(client: ComputeClient, dy: TensorHandle, w: TensorHandle, dx: TensorHandle, stride=1, padding=0, dilation=1,
                  stream=None) -> None:
    """Enqueue dx = the gradient of conv3d with respect to its input: dy [N, OD, OH, OW, Cout], w [Cout, KD, KH, KW, C], dx
    [N, D, H, W, C], with dy's shape the output rule of (dx, w).  Errors are deferred like launch."""
    _enqueue(client, "conv3d_backward_data", dy, w, dx, stride, padding, dilation, stream, 1, spatial=3)


def backward_data_alloc(client: ComputeClient, dy: TensorHandle, w: TensorHandle, input_dhw, out_dtype: str | None = None,
                        **kwargs) -> TensorHandle:
    """Convenience: allocate a compact NDHWC dx [N, D, H, W, C] with (D, H, W) = input_dhw (the forward input's extents),
    then backward_data (keyword arguments as backward_data)."""
    d, h, wd = _pair(input_dhw, "input_dhw", 3)
    dx = TensorHandle.empty_contiguous(client, [dy.shape[0], d, h, wd, w.shape[4]], out_dtype or dy.dtype)
    backward_data(client, dy, w, dx, **kwargs)
    return dx


def backward_weight(client: ComputeClient, x: TensorHandle, dy: TensorHandle, dw: TensorHandle, stride=1, padding=0, dilation=1,
                    stream=None) -> None:
    """Enqueue dw = the gradient of conv3d with respect to its weights: x [N, D, H, W, C], dy [N, OD, OH, OW, Cout], dw
    [Cout, KD, KH, KW, C], with dy's shape the output rule of (x, dw).  Errors are deferred like launch."""
    _enqueue(client, "conv3d_backward_weight", x, dy, dw, stride, padding, dilation, stream, 1, spatial=3)


def backward_weight_alloc(client: ComputeClient, x: TensorHandle, dy: TensorHandle, kernel_dhw, out_dtype: str | None = None,
                          **kwargs) -> TensorHandle:
    """Convenience: allocate a compact dw [Cout, KD, KH, KW, C] with (KD, KH, KW) = kernel_dhw, then backward_weight (keyword
    arguments as backward_weight)."""
    kd, kh, kw = _pair(kernel_dhw, "kernel_dhw", 3)
    dw = TensorHandle.empty_contiguous(client, [dy.shape[4], kd, kh, kw, x.shape[4]], out_dtype or x.dtype)
    backward_weight(client, x, dy, dw, **kwargs)
    return dw
