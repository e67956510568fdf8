"""Transposed convolution, 2-D and 3-D (PyTorch's ConvTranspose2d / 3d), with the names of conv.py.

out[n, oh, ow, co] = act(alpha * sum_{ih, iw, ky, kx, ci : oh = ih*sh - ph + ky*dh, ow = iw*sw - pw + kx*dw}
                                 x[n, ih, iw, ci] * w[ci, ky, kx, co] + bias[co])

x is NHWC [N, H, W, Cin], w is [Cin, KH, KW, Cout] (PyTorch's [Cin, Cout, KH, KW] permuted), out is NHWC [N, OH, OW, Cout]
with OH = (H-1)*sh - 2*ph + dh*(KH-1) + oph + 1 (likewise OW); 3-D adds the depth dimension with NDHWC layouts.  The
output padding is implied by out's shape; 0 <= output_padding < stride.  The rank of x (4 or 5) picks 2-D or 3-D.  See
include/cubecl_b200.h (b200_conv_transpose2d): stride 1 runs the forward convolution kernel, a larger stride every output
phase of the layer in one phase-batched wgmma launch (up to 8 phases per launch).

The gradients are the existing convolution entry points with roles swapped:
  dx    = backward_data(dy, w)       = conv2d(dy, w) with the same stride / padding / dilation (w read as [Cin, KH, KW, Cout]
                                       conv weights, no flip);
  dw    = backward_weight(x, dy)     = conv2d_backward_weight(x := dy, dy := x);
  dbias = reduce.launch(client, "sum", dy viewed as [N * OH * OW, Cout], axis=0).
"""
from __future__ import annotations

from .client import ComputeClient, TensorHandle
from .conv import ConvShapeError, _enqueue, _epilogue_check, _pair


def _spatial(t_shape, what: str) -> int:
    if len(t_shape) not in (4, 5):
        raise ConvShapeError(f"{what} needs rank 4 (NHWC) or 5 (NDHWC), got rank {len(t_shape)}")
    return len(t_shape) - 2


def calculate_conv_transpose_output(x_shape, w_shape, stride=1, padding=0, output_padding=0, dilation=1) -> list[int]:
    """[N, OH, OW, Cout] (or [N, OD, OH, OW, Cout]) of an input [N, H, W, Cin] and weights [Cin, KH, KW, Cout]; PyTorch's rule
    in each dimension: O = (I - 1) * s - 2 * p + d * (K - 1) + op + 1, with 0 <= op < s."""
    x_shape, w_shape = [int(s) for s in x_shape], [int(s) for s in w_shape]
    n = _spatial(x_shape, "conv_transpose")
    if len(w_shape) != n + 2:
        raise ConvShapeError(f"conv_transpose: x {x_shape} and w {w_shape} differ in rank")
    s, p = _pair(stride, "stride", n), _pair(padding, "padding", n)
    op, d = _pair(output_padding, "output_padding", n), _pair(dilation, "dilation", n)
    if x_shape[-1] != w_shape[0]:
        raise ConvShapeError(f"channels differ: x has {x_shape[-1]}, w has {w_shape[0]}")
    if min(s) < 1 or min(d) < 1 or min(p) < 0:
        raise ConvShapeError("strides and dilations must be >= 1 and padding >= 0")
    if any(not 0 <= op[i] < s[i] for i in range(n)):
        raise ConvShapeError(f"output_padding {op} must lie in [0, stride {s})")
    out = [x_shape[0]]
    for i in range(n):
        o = (x_shape[1 + i] - 1) * s[i] - 2 * p[i] + d[i] * (w_shape[1 + i] - 1) + op[i] + 1
        if o < 1:
            raise ConvShapeError(f"output extent {o} < 1 in dimension {i}")
        out.append(o)
    return out + [w_shape[-1]]


def launch(client: ComputeClient, x: TensorHandle, w: TensorHandle, out: TensorHandle, stride=1, padding=0, dilation=1,
           alpha: float = 1.0, bias: TensorHandle | None = None, activation: str | None = None, stream=None) -> None:
    """Enqueue the transposed convolution on the client's stream; out's shape gives the output padding.  stride / padding /
    dilation are ints or per-dimension tuples.  Optional fused epilogue: out = activation(alpha * conv_transpose + bias[co])
    with `bias` an f32 [Cout] tensor.  Errors are deferred to client.sync() / read_one() like conv.launch."""
    n = len(x.shape) - 2
    name = "conv_transpose3d" if n == 3 else "conv_transpose2d"
    _enqueue(client, name, x, w, out, stride, padding, dilation, stream, 1,
             _epilogue_check(name, w, alpha, bias, activation, cout=w.shape[-1]), spatial=3 if n == 3 else 2)


def launch_alloc(client: ComputeClient, x: TensorHandle, w: TensorHandle, output_padding=0, out_dtype: str | None = None,
                 **kwargs) -> TensorHandle:
    """Convenience: allocate a compact `out` with the output rule (and output_padding), then launch (keyword arguments as
    launch)."""
    shape = calculate_conv_transpose_output(x.shape, w.shape, kwargs.get("stride", 1), kwargs.get("padding", 0), output_padding,
                                            kwargs.get("dilation", 1))
    out = TensorHandle.empty_contiguous(client, shape, out_dtype or x.dtype)
    launch(client, x, w, out, **kwargs)
    return out


def backward_data(client: ComputeClient, dy: TensorHandle, w: TensorHandle, dx: TensorHandle, stride=1, padding=0, dilation=1,
                  stream=None) -> None:
    """Enqueue dx = the gradient of the transposed convolution with respect to x: the forward convolution of dy [N, OH, OW,
    Cout] with w [Cin, KH, KW, Cout] read as conv weights (Cout := Cin), dx [N, H, W, Cin].  Errors are deferred like launch."""
    n = len(dy.shape) - 2
    name = "conv3d" if n == 3 else "conv2d"
    _enqueue(client, name, dy, w, dx, stride, padding, dilation, stream, 1, _epilogue_check(name, w, 1.0, None, None),
             spatial=3 if n == 3 else 2)


def backward_data_alloc(client: ComputeClient, dy: TensorHandle, w: TensorHandle, out_dtype: str | None = None, **kwargs) -> TensorHandle:
    """Convenience: allocate a compact dx [N, H, W, Cin] (the convolution output rule of (dy, w)), then backward_data."""
    n = _spatial(dy.shape, "conv_transpose backward_data")
    s, p, d = (_pair(kwargs.get(k, v), k, n) for k, v in (("stride", 1), ("padding", 0), ("dilation", 1)))
    shape = [dy.shape[0]]
    for i in range(n):
        e = dy.shape[1 + i] + 2 * p[i] - d[i] * (w.shape[1 + i] - 1) - 1
        if e < 0:
            raise ConvShapeError(f"the dilated kernel {list(w.shape[1:1 + n])} is larger than the padded gradient {list(dy.shape[1:1 + n])}")
        shape.append(e // s[i] + 1)
    dx = TensorHandle.empty_contiguous(client, shape + [w.shape[0]], out_dtype or dy.dtype)
    backward_data(client, dy, w, dx, **kwargs)
    return dx


def backward_weight(client: ComputeClient, x: TensorHandle, dy: TensorHandle, dw: TensorHandle, stride=1, padding=0, dilation=1,
                    stream=None) -> None:
    """Enqueue dw [Cin, KH, KW, Cout] = the gradient of the transposed convolution with respect to w: the convolution weight
    gradient with dy [N, OH, OW, Cout] as its input and x [N, H, W, Cin] as its output gradient.  Errors are deferred like
    launch."""
    n = len(x.shape) - 2
    _enqueue(client, "conv3d_backward_weight" if n == 3 else "conv2d_backward_weight", dy, x, dw, stride, padding, dilation, stream, 1,
             spatial=3 if n == 3 else 2)


def backward_weight_alloc(client: ComputeClient, x: TensorHandle, dy: TensorHandle, kernel, out_dtype: str | None = None,
                          **kwargs) -> TensorHandle:
    """Convenience: allocate a compact dw [Cin, *kernel, Cout] (kernel = (KH, KW) or (KD, KH, KW)), then backward_weight."""
    n = _spatial(x.shape, "conv_transpose backward_weight")
    dw = TensorHandle.empty_contiguous(client, [x.shape[-1], *_pair(kernel, "kernel", n), dy.shape[-1]], out_dtype or x.dtype)
    backward_weight(client, x, dy, dw, **kwargs)
    return dw
