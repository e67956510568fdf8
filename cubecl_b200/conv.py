"""2-D convolution surface (cubek's convolution kernels are out of tree), in the std-lib op convention
`op::launch(client, &TensorHandle...)` (crates/cubecl-std/src/tensor/identity.rs:39-83).

out[n, oh, ow, co] = act(alpha * sum_{ky, kx, c} x[n, oh*sh - ph + ky*dh, ow*sw - pw + kx*dw, c] * w[co, ky, kx, c] + bias[co])

x is NHWC [N, H, W, C], w is [Cout, KH, KW, C], out is NHWC [N, OH, OW, Cout]; input outside x reads as zero, f32
accumulation.  The kernel behind it is the wgmma GEMM of csrc/gemm_wgmma.cu with its A tile loaded through a TMA im2col
map (an implicit GEMM: M = N * OH * OW output pixels, N = Cout, K = KH * KW * C), see include/cubecl_b200.h (b200_conv2d).

The gradients (b200_conv2d_backward_data / _weight) run on the same GEMM kernel:
  dx = backward_data(dy, w):    stride 1: a convolution of dy with the flipped, channel-transposed weights; stride > 1: one such
                                convolution per output phase (h % sh, w % sw), each storing its pixels straight into dx.
  dw = backward_weight(x, dy):  M = Cout, N = KH * KW * C, K = N * OH * OW pixels, with x read through im2col loads.
The bias gradient is reduce.launch(client, "sum", dy viewed as [N * OH * OW, Cout], axis=0): no separate entry point.

Grouped and depthwise convolution (groups > 1, b200_conv2d_grouped*): w and dw are [Cout, KH, KW, C / groups], group g maps
input channels [g C/groups, (g+1) C/groups) to output channels [g Cout/groups, (g+1) Cout/groups).  Groups of >= 64 channels
run one GEMM per group on channel slices; narrower groups run direct CUDA-core kernels.  groups=1 calls the plain entry points.
"""
from __future__ import annotations

import ctypes as C

from . import _ffi
from ._ffi import B200Error
from .client import ComputeClient, DTYPES, TensorHandle
from .matmul import ACTIVATIONS


class ConvShapeError(ValueError):
    """The output-shape rule does not hold: channel mismatch, rank, or an output extent < 1."""


def _pair(v, what: str, n: int = 2) -> tuple[int, ...]:
    """v as n ints: an int repeats, a sequence must have n entries."""
    if isinstance(v, int):
        return (int(v),) * n
    v = tuple(int(e) for e in v)
    if len(v) != n:
        raise ValueError(f"{what} must be an int or {'a pair' if n == 2 else f'{n} ints'}, got {v!r}")
    return v


def calculate_conv2d_output(x_shape, w_shape, stride=1, padding=0, dilation=1, groups: int = 1) -> list[int]:
    """[N, OH, OW, Cout] of an NHWC input [N, H, W, C] and weights [Cout, KH, KW, C / groups]; PyTorch's rule:
    OH = floor((H + 2*ph - dh*(KH-1) - 1) / sh) + 1, OW likewise."""
    x_shape, w_shape = [int(s) for s in x_shape], [int(s) for s in w_shape]
    if len(x_shape) != 4 or len(w_shape) != 4:
        raise ConvShapeError(f"conv2d needs rank-4 x [N,H,W,C] and w [Cout,KH,KW,C], got {x_shape} and {w_shape}")
    (sh, sw), (ph, pw), (dh, dw) = _pair(stride, "stride"), _pair(padding, "padding"), _pair(dilation, "dilation")
    n, h, w, c = x_shape
    cout, kh, kw, c2 = w_shape
    if groups < 1 or c % groups or cout % groups:
        raise ConvShapeError(f"groups = {groups} must be >= 1 and divide C = {c} and Cout = {cout}")
    if c // groups != c2:
        raise ConvShapeError(f"channels differ: x has {c} in {groups} group(s), w has {c2} per group")
    if sh < 1 or sw < 1 or dh < 1 or dw < 1 or ph < 0 or pw < 0:
        raise ConvShapeError("strides and dilations must be >= 1 and padding >= 0")
    nh, nw = h + 2 * ph - dh * (kh - 1) - 1, w + 2 * pw - dw * (kw - 1) - 1
    if nh < 0 or nw < 0:
        raise ConvShapeError(f"the dilated kernel {kh}x{kw} is larger than the padded input {h}x{w}")
    return [n, nh // sh + 1, nw // sw + 1, cout]


def launch(client: ComputeClient, x: TensorHandle, w: TensorHandle, out: TensorHandle, stride=1, padding=0, dilation=1,
           alpha: float = 1.0, bias: TensorHandle | None = None, activation: str | None = None, stream=None, groups: int = 1) -> None:
    """Enqueue the convolution on the client's stream.  stride / padding / dilation are ints or (h, w) pairs.  Optional fused
    epilogue: out = activation(alpha * conv + bias[co]) with `bias` an f32 [Cout] tensor.  groups > 1: a grouped convolution
    with w [Cout, KH, KW, C / groups].  Never raises for launch problems: errors are deferred to client.sync() / read_one()
    like matmul.launch."""
    _enqueue(client, "conv2d", x, w, out, stride, padding, dilation, stream, groups, _epilogue_check("conv2d", w, alpha, bias, activation))


def _epilogue_check(what: str, w: TensorHandle, alpha: float, bias: TensorHandle | None, activation: str | None,
                    cout: int | None = None):
    """launch's epilogue callback for _enqueue: checks the epilogue arguments, returns (b200_epilogue pointer or None,
    the extra handles it reads).  cout: the output channels (default w.shape[0])."""
    def epilogue():
        if activation not in ACTIVATIONS:
            raise B200Error(6, f"unknown activation {activation!r}")
        if bias is not None and (bias.dtype != "f32" or not bias.is_contiguous() or bias.size() != (w.shape[0] if cout is None else cout)):
            raise B200Error(6, f"{what}: bias must be a contiguous f32 tensor with Cout elements")
        if alpha == 1.0 and bias is None and activation in (None, "none"):
            return None, ()
        ep = _ffi.Epilogue(float(alpha), ACTIVATIONS[activation], bias.handle.ptr if bias is not None else 0)
        return C.byref(ep), (() if bias is None else (bias,))
    return epilogue


def launch_alloc(client: ComputeClient, x: TensorHandle, w: TensorHandle, out_dtype: str | None = None, **kwargs) -> TensorHandle:
    """Convenience: allocate a compact NHWC `out` with the output rule, then launch (keyword arguments as launch)."""
    shape = calculate_conv2d_output(x.shape, w.shape, kwargs.get("stride", 1), kwargs.get("padding", 0), kwargs.get("dilation", 1),
                                    kwargs.get("groups", 1))
    out = TensorHandle.empty_contiguous(client, shape, out_dtype or x.dtype)
    launch(client, x, w, out, **kwargs)
    return out


def _groups(groups) -> C.c_uint32:
    groups = int(groups)
    if not 0 <= groups < 2 ** 32:
        raise B200Error(6, f"conv2d: groups = {groups} out of range")
    return C.c_uint32(groups)


def _enqueue(client: ComputeClient, name: str, a: TensorHandle, b: TensorHandle, out: TensorHandle, stride, padding, dilation, stream,
             groups, epilogue=None, spatial: int = 2) -> None:
    """The body of launch, backward_data and backward_weight (and of conv3d's, spatial = 3): check the operands, mark them
    used on `stream` and call b200_<name>(a, b, out, args[, epilogue]), or its grouped form when groups != 1.  epilogue
    (launch only) checks the epilogue arguments and returns (the b200_epilogue pointer or None, the extra handles it reads).
    Errors are deferred to client.sync() / read_one()."""
    try:
        rank = spatial + 2
        if len(a.shape) != rank or len(b.shape) != rank or len(out.shape) != rank:
            raise B200Error(6, f"{name}: every operand must have rank {rank}")
        if a.dtype != b.dtype:
            raise B200Error(6, f"{name}: operand dtypes differ ({a.dtype}, {b.dtype})")
        ep, extra = epilogue() if epilogue else (None, ())
        s, p, d = _pair(stride, "stride", spatial), _pair(padding, "padding", spatial), _pair(dilation, "dilation", spatial)
        for t in (a, b, out, *extra):
            t.handle.used_on(stream)
        args = _ffi.Conv2dArgs(*s, *p, *d) if spatial == 2 else _ffi.Conv3dArgs(*s, *p, *d)
        operands = (client._ctx, stream, DTYPES[a.dtype], DTYPES[out.dtype],
                    C.c_uint64(a.handle.ptr), _ffi.u64_array(a.shape), _ffi.u64_array(a.strides),
                    C.c_uint64(b.handle.ptr), _ffi.u64_array(b.shape), _ffi.u64_array(b.strides),
                    C.c_uint64(out.handle.ptr), _ffi.u64_array(out.shape), _ffi.u64_array(out.strides), C.byref(args))
        tail = (ep,) if epilogue else ()
        if groups == 1:
            _ffi.check(getattr(client._lib, "b200_" + name)(*operands, *tail))
        else:
            _ffi.check(getattr(client._lib, "b200_" + name.replace("conv2d", "conv2d_grouped", 1))(*operands, _groups(groups), *tail))
    except (B200Error, ValueError) as e:
        client._defer(e if isinstance(e, B200Error) else B200Error(6, str(e)))


def backward_data(client: ComputeClient, dy: TensorHandle, w: TensorHandle, dx: TensorHandle, stride=1, padding=0, dilation=1,
                  stream=None, groups: int = 1) -> None:
    """Enqueue dx = the gradient of conv2d with respect to its input: dy [N, OH, OW, Cout], w [Cout, KH, KW, C / groups], dx
    [N, H, W, C] (NHWC), with dy's shape the output rule of (dx, w).  Errors are deferred like launch."""
    _enqueue(client, "conv2d_backward_data", dy, w, dx, stride, padding, dilation, stream, groups)


def backward_data_alloc(client: ComputeClient, dy: TensorHandle, w: TensorHandle, input_hw, out_dtype: str | None = None,
                        **kwargs) -> TensorHandle:
    """Convenience: allocate a compact NHWC dx [N, H, W, C] with (H, W) = input_hw (the forward input's extents; a stride > 1
    convolution maps several H to one OH) and C = groups * w.shape[3], then backward_data (keyword arguments as
    backward_data)."""
    h, wd = _pair(input_hw, "input_hw")
    dx = TensorHandle.empty_contiguous(client, [dy.shape[0], h, wd, w.shape[3] * int(kwargs.get("groups", 1))], out_dtype or dy.dtype)
    backward_data(client, dy, w, dx, **kwargs)
    return dx


def backward_weight(client: ComputeClient, x: TensorHandle, dy: TensorHandle, dw: TensorHandle, stride=1, padding=0, dilation=1,
                    stream=None, groups: int = 1) -> None:
    """Enqueue dw = the gradient of conv2d with respect to its weights: x [N, H, W, C], dy [N, OH, OW, Cout], dw
    [Cout, KH, KW, C / groups], with dy's shape the output rule of (x, dw).  Errors are deferred like launch."""
    _enqueue(client, "conv2d_backward_weight", x, dy, dw, stride, padding, dilation, stream, groups)


def backward_weight_alloc(client: ComputeClient, x: TensorHandle, dy: TensorHandle, kernel_hw, out_dtype: str | None = None,
                          **kwargs) -> TensorHandle:
    """Convenience: allocate a compact dw [Cout, KH, KW, C / groups] with (KH, KW) = kernel_hw, then backward_weight (keyword
    arguments as backward_weight)."""
    kh, kw = _pair(kernel_hw, "kernel_hw")
    groups = int(kwargs.get("groups", 1))
    if groups < 1 or x.shape[3] % groups:
        raise ValueError(f"groups = {groups} must be >= 1 and divide C = {x.shape[3]}")
    dw = TensorHandle.empty_contiguous(client, [dy.shape[3], kh, kw, x.shape[3] // groups], out_dtype or x.dtype)
    backward_weight(client, x, dy, dw, **kwargs)
    return dw
