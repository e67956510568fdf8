"""RMSNorm and LayerNorm over the innermost axis on the GPU, with a fused residual add, an fp8 block-quantized output for
b200_matmul_quantized_fp8, and the backward.  A pre-norm block:

    h, y, _, rstd = forward_alloc(c, x, weight, residual=r)        # h = x + r (rounded), y = rms_norm(h) * weight
    q, h, _, rstd = forward_quantized_alloc(c, x, scheme, weight)  # y as fp8 codes + block scales (quant.QuantizedTensor)
    dx, dw, _ = backward_alloc(c, dy, h, rstd, weight, d_h=dh)     # dx: the gradient of x and of the residual

Tensors are [T, n] with unit column stride and any row stride.  The contracts (operation order, batch invariance, fp8
schemes, refusals) are those of b200_norm* in include/cubecl_b200.h; kernels in csrc/norm.cu.  Nothing synchronises with
the host, and errors are deferred to client.sync() like every launch.
"""
from __future__ import annotations

import ctypes as C

from . import _ffi
from ._ffi import B200Error
from .client import DTYPES, ComputeClient, TensorHandle
from .quant import QuantizedTensor, QuantScheme, alloc_quantized

KINDS = {"rms": _ffi.NORM_RMS, "layer": _ffi.NORM_LAYER}


def _p(t: TensorHandle | None) -> C.c_uint64:
    return C.c_uint64(t.handle.ptr if t is not None else 0)


def _rows(t: TensorHandle | None, what: str, name: str, shape=None, dtype=None) -> None:
    """None, or a 2-D tensor with unit column stride (any row stride) of the given shape and dtype."""
    if t is None:
        return
    if len(t.shape) != 2 or (t.shape[1] > 1 and t.strides[1] != 1):
        raise B200Error(6, f"{what}: {name} must be a 2-D tensor with unit column stride, got shape {t.shape} strides {t.strides}")
    if shape is not None and list(t.shape) != list(shape):
        raise B200Error(6, f"{what}: {name} must be {list(shape)}, got {list(t.shape)}")
    if dtype is not None and t.dtype != dtype:
        raise B200Error(6, f"{what}: {name} must be {dtype}, got {t.dtype}")


def _vector(t: TensorHandle | None, what: str, name: str, n: int, dtype=None) -> None:
    if t is not None and (list(t.shape) != [n] or not t.is_contiguous() or (dtype is not None and t.dtype != dtype)):
        raise B200Error(6, f"{what}: {name} must be a compact {dtype or ''} [{n}] tensor, got {t.dtype} {list(t.shape)}")


def _args(kind: str, x_dtype: str, weight: TensorHandle | None, bias: TensorHandle | None, eps: float, what: str):
    if kind not in KINDS:
        raise B200Error(6, f"{what}: unknown kind {kind!r} (rms, layer)")
    if x_dtype not in DTYPES:
        raise B200Error(6, f"{what}: unknown dtype {x_dtype!r}")
    wdt = weight.dtype if weight is not None else bias.dtype if bias is not None else x_dtype
    if bias is not None and weight is not None and bias.dtype != weight.dtype:
        raise B200Error(6, f"{what}: weight and bias must share a dtype")
    return _ffi.NormArgs(KINDS[kind], DTYPES[x_dtype], DTYPES[wdt], float(eps))


def _stride(t: TensorHandle | None, n: int) -> int:
    return t.strides[0] if t is not None else n


def _forward_check(what, x, residual, h_out, weight, bias, mean, rstd, kind, eps):
    _rows(x, what, "x")
    T, n = x.shape
    _rows(residual, what, "residual", [T, n], x.dtype)
    _rows(h_out, what, "h_out", [T, n], x.dtype)
    _vector(weight, what, "weight", n)
    _vector(bias, what, "bias", n)
    _vector(mean, what, "mean", T, "f32")
    _vector(rstd, what, "rstd", T, "f32")
    return T, n, _args(kind, x.dtype, weight, bias, eps, what)


def forward(client: ComputeClient, x: TensorHandle, y: TensorHandle, weight: TensorHandle | None = None,
            bias: TensorHandle | None = None, kind: str = "rms", eps: float = 1e-6, residual: TensorHandle | None = None,
            h_out: TensorHandle | None = None, mean: TensorHandle | None = None, rstd: TensorHandle | None = None,
            stream=None) -> None:
    """y = norm(h) * weight (+ bias) over the last axis, h = x or, with a residual, h = x + residual rounded to x's dtype and
    written to h_out.  kind "rms" or "layer"; x f32 / bf16 / f16, weight and bias f32 or x's dtype, y f32 / bf16 / f16;
    mean (layer) and rstd optional f32 [T] outputs."""
    what = "norm"
    try:
        T, n, args = _forward_check(what, x, residual, h_out, weight, bias, mean, rstd, kind, eps)
        _rows(y, what, "y", [T, n])
        for th in (x, y, residual, h_out, weight, bias, mean, rstd):
            if th is not None:
                th.handle.used_on(stream)
        _ffi.check(client._lib.b200_norm(client._ctx, stream, C.byref(args), DTYPES[y.dtype], T, n, _p(x), x.strides[0],
                                         _p(residual), _stride(residual, n), _p(h_out), _stride(h_out, n), _p(weight), _p(bias),
                                         _p(y), y.strides[0], _p(mean), _p(rstd)))
    except B200Error as e:
        client._defer(e)


def _stats_alloc(client, x, kind, residual, want_mean, want_rstd):
    T = x.shape[0] if x.shape else 0
    h_out = TensorHandle.empty_contiguous(client, list(x.shape), x.dtype) if residual is not None else None
    mean = TensorHandle.empty_contiguous(client, [T], "f32") if want_mean and kind == "layer" else None
    rstd = TensorHandle.empty_contiguous(client, [T], "f32") if want_rstd else None
    return h_out, mean, rstd


def forward_alloc(client: ComputeClient, x: TensorHandle, weight: TensorHandle | None = None, bias: TensorHandle | None = None,
                  kind: str = "rms", eps: float = 1e-6, residual: TensorHandle | None = None, out_dtype: str | None = None,
                  stats: bool = True):
    """(h, y, mean, rstd): h is x without a residual; mean is None for rms, mean and rstd None without stats."""
    h_out, mean, rstd = _stats_alloc(client, x, kind, residual, stats, stats)
    y = TensorHandle.empty_contiguous(client, list(x.shape), out_dtype or x.dtype)
    forward(client, x, y, weight, bias, kind, eps, residual, h_out, mean, rstd)
    return (h_out if residual is not None else x), y, mean, rstd


def forward_quantized(client: ComputeClient, x: TensorHandle, q: QuantizedTensor, weight: TensorHandle | None = None,
                      bias: TensorHandle | None = None, kind: str = "rms", eps: float = 1e-6, residual: TensorHandle | None = None,
                      h_out: TensorHandle | None = None, mean: TensorHandle | None = None, rstd: TensorHandle | None = None,
                      stream=None) -> None:
    """forward() with y stored into q (quant.alloc_quantized([T, n], scheme)) exactly as quant.quantize(y_f32, scheme) would:
    e4m3 / e5m2 values, blocks of 32, 64 or 128, f32 or ue8m0 block scales, no tensor level."""
    what = "norm_quantized_fp8"
    try:
        T, n, args = _forward_check(what, x, residual, h_out, weight, bias, mean, rstd, kind, eps)
        if list(q.shape) != [T, n] or q.block_scales is None:
            raise B200Error(6, f"{what}: q must hold a block-scaled [{T}, {n}] tensor, got {q.shape}")
        s = q.scheme.to_c()
        for th in (x, q.values, q.block_scales, residual, h_out, weight, bias, mean, rstd):
            if th is not None:
                th.handle.used_on(stream)
        _ffi.check(client._lib.b200_norm_quantized_fp8(client._ctx, stream, C.byref(args), C.byref(s), T, n, _p(x), x.strides[0],
                                                       _p(residual), _stride(residual, n), _p(h_out), _stride(h_out, n),
                                                       _p(weight), _p(bias), _p(q.values), _p(q.block_scales), _p(mean), _p(rstd)))
    except B200Error as e:
        client._defer(e)


def forward_quantized_alloc(client: ComputeClient, x: TensorHandle, scheme: QuantScheme, weight: TensorHandle | None = None,
                            bias: TensorHandle | None = None, kind: str = "rms", eps: float = 1e-6,
                            residual: TensorHandle | None = None, stats: bool = True):
    """(q, h, mean, rstd) as forward_alloc, with y as the QuantizedTensor q."""
    h_out, mean, rstd = _stats_alloc(client, x, kind, residual, stats, stats)
    q = alloc_quantized(client, list(x.shape), scheme)
    forward_quantized(client, x, q, weight, bias, kind, eps, residual, h_out, mean, rstd)
    return q, (h_out if residual is not None else x), mean, rstd


def backward(client: ComputeClient, dy: TensorHandle, h: TensorHandle, rstd: TensorHandle, dx: TensorHandle,
             weight: TensorHandle | None = None, mean: TensorHandle | None = None, kind: str = "rms",
             d_h: TensorHandle | None = None, dweight: TensorHandle | None = None, dbias: TensorHandle | None = None,
             stream=None) -> None:
    """dx = the gradient of h (plus d_h, the gradient already on the residual stream), dweight and dbias (f32 [n], optional)
    from dy, the forward's input h, weight, and its rstd (and mean for layer).  dy, d_h and dx share a dtype."""
    what = "norm_backward"
    try:
        _rows(h, what, "h")
        T, n = h.shape
        _rows(dy, what, "dy", [T, n])
        _rows(d_h, what, "d_h", [T, n], dy.dtype)
        _rows(dx, what, "dx", [T, n], dy.dtype)
        _vector(weight, what, "weight", n)
        _vector(mean, what, "mean", T, "f32")
        _vector(rstd, what, "rstd", T, "f32")
        _vector(dweight, what, "dweight", n, "f32")
        _vector(dbias, what, "dbias", n, "f32")
        args = _args(kind, h.dtype, weight, None, 0.0, what)
        for th in (dy, h, rstd, dx, weight, mean, d_h, dweight, dbias):
            if th is not None:
                th.handle.used_on(stream)
        _ffi.check(client._lib.b200_norm_backward(client._ctx, stream, C.byref(args), DTYPES[dy.dtype], T, n, _p(dy), dy.strides[0],
                                                  _p(h), h.strides[0], _p(weight), _p(mean), _p(rstd), _p(d_h), _stride(d_h, n),
                                                  _p(dx), dx.strides[0], _p(dweight), _p(dbias)))
    except B200Error as e:
        client._defer(e)


def backward_alloc(client: ComputeClient, dy: TensorHandle, h: TensorHandle, rstd: TensorHandle,
                   weight: TensorHandle | None = None, mean: TensorHandle | None = None, kind: str = "rms",
                   d_h: TensorHandle | None = None, bias: bool = False):
    """(dx, dweight, dbias): dweight None without a weight, dbias only when `bias` (layer)."""
    n = h.shape[1] if len(h.shape) == 2 else 0
    dx = TensorHandle.empty_contiguous(client, list(h.shape), dy.dtype)
    dweight = TensorHandle.empty_contiguous(client, [n], "f32") if weight is not None else None
    dbias = TensorHandle.empty_contiguous(client, [n], "f32") if bias else None
    backward(client, dy, h, rstd, dx, weight, mean, kind, d_h, dweight, dbias)
    return dx, dweight, dbias
