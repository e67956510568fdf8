"""Softmax cross-entropy over the vocabulary on the GPU: per-token loss and lse, the logits gradient (in place if wanted), and
a forward that writes the gradient in the same launch.  The LM-head loss of a training step:

    loss, lse, dlogits = forward_alloc(c, logits, targets, grad=True, in_place=True)   # dlogits is logits, overwritten
    loss, lse, _ = forward_alloc(c, logits, targets)                                   # evaluation: loss only
    dlogits = backward_alloc(c, logits, targets, lse, dloss)                            # when dloss comes later

logits are [T, V] (f32 / bf16 / f16) with unit column stride and any row stride, targets a compact i32 or i64 [T].  The
contract (operation order, batch invariance, ignore_index, label smoothing, z-loss, refusals) is b200_cross_entropy's in
include/cubecl_b200.h; kernels in csrc/cross_entropy.cu.  Nothing synchronises with the host, and errors are deferred to
client.sync() like every launch.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _ffi
from ._ffi import B200Error
from .client import DTYPES, ComputeClient, TensorHandle

REDUCTIONS = {"none": _ffi.XENT_NONE, "sum": _ffi.XENT_SUM, "mean": _ffi.XENT_MEAN}


def _p(t: TensorHandle | None) -> C.c_uint64:
    return C.c_uint64(t.handle.ptr if t is not None else 0)


def _rows(t: TensorHandle, what: str, name: str, shape=None) -> None:
    if len(t.shape) != 2 or (t.shape[1] > 1 and t.strides[1] != 1):
        raise B200Error(6, f"{what}: {name} must be a 2-D tensor with unit column stride, got shape {t.shape} strides {t.strides}")
    if shape is not None and list(t.shape) != list(shape):
        raise B200Error(6, f"{what}: {name} must be {list(shape)}, got {list(t.shape)}")


def _vector(t: TensorHandle | None, what: str, name: str, n: int, dtypes=("f32",)) -> None:
    if t is not None and (list(t.shape) != [n] or not t.is_contiguous() or t.dtype not in dtypes):
        raise B200Error(6, f"{what}: {name} must be a compact {'/'.join(dtypes)} [{n}] tensor, got {t.dtype} {list(t.shape)}")


def _args(what: str, reduction: str, ignore_index: int, label_smoothing: float, z_loss: float):
    if reduction not in REDUCTIONS:
        raise B200Error(6, f"{what}: unknown reduction {reduction!r} (none, sum, mean)")
    return _ffi.XentArgs(REDUCTIONS[reduction], int(ignore_index), float(label_smoothing), float(z_loss))


def _check(what, logits, targets, reduction):
    _rows(logits, what, "logits")
    T, V = logits.shape
    _vector(targets, what, "targets", T, ("i32", "i64"))
    return T, V, (T if reduction == "none" else 1)


def forward(client: ComputeClient, logits: TensorHandle, targets: TensorHandle, loss: TensorHandle,
            lse: TensorHandle | None = None, reduction: str = "mean", ignore_index: int = -100, label_smoothing: float = 0.0,
            z_loss: float = 0.0, dloss: TensorHandle | None = None, dlogits: TensorHandle | None = None, stream=None) -> None:
    """loss (f32 [T] for "none", [1] for "sum" / "mean") and lse (f32 [T], optional) of torch's F.cross_entropy, plus
    z_loss * lse^2 per counted row.  With dloss (f32, loss's shape) and dlogits ([T, V], f32 / bf16 / f16, may be logits
    itself), the gradient is written in the same launch, bit for bit what backward() would write."""
    what = "cross_entropy"
    try:
        T, V, nl = _check(what, logits, targets, reduction)
        _vector(loss, what, "loss", nl)
        _vector(lse, what, "lse", T)
        _vector(dloss, what, "dloss", nl)
        if dlogits is not None:
            _rows(dlogits, what, "dlogits", [T, V])
        args = _args(what, reduction, ignore_index, label_smoothing, z_loss)
        for th in (logits, targets, loss, lse, dloss, dlogits):
            if th is not None:
                th.handle.used_on(stream)
        gdt = DTYPES[dlogits.dtype] if dlogits is not None else DTYPES[logits.dtype]
        _ffi.check(client._lib.b200_cross_entropy(client._ctx, stream, C.byref(args), DTYPES[logits.dtype], DTYPES[targets.dtype],
                                                  T, V, _p(logits), logits.strides[0], _p(targets), _p(loss), _p(lse), _p(dloss),
                                                  gdt, _p(dlogits), dlogits.strides[0] if dlogits is not None else V))
    except B200Error as e:
        client._defer(e)


def _dloss(client, reduction, T, dloss):
    """dloss as a device f32 tensor; a number (1.0 by default) becomes one [1] ([T] for "none") tensor of it"""
    if isinstance(dloss, TensorHandle):
        return dloss
    n = T if reduction == "none" else 1
    return TensorHandle.from_numpy(client, np.full(n, 1.0 if dloss is None else dloss, np.float32), "f32")


def _dlogits(client, logits, in_place, grad_dtype):
    if in_place:
        return logits
    return TensorHandle.empty_contiguous(client, list(logits.shape), grad_dtype or logits.dtype)


def forward_alloc(client: ComputeClient, logits: TensorHandle, targets: TensorHandle, reduction: str = "mean",
                  ignore_index: int = -100, label_smoothing: float = 0.0, z_loss: float = 0.0, want_lse: bool = True,
                  grad: bool = False, dloss=None, in_place: bool = False, grad_dtype: str | None = None):
    """(loss, lse, dlogits): lse None without want_lse; dlogits None without grad.  With grad, dloss is a device tensor or a
    number (default 1.0), and dlogits is logits itself when in_place (else a new [T, V] tensor in grad_dtype, default
    logits' dtype)."""
    T = logits.shape[0] if logits.shape else 0
    loss = TensorHandle.empty_contiguous(client, [T if reduction == "none" else 1], "f32")
    lse = TensorHandle.empty_contiguous(client, [T], "f32") if want_lse else None
    dl = _dloss(client, reduction, T, dloss) if grad else None
    dlogits = _dlogits(client, logits, in_place, grad_dtype) if grad else None
    forward(client, logits, targets, loss, lse, reduction, ignore_index, label_smoothing, z_loss, dl, dlogits)
    return loss, lse, dlogits


def backward(client: ComputeClient, logits: TensorHandle, targets: TensorHandle, lse: TensorHandle, dloss: TensorHandle,
             dlogits: TensorHandle, reduction: str = "mean", ignore_index: int = -100, label_smoothing: float = 0.0,
             z_loss: float = 0.0, stream=None) -> None:
    """dlogits ([T, V], f32 / bf16 / f16, may be logits itself) from the forward's lse and dloss (f32 [T] for "none", [1]
    otherwise); the arguments must be the forward's."""
    what = "cross_entropy_backward"
    try:
        T, V, nl = _check(what, logits, targets, reduction)
        _vector(lse, what, "lse", T)
        _vector(dloss, what, "dloss", nl)
        _rows(dlogits, what, "dlogits", [T, V])
        args = _args(what, reduction, ignore_index, label_smoothing, z_loss)
        for th in (logits, targets, lse, dloss, dlogits):
            th.handle.used_on(stream)
        _ffi.check(client._lib.b200_cross_entropy_backward(
            client._ctx, stream, C.byref(args), DTYPES[logits.dtype], DTYPES[targets.dtype], DTYPES[dlogits.dtype], T, V,
            _p(logits), logits.strides[0], _p(targets), _p(lse), _p(dloss), _p(dlogits), dlogits.strides[0]))
    except B200Error as e:
        client._defer(e)


def backward_alloc(client: ComputeClient, logits: TensorHandle, targets: TensorHandle, lse: TensorHandle, dloss=None,
                   reduction: str = "mean", ignore_index: int = -100, label_smoothing: float = 0.0, z_loss: float = 0.0,
                   in_place: bool = False, grad_dtype: str | None = None) -> TensorHandle:
    """dlogits: logits itself when in_place, else a new [T, V] tensor in grad_dtype (default logits' dtype); dloss a device
    tensor or a number (default 1.0)."""
    T = logits.shape[0] if logits.shape else 0
    dlogits = _dlogits(client, logits, in_place, grad_dtype)
    backward(client, logits, targets, lse, _dloss(client, reduction, T, dloss), dlogits, reduction, ignore_index,
             label_smoothing, z_loss)
    return dlogits
