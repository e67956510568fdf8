"""Fused scaled-dot-product attention (PyTorch's scaled_dot_product_attention), forward and backward, in the std-lib op
convention.

out[b, h, i, :] = sum_j softmax_j(scale * q[b, h, i, :] . k[b, h / G, j, :]) * v[b, h / G, j, :]      G = Hq / Hkv
lse[b, h, i]    = log sum_j exp(scale * q[b, h, i, :] . k[b, h / G, j, :])                         (natural log, f32)

q is [B, Hq, Sq, D], k and v are [B, Hkv, Sk, D], out is [B, Hq, Sq, D]: shapes and strides in elements, so [B, S, H, D]
tensors and the q / k / v slices of a fused [B, S, 3, H, D] projection arrive as stride-permuted views with no copy.
causal: key j is visible to query i only when j <= i (torch's is_causal=True, top-left aligned).  f16 or bf16 inputs, out
in the input dtype or f32, D <= 128 with D % 8 == 0.  One fused kernel (csrc/attention.cu): the score matrix never reaches
memory.  See include/cubecl_b200.h (b200_attention) for the numerics and the view rules.

The backward (launch_backward) takes the forward's out and lse with dout and writes dq [B, Hq, Sq, D] and dk, dv [B, Hkv, Sk, D]
(with GQA, dk and dv sum over the query heads of each kv head); three kernels (csrc/attention_bwd.cu), no atomics, bitwise
reproducible.  See b200_attention_backward for its numerics.
"""
from __future__ import annotations

import ctypes as C
import math

from . import _ffi
from ._ffi import B200Error
from .client import ComputeClient, DTYPES, TensorHandle


class AttentionShapeError(ValueError):
    """The shapes of q, k and v do not describe one attention problem."""


def calculate_attention_output(q_shape, k_shape, v_shape) -> list[int]:
    """[B, Hq, Sq, D] of q [B, Hq, Sq, D], k [B, Hkv, Sk, D] and v [B, Hkv, Sk, D] with Hq % Hkv == 0."""
    q, k, v = ([int(s) for s in t] for t in (q_shape, k_shape, v_shape))
    if len(q) != 4 or len(k) != 4 or len(v) != 4:
        raise AttentionShapeError(f"attention needs rank-4 q, k and v [B, H, S, D], got {q}, {k} and {v}")
    if k != v:
        raise AttentionShapeError(f"k {k} and v {v} differ")
    if q[0] != k[0] or q[3] != k[3]:
        raise AttentionShapeError(f"q {q} and k {k} differ in batch or head dim")
    if k[1] == 0 or q[1] % k[1]:
        raise AttentionShapeError(f"Hq = {q[1]} is not a multiple of Hkv = {k[1]}")
    return list(q)


def launch(client: ComputeClient, q: TensorHandle, k: TensorHandle, v: TensorHandle, out: TensorHandle, scale: float | None = None,
           causal: bool = False, lse: TensorHandle | None = None, stream=None) -> None:
    """Enqueue out = softmax(scale * q k^T) v on the client's stream (scale defaults to 1 / sqrt(D)).  lse: an optional compact
    f32 [B, Hq, Sq] tensor that receives the natural-log log-sum-exp of every row.  Never raises for launch problems: errors
    are deferred to client.sync() / read_one() like matmul.launch."""
    try:
        for name, t in (("q", q), ("k", k), ("v", v), ("out", out)):
            if len(t.shape) != 4:
                raise B200Error(6, f"attention: {name} must have rank 4 [B, H, S, D], got rank {len(t.shape)}")
        if not (q.dtype == k.dtype == v.dtype):
            raise B200Error(6, f"attention: q, k and v dtypes differ ({q.dtype}, {k.dtype}, {v.dtype})")
        if lse is not None and (lse.dtype != "f32" or not lse.is_contiguous() or lse.shape != q.shape[:3]):
            raise B200Error(6, f"attention: lse must be a compact f32 [B, Hq, Sq] = {q.shape[:3]} tensor")
        sc = 1.0 / math.sqrt(q.shape[3]) if scale is None else float(scale)
        for t in (q, k, v, out) + ((lse,) if lse is not None else ()):
            t.handle.used_on(stream)
        args = _ffi.AttentionArgs(sc, 1 if causal else 0)
        ops = []
        for t in (q, k, v, out):
            ops += [C.c_uint64(t.handle.ptr), _ffi.u64_array(t.shape), _ffi.u64_array(t.strides)]
        _ffi.check(client._lib.b200_attention(client._ctx, stream, DTYPES[q.dtype], DTYPES[out.dtype], *ops,
                                              C.c_uint64(lse.handle.ptr if lse is not None else 0), C.byref(args)))
    except (B200Error, ValueError) as e:
        client._defer(e if isinstance(e, B200Error) else B200Error(6, str(e)))


def launch_alloc(client: ComputeClient, q: TensorHandle, k: TensorHandle, v: TensorHandle, scale: float | None = None,
                 causal: bool = False, out_dtype: str | None = None, return_lse: bool = False, stream=None):
    """Convenience: allocate a compact out [B, Hq, Sq, D] (and, with return_lse, a compact f32 lse [B, Hq, Sq]), then launch.
    Returns out, or (out, lse)."""
    out = TensorHandle.empty_contiguous(client, calculate_attention_output(q.shape, k.shape, v.shape), out_dtype or q.dtype)
    lse = TensorHandle.empty_contiguous(client, q.shape[:3], "f32") if return_lse else None
    launch(client, q, k, v, out, scale=scale, causal=causal, lse=lse, stream=stream)
    return (out, lse) if return_lse else out


def launch_backward(client: ComputeClient, q: TensorHandle, k: TensorHandle, v: TensorHandle, out: TensorHandle, dout: TensorHandle,
                    lse: TensorHandle, dq: TensorHandle, dk: TensorHandle, dv: TensorHandle, scale: float | None = None,
                    causal: bool = False, stream=None) -> None:
    """Enqueue the attention backward: dq, dk and dv (one grad dtype: the input dtype or f32) from q, k, v, the forward's out
    (input dtype or f32) and lse (its compact f32 [B, Hq, Sq] output) and dout (input dtype).  scale and causal must be the
    forward's (scale defaults to 1 / sqrt(D)).  Never raises for launch problems: errors are deferred to client.sync()."""
    try:
        named = (("q", q), ("k", k), ("v", v), ("out", out), ("dout", dout), ("dq", dq), ("dk", dk), ("dv", dv))
        for name, t in named:
            if len(t.shape) != 4:
                raise B200Error(6, f"attention_backward: {name} must have rank 4 [B, H, S, D], got rank {len(t.shape)}")
        if not (q.dtype == k.dtype == v.dtype == dout.dtype):
            raise B200Error(6, f"attention_backward: q, k, v and dout dtypes differ ({q.dtype}, {k.dtype}, {v.dtype}, {dout.dtype})")
        if not (dq.dtype == dk.dtype == dv.dtype):
            raise B200Error(6, f"attention_backward: dq, dk and dv dtypes differ ({dq.dtype}, {dk.dtype}, {dv.dtype})")
        if lse.dtype != "f32" or not lse.is_contiguous() or list(lse.shape) != list(q.shape[:3]):
            raise B200Error(6, f"attention_backward: lse must be a compact f32 [B, Hq, Sq] = {list(q.shape[:3])} tensor")
        sc = 1.0 / math.sqrt(q.shape[3]) if scale is None else float(scale)
        for _, t in named + (("lse", lse),):
            t.handle.used_on(stream)
        args = _ffi.AttentionArgs(sc, 1 if causal else 0)
        ops = []
        for t in (q, k, v, out, dout):
            ops += [C.c_uint64(t.handle.ptr), _ffi.u64_array(t.shape), _ffi.u64_array(t.strides)]
        ops.append(C.c_uint64(lse.handle.ptr))
        for t in (dq, dk, dv):
            ops += [C.c_uint64(t.handle.ptr), _ffi.u64_array(t.shape), _ffi.u64_array(t.strides)]
        _ffi.check(client._lib.b200_attention_backward(client._ctx, stream, DTYPES[q.dtype], DTYPES[out.dtype], DTYPES[dq.dtype], *ops,
                                                       C.byref(args)))
    except (B200Error, ValueError) as e:
        client._defer(e if isinstance(e, B200Error) else B200Error(6, str(e)))


def launch_backward_alloc(client: ComputeClient, q: TensorHandle, k: TensorHandle, v: TensorHandle, out: TensorHandle,
                          dout: TensorHandle, lse: TensorHandle, scale: float | None = None, causal: bool = False,
                          grad_dtype: str | None = None, stream=None):
    """Convenience: allocate compact dq [B, Hq, Sq, D] and dk, dv [B, Hkv, Sk, D] in grad_dtype (default: q's dtype), then
    launch_backward.  Returns (dq, dk, dv)."""
    gd = grad_dtype or q.dtype
    dq = TensorHandle.empty_contiguous(client, list(q.shape), gd)
    dk = TensorHandle.empty_contiguous(client, list(k.shape), gd)
    dv = TensorHandle.empty_contiguous(client, list(k.shape), gd)
    launch_backward(client, q, k, v, out, dout, lse, dq, dk, dv, scale=scale, causal=causal, stream=stream)
    return dq, dk, dv
