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

Against a KV cache (launch_kvcache, for decoding): q [B, Hq, Sq, D] attends to the first L_b = cache_seqlens[b] keys of
sequence b in a paged cache k_cache, v_cache [P, page, Hkv, D] reached through an i32 block_table [B, max_pages] (None: page b
is sequence b).  causal is bottom-right there: query i also needs j <= L_b - Sq + i.  kvcache_write scatters new tokens
[B, Snew, Hkv, D] into cache slots (slot_mapping, i32 [B * Snew]; negative slots are skipped).  One split-KV kernel with a
fixed-order combine (csrc/attention_kv.cu); see b200_attention_kvcache and b200_kvcache_write.  fp8 caches (f8e4m3 / f8e5m2 with
f32 [Hkv] per-head k_scale and v_scale): launch_kvcache_fp8 widens K and V to q's dtype on chip, kvcache_write_fp8 quantizes new
tokens into them; see b200_attention_kvcache_fp8 and b200_kvcache_write_fp8.

Variable-length (packed) sequences (launch_varlen, torch's varlen_attn / flash_attn_varlen_func): q [Tq, Hq, D] and k, v
[Tk, Hkv, D] hold B sequences back to back; sequence b owns rows [cu_seqlens_q[b], cu_seqlens_q[b + 1]) of q and the matching
rows of k and v (compact i32 [B + 1] device arrays, never read by the host).  window_size = (left, right) as torch's: key j is
visible to query i iff j < Lk and i + off - left <= j <= i + off + right with off = Lk - Lq (-1: unbounded), so (-1, 0) is
bottom-right causal.  lse is a compact f32 [Hq, Tq].  The dense kernels with per-sequence addressing (-DATTN_VARLEN builds of
csrc/attention.cu and attention_bwd.cu); see b200_attention_varlen and b200_attention_varlen_backward.

Paged variable-length attention (launch_varlen_paged, for chunked prefill and prefix caching; flash_attn_varlen_func with a
block_table): packed q [Tq, Hq, D] as launch_varlen's against a paged cache as launch_kvcache's.  Sequence b's Lq_b new queries
are the last of its cache_seqlens[b] cached keys (write the chunk's keys with kvcache_write first), under launch_varlen's window
rule.  Out and lse are bit for bit those of launch_varlen on each sequence's cached keys packed contiguously.  The varlen
forward kernel with paged K / V addressing (-DATTN_VARLEN -DATTN_PAGED); see b200_attention_varlen_paged.
launch_varlen_paged_fp8 does the same against fp8 caches written by kvcache_write_fp8 (chunked prefill and prefix caching with
kv_cache_dtype="fp8"): idle producer warps widen K and V to q's dtype on chip, and power-of-two scales give the bits of
launch_varlen_paged on the dequantized cache; see b200_attention_varlen_paged_fp8.
"""
from __future__ import annotations

import ctypes as C
import functools
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


def _defers_errors(fn):
    """The launch never raises for launch problems: they are deferred to client.sync() / read_one() like matmul.launch."""
    @functools.wraps(fn)
    def wrapper(client, *args, **kwargs):
        try:
            fn(client, *args, **kwargs)
        except (B200Error, ValueError) as e:
            client._defer(e if isinstance(e, B200Error) else B200Error(6, str(e)))
    return wrapper


def _check_rank(what, rank, named, layout=""):
    for name, t in named:
        if len(t.shape) != rank:
            raise B200Error(6, f"{what}: {name} must have rank {rank}{layout}, got rank {len(t.shape)}")


def _check_same_dtype(what, named, listed=True):
    if len({t.dtype for _, t in named}) > 1:
        names = [n for n, _ in named]
        got = f" ({', '.join(t.dtype for _, t in named)})" if listed else ""
        raise B200Error(6, f"{what}: {', '.join(names[:-1])} and {names[-1]} dtypes differ{got}")


def _check_lse(what, lse, dims, want):
    """lse (None: not requested) must be a compact f32 tensor of shape `want`, named `dims` in the message."""
    if lse is not None and (lse.dtype != "f32" or not lse.is_contiguous() or list(lse.shape) != list(want)):
        raise B200Error(6, f"{what}: lse must be a compact f32 {dims} = {list(want)} tensor")


def _scale(scale, D):
    return 1.0 / math.sqrt(D) if scale is None else float(scale)


def _used_on(stream, *tensors):
    for t in tensors:
        if t is not None:
            t.handle.used_on(stream)


def _view_args(tensors):
    ops = []
    for t in tensors:
        ops += [C.c_uint64(t.handle.ptr), _ffi.u64_array(t.shape), _ffi.u64_array(t.strides)]
    return ops


def _ptr(t):
    return C.c_uint64(t.handle.ptr if t is not None else 0)


@_defers_errors
def launch(client: ComputeClient, q: TensorHandle, k: TensorHandle, v: TensorHandle, out: TensorHandle, scale: float | None = None,
           causal: bool = False, lse: TensorHandle | None = None, stream=None) -> None:
    """Enqueue out = softmax(scale * q k^T) v on the client's stream (scale defaults to 1 / sqrt(D)).  lse: an optional compact
    f32 [B, Hq, Sq] tensor that receives the natural-log log-sum-exp of every row.  Never raises for launch problems: errors
    are deferred to client.sync() / read_one() like matmul.launch."""
    what = "attention"
    _check_rank(what, 4, (("q", q), ("k", k), ("v", v), ("out", out)), " [B, H, S, D]")
    _check_same_dtype(what, (("q", q), ("k", k), ("v", v)))
    _check_lse(what, lse, "[B, Hq, Sq]", q.shape[:3])
    args = _ffi.AttentionArgs(_scale(scale, q.shape[3]), 1 if causal else 0)
    _used_on(stream, q, k, v, out, lse)
    _ffi.check(client._lib.b200_attention(client._ctx, stream, DTYPES[q.dtype], DTYPES[out.dtype], *_view_args((q, k, v, out)), _ptr(lse),
                                          C.byref(args)))


def launch_alloc(client: ComputeClient, q: TensorHandle, k: TensorHandle, v: TensorHandle, scale: float | None = None,
                 causal: bool = False, out_dtype: str | None = None, return_lse: bool = False, stream=None):
    """Convenience: allocate a compact out [B, Hq, Sq, D] (and, with return_lse, a compact f32 lse [B, Hq, Sq]), then launch.
    Returns out, or (out, lse)."""
    out = TensorHandle.empty_contiguous(client, calculate_attention_output(q.shape, k.shape, v.shape), out_dtype or q.dtype)
    lse = TensorHandle.empty_contiguous(client, q.shape[:3], "f32") if return_lse else None
    launch(client, q, k, v, out, scale=scale, causal=causal, lse=lse, stream=stream)
    return (out, lse) if return_lse else out


@_defers_errors
def launch_backward(client: ComputeClient, q: TensorHandle, k: TensorHandle, v: TensorHandle, out: TensorHandle, dout: TensorHandle,
                    lse: TensorHandle, dq: TensorHandle, dk: TensorHandle, dv: TensorHandle, scale: float | None = None,
                    causal: bool = False, stream=None) -> None:
    """Enqueue the attention backward: dq, dk and dv (one grad dtype: the input dtype or f32) from q, k, v, the forward's out
    (input dtype or f32) and lse (its compact f32 [B, Hq, Sq] output) and dout (input dtype).  scale and causal must be the
    forward's (scale defaults to 1 / sqrt(D)).  Never raises for launch problems: errors are deferred to client.sync()."""
    what = "attention_backward"
    _check_rank(what, 4, (("q", q), ("k", k), ("v", v), ("out", out), ("dout", dout), ("dq", dq), ("dk", dk), ("dv", dv)),
                " [B, H, S, D]")
    _check_same_dtype(what, (("q", q), ("k", k), ("v", v), ("dout", dout)))
    _check_same_dtype(what, (("dq", dq), ("dk", dk), ("dv", dv)))
    _check_lse(what, lse, "[B, Hq, Sq]", q.shape[:3])
    args = _ffi.AttentionArgs(_scale(scale, q.shape[3]), 1 if causal else 0)
    _used_on(stream, q, k, v, out, dout, dq, dk, dv, lse)
    _ffi.check(client._lib.b200_attention_backward(client._ctx, stream, DTYPES[q.dtype], DTYPES[out.dtype], DTYPES[dq.dtype],
                                                   *_view_args((q, k, v, out, dout)), _ptr(lse), *_view_args((dq, dk, dv)),
                                                   C.byref(args)))


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


@_defers_errors
def launch_kvcache(client: ComputeClient, q: TensorHandle, k_cache: TensorHandle, v_cache: TensorHandle, cache_seqlens: TensorHandle,
                   out: TensorHandle, block_table: TensorHandle | None = None, scale: float | None = None, causal: bool = False,
                   lse: TensorHandle | None = None, stream=None) -> None:
    """Enqueue attention of q [B, Hq, Sq, D] against a KV cache k_cache, v_cache [P, page, Hkv, D] (views by strides): sequence b
    sees its first cache_seqlens[b] keys (compact i32 [B], read on the device), key j at row j % page of page
    block_table[b, j / page] (i32 [B, max_pages]; None: page b).  causal: bottom-right (query i sees j <= L_b - Sq + i).  scale
    defaults to 1 / sqrt(D); lse: an optional compact f32 [B, Hq, Sq] tensor.  Never raises for launch problems: errors are
    deferred to client.sync()."""
    what = "attention_kvcache"
    _check_rank(what, 4, (("q", q), ("k_cache", k_cache), ("v_cache", v_cache), ("out", out)))
    _check_same_dtype(what, (("q", q), ("k_cache", k_cache), ("v_cache", v_cache)))
    if cache_seqlens.dtype != "i32" or not cache_seqlens.is_contiguous() or list(cache_seqlens.shape) != [q.shape[0]]:
        raise B200Error(6, f"{what}: cache_seqlens must be a compact i32 [B] = [{q.shape[0]}] tensor")
    if block_table is not None and (block_table.dtype != "i32" or len(block_table.shape) != 2):
        raise B200Error(6, f"{what}: block_table must be an i32 [B, max_pages] tensor")
    _check_lse(what, lse, "[B, Hq, Sq]", q.shape[:3])
    args = _ffi.AttentionArgs(_scale(scale, q.shape[3]), 1 if causal else 0)
    _used_on(stream, q, k_cache, v_cache, cache_seqlens, out, block_table, lse)
    bt = _view_args((block_table,)) if block_table is not None else [C.c_uint64(0), None, None]
    _ffi.check(client._lib.b200_attention_kvcache(
        client._ctx, stream, DTYPES[q.dtype], DTYPES[out.dtype], *_view_args((q, k_cache, v_cache)), *bt, _ptr(cache_seqlens),
        *_view_args((out,)), _ptr(lse), C.byref(args)))


def launch_kvcache_alloc(client: ComputeClient, q: TensorHandle, k_cache: TensorHandle, v_cache: TensorHandle,
                         cache_seqlens: TensorHandle, block_table: TensorHandle | None = None, scale: float | None = None,
                         causal: bool = False, out_dtype: str | None = None, return_lse: bool = False, stream=None):
    """Convenience: allocate a compact out [B, Hq, Sq, D] (and, with return_lse, a compact f32 lse [B, Hq, Sq]), then
    launch_kvcache.  Returns out, or (out, lse)."""
    out = TensorHandle.empty_contiguous(client, list(q.shape), out_dtype or q.dtype)
    lse = TensorHandle.empty_contiguous(client, list(q.shape[:3]), "f32") if return_lse else None
    launch_kvcache(client, q, k_cache, v_cache, cache_seqlens, out, block_table=block_table, scale=scale, causal=causal, lse=lse,
                   stream=stream)
    return (out, lse) if return_lse else out


@_defers_errors
def kvcache_write(client: ComputeClient, k_new: TensorHandle, v_new: TensorHandle, k_cache: TensorHandle, v_cache: TensorHandle,
                  slot_mapping: TensorHandle, stream=None) -> None:
    """Enqueue the scatter of k_new, v_new [B, Snew, Hkv, D] into k_cache, v_cache [P, page, Hkv, D]: token t of sequence b goes
    to flat slot slot_mapping[b * Snew + t] (compact i32; page slot / page, row slot % page); negative slots are skipped.  Lengths
    stay with the caller.  Errors are deferred to client.sync()."""
    what = "kvcache_write"
    named = (("k_new", k_new), ("v_new", v_new), ("k_cache", k_cache), ("v_cache", v_cache))
    _check_rank(what, 4, named)
    _check_same_dtype(what, named, listed=False)
    n = k_new.shape[0] * k_new.shape[1]
    if slot_mapping.dtype != "i32" or not slot_mapping.is_contiguous() or math.prod(slot_mapping.shape) != n:
        raise B200Error(6, f"{what}: slot_mapping must be a compact i32 tensor of B * Snew = {n} slots")
    _used_on(stream, k_new, v_new, k_cache, v_cache, slot_mapping)
    _ffi.check(client._lib.b200_kvcache_write(client._ctx, stream, DTYPES[k_cache.dtype], *_view_args((k_new, v_new, k_cache, v_cache)),
                                              _ptr(slot_mapping)))


_FP8 = ("f8e4m3", "f8e5m2")


def _check_fp8(what, k_cache, v_cache, k_scale, v_scale, Hkv):
    if k_cache.dtype != v_cache.dtype:
        raise B200Error(7, f"{what}: k_cache and v_cache dtypes differ ({k_cache.dtype}, {v_cache.dtype})")
    if k_cache.dtype not in _FP8:
        raise B200Error(7, f"{what}: cache dtype {k_cache.dtype} unsupported (f8e4m3, f8e5m2)")
    for name, t in (("k_scale", k_scale), ("v_scale", v_scale)):
        if t.dtype != "f32" or not t.is_contiguous() or list(t.shape) != [Hkv]:
            raise B200Error(6, f"{what}: {name} must be a compact f32 [Hkv] = [{Hkv}] tensor")


@_defers_errors
def launch_kvcache_fp8(client: ComputeClient, q: TensorHandle, k_cache: TensorHandle, v_cache: TensorHandle,
                       cache_seqlens: TensorHandle, k_scale: TensorHandle, v_scale: TensorHandle, out: TensorHandle,
                       block_table: TensorHandle | None = None, scale: float | None = None, causal: bool = False,
                       lse: TensorHandle | None = None, stream=None) -> None:
    """launch_kvcache against an fp8 cache: k_cache and v_cache f8e4m3 or f8e5m2 [P, page, Hkv, D] holding K = k_scale[hk] * k8
    and V = v_scale[hk] * v8, with k_scale and v_scale compact f32 [Hkv] tensors (read on the device).  K and V are widened
    exactly to q's dtype on chip; scores are scaled by scale * k_scale[hk] and out = (v_scale[hk] * O) / l.  Power-of-two
    scales give the bits of launch_kvcache on the dequantized cache.  Never raises for launch problems: errors are deferred to
    client.sync()."""
    what = "attention_kvcache_fp8"
    _check_rank(what, 4, (("q", q), ("k_cache", k_cache), ("v_cache", v_cache), ("out", out)))
    _check_fp8(what, k_cache, v_cache, k_scale, v_scale, k_cache.shape[2])
    if cache_seqlens.dtype != "i32" or not cache_seqlens.is_contiguous() or list(cache_seqlens.shape) != [q.shape[0]]:
        raise B200Error(6, f"{what}: cache_seqlens must be a compact i32 [B] = [{q.shape[0]}] tensor")
    if block_table is not None and (block_table.dtype != "i32" or len(block_table.shape) != 2):
        raise B200Error(6, f"{what}: block_table must be an i32 [B, max_pages] tensor")
    _check_lse(what, lse, "[B, Hq, Sq]", q.shape[:3])
    args = _ffi.AttentionArgs(_scale(scale, q.shape[3]), 1 if causal else 0)
    _used_on(stream, q, k_cache, v_cache, cache_seqlens, k_scale, v_scale, out, block_table, lse)
    bt = _view_args((block_table,)) if block_table is not None else [C.c_uint64(0), None, None]
    _ffi.check(client._lib.b200_attention_kvcache_fp8(
        client._ctx, stream, DTYPES[q.dtype], DTYPES[k_cache.dtype], DTYPES[out.dtype], *_view_args((q, k_cache, v_cache)), *bt,
        _ptr(cache_seqlens), _ptr(k_scale), _ptr(v_scale), *_view_args((out,)), _ptr(lse), C.byref(args)))


def launch_kvcache_fp8_alloc(client: ComputeClient, q: TensorHandle, k_cache: TensorHandle, v_cache: TensorHandle,
                             cache_seqlens: TensorHandle, k_scale: TensorHandle, v_scale: TensorHandle,
                             block_table: TensorHandle | None = None, scale: float | None = None, causal: bool = False,
                             out_dtype: str | None = None, return_lse: bool = False, stream=None):
    """Convenience: allocate a compact out [B, Hq, Sq, D] (and, with return_lse, a compact f32 lse [B, Hq, Sq]), then
    launch_kvcache_fp8.  Returns out, or (out, lse)."""
    out = TensorHandle.empty_contiguous(client, list(q.shape), out_dtype or q.dtype)
    lse = TensorHandle.empty_contiguous(client, list(q.shape[:3]), "f32") if return_lse else None
    launch_kvcache_fp8(client, q, k_cache, v_cache, cache_seqlens, k_scale, v_scale, out, block_table=block_table, scale=scale,
                       causal=causal, lse=lse, stream=stream)
    return (out, lse) if return_lse else out


@_defers_errors
def kvcache_write_fp8(client: ComputeClient, k_new: TensorHandle, v_new: TensorHandle, k_cache: TensorHandle, v_cache: TensorHandle,
                      slot_mapping: TensorHandle, k_scale: TensorHandle, v_scale: TensorHandle, stream=None) -> None:
    """kvcache_write into fp8 caches: k_new, v_new f16 or bf16 [B, Snew, Hkv, D]; each value x of kv head hk is stored as
    sat_rn(x / scale[hk]) in the cache format (saturating to +-448 for e4m3, +-57344 for e5m2; NaN stays NaN), with k_scale /
    v_scale compact f32 [Hkv] tensors.  Slots as kvcache_write.  Errors are deferred to client.sync()."""
    what = "kvcache_write_fp8"
    _check_rank(what, 4, (("k_new", k_new), ("v_new", v_new), ("k_cache", k_cache), ("v_cache", v_cache)))
    _check_same_dtype(what, (("k_new", k_new), ("v_new", v_new)))
    _check_fp8(what, k_cache, v_cache, k_scale, v_scale, k_cache.shape[2])
    n = k_new.shape[0] * k_new.shape[1]
    if slot_mapping.dtype != "i32" or not slot_mapping.is_contiguous() or math.prod(slot_mapping.shape) != n:
        raise B200Error(6, f"{what}: slot_mapping must be a compact i32 tensor of B * Snew = {n} slots")
    _used_on(stream, k_new, v_new, k_cache, v_cache, slot_mapping, k_scale, v_scale)
    _ffi.check(client._lib.b200_kvcache_write_fp8(client._ctx, stream, DTYPES[k_new.dtype], DTYPES[k_cache.dtype],
                                                  *_view_args((k_new, v_new, k_cache, v_cache)), _ptr(slot_mapping), _ptr(k_scale),
                                                  _ptr(v_scale)))


def _varlen_args(q, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k, scale, window_size, what):
    if not (cu_seqlens_q.dtype == cu_seqlens_k.dtype == "i32") or not cu_seqlens_q.is_contiguous() or not cu_seqlens_k.is_contiguous() \
            or len(cu_seqlens_q.shape) != 1 or list(cu_seqlens_k.shape) != list(cu_seqlens_q.shape) or cu_seqlens_q.shape[0] < 1:
        raise B200Error(6, f"{what}: cu_seqlens_q and cu_seqlens_k must be compact i32 [B + 1] tensors of one length")
    left, right = (int(w) for w in window_size)
    return _ffi.AttentionVarlenArgs(_scale(scale, q.shape[2]), left, right, int(max_seqlen_q), int(max_seqlen_k)), cu_seqlens_q.shape[0] - 1


@_defers_errors
def launch_varlen(client: ComputeClient, q: TensorHandle, k: TensorHandle, v: TensorHandle, cu_seqlens_q: TensorHandle,
                  cu_seqlens_k: TensorHandle, max_seqlen_q: int, max_seqlen_k: int, out: TensorHandle, scale: float | None = None,
                  window_size=(-1, -1), lse: TensorHandle | None = None, stream=None) -> None:
    """Enqueue attention over packed sequences: q [Tq, Hq, D], k and v [Tk, Hkv, D], out [Tq, Hq, D] (views by strides);
    cu_seqlens_q / cu_seqlens_k compact i32 [B + 1] offsets, max_seqlen_q / max_seqlen_k host bounds on the lengths.
    window_size (left, right), -1 unbounded: (-1, 0) is bottom-right causal.  scale defaults to 1 / sqrt(D); lse: an optional
    compact f32 [Hq, Tq] tensor.  Rows outside every sequence are not written.  Never raises for launch problems: errors are
    deferred to client.sync()."""
    what = "attention_varlen"
    _check_rank(what, 3, (("q", q), ("k", k), ("v", v), ("out", out)), " [T, H, D]")
    _check_same_dtype(what, (("q", q), ("k", k), ("v", v)))
    _check_lse(what, lse, "[Hq, Tq]", [q.shape[1], q.shape[0]])
    args, B = _varlen_args(q, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k, scale, window_size, what)
    _used_on(stream, q, k, v, cu_seqlens_q, cu_seqlens_k, out, lse)
    _ffi.check(client._lib.b200_attention_varlen(
        client._ctx, stream, DTYPES[q.dtype], DTYPES[out.dtype], *_view_args((q, k, v)), _ptr(cu_seqlens_q), _ptr(cu_seqlens_k),
        C.c_uint64(B), *_view_args((out,)), _ptr(lse), C.byref(args)))


def launch_varlen_alloc(client: ComputeClient, q: TensorHandle, k: TensorHandle, v: TensorHandle, cu_seqlens_q: TensorHandle,
                        cu_seqlens_k: TensorHandle, max_seqlen_q: int, max_seqlen_k: int, scale: float | None = None,
                        window_size=(-1, -1), out_dtype: str | None = None, return_lse: bool = False, stream=None):
    """Convenience: allocate a compact out [Tq, Hq, D] (and, with return_lse, a compact f32 lse [Hq, Tq]), then launch_varlen.
    Rows outside every sequence are left as allocated.  Returns out, or (out, lse)."""
    out = TensorHandle.empty_contiguous(client, list(q.shape), out_dtype or q.dtype)
    lse = TensorHandle.empty_contiguous(client, [q.shape[1], q.shape[0]], "f32") if return_lse else None
    launch_varlen(client, q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k, out, scale=scale, window_size=window_size,
                  lse=lse, stream=stream)
    return (out, lse) if return_lse else out


@_defers_errors
def launch_varlen_backward(client: ComputeClient, q: TensorHandle, k: TensorHandle, v: TensorHandle, out: TensorHandle,
                           dout: TensorHandle, lse: TensorHandle, cu_seqlens_q: TensorHandle, cu_seqlens_k: TensorHandle,
                           max_seqlen_q: int, max_seqlen_k: int, dq: TensorHandle, dk: TensorHandle, dv: TensorHandle,
                           scale: float | None = None, window_size=(-1, -1), stream=None) -> None:
    """Enqueue the varlen backward: dq [Tq, Hq, D], dk and dv [Tk, Hkv, D] (one grad dtype: the input dtype or f32) from q, k, v,
    the forward's out and lse (compact f32 [Hq, Tq]) and dout.  Offsets, scale and window_size must be the forward's.  Rows
    outside every sequence are not written.  Never raises for launch problems: errors are deferred to client.sync()."""
    what = "attention_varlen_backward"
    _check_rank(what, 3, (("q", q), ("k", k), ("v", v), ("out", out), ("dout", dout), ("dq", dq), ("dk", dk), ("dv", dv)), " [T, H, D]")
    _check_same_dtype(what, (("q", q), ("k", k), ("v", v), ("dout", dout)))
    _check_same_dtype(what, (("dq", dq), ("dk", dk), ("dv", dv)))
    _check_lse(what, lse, "[Hq, Tq]", [q.shape[1], q.shape[0]])
    args, B = _varlen_args(q, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k, scale, window_size, what)
    _used_on(stream, q, k, v, out, dout, dq, dk, dv, lse, cu_seqlens_q, cu_seqlens_k)
    _ffi.check(client._lib.b200_attention_varlen_backward(
        client._ctx, stream, DTYPES[q.dtype], DTYPES[out.dtype], DTYPES[dq.dtype], *_view_args((q, k, v, out, dout)), _ptr(lse),
        _ptr(cu_seqlens_q), _ptr(cu_seqlens_k), C.c_uint64(B), *_view_args((dq, dk, dv)), C.byref(args)))


def launch_varlen_backward_alloc(client: ComputeClient, q: TensorHandle, k: TensorHandle, v: TensorHandle, out: TensorHandle,
                                 dout: TensorHandle, lse: TensorHandle, cu_seqlens_q: TensorHandle, cu_seqlens_k: TensorHandle,
                                 max_seqlen_q: int, max_seqlen_k: int, scale: float | None = None, window_size=(-1, -1),
                                 grad_dtype: str | None = None, stream=None):
    """Convenience: allocate compact dq [Tq, Hq, D] and dk, dv [Tk, Hkv, D] in grad_dtype (default: q's dtype), then
    launch_varlen_backward.  Returns (dq, dk, dv)."""
    gd = grad_dtype or q.dtype
    dq = TensorHandle.empty_contiguous(client, list(q.shape), gd)
    dk = TensorHandle.empty_contiguous(client, list(k.shape), gd)
    dv = TensorHandle.empty_contiguous(client, list(k.shape), gd)
    launch_varlen_backward(client, q, k, v, out, dout, lse, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k, dq, dk, dv,
                           scale=scale, window_size=window_size, stream=stream)
    return dq, dk, dv


@_defers_errors
def launch_varlen_paged(client: ComputeClient, q: TensorHandle, k_cache: TensorHandle, v_cache: TensorHandle, cu_seqlens_q: TensorHandle,
                        cache_seqlens: TensorHandle, max_seqlen_q: int, max_seqlen_k: int, out: TensorHandle,
                        block_table: TensorHandle | None = None, scale: float | None = None, window_size=(-1, -1),
                        lse: TensorHandle | None = None, stream=None) -> None:
    """Enqueue packed queries q [Tq, Hq, D] (rows [cu_seqlens_q[b], cu_seqlens_q[b + 1]) of sequence b; compact i32 [B + 1])
    against a paged cache k_cache, v_cache [P, page, Hkv, D] in q's dtype (views by strides): sequence b has its first
    cache_seqlens[b] keys (compact i32 [B], read on the device, clamped to max_seqlen_k), key j at row j % page of page
    block_table[b, j / page] (i32 [B, max_pages]; None: page b).  window_size as launch_varlen's with off = Lk - Lq: the new
    queries are the last keys, (-1, 0) is bottom-right causal.  out [Tq, Hq, D]; lse: an optional compact f32 [Hq, Tq] tensor.
    Rows outside every sequence are not written.  Never raises for launch problems: errors are deferred to client.sync()."""
    what = "attention_varlen_paged"
    _check_rank(what, 3, (("q", q), ("out", out)), " [T, H, D]")
    _check_rank(what, 4, (("k_cache", k_cache), ("v_cache", v_cache)), " [P, page, Hkv, D]")
    if k_cache.dtype in _FP8 or v_cache.dtype in _FP8:
        raise B200Error(7, f"{what}: fp8 caches unsupported (the caches hold q's dtype)")
    _check_same_dtype(what, (("q", q), ("k_cache", k_cache), ("v_cache", v_cache)))
    if cu_seqlens_q.dtype != "i32" or not cu_seqlens_q.is_contiguous() or len(cu_seqlens_q.shape) != 1 or cu_seqlens_q.shape[0] < 1:
        raise B200Error(6, f"{what}: cu_seqlens_q must be a compact i32 [B + 1] tensor")
    B = cu_seqlens_q.shape[0] - 1
    if cache_seqlens.dtype != "i32" or not cache_seqlens.is_contiguous() or list(cache_seqlens.shape) != [B]:
        raise B200Error(6, f"{what}: cache_seqlens must be a compact i32 [B] = [{B}] tensor")
    if block_table is not None and (block_table.dtype != "i32" or len(block_table.shape) != 2):
        raise B200Error(6, f"{what}: block_table must be an i32 [B, max_pages] tensor")
    _check_lse(what, lse, "[Hq, Tq]", [q.shape[1], q.shape[0]])
    left, right = (int(w) for w in window_size)
    args = _ffi.AttentionVarlenArgs(_scale(scale, q.shape[2]), left, right, int(max_seqlen_q), int(max_seqlen_k))
    _used_on(stream, q, k_cache, v_cache, cu_seqlens_q, cache_seqlens, out, block_table, lse)
    bt = _view_args((block_table,)) if block_table is not None else [C.c_uint64(0), None, None]
    _ffi.check(client._lib.b200_attention_varlen_paged(
        client._ctx, stream, DTYPES[q.dtype], DTYPES[out.dtype], *_view_args((q, k_cache, v_cache)), *bt, _ptr(cu_seqlens_q),
        _ptr(cache_seqlens), C.c_uint64(B), *_view_args((out,)), _ptr(lse), C.byref(args)))


def launch_varlen_paged_alloc(client: ComputeClient, q: TensorHandle, k_cache: TensorHandle, v_cache: TensorHandle,
                              cu_seqlens_q: TensorHandle, cache_seqlens: TensorHandle, max_seqlen_q: int, max_seqlen_k: int,
                              block_table: TensorHandle | None = None, scale: float | None = None, window_size=(-1, -1),
                              out_dtype: str | None = None, return_lse: bool = False, stream=None):
    """Convenience: allocate a compact out [Tq, Hq, D] (and, with return_lse, a compact f32 lse [Hq, Tq]), then
    launch_varlen_paged.  Rows outside every sequence are left as allocated.  Returns out, or (out, lse)."""
    out = TensorHandle.empty_contiguous(client, list(q.shape), out_dtype or q.dtype)
    lse = TensorHandle.empty_contiguous(client, [q.shape[1], q.shape[0]], "f32") if return_lse else None
    launch_varlen_paged(client, q, k_cache, v_cache, cu_seqlens_q, cache_seqlens, max_seqlen_q, max_seqlen_k, out,
                        block_table=block_table, scale=scale, window_size=window_size, lse=lse, stream=stream)
    return (out, lse) if return_lse else out


@_defers_errors
def launch_varlen_paged_fp8(client: ComputeClient, q: TensorHandle, k_cache: TensorHandle, v_cache: TensorHandle,
                            cu_seqlens_q: TensorHandle, cache_seqlens: TensorHandle, k_scale: TensorHandle, v_scale: TensorHandle,
                            max_seqlen_q: int, max_seqlen_k: int, out: TensorHandle, block_table: TensorHandle | None = None,
                            scale: float | None = None, window_size=(-1, -1), lse: TensorHandle | None = None, stream=None) -> None:
    """launch_varlen_paged against an fp8 cache: k_cache and v_cache f8e4m3 or f8e5m2 [P, page, Hkv, D] holding
    K = k_scale[hk] * k8 and V = v_scale[hk] * v8, with k_scale and v_scale compact f32 [Hkv] tensors (read on the device).
    K and V are widened exactly to q's dtype on chip; scores are scaled by scale * k_scale[hk] and out = (v_scale[hk] * O) / l.
    Power-of-two scales give the bits of launch_varlen_paged on the dequantized cache.  Never raises for launch problems:
    errors are deferred to client.sync()."""
    what = "attention_varlen_paged_fp8"
    _check_rank(what, 3, (("q", q), ("out", out)), " [T, H, D]")
    _check_rank(what, 4, (("k_cache", k_cache), ("v_cache", v_cache)), " [P, page, Hkv, D]")
    _check_fp8(what, k_cache, v_cache, k_scale, v_scale, k_cache.shape[2])
    if cu_seqlens_q.dtype != "i32" or not cu_seqlens_q.is_contiguous() or len(cu_seqlens_q.shape) != 1 or cu_seqlens_q.shape[0] < 1:
        raise B200Error(6, f"{what}: cu_seqlens_q must be a compact i32 [B + 1] tensor")
    B = cu_seqlens_q.shape[0] - 1
    if cache_seqlens.dtype != "i32" or not cache_seqlens.is_contiguous() or list(cache_seqlens.shape) != [B]:
        raise B200Error(6, f"{what}: cache_seqlens must be a compact i32 [B] = [{B}] tensor")
    if block_table is not None and (block_table.dtype != "i32" or len(block_table.shape) != 2):
        raise B200Error(6, f"{what}: block_table must be an i32 [B, max_pages] tensor")
    _check_lse(what, lse, "[Hq, Tq]", [q.shape[1], q.shape[0]])
    left, right = (int(w) for w in window_size)
    args = _ffi.AttentionVarlenArgs(_scale(scale, q.shape[2]), left, right, int(max_seqlen_q), int(max_seqlen_k))
    _used_on(stream, q, k_cache, v_cache, cu_seqlens_q, cache_seqlens, k_scale, v_scale, out, block_table, lse)
    bt = _view_args((block_table,)) if block_table is not None else [C.c_uint64(0), None, None]
    _ffi.check(client._lib.b200_attention_varlen_paged_fp8(
        client._ctx, stream, DTYPES[q.dtype], DTYPES[k_cache.dtype], DTYPES[out.dtype], *_view_args((q, k_cache, v_cache)), *bt,
        _ptr(cu_seqlens_q), _ptr(cache_seqlens), C.c_uint64(B), _ptr(k_scale), _ptr(v_scale), *_view_args((out,)), _ptr(lse),
        C.byref(args)))


def launch_varlen_paged_fp8_alloc(client: ComputeClient, q: TensorHandle, k_cache: TensorHandle, v_cache: TensorHandle,
                                  cu_seqlens_q: TensorHandle, cache_seqlens: TensorHandle, k_scale: TensorHandle, v_scale: TensorHandle,
                                  max_seqlen_q: int, max_seqlen_k: int, block_table: TensorHandle | None = None,
                                  scale: float | None = None, window_size=(-1, -1), out_dtype: str | None = None,
                                  return_lse: bool = False, stream=None):
    """Convenience: allocate a compact out [Tq, Hq, D] (and, with return_lse, a compact f32 lse [Hq, Tq]), then
    launch_varlen_paged_fp8.  Rows outside every sequence are left as allocated.  Returns out, or (out, lse)."""
    out = TensorHandle.empty_contiguous(client, list(q.shape), out_dtype or q.dtype)
    lse = TensorHandle.empty_contiguous(client, [q.shape[1], q.shape[0]], "f32") if return_lse else None
    launch_varlen_paged_fp8(client, q, k_cache, v_cache, cu_seqlens_q, cache_seqlens, k_scale, v_scale, max_seqlen_q, max_seqlen_k,
                            out, block_table=block_table, scale=scale, window_size=window_size, lse=lse, stream=stream)
    return (out, lse) if return_lse else out
