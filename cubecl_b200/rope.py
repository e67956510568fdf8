"""Rotary position embeddings on the GPU: rotate q and k (the backward is the inverse rotation), the decode / prefill step
that rotates k straight into a paged KV cache, and the cos / sin tables of transformers' rope_parameters.  A Llama block:

    cos_sin = cos_sin_alloc(c, P, 128, 500000.0, {"rope_type": "llama3", "factor": 8.0, "low_freq_factor": 1.0,
                                                  "high_freq_factor": 4.0, "original_max_position_embeddings": 8192})
    apply(c, cos_sin, q=q, k=k, positions=pos)                       # in place, [B, S, H, D] views
    kvcache_write(c, cos_sin, q, k_new, v_new, k_cache, v_cache, slots, cache_seqlens)   # decode step, one launch

The contracts (operation order, out-of-range positions, pass-through columns, fp8 caches, table rules) are those of
b200_rope* in include/cubecl_b200.h; kernels in csrc/rope.cu.  Nothing synchronises with the host, and errors are deferred
to client.sync() like every launch.
"""
from __future__ import annotations

import ctypes as C

from . import _ffi
from ._ffi import B200Error
from .client import DTYPES, ComputeClient, TensorHandle

STYLES = {"neox": _ffi.ROPE_NEOX, "gptj": _ffi.ROPE_GPTJ}
KINDS = {"default": _ffi.ROPE_DEFAULT, "linear": _ffi.ROPE_LINEAR, "llama3": _ffi.ROPE_LLAMA3, "yarn": _ffi.ROPE_YARN}


def _p(t: TensorHandle | None) -> C.c_uint64:
    return C.c_uint64(t.handle.ptr if t is not None else 0)


def _view(t: TensorHandle | None):
    if t is None:
        return [C.c_uint64(0), None, None]
    return [C.c_uint64(t.handle.ptr), _ffi.u64_array(t.shape), _ffi.u64_array(t.strides)]


def _used_on(stream, *ts):
    for t in ts:
        if t is not None:
            t.handle.used_on(stream)


def _args(what, style, rot_dim, inverse, D):
    if style not in STYLES:
        raise B200Error(6, f"{what}: unknown style {style!r} (neox, gptj)")
    return _ffi.RopeArgs(STYLES[style], int(D if rot_dim is None else rot_dim), 1 if inverse else 0)


def _check(what, cos_sin, positions, named, B, S):
    for name, t in named:
        if t is not None and len(t.shape) != 4:
            raise B200Error(6, f"{what}: {name} must be a 4-D [B, S, H, D] view, got shape {t.shape}")
    if cos_sin.dtype != "f32" or len(cos_sin.shape) != 2 or not cos_sin.is_contiguous():
        raise B200Error(6, f"{what}: cos_sin must be a compact f32 [P, rot_dim] tensor")
    if positions is not None and (positions.dtype != "i32" or not positions.is_contiguous() or positions.size() != B * S):
        raise B200Error(6, f"{what}: positions must be a compact i32 [B, S] = [{B}, {S}] tensor")


def apply(client: ComputeClient, cos_sin: TensorHandle, q: TensorHandle | None = None, k: TensorHandle | None = None,
          positions: TensorHandle | None = None, q_out: TensorHandle | None = None, k_out: TensorHandle | None = None,
          style: str = "neox", rot_dim: int | None = None, inverse: bool = False, stream=None) -> None:
    """Rotate q [B, S, Hq, D] and / or k [B, S, Hk, D] by the rows of cos_sin (f32 [P, rot_dim]: cos then sin) at positions
    (i32 [B, S]; None: s).  In place unless q_out / k_out are given; rot_dim defaults to cos_sin's width; inverse rotates by
    -theta (the backward)."""
    what = "rope"
    try:
        ref = q if q is not None else k
        if ref is None:
            raise B200Error(6, f"{what}: q and k are both None")
        _check(what, cos_sin, positions, (("q", q), ("k", k), ("q_out", q_out), ("k_out", k_out)), ref.shape[0], ref.shape[1])
        if len({t.dtype for t in (q, k, q_out, k_out) if t is not None}) > 1:
            raise B200Error(6, f"{what}: q, k and the outputs must share a dtype")
        args = _args(what, style, cos_sin.shape[1] if rot_dim is None else rot_dim, inverse, ref.shape[3])
        _used_on(stream, cos_sin, q, k, positions, q_out, k_out)
        _ffi.check(client._lib.b200_rope(client._ctx, stream, C.byref(args), DTYPES[ref.dtype], *_view(q), *_view(k), *_view(q_out),
                                         *_view(k_out), _p(positions), _p(cos_sin), cos_sin.shape[0]))
    except B200Error as e:
        client._defer(e)


def apply_alloc(client: ComputeClient, cos_sin: TensorHandle, q: TensorHandle | None = None, k: TensorHandle | None = None,
                positions: TensorHandle | None = None, style: str = "neox", rot_dim: int | None = None, inverse: bool = False,
                stream=None):
    """(q_rot, k_rot): apply() into new compact tensors (None where the input is None); q and k are left as they are."""
    q_out = TensorHandle.empty_contiguous(client, list(q.shape), q.dtype) if q is not None else None
    k_out = TensorHandle.empty_contiguous(client, list(k.shape), k.dtype) if k is not None else None
    apply(client, cos_sin, q, k, positions, q_out, k_out, style, rot_dim, inverse, stream)
    return q_out, k_out


def kvcache_write(client: ComputeClient, cos_sin: TensorHandle, q: TensorHandle | None, k_new: TensorHandle, v_new: TensorHandle,
                  k_cache: TensorHandle, v_cache: TensorHandle, slots: TensorHandle, positions: TensorHandle | None,
                  q_out: TensorHandle | None = None, k_scale: TensorHandle | None = None, v_scale: TensorHandle | None = None,
                  style: str = "neox", rot_dim: int | None = None, stream=None) -> None:
    """One launch: q [B, Snew, Hq, D] rotated (in place, or into q_out), k_new rotated and v_new as it is written to their
    cache slots (attention.kvcache_write's rules), bit for bit apply() then attention.kvcache_write(_fp8).  The cache dtype is
    k_cache's: q's dtype, or f8e4m3 / f8e5m2 with k_scale / v_scale compact f32 [Hkv]."""
    what = "rope_kvcache_write"
    try:
        _check(what, cos_sin, positions, (("q", q), ("q_out", q_out), ("k_new", k_new), ("v_new", v_new), ("k_cache", k_cache),
                                          ("v_cache", v_cache)), k_new.shape[0], k_new.shape[1])
        if slots.dtype != "i32" or not slots.is_contiguous() or slots.size() != k_new.shape[0] * k_new.shape[1]:
            raise B200Error(6, f"{what}: slots must be a compact i32 tensor of B * Snew slots")
        if k_cache.dtype != v_cache.dtype:
            raise B200Error(6, f"{what}: k_cache and v_cache dtypes differ")
        fp8 = k_cache.dtype in ("f8e4m3", "f8e5m2")
        if fp8 and (k_scale is None or v_scale is None):
            raise B200Error(6, f"{what}: an fp8 cache needs k_scale and v_scale")
        args = _args(what, style, cos_sin.shape[1] if rot_dim is None else rot_dim, False, k_new.shape[3])
        _used_on(stream, cos_sin, q, q_out, k_new, v_new, k_cache, v_cache, slots, positions, k_scale, v_scale)
        _ffi.check(client._lib.b200_rope_kvcache_write(
            client._ctx, stream, C.byref(args), DTYPES[k_new.dtype], DTYPES[k_cache.dtype], *_view(q), *_view(q_out), *_view(k_new),
            *_view(v_new), *_view(k_cache), *_view(v_cache), _p(slots), _p(positions), _p(cos_sin), cos_sin.shape[0],
            _p(k_scale if fp8 else None), _p(v_scale if fp8 else None)))
    except B200Error as e:
        client._defer(e)


def table_args(rot_dim: int, base: float = 10000.0, scaling: dict | None = None, attention_factor: float | None = None,
               inv_freq: TensorHandle | None = None) -> "_ffi.RopeTableArgs":
    """The b200_rope_table_args of HF's rope_parameters: scaling is None (default) or {"rope_type": "default" | "linear" |
    "llama3" | "yarn", and that rule's keys}.  A yarn dict without "factor" takes max_position_embeddings /
    original_max_position_embeddings, as transformers does.  inv_freq (f32 [rot_dim / 2]) overrides every rule."""
    s = dict(scaling or {})
    kind = s.get("rope_type", s.get("type", "default"))
    if inv_freq is None and kind not in KINDS:
        raise B200Error(6, f"rope table: unsupported rope_type {kind!r} ({', '.join(KINDS)}; others: pass inv_freq)")
    factor = s.get("factor")
    if factor is None and kind == "yarn" and "max_position_embeddings" in s:
        factor = s["max_position_embeddings"] / s["original_max_position_embeddings"]
    a = _ffi.RopeTableArgs()
    a.inv_freq = inv_freq.handle.ptr if inv_freq is not None else 0
    a.kind = _ffi.ROPE_INV_FREQ if inv_freq is not None else KINDS[kind]
    a.rot_dim = int(rot_dim)
    a.base = float(s.get("rope_theta", base))
    a.factor = float(factor if factor is not None else 1.0)
    a.low_freq_factor = float(s.get("low_freq_factor", 0.0))
    a.high_freq_factor = float(s.get("high_freq_factor", 0.0))
    a.beta_fast = float(s.get("beta_fast") or 0.0)
    a.beta_slow = float(s.get("beta_slow") or 0.0)
    a.mscale = float(s.get("mscale") or 0.0)
    a.mscale_all_dim = float(s.get("mscale_all_dim") or 0.0)
    af = attention_factor if attention_factor is not None else s.get("attention_factor")
    a.attention_factor = float(af) if af is not None else 0.0
    a.original_max_position_embeddings = int(s.get("original_max_position_embeddings") or 0)
    a.truncate = 1 if s.get("truncate", True) else 0
    return a


def cos_sin(client: ComputeClient, out: TensorHandle, base: float = 10000.0, scaling: dict | None = None,
            attention_factor: float | None = None, inv_freq: TensorHandle | None = None, stream=None) -> None:
    """Fill out (compact f32 [P, rot_dim]) with the table, in f64 on the device (see b200_rope_cos_sin)."""
    what = "rope_cos_sin"
    try:
        if out.dtype != "f32" or len(out.shape) != 2 or not out.is_contiguous():
            raise B200Error(6, f"{what}: out must be a compact f32 [P, rot_dim] tensor")
        if inv_freq is not None and (inv_freq.dtype != "f32" or list(inv_freq.shape) != [out.shape[1] // 2]):
            raise B200Error(6, f"{what}: inv_freq must be an f32 [rot_dim / 2] tensor")
        a = table_args(out.shape[1], base, scaling, attention_factor, inv_freq)
        _used_on(stream, out, inv_freq)
        _ffi.check(client._lib.b200_rope_cos_sin(client._ctx, stream, C.byref(a), out.shape[0], _p(out)))
    except B200Error as e:
        client._defer(e)


def cos_sin_alloc(client: ComputeClient, P: int, rot_dim: int, base: float = 10000.0, scaling: dict | None = None,
                  attention_factor: float | None = None, inv_freq: TensorHandle | None = None, stream=None) -> TensorHandle:
    """A new compact f32 [P, rot_dim] table for positions [0, P)."""
    out = TensorHandle.empty_contiguous(client, [P, rot_dim], "f32")
    cos_sin(client, out, base, scaling, attention_factor, inv_freq, stream)
    return out
