"""Mixture-of-experts routing on the GPU: top-k gating, the expert-sorted dispatch plan the grouped matmuls take, the row
gather into expert order, and the weighted combine with its backward.  A layer:

    ids, weights = route_alloc(c, logits, k)            # [T, k] i32 / f32
    offs, row_of, slot_of = plan_alloc(c, ids, E)       # offs i32 [E], row_of i32 [T, k], slot_of i32 [T * k]
    xs = permute_alloc(c, x, slot_of, k)                # [T * k, K], rows in expert order
    ys = matmul.launch_grouped_alloc(c, xs, w, offs)    # (and its activation, the second grouped matmul, ...)
    y = combine_alloc(c, ys, row_of, weights)           # [T, N]

Nothing synchronises with the host.  Rows of xs / ys past the kept count (offs[-1]) are not written.  The contracts (order of
selection, ties, NaN, summation orders, refusals) are those of b200_moe_* in include/cubecl_b200.h.  Kernels: csrc/moe.cu.
Errors are deferred to client.sync() like every launch.
"""
from __future__ import annotations

import ctypes as C

from . import _ffi
from ._ffi import B200Error
from .client import DTYPE_SIZE, DTYPES, ComputeClient, TensorHandle

SCORES = {"softmax": _ffi.MOE_SOFTMAX, "sigmoid": _ffi.MOE_SIGMOID}


def _rows(t: TensorHandle, what: str, name: str) -> None:
    """A 2-D tensor with unit column stride (any row stride)."""
    if len(t.shape) != 2 or (t.shape[1] > 1 and t.strides[1] != 1):
        raise B200Error(6, f"{what}: {name} must be a 2-D tensor with unit column stride, got shape {t.shape} strides {t.strides}")


def _index(t: TensorHandle, what: str, name: str, shape: list[int], dtype: str = "i32") -> None:
    if t.dtype != dtype or list(t.shape) != list(shape) or not t.is_contiguous():
        raise B200Error(6, f"{what}: {name} must be a compact {dtype} {shape} tensor, got {t.dtype} {list(t.shape)}")


def route(client: ComputeClient, logits: TensorHandle, ids: TensorHandle, weights: TensorHandle, k: int, score: str = "softmax",
          renormalize: bool = True, n_group: int = 0, topk_group: int = 0, scale: float = 1.0, bias: TensorHandle | None = None,
          stream=None) -> None:
    """Top-k gating of logits [T, E] (f32 / bf16 / f16) into ids i32 [T, k] and weights f32 [T, k].  score "softmax" or
    "sigmoid"; bias: an optional f32 [E] selection bias; n_group > 1 with topk_group: group-limited routing (DeepSeek-V3)."""
    what = "moe_route"
    try:
        _rows(logits, what, "logits")
        T, E = logits.shape
        if score not in SCORES:
            raise B200Error(6, f"{what}: unknown score {score!r} (softmax, sigmoid)")
        _index(ids, what, "ids", [T, k])
        _index(weights, what, "weights", [T, k], "f32")
        if bias is not None:
            _index(bias, what, "bias", [E], "f32")
        args = _ffi.MoeRouteArgs(int(k), SCORES[score], 1 if renormalize else 0, int(n_group), int(topk_group), float(scale))
        for th in (logits, ids, weights) + ((bias,) if bias is not None else ()):
            th.handle.used_on(stream)
        _ffi.check(client._lib.b200_moe_route(client._ctx, stream, DTYPES[logits.dtype], C.c_uint64(logits.handle.ptr), T, E,
                                              logits.strides[0], C.c_uint64(bias.handle.ptr if bias is not None else 0),
                                              C.byref(args), C.c_uint64(ids.handle.ptr), C.c_uint64(weights.handle.ptr)))
    except B200Error as e:
        client._defer(e)


def route_alloc(client: ComputeClient, logits: TensorHandle, k: int, **kw) -> tuple[TensorHandle, TensorHandle]:
    T = logits.shape[0] if logits.shape else 0
    ids = TensorHandle.empty_contiguous(client, [T, k], "i32")
    weights = TensorHandle.empty_contiguous(client, [T, k], "f32")
    route(client, logits, ids, weights, k, **kw)
    return ids, weights


def plan(client: ComputeClient, ids: TensorHandle, num_experts: int, offs: TensorHandle, row_of: TensorHandle,
         slot_of: TensorHandle, stream=None) -> None:
    """The dispatch plan of ids i32 [T, k]: offs i32 [E] (cumulative ends), row_of i32 [T, k] (sorted row of each slot, -1 when
    the id is outside [0, E)) and slot_of i32 [T * k] (slot of each sorted row, -1 past the kept count).  Stable: torch's
    argsort(ids.flatten(), stable=True) without the dropped slots."""
    what = "moe_plan"
    try:
        if ids.dtype != "i32" or len(ids.shape) != 2 or not ids.is_contiguous():
            raise B200Error(6, f"{what}: ids must be a compact i32 [T, k] tensor")
        T, k = ids.shape
        _index(offs, what, "offs", [num_experts])
        _index(row_of, what, "row_of", [T, k])
        _index(slot_of, what, "slot_of", [T * k])
        for th in (ids, offs, row_of, slot_of):
            th.handle.used_on(stream)
        _ffi.check(client._lib.b200_moe_plan(client._ctx, stream, C.c_uint64(ids.handle.ptr), T, k, num_experts,
                                             C.c_uint64(offs.handle.ptr), C.c_uint64(row_of.handle.ptr),
                                             C.c_uint64(slot_of.handle.ptr)))
    except B200Error as e:
        client._defer(e)


def plan_alloc(client: ComputeClient, ids: TensorHandle, num_experts: int) -> tuple[TensorHandle, TensorHandle, TensorHandle]:
    T, k = (list(ids.shape) + [0, 0])[:2]
    offs = TensorHandle.empty_contiguous(client, [num_experts], "i32")
    row_of = TensorHandle.empty_contiguous(client, [T, k], "i32")
    slot_of = TensorHandle.empty_contiguous(client, [T * k], "i32")
    plan(client, ids, num_experts, offs, row_of, slot_of)
    return offs, row_of, slot_of


def permute(client: ComputeClient, src: TensorHandle, slot_of: TensorHandle, k: int, dst: TensorHandle, stream=None) -> None:
    """dst[r] = src[slot_of[r] // k] for every sorted row r with a slot: src [T, C] and dst [T * k, C] of one dtype (any dtype:
    activations, fp8 codes, block scales), unit column stride, any row pitch.  Rows without a slot are not written."""
    what = "moe_permute"
    try:
        _rows(src, what, "src")
        _rows(dst, what, "dst")
        T, cols = src.shape
        if dst.dtype != src.dtype or list(dst.shape) != [T * k, cols]:
            raise B200Error(6, f"{what}: dst must be {src.dtype} [{T * k}, {cols}], got {dst.dtype} {list(dst.shape)}")
        _index(slot_of, what, "slot_of", [T * k])
        esz = DTYPE_SIZE[src.dtype]
        for th in (src, slot_of, dst):
            th.handle.used_on(stream)
        _ffi.check(client._lib.b200_moe_permute(client._ctx, stream, C.c_uint64(src.handle.ptr), src.strides[0] * esz,
                                                C.c_uint64(slot_of.handle.ptr), T, k, C.c_uint64(dst.handle.ptr),
                                                dst.strides[0] * esz, cols * esz))
    except B200Error as e:
        client._defer(e)


def permute_alloc(client: ComputeClient, src: TensorHandle, slot_of: TensorHandle, k: int) -> TensorHandle:
    dst = TensorHandle.empty_contiguous(client, [src.shape[0] * k, src.shape[1] if len(src.shape) > 1 else 0], src.dtype)
    permute(client, src, slot_of, k, dst)
    return dst


def combine(client: ComputeClient, ys: TensorHandle, row_of: TensorHandle, y: TensorHandle, weights: TensorHandle | None = None,
            stream=None) -> None:
    """y[t] = sum_j weights[t, j] * ys[row_of[t, j]] (fma in increasing j, one rounding), or the plain sum without weights (the
    permute's backward).  ys [R, N] and y [T, N] in f32 / bf16 / f16 independently, unit column stride."""
    what = "moe_combine"
    try:
        _rows(ys, what, "ys")
        _rows(y, what, "y")
        if len(row_of.shape) != 2:
            raise B200Error(6, f"{what}: row_of must be a compact i32 [T, k] tensor")
        T, k = row_of.shape
        _index(row_of, what, "row_of", [T, k])
        if y.shape != [T, ys.shape[1]]:
            raise B200Error(6, f"{what}: y must be [{T}, {ys.shape[1]}], got {y.shape}")
        if weights is not None:
            _index(weights, what, "weights", [T, k], "f32")
        for th in (ys, row_of, y) + ((weights,) if weights is not None else ()):
            th.handle.used_on(stream)
        _ffi.check(client._lib.b200_moe_combine(client._ctx, stream, DTYPES[ys.dtype], DTYPES[y.dtype], C.c_uint64(ys.handle.ptr),
                                                ys.shape[0], ys.strides[0],
                                                C.c_uint64(weights.handle.ptr if weights is not None else 0),
                                                C.c_uint64(row_of.handle.ptr), T, k, ys.shape[1], C.c_uint64(y.handle.ptr),
                                                y.strides[0]))
    except B200Error as e:
        client._defer(e)


def combine_alloc(client: ComputeClient, ys: TensorHandle, row_of: TensorHandle, weights: TensorHandle | None = None,
                  out_dtype: str | None = None) -> TensorHandle:
    y = TensorHandle.empty_contiguous(client, [row_of.shape[0], ys.shape[1]], out_dtype or ys.dtype)
    combine(client, ys, row_of, y, weights)
    return y


def combine_backward(client: ComputeClient, dy: TensorHandle, ys: TensorHandle, weights: TensorHandle, row_of: TensorHandle,
                     d_ys: TensorHandle, d_w: TensorHandle, stream=None) -> None:
    """Gradients of combine with weights: d_ys[row_of[t, j]] = weights[t, j] * dy[t] (rows no slot references are not written)
    and d_w[t, j] = dot(dy[t], ys[row_of[t, j]]) (+0 for a dropped slot).  dy [T, N] and d_ys [R, N] share one dtype."""
    what = "moe_combine_backward"
    try:
        for t, name in ((dy, "dy"), (ys, "ys"), (d_ys, "d_ys")):
            _rows(t, what, name)
        if len(row_of.shape) != 2:
            raise B200Error(6, f"{what}: row_of must be a compact i32 [T, k] tensor")
        T, k = row_of.shape
        _index(row_of, what, "row_of", [T, k])
        _index(weights, what, "weights", [T, k], "f32")
        _index(d_w, what, "d_w", [T, k], "f32")
        if dy.shape != [T, ys.shape[1]] or d_ys.shape != ys.shape or d_ys.dtype != dy.dtype:
            raise B200Error(6, f"{what}: dy must be [{T}, {ys.shape[1]}] and d_ys {ys.shape} in dy's dtype")
        for th in (dy, ys, weights, row_of, d_ys, d_w):
            th.handle.used_on(stream)
        _ffi.check(client._lib.b200_moe_combine_backward(
            client._ctx, stream, DTYPES[dy.dtype], DTYPES[ys.dtype], C.c_uint64(dy.handle.ptr), dy.strides[0],
            C.c_uint64(ys.handle.ptr), ys.shape[0], ys.strides[0], C.c_uint64(weights.handle.ptr), C.c_uint64(row_of.handle.ptr),
            T, k, ys.shape[1], C.c_uint64(d_ys.handle.ptr), d_ys.strides[0], C.c_uint64(d_w.handle.ptr)))
    except B200Error as e:
        client._defer(e)


def combine_backward_alloc(client: ComputeClient, dy: TensorHandle, ys: TensorHandle, weights: TensorHandle,
                           row_of: TensorHandle) -> tuple[TensorHandle, TensorHandle]:
    d_ys = TensorHandle.empty_contiguous(client, list(ys.shape), dy.dtype)
    d_w = TensorHandle.empty_contiguous(client, list(row_of.shape), "f32")
    combine_backward(client, dy, ys, weights, row_of, d_ys, d_w)
    return d_ys, d_w
