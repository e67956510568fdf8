"""`reduce::launch` surface (cubek's reduce is out of tree; in-tree semantics: examples/sum_things/src/lib.rs:6-33,
cubecl-book/src/getting-started/src/bin/v1-cpu.rs:7-15).

Reduces one axis (or every element with axis=None) of a tensor (any strides: pitched rows and transposed views are read in
place, only views no stride description fits are compacted first); f32 accumulation; output f32 (values) or
u32 (indices for argmax/argmin: ties -> lowest index, first NaN wins).  Kernels: csrc/reduce.cu.

mean is rne_f32(S * f32(1 / len)) with S the f32 sum: the scale is applied once, to the whole sum, on every path (the
all-elements grid stage, a one-pass axis kernel, the second pass of a split reduction or the end of the fused column finish).
So on values whose partial sums are all exact (integers with sum |x| < 2^24) sum and mean are exact on every path.
"""
from __future__ import annotations

import ctypes as C

from . import _ffi
from ._ffi import B200Error
from .client import ComputeClient, DTYPES, TensorHandle

_IDS_CACHE: dict = {}


def _ids_array(device_ids):
    """(ctypes int array, n) of the sorted device set; cached -- the fused launches sit in 20 us loops."""
    key = tuple(device_ids)
    hit = _IDS_CACHE.get(key)
    if hit is None:
        ids = sorted(int(d) for d in key)
        hit = _IDS_CACHE[key] = (_ffi.int_array(ids), len(ids))
    return hit


OPS = {"sum": _ffi.REDUCE_SUM, "prod": _ffi.REDUCE_PROD, "max": _ffi.REDUCE_MAX, "min": _ffi.REDUCE_MIN,
       "argmax": _ffi.REDUCE_ARGMAX, "argmin": _ffi.REDUCE_ARGMIN, "mean": _ffi.REDUCE_MEAN}


def output_shape(shape, axis) -> list[int]:
    shape = list(shape)
    if axis is None:
        return [1]
    if not -len(shape) <= axis < len(shape):
        raise ValueError(f"axis {axis} out of range for rank {len(shape)}")
    axis %= len(shape)
    return shape[:axis] + shape[axis + 1:] or [1]


def output_dtype(op: str) -> str:
    return "u32" if op in ("argmax", "argmin") else "f32"


def launch(client: ComputeClient, input: TensorHandle, output: TensorHandle, axis, op: str = "sum", stream=None) -> None:
    """Enqueue the reduction on the client's stream; errors are deferred to sync()/read_one()."""
    try:
        if op not in OPS:
            raise B200Error(6, f"unknown reduce op {op!r}")
        if output.dtype != output_dtype(op):
            raise B200Error(6, f"reduce: output dtype must be {output_dtype(op)} for op {op}")
        rank = len(input.shape)
        ax = -1 if axis is None else axis % rank
        input.handle.used_on(stream)
        output.handle.used_on(stream)
        if not output.is_contiguous():
            raise B200Error(7, "reduce: output must be contiguous")
        # pitched / permuted inputs are reduced in place by the library (strides + row pitch go to the kernels)
        _ffi.check(client._lib.b200_reduce_strided(client._ctx, stream, OPS[op], DTYPES[input.dtype], C.c_uint64(input.handle.ptr),
                                                   C.c_uint64(output.handle.ptr), rank, _ffi.u64_array(input.shape),
                                                   _ffi.u64_array(input.strides), ax))
    except B200Error as e:
        client._defer(e)


def launch_alloc(client: ComputeClient, input: TensorHandle, axis, op: str = "sum") -> TensorHandle:
    out = TensorHandle.empty_contiguous(client, output_shape(input.shape, axis), output_dtype(op))
    launch(client, input, out, axis, op)
    return out


def launch_all_reduce(client: ComputeClient, input: TensorHandle, output: TensorHandle, device_ids) -> None:
    """Sum of every element of `input` on every rank of `device_ids`, summed over ranks, written to output[0] on each rank:
    `reduce::launch` followed by `client.all_reduce(.., Sum)` (client.rs:790) as ONE kernel -- the grid stage of the
    reduce exchanges the per-rank scalar through NVLink peer memory (csrc/reduce.cu, XgpuParams).  Collective call."""
    try:
        if input.dtype != "f32" or output.dtype != "f32":
            raise B200Error(7, "launch_all_reduce: f32 in, f32 out")
        if not input.is_contiguous():
            raise B200Error(7, "launch_all_reduce: input must be contiguous")
        ids, n_ids = _ids_array(device_ids)
        _ffi.check(client._lib.b200_reduce_all_reduce(client._ctx, None, _ffi.REDUCE_SUM, DTYPES["f32"], C.c_uint64(input.handle.ptr),
                                                      C.c_uint64(output.handle.ptr), input.size(), ids, n_ids))
    except B200Error as e:
        client._defer(e)


def launch_arg_all_reduce(client: ComputeClient, input: TensorHandle, output: TensorHandle, device_ids, index_offset: int,
                          op: str = "argmax") -> None:
    """Global argmax/argmin over the concatenation of every rank's `input` (outer-axis shards): output[0] (u32) = global
    index on every rank.  One kernel per rank; the (value, index) pairs travel through the NVLink mailboxes."""
    try:
        if op not in ("argmax", "argmin"):
            raise B200Error(6, "launch_arg_all_reduce: op must be argmax or argmin")
        if input.dtype != "f32" or output.dtype != "u32" or not input.is_contiguous():
            raise B200Error(7, "launch_arg_all_reduce: contiguous f32 in, u32 out")
        ids, n_ids = _ids_array(device_ids)
        _ffi.check(client._lib.b200_argreduce_all_reduce(client._ctx, None, OPS[op], DTYPES["f32"], C.c_uint64(input.handle.ptr),
                                                         C.c_uint64(output.handle.ptr), input.size(), int(index_offset), ids, n_ids))
    except B200Error as e:
        client._defer(e)
