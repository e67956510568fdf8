"""Cumulative scans along one axis: cumsum / cumprod / cummax / cummin, inclusive or exclusive -- the device-wide form of
the reference's plane scans (crates/cubecl-core/src/runtime_tests/plane.rs:191-405).

The output has the input's shape, is compact row-major and is f32 or the input's dtype (a 16-bit output is the f32 running
value rounded to nearest-even once).  Inputs of any strides: contiguous tensors and pitched rows are read in place, other
views are compacted first.  max / min: a NaN makes every later output NaN.  Kernels: csrc/reduce.cu (scan_rows_*,
scan_cols_*).
"""
from __future__ import annotations

import ctypes as C

from . import _ffi
from ._ffi import B200Error
from .client import ComputeClient, DTYPES, TensorHandle

OPS = {"sum": _ffi.REDUCE_SUM, "prod": _ffi.REDUCE_PROD, "max": _ffi.REDUCE_MAX, "min": _ffi.REDUCE_MIN}


def launch(client: ComputeClient, input: TensorHandle, output: TensorHandle, axis: int, op: str = "sum", exclusive: bool = False,
           stream=None) -> None:
    """Enqueue the scan of `axis` on the client's stream (or `stream`); errors are deferred to sync()/read_one()."""
    try:
        if op not in OPS:
            raise B200Error(6, f"unknown scan op {op!r} (sum, prod, max, min)")
        rank = len(input.shape)
        if not -rank <= axis < rank:
            raise B200Error(6, f"scan: axis {axis} out of range for rank {rank}")
        if list(output.shape) != list(input.shape):
            raise B200Error(6, f"scan: output shape {list(output.shape)} != input shape {list(input.shape)}")
        if not output.is_contiguous():
            raise B200Error(7, "scan: output must be contiguous")
        input.handle.used_on(stream)
        output.handle.used_on(stream)
        _ffi.check(client._lib.b200_scan(client._ctx, stream, OPS[op], 1 if exclusive else 0, DTYPES[input.dtype], DTYPES[output.dtype],
                                         C.c_uint64(input.handle.ptr), C.c_uint64(output.handle.ptr), rank,
                                         _ffi.u64_array(input.shape), _ffi.u64_array(input.strides), axis % rank))
    except B200Error as e:
        client._defer(e)


def launch_alloc(client: ComputeClient, input: TensorHandle, axis: int, op: str = "sum", exclusive: bool = False,
                 out_dtype: str = "f32") -> TensorHandle:
    out = TensorHandle.empty_contiguous(client, input.shape, out_dtype)
    launch(client, input, out, axis, op, exclusive)
    return out
