"""Token sampling from logits on the GPU: temperature, top-k, min-p and top-p, then a draw reproducible from per-row seeds, in
one launch.  The last step of a decode loop:

    ids = sample_alloc(c, logits, temperature=0.7, top_k=50, top_p=0.9, seed=seeds, offset=steps, advance_offsets=True)
    ids = sample_alloc(c, logits, temperature=0.0)                                  # greedy

logits are [B, V] (f32 / bf16 / f16) with unit column stride and any row stride; ids a compact i32 or i64 [B].  Every
parameter is a number for all rows or a compact per-row TensorHandle (temperature f32, top_k i32, top_p f32, min_p f32,
seed u64, offset u64).  The contract (integer masses, the minimal nucleus, the Philox draw, invalid rows -> -1, batch
invariance) is b200_sample's in include/cubecl_b200.h; kernels in csrc/sample.cu.  Nothing synchronises with the host, and
errors are deferred to client.sync() like every launch.
"""
from __future__ import annotations

import ctypes as C
import numbers

from . import _ffi
from ._ffi import B200Error
from .client import DTYPES, ComputeClient, TensorHandle

# parameter -> (dtypes of its per-row array, args field of the scalar, args field of the array)
PARAMS = {"temperature": (("f32",), "temperature", "temperatures"), "top_k": (("i32",), "top_k", "top_ks"),
          "top_p": (("f32",), "top_p", "top_ps"), "min_p": (("f32",), "min_p", "min_ps"),
          "seed": (("u64", "i64"), "seed", "seeds"), "offset": (("u64", "i64"), "offset", "offsets")}


def _args(what: str, B: int, values: dict, advance_offsets: bool):
    a = _ffi.SampleArgs(temperature=1.0, top_p=1.0)   # the scalars stand in for no row when every row has its array
    used = []
    for name, (dtypes, scalar, array) in PARAMS.items():
        val = values[name]
        if not isinstance(val, numbers.Real):
            if list(val.shape) != [B] or not val.is_contiguous() or val.dtype not in dtypes:
                raise B200Error(6, f"{what}: per-row {name} must be a compact {'/'.join(dtypes)} [{B}] tensor, got {val.dtype} "
                                   f"{list(val.shape)}")
            setattr(a, array, val.handle.ptr)
            used.append(val)
        elif name in ("seed", "offset"):
            setattr(a, scalar, int(val) & 0xFFFFFFFFFFFFFFFF)
        else:
            setattr(a, scalar, int(val) if name == "top_k" else float(val))
    if advance_offsets and isinstance(values["offset"], numbers.Real):
        raise B200Error(6, f"{what}: advance_offsets needs a per-row offset tensor")
    a.advance_offsets = 1 if advance_offsets else 0
    return a, used


def sample(client: ComputeClient, logits: TensorHandle, ids: TensorHandle, temperature=1.0, top_k=0, top_p=1.0, min_p=0.0,
           seed=0, offset=0, advance_offsets: bool = False, stream=None) -> None:
    """ids[r] (i32 / i64 [B]) = the token drawn from row r of logits [B, V] under b200_sample's contract; -1 for an invalid
    row.  advance_offsets adds 1 to each row's entry of the per-row offset tensor after the draw."""
    what = "sample"
    try:
        if len(logits.shape) != 2 or (logits.shape[1] > 1 and logits.strides[1] != 1):
            raise B200Error(6, f"{what}: logits must be a 2-D tensor with unit column stride, got shape {logits.shape} strides "
                               f"{logits.strides}")
        B, V = logits.shape
        if list(ids.shape) != [B] or not ids.is_contiguous() or ids.dtype not in ("i32", "i64"):
            raise B200Error(6, f"{what}: ids must be a compact i32/i64 [{B}] tensor, got {ids.dtype} {list(ids.shape)}")
        a, used = _args(what, B, dict(temperature=temperature, top_k=top_k, top_p=top_p, min_p=min_p, seed=seed,
                                      offset=offset), advance_offsets)
        for th in [logits, ids] + used:
            th.handle.used_on(stream)
        _ffi.check(client._lib.b200_sample(client._ctx, stream, C.byref(a), DTYPES[logits.dtype], DTYPES[ids.dtype], B, V,
                                           C.c_uint64(logits.handle.ptr), logits.strides[0], C.c_uint64(ids.handle.ptr)))
    except B200Error as e:
        client._defer(e)


def sample_alloc(client: ComputeClient, logits: TensorHandle, temperature=1.0, top_k=0, top_p=1.0, min_p=0.0, seed=0,
                 offset=0, advance_offsets: bool = False, ids_dtype: str = "i64") -> TensorHandle:
    """a new compact [B] ids tensor in ids_dtype (i64 by default), written by sample()"""
    B = logits.shape[0] if logits.shape else 0
    ids = TensorHandle.empty_contiguous(client, [B], ids_dtype)
    sample(client, logits, ids, temperature, top_k, top_p, min_p, seed, offset, advance_offsets)
    return ids
