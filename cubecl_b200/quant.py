"""Quantize / dequantize along the innermost axis under CubeCL's quantization schemes
(crates/cubecl-common/src/quant/scheme.rs: QuantScheme, QuantValue, ScaleDtype; the NVFP4 preset of presets.rs).

`quantize(client, x, scheme)` turns an f32 / f16 / bf16 tensor [..., K] into codes plus scales; `dequantize(client, q,
out_dtype)` reads them back as f32 / f16 / bf16.  The codes of the minifloat schemes carry the dtypes the block-scaled matmul
takes, so `matmul.launch_scaled(client, qa.values, qb.values, qa.block_scales, qb.block_scales, out, scale_block=...)` runs
on quantized operands directly (MXFP8, MXFP4, and the one-level E2M1 / 16 / ue4m3 scheme with scale_block=16).  Layout,
scale rule and encoding are stated in include/cubecl_b200.h (b200_quantize).  Kernels: csrc/quant.cu.

The two-level `nvfp4()` preset also stores a per-tensor f32 scale g; b200_matmul_scaled has no alpha, so a caller
multiplying two such operands multiplies the result by g_a * g_b itself.
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass, replace

from . import _ffi
from ._ffi import B200Error
from .client import ComputeClient, DTYPES, TensorHandle

# QuantValue, in the reference's order (b200_quant_value)
VALUES = {"q8f": _ffi.QV_Q8F, "e5m2": _ffi.QV_E5M2, "e4m3": _ffi.QV_E4M3, "q4f": _ffi.QV_Q4F, "e2m1": _ffi.QV_E2M1,
          "q2f": _ffi.QV_Q2F, "q8s": _ffi.QV_Q8S, "q4s": _ffi.QV_Q4S, "q2s": _ffi.QV_Q2S}
BITS = {"q8f": 8, "e5m2": 8, "e4m3": 8, "q4f": 4, "e2m1": 4, "q2f": 2, "q8s": 8, "q4s": 4, "q2s": 2}
# ScaleDtype -> the tensor dtype its scales are stored in (ue4m3 is an e4m3 byte with the sign clear)
SCALE_DTYPES = {"f32": "f32", "f16": "f16", "bf16": "bf16", "ue8m0": "ue8m0", "ue4m3": "f8e4m3"}
# the dtype the codes travel in: minifloats as the matmul's operand dtypes, integers as bytes
VALUE_DTYPES = {"e4m3": "f8e4m3", "e5m2": "f8e5m2", "e2m1": "f4e2m1x2", "q8f": "i8", "q8s": "i8"}


@dataclass(frozen=True)
class QuantScheme:
    """QuantScheme with the reference's builder names.  A scheme with no level resolves to per-tensor f32, as
    QuantScheme::tensor_scale does (scheme.rs:94-104)."""
    value: str = "q8f"
    block: int = 0                   # values per block scale along the innermost axis; 0 = no block level
    block_scale: str | None = None   # ScaleDtype of the block level: f32, f16, bf16, ue8m0, ue4m3
    tensor: bool = False             # the per-tensor f32 level

    def with_value(self, value: str) -> "QuantScheme":
        return replace(self, value=value)

    def per_block(self, block: int, dtype: str) -> "QuantScheme":
        return replace(self, block=int(block), block_scale=dtype)

    def per_tensor(self, dtype: str = "f32") -> "QuantScheme":
        if dtype != "f32":
            raise B200Error(7, f"per-tensor scales are stored as f32, not {dtype}")
        return replace(self, tensor=True)

    @staticmethod
    def mxfp8() -> "QuantScheme":
        return QuantScheme().with_value("e4m3").per_block(32, "ue8m0")

    @staticmethod
    def mxfp4() -> "QuantScheme":
        return QuantScheme().with_value("e2m1").per_block(32, "ue8m0")

    @staticmethod
    def nvfp4() -> "QuantScheme":
        """The reference's NVFP4 preset (presets.rs:6-12): e2m1 in blocks of 16 with ue4m3 block scales normalised by one
        per-tensor f32 scale g.  b200_matmul_scaled reads the block scales; the caller multiplies its result by g_a * g_b."""
        return QuantScheme().per_block(16, "ue4m3").per_tensor().with_value("e2m1")

    @property
    def has_tensor(self) -> bool:
        return self.tensor or self.block == 0

    @property
    def bits(self) -> int:
        return BITS[self.value]

    def to_c(self) -> _ffi.QuantScheme:
        if self.value not in VALUES:
            raise B200Error(6, f"unknown quant value {self.value!r} ({', '.join(VALUES)})")
        if self.block and self.block_scale not in SCALE_DTYPES:
            raise B200Error(6, f"unknown block-scale dtype {self.block_scale!r} ({', '.join(SCALE_DTYPES)})")
        dt = DTYPES[SCALE_DTYPES[self.block_scale]] if self.block else _ffi.F32
        return _ffi.QuantScheme(VALUES[self.value], int(self.block), dt, 1 if self.has_tensor else 0)


@dataclass
class QuantizedTensor:
    values: TensorHandle                 # codes [..., K * bits / 8] bytes (f8e4m3 / f8e5m2 / f4e2m1x2 / i8 / u8)
    block_scales: TensorHandle | None    # [..., K / block] in the block-scale dtype
    tensor_scale: TensorHandle | None    # f32 [1]
    scheme: QuantScheme
    shape: list


def _ptr(t: TensorHandle | None) -> C.c_uint64:
    return C.c_uint64(t.handle.ptr if t is not None else 0)


def alloc_quantized(client: ComputeClient, shape, scheme: QuantScheme) -> QuantizedTensor:
    """Allocate the compact outputs of quantize(x of `shape`, scheme)."""
    shape = [int(s) for s in shape]
    lead, K = shape[:-1], shape[-1] if shape else 0
    vdt = VALUE_DTYPES.get(scheme.value, "u8")
    values = TensorHandle.empty_contiguous(client, lead + [K * scheme.bits // 8], vdt)
    scales = None
    if scheme.block:
        scales = TensorHandle.empty_contiguous(client, lead + [K // scheme.block], SCALE_DTYPES.get(scheme.block_scale, "u8"))
    tensor = TensorHandle.empty_contiguous(client, [1], "f32") if scheme.has_tensor else None
    return QuantizedTensor(values, scales, tensor, scheme, shape)


def launch_quantize(client: ComputeClient, x: TensorHandle, q: QuantizedTensor, stream=None) -> None:
    """Enqueue the quantization of `x` into the buffers of `q`; errors are deferred to sync()/read_one()."""
    try:
        if x.dtype not in ("f32", "f16", "bf16"):
            raise B200Error(6, f"quantize: input dtype {x.dtype} is not f32, f16 or bf16")
        if list(q.shape) != list(x.shape):
            raise B200Error(6, f"quantize: output shape {q.shape} != input shape {x.shape}")
        s = q.scheme.to_c()
        for t in (x, q.values, q.block_scales, q.tensor_scale):
            if t is not None:
                t.handle.used_on(stream)
        _ffi.check(client._lib.b200_quantize(client._ctx, stream, C.byref(s), DTYPES[x.dtype], C.c_uint64(x.handle.ptr),
                                             _ptr(q.values), _ptr(q.block_scales), _ptr(q.tensor_scale), len(x.shape),
                                             _ffi.u64_array(x.shape), _ffi.u64_array(x.strides)))
    except B200Error as e:
        client._defer(e)


def quantize(client: ComputeClient, x: TensorHandle, scheme: QuantScheme, stream=None) -> QuantizedTensor:
    q = alloc_quantized(client, x.shape, scheme)
    launch_quantize(client, x, q, stream)
    return q


def launch_dequantize(client: ComputeClient, q: QuantizedTensor, out: TensorHandle, stream=None) -> None:
    """Enqueue out = dequantize(q) (compact, f32 / f16 / bf16); errors are deferred to sync()/read_one()."""
    try:
        if list(out.shape) != list(q.shape) or not out.is_contiguous():
            raise B200Error(6, f"dequantize: output must be contiguous with shape {q.shape}")
        s = q.scheme.to_c()
        for t in (q.values, q.block_scales, q.tensor_scale, out):
            if t is not None:
                t.handle.used_on(stream)
        _ffi.check(client._lib.b200_dequantize(client._ctx, stream, C.byref(s), DTYPES[out.dtype], _ptr(q.values),
                                               _ptr(q.block_scales), _ptr(q.tensor_scale), C.c_uint64(out.handle.ptr),
                                               len(q.shape), _ffi.u64_array(q.shape)))
    except B200Error as e:
        client._defer(e)


def dequantize(client: ComputeClient, q: QuantizedTensor, out_dtype: str = "f32", stream=None) -> TensorHandle:
    out = TensorHandle.empty_contiguous(client, q.shape, out_dtype)
    launch_dequantize(client, q, out, stream)
    return out


def values_bytes(shape, scheme: QuantScheme) -> int:
    """Bytes of the codes of a tensor of `shape` (the algorithmic write of quantize)."""
    return math.prod(shape) * scheme.bits // 8
