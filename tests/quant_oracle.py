"""numpy oracle of b200_quantize / b200_dequantize: the scale rule, the encodings and the bit layout stated in
include/cubecl_b200.h, in IEEE f32 (numpy float32 arithmetic rounds every operation, and divides with `/`), so the device
results are compared bit for bit.

round_up is ScaleDtype::round_up (crates/cubecl-common/src/quant/scheme.rs:235-270) for F32 / F16 / BF16 / UE4M3; UE8M0, which
the reference leaves unimplemented, is the smallest power of two not below the scale, clamped to codes 0..254.
"""
from __future__ import annotations

import numpy as np

from cubecl_b200 import synth

F32, U32 = np.float32, np.uint32
RANGE = {"q8f": (-128.0, 127.0), "q4f": (-8.0, 7.0), "q2f": (-2.0, 1.0), "q8s": (-127.0, 127.0), "q4s": (-7.0, 7.0),
         "q2s": (-1.0, 1.0), "e4m3": (-448.0, 448.0), "e5m2": (-57344.0, 57344.0), "e2m1": (-6.0, 6.0)}
BITS = {"q8f": 8, "e5m2": 8, "e4m3": 8, "q4f": 4, "e2m1": 4, "q2f": 2, "q8s": 8, "q4s": 4, "q2s": 2}
MAX_REPR = {"f32": F32(np.finfo(np.float32).max), "f16": F32(65504.0), "bf16": U32(0x7F7F0000).view(F32),
            "ue8m0": U32(0x7F000000).view(F32), "ue4m3": F32(448.0)}
BIT_STEP = {"f16": 1 << 13, "bf16": 1 << 16, "ue4m3": 1 << 20}
SUBNORMALS = {"f16": (F32(2.0 ** -14), F32(2.0 ** -24)), "ue4m3": (F32(0.015625), F32(0.001953125))}


def _f32(x) -> np.ndarray:
    return np.asarray(x, dtype=np.float32)


def ue8m0_code(s) -> np.ndarray:
    b = _f32(s).view(U32).astype(np.int64)
    e, m = b >> 23, b & 0x7FFFFF
    return np.where(e == 0, (m > 0x400000).astype(np.int64), np.minimum(e + (m != 0), 254)).astype(np.uint8)


def round_up(dt: str, s) -> np.ndarray:
    """The smallest value of the scale dtype not below s (s >= 0, f32)."""
    s = _f32(s)
    if dt == "f32":
        return s.copy()
    if dt == "ue8m0":
        return synth.ue8m0_to_f32(ue8m0_code(s))
    step = BIT_STEP[dt]
    bits = s.view(U32).astype(np.uint64)
    out = ((bits + (step - 1)) & (0xFFFFFFFF & ~(step - 1))).astype(U32).view(F32)
    if dt in SUBNORMALS:
        min_normal, spacing = SUBNORMALS[dt]
        with np.errstate(invalid="ignore", over="ignore"):
            sub = (np.ceil(s / spacing) * spacing).astype(F32)
        out = np.where(s < min_normal, sub, out)
    out = np.where(s >= MAX_REPR[dt], MAX_REPR[dt], out)
    return np.where(np.isnan(s), s, out).astype(F32)


def scale_store(dt: str, s) -> np.ndarray:
    """The stored representation of scales already on the dtype's grid (exact)."""
    s = _f32(s)
    if dt == "f32":
        return s.copy()
    if dt == "f16":
        return s.astype(np.float16)
    if dt == "bf16":
        return (s.view(U32) >> 16).astype(np.uint16)
    if dt == "ue4m3":
        return fp8_codes(s, "e4m3") & np.uint8(0x7F)
    return ue8m0_code(s)


def scale_load(dt: str, raw) -> np.ndarray:
    """Stored scales as f32; e4m3 with the sign ignored."""
    if dt == "f32":
        return _f32(raw)
    if dt == "f16":
        return np.asarray(raw, dtype=np.float16).astype(F32)
    if dt == "bf16":
        return synth.bf16_bits_to_f32(raw)
    if dt == "ue4m3":
        return synth.fp8_bits_to_f32(np.asarray(raw, dtype=np.uint8) & 0x7F, "f8e4m3")
    return synth.ue8m0_to_f32(raw)


FP8 = {"e4m3": (3, -6, 448.0), "e5m2": (2, -14, 57344.0)}   # mantissa bits, minimum normal exponent, largest finite


def fp8_codes(q, value: str) -> np.ndarray:
    """RNE onto the fp8 grid with satfinite, by scaling to the value's quantum (independent of synth's table search):
    +-inf saturates with its sign, NaN gives 0x7F."""
    mbits, emin, mx = FP8[value]
    q = _f32(q)
    a = np.abs(q.astype(np.float64))
    with np.errstate(divide="ignore", invalid="ignore"):
        e = np.maximum(np.floor(np.log2(np.where(a > 0, a, 1.0))), emin)
        quantum = np.exp2(e - mbits)
        r = np.minimum(np.rint(np.nan_to_num(a / quantum, posinf=1e300)) * quantum, mx)
    table = synth.fp8_bits_to_f32(np.arange(128, dtype=np.uint8), "f8" + value).astype(np.float64)
    finite = np.isfinite(table)
    codes = np.arange(128)[finite]
    code = codes[np.clip(np.searchsorted(table[finite], r), 0, len(codes) - 1)]
    code = code | (np.signbit(q).astype(np.int64) << 7)
    return np.where(np.isnan(q), 0x7F, code).astype(np.uint8)


def e2m1_codes(q) -> np.ndarray:
    """Round to nearest e2m1, ties to the even code, saturating at +-6, by the decision thresholds; NaN gives 0."""
    q = _f32(q)
    a = np.abs(q)
    c = np.select([a <= 0.25, a < 0.75, a <= 1.25, a < 1.75, a <= 2.5, a < 3.5, a <= 5.0], [0, 1, 2, 3, 4, 5, 6], 7)
    c = c | (np.signbit(q).astype(np.int64) << 3)
    return np.where(np.isnan(q), 0, c).astype(np.uint8)


def encode(x, eff, value: str) -> np.ndarray:
    """Codes (unsigned fields, low `bits` bits) of x / eff."""
    x, eff = _f32(x), _f32(eff)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        q = (x / eff).astype(F32)
    if value in ("e4m3", "e5m2"):
        c = fp8_codes(q, value).astype(np.int64)
    elif value == "e2m1":
        c = e2m1_codes(q).astype(np.int64)
    else:
        lo, hi = RANGE[value]
        c = np.where(np.isnan(q), 0, np.clip(np.rint(np.nan_to_num(q, nan=0.0)), lo, hi)).astype(np.int64)
    c = np.where(np.broadcast_to(eff, q.shape) == 0, 0, c)
    return (c & ((1 << BITS[value]) - 1)).astype(np.uint8)


def decode(fields, value: str) -> np.ndarray:
    f = np.asarray(fields, dtype=np.int64)
    if value in ("e4m3", "e5m2"):
        return synth.fp8_bits_to_f32(f.astype(np.uint8), "f8" + value)
    if value == "e2m1":
        return synth.e2m1_codes_to_f32(f.astype(np.uint8))
    sb = 1 << (BITS[value] - 1)
    return ((f ^ sb) - sb).astype(F32)


def pack(fields, bits: int) -> np.ndarray:
    """[..., K] fields -> [..., K * bits / 8] bytes, field i at bit offset i * bits from the low bits upward."""
    f = np.asarray(fields, dtype=np.uint8)
    per = 8 // bits
    g = f.reshape(f.shape[:-1] + (f.shape[-1] // per, per)).astype(np.uint32)
    return np.bitwise_or.reduce(g << (np.arange(per, dtype=np.uint32) * bits), axis=-1).astype(np.uint8)


def unpack(stream, bits: int, K: int) -> np.ndarray:
    b = np.asarray(stream, dtype=np.uint8)
    per = 8 // bits
    f = (b[..., None].astype(np.uint32) >> (np.arange(per, dtype=np.uint32) * bits)) & ((1 << bits) - 1)
    return f.reshape(b.shape[:-1] + (b.shape[-1] * per,))[..., :K].astype(np.uint8)


def words_to_bytes(words) -> np.ndarray:
    """The reference's PackedU32 words as the little-endian byte stream."""
    return np.asarray(words, dtype="<u4").view(np.uint8)


def quantize(x, scheme):
    """(values bytes [..., K * bits / 8], stored block scales [..., K / block] or None, f32 tensor scale or None)."""
    x = _f32(x)
    K = x.shape[-1]
    lo, hi = RANGE[scheme.value]
    hi = F32(hi)
    fin = np.where(np.isfinite(x), np.abs(x), F32(0)).astype(F32)
    tensor = None
    if scheme.has_tensor:
        tensor = F32(F32(fin.max() if fin.size else 0) / hi)
        if scheme.block:
            tensor = F32(tensor / MAX_REPR[scheme.block_scale])
    scales = None
    if scheme.block:
        B, dt = scheme.block, scheme.block_scale
        amax_b = fin.reshape(x.shape[:-1] + (K // B, B)).max(axis=-1)
        with np.errstate(divide="ignore", invalid="ignore"):
            q = (amax_b / hi).astype(F32)
            if tensor is not None:
                q = (q / tensor).astype(F32)
            s = np.where(amax_b == 0, F32(0), round_up(dt, q)).astype(F32)
        scales = scale_store(dt, s)
        eff = (tensor * s).astype(F32) if tensor is not None else s
        eff = np.repeat(eff, B, axis=-1)
    else:
        eff = tensor
    return pack(encode(x, eff, scheme.value), BITS[scheme.value]), scales, tensor


def effective_scale(scheme, K: int, shape_lead, block_scales=None, tensor_scale=None) -> np.ndarray:
    if scheme.block:
        s = scale_load(scheme.block_scale, block_scales).reshape(tuple(shape_lead) + (K // scheme.block,))
        if scheme.has_tensor:
            s = (F32(tensor_scale) * s).astype(F32)
        return np.repeat(s, scheme.block, axis=-1)
    return np.full(tuple(shape_lead) + (K,), F32(tensor_scale), dtype=F32)


def dequantize(values, scheme, shape, block_scales=None, tensor_scale=None, out_dtype: str = "f32") -> np.ndarray:
    """Device representation of out = RNE(f32(q) * eff) in out_dtype (bf16 as uint16 bits)."""
    shape = tuple(shape)
    K = shape[-1]
    q = decode(unpack(np.asarray(values).reshape(shape[:-1] + (-1,)), BITS[scheme.value], K), scheme.value)
    with np.errstate(over="ignore", invalid="ignore"):
        out = (q * effective_scale(scheme, K, shape[:-1], block_scales, tensor_scale)).astype(F32)
    return synth.to_device_dtype(out, out_dtype)
