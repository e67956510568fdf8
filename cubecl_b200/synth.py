"""Host mirror of the device generators in csrc/aux_kernels.cu plus bf16 bit helpers.

The counter hash lets bench/tests create operands directly in HBM and still know every value on the host
(SURVEY §8d: "generator = counter-based hash so host and device can regenerate identically without PCIe traffic").
Pure numpy; used by tests and bench only.
"""
from __future__ import annotations

import numpy as np

_M64 = np.uint64(0xFFFFFFFFFFFFFFFF)


def hash_u32(seed: int, idx: np.ndarray) -> np.ndarray:
    """splitmix64 finaliser over (seed, index) -> high 32 bits; mirrors hash_u32() in aux_kernels.cu."""
    with np.errstate(over="ignore"):
        z = (np.uint64(seed) * np.uint64(0x9E3779B97F4A7C15) + idx.astype(np.uint64) + np.uint64(0x632BE59BD9B4E019))
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
    return (z >> np.uint64(32)).astype(np.uint32)


def uniform_f32(seed: int, n: int, lo: float, hi: float, start: int = 0) -> np.ndarray:
    """lo + u * (hi - lo) with u = (hash >> 8) * 2^-24, each op rounded to f32 (no FMA) like the device kernel."""
    idx = np.arange(start, start + n, dtype=np.uint64)
    u = (hash_u32(seed, idx) >> np.uint32(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)
    scale = np.float32(np.float32(hi) - np.float32(lo))
    return (np.float32(lo) + (u * scale).astype(np.float32)).astype(np.float32)


def uniform_at(seed: int, idx: np.ndarray, lo: float, hi: float) -> np.ndarray:
    u = (hash_u32(seed, np.asarray(idx, dtype=np.uint64)) >> np.uint32(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)
    scale = np.float32(np.float32(hi) - np.float32(lo))
    return (np.float32(lo) + (u * scale).astype(np.float32)).astype(np.float32)


def f32_to_bf16_bits(x: np.ndarray) -> np.ndarray:
    """Round-to-nearest-even f32 -> bf16 bit patterns (uint16); NaN stays NaN. Mirrors __float2bfloat16_rn."""
    b = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    rounding = ((b >> np.uint32(16)) & np.uint32(1)) + np.uint32(0x7FFF)
    out = ((b + rounding) >> np.uint32(16)).astype(np.uint16)
    nan = np.isnan(x)
    if np.any(nan):
        out = np.where(nan, np.uint16(0x7FC0), out)
    return out


def bf16_bits_to_f32(bits: np.ndarray) -> np.ndarray:
    return (np.ascontiguousarray(bits, dtype=np.uint16).astype(np.uint32) << np.uint32(16)).view(np.float32)


def _fp8_table(kind: str) -> np.ndarray:
    """f32 value of every fp8 code (OCP e4m3fn: bias 7, no inf, NaN = 0x7F/0xFF; e5m2: bias 15, IEEE-like)."""
    codes = np.arange(256, dtype=np.uint32)
    sign = np.where(codes & 0x80, -1.0, 1.0)
    with np.errstate(over="ignore", invalid="ignore"):
        if kind == "f8e4m3":
            e, m, bias = (codes >> 3) & 0xF, codes & 0x7, 7
            val = np.where(e == 0, m / 8.0 * 2.0 ** (1 - bias), (1 + m / 8.0) * 2.0 ** (e.astype(np.float64) - bias))
            val = np.where((e == 15) & (m == 7), np.nan, val)
        else:
            e, m, bias = (codes >> 2) & 0x1F, codes & 0x3, 15
            val = np.where(e == 0, m / 4.0 * 2.0 ** (1 - bias), (1 + m / 4.0) * 2.0 ** (e.astype(np.float64) - bias))
            val = np.where(e == 31, np.where(m == 0, np.inf, np.nan), val)
    return (sign * val).astype(np.float32)


def fp8_bits_to_f32(bits: np.ndarray, kind: str) -> np.ndarray:
    return _fp8_table(kind)[np.ascontiguousarray(bits, dtype=np.uint8)]


def f32_to_fp8_bits(x: np.ndarray, kind: str) -> np.ndarray:
    """Round-to-nearest-even, saturating to the largest finite value (mirrors __nv_cvt_float_to_fp8(.., __NV_SATFINITE, ..));
    +-inf saturates with its sign, NaN of either sign gives 0x7F."""
    table = _fp8_table(kind).astype(np.float64)
    pos_codes = np.array([c for c in range(128) if np.isfinite(table[c])], dtype=np.int64)   # ascending magnitudes
    pos_vals = table[pos_codes]
    xf = np.ascontiguousarray(x, dtype=np.float32)
    a = np.abs(xf.astype(np.float64))
    hi = np.clip(np.searchsorted(pos_vals, a, side="left"), 0, len(pos_vals) - 1)
    lo = np.clip(hi - 1, 0, len(pos_vals) - 1)
    d_lo, d_hi = np.abs(a - pos_vals[lo]), np.abs(pos_vals[hi] - a)
    pick_hi = (d_hi < d_lo) | ((d_hi == d_lo) & (pos_codes[hi] % 2 == 0))   # ties -> even mantissa
    code = np.where(pick_hi, pos_codes[hi], pos_codes[lo])
    code = np.where(a >= pos_vals[-1], pos_codes[-1], code)                     # saturate (incl. inf)
    sign = np.signbit(xf).astype(np.int64) << 7
    return np.where(np.isnan(a), 0x7F, code | sign).astype(np.uint8)


# ---- MX formats (block-scaled matmul): e2m1 (fp4) packed two per byte, ue8m0 scales
E2M1_VALUES = np.array([0.0, 0.5, 1.0, 1.5, 2.0, 3.0, 4.0, 6.0], dtype=np.float32)   # magnitude of code & 7; bit 3 = sign


def e2m1_codes_to_f32(codes: np.ndarray) -> np.ndarray:
    codes = np.asarray(codes, dtype=np.uint8)
    v = E2M1_VALUES[codes & 7]
    return np.where(codes & 8, -v, v).astype(np.float32)


def f32_to_e2m1_codes(x: np.ndarray) -> np.ndarray:
    """Round to nearest (ties to the even code), saturating at +-6 (+-inf included); NaN gives code 0."""
    xf = np.ascontiguousarray(x, dtype=np.float32)
    a = np.minimum(np.abs(xf.astype(np.float64)), 6.0)
    hi = np.clip(np.searchsorted(E2M1_VALUES.astype(np.float64), a, side="left"), 0, 7)
    lo = np.clip(hi - 1, 0, 7)
    d_lo, d_hi = np.abs(a - E2M1_VALUES[lo]), np.abs(E2M1_VALUES[hi] - a)
    code = np.where((d_hi < d_lo) | ((d_hi == d_lo) & (hi % 2 == 0)), hi, lo)
    return np.where(np.isnan(xf), 0, code | (np.signbit(xf).astype(np.int64) << 3)).astype(np.uint8)


def pack_e2m1x2(codes: np.ndarray) -> np.ndarray:
    """[.., K] 4-bit codes -> [.., K/2] bytes, element 2i in the low nibble (e2m1x2::from_f32_slice, cubecl-common/src/float/fp4.rs:204-216)."""
    codes = np.asarray(codes, dtype=np.uint8)
    assert codes.shape[-1] % 2 == 0
    return (codes[..., 0::2] & 0xF) | ((codes[..., 1::2] & 0xF) << 4)


def unpack_e2m1x2(packed: np.ndarray) -> np.ndarray:
    packed = np.asarray(packed, dtype=np.uint8)
    out = np.empty(packed.shape[:-1] + (packed.shape[-1] * 2,), dtype=np.uint8)
    out[..., 0::2] = packed & 0xF
    out[..., 1::2] = packed >> 4
    return out


def ue8m0_to_f32(bits: np.ndarray) -> np.ndarray:
    """2^(bits - 127); 255 is NaN (ue8m0, cubecl-common float module)."""
    b = np.asarray(bits, dtype=np.uint8).astype(np.int64)
    return np.where(b == 255, np.nan, np.ldexp(1.0, b - 127)).astype(np.float32)


def pack_scale_chunks(scales: np.ndarray, pad: int = 127) -> np.ndarray:
    """[rows, n_scales] scale bytes -> the tensor core's packed chunks [ceil(rows/128)][ceil(n_scales/4)][512]:
    byte (r % 32) * 16 + (r / 32) * 4 + s; padding = 1.0 (127 for ue8m0, 0x38 for ue4m3).  The scales_packed = 1 input layout
    of b200_matmul_scaled."""
    scales = np.asarray(scales, dtype=np.uint8)
    rows, ns = scales.shape
    tiles, atoms = (rows + 127) // 128, (ns + 3) // 4
    padded = np.full((tiles * 128, atoms * 4), pad, dtype=np.uint8)
    padded[:rows, :ns] = scales
    v = padded.reshape(tiles, 4, 32, atoms, 4)          # [tile][g = r/32][r%32][atom][s]
    return np.ascontiguousarray(v.transpose(0, 3, 2, 1, 4)).reshape(tiles, atoms, 512)   # [tile][atom][r%32][g][s]


def to_device_dtype(x_f32: np.ndarray, dtype: str) -> np.ndarray:
    """f32 values -> array in the device representation of `dtype` (bf16 as uint16 bits)."""
    if dtype == "f32":
        return np.ascontiguousarray(x_f32, dtype=np.float32)
    if dtype == "f16":
        return np.ascontiguousarray(x_f32, dtype=np.float32).astype(np.float16)
    if dtype == "bf16":
        return f32_to_bf16_bits(x_f32)
    if dtype in ("f8e4m3", "f8e5m2"):
        return f32_to_fp8_bits(x_f32, dtype)
    raise ValueError(dtype)


def from_device_dtype(a: np.ndarray, dtype: str) -> np.ndarray:
    """Device representation -> f32 values."""
    if dtype == "bf16":
        return bf16_bits_to_f32(a)
    if dtype in ("f8e4m3", "f8e5m2"):
        return fp8_bits_to_f32(a, dtype)
    return np.asarray(a).astype(np.float32)
