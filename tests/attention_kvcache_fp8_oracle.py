"""f64 numpy reference of attention against an fp8 KV cache (b200_attention_kvcache_fp8) and of the quantizing cache write
(b200_kvcache_write_fp8).

An fp8 cache holds bytes k8, v8 in e4m3 (torch's float8_e4m3fn: no inf, 0x7F / 0xFF are NaN, max 448) or e5m2 (IEEE-like, max
57344) and f32 per-kv-head scales: K = k_scale[hk] * k8, V = v_scale[hk] * v8.  The attention is the 16-bit oracle on the
dequantized cache.  The write stores sat_rn(x / s): the f32 quotient rounded to nearest even in the cache format, magnitudes
past the largest finite value saturate to it (inf included), NaN stays NaN.  This module decodes and rounds from the formats'
bit layouts, without torch, so the tests can pin it to torch's casts."""
import numpy as np

import attention_kvcache_oracle as ko

FORMATS = ("f8e4m3", "f8e5m2")
MAX = {"f8e4m3": 448.0, "f8e5m2": 57344.0}


def decode(codes, fmt):
    """uint8 codes -> f64 values"""
    c = np.asarray(codes, dtype=np.uint8).astype(np.int64)
    sign = np.where(c & 0x80, -1.0, 1.0)
    if fmt == "f8e4m3":
        e, m, bias, mb = (c >> 3) & 0xF, c & 0x7, 7, 3
        nan = (c & 0x7F) == 0x7F
        inf = np.zeros_like(nan)
    else:
        e, m, bias, mb = (c >> 2) & 0x1F, c & 0x3, 15, 2
        nan = (e == 0x1F) & (m != 0)
        inf = (e == 0x1F) & (m == 0)
    mag = np.where(e == 0, m * 2.0 ** (1 - bias - mb), (1.0 + m / 2.0 ** mb) * 2.0 ** (e.astype(np.float64) - bias))
    out = sign * mag
    out = np.where(inf, sign * np.inf, out)
    return np.where(nan, np.nan, out)


def _finite_table(fmt):
    """the non-negative finite values of the format with their codes, ascending"""
    codes = np.arange(0x80, dtype=np.uint8)
    vals = decode(codes, fmt)
    keep = np.isfinite(vals)
    return vals[keep], codes[keep]


def quantize(x, scale, fmt):
    """f32 x [..., Hkv, D] and f32 scale [Hkv] -> uint8 codes of sat_rn(x / scale): the f32 quotient (rounded to nearest), then
    the nearest value of the format with ties to the even code, saturating at +-MAX; NaN gives the format's NaN (0x7F)."""
    q = (np.asarray(x, dtype=np.float32) / np.asarray(scale, dtype=np.float32)[:, None]).astype(np.float64)
    vals, codes = _finite_table(fmt)
    a = np.minimum(np.abs(np.nan_to_num(q, nan=0.0)), MAX[fmt])
    hi = np.clip(np.searchsorted(vals, a), 0, len(vals) - 1)   # first value >= a
    lo = np.maximum(hi - 1, 0)
    dlo, dhi = a - vals[lo], vals[hi] - a
    pick_hi = (dhi < dlo) | ((dhi == dlo) & (codes[hi] % 2 == 0))
    code = np.where(pick_hi, codes[hi], codes[lo]).astype(np.uint8)
    code = np.where(np.signbit(q), code | 0x80, code).astype(np.uint8)
    return np.where(np.isnan(q), np.uint8(0x7F), code).astype(np.uint8)


def dequantize(codes, scale, fmt):
    """uint8 cache codes [P, page, Hkv, D] and f32 [Hkv] scales -> the f64 cache scale[hk] * v8"""
    return decode(codes, fmt) * np.asarray(scale, dtype=np.float64)[None, None, :, None]


def attention_kvcache_fp8_f64(q, k8, v8, k_scale, v_scale, fmt, seqlens, block_table=None, scale=None, causal=False):
    """q [B, Hq, Sq, D], fp8 code caches [P, page, Hkv, D] -> (out, lse) of the dequantized cache"""
    return ko.attention_kvcache_f64(q, dequantize(k8, k_scale, fmt), dequantize(v8, v_scale, fmt), seqlens, block_table, scale,
                                    causal)
