"""numpy restatement of the b200_rope* contracts (include/cubecl_b200.h).

apply():          the f32 operation order a' = rn(rn(a c) - rn(b s)), b' = rn(rn(b c) + rn(a s)) (numpy's f32 ops round each
                  result once, and never contract into an fma), rounded once to the dtype; pass-through columns; rows whose
                  position is outside [0, P) kept bit for bit.
kvcache_write():  apply() of k, then b200_kvcache_write(_fp8)'s scatter: slots outside [0, P * page) skipped; an fp8 cache
                  stores sat_rn(x / scale[hk]) of the dtype-rounded x.
table():          the f64 inv_freq rules and attention factors, cos / sin in f64, rounded once to f32.
Values travel as f32 arrays holding dtype values; to_bits / from_bits move raw dtype bits (NaN payloads, -0)."""
import math

import numpy as np
import torch

TORCH = {"f32": torch.float32, "bf16": torch.bfloat16, "f16": torch.float16}
BITS = {"f32": np.uint32, "bf16": np.uint16, "f16": np.uint16}
FP8 = {"f8e4m3": (torch.float8_e4m3fn, 448.0), "f8e5m2": (torch.float8_e5m2, 57344.0)}


def rnd(x, dt):
    """x (f32) rounded to nearest-even in dt and widened back"""
    return torch.from_numpy(np.ascontiguousarray(x, np.float32)).to(TORCH[dt]).float().numpy()


def to_bits(x, dt):
    return torch.from_numpy(np.ascontiguousarray(x, np.float32)).to(TORCH[dt]).view(
        torch.int32 if dt == "f32" else torch.int16).numpy().view(BITS[dt])


def from_bits(b, dt):
    return torch.from_numpy(np.ascontiguousarray(b).view(np.int32 if dt == "f32" else np.int16)).view(TORCH[dt]).float().numpy()


def pairs(D, rot, style):
    """(ia, ib): the column of a and of b for every pair i < rot / 2"""
    half = rot // 2
    i = np.arange(half)
    return (i, i + half) if style == "neox" else (2 * i, 2 * i + 1)


def apply(x, cos_sin, pos, style, rot, dt, inverse=False, _mutant=None):
    """x [B, S, H, D] (f32 holding dt values), cos_sin f32 [P, rot], pos i64 [B, S] -> the rotated x, rounded to dt."""
    x = np.asarray(x, np.float32)
    out = x.copy()
    P = cos_sin.shape[0]
    half = rot // 2
    ia, ib = pairs(x.shape[-1], rot, style)
    if _mutant == "swapped_pairs":
        ia, ib = pairs(x.shape[-1], rot, "gptj" if style == "neox" else "neox")
    ok = (pos >= 0) & (pos < P)
    if _mutant == "angle_zero_out_of_range":
        ok = np.ones_like(ok)
    pc = np.where((pos >= 0) & (pos < P), pos, 0)
    c = cos_sin[pc][..., None, :half].astype(np.float32)            # [B, S, 1, half]
    s = cos_sin[pc][..., None, half:rot].astype(np.float32)
    if _mutant == "angle_zero_out_of_range":
        bad = ~((pos >= 0) & (pos < P))
        c = np.where(bad[..., None, None], np.float32(1), c)
        s = np.where(bad[..., None, None], np.float32(0), s)
    if inverse and _mutant != "inverse_sign":
        s = -s
    a, b = x[..., ia], x[..., ib]
    with np.errstate(invalid="ignore", over="ignore"):
        if _mutant == "fma":
            # rn(a c - rn(b s)) in f64: one rounding fewer, as an fma would do
            a2 = (a.astype(np.float64) * c - (b * s).astype(np.float64)).astype(np.float32)
            b2 = (b.astype(np.float64) * c + (a * s).astype(np.float64)).astype(np.float32)
        else:
            a2 = a * c - b * s
            b2 = b * c + a * s
    a2, b2 = rnd(a2, dt), rnd(b2, dt)
    okb = ok[..., None, None]
    out[..., ia] = np.where(okb, a2, a)
    out[..., ib] = np.where(okb, b2, b)
    if _mutant == "rotate_pass_through" and rot < x.shape[-1]:
        out[..., rot:] = rnd(out[..., rot:] * np.float32(0.5) + np.float32(0), dt)
    return out


def fp8_bytes(x, scale, cache):
    """sat_rn(x / scale) in the fp8 format, per kv head: x [..., Hkv, D] f32, scale [Hkv] -> uint8"""
    t, lim = FP8[cache]
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        q = (np.asarray(x, np.float32) / np.asarray(scale, np.float32)[:, None]).astype(np.float32)
    qt = torch.from_numpy(q).clamp(-lim, lim)                        # NaN stays NaN
    return qt.to(t).view(torch.uint8).numpy()


def kvcache_write(k_cache, v_cache, k_rot, v, slots, dt, cache=None, k_scale=None, v_scale=None, _mutant=None, k_raw=None):
    """scatter k_rot, v [B, S, Hkv, D] (f32 dt values) into copies of the caches (raw bits [P, page, Hkv, D]: dt bits, or fp8
    bytes); returns (k_cache, v_cache)."""
    kc, vc = k_cache.copy(), v_cache.copy()
    Pp, page = kc.shape[:2]
    B, S = k_rot.shape[:2]
    for n in range(B * S):
        b, s = divmod(n, S)
        sl = int(slots[n])
        if sl < 0 or sl >= Pp * page:
            continue
        pg, r = divmod(sl, page)
        if cache is None:
            kc[pg, r] = to_bits(k_rot[b, s], dt)
            vc[pg, r] = to_bits(v[b, s], dt)
        else:
            kx = k_raw[b, s] if _mutant == "fp8_from_f32" else k_rot[b, s]
            kc[pg, r] = fp8_bytes(kx, k_scale, cache)
            vc[pg, r] = fp8_bytes(v[b, s], v_scale, cache)
    return kc, vc


# ---------------------------------------------------------------------------------------------- tables (f64)
def _mscale(f, m=1.0):
    return 1.0 if f <= 1 else 0.1 * m * math.log(f) + 1.0


def inv_freq(rot, base=10000.0, kind="default", factor=1.0, low_freq_factor=0.0, high_freq_factor=0.0, orig=0, beta_fast=0.0,
             beta_slow=0.0, truncate=True, inv=None):
    """inv_freq [rot / 2] in f64 under the header's rules; parameters are taken as the f32 values the C struct holds"""
    f32 = lambda v: float(np.float32(v))   # noqa: E731
    base, factor, lo_f, hi_f = f32(base), f32(factor), f32(low_freq_factor), f32(high_freq_factor)
    i = np.arange(rot // 2, dtype=np.float64)
    if kind == "inv_freq":
        return np.asarray(inv, np.float32).astype(np.float64)
    d = 1.0 / np.power(base, (2.0 * i) / rot)
    if kind == "default":
        return d
    if kind == "linear":
        return d / factor
    if kind == "llama3":
        w = 2.0 * math.pi / d
        m = (orig / w - lo_f) / (hi_f - lo_f)
        mid = (1.0 - m) * d / factor + m * d
        return np.where(w > orig / lo_f, d / factor, np.where(w < orig / hi_f, d, mid))
    if kind == "yarn":
        fast = f32(beta_fast) if beta_fast else 32.0
        slow = f32(beta_slow) if beta_slow else 1.0
        corr = lambda r: rot * math.log(orig / (r * 2 * math.pi)) / (2 * math.log(base))   # noqa: E731
        lo, hi = corr(fast), corr(slow)
        if truncate:
            lo, hi = math.floor(lo), math.ceil(hi)
        lo, hi = max(lo, 0.0), min(hi, rot - 1.0)
        if lo == hi:
            hi += 0.001
        r = np.clip((i - lo) / (hi - lo), 0.0, 1.0)
        ext = 1.0 - r
        return d / factor * (1.0 - ext) + d * ext
    raise ValueError(kind)


def attention_factor(kind="default", factor=1.0, mscale=0.0, mscale_all_dim=0.0, attention_factor=0.0):
    f32 = lambda v: float(np.float32(v))   # noqa: E731
    if attention_factor and attention_factor > 0:
        return f32(attention_factor)
    if kind != "yarn":
        return 1.0
    f = f32(factor)
    if mscale and mscale_all_dim:
        return _mscale(f, f32(mscale)) / _mscale(f, f32(mscale_all_dim))
    return _mscale(f)


def table_f64(P, inv, af):
    """(cos, sin) [P, rot / 2] in f64: af * cos(p inv), af * sin(p inv)"""
    ang = np.arange(P, dtype=np.float64)[:, None] * inv[None, :]
    return af * np.cos(ang), af * np.sin(ang)


def table(P, inv, af):
    c, s = table_f64(P, inv, af)
    return np.concatenate([c, s], 1).astype(np.float32)
