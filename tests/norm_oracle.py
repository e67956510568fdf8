"""numpy oracle of b200_norm, b200_norm_quantized_fp8 and b200_norm_backward: the operation order stated in
include/cubecl_b200.h in IEEE f32 (numpy float32 arithmetic rounds every operation and never contracts), including the
fixed summation order S() of the kernels, so device results can be compared bit for bit.

Exact cases: rows built so that every sum is exact in any order (small dyadic terms) and rstd is a power of two with eps = 0;
`exact_rms_rows` / `exact_layer_rows` make them and `assert_exact` checks the preconditions on what the oracle computed.
`_mutant` names a deliberately wrong variant of the contract, used by the CPU tests to show the exact cases detect it.
"""
from __future__ import annotations

import numpy as np
import torch

F32 = np.float32
TORCH = {"f32": torch.float32, "bf16": torch.bfloat16, "f16": torch.float16}


def rnd(a, dtype: str) -> np.ndarray:
    """a (f32) rounded to nearest-even in dtype and read back as f32."""
    a = np.asarray(a, dtype=F32)
    if dtype == "f32":
        return a.copy()
    return torch.from_numpy(np.ascontiguousarray(a)).to(TORCH[dtype]).float().numpy()


def geometry(n: int) -> tuple[int, int]:
    """(threads of a row group in each CTA, CTAs per row) of the kernels' row classes."""
    nt = 32 if n <= 1024 else 64 if n <= 2048 else 128 if n <= 4096 else 256
    return nt, 1 if n <= 8192 else 2 if n <= 16384 else 4


def ksum(terms: np.ndarray, n: int) -> np.ndarray:
    """S() of include/cubecl_b200.h over the last axis of f32 terms [T, n]: 8-element chunk q to thread q % (R * NT) as its
    chunk q // (R * NT); each thread adds its values in column order from +0; an xor butterfly over each warp; the warps
    of a CTA in order; the CTAs in order."""
    terms = np.asarray(terms, dtype=F32)
    T = terms.shape[0]
    nt, ranks = geometry(n)
    g = nt * ranks
    cols = 4 * g * 8
    pad = np.zeros((T, cols), dtype=F32)
    pad[:, :n] = terms
    valid = np.zeros(cols, dtype=bool)
    valid[:n] = True
    # column j = (c * g + thread) * 8 + i
    v = pad.reshape(T, 4, g, 8)
    ok = valid.reshape(4, g, 8)
    s = np.zeros((T, g), dtype=F32)
    for c in range(4):
        for i in range(8):
            s = np.where(ok[c, :, i], s + v[:, c, :, i], s).astype(F32)
    s = s.reshape(T, ranks, nt // 32, 32)
    lane = np.arange(32)
    for m in (16, 8, 4, 2, 1):
        s = (s + s[..., lane ^ m]).astype(F32)
    w = s[..., 0]                      # [T, ranks, warps]: every lane holds its warp's sum
    cta = w[..., 0]
    for k in range(1, w.shape[2]):
        cta = (cta + w[..., k]).astype(F32)
    tot = cta[:, 0]
    for r in range(1, ranks):
        tot = (tot + cta[:, r]).astype(F32)
    return tot


def _col(a, n, default):
    return np.full(n, default, dtype=F32) if a is None else np.asarray(a, dtype=F32)


def forward(kind: str, x, eps: float, weight=None, bias=None, residual=None, x_dtype: str = "f32", _mutant: str | None = None):
    """(h, y_f32, mean, rstd) of one b200_norm call: h = x or RNE_x(x + residual); y_f32 before its rounding to y's dtype
    (a 16-bit y is rnd(y_f32, y_dtype)).  Inputs are f32 arrays holding values of their dtypes."""
    x = np.asarray(x, dtype=F32)
    T, n = x.shape
    if residual is not None:
        s = (x + np.asarray(residual, dtype=F32)).astype(F32)
        h = s if _mutant == "unrounded_residual" else rnd(s, x_dtype)
    else:
        h = x.copy()
    nn, e = F32(n - 1 if _mutant == "n_minus_1" else n), F32(eps)
    if kind == "rms":
        mu = np.zeros(T, dtype=F32)
        var = (ksum(h * h, n) / F32(n)).astype(F32)
        d = h
    else:
        mu = (ksum(h, n) / F32(n)).astype(F32)
        d = (h - mu[:, None]).astype(F32)
        if _mutant == "one_pass_var":
            var = (ksum(h * h, n) / F32(n) - mu * mu).astype(F32)
        else:
            var = (ksum(d * d, n) / nn).astype(F32)
    with np.errstate(invalid="ignore", divide="ignore"):     # var + eps = 0 gives rstd = inf, as on the device
        rstd = (F32(1.0) / np.sqrt((var + e).astype(F32))).astype(F32)
        xh = (d * rstd[:, None]).astype(F32)
    y = ((xh * _col(weight, n, 1.0)).astype(F32) + _col(bias, n, 0.0)).astype(F32)
    return h, y, mu, rstd


def units(t: int, n: int) -> tuple[int, int]:
    """(units, rows per unit) of the backward's dweight / dbias partials: a function of t and n only."""
    umax = min(1024, max(64, (1 << 21) // n))
    per = -(-t // min(t, umax))
    return -(-t // per), per


def backward(kind: str, dy, h, rstd, weight=None, mean=None, d_h=None, grad_dtype: str = "f32", _mutant: str | None = None):
    """(dx, dweight, dbias) of one b200_norm_backward call, dx rounded to grad_dtype."""
    dy, h, rstd = (np.asarray(a, dtype=F32) for a in (dy, h, rstd))
    T, n = h.shape
    d = (h - np.asarray(mean, dtype=F32)[:, None]).astype(F32) if kind == "layer" else h
    xh = (d * rstd[:, None]).astype(F32)
    g = (dy * _col(weight, n, 1.0)).astype(F32)
    c1 = (ksum(g * xh, n) / F32(n)).astype(F32)
    c2 = (ksum(g, n) / F32(n)).astype(F32)
    e = (g - (xh * c1[:, None]).astype(F32)).astype(F32)
    if kind == "layer" and _mutant != "no_c2":
        e = (e - c2[:, None]).astype(F32)
    dx = (rstd[:, None] * e).astype(F32)
    if d_h is not None:
        if _mutant == "d_h_after_round":
            dx = (rnd(dx, grad_dtype) + np.asarray(d_h, dtype=F32)).astype(F32)
        else:
            dx = (dx + np.asarray(d_h, dtype=F32)).astype(F32)
    dx = rnd(dx, grad_dtype)
    # dweight / dbias: each unit sums its rows in order from +0, then the units' partials in order
    U, per = units(T, n)
    pw = (dy * xh).astype(F32)

    def colsum(a):
        parts = []
        for u in range(U):
            acc = np.zeros(n, dtype=F32)
            for r in range(u * per, min(T, (u + 1) * per)):
                acc = (acc + a[r]).astype(F32)
            parts.append(acc)
        out = parts[0]
        for p in parts[1:]:
            out = (out + p).astype(F32)
        return out

    return dx, colsum(pw), colsum(dy)


def reference_f64(kind: str, h, eps, weight=None, bias=None):
    """y in f64 from the same h, and the bound of |y_f32 - y_f64| the contract's f32 order guarantees:
    |error| <= c * n * 2^-24 * (|x^| * |w| + |b|) + the last rounding, with x^ scaled by rstd (c a small constant)."""
    h = np.asarray(h, dtype=np.float64)
    T, n = h.shape
    w = np.ones(n) if weight is None else np.asarray(weight, dtype=np.float64)
    b = np.zeros(n) if bias is None else np.asarray(bias, dtype=np.float64)
    if kind == "rms":
        d = h
        var = (h * h).mean(1)
    else:
        d = h - h.mean(1, keepdims=True)
        var = (d * d).mean(1)
    xh = d / np.sqrt(var + eps)[:, None]
    y = xh * w + b
    bound = (4 * n + 16) * 2.0 ** -24 * (np.abs(xh) * np.abs(w) + np.abs(b) + np.abs(xh).max(1, keepdims=True) * np.abs(w))
    return y, bound


# ---------------------------------------------------------------------------------------------- exact cases
def exact_rms_rows(rng, T: int, n: int, kmin: int = -2, kmax: int = 3):
    """RMS rows of +-2^k (k per row): sum v^2 / n = 4^k, rstd = 2^-k with eps = 0, x^ = +-1."""
    k = rng.integers(kmin, kmax + 1, size=(T, 1))
    sign = np.where(rng.random((T, n)) < 0.5, -1.0, 1.0)
    return (sign * np.exp2(k)).astype(F32)


def exact_layer_rows(rng, T: int, n: int, dtype: str = "f32"):
    """Layer rows mu + s * 2^k with an integer mean mu and sum s = 0, sum s^2 = n * 4^j (var = 4^(k + j), rstd a power of two
    with eps = 0): s = +-1 balanced for even n; for odd n >= 7, (3, -3, 2, -2, 1, -1, 0) and +-2 balanced for the rest
    (var = 4^(k + 1)); n = 1 is a constant row (var = 0: give it eps = 1).  |mu| is as large as dtype holds and the sums stay
    exact (up to 2^22 / n in f32), so a one-pass E[v^2] - mu^2 loses bits."""
    mu_max = min(1 << ({"f32": 24, "f16": 11, "bf16": 8}[dtype] - 5), max(8, (1 << 22) // n))
    mu = rng.integers(-mu_max, mu_max + 1, size=(T, 1)).astype(np.float64)
    k = rng.integers(-2, 2, size=(T, 1))
    if n % 2 == 0:
        s = np.tile(np.array([1.0, -1.0]), n // 2)
    elif n == 1:
        s = np.zeros(1)
    else:
        s = np.concatenate([[3.0, -3.0, 2.0, -2.0, 1.0, -1.0, 0.0], np.tile(np.array([2.0, -2.0]), (n - 7) // 2)])
    s = np.stack([rng.permutation(s) for _ in range(T)])
    return (mu + s * np.exp2(k)).astype(F32)


def exact_weight(rng, n: int, lo: int = -4, hi: int = 4):
    """weights / biases as small multiples of 1/4: exact in every dtype, and products with dyadic x^ stay exact."""
    return (rng.integers(lo, hi + 1, size=n) / 4.0).astype(F32)


def exact_grad(rng, T: int, n: int):
    return (rng.integers(-8, 9, size=(T, n)) / 8.0).astype(F32)


def _dyadic_exact(terms, n) -> bool:
    """every partial sum of each row of these terms is exact in f32: the row's terms are integers times one 2^-e whose
    absolute total fits 24 bits."""
    t = np.asarray(terms, dtype=np.float64)
    if not np.all(np.isfinite(t)):
        return False
    for row in t.reshape(-1, t.shape[-1]):
        e = next((e for e in range(0, 60) if np.all(row * 2.0 ** e == np.round(row * 2.0 ** e))), None)
        if e is None or np.abs(row * 2.0 ** e).sum() >= 2 ** 24:
            return False
    return True


def assert_exact(kind: str, h, eps: float = 0.0, weight=None, dy=None) -> None:
    """Preconditions of the exact cases: every S() exact in any order (forward; backward when dy is given) and rstd a power
    of two."""
    h = np.asarray(h, dtype=F32)
    T, n = h.shape
    _, _, mu, r = forward(kind, h, eps)
    assert np.all(np.frexp(r)[0] == 0.5), "rstd is not a power of two"
    if kind == "rms":
        assert _dyadic_exact(h.astype(np.float64) ** 2, n)
    else:
        assert _dyadic_exact(h, n)
        assert _dyadic_exact((h - mu[:, None]).astype(np.float64) ** 2, n)
    if dy is not None:
        d = (h - mu[:, None]) if kind == "layer" else h
        xh = d.astype(np.float64) * r[:, None]
        g = np.asarray(dy, dtype=np.float64) * (1.0 if weight is None else np.asarray(weight, dtype=np.float64))
        assert _dyadic_exact(g * xh, n) and _dyadic_exact(g, n)
        assert _dyadic_exact((np.asarray(dy, dtype=np.float64) * xh).T, T) and _dyadic_exact(np.asarray(dy, dtype=np.float64).T, T)
