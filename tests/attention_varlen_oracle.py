"""f64 numpy reference of variable-length (packed) attention, forward and backward, run per sequence.

q [Tq, Hq, D], k and v [Tk, Hkv, D]; sequence b owns query rows [cu_q[b], cu_q[b + 1]) and key rows [cu_k[b], cu_k[b + 1]).
window (left, right), -1 unbounded: with off = Lk - Lq, key j is visible to query i iff j < Lk, (left < 0 or j >= i + off - left)
and (right < 0 or j <= i + off + right).  A row with no visible key gives out = 0 and lse = -inf, dq = 0, and adds nothing to
dk or dv.  Rows outside every sequence are left as the `fill` value."""
import numpy as np


def band_mask(Lq, Lk, window):
    """[Lq, Lk] boolean visibility of one sequence"""
    left, right = window
    i, j = np.arange(Lq)[:, None], np.arange(Lk)[None, :]
    off = Lk - Lq
    m = np.ones((Lq, Lk), dtype=bool)
    if left >= 0:
        m &= j >= i + off - left
    if right >= 0:
        m &= j <= i + off + right
    return m


def visible_pairs(lens_q, lens_k, window):
    return int(sum(band_mask(a, b, window).sum() for a, b in zip(lens_q, lens_k)))


def _seq(q, k, v, g, scale, mask):
    """one sequence: q [Lq, Hq, D], k, v [Lk, Hkv, D] -> s [Hq, Lq, Lk] (masked -inf), p, out [Lq, Hq, D], lse [Hq, Lq]"""
    kk, vv = np.repeat(k, g, axis=1), np.repeat(v, g, axis=1)
    s = np.where(mask[None], scale * np.einsum("ihd,jhd->hij", q, kk), -np.inf)
    m = s.max(axis=-1, keepdims=True) if s.shape[-1] else np.full(s.shape[:-1] + (1,), -np.inf)
    ms = np.where(np.isfinite(m), m, 0.0)
    p = np.exp(s - ms)
    l = p.sum(axis=-1, keepdims=True)
    out = np.einsum("hij,jhd->ihd", np.divide(p, l, out=np.zeros_like(p), where=l > 0), vv)
    with np.errstate(divide="ignore"):
        lse = (ms + np.log(l))[..., 0]
    return kk, vv, s, out, lse


def attention_varlen_f64(q, k, v, cu_q, cu_k, scale=None, window=(-1, -1), fill=0.0):
    """-> (out [Tq, Hq, D], lse [Hq, Tq]) in float64"""
    q, k, v = (np.asarray(t, dtype=np.float64) for t in (q, k, v))
    Tq, Hq, D = q.shape
    g = Hq // k.shape[1]
    scale = 1.0 / np.sqrt(D) if scale is None else float(scale)
    out, lse = np.full(q.shape, fill), np.full((Hq, Tq), fill)
    for b in range(len(cu_q) - 1):
        qa, qb, ka, kb = int(cu_q[b]), int(cu_q[b + 1]), int(cu_k[b]), int(cu_k[b + 1])
        _, _, _, o, ls = _seq(q[qa:qb], k[ka:kb], v[ka:kb], g, scale, band_mask(qb - qa, kb - ka, window))
        out[qa:qb], lse[:, qa:qb] = o, ls
    return out, lse


def attention_varlen_backward_f64(q, k, v, dout, cu_q, cu_k, scale=None, window=(-1, -1), fill=0.0):
    """-> (dq [Tq, Hq, D], dk, dv [Tk, Hkv, D]) in float64; dk and dv of kv head hk sum over its query heads"""
    q, k, v, dout = (np.asarray(t, dtype=np.float64) for t in (q, k, v, dout))
    Tq, Hq, D = q.shape
    Tk, Hkv = k.shape[0], k.shape[1]
    g = Hq // Hkv
    scale = 1.0 / np.sqrt(D) if scale is None else float(scale)
    dq, dk, dv = np.full(q.shape, fill), np.full(k.shape, fill), np.full(k.shape, fill)
    for b in range(len(cu_q) - 1):
        qa, qb, ka, kb = int(cu_q[b]), int(cu_q[b + 1]), int(cu_k[b]), int(cu_k[b + 1])
        Lq, Lk = qb - qa, kb - ka
        kk, vv, s, out, lse = _seq(q[qa:qb], k[ka:kb], v[ka:kb], g, scale, band_mask(Lq, Lk, window))
        p = np.where(np.isfinite(lse)[..., None], np.exp(s - np.where(np.isfinite(lse), lse, 0.0)[..., None]), 0.0)
        do = dout[qa:qb]
        delta = np.einsum("ihd,ihd->hi", do, out)
        ds = p * (np.einsum("ihd,jhd->hij", do, vv) - delta[..., None])
        dq[qa:qb] = scale * np.einsum("hij,jhd->ihd", ds, kk)
        dk[ka:kb] = (scale * np.einsum("hij,ihd->jhd", ds, q[qa:qb])).reshape(Lk, Hkv, g, D).sum(axis=2)
        dv[ka:kb] = np.einsum("hij,ihd->jhd", p, do).reshape(Lk, Hkv, g, D).sum(axis=2)
    return dq, dk, dv
