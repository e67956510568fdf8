"""f64 numpy reference of scaled-dot-product attention: out and the natural-log log-sum-exp per row, with a scale, top-left
causal masking (key j visible to query i iff j <= i) and GQA (query head h reads kv head h // (Hq // Hkv))."""
import numpy as np


def attention_f64(q, k, v, scale=None, causal=False):
    """q [B, Hq, Sq, D], k and v [B, Hkv, Sk, D] (any float arrays) -> (out [B, Hq, Sq, D], lse [B, Hq, Sq]) in float64."""
    q, k, v = (np.asarray(t, dtype=np.float64) for t in (q, k, v))
    B, Hq, Sq, D = q.shape
    Hkv, Sk = k.shape[1], k.shape[2]
    assert Hq % Hkv == 0 and v.shape == k.shape
    scale = 1.0 / np.sqrt(D) if scale is None else float(scale)
    g = Hq // Hkv
    kk, vv = np.repeat(k, g, axis=1), np.repeat(v, g, axis=1)
    s = scale * np.einsum("bhid,bhjd->bhij", q, kk)
    if causal:
        s = np.where(np.arange(Sk)[None, :] <= np.arange(Sq)[:, None], s, -np.inf)
    m = s.max(axis=-1, keepdims=True)
    p = np.exp(s - m)
    l = p.sum(axis=-1, keepdims=True)
    out = np.einsum("bhij,bhjd->bhid", p / l, vv)
    return out, (m + np.log(l))[..., 0]


def visible_pairs(Sq, Sk, causal):
    """the number of visible (i, j) pairs of one head: Sq * Sk, or sum_i min(i + 1, Sk) when causal"""
    if not causal:
        return Sq * Sk
    full = min(Sq, Sk)
    return full * (full + 1) // 2 + max(0, Sq - Sk) * Sk
