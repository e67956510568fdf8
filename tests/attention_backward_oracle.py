"""f64 numpy reference of the scaled-dot-product attention backward: dq, dk and dv of attention_oracle.attention_f64's out,
with a scale, top-left causal masking and GQA (dk and dv of kv head hk sum over the query heads h with h // (Hq // Hkv) == hk)."""
import numpy as np

from attention_oracle import attention_f64


def attention_backward_f64(q, k, v, dout, scale=None, causal=False):
    """q [B, Hq, Sq, D], k and v [B, Hkv, Sk, D], dout [B, Hq, Sq, D] (any float arrays) -> (dq, dk, dv) in float64.  P is
    recomputed from the f64 lse, as the kernels recompute it from the forward's."""
    q, k, v, dout = (np.asarray(t, dtype=np.float64) for t in (q, k, v, dout))
    B, Hq, Sq, D = q.shape
    Hkv, Sk = k.shape[1], k.shape[2]
    scale = 1.0 / np.sqrt(D) if scale is None else float(scale)
    g = Hq // Hkv
    out, lse = attention_f64(q, k, v, scale, causal)
    kk, vv = np.repeat(k, g, axis=1), np.repeat(v, g, axis=1)
    s = scale * np.einsum("bhid,bhjd->bhij", q, kk)
    if causal:
        s = np.where(np.arange(Sk)[None, :] <= np.arange(Sq)[:, None], s, -np.inf)
    p = np.exp(s - lse[..., None]) if Sq and Sk else np.zeros(s.shape)
    delta = np.einsum("bhid,bhid->bhi", dout, out)
    ds = p * (np.einsum("bhid,bhjd->bhij", dout, vv) - delta[..., None])
    dq = scale * np.einsum("bhij,bhjd->bhid", ds, kk)
    dk = scale * np.einsum("bhij,bhid->bhjd", ds, q).reshape(B, Hkv, g, Sk, D).sum(axis=2)
    dv = np.einsum("bhij,bhid->bhjd", p, dout).reshape(B, Hkv, g, Sk, D).sum(axis=2)
    return dq, dk, dv
