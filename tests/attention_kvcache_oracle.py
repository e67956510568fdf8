"""f64 numpy reference of attention against a paged KV cache (b200_attention_kvcache): the first L_b keys of sequence b are
gathered from their pages, and query i sees key j iff j < L_b and, when causal, j <= L_b - Sq + i (bottom-right).  A row with
no visible key gives out = 0 and lse = -inf.  Cache slots past L_b and table entries past ceil(L_b / page) are never read."""
import numpy as np


def gather_keys(cache, b, L, block_table=None):
    """the first L keys [L, Hkv, D] of sequence b: key j is row j % page of page block_table[b, j // page] (page b without a
    table)"""
    page = cache.shape[1]
    j = np.arange(L)
    pages = np.full(L, b) if block_table is None else np.asarray(block_table)[b, j // page]
    return np.asarray(cache, dtype=np.float64)[pages, j % page]


def attention_kvcache_f64(q, k_cache, v_cache, seqlens, block_table=None, scale=None, causal=False):
    """q [B, Hq, Sq, D], caches [P, page, Hkv, D], seqlens [B] (clamped to [0, capacity]) -> (out [B, Hq, Sq, D], lse [B, Hq, Sq])"""
    q = np.asarray(q, dtype=np.float64)
    B, Hq, Sq, D = q.shape
    page, Hkv = k_cache.shape[1], k_cache.shape[2]
    cap = page * (1 if block_table is None else np.asarray(block_table).shape[1])
    scale = 1.0 / np.sqrt(D) if scale is None else float(scale)
    g = Hq // Hkv
    out, lse = np.zeros((B, Hq, Sq, D)), np.full((B, Hq, Sq), -np.inf)
    for b in range(B):
        L = int(min(max(int(seqlens[b]), 0), cap))
        k = np.repeat(gather_keys(k_cache, b, L, block_table).transpose(1, 0, 2), g, axis=0)   # [Hq, L, D]
        v = np.repeat(gather_keys(v_cache, b, L, block_table).transpose(1, 0, 2), g, axis=0)
        vis = np.ones((Sq, L), bool)
        if causal:
            vis = np.arange(L)[None, :] <= L - Sq + np.arange(Sq)[:, None]
        s = np.where(vis, scale * np.einsum("hid,hjd->hij", q[b], k), -np.inf)
        rows = vis.any(axis=1)
        if not rows.any():
            continue
        m = s[:, rows].max(axis=-1, keepdims=True)
        p = np.exp(s[:, rows] - m)
        l = p.sum(axis=-1, keepdims=True)
        out[b][:, rows] = np.einsum("hij,hjd->hid", p / l, v)
        lse[b][:, rows] = (m + np.log(l))[..., 0]
    return out, lse


def kv_tile(G, Sq):
    """b200_attention_kvcache's m-tile (gt, st): fewest ceil(G / gt) * ceil(Sq / st) with gt * st <= 64, ties to the larger st"""
    best = None
    for st in range(min(Sq, 64), 0, -1):
        gt = min(G, 64 // st)
        n = -(-G // gt) * -(-Sq // st)
        if best is None or n < best[0]:
            best = (n, gt, st)
    return best[1], best[2]


def kv_splits(units, nkb, sms, cost=2, max_splits=128):
    """b200_attention_kvcache's split count for `units` CTAs per split and nkb 64-key blocks of capacity on `sms` SMs"""
    best_n, best = 1, None
    for n in range(1, min(nkb, max_splits) + 1):
        bps = -(-nkb // n)
        if -(-nkb // bps) != n:
            continue
        c = -(-units * n // sms) * (bps + cost)
        if best is None or c < best:
            best, best_n = c, n
    return best_n
