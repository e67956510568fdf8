"""numpy oracle of mixture-of-experts routing (b200_moe_* in include/cubecl_b200.h): top-k selection, the expert-sorted
dispatch plan, the row gather and the weighted combine with its backward.  tests/test_moe_cpu.py pins it to torch on the CPU
(topk, stable argsort + bincount + cumsum, index_select, weighted sums)."""
from __future__ import annotations

import numpy as np

from qmatmul_oracle import fma_f32

F32, F64 = np.float32, np.float64


def scores(logits, score: str) -> np.ndarray:
    """s_e in f64: softmax over each row (max-subtracted) or the sigmoid."""
    l = np.asarray(logits, F64)
    if score == "sigmoid":
        return 1.0 / (1.0 + np.exp(-l))
    e = np.exp(l - np.max(l, axis=1, keepdims=True))
    return e / e.sum(axis=1, keepdims=True)


def keys(logits, score: str, bias=None) -> np.ndarray:
    """Selection keys as f32: the logit without a bias, else rn(s_e + b_e) (s_e rounded to f32 first)."""
    if bias is None:
        return np.asarray(logits, F32)
    s = scores(logits, score).astype(F32)
    return (s + np.asarray(bias, F32)[None, :]).astype(F32)


def _order(v, idx) -> list:
    """Indices of v by descending value, ties to the lower index, NaN below -inf."""
    v = np.asarray(v, F64)
    return sorted(idx, key=lambda i: (1, 0.0, i) if np.isnan(v[i]) else (0, -v[i], i))


def eligible(key_row, n_group: int, topk_group: int) -> np.ndarray:
    """Experts that stay eligible under group-limited routing (all of them when n_group <= 1)."""
    E = len(key_row)
    if n_group <= 1:
        return np.ones(E, bool)
    gs = E // n_group
    gscore = np.empty(n_group, F32)
    for g in range(n_group):
        top = _order(key_row[g * gs:(g + 1) * gs], range(gs))[:2]
        gscore[g] = F32(key_row[g * gs + top[0]]) + F32(key_row[g * gs + top[1]])
    keep = np.zeros(E, bool)
    for g in _order(gscore, range(n_group))[:topk_group]:
        keep[g * gs:(g + 1) * gs] = True
    return keep


def route(logits, k: int, score: str = "softmax", renormalize: bool = True, n_group: int = 0, topk_group: int = 0,
          scale: float = 1.0, bias=None):
    """(ids i32 [T, k], weights f64 [T, k]): the selection of the contract; weights in exact arithmetic (the device's differ by
    expf's error and its summation order)."""
    kf = keys(logits, score, bias)
    s = scores(logits, score)
    T, E = kf.shape
    ids = np.zeros((T, k), np.int32)
    w = np.zeros((T, k), F64)
    for t in range(T):
        ok = eligible(kf[t], n_group, topk_group)
        ids[t] = _order(kf[t], [e for e in range(E) if ok[e]])[:k]
        w[t] = s[t, ids[t]]
        if renormalize:
            w[t] /= w[t].sum()
    return ids, w * scale


def plan(ids, E: int):
    """(offs i32 [E], row_of i32 [T, k], slot_of i32 [T * k]): a stable counting sort of the slots by expert; ids outside
    [0, E) are dropped."""
    flat = np.asarray(ids, np.int64).reshape(-1)
    keep = (flat >= 0) & (flat < E)
    order = np.argsort(np.where(keep, flat, E), kind="stable")[: int(keep.sum())]
    offs = np.cumsum(np.bincount(flat[keep], minlength=E)).astype(np.int32)
    row_of = np.full(flat.shape, -1, np.int32)
    row_of[order] = np.arange(len(order), dtype=np.int32)
    slot_of = np.full(flat.shape, -1, np.int32)
    slot_of[: len(order)] = order
    return offs, row_of.reshape(np.shape(ids)), slot_of


def permute(src, slot_of, k: int, dst):
    """dst[r] = src[slot_of[r] // k] where 0 <= slot_of[r] < len(slot_of); other rows keep dst's values."""
    out = np.array(dst, copy=True)
    n = len(slot_of)
    for r, s in enumerate(slot_of):
        if 0 <= s < n:
            out[r] = src[s // k]
    return out


def combine(ys, row_of, weights=None) -> np.ndarray:
    """y [T, N] in f32: acc = fma(w, ys[row], acc) over increasing j (acc + ys without weights), dropped slots skipped."""
    ys = np.asarray(ys, F32)
    T, k = row_of.shape
    acc = np.zeros((T, ys.shape[1]), F32)
    for j in range(k):
        r = row_of[:, j]
        live = (r >= 0) & (r < ys.shape[0])
        v = np.where(live[:, None], ys[np.where(live, r, 0)], F32(0))
        if weights is None:
            acc = np.where(live[:, None], (acc + v).astype(F32), acc)
        else:
            acc = np.where(live[:, None], fma_f32(np.asarray(weights, F32)[:, j:j + 1], v, acc), acc)
    return acc


def combine_backward(dy, ys, weights, row_of):
    """(d_ys f32 [R, N] with NaN in rows no slot references, d_w f64 [T, k]): d_ys[row] = rn(w * dy[t]); d_w the exact dot
    product (the device's matches it on integer-valued data)."""
    dy, ys, w = np.asarray(dy, F32), np.asarray(ys, F32), np.asarray(weights, F32)
    d_ys = np.full(ys.shape, np.nan, F32)
    d_w = np.zeros(row_of.shape, F64)
    for t in range(row_of.shape[0]):
        for j in range(row_of.shape[1]):
            r = row_of[t, j]
            if 0 <= r < ys.shape[0]:
                d_ys[r] = (w[t, j] * dy[t]).astype(F32)
                d_w[t, j] = np.dot(dy[t].astype(F64), ys[r].astype(F64))
    return d_ys, d_w


def weight_bound(logits, k: int, score: str) -> np.ndarray:
    """Relative bound per token on the device's weights against route()'s exact ones.  expf is within 2 ulp (2^-22 relative);
    rounding its argument l - max (softmax) costs |l - max| 2^-24 of relative error in the exponential; the softmax sum adds
    up to E - 1 roundings and its division one; renormalising adds k - 1 roundings, a division and the error of the sum; the
    scale one more.  Each error enters at most twice (numerator and denominator)."""
    l = np.asarray(logits, F64)
    T, E = l.shape
    arg = np.abs(l - np.max(l, axis=1, keepdims=True)) if score == "softmax" else np.abs(l)
    per_exp = 4.0 + arg.max(axis=1) + 1.0
    return 2.0 * (2.0 * per_exp + E + 2.0 * k + 4.0) * 2.0 ** -24
