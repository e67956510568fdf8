"""f64 oracle of the grouped matmul (b200_matmul_grouped, torch.nn.functional.grouped_mm with offs), shared by
tests/test_matmul_grouped_cpu.py and tests/test_matmul_grouped_gpu.py.

Offsets are cumulative ends; on read o_g = min(max(offs[g], o_{g-1}), T) with o_{-1} = 0, and group g owns [o_{g-1}, o_g).
  ragged M: lhs [T, K] x rhs [G, K, N] -> out [T, N]; rows >= o_{G-1} are not written (NaN here).
  ragged K: lhs [M, T] x rhs [T, N] -> out [G, M, N]; out[g] = lhs[:, o_{g-1}:o_g] @ rhs[o_{g-1}:o_g, :] (+0 when empty).
"""
from __future__ import annotations

import numpy as np


def clamp_offsets(offs, T: int) -> np.ndarray:
    """The ends the kernel reads: a running maximum (from 0) of offs, clamped to T."""
    run = np.maximum.accumulate(np.maximum(np.asarray(offs, dtype=np.int64), 0)) if len(offs) else np.zeros(0, np.int64)
    return np.minimum(run, T)


def bounds(offs, T: int) -> list[tuple[int, int]]:
    ends = clamp_offsets(offs, T)
    starts = np.concatenate([[0], ends[:-1]]) if len(ends) else ends
    return [(int(s), int(e)) for s, e in zip(starts, ends)]


def offsets(sizes) -> np.ndarray:
    """i32 cumulative ends of the group sizes"""
    return np.cumsum(np.asarray(sizes, dtype=np.int64)).astype(np.int32)


def ragged_m(a, b, offs, bias=None, alpha=1.0, activation=None):
    """out [T, N] in f64 (NaN on rows no group owns) and the mask of written rows"""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    T, N = a.shape[0], b.shape[2]
    out = np.full((T, N), np.nan)
    written = np.zeros(T, dtype=bool)
    for g, (lo, hi) in enumerate(bounds(offs, T)):
        y = alpha * (a[lo:hi] @ b[g])
        if bias is not None:
            y = y + np.asarray(bias, dtype=np.float64)[g]
        if activation == "relu":
            y = np.maximum(y, 0.0)
        out[lo:hi] = y
        written[lo:hi] = True
    return out, written


def ragged_k(a, b, offs, G: int | None = None):
    """out [G, M, N] in f64"""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    T = a.shape[1]
    G = len(offs) if G is None else G
    out = np.zeros((G, a.shape[0], b.shape[1]))
    for g, (lo, hi) in enumerate(bounds(offs, T)):
        out[g] = a[:, lo:hi] @ b[lo:hi]
    return out
