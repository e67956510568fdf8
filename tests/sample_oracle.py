"""A numpy restatement of b200_sample (include/cubecl_b200.h): temperature, top-k, min-p, top-p and the Philox draw, with the
masses and the draw in Python / u64 integers.

ex2 stands for PTX's ex2.approx.ftz: here exp2 rounded once to f32, results below 2^-126 flushed to +0.  It agrees with the
hardware on integer arguments, which is what the exact rows are built to use (an assumption about the hardware that PTX does
not promise; attention's and cross-entropy's exact tests make the same one).  On other rows the two may differ by a few ulp
of w; `sample_row` therefore also returns a margin -- the distance of the row's ex2-dependent decisions (min-p's compare,
top-p's tau, t against its interval) from their nearest boundary, in units of mass -- and the bound that distance must exceed
for the id to be the same under any such error.

Mutants (the `_mutant` argument) are wrong contracts the exact GPU cases must be able to tell apart:
  topk_drop_ties     top-k keeps exactly k tokens (the first k of a stable descending sort), dropping ties at the threshold
  topp_strict        top-p's tau needs (mass at or above tau) > P instead of >= P
  float_draw         a float draw u = f32(r0 * 2^-32) and t = floor(u * S') in place of the 64-bit integer t
  minp_of_sum        min-p relative to the kept mass, w >= min_p * sum(w), instead of to the most likely token
  topp_before_topk   top-p applied to what min-p kept, and top-k after it
  row_in_counter     the row index mixed into the Philox counter (counter word 2)
"""

import numpy as np

F32 = np.float32
LOG2E = F32(1.4426950408889634)
MASS_BITS = 40
EX2_REL = 2.0 ** -21    # relative error allowed for ex2.approx against the correctly rounded exp2 (PTX: about 2 ulp)
MUTANTS = ("topk_drop_ties", "topp_strict", "float_draw", "minp_of_sum", "topp_before_topk", "row_in_counter")

_M0, _M1, _W0, _W1, _U32 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85, 0xFFFFFFFF


def philox4x32(ctr, key, rounds=10):
    """Random123's Philox4x32-R on a counter of four and a key of two u32 words"""
    c0, c1, c2, c3 = (int(c) & _U32 for c in ctr)
    k0, k1 = (int(k) & _U32 for k in key)
    for _ in range(rounds):
        p0, p1 = _M0 * c0, _M1 * c2
        c0, c1, c2, c3 = ((p1 >> 32) ^ c1 ^ k0, p1 & _U32, (p0 >> 32) ^ c3 ^ k1, p0 & _U32)
        k0, k1 = (k0 + _W0) & _U32, (k1 + _W1) & _U32
    return c0, c1, c2, c3


def draw_bits(seed, offset, row=0, _mutant=None):
    """R = r0 + 2^32 r1 of Philox4x32-10 at key (lo, hi of seed) and counter (lo, hi of offset, 0, 0)"""
    seed, offset = int(seed), int(offset)
    c2 = row if _mutant == "row_in_counter" else 0
    r = philox4x32((offset & _U32, offset >> 32, c2, 0), (seed & _U32, seed >> 32))
    return r[0] + (r[1] << 32), r[0]


def ex2(a):
    r = np.exp2(np.asarray(a, np.float64)).astype(F32)
    return np.where(np.abs(r) < F32(2.0 ** -126), F32(0), r).astype(F32)


def masses(w):
    """q = floor(w * 2^40) as u64 (exact: w has 24 significant bits and is at most 1)"""
    return np.floor(np.asarray(w, np.float64) * float(1 << MASS_BITS)).astype(np.uint64)


def ceil_mul(p, S):
    """ceil(p * S) for an f32 p, exactly"""
    num, den = float(F32(p)).as_integer_ratio()
    return -(-num * int(S) // den)


def _nucleus(q, keep, top_p, strict=False):
    """(tau, P, F(tau), F(next larger kept value) or None) of the top-p rule over the kept masses q"""
    S = int(q[keep].sum())
    P = ceil_mul(top_p, S)
    vals, cnt = np.unique(q[keep & (q > 0)], return_counts=True)
    vals, cnt = vals[::-1], cnt[::-1]                                  # descending distinct values
    F = np.cumsum([int(a) * int(c) for a, c in zip(vals, cnt)], dtype=object)
    j = next(i for i in range(len(vals)) if (F[i] > P if strict else F[i] >= P))
    return int(vals[j]), P, int(F[j]), (int(F[j - 1]) if j > 0 else None), vals


def sample_row(x, temperature=1.0, top_k=0, top_p=1.0, min_p=0.0, seed=0, offset=0, row=0, _mutant=None, _keep=None):
    """(id, margin, bound) for one row x (f32 values of the logits).  margin = inf when no decision depends on ex2 (greedy,
    invalid, one surviving token); the id is robust to ex2's error wherever margin > bound.  A list passed as _keep receives
    the surviving tokens' mask and their masses."""
    x = np.asarray(x, F32)
    v = x.size
    T, tp, mp = F32(temperature), F32(top_p), F32(min_p)
    if not (T >= 0) or T == np.inf or not (0 < tp <= 1) or not (0 <= mp <= 1):
        return -1, np.inf, 0.0
    if T == 0:
        if np.isnan(x).any() or (x == np.inf).any() or (x == -np.inf).all():
            return -1, np.inf, 0.0
        return int(np.argmax(x)), np.inf, 0.0
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        z = (x / T).astype(F32)
    if np.isnan(z).any() or (z == np.inf).any() or (z == -np.inf).all():
        return -1, np.inf, 0.0
    m = z.max()
    with np.errstate(invalid="ignore"):
        w = ex2(((z - m).astype(F32) * LOG2E).astype(F32))
    q = masses(w)
    keep_k = np.ones(v, bool)
    if 1 <= top_k < v:
        if _mutant == "topk_drop_ties":
            keep_k = np.zeros(v, bool)
            keep_k[np.argsort(-z.astype(np.float64), kind="stable")[:top_k]] = True
        else:
            keep_k = z >= np.sort(z)[v - top_k]
    if _mutant == "minp_of_sum":
        keep_p = w >= F32(mp * w[keep_k].astype(np.float64).sum())
    else:
        keep_p = w >= mp
    margins = []
    S_all = int(q[keep_k & keep_p].sum())
    bound = EX2_REL * S_all * 2 + 2 * v + 4
    if mp > 0:
        sel = keep_k & (q > 0)
        if sel.any():
            margins.append(float(np.min(np.abs(w[sel].astype(np.float64) - float(mp)))) * float(1 << MASS_BITS))
    if not (keep_k & keep_p & (q > 0)).any():      # only a mutant can drop the max
        return -1, np.inf, 0.0
    if _mutant == "topp_before_topk":
        keep = keep_p.copy()
        if tp < 1:
            tau = _nucleus(q, keep, tp)[0]
            keep &= q >= tau
        keep &= keep_k
    else:
        keep = keep_k & keep_p
        if tp < 1:
            tau, P, Ft, Fn, vals = _nucleus(q, keep, tp, strict=_mutant == "topp_strict")
            margins.append(Ft - P)
            if Fn is not None:
                margins.append(P - 1 - Fn)
            other = vals[vals != tau].astype(np.float64)
            if other.size:
                margins.append(float(np.min(np.abs(other - tau))))
            keep &= q >= tau
    qn = np.where(keep, q, np.uint64(0))
    if _keep is not None:
        _keep.extend([keep & (q > 0), qn])
    Sp = int(qn.sum())
    R, r0 = draw_bits(seed, offset, row, _mutant)
    if _mutant == "float_draw":
        t = int(np.floor(float(F32(r0 * 2.0 ** -32)) * Sp))
        t = min(t, Sp - 1)
    else:
        t = (R * Sp) >> 64
    C = np.cumsum(qn, dtype=np.uint64)
    i = int(np.searchsorted(C, np.uint64(t), side="right"))
    if int(np.count_nonzero(qn)) > 1:
        lo = int(C[i]) - int(qn[i])
        margins.append(min(t - lo, int(C[i]) - 1 - t))
    return i, (min(margins) if margins else np.inf), bound


def sample(x, temperature=1.0, top_k=0, top_p=1.0, min_p=0.0, seed=0, offset=0, _mutant=None):
    """(ids, margins, bounds) for rows x [b, v]; each parameter a scalar or a per-row sequence"""
    x = np.asarray(x, F32)
    b = x.shape[0]

    def at(p, r):
        return p[r] if np.ndim(p) else p
    out = [sample_row(x[r], at(temperature, r), int(at(top_k, r)), at(top_p, r), at(min_p, r), int(at(seed, r)),
                      int(at(offset, r)), r, _mutant) for r in range(b)]
    return (np.array([o[0] for o in out], np.int64), np.array([o[1] for o in out], np.float64),
            np.array([o[2] for o in out], np.float64))


# ---------------------------------------------------------------------------------------------- exact rows
def exact_steps(jmin=-45):
    """{j: d} for the integers j in [jmin, 0] that have an f32 d (within 8 ulps of j ln2) with rn(d * log2e) = j exactly, so
    that a logit d below the max has w = ex2(j) = 2^j"""
    out = {0: F32(0)}
    for j in range(-1, jmin - 1, -1):
        c = F32(j * np.log(2.0))
        for s in range(-8, 9):
            d = np.nextafter(c, F32(np.inf if s > 0 else -np.inf), dtype=F32) if s else c
            for _ in range(abs(s) - 1):
                d = np.nextafter(d, F32(np.inf if s > 0 else -np.inf), dtype=F32)
            if F32(d * LOG2E) == F32(j):
                out[j] = F32(d)
                break
    return out


def exact_rows(rng, b, v, dtype, T=1.0):
    """rows [b, v] whose every w is a power of two or +0 at temperature T (a power of two): f32 rows draw their logits from
    the exact steps d_j * T below a max of 0, with -inf and signed-zero ties mixed in; 16-bit rows hold tied maxima and values
    far below them (w = 1 or +0), as cross-entropy's exact rows do"""
    x = np.empty((b, v), F32)
    T = F32(T)
    if dtype == "f32":
        steps = exact_steps()
        js = np.array(sorted(j for j in steps if j < 0), np.int64)
        for r in range(b):
            # mostly the largest few steps below the max, so that a sizable part of the mass sits on many tokens
            pick = js[np.clip(len(js) - rng.geometric(0.25, size=v), 0, len(js) - 1)]
            row = np.array([steps[int(j)] for j in pick], F32) * T
            row[rng.random(v) < 0.02] = -np.inf
            n0 = max(1, min(v, int(rng.integers(1, 9))))
            z = rng.choice(v, size=n0, replace=False)
            row[z] = np.where(rng.random(n0) < 0.5, F32(0.0), F32(-0.0))
            x[r] = row
    else:
        for r in range(b):
            row = np.full(v, F32(-256.0) * T if dtype == "f16" else F32(-2048.0) * T, F32)
            n = int(min(v, 2 ** int(rng.integers(0, 6))))
            row[rng.choice(v, size=n, replace=False)] = F32(8.0) * T
            x[r] = row
    return x


# per-row configurations of the exact cases: (temperature, top_k, top_p, min_p); in f32 the last two rows are crafted
EXACT_CONF = [(0.0, 0, 1.0, 0.0), (1.0, 0, 1.0, 0.0), (1.0, 1, 1.0, 0.0), (0.5, 3, 1.0, 0.0), (2.0, 50, 1.0, 0.0),
              (1.0, 0, 0.5, 0.0), (1.0, 0, 0.9, 0.0), (0.5, 0, 1.0, 0.25), (1.0, 0, 1.0, 2.0 ** -20),
              (1.0, 40, 0.7, 2.0 ** -6), (2.0, 7, 0.3, 0.5), (1.0, 100000, 0.99, 0.0), (1.0, 0, 0.5, 0.0),
              (1.0, 2, 0.6, 0.0)]


def exact_batch(rng, v, dtype):
    """(x, per-row parameters) of one exact call: a row per EXACT_CONF entry, built at its temperature, with random seeds and
    offsets.  In f32 two rows are crafted.  The next-to-last holds one max (w = 1), two tokens at w = 1/2 and the rest far
    below, so that at top_p = 1/2 the mass at or above 2^40 is exactly P: the case where top-p's >= and > differ.  The last
    holds one max, one token at w = 1/2 and the rest at w = 1/4: top-k 2 then top-p 0.6 keeps the max alone, while top-p
    over the whole row keeps every token and top-k after it two."""
    b = len(EXACT_CONF)
    x = np.concatenate([exact_rows(rng, 1, v, dtype, T=t if t else 1.0) for t, *_ in EXACT_CONF])
    if dtype == "f32" and v >= 3:
        steps = exact_steps()
        x[-2] = F32(-1000.0)
        pos = rng.choice(v, size=3, replace=False)
        x[-2, pos] = [F32(0.0), steps[-1], steps[-1]]
        x[-1] = steps[-2]
        x[-1, pos[:2]] = [F32(0.0), steps[-1]]
    cols = list(zip(*EXACT_CONF))
    seeds = rng.integers(0, 2 ** 63, size=b, dtype=np.int64).astype(np.uint64) * np.uint64(2) + np.uint64(1)
    offs = rng.integers(0, 2 ** 62, size=b, dtype=np.int64).astype(np.uint64)
    return x, dict(temperature=np.array(cols[0], F32), top_k=np.array(cols[1]), top_p=np.array(cols[2], F32),
                   min_p=np.array(cols[3], F32), seed=seeds, offset=offs)
