"""Exact model of the attention kernels on power-of-two softmax weights, shared by tests/test_attention_exact_weights_cpu.py
and tests/test_attention_exact_weights_gpu.py.

With scale = ln 2 the kernels' scale_log2 is exactly 1.0f, so on integer scores every p = ex2(t - m) is ex2 of an integer.
Every row is required to keep each visible score either within NEAR of the row maximum or at least FAR below it.  Then, in
whatever order the kernels meet the keys (128-key blocks, 64-key blocks, KV-cache splits):
  * a key within NEAR gets p = 2^-k (k <= NEAR), and every rescale or merge factor ex2(m_old - m_new) is 2^-k as well, or
    +0 when m_old was itself a far score;
  * a far key gets p = +0: it is at least FAR - NEAR = 2^7 + 1 below any running maximum it meets (ex2.approx.ftz of an
    argument <= -127 is +0), so no subnormal ever reaches l or O;
  * P rounded to 16 bits is exact, and O = sum w v and l = sum w are exact f32 sums while the weighted keys' integer |v| sum below 2^(24 - NEAR).
So the forward (and the KV-cache split merge) gives out = rne_out(f32(O) / f32(l)): the kernels divide with __fdiv_rn, and
numpy's f32 division rounds the same way.
The backward is modelled on rows with l = 2^n, where out and delta = dout . out are exact: dS = (w / l)(dP - delta) must be
exactly representable in the input dtype (checked), so the few-ulp error of p from the lse round trip (lse in natural log,
L = lse * log2 e in f32) cannot change its rounding while |scores| stay small.  Then dv = rne_grad(sum P dout),
dq = rne_grad(f32(f32(ln 2) sum dS k)) and dk = rne_grad(f32(f32(ln 2) sum over group heads and rows of dS q)).
Every function checks its preconditions and refuses a case that breaks them.

Inputs are built on a grid of tie classes: key j has one-hot features for its class and for its slot, so a query row picks a
class with a large weight and gives each slot of that class an integer offset: weighted (0 .. -NEAR), far, or a decoy that
would dominate the row if a mask let it through.  Every value is a small integer both 16-bit dtypes hold exactly."""
from __future__ import annotations

import math

import numpy as np

import gemm_exact_oracle as ge

LN2 = math.log(2.0)
NEAR = 8                 # weights 2^0 .. 2^-8
FAR = 136                # far keys: p = +0 against every running maximum
CLASS_W = 160            # class weight: keys of other classes score at least this far below the row's keys
FAR_OFFSET = -200        # slot offset of a key of the row's class that must not count
DECOY = 16               # slot offset of a masked key that would dominate its row
MAX_SCORE = 60           # |row maximum| bound: keeps the backward's lse round-trip error of p a few ulps


def scale_log2():
    return np.float32(np.float64(np.float32(LN2)) * 1.4426950408889634074)


def _f32_exact_sum(terms, axis) -> None:
    """Every partial sum of `terms` (dyadic values) along `axis`, in any order, is a multiple of the finest term's last bit
    below 2^24 of them, so exact in f32."""
    t = np.abs(np.asarray(terms, dtype=np.float64))
    nz = t[t > 0]
    if nz.size == 0:
        return
    m, e = np.frexp(nz)
    n = (m * 2.0 ** 53).astype(np.int64)
    grain = float(((n & -n).astype(np.float64) * np.exp2(e - 53.0)).min())
    assert t.sum(axis=axis).max() < 2.0 ** 24 * grain, "a partial sum could round in f32"


# ------------------------------------------------------------------------------------------------ inputs
def grid_keys(Sk, D, P, slots, order="periodic"):
    """k [Sk, D] of the class grid: dims [0, P) one-hot class, [P, P + slots) one-hot slot, P + slots the bias dim.
    periodic: class j % P, slot j // P (keys P apart share a class); blocked: class j // slots, slot j % slots."""
    assert P + slots + 1 <= D, "the class grid does not fit in the head dim"
    assert Sk <= P * slots
    j = np.arange(Sk)
    cls, slot = (j % P, j // P) if order == "periodic" else (j // slots, j % slots)
    k = np.zeros((Sk, D))
    k[j, cls] = 1.0
    k[j, P + slot] = 1.0
    k[:, P + slots] = 1.0
    return k, cls, slot


def grid_query(D, P, slots, cls, offsets, r):
    """One query row: class `cls`, slot offsets {slot: integer offset} (every other slot FAR_OFFSET), row maximum -r."""
    q = np.zeros(D)
    q[cls] = CLASS_W
    q[P:P + slots] = FAR_OFFSET
    for s, o in offsets.items():
        q[P + s] = o
    q[P + slots] = -(CLASS_W + r)
    return q


def key_of(cls, slot, P, slots, order="periodic"):
    return slot * P + cls if order == "periodic" else cls * slots + slot


# ------------------------------------------------------------------------------------------------ the model
def scores(q, k):
    """Integer scores q . k, exact in f32 (checked)."""
    s = np.einsum("...id,...jd->...ij", q, k)
    assert np.array_equal(s, np.round(s)), "scores must be integers"
    assert np.einsum("...id,...jd->...ij", np.abs(q), np.abs(k)).max() < 2.0 ** 24
    return s


def weights(s, vis):
    """(w, m): w = 2^(s - m) on visible keys within NEAR of the row maximum m, else 0; asserts the score bands."""
    s = np.where(vis, s, -np.inf)
    m = s.max(axis=-1, keepdims=True)
    rows = np.isfinite(m)
    assert np.all(np.abs(m[rows]) <= MAX_SCORE), "a row maximum is too large for the lse round trip"
    with np.errstate(invalid="ignore"):
        e = np.where(vis & rows, m - s, 0.0)
    assert np.all((e <= NEAR) | (e >= FAR)), "a visible score lies between NEAR and FAR below its row maximum"
    w = np.where(vis & rows & (e <= NEAR), np.exp2(-e), 0.0)
    return w, np.where(rows, m, -np.inf)[..., 0]


def forward(q, k, v, vis, out_dtype):
    """q [B, Hq, Sq, D], k, v [B, Hkv, Sk, D], vis broadcastable to [B, Hq, Sq, Sk] -> (out bits, w, l).  Rows with no visible
    key give +0."""
    G = q.shape[1] // k.shape[1]
    kk, vv = np.repeat(k, G, axis=1), np.repeat(v, G, axis=1)
    vis = np.broadcast_to(vis, q.shape[:3] + (k.shape[2],))
    w, _ = weights(scores(q, kk), vis)
    # a running O or l sums p <= 1 times v on a grain of 2^-NEAR (times v's): exact below 2^(24 - NEAR) of integer v
    assert np.array_equal(vv, np.round(vv)), "v must be integers"
    assert np.einsum("bhij,bhjd->bhid", (w > 0).astype(np.float64), np.abs(vv)).max() < 2.0 ** (24 - NEAR)
    l = w.sum(axis=-1)
    O = np.einsum("bhij,bhjd->bhid", w, vv)
    with np.errstate(invalid="ignore", divide="ignore"):
        out = np.where(l[..., None] > 0, O.astype(np.float32) / l[..., None].astype(np.float32), np.float32(0))
    return ge.rne(out, out_dtype), w, l


def rounds_exactly(x, dtype):
    return np.array_equal(ge.bits_to_f64(ge.rne(x, dtype), dtype), np.asarray(x, dtype=np.float64))


def backward(q, k, v, dout, vis, in_dtype, out_dtype, grad_dtype, mutant=None, vis_dq=None, vis_dkdv=None):
    """(dq, dk, dv) bits for rows with l = 2^n.  mutant: one of BACKWARD_MUTANTS, a kernel that gets one step wrong.
    vis_dq / vis_dkdv: a wrong mask in the dq kernel or in the dk / dv kernel alone (each recomputes p = 2^(t - L) from the
    forward's L = m + log2 l, so a key it wrongly lets through gets its unnormalised weight, a masked decoy 2^DECOY)."""
    B, Hq, Sq, D = q.shape
    Hkv, Sk = k.shape[1], k.shape[2]
    G = Hq // Hkv
    out_bits, w, l = forward(q, k, v, vis, out_dtype)
    live = l > 0
    assert np.all(l[live] == np.exp2(np.round(np.log2(l[live])))), "backward rows need l = 2^n"
    out = ge.bits_to_f64(out_bits, out_dtype)
    kk, vv = np.repeat(k, G, axis=1), np.repeat(v, G, axis=1)
    dterms = dout * out
    _f32_exact_sum(dterms, axis=-1)
    delta = dterms.sum(axis=-1)
    if mutant == "delta_from_next_row":
        delta = np.concatenate([delta[..., 1:], delta[..., :1]], axis=-1)
    dp = np.einsum("bhid,bhjd->bhij", dout, vv)
    s = scores(q, kk)
    m = np.where(np.broadcast_to(vis, s.shape), s, -np.inf).max(axis=-1)
    L = np.where(live, m + np.log2(np.where(live, l, 1.0)), np.inf)[..., None]   # rows that see nothing: L = +inf, p = +0
    wrong = vis_dq is not None or vis_dkdv is not None

    def p_ds(mask):
        with np.errstate(invalid="ignore"):
            t = np.where(np.broadcast_to(mask, s.shape), s - L, -np.inf)
        P = np.where(t > -127, np.exp2(np.minimum(t, 1000)), 0.0)
        ds = P * (dp - delta[..., None])
        assert mutant or wrong or rounds_exactly(ds, in_dtype), "dS is not exactly representable in the input dtype"
        return P, ge.bits_to_f64(ge.rne(ds, in_dtype), in_dtype)

    P, ds = p_ds(vis)
    assert np.array_equal(P, np.where(live[..., None], w / np.where(live, l, 1.0)[..., None], 0.0))
    ds_q = ds if vis_dq is None else p_ds(vis_dq)[1]
    if vis_dkdv is not None:
        P, ds = p_ds(vis_dkdv)
    check = _f32_exact_sum if not (mutant or wrong) else (lambda *a, **kw: None)
    s32 = np.float32(LN2)
    vt = P[..., None] * dout[..., :, None, :]                       # [B, Hq, Sq, Sk, D]
    check(vt.reshape(B, Hkv, G * Sq, Sk, D), axis=2)
    dv = vt.reshape(B, Hkv, G, Sq, Sk, D).sum(axis=(2, 3))
    qt = ds_q[..., None] * kk[..., None, :, :]
    check(qt, axis=-2)
    dq_sum = qt.sum(axis=-2).astype(np.float32)
    dq = dq_sum if mutant == "dq_without_scale" else s32 * dq_sum
    kt = (ds[..., None] * q[..., :, None, :]).reshape(B, Hkv, G, Sq, Sk, D)
    if mutant == "dk_missing_a_group_head":
        kt = kt[:, :, :-1]
    check(kt.reshape(B, Hkv, -1, Sk, D), axis=2)
    dk = s32 * kt.sum(axis=(2, 3)).astype(np.float32)
    with np.errstate(over="ignore"):
        return ge.rne(dq, grad_dtype), ge.rne(dk, grad_dtype), ge.rne(dv, grad_dtype)


BACKWARD_MUTANTS = ("dq_without_scale", "dk_missing_a_group_head", "delta_from_next_row")


# ------------------------------------------------------------------------------------------------ online order (mutants)
def online_forward(s, v, vis, block, out_dtype, rescale=True):
    """The forward as the kernels run it, key block by key block in f64 (exact on these inputs): p = 2^(t - m) (+0 below
    -126), O and l rescaled by 2^(m_old - m_new) (or not at all: rescale=False, the mutant).  s [.., Sq, Sk] scores,
    v [.., Sk, D] values."""
    sk = s.shape[-1]
    s = np.where(vis, s, -np.inf)
    m = np.full(s.shape[:-1], -np.inf)
    l = np.zeros(s.shape[:-1])
    O = np.zeros(s.shape[:-1] + (v.shape[-1],))
    ex2 = lambda x: np.where(x > -127, np.exp2(np.maximum(x, -127)), 0.0)  # noqa: E731
    for j0 in range(0, sk, block):
        blk = s[..., j0:j0 + block]
        mn = np.maximum(m, blk.max(axis=-1))
        z = np.where(np.isfinite(mn), mn, 0.0)
        a = ex2(np.where(np.isfinite(m), m - z, -np.inf)) if rescale else np.ones_like(m)
        p = ex2(blk - z[..., None])
        l = l * a + p.sum(axis=-1)
        O = O * a[..., None] + np.einsum("...ij,...jd->...id", p, v[..., j0:j0 + block, :])
        m = mn
    with np.errstate(invalid="ignore", divide="ignore"):
        out = np.where(l[..., None] > 0, O.astype(np.float32) / l[..., None].astype(np.float32), np.float32(0))
    return ge.rne(out, out_dtype)


def rescale_exponents(s, vis, block):
    """Set of k > 0 for which some row meets a rescale factor 2^-k (m_old finite and within NEAR of the new maximum)."""
    s = np.where(vis, s, -np.inf)
    m = np.full(s.shape[:-1], -np.inf)
    seen = set()
    for j0 in range(0, s.shape[-1], block):
        mn = np.maximum(m, s[..., j0:j0 + block].max(axis=-1))
        d = (mn - m)[np.isfinite(m)]
        seen |= {int(x) for x in np.unique(d) if 0 < x <= NEAR}
        m = mn
    return seen


def split_forward(s, v, vis, splits, out_dtype, merge=True):
    """The split-KV forward: each key range [a, b) of `splits` gives (m_s, l_s, O_s) and the combine merges them with weights
    2^(m_s - m) (merge=False: weights forced to 1, the mutant)."""
    s = np.where(vis, s, -np.inf)
    parts = []
    for a, b in splits:
        blk = s[..., a:b]
        ms = blk.max(axis=-1)
        z = np.where(np.isfinite(ms), ms, 0.0)
        p = np.where(np.isfinite(blk), np.exp2(np.maximum(blk - z[..., None], -1074)), 0.0)
        p = np.where(blk - z[..., None] > -127, p, 0.0)
        parts.append((ms, p.sum(axis=-1), np.einsum("...ij,...jd->...id", p, v[..., a:b, :])))
    m = np.max([ms for ms, _, _ in parts], axis=0)
    l = np.zeros(m.shape)
    O = np.zeros(m.shape + (v.shape[-1],))
    for ms, ls, Os in parts:
        wgt = np.where(np.isfinite(ms), np.exp2(np.where(np.isfinite(ms), ms - np.where(np.isfinite(m), m, 0.0), 0.0)), 0.0)
        wgt = np.where(wgt >= 2.0 ** -126, wgt, 0.0)
        if not merge:
            wgt = np.where(np.isfinite(ms), 1.0, 0.0)
        l = l + wgt * ls
        O = O + wgt[..., None] * Os
    with np.errstate(invalid="ignore", divide="ignore"):
        out = np.where(l[..., None] > 0, O.astype(np.float32) / l[..., None].astype(np.float32), np.float32(0))
    return ge.rne(out, out_dtype)


def merge_exponents(s, vis, splits):
    """Set of k >= 0 for which some row merges a split with weight 2^-k (k <= NEAR)."""
    s = np.where(vis, s, -np.inf)
    ms = np.stack([s[..., a:b].max(axis=-1) for a, b in splits], axis=-1)
    m = ms.max(axis=-1, keepdims=True)
    d = (m - ms)[np.isfinite(ms) & np.isfinite(m)]
    return {int(x) for x in np.unique(d) if x <= NEAR}
