"""GPU: attention outputs checked bit for bit on power-of-two softmax weights (tests/attention_exact_oracle.py).

The one-hot and uniform exact tests only ever give p = 0 or 1, and their backward has dS = 0.  Here every row has several
weighted keys with p = 2^-k, the row maximum arrives after earlier weighted blocks (so the online rescale factors 2^-1 ..
2^-8 occur), KV-cache rows weight keys in several splits with the maximum in a later one (merge weights 2^-k), and backward
rows have l = 2^n with nonzero dS, so the dS products, the final multiply by scale and the GQA sum of dK are exact too.
tests/test_attention_exact_weights_cpu.py checks the generators against the model's preconditions, the model against the
f64 oracles, and that each case would fail under a kernel that gets the rescale, merge, mask, scale, group sum or delta
wrong."""
import numpy as np
import pytest

import attention_exact_oracle as xo
import attention_kvcache_oracle as ko
import attention_varlen_oracle as vo
from cubecl_b200 import attention
from test_attention_gpu import bits, up
from test_attention_kvcache_gpu import layout, up_i32

pytestmark = pytest.mark.gpu

# backward rows: exponent patterns (relative to the row maximum) whose weights sum to a power of two
POW2_PATTERNS = ((0,), (0, 0), (1, 1, 0), (0, 0, 0, 0), (2, 2, 1, 0), (2, 2, 2, 2, 0), (3, 3, 2, 1, 0))


def _grid(Sk, D):
    slots = min((D - 1) // 2, 24)
    P = -(-Sk // slots)
    assert P + slots + 1 <= D
    return P, slots


def _visible_slots(c, P, slots, limit):
    return [s for s in range(slots) if s * P + c < limit]


def dense_problem(B, Hq, Hkv, Sq, Sk, D, causal, seed, backward=False):
    """q, k, v (and dout) on the periodic class grid.  Forward rows weight a random subset of their class's visible keys with
    2^-1 .. 2^-8 and put the maximum on the last visible one.  When causal, every third row's maximum is the diagonal key
    itself, and in every third row the masked key i + 1 is a decoy that would dominate the row (forward and backward).
    Backward rows
    use POW2_PATTERNS, so l = 2^n, with small v and a dout of two +-1 entries per row."""
    rng = np.random.default_rng(seed)
    P, slots = _grid(Sk, D)
    k1, _, _ = xo.grid_keys(Sk, D, P, slots)
    k = np.broadcast_to(k1, (B, Hkv, Sk, D)).copy()
    q = np.zeros((B, Hq, Sq, D))
    for b in range(B):
        for h in range(Hq):
            for i in range(Sq):
                limit = min(i + 1, Sk) if causal else Sk
                decoy = causal and i % 3 == 1 and P <= i + 1 < Sk   # key i + 1, masked, would dominate the row
                if causal and i % 3 == 0 and i < Sk:
                    c = i % P                                      # the diagonal key itself is the row maximum
                elif decoy:
                    c = (i + 1) % P
                else:
                    c = int(rng.integers(0, min(P, limit)))
                vs = _visible_slots(c, P, slots, limit)
                if backward:
                    pats = [p for p in POW2_PATTERNS if len(p) <= len(vs)]
                    pat = pats[int(rng.integers(0, len(pats)))]
                    chosen = sorted(rng.choice(vs[:-1], size=len(pat) - 1, replace=False).tolist()) + [vs[-1]] if len(pat) > 1 else [vs[-1]]
                    offsets = {s: -e for s, e in zip(chosen, pat)}
                else:
                    offsets = {s: -int(rng.integers(1, xo.NEAR + 1)) for s in vs[:-1] if rng.random() < 0.6}
                    offsets[vs[-1]] = 0
                if decoy:
                    offsets[(i + 1) // P] = xo.DECOY
                q[b, h, i] = xo.grid_query(D, P, slots, c, offsets, int(rng.integers(1, 50)))
    if backward:
        v = rng.integers(-3, 4, (B, Hkv, Sk, D)).astype(np.float64)
        dout = np.zeros((B, Hq, Sq, D))
        i4 = np.arange(Sq)
        for d0 in (0, 7):
            dout[..., i4, (i4 * 5 + d0) % D] = rng.choice([-1.0, 1.0], (B, Hq, Sq))
        return q, k, v, dout
    v = rng.integers(-64, 65, (B, Hkv, Sk, D)).astype(np.float64)
    return q, k, v


def dense_vis(Sq, Sk, causal):
    if not causal:
        return np.ones((Sq, Sk), bool)
    return np.arange(Sk)[None, :] <= np.arange(Sq)[:, None]


# ---------------------------------------------------------------------------------------------- dense forward
FORWARD_CASES = [   # B, Hq, Hkv, Sq, Sk, D, causal
    (1, 4, 2, 300, 333, 40, False), (2, 2, 1, 333, 333, 40, True), (1, 4, 1, 257, 429, 64, False), (1, 2, 2, 429, 429, 64, True),
    (1, 3, 1, 200, 390, 96, False), (1, 4, 2, 390, 390, 96, True), (1, 2, 1, 150, 555, 128, False), (1, 4, 2, 555, 555, 128, True),
]
FORWARD_IDS = [f"D{c[5]}-{'causal' if c[6] else 'full'}-G{c[1] // c[2]}-{c[3]}x{c[4]}" for c in FORWARD_CASES]


@pytest.mark.parametrize("dtype", ["bf16", "f16"])
@pytest.mark.parametrize("B,Hq,Hkv,Sq,Sk,D,causal", FORWARD_CASES, ids=FORWARD_IDS)
def test_dense_forward_is_exact_on_power_of_two_weights(client, dtype, B, Hq, Hkv, Sq, Sk, D, causal):
    q, k, v = dense_problem(B, Hq, Hkv, Sq, Sk, D, causal, seed=Sq + Sk + D)
    qh, kh, vh = (up(client, t, dtype) for t in (q, k, v))
    for od in (dtype, "f32"):
        want, _, _ = xo.forward(q, k, v, dense_vis(Sq, Sk, causal), od)
        out = attention.launch_alloc(client, qh, kh, vh, scale=xo.LN2, causal=causal, out_dtype=od)
        client.sync()
        xo.ge.assert_bits_equal(bits(client, out).reshape(want.shape), want, od, f"forward -> {od}")


# ---------------------------------------------------------------------------------------------- dense backward
BACKWARD_CASES = [   # B, Hq, Hkv, Sq, Sk, D, causal
    (1, 4, 2, 150, 190, 40, False), (1, 4, 2, 190, 190, 40, True), (1, 3, 1, 100, 250, 64, False), (2, 2, 1, 129, 129, 64, True),
    (1, 4, 1, 77, 300, 128, False), (1, 4, 2, 200, 200, 128, True),
]
BACKWARD_IDS = [f"D{c[5]}-{'causal' if c[6] else 'full'}-G{c[1] // c[2]}-{c[3]}x{c[4]}" for c in BACKWARD_CASES]


@pytest.mark.parametrize("dtype", ["bf16", "f16"])
@pytest.mark.parametrize("B,Hq,Hkv,Sq,Sk,D,causal", BACKWARD_CASES, ids=BACKWARD_IDS)
def test_dense_backward_is_exact_with_nonzero_ds(client, dtype, B, Hq, Hkv, Sq, Sk, D, causal):
    q, k, v, dout = dense_problem(B, Hq, Hkv, Sq, Sk, D, causal, seed=Sq + Sk + D, backward=True)
    qh, kh, vh, doh = (up(client, t, dtype) for t in (q, k, v, dout))
    vis = dense_vis(Sq, Sk, causal)
    for od, gd in ((dtype, dtype), ("f32", "f32"), (dtype, "f32")):
        want = xo.backward(q, k, v, dout, vis, dtype, od, gd)
        out, lse = attention.launch_alloc(client, qh, kh, vh, scale=xo.LN2, causal=causal, out_dtype=od, return_lse=True)
        grads = attention.launch_backward_alloc(client, qh, kh, vh, out, doh, lse, scale=xo.LN2, causal=causal, grad_dtype=gd)
        client.sync()
        for name, g, w in zip(("dq", "dk", "dv"), grads, want):
            xo.ge.assert_bits_equal(bits(client, g).reshape(w.shape), w, gd, f"{name} (out {od}, grad {gd})")


# ---------------------------------------------------------------------------------------------- KV cache with several splits
KV_CASES = [   # B, Hq, Hkv, Sq, D, page, pages per sequence, causal, dtype
    (2, 4, 1, 1, 64, 64, 12, False, "bf16"),
    (2, 8, 2, 3, 128, 16, 64, True, "bf16"),
    (1, 4, 1, 3, 64, 256, 3, True, "f16"),
    (3, 2, 1, 1, 128, 64, 12, True, "f16"),
]


def kv_splits(B, Hq, Hkv, Sq, cap, sms=132):
    """the key ranges of the split-KV launch, as b200_attention_kvcache plans it on `sms` SMs (an H100 SXM has 132)"""
    gt, st = ko.kv_tile(Hq // Hkv, Sq)
    nkb = -(-cap // 64)
    n = ko.kv_splits(B * Hkv * -(-(Hq // Hkv) // gt) * -(-Sq // st), nkb, sms)
    bps = -(-nkb // n)
    return [(s * bps * 64, min((s + 1) * bps * 64, cap)) for s in range(n)]


def kv_problem(B, Hq, Hkv, Sq, D, cap, lens, causal, seed):
    """q, k, v [B, Hkv, cap, D] and vis [B, 1, Sq, cap]: each row weights keys of its class in several splits, the maximum on
    its last visible key of the class, earlier ones 2^-1 .. 2^-8.  Even heads take the class of the row's last visible key;
    when causal, odd heads of rows that stop short of L_b take the class of the first masked key, a decoy that would
    dominate the row."""
    rng = np.random.default_rng(seed)
    P, slots = _grid(cap, D)
    k1, _, _ = xo.grid_keys(cap, D, P, slots)
    k = np.broadcast_to(k1, (B, Hkv, cap, D)).copy()
    q = np.zeros((B, Hq, Sq, D))
    vis = np.zeros((B, 1, Sq, cap), bool)
    for b, L in enumerate(lens):
        for i in range(Sq):
            limit = min(L, L - Sq + i + 1) if causal else L
            vis[b, 0, i, :max(limit, 0)] = True
            if limit <= 0:
                continue
            for h in range(Hq):
                decoy = causal and h % 2 == 1 and P <= limit < L   # the first masked key would dominate the row
                c = limit % P if decoy else (limit - 1) % P if h % 2 == 0 else int(rng.integers(0, min(P, limit)))
                vs = _visible_slots(c, P, slots, limit)
                offsets = {s: -int(rng.integers(1, xo.NEAR + 1)) for s in vs[:-1] if rng.random() < 0.5}
                offsets[vs[-1]] = 0
                if decoy:
                    offsets[limit // P] = xo.DECOY
                q[b, h, i] = xo.grid_query(D, P, slots, c, offsets, int(rng.integers(1, 50)))
    v = rng.integers(-64, 65, (B, Hkv, cap, D)).astype(np.float64)
    return q, k, v, vis


def kv_lens(B, cap):
    return [cap - 1 - 37 * b if b % 2 == 0 else cap - 64 * b - 5 for b in range(B)]


@pytest.mark.parametrize("B,Hq,Hkv,Sq,D,page,mp,causal,dtype", KV_CASES)
def test_kvcache_split_merge_is_exact_on_power_of_two_weights(client, B, Hq, Hkv, Sq, D, page, mp, causal, dtype):
    cap = page * mp
    lens = kv_lens(B, cap)
    q, k, v, vis = kv_problem(B, Hq, Hkv, Sq, D, cap, lens, causal, seed=cap + Sq)
    assert len(kv_splits(B, Hq, Hkv, Sq, cap, client.properties["num_streaming_multiprocessors"])) > 1
    kc, vc, bt = layout(client, k, v, lens, page, "paged", dtype, seed=Sq)
    qh = up(client, q, dtype)
    for od in (dtype, "f32"):
        want, _, _ = xo.forward(q, k, v, vis, od)
        out = attention.launch_kvcache_alloc(client, qh, kc, vc, up_i32(client, lens), block_table=bt, scale=xo.LN2, causal=causal,
                                             out_dtype=od)
        client.sync()
        assert "combine" in client.last_kernel(), client.last_kernel()   # several splits, merged by the combine kernel
        xo.ge.assert_bits_equal(bits(client, out).reshape(want.shape), want, od, f"kvcache -> {od}")


# ---------------------------------------------------------------------------------------------- varlen forward and backward
# (lens_q, lens_k) per case: Lq > Lk and Lq < Lk, an empty sequence and length-1 sequences
VARLEN_LENS = ([150, 0, 1, 1, 97, 200], [110, 0, 1, 5, 130, 200])
VARLEN_WINDOWS = [(-1, 0), (40, 0), (40, 20), (0, 40)]
VARLEN_IDS = [f"w{a}_{b}" for a, b in VARLEN_WINDOWS]


def varlen_edges(i, Lq, Lk, window):
    """the unclipped band edges of row i: (edge key, the key one position outside it) for the left and right edge"""
    left, right = window
    off = Lk - Lq
    edges = []
    if left >= 0 and 1 <= i + off - left <= Lk - 1:
        edges.append((i + off - left, i + off - left - 1))
    if right >= 0 and 0 <= i + off + right <= Lk - 2:
        edges.append((i + off + right, i + off + right + 1))
    return edges


def varlen_problem(lens_q, lens_k, Hq, Hkv, D, window, seed, backward=False):
    """Packed q [Tq, Hq, D], k, v [Tk, Hkv, D] (and dout) on the blocked class grid of each sequence (class = j // slots, so
    consecutive keys share a class).  Each row with an unclipped band edge takes the class of an edge key, weights it, and
    makes the key one position outside the band a decoy when it is of the same class; other rows take the class of a random
    visible key.  Forward weights are 2^0 .. 2^-8, backward rows follow POW2_PATTERNS (l = 2^n)."""
    rng = np.random.default_rng(seed)
    Tq, Tk = sum(lens_q), sum(lens_k)
    q, k = np.zeros((Tq, Hq, D)), np.zeros((Tk, Hkv, D))
    qa = ka = 0
    for Lq, Lk in zip(lens_q, lens_k):
        if Lk:
            P, slots = _grid(Lk, D)
            k[ka:ka + Lk] = xo.grid_keys(Lk, D, P, slots, order="blocked")[0][:, None, :]
        vis = vo.band_mask(Lq, Lk, window)
        for i in range(Lq):
            seen = np.flatnonzero(vis[i])
            if seen.size == 0:
                continue
            for h in range(Hq):
                edges = varlen_edges(i, Lq, Lk, window)
                edge, out = edges[(i + h) % len(edges)] if edges and (i + h) % 4 else (int(rng.choice(seen)), -1)
                c = edge // slots
                vs = [j % slots for j in seen if j // slots == c]
                es = edge % slots
                others = [x for x in vs if x != es]
                if backward:
                    pats = [p for p in POW2_PATTERNS if len(p) <= len(vs)]
                    pat = pats[int(rng.integers(0, len(pats)))]
                    chosen = [es] + (rng.choice(others, size=len(pat) - 1, replace=False).tolist() if len(pat) > 1 else [])
                    rng.shuffle(chosen)
                    offsets = {x: -e for x, e in zip(chosen, pat)}
                else:
                    offsets = {x: -int(rng.integers(1, xo.NEAR + 1)) for x in others if rng.random() < 0.6}
                    offsets[es] = -int(rng.integers(0, 3))
                    offsets[int(rng.choice(vs)) if offsets[es] else es] = 0
                if 0 <= out and out // slots == c:
                    offsets[out % slots] = xo.DECOY
                q[qa + i, h] = xo.grid_query(D, P, slots, c, offsets, int(rng.integers(1, 50)))
        qa, ka = qa + Lq, ka + Lk
    if backward:
        v = rng.integers(-3, 4, (Tk, Hkv, D)).astype(np.float64)
        dout = np.zeros((Tq, Hq, D))
        r = np.arange(Tq)
        for d0 in (0, 7):
            dout[r, :, (r * 5 + d0) % D] = rng.choice([-1.0, 1.0], (Tq, Hq))
        return q, k, v, dout
    return q, k, rng.integers(-64, 65, (Tk, Hkv, D)).astype(np.float64)


def varlen_seqs(lens_q, lens_k):
    """(query rows, key rows) slices of every sequence"""
    cq, ck = np.cumsum([0] + list(lens_q)), np.cumsum([0] + list(lens_k))
    return [(slice(cq[b], cq[b + 1]), slice(ck[b], ck[b + 1])) for b in range(len(lens_q))]


def _bhsd(t):
    return t.transpose(1, 0, 2)[None]


def varlen_forward(q, k, v, lens_q, lens_k, window, out_dtype):
    """the model per sequence, packed back: out bits [Tq, Hq, D]"""
    out = np.zeros(q.shape, xo.ge.OUT_BITS_VIEW[out_dtype])
    for (sq, sk), Lq, Lk in zip(varlen_seqs(lens_q, lens_k), lens_q, lens_k):
        if Lq and Lk:
            out[sq] = xo.forward(_bhsd(q[sq]), _bhsd(k[sk]), _bhsd(v[sk]), vo.band_mask(Lq, Lk, window), out_dtype)[0][0].transpose(1, 0, 2)
    return out


def varlen_backward(q, k, v, dout, lens_q, lens_k, window, in_dtype, out_dtype, grad_dtype, mask_dq=None, mask_dkdv=None):
    """(dq, dk, dv) bits packed; mask_dq / mask_dkdv: (Lq, Lk) -> a wrong [Lq, Lk] mask in one backward kernel only"""
    view = xo.ge.OUT_BITS_VIEW[grad_dtype]
    dq, dk, dv = np.zeros(q.shape, view), np.zeros(k.shape, view), np.zeros(k.shape, view)
    for (sq, sk), Lq, Lk in zip(varlen_seqs(lens_q, lens_k), lens_q, lens_k):
        if not (Lq and Lk):
            continue
        mask = lambda f: None if f is None else f(Lq, Lk)   # noqa: E731
        g = xo.backward(_bhsd(q[sq]), _bhsd(k[sk]), _bhsd(v[sk]), _bhsd(dout[sq]), vo.band_mask(Lq, Lk, window), in_dtype, out_dtype,
                        grad_dtype, vis_dq=mask(mask_dq), vis_dkdv=mask(mask_dkdv))
        dq[sq], dk[sk], dv[sk] = (x[0].transpose(1, 0, 2) for x in g)
    return dq, dk, dv


VARLEN_SHAPE = dict(Hq=4, Hkv=2, D=64)


@pytest.mark.parametrize("dtype", ["bf16", "f16"])
@pytest.mark.parametrize("window", VARLEN_WINDOWS, ids=VARLEN_IDS)
def test_varlen_forward_and_backward_are_exact_at_the_window_edges(client, dtype, window):
    lq, lk = VARLEN_LENS
    Hq, Hkv, D = VARLEN_SHAPE["Hq"], VARLEN_SHAPE["Hkv"], VARLEN_SHAPE["D"]
    cq, ck = (up_i32(client, np.cumsum([0] + list(x))) for x in (lq, lk))
    mq, mk = max(lq), max(lk)
    q, k, v = varlen_problem(lq, lk, Hq, Hkv, D, window, seed=sum(window) + 11)
    qh, kh, vh = (up(client, t, dtype) for t in (q, k, v))
    for od in (dtype, "f32"):
        out = attention.launch_varlen_alloc(client, qh, kh, vh, cq, ck, mq, mk, scale=xo.LN2, window_size=window, out_dtype=od)
        client.sync()
        xo.ge.assert_bits_equal(bits(client, out).reshape(q.shape), varlen_forward(q, k, v, lq, lk, window, od), od, f"varlen -> {od}")
    q, k, v, dout = varlen_problem(lq, lk, Hq, Hkv, D, window, seed=sum(window) + 12, backward=True)
    qh, kh, vh, doh = (up(client, t, dtype) for t in (q, k, v, dout))
    for od, gd in ((dtype, dtype), ("f32", "f32")):
        want = varlen_backward(q, k, v, dout, lq, lk, window, dtype, od, gd)
        out, lse = attention.launch_varlen_alloc(client, qh, kh, vh, cq, ck, mq, mk, scale=xo.LN2, window_size=window, out_dtype=od,
                                                 return_lse=True)
        grads = attention.launch_varlen_backward_alloc(client, qh, kh, vh, out, doh, lse, cq, ck, mq, mk, scale=xo.LN2,
                                                       window_size=window, grad_dtype=gd)
        client.sync()
        for name, g, w in zip(("dq", "dk", "dv"), grads, want):
            xo.ge.assert_bits_equal(bits(client, g).reshape(w.shape), w, gd, f"varlen {name} (out {od}, grad {gd})")
