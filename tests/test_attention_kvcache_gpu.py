"""GPU: b200_attention_kvcache and b200_kvcache_write on an H100.

Exact contracts (integer-valued operands, so every score and every p is exact):
- one-hot rows: every row's chosen visible key scores at least 128 / scale above every other visible key and below 0, so a
  zero-filled or stale key that leaked through the length mask would win; with causal, the last valid key is a decoy that
  scores higher still for every row that must not see it.  out must be v[chosen] bit for bit, rows with no visible key +0
  with lse -inf.  Shuffled pages of 16, 64 and 256 keys and the identity table, ragged lengths (0, 1, a page boundary +- 1,
  full capacity), Sq in {1, 3, 17}, G in {1, 4, 8, 128}, shapes with one split and with several.
- uniform rows: q = 0 gives the exact column mean of v[:L_b], for one split and several.
Stale slots (NaN, +-inf) against a zero-filled cache, layout invariance, random data against the f64 oracle and against
b200_attention, reproducibility across repeats and streams, and the cache scatter."""
import numpy as np
import pytest

import attention_kvcache_oracle as ko
from cubecl_b200 import ServerError, TensorHandle, attention
from test_attention_gpu import ONE_HOT, _bound, _digits, bits, rounded, up, values

pytestmark = pytest.mark.gpu


def up_i32(client, a):
    return TensorHandle.from_numpy(client, np.ascontiguousarray(a, dtype=np.int32), "i32")


def layout(client, k, v, lens, page, kind, dtype, fill=0.0, seed=0):
    """k, v [B, Hkv, cap, D] (logical) -> (k_cache, v_cache, block_table) handles.  Slots at or past L_b and unused pages hold
    `fill` (a value, or "nan" / "inf" for NaN / alternating +-inf); table entries past ceil(L_b / page) are -1.
    kind: "identity" (no table, [B, cap, Hkv, D]), "paged" (shuffled [P, page, Hkv, D] pages plus 3 unused ones), "headmajor"
    (the same pages stored [P, Hkv, page, D] and passed as a view)."""
    B, Hkv, cap, D = k.shape
    rng = np.random.default_rng(seed)

    def stale(shape):
        if fill == "nan":
            return np.full(shape, np.nan)
        if fill == "inf":
            return np.where(rng.random(shape) < 0.5, np.inf, -np.inf)
        return np.full(shape, float(fill))

    out = []
    mp = cap // page
    P = B * mp + 3
    perm = rng.permutation(P)
    table = perm[:B * mp].reshape(B, mp).copy()
    for b, L in enumerate(lens):
        table[b, -(-L // page):] = -1
    for t in (k, v):
        t = t.copy()
        for b, L in enumerate(lens):
            t[b, :, L:] = stale(t[b, :, L:].shape)
        if kind == "identity":
            out.append(up(client, t.transpose(0, 2, 1, 3), dtype))
            continue
        cache = stale((P, page, Hkv, D))
        for b in range(B):
            for p in range(mp):
                cache[perm[b * mp + p]] = t[b, :, p * page:(p + 1) * page].transpose(1, 0, 2)
        if kind == "paged":
            out.append(up(client, cache, dtype))
        else:
            h = up(client, cache.transpose(0, 2, 1, 3), dtype)
            out.append(TensorHandle(h.handle, [P, page, Hkv, D], [Hkv * page * D, D, page * D, 1], dtype))
    return out[0], out[1], (None if kind == "identity" else up_i32(client, table))


def run(client, q, kc, vc, bt, lens, dtype, out_dtype, scale=None, causal=False, q_view=None):
    qh = up(client, q, dtype) if q_view is None else q_view
    res = attention.launch_kvcache_alloc(client, qh, kc, vc, up_i32(client, lens), block_table=bt, scale=scale, causal=causal,
                                         out_dtype=out_dtype, return_lse=True)
    client.sync()
    return values(client, res[0]), values(client, res[1]), bits(client, res[0])


def nsplit(B, Hq, Hkv, Sq, cap, sms=132):
    gt, st = ko.kv_tile(Hq // Hkv, Sq)
    return ko.kv_splits(B * Hkv * -(-(Hq // Hkv) // gt) * -(-Sq // st), -(-cap // 64), sms)


def ragged(B, cap, page, rng):
    """lengths cycling through 0, 1, page - 1, page, page + 1, cap and a random one"""
    pool = [0, 1, page - 1, page, page + 1, cap, int(rng.integers(2, cap))]
    off = int(rng.integers(0, 7))
    return [min(pool[(b + off) % 7], cap) for b in range(B)]


# ---------------------------------------------------------------------------------------------- exact: one-hot rows
def one_hot_kv(B, Hq, Hkv, Sq, cap, D, lens, causal, dtype, seed):
    G, C, _ = ONE_HOT[dtype]
    rng = np.random.default_rng(seed)
    j = np.arange(cap)
    k = np.zeros((B, Hkv, cap, D))
    k[..., 0:3] = _digits(j)
    k[..., 3:6] = _digits(j) ** 2
    k[..., 6] = 1.0
    chosen = np.full((B, Hq, Sq), -1)
    for b, L in enumerate(lens):
        if L:
            k[b, :, L - 1, 7] = 1.0   # decoy for the rows that must not see the last key
        for i in range(Sq):
            vis = min(L, L - Sq + i + 1) if causal else L
            if vis > 0:
                c = rng.integers(0, vis, Hq)
                c[::3] = vis - 1
                chosen[b, :, i] = c
    q = np.zeros((B, Hq, Sq, D))
    q[..., 0:3] = 2 * G * _digits(np.maximum(chosen, 0))
    q[..., 3:6] = -G
    q[..., 6] = -C
    if causal:
        q[..., 7] = np.where(np.arange(Sq) < Sq - 1, C, 0.0)
    bb, hk, jj, dd = np.meshgrid(np.arange(B), np.arange(Hkv), j, np.arange(D), indexing="ij")
    v = ((jj * 7 + dd * 3 + hk * 5 + bb) % 257 - 128).astype(np.float64)
    want = np.zeros((B, Hq, Sq, D))
    g = Hq // Hkv
    for b in range(B):
        for h in range(Hq):
            for i in range(Sq):
                if chosen[b, h, i] >= 0:
                    want[b, h, i] = v[b, h // g, chosen[b, h, i]]
    return q, k, v, want, chosen < 0


ONE_HOT_CASES = [   # B, Hq, Hkv, Sq, D, page, max_pages, kind, causal, dtype
    (7, 4, 1, 1, 128, 16, 16, "paged", False, "bf16"),
    (7, 4, 1, 3, 128, 64, 8, "paged", True, "bf16"),
    (7, 8, 1, 17, 64, 256, 4, "paged", True, "bf16"),
    (7, 8, 1, 17, 64, 256, 4, "paged", False, "f16"),
    (3, 128, 1, 1, 64, 16, 20, "paged", False, "bf16"),
    (7, 1, 1, 3, 128, 320, 1, "identity", True, "bf16"),
    (8, 16, 16, 1, 128, 64, 4, "paged", False, "bf16"),     # 128 CTAs: one split
    (8, 16, 16, 3, 64, 256, 1, "identity", True, "bf16"),   # one split
    (8, 64, 16, 1, 128, 16, 4, "paged", True, "f16"),       # one split
]


@pytest.mark.parametrize("B,Hq,Hkv,Sq,D,page,mp,kind,causal,dtype", ONE_HOT_CASES)
def test_one_hot_rows_exact(client, B, Hq, Hkv, Sq, D, page, mp, kind, causal, dtype):
    cap = page * mp
    rng = np.random.default_rng(B * Hq + Sq + page)
    lens = ragged(B, cap, page, rng)
    q, k, v, want, empty = one_hot_kv(B, Hq, Hkv, Sq, cap, D, lens, causal, dtype, Sq + page)
    kc, vc, bt = layout(client, k, v, lens, page, kind, dtype, seed=page)
    for out_dtype in (dtype, "f32"):
        got, lse, _ = run(client, q, kc, vc, bt, lens, dtype, out_dtype, scale=ONE_HOT[dtype][2], causal=causal)
        if out_dtype == "f32":
            np.testing.assert_allclose(got, want, rtol=2.0 ** -20, atol=0)
        else:
            np.testing.assert_array_equal(got, want)
        assert np.all(lse[empty] == -np.inf) and np.isfinite(lse[~empty]).all()
        assert not np.signbit(got[empty]).any()


def test_one_hot_cases_cover_both_split_kinds():
    kinds = {nsplit(B, Hq, Hkv, Sq, page * mp) > 1 for B, Hq, Hkv, Sq, D, page, mp, *_ in ONE_HOT_CASES}
    assert kinds == {False, True}


# ---------------------------------------------------------------------------------------------- exact: uniform rows
@pytest.mark.parametrize("B,Hq,Hkv,cap,page", [(2, 4, 2, 1024, 16), (4, 8, 8, 4096, 64), (64, 8, 2, 256, 256), (8, 32, 16, 512, 32)])
def test_uniform_rows_give_the_exact_column_mean(client, B, Hq, Hkv, cap, page):
    D, Sq, dtype = 128, 2, "bf16"
    lens = [max(4, (cap * (b + 1) // B) // 4 * 4) for b in range(B)]
    k = np.random.default_rng(cap).integers(-8, 9, (B, Hkv, cap, D)).astype(np.float64)
    jj, dd = np.meshgrid(np.arange(cap), np.arange(D), indexing="ij")
    v = np.broadcast_to((jj % 4 - 1 + dd % 3).astype(np.float64), (B, Hkv, cap, D))
    want = np.broadcast_to((0.5 + np.arange(D) % 3).astype(np.float64), (B, Hq, Sq, D))
    kc, vc, bt = layout(client, k, v, lens, page, "paged", dtype)
    for out_dtype in (dtype, "f32"):
        got, _, _ = run(client, np.zeros((B, Hq, Sq, D)), kc, vc, bt, lens, dtype, out_dtype, scale=0.3)
        np.testing.assert_array_equal(got, want)


def test_uniform_cases_cover_both_split_kinds():
    kinds = {nsplit(B, Hq, Hkv, 2, cap) > 1 for B, Hq, Hkv, cap, _ in [(2, 4, 2, 1024, 16), (64, 8, 2, 256, 256)]}
    assert kinds == {False, True}


# ---------------------------------------------------------------------------------------------- stale slots, layouts
@pytest.mark.parametrize("causal", [False, True])
def test_stale_slots_never_reach_out(client, causal):
    B, Hq, Hkv, Sq, D, page, mp, dtype = 6, 8, 2, 3, 128, 16, 12, "bf16"
    cap = page * mp
    rng = np.random.default_rng(11)
    lens = [0, 1, 15, 17, 100, cap]
    q, k, v = (rounded(rng.uniform(-2, 2, s), dtype) for s in ((B, Hq, Sq, D), (B, Hkv, cap, D), (B, Hkv, cap, D)))
    ref = None
    for fill in (0.0, "nan", "inf"):
        kc, vc, bt = layout(client, k, v, lens, page, "paged", dtype, fill=fill, seed=5)
        vals, _, got = run(client, q, kc, vc, bt, lens, dtype, dtype, causal=causal)
        assert np.isfinite(vals).all()
        if ref is None:
            ref = got
        assert np.array_equal(got, ref), fill


def test_layouts_give_identical_bits(client):
    B, Hq, Hkv, Sq, D, dtype = 4, 16, 4, 2, 128, "bf16"
    cap = 1024
    rng = np.random.default_rng(13)
    lens = [1000, 17, 1024, 64]
    q, k, v = (rounded(rng.uniform(-2, 2, s), dtype) for s in ((B, Hq, Sq, D), (B, Hkv, cap, D), (B, Hkv, cap, D)))
    qb = up(client, np.ascontiguousarray(q.transpose(0, 2, 1, 3)), dtype)   # [B, Sq, Hq, D] as a [B, Hq, Sq, D] view
    q_view = TensorHandle(qb.handle, [B, Hq, Sq, D], [Sq * Hq * D, D, Hq * D, 1], dtype)
    outs = []
    for kind, page in (("identity", cap), ("paged", 16), ("paged", 256), ("headmajor", 64)):
        kc, vc, bt = layout(client, k, v, lens, page, kind, dtype, seed=page)
        for qv in (None, q_view):
            outs.append(run(client, q, kc, vc, bt, lens, dtype, "f32", causal=True, q_view=qv)[2])
    for o in outs[1:]:
        assert np.array_equal(o, outs[0])


# ---------------------------------------------------------------------------------------------- random data
@pytest.mark.parametrize("dtype", ["bf16", "f16"])
@pytest.mark.parametrize("B,Hq,Hkv,Sq,D,page,mp,causal", [
    (3, 32, 8, 1, 128, 16, 64, False), (2, 8, 2, 4, 64, 64, 10, True), (5, 4, 4, 17, 128, 256, 2, True),
    (64, 8, 8, 1, 96, 32, 8, False), (2, 128, 1, 1, 128, 16, 40, False), (3, 6, 3, 33, 40, 128, 3, True),
])
def test_random_against_the_oracle(client, dtype, B, Hq, Hkv, Sq, D, page, mp, causal):
    cap = page * mp
    rng = np.random.default_rng(B + Sq + D + page)
    lens = ragged(B, cap, page, rng)
    q, k, v = (rounded(rng.uniform(-2, 2, s), dtype) for s in ((B, Hq, Sq, D), (B, Hkv, cap, D), (B, Hkv, cap, D)))
    kc, vc, bt = layout(client, k, v, lens, page, "paged", dtype, fill="nan", seed=3)
    kn, vn = (np.ascontiguousarray(t.transpose(0, 2, 1, 3)) for t in (k, v))   # the identity layout of the oracle
    ref, ref_lse = ko.attention_kvcache_f64(q, kn, vn, lens, None, None, causal)
    for out_dtype in (dtype, "f32"):
        got, lse, _ = run(client, q, kc, vc, bt, lens, dtype, out_dtype, causal=causal)
        err = np.abs(got - ref) - _bound(ref, v, dtype, out_dtype)
        assert err.max() <= 0, float(err.max())
        fin = np.isfinite(ref_lse)
        assert np.array_equal(lse[~fin], ref_lse[~fin])
        np.testing.assert_allclose(lse[fin], ref_lse[fin], rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("B,Hq,Hkv,Sk", [(1, 32, 8, 8192), (16, 32, 32, 700), (2, 8, 1, 3000)])
def test_decode_agrees_with_b200_attention(client, B, Hq, Hkv, Sk):
    D, dtype = 128, "bf16"
    rng = np.random.default_rng(Sk)
    q, k, v = (rounded(rng.uniform(-2, 2, s), dtype) for s in ((B, Hq, 1, D), (B, Hkv, Sk, D), (B, Hkv, Sk, D)))
    kc, vc = (up(client, t.transpose(0, 2, 1, 3), dtype) for t in (k, v))
    got, lse, _ = run(client, q, kc, vc, None, [Sk] * B, dtype, dtype)
    kh, vh = (TensorHandle(t.handle, [B, Hkv, Sk, D], [Sk * Hkv * D, D, Hkv * D, 1], dtype) for t in (kc, vc))
    dense, dense_lse = attention.launch_alloc(client, up(client, q, dtype), kh, vh, return_lse=True)
    client.sync()
    ref = values(client, dense)
    assert (np.abs(got - ref) - 2 * _bound(ref, v, dtype, dtype)).max() <= 0
    np.testing.assert_allclose(lse, values(client, dense_lse), rtol=2e-5, atol=2e-5)


# ---------------------------------------------------------------------------------------------- reproducibility
def test_repeats_and_two_streams_give_the_same_bits(client):
    B, Hq, Hkv, D, page, mp, dtype = 2, 32, 8, 128, 16, 256, "f16"
    cap = page * mp
    assert nsplit(B, Hq, Hkv, 1, cap) > 1
    rng = np.random.default_rng(17)
    lens = [4000, 1234]
    q, k, v = (rounded(rng.uniform(-2, 2, s), dtype) for s in ((B, Hq, 1, D), (B, Hkv, cap, D), (B, Hkv, cap, D)))
    kc, vc, bt = layout(client, k, v, lens, page, "paged", dtype)
    qh, sl = up(client, q, dtype), up_i32(client, lens)
    streams = [client.create_stream(), client.create_stream()]
    outs = [[TensorHandle.empty_contiguous(client, [B, Hq, 1, D], "f32") for _ in range(3)] for _ in streams]
    try:
        for st, row in zip(streams, outs):
            for o in row:
                attention.launch_kvcache(client, qh, kc, vc, sl, o, block_table=bt, stream=st)
        for st in streams:
            client.sync_stream(st)
        client.sync()
        ref = bits(client, outs[0][0])
        for row in outs:
            for o in row:
                assert np.array_equal(bits(client, o), ref)
    finally:
        for st in streams:
            client.destroy_stream(st)


# ---------------------------------------------------------------------------------------------- kvcache_write
def test_write_scatters_exact_bits_and_skips_negative_slots(client):
    B, Snew, Hkv, D, P, page, dtype = 3, 5, 4, 64, 6, 16, "bf16"
    rng = np.random.default_rng(19)
    kn, vn = (rounded(rng.uniform(-100, 100, (B, Snew, Hkv, D)), dtype) for _ in range(2))
    slots = rng.permutation(P * page)[:B * Snew]
    slots[[2, 7]] = -1
    base = rounded(rng.uniform(-1, 1, (P, page, Hkv, D)), dtype)
    kc, vc = up(client, base, dtype), up(client, base, dtype)
    attention.kvcache_write(client, up(client, kn, dtype), up(client, vn, dtype), kc, vc, up_i32(client, slots))
    client.sync()
    for cache, new in ((kc, kn), (vc, vn)):
        want = base.copy()
        for n, s in enumerate(slots):
            if s >= 0:
                want[s // page, s % page] = new.reshape(B * Snew, Hkv, D)[n]
        np.testing.assert_array_equal(values(client, cache), want)


def test_prefill_through_write_equals_the_built_cache(client):
    B, Hq, Hkv, Sq, D, page, mp, dtype = 3, 8, 2, 4, 128, 16, 8, "bf16"
    cap = page * mp
    rng = np.random.default_rng(23)
    lens = [100, 37, 128]
    q, k, v = (rounded(rng.uniform(-2, 2, s), dtype) for s in ((B, Hq, Sq, D), (B, Hkv, cap, D), (B, Hkv, cap, D)))
    kc, vc, bt = layout(client, k, v, lens, page, "paged", dtype, seed=9)
    want = run(client, q, kc, vc, bt, lens, dtype, dtype, causal=True)[2]
    table = np.random.default_rng(29).permutation(B * mp).reshape(B, mp)
    kc2, vc2 = (up(client, np.zeros((B * mp, page, Hkv, D)), dtype) for _ in range(2))
    slots = np.full((B, cap), -1)
    for b, L in enumerate(lens):
        j = np.arange(L)
        slots[b, :L] = table[b, j // page] * page + j % page
    # the new tokens [B, cap, Hkv, D] as a stride-permuted view of [B, Hkv, cap, D]
    kn, vn = (up(client, t, dtype) for t in (k, v))
    views = [TensorHandle(t.handle, [B, cap, Hkv, D], [Hkv * cap * D, D, cap * D, 1], dtype) for t in (kn, vn)]
    attention.kvcache_write(client, *views, kc2, vc2, up_i32(client, slots))
    got = run(client, q, kc2, vc2, up_i32(client, table), lens, dtype, dtype, causal=True)[2]
    assert np.array_equal(got, want)


def test_errors_are_deferred_to_sync(client):
    q = up(client, np.zeros((2, 4, 1, 64)), "bf16")
    kc = up(client, np.zeros((2, 16, 3, 64)), "bf16")
    sl = up_i32(client, [1, 2])
    out = TensorHandle.empty_contiguous(client, [2, 4, 1, 64], "bf16")
    attention.launch_kvcache(client, q, kc, kc, sl, out)   # Hq = 4 is not a multiple of Hkv = 3: no raise here
    with pytest.raises(ServerError, match="multiple of Hkv"):
        client.sync()
    kn = up(client, np.zeros((2, 1, 2, 64)), "bf16")
    attention.kvcache_write(client, kn, kn, kc, kc, sl)
    with pytest.raises(ServerError, match="heads or head dim"):
        client.sync()
