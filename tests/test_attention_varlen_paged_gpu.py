"""GPU: b200_attention_varlen_paged on an H100.

- Bitwise equal to b200_attention_varlen: out and lse equal a varlen call whose k and v are every sequence's cached keys packed
  contiguously, over both dtypes, 16-bit and f32 out, D in {40, 64, 96, 128}, (Hq, Hkv) in {(8, 8), (16, 4), (8, 1)}, windows
  (-1, -1), (-1, 0), (W, 0) and (W, W'), shuffled pages of 16 to 256 keys, no table and one page per sequence through a table,
  Lq in {0, 1, 5, 127, 128, 129, 1000} and Lk >= Lq, Lk < Lq and Lk = 0, Lk not a multiple of the page.
- Random data with a non-default scale against the f64 oracle (a page gather, then the varlen oracle).
- Stale NaN and inf in unused slots and in pages no sequence owns change no bit; rows outside every sequence keep their
  sentinel bytes; sequences that share prefix pages each equal their own varlen call.
- A kvcache_write of a chunk into the pages, then a paged call, gives the bits of varlen on the prefix and chunk concatenated.
- A uniform causal batch agrees with b200_attention_kvcache within bf16 rounding (the key blocking differs, so bits do not).
- Reproducible across repeats and two streams."""
import numpy as np
import pytest

from cubecl_b200 import TensorHandle, attention
from test_attention_varlen_gpu import SENT, _close, bits, cu, up, values
from test_attention_varlen_paged_cpu import attention_varlen_paged_f64, cache_lengths

pytestmark = pytest.mark.gpu


def paged_cache(rng, lens_k, Hkv, D, page, mode, stale="nan", spare=3):
    """Keys and values of every sequence in a paged cache.  mode: "table" (shuffled pages of `page` keys plus `spare` pages no
    sequence owns; table entries past ceil(Lk / page) are -1), "none" (no table: sequence b is page b, one page of the longest
    length) or "one" (a [B, 1] table of shuffled single pages).  Slots past Lk and unowned pages hold `stale`: "nan", "inf"
    (+-inf) or a value.  -> (k_cache, v_cache [P, page, Hkv, D] f32, table [B, max_pages] i32 or None, packed k, v, cu_k)"""
    B = len(lens_k)
    if mode != "table":
        page = max(max(lens_k), 1) + 5
    mp = max(1, -(-max(lens_k) // page)) if mode == "table" else 1
    P = B * mp + (spare if mode != "none" else 0)
    signs = np.random.default_rng(99)   # its own generator: the keys and the page order do not depend on `stale`

    def fill(shape):
        if stale == "nan":
            return np.full(shape, np.nan, np.float32)
        if stale == "inf":
            return np.where(signs.random(shape) < 0.5, np.inf, -np.inf).astype(np.float32)
        return np.full(shape, float(stale), np.float32)

    kc, vc = fill((P, page, Hkv, D)), fill((P, page, Hkv, D))
    perm = rng.permutation(P) if mode != "none" else np.arange(P)
    table = perm[:B * mp].reshape(B, mp).astype(np.int32)
    k, v = rng.standard_normal((sum(lens_k), Hkv, D)).astype(np.float32), rng.standard_normal((sum(lens_k), Hkv, D)).astype(np.float32)
    cuk = cu(lens_k)
    for b, L in enumerate(lens_k):
        for j in range(L):
            kc[table[b, j // page], j % page] = k[cuk[b] + j]
            vc[table[b, j // page], j % page] = v[cuk[b] + j]
        table[b, -(-L // page):] = -1
    return kc, vc, (table if mode != "none" else None), k, v, cuk


def paged(client, q, kc, vc, table, seqlens, cuq, maxq, maxk, dtype, odt, window, scale=None, out=None, lse=None, stream=None):
    qh, kh, vh = up(client, q, dtype), up(client, kc, dtype), up(client, vc, dtype)
    bt = up(client, table, "i32") if table is not None else None
    if out is None:
        out = TensorHandle.empty_contiguous(client, list(q.shape), odt)
        lse = TensorHandle.empty_contiguous(client, [q.shape[1], q.shape[0]], "f32")
    attention.launch_varlen_paged(client, qh, kh, vh, up(client, cuq, "i32"), up(client, np.asarray(seqlens), "i32"), maxq, maxk, out,
                                  block_table=bt, scale=scale, window_size=window, lse=lse, stream=stream)
    return out, lse


def varlen_ref(client, q, k, v, cuq, cuk, maxq, maxk, dtype, odt, window, scale=None):
    out, lse = attention.launch_varlen_alloc(client, up(client, q, dtype), up(client, k, dtype), up(client, v, dtype), up(client, cuq, "i32"),
                                             up(client, cuk, "i32"), maxq, maxk, scale=scale, window_size=window, out_dtype=odt,
                                             return_lse=True)
    return out, lse


# ---------------------------------------------------------------------------------------------- bitwise against varlen
LENS_Q = [0, 1, 5, 127, 128, 129, 1000]
LENS_K = [37, 1, 700, 0, 200, 100, 1811]     # Lk >= Lq, Lk < Lq (129 / 100), Lk = 0 with queries, Lq = 0 with keys
PAGES = [("table", 16), ("table", 32), ("table", 64), ("table", 128), ("table", 192), ("table", 256), ("none", 0), ("one", 0)]
WINDOWS = [(-1, -1), (-1, 0), (100, 0), (64, 32)]
HEADS = [(8, 8), (16, 4), (8, 1)]


@pytest.mark.parametrize("dtype", ["bf16", "f16"])
@pytest.mark.parametrize("D", [40, 64, 96, 128])
@pytest.mark.parametrize("f32", [False, True])
def test_bits_equal_varlen_on_the_gathered_keys(client, dtype, D, f32):
    odt = "f32" if f32 else dtype
    n = 0
    for window in WINDOWS:
        for mode, page in PAGES:
            Hq, Hkv = HEADS[n % len(HEADS)]
            n += 1
            rng = np.random.default_rng(D + 1000 * n + 7 * f32)
            kc, vc, table, k, v, cuk = paged_cache(rng, LENS_K, Hkv, D, page, mode)
            cuq = cu(LENS_Q)
            q = rng.standard_normal((int(cuq[-1]), Hq, D)).astype(np.float32)
            out, lse = paged(client, q, kc, vc, table, LENS_K, cuq, max(LENS_Q), max(LENS_K), dtype, odt, window)
            rout, rlse = varlen_ref(client, q, k, v, cuq, cuk, max(LENS_Q), max(LENS_K), dtype, odt, window)
            client.sync()
            what = f"{window} {mode} page={page} heads={Hq},{Hkv}"
            np.testing.assert_array_equal(bits(client, out), bits(client, rout), err_msg=f"out: {what}")
            np.testing.assert_array_equal(bits(client, lse), bits(client, rlse), err_msg=f"lse: {what}")


# ---------------------------------------------------------------------------------------------- against the oracle
@pytest.mark.parametrize("dtype", ["bf16", "f16"])
@pytest.mark.parametrize("window,page", [((-1, 0), 16), ((-1, -1), 64), ((200, 0), 32), ((48, 48), 256)])
def test_random_data_against_the_oracle(client, dtype, window, page):
    rng = np.random.default_rng(page + window[0])
    lens_q, lens_k = [300, 0, 129, 77, 5], [200, 9, 900, 77, 0]
    Hq, Hkv, D, scale = 8, 2, 64, 0.3
    kc, vc, table, _, _, _ = paged_cache(rng, lens_k, Hkv, D, page, "table")
    cuq = cu(lens_q)
    q = rng.standard_normal((int(cuq[-1]), Hq, D)).astype(np.float32)
    out, lse = paged(client, q, kc, vc, table, lens_k, cuq, max(lens_q), max(lens_k), dtype, "f32", window, scale=scale)
    client.sync()
    rq, rkc, rvc = (values(client, up(client, t, dtype)) for t in (q, kc, vc))
    ref_out, ref_lse = attention_varlen_paged_f64(rq, rkc, rvc, table, lens_k, cuq, max(lens_k), scale, window)
    got_lse = values(client, lse)
    np.testing.assert_array_equal(np.isneginf(got_lse), np.isneginf(ref_lse))
    fin = np.isfinite(ref_lse)
    np.testing.assert_allclose(got_lse[fin], ref_lse[fin], rtol=0, atol=1e-3)
    got_out = values(client, out)
    assert np.all(got_out[np.isneginf(ref_lse).T] == 0)   # rows without keys: +0
    _close(got_out, ref_out, dtype, "out")


def test_lengths_are_clamped_to_max_seqlen_k_and_capacity(client):
    rng = np.random.default_rng(5)
    lens_q, lens_k, page = [50, 60, 70], [300, 500, 100], 64
    kc, vc, table, k, v, cuk = paged_cache(rng, lens_k, 2, 64, page, "table")
    cuq = cu(lens_q)
    q = rng.standard_normal((int(cuq[-1]), 4, 64)).astype(np.float32)
    seqlens, maxk = [300, 10 ** 6, -4], 400     # 10^6 clamps to max_seqlen_k = 400 (below the capacity), -4 to 0
    out, lse = paged(client, q, kc, vc, table, seqlens, cuq, 70, maxk, "bf16", "bf16", (-1, 0))
    lens = cache_lengths(seqlens, maxk, page * table.shape[1])
    assert lens == [300, 400, 0]
    kk = np.concatenate([k[cuk[b]:cuk[b] + L] for b, L in enumerate(lens)])
    vv = np.concatenate([v[cuk[b]:cuk[b] + L] for b, L in enumerate(lens)])
    rout, rlse = varlen_ref(client, q, kk, vv, cuq, cu(lens), 70, maxk, "bf16", "bf16", (-1, 0))
    client.sync()
    np.testing.assert_array_equal(bits(client, out), bits(client, rout))
    np.testing.assert_array_equal(bits(client, lse), bits(client, rlse))


# ---------------------------------------------------------------------------------------------- stale data, sentinels, sharing
@pytest.mark.parametrize("page", [16, 192, 256])
def test_stale_nan_and_inf_change_no_bit(client, page):
    lens_q, lens_k = [100, 31, 400], [250, 31, 999]
    cuq = cu(lens_q)
    results = []
    for stale in (0.0, "nan", "inf"):
        rng = np.random.default_rng(page)   # the same keys, queries and page order every time: only the stale slots differ
        kc, vc, table, _, _, _ = paged_cache(rng, lens_k, 2, 128, page, "table", stale=stale)
        q = np.random.default_rng(1).standard_normal((int(cuq[-1]), 8, 128)).astype(np.float32)
        out, lse = paged(client, q, kc, vc, table, lens_k, cuq, 400, 999, "bf16", "f32", (-1, 0))
        client.sync()
        results.append((bits(client, out), bits(client, lse)))
    for got in results[1:]:
        np.testing.assert_array_equal(got[0], results[0][0])
        np.testing.assert_array_equal(got[1], results[0][1])


@pytest.mark.parametrize("f32", [False, True])
def test_rows_outside_every_sequence_keep_their_sentinels(client, f32):
    rng = np.random.default_rng(12)
    lens_q, lens_k, pad = [100, 0, 190], [130, 7, 65], (5, 77)
    Hq, D = 4, 96
    kc, vc, table, _, _, _ = paged_cache(rng, lens_k, 4, D, 32, "table")
    Tq = sum(lens_q) + sum(pad)
    cuq = cu(lens_q, pad[0])
    q = rng.standard_normal((Tq, Hq, D)).astype(np.float32)
    dt = "f32" if f32 else "f16"
    raw = lambda shape, d: TensorHandle.from_numpy(  # noqa: E731
        client, np.full(int(np.prod(shape)), SENT[d], dtype=np.uint32 if d == "f32" else np.uint16).reshape(shape), d)
    out, lse = raw([Tq, Hq, D], dt), raw([Hq, Tq], "f32")
    paged(client, q, kc, vc, table, lens_k, cuq, 190, 130, "f16", dt, (50, 0), out=out, lse=lse)
    client.sync()
    for name, arr, axis in (("out", bits(client, out), 0), ("lse", bits(client, lse), 1)):
        s = SENT["f32" if name == "lse" else dt]
        a = np.moveaxis(arr, axis, 0)
        assert np.all(a[:cuq[0]] == s) and np.all(a[cuq[-1]:] == s), name
        assert not np.any(a[cuq[0]:cuq[-1]] == s), name   # every owned row was written


def test_sequences_sharing_prefix_pages_each_equal_their_own_varlen_call(client):
    rng = np.random.default_rng(21)
    page, Hkv, D, Hq = 64, 2, 128, 8
    prefix, tails, lens_q = 640, [150, 333], [150, 333]   # a shared system prompt of 10 pages, then each request's own pages
    P = 10 + 2 * 6 + 2
    kc = rng.standard_normal((P, page, Hkv, D)).astype(np.float32)
    vc = rng.standard_normal((P, page, Hkv, D)).astype(np.float32)
    perm = rng.permutation(P)
    shared, own = perm[:10], [perm[10:16], perm[16:22]]
    table = np.full((2, 16), -1, np.int32)
    lens_k = [prefix + t for t in tails]
    for b in range(2):
        table[b, :10] = shared
        table[b, 10:10 + -(-tails[b] // page)] = own[b][:-(-tails[b] // page)]
    cuq = cu(lens_q)
    q = rng.standard_normal((int(cuq[-1]), Hq, D)).astype(np.float32)
    out, lse = paged(client, q, kc, vc, table, lens_k, cuq, 333, max(lens_k), "bf16", "bf16", (-1, 0))
    ob, lb = bits(client, out), bits(client, lse)
    for b in range(2):
        rows = [(table[b, j // page], j % page) for j in range(lens_k[b])]
        k = np.stack([kc[p, r] for p, r in rows])
        v = np.stack([vc[p, r] for p, r in rows])
        qs = q[cuq[b]:cuq[b + 1]]
        rout, rlse = varlen_ref(client, qs, k, v, cu([lens_q[b]]), cu([lens_k[b]]), lens_q[b], lens_k[b], "bf16", "bf16", (-1, 0))
        client.sync()
        np.testing.assert_array_equal(ob[cuq[b]:cuq[b + 1]], bits(client, rout), err_msg=f"out of sequence {b}")
        np.testing.assert_array_equal(lb[:, cuq[b]:cuq[b + 1]], bits(client, rlse), err_msg=f"lse of sequence {b}")


# ---------------------------------------------------------------------------------------------- chunked prefill round trip
def test_kvcache_write_then_paged_call_equals_varlen_on_prefix_and_chunk(client):
    rng = np.random.default_rng(31)
    page, Hkv, D, Hq, dtype = 64, 4, 128, 16, "bf16"
    prefixes, chunks = [500, 1000], [300, 180]
    mp = -(-(max(p + c for p, c in zip(prefixes, chunks))) // page)
    P = 2 * mp + 1
    kc = np.zeros((P, page, Hkv, D), np.float32)
    vc = np.zeros((P, page, Hkv, D), np.float32)
    table = rng.permutation(P)[:2 * mp].reshape(2, mp).astype(np.int32)
    pk = [rng.standard_normal((L, Hkv, D)).astype(np.float32) for L in prefixes]
    pv = [rng.standard_normal((L, Hkv, D)).astype(np.float32) for L in prefixes]
    for b, L in enumerate(prefixes):
        for j in range(L):
            kc[table[b, j // page], j % page], vc[table[b, j // page], j % page] = pk[b][j], pv[b][j]
    Snew = max(chunks)
    kn = rng.standard_normal((2, Snew, Hkv, D)).astype(np.float32)
    vn = rng.standard_normal((2, Snew, Hkv, D)).astype(np.float32)
    slots = np.full((2, Snew), -1, np.int32)
    for b, (L, c) in enumerate(zip(prefixes, chunks)):
        j = L + np.arange(c)
        slots[b, :c] = table[b, j // page] * page + j % page
    kch, vch = up(client, kc, dtype), up(client, vc, dtype)
    attention.kvcache_write(client, up(client, kn, dtype), up(client, vn, dtype), kch, vch, up(client, slots.reshape(-1), "i32"))
    lens_k = [L + c for L, c in zip(prefixes, chunks)]
    cuq = cu(chunks)
    q = rng.standard_normal((int(cuq[-1]), Hq, D)).astype(np.float32)
    out, lse = attention.launch_varlen_paged_alloc(client, up(client, q, dtype), kch, vch, up(client, cuq, "i32"),
                                                   up(client, np.array(lens_k), "i32"), max(chunks), max(lens_k),
                                                   block_table=up(client, table, "i32"), window_size=(-1, 0), return_lse=True)
    k = np.concatenate([np.concatenate([pk[b], kn[b, :c]]) for b, c in enumerate(chunks)])
    v = np.concatenate([np.concatenate([pv[b], vn[b, :c]]) for b, c in enumerate(chunks)])
    rout, rlse = varlen_ref(client, q, k, v, cuq, cu(lens_k), max(chunks), max(lens_k), dtype, dtype, (-1, 0))
    client.sync()
    np.testing.assert_array_equal(bits(client, out), bits(client, rout))
    np.testing.assert_array_equal(bits(client, lse), bits(client, rlse))


# ---------------------------------------------------------------------------------------------- against the decode kernel
def test_uniform_causal_batch_agrees_with_the_kvcache_kernel(client):
    rng = np.random.default_rng(41)
    B, Sq, Hq, Hkv, D, page = 4, 200, 8, 2, 128, 16
    lens_k = [700, 200, 1333, 999]
    kc, vc, table, _, _, _ = paged_cache(rng, lens_k, Hkv, D, page, "table")
    q = rng.standard_normal((B * Sq, Hq, D)).astype(np.float32)
    cuq = cu([Sq] * B)
    out, lse = paged(client, q, kc, vc, table, lens_k, cuq, Sq, max(lens_k), "bf16", "f32", (-1, 0))
    qd = up(client, np.ascontiguousarray(q.reshape(B, Sq, Hq, D).transpose(0, 2, 1, 3)), "bf16")
    kout, klse = attention.launch_kvcache_alloc(client, qd, up(client, kc, "bf16"), up(client, vc, "bf16"), up(client, np.array(lens_k), "i32"),
                                                block_table=up(client, table, "i32"), causal=True, out_dtype="f32", return_lse=True)
    client.sync()
    got = values(client, out).reshape(B, Sq, Hq, D)
    want = values(client, kout).transpose(0, 2, 1, 3)
    assert float(np.abs(got - want).max()) <= 4 * 2.0 ** -8 * max(1.0, float(np.abs(want).max()))
    got_lse = values(client, lse).reshape(Hq, B, Sq).transpose(1, 0, 2)
    np.testing.assert_allclose(got_lse, values(client, klse), rtol=0, atol=1e-4)


# ---------------------------------------------------------------------------------------------- reproducibility
def test_repeats_and_two_streams_give_the_same_bits(client):
    rng = np.random.default_rng(13)
    lens_q, lens_k = [333, 1000, 64, 5], [900, 1000, 2000, 5]
    kc, vc, table, _, _, _ = paged_cache(rng, lens_k, 2, 128, 16, "table")
    cuq = cu(lens_q)
    q = rng.standard_normal((int(cuq[-1]), 8, 128)).astype(np.float32)
    ref = paged(client, q, kc, vc, table, lens_k, cuq, 1000, 2000, "bf16", "bf16", (256, 0))
    client.sync()
    ref = [bits(client, t) for t in ref]
    qh, kh, vh = up(client, q, "bf16"), up(client, kc, "bf16"), up(client, vc, "bf16")
    cq, sl, bt = up(client, cuq, "i32"), up(client, np.array(lens_k), "i32"), up(client, table, "i32")
    streams = [client.create_stream(), client.create_stream()]
    try:
        results = []
        for _ in range(2):
            for st in streams:
                results.append(attention.launch_varlen_paged_alloc(client, qh, kh, vh, cq, sl, 1000, 2000, block_table=bt, window_size=(256, 0),
                                                                   return_lse=True, stream=st))
        for st in streams:
            client.sync_stream(st)
        client.sync()
        for r in results:
            for want, got in zip(ref, r):
                np.testing.assert_array_equal(want, bits(client, got))
    finally:
        for st in streams:
            client.destroy_stream(st)
