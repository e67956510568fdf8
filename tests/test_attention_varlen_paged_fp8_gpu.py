"""GPU: b200_attention_varlen_paged_fp8 on an H100.

- Bitwise equal to b200_attention_varlen_paged on the dequantized 16-bit cache (scale * code in q's dtype) with per-head
  power-of-two scales and scales of 1: both fp8 formats, f16 and bf16 q, 16-bit and f32 out, D in {48, 64, 112, 128},
  (Hq, Hkv) in {(8, 8), (16, 4), (8, 1)}, windows (-1, -1), (-1, 0), (W, 0) and (W, W'), shuffled pages of 16 to 256 keys,
  no table and one page per sequence, Lq in {0, 1, 5, 127, 128, 129, 300} with Lk >= Lq, Lk < Lq, Lk = 0 and Lk not a
  multiple of the page.
- Random codes with non-power-of-two scales and a non-default scale against the f64 oracle (the fp8 dequantization, then the
  paged varlen oracle).
- Stale e4m3 NaN and e5m2 inf / NaN bytes in unused slots and unowned pages change no bit; rows outside every sequence keep
  their sentinel bytes.
- Chunked prefill end to end: a prefix and then a chunk written with kvcache_write_fp8, then a paged fp8 call, equal the 16-bit
  paged call on the dequantized cache; a following fp8 decode step agrees with a paged fp8 call within bf16 rounding.
- Reproducible across repeats and two streams."""
import numpy as np
import pytest

import attention_kvcache_fp8_oracle as fo
from cubecl_b200 import TensorHandle, attention
from test_attention_kvcache_fp8_gpu import STALE, up8, up_f32
from test_attention_varlen_gpu import SENT, _close, bits, cu, up, values
from test_attention_varlen_paged_cpu import attention_varlen_paged_f64
from test_attention_varlen_paged_gpu import HEADS, PAGES, WINDOWS, paged

pytestmark = pytest.mark.gpu

FORMATS = ("f8e4m3", "f8e5m2")
LENS_Q = [0, 1, 5, 127, 128, 129, 300]
LENS_K = [37, 1, 700, 0, 200, 100, 555]   # Lk >= Lq, Lk < Lq (129 / 100), Lk = 0 with queries, Lq = 0 with keys


def paged_cache8(rng, lens_k, Hkv, D, page, mode, fmt, stale=0):
    """fp8 codes of random keys and values in paged_cache's layouts: "table" (shuffled pages of `page` keys plus three pages no
    sequence owns; entries past ceil(Lk / page) are -1), "none" (no table, one page of the longest length per sequence) or
    "one" (a [B, 1] table of shuffled single pages).  Slots past Lk and unowned pages hold the byte `stale` (an int, or a
    tuple cycled through).  -> (k8, v8 [P, page, Hkv, D] uint8, table or None)"""
    B = len(lens_k)
    if mode != "table":
        page = max(max(lens_k), 1) + 5
    mp = max(1, -(-max(lens_k) // page)) if mode == "table" else 1
    P = B * mp + (3 if mode != "none" else 0)
    perm = rng.permutation(P) if mode != "none" else np.arange(P)
    table = perm[:B * mp].reshape(B, mp).astype(np.int32)
    one = np.ones(Hkv, np.float32)
    fill = np.resize(np.asarray(stale, dtype=np.uint8), (P, page, Hkv, D))
    caches = []
    for _ in range(2):
        codes = fo.quantize(rng.standard_normal((sum(lens_k), Hkv, D)).astype(np.float32), one, fmt)
        c, cuk = fill.copy(), cu(lens_k)
        for b, L in enumerate(lens_k):
            j = np.arange(L)
            c[table[b, j // page], j % page] = codes[cuk[b]:cuk[b] + L]
        caches.append(c)
    for b, L in enumerate(lens_k):
        table[b, -(-L // page):] = -1
    return caches[0], caches[1], (table if mode != "none" else None)


def scales(rng, Hkv, kind):
    """f32 [Hkv]: "one", "pow2" (2^-3 .. 2^2: scale * code is exact in f16 and bf16 for every finite e4m3 code and every e5m2
    code below 2^13) or "any" """
    if kind == "one":
        return np.ones(Hkv, np.float32)
    if kind == "pow2":
        return (2.0 ** rng.integers(-3, 3, Hkv)).astype(np.float32)
    return rng.uniform(0.05, 3.0, Hkv).astype(np.float32)


def paged8(client, q, k8, v8, table, seqlens, cuq, maxq, maxk, ks, vs, fmt, dtype, odt, window, scale=None, out=None, lse=None,
           stream=None):
    qh = up(client, q, dtype)
    bt = up(client, table, "i32") if table is not None else None
    if out is None:
        out = TensorHandle.empty_contiguous(client, list(q.shape), odt)
        lse = TensorHandle.empty_contiguous(client, [q.shape[1], q.shape[0]], "f32")
    attention.launch_varlen_paged_fp8(client, qh, up8(client, k8, fmt), up8(client, v8, fmt), up(client, cuq, "i32"),
                                      up(client, np.asarray(seqlens), "i32"), up_f32(client, ks), up_f32(client, vs), maxq, maxk, out,
                                      block_table=bt, scale=scale, window_size=window, lse=lse, stream=stream)
    return out, lse


def dequant(codes, s, fmt):
    """the dequantized cache scale[hk] * code as f32 (exact in f16 and bf16 for the scales and codes used here), through a
    table of the 256 codes"""
    with np.errstate(invalid="ignore"):
        return fo.decode(np.arange(256), fmt).astype(np.float32)[codes] * np.asarray(s, np.float32)[:, None]


# ---------------------------------------------------------------------------------------------- bitwise against 16-bit paged
@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("dtype", ["bf16", "f16"])
@pytest.mark.parametrize("D", [48, 64, 112, 128])
@pytest.mark.parametrize("f32", [False, True])
def test_bits_equal_paged_on_the_dequantized_cache(client, fmt, dtype, D, f32):
    odt = "f32" if f32 else dtype
    half = (D // 16 + f32 + (fmt == "f8e5m2")) % 2   # half of the page layouts per case: each layout in 16 of the 32 cases
    for n, (mode, page) in enumerate(PAGES[half::2]):
        window, (Hq, Hkv) = WINDOWS[(n + half) % len(WINDOWS)], HEADS[(n + D // 16) % len(HEADS)]
        rng = np.random.default_rng(D + 1000 * n + 7 * f32 + 31 * (fmt == "f8e5m2"))
        k8, v8, table = paged_cache8(rng, LENS_K, Hkv, D, page, mode, fmt, stale=STALE[fmt])
        ks, vs = scales(rng, Hkv, "one" if n == 0 else "pow2"), scales(rng, Hkv, "pow2")
        cuq = cu(LENS_Q)
        q = rng.standard_normal((int(cuq[-1]), Hq, D)).astype(np.float32)
        out, lse = paged8(client, q, k8, v8, table, LENS_K, cuq, max(LENS_Q), max(LENS_K), ks, vs, fmt, dtype, odt, window)
        rout, rlse = paged(client, q, dequant(k8, ks, fmt), dequant(v8, vs, fmt), table, LENS_K, cuq, max(LENS_Q), max(LENS_K), dtype,
                           odt, window)
        client.sync()
        what = f"{window} {mode} page={page} heads={Hq},{Hkv}"
        np.testing.assert_array_equal(bits(client, out), bits(client, rout), err_msg=f"out: {what}")
        np.testing.assert_array_equal(bits(client, lse), bits(client, rlse), err_msg=f"lse: {what}")


# ---------------------------------------------------------------------------------------------- against the oracle
@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("dtype", ["bf16", "f16"])
@pytest.mark.parametrize("window,page", [((-1, 0), 16), ((200, 0), 64), ((48, 48), 256)])
def test_random_codes_against_the_oracle(client, fmt, dtype, window, page):
    rng = np.random.default_rng(page + window[0] + 3 * (fmt == "f8e5m2"))
    lens_q, lens_k = [300, 0, 129, 77, 5], [200, 9, 900, 77, 0]
    Hq, Hkv, D, scale = 8, 2, 64, 0.3
    k8, v8, table = paged_cache8(rng, lens_k, Hkv, D, page, "table", fmt)
    ks, vs = scales(rng, Hkv, "any"), scales(rng, Hkv, "any")
    cuq = cu(lens_q)
    q = rng.standard_normal((int(cuq[-1]), Hq, D)).astype(np.float32)
    out, lse = paged8(client, q, k8, v8, table, lens_k, cuq, max(lens_q), max(lens_k), ks, vs, fmt, dtype, "f32", window, scale=scale)
    client.sync()
    rq = values(client, up(client, q, dtype))
    ref_out, ref_lse = attention_varlen_paged_f64(rq, fo.dequantize(k8, ks, fmt), fo.dequantize(v8, vs, fmt), table, lens_k, cuq,
                                                  max(lens_k), scale, window)
    got_lse = values(client, lse)
    np.testing.assert_array_equal(np.isneginf(got_lse), np.isneginf(ref_lse))
    fin = np.isfinite(ref_lse)
    np.testing.assert_allclose(got_lse[fin], ref_lse[fin], rtol=0, atol=1e-3)
    got_out = values(client, out)
    assert np.all(got_out[np.isneginf(ref_lse).T] == 0)   # rows without keys: +0
    _close(got_out, ref_out, dtype, "out")


# ---------------------------------------------------------------------------------------------- stale bytes, sentinels
@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("page", [16, 192, 256])
def test_stale_bytes_change_no_bit(client, fmt, page):
    lens_q, lens_k = [100, 31, 400], [250, 31, 999]
    cuq = cu(lens_q)
    results = []
    for stale in (0, STALE[fmt]):
        rng = np.random.default_rng(page)   # the same codes, queries and page order every time: only the stale slots differ
        k8, v8, table = paged_cache8(rng, lens_k, 2, 128, page, "table", fmt, stale=stale)
        ks, vs = np.array([0.5, 2.0], np.float32), np.array([0.25, 1.0], np.float32)
        q = np.random.default_rng(1).standard_normal((int(cuq[-1]), 8, 128)).astype(np.float32)
        out, lse = paged8(client, q, k8, v8, table, lens_k, cuq, 400, 999, ks, vs, fmt, "bf16", "f32", (-1, 0))
        client.sync()
        results.append((bits(client, out), bits(client, lse)))
    np.testing.assert_array_equal(results[1][0], results[0][0])
    np.testing.assert_array_equal(results[1][1], results[0][1])


@pytest.mark.parametrize("f32", [False, True])
def test_rows_outside_every_sequence_keep_their_sentinels(client, f32):
    rng = np.random.default_rng(12)
    lens_q, lens_k, pad = [100, 0, 190], [130, 7, 65], (5, 77)
    Hq, D = 4, 96
    k8, v8, table = paged_cache8(rng, lens_k, 4, D, 32, "table", "f8e4m3", stale=STALE["f8e4m3"])
    Tq = sum(lens_q) + sum(pad)
    cuq = cu(lens_q, pad[0])
    q = rng.standard_normal((Tq, Hq, D)).astype(np.float32)
    dt = "f32" if f32 else "f16"
    raw = lambda shape, d: TensorHandle.from_numpy(  # noqa: E731
        client, np.full(int(np.prod(shape)), SENT[d], dtype=np.uint32 if d == "f32" else np.uint16).reshape(shape), d)
    out, lse = raw([Tq, Hq, D], dt), raw([Hq, Tq], "f32")
    one = np.ones(4, np.float32)
    paged8(client, q, k8, v8, table, lens_k, cuq, 190, 130, one, one, "f8e4m3", "f16", dt, (50, 0), out=out, lse=lse)
    client.sync()
    for name, arr, axis in (("out", bits(client, out), 0), ("lse", bits(client, lse), 1)):
        s = SENT["f32" if name == "lse" else dt]
        a = np.moveaxis(arr, axis, 0)
        assert np.all(a[:cuq[0]] == s) and np.all(a[cuq[-1]:] == s), name
        assert not np.any(a[cuq[0]:cuq[-1]] == s), name   # every owned row was written


# ---------------------------------------------------------------------------------------------- chunked prefill end to end
@pytest.mark.parametrize("fmt", FORMATS)
def test_chunked_prefill_into_an_fp8_cache_then_decode(client, fmt):
    rng = np.random.default_rng(31)
    page, Hkv, D, Hq, dtype = 64, 4, 128, 16, "bf16"
    prefixes, chunks = [500, 1000], [300, 180]
    mp = -(-(max(p + c for p, c in zip(prefixes, chunks)) + 1) // page)
    P = 2 * mp + 1
    table = rng.permutation(P)[:2 * mp].reshape(2, mp).astype(np.int32)
    ks, vs = scales(rng, Hkv, "pow2"), scales(rng, Hkv, "pow2")
    kch = up8(client, np.zeros((P, page, Hkv, D), np.uint8), fmt)
    vch = up8(client, np.zeros((P, page, Hkv, D), np.uint8), fmt)
    ksh, vsh = up_f32(client, ks), up_f32(client, vs)

    def write(starts, counts):   # tokens [starts[b], starts[b] + counts[b]) of each sequence into their slots
        S = max(counts)
        kn = rng.standard_normal((2, S, Hkv, D)).astype(np.float32)
        vn = rng.standard_normal((2, S, Hkv, D)).astype(np.float32)
        slots = np.full((2, S), -1, np.int32)
        for b, (s0, c) in enumerate(zip(starts, counts)):
            j = s0 + np.arange(c)
            slots[b, :c] = table[b, j // page] * page + j % page
        attention.kvcache_write_fp8(client, up(client, kn, dtype), up(client, vn, dtype), kch, vch, up(client, slots.reshape(-1), "i32"),
                                    ksh, vsh)

    write([0, 0], prefixes)   # the cached prefix
    write(prefixes, chunks)   # this step's chunk
    lens_k = [L + c for L, c in zip(prefixes, chunks)]
    cuq = cu(chunks)
    q = rng.standard_normal((int(cuq[-1]), Hq, D)).astype(np.float32)
    qh, bt = up(client, q, dtype), up(client, table, "i32")
    out, lse = attention.launch_varlen_paged_fp8_alloc(client, qh, kch, vch, up(client, cuq, "i32"), up(client, np.array(lens_k), "i32"),
                                                       ksh, vsh, max(chunks), max(lens_k), block_table=bt, window_size=(-1, 0),
                                                       return_lse=True)
    k8, v8 = (np.asarray(h.to_numpy(client)).view(np.uint8).reshape(P, page, Hkv, D) for h in (kch, vch))
    rout, rlse = paged(client, q, dequant(k8, ks, fmt), dequant(v8, vs, fmt), table, lens_k, cuq, max(chunks), max(lens_k), dtype,
                       dtype, (-1, 0))
    client.sync()
    np.testing.assert_array_equal(bits(client, out), bits(client, rout))
    np.testing.assert_array_equal(bits(client, lse), bits(client, rlse))

    # one decode step: write the next token, then the fp8 decode kernel and a paged fp8 call with Lq = 1 per sequence
    write(lens_k, [1, 1])
    lens_d = [L + 1 for L in lens_k]
    qd = rng.standard_normal((2, Hq, D)).astype(np.float32)
    sl = up(client, np.array(lens_d), "i32")
    dout = attention.launch_kvcache_fp8_alloc(client, up(client, qd.reshape(2, Hq, 1, D), dtype), kch, vch, sl, ksh, vsh,
                                              block_table=bt, causal=True, out_dtype="f32")
    pout = attention.launch_varlen_paged_fp8_alloc(client, up(client, qd, dtype), kch, vch, up(client, cu([1, 1]), "i32"), sl, ksh, vsh,
                                                   1, max(lens_d), block_table=bt, window_size=(-1, 0), out_dtype="f32")
    client.sync()
    want, got = values(client, dout).reshape(2, Hq, D), values(client, pout)
    assert float(np.abs(got - want).max()) <= 4 * 2.0 ** -8 * max(1.0, float(np.abs(want).max()))


# ---------------------------------------------------------------------------------------------- reproducibility
def test_repeats_and_two_streams_give_the_same_bits(client):
    rng = np.random.default_rng(13)
    lens_q, lens_k, fmt = [333, 1000, 64, 5], [900, 1000, 2000, 5], "f8e4m3"
    k8, v8, table = paged_cache8(rng, lens_k, 2, 128, 16, "table", fmt, stale=STALE[fmt])
    ks, vs = scales(rng, 2, "any"), scales(rng, 2, "any")
    cuq = cu(lens_q)
    q = rng.standard_normal((int(cuq[-1]), 8, 128)).astype(np.float32)
    ref = paged8(client, q, k8, v8, table, lens_k, cuq, 1000, 2000, ks, vs, fmt, "bf16", "bf16", (256, 0))
    client.sync()
    ref = [bits(client, t) for t in ref]
    qh, kh, vh = up(client, q, "bf16"), up8(client, k8, fmt), up8(client, v8, fmt)
    cq, sl, bt = up(client, cuq, "i32"), up(client, np.array(lens_k), "i32"), up(client, table, "i32")
    ksh, vsh = up_f32(client, ks), up_f32(client, vs)
    streams = [client.create_stream(), client.create_stream()]
    try:
        results = []
        for _ in range(2):
            for st in streams:
                results.append(attention.launch_varlen_paged_fp8_alloc(client, qh, kh, vh, cq, sl, ksh, vsh, 1000, 2000, block_table=bt,
                                                                       window_size=(256, 0), return_lse=True, stream=st))
        for st in streams:
            client.sync_stream(st)
        client.sync()
        for r in results:
            for want, got in zip(ref, r):
                np.testing.assert_array_equal(want, bits(client, got))
    finally:
        for st in streams:
            client.destroy_stream(st)
