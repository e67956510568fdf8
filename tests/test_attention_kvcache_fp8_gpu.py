"""GPU: b200_attention_kvcache_fp8 and b200_kvcache_write_fp8 on an H100.

- Bits equal to b200_attention_kvcache on the dequantized 16-bit cache with scales of 1 and with power-of-two per-head scales:
  both fp8 formats, f16 and bf16 q, 16-bit and f32 out with lse, D in {48, 64, 112, 128}, GQA, Sq > 1 causal, one split and
  several, the identity table and shuffled pages of 16, 32 and 128 keys.
- Random data with arbitrary scales against the f64 oracle.
- Stale NaN and inf bytes past L_b change no bit of out.
- The quantizing write bit for bit against the oracle (saturation, NaN, inf), with skipped slots and sentinel bytes kept.
- A write-then-attend round trip, and identical bits across repeats and two streams."""
import numpy as np
import pytest

import attention_kvcache_fp8_oracle as fo
from cubecl_b200 import ServerError, TensorHandle, attention
from test_attention_gpu import _bound, bits, rounded, up, values
from test_attention_kvcache_gpu import nsplit, ragged, up_i32

pytestmark = pytest.mark.gpu

# a stale byte per format: NaN and +-inf where the format has them
STALE = {"f8e4m3": (0x7F, 0xFF), "f8e5m2": (0x7F, 0x7C, 0xFC)}


def up8(client, codes, fmt):
    return TensorHandle.from_numpy(client, np.ascontiguousarray(codes, dtype=np.uint8), fmt)


def up_f32(client, a):
    return TensorHandle.from_numpy(client, np.ascontiguousarray(a, dtype=np.float32), "f32")


def layout8(k8, lens, page, kind, fill=0, seed=0):
    """logical codes [B, Hkv, cap, D] -> (cache codes [P, page, Hkv, D] or the identity [B, cap, Hkv, D], table or None).  Slots
    at or past L_b and unused pages hold the byte `fill` (an int, or a tuple cycled through); table entries past ceil(L_b /
    page) are -1.  The same seed gives the same page permutation."""
    B, Hkv, cap, D = k8.shape
    rng = np.random.default_rng(seed)

    def stale(shape):
        f = np.atleast_1d(np.asarray(fill, dtype=np.uint8))
        return np.resize(f, int(np.prod(shape))).reshape(shape)

    t = k8.copy()
    for b, L in enumerate(lens):
        t[b, :, L:] = stale(t[b, :, L:].shape)
    if kind == "identity":
        return np.ascontiguousarray(t.transpose(0, 2, 1, 3)), None
    mp = cap // page
    P = B * mp + 3
    perm = rng.permutation(P)
    table = perm[:B * mp].reshape(B, mp).copy()
    for b, L in enumerate(lens):
        table[b, -(-L // page):] = -1
    cache = stale((P, page, Hkv, D))
    for b in range(B):
        for p in range(mp):
            cache[perm[b * mp + p]] = t[b, :, p * page:(p + 1) * page].transpose(1, 0, 2)
    return cache, table


def random_codes(rng, shape, fmt, spread=2.0):
    """finite fp8 codes of values uniform in [-spread, spread]"""
    return fo.quantize(rng.uniform(-spread, spread, (int(np.prod(shape[:-2])), shape[-2], shape[-1])).astype(np.float32),
                       np.ones(shape[-2], np.float32), fmt).reshape(shape)


def run8(client, q, kc8, vc8, table, lens, ks, vs, fmt, dtype, out_dtype, causal=False, scale=None, stream=None):
    qh = up(client, q, dtype)
    bt = None if table is None else up_i32(client, table)
    out, lse = attention.launch_kvcache_fp8_alloc(client, qh, up8(client, kc8, fmt), up8(client, vc8, fmt), up_i32(client, lens),
                                                  up_f32(client, ks), up_f32(client, vs), block_table=bt, scale=scale,
                                                  causal=causal, out_dtype=out_dtype, return_lse=True)
    client.sync()
    return values(client, out), values(client, lse), bits(client, out), bits(client, lse)


def run16(client, q, kc, vc, table, lens, dtype, out_dtype, causal=False, scale=None):
    bt = None if table is None else up_i32(client, table)
    out, lse = attention.launch_kvcache_alloc(client, up(client, q, dtype), up(client, kc, dtype), up(client, vc, dtype),
                                              up_i32(client, lens), block_table=bt, scale=scale, causal=causal,
                                              out_dtype=out_dtype, return_lse=True)
    client.sync()
    return bits(client, out), bits(client, lse)


# ---------------------------------------------------------------------------------------------- bits of the 16-bit kernel
BIT_CASES = [   # B, Hq, Hkv, Sq, D, page, max_pages, kind, causal, fmt, dtype
    (3, 32, 8, 1, 128, 16, 64, "paged", False, "f8e4m3", "bf16"),     # several splits
    (3, 32, 8, 1, 128, 16, 64, "paged", False, "f8e5m2", "f16"),
    (64, 8, 8, 1, 64, 32, 4, "paged", False, "f8e4m3", "f16"),        # one split
    (64, 8, 8, 1, 48, 32, 4, "paged", False, "f8e5m2", "bf16"),
    (5, 12, 4, 4, 112, 128, 3, "paged", True, "f8e4m3", "bf16"),      # Sq > 1 causal, GQA
    (5, 12, 4, 4, 112, 128, 3, "paged", True, "f8e5m2", "f16"),
    (4, 8, 2, 3, 128, 700, 1, "identity", True, "f8e4m3", "f16"),
    (2, 16, 2, 1, 64, 4096, 1, "identity", False, "f8e5m2", "bf16"),  # several splits, identity table
    (48, 4, 4, 17, 48, 32, 8, "paged", True, "f8e4m3", "f16"),
]


def test_bit_cases_cover_both_split_kinds():
    kinds = {nsplit(B, Hq, Hkv, Sq, page * mp) > 1 for B, Hq, Hkv, Sq, D, page, mp, *_ in BIT_CASES}
    assert kinds == {False, True}


@pytest.mark.parametrize("B,Hq,Hkv,Sq,D,page,mp,kind,causal,fmt,dtype", BIT_CASES)
@pytest.mark.parametrize("scales", ["ones", "pow2"])
def test_bits_equal_the_16_bit_kernel_on_the_dequantized_cache(client, B, Hq, Hkv, Sq, D, page, mp, kind, causal, fmt, dtype, scales):
    cap = page * mp
    rng = np.random.default_rng(B * Hq + Sq + D + page)
    lens = ragged(B, cap, min(page, cap), rng)
    q = rounded(rng.uniform(-2, 2, (B, Hq, Sq, D)), dtype)
    k8, v8 = random_codes(rng, (B, Hkv, cap, D), fmt), random_codes(rng, (B, Hkv, cap, D), fmt)
    if scales == "ones":
        ks = vs = np.ones(Hkv, np.float32)
    else:
        ks = (2.0 ** rng.integers(-3, 3, Hkv)).astype(np.float32)
        vs = (2.0 ** rng.integers(-3, 3, Hkv)).astype(np.float32)
    kc8, table = layout8(k8, lens, page, kind, seed=page)
    vc8, _ = layout8(v8, lens, page, kind, seed=page)
    kc16, vc16 = fo.dequantize(kc8, ks, fmt), fo.dequantize(vc8, vs, fmt)
    for out_dtype in (dtype, "f32"):
        _, _, got, got_lse = run8(client, q, kc8, vc8, table, lens, ks, vs, fmt, dtype, out_dtype, causal=causal)
        want, want_lse = run16(client, q, kc16, vc16, table, lens, dtype, out_dtype, causal=causal)
        assert np.array_equal(got, want), out_dtype
        assert np.array_equal(got_lse, want_lse), out_dtype


# ---------------------------------------------------------------------------------------------- random data, any scales
@pytest.mark.parametrize("fmt", fo.FORMATS)
@pytest.mark.parametrize("dtype", ["bf16", "f16"])
@pytest.mark.parametrize("B,Hq,Hkv,Sq,D,page,mp,causal", [
    (3, 32, 8, 1, 128, 16, 64, False), (2, 8, 2, 4, 64, 64, 10, True), (64, 8, 8, 1, 112, 32, 8, False), (3, 6, 3, 33, 48, 128, 3, True),
])
def test_random_against_the_oracle(client, fmt, dtype, B, Hq, Hkv, Sq, D, page, mp, causal):
    cap = page * mp
    rng = np.random.default_rng(B + Sq + D + page)
    lens = ragged(B, cap, page, rng)
    q = rounded(rng.uniform(-2, 2, (B, Hq, Sq, D)), dtype)
    k8, v8 = random_codes(rng, (B, Hkv, cap, D), fmt), random_codes(rng, (B, Hkv, cap, D), fmt)
    ks, vs = rng.uniform(0.05, 1.5, Hkv).astype(np.float32), rng.uniform(0.05, 3.0, Hkv).astype(np.float32)
    kc8, table = layout8(k8, lens, page, "paged", fill=STALE[fmt], seed=3)
    vc8, _ = layout8(v8, lens, page, "paged", fill=STALE[fmt], seed=3)
    ref, ref_lse = fo.attention_kvcache_fp8_f64(q, kc8, vc8, ks, vs, fmt, lens, table, None, causal)
    vmax = fo.dequantize(v8.transpose(0, 2, 1, 3), vs, fmt)
    for out_dtype in (dtype, "f32"):
        got, lse, _, _ = run8(client, q, kc8, vc8, table, lens, ks, vs, fmt, dtype, out_dtype, causal=causal)
        err = np.abs(got - ref) - _bound(ref, vmax, dtype, out_dtype)
        assert err.max() <= 0, float(err.max())
        fin = np.isfinite(ref_lse)
        assert np.array_equal(lse[~fin], ref_lse[~fin])
        np.testing.assert_allclose(lse[fin], ref_lse[fin], rtol=1e-5, atol=1e-5)


# ---------------------------------------------------------------------------------------------- stale slots
@pytest.mark.parametrize("fmt", fo.FORMATS)
@pytest.mark.parametrize("causal", [False, True])
def test_stale_nan_and_inf_bytes_never_reach_out(client, fmt, causal):
    B, Hq, Hkv, Sq, D, page, mp, dtype = 6, 8, 2, 3, 128, 16, 12, "bf16"
    cap = page * mp
    rng = np.random.default_rng(11)
    lens = [0, 1, 15, 17, 100, cap]
    q = rounded(rng.uniform(-2, 2, (B, Hq, Sq, D)), dtype)
    k8, v8 = random_codes(rng, (B, Hkv, cap, D), fmt), random_codes(rng, (B, Hkv, cap, D), fmt)
    ks, vs = np.array([0.3, 1.1], np.float32), np.array([2.5, 0.7], np.float32)
    ref = None
    for fill in (0,) + tuple((s,) for s in STALE[fmt]) + (STALE[fmt],):
        kc8, table = layout8(k8, lens, page, "paged", fill=fill, seed=5)
        vc8, _ = layout8(v8, lens, page, "paged", fill=fill, seed=5)
        vals, _, got, got_lse = run8(client, q, kc8, vc8, table, lens, ks, vs, fmt, dtype, dtype, causal=causal)
        assert np.isfinite(vals).all()
        if ref is None:
            ref = (got, got_lse)
        assert np.array_equal(got, ref[0]) and np.array_equal(got_lse, ref[1]), fill


# ---------------------------------------------------------------------------------------------- reproducibility
def test_repeats_and_two_streams_give_the_same_bits(client):
    B, Hq, Hkv, D, page, mp, dtype, fmt = 2, 32, 8, 128, 16, 256, "f16", "f8e4m3"
    cap = page * mp
    assert nsplit(B, Hq, Hkv, 1, cap) > 1
    rng = np.random.default_rng(17)
    lens = [4000, 1234]
    q = rounded(rng.uniform(-2, 2, (B, Hq, 1, D)), dtype)
    k8, v8 = random_codes(rng, (B, Hkv, cap, D), fmt), random_codes(rng, (B, Hkv, cap, D), fmt)
    kc8, table = layout8(k8, lens, page, "paged")
    vc8, _ = layout8(v8, lens, page, "paged")
    qh, sl, bt = up(client, q, dtype), up_i32(client, lens), up_i32(client, table)
    kh, vh = up8(client, kc8, fmt), up8(client, vc8, fmt)
    ksh, vsh = up_f32(client, rng.uniform(0.1, 1, Hkv)), up_f32(client, rng.uniform(0.1, 1, Hkv))
    streams = [client.create_stream(), client.create_stream()]
    outs = [[TensorHandle.empty_contiguous(client, [B, Hq, 1, D], "f32") for _ in range(3)] for _ in streams]
    try:
        for st, row in zip(streams, outs):
            for o in row:
                attention.launch_kvcache_fp8(client, qh, kh, vh, sl, ksh, vsh, o, block_table=bt, stream=st)
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


# ---------------------------------------------------------------------------------------------- kvcache_write_fp8
@pytest.mark.parametrize("fmt", fo.FORMATS)
@pytest.mark.parametrize("dtype", ["bf16", "f16"])
def test_write_quantizes_exactly_and_skips_slots(client, fmt, dtype):
    B, Snew, Hkv, D, P, page = 3, 5, 4, 64, 6, 16
    rng = np.random.default_rng(19)
    top = 60000.0 if dtype == "f16" else 1e6
    kn, vn = (rounded(rng.standard_normal((B, Snew, Hkv, D)) * 10.0 ** rng.uniform(-3, 2.5, (B, Snew, Hkv, 1)), dtype) for _ in range(2))
    kn[0, 0, 0, :4] = [np.nan, np.inf, -np.inf, top]
    vn[1, 2, 3, :3] = [-top, np.nan, 0.0]
    kn[2, 1, 1, 0] = -0.0
    kn, vn = rounded(kn, dtype), rounded(vn, dtype)
    ks, vs = np.array([0.5, 1.0, 0.013, 7.7], np.float32), np.array([2.0, 0.3, 1.0, 100.0], np.float32)
    slots = rng.permutation(P * page)[:B * Snew]
    slots[[2, 7]] = -1
    slots[9] = P * page   # past the cache: skipped
    sentinel = np.full((P, page, Hkv, D), 0xA5, np.uint8)
    kc, vc = up8(client, sentinel, fmt), up8(client, sentinel, fmt)
    attention.kvcache_write_fp8(client, up(client, kn, dtype), up(client, vn, dtype), kc, vc, up_i32(client, slots), up_f32(client, ks),
                                up_f32(client, vs))
    client.sync()
    for cache, new, s in ((kc, kn, ks), (vc, vn, vs)):
        want = sentinel.copy()
        codes = fo.quantize(new.reshape(B * Snew, Hkv, D), s, fmt)
        for n, sl in enumerate(slots):
            if 0 <= sl < P * page:
                want[sl // page, sl % page] = codes[n]
        got = cache.to_numpy(client).reshape(want.shape)
        nan = np.isnan(fo.decode(want, fmt))
        assert np.array_equal(np.isnan(fo.decode(got, fmt)), nan)
        assert np.array_equal(got[~nan], want[~nan])


def test_write_then_attend_round_trip(client):
    B, Hq, Hkv, Sq, D, page, mp, dtype, fmt = 3, 8, 2, 4, 128, 16, 8, "bf16", "f8e4m3"
    cap = page * mp
    rng = np.random.default_rng(23)
    lens = [100, 37, 128]
    q, k, v = (rounded(rng.uniform(-2, 2, s), dtype) for s in ((B, Hq, Sq, D), (B, Hkv, cap, D), (B, Hkv, cap, D)))
    ks, vs = np.array([0.01, 0.02], np.float32), np.array([0.015, 0.005], np.float32)
    table = np.random.default_rng(29).permutation(B * mp).reshape(B, mp)
    slots = np.full((B, cap), -1)
    for b, L in enumerate(lens):
        j = np.arange(L)
        slots[b, :L] = table[b, j // page] * page + j % page
    kc, vc = (up8(client, np.zeros((B * mp, page, Hkv, D), np.uint8), fmt) for _ in range(2))
    kn, vn = (up(client, t, dtype) for t in (k, v))   # [B, Hkv, cap, D] seen as [B, cap, Hkv, D] views
    views = [TensorHandle(t.handle, [B, cap, Hkv, D], [Hkv * cap * D, D, cap * D, 1], dtype) for t in (kn, vn)]
    ksh, vsh = up_f32(client, ks), up_f32(client, vs)
    attention.kvcache_write_fp8(client, *views, kc, vc, up_i32(client, slots), ksh, vsh)
    out = attention.launch_kvcache_fp8_alloc(client, up(client, q, dtype), kc, vc, up_i32(client, lens), ksh, vsh,
                                             block_table=up_i32(client, table), causal=True)
    client.sync()
    # the cache the host builds from the oracle's codes
    k8, v8 = (fo.quantize(np.ascontiguousarray(t.transpose(0, 2, 1, 3)).reshape(B * cap, Hkv, D), s, fmt).reshape(B, cap, Hkv, D)
              for t, s in ((k, ks), (v, vs)))
    hk, hv = np.zeros((B * mp, page, Hkv, D), np.uint8), np.zeros((B * mp, page, Hkv, D), np.uint8)
    for b, L in enumerate(lens):
        for j in range(L):
            hk[table[b, j // page], j % page] = k8[b, j]
            hv[table[b, j // page], j % page] = v8[b, j]
    assert np.array_equal(kc.to_numpy(client).reshape(hk.shape), hk)
    want = run8(client, q, hk, hv, table, lens, ks, vs, fmt, dtype, dtype, causal=True)[2]
    assert np.array_equal(bits(client, out), want)


def test_errors_are_deferred_to_sync(client):
    q = up(client, np.zeros((2, 4, 1, 64)), "bf16")
    kc = up8(client, np.zeros((2, 16, 3, 64), np.uint8), "f8e4m3")
    sl = up_i32(client, [1, 2])
    sc = up_f32(client, np.ones(3))
    out = TensorHandle.empty_contiguous(client, [2, 4, 1, 64], "bf16")
    attention.launch_kvcache_fp8(client, q, kc, kc, sl, sc, sc, out)   # Hq = 4 is not a multiple of Hkv = 3
    with pytest.raises(ServerError, match="multiple of Hkv"):
        client.sync()
