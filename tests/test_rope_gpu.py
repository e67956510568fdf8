"""GPU: b200_rope, b200_rope_kvcache_write and b200_rope_cos_sin against tests/rope_oracle.py -- bit for bit for every dtype
and style, head dims 64 to 512, full and partial rotary, in place and out of place, GQA, q-only and k-only calls, head-major
views and the q / k slices of a fused QKV buffer, the 16-byte and the element-wise path, null / random / out-of-range
positions with -0, inf and NaN rows, token rows past the grid cap, the inverse against the oracle and against autograd;
sentinels around every output, two streams; the fused cache write against b200_rope + b200_kvcache_write(_fp8), and a
decode step through b200_attention_kvcache; the tables within one f32 ulp of their f64 value."""
import numpy as np
import pytest
import torch

import rope_oracle as ro
from cubecl_b200 import TensorHandle, attention, rope

pytestmark = pytest.mark.gpu

ESZ = {"f32": 4, "bf16": 2, "f16": 2}


def up_bits(c, b, dt):
    return TensorHandle.from_numpy(c, np.ascontiguousarray(b), dt)


def up(c, x, dt):
    return up_bits(c, ro.to_bits(x, dt), dt)


def bits(c, t):
    return t.to_numpy(c).view(ro.BITS[t.dtype] if t.dtype in ro.BITS else np.uint8)


def table_dev(c, tab):
    return TensorHandle.from_numpy(c, np.ascontiguousarray(tab, np.float32), "f32")


def rand_table(rng, P, rot):
    ang = rng.uniform(0, 6.3, (P, rot // 2))
    return np.concatenate([np.cos(ang), np.sin(ang)], 1).astype(np.float32)


def rand_x(rng, shape, dt):
    return ro.rnd(rng.standard_normal(shape).astype(np.float32) * 3, dt)


def view_in(c, x, dt, layout="bshd", lead=0, pad=0, fill=7.0):
    """x [B, S, H, D] stored as a view: "bshd" rows padded by `pad` elements, or head-major "bhsd"; the buffer starts `lead`
    elements before the view and is filled with `fill` elsewhere.  Returns (view, buffer, buffer values)."""
    B, S, H, D = x.shape
    if layout == "bshd":
        st = [S * H * (D + pad), H * (D + pad), D + pad, 1]
    else:
        st = [H * S * (D + pad), D + pad, S * (D + pad), 1]
    n = lead + B * S * H * (D + pad) + 8
    flat = np.full(n, fill, np.float32)
    idx = lead + np.arange(B)[:, None, None, None] * st[0] + np.arange(S)[None, :, None, None] * st[1] + \
        np.arange(H)[None, None, :, None] * st[2] + np.arange(D)[None, None, None, :]
    flat[idx] = x
    buf = up(c, flat, dt)
    return TensorHandle(buf.handle.offset(lead * ESZ[dt]), [B, S, H, D], st, dt), buf, flat, idx


CASES = [(64, 64), (80, 80), (96, 24), (128, 128), (128, 64), (256, 256), (512, 512), (128, 2), (80, 32)]


@pytest.mark.parametrize("dt", ["f32", "bf16", "f16"])
@pytest.mark.parametrize("style", ["neox", "gptj"])
@pytest.mark.parametrize("D,rot", CASES)
def test_rope_matches_oracle_bitwise(client, dt, style, D, rot):
    rng = np.random.default_rng(D * 7 + rot)
    B, S, Hq, Hk, P = 2, 9, 4, 2, 40
    tab = rand_table(rng, P, rot)
    cs = table_dev(client, tab)
    q, k = rand_x(rng, (B, S, Hq, D), dt), rand_x(rng, (B, S, Hk, D), dt)
    pos = rng.integers(0, P, (B, S)).astype(np.int32)
    pd = TensorHandle.from_numpy(client, pos, "i32")
    for inverse in (False, True):
        want_q = ro.apply(q, tab, pos, style, rot, dt, inverse)
        want_k = ro.apply(k, tab, pos, style, rot, dt, inverse)
        # out of place, 16-byte path
        qo, ko = rope.apply_alloc(client, cs, up(client, q, dt), up(client, k, dt), pd, style=style, inverse=inverse)
        client.sync()
        assert np.array_equal(bits(client, qo), ro.to_bits(want_q, dt)) and np.array_equal(bits(client, ko), ro.to_bits(want_k, dt))
        # in place through misaligned, padded views (element-wise path), q-only then k-only, sentinels untouched
        for name, x, want in (("q", q, want_q), ("k", k, want_k)):
            v, buf, flat, idx = view_in(client, x, dt, lead=1, pad=3)
            rope.apply(client, cs, **{name: v}, positions=pd, style=style, inverse=inverse)
            client.sync()
            exp = ro.to_bits(flat, dt)
            exp[idx] = ro.to_bits(want, dt)
            assert np.array_equal(bits(client, buf), exp), name


@pytest.mark.parametrize("dt", ["bf16", "f32"])
@pytest.mark.parametrize("style", ["neox", "gptj"])
def test_views_fused_qkv_head_major_and_null_positions(client, dt, style):
    rng = np.random.default_rng(3)
    T, Hq, Hk, D, rot, P = 37, 8, 2, 128, 128, 64
    tab = rand_table(rng, P, rot)
    cs = table_dev(client, tab)
    qkv = rand_x(rng, (T, Hq + 2 * Hk, D), dt)
    buf = up(client, qkv, dt)
    e = ESZ[dt]
    st = [T * (Hq + 2 * Hk) * D, (Hq + 2 * Hk) * D, D, 1]
    qv = TensorHandle(buf.handle, [1, T, Hq, D], st, dt)
    kv = TensorHandle(buf.handle.offset(Hq * D * e), [1, T, Hk, D], st, dt)
    rope.apply(client, cs, qv, kv, None, style=style)                 # positions = s
    client.sync()
    pos = np.arange(T)[None, :]
    want = qkv.copy()
    want[:, :Hq] = ro.apply(qkv[None, :, :Hq], tab, pos, style, rot, dt)[0]
    want[:, Hq:Hq + Hk] = ro.apply(qkv[None, :, Hq:Hq + Hk], tab, pos, style, rot, dt)[0]
    assert np.array_equal(bits(client, buf), ro.to_bits(want, dt))     # v's bytes unchanged
    # head-major [B, H, S, D] views in and out
    x = rand_x(rng, (2, 11, 3, D), dt)
    v, _, _, _ = view_in(client, x, dt, layout="bhsd")
    o, obuf, oflat, oidx = view_in(client, np.zeros_like(x), dt, layout="bhsd", fill=5.0)
    rope.apply(client, cs, k=v, k_out=o, style=style)
    client.sync()
    exp = ro.to_bits(oflat, dt)
    exp[oidx] = ro.to_bits(ro.apply(x, tab, np.tile(np.arange(11), (2, 1)), style, rot, dt), dt)
    assert np.array_equal(bits(client, obuf), exp)


@pytest.mark.parametrize("dt", ["f32", "bf16", "f16"])
@pytest.mark.parametrize("inplace", [True, False])
def test_out_of_range_rows_are_kept_bit_for_bit(client, dt, inplace):
    rng = np.random.default_rng(5)
    B, S, H, D, rot, P = 2, 8, 3, 96, 64, 16
    tab = rand_table(rng, P, rot)
    x = rand_x(rng, (B, S, H, D), dt)
    x[:, ::2, :, 0] = -0.0
    x[:, 1::4, :, 1] = np.inf
    x[:, 3::4, :, 2] = np.nan
    pos = rng.integers(0, P, (B, S)).astype(np.int32)
    pos[0, :4] = [-1, P, P + 100, -(2 ** 31)]
    pos[1, 5] = 2 ** 31 - 1
    xb = ro.to_bits(x, dt)
    xd = up_bits(client, xb, dt)
    pd = TensorHandle.from_numpy(client, pos, "i32")
    if inplace:
        rope.apply(client, table_dev(client, tab), q=xd, positions=pd)
        out = xd
    else:
        out = rope.apply_alloc(client, table_dev(client, tab), q=xd, positions=pd)[0]
    client.sync()
    got = bits(client, out)
    bad = (pos < 0) | (pos >= P)
    assert np.array_equal(got[bad], xb[bad])
    # a rotated NaN is a NaN (its payload is the GPU's); every other element bit for bit
    want = ro.to_bits(ro.apply(x, tab, pos, "neox", rot, dt), dt)[~bad]
    nan = np.isnan(ro.from_bits(want, dt))
    assert np.array_equal(np.isnan(ro.from_bits(got[~bad], dt)), nan) and np.array_equal(got[~bad][~nan], want[~nan])


def test_rows_past_the_grid_cap(client):
    rng = np.random.default_rng(9)
    sms = client.properties["num_streaming_multiprocessors"]
    T = sms * 4 * 256 // 8 * 3 + 1001        # token * group units three times the capped grid
    D, rot, P = 128, 128, 4096
    tab = rand_table(rng, P, rot)
    x = rand_x(rng, (1, T, 1, D), "bf16")
    pos = rng.integers(-3, P + 3, (1, T)).astype(np.int32)
    xd = up(client, x, "bf16")
    rope.apply(client, table_dev(client, tab), k=xd, positions=TensorHandle.from_numpy(client, pos, "i32"), style="gptj")
    client.sync()
    assert np.array_equal(bits(client, xd), ro.to_bits(ro.apply(x, tab, pos, "gptj", rot, "bf16"), "bf16"))


def test_inverse_is_the_autograd_backward(client):
    rng = np.random.default_rng(11)
    B, S, H, D, P = 2, 16, 4, 64, 32
    inv = ro.inv_freq(D, 10000.0)
    cos, sin = ro.table_f64(P, inv, 1.0)
    tab = np.concatenate([cos, sin], 1).astype(np.float32)
    x = rng.standard_normal((B, S, H, D))
    dy = rng.standard_normal((B, S, H, D)).astype(np.float32)
    pos = rng.integers(0, P, (B, S))
    xt = torch.tensor(x, requires_grad=True)
    ct = torch.tensor(tab[:, :D // 2], dtype=torch.float64)[pos][:, :, None].repeat(1, 1, 1, 2)
    st = torch.tensor(tab[:, D // 2:], dtype=torch.float64)[pos][:, :, None].repeat(1, 1, 1, 2)
    rot_half = lambda t: torch.cat([-t[..., D // 2:], t[..., :D // 2]], -1)   # noqa: E731
    (xt * ct + rot_half(xt) * st).mul(torch.tensor(dy, dtype=torch.float64)).sum().backward()
    dq = rope.apply_alloc(client, table_dev(client, tab), q=up(client, dy, "f32"),
                          positions=TensorHandle.from_numpy(client, pos.astype(np.int32), "i32"), inverse=True)[0]
    client.sync()
    got = dq.to_numpy(client)
    assert np.array_equal(got, ro.apply(dy, tab, pos, "neox", D, "f32", inverse=True))
    assert np.max(np.abs(got - xt.grad.numpy())) <= 4 * 2.0 ** -24 * (np.abs(dy).max() * 2)


def test_two_streams_give_identical_bits(client):
    rng = np.random.default_rng(13)
    tab = rand_table(rng, 64, 128)
    cs = table_dev(client, tab)
    x = up(client, rand_x(rng, (4, 64, 8, 128), "bf16"), "bf16")
    outs = []
    for _ in range(2):
        s = client.create_stream()
        o = TensorHandle.empty_contiguous(client, x.shape, "bf16")
        rope.apply(client, cs, q=x, q_out=o, stream=s)
        client.sync_stream(s)
        outs.append(bits(client, o))
        client.destroy_stream(s)
    assert np.array_equal(outs[0], outs[1])


# ---------------------------------------------------------------------------------------------- fused cache write
@pytest.mark.parametrize("dt", ["bf16", "f16"])
@pytest.mark.parametrize("cache", ["same", "f8e4m3", "f8e5m2"])
@pytest.mark.parametrize("style,rot", [("neox", 128), ("gptj", 128), ("neox", 64)])
@pytest.mark.parametrize("page,q_inplace", [(16, True), (16, False), (None, True)])
def test_fused_cache_write_equals_rope_then_kvcache_write(client, dt, cache, style, rot, page, q_inplace):
    rng = np.random.default_rng(17)
    B, Sn, Hq, Hkv, D, P = 3, 5, 8, 2, 128, 64
    pg = page or 32                                           # None: an identity cache, one page per sequence
    Pp = 12 if page else B
    cd = dt if cache == "same" else cache
    tab = rand_table(rng, P, rot)
    cs = table_dev(client, tab)
    q, k, v = rand_x(rng, (B, Sn, Hq, D), dt), rand_x(rng, (B, Sn, Hkv, D), dt), rand_x(rng, (B, Sn, Hkv, D), dt)
    pos = rng.integers(0, P, (B, Sn)).astype(np.int32)
    pos[0, 0] = P + 1                                        # out of range: k kept, still written
    slots = rng.permutation(Pp * pg)[:B * Sn].astype(np.int32)
    slots[1], slots[4] = -1, Pp * pg                          # skipped
    ks, vs = np.float32([0.5, 0.25]), np.float32([2.0, 0.125])
    kcb = np.zeros((Pp, pg, Hkv, D), ro.BITS[dt] if cache == "same" else np.uint8) + 3
    args = dict(cache=None if cache == "same" else cache, k_scale=ks, v_scale=vs)
    dev = lambda a, d: TensorHandle.from_numpy(client, a, d)   # noqa: E731
    # fused
    kc, vc = dev(kcb, cd), dev(kcb.copy(), cd)
    qd = up(client, q, dt)
    qo = None if q_inplace else TensorHandle.empty_contiguous(client, q.shape, dt)
    f8 = cache != "same"
    rope.kvcache_write(client, cs, qd, up(client, k, dt), up(client, v, dt), kc, vc, dev(slots, "i32"), dev(pos, "i32"), q_out=qo,
                       k_scale=dev(ks, "f32") if f8 else None, v_scale=dev(vs, "f32") if f8 else None, style=style)
    # unfused: b200_rope + b200_kvcache_write(_fp8)
    kc2, vc2 = dev(kcb, cd), dev(kcb.copy(), cd)
    q2, k2 = up(client, q, dt), up(client, k, dt)
    rope.apply(client, cs, q2, k2, dev(pos, "i32"), style=style)
    if f8:
        attention.kvcache_write_fp8(client, k2, up(client, v, dt), kc2, vc2, dev(slots, "i32"), dev(ks, "f32"), dev(vs, "f32"))
    else:
        attention.kvcache_write(client, k2, up(client, v, dt), kc2, vc2, dev(slots, "i32"))
    client.sync()
    assert np.array_equal(bits(client, qo if qo is not None else qd), bits(client, q2))
    assert np.array_equal(bits(client, kc), bits(client, kc2)) and np.array_equal(bits(client, vc), bits(client, vc2))
    # and the oracle
    kr = ro.apply(k, tab, pos, style, rot, dt)
    wk, wv = ro.kvcache_write(kcb, kcb.copy(), kr, v, slots, dt, args["cache"], ks, vs)
    assert np.array_equal(bits(client, kc), wk) and np.array_equal(bits(client, vc), wv)
    if f8:   # the mutant that encodes K from the unrounded f32 rotation differs somewhere (it is what the contract rules out)
        kr32 = ro.apply(k, tab, pos, style, rot, "f32")
        bad = ro.kvcache_write(kcb, kcb.copy(), kr, v, slots, dt, args["cache"], ks, vs, _mutant="fp8_from_f32", k_raw=kr32)[0]
        assert not np.array_equal(bad, wk)


def test_decode_step_through_attention_matches_unfused(client):
    rng = np.random.default_rng(19)
    B, Hq, Hkv, D, page, Pp, P = 4, 8, 2, 128, 16, 32, 256
    tab = ro.table(P, ro.inv_freq(D, 10000.0), 1.0)
    cs = table_dev(client, tab)
    lens = np.int32([5, 17, 33, 1])
    bt = np.arange(B * 8, dtype=np.int32).reshape(B, 8)
    slots = np.int32([bt[b, lens[b] // page] * page + lens[b] % page for b in range(B)])
    q, k, v = (rand_x(rng, (B, 1, h, D), "bf16") for h in (Hq, Hkv, Hkv))
    kc0 = ro.to_bits(rand_x(rng, (Pp, page, Hkv, D), "bf16"), "bf16")
    dev = lambda a, d: TensorHandle.from_numpy(client, a, d)   # noqa: E731
    outs = []
    for fused in (True, False):
        kc, vc = dev(kc0, "bf16"), dev(kc0.copy(), "bf16")
        qd = up(client, q, "bf16")
        if fused:
            rope.kvcache_write(client, cs, qd, up(client, k, "bf16"), up(client, v, "bf16"), kc, vc, dev(slots, "i32"), dev(lens, "i32"))
        else:
            kd = up(client, k, "bf16")
            rope.apply(client, cs, qd, kd, dev(lens, "i32"))
            attention.kvcache_write(client, kd, up(client, v, "bf16"), kc, vc, dev(slots, "i32"))
        qh = TensorHandle(qd.handle, [B, Hq, 1, D], [Hq * D, D, D, 1], "bf16")
        out = attention.launch_kvcache_alloc(client, qh, kc, vc, dev(lens + 1, "i32"), block_table=dev(bt, "i32"))
        client.sync()
        outs.append(bits(client, out))
    assert np.array_equal(outs[0], outs[1])


# ---------------------------------------------------------------------------------------------- tables
TABLES = [
    dict(kind="default", base=10000.0),
    dict(kind="default", base=500000.0),
    dict(kind="linear", base=10000.0, factor=4.0),
    dict(kind="llama3", base=500000.0, factor=8.0, low_freq_factor=1.0, high_freq_factor=4.0, orig=8192),
    dict(kind="yarn", base=10000.0, factor=40.0, orig=4096, beta_fast=32.0, beta_slow=1.0, mscale=1.0, mscale_all_dim=1.0),
    dict(kind="yarn", base=1000000.0, factor=4.0, orig=32768, truncate=False),
]


@pytest.mark.parametrize("case", range(len(TABLES)))
def test_table_within_one_ulp_of_f64(client, case):
    t = dict(TABLES[case])
    P, rot = 1 << 20, 128
    scaling = {"rope_type": t["kind"], "factor": t.get("factor"), "low_freq_factor": t.get("low_freq_factor"),
               "high_freq_factor": t.get("high_freq_factor"), "original_max_position_embeddings": t.get("orig"),
               "beta_fast": t.get("beta_fast"), "beta_slow": t.get("beta_slow"), "mscale": t.get("mscale"),
               "mscale_all_dim": t.get("mscale_all_dim"), "truncate": t.get("truncate", True)}
    scaling = {k: v for k, v in scaling.items() if v is not None}
    got = rope.cos_sin_alloc(client, P, rot, t["base"], scaling).to_numpy(client)
    inv = ro.inv_freq(rot, t["base"], t["kind"], t.get("factor", 1.0), t.get("low_freq_factor", 0.0), t.get("high_freq_factor", 0.0),
                      t.get("orig", 0), t.get("beta_fast", 0.0), t.get("beta_slow", 0.0), t.get("truncate", True))
    af = ro.attention_factor(t["kind"], t.get("factor", 1.0), t.get("mscale", 0.0), t.get("mscale_all_dim", 0.0))
    c, s = ro.table_f64(P, inv, af)
    ref = np.concatenate([c, s], 1)
    ulp = np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64)
    # one f32 ulp, plus the conditioning of cos / sin on the f64 angle itself: p * inv_freq_i carries a few f64 ulps (pow
    # and the product round on both sides), which near a zero of cos or sin at large angles exceeds an f32 ulp of the value
    ang = np.arange(P, dtype=np.float64)[:, None] * inv[None, :]
    cond = 8 * 2.0 ** -53 * np.concatenate([ang, ang], 1) * af
    err = np.abs(got - ref)
    assert np.all(err <= ulp + cond)
    print(f"{t['kind']}: {np.count_nonzero(got != ref.astype(np.float32))} of {ref.size} entries not identical to rn_f32(f64), "
          f"{np.count_nonzero(err > ulp)} beyond one f32 ulp (all within the angle's f64 conditioning)")


def test_table_from_inv_freq(client):
    inv = (1.0 / 10000.0 ** (np.arange(0, 64, 2) / 64)).astype(np.float32)
    got = rope.cos_sin_alloc(client, 4096, 64, inv_freq=TensorHandle.from_numpy(client, inv, "f32"), attention_factor=0.5).to_numpy(client)
    c, s = ro.table_f64(4096, inv.astype(np.float64), 0.5)
    ref = np.concatenate([c, s], 1)
    assert np.all(np.abs(got - ref) <= np.spacing(np.abs(ref).astype(np.float32)))


def test_flash_attn_rotary_agrees_within_bound(client):
    fa = pytest.importorskip("flash_attn.layers.rotary")
    rng = np.random.default_rng(23)
    B, S, H, D, rot = 2, 64, 4, 128, 64
    tab = ro.table(S, ro.inv_freq(rot), 1.0)
    x = rand_x(rng, (B, S, H, D), "bf16")
    xt = torch.tensor(x, dtype=torch.bfloat16, device="cuda")
    ct = torch.tensor(tab[:, :rot // 2], device="cuda")
    st = torch.tensor(tab[:, rot // 2:], device="cuda")
    ref = fa.apply_rotary_emb(xt, ct, st, interleaved=True).float().cpu().numpy()
    got = ro.from_bits(bits(client, rope.apply_alloc(client, table_dev(client, tab), q=up(client, x, "bf16"), style="gptj", rot_dim=rot)[0]), "bf16")
    assert np.max(np.abs(got - ref)) <= 2 * 2.0 ** -8 * (np.abs(x).max() * 2)
