"""GPU: b200_attention on an H100.

Exact contracts (integer-valued operands, so every score and every p is exact):
- one-hot rows: in every row one visible key scores at least 128 / scale above every other visible key (every other exp2
  argument is <= -184, which is +0 in f32) and below 0, so an unmasked zero-filled tail key would win; when causal, a
  masked key scores higher still.  out must be v[chosen] bit for bit.  This pins the masks, the tails, the online rescale,
  the GQA head mapping and every index.
- uniform rows: q = 0 makes every p = 1, so out is the exact column mean of v.
Random data against the f64 oracle and against torch, views, streams and deferred errors."""
import numpy as np
import pytest
import torch

import attention_oracle as ao
from cubecl_b200 import ServerError, TensorHandle, attention, synth

pytestmark = pytest.mark.gpu


def up(client, vals, dtype):
    return TensorHandle.from_numpy(client, synth.to_device_dtype(np.ascontiguousarray(vals, np.float32), dtype), dtype)


def rounded(vals, dtype):
    return synth.from_device_dtype(synth.to_device_dtype(np.asarray(vals, np.float32), dtype), dtype).astype(np.float64)


def values(client, t):
    return synth.from_device_dtype(t.to_numpy(client), t.dtype).astype(np.float64).reshape(t.shape)


def bits(client, t):
    return np.asarray(t.to_numpy(client)).view(np.uint32 if t.dtype == "f32" else np.uint16)


def run(client, q, k, v, dtype, out_dtype, scale=None, causal=False, lse=False):
    qh, kh, vh = up(client, q, dtype), up(client, k, dtype), up(client, v, dtype)
    res = attention.launch_alloc(client, qh, kh, vh, scale=scale, causal=causal, out_dtype=out_dtype, return_lse=lse)
    client.sync()
    if lse:
        return values(client, res[0]), values(client, res[1])
    return values(client, res)


# ---------------------------------------------------------------------------------------------- exact: one-hot rows
# per input dtype: score step G between keys, offset C that makes every real score negative (also the decoy bonus), and the
# scale that makes the step 128 (f16 holds integers up to 65504, so its scores are 8x smaller)
ONE_HOT = {"bf16": (128, 131072.0, 1.0), "f16": (16, 16384.0, 8.0)}


def _digits(j):
    return np.stack([(j >> 8) & 15, (j >> 4) & 15, j & 15], axis=-1)


def one_hot_problem(B, Hq, Hkv, Sq, Sk, D, causal, where, dtype):
    """q, k, v and the chosen key of every (b, h, i).  A key j is the base-16 digits (d2, d1, d0) with their squares; q of a
    row whose chosen key has digits c scores G * (sum c^2 - sum (d - c)^2) - C: the chosen key is the unique maximum, every
    other key at least G below (G * scale = 128), every score negative.  Key Sk - 1 is a decoy with a +C bonus for rows that
    must not see it (causal, i < Sk - 1).  Every value is an integer a 16-bit float holds exactly, and every sum is exact in f32."""
    assert D >= 8 and Sk <= 4096
    G, C, _ = ONE_HOT[dtype]
    i = np.arange(Sq)
    vis = np.minimum(i + 1, Sk) if causal else np.full(Sq, Sk)
    chosen = np.zeros((B, Hq, Sq), np.int64)
    for b in range(B):
        for h in range(Hq):
            if where == "first":
                c = (i * 7 + h + b) % np.minimum(128, vis)
            elif where == "last":
                c = vis - 1 - (i + h + b) % np.minimum(vis, 5)
            else:   # the last visible block: the diagonal block when causal, the tail block otherwise
                c = 128 * ((vis - 1) // 128) + (i * 3 + h + b) % ((vis - 1) % 128 + 1)
            chosen[b, h] = c
    j = np.arange(Sk)
    dk = _digits(j)
    k = np.zeros((B, Hkv, Sk, D))
    k[..., 0:3] = dk
    k[..., 3:6] = dk ** 2
    k[..., 6] = 1.0
    k[..., Sk - 1, 7] = 1.0
    dc = _digits(chosen)
    q = np.zeros((B, Hq, Sq, D))
    q[..., 0:3] = 2 * G * dc
    q[..., 3:6] = -G
    q[..., 6] = -C
    if causal:
        q[..., 7] = np.where(i < Sk - 1, C, 0.0)
    bb, hk, jj, dd = np.meshgrid(np.arange(B), np.arange(Hkv), j, np.arange(D), indexing="ij")
    v = ((jj * 7 + dd * 3 + hk * 5 + bb) % 257 - 128).astype(np.float64)
    return q, k, v, chosen


@pytest.mark.parametrize("dtype", ["bf16", "f16"])
@pytest.mark.parametrize("D,Sq,Sk,Hq,Hkv,causal", [
    (8, 200, 300, 4, 2, False), (40, 300, 200, 2, 1, True), (64, 129, 129, 2, 2, True), (72, 100, 390, 6, 3, False),
    (128, 257, 257, 2, 1, True), (128, 60, 140, 2, 2, False),
])
@pytest.mark.parametrize("where", ["first", "last", "diag"])
def test_one_hot_rows_exact(client, dtype, D, Sq, Sk, Hq, Hkv, causal, where):
    B = 2
    q, k, v, chosen = one_hot_problem(B, Hq, Hkv, Sq, Sk, D, causal, where, dtype)
    g = Hq // Hkv
    want = np.empty((B, Hq, Sq, D))
    for b in range(B):
        for h in range(Hq):
            want[b, h] = v[b, h // g, chosen[b, h]]
    for out_dtype in (dtype, "f32"):
        got = run(client, q, k, v, dtype, out_dtype, scale=ONE_HOT[dtype][2], causal=causal)
        if out_dtype == "f32":
            np.testing.assert_allclose(got, want, rtol=2.0 ** -20, atol=0)
        else:
            np.testing.assert_array_equal(got, want)


# ---------------------------------------------------------------------------------------------- exact: uniform rows
@pytest.mark.parametrize("dtype", ["bf16", "f16"])
@pytest.mark.parametrize("D,Sk", [(64, 256), (128, 512), (40, 128), (96, 1024)])
def test_uniform_rows_give_the_exact_column_mean(client, dtype, D, Sk):
    B, H, Sq = 2, 3, 77
    q = np.zeros((B, H, Sq, D))
    k = np.random.default_rng(D + Sk).integers(-8, 9, (B, H, Sk, D)).astype(np.float64)
    jj, dd = np.meshgrid(np.arange(Sk), np.arange(D), indexing="ij")
    v = np.broadcast_to((jj % 4 - 1 + dd % 3).astype(np.float64), (B, H, Sk, D))   # column mean 0.5 + d % 3
    want = np.broadcast_to(v.mean(axis=2, keepdims=True), (B, H, Sq, D))
    for out_dtype in (dtype, "f32"):
        np.testing.assert_array_equal(run(client, q, k, v, dtype, out_dtype, scale=0.3), want)


# ---------------------------------------------------------------------------------------------- random data
def _bound(ref, v, dtype, out_dtype):
    """P rounded to the input dtype (unit roundoff u) moves out by at most u * max|v| per row; twice that for slack, plus the
    output rounding and the f32 / ex2.approx terms"""
    u = 2.0 ** -8 if dtype == "bf16" else 2.0 ** -11
    uo = {"bf16": 2.0 ** -8, "f16": 2.0 ** -11, "f32": 0.0}[out_dtype]
    return 2 * u * np.abs(v).max() + uo * np.abs(ref) + 1e-5


@pytest.mark.parametrize("dtype", ["bf16", "f16"])
@pytest.mark.parametrize("B,Hq,Hkv,Sq,Sk,D,causal", [
    (2, 4, 4, 333, 333, 64, False), (1, 8, 2, 300, 513, 128, True), (2, 4, 1, 517, 200, 128, False), (1, 2, 2, 1, 700, 64, False),
    (1, 3, 3, 250, 250, 40, True), (1, 2, 1, 1000, 1000, 96, True),
])
def test_random_against_the_oracle(client, dtype, B, Hq, Hkv, Sq, Sk, D, causal):
    rng = np.random.default_rng(Sq + Sk + D)
    q, k, v = (rounded(rng.uniform(-2, 2, s), dtype) for s in ((B, Hq, Sq, D), (B, Hkv, Sk, D), (B, Hkv, Sk, D)))
    ref, ref_lse = ao.attention_f64(q, k, v, None, causal)
    for out_dtype in (dtype, "f32"):
        got, lse = run(client, q, k, v, dtype, out_dtype, causal=causal, lse=True)
        err = np.abs(got - ref) - _bound(ref, v, dtype, out_dtype)
        assert err.max() <= 0, float(err.max())
        np.testing.assert_allclose(lse, ref_lse, rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("causal", [False, True])
def test_matches_torch_on_the_gpu(client, causal):
    B, H, S, D = 1, 8, 2048, 128
    g = torch.Generator(device="cuda").manual_seed(7)
    qt, kt, vt = (torch.rand((B, H, S, D), device="cuda", generator=g, dtype=torch.float32).mul_(4).sub_(2).to(torch.bfloat16)
                  for _ in range(3))
    ref = torch.nn.functional.scaled_dot_product_attention(qt, kt, vt, is_causal=causal).float().cpu().numpy().astype(np.float64)
    q, k, v = (t.float().cpu().numpy().astype(np.float64) for t in (qt, kt, vt))
    got = run(client, q, k, v, "bf16", "bf16", causal=causal)
    # both round P to bf16: the difference is within the sum of the two bounds
    assert (np.abs(got - ref) - 2 * _bound(ref, v, "bf16", "bf16")).max() <= 0


# ---------------------------------------------------------------------------------------------- views, streams, errors
def test_views_give_identical_bits(client):
    B, H, S, D = 2, 4, 300, 64
    rng = np.random.default_rng(3)
    qkv = rounded(rng.uniform(-2, 2, (B, S, 3, H, D)), "bf16")
    fused = up(client, qkv, "bf16")
    st5 = [S * 3 * H * D, D, 3 * H * D, 1]
    sl = [TensorHandle(fused.handle.offset(i * H * D * 2), [B, H, S, D], st5, "bf16") for i in range(3)]
    compact = [up(client, np.ascontiguousarray(qkv[:, :, i].transpose(0, 2, 1, 3)), "bf16") for i in range(3)]
    bshd = []
    for i in range(3):
        t = up(client, np.ascontiguousarray(qkv[:, :, i]), "bf16")   # [B, S, H, D] as a [B, H, S, D] view
        bshd.append(TensorHandle(t.handle, [B, H, S, D], [S * H * D, D, H * D, 1], "bf16"))
    # a misaligned k: one element into a buffer, so the base is not 16-byte aligned and the operand is gathered
    kbuf = up(client, np.concatenate([[0.0], qkv[:, :, 1].transpose(0, 2, 1, 3).reshape(-1)]), "bf16")
    mis = [compact[0], TensorHandle(kbuf.handle.offset(2), [B, H, S, D], compact[1].strides, "bf16"), compact[2]]
    outs = []
    for ops in (compact, sl, bshd, mis):
        o = TensorHandle.empty_contiguous(client, [B, H, S, D], "bf16")
        attention.launch(client, *ops, o, causal=True)
        outs.append(o)
    client.sync()
    ref = bits(client, outs[0])
    for o in outs[1:]:
        assert np.array_equal(bits(client, o), ref)
    # a [B, S, H, D] output view of the same values
    ob = TensorHandle.empty_contiguous(client, [B, S, H, D], "bf16")
    attention.launch(client, *compact, TensorHandle(ob.handle, [B, H, S, D], [S * H * D, D, H * D, 1], "bf16"), causal=True)
    client.sync()
    assert np.array_equal(bits(client, ob).reshape(B, S, H, D).transpose(0, 2, 1, 3), ref.reshape(B, H, S, D))


def test_two_streams_and_repeats_give_the_same_bits(client):
    B, H, S, D = 2, 4, 700, 128
    rng = np.random.default_rng(5)
    q, k, v = (up(client, rng.uniform(-2, 2, (B, H, S, D)), "f16") for _ in range(3))
    streams = [client.create_stream(), client.create_stream()]
    outs = [[TensorHandle.empty_contiguous(client, [B, H, S, D], "f32") for _ in range(3)] for _ in streams]
    try:
        for st, row in zip(streams, outs):
            for o in row:
                attention.launch(client, q, k, v, o, causal=True, stream=st)
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


def test_errors_are_deferred_to_sync(client):
    q = up(client, np.zeros((1, 4, 8, 64)), "bf16")
    k = up(client, np.zeros((1, 3, 8, 64)), "bf16")
    out = TensorHandle.empty_contiguous(client, [1, 4, 8, 64], "bf16")
    attention.launch(client, q, k, k, out)   # Hq = 4 is not a multiple of Hkv = 3: no raise here
    with pytest.raises(ServerError, match="multiple of Hkv"):
        client.sync()
    attention.launch(client, q, q, q, TensorHandle.empty_contiguous(client, [1, 4, 8, 64], "f16"))
    with pytest.raises(ServerError, match="output dtype"):
        client.sync()
