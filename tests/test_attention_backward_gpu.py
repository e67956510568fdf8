"""GPU: b200_attention_backward on an H100.  Every test takes out and lse from the library's own forward.

Exact contracts (integer-valued operands, scale = ln 2 so the forward's scale_log2 is exactly 1.0f and t = s):
- one-hot rows: in every row one visible key scores t = -r (1 <= r <= 60) and every other visible key scores at least 160
  below it, so p rounds to exactly 1 for the chosen key and to +0 elsewhere (exp2 of <= -150 is +0 under ftz).  A zero-filled
  key past Sk would score 0, above the chosen key; when causal, key Sk - 1 carries a bonus that puts it above the chosen key
  for the rows that must not see it.  out = v[chosen] exactly, so delta = dout . v[chosen] = dP[chosen] and dS = 0: dq and
  dk must be exactly 0, and dv[j] the exact sum of dout over every (group head, row) that chose j (rounded once, RNE, for a
  16-bit grad dtype).  This pins the masks, the tails, the GQA sums, the causal skips and every index of P.
- uniform rows: q = 0 and Sk = 2^k make every 16-bit P exactly 2^-k, so dv = 2^-k * (sum of dout over all rows and group
  heads), exactly: every query block reaches every key.
Random data against the f64 oracle within a bound derived from where the kernels round, one S = 2048 case against torch's
backward on the GPU, bit-identical results across repeats, streams and views, and deferred errors."""
import math

import numpy as np
import pytest
import torch

import attention_oracle as ao
from cubecl_b200 import ServerError, TensorHandle, attention, synth

pytestmark = pytest.mark.gpu

LN2 = math.log(2.0)


def ein(spec, *ops):
    return np.einsum(spec, *ops, optimize=True)


U = {"bf16": 2.0 ** -8, "f16": 2.0 ** -11, "f32": 0.0}   # unit roundoff of each dtype (f32 outputs: no output rounding)


def up(client, vals, dtype):
    return TensorHandle.from_numpy(client, synth.to_device_dtype(np.ascontiguousarray(vals, np.float32), dtype), dtype)


def rounded(vals, dtype):
    if dtype == "f32":
        return np.asarray(vals, np.float32).astype(np.float64)
    return synth.from_device_dtype(synth.to_device_dtype(np.asarray(vals, np.float32), dtype), dtype).astype(np.float64)


def values(client, t):
    return synth.from_device_dtype(t.to_numpy(client), t.dtype).astype(np.float64).reshape(t.shape)


def bits(client, t):
    return np.asarray(t.to_numpy(client)).view(np.uint32 if t.dtype == "f32" else np.uint16)


def forward(client, qh, kh, vh, out_dtype, scale, causal):
    return attention.launch_alloc(client, qh, kh, vh, scale=scale, causal=causal, out_dtype=out_dtype, return_lse=True)


def run(client, q, k, v, dout, dtype, out_dtype, grad_dtype, scale=None, causal=False):
    qh, kh, vh, doh = (up(client, t, dtype) for t in (q, k, v, dout))
    out, lse = forward(client, qh, kh, vh, out_dtype, scale, causal)
    dq, dk, dv = attention.launch_backward_alloc(client, qh, kh, vh, out, doh, lse, scale=scale, causal=causal, grad_dtype=grad_dtype)
    client.sync()
    return values(client, dq), values(client, dk), values(client, dv)


# ---------------------------------------------------------------------------------------------- exact: one-hot rows
G_STEP = 160          # score step between the chosen key and the next best
DECOY = 61440.0       # 15 * 2^12: a 16-bit value in both dtypes, above every score gap of the problem


def one_hot_problem(B, Hq, Hkv, Sq, Sk, D, causal, where):
    """q, k, v, dout and the chosen key of every (b, h, i).  Key j is its base-`base` digits d with their squares; a row whose
    chosen key has digits c scores G (|c|^2 - |d - c|^2) - G |c|^2 - r = -r - G |d - c|^2 (the bias -G |c|^2 - r split over
    two dims so each part is a 16-bit value).  Every operand is an integer both 16-bit dtypes hold, every sum exact in f32."""
    ndig = 2 if D < 9 else 3
    base = 2
    while base ** ndig < Sk:
        base += 1
    assert G_STEP * ndig * (base - 1) ** 2 + 64 < DECOY and 2 * ndig + 3 <= D
    i = np.arange(Sq)
    vis = np.minimum(i + 1, Sk) if causal else np.full(Sq, Sk)
    chosen = np.zeros((B, Hq, Sq), np.int64)
    for b in range(B):
        for h in range(Hq):
            if where == "first":
                c = (i * 7 + h + b) % np.minimum(128, vis)
            elif where == "last":
                c = vis - 1 - (i + h + b) % np.minimum(vis, 5)
            else:   # the last visible 64-key block
                c = 64 * ((vis - 1) // 64) + (i * 3 + h + b) % ((vis - 1) % 64 + 1)
            chosen[b, h] = c
    dig = lambda j: np.stack([(j // base ** m) % base for m in range(ndig)], axis=-1)  # noqa: E731
    j = np.arange(Sk)
    dk = dig(j)
    k = np.zeros((B, Hkv, Sk, D))
    k[..., 0:ndig] = dk
    k[..., ndig:2 * ndig] = dk ** 2
    k[..., Sk - 1, 2 * ndig] = 1.0
    k[..., 2 * ndig + 1:2 * ndig + 3] = 1.0
    dc = dig(chosen)
    bb, hh, ii = np.meshgrid(np.arange(B), np.arange(Hq), i, indexing="ij")
    r = 1 + (ii * 5 + hh * 3 + bb) % 60
    n = G_STEP * (dc ** 2).sum(axis=-1) + r
    q = np.zeros((B, Hq, Sq, D))
    q[..., 0:ndig] = 2 * G_STEP * dc
    q[..., ndig:2 * ndig] = -G_STEP
    if causal:
        q[..., 2 * ndig] = np.where(i < Sk - 1, DECOY, 0.0)
    q[..., 2 * ndig + 1] = -(n & ~0xFF)
    q[..., 2 * ndig + 2] = -(n & 0xFF)
    b4, hk, jj, dd = np.meshgrid(np.arange(B), np.arange(Hkv), j, np.arange(D), indexing="ij")
    v = ((jj * 7 + dd * 3 + hk * 5 + b4) % 257 - 128).astype(np.float64)
    b4, h4, i4, d4 = np.meshgrid(np.arange(B), np.arange(Hq), i, np.arange(D), indexing="ij")
    dout = ((i4 * 3 + d4 * 5 + h4 * 7 + b4) % 9 - 4).astype(np.float64)
    return q, k, v, dout, chosen


@pytest.mark.parametrize("dtype", ["bf16", "f16"])
@pytest.mark.parametrize("D,Sq,Sk,Hq,Hkv,causal", [
    (8, 150, 190, 4, 2, False), (8, 100, 64, 2, 1, True), (40, 300, 200, 2, 1, True), (64, 129, 129, 2, 2, True),
    (72, 100, 390, 6, 3, False), (128, 257, 257, 2, 1, True), (128, 60, 300, 4, 2, True),
])
@pytest.mark.parametrize("where", ["first", "last", "diag"])
def test_one_hot_rows_exact(client, dtype, D, Sq, Sk, Hq, Hkv, causal, where):
    B = 2
    q, k, v, dout, chosen = one_hot_problem(B, Hq, Hkv, Sq, Sk, D, causal, where)
    g = Hq // Hkv
    want = np.zeros((B, Hkv, Sk, D))
    for b in range(B):
        for h in range(Hq):
            np.add.at(want[b, h // g], chosen[b, h], dout[b, h])
    for out_dtype, grad_dtype in ((dtype, dtype), ("f32", "f32"), (dtype, "f32")):
        dq, dk, dv = run(client, q, k, v, dout, dtype, out_dtype, grad_dtype, scale=LN2, causal=causal)
        np.testing.assert_array_equal(dq, 0.0)
        np.testing.assert_array_equal(dk, 0.0)
        np.testing.assert_array_equal(dv, rounded(want, grad_dtype))


# ---------------------------------------------------------------------------------------------- exact: uniform rows
@pytest.mark.parametrize("dtype", ["bf16", "f16"])
@pytest.mark.parametrize("D,Sk,Hq,Hkv", [(64, 256, 2, 2), (128, 512, 4, 2), (40, 128, 3, 1), (96, 1024, 2, 2)])
def test_uniform_rows_give_the_exact_mean_gradient(client, dtype, D, Sk, Hq, Hkv):
    B, Sq = 2, 333
    rng = np.random.default_rng(D + Sk)
    q = np.zeros((B, Hq, Sq, D))
    k = rng.integers(-8, 9, (B, Hkv, Sk, D)).astype(np.float64)
    v = rng.integers(-8, 9, (B, Hkv, Sk, D)).astype(np.float64)
    dout = rng.integers(-4, 5, (B, Hq, Sq, D)).astype(np.float64)
    s = dout.reshape(B, Hkv, Hq // Hkv, Sq, D).sum(axis=(2, 3)) / Sk
    want = np.broadcast_to(s[:, :, None, :], (B, Hkv, Sk, D))
    for grad_dtype in (dtype, "f32"):
        _, _, dv = run(client, q, k, v, dout, dtype, dtype, grad_dtype, scale=0.3)
        np.testing.assert_array_equal(dv, rounded(want, grad_dtype))


# ---------------------------------------------------------------------------------------------- random data
def bounds(q, k, v, dout, dtype, out_dtype, grad_dtype, scale, causal):
    """(dq, dk, dv) of the f64 oracle and elementwise error bounds derived from where the kernels round:
    - the forward's out carries at most 2 u max|v| (its P rounding) plus its output rounding u_out |out|, so delta carries
      sum_d |dout| (2 u max|v| + u_out |out|); f32 sums of n terms add n 2^-24 of their absolute sums (dP: n = D);
    - p carries the lse round trip and ex2.approx: eps_p = 2^-16 relative;
    - dS (and P for dV) rounded to the input dtype: u relative;
    - dq, dk and dv are f32 sums over n = Sk, G * Sq terms, then rounded once to the grad dtype: u_grad |ref|.
    The bound is twice the sum of these first-order terms (second-order terms and slack)."""
    u, uo, ug, eps_p = U[dtype], U[out_dtype], U[grad_dtype], 2.0 ** -16
    B, Hq, Sq, D = q.shape
    Hkv, Sk = k.shape[1], k.shape[2]
    g = Hq // Hkv
    out, lse = ao.attention_f64(q, k, v, scale, causal)
    kk, vv = np.repeat(k, g, axis=1), np.repeat(v, g, axis=1)
    s = scale * ein("bhid,bhjd->bhij", q, kk)
    if causal:
        s = np.where(np.arange(Sk)[None, :] <= np.arange(Sq)[:, None], s, -np.inf)
    p = np.exp(s - lse[..., None])
    dp = ein("bhid,bhjd->bhij", dout, vv)
    delta = ein("bhid,bhid->bhi", dout, out)
    ds = p * (dp - delta[..., None])
    dq = scale * ein("bhij,bhjd->bhid", ds, kk)
    dk = scale * ein("bhij,bhid->bhjd", ds, q).reshape(B, Hkv, g, Sk, D).sum(axis=2)
    dv = ein("bhij,bhid->bhjd", p, dout).reshape(B, Hkv, g, Sk, D).sum(axis=2)
    ad = np.abs(dout)
    delta_err = ein("bhid,bhid->bhi", ad, 2 * u * np.abs(v).max() + uo * np.abs(out) + D * 2.0 ** -24 * np.abs(out))
    dp_err = D * 2.0 ** -24 * ein("bhid,bhjd->bhij", ad, np.abs(vv))
    e_ds = (u + eps_p) * np.abs(ds) + p * (dp_err + delta_err[..., None])
    nq, nk = Sk * 2.0 ** -24, g * Sq * 2.0 ** -24
    b_dq = scale * ein("bhij,bhjd->bhid", e_ds + nq * np.abs(ds), np.abs(kk)) + ug * np.abs(dq)
    b_dk = scale * ein("bhij,bhid->bhjd", e_ds + nk * np.abs(ds), np.abs(q)).reshape(B, Hkv, g, Sk, D).sum(axis=2) \
        + ug * np.abs(dk)
    b_dv = (u + eps_p + nk) * ein("bhij,bhid->bhjd", p, ad).reshape(B, Hkv, g, Sk, D).sum(axis=2) + ug * np.abs(dv)
    return (dq, dk, dv), tuple(2 * b + 1e-7 for b in (b_dq, b_dk, b_dv))


@pytest.mark.parametrize("dtype", ["bf16", "f16"])
@pytest.mark.parametrize("B,Hq,Hkv,Sq,Sk,D,causal", [
    (2, 4, 4, 333, 333, 64, False), (1, 8, 2, 300, 513, 128, True), (2, 4, 1, 517, 200, 128, False), (1, 2, 2, 1, 700, 64, False),
    (1, 3, 3, 250, 250, 40, True), (1, 2, 1, 600, 600, 96, True), (1, 4, 2, 77, 130, 40, False),
])
def test_random_against_the_oracle(client, dtype, B, Hq, Hkv, Sq, Sk, D, causal):
    rng = np.random.default_rng(Sq + Sk + D)
    q, k, v, dout = (rounded(rng.uniform(-2, 2, s), dtype) for s in ((B, Hq, Sq, D), (B, Hkv, Sk, D), (B, Hkv, Sk, D), (B, Hq, Sq, D)))
    scale = 1 / math.sqrt(D)
    for out_dtype, grad_dtype in ((dtype, dtype), ("f32", "f32")):
        refs, bnds = bounds(q, k, v, dout, dtype, out_dtype, grad_dtype, scale, causal)
        got = run(client, q, k, v, dout, dtype, out_dtype, grad_dtype, causal=causal)
        for name, x, ref, bnd in zip(("dq", "dk", "dv"), got, refs, bnds):
            err = np.abs(x - ref) - bnd
            assert err.max() <= 0, (name, out_dtype, grad_dtype, float(err.max()))


@pytest.mark.parametrize("causal", [False, True])
def test_matches_torch_backward_on_the_gpu(client, causal):
    B, H, S, D = 1, 8, 2048, 128
    gen = torch.Generator(device="cuda").manual_seed(11)
    qt, kt, vt, dot = (torch.rand((B, H, S, D), device="cuda", generator=gen, dtype=torch.float32).mul_(4).sub_(2).to(torch.bfloat16)
                       for _ in range(4))
    qr, kr, vr = (t.clone().requires_grad_() for t in (qt, kt, vt))
    o = torch.nn.functional.scaled_dot_product_attention(qr, kr, vr, is_causal=causal)
    ref_t = [t.float().cpu().numpy().astype(np.float64) for t in torch.autograd.grad(o, (qr, kr, vr), dot)]
    q, k, v, dout = (t.float().cpu().numpy().astype(np.float64) for t in (qt, kt, vt, dot))
    got = run(client, q, k, v, dout, "bf16", "bf16", "bf16", causal=causal)
    _, bnds = bounds(q, k, v, dout, "bf16", "bf16", "bf16", 1 / math.sqrt(D), causal)
    # both round P and dS to bf16 and the outputs to bf16: the difference is within the sum of the two bounds
    for name, x, r, bnd in zip(("dq", "dk", "dv"), got, ref_t, bnds):
        assert (np.abs(x - r) - 2 * bnd).max() <= 0, name


# ---------------------------------------------------------------------------------------------- views, streams, errors
def test_two_streams_and_repeats_give_the_same_bits(client):
    B, Hq, Hkv, S, D = 2, 4, 2, 700, 128
    rng = np.random.default_rng(5)
    q, do = (up(client, rng.uniform(-2, 2, (B, Hq, S, D)), "f16") for _ in range(2))
    k, v = (up(client, rng.uniform(-2, 2, (B, Hkv, S, D)), "f16") for _ in range(2))
    out, lse = forward(client, q, k, v, "f16", None, True)
    client.sync()
    streams = [client.create_stream(), client.create_stream()]
    grads = [[attention.launch_backward_alloc(client, q, k, v, out, do, lse, causal=True, grad_dtype="f32", stream=st) for _ in range(3)]
             for st in streams]
    try:
        for st in streams:
            client.sync_stream(st)
        client.sync()
        ref = [bits(client, t) for t in grads[0][0]]
        for row in grads:
            for gs in row:
                for t, r in zip(gs, ref):
                    assert np.array_equal(bits(client, t), r)
    finally:
        for st in streams:
            client.destroy_stream(st)


def test_views_give_identical_bits(client):
    B, H, S, D = 2, 4, 300, 64
    rng = np.random.default_rng(3)
    qkv = rounded(rng.uniform(-2, 2, (B, S, 3, H, D)), "bf16")
    dout_bshd = rounded(rng.uniform(-2, 2, (B, S, H, D)), "bf16")
    fused = up(client, qkv, "bf16")
    st5 = [S * 3 * H * D, D, 3 * H * D, 1]
    bshd_st = [S * H * D, D, H * D, 1]
    sl = [TensorHandle(fused.handle.offset(i * H * D * 2), [B, H, S, D], st5, "bf16") for i in range(3)]
    compact = [up(client, np.ascontiguousarray(qkv[:, :, i].transpose(0, 2, 1, 3)), "bf16") for i in range(3)]
    bshd = []
    for i in range(3):
        t = up(client, np.ascontiguousarray(qkv[:, :, i]), "bf16")   # [B, S, H, D] as a [B, H, S, D] view
        bshd.append(TensorHandle(t.handle, [B, H, S, D], bshd_st, "bf16"))
    # a misaligned k: one element into a buffer, so the base is not 16-byte aligned and the operand is gathered
    kbuf = up(client, np.concatenate([[0.0], qkv[:, :, 1].transpose(0, 2, 1, 3).reshape(-1)]), "bf16")
    mis = [compact[0], TensorHandle(kbuf.handle.offset(2), [B, H, S, D], compact[1].strides, "bf16"), compact[2]]
    do_c = up(client, np.ascontiguousarray(dout_bshd.transpose(0, 2, 1, 3)), "bf16")
    do_b = TensorHandle(up(client, dout_bshd, "bf16").handle, [B, H, S, D], bshd_st, "bf16")
    out, lse = forward(client, *compact, "bf16", None, True)
    client.sync()
    res = []
    for ops, do in ((compact, do_c), (sl, do_c), (bshd, do_b), (mis, do_c)):
        res.append(attention.launch_backward_alloc(client, *ops, out, do, lse, causal=True))
    client.sync()
    ref = [bits(client, t) for t in res[0]]
    assert any(r.any() for r in ref)
    for gs in res[1:]:
        for t, r in zip(gs, ref):
            assert np.array_equal(bits(client, t), r)
    # dq, dk and dv as the slices of one fused [B, S, 3, H, D] gradient buffer
    gbuf = TensorHandle.empty_contiguous(client, [B, S, 3, H, D], "bf16")
    gsl = [TensorHandle(gbuf.handle.offset(i * H * D * 2), [B, H, S, D], st5, "bf16") for i in range(3)]
    attention.launch_backward(client, *compact, out, do_c, lse, *gsl, causal=True)
    client.sync()
    g = bits(client, gbuf).reshape(B, S, 3, H, D)
    for i in range(3):
        assert np.array_equal(g[:, :, i].transpose(0, 2, 1, 3), ref[i].reshape(B, H, S, D))


def test_errors_are_deferred_to_sync(client):
    q = up(client, np.zeros((1, 4, 8, 64)), "bf16")
    k = up(client, np.zeros((1, 3, 8, 64)), "bf16")
    lse = TensorHandle.empty_contiguous(client, [1, 4, 8], "f32")
    attention.launch_backward_alloc(client, q, k, k, q, q, lse)   # Hq = 4 is not a multiple of Hkv = 3: no raise here
    with pytest.raises(ServerError, match="multiple of Hkv"):
        client.sync()
    g = [TensorHandle.empty_contiguous(client, [1, 4, 8, 64], "f16") for _ in range(3)]
    attention.launch_backward(client, q, q, q, q, q, lse, *g)
    with pytest.raises(ServerError, match="grad dtype"):
        client.sync()
