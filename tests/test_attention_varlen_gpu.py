"""GPU: b200_attention_varlen and b200_attention_varlen_backward on an H100.

- Bitwise equal to the dense kernels: with Lq == Lk and window (-1, -1) or (-1, 0), every sequence's out, lse, dq, dk and dv
  equal a dense b200_attention / b200_attention_backward call on that sequence alone (the only difference is addressing).
- Random data against the f64 oracle: Lq != Lk (bottom-right, rows that see nothing), windows (W, 0), (W, W) and (0, W), and an
  empty sequence between non-empty ones.
- Against torch's varlen attention (or, where it refuses the call, torch's SDPA per sequence with an explicit mask) on the GPU.
- Sequences are independent: NaN in one sequence's rows and outside every sequence changes no bit of the others, and rows
  outside every sequence of out, lse, dq, dk and dv keep their sentinel bytes.
- Reproducible across repeats and two streams.
- Views read in place (fused-QKV slices, pitched outputs and gradients) or gathered (a misaligned q) give the bits of compact
  operands."""

import numpy as np
import pytest
import torch

import attention_varlen_oracle as vo
from cubecl_b200 import TensorHandle, attention, synth

pytestmark = pytest.mark.gpu

U = {"bf16": 2.0 ** -8, "f16": 2.0 ** -11, "f32": 0.0}


def up(client, vals, dtype):
    if dtype == "i32":
        return TensorHandle.from_numpy(client, np.ascontiguousarray(vals, np.int32), "i32")
    return TensorHandle.from_numpy(client, synth.to_device_dtype(np.ascontiguousarray(vals, np.float32), dtype), dtype)


def values(client, t):
    return synth.from_device_dtype(t.to_numpy(client), t.dtype).astype(np.float64).reshape(t.shape)


def bits(client, t):
    return np.asarray(t.to_numpy(client)).view(np.uint32 if t.dtype == "f32" else np.uint16).reshape(t.shape)


def cu(lens, start=0):
    return np.concatenate([[start], start + np.cumsum(lens)]).astype(np.int32)


def varlen(client, q, k, v, dout, cuq, cuk, maxq, maxk, dtype, odt, gdt, window, scale=None, sentinel=None):
    """forward and backward; with `sentinel`, every output buffer starts filled with that byte pattern"""
    qh, kh, vh, doh = (up(client, t, dtype) for t in (q, k, v, dout))
    cq, ck = up(client, cuq, "i32"), up(client, cuk, "i32")

    def buf(shape, dt):
        if sentinel is None:
            return TensorHandle.empty_contiguous(client, shape, dt)
        raw = np.full(int(np.prod(shape)), sentinel[dt], dtype=np.uint32 if dt == "f32" else np.uint16).reshape(shape)
        return TensorHandle.from_numpy(client, raw, dt)

    out, lse = buf(list(q.shape), odt), buf([q.shape[1], q.shape[0]], "f32")
    attention.launch_varlen(client, qh, kh, vh, cq, ck, maxq, maxk, out, scale=scale, window_size=window, lse=lse)
    dq, dk, dv = buf(list(q.shape), gdt), buf(list(k.shape), gdt), buf(list(k.shape), gdt)
    attention.launch_varlen_backward(client, qh, kh, vh, out, doh, lse, cq, ck, maxq, maxk, dq, dk, dv, scale=scale, window_size=window)
    client.sync()
    return out, lse, dq, dk, dv


def problem(rng, lens_q, lens_k, Hq, Hkv, D, pad=(0, 0)):
    Tq, Tk = sum(lens_q) + sum(pad), sum(lens_k) + sum(pad)
    q, k, v = rng.standard_normal((Tq, Hq, D)), rng.standard_normal((Tk, Hkv, D)), rng.standard_normal((Tk, Hkv, D))
    return q, k, v, rng.standard_normal((Tq, Hq, D)), cu(lens_q, pad[0]), cu(lens_k, pad[0])


# ---------------------------------------------------------------------------------------------- bitwise against dense
LENS = [1, 63, 64, 127, 128, 129, 1000, 0]


@pytest.mark.parametrize("dtype", ["bf16", "f16"])
@pytest.mark.parametrize("D", [40, 64, 96, 128])
@pytest.mark.parametrize("window", [(-1, -1), (-1, 0)])
@pytest.mark.parametrize("f32", [False, True])
def test_each_sequence_equals_a_dense_call_bit_for_bit(client, dtype, D, window, f32):
    rng = np.random.default_rng(D + 7 * (window[1] + 2) + 31 * f32)
    Hq, Hkv = 4, 2
    q, k, v, dout, cuq, cuk = problem(rng, LENS, LENS, Hq, Hkv, D)
    odt = gdt = "f32" if f32 else dtype
    out, lse, dq, dk, dv = varlen(client, q, k, v, dout, cuq, cuk, max(LENS), max(LENS), dtype, odt, gdt, window)
    ob, lb, dqb, dkb, dvb = (bits(client, t) for t in (out, lse, dq, dk, dv))
    causal = window == (-1, 0)
    for b, L in enumerate(LENS):
        if L == 0:
            continue
        a, z = cuq[b], cuq[b + 1]
        per = lambda t: up(client, np.ascontiguousarray(t[a:z].transpose(1, 0, 2))[None], dtype)  # noqa: E731
        qh, kh, vh, doh = per(q), per(k), per(v), per(dout)
        dout_, dlse = attention.launch_alloc(client, qh, kh, vh, causal=causal, out_dtype=odt, return_lse=True)
        ddq, ddk, ddv = attention.launch_backward_alloc(client, qh, kh, vh, dout_, doh, dlse, causal=causal, grad_dtype=gdt)
        client.sync()
        back = lambda t: bits(client, t)[0].transpose(1, 0, 2)  # noqa: E731
        np.testing.assert_array_equal(ob[a:z], back(dout_), err_msg=f"out of sequence {b} (L = {L})")
        np.testing.assert_array_equal(lb[:, a:z], bits(client, dlse)[0], err_msg=f"lse of sequence {b}")
        np.testing.assert_array_equal(dqb[a:z], back(ddq), err_msg=f"dq of sequence {b}")
        np.testing.assert_array_equal(dkb[a:z], back(ddk), err_msg=f"dk of sequence {b}")
        np.testing.assert_array_equal(dvb[a:z], back(ddv), err_msg=f"dv of sequence {b}")


# ---------------------------------------------------------------------------------------------- against the oracle
def _close(got, want, dtype, what, k=4.0):
    """|got - want| <= k * (u_in + u_out) * max|want| + small: the inputs are rounded once, every output once"""
    scale = max(1.0, float(np.abs(want).max()))
    err = float(np.abs(got - want).max())
    assert err <= k * (U[dtype] + 2 ** -8) * scale, (what, err, scale)


@pytest.mark.parametrize("lens_q,lens_k,window", [
    ([300, 0, 129, 77], [200, 0, 400, 77], (-1, 0)),      # Lq > Lk: rows that see nothing; an empty sequence between
    ([500, 260], [500, 700], (-1, 0)),                     # chunked prefill against its own prefix
    ([700, 333], [700, 333], (100, 0)), ([700, 333], [700, 400], (64, 64)), ([700, 333], [700, 333], (0, 96)),
    ([257, 1, 64], [300, 5, 1], (-1, -1)),
])
@pytest.mark.parametrize("dtype", ["bf16", "f16"])
def test_random_data_against_the_oracle(client, lens_q, lens_k, window, dtype):
    rng = np.random.default_rng(sum(lens_q) + sum(lens_k) + window[0])
    Hq, Hkv, D = 4, 1, 64
    q, k, v, dout, cuq, cuk = problem(rng, lens_q, lens_k, Hq, Hkv, D)
    rq, rk, rv, rdo = (values(client, up(client, t, dtype)) for t in (q, k, v, dout))
    out, lse, dq, dk, dv = varlen(client, q, k, v, dout, cuq, cuk, max(lens_q), max(lens_k), dtype, "f32", "f32", window)
    ref_out, ref_lse = vo.attention_varlen_f64(rq, rk, rv, cuq, cuk, None, window)
    got_lse = values(client, lse)
    np.testing.assert_array_equal(np.isneginf(got_lse), np.isneginf(ref_lse))
    fin = np.isfinite(ref_lse)
    np.testing.assert_allclose(got_lse[fin], ref_lse[fin], rtol=0, atol=1e-3)
    got_out = values(client, out)
    assert np.all(got_out[np.isneginf(ref_lse).T] == 0)   # rows without keys: +0
    _close(got_out, ref_out, dtype, "out")
    rdq, rdk, rdv = vo.attention_varlen_backward_f64(rq, rk, rv, rdo, cuq, cuk, None, window)
    for name, g, r in (("dq", dq, rdq), ("dk", dk, rdk), ("dv", dv, rdv)):
        _close(values(client, g), r, dtype, name, k=16.0)
    assert np.all(values(client, dq)[np.isneginf(ref_lse).T] == 0)


# ---------------------------------------------------------------------------------------------- against torch
def test_against_torch_varlen_attention(client):
    lens = [1000, 37, 512, 2048, 129]
    Hq, Hkv, D, dtype = 8, 2, 128, "bf16"
    rng = np.random.default_rng(5)
    q, k, v, dout, cuq, cuk = problem(rng, lens, lens, Hq, Hkv, D)
    out, lse, dq, dk, dv = varlen(client, q, k, v, dout, cuq, cuk, max(lens), max(lens), dtype, dtype, dtype, (-1, 0))
    dev = torch.device("cuda")
    qt, kt, vt, dot = (torch.tensor(t, dtype=torch.bfloat16, device=dev) for t in (q, k, v, dout))
    kt, vt = (t.repeat_interleave(Hq // Hkv, dim=1) for t in (kt, vt))   # torch's varlen path takes equal head counts
    for t in (qt, kt, vt):
        t.requires_grad_(True)
    cq = torch.tensor(cuq, dtype=torch.int32, device=dev)
    try:
        from torch.nn.attention.varlen import varlen_attn
        ref = varlen_attn(qt, kt, vt, cq, cq, max(lens), max(lens), window_size=(-1, 0))
        backend = "varlen_attn"
    except (RuntimeError, NotImplementedError):   # a torch build without the varlen kernel: SDPA per sequence, explicit mask
        pieces = []
        for b, L in enumerate(lens):
            a, z = cuq[b], cuq[b + 1]
            mask = torch.ones(L, L, dtype=torch.bool, device=dev).tril()
            pieces.append(torch.nn.functional.scaled_dot_product_attention(
                *(t[a:z].transpose(0, 1)[None] for t in (qt, kt, vt)), attn_mask=mask)[0].transpose(0, 1))
        ref = torch.cat(pieces)
        backend = "scaled_dot_product_attention"
    ref.backward(dot)
    gk = kt.grad.view(-1, Hkv, Hq // Hkv, D).sum(2)
    gv = vt.grad.view(-1, Hkv, Hq // Hkv, D).sum(2)
    for name, got, want in (("out", out, ref), ("dq", dq, qt.grad), ("dk", dk, gk), ("dv", dv, gv)):
        w = want.detach().float().cpu().numpy().astype(np.float64)
        err = float(np.abs(values(client, got) - w).max())
        assert err <= 0.05 * max(1.0, float(np.abs(w).max())), (backend, name, err)


# ---------------------------------------------------------------------------------------------- independence
SENT = {"bf16": 0x7FA1, "f16": 0x7E01, "f32": 0x7FC0_1234}


def test_nan_in_one_sequence_and_outside_changes_no_other_bit(client):
    rng = np.random.default_rng(11)
    lens_q, lens_k = [200, 129, 64, 300], [250, 129, 130, 300]
    pad = (3, 70)
    q, k, v, dout, cuq, cuk = problem(rng, lens_q, lens_k, 4, 2, 64, pad=pad)
    clean = [bits(client, t) for t in varlen(client, q, k, v, dout, cuq, cuk, 300, 300, "bf16", "bf16", "bf16", (-1, 0))]
    poisoned = []
    for t, c in ((q, cuq), (k, cuk), (v, cuk), (dout, cuq)):
        t = t.copy()
        t[c[1]:c[2]] = np.nan              # sequence 1
        t[:c[0]] = np.inf                  # rows before the first sequence
        t[c[-1]:] = np.nan                 # rows past cu[B]
        poisoned.append(t)
    dirty = [bits(client, t) for t in varlen(client, *poisoned, cuq, cuk, 300, 300, "bf16", "bf16", "bf16", (-1, 0))]
    for b in (0, 2, 3):
        (qa, qb), (ka, kb) = (cuq[b], cuq[b + 1]), (cuk[b], cuk[b + 1])
        for i, (c, d) in enumerate(zip(clean, dirty)):
            if i == 1:
                np.testing.assert_array_equal(c[:, qa:qb], d[:, qa:qb], err_msg=f"lse of sequence {b}")
            elif i < 3:
                np.testing.assert_array_equal(c[qa:qb], d[qa:qb], err_msg=f"output {i} of sequence {b}")
            else:
                np.testing.assert_array_equal(c[ka:kb], d[ka:kb], err_msg=f"output {i} of sequence {b}")


@pytest.mark.parametrize("f32", [False, True])
def test_rows_outside_every_sequence_keep_their_sentinels(client, f32):
    rng = np.random.default_rng(12)
    lens_q, lens_k = [100, 0, 190], [130, 7, 65]
    pad = (5, 77)
    q, k, v, dout, cuq, cuk = problem(rng, lens_q, lens_k, 4, 4, 96, pad=pad)
    dt = "f32" if f32 else "f16"
    res = varlen(client, q, k, v, dout, cuq, cuk, 190, 130, "f16", dt, dt, (50, 0), sentinel=SENT)
    out, lse, dq, dk, dv = (bits(client, t) for t in res)
    for name, arr, c, axis in (("out", out, cuq, 0), ("lse", lse, cuq, 1), ("dq", dq, cuq, 0), ("dk", dk, cuk, 0), ("dv", dv, cuk, 0)):
        s = SENT["f32" if name == "lse" else dt]
        a = np.moveaxis(arr, axis, 0)
        assert np.all(a[:c[0]] == s) and np.all(a[c[-1]:] == s), name
        assert not np.any(a[c[0]:c[-1]] == s), name   # every owned row was written


def test_repeats_and_two_streams_give_the_same_bits(client):
    rng = np.random.default_rng(13)
    lens = [333, 1000, 64, 5]
    q, k, v, dout, cuq, cuk = problem(rng, lens, lens, 8, 2, 128)
    ref = [bits(client, t) for t in varlen(client, q, k, v, dout, cuq, cuk, 1000, 1000, "bf16", "bf16", "bf16", (256, 0))]
    qh, kh, vh, doh = (up(client, t, "bf16") for t in (q, k, v, dout))
    cq, ck = up(client, cuq, "i32"), up(client, cuk, "i32")
    streams = [client.create_stream(), client.create_stream()]
    try:
        results = []
        for _ in range(2):
            for st in streams:
                out, lse = attention.launch_varlen_alloc(client, qh, kh, vh, cq, ck, 1000, 1000, window_size=(256, 0), return_lse=True,
                                                         stream=st)
                g = attention.launch_varlen_backward_alloc(client, qh, kh, vh, out, doh, lse, cq, ck, 1000, 1000, window_size=(256, 0),
                                                           stream=st)
                results.append((out, lse) + tuple(g))
        for st in streams:
            client.sync_stream(st)
        client.sync()
        for r in results:
            for want, got in zip(ref, r):
                np.testing.assert_array_equal(want, bits(client, got))
    finally:
        for st in streams:
            client.destroy_stream(st)


@pytest.mark.parametrize("f32", [False, True])
def test_views_give_identical_bits(client, f32):
    """q, k and v as slices of one [T, 3, H, D] projection with pitched out, dout, dq, dk and dv, and a misaligned q (gathered),
    give the bits of compact operands, forward and backward"""
    rng = np.random.default_rng(14)
    lens = [100, 0, 190, 7]
    T, H, D, P = sum(lens), 4, 64, 72
    cuq = cu(lens)
    qkv, dout = rng.standard_normal((T, 3, H, D)), rng.standard_normal((T, H, D))
    dt = "f32" if f32 else "bf16"
    ref = [bits(client, t) for t in varlen(client, qkv[:, 0], qkv[:, 1], qkv[:, 2], dout, cuq, cuq, 190, 190, "bf16", dt, dt, (-1, 0))]
    cq = up(client, cuq, "i32")

    def pitched(dtype, vals=None):   # [T, H, D] rows of P elements per head: a view, and the buffer behind it
        buf = up(client, np.pad(vals, ((0, 0), (0, 0), (0, P - D))), dtype) if vals is not None else \
            TensorHandle.empty_contiguous(client, [T, H, P], dtype)
        return TensorHandle(buf.handle, [T, H, D], [H * P, P, 1], dtype), buf

    fused = up(client, qkv, "bf16")
    q, k, v = (TensorHandle(fused.handle.offset(i * H * D * 2), [T, H, D], [3 * H * D, D, 1], "bf16") for i in range(3))
    (out, ob), (do, _), (dq, dqb), (dk, dkb), (dv, dvb) = (pitched(dt), pitched("bf16", dout), pitched(dt), pitched(dt), pitched(dt))
    lse = TensorHandle.empty_contiguous(client, [H, T], "f32")
    attention.launch_varlen(client, q, k, v, cq, cq, 190, 190, out, window_size=(-1, 0), lse=lse)
    attention.launch_varlen_backward(client, q, k, v, out, do, lse, cq, cq, 190, 190, dq, dk, dv, window_size=(-1, 0))
    client.sync()
    for name, want, got in zip(("out", "lse", "dq", "dk", "dv"), ref, (ob, lse, dqb, dkb, dvb)):
        g = bits(client, got)
        np.testing.assert_array_equal(g[..., :D] if name != "lse" else g, want, err_msg=name)
    # a q one element into its buffer: the base is not 16-byte aligned, so both calls read a gathered copy
    qbuf = up(client, np.concatenate([[0.0], qkv[:, 0].reshape(-1)]), "bf16")
    qm = TensorHandle(qbuf.handle.offset(2), [T, H, D], [H * D, D, 1], "bf16")
    kc, vc, doc = (up(client, t, "bf16") for t in (qkv[:, 1], qkv[:, 2], dout))
    out, lse = attention.launch_varlen_alloc(client, qm, kc, vc, cq, cq, 190, 190, window_size=(-1, 0), out_dtype=dt, return_lse=True)
    grads = attention.launch_varlen_backward_alloc(client, qm, kc, vc, out, doc, lse, cq, cq, 190, 190, window_size=(-1, 0), grad_dtype=dt)
    client.sync()
    for name, want, got in zip(("out", "lse", "dq", "dk", "dv"), ref, (out, lse) + tuple(grads)):
        np.testing.assert_array_equal(bits(client, got), want, err_msg=f"misaligned q: {name}")
