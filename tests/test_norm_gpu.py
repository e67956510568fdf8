"""GPU: b200_norm, b200_norm_quantized_fp8 and b200_norm_backward against tests/norm_oracle.py -- bit for bit on exact rows
(every sum exact in any order, rstd a power of two) for every dtype cell, kind and optional operand at n from 1 to 32768;
random rows within the oracle's bound of an f64 reference and within bf16 tolerance of torch; dweight and dbias bit for bit
when each backward unit sums several rows; rows past the forward's grid cap; batch invariance of a planted
row across positions, batch sizes and the 128-bit / element-wise paths; the fused residual against the unfused call; the
fp8 output against b200_quantize and through b200_matmul_quantized_fp8; sentinels, repeats and pooled temporaries."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import norm_oracle as no
from cubecl_b200 import TensorHandle, matmul, norm, quant, synth
from cubecl_b200.quant import QuantScheme

pytestmark = pytest.mark.gpu

NP16 = {"bf16": np.uint16, "f16": np.uint16, "f32": np.uint32}


def up(c, arr, dtype):
    return TensorHandle.from_numpy(c, synth.to_device_dtype(np.asarray(arr, np.float32), dtype), dtype)


def down(c, t):
    return synth.from_device_dtype(t.to_numpy(c), t.dtype)


def bits(c, t):
    """the raw element bits of a device tensor (exact comparison, NaN and -0 included)"""
    return t.to_numpy(c).view(NP16[t.dtype])


def hbits(a, dtype):
    return synth.to_device_dtype(np.asarray(a, np.float32), dtype).view(NP16[dtype])


def pitched(c, arr, dtype, pad=3, lead=1, fill=0.0):
    """arr [T, n] in a wider buffer [T, n + pad] starting `lead` elements in: a misaligned, pitched view (element-wise path)"""
    T, n = arr.shape
    buf = np.full((T * (n + pad) + lead,), fill, np.float32)
    buf[lead:].reshape(T, n + pad)[:, :n] = arr
    h = up(c, buf, dtype)
    esz = 2 if dtype != "f32" else 4
    return TensorHandle(h.handle.offset(lead * esz), [T, n], [n + pad, 1], dtype)


# ---------------------------------------------------------------------------------------------- exact rows
NS = [1, 7, 128, 1000, 4096, 7168, 16384, 32768]
CELLS = [("f32", "f32", "f32", "f32"), ("bf16", "f32", "bf16", "bf16"), ("bf16", "bf16", "f32", "f32"),
         ("f16", "f16", "f16", "f16"), ("f16", "f32", "bf16", "f32"), ("f32", "f32", "f16", "bf16")]
OPTS = [dict(residual=False, weight=False, bias=False, d_h=False), dict(residual=True, weight=True, bias=True, d_h=True),
        dict(residual=False, weight=True, bias=False, d_h=True), dict(residual=True, weight=False, bias=True, d_h=False)]


def exact_case(kind, n, xdt, T, seed):
    rng = np.random.default_rng(seed)
    h = no.exact_rms_rows(rng, T, n) if kind == "rms" else no.exact_layer_rows(rng, T, n, xdt)
    eps = 1.0 if (kind == "layer" and n == 1) else 0.0
    return rng, h, eps


def exact_residual(rng, h, xdt):
    """(x, residual) with RNE_x(x + residual) = h.  16-bit x: x = h and residual = +-2^(e - m - 3) for h in [2^e, 2^(e+1)) (m
    mantissa bits), below half an ulp of h, so the f32 sum is not h and only its rounding gives h back.  f32 x: x = h - r with
    r in {0, +-1/4}, both exact."""
    if xdt == "f32":
        r = (rng.integers(-1, 2, size=h.shape) * 0.25).astype(np.float32)
        x = (h - r).astype(np.float32)
    else:
        m = {"bf16": 7, "f16": 10}[xdt]
        e = np.floor(np.log2(np.where(h == 0, 1.0, np.abs(h))))
        r = np.where(h == 0, 0.0, np.where(rng.random(h.shape) < 0.5, -1.0, 1.0) * np.exp2(e - m - 3)).astype(np.float32)
        x = h.copy()
        assert np.array_equal(no.rnd(x + r, xdt), h) and not np.array_equal((x + r).astype(np.float32), h)
    assert np.array_equal(no.rnd(x, xdt), x) and np.array_equal(no.rnd(r, xdt), r)
    return x, r


@pytest.mark.parametrize("cell", CELLS, ids=lambda c: "-".join(c))
@pytest.mark.parametrize("kind", ["rms", "layer"])
@pytest.mark.parametrize("n", NS)
def test_exact_rows_match_oracle_bitwise(client, n, kind, cell):
    xdt, wdt, ydt, gdt = cell
    T = 12
    for oi, o in enumerate(OPTS):
        rng, h, eps = exact_case(kind, n, xdt, T, n * 10 + oi)
        w = no.exact_weight(rng, n) if o["weight"] else None
        b = no.exact_weight(rng, n) if (o["bias"] and kind == "layer") else None
        r = None
        x = h
        if o["residual"]:
            x, r = exact_residual(rng, h, xdt)
        dy = no.exact_grad(rng, T, n)
        dh = no.exact_grad(rng, T, n) if o["d_h"] else None
        no.assert_exact(kind, h, eps, w, dy)
        oh, oy, omu, orstd = no.forward(kind, x, eps, w, b, r, xdt)
        assert np.array_equal(oh, h)
        if r is not None and xdt != "f32":     # these rows tell statistics of the rounded h from those of the f32 sum
            _, _, bmu, brstd = no.forward(kind, x, eps, w, b, r, xdt, _mutant="unrounded_residual")
            assert not (np.array_equal(bmu, omu) and np.array_equal(brstd, orstd))
        tx = up(client, x, xdt)
        tr = up(client, r, xdt) if r is not None else None
        tw = up(client, w, wdt) if w is not None else None
        tb = up(client, b, wdt) if b is not None else None
        hh, y, mean, rstd = norm.forward_alloc(client, tx, tw, tb, kind, eps, tr, ydt)
        client.sync()
        np.testing.assert_array_equal(bits(client, y), hbits(no.rnd(oy, ydt), ydt), err_msg=f"y {o}")
        np.testing.assert_array_equal(rstd.to_numpy(client).view(np.uint32), orstd.view(np.uint32))
        if kind == "layer":
            np.testing.assert_array_equal(mean.to_numpy(client).view(np.uint32), omu.view(np.uint32))
        if r is not None:
            np.testing.assert_array_equal(bits(client, hh), hbits(h, xdt))
        odx, odw, odb = no.backward(kind, no.rnd(dy, gdt), h, orstd, w, omu, None if dh is None else no.rnd(dh, gdt), gdt)
        dx, dw, db = norm.backward_alloc(client, up(client, dy, gdt), hh, rstd, tw, mean if kind == "layer" else None, kind,
                                         up(client, dh, gdt) if dh is not None else None, bias=kind == "layer")
        client.sync()
        np.testing.assert_array_equal(bits(client, dx), hbits(odx, gdt), err_msg=f"dx {o}")
        if dw is not None:
            np.testing.assert_array_equal(dw.to_numpy(client).view(np.uint32), odw.view(np.uint32))
        if db is not None:
            np.testing.assert_array_equal(db.to_numpy(client).view(np.uint32), odb.view(np.uint32))


# ---------------------------------------------------------------------------------------------- random rows
@pytest.mark.parametrize("kind", ["rms", "layer"])
@pytest.mark.parametrize("n", [7, 1000, 4096, 7168, 16384, 32768])
def test_random_rows_within_bound_and_match_torch(client, kind, n):
    rng = np.random.default_rng(n)
    T = 64
    x = no.rnd(rng.standard_normal((T, n)).astype(np.float32) * 3 + 0.5, "bf16")
    w = no.rnd(rng.standard_normal(n).astype(np.float32), "bf16")
    b = no.rnd(rng.standard_normal(n).astype(np.float32), "bf16") if kind == "layer" else None
    tw, tb = up(client, w, "bf16"), (up(client, b, "bf16") if b is not None else None)
    _, y, mean, rstd = norm.forward_alloc(client, up(client, x, "bf16"), tw, tb, kind, 1e-5, out_dtype="f32")
    client.sync()
    got = y.to_numpy(client)
    # the contract's own order, bit for bit, and within the derived bound of f64
    _, oy, omu, orstd = no.forward(kind, x, 1e-5, w, b)
    np.testing.assert_array_equal(got.view(np.uint32), oy.view(np.uint32))
    ref, bound = no.reference_f64(kind, x, 1e-5, w, b)
    assert np.all(np.abs(got - ref) <= bound)
    # torch on the GPU in bf16, and autograd for the backward
    xt = torch.tensor(x, dtype=torch.bfloat16, device="cuda", requires_grad=True)
    wt = torch.tensor(w, dtype=torch.bfloat16, device="cuda", requires_grad=True)
    bt = torch.tensor(b, dtype=torch.bfloat16, device="cuda", requires_grad=True) if b is not None else None
    yt = F.rms_norm(xt, (n,), wt, 1e-5) if kind == "rms" else F.layer_norm(xt, (n,), wt, bt, 1e-5)
    torch.testing.assert_close(torch.tensor(got), yt.float().cpu(), atol=6e-2, rtol=1.6e-2)
    dy = no.rnd(rng.standard_normal((T, n)).astype(np.float32), "bf16")
    yt.backward(torch.tensor(dy, dtype=torch.bfloat16, device="cuda"))
    dx, dw, db = norm.backward_alloc(client, up(client, dy, "bf16"), up(client, x, "bf16"), rstd, tw, mean, kind,
                                     bias=kind == "layer")
    client.sync()
    odx, odw, odb = no.backward(kind, dy, x, orstd, w, omu, grad_dtype="bf16")
    np.testing.assert_array_equal(bits(client, dx), hbits(odx, "bf16"))
    np.testing.assert_array_equal(dw.to_numpy(client).view(np.uint32), odw.view(np.uint32))
    torch.testing.assert_close(torch.tensor(down(client, dx)), xt.grad.float().cpu(), atol=6e-2, rtol=3e-2)
    scale = float(np.abs(wt.grad.float().cpu().numpy()).max()) + 1e-3
    assert np.max(np.abs(dw.to_numpy(client) - wt.grad.float().cpu().numpy())) <= 2e-2 * scale
    if b is not None:
        np.testing.assert_allclose(db.to_numpy(client), bt.grad.float().cpu().numpy(), rtol=1e-2, atol=1e-2)   # torch's is bf16


# ---------------------------------------------------------------------------------------------- multi-row backward units
@pytest.mark.parametrize("kind", ["rms", "layer"])
@pytest.mark.parametrize("n,T", [(1000, 3001), (4096, 3001), (16384, 1001)])
def test_multi_row_units_give_dweight_dbias_bitwise(client, kind, n, T):
    """t well above the unit count: each unit sums several rows in shared memory and the last unit is short."""
    units, per = no.units(T, n)
    assert per > 1 and T % per != 0 and units * per > T
    rng = np.random.default_rng(T + n)
    bias = kind == "layer"
    for data in ("exact", "random"):
        if data == "exact":
            h = no.exact_rms_rows(rng, T, n) if kind == "rms" else no.exact_layer_rows(rng, T, n, "bf16")
            w, dy, dh = no.exact_weight(rng, n), no.exact_grad(rng, T, n), no.exact_grad(rng, T, n)
            eps = 0.0
            no.assert_exact(kind, h, eps, w, dy)
        else:
            h = no.rnd(rng.standard_normal((T, n)).astype(np.float32) * 2 + 0.3, "bf16")
            w = no.rnd(rng.standard_normal(n).astype(np.float32), "bf16")
            dy = no.rnd(rng.standard_normal((T, n)).astype(np.float32), "bf16")
            dh = no.rnd(rng.standard_normal((T, n)).astype(np.float32), "bf16")
            eps = 1e-5
        _, _, omu, orstd = no.forward(kind, h, eps, w)
        odx, odw, odb = no.backward(kind, dy, h, orstd, w, omu, dh, "bf16")
        if data == "exact":       # the column sums are exact, so the oracle's equal the f64 ones
            xh = ((h - omu[:, None]) if bias else h).astype(np.float64) * orstd[:, None]
            np.testing.assert_array_equal(odw, (dy.astype(np.float64) * xh).sum(0).astype(np.float32))
            np.testing.assert_array_equal(odb, dy.astype(np.float64).sum(0).astype(np.float32))
        tw, th = up(client, w, "f32"), up(client, h, "bf16")
        _, _, mean, rstd = norm.forward_alloc(client, th, tw, None, kind, eps)
        dx, dw, db = norm.backward_alloc(client, up(client, dy, "bf16"), th, rstd, tw, mean, kind, up(client, dh, "bf16"),
                                         bias=bias)
        client.sync()
        np.testing.assert_array_equal(rstd.to_numpy(client).view(np.uint32), orstd.view(np.uint32))
        np.testing.assert_array_equal(bits(client, dx), hbits(odx, "bf16"), err_msg=data)
        np.testing.assert_array_equal(dw.to_numpy(client).view(np.uint32), odw.view(np.uint32), err_msg=data)
        if bias:
            np.testing.assert_array_equal(db.to_numpy(client).view(np.uint32), odb.view(np.uint32), err_msg=data)


# ---------------------------------------------------------------------------------------------- rows past the grid cap
@pytest.mark.parametrize("n,rows_per_group", [(8, 8), (4104, 1), (8200, 1)])
def test_rows_past_the_grid_cap_are_normalized(client, n, rows_per_group):
    """More row groups than the forward launches CTAs (or clusters) for: the groups loop over the rows past the cap.  Every
    row is x = (1, -2, 1, -2, ...), filled on the device, so every row's y and rstd equal the oracle's one row."""
    t = (1 << 20) * rows_per_group + 1001
    x = TensorHandle.empty_contiguous(client, [t, n], "bf16")
    assert client._lib.b200_memset32(client._ctx, None, C.c_uint64(x.handle.ptr), C.c_uint32(0xC0003F80), C.c_size_t(t * n // 2)) == 0
    w = no.rnd(np.linspace(-1, 1, n).astype(np.float32), "bf16")
    y = TensorHandle.empty_contiguous(client, [t, n], "bf16")
    rstd = TensorHandle.empty_contiguous(client, [t], "f32")
    norm.forward(client, x, y, up(client, w, "bf16"), rstd=rstd)
    client.sync()
    row = np.tile(np.array([1.0, -2.0], np.float32), n // 2)[None, :]
    _, oy, _, orstd = no.forward("rms", row, 1e-6, w)
    np.testing.assert_array_equal(rstd.to_numpy(client).view(np.uint32), np.full(t, orstd.view(np.uint32)[0]))
    for r0 in (0, t // 2, t - 1100):     # the head, the middle and the tail past the cap
        k = 1100 if r0 else 8
        view = TensorHandle(y.handle.offset(r0 * n * 2, k * n * 2), [k, n], [n, 1], "bf16")
        np.testing.assert_array_equal(bits(client, view), np.broadcast_to(hbits(no.rnd(oy, "bf16"), "bf16"), (k, n)))
    del x, y, rstd
    client.memory_cleanup()


# ---------------------------------------------------------------------------------------------- batch invariance
@pytest.mark.parametrize("kind", ["rms", "layer"])
@pytest.mark.parametrize("n,ts", [(1000, (1, 3, 4096, 65537)), (4096, (1, 3, 4096, 65537)), (7168, (1, 3, 4096)),
                                  (32768, (1, 3, 4096))])
def test_planted_row_is_batch_invariant(client, kind, n, ts):
    rng = np.random.default_rng(n + 1)
    row = no.rnd(rng.standard_normal(n).astype(np.float32) * 2 + 0.25, "bf16")
    dyr = no.rnd(rng.standard_normal(n).astype(np.float32), "bf16")
    w = up(client, no.rnd(rng.standard_normal(n).astype(np.float32), "bf16"), "f32")
    seen = None
    for t in ts:
        for pos in sorted({0, t // 2, t - 1}):
            x = np.zeros((t, n), np.float32)
            x[:] = row[::-1]          # other rows differ from the planted one
            x[pos] = row
            dy = np.zeros((t, n), np.float32)
            dy[:] = dyr[::-1]
            dy[pos] = dyr
            for view in ("compact", "pitched") if t <= 4096 else ("compact",):
                mk = (lambda a: up(client, a, "bf16")) if view == "compact" else (lambda a: pitched(client, a, "bf16"))
                tx = mk(x)
                _, y, mean, rstd = norm.forward_alloc(client, tx, w, None, kind, 1e-6)
                dx, dwt, _ = norm.backward_alloc(client, mk(dy), tx, rstd, w, mean, kind)
                client.sync()
                got = (bits(client, y)[pos].copy(), rstd.to_numpy(client)[pos].view(np.uint32).copy(), bits(client, dx)[pos].copy())
                if seen is None:
                    seen = got
                for a, b_ in zip(got, seen):
                    np.testing.assert_array_equal(a, b_, err_msg=f"t={t} pos={pos} {view}")


# ---------------------------------------------------------------------------------------------- fused residual
@pytest.mark.parametrize("kind", ["rms", "layer"])
@pytest.mark.parametrize("n", [1000, 4096, 16384])
def test_fused_residual_equals_unfused(client, kind, n):
    rng = np.random.default_rng(7 * n)
    T = 33
    x = no.rnd(rng.standard_normal((T, n)).astype(np.float32), "bf16")
    r = no.rnd(rng.standard_normal((T, n)).astype(np.float32) * 0.37, "bf16")
    w = up(client, no.rnd(rng.standard_normal(n).astype(np.float32), "bf16"), "bf16")
    h, y1, m1, s1 = norm.forward_alloc(client, up(client, x, "bf16"), w, None, kind, 1e-5, up(client, r, "bf16"))
    client.sync()
    np.testing.assert_array_equal(bits(client, h), hbits(no.rnd(x + r, "bf16"), "bf16"))
    _, y2, m2, s2 = norm.forward_alloc(client, up(client, down(client, h), "bf16"), w, None, kind, 1e-5)
    client.sync()
    np.testing.assert_array_equal(bits(client, y1), bits(client, y2))
    np.testing.assert_array_equal(s1.to_numpy(client).view(np.uint32), s2.to_numpy(client).view(np.uint32))


# ---------------------------------------------------------------------------------------------- fp8 output
SCHEMES = [(v, blk, sdt) for v in ("e4m3", "e5m2") for blk in (32, 64, 128) for sdt in ("f32", "ue8m0")]


@pytest.mark.parametrize("value,block,sdt", SCHEMES)
def test_fp8_output_equals_quantize_of_f32_output(client, value, block, sdt):
    rng = np.random.default_rng(block)
    T, n = 70, 4096 if block != 64 else 1024
    scheme = QuantScheme().with_value(value).per_block(block, sdt)
    x = no.rnd(rng.standard_normal((T, n)).astype(np.float32) * 4, "bf16")
    x[3, :block] = 0.0            # an all-zero block: scale 0, codes 0
    w = up(client, no.rnd(rng.standard_normal(n).astype(np.float32), "bf16"), "bf16")
    tx = up(client, x, "bf16")
    q, _, _, _ = norm.forward_quantized_alloc(client, tx, scheme, w, None, "rms", 1e-6)
    _, yf, _, _ = norm.forward_alloc(client, tx, w, None, "rms", 1e-6, out_dtype="f32")
    ref = quant.quantize(client, yf, scheme)
    client.sync()
    np.testing.assert_array_equal(q.values.to_numpy(client), ref.values.to_numpy(client))
    np.testing.assert_array_equal(q.block_scales.to_numpy(client), ref.block_scales.to_numpy(client))


def test_fp8_output_feeds_the_fp8_matmul(client):
    rng = np.random.default_rng(5)
    T, K, N = 256, 2048, 384
    scheme = QuantScheme().with_value("e4m3").per_block(128, "f32")
    x = no.rnd(rng.standard_normal((T, K)).astype(np.float32), "bf16")
    r = no.rnd(rng.standard_normal((T, K)).astype(np.float32), "bf16")
    wn = up(client, no.rnd(rng.standard_normal(K).astype(np.float32), "bf16"), "f32")
    wm = quant.quantize(client, up(client, rng.standard_normal((N, K)).astype(np.float32) / 32, "bf16"), scheme)
    q, h, _, _ = norm.forward_quantized_alloc(client, up(client, x, "bf16"), scheme, wn, None, "rms", 1e-6, up(client, r, "bf16"))
    _, yb, _, _ = norm.forward_alloc(client, h, wn, None, "rms", 1e-6, out_dtype="f32")
    q2 = quant.quantize(client, yb, scheme)
    out1 = TensorHandle.empty_contiguous(client, [T, N], "bf16")
    out2 = TensorHandle.empty_contiguous(client, [T, N], "bf16")
    matmul.launch_quantized_fp8(client, q, wm, out1)
    matmul.launch_quantized_fp8(client, q2, wm, out2)
    client.sync()
    np.testing.assert_array_equal(bits(client, out1), bits(client, out2))
    assert np.abs(down(client, out1)).max() > 0


# ---------------------------------------------------------------------------------------------- sentinels and repeats
def test_padding_untouched_repeats_bitwise_and_pool_returned(client):
    rng = np.random.default_rng(11)
    T, n = 300, 5000
    x = no.rnd(rng.standard_normal((T, n)).astype(np.float32), "bf16")
    dy = no.rnd(rng.standard_normal((T, n)).astype(np.float32), "bf16")
    SENT = -7.5        # exact in bf16 and f32
    tx, tr = pitched(client, x, "bf16", pad=8, lead=0), pitched(client, x * 0.5, "bf16", pad=8, lead=0)
    y, hh = pitched(client, np.zeros((T, n)), "bf16", pad=8, lead=0, fill=SENT), pitched(client, np.zeros((T, n)), "bf16", pad=8, lead=0, fill=SENT)
    mean, rstd = up(client, np.full(T, SENT), "f32"), up(client, np.full(T, SENT), "f32")
    w = up(client, rng.standard_normal(n).astype(np.float32), "f32")
    norm.forward(client, tx, y, w, None, "layer", 1e-5, tr, hh, mean=None, rstd=rstd)
    client.sync()
    raw_y = down(client, TensorHandle(y.handle, [T, n + 8], [n + 8, 1], "bf16"))
    raw_h = down(client, TensorHandle(hh.handle, [T, n + 8], [n + 8, 1], "bf16"))
    assert np.all(raw_y[:, n:] == SENT) and np.all(raw_h[:, n:] == SENT)
    assert np.all(mean.to_numpy(client) == SENT)     # not asked for: not written
    used = client.memory_usage().bytes_in_use
    runs = []
    for _ in range(3):
        mean2 = TensorHandle.empty_contiguous(client, [T], "f32")
        norm.forward(client, tx, y, w, None, "layer", 1e-5, tr, hh, mean=mean2, rstd=rstd)
        dx, dw, db = norm.backward_alloc(client, up(client, dy, "bf16"), hh, rstd, w, mean2, "layer", bias=True)
        client.sync()
        runs.append((bits(client, y), bits(client, dx), dw.to_numpy(client).view(np.uint32), db.to_numpy(client).view(np.uint32)))
        del dx, dw, db, mean2
    for a, b_ in zip(runs[0], runs[1]):
        np.testing.assert_array_equal(a, b_)
    for a, b_ in zip(runs[0], runs[2]):
        np.testing.assert_array_equal(a, b_)
    client.sync()
    assert client.memory_usage().bytes_in_use <= used + 4 * T + 2 * T * n * 2 + 2 * n * 4 + (1 << 20)
