"""GPU: b200_cross_entropy and b200_cross_entropy_backward against tests/cross_entropy_oracle.py -- bit for bit on exact rows
(2^k tied maxima, every other logit at least 152 below, so every ex2 term is 1 or +0) for every logits and gradient dtype at
vocabularies from 1 to 262144; random rows within the oracle's bound of an f64 reference and within bf16 tolerance of torch;
the fused forward-with-gradient against forward then backward, in place against out of place, a planted row at several
positions and batch sizes, pitched misaligned views against compact ones, repeats, sentinels; ignored and out-of-range
targets, i32 / i64 targets, MEAN over zero counted rows; and an LM-head chain through b200_matmul."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import cross_entropy_oracle as xo
from cubecl_b200 import TensorHandle, cross_entropy as xent, synth

pytestmark = pytest.mark.gpu

NPBITS = {"bf16": np.uint16, "f16": np.uint16, "f32": np.uint32}
VS = [1, 2, 7, 1000, 32000, 50257, 128256, 151936, 262144]
SENT = 12345.0


def up(c, arr, dtype):
    return TensorHandle.from_numpy(c, synth.to_device_dtype(np.asarray(arr, np.float32), dtype), dtype)


def down(c, t):
    return synth.from_device_dtype(t.to_numpy(c), t.dtype)


def bits(a, dtype):
    return synth.to_device_dtype(np.asarray(a, np.float32), dtype).view(NPBITS[dtype])


def dev_bits(c, t):
    return t.to_numpy(c).view(NPBITS[t.dtype])


def tgt(c, y, dtype="i64"):
    return TensorHandle.from_numpy(c, np.asarray(y, np.int64 if dtype == "i64" else np.int32), dtype)


def f32(c, a):
    return TensorHandle.from_numpy(c, np.asarray(a, np.float32).reshape(-1), "f32")


def filled(c, shape, dtype, value=SENT):
    return up(c, np.full(shape, value, np.float32), dtype)


def pitched(c, arr, dtype, pad=3, lead=1, fill=SENT):
    """arr [T, V] in a wider buffer [T, V + pad] starting `lead` elements in: a misaligned, pitched view (element-wise path)"""
    T, V = arr.shape
    buf = np.full((T * (V + pad) + lead,), fill, np.float32)
    buf[lead:].reshape(T, V + pad)[:, :V] = arr
    h = up(c, buf, dtype)
    esz = 2 if dtype != "f32" else 4
    return TensorHandle(h.handle.offset(lead * esz), [T, V], [V + pad, 1], dtype), h


def run(c, x, y, reduction, dtype, gdt, eps=0.0, z=0.0, dloss=None, fused=True, ignore_index=-100):
    """(loss, lse, dlogits) of the fused call, or of forward then backward"""
    T, V = x.shape
    X, Y = up(c, x, dtype), tgt(c, y)
    nl = T if reduction == "none" else 1
    loss, lse, dx = filled(c, [nl], "f32"), filled(c, [T], "f32"), filled(c, [T, V], gdt)
    dl = f32(c, dloss)
    if fused:
        xent.forward(c, X, Y, loss, lse, reduction, ignore_index, eps, z, dl, dx)
    else:
        xent.forward(c, X, Y, loss, lse, reduction, ignore_index, eps, z)
        xent.backward(c, X, Y, lse, dl, dx, reduction, ignore_index, eps, z)
    c.sync()
    return loss, lse, dx


# ---------------------------------------------------------------------------------------------- exact rows
# each grad dtype appears once per logits dtype; label smoothing and z-loss are dyadic, and with them v a power of two
CELLS = [("f32", "f32", "mean"), ("bf16", "bf16", "sum"), ("f16", "f16", "none"), ("bf16", "f32", "none"),
         ("f16", "bf16", "mean"), ("f32", "f16", "sum")]


@pytest.mark.parametrize("cell", CELLS, ids=lambda c: "-".join(c))
@pytest.mark.parametrize("v", VS)
def test_exact_rows_match_oracle_bitwise(client, v, cell):
    dtype, gdt, reduction = cell
    rng = np.random.default_rng(v)
    T = 9
    x, _ = xo.exact_rows(rng, T, v, dtype)
    y = xo.exact_targets(rng, x)
    pow2 = v & (v - 1) == 0
    for eps, z in ((0.0, 0.0), (0.25 if pow2 else 0.0, 2.0 ** -6)):
        dloss = (rng.integers(1, 8, size=T if reduction == "none" else 1) / 4.0).astype(np.float32)
        ref, rlse, _, _ = xo.forward(x, y, reduction, -100, eps, z)
        rdx = xo.backward(x, y, rlse, dloss, reduction, -100, eps, z, gdt)
        for fused in (True, False):
            loss, lse, dx = run(client, x, y, reduction, dtype, gdt, eps, z, dloss, fused)
            np.testing.assert_array_equal(dev_bits(client, lse), bits(rlse, "f32"))
            np.testing.assert_array_equal(dev_bits(client, loss), bits(np.atleast_1d(ref), "f32"))
            np.testing.assert_array_equal(dev_bits(client, dx), bits(rdx, gdt))


# ---------------------------------------------------------------------------------------------- random rows
@pytest.mark.parametrize("reduction", ["none", "sum", "mean"])
@pytest.mark.parametrize("v", [7, 1000, 32000, 50257, 128256])
def test_random_rows_within_bound_and_torch(client, v, reduction):
    rng = np.random.default_rng(v + 1)
    T = 33
    x = xo.rnd(rng.standard_normal((T, v)).astype(np.float32) * 3, "bf16")
    y = rng.integers(0, v, size=T)
    y[::4] = -100
    eps, z = 0.1, 1e-4
    loss, lse, dx = run(client, x, y, reduction, "bf16", "f32", eps, z, np.ones(T if reduction == "none" else 1))
    rl, rlse, rg, bound = xo.reference_f64(x, y, reduction, -100, eps, z)
    got_lse = down(client, lse)
    assert np.all(np.abs(got_lse - rlse) <= bound), np.max(np.abs(got_lse - rlse) - bound)
    got = down(client, loss)
    tol = bound.sum() if reduction != "none" else bound
    assert np.all(np.abs(got - np.atleast_1d(rl)) <= tol + 1e-6 * np.abs(rl))
    g = down(client, dx)
    scale = np.abs(rg).max() + 1e-30
    assert np.max(np.abs(g - rg)) <= 1e-5 * scale + 4 * 2.0 ** -24 * v * np.abs(rg).max(), np.max(np.abs(g - rg))
    # torch's own bf16 cross-entropy and autograd
    xt = torch.tensor(x, dtype=torch.bfloat16, device="cuda", requires_grad=True)
    lt = F.cross_entropy(xt.float(), torch.tensor(y, device="cuda"), reduction=reduction, label_smoothing=eps)
    lt.backward(torch.ones_like(lt))
    np.testing.assert_allclose(down(client, loss) if reduction == "none" else got[0],
                               (lt.detach().cpu().numpy() if reduction == "none" else lt.item()), rtol=2e-2, atol=2e-2)


# ---------------------------------------------------------------------------------------------- bitwise invariants
@pytest.mark.parametrize("v", [1000, 50257, 128256])
def test_fused_equals_forward_then_backward_and_in_place_equals_out_of_place(client, v):
    rng = np.random.default_rng(v + 2)
    T = 40
    x = xo.rnd(rng.standard_normal((T, v)).astype(np.float32) * 4, "bf16")
    y = rng.integers(0, v, size=T)
    y[3] = -100
    y[5] = v + 3          # out of range: NaN row
    outs = [run(client, x, y, "mean", "bf16", "bf16", 0.05, 1e-4, [0.5], fused) for fused in (True, False)]
    for a, b in zip(outs[0], outs[1]):
        np.testing.assert_array_equal(dev_bits(client, a), dev_bits(client, b))
    X = up(client, x, "bf16")
    loss, lse, g = xent.forward_alloc(client, X, tgt(client, y), "mean", -100, 0.05, 1e-4, grad=True, dloss=0.5, in_place=True)
    client.sync()
    assert g is X
    np.testing.assert_array_equal(dev_bits(client, g), dev_bits(client, outs[0][2]))
    np.testing.assert_array_equal(dev_bits(client, loss), dev_bits(client, outs[0][0]))
    # the backward in place
    X2 = up(client, x, "bf16")
    g2 = xent.backward_alloc(client, X2, tgt(client, y), outs[0][1], 0.5, "mean", -100, 0.05, 1e-4, in_place=True)
    client.sync()
    np.testing.assert_array_equal(dev_bits(client, g2), dev_bits(client, outs[0][2]))
    d = down(client, g2)
    assert np.all(np.isnan(d[5])) and np.all(dev_bits(client, g2)[3] == 0) and np.isnan(down(client, loss)[0])


@pytest.mark.parametrize("v", [7, 1000, 4000, 32000, 50257, 128256])
def test_planted_row_is_batch_invariant(client, v):
    rng = np.random.default_rng(v + 3)
    row = xo.rnd(rng.standard_normal(v).astype(np.float32) * 5, "bf16")
    yr = int(rng.integers(0, v))
    ref = None
    for T, pos in ((1, 0), (3, 2), (4096, 1), (4096, 4095), (5000, 2500)):
        if T * v > 2 ** 29:
            continue
        x = xo.rnd(rng.standard_normal((T, v)).astype(np.float32), "bf16")
        x[pos] = row
        y = rng.integers(0, v, size=T)
        y[pos] = yr
        loss, lse, dx = run(client, x, y, "none", "bf16", "bf16", 0.1, 1e-3, np.ones(T))
        got = (dev_bits(client, loss)[pos], dev_bits(client, lse)[pos], dev_bits(client, dx)[pos])
        if ref is None:
            ref = got
        assert got[0] == ref[0] and got[1] == ref[1] and np.array_equal(got[2], ref[2]), (T, pos)


@pytest.mark.parametrize("dtype", ["f32", "bf16"])
@pytest.mark.parametrize("v", [1000, 32000, 128256])
def test_pitched_misaligned_views_match_compact_and_leave_padding(client, v, dtype):
    rng = np.random.default_rng(v + 4)
    T = 17
    x = xo.rnd(rng.standard_normal((T, v)).astype(np.float32) * 2, dtype)
    y = rng.integers(0, v, size=T)
    loss, lse, dx = run(client, x, y, "none", dtype, dtype, 0.0, 0.0, np.ones(T))
    X, _ = pitched(client, x, dtype)
    G, gbuf = pitched(client, np.zeros_like(x), dtype, pad=5, lead=3)
    l2, s2 = filled(client, [T], "f32"), filled(client, [T], "f32")
    xent.forward(client, X, tgt(client, y, "i32"), l2, s2, "none", dloss=f32(client, np.ones(T)), dlogits=G)
    client.sync()
    np.testing.assert_array_equal(dev_bits(client, l2), dev_bits(client, loss))
    np.testing.assert_array_equal(dev_bits(client, s2), dev_bits(client, lse))
    full = down(client, gbuf)
    got = full[3:].reshape(T, v + 5)
    np.testing.assert_array_equal(bits(got[:, :v], dtype), dev_bits(client, dx))
    sent = xo.rnd(np.float32(SENT), dtype)                               # the sentinel as the buffer holds it
    assert np.all(got[:, v:] == sent) and np.all(full[:3] == sent)       # padding untouched
    # repeated calls are bitwise equal
    l3 = filled(client, [T], "f32")
    xent.forward(client, X, tgt(client, y, "i32"), l3, reduction="none")
    client.sync()
    np.testing.assert_array_equal(dev_bits(client, l3), dev_bits(client, loss))


def test_targets_and_reductions(client):
    rng = np.random.default_rng(5)
    T, v = 64, 1000
    x = xo.rnd(rng.standard_normal((T, v)).astype(np.float32), "bf16")
    y = rng.integers(0, v, size=T)
    y[::3] = 7                      # ignore_index = 7
    y[1] = -1
    y[2] = v
    for tdt in ("i32", "i64"):
        loss, lse = filled(client, [T], "f32"), filled(client, [T], "f32")
        xent.forward(client, up(client, x, "bf16"), tgt(client, y, tdt), loss, lse, "none", ignore_index=7)
        client.sync()
        l = down(client, loss)
        assert np.all(dev_bits(client, loss)[::3] == 0) and np.isnan(l[1]) and np.isnan(l[2])
        ok = (y != 7) & (y >= 0) & (y < v)
        ref = F.cross_entropy(torch.tensor(x, dtype=torch.float64), torch.tensor(np.where(ok, y, 0)), reduction="none").numpy()
        np.testing.assert_allclose(l[ok], ref[ok], rtol=1e-5, atol=1e-5)
        assert np.all(np.isfinite(down(client, lse)))
    # MEAN over zero counted rows is NaN (0 / 0), and so is its gradient scale; the rows' gradients stay +0
    yi = np.full(T, -100)
    loss, lse, dx = run(client, x, yi, "mean", "bf16", "bf16", dloss=[1.0])
    assert np.isnan(down(client, loss)[0]) and np.all(dev_bits(client, dx) == 0)
    # SUM without lse: the total in the kernel's order over the oracle's row losses
    loss = filled(client, [1], "f32")
    l_rows = filled(client, [T], "f32")
    xent.forward(client, up(client, x, "bf16"), tgt(client, y % v), l_rows, None, "none")
    xent.forward(client, up(client, x, "bf16"), tgt(client, y % v), loss, None, "sum")
    client.sync()
    np.testing.assert_array_equal(dev_bits(client, loss), bits([xo.total(down(client, l_rows), "sum", T)], "f32"))


def test_lm_head_chain_matches_torch_autograd(client):
    from cubecl_b200 import matmul
    rng = np.random.default_rng(6)
    T, H, V = 256, 512, 32000
    h = xo.rnd(rng.standard_normal((T, H)).astype(np.float32) * 0.5, "bf16")
    W = xo.rnd(rng.standard_normal((V, H)).astype(np.float32) * 0.05, "bf16")
    y = rng.integers(0, V, size=T)
    Hd, Wd = up(client, h, "bf16"), up(client, W, "bf16")
    WT = TensorHandle(Wd.handle, [H, V], [1, H], "bf16")
    logits = TensorHandle.empty_contiguous(client, [T, V], "bf16")
    matmul.launch(client, Hd, WT, logits)
    loss, _, dlogits = xent.forward_alloc(client, logits, tgt(client, y), "mean", grad=True, in_place=True)
    dh = TensorHandle.empty_contiguous(client, [T, H], "bf16")
    matmul.launch(client, dlogits, Wd, dh)
    client.sync()
    ht = torch.tensor(h, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    Wt = torch.tensor(W, device="cuda", dtype=torch.bfloat16)
    lt = F.cross_entropy((ht @ Wt.T).float(), torch.tensor(y, device="cuda"))
    lt.backward()
    np.testing.assert_allclose(down(client, loss)[0], lt.item(), rtol=1e-2)
    ref = ht.grad.float().cpu().numpy()
    assert np.max(np.abs(down(client, dh) - ref)) <= 2e-2 * np.abs(ref).max()
