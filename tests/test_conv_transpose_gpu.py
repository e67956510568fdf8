"""GPU: b200_conv_transpose2d / 3d -- integer-valued operands bit for bit (rne of the f64 oracle) over strides 1-4 and mixed,
kernels 1-7, dilations, every output padding, odd channel counts, both tiles, both output dtypes and f16 / bf16, a channel-
slice output and the fused epilogue, with out pre-filled with NaN so every pixel is shown written (phases no tap reaches
are exactly act(bias)); without an epilogue bit-identical to the data gradient on the same operands; random bf16 against
torch; the gradient helpers against torch autograd; two streams give the same bits."""
import contextlib

import numpy as np
import pytest
import torch

import conv_transpose_oracle as cto
import gemm_exact_oracle as ge
from cubecl_b200 import TensorHandle, conv, conv3d, conv_transpose, reduce, synth

pytestmark = pytest.mark.gpu

TOL = {"bf16": 1e-2, "f16": 1e-2, "f32": 1e-5}
DEFAULTS = {"gemm.variant": "auto"}


@contextlib.contextmanager
def variant(client, v):
    try:
        client.set_option("gemm.variant", v)
        yield
    finally:
        client.set_option("gemm.variant", DEFAULTS["gemm.variant"])


def up(client, vals, dtype):
    return TensorHandle.from_numpy(client, synth.to_device_dtype(np.asarray(vals, np.float32), dtype), dtype)


def nan_out(client, shape, dtype):
    return up(client, np.full(shape, np.nan, np.float32), dtype)


def bits(client, t):
    return np.asarray(t.to_numpy(client)).view(ge.OUT_BITS_VIEW[t.dtype]).reshape(t.shape)


def values(client, t):
    return synth.from_device_dtype(np.asarray(t.to_numpy(client)), t.dtype).reshape(t.shape).astype(np.float64)


def rounded(vals, dtype):
    return synth.from_device_dtype(synth.to_device_dtype(np.asarray(vals, np.float32), dtype), dtype).reshape(np.shape(vals)).astype(np.float64)


def run(client, x, w, out_shape, od, s, p, d, ep=None, dtype="bf16"):
    """one call into a NaN-filled out; returns the out handle"""
    out = nan_out(client, out_shape, od)
    kw = {}
    if ep is not None:
        alpha, bias, act = ep
        kw = dict(alpha=alpha, bias=TensorHandle.from_numpy(client, np.asarray(bias, np.float32), "f32"), activation=act)
    conv_transpose.launch(client, up(client, x, dtype), up(client, w, dtype), out, stride=s, padding=p, dilation=d, **kw)
    client.sync()
    return out


def expected(x, w, s, p, op, d, ep=None):
    ref, aref = cto.conv_transpose_f64(x, w, s, p, op, d)
    ge.assert_exact_bound(aref)
    if ep is None:
        return ref
    alpha, bias, act = ep
    y = alpha * ref + np.asarray(bias, np.float64)
    return np.maximum(y, 0.0) if act == "relu" else y


# (x shape, Cout, kernel, stride, padding, output padding, dilation)
EXACT_GEOMS = [
    ((2, 9, 11, 64), 64, (2, 2), 2, 0, 0, 1),                  # U-Net 2x2 / 2
    ((2, 7, 8, 72), 96, (3, 3), 2, 1, 1, 1),                   # 3x3 / 2, output padding 1, C and Cout not multiples of 64
    ((1, 6, 7, 48), 40, (4, 4), 2, 1, 0, 1),                   # DCGAN 4x4 / 2
    ((2, 5, 6, 3), 20, (7, 7), 3, 3, 2, 1),                    # stride 3 (two launches), C * 2 % 16 != 0 on both sides
    ((1, 5, 5, 24), 36, (1, 1), 4, 0, 3, 1),                   # 1x1 / 4: fifteen phases without taps
    ((2, 6, 6, 32), 30, (3, 2), (2, 3), (2, 0), (1, 2), (3, 2)),   # dilation 2-3
    ((2, 8, 9, 80), 72, (3, 3), 1, 1, 0, 2),                   # stride 1: the forward kernel
    ((1, 4, 5, 6, 24), 40, (2, 2, 2), 2, 0, 1, 1),             # 3-D 2x2x2 / 2
    ((1, 3, 6, 5, 16), 24, (1, 3, 3), (1, 2, 2), (0, 1, 1), (0, 1, 0), (1, 1, 2)),   # 3-D mixed (1, 2, 2)
    ((1, 4, 4, 4, 72), 24, (3, 3, 3), 1, 1, 0, 1),             # 3-D stride 1
    ((1, 3, 3, 4, 8), 12, (4, 1, 2), (3, 1, 4), (1, 0, 0), (2, 0, 1), (1, 1, 1)),   # 3-D strides 3 and 4
]


def _ints(geom, seed, bound=4):
    xs, cout, k, s, p, op, d = geom
    x = ge.int_values(xs, bound, seed)
    w = ge.int_values((xs[-1], *k, cout), bound, seed + 1)
    return x, w


def _ep(cout, seed):
    rng = np.random.default_rng(seed)
    return 0.5, rng.integers(-16, 17, cout) / 4.0, "relu"


@pytest.mark.parametrize("tile", ["2sm_n128", "1sm_n128"])
@pytest.mark.parametrize("od", ["bf16", "f32"])
def test_integer_operands_are_exact(client, tile, od):
    for i, geom in enumerate(EXACT_GEOMS):
        xs, cout, k, s, p, op, d = geom
        x, w = _ints(geom, 10 * i)
        shape = cto.output_shape(xs, w.shape, s, p, op, d)
        for ep in (None, _ep(cout, i)):
            with variant(client, tile):
                out = run(client, x, w, shape, od, s, p, d, ep)
                kernel = client.last_kernel()
            assert kernel.endswith(tile), kernel
            ge.assert_exact(bits(client, out), expected(x, w, s, p, op, d, ep), od, f"{geom} ep={ep is not None} {kernel}")


def test_integer_f16_is_exact_and_16_bit_outputs_are_one_rounding(client):
    for i, geom in enumerate(EXACT_GEOMS[1::2]):
        xs, cout, k, s, p, op, d = geom
        x, w = _ints(geom, 100 + i)
        shape = cto.output_shape(xs, w.shape, s, p, op, d)
        ep = _ep(cout, 50 + i)
        f32 = run(client, x, w, shape, "f32", s, p, d, ep, dtype="f16")
        f16 = run(client, x, w, shape, "f16", s, p, d, ep, dtype="f16")
        ge.assert_exact(bits(client, f16), expected(x, w, s, p, op, d, ep), "f16", str(geom))
        ge.assert_bits_equal(bits(client, f16), ge.f32_run_rounded(values(client, f32), "f16"), "f16", str(geom))


def test_phases_without_taps_store_act_bias(client):
    """1x1 / 2: three of four phases receive no tap; every one of their pixels is exactly act(alpha * 0 + bias)"""
    xs, cout = (2, 7, 9, 64), 48
    x, w = _ints((xs, cout, (1, 1), 2, 0, 1, 1), 3)
    bias = np.arange(cout) / 4.0 - 5.0
    out = run(client, x, w, cto.output_shape(xs, w.shape, 2, 0, 1, 1), "f32", 2, 0, 1, (2.0, bias, "relu"))
    got = values(client, out)
    want = np.maximum(bias, 0.0)
    for rh, rw in ((0, 1), (1, 0), (1, 1)):
        assert np.array_equal(got[:, rh::2, rw::2, :], np.broadcast_to(want, got[:, rh::2, rw::2, :].shape))
    ge.assert_exact(bits(client, out), expected(x, w, 2, 0, 1, 1, (2.0, bias, "relu")), "f32")


def test_channel_slice_output(client):
    geom = EXACT_GEOMS[1]
    xs, cout, k, s, p, op, d = geom
    x, w = _ints(geom, 5)
    shape = cto.output_shape(xs, w.shape, s, p, op, d)
    n, oh, ow = shape[:3]
    big = TensorHandle.from_numpy(client, np.full((n, oh, ow, 256), 7.0, np.float32), "f32")
    view = TensorHandle(big.handle.offset(64 * 4), [n, oh, ow, cout], [oh * ow * 256, ow * 256, 256, 1], "f32")
    conv_transpose.launch(client, up(client, x, "bf16"), up(client, w, "bf16"), view, stride=s, padding=p, dilation=d)
    client.sync()
    full = big.to_numpy(client).astype(np.float64).reshape(n, oh, ow, 256)
    ge.assert_exact(full[..., 64:64 + cout].astype(np.float32).view(np.uint32), expected(x, w, s, p, op, d), "f32")
    assert np.all(full[..., :64] == 7.0) and np.all(full[..., 64 + cout:] == 7.0)


@pytest.mark.parametrize("geom", [EXACT_GEOMS[i] for i in (0, 1, 3, 4, 5, 7, 8, 10)])
def test_without_epilogue_bit_identical_to_the_data_gradient(client, geom):
    xs, cout, k, s, p, op, d = geom
    rng = np.random.default_rng(sum(xs))
    x, w = rounded(rng.uniform(-1, 1, xs), "bf16"), rounded(rng.uniform(-1, 1, (xs[-1], *k, cout)), "bf16")
    shape = cto.output_shape(xs, w.shape, s, p, op, d)
    for od in ("bf16", "f32"):
        a = run(client, x, w, shape, od, s, p, d)
        b = nan_out(client, shape, od)
        (conv3d if len(xs) == 5 else conv).backward_data(client, up(client, x, "bf16"), up(client, w, "bf16"), b, stride=s, padding=p,
                                                        dilation=d)
        client.sync()
        assert np.array_equal(bits(client, a), bits(client, b)), (geom, od)


@pytest.mark.parametrize("xs,cout,k,s,p,op", [((4, 28, 28, 128), 96, (3, 3), 2, 1, 1), ((2, 8, 12, 10, 64), 80, (2, 2, 2), 2, 0, 0)])
def test_random_bf16_against_torch(client, xs, cout, k, s, p, op):
    rng = np.random.default_rng(9)
    x, w = rounded(rng.uniform(-1, 1, xs), "bf16"), rounded(rng.uniform(-1, 1, (xs[-1], *k, cout)), "bf16")
    shape = cto.output_shape(xs, w.shape, s, p, op, 1)
    n = len(xs) - 2
    f = torch.nn.functional.conv_transpose3d if n == 3 else torch.nn.functional.conv_transpose2d
    t = lambda a: torch.from_numpy(np.ascontiguousarray(np.moveaxis(a, -1, 1)))  # noqa: E731
    want = np.moveaxis(f(t(x), t(w), stride=s, padding=p, output_padding=op).numpy(), 1, -1)
    aref = np.moveaxis(f(t(np.abs(x)), t(np.abs(w)), stride=s, padding=p, output_padding=op).numpy(), 1, -1)
    for od in ("bf16", "f32"):
        got = values(client, run(client, x, w, shape, od, s, p, 1))
        err = float(np.max(np.abs(got - want) / np.maximum(aref, 1e-30)))
        assert err <= TOL[od], (od, err)


@pytest.mark.parametrize("xs,cout,k,s,p,op,d", [((2, 9, 10, 72), 64, (3, 3), 2, 1, 1, 1), ((1, 4, 5, 6, 32), 48, (2, 3, 2), (2, 1, 2), (0, 1, 0),
                                                                                             (1, 0, 0), 1)])
def test_gradient_helpers_match_torch_autograd(client, xs, cout, k, s, p, op, d):
    rng = np.random.default_rng(21)
    n = len(xs) - 2
    x, w = rounded(rng.uniform(-1, 1, xs), "bf16"), rounded(rng.uniform(-1, 1, (xs[-1], *k, cout)), "bf16")
    shape = cto.output_shape(xs, w.shape, s, p, op, d)
    dy = rounded(rng.uniform(-1, 1, shape), "bf16")
    f = torch.nn.functional.conv_transpose3d if n == 3 else torch.nn.functional.conv_transpose2d
    t = lambda a: torch.from_numpy(np.ascontiguousarray(np.moveaxis(a, -1, 1))).requires_grad_()  # noqa: E731
    back = lambda a: np.moveaxis(a.grad.numpy(), 1, -1)  # noqa: E731

    def grads(xv, wv, dyv):
        xt, wt, bt = t(xv), t(wv), torch.zeros(cout, dtype=torch.float64, requires_grad=True)
        f(xt, wt, bt, stride=s, padding=p, output_padding=op, dilation=d).backward(torch.from_numpy(np.ascontiguousarray(np.moveaxis(dyv, -1, 1))))
        return back(xt), back(wt), bt.grad.numpy()

    want = grads(x, w, dy)
    absum = grads(np.abs(x), np.abs(w), np.abs(dy))
    kw = dict(stride=s, padding=p, dilation=d)
    dx = conv_transpose.backward_data_alloc(client, up(client, dy, "bf16"), up(client, w, "bf16"), "f32", **kw)
    dw = conv_transpose.backward_weight_alloc(client, up(client, x, "bf16"), up(client, dy, "bf16"), k, "f32", **kw)
    dyh = up(client, dy, "bf16")
    db = reduce.launch_alloc(client, TensorHandle(dyh.handle, [int(np.prod(shape[:-1])), cout], [cout, 1], "bf16"), 0, "sum")
    client.sync()
    for got, ref, a in zip((values(client, dx), values(client, dw), db.to_numpy(client).reshape(-1).astype(np.float64)), want, absum):
        assert got.shape == ref.shape
        assert float(np.max(np.abs(got - ref) / np.maximum(a, 1e-30))) <= TOL["f32"]


def test_two_streams_give_the_same_bits(client):
    geom = EXACT_GEOMS[2]
    xs, cout, k, s, p, op, d = geom
    rng = np.random.default_rng(4)
    x, w = rounded(rng.uniform(-1, 1, xs), "bf16"), rounded(rng.uniform(-1, 1, (xs[-1], *k, cout)), "bf16")
    shape = cto.output_shape(xs, w.shape, s, p, op, d)
    xh, wh = up(client, x, "bf16"), up(client, w, "bf16")
    streams = [client.create_stream(), client.create_stream()]
    outs = [[nan_out(client, shape, "f32") for _ in range(3)] for _ in streams]
    try:
        for st, row in zip(streams, outs):
            for o in row:
                conv_transpose.launch(client, xh, wh, o, stride=s, padding=p, dilation=d, stream=st)
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


@pytest.mark.parametrize("geom", [EXACT_GEOMS[1], EXACT_GEOMS[3], EXACT_GEOMS[8]])
def test_16_bit_channel_slice_output_with_the_epilogue(client, geom):
    """a bf16 channel slice at an odd channel offset of a wider tensor (rows not 16-byte aligned: the scalar direct stores)
    under alpha, bias and relu; every other channel keeps its sentinel"""
    xs, cout, k, s, p, op, d = geom
    x, w = _ints(geom, 31)
    shape = cto.output_shape(xs, w.shape, s, p, op, d)
    lead, pitch = shape[:-1], cout + 37
    alpha, bias, act = _ep(cout, 7)
    sentinel = up(client, np.full([*lead, pitch], 3.0, np.float32), "bf16")
    strides, acc = [], 1
    for e in reversed([*lead, pitch]):
        strides.insert(0, acc)
        acc *= e
    view = TensorHandle(sentinel.handle.offset(5 * 2), [*lead, cout], strides, "bf16")
    conv_transpose.launch(client, up(client, x, "bf16"), up(client, w, "bf16"), view, stride=s, padding=p, dilation=d, alpha=alpha,
                          bias=TensorHandle.from_numpy(client, np.asarray(bias, np.float32), "f32"), activation=act)
    client.sync()
    full = np.asarray(sentinel.to_numpy(client)).view(np.uint16).reshape(*lead, pitch)
    ge.assert_exact(full[..., 5:5 + cout], expected(x, w, s, p, op, d, (alpha, bias, act)), "bf16", str(geom))
    rest = np.concatenate([full[..., :5].reshape(-1), full[..., 5 + cout:].reshape(-1)])
    assert np.all(rest == ge.rne(np.float32(3.0), "bf16")), geom
