"""GPU: grouped and depthwise convolution (b200_conv2d_grouped*).  The direct route (Cg < 64) bit for bit against the serial-f32
orders of tests/conv_grouped_oracle.py; the wide route (Cg >= 64) exact on integer operands and bit-identical to b200_conv2d
called by hand on channel slices; groups == 1 identical to the plain entry points; NaN isolation; views; zero extents;
determinism; and a ConvNeXt depthwise and a ResNeXt grouped layer against torch on the CPU."""
import numpy as np
import pytest
import torch

import conv_grouped_oracle as go
import gemm_exact_oracle as eo
from cubecl_b200 import TensorHandle, conv, synth

pytestmark = pytest.mark.gpu

TOL = {"bf16": 1e-2, "f16": 1e-2, "f32": 1e-5}   # relative to sum |a||b|, as tests/test_conv_gpu.py


def operand(shape, dtype, seed, integer=None, lo=-1.0, hi=1.0):
    rng = np.random.default_rng(seed)
    vals = (rng.integers(-integer, integer + 1, size=shape) if integer else rng.uniform(lo, hi, size=shape)).astype(np.float32)
    dev = synth.to_device_dtype(vals, dtype)
    return dev, synth.from_device_dtype(dev, dtype).reshape(shape).astype(np.float32)


def upload(client, dev, dtype):
    return TensorHandle.from_numpy(client, dev, dtype)


def bits(client, t):
    vals = synth.from_device_dtype(t.to_numpy(client), t.dtype).reshape(t.shape).astype(np.float32)
    return eo.rne(vals, t.dtype)


def values(client, t):
    return synth.from_device_dtype(t.to_numpy(client), t.dtype).reshape(t.shape).astype(np.float64)


def mult_cout(c, groups, mult):
    return groups * mult * (c // groups) if mult >= 1 else groups


# ---------------------------------------------------------------------------------------------- direct route, bit for bit
DIRECT = [
    # (x shape, groups, multiplier, kernel, stride, padding, dilation)
    ((2, 13, 11, 32), 32, 1, 3, 1, 1, 1),
    ((2, 15, 17, 24), 24, 2, 3, 2, 1, 1),
    ((1, 19, 13, 16), 16, 1, 7, 1, 3, 1),
    ((2, 12, 12, 32), 8, 1, 3, 1, 1, 1),
    ((1, 11, 14, 64), 4, 1, 5, 3, 2, 2),
    ((2, 9, 9, 40), 5, 2, 1, 1, 0, 1),
    ((1, 10, 10, 96), 3, 1, 3, 2, (0, 1), (1, 2)),
    ((2, 7, 9, 6), 6, 3, 2, 1, 1, 1),
    ((1, 23, 21, 48), 48, 1, 7, 2, 3, 1),
]
IDS = [f"x{c[0]}-g{c[1]}-m{c[2]}-k{c[3]}-s{c[4]}-p{c[5]}-d{c[6]}" for c in DIRECT]


@pytest.mark.parametrize("dtype,out_dtype", [("bf16", "bf16"), ("bf16", "f32"), ("f16", "f16"), ("f16", "f32")])
@pytest.mark.parametrize("case", DIRECT, ids=IDS)
def test_direct_forward_and_dgrad_bit_exact(client, dtype, out_dtype, case):
    xs, groups, mult, k, s, p, d = case
    cout = mult_cout(xs[3], groups, mult)
    x_dev, x = operand(xs, dtype, 1)
    w_dev, w = operand((cout, k, k, xs[3] // groups), dtype, 2)
    xt, wt = upload(client, x_dev, dtype), upload(client, w_dev, dtype)
    out = conv.launch_alloc(client, xt, wt, out_dtype, stride=s, padding=p, dilation=d, groups=groups)
    client.sync()
    assert client.last_kernel().startswith("conv2d_grp_")
    eo.assert_bits_equal(bits(client, out), eo.rne(go.forward_f32(x, w, groups, s, p, d), out_dtype), out_dtype, "forward")
    dy_dev, dy = operand(out.shape, dtype, 3)
    dx = conv.backward_data_alloc(client, upload(client, dy_dev, dtype), wt, xs[1:3], out_dtype, stride=s, padding=p, dilation=d,
                                  groups=groups)
    client.sync()
    eo.assert_bits_equal(bits(client, dx), eo.rne(go.dgrad_f32(dy, w, xs[1:3], groups, s, p, d), out_dtype), out_dtype, "dgrad")


@pytest.mark.parametrize("out_dtype", ["bf16", "f32"])
@pytest.mark.parametrize("epi", ["alpha", "bias", "relu", "all"])
def test_direct_fused_epilogue_bit_exact(client, out_dtype, epi):
    xs, groups, k = (2, 14, 13, 32), 16, 3
    x_dev, x = operand(xs, "bf16", 4)
    w_dev, w = operand((64, k, k, 2), "bf16", 5)
    b = np.random.default_rng(6).uniform(-1, 1, 64).astype(np.float32)
    alpha = 0.75 if epi in ("alpha", "all") else None
    bias = b if epi in ("bias", "all") else None
    relu = epi in ("relu", "all")
    out = conv.launch_alloc(client, upload(client, x_dev, "bf16"), upload(client, w_dev, "bf16"), out_dtype, padding=1, groups=groups,
                            alpha=1.0 if alpha is None else alpha, bias=upload(client, b, "f32") if bias is not None else None,
                            activation="relu" if relu else None)
    client.sync()
    want = go.forward_f32(x, w, groups, 1, 1, 1, alpha=alpha, bias=bias, relu=relu)
    eo.assert_bits_equal(bits(client, out), eo.rne(want, out_dtype), out_dtype, epi)


def test_direct_gelu_within_a_few_ulps(client):
    x_dev, x = operand((2, 12, 12, 32), "bf16", 7)
    w_dev, w = operand((32, 3, 3, 1), "bf16", 8)
    out = conv.launch_alloc(client, upload(client, x_dev, "bf16"), upload(client, w_dev, "bf16"), "f32", padding=1, groups=32,
                            activation="gelu")
    client.sync()
    acc = go.forward_f32(x, w, 32, 1, 1, 1).astype(np.float64)
    want = np.asarray(torch.nn.functional.gelu(torch.from_numpy(acc)))
    got = values(client, out)
    # erff is not correctly rounded: a few ulps of the pre-activation value, the bound of tests/test_gemm_exact_gpu.py
    assert np.max(np.abs(got - want) / np.maximum(np.abs(acc), 1.0)) <= 8 * 2.0 ** -24


WGRAD = [
    ((2, 13, 11, 32), 32, 1, 3, 1, 1, 1),
    ((2, 15, 17, 24), 24, 2, 3, 2, 1, 1),
    ((4, 20, 20, 16), 16, 1, 7, 1, 3, 1),
    ((2, 12, 12, 32), 8, 1, 3, 1, 1, 1),
    ((1, 11, 14, 64), 4, 1, 5, 3, 2, 2),
    ((2, 9, 9, 40), 5, 2, 1, 1, 0, 1),
]


@pytest.mark.parametrize("dtype,out_dtype", [("bf16", "bf16"), ("bf16", "f32"), ("f16", "f32")])
@pytest.mark.parametrize("case", WGRAD, ids=[f"x{c[0]}-g{c[1]}-m{c[2]}-k{c[3]}-s{c[4]}" for c in WGRAD])
def test_direct_wgrad_bit_exact_in_segment_order(client, dtype, out_dtype, case):
    xs, groups, mult, k, s, p, d = case
    cout = mult_cout(xs[3], groups, mult)
    x_dev, x = operand(xs, dtype, 9)
    oshape = conv.calculate_conv2d_output(xs, (cout, k, k, xs[3] // groups), s, p, d, groups)
    dy_dev, dy = operand(oshape, dtype, 10)
    dw = conv.backward_weight_alloc(client, upload(client, x_dev, dtype), upload(client, dy_dev, dtype), (k, k), out_dtype, stride=s,
                                    padding=p, dilation=d, groups=groups)
    client.sync()
    want, (seg, nseg) = go.wgrad_f32(x, dy, (k, k), groups, s, p, d)
    eo.assert_bits_equal(bits(client, dw), eo.rne(want, out_dtype), out_dtype, f"wgrad L={seg} S={nseg}")


def test_direct_wgrad_exact_on_integers(client):
    xs, groups, k = (4, 16, 16, 32), 32, 3
    x_dev, x = operand(xs, "bf16", 11, integer=3)
    dy_dev, dy = operand((4, 16, 16, 64), "bf16", 12, integer=3)
    dw = conv.backward_weight_alloc(client, upload(client, x_dev, "bf16"), upload(client, dy_dev, "bf16"), (k, k), "f32", padding=1,
                                    groups=groups)
    client.sync()
    want, _ = go.grouped_weight_grad_f64(x.astype(np.float64), dy.astype(np.float64), (k, k), groups, 1, 1)
    assert np.array_equal(values(client, dw), want)


# ---------------------------------------------------------------------------------------------- wide route
WIDE = ((2, 10, 12, 256), 2, 64, 3, 1, 1)   # x, groups, Coutg, kernel, stride, padding: Cg = 128


def test_wide_groups_exact_on_integers(client):
    xs, groups, coutg, k, s, p = WIDE
    cout, cg = groups * coutg, xs[3] // groups
    x_dev, x = operand(xs, "bf16", 13, integer=2)
    w_dev, w = operand((cout, k, k, cg), "bf16", 14, integer=2)
    xt, wt = upload(client, x_dev, "bf16"), upload(client, w_dev, "bf16")
    out = conv.launch_alloc(client, xt, wt, "f32", stride=s, padding=p, groups=groups)
    client.sync()
    assert client.last_kernel().startswith("conv2d_bf16_f32_")
    assert np.array_equal(values(client, out), go.grouped_f64(x, w, groups, s, p)[0])
    dy_dev, dy = operand(out.shape, "bf16", 15, integer=2)
    dyt = upload(client, dy_dev, "bf16")
    dx = conv.backward_data_alloc(client, dyt, wt, xs[1:3], "f32", stride=s, padding=p, groups=groups)
    dw = conv.backward_weight_alloc(client, xt, dyt, (k, k), "f32", stride=s, padding=p, groups=groups)
    client.sync()
    assert np.array_equal(values(client, dx), go.grouped_input_grad_f64(dy, w, xs[1:3], groups, s, p)[0])
    assert np.array_equal(values(client, dw), go.grouped_weight_grad_f64(x, dy, (k, k), groups, s, p)[0])


def _slice(t, c0, width, esz):
    return TensorHandle(t.handle.offset(c0 * esz), [*t.shape[:3], width], list(t.strides), t.dtype)


def test_wide_groups_match_per_slice_calls(client):
    xs, groups, coutg, k, s, p = WIDE
    cout, cg = groups * coutg, xs[3] // groups
    x_dev, _ = operand(xs, "bf16", 16)
    w_dev, _ = operand((cout, k, k, cg), "bf16", 17)
    xt, wt = upload(client, x_dev, "bf16"), upload(client, w_dev, "bf16")
    b = upload(client, np.random.default_rng(18).uniform(-1, 1, cout).astype(np.float32), "f32")
    got = conv.launch_alloc(client, xt, wt, "bf16", padding=p, groups=groups, alpha=0.5, bias=b, activation="relu")
    ref = TensorHandle.empty_contiguous(client, got.shape, "bf16")
    for g in range(groups):
        wg = TensorHandle(wt.handle.offset(g * coutg * k * k * cg * 2), [coutg, k, k, cg], list(wt.strides), "bf16")
        bg = TensorHandle(b.handle.offset(g * coutg * 4), [coutg], [1], "f32")
        conv.launch(client, _slice(xt, g * cg, cg, 2), wg, _slice(ref, g * coutg, coutg, 2), padding=p, alpha=0.5, bias=bg,
                    activation="relu")
    client.sync()
    assert np.array_equal(got.to_numpy(client), ref.to_numpy(client))
    dy_dev, _ = operand(got.shape, "bf16", 19)
    dyt = upload(client, dy_dev, "bf16")
    dx = conv.backward_data_alloc(client, dyt, wt, xs[1:3], "f32", padding=p, groups=groups)
    dw = conv.backward_weight_alloc(client, xt, dyt, (k, k), "f32", padding=p, groups=groups)
    dx_ref = TensorHandle.empty_contiguous(client, dx.shape, "f32")
    dw_ref = TensorHandle.empty_contiguous(client, dw.shape, "f32")
    for g in range(groups):
        wg = TensorHandle(wt.handle.offset(g * coutg * k * k * cg * 2), [coutg, k, k, cg], list(wt.strides), "bf16")
        dwg = TensorHandle(dw_ref.handle.offset(g * coutg * k * k * cg * 4), [coutg, k, k, cg], list(dw_ref.strides), "f32")
        conv.backward_data(client, _slice(dyt, g * coutg, coutg, 2), wg, _slice(dx_ref, g * cg, cg, 4), padding=p)
        conv.backward_weight(client, _slice(xt, g * cg, cg, 2), _slice(dyt, g * coutg, coutg, 2), dwg, padding=p)
    client.sync()
    assert np.array_equal(dx.to_numpy(client), dx_ref.to_numpy(client))
    assert np.array_equal(dw.to_numpy(client), dw_ref.to_numpy(client))


def test_groups_one_gives_the_plain_bits(client):
    x_dev, _ = operand((2, 14, 14, 64), "bf16", 20)
    w_dev, _ = operand((96, 3, 3, 64), "bf16", 21)
    xt, wt = upload(client, x_dev, "bf16"), upload(client, w_dev, "bf16")
    a = conv.launch_alloc(client, xt, wt, "f32", padding=1)
    out = TensorHandle.empty_contiguous(client, a.shape, "f32")
    from cubecl_b200 import _ffi
    import ctypes as C
    args = _ffi.Conv2dArgs(1, 1, 1, 1, 1, 1)
    _ffi.check(client._lib.b200_conv2d_grouped(
        client._ctx, None, _ffi.BF16, _ffi.F32, C.c_uint64(xt.handle.ptr), _ffi.u64_array(xt.shape), _ffi.u64_array(xt.strides),
        C.c_uint64(wt.handle.ptr), _ffi.u64_array(wt.shape), _ffi.u64_array(wt.strides), C.c_uint64(out.handle.ptr),
        _ffi.u64_array(out.shape), _ffi.u64_array(out.strides), C.byref(args), C.c_uint32(1), None))
    client.sync()
    assert np.array_equal(a.to_numpy(client).view(np.uint32), out.to_numpy(client).view(np.uint32))


# ---------------------------------------------------------------------------------------------- NaN isolation
@pytest.mark.parametrize("route", ["direct", "wide"])
def test_nan_reaches_only_its_group_and_windows(client, route):
    xs, groups, k, s, p = ((2, 11, 12, 32), 8, 3, 2, 1) if route == "direct" else ((1, 9, 10, 256), 2, 3, 2, 1)
    cg = xs[3] // groups
    cout = 2 * xs[3]
    coutg = cout // groups
    x_dev, _ = operand(xs, "bf16", 22)
    w_dev, _ = operand((cout, k, k, cg), "bf16", 23)
    x_dev = x_dev.copy()
    g = 1
    x_dev[1 if xs[0] > 1 else 0, 5, 7, g * cg + 1] = 0x7FC0
    out = conv.launch_alloc(client, upload(client, x_dev, "bf16"), upload(client, w_dev, "bf16"), "f32", stride=s, padding=p, groups=groups)
    client.sync()
    mask = np.zeros(xs)
    mask[1 if xs[0] > 1 else 0, 5, 7, g * cg + 1] = 1.0
    hit, _ = go.grouped_f64(mask, np.ones((cout, k, k, cg)), groups, s, p)
    got = values(client, out)
    assert np.array_equal(np.isnan(got), hit > 0)
    assert np.isnan(got[..., g * coutg:(g + 1) * coutg]).any() and not np.isnan(np.delete(got, np.s_[g * coutg:(g + 1) * coutg], axis=3)).any()
    # the same NaN in dy reaches only group g's dx channels
    dy_dev, _ = operand(out.shape, "bf16", 24)
    dy_dev = dy_dev.copy()
    dy_dev[0, 2, 3, g * coutg] = 0x7FC0
    dx = conv.backward_data_alloc(client, upload(client, dy_dev, "bf16"), upload(client, w_dev, "bf16"), xs[1:3], "f32", stride=s,
                                  padding=p, groups=groups)
    client.sync()
    dmask = np.zeros(out.shape)
    dmask[0, 2, 3, g * coutg] = 1.0
    dhit, _ = go.grouped_input_grad_f64(dmask, np.ones((cout, k, k, cg)), xs[1:3], groups, s, p)
    assert np.array_equal(np.isnan(values(client, dx)), dhit > 0)


# ---------------------------------------------------------------------------------------------- views and extents
def test_nchw_input_and_oihw_weight_views(client):
    n, c, h, wd, groups, k = 2, 32, 13, 11, 8, 3
    x_dev, x = operand((n, c, h, wd), "bf16", 25)
    w_dev, w = operand((64, c // groups, k, k), "bf16", 26)
    perm = lambda t: TensorHandle(t.handle, [t.shape[i] for i in (0, 2, 3, 1)], [t.strides[i] for i in (0, 2, 3, 1)], t.dtype)  # noqa: E731
    out = conv.launch_alloc(client, perm(upload(client, x_dev, "bf16")), perm(upload(client, w_dev, "bf16")), "f32", padding=1,
                            groups=groups)
    client.sync()
    want = go.forward_f32(x.transpose(0, 2, 3, 1), w.transpose(0, 2, 3, 1), groups, 1, 1)
    eo.assert_bits_equal(bits(client, out), eo.rne(want, "f32"), "f32", "views")


def test_output_channel_slice(client):
    x_dev, x = operand((2, 10, 12, 32), "bf16", 27)
    w_dev, w = operand((32, 3, 3, 1), "bf16", 28)
    big = TensorHandle.from_numpy(client, np.full((2, 10, 12, 96), 7.0, np.float32), "f32")
    view = TensorHandle(big.handle.offset(40 * 4), [2, 10, 12, 32], [10 * 12 * 96, 12 * 96, 96, 1], "f32")
    conv.launch(client, upload(client, x_dev, "bf16"), upload(client, w_dev, "bf16"), view, padding=1, groups=32)
    client.sync()
    full = big.to_numpy(client)
    eo.assert_bits_equal(eo.rne(full[..., 40:72], "f32"), eo.rne(go.forward_f32(x, w, 32, 1, 1), "f32"), "f32", "slice")
    assert np.all(full[..., :40] == 7.0) and np.all(full[..., 72:] == 7.0)


@pytest.mark.parametrize("c", [3, 5])
def test_odd_channel_depthwise_read_in_place(client, c):
    x_dev, x = operand((2, 17, 15, c), "f16", 29)
    w_dev, w = operand((2 * c, 5, 5, 1), "f16", 30)
    out = conv.launch_alloc(client, upload(client, x_dev, "f16"), upload(client, w_dev, "f16"), "f16", stride=2, padding=2, groups=c)
    client.sync()
    assert client.last_kernel() == "conv2d_grp_f16_f16"
    eo.assert_bits_equal(bits(client, out), eo.rne(go.forward_f32(x, w, c, 2, 2), "f16"), "f16", f"C={c}")


def test_zero_extents(client):
    x = TensorHandle.empty_contiguous(client, [0, 8, 8, 16], "bf16")
    w = TensorHandle.empty_contiguous(client, [32, 3, 3, 2], "bf16")
    out = conv.launch_alloc(client, x, w, "f32", groups=8)
    client.sync()
    assert out.shape == [0, 6, 6, 32]
    dy = TensorHandle.empty_contiguous(client, [0, 6, 6, 32], "bf16")
    dw = TensorHandle.from_numpy(client, np.full((32, 3, 3, 2), 5.0, np.float32), "f32")
    conv.backward_weight(client, x, dy, dw, groups=8)
    client.sync()
    assert np.all(dw.to_numpy(client) == 0.0)


def test_two_runs_give_the_same_bits(client):
    x_dev, _ = operand((8, 28, 28, 64), "bf16", 31)
    dy_dev, _ = operand((8, 28, 28, 64), "bf16", 32)
    xt, dyt = upload(client, x_dev, "bf16"), upload(client, dy_dev, "bf16")
    a = conv.backward_weight_alloc(client, xt, dyt, (7, 7), "f32", padding=3, groups=64)
    b = conv.backward_weight_alloc(client, xt, dyt, (7, 7), "f32", padding=3, groups=64)
    client.sync()
    assert np.array_equal(a.to_numpy(client).view(np.uint32), b.to_numpy(client).view(np.uint32))


# ---------------------------------------------------------------------------------------------- model layers against torch
@pytest.mark.parametrize("layer", ["convnext_7x7_dw", "resnext_32x4d"])
def test_model_layers_against_torch_cpu(client, layer):
    if layer == "convnext_7x7_dw":
        xs, cout, groups, k, p = (8, 28, 28, 192), 192, 192, 7, 3
    else:
        xs, cout, groups, k, p = (8, 28, 28, 256), 256, 32, 3, 1
    x_dev, x = operand(xs, "bf16", 33)
    w_dev, w = operand((cout, k, k, xs[3] // groups), "bf16", 34)
    out = conv.launch_alloc(client, upload(client, x_dev, "bf16"), upload(client, w_dev, "bf16"), "bf16", padding=p, groups=groups)
    client.sync()
    xt = torch.from_numpy(x).permute(0, 3, 1, 2)
    wt = torch.from_numpy(w).permute(0, 3, 1, 2)
    ref = torch.nn.functional.conv2d(xt, wt, padding=p, groups=groups).permute(0, 2, 3, 1).double().numpy()
    aref = torch.nn.functional.conv2d(xt.abs(), wt.abs(), padding=p, groups=groups).permute(0, 2, 3, 1).double().numpy()
    err = float(np.max(np.abs(values(client, out) - ref) / np.maximum(aref, 1e-30)))
    assert err <= TOL["bf16"], err
