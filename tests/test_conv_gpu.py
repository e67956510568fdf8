"""GPU: b200_conv2d against the f64 direct convolution of tests/conv_oracle.py -- the reference's im2col known-answer test bit
for bit, integer-valued operands bit for bit, uniform operands at the repository's bounds over kernels, strides, padding,
dilations, channel counts and views, every tile and epilogue path, NaN placement, determinism, and one ResNet-scale layer
against torch's CPU conv2d."""
import numpy as np
import pytest
import torch

import conv_oracle as co
from cubecl_b200 import TensorHandle, conv, synth

pytestmark = pytest.mark.gpu

# error bounds relative to sum |x||w| (keyed by output dtype): 16-bit outputs round once, f32 outputs accumulate in f32
TOL = {"bf16": 1e-2, "f16": 1e-2, "f32": 1e-5}


def operand(shape, dtype, seed, integer=None):
    rng = np.random.default_rng(seed)
    vals = rng.integers(-integer, integer + 1, size=shape).astype(np.float32) if integer else rng.uniform(-1, 1, size=shape).astype(np.float32)
    dev = synth.to_device_dtype(vals, dtype)
    return dev, synth.from_device_dtype(dev, dtype).reshape(shape).astype(np.float64)


def run(client, x_dev, w_dev, dtype, out_dtype, stride=1, padding=0, dilation=1, x_view=None, w_view=None, **kw):
    x = TensorHandle.from_numpy(client, x_dev, dtype)
    w = TensorHandle.from_numpy(client, w_dev, dtype)
    if x_view:
        x = x_view(x)
    if w_view:
        w = w_view(w)
    out = conv.launch_alloc(client, x, w, out_dtype, stride=stride, padding=padding, dilation=dilation, **kw)
    client.sync()
    return synth.from_device_dtype(out.to_numpy(client), out_dtype).reshape(out.shape).astype(np.float64)


def check(got, x, w, out_dtype, stride=1, padding=0, dilation=1, bias=None, act=None):
    ref, aref = co.conv2d_f64(x, w, stride, padding, dilation)
    if bias is not None:
        ref = ref + bias
        aref = aref + np.abs(bias)
    if act == "relu":
        ref = np.maximum(ref, 0)
    elif act == "gelu":
        ref = np.asarray(torch.nn.functional.gelu(torch.from_numpy(ref)))
    assert got.shape == ref.shape
    err = float(np.max(np.abs(got - ref) / np.maximum(aref, 1e-30)))
    assert err <= TOL[out_dtype], f"max |gpu - f64| / sum|x||w| = {err:.3e} > {TOL[out_dtype]:.0e}"
    return err


@pytest.mark.parametrize("dtype", ["bf16", "f16"])
@pytest.mark.parametrize("out_dtype", ["same", "f32"])
def test_im2col_kat_bit_exact(client, dtype, out_dtype):
    """The reference's test_tensormap_load_im2col through b200_conv2d: one-hot weights make output channel (ky*2 + kx)*8 + c the
    im2col column of kernel position (ky, kx), channel c."""
    x, w, exp, kat = co.im2col_kat()
    od = dtype if out_dtype == "same" else "f32"
    got = run(client, synth.to_device_dtype(x.astype(np.float32), dtype), synth.to_device_dtype(w.astype(np.float32), dtype), dtype, od,
              padding=(kat["pad_h"], kat["pad_w"]))
    assert np.array_equal(got, exp)


@pytest.mark.parametrize("case", [
    # (x shape, w shape, stride, padding, dilation)
    ((1, 3, 3, 8), (32, 2, 2, 8), 1, 1, 1),
    ((2, 17, 13, 64), (64, 3, 3, 64), 1, 1, 1),
    ((3, 11, 19, 96), (200, 5, 3, 96), 2, (2, 1), (1, 2)),
    ((2, 9, 9, 24), (32, 7, 7, 24), 1, 3, 1),
    ((1, 20, 20, 3), (64, 7, 7, 3), 2, 3, 1),
])
def test_integer_operands_bit_exact(client, case):
    xs, ws, s, p, d = case
    x_dev, x = operand(xs, "bf16", 1, integer=3)
    w_dev, w = operand(ws, "bf16", 2, integer=3)
    got = run(client, x_dev, w_dev, "bf16", "f32", s, p, d)
    ref, _ = co.conv2d_f64(x, w, s, p, d)
    assert np.array_equal(got, ref)


GRID = [
    # (x shape [N,H,W,C], Cout, kernel, stride, padding, dilation)
    ((2, 16, 16, 64), 64, 1, 1, 0, 1),
    ((2, 15, 17, 64), 32, 3, 1, 1, 1),
    ((1, 23, 21, 8), 256, 3, 2, 1, 1),
    ((4, 10, 12, 24), 200, 5, 1, 2, 1),
    ((2, 19, 19, 3), 64, 7, 2, 3, 1),
    ((1, 33, 29, 256), 384, 3, 1, 1, 1),
    ((3, 14, 14, 96), 200, 3, 4, 3, 2),
    ((2, 12, 12, 64), 64, 3, 1, 0, 3),
    ((2, 7, 7, 256), 256, 3, 1, 1, 1),
    ((5, 4, 6, 64), 32, 5, 1, 3, 1),          # padding wider than the kernel's reach on one side
    ((2, 3, 2, 24), 64, 5, 1, 2, 1),          # H and W smaller than the kernel extent
    ((3, 9, 11, 8), 384, 1, 2, 0, 1),
    ((1, 31, 31, 64), 200, 3, 2, (0, 2), (2, 1)),
]


@pytest.mark.parametrize("dtype,out_dtype", [("bf16", "bf16"), ("bf16", "f32"), ("f16", "f16"), ("f16", "f32")])
@pytest.mark.parametrize("case", GRID, ids=[f"x{c[0]}-co{c[1]}-k{c[2]}-s{c[3]}-p{c[4]}-d{c[5]}" for c in GRID])
def test_uniform_operands_against_oracle(client, dtype, out_dtype, case):
    xs, cout, k, s, p, d = case
    x_dev, x = operand(xs, dtype, 11)
    w_dev, w = operand((cout, k, k, xs[3]), dtype, 12)
    got = run(client, x_dev, w_dev, dtype, out_dtype, s, p, d)
    check(got, x, w, out_dtype, s, p, d)


@pytest.mark.parametrize("act", ["relu", "gelu"])
def test_bias_and_activation(client, act):
    x_dev, x = operand((2, 13, 15, 64), "bf16", 3)
    w_dev, w = operand((200, 3, 3, 64), "bf16", 4)
    b = np.random.default_rng(5).uniform(-2, 2, 200).astype(np.float32)
    bias = TensorHandle.from_numpy(client, b, "f32")
    for od in ("bf16", "f32"):
        got = run(client, x_dev, w_dev, "bf16", od, padding=1, alpha=0.5, bias=bias, activation=act)
        check(got, 0.5 * x, w, od, padding=1, bias=b.astype(np.float64), act=act)


def test_nchw_input_and_oihw_weight_views(client):
    """torch's NCHW activations and OIHW weights passed as stride-permuted [N,H,W,C] / [Cout,KH,KW,C] views."""
    n, c, h, wd, cout, k = 2, 64, 13, 11, 96, 3
    x_nchw_dev, x_nchw = operand((n, c, h, wd), "bf16", 6)
    w_oihw_dev, w_oihw = operand((cout, c, k, k), "bf16", 7)
    perm = lambda t: TensorHandle(t.handle, [t.shape[i] for i in (0, 2, 3, 1)], [t.strides[i] for i in (0, 2, 3, 1)], t.dtype)  # noqa: E731
    got = run(client, x_nchw_dev, w_oihw_dev, "bf16", "f32", padding=1, x_view=perm, w_view=perm)
    check(got, x_nchw.transpose(0, 2, 3, 1), w_oihw.transpose(0, 2, 3, 1), "f32", padding=1)
    # the 3-channel stem as OIHW weights
    x3_dev, x3 = operand((2, 3, 21, 21), "bf16", 8)
    w3_dev, w3 = operand((64, 3, 7, 7), "bf16", 9)
    got = run(client, x3_dev, w3_dev, "bf16", "bf16", stride=2, padding=3, x_view=perm, w_view=perm)
    check(got, x3.transpose(0, 2, 3, 1), w3.transpose(0, 2, 3, 1), "bf16", stride=2, padding=3)


def test_output_channel_slice(client):
    """out is channels [64, 64 + 96) of a wider 256-channel NHWC tensor; the rest is left untouched."""
    x_dev, x = operand((2, 10, 12, 64), "bf16", 10)
    w_dev, w = operand((96, 3, 3, 64), "bf16", 11)
    oh, ow = 10, 12
    big = TensorHandle.from_numpy(client, np.full((2, oh, ow, 256), 7.0, np.float32), "f32")
    view = TensorHandle(big.handle.offset(64 * 4), [2, oh, ow, 96], [oh * ow * 256, ow * 256, 256, 1], "f32")
    conv.launch(client, TensorHandle.from_numpy(client, x_dev, "bf16"), TensorHandle.from_numpy(client, w_dev, "bf16"), view, padding=1)
    client.sync()
    full = big.to_numpy(client).astype(np.float64)
    check(full[..., 64:160], x, w, "f32", padding=1)
    assert np.all(full[..., :64] == 7.0) and np.all(full[..., 160:] == 7.0)


@pytest.mark.parametrize("opt", [("gemm.variant", "2sm_n128"), ("gemm.variant", "1sm_n128"), ("gemm.epilogue", "direct"),
                                 ("gemm.split_k", "on")])
def test_every_tile_and_epilogue_path(client, opt):
    key, val = opt
    dflt = {"gemm.variant": "auto", "gemm.epilogue": "tma", "gemm.split_k": "auto"}[key]
    client.set_option(key, val)
    try:
        for xs, cout, k, s, p in (((3, 17, 19, 64), 200, 3, 1, 1), ((2, 28, 28, 256), 256, 3, 2, 1), ((1, 9, 9, 3), 32, 7, 1, 3)):
            for od in ("bf16", "f32"):
                x_dev, x = operand(xs, "bf16", 20)
                w_dev, w = operand((cout, k, k, xs[3]), "bf16", 21)
                got = run(client, x_dev, w_dev, "bf16", od, s, p)
                check(got, x, w, od, s, p)
    finally:
        client.set_option(key, dflt)


def test_nan_reaches_exactly_the_windows_that_cover_it(client):
    """A NaN in input pixel (n, 5, 7) must make exactly the outputs whose receptive field holds it NaN: wrong im2col coordinates
    or a NaN out-of-bounds fill would show elsewhere."""
    xs, ws, s, p, d = (2, 12, 14, 64), (64, 3, 3, 64), 2, 1, 2
    x_dev, x = operand(xs, "bf16", 30)
    w_dev, w = operand(ws, "bf16", 31)
    x_dev = x_dev.copy()
    x_dev[1, 5, 7, :] = 0x7FC0   # bf16 NaN in every channel of one pixel
    got = run(client, x_dev, w_dev, "bf16", "f32", s, p, d)
    mask = np.zeros(xs, np.float64)
    mask[1, 5, 7, :] = 1.0
    hit, _ = co.conv2d_f64(mask, np.ones(ws), s, p, d)
    assert np.array_equal(np.isnan(got), hit > 0)


def test_two_runs_give_the_same_bits(client):
    x_dev, _ = operand((4, 21, 21, 128), "bf16", 40)
    w_dev, _ = operand((200, 3, 3, 128), "bf16", 41)
    client.set_option("gemm.split_k", "on")
    try:
        a = run(client, x_dev, w_dev, "bf16", "f32", padding=1)
        b = run(client, x_dev, w_dev, "bf16", "f32", padding=1)
    finally:
        client.set_option("gemm.split_k", "auto")
    assert np.array_equal(a.view(np.uint64), b.view(np.uint64))


def test_resnet_layer_against_torch_cpu(client):
    """[32, 28, 28, 256] -> 256, 3 x 3, pad 1, bf16: every output against torch's CPU f32 conv2d of the bf16-rounded operands."""
    x_dev, x = operand((32, 28, 28, 256), "bf16", 50)
    w_dev, w = operand((256, 3, 3, 256), "bf16", 51)
    got = run(client, x_dev, w_dev, "bf16", "f32", padding=1)
    xt = torch.from_numpy(x.astype(np.float32)).permute(0, 3, 1, 2)
    wt = torch.from_numpy(w.astype(np.float32)).permute(0, 3, 1, 2)
    ref = torch.nn.functional.conv2d(xt, wt, padding=1).permute(0, 2, 3, 1).double().numpy()
    aref = torch.nn.functional.conv2d(xt.abs(), wt.abs(), padding=1).permute(0, 2, 3, 1).double().numpy()
    err = float(np.max(np.abs(got - ref) / aref))
    assert err <= TOL["f32"], err
