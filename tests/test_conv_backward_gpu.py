"""GPU: b200_conv2d_backward_data / _weight against the f64 gradients of tests/conv_backward_oracle.py -- integer-valued
operands bit for bit, uniform operands at the repository's bounds over the forward's geometry grid plus strided / dilated /
odd-channel cases, the bias gradient through reduce, every tile and epilogue path, views and a pitched dx, NaN placement,
reproducibility, and ResNet-scale layers against torch autograd on the GPU."""
import math

import numpy as np
import pytest
import torch

import conv_backward_oracle as cbo
import conv_oracle as co
from cubecl_b200 import TensorHandle, conv, reduce, synth
from test_conv_gpu import GRID, operand

pytestmark = pytest.mark.gpu


def tol(out_dtype, k_chain):
    """error bound relative to sum |dy||w| (dx) or sum |dy||x| (dw).  16-bit outputs: 1e-2 (one output rounding).  f32: wgmma
    adds each k = 16 step into the f32 accumulator truncating (at most one ulp of the running sum, <= 2^-23 of the scale, DESIGN
    §4), so a chain of k_chain products is bounded by ceil(k_chain / 16) * 2^-23, and never tighter than the forward's 1e-5."""
    if out_dtype != "f32":
        return 1e-2
    return max(1e-5, math.ceil(k_chain / 16) * 2.0 ** -23)


def to_np(client, t, dtype):
    return synth.from_device_dtype(t.to_numpy(client), dtype).reshape(t.shape).astype(np.float64)


def run_dx(client, dy_dev, w_dev, dtype, out_dtype, input_hw, stride=1, padding=0, dilation=1, dy_view=None, w_view=None):
    dy = TensorHandle.from_numpy(client, dy_dev, dtype)
    w = TensorHandle.from_numpy(client, w_dev, dtype)
    dy = dy_view(dy) if dy_view else dy
    w = w_view(w) if w_view else w
    dx = conv.backward_data_alloc(client, dy, w, input_hw, out_dtype, stride=stride, padding=padding, dilation=dilation)
    client.sync()
    return to_np(client, dx, out_dtype)


def run_dw(client, x_dev, dy_dev, dtype, out_dtype, kernel_hw, stride=1, padding=0, dilation=1, x_view=None, dy_view=None):
    x = TensorHandle.from_numpy(client, x_dev, dtype)
    dy = TensorHandle.from_numpy(client, dy_dev, dtype)
    x = x_view(x) if x_view else x
    dy = dy_view(dy) if dy_view else dy
    dw = conv.backward_weight_alloc(client, x, dy, kernel_hw, out_dtype, stride=stride, padding=padding, dilation=dilation)
    client.sync()
    return to_np(client, dw, out_dtype)


def check_dx(got, dy, w, input_hw, out_dtype, stride=1, padding=0, dilation=1):
    ref, aref = cbo.conv2d_input_grad_f64(dy, w, input_hw, stride, padding, dilation)
    assert got.shape == ref.shape
    kh, kw = w.shape[1], w.shape[2]
    bound = tol(out_dtype, kh * kw * ((w.shape[0] + 63) // 64 * 64))
    err = float(np.max(np.abs(got - ref) / np.maximum(aref, 1e-30)))
    assert err <= bound, f"dx: max |gpu - f64| / sum|dy||w| = {err:.3e} > {bound:.1e}"


def check_dw(got, x, dy, kernel_hw, out_dtype, stride=1, padding=0, dilation=1):
    ref, aref = cbo.conv2d_weight_grad_f64(x, dy, kernel_hw, stride, padding, dilation)
    assert got.shape == ref.shape
    bound = tol(out_dtype, dy.shape[0] * dy.shape[1] * dy.shape[2])
    err = float(np.max(np.abs(got - ref) / np.maximum(aref, 1e-30)))
    assert err <= bound, f"dw: max |gpu - f64| / sum|dy||x| = {err:.3e} > {bound:.1e}"


EXTRA = [
    # (x shape [N,H,W,C], Cout, kernel, stride, padding, dilation): strides 2-3 with dilation, odd channel counts, 1x1 stride 2
    ((2, 17, 15, 40), 72, 3, 2, 2, 2),
    ((2, 19, 16, 64), 96, 5, 3, (2, 1), (1, 2)),
    ((3, 14, 14, 64), 128, 1, 2, 0, 1),
    ((2, 12, 13, 3), 64, 7, 2, 3, 1),
    ((2, 11, 10, 100), 3, 3, (3, 2), 1, 3),
]
CASES = GRID + EXTRA
IDS = [f"x{c[0]}-co{c[1]}-k{c[2]}-s{c[3]}-p{c[4]}-d{c[5]}" for c in CASES]


def dy_shape(xs, cout, k, s, p, d):
    return (xs[0], *co.out_hw(xs[1], xs[2], k, k, s, p, d), cout)


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_integer_operands_bit_exact(client, case):
    xs, cout, k, s, p, d = case
    x_dev, x = operand(xs, "bf16", 1, integer=3)
    w_dev, w = operand((cout, k, k, xs[3]), "bf16", 2, integer=3)
    dy_dev, dy = operand(dy_shape(xs, cout, k, s, p, d), "bf16", 3, integer=3)
    got = run_dx(client, dy_dev, w_dev, "bf16", "f32", xs[1:3], s, p, d)
    assert np.array_equal(got, cbo.conv2d_input_grad_f64(dy, w, xs[1:3], s, p, d)[0])
    got = run_dw(client, x_dev, dy_dev, "bf16", "f32", (k, k), s, p, d)
    assert np.array_equal(got, cbo.conv2d_weight_grad_f64(x, dy, (k, k), s, p, d)[0])


@pytest.mark.parametrize("dtype,out_dtype", [("bf16", "bf16"), ("bf16", "f32"), ("f16", "f16"), ("f16", "f32")])
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_uniform_operands_against_oracle(client, dtype, out_dtype, case):
    xs, cout, k, s, p, d = case
    x_dev, x = operand(xs, dtype, 11)
    w_dev, w = operand((cout, k, k, xs[3]), dtype, 12)
    dy_dev, dy = operand(dy_shape(xs, cout, k, s, p, d), dtype, 13)
    check_dx(run_dx(client, dy_dev, w_dev, dtype, out_dtype, xs[1:3], s, p, d), dy, w, xs[1:3], out_dtype, s, p, d)
    check_dw(run_dw(client, x_dev, dy_dev, dtype, out_dtype, (k, k), s, p, d), x, dy, (k, k), out_dtype, s, p, d)


def test_bias_gradient_is_a_reduce_over_pixels(client):
    dy_dev, dy = operand((3, 9, 11, 200), "bf16", 14)
    t = TensorHandle.from_numpy(client, dy_dev, "bf16")
    flat = TensorHandle(t.handle, [3 * 9 * 11, 200], [200, 1], "bf16")
    db = reduce.launch_alloc(client, flat, 0, "sum")
    client.sync()
    got = db.to_numpy(client).reshape(-1).astype(np.float64)
    ref = dy.reshape(-1, 200).sum(axis=0)
    assert np.max(np.abs(got - ref) / np.abs(dy).reshape(-1, 200).sum(axis=0)) <= 1e-5


@pytest.mark.parametrize("opt", [("gemm.variant", "2sm_n128"), ("gemm.variant", "1sm_n128"), ("gemm.epilogue", "direct"),
                                 ("gemm.split_k", "on"), ("gemm.split_k", "off")])
def test_every_tile_and_epilogue_path(client, opt):
    key, val = opt
    dflt = {"gemm.variant": "auto", "gemm.epilogue": "tma", "gemm.split_k": "auto"}[key]
    client.set_option(key, val)
    try:
        for xs, cout, k, s, p in (((3, 17, 19, 64), 200, 3, 1, 1), ((2, 28, 28, 256), 256, 3, 2, 1), ((1, 9, 9, 3), 32, 7, 1, 3)):
            x_dev, x = operand(xs, "bf16", 20)
            w_dev, w = operand((cout, k, k, xs[3]), "bf16", 21)
            dy_dev, dy = operand(dy_shape(xs, cout, k, s, p, 1), "bf16", 22)
            for od in ("bf16", "f32"):
                check_dx(run_dx(client, dy_dev, w_dev, "bf16", od, xs[1:3], s, p), dy, w, xs[1:3], od, s, p)
                check_dw(run_dw(client, x_dev, dy_dev, "bf16", od, (k, k), s, p), x, dy, (k, k), od, s, p)
    finally:
        client.set_option(key, dflt)


def test_nchw_and_oihw_views_and_a_pitched_dx(client):
    n, c, h, wd, cout, k = 2, 64, 13, 11, 96, 3
    perm = lambda t: TensorHandle(t.handle, [t.shape[i] for i in (0, 2, 3, 1)], [t.strides[i] for i in (0, 2, 3, 1)], t.dtype)  # noqa: E731
    x_dev, x = operand((n, c, h, wd), "bf16", 6)
    w_dev, w = operand((cout, c, k, k), "bf16", 7)
    oh, ow = co.out_hw(h, wd, k, k, 2, 1, 1)
    dy_dev, dy = operand((n, cout, oh, ow), "bf16", 8)
    xn, wn, dyn = x.transpose(0, 2, 3, 1), w.transpose(0, 2, 3, 1), dy.transpose(0, 2, 3, 1)
    check_dx(run_dx(client, dy_dev, w_dev, "bf16", "f32", (h, wd), 2, 1, dy_view=perm, w_view=perm), dyn, wn, (h, wd), "f32", 2, 1)
    check_dw(run_dw(client, x_dev, dy_dev, "bf16", "f32", (k, k), 2, 1, x_view=perm, dy_view=perm), xn, dyn, (k, k), "f32", 2, 1)
    # dx as channels [64, 128) of a 256-channel NHWC tensor: the other channels are left untouched
    for s in (1, 2):
        oh, ow = co.out_hw(h, wd, k, k, s, 1, 1)
        dyc_dev, dyc = operand((n, oh, ow, cout), "bf16", 9)
        wc_dev, wc = operand((cout, k, k, c), "bf16", 10)
        big = TensorHandle.from_numpy(client, np.full((n, h, wd, 256), 7.0, np.float32), "f32")
        view = TensorHandle(big.handle.offset(64 * 4), [n, h, wd, c], [h * wd * 256, wd * 256, 256, 1], "f32")
        conv.backward_data(client, TensorHandle.from_numpy(client, dyc_dev, "bf16"), TensorHandle.from_numpy(client, wc_dev, "bf16"), view,
                           stride=s, padding=1)
        client.sync()
        full = big.to_numpy(client).astype(np.float64)
        check_dx(full[..., 64:128], dyc, wc, (h, wd), "f32", s, 1)
        assert np.all(full[..., :64] == 7.0) and np.all(full[..., 128:] == 7.0)


def test_nan_in_dy_reaches_exactly_the_covering_dx_pixels(client):
    xs, ws, s, p, d = (2, 12, 14, 64), (64, 3, 3, 64), 2, 1, 2
    oh, ow = co.out_hw(xs[1], xs[2], 3, 3, s, p, d)
    w_dev, _ = operand(ws, "bf16", 31)
    dy_dev, _ = operand((2, oh, ow, 64), "bf16", 32)
    dy_dev = dy_dev.copy()
    dy_dev[1, 2, 3, :] = 0x7FC0   # bf16 NaN in every channel of one dy pixel
    got = run_dx(client, dy_dev, w_dev, "bf16", "f32", xs[1:3], s, p, d)
    mask = np.zeros((2, oh, ow, 64))
    mask[1, 2, 3, :] = 1.0
    hit, _ = cbo.conv2d_input_grad_f64(mask, np.ones(ws), xs[1:3], s, p, d)
    assert np.array_equal(np.isnan(got), hit > 0)


def test_two_runs_give_the_same_bits(client):
    xs, cout, k = (8, 28, 28, 128), 128, 3
    x_dev, _ = operand(xs, "bf16", 40)
    w_dev, _ = operand((cout, k, k, 128), "bf16", 41)
    for s in (1, 2):
        dy_dev, _ = operand(dy_shape(xs, cout, k, s, 1, 1), "bf16", 42)
        a = run_dx(client, dy_dev, w_dev, "bf16", "f32", xs[1:3], s, 1)
        b = run_dx(client, dy_dev, w_dev, "bf16", "f32", xs[1:3], s, 1)
        assert np.array_equal(a.view(np.uint64), b.view(np.uint64))
        a = run_dw(client, x_dev, dy_dev, "bf16", "f32", (k, k), s, 1)
        b = run_dw(client, x_dev, dy_dev, "bf16", "f32", (k, k), s, 1)
        assert np.array_equal(a.view(np.uint64), b.view(np.uint64))


@pytest.mark.parametrize("xs,cout,k,s,p", [((32, 28, 28, 128), 128, 3, 1, 1), ((32, 56, 56, 64), 128, 3, 2, 1)])
def test_resnet_layer_against_torch_autograd(client, xs, cout, k, s, p):
    """bf16 operands; torch autograd on the GPU in f32 with TF32 off on the same (bf16-rounded) values."""
    x_dev, x = operand(xs, "bf16", 50)
    w_dev, w = operand((cout, k, k, xs[3]), "bf16", 51)
    dy_dev, dy = operand(dy_shape(xs, cout, k, s, p, 1), "bf16", 52)
    got_dx = run_dx(client, dy_dev, w_dev, "bf16", "f32", xs[1:3], s, p)
    got_dw = run_dw(client, x_dev, dy_dev, "bf16", "f32", (k, k), s, p)
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        xt = torch.from_numpy(x.astype(np.float32)).permute(0, 3, 1, 2).cuda().requires_grad_()
        wt = torch.from_numpy(w.astype(np.float32)).permute(0, 3, 1, 2).cuda().requires_grad_()
        dyt = torch.from_numpy(dy.astype(np.float32)).permute(0, 3, 1, 2).cuda()
        torch.nn.functional.conv2d(xt, wt, stride=s, padding=p).backward(dyt)
        ref_dx = xt.grad.permute(0, 2, 3, 1).double().cpu().numpy()
        ref_dw = wt.grad.permute(0, 2, 3, 1).double().cpu().numpy()
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
    _, adx = cbo.conv2d_input_grad_f64(np.abs(dy), np.abs(w), xs[1:3], s, p)
    _, adw = cbo.conv2d_weight_grad_f64(np.abs(x), np.abs(dy), (k, k), s, p)
    assert float(np.max(np.abs(got_dx - ref_dx) / np.maximum(adx, 1e-30))) <= 1e-5
    p_px = dy.shape[0] * dy.shape[1] * dy.shape[2]
    assert float(np.max(np.abs(got_dw - ref_dw) / np.maximum(adw, 1e-30))) <= tol("f32", p_px)
