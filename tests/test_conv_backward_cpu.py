"""CPU: the f64 gradient oracle (pinned to torch.nn.grad), dx rebuilt from the phases the dry-run plan of
b200_conv2d_backward_data records, the launch plans of both gradients (prep, phases, zero fill, stream-K head, gathers,
channel padding, forced tiles), every validation code, the zero-extent rules, and the SASS of the backward kernels."""
import ctypes as C
import re
import subprocess

import numpy as np
import pytest
import torch

import conv_backward_oracle as cbo
import conv_oracle as co
from cubecl_b200 import _ffi
from plan_context import PlanContext
from test_conv_cpu import ROOT, _tool

F32, F16, BF16 = _ffi.F32, _ffi.F16, _ffi.BF16
DY, W, X, OUT = 0x10000000, 0x20000000, 0x30000000, 0x40000000
INVALID, UNSUPPORTED = 6, 7


def _torch_grads(x, w, dy, stride, padding, dilation):
    xt = torch.from_numpy(np.ascontiguousarray(x.transpose(0, 3, 1, 2)))
    wt = torch.from_numpy(np.ascontiguousarray(w.transpose(0, 3, 1, 2)))
    dyt = torch.from_numpy(np.ascontiguousarray(dy.transpose(0, 3, 1, 2)))
    dx = torch.nn.grad.conv2d_input(xt.shape, wt, dyt, stride=stride, padding=padding, dilation=dilation)
    dw = torch.nn.grad.conv2d_weight(xt, wt.shape, dyt, stride=stride, padding=padding, dilation=dilation)
    return dx.numpy().transpose(0, 2, 3, 1), dw.numpy().transpose(0, 2, 3, 1)


def _geometries(seed, count):
    """seeded random (N, H, W, C, Cout, KH, KW, stride, padding, dilation) with a valid output, H / W often below the kernel's
    extent"""
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < count:
        kh, kw = (int(v) for v in rng.integers(1, 8, 2))
        s = tuple(int(v) for v in rng.integers(1, 5, 2))
        p = tuple(int(v) for v in rng.integers(0, 4, 2))
        d = tuple(int(v) for v in rng.integers(1, 4, 2))
        h, w = (int(v) for v in rng.integers(1, 14, 2))
        if min(co.out_hw(h, w, kh, kw, s, p, d)) < 1:
            continue
        out.append((2, h, w, 3, 4, kh, kw, s, p, d))
    return out


# ---------------------------------------------------------------------------------------------- oracle
@pytest.mark.parametrize("geom", _geometries(1, 60))
def test_oracle_matches_torch_grad(geom):
    n, h, w, c, cout, kh, kw, s, p, d = geom
    rng = np.random.default_rng(h * 31 + w)
    x = rng.uniform(-1, 1, (n, h, w, c))
    wt = rng.uniform(-1, 1, (cout, kh, kw, c))
    oh, ow = co.out_hw(h, w, kh, kw, s, p, d)
    dy = rng.uniform(-1, 1, (n, oh, ow, cout))
    want_dx, want_dw = _torch_grads(x, wt, dy, s, p, d)
    dx, adx = cbo.conv2d_input_grad_f64(dy, wt, (h, w), s, p, d)
    dw, adw = cbo.conv2d_weight_grad_f64(x, dy, (kh, kw), s, p, d)
    np.testing.assert_allclose(dx, want_dx, rtol=0, atol=1e-12 * max(1.0, float(adx.max())))
    np.testing.assert_allclose(dw, want_dw, rtol=0, atol=1e-12 * max(1.0, float(adw.max())))


# ---------------------------------------------------------------------------------------------- dry-run plans
class Planner(PlanContext):
    def _call(self, fn, a_shape, b_shape, out_shape, dy_shape, idt, odt, stride, pad, dil, a_strides, b_strides, o_strides, ptrs):
        (sh, sw), (ph, pw), (dh, dw) = co.pair(stride), co.pair(pad), co.pair(dil)
        args = _ffi.Conv2dArgs(sh, sw, ph, pw, dh, dw)
        arr = lambda v: _ffi.u64_array(v) if v is not None else None  # noqa: E731
        rc = fn(self.ctx, None, idt, odt, ptrs[0], arr(a_shape), arr(a_strides), ptrs[1], arr(b_shape), arr(b_strides), ptrs[2],
                arr(out_shape), arr(o_strides), C.byref(args))
        return rc, self.text()

    def dgrad(self, dxs, ws, dys=None, idt=BF16, odt=BF16, stride=1, pad=0, dil=1, dy_strides=None, w_strides=None, dx_strides=None,
              ptrs=(DY, W, OUT)):
        if dys is None:
            dys = [dxs[0], *co.out_hw(dxs[1], dxs[2], ws[1], ws[2], stride, pad, dil), ws[0]]
        return self._call(self.lib.b200_conv2d_backward_data, dys, ws, dxs, dys, idt, odt, stride, pad, dil, dy_strides, w_strides,
                          dx_strides, ptrs)

    def wgrad(self, xs, dws, dys=None, idt=BF16, odt=BF16, stride=1, pad=0, dil=1, x_strides=None, dy_strides=None, dw_strides=None,
              ptrs=(X, DY, OUT)):
        if dys is None:
            dys = [xs[0], *co.out_hw(xs[1], xs[2], dws[1], dws[2], stride, pad, dil), dws[0]]
        return self._call(self.lib.b200_conv2d_backward_weight, xs, dys, dws, dys, idt, odt, stride, pad, dil, x_strides, dy_strides,
                          dw_strides, ptrs)


@pytest.fixture
def plan():
    with Planner() as p:
        yield p


def _names(t):
    return [ln.split()[1] for ln in t.splitlines() if ln.startswith("launch ")]


@pytest.mark.parametrize("geom", _geometries(2, 40))
def test_dx_rebuilt_from_the_plan_matches_torch(plan, geom):
    n, h, w, c, cout, kh, kw, s, p, d = geom
    rc, t = plan.dgrad([n, h, w, c], [cout, kh, kw, c], stride=s, pad=p, dil=d)
    assert rc == 0, (t, _ffi.load().b200_last_error())
    rng = np.random.default_rng(kh * 10 + kw)
    x = rng.uniform(-1, 1, (n, h, w, c))
    wt = rng.uniform(-1, 1, (cout, kh, kw, c))
    oh, ow = co.out_hw(h, w, kh, kw, s, p, d)
    dy = rng.uniform(-1, 1, (n, oh, ow, cout))
    want, _ = _torch_grads(x, wt, dy, s, p, d)
    got, phases = cbo.rebuild_dx_from_plan(t, dy, wt, (h, w), s)
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-10)
    # one GEMM per listed phase; a memset exactly when some phase with pixels has no taps
    names = _names(t)
    gemms = [nm for nm in names if nm.startswith("conv2d_")]
    assert len(gemms) == len(phases) and names.count("conv_dgrad_weights") == 1
    sh, sw = co.pair(s)
    listed = set(phases)
    with_pixels = {(rh, rw) for rh in range(min(sh, h)) for rw in range(min(sw, w))}
    assert listed <= with_pixels
    assert ("memset2d" in t) == (listed != with_pixels)


def test_stride_one_is_prep_and_one_forward_conv_launch(plan):
    rc, t = plan.dgrad([8, 28, 28, 128], [128, 3, 3, 128], pad=1)
    assert rc == 0, t
    names = _names(t)
    assert names[0] == "conv_dgrad_weights" and len(names) == 2
    assert re.match(r"conv2d_bf16_bf16_(2sm_n128|1sm_n128)$", names[1]), names
    # dy through im2col with the flipped kernel's corners: lower = -(dh (KH-1) - ph), upper = -ph
    assert "lower=(-1,-1) upper=(-1,-1) channels=64 pixels=128 estrides=(1,1,1,1)" in t, t
    assert "memset2d" not in t


def test_three_by_three_stride_two_is_four_dgrad_phases(plan):
    rc, t = plan.dgrad([8, 56, 56, 128], [128, 3, 3, 128], stride=2, pad=1)
    assert rc == 0, t
    names = _names(t)
    assert names[0] == "conv_dgrad_weights" and len(names) == 5
    assert all(re.match(r"conv2d_dgrad_bf16_bf16_(2sm_n128|1sm_n128)$", nm) for nm in names[1:]), names
    assert "memset2d" not in t
    assert t.count("conv dgrad phase") == 4
    # phase (0, 0): taps ky = 1 only; phase (1, 1): taps 2, 0 (ascending dy offset), dilation 1
    assert "conv dgrad phase r=(0,0) taps_h=1 taps_w=1 dil=(1,1) lower=(0,0)" in t, t
    assert "conv dgrad phase r=(1,1) taps_h=2,0 taps_w=2,0 dil=(1,1) lower=(0,0)" in t, t


def test_one_by_one_stride_two_zero_fills_once(plan):
    rc, t = plan.dgrad([8, 56, 56, 256], [512, 1, 1, 256], stride=2)
    assert rc == 0, t
    names = _names(t)
    assert names[0] == "conv_dgrad_weights" and len(names) == 2 and names[1].startswith("conv2d_dgrad_")
    assert t.count("memset2d") == 1 and "memset2d esz=2 cols=256 rows=25088" in t, t
    assert t.count("conv dgrad phase") == 1


def test_wgrad_is_one_launch_with_a_wide_stream_k_head(plan):
    rc, t = plan.wgrad([64, 56, 56, 64], [64, 3, 3, 64], pad=1)
    assert rc == 0, t
    names = _names(t)
    assert len(names) == 1 and re.match(r"conv2d_wgrad_bf16_bf16_1sm_n128$", names[0]), names
    m = re.search(r"gemm stream-k head: (\d+) whole tiles \+ (\d+) tiles in (\d+) k-ranges", t)
    assert m, t
    whole, tiles, ranges = (int(v) for v in m.groups())
    assert whole == 0 and tiles == 5 and ranges > 8 * tiles
    # every range keeps >= 8 k-blocks of 64 pixels
    assert 64 * 56 * 56 // 64 // (ranges // tiles) >= 8
    # x through im2col, 64 pixels x 64 channels; dy as (Cout, pixels) in 64 x 64 boxes; dw as (C, Cout, KH * KW)
    assert "tmap im2col esz=2 dims=(64,56,56,64) strides=(128,7168,401408) lower=(-1,-1) upper=(-1,-1) channels=64 pixels=64" in t, t
    assert "tmap esz=2 dims=(64,200704,1) strides=(128,25690112) box=(64,64)" in t, t
    assert "tmap esz=2 dims=(64,64,9) strides=(1152,128) box=(64,64)" in t, t


def test_existing_gemm_plans_keep_eight_parts(plan):
    """The stream-K cap is per problem: a matmul whose head could take more than 8 parts per tile still gets at most 8."""
    m, n, k = 256, 256, 65536
    u = _ffi.u64_array
    rc = plan.lib.b200_matmul(plan.ctx, None, BF16, F32, X, W, OUT, 2, u([m, k]), u([k, 1]), u([k, n]), u([n, 1]), u([m, n]), u([n, 1]))
    t = plan.text()
    assert rc == 0, t
    mm = re.search(r"gemm stream-k head: (\d+) whole tiles \+ (\d+) tiles in (\d+) k-ranges", t)
    assert mm, t
    assert int(mm.group(3)) <= 8 * int(mm.group(2))


def test_three_channel_stem_pads_the_operands(plan):
    rc, t = plan.wgrad([4, 32, 32, 3], [64, 7, 7, 3], stride=2, pad=3)
    assert rc == 0, t
    assert _names(t)[:-1] == ["repitch_rows"] and _names(t)[-1].startswith("conv2d_wgrad_")
    assert "dims=(8,32,32,4)" in t, t
    rc, t = plan.dgrad([4, 32, 32, 3], [64, 7, 7, 3], stride=2, pad=3)
    assert rc == 0, t
    assert _names(t)[0] == "conv_dgrad_weights" and all(nm.startswith("conv2d_dgrad_") for nm in _names(t)[1:])
    # Cout = 3 channels of dy are padded to 8
    rc, t = plan.dgrad([4, 16, 16, 64], [3, 3, 3, 64], pad=1)
    assert rc == 0 and _names(t)[0] == "repitch_rows", t


def test_nchw_and_oihw_views_add_gathers(plan):
    n, h, w, c, cout, k = 2, 14, 14, 64, 128, 3
    nchw_x = [c * h * w, w, 1, h * w]
    nchw_dy = [cout * h * w, w, 1, h * w]
    oihw = [c * k * k, 1, k, k * k]
    rc, t = plan.wgrad([n, h, w, c], [cout, k, k, c], pad=1, x_strides=nchw_x, dy_strides=nchw_dy)
    assert rc == 0, t
    assert _names(t)[:-1] == ["gather_strided", "gather_strided"]
    # backward_data reads OIHW weights in place through the prep kernel; an NCHW dy is gathered
    rc, t = plan.dgrad([n, h, w, c], [cout, k, k, c], pad=1, w_strides=oihw, dy_strides=nchw_dy)
    assert rc == 0, t
    assert _names(t)[:2] == ["gather_strided", "conv_dgrad_weights"] and len(_names(t)) == 3


@pytest.mark.parametrize("variant", ["2sm_n128", "1sm_n128"])
def test_forced_tiles_are_honoured(plan, variant):
    plan.option("gemm.variant", variant)
    rc, t = plan.dgrad([8, 28, 28, 256], [256, 3, 3, 256], stride=2, pad=1, odt=F32)
    assert rc == 0 and all(nm.endswith(variant) for nm in _names(t)[1:]), t
    rc, t = plan.wgrad([8, 28, 28, 256], [256, 3, 3, 256], pad=1, odt=F32)
    assert rc == 0 and _names(t)[-1] == f"conv2d_wgrad_bf16_f32_{variant}", t


def test_forced_tile_without_a_conv_kernel_is_refused(plan):
    plan.option("gemm.variant", "2sm_n256")
    assert plan.wgrad([8, 28, 28, 128], [128, 3, 3, 128], pad=1)[0] == INVALID
    assert plan.dgrad([8, 28, 28, 128], [128, 3, 3, 128], pad=1)[0] == INVALID


@pytest.mark.parametrize("case,status,words", [
    ("channel_mismatch", INVALID, "channels"), ("bad_dy_shape", INVALID, "expected"), ("zero_stride", INVALID, "stride"),
    ("f32_input", UNSUPPORTED, "dtype"), ("bf16_to_f16", UNSUPPORTED, "dtype"), ("stride_9", UNSUPPORTED, "stride"),
    ("corner", UNSUPPORTED, "corner"), ("too_many_pixels", UNSUPPORTED, "2^31"), ("out_layout", UNSUPPORTED, "unit channel stride"),
    ("kernel_too_large", INVALID, "larger"),
])
@pytest.mark.parametrize("which", ["dgrad", "wgrad"])
def test_malformed_and_out_of_limit_cases(plan, which, case, status, words):
    a, ws, kw = [1, 8, 8, 16], [32, 3, 3, 16], {}
    if case == "channel_mismatch":
        ws = [32, 3, 3, 8]
        kw["dys"] = [1, 6, 6, 32]
    elif case == "bad_dy_shape":
        kw["dys"] = [1, 7, 6, 32]
    elif case == "zero_stride":
        kw.update(stride=(0, 1), dys=[1, 6, 6, 32])
    elif case == "f32_input":
        kw["idt"] = kw["odt"] = F32
    elif case == "bf16_to_f16":
        kw["odt"] = F16
    elif case == "stride_9":
        kw["stride"] = 9
    elif case == "corner":
        a = [1, 400, 8, 16]
        kw["pad"] = (129, 0) if which == "wgrad" else (0, 0)
        if which == "dgrad":   # a phase whose extent reaches 128 pixels past dy: lower + extent - OH > 127
            kw.update(pad=(0, 0), dil=(1, 1))
            a, ws = [1, 300, 8, 16], [32, 150, 1, 16]
    elif case == "too_many_pixels":
        a, ws = [1 << 17, 128, 128, 16], [32, 1, 1, 16]
    elif case == "out_layout":
        if which == "dgrad":
            kw["dx_strides"] = [8 * 8 * 16 * 2, 8 * 16 * 2, 16 * 2, 2]
        else:
            kw["dw_strides"] = [3 * 3 * 16 * 2, 3 * 16 * 2, 16 * 2, 2]
    elif case == "kernel_too_large":
        a = [1, 2, 8, 16]
        kw["dys"] = [1, 1, 6, 32]
    rc, _ = plan.dgrad(a, ws, **kw) if which == "dgrad" else plan.wgrad(a, ws, **kw)
    msg = _ffi.load().b200_last_error().decode()
    assert rc == status, (which, case, rc, msg)
    assert words in msg, msg


def test_zero_extents(plan):
    # empty dx / dw: no-op
    rc, t = plan.dgrad([0, 8, 8, 16], [32, 3, 3, 16], dys=[0, 6, 6, 32])
    assert rc == 0 and _names(t) == [] and "memset" not in t
    rc, t = plan.wgrad([1, 8, 8, 16], [0, 3, 3, 16], dys=[1, 6, 6, 0])
    assert rc == 0 and _names(t) == [] and "memset" not in t
    # no pixels (N = 0) but a non-empty dw: dw is written as zeros
    rc, t = plan.wgrad([0, 8, 8, 16], [32, 3, 3, 16], dys=[0, 6, 6, 32])
    assert rc == 0 and _names(t) == [] and "memset2d esz=2 cols=16 rows=288" in t, t
    # Cout = 0 but a non-empty dx: dx is written as zeros
    rc, t = plan.dgrad([1, 8, 8, 16], [0, 3, 3, 16], dys=[1, 6, 6, 0])
    assert rc == 0 and _names(t) == [] and "memset2d esz=2 cols=16 rows=64" in t, t


# ---------------------------------------------------------------------------------------------- kernels
def test_backward_kernels_use_wgmma_and_im2col_tma_and_do_not_spill():
    tool = _tool("cuobjdump")
    _ffi.load()
    cubin = ROOT / "cubecl_b200" / "build" / "gemm_convbwd.cubin"
    out = subprocess.run([tool, "-res-usage", str(cubin)], capture_output=True, text=True, check=True).stdout
    funcs = re.findall(r"Function (\w+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)
    assert {f for f, *_ in funcs} == {f"conv2d_{g}_{i}_{o}_{t}" for g in ("dgrad", "wgrad")
                                      for i, o in (("bf16", "bf16"), ("bf16", "f32"), ("f16", "f16"), ("f16", "f32"))
                                      for t in ("2sm_n128", "1sm_n128")}
    for name, reg, stack, local in funcs:
        assert int(stack) == 0 and int(local) == 0, (name, stack, local)
    sass = subprocess.run([tool, "-sass", str(cubin)], capture_output=True, text=True, check=True).stdout
    for body in re.split(r"\n\s*Function : ", sass)[1:]:
        name = body.split()[0]
        assert "HGMMA.64x128x16.F32" in body, name
        assert "UTMALDG.4D.IM2COL" in body, name
