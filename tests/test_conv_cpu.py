"""CPU: the conv2d oracle (pinned to torch's CPU conv2d and to the reference's im2col known-answer test), the output-shape
rule, the host plans of b200_conv2d through a dry-run planning context (launches, im2col and weight tensor maps, views, tile
choice), every validation code, and the SASS and register report of the conv2d kernels."""
import ctypes as C
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch

import conv_oracle as co
from cubecl_b200 import _ffi, conv
from plan_context import PlanContext

ROOT = Path(__file__).resolve().parent.parent
F32, F16, BF16, I8 = _ffi.F32, _ffi.F16, _ffi.BF16, _ffi.I8
X, W, O = 0x10000000, 0x20000000, 0x30000000
INVALID, UNSUPPORTED = 6, 7


def _torch_conv(x, w, stride, padding, dilation):
    xt = torch.from_numpy(np.ascontiguousarray(x.transpose(0, 3, 1, 2)))
    wt = torch.from_numpy(np.ascontiguousarray(w.transpose(0, 3, 1, 2)))
    return torch.nn.functional.conv2d(xt, wt, stride=stride, padding=padding, dilation=dilation).numpy().transpose(0, 2, 3, 1)


# ---------------------------------------------------------------------------------------------- oracle
@pytest.mark.parametrize("k", [1, 2, 3, 5])
@pytest.mark.parametrize("stride", [1, 2, 3, (2, 1)])
@pytest.mark.parametrize("padding", [0, 1, 3, (2, 0)])
@pytest.mark.parametrize("dilation", [1, 2, (1, 3)])
def test_oracle_matches_torch_conv2d(k, stride, padding, dilation):
    rng = np.random.default_rng(k * 100 + hash((stride, padding, dilation)) % 97)
    x = rng.uniform(-1, 1, (2, 9, 11, 5))
    w = rng.uniform(-1, 1, (4, k, k, 5))
    try:
        want = _torch_conv(x, w, co.pair(stride), co.pair(padding), co.pair(dilation))
    except RuntimeError:
        with pytest.raises(conv.ConvShapeError):
            conv.calculate_conv2d_output(x.shape, w.shape, stride, padding, dilation)
        return
    got, aout = co.conv2d_f64(x, w, stride, padding, dilation)
    assert got.shape == want.shape
    assert list(got.shape) == conv.calculate_conv2d_output(x.shape, w.shape, stride, padding, dilation)
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-12 * max(1.0, float(aout.max())))


def test_oracle_reproduces_the_im2col_kat():
    x, w, exp, kat = co.im2col_kat()
    got, _ = co.conv2d_f64(x, w, 1, (kat["pad_h"], kat["pad_w"]))
    assert np.array_equal(got, exp)
    # the table is the reference's: row 0 (ky = kx = 0) reads pixel (oh - 1, ow - 1)
    assert kat["expected_pixels"][0] == [0, 0, 0, 0, 0, 1, 2, 3, 0, 4, 5, 6, 0, 7, 8, 9]


@pytest.mark.parametrize("hw,k,s,p,d", [((7, 7), 7, 2, 3, 1), ((1, 1), 1, 1, 0, 1), ((5, 3), 3, 2, (0, 1), 2), ((2, 2), 5, 1, 2, 1)])
def test_shape_rule_matches_torch(hw, k, s, p, d):
    x = np.zeros((1, *hw, 3))
    w = np.zeros((2, k, k, 3))
    want = _torch_conv(x, w, co.pair(s), co.pair(p), co.pair(d)).shape
    assert conv.calculate_conv2d_output(x.shape, w.shape, s, p, d) == list(want)


# ---------------------------------------------------------------------------------------------- dry-run plans
class Planner(PlanContext):
    def conv(self, xs, ws, os_=None, idt=BF16, odt=BF16, stride=1, pad=0, dil=1, x_strides=None, w_strides=None, o_strides=None,
             x=X, w=W, o=O, ep=None):
        (sh, sw), (ph, pw), (dh, dw) = co.pair(stride), co.pair(pad), co.pair(dil)
        if os_ is None:
            os_ = [xs[0], *co.out_hw(xs[1], xs[2], ws[1], ws[2], stride, pad, dil), ws[0]]
        args = _ffi.Conv2dArgs(sh, sw, ph, pw, dh, dw)
        arr = lambda v: _ffi.u64_array(v) if v is not None else None  # noqa: E731
        rc = self.lib.b200_conv2d(self.ctx, None, idt, odt, x, arr(xs), arr(x_strides), w, arr(ws), arr(w_strides), o, arr(os_),
                                  arr(o_strides), C.byref(args), C.byref(ep) if ep is not None else None)
        return rc, self.text()


@pytest.fixture
def plan():
    with Planner() as p:
        yield p


def _launches(t):
    return [ln for ln in t.splitlines() if ln.startswith("launch ")]


def test_compact_nhwc_is_one_conv_launch_with_im2col_and_weight_maps(plan):
    rc, t = plan.conv([8, 28, 28, 256], [256, 3, 3, 256], pad=1)
    assert rc == 0, t
    launches = _launches(t)
    assert len(launches) == 1 and re.match(r"launch conv2d_bf16_bf16_(2sm_n128|1sm_n128) grid=\(\d+,1,1\) block=384", launches[0]), t
    # x as (C, W, H, N), 128 pixels x 64 channels per load; corners (-pad, pad - dilation * (K - 1)) per (w, h)
    assert ("tmap im2col esz=2 dims=(256,28,28,8) strides=(512,14336,401408) lower=(-1,-1) upper=(-1,-1) channels=64 pixels=128 "
            "estrides=(1,1,1,1) swizzle=3") in t, t
    # weights as (C, KH * KW, Cout), one kernel position of 64 channels x n_local output channels per load
    n_local = 64 if "2sm_n128" in launches[0] else 128
    assert f"tmap esz=2 dims=(256,9,256) strides=(512,4608) box=(64,1,{n_local}) swizzle=3" in t, t


def test_stride_dilation_and_asymmetric_padding_reach_the_map(plan):
    rc, t = plan.conv([2, 30, 20, 64], [128, 3, 5, 64], stride=(2, 3), pad=(1, 4), dil=(3, 2))
    assert rc == 0, t
    assert "lower=(-4,-1) upper=(-4,-5) channels=64 pixels=128 estrides=(1,3,2,1)" in t, t
    assert len(_launches(t)) == 1


def test_oihw_weights_and_nchw_input_each_add_one_gather(plan):
    n, h, w, c, cout, k = 2, 14, 14, 64, 128, 3
    oihw = [c * k * k, 1, k, k * k]               # torch OIHW storage seen as [Cout, KH, KW, C]
    nchw = [c * h * w, w, 1, h * w]               # torch NCHW storage seen as [N, H, W, C]
    rc, t = plan.conv([n, h, w, c], [cout, k, k, c], pad=1, w_strides=oihw)
    assert rc == 0, t
    assert [ln.split()[1] for ln in _launches(t)][:-1] == ["gather_strided"]
    rc, t = plan.conv([n, h, w, c], [cout, k, k, c], pad=1, x_strides=nchw, w_strides=oihw)
    assert rc == 0, t
    names = [ln.split()[1] for ln in _launches(t)]
    assert names[:-1] == ["gather_strided", "gather_strided"] and names[-1].startswith("conv2d_bf16_bf16_")


def test_three_channel_stem_pads_both_operands_to_eight_channels(plan):
    rc, t = plan.conv([4, 32, 32, 3], [64, 7, 7, 3], stride=2, pad=3)
    assert rc == 0, t
    names = [ln.split()[1] for ln in _launches(t)]
    assert names[:-1] == ["repitch_rows", "repitch_rows"] and names[-1].startswith("conv2d_")
    assert "tmap im2col esz=2 dims=(8,32,32,4) strides=(16,512,16384) lower=(-3,-3) upper=(-3,-3)" in t, t
    assert "tmap esz=2 dims=(8,49,64) strides=(16,784)" in t, t
    # a stride-permuted (OIHW) 3-channel weight view flattens (KH, KW): still one copy per operand
    rc, t = plan.conv([4, 32, 32, 3], [64, 7, 7, 3], stride=2, pad=3, w_strides=[3 * 49, 7, 1, 49])
    assert rc == 0 and [ln.split()[1] for ln in _launches(t)][:-1] == ["repitch_rows", "repitch_rows"], t


def test_output_channel_slice_keeps_the_pixel_pitch(plan):
    rc, t = plan.conv([2, 16, 16, 64], [96, 3, 3, 64], pad=1, o_strides=[16 * 16 * 256, 16 * 256, 256, 1], o=O + 64 * 2)
    assert rc == 0, t
    # TMA stores need a 16-byte aligned base: the slice at channel 64 of bf16 keeps it; the out map has the 256-channel pitch
    assert "dims=(96,512,1) strides=(512," in t, t


@pytest.mark.parametrize("variant", ["2sm_n128", "1sm_n128"])
def test_forced_variant_picks_the_named_tile(plan, variant):
    plan.option("gemm.variant", variant)
    rc, t = plan.conv([8, 28, 28, 128], [128, 3, 3, 128], pad=1, odt=F32)
    assert rc == 0, t
    assert _launches(t)[-1].startswith(f"launch conv2d_bf16_f32_{variant} ")


def test_forced_tile_without_a_conv_kernel_is_refused(plan):
    plan.option("gemm.variant", "2sm_n256")
    rc, _ = plan.conv([8, 28, 28, 128], [128, 3, 3, 128], pad=1)
    assert rc == INVALID


def test_split_k_on_plans_a_stream_k_head(plan):
    plan.option("gemm.split_k", "on")
    rc, t = plan.conv([1, 20, 20, 256], [200, 3, 3, 256], pad=1, odt=F32, idt=F16)
    assert rc == 0, t
    assert "stream-k head" in t and _launches(t)[-1].startswith("launch conv2d_f16_f32_")


@pytest.mark.parametrize("case,status", [
    ("channel_mismatch", INVALID), ("bad_out_shape", INVALID), ("oh_below_one", INVALID), ("zero_stride", INVALID),
    ("f32_input", UNSUPPORTED), ("i8_input", UNSUPPORTED), ("bf16_to_f16", UNSUPPORTED), ("corner", UNSUPPORTED),
    ("dilated_corner", UNSUPPORTED), ("stride_9", UNSUPPORTED), ("too_many_pixels", UNSUPPORTED), ("out_channel_stride", UNSUPPORTED),
    ("activation", INVALID),
])
def test_malformed_and_out_of_limit_cases(plan, case, status):
    kw = {}
    xs, ws = [1, 8, 8, 16], [32, 3, 3, 16]
    if case == "channel_mismatch":
        ws = [32, 3, 3, 8]
        kw["os_"] = [1, 6, 6, 32]
    elif case == "bad_out_shape":
        kw["os_"] = [1, 7, 6, 32]
    elif case == "oh_below_one":
        xs = [1, 2, 8, 16]
        kw["os_"] = [1, 1, 6, 32]
    elif case == "zero_stride":
        kw.update(stride=(0, 1), os_=[1, 6, 6, 32])
    elif case == "f32_input":
        kw["idt"] = kw["odt"] = F32
    elif case == "i8_input":
        kw["idt"] = I8
    elif case == "bf16_to_f16":
        kw["odt"] = F16
    elif case == "corner":
        xs = [1, 300, 8, 16]
        kw["pad"] = (129, 0)
    elif case == "dilated_corner":
        ws = [32, 3, 3, 16]
        xs = [1, 400, 8, 16]
        kw["dil"] = (70, 1)
    elif case == "stride_9":
        kw["stride"] = 9
    elif case == "too_many_pixels":
        xs = [1 << 17, 128, 128, 16]
        ws = [32, 1, 1, 16]
    elif case == "out_channel_stride":
        kw["o_strides"] = [6 * 6 * 32 * 2, 6 * 32 * 2, 32 * 2, 2]
    elif case == "activation":
        kw["ep"] = _ffi.Epilogue(1.0, 7, 0)
    rc, _ = plan.conv(xs, ws, **kw)
    assert rc == status, (case, rc, _ffi.load().b200_last_error())
    if status == UNSUPPORTED and case in ("corner", "dilated_corner", "stride_9", "too_many_pixels"):
        msg = _ffi.load().b200_last_error().decode()
        assert any(word in msg for word in ("corner", "stride", "2^31")), msg


def test_zero_extent_is_a_no_op(plan):
    rc, t = plan.conv([0, 8, 8, 16], [32, 3, 3, 16], os_=[0, 6, 6, 32])
    assert rc == 0 and _launches(t) == []
    rc, t = plan.conv([1, 8, 8, 16], [0, 3, 3, 16], os_=[1, 6, 6, 0])
    assert rc == 0 and _launches(t) == []


# ---------------------------------------------------------------------------------------------- kernels
def _tool(name):
    t = shutil.which(name) or (f"/usr/local/cuda/bin/{name}" if Path(f"/usr/local/cuda/bin/{name}").exists() else None)
    if t is None:
        pytest.skip(f"{name} is not installed")
    return t


def test_conv_kernels_use_wgmma_and_im2col_tma_and_do_not_spill():
    tool = _tool("cuobjdump")
    _ffi.load()   # builds the cubins when they are missing
    cubin = ROOT / "cubecl_b200" / "build" / "gemm_conv.cubin"
    out = subprocess.run([tool, "-res-usage", str(cubin)], capture_output=True, text=True, check=True).stdout
    funcs = re.findall(r"Function (\w+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)
    assert {f for f, *_ in funcs} == {f"conv2d_{i}_{o}_{t}" for i, o in (("bf16", "bf16"), ("bf16", "f32"), ("f16", "f16"), ("f16", "f32"))
                                      for t in ("2sm_n128", "1sm_n128")}
    for name, reg, stack, local in funcs:
        assert int(stack) == 0 and int(local) == 0, (name, stack, local)
    sass = subprocess.run([tool, "-sass", str(cubin)], capture_output=True, text=True, check=True).stdout
    for body in re.split(r"\n\s*Function : ", sass)[1:]:
        name = body.split()[0]
        assert "HGMMA.64x128x16.F32" in body, name
        assert "UTMALDG.4D.IM2COL" in body, name
