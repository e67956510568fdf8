"""CPU: the grouped-convolution oracle against torch (f64 reference, and the serial-f32 orders against f64), the routing of
b200_conv2d_grouped* through dry-run plans (groups == 1 delegates, narrow groups run one direct launch, wide groups run the
GEMM per group on in-place slices, the weight gradient records its segments), every new error status, and the register
report of the direct kernels."""
import ctypes as C
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch

import conv_grouped_oracle as go
from conv_oracle import out_hw, pair
from cubecl_b200 import _ffi, conv
from plan_context import PlanContext

ROOT = Path(__file__).resolve().parent.parent
F32, F16, BF16 = _ffi.F32, _ffi.F16, _ffi.BF16
X, W, O = 0x10000000, 0x20000000, 0x30000000
INVALID, UNSUPPORTED = 6, 7


def _nchw(a):
    return torch.from_numpy(np.ascontiguousarray(a.transpose(0, 3, 1, 2)))


# ---------------------------------------------------------------------------------------------- oracle
ORACLE_CASES = [
    # (x shape, groups, multiplier, kernel, stride, padding, dilation)
    ((2, 9, 11, 8), 8, 1, 3, 1, 1, 1),
    ((2, 9, 11, 8), 8, 2, 5, 2, 2, 1),
    ((1, 13, 7, 16), 8, 1, 7, 1, 3, 1),
    ((2, 10, 9, 16), 4, 2, 3, 3, 1, 2),
    ((1, 11, 11, 16), 2, 1, 1, 1, 0, 1),
    ((2, 8, 12, 24), 3, 1, 3, (2, 1), (0, 2), (1, 3)),
    ((1, 15, 13, 4), 4, 2, 7, 2, 3, 1),
    ((1, 9, 9, 32), 32, 1, 2, 1, 1, 2),
]


@pytest.mark.parametrize("case", ORACLE_CASES, ids=[f"x{c[0]}-g{c[1]}-m{c[2]}-k{c[3]}-s{c[4]}-p{c[5]}-d{c[6]}" for c in ORACLE_CASES])
def test_oracle_matches_torch(case):
    xs, groups, mult, k, s, p, d = case
    rng = np.random.default_rng(7)
    c = xs[3]
    cout = groups * mult * (c // groups)
    x = rng.uniform(-1, 1, xs)
    w = rng.uniform(-1, 1, (cout, k, k, c // groups))
    sp, pp, dp = pair(s), pair(p), pair(d)
    xt, wt = _nchw(x), _nchw(w)
    want = torch.nn.functional.conv2d(xt, wt, stride=sp, padding=pp, dilation=dp, groups=groups).numpy().transpose(0, 2, 3, 1)
    got, aout = go.grouped_f64(x, w, groups, s, p, d)
    assert list(got.shape) == conv.calculate_conv2d_output(xs, w.shape, s, p, d, groups)
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-12 * max(1.0, float(aout.max())))
    dy = rng.uniform(-1, 1, got.shape)
    dyt = _nchw(dy)
    dx_want = torch.nn.grad.conv2d_input(xt.shape, wt, dyt, stride=sp, padding=pp, dilation=dp, groups=groups).numpy().transpose(0, 2, 3, 1)
    dw_want = torch.nn.grad.conv2d_weight(xt, wt.shape, dyt, stride=sp, padding=pp, dilation=dp, groups=groups).numpy().transpose(0, 2, 3, 1)
    dx, adx = go.grouped_input_grad_f64(dy, w, xs[1:3], groups, s, p, d)
    dw, adw = go.grouped_weight_grad_f64(x, dy, (k, k), groups, s, p, d)
    np.testing.assert_allclose(dx, dx_want, rtol=0, atol=1e-12 * max(1.0, float(adx.max())))
    np.testing.assert_allclose(dw, dw_want, rtol=0, atol=1e-12 * max(1.0, float(adw.max())))
    # the serial-f32 orders are the same sums: within f32 accumulation error of f64
    x32, w32, dy32 = (a.astype(np.float32) for a in (x, w, dy))
    f, _ = go.grouped_f64(x32, w32, groups, s, p, d)
    np.testing.assert_allclose(go.forward_f32(x32, w32, groups, s, p, d), f, rtol=0, atol=1e-5 * max(1.0, float(aout.max())))
    gx, _ = go.grouped_input_grad_f64(dy32, w32, xs[1:3], groups, s, p, d)
    np.testing.assert_allclose(go.dgrad_f32(dy32, w32, xs[1:3], groups, s, p, d), gx, rtol=0, atol=1e-5 * max(1.0, float(adx.max())))
    gw, _ = go.grouped_weight_grad_f64(x32, dy32, (k, k), groups, s, p, d)
    got_w, _ = go.wgrad_f32(x32, dy32, (k, k), groups, s, p, d)
    np.testing.assert_allclose(got_w, gw, rtol=0, atol=1e-5 * max(1.0, float(adw.max())))


def test_shape_rule_checks_groups():
    assert conv.calculate_conv2d_output([2, 8, 8, 32], [64, 3, 3, 4], 1, 1, 1, 8) == [2, 8, 8, 64]
    for groups, wc in ((3, 4), (8, 8), (0, 4)):
        with pytest.raises(conv.ConvShapeError):
            conv.calculate_conv2d_output([2, 8, 8, 32], [64, 3, 3, wc], 1, 1, 1, groups)


def test_wgrad_segments_formula():
    assert go.wgrad_segments(0, 100) == (64, 1)
    assert go.wgrad_segments(100, 1 << 20) == (100, 1)            # one segment: a single launch
    assert go.wgrad_segments(64 * 56 * 56, 96 * 49) == (3584, 56)  # ConvNeXt-T 56^2 x 96, 7x7 depthwise


# ---------------------------------------------------------------------------------------------- dry-run plans
class Planner(PlanContext):
    def call(self, fn, a_shape, b_shape, o_shape, groups, idt=BF16, odt=BF16, stride=1, pad=0, dil=1, a_strides=None, b_strides=None,
             o_strides=None, a=X, b=W, o=O, ep=None, forward=False):
        (sh, sw), (ph, pw), (dh, dw) = pair(stride), pair(pad), pair(dil)
        args = _ffi.Conv2dArgs(sh, sw, ph, pw, dh, dw)
        arr = lambda v: _ffi.u64_array(v) if v is not None else None  # noqa: E731
        operands = (self.ctx, None, idt, odt, a, arr(a_shape), arr(a_strides), b, arr(b_shape), arr(b_strides), o, arr(o_shape), arr(o_strides),
                    C.byref(args))
        extra = (C.byref(ep) if ep is not None else None,) if forward else ()
        if groups is None:
            rc = getattr(self.lib, fn)(*operands, *extra)
        else:
            rc = getattr(self.lib, _grouped(fn))(*operands, C.c_uint32(groups), *extra)
        return rc, self.text()

    def fwd(self, xs, ws, groups, os_=None, stride=1, pad=0, dil=1, **kw):
        if os_ is None:
            os_ = [xs[0], *out_hw(xs[1], xs[2], ws[1], ws[2], stride, pad, dil), ws[0]]
        return self.call("b200_conv2d", xs, ws, os_, groups, stride=stride, pad=pad, dil=dil, forward=True, **kw)

    def dgrad(self, xs, ws, groups, stride=1, pad=0, dil=1, **kw):
        ys = [xs[0], *out_hw(xs[1], xs[2], ws[1], ws[2], stride, pad, dil), ws[0]]
        return self.call("b200_conv2d_backward_data", ys, ws, xs, groups, stride=stride, pad=pad, dil=dil, **kw)

    def wgrad(self, xs, ws, groups, stride=1, pad=0, dil=1, **kw):
        ys = [xs[0], *out_hw(xs[1], xs[2], ws[1], ws[2], stride, pad, dil), ws[0]]
        return self.call("b200_conv2d_backward_weight", xs, ys, ws, groups, stride=stride, pad=pad, dil=dil, **kw)


def _grouped(fn):
    return fn.replace("b200_conv2d", "b200_conv2d_grouped")


@pytest.fixture
def plan():
    with Planner() as p:
        yield p


def _launches(t):
    return [ln.split()[1] for ln in t.splitlines() if ln.startswith("launch ")]


@pytest.mark.parametrize("which", ["fwd", "dgrad", "wgrad"])
@pytest.mark.parametrize("case", [((4, 14, 14, 64), (128, 3, 3, 64), 2, 1), ((2, 9, 9, 3), (32, 7, 7, 3), 2, 3),
                                  ((1, 20, 20, 256), (200, 3, 3, 256), 1, 1)])
def test_groups_one_is_the_plain_entry_point(plan, which, case):
    xs, ws, s, p = case
    rc0, t0 = getattr(plan, which)(xs, ws, None, stride=s, pad=p)
    rc1, t1 = getattr(plan, which)(xs, ws, 1, stride=s, pad=p)
    assert rc0 == rc1 == 0 and t0 == t1 and t0, (t0, t1)


@pytest.mark.parametrize("odt", [BF16, F32])
def test_depthwise_is_one_direct_launch(plan, odt):
    rc, t = plan.fwd([8, 56, 56, 144], [144, 3, 3, 1], 144, pad=1, odt=odt)
    assert rc == 0, t
    tag = "bf16" if odt == BF16 else "f32"
    assert _launches(t) == [f"conv2d_grp_bf16_{tag}"], t
    # 7 x 7 tiles of 8 x 8 pixels per image, ceil(144 / 32) channel chunks, the halo staged in shared memory
    assert re.search(r"grid=\(392,5,1\) block=256 smem=(\d+)", t) and int(re.search(r"smem=(\d+)", t).group(1)) > 0, t
    rc, t = plan.dgrad([8, 56, 56, 144], [144, 3, 3, 1], 144, pad=1, odt=odt)
    assert rc == 0 and _launches(t) == [f"conv2d_grp_dgrad_bf16_{tag}"], t
    rc, t = plan.wgrad([8, 56, 56, 144], [144, 3, 3, 1], 144, pad=1, odt=odt)
    assert rc == 0 and _launches(t) == [f"conv2d_grp_wgrad_bf16_{tag}", f"conv2d_grp_wgrad_combine_{tag}"], t


def test_last_kernel_names_the_direct_kernel(plan):
    rc, _ = plan.fwd([2, 16, 16, 32], [64, 3, 3, 4], 8, pad=1)
    assert rc == 0
    buf = C.create_string_buffer(128)
    _ffi.check(plan.lib.b200_last_kernel(plan.ctx, buf, 128))
    assert buf.value == b"conv2d_grp_bf16_bf16"


def test_wide_groups_are_one_gemm_per_group_on_in_place_slices(plan):
    xs, ws = [4, 28, 28, 512], [512, 3, 3, 128]
    for which in ("fwd", "dgrad", "wgrad"):
        rc, t = getattr(plan, which)(xs, ws, 4, pad=1)
        assert rc == 0, t
        names = _launches(t)
        kind = {"fwd": "conv2d_bf16", "dgrad": "conv2d_bf16", "wgrad": "conv2d_wgrad_bf16"}[which]
        gemms = [n for n in names if n.startswith(kind)]
        assert len(gemms) == 4, t
        assert "gather_strided" not in names and "repitch_rows" not in names, t
    # the forward reads each group's slice through the full tensor's pixel pitch
    rc, t = plan.fwd(xs, ws, 4, pad=1)
    assert t.count("tmap im2col esz=2 dims=(128,28,28,4) strides=(1024,28672,802816)") == 4, t


def test_misaligned_wide_slices_take_the_existing_copy(plan):
    # Cg = 68: the second group's slice starts 136 bytes in and its rows are not 16-byte multiples: b200_conv2d copies each
    # group's operands with the channels padded to 72
    rc, t = plan.fwd([2, 10, 10, 136], [64, 3, 3, 68], 2, pad=1)
    assert rc == 0, t
    names = _launches(t)
    assert names == ["repitch_rows", "repitch_rows", "conv2d_bf16_bf16_2sm_n128"] * 2 or \
        names == ["repitch_rows", "repitch_rows", "conv2d_bf16_bf16_1sm_n128"] * 2, t


def test_wgrad_records_its_segment_plan(plan):
    xs, ws = [4, 28, 28, 192], [192, 7, 7, 1]
    rc, t = plan.wgrad(xs, ws, 192, pad=3)
    assert rc == 0, t
    P, E = 4 * 28 * 28, 192 * 49
    L, S = go.wgrad_segments(P, E)
    assert f"conv grouped wgrad pixels={P} elements={E} segments={S} length={L}" in t, t
    assert S > 1 and "alloc " in t and _launches(t) == ["conv2d_grp_wgrad_bf16_bf16", "conv2d_grp_wgrad_combine_bf16"], t
    # one segment: a single launch, no partials buffer
    rc, t = plan.wgrad([1, 6, 6, 8], [8, 3, 3, 1], 8, pad=1)
    assert rc == 0 and "segments=1 " in t and _launches(t) == ["conv2d_grp_wgrad_bf16_bf16"] and "alloc" not in t, t


def test_views_without_unit_channel_stride_are_gathered(plan):
    n, h, w, c = 2, 12, 12, 32
    nchw = [c * h * w, w, 1, h * w]
    rc, t = plan.fwd([n, h, w, c], [64, 3, 3, 4], 8, pad=1, a_strides=nchw)
    assert rc == 0 and _launches(t) == ["gather_strided", "conv2d_grp_bf16_bf16"], t
    oihw = [4 * 9, 1, 3, 9]
    rc, t = plan.fwd([n, h, w, c], [64, 3, 3, 4], 8, pad=1, b_strides=oihw)
    assert rc == 0 and _launches(t) == ["gather_strided", "conv2d_grp_bf16_bf16"], t
    # odd channel counts with a unit channel stride are read in place
    rc, t = plan.fwd([n, h, w, 5], [5, 3, 3, 1], 5, pad=1)
    assert rc == 0 and _launches(t) == ["conv2d_grp_bf16_bf16"], t


@pytest.mark.parametrize("case,status", [
    ("groups_zero", INVALID), ("c_not_divisible", INVALID), ("cout_not_divisible", INVALID), ("weight_channels", INVALID),
    ("f32_input", UNSUPPORTED), ("bf16_to_f16", UNSUPPORTED), ("stride_9", UNSUPPORTED), ("corner", UNSUPPORTED),
    ("out_channel_stride", UNSUPPORTED), ("bad_out_shape", INVALID),
])
@pytest.mark.parametrize("which", ["fwd", "dgrad", "wgrad"])
def test_error_statuses(plan, case, status, which):
    xs, ws, groups, kw = [1, 8, 8, 16], [32, 3, 3, 2], 8, {}
    if case == "groups_zero":
        groups = 0
    elif case == "c_not_divisible":
        xs, ws, groups = [1, 8, 8, 18], [32, 3, 3, 2], 8
    elif case == "cout_not_divisible":
        ws = [36, 3, 3, 2]
    elif case == "weight_channels":
        ws = [32, 3, 3, 4]
    elif case == "f32_input":
        kw["idt"] = kw["odt"] = F32
    elif case == "bf16_to_f16":
        kw["odt"] = F16
    elif case == "stride_9":
        kw["stride"] = 9
        xs = [1, 20, 20, 16]
    elif case == "corner":
        xs = [1, 300, 8, 16]
        kw["pad"] = (129, 0)
    elif case == "out_channel_stride":
        if which == "fwd":
            kw["o_strides"] = [6 * 6 * 64, 6 * 64, 64, 2]
        elif which == "dgrad":
            kw["o_strides"] = [8 * 8 * 32, 8 * 32, 32, 2]
        else:
            kw["o_strides"] = [9 * 16, 16, 1, 8]   # dw without a unit channel stride
    elif case == "bad_out_shape":
        if which == "fwd":
            kw["os_"] = [1, 7, 6, 32]
        else:
            xs = [1, 8, 8, 16]
            # dy of the wrong shape: shrink the spatial extent seen by the gradient entry points
            ys = [1, 5, 6, 32]
            args = (ys, ws, xs) if which == "dgrad" else (xs, ys, ws)
            fn = "b200_conv2d_backward_data" if which == "dgrad" else "b200_conv2d_backward_weight"
            rc, _ = plan.call(fn, *args, groups)
            assert rc == status
            return
    rc, _ = getattr(plan, which)(xs, ws, groups, **kw)
    assert rc == status, (case, which, rc, _ffi.load().b200_last_error())


def test_zero_extents(plan):
    rc, t = plan.fwd([0, 8, 8, 16], [32, 3, 3, 2], 8, os_=[0, 6, 6, 32])
    assert rc == 0 and _launches(t) == []
    rc, t = plan.dgrad([0, 8, 8, 16], [32, 3, 3, 2], 8)
    assert rc == 0 and _launches(t) == []
    # no pixels in dy: dw is written as zeros by the one direct launch
    rc, t = plan.wgrad([0, 8, 8, 16], [32, 3, 3, 2], 8)
    assert rc == 0 and _launches(t) == ["conv2d_grp_wgrad_bf16_bf16"], t


# ---------------------------------------------------------------------------------------------- kernels
def test_direct_kernels_do_not_spill():
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not Path(tool).exists():
        pytest.skip("cuobjdump is not installed")
    _ffi.load()
    cubin = ROOT / "cubecl_b200" / "build" / "conv_grouped.cubin"
    out = subprocess.run([tool, "-res-usage", str(cubin)], capture_output=True, text=True, check=True).stdout
    funcs = re.findall(r"Function (\w+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)
    pairs = (("bf16", "bf16"), ("bf16", "f32"), ("f16", "f16"), ("f16", "f32"))
    want = {f"conv2d_grp_{k}{i}_{o}" for i, o in pairs for k in ("", "dgrad_", "wgrad_")}
    want |= {f"conv2d_grp_wgrad_combine_{o}" for o in ("bf16", "f16", "f32")}
    assert {f for f, *_ in funcs} == want
    for name, reg, stack, local in funcs:
        assert int(stack) == 0 and int(local) == 0, (name, stack, local)
