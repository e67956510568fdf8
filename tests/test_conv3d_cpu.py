"""CPU: the f64 3-D convolution oracle (pinned to torch's conv3d and its autograd gradients), the dry-run plans of
b200_conv3d and both gradients (5-D im2col maps, kernels, forced tiles, stream-K head, staging copies), dx rebuilt from the
data gradient's phase lines alone, the rank-5 corner / offset / stride limits, the other refusals, zero extents, and the
gemm_conv3d cubin."""
import ctypes as C
import re
import subprocess

import numpy as np
import pytest
import torch

import conv3d_oracle as o3
from cubecl_b200 import _ffi, conv3d
from test_conv_cpu import ROOT, _tool

F32, F16, BF16, I8 = _ffi.F32, _ffi.F16, _ffi.BF16, _ffi.I8
X, W, DY, OUT = 0x10000000, 0x20000000, 0x30000000, 0x40000000
INVALID, UNSUPPORTED = 6, 7


def _ncdhw(a):
    return torch.from_numpy(np.ascontiguousarray(np.moveaxis(a, -1, 1)))


def _ndhwc(t):
    return np.moveaxis(t.detach().numpy(), 1, -1)


def _torch_all(x, w, dy, s, p, d):
    xt, wt = _ncdhw(x).requires_grad_(True), _ncdhw(w).requires_grad_(True)
    y = torch.nn.functional.conv3d(xt, wt, stride=s, padding=p, dilation=d)
    y.backward(_ncdhw(dy))
    return _ndhwc(y), _ndhwc(xt.grad), _ndhwc(wt.grad)


GEOMS = [  # (N, D, H, W, C, Cout, K, stride, padding, dilation)
    (2, 5, 6, 7, 3, 4, (3, 3, 3), 1, 1, 1),
    (1, 6, 9, 8, 2, 3, (3, 7, 7), (1, 2, 2), (1, 3, 3), 1),
    (2, 7, 7, 7, 3, 2, (3, 3, 3), 2, 1, 1),
    (1, 5, 8, 9, 2, 3, (1, 3, 3), (3, 1, 2), (0, 1, 2), 1),
    (1, 9, 9, 9, 2, 2, (3, 3, 3), 1, 2, 2),
    (2, 6, 6, 6, 3, 3, (1, 1, 1), 2, 0, 1),
    (1, 4, 5, 6, 2, 2, (2, 3, 1), (2, 3, 1), (1, 0, 0), (1, 2, 1)),
]


@pytest.mark.parametrize("geom", GEOMS)
def test_oracle_matches_torch(geom):
    n, dd, h, w, c, cout, k, s, p, d = geom
    rng = np.random.default_rng(sum(k) + dd)
    x = rng.uniform(-1, 1, (n, dd, h, w, c))
    wt = rng.uniform(-1, 1, (cout, *k, c))
    o = o3.out_dhw((dd, h, w), k, s, p, d)
    dy = rng.uniform(-1, 1, (n, *o, cout))
    y, dx, dw = _torch_all(x, wt, dy, o3.triple(s), o3.triple(p), o3.triple(d))
    got, ay = o3.conv3d_f64(x, wt, s, p, d)
    np.testing.assert_allclose(got, y, rtol=0, atol=1e-12 * max(1.0, float(ay.max())))
    gdx, _ = o3.conv3d_input_grad_f64(dy, wt, (dd, h, w), s, p, d)
    np.testing.assert_allclose(gdx, dx, rtol=0, atol=1e-11)
    gdw, _ = o3.conv3d_weight_grad_f64(x, dy, k, s, p, d)
    np.testing.assert_allclose(gdw, dw, rtol=0, atol=1e-11)
    assert conv3d.calculate_conv3d_output(x.shape, wt.shape, s, p, d) == [n, *o, cout]


# ---------------------------------------------------------------------------------------------- dry-run plans
class Planner:
    def __init__(self, sms=132):   # H100 SXM
        self.lib = _ffi.load()
        self.ctx = C.c_void_p()
        _ffi.check(self.lib.b200_plan_begin(sms, C.byref(self.ctx)))

    def text(self):
        need = C.c_size_t()
        _ffi.check(self.lib.b200_plan_text(self.ctx, None, 0, C.byref(need)))
        buf = C.create_string_buffer(need.value)
        _ffi.check(self.lib.b200_plan_text(self.ctx, buf, need.value, None))
        return buf.value.decode()

    def option(self, k, v):
        _ffi.check(self.lib.b200_set_option(self.ctx, k.encode(), str(v).encode()))

    def _call(self, fn, a, b, out, idt, odt, stride, pad, dil, strides, ptrs, ep=()):
        args = _ffi.Conv3dArgs(*o3.triple(stride), *o3.triple(pad), *o3.triple(dil))
        arr = lambda v: _ffi.u64_array(v) if v is not None else None  # noqa: E731
        rc = fn(self.ctx, None, idt, odt, ptrs[0], arr(a), arr(strides[0]), ptrs[1], arr(b), arr(strides[1]), ptrs[2], arr(out),
                arr(strides[2]), C.byref(args), *ep)
        return rc, self.text()

    def fwd(self, xs, ws, os_=None, idt=BF16, odt=BF16, stride=1, pad=0, dil=1, strides=(None, None, None), ptrs=(X, W, OUT), ep=None):
        if os_ is None:
            os_ = [xs[0], *o3.out_dhw(xs[1:4], ws[1:4], stride, pad, dil), ws[0]]
        return self._call(self.lib.b200_conv3d, xs, ws, os_, idt, odt, stride, pad, dil, strides, ptrs,
                          (C.byref(ep) if ep is not None else None,))

    def dgrad(self, dxs, ws, dys=None, idt=BF16, odt=BF16, stride=1, pad=0, dil=1, strides=(None, None, None), ptrs=(DY, W, OUT)):
        if dys is None:
            dys = [dxs[0], *o3.out_dhw(dxs[1:4], ws[1:4], stride, pad, dil), ws[0]]
        return self._call(self.lib.b200_conv3d_backward_data, dys, ws, dxs, idt, odt, stride, pad, dil, strides, ptrs)

    def wgrad(self, xs, dws, dys=None, idt=BF16, odt=BF16, stride=1, pad=0, dil=1, strides=(None, None, None), ptrs=(X, DY, OUT)):
        if dys is None:
            dys = [xs[0], *o3.out_dhw(xs[1:4], dws[1:4], stride, pad, dil), dws[0]]
        return self._call(self.lib.b200_conv3d_backward_weight, xs, dys, dws, idt, odt, stride, pad, dil, strides, ptrs)

    def close(self):
        self.lib.b200_destroy(self.ctx)


@pytest.fixture
def plan():
    p = Planner()
    yield p
    p.close()


def _names(t):
    return [ln.split()[1] for ln in t.splitlines() if ln.startswith("launch ")]


def test_forward_is_one_launch_with_a_5d_im2col_map(plan):
    rc, t = plan.fwd([4, 8, 14, 14, 128], [256, 3, 3, 3, 128], pad=1, stride=(1, 2, 2), dil=(2, 1, 1))
    assert rc == 0, t
    names = _names(t)
    assert len(names) == 1 and re.match(r"conv3d_bf16_bf16_(2sm_n128|1sm_n128)$", names[0]), names
    # x as (C, W, H, D, N) with the W, H, D, N strides in bytes; corners (w, h, d); element strides (1, sw, sh, sd, 1)
    assert ("tmap im2col5d esz=2 dims=(128,14,14,8,4) strides=(256,3584,50176,401408) lower=(-1,-1,-1) upper=(-1,-1,-3) "
            "channels=64 pixels=128 estrides=(1,2,2,1,1) swizzle=3") in t, t
    # weights as (C, KD * KH * KW, Cout)
    n_local = 64 if "2sm_n128" in names[0] else 128
    assert f"tmap esz=2 dims=(128,27,256) strides=(256,6912) box=(64,1,{n_local}) swizzle=3" in t, t


@pytest.mark.parametrize("variant", ["2sm_n128", "1sm_n128"])
def test_forced_variant_names_the_kernel_of_every_pass(plan, variant):
    plan.option("gemm.variant", variant)
    rc, t = plan.fwd([2, 8, 16, 16, 64], [64, 3, 3, 3, 64], pad=1, odt=F32)
    assert rc == 0 and _names(t) == [f"conv3d_bf16_f32_{variant}"], t
    rc, t = plan.dgrad([2, 8, 16, 16, 64], [64, 3, 3, 3, 64], pad=1, stride=2, idt=F16, odt=F16)
    assert rc == 0 and all(nm == f"conv3d_dgrad_f16_f16_{variant}" for nm in _names(t)[1:]), t
    rc, t = plan.wgrad([2, 8, 16, 16, 64], [64, 3, 3, 3, 64], pad=1)
    assert rc == 0 and _names(t) == [f"conv3d_wgrad_bf16_bf16_{variant}"], t


def test_tile_without_a_conv_kernel_is_refused(plan):
    plan.option("gemm.variant", "2sm_n256")
    rc, _ = plan.fwd([2, 8, 16, 16, 64], [64, 3, 3, 3, 64], pad=1)
    assert rc == INVALID


def test_wgrad_plans_a_stream_k_head_and_5d_maps(plan):
    rc, t = plan.wgrad([16, 16, 56, 56, 64], [64, 3, 3, 3, 64], pad=1)
    assert rc == 0, t
    assert len(_names(t)) == 1 and _names(t)[0].startswith("conv3d_wgrad_bf16_bf16_"), t
    m = re.search(r"gemm stream-k head: (\d+) whole tiles \+ (\d+) tiles in (\d+) k-ranges", t)
    assert m and int(m.group(3)) > 8 * int(m.group(2)), t
    assert "tmap im2col5d esz=2 dims=(64,56,56,16,16) strides=(128,7168,401408,6422528) lower=(-1,-1,-1) upper=(-1,-1,-1) channels=64 pixels=64" in t, t
    # dy as (Cout, pixels); dw as (C, Cout, KD * KH * KW)
    assert "tmap esz=2 dims=(64,802816,1) strides=(128,102760448) box=(64,64)" in t, t
    assert "tmap esz=2 dims=(64,64,27) strides=(3456,128) box=(64,64)" in t, t


def test_views_and_channel_padding_add_copies(plan):
    n, dd, h, w, c, cout = 2, 4, 8, 8, 64, 64
    ncdhw = [c * dd * h * w, h * w, w, 1, dd * h * w]      # torch NCDHW storage seen as NDHWC
    oidhw = [c * 27, 9, 3, 1, 27]                          # torch OIDHW storage seen as [Cout, KD, KH, KW, C]
    rc, t = plan.fwd([n, dd, h, w, c], [cout, 3, 3, 3, c], pad=1, strides=(ncdhw, oidhw, None))
    assert rc == 0 and _names(t)[:-1] == ["gather_strided", "gather_strided"], t
    # an R3D stem (C = 3): both operands copied with 8 channels
    rc, t = plan.fwd([1, 8, 32, 32, 3], [64, 3, 7, 7, 3], stride=(1, 2, 2), pad=(1, 3, 3))
    assert rc == 0 and _names(t)[:-1] == ["repitch_rows", "repitch_rows"], t
    assert "tmap im2col5d esz=2 dims=(8,32,32,8,1) strides=(16,512,16384,131072) lower=(-3,-3,-1) upper=(-3,-3,-1)" in t, t
    # a channel slice of out keeps the pixel pitch
    rc, t = plan.fwd([1, 4, 8, 8, 64], [64, 3, 3, 3, 64], pad=1, strides=(None, None, [4 * 64 * 128, 64 * 128, 8 * 128, 128, 1]))
    assert rc == 0 and len(_names(t)) == 1, t
    # the weight gradient gathers a dy whose pixels do not share one pitch
    rc, t = plan.wgrad([1, 4, 8, 8, 64], [64, 3, 3, 3, 64], pad=1, strides=(None, [4 * 8 * 9 * 64, 8 * 9 * 64, 9 * 64, 64, 1], None))
    assert rc == 0 and _names(t)[:-1] == ["gather_strided"], t


# ---------------------------------------------------------------------------------------------- data gradient phases
@pytest.mark.parametrize("dhw,k,s,p,d", [
    ((7, 8, 9), (3, 3, 3), (2, 2, 2), 1, 1),
    ((5, 8, 8), (3, 3, 3), (1, 2, 2), 1, 1),
    ((7, 6, 8), (3, 3, 3), (3, 1, 2), (1, 1, 1), 1),
    ((7, 7, 7), (3, 3, 3), 2, 2, 2),
    ((6, 6, 6), (1, 1, 1), 2, 0, 1),
    ((6, 7, 8), (3, 1, 2), (2, 1, 3), (1, 0, 1), (1, 1, 2)),
])
def test_dx_rebuilt_from_the_plan_matches_torch(plan, dhw, k, s, p, d):
    n, c, cout = 2, 3, 4
    rc, t = plan.dgrad([n, *dhw, c], [cout, *k, c], stride=s, pad=p, dil=d)
    assert rc == 0, (t, _ffi.load().b200_last_error())
    rng = np.random.default_rng(sum(dhw))
    x = rng.uniform(-1, 1, (n, *dhw, c))
    wt = rng.uniform(-1, 1, (cout, *k, c))
    o = o3.out_dhw(dhw, k, s, p, d)
    dy = rng.uniform(-1, 1, (n, *o, cout))
    _, want, _ = _torch_all(x, wt, dy, o3.triple(s), o3.triple(p), o3.triple(d))
    got, phases = o3.rebuild_dx_from_plan(t, dy, wt, dhw, s)
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-10)
    names = _names(t)
    gemms = [nm for nm in names if nm.startswith("conv3d_") and nm != "conv3d_dgrad_weights"]
    assert len(gemms) == len(phases) and names.count("conv3d_dgrad_weights") == 1
    st = o3.triple(s)
    with_pixels = {(a, b, e) for a in range(min(st[0], dhw[0])) for b in range(min(st[1], dhw[1])) for e in range(min(st[2], dhw[2]))}
    assert set(phases) <= with_pixels
    assert ("memset2d" in t) == (set(phases) != with_pixels)
    if st == (1, 1, 1):
        assert len(gemms) == 1 and gemms[0].startswith("conv3d_bf16_")
    else:
        assert all(nm.startswith("conv3d_dgrad_") for nm in gemms)


def test_one_by_one_stride_two_plans_the_memset(plan):
    rc, t = plan.dgrad([2, 8, 8, 8, 64], [128, 1, 1, 1, 64], stride=2)
    assert rc == 0, t
    assert t.count("conv3d dgrad phase") == 1 and t.count("memset2d") == 1 and "memset2d esz=2 cols=64 rows=1024" in t, t
    assert "conv3d dgrad phase r=(0,0,0) taps_d=0 taps_h=0 taps_w=0 dil=(1,1,1) lower=(0,0,0) upper=(0,0,0) extent=(4,4,4)" in t, t


# ---------------------------------------------------------------------------------------------- limits and refusals
def _err():
    return _ffi.load().b200_last_error().decode()


@pytest.mark.parametrize("pad,ok", [(16, True), (17, False)])
def test_padding_corner_boundary(plan, pad, ok):
    rc, _ = plan.fwd([1, 40, 40, 40, 16], [16, 33, 1, 1, 16], pad=(pad, 0, 0)) if pad == 16 else plan.fwd([1, 40, 40, 40, 16], [16, 1, 1, 1, 16], pad=(pad, 0, 0))
    if ok:
        assert rc == UNSUPPORTED and "offset" in _err()   # 16 - (33 - 1) = -16 is a valid corner, but offset 32 > 31
        rc, _ = plan.fwd([1, 40, 40, 40, 16], [16, 3, 1, 1, 16], pad=(pad, 0, 0))
        assert rc == 0, _err()
    else:
        assert rc == UNSUPPORTED and "corner" in _err(), _err()


@pytest.mark.parametrize("k,ok", [(17, True), (18, False)])
def test_upper_corner_boundary(plan, k, ok):
    # p - d (K - 1) = 0 - (K - 1): -16 accepted, -17 refused
    rc, _ = plan.fwd([1, 20, 20, 40, 16], [16, 1, 1, k, 16])
    assert (rc == 0) == ok, _err()
    if not ok:
        assert rc == UNSUPPORTED and "corner" in _err(), _err()
    rc, _ = plan.wgrad([1, 20, 20, 40, 16], [16, 1, 1, k, 16])
    assert (rc == 0) == ok and (ok or "corner" in _err()), _err()


def test_dgrad_phase_corners_are_checked(plan):
    rc, _ = plan.dgrad([1, 8, 8, 40, 16], [16, 1, 1, 17, 16])
    assert rc == 0, _err()
    rc, _ = plan.dgrad([1, 8, 8, 40, 16], [16, 1, 1, 18, 16])
    assert rc == UNSUPPORTED and "corner" in _err(), _err()


@pytest.mark.parametrize("case,status", [
    ("stride_9", UNSUPPORTED), ("f32_input", UNSUPPORTED), ("i8_input", UNSUPPORTED), ("bf16_to_f16", UNSUPPORTED),
    ("channel_mismatch", INVALID), ("bad_out_shape", INVALID), ("zero_stride", INVALID), ("too_many_pixels", UNSUPPORTED),
    ("out_channel_stride", UNSUPPORTED),
])
def test_refusals(plan, case, status):
    xs, ws, kw = [1, 6, 8, 8, 16], [32, 3, 3, 3, 16], {}
    if case == "stride_9":
        kw["stride"] = (9, 1, 1)
    elif case == "f32_input":
        kw["idt"] = kw["odt"] = F32
    elif case == "i8_input":
        kw["idt"] = I8
    elif case == "bf16_to_f16":
        kw["odt"] = F16
    elif case == "channel_mismatch":
        ws = [32, 3, 3, 3, 8]
        kw["os_"] = [1, 4, 6, 6, 32]
    elif case == "bad_out_shape":
        kw["os_"] = [1, 5, 6, 6, 32]
    elif case == "zero_stride":
        kw.update(stride=(0, 1, 1), os_=[1, 4, 6, 6, 32])
    elif case == "too_many_pixels":
        xs, ws = [1 << 13, 64, 64, 64, 16], [32, 1, 1, 1, 16]
    elif case == "out_channel_stride":
        kw["strides"] = (None, None, [4 * 6 * 6 * 64, 6 * 6 * 64, 6 * 64, 64, 2])
    rc, _ = plan.fwd(xs, ws, **kw)
    assert rc == status, (case, rc, _err())
    if case == "stride_9":
        assert "stride" in _err()
        rc, _ = plan.dgrad(xs, ws, stride=(1, 9, 1))
        assert rc == UNSUPPORTED


def test_wrong_rank_is_invalid_in_python():
    from cubecl_b200.conv import ConvShapeError
    with pytest.raises(ConvShapeError):
        conv3d.calculate_conv3d_output([1, 8, 8, 16], [32, 3, 3, 16])


def test_zero_extents_plan_no_launch(plan):
    rc, t = plan.fwd([0, 4, 8, 8, 16], [32, 3, 3, 3, 16], os_=[0, 2, 6, 6, 32])
    assert rc == 0 and _names(t) == []
    rc, t = plan.fwd([1, 4, 8, 8, 16], [0, 3, 3, 3, 16], os_=[1, 2, 6, 6, 0])
    assert rc == 0 and _names(t) == []
    # the gradients' zero fills: Cout = 0 writes dx as zeros, N = 0 in dy writes dw as zeros
    rc, t = plan.dgrad([1, 4, 8, 8, 16], [0, 3, 3, 3, 16])
    assert rc == 0 and _names(t) == [] and t.count("memset2d") == 1, t
    rc, t = plan.wgrad([0, 4, 8, 8, 16], [32, 3, 3, 3, 16])
    assert rc == 0 and _names(t) == [] and "memset2d esz=2 cols=16 rows=864" in t, t


# ---------------------------------------------------------------------------------------------- kernels
def test_conv3d_cubin_has_the_kernel_set_and_5d_im2col_loads():
    tool = _tool("cuobjdump")
    _ffi.load()
    cubin = ROOT / "cubecl_b200" / "build" / "gemm_conv3d.cubin"
    out = subprocess.run([tool, "-res-usage", str(cubin)], capture_output=True, text=True, check=True).stdout
    funcs = re.findall(r"Function (\w+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)
    want = {f"conv3d_{pfx}{i}_{o}_{t}" for pfx in ("", "dgrad_", "wgrad_") for i, o in (("bf16", "bf16"), ("bf16", "f32"), ("f16", "f16"),
                                                                                       ("f16", "f32")) for t in ("2sm_n128", "1sm_n128")}
    assert {f for f, *_ in funcs} == want
    for name, _, stack, local in funcs:
        assert int(stack) == 0 and int(local) == 0, (name, stack, local)
    sass = subprocess.run([tool, "-sass", str(cubin)], capture_output=True, text=True, check=True).stdout
    for body in re.split(r"\n\s*Function : ", sass)[1:]:
        name = body.split()[0]
        assert "HGMMA.64x128x16.F32" in body, name
        assert "UTMALDG.5D.IM2COL" in body, name
