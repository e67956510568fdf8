"""CPU: the f64 transposed-convolution oracle (pinned to torch.nn.functional.conv_transpose2d / 3d), the output rule, the
dry-run plans of b200_conv_transpose2d / 3d (stride 1 on the forward kernel, every stride phase in phase-batched launches,
no memset), the output rebuilt from the plan's phase lines alone, the longest-first phase order, every refusal, the
zero-extent rules, and the SASS of the phase-batched kernels."""
import ctypes as C
import itertools
import re
import subprocess

import numpy as np
import pytest
import torch

import conv_transpose_oracle as cto
from cubecl_b200 import _ffi
from cubecl_b200.conv_transpose import calculate_conv_transpose_output
from plan_context import PlanContext
from test_conv_cpu import ROOT, _tool

F32, F16, BF16, I8 = _ffi.F32, _ffi.F16, _ffi.BF16, _ffi.I8
X, W, OUT = 0x10000000, 0x20000000, 0x40000000
INVALID, UNSUPPORTED = 6, 7


def _torch(x, w, s, p, op, d, bias=None):
    """torch's transposed convolution in float64 on channels-last numpy operands ([Cin, *k, Cout] weights)"""
    n = x.ndim - 2
    xt = torch.from_numpy(np.ascontiguousarray(np.moveaxis(x, -1, 1)))
    wt = torch.from_numpy(np.ascontiguousarray(np.moveaxis(w, -1, 1)))
    bt = None if bias is None else torch.from_numpy(np.asarray(bias, dtype=np.float64))
    f = torch.nn.functional.conv_transpose3d if n == 3 else torch.nn.functional.conv_transpose2d
    return np.moveaxis(f(xt, wt, bt, stride=s, padding=p, output_padding=op, dilation=d).numpy(), 1, -1)


def _geometries(seed, count, n):
    """seeded random (x shape, w shape, stride, padding, output_padding, dilation) with a valid output: kernels 1-7,
    strides 1-4, output_padding any value in [0, stride)"""
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < count:
        k = tuple(int(v) for v in rng.integers(1, 8 if n == 2 else 5, n))
        s = tuple(int(v) for v in rng.integers(1, 5, n))
        d = tuple(int(v) for v in rng.integers(1, 4, n))
        p = tuple(int(v) for v in rng.integers(0, 4, n))
        op = tuple(int(rng.integers(0, si)) for si in s)
        xs = [2, *(int(v) for v in rng.integers(1, 7 if n == 2 else 4, n)), 3]
        ws = [3, *k, 5]
        if min(cto.output_shape(xs, ws, s, p, op, d)[1:-1]) < 1:
            continue
        out.append((xs, ws, s, p, op, d))
    return out


# ---------------------------------------------------------------------------------------------- oracle
@pytest.mark.parametrize("geom", _geometries(11, 60, 2) + _geometries(12, 25, 3))
def test_oracle_matches_torch(geom):
    xs, ws, s, p, op, d = geom
    rng = np.random.default_rng(sum(xs) * 7 + sum(ws))
    x, w, b = rng.uniform(-1, 1, xs), rng.uniform(-1, 1, ws), rng.uniform(-1, 1, ws[-1])
    for bias in (None, b):
        got, aout = cto.conv_transpose_f64(x, w, s, p, op, d, bias)
        np.testing.assert_allclose(got, _torch(x, w, s, p, op, d, bias), rtol=0, atol=1e-12 * max(1.0, float(aout.max())))


@pytest.mark.parametrize("geom", _geometries(13, 30, 2) + _geometries(14, 15, 3))
def test_output_rule_matches_torch(geom):
    xs, ws, s, p, op, d = geom
    x, w = np.zeros(xs), np.zeros(ws)
    assert calculate_conv_transpose_output(xs, ws, s, p, op, d) == list(_torch(x, w, s, p, op, d).shape)


# ---------------------------------------------------------------------------------------------- dry-run plans
class Planner(PlanContext):
    def run(self, xs, ws, s=1, p=0, op=0, d=1, outs=None, idt=BF16, odt=BF16, strides=(None, None, None), ptrs=(X, W, OUT), ep=None):
        n = len(xs) - 2
        if outs is None:
            outs = cto.output_shape(xs, ws, s, p, op, d)
        t = lambda v: cto._tuple(v, n)  # noqa: E731
        args = (_ffi.Conv3dArgs if n == 3 else _ffi.Conv2dArgs)(*t(s), *t(p), *t(d))
        fn = self.lib.b200_conv_transpose3d if n == 3 else self.lib.b200_conv_transpose2d
        arr = lambda v: _ffi.u64_array(v) if v is not None else None  # noqa: E731
        rc = fn(self.ctx, None, idt, odt, ptrs[0], arr(xs), arr(strides[0]), ptrs[1], arr(ws), arr(strides[1]), ptrs[2], arr(outs),
                arr(strides[2]), C.byref(args), C.byref(ep) if ep is not None else None)
        return rc, self.text()


@pytest.fixture
def plan():
    with Planner() as p:
        yield p


def _names(t):
    return [ln.split()[1] for ln in t.splitlines() if ln.startswith("launch ")]


_PHASE = re.compile(r"conv(3d)? tconv phase r=\(([\d,]+)\)((?: taps_[dhw]=[\d,]*)+) dil=\(([\d,]+)\) lower=\(([-\d,]+)\) "
                    r"upper=\(([-\d,]+)\) extent=\(([\d,]+)\) kblocks=(\d+)")


def _phases(t):
    """the plan's phase lines: (residue, taps per dimension in walk order, dilation, lower, upper, extent, k-blocks)"""
    out = []
    for m in _PHASE.finditer(t):
        ints = lambda g: tuple(int(v) for v in g.split(","))  # noqa: E731
        taps = tuple(tuple(int(v) for v in grp.split("=")[1].split(",") if v) for grp in m.group(3).split())
        out.append((ints(m.group(2)), taps, ints(m.group(4)), ints(m.group(5)), ints(m.group(6)), ints(m.group(7)), int(m.group(8))))
    return out


def _rebuild_from_plan(t, x, w, out_shape, s):
    """out rebuilt from the phase lines alone: phase r is the stride-1 correlation of x over its taps (walk order, `dil`
    apart, from x offset `lower`) written to out[r::s] over `extent` pixels.  Pixels of phases not listed stay NaN."""
    n = x.ndim - 2
    s = cto._tuple(s, n)
    out = np.full(out_shape, np.nan)
    I = x.shape[1:1 + n]
    for r, taps, dil, lower, upper, extent, kb in _phases(t):
        for i in range(n):
            assert upper[i] == lower[i] + extent[i] - I[i]   # the walk covers exactly the phase extent
        ph = np.zeros((x.shape[0], *extent, w.shape[-1]))
        for tt in itertools.product(*(range(len(tp)) for tp in taps)):
            k = tuple(taps[i][tt[i]] for i in range(n))
            for px in itertools.product(*(range(e) for e in extent)):
                src = tuple(px[i] + lower[i] + tt[i] * dil[i] for i in range(n))
                if all(0 <= src[i] < I[i] for i in range(n)):
                    ph[(slice(None),) + px] += x[(slice(None),) + src] @ w[(slice(None),) + k]
        dst = (slice(None),) + tuple(slice(r[i], r[i] + s[i] * extent[i], s[i]) for i in range(n))
        out[dst] = ph
    return out


@pytest.mark.parametrize("geom", _geometries(21, 30, 2) + _geometries(22, 10, 3))
def test_output_rebuilt_from_the_plan_matches_the_oracle(plan, geom):
    xs, ws, s, p, op, d = geom
    rc, t = plan.run(xs, ws, s, p, op, d)
    assert rc == 0, (t, _ffi.load().b200_last_error())
    rng = np.random.default_rng(len(t))
    x, w = rng.uniform(-1, 1, xs), rng.uniform(-1, 1, ws)
    want, _ = cto.conv_transpose_f64(x, w, s, p, op, d)
    got = _rebuild_from_plan(t, x, w, want.shape, s)
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-10)   # NaN anywhere: a pixel no phase line covers
    names = _names(t)
    assert "memset" not in t
    assert names[0] == "conv_dgrad_weights" or names[0] == "conv3d_dgrad_weights" or names[0] == "repitch_rows"
    n = len(xs) - 2
    phases = _phases(t)
    # every phase with pixels is listed once; at most 8 per batched launch, most k-blocks first
    assert len({ph[0] for ph in phases}) == len(phases) == int(np.prod([min(si, oi) for si, oi in zip(cto._tuple(s, n), want.shape[1:-1])]))
    kbs = [ph[-1] for ph in phases]
    assert kbs == sorted(kbs, reverse=True)
    batched = [nm for nm in names if "_tconv_" in nm]
    if all(v == 1 for v in cto._tuple(s, n)):
        assert not batched and re.match(rf"conv{n}d_bf16_bf16_(2sm|1sm)_n128$", names[-1]), names
    else:
        assert len(batched) == (len(phases) + 7) // 8 and batched == names[-len(batched):], names


def test_stride_one_is_prep_and_one_forward_launch(plan):
    rc, t = plan.run([8, 28, 28, 128], [128, 3, 3, 64], p=1)
    assert rc == 0, t
    assert _names(t)[0] == "conv_dgrad_weights" and len(_names(t)) == 2
    assert re.match(r"conv2d_bf16_bf16_(2sm_n128|1sm_n128)$", _names(t)[1]), t
    assert "memset" not in t and t.count("conv tconv phase") == 1
    rc, t = plan.run([2, 8, 8, 8, 64], [64, 3, 3, 3, 32], p=1)
    assert rc == 0 and _names(t)[0] == "conv3d_dgrad_weights" and re.match(r"conv3d_bf16_bf16_(2sm|1sm)_n128$", _names(t)[1]), t
    assert len(_names(t)) == 2


def test_stride_two_is_prep_and_one_batched_launch(plan):
    # U-Net decoder 2x2 / 2: four phases of one tap each
    rc, t = plan.run([8, 28, 28, 128], [128, 2, 2, 128], s=2)
    assert rc == 0, t
    assert _names(t) == ["conv_dgrad_weights", _names(t)[1]] and re.match(r"conv2d_tconv_bf16_bf16_(2sm|1sm)_n128$", _names(t)[1]), t
    assert len(_phases(t)) == 4 and "memset" not in t
    # 3x3 / 2 with output_padding 1: phases of 4, 2, 2 and 1 taps, longest first
    rc, t = plan.run([8, 28, 28, 128], [128, 3, 3, 64], s=2, p=1, op=1, odt=F32)
    assert rc == 0 and len(_names(t)) == 2 and _names(t)[1].startswith("conv2d_tconv_bf16_f32_"), t
    assert [ph[-1] for ph in _phases(t)] == [8, 4, 4, 2]
    assert _phases(t)[0][0] == (1, 1) and "memset" not in t
    # 1x1 / 2: three of the four phases have no tap -- still one launch, no memset
    rc, t = plan.run([8, 28, 28, 256], [256, 1, 1, 128], s=2, op=1)
    assert rc == 0 and len(_names(t)) == 2 and "_tconv_" in _names(t)[1] and "memset" not in t, t
    assert [ph[-1] for ph in _phases(t)] == [4, 0, 0, 0]
    # 3-D stride 2 in every dimension: eight phases in one launch
    rc, t = plan.run([1, 16, 16, 16, 64], [64, 2, 2, 2, 64], s=2)
    assert rc == 0 and _names(t)[0] == "conv3d_dgrad_weights" and len(_names(t)) == 2, t
    assert re.match(r"conv3d_tconv_bf16_bf16_(2sm|1sm)_n128$", _names(t)[1]) and len(_phases(t)) == 8, t
    rc, t = plan.run([1, 8, 8, 8, 64], [64, 1, 3, 3, 64], s=(1, 2, 2), p=(0, 1, 1), op=(0, 1, 1))
    assert rc == 0 and len(_names(t)) == 2 and "conv3d_tconv_" in _names(t)[1] and len(_phases(t)) == 4, t


def test_stride_three_is_two_batched_launches(plan):
    rc, t = plan.run([4, 16, 16, 64], [64, 3, 3, 64], s=3)
    assert rc == 0, t
    assert _names(t)[0] == "conv_dgrad_weights" and len(_names(t)) == 3 and all("_tconv_" in nm for nm in _names(t)[1:]), t
    assert len(_phases(t)) == 9 and "memset" not in t
    # stride 4 (16 phases) takes two launches too; a 1 x 1 kernel leaves 15 of them without taps
    rc, t = plan.run([4, 16, 16, 64], [64, 1, 1, 64], s=4)
    assert rc == 0 and len(_names(t)) == 3 and len(_phases(t)) == 16 and _phases(t)[0][-1] == 1, t


def test_no_input_channels_store_the_bias_alone(plan):
    ep = _ffi.Epilogue(1.0, 1, 0x50000000)
    rc, t = plan.run([2, 8, 8, 0], [0, 3, 3, 16], s=2, p=1, op=1, ep=ep)
    assert rc == 0, t
    assert len(_names(t)) == 1 and "_tconv_" in _names(t)[0] and all(ph[-1] == 0 for ph in _phases(t)), t
    rc, t = plan.run([2, 8, 8, 0], [0, 3, 3, 16], p=1)
    assert rc == 0 and len(_names(t)) == 1 and "_tconv_" in _names(t)[0], t


def test_data_gradient_plans_are_unchanged_by_the_shared_planning(plan):
    """the transposed convolution and the data gradient plan the same phases: same taps, dilation, corners and extents"""
    rc, tt = plan.run([2, 14, 14, 64], [64, 5, 5, 32], s=3, p=2, op=1, d=2)
    assert rc == 0, tt
    args = _ffi.Conv2dArgs(3, 3, 2, 2, 2, 2)
    u = _ffi.u64_array
    rc = plan.lib.b200_conv2d_backward_data(plan.ctx, None, BF16, BF16, X, u([2, 14, 14, 64]), None, W, u([64, 5, 5, 32]), None, OUT,
                                            u(cto.output_shape([2, 14, 14, 64], [64, 5, 5, 32], 3, 2, 1, 2)), None, C.byref(args))
    td = plan.text()
    assert rc == 0, td
    dg = {m.group(1) for m in re.finditer(r"conv dgrad phase (r=.*)", td)}
    tc = {re.sub(r" kblocks=\d+", "", m.group(1)) for m in re.finditer(r"conv tconv phase (r=.*)", tt)}
    assert dg and dg <= tc and all("taps_h= " in ln or "taps_w= " in ln for ln in tc - dg)


@pytest.mark.parametrize("variant", ["2sm_n128", "1sm_n128"])
def test_forced_tiles_are_honoured(plan, variant):
    plan.option("gemm.variant", variant)
    rc, t = plan.run([8, 28, 28, 256], [256, 3, 3, 256], s=2, p=1, op=1, odt=F32)
    assert rc == 0 and all(nm.endswith(variant) for nm in _names(t)[1:]), t
    plan.option("gemm.variant", "2sm_n256")
    assert plan.run([8, 28, 28, 256], [256, 3, 3, 256], s=2, p=1, op=1)[0] == INVALID


@pytest.mark.parametrize("case,status,words", [
    ("output_padding_ge_stride", UNSUPPORTED, "output_padding"), ("output_padding_too_large", INVALID, "expected"),
    ("f32_input", UNSUPPORTED, "dtype"), ("i8_input", UNSUPPORTED, "dtype"), ("bf16_to_f16", UNSUPPORTED, "dtype"),
    ("corner_4d", UNSUPPORTED, "corner"), ("corner_5d", UNSUPPORTED, "corner"), ("offset_5d", UNSUPPORTED, "offset"),
    ("stride_9", UNSUPPORTED, "stride"), ("too_many_pixels", UNSUPPORTED, "2^31"), ("null_pointer", INVALID, "null"),
    ("channel_mismatch", INVALID, "channels"), ("out_layout", UNSUPPORTED, "unit channel stride"), ("activation", INVALID, "activation"),
])
def test_refusals(plan, case, status, words):
    xs, ws, kw = [1, 8, 8, 16], [16, 3, 3, 32], dict(s=2, p=1, op=1)
    if case == "output_padding_ge_stride":     # PyTorch takes op = 2 with stride 2 when dilation is 3
        kw = dict(s=2, p=1, d=3, outs=[1, (8 - 1) * 2 - 2 + 3 * 2 + 1 + 2, (8 - 1) * 2 - 2 + 3 * 2 + 1, 32])
    elif case == "output_padding_too_large":
        kw["outs"] = [1, 17, 17, 32]
    elif case == "f32_input":
        kw.update(idt=F32, odt=F32)
    elif case == "i8_input":
        kw.update(idt=I8, odt=F32)
    elif case == "bf16_to_f16":
        kw["odt"] = F16
    elif case == "corner_4d":   # the phase's lower corner -(KH - 1) = -149 < -128
        xs, ws, kw = [1, 151, 8, 16], [16, 150, 1, 32], dict(s=1)
    elif case == "corner_5d":   # lower corner p - (K - 1) = 15, upper corner 15 + 1 - 33 = -17 < -16
        xs, ws, kw = [1, 33, 4, 4, 16], [16, 3, 1, 1, 32], dict(s=1, p=(17, 0, 0))
    elif case == "offset_5d":   # corners -16 and -16, but the im2col offset (3 - 1) * 16 = 32 > 31
        xs, ws, kw = [1, 8, 4, 4, 16], [16, 3, 1, 1, 32], dict(s=1, p=(16, 0, 0), d=(16, 1, 1))
    elif case == "stride_9":
        kw = dict(s=9)
    elif case == "too_many_pixels":
        xs, ws, kw = [1 << 17, 128, 128, 16], [16, 1, 1, 32], dict(s=1)
    elif case == "null_pointer":
        kw["ptrs"] = (X, 0, OUT)
    elif case == "channel_mismatch":   # out has 16 channels, w writes 32
        kw["outs"] = [1, 16, 16, 16]
    elif case == "out_layout":
        kw["strides"] = (None, None, [16 * 16 * 32 * 2, 16 * 32 * 2, 32 * 2, 2])
    elif case == "activation":
        kw["ep"] = _ffi.Epilogue(1.0, 7, 0)
    rc, t = plan.run(xs, ws, **kw)
    msg = _ffi.load().b200_last_error().decode()
    assert rc == status, (case, rc, msg, t)
    assert words in msg, msg


def test_zero_extents(plan):
    # empty output: no-op
    rc, t = plan.run([0, 8, 8, 16], [16, 3, 3, 32], s=2, p=1, op=1)
    assert rc == 0 and _names(t) == [] and "memset" not in t
    rc, t = plan.run([1, 8, 8, 16], [16, 3, 3, 0], s=2, p=1, op=1)
    assert rc == 0 and _names(t) == []
    rc, t = plan.run([0, 4, 4, 4, 16], [16, 2, 2, 2, 8], s=2)
    assert rc == 0 and _names(t) == []


# ---------------------------------------------------------------------------------------------- kernels
def test_batched_kernels_use_wgmma_and_im2col_tma_and_do_not_spill():
    tool = _tool("cuobjdump")
    _ffi.load()
    cubin = ROOT / "cubecl_b200" / "build" / "gemm_convt.cubin"
    out = subprocess.run([tool, "-res-usage", str(cubin)], capture_output=True, text=True, check=True).stdout
    funcs = re.findall(r"Function (\w+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)
    assert {f for f, *_ in funcs} == {f"conv{n}d_tconv_{i}_{o}_{t}" for n in (2, 3)
                                      for i, o in (("bf16", "bf16"), ("bf16", "f32"), ("f16", "f16"), ("f16", "f32"))
                                      for t in ("2sm_n128", "1sm_n128")}
    for name, reg, stack, local in funcs:
        assert int(stack) == 0 and int(local) == 0, (name, stack, local)
    sass = subprocess.run([tool, "-sass", str(cubin)], capture_output=True, text=True, check=True).stdout
    for body in re.split(r"\n\s*Function : ", sass)[1:]:
        name = body.split()[0]
        assert "HGMMA.64x128x16.F32" in body, name
        assert ("UTMALDG.5D.IM2COL" if name.startswith("conv3d_") else "UTMALDG.4D.IM2COL") in body, name


# ---------------------------------------------------------------------------------------------- empty kernels, options
@pytest.mark.parametrize("stride", [9, 1000])
def test_stride_limit_holds_for_empty_kernels(plan, stride):
    """an empty kernel takes no shape rule from the convolution, but the stride limit still holds (it bounds the per-phase
    tables the plan fills)"""
    for xs, ws in (([1, 2, 2, 2, 16], [16, 0, 1, 1, 32]), ([1, 2, 2, 16], [16, 0, 1, 32]), ([1, 2, 2, 2, 16], [16, 1, 1, 0, 32])):
        n = len(xs) - 2
        outs = [1, *([(2 - 1) * stride - 1 + 1 + 1] * n), 32]   # the transposed rule with K = 0 where it applies
        rc, t = plan.run(xs, ws, s=stride, outs=outs)
        msg = _ffi.load().b200_last_error().decode()
        assert rc == UNSUPPORTED and "stride" in msg, (xs, ws, rc, msg, t)
        assert _names(t) == []


def test_empty_kernel_stores_bias_under_the_transposed_output_rule(plan):
    ep = _ffi.Epilogue(1.0, 0, 0x50000000)
    # K = 0 in H: OH = (H - 1) * s - 2p + d * (0 - 1) + op + 1 = 7 * 2 - 0 - 1 + op + 1 = 14 + op
    for op in (0, 1):
        rc, t = plan.run([2, 8, 8, 16], [16, 0, 3, 24], s=2, outs=[2, 14 + op, 17, 24], ep=ep)
        assert rc == 0, (t, _ffi.load().b200_last_error())
        assert len(_names(t)) == 1 and "_tconv_" in _names(t)[0] and all(ph[-1] == 0 for ph in _phases(t)), t
    rc, t = plan.run([1, 2, 3, 3, 16], [16, 2, 0, 2, 8], s=2, outs=[1, 4, 4, 6, 8])
    assert rc == 0 and len(_names(t)) == 1 and "conv3d_tconv_" in _names(t)[0], (t, _ffi.load().b200_last_error())
    # extents outside the rule, another batch, or mismatched channels are refused
    for xs, ws, outs in (([2, 8, 8, 16], [16, 0, 3, 24], [2, 16, 17, 24]), ([2, 8, 8, 16], [16, 0, 3, 24], [2, 13, 17, 24]),
                         ([2, 8, 8, 16], [16, 0, 3, 24], [1, 14, 17, 24]), ([2, 8, 8, 16], [8, 0, 3, 24], [2, 14, 17, 24]),
                         ([1, 2, 3, 3, 16], [16, 2, 0, 2, 8], [1, 4, 7, 6, 8])):
        rc, t = plan.run(xs, ws, s=2, outs=outs)
        assert rc == INVALID and "empty kernel" in _ffi.load().b200_last_error().decode(), (xs, ws, outs, t)


def test_split_k_option_is_validated_and_plans_no_stream_k_head(plan):
    for v in ("auto", "off", "on", "3"):
        plan.option("gemm.split_k", v)
        rc, t = plan.run([8, 28, 28, 256], [256, 3, 3, 256], s=2, p=1, op=1)
        assert rc == 0 and "stream-k" not in t, (v, t)
    plan.option("gemm.split_k", "9")
    rc, t = plan.run([8, 28, 28, 256], [256, 3, 3, 256], s=2, p=1, op=1)
    assert rc == INVALID and "split_k" in _ffi.load().b200_last_error().decode()
