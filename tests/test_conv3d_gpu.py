"""GPU: b200_conv3d and its gradients -- integer-valued operands bit for bit (rne of the f64 result) on both tiles, both store
paths and with the stream-K head on and off; D = KD = 1 bit-identical to b200_conv2d and its gradients; the reference's
im2col known-answer test through the 5-D path; uniform operands against the f64 oracle at the repository's bounds over
anisotropic kernels, strides, padding and dilations; a full layer against torch's GPU conv3d; views; the fused epilogue;
determinism; deferred errors."""
import contextlib

import numpy as np
import pytest
import torch

import conv3d_oracle as o3
import conv_oracle as co
import gemm_exact_oracle as ge
from cubecl_b200 import ServerError, TensorHandle, conv, conv3d, synth

pytestmark = pytest.mark.gpu

TOL = {"bf16": 1e-2, "f16": 1e-2, "f32": 1e-5}
DEFAULTS = {"gemm.variant": "auto", "gemm.epilogue": "tma", "gemm.split_k": "auto"}


@contextlib.contextmanager
def options(client, **kw):
    try:
        for k, v in kw.items():
            client.set_option(k.replace("_", ".", 1), v)
        yield
    finally:
        for k in kw:
            key = k.replace("_", ".", 1)
            client.set_option(key, DEFAULTS[key])


def up(client, vals, dtype):
    return TensorHandle.from_numpy(client, synth.to_device_dtype(np.asarray(vals, np.float32), dtype), dtype)


def bits(client, t):
    return np.asarray(t.to_numpy(client)).view(ge.OUT_BITS_VIEW[t.dtype])


def values(client, t):
    return synth.from_device_dtype(np.asarray(t.to_numpy(client)), t.dtype).reshape(t.shape).astype(np.float64)


def rounded(vals, dtype):
    """vals rounded to dtype and back (the operand values the GPU sees)"""
    return synth.from_device_dtype(synth.to_device_dtype(np.asarray(vals, np.float32), dtype), dtype).reshape(np.shape(vals)).astype(np.float64)


def run(client, which, geom, vals, dtype, od):
    """one pass; returns the output handle.  geom = (xs, cout, k, s, p, d)"""
    xs, cout, k, s, p, d = geom
    if which == "fwd":
        return conv3d.launch_alloc(client, up(client, vals["x"], dtype), up(client, vals["w"], dtype), od, stride=s, padding=p, dilation=d)
    if which == "dgrad":
        return conv3d.backward_data_alloc(client, up(client, vals["dy"], dtype), up(client, vals["w"], dtype), xs[1:4], od, stride=s,
                                          padding=p, dilation=d)
    return conv3d.backward_weight_alloc(client, up(client, vals["x"], dtype), up(client, vals["dy"], dtype), k, od, stride=s, padding=p,
                                        dilation=d)


def exact(which, geom, vals):
    xs, cout, k, s, p, d = geom
    if which == "fwd":
        return o3.conv3d_f64(vals["x"], vals["w"], s, p, d)
    if which == "dgrad":
        return o3.conv3d_input_grad_f64(vals["dy"], vals["w"], xs[1:4], s, p, d)
    return o3.conv3d_weight_grad_f64(vals["x"], vals["dy"], k, s, p, d)


def int_values(geom, seed, bound=8):
    xs, cout, k, s, p, d = geom
    o = o3.out_dhw(xs[1:4], k, s, p, d)
    vals = {"x": ge.int_values(xs, bound, seed), "w": ge.int_values((cout, *k, xs[4]), bound, seed + 1),
            "dy": ge.int_values((xs[0], *o, cout), bound, seed + 2)}
    for which in ("fwd", "dgrad", "wgrad"):
        ge.assert_exact_bound(exact(which, geom, {kk: np.abs(v) for kk, v in vals.items()})[0])
    return vals


# (x shape, Cout, kernel, stride, padding, dilation): stride 1 (dgrad = one forward GEMM) and phased dgrad
EXACT_GEOMS = [((2, 6, 10, 12, 64), 96, (3, 3, 3), 1, 1, 1), ((1, 7, 12, 10, 72), 130, (3, 3, 3), (2, 2, 1), (1, 1, 1), 1),
               ((2, 5, 9, 9, 32), 64, (1, 3, 3), (1, 2, 2), (0, 2, 1), (1, 1, 2))]
PATHS = [{"gemm_variant": "2sm_n128"}, {"gemm_variant": "1sm_n128"}, {"gemm_epilogue": "direct"}, {"gemm_split_k": "on"},
         {"gemm_split_k": "off"}]


@pytest.mark.parametrize("path", PATHS, ids=lambda p: "-".join(f"{k}={v}" for k, v in p.items()))
@pytest.mark.parametrize("od", ["bf16", "f32"])
@pytest.mark.parametrize("which", ["fwd", "dgrad", "wgrad"])
def test_integer_operands_are_exact(client, which, od, path):
    for i, geom in enumerate(EXACT_GEOMS):
        vals = int_values(geom, 10 * i)
        with options(client, **path):
            out = run(client, which, geom, vals, "bf16", od)
            client.sync()
            kernel = client.last_kernel()
        ge.assert_exact(bits(client, out), exact(which, geom, vals)[0], od, f"{which} {geom} {path} {kernel}")
        if "gemm_variant" in path:
            assert kernel.endswith(path["gemm_variant"]), kernel


def test_integer_f16_is_exact(client):
    geom = EXACT_GEOMS[1]
    vals = int_values(geom, 77)
    for which in ("fwd", "dgrad", "wgrad"):
        out = run(client, which, geom, vals, "f16", "f16")
        client.sync()
        ge.assert_exact(bits(client, out), exact(which, geom, vals)[0], "f16", which)


# ---------------------------------------------------------------------------------------------- D = KD = 1 is conv2d
@pytest.mark.parametrize("variant", ["2sm_n128", "1sm_n128"])
@pytest.mark.parametrize("s,p,d", [(1, 1, 1), (2, 1, 1), ((1, 2), (2, 0), (1, 2))])
def test_depth_one_is_bit_identical_to_conv2d(client, variant, s, p, d):
    rng = np.random.default_rng(5)
    n, h, w, c, cout, k = 2, 15, 13, 72, 80, 3
    x = rng.uniform(-1, 1, (n, h, w, c))
    wt = rng.uniform(-1, 1, (cout, k, k, c))
    oh, ow = co.out_hw(h, w, k, k, s, p, d)
    dy = rng.uniform(-1, 1, (n, oh, ow, cout))
    s2, p2, d2 = co.pair(s), co.pair(p), co.pair(d)
    s3, p3, d3 = (1, *s2), (0, *p2), (1, *d2)
    with options(client, gemm_variant=variant):
        x2, w2, dy2 = up(client, x, "bf16"), up(client, wt, "bf16"), up(client, dy, "bf16")
        x3, w3, dy3 = up(client, x[:, None], "bf16"), up(client, wt[:, None], "bf16"), up(client, dy[:, None], "bf16")
        pairs = [(conv.launch_alloc(client, x2, w2, "f32", stride=s2, padding=p2, dilation=d2),
                  conv3d.launch_alloc(client, x3, w3, "f32", stride=s3, padding=p3, dilation=d3)),
                 (conv.backward_data_alloc(client, dy2, w2, (h, w), "bf16", stride=s2, padding=p2, dilation=d2),
                  conv3d.backward_data_alloc(client, dy3, w3, (1, h, w), "bf16", stride=s3, padding=p3, dilation=d3)),
                 (conv.backward_weight_alloc(client, x2, dy2, (k, k), "f32", stride=s2, padding=p2, dilation=d2),
                  conv3d.backward_weight_alloc(client, x3, dy3, (1, k, k), "f32", stride=s3, padding=p3, dilation=d3))]
        client.sync()
    for i, (a, b) in enumerate(pairs):
        ga, gb = bits(client, a), bits(client, b)
        assert np.array_equal(ga.reshape(-1), gb.reshape(-1)), f"pass {i}: conv3d with D = 1 differs from conv2d"


@pytest.mark.parametrize("dtype", ["bf16", "f16"])
def test_im2col_kat_through_conv3d(client, dtype):
    """The reference's test_tensormap_load_im2col (tests/golden/conv_golden.json) through b200_conv3d with D = KD = 1."""
    x, w, exp, kat = co.im2col_kat()
    out = conv3d.launch_alloc(client, up(client, x[:, None], dtype), up(client, w[:, None], dtype), dtype, padding=(0, kat["pad_h"], kat["pad_w"]))
    client.sync()
    got = values(client, out)[:, 0]
    assert np.array_equal(got, exp)


# ---------------------------------------------------------------------------------------------- random operands
SWEEP = [((2, 6, 14, 14, 64), 64, (3, 3, 3), 1, 1, 1), ((1, 8, 20, 20, 16), 64, (3, 7, 7), (1, 2, 2), (1, 3, 3), 1),
         ((2, 5, 12, 12, 64), 96, (1, 3, 3), 1, (0, 1, 1), 1), ((1, 9, 11, 13, 40), 48, (3, 3, 3), (2, 3, 1), (2, 0, 3), (1, 2, 2)),
         ((2, 7, 9, 9, 128), 72, (2, 3, 3), 3, 1, 2), ((1, 6, 10, 10, 24), 130, (3, 1, 3), (1, 1, 2), (1, 0, 1), (2, 1, 1))]


@pytest.mark.parametrize("dtype,od", [("bf16", "bf16"), ("f16", "f16"), ("bf16", "f32"), ("f16", "f32")])
@pytest.mark.parametrize("which", ["fwd", "dgrad", "wgrad"])
def test_random_operands_within_bounds(client, which, dtype, od):
    for i, geom in enumerate(SWEEP):
        xs, cout, k, s, p, d = geom
        rng = np.random.default_rng(i)
        o = o3.out_dhw(xs[1:4], k, s, p, d)
        vals = {"x": rounded(rng.uniform(-1, 1, xs), dtype), "w": rounded(rng.uniform(-1, 1, (cout, *k, xs[4])), dtype),
                "dy": rounded(rng.uniform(-1, 1, (xs[0], *o, cout)), dtype)}
        out = run(client, which, geom, vals, dtype, od)
        client.sync()
        ref, aref = exact(which, geom, vals)
        got = values(client, out)
        err = float(np.max(np.abs(got - ref) / np.maximum(aref, 1e-30)))
        assert err <= TOL[od], f"{which} {geom}: {err:.3e}"


def test_full_layer_against_torch_gpu(client):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    n, dd, h, w, c, cout = 4, 8, 28, 28, 128, 128
    g = torch.Generator().manual_seed(3)
    x = torch.randn(n, c, dd, h, w, generator=g).bfloat16().float()
    wt = (torch.randn(cout, c, 3, 3, 3, generator=g) * 0.05).bfloat16().float()
    dy = torch.randn(n, cout, dd, h, w, generator=g).bfloat16().float()
    xg, wg = x.cuda().requires_grad_(True), wt.cuda().requires_grad_(True)
    yg = torch.nn.functional.conv3d(xg, wg, padding=1)
    yg.backward(dy.cuda())
    nd = lambda t: np.moveaxis(t.detach().cpu().numpy().astype(np.float64), 1, -1)  # noqa: E731
    xv, wv, dyv = nd(x), nd(wt), nd(dy)
    y3 = conv3d.launch_alloc(client, up(client, xv, "bf16"), up(client, wv, "bf16"), "f32", padding=1)
    dx3 = conv3d.backward_data_alloc(client, up(client, dyv, "bf16"), up(client, wv, "bf16"), (dd, h, w), "f32", padding=1)
    dw3 = conv3d.backward_weight_alloc(client, up(client, xv, "bf16"), up(client, dyv, "bf16"), (3, 3, 3), "f32", padding=1)
    client.sync()
    _, ay = o3.conv3d_f64(xv[:1], wv, 1, 1, 1)
    for got, want, scale in ((y3, yg, float(ay.max())), (dx3, xg.grad, None), (dw3, wg.grad, None)):
        g64, w64 = values(client, got), nd(want)
        tol = 1e-4 * (scale or float(np.abs(w64).max()))
        assert float(np.max(np.abs(g64 - w64))) <= tol


# ---------------------------------------------------------------------------------------------- views, epilogue, errors
def test_views(client):
    rng = np.random.default_rng(9)
    n, dd, h, w, c, cout = 2, 5, 9, 10, 64, 80
    x = rounded(rng.uniform(-1, 1, (n, dd, h, w, c)), "bf16")
    wt = rounded(rng.uniform(-1, 1, (cout, 3, 3, 3, c)), "bf16")
    want, aref = o3.conv3d_f64(x, wt, 1, 1, 1)
    # NCDHW x and OIDHW w as stride-permuted views
    xn = up(client, np.moveaxis(x, -1, 1), "bf16")
    wn = up(client, np.moveaxis(wt, -1, 1), "bf16")
    xv = TensorHandle(xn.handle, [n, dd, h, w, c], [c * dd * h * w, h * w, w, 1, dd * h * w], "bf16")
    wv = TensorHandle(wn.handle, [cout, 3, 3, 3, c], [c * 27, 9, 3, 1, 27], "bf16")
    # out as a channel slice [64, 64 + Cout) of a 64 + Cout + 64 channel tensor
    full = TensorHandle.empty_contiguous(client, [n, dd, h, w, cout + 128], "f32")
    out = TensorHandle(full.handle.offset(64 * 4), [n, dd, h, w, cout], full.strides, "f32")
    conv3d.launch(client, xv, wv, out, padding=1)
    client.sync()
    got = np.asarray(full.to_numpy(client))[..., 64:64 + cout].astype(np.float64)
    assert float(np.max(np.abs(got - want) / aref)) <= TOL["f32"]
    # a C = 3 stem (channels padded to 8) and a misaligned x base (gathered)
    xs = rounded(rng.uniform(-1, 1, (1, 6, 20, 20, 3)), "bf16")
    ws = rounded(rng.uniform(-1, 1, (64, 3, 7, 7, 3)), "bf16")
    y = conv3d.launch_alloc(client, up(client, xs, "bf16"), up(client, ws, "bf16"), "f32", stride=(1, 2, 2), padding=(1, 3, 3))
    buf = up(client, np.concatenate([np.zeros(1), x.reshape(-1)]), "bf16")
    xm = TensorHandle(buf.handle.offset(2), list(x.shape), [dd * h * w * c, h * w * c, w * c, c, 1], "bf16")
    ym = conv3d.launch_alloc(client, xm, up(client, wt, "bf16"), "f32", padding=1)
    client.sync()
    ref, aref2 = o3.conv3d_f64(xs, ws, (1, 2, 2), (1, 3, 3), 1)
    assert float(np.max(np.abs(values(client, y) - ref) / aref2)) <= TOL["f32"]
    assert float(np.max(np.abs(values(client, ym) - want) / aref)) <= TOL["f32"]


@pytest.mark.parametrize("act", ["relu", "gelu"])
def test_fused_epilogue(client, act):
    rng = np.random.default_rng(11)
    x = rounded(rng.uniform(-1, 1, (2, 4, 8, 8, 64)), "bf16")
    wt = rounded(rng.uniform(-1, 1, (96, 3, 3, 3, 64)), "bf16")
    bias = rng.uniform(-1, 1, 96).astype(np.float32)
    b = TensorHandle.from_numpy(client, bias, "f32")
    out = conv3d.launch_alloc(client, up(client, x, "bf16"), up(client, wt, "bf16"), "f32", padding=1, alpha=0.5, bias=b, activation=act)
    client.sync()
    ref, aref = o3.conv3d_f64(x, wt, 1, 1, 1)
    ref = 0.5 * ref + bias
    ref = np.maximum(ref, 0) if act == "relu" else np.asarray(torch.nn.functional.gelu(torch.from_numpy(ref)))
    assert float(np.max(np.abs(values(client, out) - ref) / (0.5 * aref + np.abs(bias)))) <= TOL["f32"]


def test_two_runs_give_identical_bits(client):
    geom = ((2, 8, 14, 14, 64), 64, (3, 3, 3), (1, 2, 2), 1, 1)
    rng = np.random.default_rng(13)
    o = o3.out_dhw(geom[0][1:4], geom[2], geom[3], geom[4], geom[5])
    vals = {"x": rng.uniform(-1, 1, geom[0]), "w": rng.uniform(-1, 1, (64, 3, 3, 3, 64)), "dy": rng.uniform(-1, 1, (2, *o, 64))}
    for which in ("fwd", "dgrad", "wgrad"):
        a, b = run(client, which, geom, vals, "bf16", "f32"), run(client, which, geom, vals, "bf16", "f32")
        client.sync()
        assert np.array_equal(bits(client, a), bits(client, b)), which


def test_errors_are_deferred_to_sync(client):
    x = TensorHandle.empty_contiguous(client, [1, 4, 8, 8, 16], "bf16")
    w = TensorHandle.empty_contiguous(client, [16, 3, 3, 3, 8], "bf16")          # channel mismatch
    out = TensorHandle.empty_contiguous(client, [1, 2, 6, 6, 16], "bf16")
    conv3d.launch(client, x, w, out)                                            # returns: the error waits for sync()
    with pytest.raises(ServerError) as e:
        client.sync()
    assert [err.status for err in e.value.errors] == [6] and "channels" in str(e.value)
    w = TensorHandle.empty_contiguous(client, [16, 3, 3, 3, 16], "bf16")
    out = TensorHandle.empty_contiguous(client, [1, 1, 6, 6, 16], "bf16")
    conv3d.launch(client, x, w, out, stride=(9, 1, 1))
    with pytest.raises(ServerError) as e:
        client.sync()
    assert [err.status for err in e.value.errors] == [7] and "stride" in str(e.value)
