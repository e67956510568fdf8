"""GPU: GEMM and convolution outputs checked exactly (tests/gemm_exact_oracle.py).

Integer-valued operands make every f32 partial sum exact, so each tile, store path (TMA store, vectorised and scalar direct
stores), stream-K reduction and 16-bit conversion must give rne(exact) bit for bit; on random data a 16-bit output must be the
single RNE rounding of the same plan's f32 output.  Every case asserts, through a dry-run plan of the same call, which kernel,
store path and stream-K head it took, and tests/test_gemm_exact_cpu.py checks that the case lists below cover every path."""
import math

import numpy as np
import pytest

import conv_backward_oracle as cbo
import conv_oracle as co
import gemm_exact_oracle as ge
from cubecl_b200 import TensorHandle, conv, matmul, reduce, synth
from cubecl_b200.client import DTYPE_SIZE

pytestmark = pytest.mark.gpu

GEMM_OPTIONS = {"gemm.variant": "auto", "gemm.split_k": "auto", "gemm.epilogue": "tma", "gemm.group_m": 8, "gemm.f32": "hybrid"}
IN_FOR_OUT = {"bf16": "bf16", "f16": "f16", "f32": "bf16"}


@pytest.fixture(autouse=True)
def _reset_options(client):
    yield
    for k, v in GEMM_OPTIONS.items():
        client.set_option(k, v)


def _opts(**kw):
    return tuple(sorted((f"gemm.{k}", str(v)) for k, v in kw.items()))


# ------------------------------------------------------------------------------------------------ case lists
# Per variant, a ragged shape with more tiles than clusters: split_k "2" gives a stream-K head AND whole tiles.
VARIANT_SHAPES = {"2sm_n256": (2300, 2056, 200), "2sm_n128": (1300, 1544, 200), "1sm_n128": (1400, 1672, 200),
                  "2sm_m512": (1100, 1000, 200), "simt": (130, 90, 600)}
HEAD_VARIANTS = ("2sm_n256", "2sm_n128", "1sm_n128")


def _plan_grid():
    cases = []
    for variant, (M, N, K) in VARIANT_SHAPES.items():
        for epi in ("tma", "direct"):
            for split in (("off", "2") if variant in HEAD_VARIANTS else ("off",)):
                for od in ("f32", "bf16", "f16"):
                    cases.append(ge.GemmCase(f"{variant}-{epi}-sk{split}-{od}", IN_FOR_OUT[od], od, M, N, K,
                                             opts=_opts(variant=variant, epilogue=epi, split_k=split)))
    return cases


PLAN_GRID = _plan_grid()

LAYOUT_CASES = [
    ge.GemmCase("batched-bf16", "bf16", "bf16", 300, 264, 136, batch=3),
    ge.GemmCase("bcast-f16", "f16", "f16", 300, 264, 136, batch=3, bcast=True),
    ge.GemmCase("lhs_t-bf16", "bf16", "bf16", 264, 200, 136, lhs_t=True),
    ge.GemmCase("rhs_t-f16", "f16", "f16", 264, 200, 136, rhs_t=True),
    ge.GemmCase("both_t-f32out", "bf16", "f32", 264, 200, 136, lhs_t=True, rhs_t=True),
    ge.GemmCase("window-bf16", "bf16", "bf16", 300, 264, 136, window=True),
    ge.GemmCase("window-batched-f16-direct", "f16", "f16", 300, 264, 136, batch=2, window=True, opts=_opts(epilogue="direct")),
    ge.GemmCase("window-f32-sk2", "bf16", "f32", 300, 264, 136, window=True, opts=_opts(split_k=2)),
    # N = 2 mod 8: 16-bit rows are not 16-byte multiples, so the scalar direct stores run (K-major rhs keeps B on TMA)
    ge.GemmCase("n2mod8-bf16", "bf16", "bf16", 200, 258, 128, rhs_t=True),
    ge.GemmCase("n2mod8-f16-sk2", "f16", "f16", 200, 258, 128, rhs_t=True, opts=_opts(split_k=2)),
    ge.GemmCase("groupm1-bf16", "bf16", "bf16", 1300, 1544, 200, opts=_opts(group_m=1, variant="2sm_n128")),
    ge.GemmCase("groupm8-f16", "f16", "f16", 1300, 1544, 200, opts=_opts(group_m=8, variant="2sm_n128")),
    # split_k auto where the model plans a head (8 tiles, long K); and 3 ranges per tile
    ge.GemmCase("skauto-bf16", "bf16", "bf16", 512, 512, 16384),
    ge.GemmCase("sk3-f16", "f16", "f16", 520, 392, 1000, opts=_opts(split_k=3)),
    ge.GemmCase("sk3-f32-1sm", "bf16", "f32", 520, 392, 1000, opts=_opts(split_k=3, variant="1sm_n128")),
    # fp8 operands (widened exactly to f16), a mixed e4m3 x e5m2 pair, and f32 operands in all three tf32 schedules
    ge.GemmCase("e4m3-bf16", "f8e4m3", "bf16", 300, 264, 256),
    ge.GemmCase("e4m3-f16-sk2", "f8e4m3", "f16", 300, 264, 256, opts=_opts(split_k=2)),
    ge.GemmCase("e4m3-f32-m512", "f8e4m3", "f32", 600, 272, 256, opts=_opts(variant="2sm_m512")),
    ge.GemmCase("mixed-f32", "mixed", "f32", 300, 264, 256),
    ge.GemmCase("mixed-bf16", "mixed", "bf16", 300, 264, 256),
    ge.GemmCase("f32-tf32", "f32", "f32", 300, 264, 200, opts=_opts(f32="tf32")),
    ge.GemmCase("f32-3xtf32", "f32", "f32", 300, 264, 200, opts=_opts(f32="3xtf32")),
    ge.GemmCase("f32-hybrid-sk2", "f32", "f32", 300, 264, 200, opts=_opts(f32="hybrid", split_k=2)),
]
GEMM_CASES = PLAN_GRID + LAYOUT_CASES


def _bound(case):
    return 8 if case.in_dtype == "mixed" else 16   # integers exact in every input format (e5m2: up to 8)


def _options(case):
    return {**GEMM_OPTIONS, **case.options}


def _read_bits(client, out, buf=None):
    """Output bits of a TensorHandle (and, for a window, the whole buffer's bits)."""
    bits = out.to_numpy(client)
    if out.dtype == "f16":
        bits = bits.view(np.uint16)
    elif out.dtype == "f32":
        bits = bits.view(np.uint32)
    whole = None
    if buf is not None:
        whole = np.frombuffer(client.read_one(buf[0]), dtype=buf[1].dtype).reshape(buf[1].shape)
    return bits, whole


def run_gemm(client, case, a, b, **epilogue):
    """Run a case on the device and on the planner; returns (output bits, plan)."""
    opts = _options(case)
    for k, v in opts.items():
        client.set_option(k, v)
    lhs, rhs, out, buf = ge.gemm_tensors(case, a, b, ge.device_alloc(client))
    ep = dict(epilogue)
    if "bias" in ep:
        ep["bias"] = TensorHandle.from_numpy(client, ep["bias"].astype(np.float32), "f32")
    matmul.launch(client, lhs, rhs, out, **ep)
    client.sync()
    kernel = client.last_kernel()
    bits, whole = _read_bits(client, out, buf)
    plan = ge.probe(client.properties["num_streaming_multiprocessors"], opts, lambda pc: matmul.launch(pc, lhs, rhs, out, **ep))
    assert plan.kernel == kernel, (plan.kernel, kernel)
    if buf is not None:   # the window's neighbours are untouched
        mask = np.ones(whole.shape, bool)
        mask[..., ge.WINDOW_COL0:ge.WINDOW_COL0 + case.N] = False
        assert np.all(whole[mask] == ge.SENTINEL[case.out_dtype])
    return bits, plan


def _expect_path(case, plan):
    o = case.options
    if o.get("gemm.variant", "auto") not in ("auto", "simt"):
        assert o["gemm.variant"] in plan.kernel, (case.name, plan.kernel)
    if o.get("gemm.split_k") == "2" and o.get("gemm.variant") in HEAD_VARIANTS:
        assert plan.head and plan.whole_tiles > 0, (case.name, plan.text)
    if o.get("gemm.split_k") == "off":
        assert not plan.head


# ------------------------------------------------------------------------------------------------ 1. integer-exact matmul
@pytest.mark.parametrize("case", GEMM_CASES, ids=[c.name for c in GEMM_CASES])
def test_integer_matmul_is_exact_on_every_plan(client, case):
    ls, rs = ge.gemm_shapes(case)
    a, b, exact = ge.matmul_operands(ls, rs, _bound(case), seed=case.M + case.N, out_dtype=case.out_dtype)
    bits, plan = run_gemm(client, case, a, b)
    _expect_path(case, plan)
    ge.assert_exact(bits, exact, case.out_dtype, f"{case.name} on {plan.kernel}")


# ------------------------------------------------------------------------------------------------ 2. fused epilogue
EPILOGUE_CASES = [c for c in PLAN_GRID if "m512" not in c.name] + [c for c in LAYOUT_CASES if c.in_dtype != "mixed"]


@pytest.mark.parametrize("alpha,act", [(0.5, None), (0.125, "relu")])
@pytest.mark.parametrize("case", EPILOGUE_CASES, ids=[c.name for c in EPILOGUE_CASES])
def test_fused_epilogue_is_exact_where_the_arithmetic_is(client, case, alpha, act):
    ls, rs = ge.gemm_shapes(case)
    a, b, exact = ge.matmul_operands(ls, rs, _bound(case), seed=case.K, out_dtype=case.out_dtype)
    bias = np.arange(case.N) % 129 / 8.0 - 8.0   # dyadic: alpha * exact + bias needs < 24 bits
    bits, plan = run_gemm(client, case, a, b, alpha=alpha, bias=bias, activation=act)
    want = alpha * exact + bias
    if act == "relu":
        want = np.maximum(want, 0.0)
    ge.assert_exact(bits, want, case.out_dtype, f"{case.name} on {plan.kernel}")


GELU_CASES = [c for c in PLAN_GRID if c.out_dtype == "f32" and "m512" not in c.name]


@pytest.mark.parametrize("case", GELU_CASES, ids=[c.name for c in GELU_CASES])
def test_gelu_f32_is_within_a_few_ulps_and_16bit_is_its_rounding(client, case):
    ls, rs = ge.gemm_shapes(case)
    a, b, exact = ge.matmul_operands(ls, rs, _bound(case), seed=case.K + 1, out_dtype="f32")
    alpha, bias = 1.0 / 1024, (np.arange(case.N) % 17 - 8) / 4.0
    bits, _ = run_gemm(client, case, a, b, alpha=alpha, bias=bias, activation="gelu")
    x = alpha * exact + bias
    ref = 0.5 * x * (1.0 + np.vectorize(math.erf)(x / math.sqrt(2.0)))
    got = ge.bits_to_f64(bits, "f32")
    # erff is not correctly rounded: a few ulps of the pre-activation value
    assert np.max(np.abs(got - ref) / np.maximum(np.abs(x), 1.0)) <= 8 * 2.0 ** -24
    for od in ("bf16",):   # bf16 inputs: bf16 output; the plan differs only in the output tag
        c16 = ge.GemmCase(case.name + "-16", case.in_dtype, od, case.M, case.N, case.K, opts=case.opts)
        bits16, _ = run_gemm(client, c16, a, b, alpha=alpha, bias=bias, activation="gelu")
        ge.assert_bits_equal(bits16, ge.f32_run_rounded(got, od), od, "gelu 16-bit output")


# ------------------------------------------------------------------------------------------------ 3. one rounding on random data
ONE_ROUNDING = [c for c in PLAN_GRID if c.out_dtype != "f32"] + [c for c in LAYOUT_CASES if c.out_dtype in ("bf16", "f16") and c.in_dtype != "mixed"]


def _uniform(shape, dtype, seed):
    vals = synth.uniform_f32(seed, int(np.prod(shape)), -1.0, 1.0).reshape(shape)
    return synth.from_device_dtype(synth.to_device_dtype(vals, dtype), dtype).reshape(shape).astype(np.float64)


@pytest.mark.parametrize("epilogue", ["plain", "fused"])
@pytest.mark.parametrize("case", ONE_ROUNDING, ids=[c.name for c in ONE_ROUNDING])
def test_16bit_output_is_the_f32_run_rounded_once(client, case, epilogue):
    ld, rd = case.dtypes()
    ls, rs = ge.gemm_shapes(case)
    a, b = _uniform(ls, ld, 3), _uniform(rs, rd, 4)
    ep = {} if epilogue == "plain" else {"alpha": 0.3713, "bias": synth.uniform_f32(5, case.N, -2.0, 2.0).astype(np.float64), "activation": "relu"}
    c32 = ge.GemmCase(case.name + "-f32", case.in_dtype, "f32", case.M, case.N, case.K, case.batch, case.bcast, case.lhs_t,
                      case.rhs_t, case.window, case.opts)
    bits32, p32 = run_gemm(client, c32, a, b, **ep)
    bits16, p16 = run_gemm(client, case, a, b, **ep)
    assert ge.out_tag_free(p32.kernel) == ge.out_tag_free(p16.kernel) and p32.head == p16.head, (p32.text, p16.text)
    assert p32.whole_tiles == p16.whole_tiles and p32.tma_store == p16.tma_store
    f32 = bits32.view(np.float32)
    ge.assert_bits_equal(bits16, ge.f32_run_rounded(f32, case.out_dtype), case.out_dtype, f"{case.name} ({epilogue}) on {p16.kernel}")
    assert ge.bit_mismatches(ge.rz(f32, case.out_dtype), bits16, case.out_dtype).any()   # truncation would not pass


# ------------------------------------------------------------------------------------------------ 4. block-scaled exact
TC_VARIANTS = ["2sm_n256", "2sm_n224", "2sm_n128", "1sm_n128"]
SCALED_KINDS = {"e4m3": ("f8e4m3", 32), "e5m2": ("f8e5m2", 32), "e2m1": ("f4e2m1x2", 32), "nvfp4": ("f4e2m1x2", 16)}


def run_scaled(client, variant, kind, od, M, N, K, packed=False, split="auto", seed=0):
    dt, block = SCALED_KINDS[kind]
    a_dev, b_dev, sa, sb, a, b = ge.block_scaled_operands(M, N, K, kind, seed=seed + M + N)
    client.set_option("gemm.variant", variant)
    client.set_option("gemm.split_k", split)
    one = 0x38 if block == 16 else 127
    if packed:
        sa, sb = synth.pack_scale_chunks(sa, one), synth.pack_scale_chunks(sb, one)
    sdt = "f8e4m3" if block == 16 else "ue8m0"
    lhs, rhs = TensorHandle.from_numpy(client, a_dev, dt), TensorHandle.from_numpy(client, b_dev, dt)
    ls, rs = TensorHandle.from_numpy(client, sa, sdt), TensorHandle.from_numpy(client, sb, sdt)
    out = TensorHandle.empty_contiguous(client, [M, N], od)
    matmul.launch_scaled(client, lhs, rhs, ls, rs, out, scale_block=block, scales_packed=packed)
    client.sync()
    assert variant in client.last_kernel()
    bits, _ = _read_bits(client, out)
    return bits, np.matmul(a, b.T)


@pytest.mark.parametrize("od", ["f32", "bf16", "f16"])
@pytest.mark.parametrize("kind", list(SCALED_KINDS))
@pytest.mark.parametrize("variant", TC_VARIANTS)
def test_block_scaled_integer_products_are_exact(client, variant, kind, od):
    # N = 520: two 224-wide tiles and a ragged third, so the direct-store tail columns [192, 224) of every tile run
    bits, exact = run_scaled(client, variant, kind, od, 300, 520, 256)
    ge.assert_exact(bits, exact, od, f"{kind} {variant} -> {od}")
    bits_p, _ = run_scaled(client, variant, kind, od, 300, 520, 256, packed=True)
    assert np.array_equal(bits_p, bits)


@pytest.mark.parametrize("od", ["f32", "bf16", "f16"])
@pytest.mark.parametrize("variant", TC_VARIANTS)
def test_block_scaled_stream_k_head_is_exact(client, variant, od):
    bits, exact = run_scaled(client, variant, "e4m3", od, 256, 448, 1024, split="3", seed=7)
    ge.assert_exact(bits, exact, od, f"split {variant} -> {od}")


# ------------------------------------------------------------------------------------------------ 5. convolution exact
from test_conv_backward_gpu import CASES as CONV_CASES, IDS as CONV_IDS, dy_shape  # noqa: E402

CONV_PATH_OPTIONS = [("gemm.variant", "2sm_n128"), ("gemm.variant", "1sm_n128"), ("gemm.epilogue", "direct"),
                     ("gemm.split_k", "on"), ("gemm.split_k", "off")]
CONV_PATH_GEOMS = [((3, 17, 19, 64), 200, 3, 1, 1), ((2, 28, 28, 256), 256, 3, 2, 1), ((1, 9, 9, 3), 32, 7, 1, 3)]


def conv_issue(which, xs, cout, k, s, p, d, dtype, od, alloc, vals=None, window=False):
    """(issue(client), out handle, window buffer) of one convolution call.  which: fwd / dgrad / wgrad."""
    def up(shape, key):
        v = vals[key] if vals is not None else np.zeros(shape)
        dev = synth.to_device_dtype(v.astype(np.float32), dtype)
        return TensorHandle.new_contiguous(list(shape), alloc(dev), dtype)
    ws, dys = (cout, k, k, xs[3]), dy_shape(xs, cout, k, s, p, d)
    osz = DTYPE_SIZE[od]
    if which == "fwd":
        x, w = up(xs, "x"), up(ws, "w")
        oshape = list(dys)
    elif which == "dgrad":
        dy, w = up(dys, "dy"), up(ws, "w")
        oshape = list(xs)
    else:
        x, dy = up(xs, "x"), up(dys, "dy")
        oshape = list(ws)
    buf = None
    if window:   # channels [64, 64 + C) of a 64 + C + 64 channel tensor filled with sentinels
        full = oshape[:-1] + [oshape[-1] + 128]
        host = np.full(full, ge.SENTINEL[od], dtype=ge.OUT_BITS_VIEW[od])
        h = alloc(host)
        strides = [int(np.prod(full[i + 1:])) for i in range(4)]
        out = TensorHandle(h.offset(64 * osz), oshape, strides, od)
        buf = (h, host)
    else:
        out = TensorHandle.new_contiguous(oshape, alloc(np.zeros(oshape, ge.OUT_BITS_VIEW[od])), od)

    def issue(c, stream=None):
        if which == "fwd":
            conv.launch(c, x, w, out, stride=s, padding=p, dilation=d, stream=stream)
        elif which == "dgrad":
            conv.backward_data(c, dy, w, out, stride=s, padding=p, dilation=d, stream=stream)
        else:
            conv.backward_weight(c, x, dy, out, stride=s, padding=p, dilation=d, stream=stream)
    return issue, out, buf


def conv_exact(which, vals, xs, cout, k, s, p, d):
    if which == "fwd":
        return co.conv2d_f64(vals["x"], vals["w"], s, p, d)
    if which == "dgrad":
        return cbo.conv2d_input_grad_f64(vals["dy"], vals["w"], xs[1:3], s, p, d)
    return cbo.conv2d_weight_grad_f64(vals["x"], vals["dy"], (k, k), s, p, d)


def run_conv(client, which, geom, od, vals, options=None, window=False):
    xs, cout, k, s, p, d = geom
    dtype = "f16" if od == "f16" else "bf16"
    issue, out, buf = conv_issue(which, xs, cout, k, s, p, d, dtype, od, ge.device_alloc(client), vals, window)
    issue(client)
    client.sync()
    bits, whole = _read_bits(client, out, buf)
    if buf is not None:
        assert np.all(whole[..., :64] == ge.SENTINEL[od]) and np.all(whole[..., 64 + out.shape[-1]:] == ge.SENTINEL[od])
    plan = ge.probe(client.properties["num_streaming_multiprocessors"], {**GEMM_OPTIONS, **(options or {})}, issue)
    assert plan.kernel == client.last_kernel(), (plan.kernels, client.last_kernel())
    return bits, plan


def conv_values(geom, seed, bound=16):
    xs, cout, k, s, p, d = geom
    vals = {"x": ge.int_values(xs, bound, seed), "w": ge.int_values((cout, k, k, xs[3]), bound, seed + 1),
            "dy": ge.int_values(dy_shape(xs, cout, k, s, p, d), bound, seed + 2)}
    for which in ("fwd", "dgrad", "wgrad"):
        ge.assert_exact_bound(conv_exact(which, {kk: np.abs(v) for kk, v in vals.items()}, xs, cout, k, s, p, d)[0])
    return vals


@pytest.mark.parametrize("which", ["fwd", "dgrad", "wgrad"])
@pytest.mark.parametrize("od", ["bf16", "f16", "f32"])
@pytest.mark.parametrize("geom", CONV_CASES, ids=CONV_IDS)
def test_integer_convolution_is_exact(client, geom, od, which):
    vals = conv_values(geom, 100)
    bits, plan = run_conv(client, which, geom, od, vals)
    ge.assert_exact(bits, conv_exact(which, vals, *geom)[0], od, f"{which} on {plan.kernels}")


CONV_PATH_CASES = [(which, (*g, 1), od, opt) for opt in CONV_PATH_OPTIONS for g in CONV_PATH_GEOMS for od in ("bf16", "f16")
                   for which in ("fwd", "dgrad", "wgrad")]


@pytest.mark.parametrize("opt", CONV_PATH_OPTIONS, ids=[f"{k}={v}" for k, v in CONV_PATH_OPTIONS])
def test_integer_convolution_is_exact_on_every_tile_and_epilogue(client, opt):
    client.set_option(*opt)
    for which, geom, od, o in CONV_PATH_CASES:
        if o != opt:
            continue
        vals = conv_values(geom, 200)
        bits, plan = run_conv(client, which, geom, od, vals, dict([opt]))
        ge.assert_exact(bits, conv_exact(which, vals, *geom)[0], od, f"{which} {geom} {opt} on {plan.kernels}")


@pytest.mark.parametrize("which", ["fwd", "dgrad", "wgrad"])
@pytest.mark.parametrize("od", ["bf16", "f16"])
def test_integer_convolution_into_a_channel_slice_is_exact(client, which, od):
    geom = ((2, 13, 11, 64), 96, 3, 2, 1, 1)
    vals = conv_values(geom, 300)
    bits, plan = run_conv(client, which, geom, od, vals, window=True)
    ge.assert_exact(bits, conv_exact(which, vals, *geom)[0], od, f"{which} slice on {plan.kernels}")


ROUNDING_CONV = [("fwd", ((2, 17, 13, 64), 200, 3, 1, 1, 1)), ("dgrad", ((2, 17, 13, 64), 200, 3, 1, 1, 1)),
                 ("dgrad", ((2, 19, 16, 64), 96, 3, 2, 1, 1)), ("wgrad", ((8, 28, 28, 64), 64, 3, 1, 1, 1))]


@pytest.mark.parametrize("od", ["bf16", "f16"])
@pytest.mark.parametrize("which,geom", ROUNDING_CONV, ids=[f"{w}-s{g[3]}" for w, g in ROUNDING_CONV])
def test_16bit_convolution_is_the_f32_run_rounded_once(client, which, geom, od):
    xs, cout, k, s, p, d = geom
    dtype = "f16" if od == "f16" else "bf16"
    vals = {"x": _uniform(xs, dtype, 1), "w": _uniform((cout, k, k, xs[3]), dtype, 2), "dy": _uniform(dy_shape(xs, cout, k, s, p, d), dtype, 3)}
    # f32 outputs of the same (16-bit) operands: run_conv picks the input dtype from the output, so pass it explicitly
    issue32, out32, _ = conv_issue(which, xs, cout, k, s, p, d, dtype, "f32", ge.device_alloc(client), vals)
    issue32(client)
    client.sync()
    p32 = ge.probe(client.properties["num_streaming_multiprocessors"], GEMM_OPTIONS, issue32)
    bits32, _ = _read_bits(client, out32)
    bits16, p16 = run_conv(client, which, geom, od, vals)
    assert [ge.out_tag_free(kk) for kk in p32.kernels] == [ge.out_tag_free(kk) for kk in p16.kernels] and p32.head == p16.head
    ge.assert_bits_equal(bits16, ge.f32_run_rounded(bits32.view(np.float32), od), od, f"{which} on {p16.kernels}")


# ------------------------------------------------------------------------------------------------ 6. conversion edges
EDGE_PATHS = [_opts(epilogue="tma", split_k="off"), _opts(epilogue="direct", split_k="off"), _opts(split_k="2")]


@pytest.mark.parametrize("opts", EDGE_PATHS, ids=["tma", "direct", "stream-k"])
def test_conversion_edges_round_like_numpy(client, opts):
    f16_targets = [65504, 65519, 65520, 70000, -70000, 2.0 ** -7, 2.0 ** -12, 3 * 2.0 ** -13, 2049, 2051, 4097]
    bf16_targets = [257, 259, 385, -257, 511, 1025.0, 2 ** 20 + 2 ** 12, 3.0]
    for in_dt, od, targets in (("f16", "f16", f16_targets), ("f16", "f32", f16_targets), ("bf16", "bf16", bf16_targets)):
        # column scales: 1, -1, and 2^-13 (f16 results 2^-20, 2^-25 (a tie: rounds to 0) and 3 * 2^-26 (-> 2^-24))
        a, b, exact = ge.edge_operands(targets * 12, in_dt, K=256, col_signs=(1.0, -1.0, 2.0 ** -13, 0.5) * 4)
        case = ge.GemmCase("edges", in_dt, od, a.shape[0], b.shape[1], a.shape[1], rhs_t=True, opts=opts)
        bits, plan = run_gemm(client, case, a, b)
        if dict(opts).get("gemm.split_k") == "2":
            assert plan.head
        want = ge.rne(exact, od)
        ge.assert_bits_equal(bits, want, od, f"edges {in_dt}->{od} on {plan.kernel}")
        if od == "f16":   # the checks numpy's own f64 -> f16 rounding agrees with (no double-rounding case among these)
            with np.errstate(over="ignore"):
                assert np.array_equal(want, exact.astype(np.float16).view(np.uint16))
            sub = ge.bits_to_f64(bits, od)[[5, 6, 7], 2]
            assert list(sub) == [2.0 ** -20, 0.0, 2.0 ** -24]
            assert list(ge.bits_to_f64(bits, od)[[1, 2, 3, 4], 0]) == [65504.0, np.inf, np.inf, -np.inf]


# ------------------------------------------------------------------------------------------------ 7. non-finite operands
@pytest.mark.parametrize("opts", EDGE_PATHS, ids=["tma", "direct", "stream-k"])
@pytest.mark.parametrize("dtype", ["bf16", "f16"])
def test_nonfinite_operands_land_where_f64_puts_them(client, dtype, opts):
    M, N, K = 200, 136, 256
    a, b = ge.int_values((M, K), 4, 1), ge.int_values((K, N), 4, 2)
    a[3, 10], a[7, 100], a[9, 200] = np.inf, -np.inf, np.nan
    b[10, 5], b[150, 8], b[30, 60] = -np.inf, np.inf, np.nan
    a[11, 150] = np.inf                     # meets b's +inf in column 8: +inf + ... ; a[7,100] * b[100, :] = -inf everywhere
    b[20, :] = 0.0
    a[13, 20] = np.inf                      # inf * 0 = NaN for the whole row 13
    exact = ge.matmul_f64_ieee(a, b)
    for od in (dtype, "f32"):
        case = ge.GemmCase("nonfinite", dtype, od, M, N, K, opts=opts)
        bits, plan = run_gemm(client, case, a, b)
        got = ge.bits_to_f64(bits, od)
        for mask in (np.isnan, np.isposinf, np.isneginf):
            assert np.array_equal(mask(got), mask(exact)), (mask.__name__, od, plan.kernel)
        fin = np.isfinite(exact)
        ge.assert_bits_equal(bits[fin], ge.rne(exact[fin], od), od, "finite outputs next to non-finite ones")


# ------------------------------------------------------------------------------------------------ 8. state across launches and streams
def test_stream_k_tickets_and_workspace_across_queued_launches_and_two_streams(client):
    """Stream-K GEMMs of different tile counts back to back (the tickets must reset themselves), reduce_all launches between them
    (sharing the stream's workspace, chained through PDL) and a weight gradient with a head, queued with no sync, on the
    client's stream and on a second stream at the same time."""
    client.set_option("gemm.split_k", "2")
    sms = client.properties["num_streaming_multiprocessors"]
    shapes = [(520, 392, 1000), (1300, 1544, 200), (300, 264, 640)]   # different tile and range counts, each with a head
    geom = ((4, 28, 28, 64), 64, 3, 1, 1, 1)
    stream2 = client.create_stream()
    try:
        queues = []
        for si in range(2):
            q = []
            for i, (M, N, K) in enumerate(shapes):
                a, b, exact = ge.matmul_operands((M, K), (K, N), 16, seed=10 * si + i, out_dtype="bf16")
                case = ge.GemmCase("queued", "bf16", "bf16", M, N, K, opts=_opts(split_k=2))
                lhs, rhs, out, _ = ge.gemm_tensors(case, a, b, ge.device_alloc(client))
                assert ge.probe(sms, _options(case), lambda pc, lhs=lhs, rhs=rhs, out=out: matmul.launch(pc, lhs, rhs, out)).head
                q.append((lambda st, lhs=lhs, rhs=rhs, out=out: matmul.launch(client, lhs, rhs, out, stream=st), out, exact, "bf16"))
                x = ge.int_values((1 << 20) + 7, 100, 3 * si + i)
                xt = TensorHandle.from_numpy(client, x.astype(np.float32), "f32")
                rt = TensorHandle.empty_contiguous(client, [1], "f32")
                q.append((lambda st, xt=xt, rt=rt: reduce.launch(client, xt, rt, None, "sum", stream=st), rt, np.array([x.sum()]), "f32"))
            vals = conv_values(geom, 400 + si, bound=4)
            issue, dw, _ = conv_issue("wgrad", *geom, "bf16", "bf16", ge.device_alloc(client), vals)
            assert ge.probe(sms, {**GEMM_OPTIONS, "gemm.split_k": "2"}, issue).head
            q.append((lambda st, issue=issue: issue(client, st), dw, conv_exact("wgrad", vals, *geom)[0], "bf16"))
            queues.append(q)
        for i in range(len(queues[0])):           # interleaved launch by launch, no sync in between
            for q, st in zip(queues, (None, stream2)):
                q[i][0](st)
        client.sync_stream(stream2)
        client.sync()
        for q in queues:
            for _, out, exact, od in q:
                ge.assert_exact(_read_bits(client, out)[0], exact, od, "queued launch")
    finally:
        client.sync_stream(stream2)
        client.destroy_stream(stream2)
