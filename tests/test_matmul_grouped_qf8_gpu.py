"""GPU: b200_matmul_grouped_quantized_fp8 bit for bit against the per-group fp8 oracle (tests/qmatmul_fp8_oracle.py) on
integer-valued codes, against the dense b200_matmul_quantized_fp8 on b200_quantize'd data, its error bound and the 128 x 128
weight-scale recipe, non-finite values, offsets (malformed, rewritten on the stream), group counts, staged codes and the
short last block, determinism, and torch's F.scaled_grouped_mm as a yardstick."""
import ctypes as C

import numpy as np
import pytest

import qmatmul_fp8_oracle as qf8
import qmatmul_oracle as qmo
import quant_oracle as qo
from cubecl_b200 import TensorHandle, _ffi, matmul, quant, synth
from cubecl_b200.quant import QuantScheme, QuantizedTensor

pytestmark = pytest.mark.gpu

FP8 = ["e4m3", "e5m2"]
SENT = {"bf16": 0x7FA1, "f16": 0x7E01, "f32": 0x7FC0_1234}
# group sizes (T = their sum): empty first, middle and last groups; 1-row groups; ends mid-tile (128 rows) and mid-pair (256)
ROUTES = {"balanced": [192] * 4, "skewed": [0, 300, 0, 17, 400, 0], "one_row": [1, 1, 0, 1, 129, 1],
          "mid_tile": [65, 127, 129, 255, 257, 3]}


def scheme_of(value, block=0, dt=None, tensor=False):
    return QuantScheme(value=value, block=block, block_scale=dt if block else None, tensor=tensor or block == 0)


def make(client, scheme, batch, rows, K, seed, scale_values=None, q=None, shape=None):
    """Integer-valued codes in [-4, 4] (every partial sum of a block of <= 128 stays within 2^11) and random scales on the scale
    dtype's grid: (QuantizedTensor of `shape`, default [batch, rows, K]; host copy with batch x rows)."""
    rng = np.random.default_rng(seed)
    if q is None:
        q = rng.integers(-4, 5, size=(batch, rows, K)).astype(np.float32)
    values = qo.fp8_codes(q, scheme.value)
    raw = None
    if scheme.block:
        nb = K // scheme.block
        s = scale_values if scale_values is not None else \
            (rng.uniform(0.5, 2.0, size=(batch, rows, nb)) * np.exp2(rng.integers(-4, 4, size=(batch, rows, nb))))
        raw = qo.scale_store(scheme.block_scale, qo.round_up(scheme.block_scale, np.asarray(s, np.float32)))
    g = np.float32(rng.uniform(0.001, 0.01)) if scheme.has_tensor else None
    vt = TensorHandle.from_numpy(client, values, quant.VALUE_DTYPES[scheme.value])
    st = TensorHandle.from_numpy(client, np.ascontiguousarray(raw), quant.SCALE_DTYPES[scheme.block_scale]) if raw is not None else None
    tt = TensorHandle.from_numpy(client, np.array([g], np.float32), "f32") if g is not None else None
    return (QuantizedTensor(vt, st, tt, scheme, shape or [batch, rows, K]), qmo.Operand(scheme, values, raw, g, batch, rows, K))


def make_x(client, scheme, T, K, seed, **kw):
    return make(client, scheme, 1, T, K, seed, shape=[T, K], **kw)


def clamp(offs, T):
    ends, prev = [], 0
    for v in offs:
        prev = min(max(int(v), prev), T)
        ends.append(prev)
    return ends


def expert(hw, g):
    """Host operand of expert g of a [G, N, K] operand."""
    return qmo.Operand(hw.scheme, hw.values[g:g + 1], None if hw.scales is None else hw.scales[g:g + 1], hw.tensor, 1, hw.rows, hw.K)


def oracle(hx, hw, offs):
    """f32 result [T, N] of the contract before the output rounding, and the written rows."""
    T, N = hx.rows, hw.rows
    out, written, lo = np.zeros((T, N), np.float32), np.zeros(T, bool), 0
    for g, hi in enumerate(clamp(offs, T)):
        if hi > lo:
            out[lo:hi] = qf8.matmul(hx, expert(hw, g), rows=np.arange(lo, hi))[0]
            written[lo:hi] = True
        lo = hi
    return out, written


def sentinel(client, shape, odt):
    return TensorHandle.from_numpy(client, np.full(shape, SENT[odt], np.uint32 if odt == "f32" else np.uint16), odt)


def bits(client, t):
    return np.asarray(t.to_numpy(client)).view(np.uint32 if t.dtype == "f32" else np.uint16).reshape(t.shape)


def i32(client, offs):
    return TensorHandle.from_numpy(client, np.asarray(offs, np.int32), "i32")


def run(client, qx, qw, offs, odt, stream=None):
    out = sentinel(client, [qx.shape[0], qw.shape[1]], odt)
    matmul.launch_grouped_quantized_fp8(client, qx, qw, offs if isinstance(offs, TensorHandle) else i32(client, offs), out, stream)
    return out


def check(client, qx, hx, qw, hw, offs, odt="f32"):
    got = bits(client, run(client, qx, qw, offs, odt))
    client.sync()
    acc, written = oracle(hx, hw, offs)
    want = np.asarray(qmo.to_out(acc, odt)).view(got.dtype).reshape(got.shape)
    bad = np.argwhere(got[written] != want[written])
    assert bad.size == 0, bad[:4]
    assert (got[~written] == SENT[odt]).all()
    return got


def offsets(sizes):
    return list(np.cumsum(sizes))


# ---------------------------------------------------------------------------------------------- exact contract
@pytest.mark.parametrize("vx", FP8)
@pytest.mark.parametrize("vw", FP8)
def test_every_value_pair(client, vx, vw):
    sizes = ROUTES["skewed"]
    T, G = sum(sizes), len(sizes)
    qx, hx = make_x(client, scheme_of(vx, 128, "f32"), T, 512, 1)
    qw, hw = make(client, scheme_of(vw, 128, "f32"), G, 200, 512, 2)
    check(client, qx, hx, qw, hw, offsets(sizes), "bf16")
    qx, hx = make_x(client, scheme_of(vx, 32, "f16"), T, 256, 3)
    qw, hw = make(client, scheme_of(vw), G, 72, 256, 4)
    check(client, qx, hx, qw, hw, offsets(sizes))


@pytest.mark.parametrize("dt", ["f32", "f16", "bf16", "ue8m0", "ue4m3"])
@pytest.mark.parametrize("block", [32, 64, 128])
def test_block_sizes_and_scale_dtypes(client, block, dt):
    sizes = ROUTES["mid_tile"]
    T, G = sum(sizes), len(sizes)
    qx, hx = make_x(client, scheme_of("e4m3", block, dt), T, 512, 5)
    qw, hw = make(client, scheme_of("e4m3", block, dt), G, 136, 512, 6)
    check(client, qx, hx, qw, hw, offsets(sizes))
    # two levels on both sides, e5m2 weights
    qx, hx = make_x(client, scheme_of("e4m3", block, dt, tensor=True), T, 512, 7)
    qw, hw = make(client, scheme_of("e5m2", block, dt, tensor=True), G, 136, 512, 8)
    check(client, qx, hx, qw, hw, offsets(sizes), "bf16")


@pytest.mark.parametrize("route", list(ROUTES))
@pytest.mark.parametrize("tile", ["2sm_n128", "1sm_n128"])
@pytest.mark.parametrize("store", ["tma", "direct"])
@pytest.mark.parametrize("odt", ["f32", "bf16", "f16"])
def test_routes_tiles_store_paths_outputs(client, route, tile, store, odt):
    sizes = ROUTES[route]
    T, G = sum(sizes), len(sizes)
    client.set_option("gemm.variant", tile)
    client.set_option("gemm.epilogue", store)
    try:
        qx, hx = make_x(client, scheme_of("e4m3", 64, "bf16"), T, 384, 9)
        qw, hw = make(client, scheme_of("e5m2", 128, "f32", tensor=True), G, 264, 384, 10)
        check(client, qx, hx, qw, hw, offsets(sizes), odt)
    finally:
        client.set_option("gemm.variant", "auto")
        client.set_option("gemm.epilogue", "tma")


@pytest.mark.parametrize("sx,sw", [(("e4m3", 0), ("e4m3", 128)), (("e5m2", 128), ("e4m3", 0)), (("e4m3", 0), ("e5m2", 0))])
def test_per_tensor_sides(client, sx, sw):
    sizes = ROUTES["mid_tile"]
    T, G = sum(sizes), len(sizes)
    qx, hx = make_x(client, scheme_of(sx[0], sx[1], "f16"), T, 384, 11)
    qw, hw = make(client, scheme_of(sw[0], sw[1], "bf16"), G, 96, 384, 12)
    check(client, qx, hx, qw, hw, offsets(sizes), "bf16")


def test_staged_unaligned_codes_and_short_last_block(client):
    # K = 200: not a multiple of 16 (both code operands are staged) nor of 128 (per-tensor sides fold a short last block of 72)
    sizes = [70, 0, 33, 100]
    T, G = sum(sizes), len(sizes)
    qx, hx = make_x(client, scheme_of("e4m3"), T, 200, 15)
    qw, hw = make(client, scheme_of("e5m2"), G, 33, 200, 16)
    check(client, qx, hx, qw, hw, offsets(sizes))
    # an unaligned lhs code base: a view 8 bytes into a larger buffer
    qx, hx = make_x(client, scheme_of("e4m3", 64, "f32"), T, 256, 17)
    qw, hw = make(client, scheme_of("e4m3", 64, "f32"), G, 80, 256, 18)
    big = TensorHandle.from_numpy(client, np.concatenate([np.zeros(8, np.uint8), hx.values.reshape(-1)]), "u8")
    qx.values = TensorHandle.new_contiguous([T, 256], big.handle.offset(8, hx.values.size), "f8e4m3")
    check(client, qx, hx, qw, hw, offsets(sizes), "bf16")


# ---------------------------------------------------------------------------------------------- offsets and group counts
@pytest.mark.parametrize("table", [[50, 30, 400, 10000, -5], [100, 90, 80], [-7, -1, 2000, 3], [0, 0, 0]])
def test_malformed_offsets_are_clamped(client, table):
    T, G = 600, len(table)
    qx, hx = make_x(client, scheme_of("e4m3", 128, "f32"), T, 256, 19)
    qw, hw = make(client, scheme_of("e4m3", 32, "ue8m0"), G, 136, 256, 20)
    check(client, qx, hx, qw, hw, table)


def test_offsets_rewritten_on_the_stream_are_followed(client):
    """two calls enqueued back to back with the offsets rewritten on the stream between them (no host sync)"""
    T, G = 1500, 5
    first, second = offsets([300, 0, 500, 200, 100]), offsets([10, 700, 1, 300, 489])
    qx, hx = make_x(client, scheme_of("e4m3", 128, "f32"), T, 256, 21)
    qw, hw = make(client, scheme_of("e5m2", 128, "f32"), G, 128, 256, 22)
    src1, src2, offs = i32(client, first), i32(client, second), i32(client, np.zeros(G))
    o1, o2 = sentinel(client, [T, 128], "f32"), sentinel(client, [T, 128], "f32")
    lib = client._lib
    _ffi.check(lib.b200_copy(client._ctx, None, C.c_uint64(offs.handle.ptr), C.c_uint64(src1.handle.ptr), 4 * G))
    matmul.launch_grouped_quantized_fp8(client, qx, qw, offs, o1)
    _ffi.check(lib.b200_copy(client._ctx, None, C.c_uint64(offs.handle.ptr), C.c_uint64(src2.handle.ptr), 4 * G))
    matmul.launch_grouped_quantized_fp8(client, qx, qw, offs, o2)
    client.sync()
    for o, table in ((o1, first), (o2, second)):
        acc, written = oracle(hx, hw, table)
        got = bits(client, o)
        assert np.array_equal(got[written], acc.view(np.uint32)[written])
        assert (got[~written] == SENT["f32"]).all()


def test_one_group_equals_the_dense_call(client):
    T, N, K = 700, 300, 512
    qx, _ = make_x(client, scheme_of("e4m3", 64, "f16", tensor=True), T, K, 23)
    qw, _ = make(client, scheme_of("e5m2", 128, "f32"), 1, N, K, 24, shape=[1, N, K])
    got = bits(client, run(client, qx, qw, [T], "bf16"))
    dense = TensorHandle.empty_contiguous(client, [T, N], "bf16")
    matmul.launch_quantized_fp8(client, qx, QuantizedTensor(qw.values, qw.block_scales, qw.tensor_scale, qw.scheme, [N, K]), dense)
    assert np.array_equal(got, bits(client, dense))


def test_1024_groups(client):
    rng = np.random.default_rng(25)
    sizes = list(rng.integers(0, 5, 1024))
    T, G = sum(sizes), 1024
    qx, hx = make_x(client, scheme_of("e4m3", 128, "f32"), T, 128, 26)
    qw, hw = make(client, scheme_of("e4m3", 128, "f32"), G, 16, 128, 27)
    check(client, qx, hx, qw, hw, offsets(sizes))


# ---------------------------------------------------------------------------------------------- real data
def quantized_layer(client, T, G, N, K, seed, scheme=None):
    """b200_quantize'd random activations [T, K] and expert weights [G, N, K] (e4m3, per-block 128 f32 by default)."""
    s = scheme or QuantScheme().with_value("e4m3").per_block(128, "f32")
    x = synth.uniform_f32(seed, T * K, -2.0, 2.0).reshape(T, K) * np.exp2(synth.uniform_f32(seed + 1, T * K, -3.0, 3.0).reshape(T, K))
    w = synth.uniform_f32(seed + 2, G * N * K, -1.0, 1.0).reshape(G, N, K)
    xd = TensorHandle.from_numpy(client, synth.to_device_dtype(x.astype(np.float32), "bf16"), "bf16")
    wd = TensorHandle.from_numpy(client, synth.to_device_dtype(w, "bf16"), "bf16")
    return quant.quantize(client, xd, s), quant.quantize(client, wd, s)


def view(q, shape, v_off, s_off, rows):
    """A QuantizedTensor over `rows` rows of q starting at element offsets (v_off codes, s_off block scales)."""
    K = q.shape[-1]
    nb = K // q.scheme.block
    vals = TensorHandle.new_contiguous(shape, q.values.handle.offset(v_off, rows * K), q.values.dtype)
    sc = TensorHandle.new_contiguous(shape[:-1] + [nb], q.block_scales.handle.offset(s_off * 4, rows * nb * 4), "f32")
    return QuantizedTensor(vals, sc, q.tensor_scale, q.scheme, shape)


@pytest.mark.parametrize("tile", ["2sm_n128", "1sm_n128"])
def test_each_group_equals_the_dense_call_on_its_slices(client, tile):
    sizes = [0, 1000, 13, 0, 700, 335]
    T, G, N, K = sum(sizes), len(sizes), 384, 1024
    qx, qw = quantized_layer(client, T, G, N, K, 31)
    client.set_option("gemm.variant", tile)
    try:
        got = bits(client, run(client, qx, qw, offsets(sizes), "bf16"))
        lo, nb = 0, K // 128
        for g, n in enumerate(sizes):
            if n:
                d = TensorHandle.empty_contiguous(client, [n, N], "bf16")
                matmul.launch_quantized_fp8(client, view(qx, [n, K], lo * K, lo * nb, n), view(qw, [N, K], g * N * K, g * N * nb, N), d)
                assert np.array_equal(got[lo:lo + n], bits(client, d)), g
            lo += n
        assert (got[lo:] == SENT["bf16"]).all()
    finally:
        client.set_option("gemm.variant", "auto")


def test_balanced_groups_equal_the_batched_call(client):
    T, G, N, K = 4096, 8, 512, 1024
    qx, qw = quantized_layer(client, T, G, N, K, 41)
    got = bits(client, run(client, qx, qw, offsets([T // G] * G), "bf16"))
    out = TensorHandle.empty_contiguous(client, [G, T // G, N], "bf16")
    matmul.launch_quantized_fp8(client, QuantizedTensor(qx.values, qx.block_scales, qx.tensor_scale, qx.scheme, [G, T // G, K]), qw, out)
    assert np.array_equal(got, bits(client, out).reshape(T, N))


def _host(client, q, batch, rows, K):
    v = q.values.to_numpy(client).view(np.uint8)
    s = q.block_scales.to_numpy(client) if q.block_scales is not None else None
    t = np.float32(q.tensor_scale.to_numpy(client)[0]) if q.tensor_scale is not None else None
    return qmo.Operand(q.scheme, v.reshape(batch, rows, K), None if s is None else s.reshape(batch, rows, -1), t, batch, rows, K)


def within_bound(got, hx, hw, sizes):
    """|out - ref| <= 2^-10 sum_k |a_k b_k| + one f32 ulp of ref, ref the f64 product of the dequantized operands of each group"""
    dx, dw = hx.dequantized()[0], hw.dequantized()
    worst, lo = 0.0, 0
    for g, n in enumerate(sizes):
        ref, mag = dx[lo:lo + n] @ dw[g].T, np.abs(dx[lo:lo + n]) @ np.abs(dw[g]).T
        err = np.abs(got[lo:lo + n] - ref)
        assert np.all(err <= 2.0 ** -10 * mag + 2.0 ** -23 * np.abs(ref)), g
        worst = max(worst, float(np.max(err / np.maximum(mag, 1e-300)))) if n else worst
        lo += n
    return worst


def test_error_bound_on_quantized_real_data(client):
    sizes = [512, 0, 1024, 300, 212]
    T, G, N, K = sum(sizes), len(sizes), 256, 2048
    qx, qw = quantized_layer(client, T, G, N, K, 51)
    got = run(client, qx, qw, offsets(sizes), "f32").to_numpy(client)
    worst = within_bound(got, _host(client, qx, 1, T, K), _host(client, qw, G, N, K), sizes)
    print(f"\ngrouped fp8 error bound: max |out - ref| / sum|a b| = {worst:.3e} (2^{np.log2(max(worst, 1e-300)):.2f})")


def test_128x128_weight_scale_recipe(client):
    """DeepSeek-style weights: e4m3 codes with one f32 scale per 128 x 128 block, [G, N / 128, K / 128], passed as a per-block-128
    operand whose scale rows repeat each 128 x 128 scale row 128 times"""
    sizes = [256, 0, 384, 130]
    T, G, N, K = sum(sizes), len(sizes), 256, 1024
    rng = np.random.default_rng(61)
    w = rng.standard_normal((G, N // 128, 128, K // 128, 128)) * np.exp2(rng.integers(-3, 3, size=(G, N // 128, 1, K // 128, 1)))
    s2 = (np.abs(w).max(axis=(2, 4)) / 448.0).astype(np.float32)                       # [G, N / 128, K / 128]
    codes = qo.fp8_codes((w / s2[:, :, None, :, None]).reshape(G, N, K).astype(np.float32), "e4m3")
    s_rows = np.ascontiguousarray(np.repeat(s2, 128, axis=1))                           # [G, N, K / 128]
    sw = QuantScheme().with_value("e4m3").per_block(128, "f32")
    qw = QuantizedTensor(TensorHandle.from_numpy(client, codes, "f8e4m3"), TensorHandle.from_numpy(client, s_rows, "f32"), None, sw, [G, N, K])
    x = synth.uniform_f32(62, T * K, -1.0, 1.0).reshape(T, K)
    qx = quant.quantize(client, TensorHandle.from_numpy(client, synth.to_device_dtype(x, "bf16"), "bf16"), sw)
    got = run(client, qx, qw, offsets(sizes), "f32").to_numpy(client)
    hw = qmo.Operand(sw, codes, s_rows, None, G, N, K)
    wq = synth.fp8_bits_to_f32(codes, "f8e4m3").reshape(G, N // 128, 128, K // 128, 128)
    assert np.array_equal(hw.dequantized(), (wq * s2[:, :, None, :, None]).astype(np.float32).reshape(G, N, K).astype(np.float64))
    within_bound(got, _host(client, qx, 1, T, K), hw, sizes)


# ---------------------------------------------------------------------------------------------- non-finite values, determinism
def test_non_finite_values_stay_local(client):
    sizes = [100, 200, 0, 156]
    T, G, N, K = sum(sizes), len(sizes), 144, 256
    sx = scheme_of("e4m3", 32, "f32")
    qx, hx = make_x(client, sx, T, K, 71)
    qw, hw = make(client, scheme_of("e4m3", 32, "f32"), G, N, K, 72)
    base = bits(client, run(client, qx, qw, offsets(sizes), "f32"))
    # a NaN code in lhs row 150 (group 1): only that row changes
    codes = hx.values.copy()
    codes[0, 150, 7] = 0x7F
    qx2 = QuantizedTensor(TensorHandle.from_numpy(client, codes, "f8e4m3"), qx.block_scales, qx.tensor_scale, sx, [T, K])
    got = bits(client, run(client, qx2, qw, offsets(sizes), "f32"))
    assert np.isnan(got[150].view(np.float32)).all()
    rest = np.arange(T) != 150
    assert np.array_equal(got[rest], base[rest])
    # an inf block scale of expert 3 (rows [300, 456)), row 20, block 2: only column 20 of group 3's rows changes
    sc = hw.scales.copy()
    sc[3, 20, 2] = np.inf
    qw2 = QuantizedTensor(qw.values, TensorHandle.from_numpy(client, sc, "f32"), None, qw.scheme, [G, N, K])
    got = bits(client, run(client, qx, qw2, offsets(sizes), "f32"))
    changed = np.argwhere(got != base)
    assert set(changed[:, 1]) == {20} and set(changed[:, 0]) == set(range(300, 456))
    assert not np.isfinite(got[300:456, 20].view(np.float32)).any()


def test_repeats_give_the_same_bits(client):
    rng = np.random.default_rng(81)
    sizes = list(rng.integers(0, 300, 64))
    T, G = sum(sizes), 64
    qx, _ = make_x(client, scheme_of("e4m3", 128, "f32", tensor=True), T, 512, 82)
    qw, _ = make(client, scheme_of("e5m2", 64, "bf16"), G, 200, 512, 83)
    s = client.create_stream()
    try:
        outs = [run(client, qx, qw, offsets(sizes), "bf16", s) for _ in range(3)]
        client.sync_stream(s)
        got = [bits(client, o) for o in outs]
    finally:
        client.destroy_stream(s)
    assert all(np.array_equal(got[0], g) for g in got[1:])


# ---------------------------------------------------------------------------------------------- yardstick
def test_agrees_with_torch_scaled_grouped_mm(client):
    """row-wise scales (one per token, one per expert output row) through both: ours as per-block-128 f32 scales repeated along K"""
    torch = pytest.importorskip("torch")
    F = torch.nn.functional
    if not torch.cuda.is_available() or not hasattr(F, "scaled_grouped_mm"):
        pytest.skip("this torch has no F.scaled_grouped_mm on this GPU")
    sizes = [256, 0, 128, 384]   # torch's grouped GEMMs want group ends aligned to 16
    T, G, N, K = sum(sizes), len(sizes), 256, 512
    rng = np.random.default_rng(91)
    xq, wq = rng.integers(-4, 5, (T, K)).astype(np.float32), rng.integers(-4, 5, (G, N, K)).astype(np.float32)
    sa, sb = rng.uniform(0.5, 2.0, T).astype(np.float32), rng.uniform(0.5, 2.0, (G, N)).astype(np.float32)
    xc, wc = qo.fp8_codes(xq, "e4m3"), qo.fp8_codes(wq, "e4m3")
    s = QuantScheme().with_value("e4m3").per_block(128, "f32")
    qx = QuantizedTensor(TensorHandle.from_numpy(client, xc, "f8e4m3"),
                         TensorHandle.from_numpy(client, np.ascontiguousarray(np.repeat(sa[:, None], K // 128, 1)), "f32"), None, s, [T, K])
    qw = QuantizedTensor(TensorHandle.from_numpy(client, wc, "f8e4m3"),
                         TensorHandle.from_numpy(client, np.ascontiguousarray(np.repeat(sb[:, :, None], K // 128, 2)), "f32"), None, s,
                         [G, N, K])
    got = run(client, qx, qw, offsets(sizes), "bf16").to_numpy(client)
    got = synth.bf16_bits_to_f32(np.asarray(got).view(np.uint16)).reshape(T, N).astype(np.float64)
    a8 = torch.from_numpy(xc.copy()).view(torch.float8_e4m3fn).cuda()
    b8 = torch.from_numpy(wc.copy()).view(torch.float8_e4m3fn).cuda()
    toffs = torch.tensor(offsets(sizes), dtype=torch.int32).cuda()
    try:
        ref = F.scaled_grouped_mm(a8, b8.transpose(-2, -1), torch.from_numpy(sa).cuda(), F.ScalingType.RowWise,
                                  torch.from_numpy(sb).cuda(), F.ScalingType.RowWise, offs=toffs, output_dtype=torch.bfloat16)
        torch.cuda.synchronize()
    except Exception as e:   # noqa: BLE001 -- an unsupported recipe is reported, not failed
        pytest.skip(f"torch refuses F.scaled_grouped_mm(RowWise, RowWise) here: {type(e).__name__}: {e}")
    t = ref.float().cpu().numpy().astype(np.float64)
    ex = (xq * sa[:, None]).astype(np.float64)
    lo = 0
    for g, n in enumerate(sizes):
        ew = (wq[g] * sb[g][:, None]).astype(np.float64)
        mag = np.abs(ex[lo:lo + n]) @ np.abs(ew).T
        assert np.all(np.abs(got[lo:lo + n] - t[lo:lo + n]) <= 2.0 ** -10 * mag + 2.0 ** -7 * np.abs(t[lo:lo + n])), g
        lo += n
