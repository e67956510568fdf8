"""GPU parity: b200_quantize / b200_dequantize through the C ABI against the reference's known answers and the numpy oracle
(tests/quant_oracle.py), bit for bit, and the bridge into the block-scaled matmul."""
import json
from pathlib import Path

import numpy as np
import pytest

import oracle
import quant_oracle as qo
from cubecl_b200 import TensorHandle, matmul, quant, reduce, synth
from cubecl_b200.quant import QuantScheme, QuantizedTensor

pytestmark = pytest.mark.gpu

REF_DTYPES = {"F32": "f32", "F16": "f16", "BF16": "bf16", "UE4M3": "ue4m3", "UE8M0": "ue8m0"}


@pytest.fixture(scope="module")
def golden():
    return json.loads((Path(__file__).resolve().parent / "golden" / "quant_golden.json").read_text())


def _upload(client, x, dtype):
    dev = synth.to_device_dtype(np.asarray(x, dtype=np.float32), dtype)
    return TensorHandle.from_numpy(client, dev, dtype), synth.from_device_dtype(dev, dtype).reshape(np.shape(x))


def _read(client, q: QuantizedTensor):
    v = q.values.to_numpy(client).view(np.uint8).reshape(q.values.shape)
    s = q.block_scales.to_numpy(client).reshape(q.block_scales.shape) if q.block_scales is not None else None
    if s is not None and q.scheme.block_scale in ("ue4m3", "ue8m0"):
        s = s.view(np.uint8)
    t = np.float32(q.tensor_scale.to_numpy(client)[0]) if q.tensor_scale is not None else None
    return v, s, t


def _check_parity(client, x_dev_handle, vals, scheme):
    q = quant.quantize(client, x_dev_handle, scheme)
    client.sync()
    v, s, t = _read(client, q)
    ev, es, et = qo.quantize(vals, scheme)
    assert np.array_equal(v, ev), ("codes", scheme, np.argwhere(v != ev)[:5])
    if es is not None:
        assert np.array_equal(s.view(np.uint8), np.ascontiguousarray(es).view(np.uint8)), ("scales", scheme)
    if et is not None:
        assert t.view(np.uint32) == et.view(np.uint32), ("tensor scale", scheme, t, et)
    return q


def _kat(kat):
    value = kat["value"].lower()
    values = qo.words_to_bytes(kat["words"])
    i = np.arange(16)
    if kat["block"] == 0:
        scheme = QuantScheme().with_value(value).per_tensor()
        ts = np.float32(kat["tensor_scale"])
        base = np.arange(-8, 8).astype(np.float32) if kat["formula"] == "int_range_times_scale" else synth.e2m1_codes_to_f32(i.astype(np.uint8))
        return scheme, values, None, ts, (base * ts).astype(np.float32)
    dt = REF_DTYPES[kat["block_scale"]]
    scheme = QuantScheme().per_block(kat["block"], dt).per_tensor().with_value(value)
    g = np.float32(np.ldexp(1.0, kat["global_scale_pow2"]))
    bs = np.array(kat["block_scales"], dtype=np.float32)
    exp = ((g * bs[i // kat["block"]]).astype(np.float32) * (i - 8).astype(np.float32)).astype(np.float32)
    return scheme, values, qo.scale_store(dt, bs), g, exp


# ---------------------------------------------------------------------------------------------- reference vectors
@pytest.mark.parametrize("out_dtype", ["f32", "f16", "bf16"])
@pytest.mark.parametrize("name", ["test_quantized_per_tensor_int", "test_quantized_per_tensor_fp4", "test_quantized_global_scale",
                                  "test_quantized_two_level_int", "test_quantized_two_level_ue4m3"])
def test_reference_kats_through_the_cuda_path(client, golden, name, out_dtype):
    scheme, values, scales, ts, exp = _kat(golden["kats"][name])
    vt = TensorHandle.from_numpy(client, values, quant.VALUE_DTYPES.get(scheme.value, "u8"))
    st = TensorHandle.from_numpy(client, np.ascontiguousarray(scales), quant.SCALE_DTYPES[scheme.block_scale]) if scales is not None else None
    q = QuantizedTensor(vt, st, TensorHandle.from_numpy(client, np.array([ts], np.float32), "f32"), scheme, [16])
    got = quant.dequantize(client, q, out_dtype).to_numpy(client)
    assert np.array_equal(got.view(np.uint8), synth.to_device_dtype(exp, out_dtype).view(np.uint8)), (got, exp)


@pytest.mark.parametrize("ref_dt", ["F16", "BF16", "UE4M3", "F32", "UE8M0"])
def test_device_round_up_matches_the_oracle_on_the_probe_grid(client, golden, ref_dt):
    # Q2S has range_max 1, so a block whose absmax is v stores round_up(v) as its scale
    dt = REF_DTYPES[ref_dt]
    spec = golden["round_up_grid"]
    grid = [np.float32(step / spec["step_div"]) * np.float32(2.0 ** e) for e in range(*spec["exp"]) for step in range(*spec["step"])]
    mx = np.float32(golden["scale_dtypes"][ref_dt]["max"])
    with np.errstate(over="ignore"):
        grid += [np.float32(mx * np.float32(m)) for m in spec["max_multipliers"]] + [np.float32(np.finfo(np.float32).max)]
    grid = np.array([g for g in grid if np.isfinite(g)], dtype=np.float32)   # absmax only takes finite inputs
    x = np.zeros((len(grid), 8), np.float32)
    x[:, 3] = grid
    t, _ = _upload(client, x, "f32")
    q = quant.quantize(client, t, QuantScheme().with_value("q2s").per_block(8, dt))
    client.sync()
    _, s, _ = _read(client, q)
    got = qo.scale_load(dt, s.reshape(-1))
    assert np.array_equal(got.view(np.uint32), qo.round_up(dt, grid).view(np.uint32))
    if ref_dt in golden["round_up_grid"]["dtypes"]:
        assert np.all(got >= np.minimum(grid, mx))


# ---------------------------------------------------------------------------------------------- quantize parity
SCHEMES = [("per_block", dt) for dt in ("f32", "f16", "bf16", "ue8m0", "ue4m3")] + [("two_level", "f16"), ("two_level", "ue4m3"),
                                                                                   ("per_tensor", None)]


def _scheme(value, kind, dt, block=32):
    s = QuantScheme().with_value(value)
    if kind == "per_tensor":
        return s.per_tensor()
    s = s.per_block(block, dt)
    return s.per_tensor() if kind == "two_level" else s


@pytest.mark.parametrize("in_dtype", ["f32", "f16", "bf16"])
@pytest.mark.parametrize("value", list(quant.VALUES))
def test_quantize_parity_every_scheme(client, value, in_dtype):
    x = synth.uniform_f32(100 + quant.VALUES[value], 6 * 128, -5.0, 5.0).reshape(6, 128)
    x[1] *= 1e-3    # blocks of different magnitudes
    x[2, :16] = 0   # a zero block
    t, vals = _upload(client, x, in_dtype)
    for kind, dt in SCHEMES:
        for block in ((8, 16, 32, 64, 128) if kind == "per_block" and dt == "f16" else (32,)):
            _check_parity(client, t, vals, _scheme(value, kind, dt, block))


@pytest.mark.parametrize("shape,block", [([5], 0), ([7, 96], 32), ([3, 5, 64], 16), ([1, 1, 1024], 128), ([1000, 24], 8), ([2, 3, 10], 0)])
@pytest.mark.parametrize("in_dtype", ["f32", "bf16"])
def test_quantize_ragged_shapes(client, shape, block, in_dtype):
    x = synth.uniform_f32(77, int(np.prod(shape)), -2.0, 2.0).reshape(shape)
    t, vals = _upload(client, x, in_dtype)
    for value in ("q8s", "e4m3", "e2m1", "q2f"):
        if shape[-1] * quant.BITS[value] % 8:
            continue
        scheme = QuantScheme().with_value(value).per_tensor() if block == 0 else QuantScheme().with_value(value).per_block(block, "ue8m0")
        _check_parity(client, t, vals, scheme)
        if block:
            _check_parity(client, t, vals, scheme.per_block(block, "ue4m3").per_tensor())


def test_views_in_place_and_gathered(client):
    rows, K, pitch = 64, 64, 96
    base = synth.uniform_f32(3, rows * pitch, -1.0, 1.0).reshape(rows, pitch)
    dev = synth.to_device_dtype(base, "bf16")
    vals = synth.from_device_dtype(dev, "bf16").reshape(rows, pitch)
    full = TensorHandle.from_numpy(client, dev, "bf16")
    for scheme in (QuantScheme.mxfp8(), QuantScheme.nvfp4(), QuantScheme().with_value("q4s").per_tensor()):
        n_launch = 1 if scheme.block and not scheme.tensor else 2
        # pitched rows, 16-byte aligned: read in place
        view = TensorHandle(full.handle, [rows, K], [pitch, 1], "bf16")
        before = client.launch_count()
        q = _check_parity(client, view, vals[:, :K], scheme)
        assert client.launch_count() - before == n_launch
        # base shifted by one element: gathered first, exactly one extra launch, same bits as the compact input
        shifted = TensorHandle(full.handle.offset(2), [rows, K], [pitch, 1], "bf16")
        before = client.launch_count()
        _check_parity(client, shifted, vals[:, 1:K + 1], scheme)
        assert client.launch_count() - before == n_launch + 1
        # a transposed view: gathered first
        tr = TensorHandle(full.handle, [K, rows], [1, pitch], "bf16")
        before = client.launch_count()
        _check_parity(client, tr, np.ascontiguousarray(vals[:, :K].T), scheme)
        assert client.launch_count() - before == n_launch + 1
        del q


@pytest.mark.parametrize("value", ["q8f", "q4f", "q2f", "q8s", "q4s", "q2s"])
def test_round_trip_bound(client, value):
    x = synth.uniform_f32(9, 16 * 256, -3.0, 3.0).reshape(16, 256)
    t, vals = _upload(client, x, "f32")
    for scheme in (QuantScheme().with_value(value).per_tensor(), QuantScheme().with_value(value).per_block(32, "f16"),
                   QuantScheme().with_value(value).per_block(16, "ue4m3").per_tensor()):
        q = quant.quantize(client, t, scheme)
        back = quant.dequantize(client, q, "f32").to_numpy(client).reshape(x.shape)
        v, s, ts = _read(client, q)
        eff = qo.effective_scale(scheme, 256, (16,), s, ts)
        assert np.all(np.abs(back - vals) <= eff / 2 * np.float32(1 + 2.0 ** -20)), scheme   # up to the f32 roundings
        for odt in ("f32", "f16", "bf16"):
            got = quant.dequantize(client, q, odt).to_numpy(client).reshape(x.shape)
            assert np.array_equal(got.view(np.uint8), qo.dequantize(v, scheme, x.shape, s, ts, odt).reshape(x.shape).view(np.uint8))


def test_non_finite_rule(client):
    x = synth.uniform_f32(4, 4 * 32, -1.0, 1.0).reshape(4, 32)
    x[0, 1], x[0, 2], x[0, 3] = np.inf, -np.inf, np.nan
    x[1, :] = np.nan                     # a block with no finite value: scale 0, every code 0
    x[2, 5] = -np.nan
    t, vals = _upload(client, x, "f32")
    for value in ("q8s", "q4f", "e4m3", "e5m2", "e2m1"):
        for scheme in (QuantScheme().with_value(value).per_block(32, "f16"), QuantScheme().with_value(value).per_tensor(),
                       QuantScheme().with_value(value).per_block(16, "ue4m3").per_tensor()):
            _check_parity(client, t, vals, scheme)
        q = quant.quantize(client, t, QuantScheme().with_value(value).per_block(32, "f32"))
        v, s, _ = _read(client, q)
        f = qo.unpack(v, quant.BITS[value], 32)
        nan_code = 0x7F if value in ("e4m3", "e5m2") else 0
        assert f[0, 3] == nan_code and f[2, 5] == nan_code and np.all(f[1] == 0) and s[1] == 0
        lo, hi = qo.RANGE[value]
        dec = qo.decode(f[0, 1:3], value)
        assert dec[0] == hi and dec[1] == lo          # +-inf saturates to the range end


def test_determinism(client):
    x = synth.uniform_f32(12, 4096 * 512, -4.0, 4.0).reshape(4096, 512)
    t, _ = _upload(client, x, "bf16")
    for scheme in (QuantScheme.nvfp4(), QuantScheme().with_value("q8s").per_tensor()):
        a, b = _read(client, quant.quantize(client, t, scheme)), _read(client, quant.quantize(client, t, scheme))
        assert all(np.array_equal(np.atleast_1d(p).view(np.uint8), np.atleast_1d(r).view(np.uint8)) for p, r in zip(a, b) if p is not None)


def test_full_size_mxfp8(client):
    M = K = 8192
    buf = TensorHandle.empty_contiguous(client, [M, K], "bf16")
    client.fill_uniform(buf.handle, "bf16", M * K, 2024, -3.0, 3.0)
    q = quant.quantize(client, buf, QuantScheme.mxfp8())
    client.sync()
    vals = synth.bf16_bits_to_f32(buf.to_numpy(client)).reshape(M, K)
    v, s, _ = _read(client, q)
    for r0 in range(0, M, 1024):   # every code and scale, a slab of rows at a time
        ev, es, _ = qo.quantize(vals[r0:r0 + 1024], QuantScheme.mxfp8())
        assert np.array_equal(v[r0:r0 + 1024], ev) and np.array_equal(s[r0:r0 + 1024], es), r0
    back = quant.dequantize(client, q, "bf16").to_numpy(client).reshape(M, K)
    rows = np.arange(0, M, 97)
    assert np.array_equal(back[rows], qo.dequantize(v[rows], QuantScheme.mxfp8(), (len(rows), K), s[rows], None, "bf16").reshape(len(rows), K))


# ---------------------------------------------------------------------------------------------- the bridge into the matmul
@pytest.mark.parametrize("kind", ["mxfp8", "mxfp4", "e2m1_16_ue4m3"])
def test_quantized_operands_feed_the_scaled_matmul(client, kind):
    M, N, K = 256, 192, 512
    scheme = {"mxfp8": QuantScheme.mxfp8(), "mxfp4": QuantScheme.mxfp4(),
              "e2m1_16_ue4m3": QuantScheme().with_value("e2m1").per_block(16, "ue4m3")}[kind]
    sb = scheme.block
    ta, a = _upload(client, synth.uniform_f32(31, M * K, -2.0, 2.0).reshape(M, K), "bf16")
    tb, b = _upload(client, synth.uniform_f32(32, N * K, -2.0, 2.0).reshape(N, K), "bf16")
    qa, qb = quant.quantize(client, ta, scheme), quant.quantize(client, tb, scheme)
    out = TensorHandle.empty_contiguous(client, [M, N], "f32")
    matmul.launch_scaled(client, qa.values, qb.values, qa.block_scales, qb.block_scales, out, scale_block=sb)
    got = out.to_numpy(client).reshape(M, N)
    # the same launch on operands quantized by the oracle on the host
    (va, sa, _), (vb, sbb, _) = qo.quantize(a, scheme), qo.quantize(b, scheme)
    vdt, sdt = quant.VALUE_DTYPES[scheme.value], quant.SCALE_DTYPES[scheme.block_scale]
    host = TensorHandle.empty_contiguous(client, [M, N], "f32")
    matmul.launch_scaled(client, TensorHandle.from_numpy(client, va, vdt), TensorHandle.from_numpy(client, vb, vdt),
                         TensorHandle.from_numpy(client, sa, sdt), TensorHandle.from_numpy(client, sbb, sdt), host, scale_block=sb)
    assert np.array_equal(got, host.to_numpy(client).reshape(M, N))
    # and within the scaled matmul's tolerance of its oracle
    if scheme.value == "e4m3":
        fa, fb = synth.fp8_bits_to_f32(va, "f8e4m3"), synth.fp8_bits_to_f32(vb, "f8e4m3")
    else:
        fa, fb = synth.e2m1_codes_to_f32(synth.unpack_e2m1x2(va)), synth.e2m1_codes_to_f32(synth.unpack_e2m1x2(vb))
    _, f64, fabs = oracle.matmul_scaled(fa, fb, qo.scale_load(scheme.block_scale, sa), qo.scale_load(scheme.block_scale, sbb), sb)
    assert float(np.max(np.abs(got - f64) / fabs)) <= 2e-6


def test_stream_order_and_pool(client):
    # quantize reading a reduce-free input, dequantize feeding a reduce, on the client's stream; temporaries go back to the pool
    shape = [2048, 1024]
    x = synth.uniform_f32(55, int(np.prod(shape)), -1.0, 1.0).reshape(shape)
    t, vals = _upload(client, x, "f32")
    q = quant.alloc_quantized(client, shape, QuantScheme.nvfp4())
    y = TensorHandle.empty_contiguous(client, shape, "f32")
    r = TensorHandle.empty_contiguous(client, [shape[0]], "f32")
    client.sync()
    base = client.memory_usage().bytes_in_use
    quant.launch_quantize(client, t, q)
    quant.launch_dequantize(client, q, y)
    reduce.launch(client, y, r, 1, "sum")                        # reads the dequantized output
    quant.launch_quantize(client, y, q)                          # overwrites q after the reduce's read of y
    client.sync()
    assert client.memory_usage().bytes_in_use == base
    v0, s0, t0 = qo.quantize(vals, QuantScheme.nvfp4())
    y_exp = qo.dequantize(v0, QuantScheme.nvfp4(), shape, s0, t0)
    assert np.array_equal(y.to_numpy(client).reshape(shape), y_exp)
    assert np.all(np.abs(r.to_numpy(client) - oracle.reduce_f64(y_exp, 1, "sum")) <= 1e-5 * oracle.reduce_f64(np.abs(y_exp), 1, "sum") + 1e-30)
    v1, s1, t1 = qo.quantize(y_exp, QuantScheme.nvfp4())
    v, s, ts = _read(client, q)
    assert np.array_equal(v, v1) and np.array_equal(s, s1) and ts == t1
