"""GPU parity: axis scans (cumsum / cumprod / cummax / cummin) through the C ABI vs the reference vectors and the oracle."""
import json
from pathlib import Path

import numpy as np
import pytest

import oracle
from cubecl_b200 import TensorHandle, reduce, scan, synth
from scan_oracle import scan_axis_f32, scan_axis_f64

pytestmark = pytest.mark.gpu

TYPE_EPS = {"f32": float(np.finfo(np.float32).eps), "f16": float(np.finfo(np.float16).eps), "bf16": 2.0 ** -7}


@pytest.fixture(scope="module")
def scan_golden():
    """The reference's plane-scan vectors (tests/golden/make_scan_golden.py)."""
    return json.loads((Path(__file__).resolve().parent / "golden" / "scan_golden.json").read_text())


def _upload(client, x, dtype="f32"):
    dev = synth.to_device_dtype(np.asarray(x, dtype=np.float32), dtype)
    return TensorHandle.from_numpy(client, dev, dtype), synth.from_device_dtype(dev, dtype).reshape(np.shape(x))


def _scan(client, t, axis, op="sum", exclusive=False, out_dtype="f32"):
    out = scan.launch_alloc(client, t, axis, op, exclusive, out_dtype)
    return synth.from_device_dtype(out.to_numpy(client), out_dtype).reshape(t.shape)


def mod8_prefix_sum(index):
    """sum_{i <= l} (i % 8), closed form."""
    l = np.asarray(index, dtype=np.int64)
    return (l + 1) // 8 * 28 + ((l + 1) % 8) * ((l + 1) % 8 - 1) // 2


# ---------------------------------------------------------------------------------------------- reference vectors
@pytest.mark.parametrize("dtype", ["f32", "f16", "bf16"])
@pytest.mark.parametrize("kind", ["inclusive_sum", "exclusive_sum", "inclusive_prod", "exclusive_prod"])
@pytest.mark.parametrize("vec", [1, 2, 4])
def test_plane_scan_goldens_through_the_cuda_path(client, scan_golden, dtype, kind, vec):
    # plane.rs:191-405 (vectorisation 1 / 2 / 4): 32 lanes x vec values; lane k holds the scan over lanes of its vector
    # slot -- the [32, vec] tensor scanned along the lane axis, in and out in the element type
    g = scan_golden[f"plane_{kind}"]
    n = 32 * vec
    if g["generator"] == "index":
        x = np.arange(n, dtype=np.float32)
    else:
        x = np.array([(0.5, 1.25, 1.75)[i % 3] for i in range(n)], dtype=np.float32)
    t, _ = _upload(client, x.reshape(32, vec), dtype)
    got = _scan(client, t, 0, g["op"], g["exclusive"], dtype).ravel().astype(np.float64)
    exp = np.array(g["expected"][str(vec)], dtype=np.float32).astype(np.float64)
    # assert_equals_approx (runtime_tests/binary.rs:15-53): epsilon normalised to the element type
    eps = max(g["epsilon"] / TYPE_EPS["f32"] * TYPE_EPS[dtype], g["epsilon"])
    assert np.all(np.abs(got - exp) < np.maximum(eps * np.abs(exp), eps)), (got, exp)


# ---------------------------------------------------------------------------------------------- exact integer pattern
INT_CASES = [
    ([1000, 3], 1, "rows, one thread per row"),
    ([300, 1000], 1, "rows, sub-warp groups"),
    ([64, 20000], 1, "rows, a block per row"),
    ([2, 1 << 22], 1, "rows, three-pass"),
    ([300, 64, 40], 1, "columns, vector units"),
    ([50, 1000, 7], 1, "columns, scalar units"),
    ([8192, 2048], 0, "columns, three-pass"),
    ([1 << 20, 4], 0, "columns, three-pass, few outputs"),
]


@pytest.mark.parametrize("shape,axis,family", INT_CASES)
def test_integer_pattern_exact(client, shape, axis, family):
    # x[i] = i % 8 with every prefix below 2^24: exact integers in any summation order
    x = (np.arange(int(np.prod(shape))) % 8).astype(np.float32).reshape(shape)
    t, _ = _upload(client, x)
    for exclusive in (False, True):
        got = _scan(client, t, axis, "sum", exclusive)
        assert np.array_equal(got, scan_axis_f32(x, axis, "sum", exclusive)), (family, exclusive)


def test_integer_pattern_views(client):
    # pitched rows (TensorHandle::empty) in place, an element-aligned base, and a transposed view (gathered first)
    rows, cols = 100, 72
    x = (np.arange(rows * cols) % 8).astype(np.float32).reshape(rows, cols)
    t = TensorHandle.empty(client, [rows, cols], "f32")
    assert t.strides[0] > cols
    host = np.full((rows, t.strides[0]), 1e30, dtype=np.float32)      # the padding must never be read
    host[:, :cols] = x
    client.write(t.handle, host)
    for axis in (0, 1):
        for exclusive in (False, True):
            before = client.launch_count()
            got = _scan(client, t, axis, "sum", exclusive)
            assert client.launch_count() - before == 1
            assert np.array_equal(got, scan_axis_f32(x, axis, "sum", exclusive)), (axis, exclusive)
    r2, c2 = 257, 2041                                                  # odd rows: every row starts at another alignment
    n = r2 * c2
    flat = (np.arange(n + 3) % 8).astype(np.float32)
    whole = client.create_from_slice(flat)
    for off in (1, 3):
        view = TensorHandle.new_contiguous([r2, c2], whole.offset(off * 4, n * 4), "f32")
        x2 = flat[off:off + n].reshape(r2, c2)
        for axis in (0, 1):
            for exclusive in (False, True):
                assert np.array_equal(_scan(client, view, axis, "sum", exclusive), scan_axis_f32(x2, axis, "sum", exclusive)), (off, axis)
    tt = TensorHandle.from_numpy(client, x, "f32").transposed()          # logical [cols, rows]
    for axis in (0, 1):
        for exclusive in (False, True):
            got = _scan(client, tt, axis, "sum", exclusive)
            assert np.array_equal(got, scan_axis_f32(np.ascontiguousarray(x.T), axis, "sum", exclusive)), (axis, exclusive)


# ---------------------------------------------------------------------------------------------- random data
RANDOM_CASES = [([512, 8192], 1), ([64, 20000], 1), ([2, 1 << 22], 1), ([255, 20000], 0), ([4096, 512], 0), ([30, 500, 33], 1)]


@pytest.mark.parametrize("shape,axis", RANDOM_CASES)
@pytest.mark.parametrize("exclusive", [False, True])
def test_random_sum_vs_f64(client, shape, axis, exclusive):
    x = synth.uniform_f32(61, int(np.prod(shape)), -1.0, 1.0).reshape(shape)
    t, vals = _upload(client, x)
    got = _scan(client, t, axis, "sum", exclusive).astype(np.float64)
    ref, pabs = scan_axis_f64(vals, axis, "sum", exclusive)
    serial = scan_axis_f32(vals, axis, "sum", exclusive)
    err = np.abs(got - ref)
    # per line along the axis: never much worse than the reference's own serial order
    line_err = err.max(axis=axis)
    serial_err = np.abs(serial.astype(np.float64) - ref).max(axis=axis)
    total_abs = np.take(pabs, [-1], axis=axis).squeeze(axis) + np.take(np.abs(vals), [-1], axis=axis).squeeze(axis) * exclusive
    assert np.all(line_err <= serial_err + 1e-6 * total_abs)
    assert np.all(err <= 1e-3 * pabs + 1e-30)                             # north-star bound, element by element
    if (shape, axis) == ([255, 20000], 0):                                # unsegmented columns: exactly the serial order
        assert np.array_equal(got.astype(np.float32), serial)


@pytest.mark.parametrize("op", ["max", "min"])
def test_max_min_exact_with_special_values(client, op):
    for shape, axis in (([64, 5000], 1), ([5000, 64], 0), ([1 << 16, 8], 0), ([3, 1 << 18], 1)):
        x = synth.uniform_f32(71, int(np.prod(shape)), -1.0, 1.0).reshape(shape)
        m = np.moveaxis(x, axis, -1)                                      # a view: plant values along the axis
        L = m.shape[-1]
        m[..., L // 3] = np.inf
        m[..., L // 5] = -np.inf
        m[..., L // 7] = 0.0
        m[..., L // 7 + 1] = -0.0
        m[1, ...] = -0.0
        m[0, L // 2] = np.nan                                             # every later output of line 0 is NaN
        t, vals = _upload(client, x)
        for exclusive in (False, True):
            got = _scan(client, t, axis, op, exclusive)
            exp = scan_axis_f32(vals, axis, op, exclusive)
            assert np.array_equal(got, exp, equal_nan=True), (shape, axis, exclusive)
            assert np.isnan(np.moveaxis(got, axis, -1)[0, L // 2 + 1:]).all()


def test_prod_vs_f64(client):
    for shape, axis in (([64, 5000], 1), ([5000, 64], 0), ([40, 3000, 9], 1)):
        x = synth.uniform_f32(81, int(np.prod(shape)), 0.99, 1.01).reshape(shape)
        t, vals = _upload(client, x)
        for exclusive in (False, True):
            got = _scan(client, t, axis, "prod", exclusive)
            ref, _ = scan_axis_f64(vals, axis, "prod", exclusive)
            # each of the <= 5000 f32 products rounds by <= 2^-24: 5000 * 6e-8 = 3e-4 worst case
            assert np.allclose(got, ref, rtol=5e-4, atol=0), (shape, axis, exclusive)


@pytest.mark.parametrize("dtype", ["f16", "bf16"])
def test_16bit_output_is_the_f32_run_rounded(client, dtype):
    for shape, axis, op in (([64, 5000], 1, "sum"), ([5000, 64], 0, "sum"), ([300, 40, 16], 1, "max"), ([2, 1 << 22], 1, "sum")):
        x = synth.uniform_f32(91, int(np.prod(shape)), -1.0, 1.0).reshape(shape)
        t, _ = _upload(client, x, dtype)
        for exclusive in (False, True):
            f32 = _scan(client, t, axis, op, exclusive, "f32")
            o16 = scan.launch_alloc(client, t, axis, op, exclusive, dtype).to_numpy(client).reshape(shape)
            assert np.array_equal(o16, synth.to_device_dtype(f32, dtype)), (shape, axis, op, exclusive)


def test_three_pass_is_deterministic(client):
    for shape, axis in (([2, 1 << 22], 1), ([8192, 2048], 0)):
        x = synth.uniform_f32(101, int(np.prod(shape)), -1.0, 1.0).reshape(shape)
        t, _ = _upload(client, x)
        a = scan.launch_alloc(client, t, axis, "sum").to_numpy(client)
        b = scan.launch_alloc(client, t, axis, "sum").to_numpy(client)
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), shape


def test_cumsum_2pow28_closed_form(client):
    n = 1 << 28
    t = TensorHandle.empty_contiguous(client, [n], "f32")
    client.fill_modulo(t.handle, "f32", n, 8)
    got = scan.launch_alloc(client, t, 0, "sum").to_numpy(client)
    idx = np.unique(np.concatenate([np.random.default_rng(5).integers(0, n, 4096), [n - 1]]))
    exp = mod8_prefix_sum(idx).astype(np.float64)
    assert np.all(np.abs(got[idx].astype(np.float64) - exp) <= 1e-6 * np.maximum(exp, 1.0))
    assert abs(float(got[-1]) - 939524096.0) <= 1e-6 * 939524096.0
    del got
    cm = scan.launch_alloc(client, t, 0, "max").to_numpy(client)
    assert cm[:7].tolist() == list(range(7)) and bool(np.all(cm[7:] == 7.0))


def test_stream_order_and_pool(client):
    # a scan feeding a reduce and a reduce feeding a scan on the client's stream give the serial-execution results, and
    # the three-pass temporaries go back to the pool
    shape = [8192, 2048]
    x = synth.uniform_f32(111, int(np.prod(shape)), -1.0, 1.0).reshape(shape)
    t, vals = _upload(client, x)
    y = TensorHandle.empty_contiguous(client, shape, "f32")
    s = TensorHandle.empty_contiguous(client, [shape[1]], "f32")
    r = TensorHandle.empty_contiguous(client, [shape[0]], "f32")
    z = TensorHandle.empty_contiguous(client, [shape[0]], "f32")
    client.sync()
    base = client.memory_usage().bytes_in_use
    scan.launch(client, t, y, 0, "max")
    reduce.launch(client, y, s, 0, "sum")                                 # reads the scan's output
    reduce.launch(client, t, r, 1, "max")
    scan.launch(client, r, z, 0, "sum", exclusive=True)                  # reads the reduce's output
    client.sync()
    assert client.memory_usage().bytes_in_use == base
    y_exp = scan_axis_f32(vals, 0, "max")
    assert np.array_equal(y.to_numpy(client).reshape(shape), y_exp)
    assert np.all(np.abs(s.to_numpy(client) - oracle.reduce_f64(y_exp, 0, "sum")) <= 1e-5 * oracle.reduce_f64(np.abs(y_exp), 0, "sum"))
    r_exp = oracle.reduce(vals, 1, "max")
    assert np.array_equal(r.to_numpy(client), r_exp)
    ref, pabs = scan_axis_f64(r_exp, 0, "sum", True)
    assert np.all(np.abs(z.to_numpy(client) - ref) <= 1e-5 * pabs + 1e-30)
