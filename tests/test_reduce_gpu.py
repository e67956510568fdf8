"""GPU parity: reductions through the C ABI vs the oracle."""
import numpy as np
import pytest

import oracle
from cubecl_b200 import ServerError, TensorHandle, reduce, synth

pytestmark = pytest.mark.gpu


def _run(client, x_f32, axis, op, dtype="f32"):
    dev = synth.to_device_dtype(x_f32, dtype)
    vals = synth.from_device_dtype(dev, dtype).reshape(x_f32.shape)
    t = TensorHandle.from_numpy(client, dev, dtype)
    out = reduce.launch_alloc(client, t, axis, op)
    return out.to_numpy(client), vals


def test_sum_things_kat(client, golden):
    # examples/sum_things/src/lib.rs:180,222-225: [-1,10,1,5] -> 15
    got, _ = _run(client, np.array(golden["sum_things"]["input"], dtype=np.float32), None, "sum")
    assert got.tolist() == [golden["sum_things"]["expected_sum"]]


@pytest.mark.parametrize("variant", ["auto", "u2", "u4", "u16", "b4", "b8", "w2", "w4", "tma"])
@pytest.mark.parametrize("n", [1, 3, 4, 1000, (1 << 20) + 5, (1 << 23) + 4099])
def test_sum_all_integer_pattern_exact(client, variant, n):
    # BASELINE config 1 pattern x[i] = i % 8: every partial is an exact integer, so the result must be exact
    client.set_option("reduce.variant", variant)
    try:
        x = (np.arange(n) % 8).astype(np.float32)
        got, _ = _run(client, x, None, "sum")
        # exact integer partials everywhere; the only rounding is the final f64 -> f32 conversion of the total
        assert float(got[0]) == float(np.float32(x.astype(np.float64).sum()))
    finally:
        client.set_option("reduce.variant", "auto")


@pytest.mark.parametrize("dtype", ["f32", "f16", "bf16"])
def test_sum_all_random_vs_f64(client, dtype):
    n = (1 << 22) + 13
    x = synth.uniform_f32(5, n, 0.0, 1.0)
    got, vals = _run(client, x, None, "sum", dtype)
    ref = oracle.sum_f64(vals)
    serial_err = abs(float(oracle.sum_serial_f32(vals)) - ref)
    gpu_err = abs(float(got[0]) - ref)
    assert gpu_err <= 1e-3 * oracle.sum_abs_f64(vals)      # north-star tolerance
    assert gpu_err <= 1e-6 * oracle.sum_abs_f64(vals)      # what a blocked f32 sum should achieve
    assert gpu_err <= serial_err + 1e-6 * abs(ref)          # never worse than the reference's own serial order


def test_sum_2pow28_exact_and_tolerance(client):
    # BASELINE config 4 at full size, data generated in HBM: (i) i%8 pattern -> 939,524,096 exactly
    n = 1 << 28
    t = TensorHandle.empty_contiguous(client, [n], "f32")
    client.fill_modulo(t.handle, "f32", n, 8)
    out = reduce.launch_alloc(client, t, None, "sum")
    assert float(out.to_numpy(client)[0]) == 939524096.0
    # (ii) U[0,1) seed 5: compare with the f64 sum of the host-regenerated stream (chunked)
    client.fill_uniform(t.handle, "f32", n, 5, 0.0, 1.0)
    out = reduce.launch_alloc(client, t, None, "sum")
    got = float(out.to_numpy(client)[0])
    ref = 0.0
    step = 1 << 24
    for s in range(0, n, step):
        ref += float(synth.uniform_f32(5, step, 0.0, 1.0, start=s).astype(np.float64).sum())
    assert abs(got - ref) <= 1e-6 * ref
    # idempotence: same input, same grid -> bitwise same answer
    out2 = reduce.launch_alloc(client, t, None, "sum")
    assert out2.to_numpy(client)[0] == np.float32(got)


@pytest.mark.parametrize("shape,axis", [([512, 8192], 1), ([128, 32768], 1), ([64, 256, 1024], 2), ([64, 64, 4096], 2),
                                        ([7, 33], 1), ([1000, 3], 1), ([4, 1 << 18], 1), ([5, 1 << 17], 0), ([3, 70, 11], 1),
                                        ([4096, 64], 0), ([2, 3, 4, 5], 2), ([9], 0)])
@pytest.mark.parametrize("op", ["sum", "mean", "max", "min", "prod", "argmax", "argmin"])
def test_axis_reductions(client, shape, axis, op):
    # row-sum shapes are the book's benchmarks (cubecl-book/.../benchmark.md, parallel_reduction*.md)
    n = int(np.prod(shape))
    if op == "prod":
        x = synth.uniform_f32(8, n, 0.9, 1.1).reshape(shape)
    else:
        x = synth.uniform_f32(8, n, -1.0, 1.0).reshape(shape)
    got, vals = _run(client, x, axis, op)
    exp = oracle.reduce(vals, axis, op)
    if op in ("argmax", "argmin", "max", "min"):
        assert np.array_equal(got, exp)
    elif op == "prod":
        assert np.allclose(got, exp, rtol=1e-3)
    else:
        ref = oracle.reduce_f64(vals, axis, op)
        scale = oracle.reduce_f64(np.abs(vals), axis, op)
        assert np.all(np.abs(got - ref) <= 1e-5 * scale + 1e-30)


@pytest.mark.parametrize("dtype", ["f16", "bf16"])
def test_axis_reductions_16bit(client, dtype):
    x = synth.uniform_f32(9, 64 * 1000, -1.0, 1.0).reshape(64, 1000)
    for axis in (0, 1):
        got, vals = _run(client, x, axis, "sum", dtype)
        assert np.allclose(got, oracle.reduce_f64(vals, axis, "sum"), rtol=0, atol=1e-3)
        got, vals = _run(client, x, axis, "argmax", dtype)
        assert np.array_equal(got, oracle.reduce(vals, axis, "argmax"))


def test_argmax_ties_and_nan_rules(client):
    # unpinned by the reference: lowest index among equal maxima; NaN is the extreme and the first NaN wins
    x = np.zeros(100003, dtype=np.float32)
    x[[777, 50000, 99999]] = 7.0
    got, _ = _run(client, x, None, "argmax")
    assert got.tolist() == [777]
    x[60000] = np.nan
    x[90000] = np.nan
    got, _ = _run(client, x, None, "argmax")
    assert got.tolist() == [60000]
    got, _ = _run(client, x, None, "argmin")
    assert got.tolist() == [60000]
    got, _ = _run(client, x, None, "max")
    assert np.isnan(got[0])
    rows = np.array([[1, 5, 5, 2], [np.nan, 9, np.nan, 0], [3, 3, 3, 3]], dtype=np.float32)
    got, vals = _run(client, rows, 1, "argmax")
    assert got.tolist() == oracle.reduce(vals, 1, "argmax").tolist() == [1, 0, 0]
    got, _ = _run(client, rows, 0, "argmin")
    assert got.tolist() == oracle.reduce(rows, 0, "argmin").tolist()


def test_bad_axis_is_deferred(client):
    t = TensorHandle.from_numpy(client, np.ones((4, 4), dtype=np.float32), "f32")
    out = TensorHandle.empty_contiguous(client, [4], "u32")  # wrong output dtype for a sum
    reduce.launch(client, t, out, 1, "sum")
    with pytest.raises(ServerError):
        client.sync()


def test_pitched_and_permuted_inputs(client):
    # TensorHandle::empty pitches rows (allocator.rs:21-72): [100, 72] f32 rows of 288 B pitch to 512 B; the reduce must
    # see the logical tensor -- IN PLACE: one kernel launch per reduction (no into_contiguous gather), padding never read.
    rows, cols = 100, 72
    x = synth.uniform_f32(12, rows * cols, -1.0, 1.0).reshape(rows, cols)
    t = TensorHandle.empty(client, [rows, cols], "f32")
    assert t.strides[0] > cols
    host = np.zeros((rows, t.strides[0]), dtype=np.float32)
    host[:, :cols] = x
    host[:, cols:] = 1e30  # padding must never be read
    client.write(t.handle, host)
    for axis in (0, 1, None):
        for op in ("sum", "argmax", "max"):
            out = TensorHandle.empty_contiguous(client, reduce.output_shape([rows, cols], axis), reduce.output_dtype(op))
            before = client.launch_count()
            reduce.launch(client, t, out, axis, op)
            assert client.launch_count() - before == 1, (axis, op)
            got = out.to_numpy(client)
            if op == "sum":
                assert np.allclose(got, oracle.reduce_f64(x, axis, "sum"), rtol=0, atol=1e-4)
            else:
                assert np.array_equal(got, oracle.reduce(x, axis, op)), (axis, op)
    # a transposed (stride-swapped) view: reducing its last axis is a column reduction of the buffer, again one launch
    tt = TensorHandle.from_numpy(client, x, "f32").transposed()          # logical [cols, rows]
    for axis, op in ((1, "max"), (0, "sum"), (1, "argmin"), (None, "sum")):
        out = TensorHandle.empty_contiguous(client, reduce.output_shape([cols, rows], axis), reduce.output_dtype(op))
        before = client.launch_count()
        reduce.launch(client, tt, out, axis, op)
        assert client.launch_count() - before == 1, (axis, op)
        got = out.to_numpy(client)
        if op == "sum":
            assert np.allclose(got, oracle.reduce_f64(np.ascontiguousarray(x.T), axis, "sum"), rtol=0, atol=1e-4)
        else:
            assert np.array_equal(got, oracle.reduce(np.ascontiguousarray(x.T), axis, op)), (axis, op)
    # views nothing but a gather describes still work: flat argmax of a transposed view (the index is logical)
    got = reduce.launch_alloc(client, tt, None, "argmax").to_numpy(client)
    assert got.tolist() == [int(np.argmax(x.T))]


@pytest.mark.parametrize("dtype", ["f32", "bf16"])
def test_pitched_rank3_and_unaligned_pitch(client, dtype):
    # rank 3 with a pitched last-but-one dimension (outer strides compact over the pitch), every axis and every element; and a
    # row length / pitch that is NOT a multiple of the 128-bit vector (scalar path of the pitched kernels)
    esz = 4 if dtype == "f32" else 2
    for shape in ([6, 50, 72], [5, 33, 7]):
        t = TensorHandle.empty(client, shape, dtype)
        pitch = t.strides[1]
        assert t.strides == [shape[1] * pitch, pitch, 1]
        vals = synth.uniform_f32(21, int(np.prod(shape)), -1.0, 1.0).reshape(shape)
        dev = synth.to_device_dtype(vals, dtype)
        x = synth.from_device_dtype(dev, dtype).reshape(shape)
        host = np.full((shape[0], shape[1], pitch), synth.to_device_dtype(np.array([3e4], np.float32), dtype)[0], dtype=dev.dtype)
        host[:, :, :shape[2]] = dev.reshape(shape)
        assert host.nbytes <= t.handle.size and host.dtype.itemsize == esz
        client.write(t.handle, host)
        for axis in (0, 1, 2, None):
            for op in ("sum", "argmax"):
                out = TensorHandle.empty_contiguous(client, reduce.output_shape(shape, axis), reduce.output_dtype(op))
                before = client.launch_count()
                reduce.launch(client, t, out, axis, op)
                assert client.launch_count() - before == 1, (shape, axis, op)
                got = out.to_numpy(client)
                if op == "sum":
                    assert np.allclose(got, oracle.reduce_f64(x, axis, "sum"), rtol=0, atol=2e-4), (shape, axis)
                else:
                    assert np.array_equal(got, oracle.reduce(x, axis, op)), (shape, axis)


@pytest.mark.parametrize("dtype,offset", [("f32", 1), ("f32", 2), ("f32", 3), ("bf16", 1), ("bf16", 5), ("f16", 7)])
def test_offset_views_need_element_alignment_only(client, dtype, offset):
    # a sub-slice view (Handle::offset) starts on an element boundary, not a 16-byte one: the all / rows / columns kernels and
    # their wide / bulk variants peel a scalar head instead of issuing a misaligned vector load (which would be a sticky fault)
    esz = 4 if dtype == "f32" else 2
    n = (1 << 19) + 301                                                  # >= 257 * 2041, the row / column case below
    vals = synth.uniform_f32(31, n + offset, -1.0, 1.0)
    dev = synth.to_device_dtype(vals, dtype)
    x = synth.from_device_dtype(dev, dtype)[offset:]
    whole = client.create_from_slice(dev)
    view = TensorHandle.new_contiguous([n], whole.offset(offset * esz, n * esz), dtype)
    for variant in ("auto", "w2", "w4", "b8", "tma") if dtype == "f32" else ("auto", "tma"):
        client.set_option("reduce.variant", variant)
        try:
            got = reduce.launch_alloc(client, view, None, "sum").to_numpy(client)
        finally:
            client.set_option("reduce.variant", "auto")
        assert abs(float(got[0]) - oracle.sum_f64(x)) <= 1e-6 * oracle.sum_abs_f64(x), variant
    for op in ("argmax", "argmin", "max"):
        got = reduce.launch_alloc(client, view, None, op).to_numpy(client)
        assert np.array_equal(got, oracle.reduce(x, None, op).reshape(got.shape)), op
    rows, cols = 257, 2041                                               # odd row length: every row starts at a different alignment
    v2 = TensorHandle.new_contiguous([rows, cols], whole.offset(offset * esz, rows * cols * esz), dtype)
    x2 = x[:rows * cols].reshape(rows, cols)
    for axis in (0, 1):
        got = reduce.launch_alloc(client, v2, axis, "sum").to_numpy(client)
        assert np.allclose(got, oracle.reduce_f64(x2, axis, "sum"), rtol=0, atol=2e-3 if dtype != "f32" else 5e-4), axis
        got = reduce.launch_alloc(client, v2, axis, "argmin").to_numpy(client)
        assert np.array_equal(got, oracle.reduce(x2, axis, "argmin")), axis
    client.sync()


@pytest.mark.parametrize("dtype", ["f32", "f16", "bf16"])
@pytest.mark.parametrize("vec", [1, 2, 4])
def test_plane_sum_golden_through_the_cuda_path(client, golden, dtype, vec):
    # crates/cubecl-core/src/runtime_tests/plane.rs:154-189 (test_plane_sum, vectorisation 1 / 2 / 4): 32 lanes x vec values =
    # flat index; every lane ends up with expected[v] = sum_k input[v + k * vec] (vec 1: 496).  On this path plane_sum is the
    # warp stage of the reduction, so the KAT is the [32, vec] tensor reduced over the lane axis.
    assert vec in golden["plane_sum"]["vec_sizes"]
    inp = np.arange(32 * vec, dtype=np.float32).reshape(32, vec)
    got, _ = _run(client, inp, 0, "sum", dtype)
    exp = np.array([sum(v + k * vec for k in range(32)) for v in range(vec)], dtype=np.float32)
    assert got.tolist() == exp.tolist()
    if vec == 1:
        assert got.tolist() == [496.0]
        got_all, _ = _run(client, inp, None, "sum", dtype)               # the same 32 values through the all-elements kernel
        assert got_all.tolist() == [496.0]


def test_back_to_back_reductions_overlap_safely(client):
    # consecutive all-element reductions on the client's stream overlap (programmatic dependent launch: the next launch
    # streams its input while the previous one's last block finishes).  Results must be what serial execution gives:
    # alternating inputs and outputs, the shared workspace reused every launch, and a chain whose input IS the previous
    # output (that pair must not overlap)
    n = (1 << 24) + 1024
    xs, exp = [], []
    for i in range(3):
        x = ((np.arange(n) + i) % (5 + i)).astype(np.float32)
        xs.append(TensorHandle.from_numpy(client, x, "f32"))
        exp.append(float(np.float32(x.astype(np.float64).sum())))
    outs = [TensorHandle.empty_contiguous(client, [1], "f32") for _ in range(60)]
    aouts = [TensorHandle.empty_contiguous(client, [1], "u32") for _ in range(6)]
    for variant in ("auto", "u8"):
        client.set_option("reduce.variant", variant)
        for k, o in enumerate(outs):
            reduce.launch(client, xs[k % 3], o, None, "sum")
        for k, o in enumerate(aouts):
            reduce.launch(client, xs[k % 3], o, None, "argmax")
        client.sync()
        for k, o in enumerate(outs):
            assert float(o.to_numpy(client)[0]) == exp[k % 3], (variant, k)
        for k, o in enumerate(aouts):
            assert int(o.to_numpy(client)[0]) == 4, (variant, k)   # first index holding the largest value of every pattern
    client.set_option("reduce.variant", "auto")
    chain = TensorHandle.empty_contiguous(client, [1], "f32")
    reduce.launch(client, xs[0], outs[0], None, "sum")
    reduce.launch(client, outs[0], chain, None, "sum")      # reads the predecessor's 4-byte result
    assert float(chain.to_numpy(client)[0]) == exp[0]
    client.set_option("reduce.pdl", "off")
    reduce.launch(client, xs[1], outs[1], None, "sum")
    assert float(outs[1].to_numpy(client)[0]) == exp[1]
    client.set_option("reduce.pdl", "on")


def test_arg_reductions_special_values(client):
    # the integer-key form of the arg ops: -0.0 ties with +0.0, infinities order correctly, all-equal / all -inf inputs give
    # index 0, NaN is the extreme for both ops, and long rows and segmented columns agree with the oracle
    x = np.full(70001, -np.inf, dtype=np.float32)
    assert _run(client, x, None, "argmax")[0].tolist() == [0]
    assert _run(client, x, None, "argmin")[0].tolist() == [0]
    x = np.zeros(5000, dtype=np.float32); x[17] = -0.0; x[40] = 0.0
    assert _run(client, x, None, "argmax")[0].tolist() == [0]
    x[:] = -1.0; x[33] = -0.0; x[77] = 0.0
    assert _run(client, x, None, "argmax")[0].tolist() == [33]          # -0.0 == +0.0: the earlier one wins
    x[:] = 1.0; x[33] = 0.0; x[77] = -0.0
    assert _run(client, x, None, "argmin")[0].tolist() == [33]
    x = synth.uniform_f32(3, 4 * (1 << 20), -1.0, 1.0).reshape(4, 1 << 20)     # few long rows (16 MB: one rows launch)
    x[1, 999999] = np.inf; x[2, 5] = -np.inf; x[3, 123456] = np.nan; x[3, 654321] = np.nan
    for op in ("argmax", "argmin"):
        got, vals = _run(client, x, 1, op)
        assert np.array_equal(got, oracle.reduce(vals, 1, op)), op
    y = np.ascontiguousarray(x.T)                                              # [2^20, 4]: long axis, 4 columns -> segmented columns
    for op in ("argmax", "argmin", "sum", "max"):
        got, vals = _run(client, y, 0, op)
        if op == "sum":
            ok = ~np.isnan(oracle.reduce_f64(vals, 0, "sum"))
            assert np.allclose(got[ok], oracle.reduce_f64(vals, 0, "sum")[ok], rtol=1e-4)
        else:
            assert np.array_equal(got, oracle.reduce(vals, 0, op), equal_nan=True), op


@pytest.mark.parametrize("shape,axis", [([3, 40000, 5], 1), ([1, 100003, 64], 1), ([2, 777, 4096], 1), ([100003, 3], 0),
                                        ([7, 20011], 1), ([300, 20011], 1), ([2, 3, 50000], 2), ([100000, 33], 1)])
@pytest.mark.parametrize("op", ["sum", "argmax", "min"])
def test_segmented_and_ragged_axis_reductions(client, shape, axis, op):
    # extents that do not divide the segment / tile / vector sizes: last segments shorter, partial column tiles, scalar tails
    n = int(np.prod(shape))
    x = synth.uniform_f32(41, n, -1.0, 1.0).reshape(shape)
    got, vals = _run(client, x, axis, op)
    if op == "sum":
        ref = oracle.reduce_f64(vals, axis, "sum")
        scale = oracle.reduce_f64(np.abs(vals), axis, "sum")
        assert np.all(np.abs(got - ref) <= 1e-5 * scale + 1e-30)
    else:
        assert np.array_equal(got, oracle.reduce(vals, axis, op))


def test_fuzz_shapes_axes_ops_dtypes(client):
    # 80 seeded random reductions: rank 1-4, any axis or all, every op and input dtype, odd extents (vector tails, short
    # and long rows, split paths) -- value ops vs the f64 oracle, index/extremum ops exactly
    rng = np.random.default_rng(77)
    ops = ["sum", "mean", "max", "min", "prod", "argmax", "argmin"]
    for case in range(80):
        rank = int(rng.integers(1, 5))
        budget = int(rng.choice([300, 5000, 200000, 3000000]))
        shape = []
        for d in range(rank):
            hi = max(2, int(round(budget ** (1.0 / (rank - d)))) * 2)
            ext = int(rng.integers(1, hi))
            shape.append(ext)
            budget = max(1, budget // ext)
        axis = None if rng.random() < 0.2 else int(rng.integers(0, rank))
        op = ops[case % len(ops)]
        dtype = ["f32", "f16", "bf16"][case % 3]
        n = int(np.prod(shape))
        lo, hi = (0.97, 1.03) if op == "prod" else (-1.0, 1.0)
        x = synth.uniform_f32(500 + case, n, lo, hi).reshape(shape)
        if op in ("argmax", "argmin", "max", "min") and n > 8:      # plant ties so the lowest-index rule is exercised
            flat = x.reshape(-1)
            flat[rng.integers(0, n, 4)] = 2.0 if op in ("argmax", "max") else -2.0
        got, vals = _run(client, x, axis, op, dtype)
        exp = oracle.reduce(vals, axis, op)
        tag = (case, shape, axis, op, dtype)
        if op in ("argmax", "argmin", "max", "min"):
            assert np.array_equal(got, exp), tag
        elif op == "prod":
            assert np.allclose(got, oracle.reduce_f64(vals, axis, "prod"), rtol=2e-3), tag
        else:
            ref = oracle.reduce_f64(vals, axis, op)
            scale = oracle.reduce_f64(np.abs(vals), axis, op)
            assert np.all(np.abs(got - ref) <= 2e-5 * scale + 1e-30), tag
