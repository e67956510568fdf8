"""GPU parity: wgmma/TMA matmul through the C ABI vs the oracle -- reference goldens, seeded random cases for every
kernel variant / dtype / rhs layout, edge cases, and size-independent properties at the BASELINE sizes."""
import numpy as np
import pytest

import oracle
from cubecl_b200 import ServerError, TensorHandle, matmul, synth
from gpu_util import check_against_oracle, make_operand, run_matmul

pytestmark = pytest.mark.gpu

VARIANTS = ["2sm_n256", "2sm_n128", "1sm_n128"]


@pytest.fixture(autouse=True)
def _reset_options(client):
    yield
    client.set_option("gemm.variant", "auto")
    client.set_option("gemm.f32", "hybrid")
    client.set_option("gemm.split_k", "auto")
    client.set_option("gemm.epilogue", "tma")
    client.set_option("gemm.stage", "on")


# ------------------------------------------------------------------------------------------------ reference goldens
@pytest.mark.parametrize("variant", ["auto", "simt"] + VARIANTS)
def test_golden_cmma_simple_1(client, golden, variant):
    # cmma.rs:386-519 / 552-576: f16, Out = Lhs @ Rhs.T, exact
    client.set_option("gemm.variant", variant)
    lhs = np.arange(256, dtype=np.float32).astype(np.float16).reshape(16, 16)
    rhs_nk = (np.arange(256) % 8).astype(np.float16).reshape(16, 16)
    got = run_matmul(client, lhs, rhs_nk, "f16", "f32", rhs_transposed=True)
    assert got.ravel().tolist() == golden["cmma_simple_1"]["expected"]


@pytest.mark.parametrize("mode", ["tf32", "3xtf32", "hybrid"])
def test_golden_cmma_tf32(client, golden, mode):
    # cmma.rs:834-891: f32 inputs on the tf32 pipe, rhs row-major [8,16]; small integers are exact in tf32
    client.set_option("gemm.f32", mode)
    lhs = np.arange(128, dtype=np.float32).reshape(16, 8)
    rhs = (np.arange(128) % 8).astype(np.float32).reshape(8, 16)
    got = run_matmul(client, lhs, rhs, "f32", "f32")
    assert got.ravel().tolist() == golden["cmma_tf32"]["expected"]


def test_golden_cmma_strided(client, golden):
    # cmma.rs:932-1005: lhs tile read with row stride 32 out of a [16,32] buffer
    i = np.arange(16 * 32)
    lhs_buf = np.where((i % 32) < 16, i - (i // 32) * 16, 0).astype(np.float16).reshape(16, 32)
    rhs_buf = (np.arange(16 * 32) % 8).astype(np.float16)
    lhs_full = TensorHandle.from_numpy(client, lhs_buf, "f16")
    lhs = TensorHandle(lhs_full.handle, [16, 16], [32, 1], "f16")
    rhs_full = TensorHandle.from_numpy(client, rhs_buf, "f16")
    rhs = TensorHandle(rhs_full.handle, [16, 16], [1, 16], "f16")  # col-major, stride 16
    out = TensorHandle.empty_contiguous(client, [16, 16], "f32")
    matmul.launch(client, lhs, rhs, out)
    got = out.to_numpy(client)
    assert got.ravel().tolist() == golden["cmma_strided"]["expected"]


@pytest.mark.parametrize("dtype", ["bf16", "f16"])
@pytest.mark.parametrize("m,n,k", [(16, 8, 16), (16, 8, 8)])
def test_golden_cmma_manual(client, dtype, m, n, k):
    # cmma.rs:1099-1196: lhs[i,j]=2i+j, rhs[i,j]=3i+j row-major; integer dot products (reference tolerance 3%, exact here)
    lhs = np.array([[2 * i + j for j in range(k)] for i in range(m)], dtype=np.float32)
    rhs = np.array([[3 * i + j for j in range(n)] for i in range(k)], dtype=np.float32)
    exp = lhs.astype(np.float64) @ rhs.astype(np.float64)
    got = run_matmul(client, synth.to_device_dtype(lhs, dtype), synth.to_device_dtype(rhs, dtype), dtype, "f32")
    assert np.array_equal(got.astype(np.float64), exp)


@pytest.mark.parametrize("m,n,k", [(16, 16, 32), (32, 8, 16), (128, 256, 128)])
def test_golden_simple_cube_formula(client, m, n, k):
    # cmma.rs:578-721: lhs[i]=i, rhs[i]=i%8 stored [n,k]; expectation = reference-order oracle (integers: exact)
    lhs = np.arange(m * k, dtype=np.float32).astype(np.float16).reshape(m, k)
    rhs_nk = (np.arange(n * k) % 8).astype(np.float16).reshape(n, k)
    exp = oracle.matmul_f32(lhs.astype(np.float32), rhs_nk.astype(np.float32).T)
    if float(exp.max()) < 2 ** 24:
        got = run_matmul(client, lhs, rhs_nk, "f16", "f32", rhs_transposed=True)
        assert np.array_equal(got, exp)


# ------------------------------------------------------------------------------------------------ seeded parity, all variants
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("rhs_t", [False, True], ids=["rhs_kn", "rhs_nk"])
@pytest.mark.parametrize("in_dtype,out_dtype", [("bf16", "bf16"), ("bf16", "f32"), ("f16", "f16"), ("f16", "f32")])
def test_parity_16bit(client, variant, rhs_t, in_dtype, out_dtype):
    client.set_option("gemm.variant", variant)
    M, N, K = 384, 512, 320  # several tiles, 5 k-blocks: exercises the smem ring wrap and both accumulator stages
    a_dev, a = make_operand((M, K), in_dtype, 11)
    b_dev, b = make_operand((N, K) if rhs_t else (K, N), in_dtype, 12)
    got = run_matmul(client, a_dev, b_dev, in_dtype, out_dtype, rhs_transposed=rhs_t)
    check_against_oracle(got, a, b.T if rhs_t else b, out_dtype, tight=1e-5 if out_dtype == "f32" else None)


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("rhs_t", [False, True], ids=["rhs_kn", "rhs_nk"])
# hybrid (the default): tf32 product + bf16 cross terms -- the cross terms (~2^-11 of a product) carry bf16 rounding (2^-9)
@pytest.mark.parametrize("mode,tol", [("tf32", 1e-3), ("3xtf32", 2e-6), ("hybrid", 3e-6)])
def test_parity_f32(client, variant, rhs_t, mode, tol):
    client.set_option("gemm.variant", variant)
    client.set_option("gemm.f32", mode)
    M, N, K = 256, 384, 200
    a_dev, a = make_operand((M, K), "f32", 21)
    b_dev, b = make_operand((N, K) if rhs_t else (K, N), "f32", 22)
    got = run_matmul(client, a_dev, b_dev, "f32", "f32", rhs_transposed=rhs_t)
    check_against_oracle(got, a, b.T if rhs_t else b, "f32", tight=tol)


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("rhs_t", [False, True], ids=["rhs_kn", "rhs_nk"])
@pytest.mark.parametrize("in_dtype,mode,tol", [("bf16", "-", 1e-5), ("f16", "-", 1e-5), ("f32", "tf32", 1e-3), ("f32", "3xtf32", 2e-6),
                                                 ("f32", "hybrid", 3e-6)])
def test_parity_transposed_lhs(client, variant, rhs_t, in_dtype, mode, tol):
    # lhs given as a transposed view of a [K, M] buffer (MildlyPermuted{transposed}, matrix_batch_layout.rs:8-19):
    # MN-major A operand through TMA, no into_contiguous copy
    client.set_option("gemm.variant", variant)
    if in_dtype == "f32":
        client.set_option("gemm.f32", mode)
    M, N, K = 320, 384, 264
    a_dev, a_km = make_operand((K, M), in_dtype, 71)
    b_dev, b = make_operand((N, K) if rhs_t else (K, N), in_dtype, 72)
    before = client.launch_count()
    got = run_matmul(client, a_dev, b_dev, in_dtype, "f32", rhs_transposed=rhs_t, lhs_transposed=True)
    # wgmma path (+2 split kernels), not SIMT; wgmma reads MN-major operands for 16-bit types only, so f32 operands in that
    # layout (the lhs, and a [K, N] rhs) take one K-major staging copy each
    staged = 0 if in_dtype != "f32" else 1 + (0 if rhs_t else 1)
    assert client.launch_count() - before == staged + (3 if mode in ("3xtf32", "hybrid") else 1)
    check_against_oracle(got, np.ascontiguousarray(a_km.T), b.T if rhs_t else b, "f32", tight=tol)


# ------------------------------------------------------------------------------------------------ fp8 (kind::f8f6f4)
@pytest.mark.parametrize("dtype", ["f8e4m3", "f8e5m2"])
def test_golden_cmma_manual_fp8(client, dtype):
    # cmma.rs:1099-1196 instantiated (16, 8, 32) for e4m3 / e5m2 (cmma.rs:1856-1859): lhs[i,j]=2i+j, rhs[i,j]=3i+j.
    # fp8 cannot hold every integer up to 100, which is why the reference allows 3 %; against the fp8-ROUNDED operands
    # the f32-accumulated result is exact, and it is within the reference's 3 % of the integer expectation.
    m, n, k = 16, 8, 32
    lhs = np.array([[2 * i + j for j in range(k)] for i in range(m)], dtype=np.float32)
    rhs = np.array([[3 * i + j for j in range(n)] for i in range(k)], dtype=np.float32)
    l8, r8 = synth.to_device_dtype(lhs, dtype), synth.to_device_dtype(rhs, dtype)
    got = run_matmul(client, l8, r8, dtype, "f32")
    exp_rounded = synth.from_device_dtype(l8, dtype).astype(np.float64) @ synth.from_device_dtype(r8, dtype).astype(np.float64)
    assert np.array_equal(got.astype(np.float64), exp_rounded)
    exp_int = lhs.astype(np.float64) @ rhs.astype(np.float64)
    assert np.all(np.abs(got - exp_int) <= 0.03 * exp_int + 1e-9)   # the reference's own criterion (cmma.rs:1180-1194)


@pytest.mark.parametrize("variant", ["2sm_n256", "1sm_n128"])
@pytest.mark.parametrize("lhs_t", [False, True], ids=["lhs_mk", "lhs_km"])
@pytest.mark.parametrize("rhs_t", [False, True], ids=["rhs_kn", "rhs_nk"])
@pytest.mark.parametrize("dtype,out_dtype", [("f8e4m3", "f32"), ("f8e4m3", "bf16"), ("f8e5m2", "f16"), ("f8e5m2", "f32")])
def test_parity_fp8(client, variant, lhs_t, rhs_t, dtype, out_dtype):
    client.set_option("gemm.variant", variant)
    M, N, K = 384, 512, 640   # 5 k-blocks of 128 fp8 elements
    a_dev, a = make_operand((K, M) if lhs_t else (M, K), dtype, 81)
    b_dev, b = make_operand((N, K) if rhs_t else (K, N), dtype, 82)
    got = run_matmul(client, a_dev, b_dev, dtype, out_dtype, rhs_transposed=rhs_t, lhs_transposed=lhs_t)
    check_against_oracle(got, np.ascontiguousarray(a.T) if lhs_t else a, b.T if rhs_t else b, out_dtype,
                         tight=1e-5 if out_dtype == "f32" else None)


def test_fp8_ragged_and_simt_fallback(client):
    for (M, N, K) in ((1, 16, 16), (130, 48, 272), (33, 7, 5)):   # the last one is not TMA-describable -> SIMT kernel
        a_dev, a = make_operand((M, K), "f8e4m3", 83)
        b_dev, b = make_operand((K, N), "f8e4m3", 84)
        got = run_matmul(client, a_dev, b_dev, "f8e4m3", "f32")
        check_against_oracle(got, a, b, "f32", tight=1e-5)


# ------------------------------------------------------------------------------------------------ u8 / i8 -> i32 (kind::i8)
@pytest.mark.parametrize("dtype", ["i8", "u8"])
def test_golden_cmma_manual_int8(client, dtype):
    # cmma.rs:1099-1196 instantiated test::<i8, i8, i32>(16, 8, 32) / <u8, u8, i32> (cmma.rs:1860-1863): exact integers
    m, n, k = 16, 8, 32
    lhs = np.array([[2 * i + j for j in range(k)] for i in range(m)], dtype=np.int64)
    rhs = np.array([[3 * i + j for j in range(n)] for i in range(k)], dtype=np.int64)
    npdt = np.int8 if dtype == "i8" else np.uint8
    got = run_matmul_int(client, lhs.astype(npdt), rhs.astype(npdt), dtype)
    assert np.array_equal(got.astype(np.int64), lhs @ rhs)


@pytest.mark.parametrize("variant", ["auto", "2sm_n256", "1sm_n128", "simt"])
@pytest.mark.parametrize("lhs_t", [False, True], ids=["lhs_mk", "lhs_km"])
@pytest.mark.parametrize("rhs_t", [False, True], ids=["rhs_kn", "rhs_nk"])
@pytest.mark.parametrize("dtype", ["i8", "u8"])
def test_parity_int8_exact(client, variant, lhs_t, rhs_t, dtype):
    client.set_option("gemm.variant", variant)
    M, N, K = 272, 320, 640
    rng = np.random.default_rng(91)
    lo, hi, npdt = (-128, 128, np.int8) if dtype == "i8" else (0, 256, np.uint8)
    a = rng.integers(lo, hi, size=(K, M) if lhs_t else (M, K)).astype(npdt)
    b = rng.integers(lo, hi, size=(N, K) if rhs_t else (K, N)).astype(npdt)
    got = run_matmul_int(client, a, b, dtype, lhs_t=lhs_t, rhs_t=rhs_t)
    exp = (a.T if lhs_t else a).astype(np.int64) @ (b.T if rhs_t else b).astype(np.int64)
    assert np.array_equal(got.astype(np.int64), exp)   # integer work: bit-exact


def run_matmul_int(client, a, b, dtype, lhs_t=False, rhs_t=False):
    lhs = TensorHandle.from_numpy(client, a, dtype)
    rhs = TensorHandle.from_numpy(client, b, dtype)
    lhs = lhs.transposed() if lhs_t else lhs
    rhs = rhs.transposed() if rhs_t else rhs
    out = TensorHandle.empty_contiguous(client, matmul.calculate_matmul_output(lhs.shape, rhs.shape), "i32")
    matmul.launch(client, lhs, rhs, out)
    return out.to_numpy(client)


# ------------------------------------------------------------------------------------------------ mixed 8-bit operand formats
@pytest.mark.parametrize("variant", ["auto", "2sm_n256", "1sm_n128", "simt"])
@pytest.mark.parametrize("lhs_dtype,rhs_dtype", [("i8", "u8"), ("u8", "i8")])
def test_mixed_sign_int8_exact(client, variant, lhs_dtype, rhs_dtype):
    # crates/cubecl-cpp/src/cuda/mma/manual.rs:151-166: the reference instantiates i8 x u8 and u8 x i8 -> i32 for its manual
    # MMA; here the golden generator of cmma.rs:1099-1196 (lhs[i,j] = 2i+j, rhs[i,j] = 3i+j) shifted so the signed operand is
    # negative, plus a seeded full-range problem; exact integers either way
    client.set_option("gemm.variant", variant)
    m, n, k = 16, 8, 32
    lhs = np.array([[2 * i + j for j in range(k)] for i in range(m)], dtype=np.int64)
    rhs = np.array([[3 * i + j for j in range(n)] for i in range(k)], dtype=np.int64)
    if lhs_dtype == "i8":
        lhs = lhs - 60
    else:
        rhs = rhs - 60
    npdt = {"i8": np.int8, "u8": np.uint8}
    l8 = TensorHandle.from_numpy(client, lhs.astype(npdt[lhs_dtype]), lhs_dtype)
    # rhs handed over K-major (a transposed view of [n, k]): 32-byte rows, describable by TMA for the forced tile variants
    r8 = TensorHandle.from_numpy(client, np.ascontiguousarray(rhs.T).astype(npdt[rhs_dtype]), rhs_dtype).transposed()
    out = TensorHandle.empty_contiguous(client, [m, n], "i32")
    matmul.launch(client, l8, r8, out)
    assert np.array_equal(out.to_numpy(client).astype(np.int64), lhs @ rhs)
    rng = np.random.default_rng(93)
    M, N, K = 272, 320, 640
    rng_of = {"i8": (-128, 128), "u8": (0, 256)}
    a = rng.integers(*rng_of[lhs_dtype], size=(M, K)).astype(npdt[lhs_dtype])
    b = rng.integers(*rng_of[rhs_dtype], size=(N, K)).astype(npdt[rhs_dtype])      # rhs given transposed (K-major)
    out = TensorHandle.empty_contiguous(client, [M, N], "i32")
    matmul.launch(client, TensorHandle.from_numpy(client, a, lhs_dtype), TensorHandle.from_numpy(client, b, rhs_dtype).transposed(), out)
    assert np.array_equal(out.to_numpy(client).astype(np.int64), a.astype(np.int64) @ b.T.astype(np.int64))


@pytest.mark.parametrize("variant", ["auto", "2sm_n256", "2sm_m512", "1sm_n128", "simt"])
@pytest.mark.parametrize("lhs_dtype,rhs_dtype", [("f8e4m3", "f8e5m2"), ("f8e5m2", "f8e4m3")])
def test_mixed_fp8_formats(client, variant, lhs_dtype, rhs_dtype):
    # manual.rs:170-186: kind::f8f6f4 takes one format per operand.  The reference's fp8 golden generator with one operand in
    # each format (exact against the fp8-rounded operands, within its 3 % of the integer expectation), then a seeded problem
    client.set_option("gemm.variant", variant)
    m, n, k = 16, 8, 32
    lhs = np.array([[2 * i + j for j in range(k)] for i in range(m)], dtype=np.float32)
    rhs = np.array([[3 * i + j for j in range(n)] for i in range(k)], dtype=np.float32)
    l8, r8 = synth.to_device_dtype(lhs, lhs_dtype), synth.to_device_dtype(rhs, rhs_dtype)
    out_dt = "bf16" if variant == "2sm_m512" else "f32"
    out = TensorHandle.empty_contiguous(client, [m, n], out_dt)
    # rhs handed over K-major (a transposed view of [n, k]): 32-byte rows, describable by TMA for the forced tile variants
    matmul.launch(client, TensorHandle.from_numpy(client, l8, lhs_dtype), TensorHandle.from_numpy(client, np.ascontiguousarray(r8.T), rhs_dtype).transposed(), out)
    got = synth.from_device_dtype(out.to_numpy(client), out_dt).astype(np.float64)
    exp_rounded = synth.from_device_dtype(l8, lhs_dtype).astype(np.float64) @ synth.from_device_dtype(r8, rhs_dtype).astype(np.float64)
    if out_dt == "f32":
        assert np.array_equal(got, exp_rounded)
    exp_int = lhs.astype(np.float64) @ rhs.astype(np.float64)
    assert np.all(np.abs(got - exp_int) <= (0.03 if out_dt == "f32" else 0.04) * exp_int + 1e-9)
    M, N, K = 384, 512, 640
    a_dev, a = make_operand((M, K), lhs_dtype, 181)
    b_dev, b = make_operand((K, N), rhs_dtype, 182)
    out = TensorHandle.empty_contiguous(client, [M, N], out_dt)
    matmul.launch(client, TensorHandle.from_numpy(client, a_dev, lhs_dtype), TensorHandle.from_numpy(client, b_dev, rhs_dtype), out)
    check_against_oracle(synth.from_device_dtype(out.to_numpy(client), out_dt).reshape(M, N), a, b, out_dt, tight=1e-5 if out_dt == "f32" else None)


def test_mixed_formats_outside_the_8bit_families_are_refused(client):
    a = TensorHandle.empty_contiguous(client, [16, 16], "bf16")
    b = TensorHandle.empty_contiguous(client, [16, 16], "f16")
    out = TensorHandle.empty_contiguous(client, [16, 16], "f32")
    matmul.launch(client, a, b, out)
    with pytest.raises(ServerError):
        client.sync()


# ------------------------------------------------------------------------------------------------ operands TMA cannot describe
@pytest.mark.parametrize("dtype,out_dtype,tol", [("bf16", "bf16", None), ("bf16", "f32", 1e-5), ("f16", "f32", 1e-5), ("f32", "f32", 2e-6), ("f8e4m3", "f32", 1e-5)])
def test_unaligned_row_pitch_is_staged_onto_the_tensor_cores(client, dtype, out_dtype, tol):
    # K = 1001: lhs rows are not 16-byte aligned, so TMA cannot describe lhs [M, K] in place.  One staging pass copies it into
    # an aligned pooled buffer and the wgmma kernel runs (no cliff down to the strided SIMT kernel).
    M, N, K = 320, 256, 1001
    a_dev, a = make_operand((M, K), dtype, 191)
    b_dev, b = make_operand((K, N), dtype, 192)
    before = client.launch_count()
    got = run_matmul(client, a_dev, b_dev, dtype, out_dtype)
    launches = client.launch_count() - before
    # repitch (+ 2 lo splits) + GEMM; f32 / fp8 rhs [K, N] is MN-major, which wgmma reads for 16-bit types only: one more staging copy
    assert "gemm_simt" not in client.last_kernel() and launches == {"f32": 5, "f8e4m3": 3}.get(dtype, 2)
    check_against_oracle(got, a, b, out_dtype, tight=tol)
    # rhs given transposed [N, K] with the same odd K (both operands staged), a batch with a broadcast rhs, and an odd N for
    # a row-major rhs (MN-major copy: rows of N stay rows)
    bt_dev, bt = make_operand((N, K), dtype, 193)
    got = run_matmul(client, a_dev, bt_dev, dtype, out_dtype, rhs_transposed=True)
    check_against_oracle(got, a, np.ascontiguousarray(bt.T), out_dtype, tight=tol)
    if dtype in ("bf16", "f32"):
        a3_dev, a3 = make_operand((3, M, K), dtype, 194)
        b1_dev, b1 = make_operand((1, K, N - 3), dtype, 195)
        got = run_matmul(client, a3_dev, b1_dev, dtype, out_dtype)
        for i in range(3):
            check_against_oracle(got[i], a3[i], b1[0], out_dtype, tight=tol)
    client.set_option("gemm.stage", "off")                      # the reference-order SIMT kernel is still there
    try:
        got = run_matmul(client, a_dev, b_dev, dtype, out_dtype)
        assert "gemm_simt" in client.last_kernel()
        check_against_oracle(got, a, b, out_dtype, tight=tol)
    finally:
        client.set_option("gemm.stage", "on")


# ------------------------------------------------------------------------------------------------ fused epilogue
@pytest.mark.parametrize("variant", ["auto", "1sm_n128", "simt"])
@pytest.mark.parametrize("in_dtype,out_dtype", [("bf16", "bf16"), ("bf16", "f32"), ("f32", "f32"), ("f8e4m3", "f16")])
@pytest.mark.parametrize("activation", [None, "relu", "gelu"])
def test_fused_epilogue(client, variant, in_dtype, out_dtype, activation):
    # out = act(alpha * (A @ B) + bias[n]) inside the GEMM epilogue (SURVEY 8f-4); oracle: the same formula in f64
    from math import erf
    client.set_option("gemm.variant", variant)
    M, N, K = 300, 272, 192   # N % 16 == 0 keeps the 1-byte rhs rows TMA-describable (16-byte strides)
    a_dev, a = make_operand((M, K), in_dtype, 101)
    b_dev, b = make_operand((K, N), in_dtype, 102)
    bias = synth.uniform_f32(103, N, -2.0, 2.0)
    alpha = 0.125
    lhs, rhs = TensorHandle.from_numpy(client, a_dev, in_dtype), TensorHandle.from_numpy(client, b_dev, in_dtype)
    out = TensorHandle.empty_contiguous(client, [M, N], out_dtype)
    matmul.launch(client, lhs, rhs, out, alpha=alpha, bias=TensorHandle.from_numpy(client, bias, "f32"), activation=activation)
    got = synth.from_device_dtype(out.to_numpy(client), out_dtype).astype(np.float64)
    f64, fabs = oracle.matmul_f64(a, b)
    x = alpha * f64 + bias.astype(np.float64)[None, :]
    if activation == "relu":
        exp = np.maximum(x, 0.0)
    elif activation == "gelu":
        exp = 0.5 * x * (1.0 + np.vectorize(erf)(x / np.sqrt(2.0)))
    else:
        exp = x
    scale = alpha * fabs + np.abs(bias)[None, :] + 1e-6
    tol = {"f32": 1e-5 if in_dtype != "f32" else 1e-4, "bf16": 1e-2, "f16": 2e-3}[out_dtype]
    assert np.max(np.abs(got - exp) / scale) <= tol


# ------------------------------------------------------------------------------------------------ epilogue store paths
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("in_dtype,out_dtype", [("bf16", "bf16"), ("bf16", "f32"), ("f16", "f16"), ("f8e4m3", "bf16"), ("f32", "f32")])
@pytest.mark.parametrize("M,N,K", [(300, 520, 192), (128, 256, 64), (33, 72, 128), (1, 8, 64)])
def test_tma_store_epilogue_equals_direct_stores(client, variant, in_dtype, out_dtype, M, N, K):
    # staged TMA stores (ragged edges clipped by the tensor map) must write exactly what the per-thread stores write,
    # and nothing outside the M x N window of a larger, pre-filled buffer
    client.set_option("gemm.variant", variant)
    a_dev, a = make_operand((M, K), in_dtype, 401)
    b_dev, b = make_operand((N, K), in_dtype, 402)
    outs = []
    for mode in ("tma", "direct"):
        client.set_option("gemm.epilogue", mode)
        outs.append(run_matmul(client, a_dev, b_dev, in_dtype, out_dtype, rhs_transposed=True))
    assert np.array_equal(outs[0], outs[1])
    check_against_oracle(outs[0], a, np.ascontiguousarray(b.T), out_dtype)


def test_tma_store_respects_pitched_output_window(client):
    # out is a [M, N] window with a row pitch of N + 24 elements inside a buffer pre-filled with a sentinel
    M, N, K, pitch = 200, 136, 96, 160
    a_dev, a = make_operand((M, K), "bf16", 411)
    b_dev, b = make_operand((K, N), "bf16", 412)
    lhs, rhs = TensorHandle.from_numpy(client, a_dev, "bf16"), TensorHandle.from_numpy(client, b_dev, "bf16")
    backing = TensorHandle.from_numpy(client, np.full((M, pitch), -7.0, np.float32), "f32")
    out = TensorHandle(backing.handle, [M, N], [pitch, 1], "f32")
    matmul.launch(client, lhs, rhs, out)
    client.sync()
    full = backing.to_numpy(client).reshape(M, pitch)
    assert np.all(full[:, N:] == -7.0)
    check_against_oracle(full[:, :N], a, b, "f32", tight=1e-5)


# ------------------------------------------------------------------------------------------------ tail split (split-K)
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("split", ["2", "3", "4"])
@pytest.mark.parametrize("in_dtype,out_dtype,mode,tol", [("bf16", "f32", "-", 1e-5), ("bf16", "bf16", "-", 1e-2),
                                                         ("f32", "f32", "3xtf32", 2e-6), ("f32", "f32", "tf32", 1e-3),
                                                         ("f32", "f32", "hybrid", 3e-6)])
def test_tail_split_all_tiles(client, variant, split, in_dtype, out_dtype, mode, tol):
    # fewer tiles than CTA pairs: every tile is cut into K-slices; ragged M/N, K not a multiple of the slice count
    client.set_option("gemm.variant", variant)
    client.set_option("gemm.split_k", split)
    if mode != "-":
        client.set_option("gemm.f32", mode)
    M, N, K = 300, 520, 1096
    a_dev, a = make_operand((M, K), in_dtype, 301)
    b_dev, b = make_operand((K, N), in_dtype, 302)
    got = run_matmul(client, a_dev, b_dev, in_dtype, out_dtype)
    check_against_oracle(got, a, b, out_dtype, tight=tol)
    again = run_matmul(client, a_dev, b_dev, in_dtype, out_dtype)
    assert np.array_equal(got, again)          # slabs are added in slice order: bit-reproducible


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("split", ["off", "2", "4"])
def test_tail_split_after_full_waves(client, variant, split):
    # 80 (2-CTA) / 160 / 320 (1-CTA) tiles: full waves of whole tiles first, then the sliced remainder; batch of 2 on top
    client.set_option("gemm.variant", variant)
    client.set_option("gemm.split_k", split)
    M, N, K = 2560, 2048, 512
    a_dev, a = make_operand((M, K), "bf16", 311)
    b_dev, b = make_operand((N, K), "bf16", 312)
    got = run_matmul(client, a_dev, b_dev, "bf16", "f32", rhs_transposed=True)
    check_against_oracle(got, a, np.ascontiguousarray(b.T), "f32", tight=1e-5)
    client.set_option("gemm.split_k", "off")
    ref = run_matmul(client, a_dev, b_dev, "bf16", "f32", rhs_transposed=True)
    # f32 accumulation in a different association: tiny differences only, and none in the whole-tile region for "off"
    assert np.max(np.abs(got - ref)) <= 1e-4 * np.max(np.abs(ref))
    if split == "off":
        assert np.array_equal(got, ref)


def test_tail_split_batched_fused_epilogue_and_fp8(client):
    from math import erf
    client.set_option("gemm.split_k", "3")
    Bn, M, N, K = 3, 260, 272, 1536
    a_dev, a = make_operand((Bn, M, K), "f8e4m3", 321)
    b_dev, b = make_operand((1, K, N), "f8e4m3", 322)
    bias = synth.uniform_f32(323, N, -2.0, 2.0)
    lhs, rhs = TensorHandle.from_numpy(client, a_dev, "f8e4m3"), TensorHandle.from_numpy(client, b_dev, "f8e4m3")
    out = TensorHandle.empty_contiguous(client, [Bn, M, N], "f16")
    matmul.launch(client, lhs, rhs, out, alpha=0.25, bias=TensorHandle.from_numpy(client, bias, "f32"), activation="gelu")
    got = synth.from_device_dtype(out.to_numpy(client), "f16").astype(np.float64).reshape(Bn, M, N)
    for i in range(Bn):
        f64, fabs = oracle.matmul_f64(a[i], b[0])
        x = 0.25 * f64 + bias.astype(np.float64)[None, :]
        exp = 0.5 * x * (1.0 + np.vectorize(erf)(x / np.sqrt(2.0)))
        scale = 0.25 * fabs + np.abs(bias)[None, :] + 1e-6
        assert np.max(np.abs(got[i] - exp) / scale) <= 2e-3


def test_tail_split_leaves_integer_paths_alone(client):
    client.set_option("gemm.split_k", "4")
    a = (np.arange(256 * 2048) % 251).astype(np.uint8).reshape(256, 2048)
    b = (np.arange(2048 * 256) % 241).astype(np.uint8).reshape(2048, 256)
    got = run_matmul_int(client, a, b, "u8")
    assert np.array_equal(got, a.astype(np.int64) @ b.astype(np.int64))


def test_fuzz_shapes_layouts_dtypes(client):
    # 60 seeded random problems (ragged M/N/K, both operand majors, batch, every dtype); TMA-describable or not, each must
    # match the f64 oracle -- integer dtypes exactly
    rng = np.random.default_rng(2024)
    seen_paths = set()
    for case in range(60):
        dtype = ["bf16", "f16", "f32", "f8e4m3", "f8e5m2", "i8", "u8"][case % 7]
        align = {"bf16": 8, "f16": 8, "f32": 4, "f8e4m3": 16, "f8e5m2": 16, "i8": 16, "u8": 16}[dtype]
        aligned = rng.random() < 0.75
        def dim(hi):
            d = int(rng.integers(1, hi))
            return max(align, d // align * align) if aligned else d
        M, N, K = dim(500), dim(600), dim(700)
        lhs_t, rhs_t = bool(rng.integers(0, 2)), bool(rng.integers(0, 2))
        batch = int(rng.integers(1, 4)) if case % 5 == 0 else 1
        a_shape = ((batch,) if batch > 1 else ()) + ((K, M) if lhs_t else (M, K))
        b_shape = ((batch,) if batch > 1 else ()) + ((N, K) if rhs_t else (K, N))
        before = client.launch_count()
        if dtype in ("i8", "u8"):
            lo, hi, npdt = (-128, 128, np.int8) if dtype == "i8" else (0, 256, np.uint8)
            a = rng.integers(lo, hi, size=a_shape).astype(npdt)
            b = rng.integers(lo, hi, size=b_shape).astype(npdt)
            lhs, rhs = TensorHandle.from_numpy(client, a, dtype), TensorHandle.from_numpy(client, b, dtype)
            lhs = lhs.transposed() if lhs_t else lhs
            rhs = rhs.transposed() if rhs_t else rhs
            out = TensorHandle.empty_contiguous(client, matmul.calculate_matmul_output(lhs.shape, rhs.shape), "i32")
            matmul.launch(client, lhs, rhs, out)
            got = out.to_numpy(client).astype(np.int64)
            al = np.swapaxes(a, -1, -2) if lhs_t else a
            bl = np.swapaxes(b, -1, -2) if rhs_t else b
            assert np.array_equal(got, np.matmul(al.astype(np.int64), bl.astype(np.int64))), (case, dtype, M, N, K, lhs_t, rhs_t)
        else:
            a_dev, a = make_operand(a_shape, dtype, 1000 + case)
            b_dev, b = make_operand(b_shape, dtype, 2000 + case)
            client.set_option("gemm.f32", ("3xtf32", "tf32", "hybrid")[case % 3])
            got = run_matmul(client, a_dev, b_dev, dtype, "f32", rhs_transposed=rhs_t, lhs_transposed=lhs_t)
            al = np.swapaxes(a, -1, -2) if lhs_t else a
            bl = np.swapaxes(b, -1, -2) if rhs_t else b
            exp = np.matmul(al.astype(np.float64), bl.astype(np.float64))
            scale = np.matmul(np.abs(al).astype(np.float64), np.abs(bl).astype(np.float64)) + 1e-30
            tol = 1e-3 if dtype == "f32" else 1e-5
            assert np.max(np.abs(got - exp) / scale) <= tol, (case, dtype, M, N, K, lhs_t, rhs_t, batch)
        seen_paths.add(client.launch_count() - before)
    assert len(seen_paths) >= 2   # both the single-launch wgmma/SIMT path and the split + GEMM path were exercised


def test_simt_is_bit_exact_with_reference_order(client):
    # the strided SIMT kernel accumulates exactly like cmma.rs:695-721 (f32, ascending k, separate mul/add)
    client.set_option("gemm.variant", "simt")
    for dtype in ("f32", "bf16", "f16"):
        a_dev, a = make_operand((37, 53), dtype, 31)
        b_dev, b = make_operand((53, 29), dtype, 32)
        got = run_matmul(client, a_dev, b_dev, dtype, "f32")
        assert np.array_equal(got, oracle.matmul_f32(a, b))


# ------------------------------------------------------------------------------------------------ edge cases
@pytest.mark.parametrize("M,N,K", [(1, 8, 8), (1, 1, 8), (7, 24, 40), (129, 257, 72), (300, 72, 8), (128, 256, 64), (255, 8, 1000)])
def test_ragged_shapes(client, M, N, K):
    a_dev, a = make_operand((M, K), "bf16", 41)
    b_dev, b = make_operand((K, N), "bf16", 42)
    got = run_matmul(client, a_dev, b_dev, "bf16", "f32")
    check_against_oracle(got, a, b, "f32", tight=1e-5)


def test_unaligned_strides_take_the_simt_path(client):
    # K = 5: rows are 10 bytes, not TMA-describable -> strided SIMT kernel, still on the GPU
    before = client.launch_count()
    a_dev, a = make_operand((9, 5), "bf16", 43)
    b_dev, b = make_operand((5, 3), "bf16", 44)
    got = run_matmul(client, a_dev, b_dev, "bf16", "f32")
    assert client.launch_count() == before + 1
    assert np.array_equal(got, oracle.matmul_f32(a, b))


def test_empty_and_zero_k(client):
    out = TensorHandle.empty_contiguous(client, [0, 8], "f32")
    a = TensorHandle.empty_contiguous(client, [0, 16], "bf16")
    b = TensorHandle.empty_contiguous(client, [16, 8], "bf16")
    matmul.launch(client, a, b, out)
    client.sync()


def test_batched_and_broadcast(client):
    # shape.rs:1030-1036: [1,3,M,K] x [2,1,K,N] -> [2,3,M,N]; plus plain batch and fully broadcast rhs
    M, N, K = 64, 72, 96
    a_dev, a = make_operand((1, 3, M, K), "bf16", 51)
    b_dev, b = make_operand((2, 1, K, N), "bf16", 52)
    got = run_matmul(client, a_dev, b_dev, "bf16", "f32")
    exp = np.matmul(a.astype(np.float64), b.astype(np.float64))
    assert got.shape == (2, 3, M, N) and np.allclose(got, exp, rtol=0, atol=1e-4)
    a_dev, a = make_operand((5, M, K), "bf16", 53)
    b_dev, b = make_operand((5, K, N), "bf16", 54)
    got = run_matmul(client, a_dev, b_dev, "bf16", "bf16")
    check_against_oracle(got, a, b, "bf16")
    b_dev, b = make_operand((1, K, N), "bf16", 55)
    got = run_matmul(client, a_dev, b_dev, "bf16", "f32")
    assert np.allclose(got, np.matmul(a.astype(np.float64), b.astype(np.float64)), rtol=0, atol=1e-4)


@pytest.mark.parametrize("mode,tol", [("hybrid", 4e-6), ("3xtf32", 4e-6)])   # K = 333 / 520: accumulation truncation shows (measured 2.7e-6)
def test_f32_split_modes_batched_broadcast_ragged(client, mode, tol):
    # the split-operand f32 schedules on batched / broadcast operands (pair-buffer planes are indexed per batch entry), every
    # operand-major combination, K that is neither a multiple of 32 nor of 64, unaligned row pitches (pad to 16 bytes)
    client.set_option("gemm.f32", mode)
    M, N, K = 136, 200, 333
    a_dev, a = make_operand((3, M, K), "f32", 81)
    b_dev, b = make_operand((3, K, N), "f32", 82)
    check_against_oracle(run_matmul(client, a_dev, b_dev, "f32", "f32"), a, b, "f32", tight=tol)
    b1_dev, b1 = make_operand((1, K, N), "f32", 83)          # rhs broadcast over the batch: ONE pair buffer entry
    check_against_oracle(run_matmul(client, a_dev, b1_dev, "f32", "f32"), a, b1, "f32", tight=tol)
    a1_dev, a1 = make_operand((1, M, K), "f32", 84)
    check_against_oracle(run_matmul(client, a1_dev, b_dev, "f32", "f32"), a1, b, "f32", tight=tol)
    M, N, K = 264, 328, 520                                   # 16-byte aligned pitches for the transposed views
    for lhs_t in (False, True):
        for rhs_t in (False, True):
            a_dev, a = make_operand((2, K, M) if lhs_t else (2, M, K), "f32", 85)
            b_dev, b = make_operand((2, N, K) if rhs_t else (2, K, N), "f32", 86)
            got = run_matmul(client, a_dev, b_dev, "f32", "f32", rhs_transposed=rhs_t, lhs_transposed=lhs_t)
            check_against_oracle(got, np.swapaxes(a, -1, -2) if lhs_t else a, np.swapaxes(b, -1, -2) if rhs_t else b, "f32", tight=tol)


@pytest.mark.parametrize("mode", ["hybrid", "tf32"])
def test_f32_nonfinite_operands_propagate_like_f32(client, mode):
    # hybrid: an infinite operand has no low part and is dropped from the cross terms (inf - inf, inf * 0 would poison them):
    # inf * finite stays inf, NaN stays NaN.  (3xtf32 multiplies the ORIGINAL lhs by rhs_lo, so inf * 0 = NaN there: documented.)
    client.set_option("gemm.f32", mode)
    M, N, K = 128, 128, 64
    a = np.ones((M, K), dtype=np.float32)
    b = np.ones((K, N), dtype=np.float32)
    a[3, 5] = np.inf
    a[7, 9] = -np.inf
    b[11, 13] = np.nan
    got = run_matmul(client, a, b, "f32", "f32")
    exp = a.astype(np.float64) @ b.astype(np.float64)
    assert np.array_equal(np.isnan(got), np.isnan(exp))
    fin = np.isfinite(exp)
    assert np.array_equal(got[~fin & ~np.isnan(exp)], exp[~fin & ~np.isnan(exp)].astype(np.float32))
    assert np.array_equal(got[fin], exp[fin].astype(np.float32))


def test_pitched_output_and_inputs(client):
    # TensorHandle::empty applies the pitched layout (allocator.rs:21-72): [100, 72] bf16 rows of 144 B pitch to 256 B
    M, N, K = 100, 72, 136
    a_dev, a = make_operand((M, K), "bf16", 61)
    b_dev, b = make_operand((K, N), "bf16", 62)
    lhs = TensorHandle.empty(client, [M, K], "bf16")
    assert lhs.strides[0] * 2 % 16 == 0 and lhs.strides[0] >= K
    host = np.zeros((M, lhs.strides[0]), dtype=np.uint16)
    host[:, :K] = a_dev
    client.write(lhs.handle, host)
    rhs = TensorHandle.from_numpy(client, b_dev, "bf16")
    out = TensorHandle.empty(client, [M, N], "f32")
    assert out.strides[0] >= N
    matmul.launch(client, lhs, rhs, out)
    got = out.to_numpy(client)
    check_against_oracle(got, a, b, "f32", tight=1e-5)


def test_shape_errors_are_deferred_to_sync(client):
    # launch never fails synchronously; the error surfaces at sync (server.rs:269-284,981-1002)
    a = TensorHandle.empty_contiguous(client, [8, 16], "bf16")
    b = TensorHandle.empty_contiguous(client, [24, 8], "bf16")
    out = TensorHandle.empty_contiguous(client, [8, 8], "bf16")
    matmul.launch(client, a, b, out)  # inner dims differ: no exception here
    with pytest.raises(ServerError):
        client.sync()
    client.sync()  # error list drained; the client is healthy again


# ------------------------------------------------------------------------------------------------ BASELINE sizes: properties
def _device_operand(client, shape, dtype, seed):
    t = TensorHandle.empty_contiguous(client, shape, dtype)
    client.fill_uniform(t.handle, dtype, int(np.prod(shape)), seed, -1.0, 1.0)
    return t


def _host_rows(seed, rows, ncols, dtype):
    """Regenerate selected rows of a device-filled [R, ncols] operand on the host (counter hash)."""
    out = np.empty((len(rows), ncols), dtype=np.float32)
    for i, r in enumerate(rows):
        out[i] = synth.uniform_f32(seed, ncols, -1.0, 1.0, start=int(r) * ncols)
    return synth.from_device_dtype(synth.to_device_dtype(out, dtype), dtype)


@pytest.mark.parametrize("variant", ["auto", "2sm_n256", "2sm_n128"])
def test_bf16_8192_sampled_points_and_linearity(client, variant):
    # BASELINE config 3 at full size: 256 sampled outputs vs f64 dot products of host-regenerated operands
    client.set_option("gemm.variant", variant)
    n = 8192
    a = _device_operand(client, [n, n], "bf16", 3)
    b = _device_operand(client, [n, n], "bf16", 4)
    out = TensorHandle.empty_contiguous(client, [n, n], "bf16")
    matmul.launch(client, a, b, out)
    got = synth.bf16_bits_to_f32(out.to_numpy(client))
    rng = np.random.default_rng(9)
    ms = np.concatenate([rng.integers(0, n, 24), [0, 127, 128, 255, 256, n - 1, 4095, 4096]])
    ns = np.concatenate([rng.integers(0, n, 24), [0, 63, 64, 255, 256, n - 1, 4097, 8000]])
    a_rows = _host_rows(3, ms, n, "bf16")                      # [32, K]
    b_full_cols = np.stack([synth.from_device_dtype(synth.to_device_dtype(synth.uniform_at(4, np.arange(n, dtype=np.uint64) * n + c, -1.0, 1.0), "bf16"), "bf16") for c in ns])  # [32, K]
    f64 = a_rows.astype(np.float64) @ b_full_cols.astype(np.float64).T   # [32 m, 32 n]
    fabs = np.abs(a_rows).astype(np.float64) @ np.abs(b_full_cols).astype(np.float64).T
    sub = got[np.ix_(ms, ns)].astype(np.float64)
    assert np.max(np.abs(sub - f64) / fabs) <= 1e-2
    assert np.max(np.abs(sub - f64)) <= 0.02 * np.max(np.abs(f64)) + 0.5  # bf16 output rounding only


def _host_operand(seed, rows, cols, dtype, chunk_rows=1024):
    """A whole device-filled [rows, cols] operand regenerated on the host (counter hash), as the f32 values the device holds."""
    out = np.empty((rows, cols), dtype=np.float32)
    for r0 in range(0, rows, chunk_rows):
        r1 = min(rows, r0 + chunk_rows)
        v = synth.uniform_f32(seed, (r1 - r0) * cols, -1.0, 1.0, start=r0 * cols)
        out[r0:r1] = synth.from_device_dtype(synth.to_device_dtype(v, dtype), dtype).reshape(r1 - r0, cols)
    return out


def _block_checksums_ok(got, a, b, out_dtype, bm=32, bn=64, rel=None):
    """Checksum identity over EVERY [bm x bn] block of the product (the epilogue's staging-tile granularity, so every
    512 x 256 / 256 x 256 tile, every CTA half and every epilogue warp's rows are covered):
        sum_{m in rows, n in cols} C[m, n] == sum_k (sum_{m in rows} A[m, k]) * (sum_{n in cols} B[k, n])      (f64)
    The only differences are the output rounding (one ulp of the output type per element, random sign) and the f32
    accumulation; the bound is 12 standard deviations of that noise, against block sums of magnitude ~1e3-1e4.  Any wrong
    row segment, swapped tile, missing K-slice or stale accumulator moves a block sum by far more."""
    M, K = a.shape
    N = b.shape[1]
    asum = a.astype(np.float64).reshape(M // bm, bm, K).sum(axis=1)             # [M/bm, K]
    bsum = b.astype(np.float64).reshape(K, N // bn, bn).sum(axis=2)             # [K, N/bn]
    expect = asum @ bsum                                                        # [M/bm, N/bn]
    have = got.astype(np.float64).reshape(M // bm, bm, N // bn, bn).sum(axis=(1, 3))
    # per-element rounding noise: |c| * 2^-9 (bf16) / 2^-12 (f16) / 2^-25 (f32, plus accumulation ~1e-6 |a||b| K)
    rel = rel if rel is not None else {"bf16": 2.0 ** -9, "f16": 2.0 ** -12, "f32": 2.0 ** -20}[out_dtype]
    rms_c = np.sqrt(np.mean(got.astype(np.float64) ** 2))
    sigma = rel * rms_c * np.sqrt(bm * bn) / np.sqrt(3.0)
    worst = float(np.max(np.abs(have - expect)))
    return worst <= 12.0 * sigma + 1e-6 * np.max(np.abs(expect)), worst, 12.0 * sigma


def test_bf16_8192_every_block_checksum(client):
    # BASELINE config 3 at full size on the DEFAULT path (auto -> the 256 x 256 cluster tile): all 67 M outputs take part,
    # through 32,768 block checksums against f64 sums of the host-regenerated operands
    n = 8192
    a = _device_operand(client, [n, n], "bf16", 3)
    b = _device_operand(client, [n, n], "bf16", 4)
    out = TensorHandle.empty_contiguous(client, [n, n], "bf16")
    matmul.launch(client, a, b, out)
    got = synth.bf16_bits_to_f32(out.to_numpy(client))
    assert "2sm_n256" in client.last_kernel()
    ah, bh = _host_operand(3, n, n, "bf16"), _host_operand(4, n, n, "bf16")
    ok, worst, bound = _block_checksums_ok(got, ah, bh, "bf16")
    assert ok, f"block checksum off by {worst:.3f} (bound {bound:.3f})"
    # the check has teeth: one corrupted 32-element row segment is caught
    bad = got.copy()
    bad[4100, 4096:4128] += 4.0
    assert not _block_checksums_ok(bad, ah, bh, "bf16")[0]
    # checksum of checksums: the grand total equals colsum(A) . rowsum(B)
    total = float(ah.astype(np.float64).sum(axis=0) @ bh.astype(np.float64).sum(axis=1))
    assert abs(float(got.astype(np.float64).sum()) - total) <= 12.0 * (2.0 ** -9) * np.sqrt(np.mean(got.astype(np.float64) ** 2)) * n / np.sqrt(3.0)


@pytest.mark.parametrize("mode,rel", [("tf32", 2.0 ** -11), ("3xtf32", 2.0 ** -14), ("hybrid", 2.0 ** -14)])
def test_f32_4096_every_block_checksum(client, mode, rel):
    # BASELINE config 2 at full size on the default plan (256 x 256 tiles with a stream-K head: 34 tiles are summed from two
    # K-halves): every output through the block checksums.  Noise model: tf32 rounds each operand to 11 bits (relative 2^-11 of the
    # element magnitude, accumulated as a random walk over K -- bounded above by 2^-11 of rms(C) sqrt(block)); 3xTF32 restores
    # the operands to ~f32, but the tensor core adds each 8-deep partial product into the f32 accumulator with truncation, a bias
    # of half an ulp TOWARD ZERO per instruction: 3 * 4096 / 8 = 1536 instructions * 1e-6 (ulp of 16..32) = ~1.5e-3 per element,
    # signed like the element (measured: worst block sum 0.16, i.e. ~1e-3 per element) -- hence 2^-14 of rms(C)
    client.set_option("gemm.f32", mode)
    n = 4096
    a = _device_operand(client, [n, n], "f32", 1)
    b = _device_operand(client, [n, n], "f32", 2)
    out = TensorHandle.empty_contiguous(client, [n, n], "f32")
    matmul.launch(client, a, b, out)
    got = out.to_numpy(client)
    ah, bh = _host_operand(1, n, n, "f32"), _host_operand(2, n, n, "f32")
    ok, worst, bound = _block_checksums_ok(got, ah, bh, "f32", rel=rel)
    assert ok, f"{mode}: block checksum off by {worst:.4f} (bound {bound:.4f})"
    bad = got.copy()
    bad[1000, 2048:2080] += 0.5 if mode == "tf32" else 0.05
    assert not _block_checksums_ok(bad, ah, bh, "f32", rel=rel)[0]


def test_batched_8x4096_every_block_checksum(client):
    # BASELINE config 5, the per-GPU slice (8 x 4096^3 bf16): every output of every batch through block checksums
    n, B = 4096, 8
    a = _device_operand(client, [B, n, n], "bf16", 6)
    b = _device_operand(client, [B, n, n], "bf16", 7)
    out = TensorHandle.empty_contiguous(client, [B, n, n], "bf16")
    matmul.launch(client, a, b, out)
    got = synth.bf16_bits_to_f32(out.to_numpy(client)).reshape(B, n, n)
    for bi in range(B):
        ah = synth.from_device_dtype(synth.to_device_dtype(synth.uniform_f32(6, n * n, -1.0, 1.0, start=bi * n * n), "bf16"), "bf16").reshape(n, n)
        bh = synth.from_device_dtype(synth.to_device_dtype(synth.uniform_f32(7, n * n, -1.0, 1.0, start=bi * n * n), "bf16"), "bf16").reshape(n, n)
        ok, worst, bound = _block_checksums_ok(got[bi], ah, bh, "bf16")
        assert ok, f"batch {bi}: block checksum off by {worst:.3f} (bound {bound:.3f})"


def test_f32_4096_sampled_points(client):
    # BASELINE config 2: f32 4096^3, both f32 modes, sampled against f64
    n = 4096
    a = _device_operand(client, [n, n], "f32", 1)
    b = _device_operand(client, [n, n], "f32", 2)
    rng = np.random.default_rng(10)
    ms, ns = rng.integers(0, n, 32), rng.integers(0, n, 32)
    a_rows = _host_rows(1, ms, n, "f32")
    b_cols = np.stack([synth.uniform_at(2, np.arange(n, dtype=np.uint64) * n + c, -1.0, 1.0) for c in ns])
    f64 = a_rows.astype(np.float64) @ b_cols.astype(np.float64).T
    fabs = np.abs(a_rows).astype(np.float64) @ np.abs(b_cols).astype(np.float64).T
    # 3xtf32 at K = 4096: f32 accumulation of 3K products dominates (measured 4e-6); the reference-order f32 loop itself
    # is only good to ~K * 2^-24 = 2.4e-4 in the worst case
    for mode, tol in (("tf32", 1e-3), ("3xtf32", 1e-5), ("hybrid", 1e-5)):
        client.set_option("gemm.f32", mode)
        out = TensorHandle.empty_contiguous(client, [n, n], "f32")
        matmul.launch(client, a, b, out)
        got = out.to_numpy(client)
        assert np.max(np.abs(got[np.ix_(ms, ns)].astype(np.float64) - f64) / fabs) <= tol


def test_batched_4096_matches_single(client):
    # BASELINE config 5 shape family (per-GPU slice: 8 x 4096^3): every batch equals the same product run alone -- bit for bit
    # when both run the same plan (the K association of a stream-K head depends on the tile count, so it is switched off for
    # that comparison), and to one output rounding under the default plans
    n, B = 4096, 3
    a = _device_operand(client, [B, n, n], "bf16", 6)
    b = _device_operand(client, [B, n, n], "bf16", 7)
    for split, exact in (("off", True), ("auto", False)):
        client.set_option("gemm.split_k", split)
        client.set_option("gemm.variant", "2sm_n256" if exact else "auto")
        out = TensorHandle.empty_contiguous(client, [B, n, n], "bf16")
        matmul.launch(client, a, b, out)
        got = out.to_numpy(client)
        for bi in (0, B - 1):
            a1 = TensorHandle(a.handle.offset(bi * n * n * 2, n * n * 2), [n, n], [n, 1], "bf16")
            b1 = TensorHandle(b.handle.offset(bi * n * n * 2, n * n * 2), [n, n], [n, 1], "bf16")
            o1 = TensorHandle.empty_contiguous(client, [n, n], "bf16")
            matmul.launch(client, a1, b1, o1)
            one = o1.to_numpy(client)
            if exact:
                assert np.array_equal(one, got[bi])
            else:
                x, y = synth.bf16_bits_to_f32(one).astype(np.float64), synth.bf16_bits_to_f32(got[bi]).astype(np.float64)
                assert np.max(np.abs(x - y) / (np.abs(y) + 1.0)) <= 2.0 ** -7      # at most one bf16 rounding step apart
                assert np.mean(one != got[bi]) < 0.02                               # and almost everywhere identical
