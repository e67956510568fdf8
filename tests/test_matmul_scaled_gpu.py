"""GPU parity: block-scaled (MX) matmul through the C ABI -- operands expanded exactly to bf16 x * scale, then the bf16 wgmma GEMM --
against the oracle's restatement of the reference's expected loops (test_cmma_scaled / test_cmma_scaled_fp4,
crates/cubecl-core/src/runtime_tests/cmma.rs:1476-1700)."""
import numpy as np
import pytest

import oracle
from cubecl_b200 import ServerError, TensorHandle, matmul, synth

pytestmark = pytest.mark.gpu

TC_VARIANTS = ["2sm_n256", "2sm_n224", "2sm_n128", "1sm_n128"]


@pytest.fixture(autouse=True)
def _reset_options(client):
    yield
    client.set_option("gemm.variant", "auto")
    client.set_option("gemm.split_k", "auto")


def quantise(vals, dtype):
    """f32 values -> (device bytes [rows, K or K/2], the f32 values those bytes represent)"""
    if dtype == "f4e2m1x2":
        codes = synth.f32_to_e2m1_codes(vals)
        return synth.pack_e2m1x2(codes), synth.e2m1_codes_to_f32(codes)
    bits = synth.f32_to_fp8_bits(vals, dtype)
    return bits, synth.fp8_bits_to_f32(bits, dtype)


def run_scaled(client, a_dev, b_dev, sa_bits, sb_bits, lhs_dtype, rhs_dtype, out_dtype, packed=False, scale_block=32):
    lhs, rhs = TensorHandle.from_numpy(client, a_dev, lhs_dtype), TensorHandle.from_numpy(client, b_dev, rhs_dtype)
    one = 0x38 if scale_block == 16 else 127
    if packed:
        sa = np.stack([synth.pack_scale_chunks(x, one) for x in sa_bits.reshape(-1, *sa_bits.shape[-2:])])
        sb = np.stack([synth.pack_scale_chunks(x, one) for x in sb_bits.reshape(-1, *sb_bits.shape[-2:])])
    else:
        sa, sb = sa_bits, sb_bits
    sdt = "f8e4m3" if scale_block == 16 else "ue8m0"
    ls, rs = TensorHandle.from_numpy(client, sa, sdt), TensorHandle.from_numpy(client, sb, sdt)
    shape = list(a_dev.shape[:-2]) + [a_dev.shape[-2], b_dev.shape[-2]]
    out = TensorHandle.empty_contiguous(client, shape, out_dtype)
    matmul.launch_scaled(client, lhs, rhs, ls, rs, out, scales_packed=packed, scale_block=scale_block)
    client.sync()
    return synth.from_device_dtype(out.to_numpy(client), out_dtype).reshape(shape)


def random_problem(M, N, K, lhs_dtype, rhs_dtype, seed, batch=(), scale_lo=117, scale_hi=138):
    rng = np.random.default_rng(seed)
    a_dev, a = quantise(rng.uniform(-3, 3, size=batch + (M, K)).astype(np.float32), lhs_dtype)
    b_dev, b = quantise(rng.uniform(-3, 3, size=batch + (N, K)).astype(np.float32), rhs_dtype)
    sa = rng.integers(scale_lo, scale_hi, size=batch + (M, K // 32), dtype=np.uint8)   # default 2^-10 .. 2^10
    sb = rng.integers(scale_lo, scale_hi, size=batch + (N, K // 32), dtype=np.uint8)
    return a_dev, a, b_dev, b, sa, sb


def check(got, a, b, sa, sb, tol):
    o32, f64, fabs = oracle.matmul_scaled(a, b, synth.ue8m0_to_f32(sa), synth.ue8m0_to_f32(sb), 32)
    err = np.max(np.abs(got.astype(np.float64) - f64) / np.maximum(fabs, 1e-30))
    assert err <= tol, f"max |gpu - f64| / sum|terms| = {err:.3e} > {tol:.1e}"
    return o32


# ------------------------------------------------------------------------------------------------ reference goldens
@pytest.mark.parametrize("variant", ["auto", "simt"] + TC_VARIANTS)
@pytest.mark.parametrize("lhs_dtype,rhs_dtype", [("f8e5m2", "f8e5m2"), ("f8e4m3", "f8e4m3"), ("f8e5m2", "f8e4m3"), ("f8e4m3", "f8e5m2")])
def test_golden_cmma_scaled(client, variant, lhs_dtype, rhs_dtype):
    # test_cmma_scaled (cmma.rs:1518-1593, instantiated :1914-1917): m16 n8 k32, one ue8m0 scale per row (factor 1)
    client.set_option("gemm.variant", variant)
    m, n, k = 16, 8, 32
    lhs_f = np.array([[i * 2 + j for j in range(k)] for i in range(m)], dtype=np.float32)
    rhs_f = np.array([[i * 3 + j for i in range(k)] for j in range(n)], dtype=np.float32)      # [n, k]: the test's col-major rhs
    sa = np.array([[i * 2 + j + 120 for j in range(1)] for i in range(m)], dtype=np.uint8)
    sb = np.array([[i * 3 + j + 120 for i in range(1)] for j in range(n)], dtype=np.uint8)
    a_dev, a = quantise(lhs_f, lhs_dtype)       # A::from(i * 2 + j): rounded to the fp8 type, as the reference uploads it
    b_dev, b = quantise(rhs_f, rhs_dtype)
    got = run_scaled(client, a_dev, b_dev, sa, sb, lhs_dtype, rhs_dtype, "f32")
    o32 = check(got, a, b, sa, sb, 1e-6)
    if variant == "simt":
        assert np.array_equal(got, o32)          # reference order, bit for bit
    # the reference's own criterion: 3 % of the expected values computed from the UNROUNDED generators (cmma.rs:1572-1592)
    exp, _, _ = oracle.matmul_scaled(lhs_f, rhs_f, synth.ue8m0_to_f32(sa), synth.ue8m0_to_f32(sb), 32)
    if lhs_dtype == rhs_dtype == "f8e4m3":       # e5m2 rounds these integers by up to 12.5 %; the reference test is loose there too
        assert np.max(np.abs(got - exp) / np.abs(exp)) <= 0.03


@pytest.mark.parametrize("variant", ["auto", "simt"] + TC_VARIANTS)
def test_golden_cmma_scaled_fp4(client, variant):
    # test_cmma_scaled_fp4 (cmma.rs:1595-1710): m16 n8 k64, e2m1 codes ((i + j) % 15) + 1, two scales per row (factor 2)
    client.set_option("gemm.variant", variant)
    m, n, k = 16, 8, 64
    a_codes = np.array([[((i + j) % 15) + 1 for j in range(k)] for i in range(m)], dtype=np.uint8)
    b_codes = np.array([[((i + j) % 15) + 1 for i in range(k)] for j in range(n)], dtype=np.uint8)
    sa = np.array([[i * 2 + j + 120 for j in range(2)] for i in range(m)], dtype=np.uint8)
    sb = np.array([[i * 3 + j + 120 for i in range(2)] for j in range(n)], dtype=np.uint8)
    a, b = synth.e2m1_codes_to_f32(a_codes), synth.e2m1_codes_to_f32(b_codes)
    got = run_scaled(client, synth.pack_e2m1x2(a_codes), synth.pack_e2m1x2(b_codes), sa, sb, "f4e2m1x2", "f4e2m1x2", "f32")
    o32 = check(got, a, b, sa, sb, 1e-6)
    if variant == "simt":
        assert np.array_equal(got, o32)
    assert np.max(np.abs(got - o32)) <= 0.03 * np.max(np.abs(o32))


# ------------------------------------------------------------------------------------------------ seeded parity
@pytest.mark.parametrize("variant", TC_VARIANTS)
@pytest.mark.parametrize("lhs_dtype,rhs_dtype,out_dtype,tol", [("f8e4m3", "f8e4m3", "f32", 2e-6), ("f8e4m3", "f8e5m2", "bf16", 1e-2),
                                                               ("f8e5m2", "f8e5m2", "f16", 2e-3), ("f4e2m1x2", "f4e2m1x2", "f32", 2e-6),
                                                               ("f4e2m1x2", "f4e2m1x2", "bf16", 1e-2)])
@pytest.mark.parametrize("M,N,K", [(300, 520, 1024), (128, 256, 96), (1, 8, 32), (257, 129, 4096)])
def test_parity_scaled(client, variant, lhs_dtype, rhs_dtype, out_dtype, tol, M, N, K):
    # ragged M / N, K that is not a whole k-block (96: padded scale atoms), a single row, a long K
    client.set_option("gemm.variant", variant)
    hi = 129 if out_dtype == "f16" else 138      # keep the results inside f16's range
    a_dev, a, b_dev, b, sa, sb = random_problem(M, N, K, lhs_dtype, rhs_dtype, seed=M + N + K, scale_hi=hi)
    got = run_scaled(client, a_dev, b_dev, sa, sb, lhs_dtype, rhs_dtype, out_dtype)
    check(got, a, b, sa, sb, tol)


@pytest.mark.parametrize("dtype", ["f8e4m3", "f4e2m1x2"])
def test_simt_path_is_reference_order_and_agrees_with_tcgen05(client, dtype):
    M, N, K = 70, 90, 160
    a_dev, a, b_dev, b, sa, sb = random_problem(M, N, K, dtype, dtype, seed=5)
    client.set_option("gemm.variant", "simt")
    simt = run_scaled(client, a_dev, b_dev, sa, sb, dtype, dtype, "f32")
    o32 = check(simt, a, b, sa, sb, 2e-6)
    assert np.array_equal(simt, o32)
    client.set_option("gemm.variant", "auto")
    tc = run_scaled(client, a_dev, b_dev, sa, sb, dtype, dtype, "f32")
    _, _, fabs = oracle.matmul_scaled(a, b, synth.ue8m0_to_f32(sa), synth.ue8m0_to_f32(sb), 32)
    assert np.max(np.abs(tc - simt) / fabs) <= 2e-6


@pytest.mark.parametrize("dtype", ["f8e5m2", "f4e2m1x2"])
def test_prepacked_scales_and_batches(client, dtype):
    # [batch, rows, K] operands; the same scales handed over row-major and already in the tensor core's chunk layout
    batch, M, N, K = (3,), 200, 136, 384
    a_dev, a, b_dev, b, sa, sb = random_problem(M, N, K, dtype, dtype, seed=11, batch=batch)
    plain = run_scaled(client, a_dev, b_dev, sa, sb, dtype, dtype, "f32")
    packed = run_scaled(client, a_dev, b_dev, sa, sb, dtype, dtype, "f32", packed=True)
    assert np.array_equal(plain, packed)
    for i in range(batch[0]):
        check(plain[i], a[i], b[i], sa[i], sb[i], 2e-6)


# ------------------------------------------------------------------------------------------------ NVFP4 (ue4m3 scale per 16)
def nvfp4_problem(M, N, K, seed, batch=()):
    """packed e2m1 operands + e4m3 scale bytes per 16 elements; some scale bytes carry a sign bit, which the hardware ignores
    (third ScaledMmaConfig row, crates/cubecl-cpp/src/cuda/mma/manual.rs:240-250: "Sign of scales is ignored")"""
    rng = np.random.default_rng(seed)
    a_dev, a = quantise(rng.uniform(-6, 6, size=batch + (M, K)).astype(np.float32), "f4e2m1x2")
    b_dev, b = quantise(rng.uniform(-6, 6, size=batch + (N, K)).astype(np.float32), "f4e2m1x2")
    sa = synth.f32_to_fp8_bits(rng.uniform(0.05, 8.0, size=batch + (M, K // 16)).astype(np.float32), "f8e4m3")
    sb = synth.f32_to_fp8_bits(rng.uniform(0.05, 8.0, size=batch + (N, K // 16)).astype(np.float32), "f8e4m3")
    sa[..., 0::7] |= 0x80
    sb[..., 0::5] |= 0x80
    return a_dev, a, b_dev, b, sa, sb


def check_nvfp4(got, a, b, sa, sb, tol):
    fa, fb = np.abs(synth.fp8_bits_to_f32(sa, "f8e4m3")), np.abs(synth.fp8_bits_to_f32(sb, "f8e4m3"))
    o32, f64, fabs = oracle.matmul_scaled(a, b, fa, fb, 16)
    err = np.max(np.abs(got.astype(np.float64) - f64) / np.maximum(fabs, 1e-30))
    assert err <= tol, f"max |gpu - f64| / sum|terms| = {err:.3e} > {tol:.1e}"
    return o32


@pytest.mark.parametrize("variant", ["simt"] + TC_VARIANTS)
@pytest.mark.parametrize("out_dtype,tol", [("f32", 2e-6), ("bf16", 1e-2)])
@pytest.mark.parametrize("M,N,K", [(16, 8, 64), (300, 520, 1024), (128, 256, 96), (257, 129, 2048)])
def test_parity_nvfp4(client, variant, out_dtype, tol, M, N, K):
    # (16, 8, 64) with four scales per row is the shape of the reference's e2m1x2 / E4M3-scale feature row (k 64, factor 4)
    client.set_option("gemm.variant", variant)
    a_dev, a, b_dev, b, sa, sb = nvfp4_problem(M, N, K, seed=M + N + K)
    got = run_scaled(client, a_dev, b_dev, sa, sb, "f4e2m1x2", "f4e2m1x2", out_dtype, scale_block=16)
    o32 = check_nvfp4(got, a, b, sa, sb, tol)
    if variant == "simt" and out_dtype == "f32":
        assert np.array_equal(got, o32)              # reference-order loop, bit for bit


def test_nvfp4_prepacked_scales_and_batches(client):
    batch, M, N, K = (2,), 200, 136, 384
    a_dev, a, b_dev, b, sa, sb = nvfp4_problem(M, N, K, seed=13, batch=batch)
    plain = run_scaled(client, a_dev, b_dev, sa, sb, "f4e2m1x2", "f4e2m1x2", "f32", scale_block=16)
    packed = run_scaled(client, a_dev, b_dev, sa, sb, "f4e2m1x2", "f4e2m1x2", "f32", packed=True, scale_block=16)
    assert np.array_equal(plain, packed)
    for i in range(batch[0]):
        check_nvfp4(plain[i], a[i], b[i], sa[i], sb[i], 2e-6)


def test_split_k_tail_on_scaled_problem(client):
    # few tiles, long K: the cost model slices K (partial accumulators meet in the slab exchange); forced here
    client.set_option("gemm.split_k", "3")
    a_dev, a, b_dev, b, sa, sb = random_problem(256, 256, 3072, "f8e4m3", "f8e4m3", seed=21)
    got = run_scaled(client, a_dev, b_dev, sa, sb, "f8e4m3", "f8e4m3", "f32")
    check(got, a, b, sa, sb, 2e-6)


def test_extreme_and_nan_scales(client):
    # scale exponents at the ends of ue8m0; 0xFF is NaN and poisons exactly its row of A / column of B
    M, N, K = 64, 64, 64
    a_dev, a, b_dev, b, sa, sb = random_problem(M, N, K, "f8e4m3", "f8e4m3", seed=31)
    sa[:] = 127
    sb[:] = 127
    sa[3, 0], sb[5, 1] = 1, 227          # 2^-126, 2^100 (products stay finite in f32)
    got = run_scaled(client, a_dev, b_dev, sa, sb, "f8e4m3", "f8e4m3", "f32")
    check(got, a, b, sa, sb, 2e-6)
    sa[7, 1] = 255
    got = run_scaled(client, a_dev, b_dev, sa, sb, "f8e4m3", "f8e4m3", "f32")
    assert np.isnan(got[7]).all() and not np.isnan(np.delete(got, 7, axis=0)).any()


def test_scaled_argument_errors_are_deferred(client):
    a = TensorHandle.from_numpy(client, np.zeros((16, 48), np.uint8), "f8e4m3")
    s = TensorHandle.from_numpy(client, np.full((16, 1), 127, np.uint8), "ue8m0")
    out = TensorHandle.empty_contiguous(client, [16, 16], "f32")
    matmul.launch_scaled(client, a, a, s, s, out)                 # K = 48 is not a multiple of 32
    with pytest.raises(ServerError):
        client.sync()
    a64 = TensorHandle.from_numpy(client, np.zeros((16, 64), np.uint8), "f8e4m3")
    s2 = TensorHandle.from_numpy(client, np.full((16, 2), 127, np.uint8), "ue8m0")
    matmul.launch_scaled(client, a64, a64, s2, s2, out, scale_block=16)
    with pytest.raises(ServerError):
        client.sync()
    matmul.launch_scaled(client, a64, a64, s2, s2, out)           # and the context still works afterwards
    client.sync()
    assert np.array_equal(out.to_numpy(client), np.zeros((16, 16), np.float32))
