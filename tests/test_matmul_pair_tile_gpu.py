"""GPU parity of the 512 x 128 pair tile (2sm_m512, forced through gemm.variant) against the oracle.

2sm_m512 is a 2-CTA cluster tile of 512 x 128: each CTA holds 256 rows of A per stage, and each consumer warpgroup issues
two m64 wgmma blocks that share every B stage (4 x 48 KB stages).  Same oracle, same tolerances and the same operand-layout
matrix as tests/test_matmul_gpu.py; shapes are chosen so that the 4-stage ring wraps, tiles are ragged in M, N and K, and
every CTA pair walks several tiles (barrier parities flip).
"""
import numpy as np
import pytest

import oracle
from cubecl_b200 import TensorHandle, matmul, synth
from gpu_util import check_against_oracle, make_operand, run_matmul

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _reset_options(client):
    yield
    client.set_option("gemm.variant", "auto")
    client.set_option("gemm.epilogue", "tma")
    client.set_option("gemm.split_k", "auto")


@pytest.mark.parametrize("lhs_t", [False, True], ids=["lhs_mk", "lhs_km"])
@pytest.mark.parametrize("rhs_t", [False, True], ids=["rhs_kn", "rhs_nk"])
@pytest.mark.parametrize("in_dtype,out_dtype", [("bf16", "bf16"), ("bf16", "f32"), ("f16", "f16"), ("f16", "f32")])
def test_pair_tile_512_parity_ragged(client, lhs_t, rhs_t, in_dtype, out_dtype):
    client.set_option("gemm.variant", "2sm_m512")
    M, N, K = 704, 520, 328   # 2 x 3 tiles, ragged in M (704 = 512 + 192), N and K (5.1 k-blocks: the 4-stage ring wraps)
    a_dev, a = make_operand((K, M) if lhs_t else (M, K), in_dtype, 311)
    b_dev, b = make_operand((N, K) if rhs_t else (K, N), in_dtype, 312)
    before = client.launch_count()
    got = run_matmul(client, a_dev, b_dev, in_dtype, out_dtype, rhs_transposed=rhs_t, lhs_transposed=lhs_t)
    assert client.launch_count() - before == 1
    check_against_oracle(got, np.ascontiguousarray(a.T) if lhs_t else a, b.T if rhs_t else b, out_dtype,
                         tight=1e-5 if out_dtype == "f32" else None)


@pytest.mark.parametrize("lhs_t", [False, True], ids=["lhs_mk", "lhs_km"])
@pytest.mark.parametrize("rhs_t", [False, True], ids=["rhs_kn", "rhs_nk"])
@pytest.mark.parametrize("dtype,out_dtype", [("f8e4m3", "bf16"), ("f8e5m2", "f16")])
def test_pair_tile_512_parity_fp8(client, lhs_t, rhs_t, dtype, out_dtype):
    client.set_option("gemm.variant", "2sm_m512")
    M, N, K = 704, 528, 720   # 16-byte multiples for 1-byte rows; 5.6 k-blocks of 128 fp8 elements
    a_dev, a = make_operand((K, M) if lhs_t else (M, K), dtype, 351)
    b_dev, b = make_operand((N, K) if rhs_t else (K, N), dtype, 352)
    before = client.launch_count()
    got = run_matmul(client, a_dev, b_dev, dtype, out_dtype, rhs_transposed=rhs_t, lhs_transposed=lhs_t)
    assert client.launch_count() - before == 3   # fp8 operands widened exactly to f16 (one pass each), then the f16 kernel
    check_against_oracle(got, np.ascontiguousarray(a.T) if lhs_t else a, b.T if rhs_t else b, out_dtype)
    client.set_option("gemm.variant", "2sm_n256")   # and bit-identical to the 256 x 256 tile
    ref = run_matmul(client, a_dev, b_dev, dtype, out_dtype, rhs_transposed=rhs_t, lhs_transposed=lhs_t)
    assert np.array_equal(got, ref)


@pytest.mark.parametrize("variant", ["2sm_m512"])
@pytest.mark.parametrize("epilogue", ["tma", "direct"])
def test_pair_tile_many_tiles_per_cta_pair(client, variant, epilogue):
    # 9 x 34 = 306 tiles of 512 x 128 on 66 CTA pairs: every pair runs 4-5 tiles back to back, so the stage barriers change
    # parity across tiles and the epilogue of one tile overlaps the next tile's loads
    client.set_option("gemm.variant", variant)
    client.set_option("gemm.epilogue", epilogue)
    M, N, K = 4608, 4352, 640
    a_dev, a = make_operand((M, K), "bf16", 321)
    b_dev, b = make_operand((K, N), "bf16", 322)
    got = run_matmul(client, a_dev, b_dev, "bf16", "bf16")
    check_against_oracle(got, a, b, "bf16")
    # and bit-identical to the default tile (same k order within a tile row, f32 accumulate, one rounding to bf16)
    client.set_option("gemm.variant", "2sm_n256")
    ref = run_matmul(client, a_dev, b_dev, "bf16", "bf16")
    assert np.array_equal(got, ref)


def test_pair_tile_512_batched_fused_epilogue_and_pitched_output(client):
    from math import erf
    client.set_option("gemm.variant", "2sm_m512")
    B, M, N, K = 3, 520, 264, 192
    a_dev, a = make_operand((B, M, K), "bf16", 331)
    b_dev, b = make_operand((K, N), "bf16", 332)                       # rhs broadcast over the batch
    bias = synth.uniform_f32(333, N, -2.0, 2.0)
    lhs, rhs = TensorHandle.from_numpy(client, a_dev, "bf16"), TensorHandle.from_numpy(client, b_dev, "bf16")
    pitch = 272                                                         # output rows pitched: 264 columns inside 272
    buf = TensorHandle.from_numpy(client, np.full((B, M, pitch), -7.0, np.float32), "f32")
    out = TensorHandle(buf.handle, [B, M, N], [M * pitch, pitch, 1], "f32")
    rhs3 = TensorHandle(rhs.handle, [1, K, N], [K * N, N, 1], "bf16")
    matmul.launch(client, lhs, rhs3, out, alpha=0.25, bias=TensorHandle.from_numpy(client, bias, "f32"), activation="gelu")
    full = buf.to_numpy(client).reshape(B, M, pitch)
    assert np.all(full[:, :, N:] == -7.0)                                # nothing written outside the M x N window
    for i in range(B):
        f64, fabs = oracle.matmul_f64(a[i], b)
        x = 0.25 * f64 + bias.astype(np.float64)[None, :]
        exp = 0.5 * x * (1.0 + np.vectorize(erf)(x / np.sqrt(2.0)))
        scale = 0.25 * fabs + np.abs(bias)[None, :] + 1e-6
        assert np.max(np.abs(full[i, :, :N] - exp) / scale) <= 1e-5


def test_pair_tile_512_rejects_dtypes_it_is_not_built_for(client):
    from cubecl_b200 import ServerError
    a_dev, _ = make_operand((256, 64), "f32", 341)
    b_dev, _ = make_operand((64, 256), "f32", 342)
    client.set_option("gemm.variant", "2sm_m512")
    with pytest.raises(ServerError):
        run_matmul(client, a_dev, b_dev, "f32", "f32")
