"""GPU: b200_matmul_quantized_fp8 bit for bit against the exact-input oracle (tests/qmatmul_fp8_oracle.py) on integer-valued
codes, its error bound on real data quantized by b200_quantize, the 128 x 128 weight-scale recipe, non-finite codes and
scales, ordering, pool use and determinism, and the full-size 8192^3 e4m3/128 case."""
import numpy as np
import pytest

import qmatmul_fp8_oracle as qf8
import qmatmul_oracle as qmo
import quant_oracle as qo
from cubecl_b200 import TensorHandle, matmul, quant, synth
from cubecl_b200.quant import QuantScheme, QuantizedTensor

pytestmark = pytest.mark.gpu

FP8 = ["e4m3", "e5m2"]


def scheme_of(value, block=0, dt=None, tensor=False):
    return QuantScheme(value=value, block=block, block_scale=dt if block else None, tensor=tensor or block == 0)


def make(client, scheme, batch, rows, K, seed, scale_values=None, q=None):
    """Integer-valued codes in [-4, 4] (every partial sum of a block of <= 128 stays within 2^11) and random scales on the scale
    dtype's grid: (device tensor, host copy)."""
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
    return QuantizedTensor(vt, st, tt, scheme, [batch, rows, K]), qmo.Operand(scheme, values, raw, g, batch, rows, K)


def run(client, qa, qb, out_dtype, stream=None):
    batch, M, N = qa.shape[0], qa.shape[1], qb.shape[1]
    out = TensorHandle.empty_contiguous(client, [batch, M, N], out_dtype)
    matmul.launch_quantized_fp8(client, qa, qb, out, stream)
    return out


def check(client, qa, ha, qb, hb, out_dtype="f32"):
    got = run(client, qa, qb, out_dtype).to_numpy(client)
    exp = np.ascontiguousarray(qmo.to_out(qf8.matmul(ha, hb), out_dtype))
    g8, e8 = got.view(np.uint8).reshape(exp.shape + (-1,)), exp.view(np.uint8).reshape(exp.shape + (-1,))
    assert np.array_equal(g8, e8), np.argwhere((g8 != e8).any(-1))[:4]


@pytest.mark.parametrize("va", FP8)
@pytest.mark.parametrize("vb", FP8)
def test_every_value_pair(client, va, vb):
    qa, ha = make(client, scheme_of(va, 128, "f32"), 1, 130, 512, 1)
    qb, hb = make(client, scheme_of(vb, 128, "f32"), 1, 200, 512, 2)
    check(client, qa, ha, qb, hb, "bf16")
    qa, ha = make(client, scheme_of(va, 32, "f16"), 1, 130, 256, 3)
    qb, hb = make(client, scheme_of(vb), 1, 72, 256, 4)
    check(client, qa, ha, qb, hb)


@pytest.mark.parametrize("dt", ["f32", "f16", "bf16", "ue8m0", "ue4m3"])
@pytest.mark.parametrize("block", [32, 64, 128])
def test_block_sizes_and_scale_dtypes(client, block, dt):
    qa, ha = make(client, scheme_of("e4m3", block, dt), 1, 200, 512, 5)
    qb, hb = make(client, scheme_of("e4m3", block, dt), 1, 136, 512, 6)
    check(client, qa, ha, qb, hb)
    # two levels on both sides, e5m2 on the rhs
    qa, ha = make(client, scheme_of("e4m3", block, dt, tensor=True), 1, 200, 512, 7)
    qb, hb = make(client, scheme_of("e5m2", block, dt, tensor=True), 1, 136, 512, 8)
    check(client, qa, ha, qb, hb, "bf16")


@pytest.mark.parametrize("out_dtype", ["f32", "bf16", "f16"])
@pytest.mark.parametrize("sa,sb", [(("e4m3", 0), ("e4m3", 128)), (("e5m2", 128), ("e4m3", 0)), (("e4m3", 32), ("e5m2", 128)),
                                   (("e4m3", 64), ("e4m3", 32)), (("e5m2", 0), ("e4m3", 0))])
def test_mixed_levels_outputs_ragged_batch(client, sa, sb, out_dtype):
    qa, ha = make(client, scheme_of(sa[0], sa[1], "f16"), 3, 77, 384, 9)
    qb, hb = make(client, scheme_of(sb[0], sb[1], "bf16"), 3, 45, 384, 10)
    check(client, qa, ha, qb, hb, out_dtype)


@pytest.mark.parametrize("variant", ["2sm_n128", "1sm_n128"])
def test_each_tile_variant(client, variant):
    client.set_option("gemm.variant", variant)
    try:
        qa, ha = make(client, scheme_of("e4m3"), 1, 300, 640, 11)
        qb, hb = make(client, scheme_of("e5m2"), 1, 520, 640, 12)
        check(client, qa, ha, qb, hb, "bf16")
        qa, ha = make(client, scheme_of("e4m3", 32, "f32"), 1, 300, 640, 13)
        qb, hb = make(client, scheme_of("e4m3", 64, "f16", tensor=True), 1, 520, 640, 14)
        check(client, qa, ha, qb, hb, "f32")
    finally:
        client.set_option("gemm.variant", "auto")


def test_staged_unaligned_codes_and_short_last_block(client):
    # K = 200: not a multiple of 16 (the codes are staged) nor of 128 (per-tensor sides fold a short last block of 72)
    qa, ha = make(client, scheme_of("e4m3"), 2, 70, 200, 15)
    qb, hb = make(client, scheme_of("e5m2"), 2, 33, 200, 16)
    check(client, qa, ha, qb, hb, "f32")
    # an unaligned code base: a view 8 bytes into a larger buffer
    qa, ha = make(client, scheme_of("e4m3", 64, "f32"), 1, 96, 256, 17)
    qb, hb = make(client, scheme_of("e4m3", 64, "f32"), 1, 80, 256, 18)
    big = TensorHandle.from_numpy(client, np.concatenate([np.zeros(8, np.uint8), ha.values.reshape(-1)]), "u8")
    qa.values = TensorHandle.new_contiguous([1, 96, 256], big.handle.offset(8, ha.values.size), "f8e4m3")
    check(client, qa, ha, qb, hb, "bf16")


def _bound_ratio(got, ref, mag, out_dtype):
    """max |out - ref| / (sum_k |a_k b_k|), and whether |out - ref| <= 2^-10 sum |a_k b_k| + one output ulp everywhere."""
    ulp = {"f32": 2.0 ** -23, "bf16": 2.0 ** -7, "f16": 2.0 ** -10}[out_dtype] * np.abs(ref)
    err = np.abs(got - ref)
    return float(np.max(err / np.maximum(mag, 1e-300))), bool(np.all(err <= 2.0 ** -10 * mag + ulp))


def _host_operand(client, q, rows, K):
    v = q.values.to_numpy(client).view(np.uint8)
    s = q.block_scales.to_numpy(client) if q.block_scales is not None else None
    t = np.float32(q.tensor_scale.to_numpy(client)[0]) if q.tensor_scale is not None else None
    return qmo.Operand(q.scheme, v, s, t, 1, rows, K)


@pytest.mark.parametrize("M,N,K,sample", [(8192, 8192, 8192, 128), (256, 256, 16384, None)])
def test_error_bound_on_quantized_real_data(client, M, N, K, sample):
    x = synth.uniform_f32(21, M * K, -2.0, 2.0).reshape(M, K) * np.exp2(synth.uniform_f32(23, M * K, -3.0, 3.0).reshape(M, K))
    w = synth.uniform_f32(22, N * K, -1.0, 1.0).reshape(N, K)
    xd = TensorHandle.from_numpy(client, synth.to_device_dtype(x.astype(np.float32), "bf16"), "bf16")
    wd = TensorHandle.from_numpy(client, synth.to_device_dtype(w, "bf16"), "bf16")
    del x, w
    s = QuantScheme().with_value("e4m3").per_block(128, "f32")
    qa, qb = quant.quantize(client, xd, s), quant.quantize(client, wd, s)
    out = TensorHandle.empty_contiguous(client, [M, N], "f32")
    matmul.launch_quantized_fp8(client, qa, qb, out)          # no sync between quantize and the matmul
    # the same operands dequantized to bf16 through b200_dequantize, then the bf16 GEMM: the yardstick
    da16 = TensorHandle.empty_contiguous(client, [M, K], "bf16")
    db16 = TensorHandle.empty_contiguous(client, [N, K], "bf16")
    quant.launch_dequantize(client, qa, da16)
    quant.launch_dequantize(client, qb, db16)
    out16 = TensorHandle.empty_contiguous(client, [M, N], "f32")
    matmul.launch(client, da16, db16.transposed(), out16)
    got, got16 = out.to_numpy(client), out16.to_numpy(client)
    rows = np.arange(M) if sample is None else np.random.default_rng(24).choice(M, sample, replace=False)
    ha, hb = _host_operand(client, qa, M, K), _host_operand(client, qb, N, K)
    da, db = ha.dequantized()[0][rows], hb.dequantized()[0]
    ref = da @ db.T
    mag = np.abs(da) @ np.abs(db).T
    ratio, ok = _bound_ratio(got[rows], ref, mag, "f32")
    ratio16, _ = _bound_ratio(got16[rows], ref, mag, "f32")
    print(f"\nfp8 error bound {M}x{N}x{K}: max |out - ref| / sum|a b| = {ratio:.3e} (2^{np.log2(max(ratio, 1e-300)):.2f}); "
          f"dequantize + bf16 matmul on the same data: {ratio16:.3e} (2^{np.log2(max(ratio16, 1e-300)):.2f})")
    assert ok, ratio


def _blockwise_weight(N, K, seed):
    """A DeepSeek-style weight: e4m3 codes [N, K] with one f32 scale per 128 x 128 block ([N / 128, K / 128])."""
    rng = np.random.default_rng(seed)
    w = (rng.standard_normal((N // 128, 128, K // 128, 128)) * np.exp2(rng.integers(-3, 3, size=(N // 128, 1, K // 128, 1))))
    w = w.reshape(N, K).astype(np.float32)
    blk = np.abs(w.reshape(N // 128, 128, K // 128, 128)).max(axis=(1, 3)).astype(np.float32)
    s2 = (blk / np.float32(448.0)).astype(np.float32)
    codes = qo.fp8_codes((w.reshape(N // 128, 128, K // 128, 128) / s2[:, None, :, None]).reshape(N, K), "e4m3")
    return codes, s2


def _recipe_run(client, M, N, K):
    x = synth.uniform_f32(31, M * K, -1.0, 1.0).reshape(M, K)
    qa = quant.quantize(client, TensorHandle.from_numpy(client, synth.to_device_dtype(x, "bf16"), "bf16"),
                        QuantScheme().with_value("e4m3").per_block(128, "f32"))
    codes, s2 = _blockwise_weight(N, K, 32)
    s_rows = np.ascontiguousarray(np.repeat(s2, 128, axis=0))   # the recipe: each scale row repeated 128 times -> [N, K / 128]
    sb = QuantScheme().with_value("e4m3").per_block(128, "f32")
    qb = QuantizedTensor(TensorHandle.from_numpy(client, codes, "f8e4m3"), TensorHandle.from_numpy(client, s_rows, "f32"), None, sb, [N, K])
    out = TensorHandle.empty_contiguous(client, [M, N], "f32")
    matmul.launch_quantized_fp8(client, qa, qb, out)
    ha = _host_operand(client, qa, M, K)
    hb = qmo.Operand(sb, codes, s_rows, None, 1, N, K)
    return qa, ha, codes, s2, hb, out.to_numpy(client)


def test_128x128_weight_scale_recipe(client):
    M, N, K = 256, 384, 1024
    _, ha, codes, s2, hb, got = _recipe_run(client, M, N, K)
    # the effective scales of the expanded operand are the 128 x 128 scales themselves
    wq = synth.fp8_bits_to_f32(codes, "f8e4m3").reshape(N // 128, 128, K // 128, 128)
    w_deq = (wq * s2[:, None, :, None]).astype(np.float32).reshape(N, K).astype(np.float64)
    assert np.array_equal(hb.dequantized()[0], w_deq)
    da = ha.dequantized()[0]
    ref, mag = da @ w_deq.T, np.abs(da) @ np.abs(w_deq).T
    ratio, ok = _bound_ratio(got, ref, mag, "f32")
    assert ok, ratio


def test_128x128_weight_scales_agree_with_torch_scaled_mm(client):
    torch = pytest.importorskip("torch")
    F = torch.nn.functional
    if not torch.cuda.is_available() or not hasattr(F, "scaled_mm") or not hasattr(F, "ScalingType"):
        pytest.skip("this torch has no F.scaled_mm with block-wise scaling on this GPU")
    M, N, K = 256, 384, 1024
    qa, ha, codes, s2, hb, got = _recipe_run(client, M, N, K)
    a8 = torch.from_numpy(qa.values.to_numpy(client).view(np.uint8).reshape(M, K).copy()).view(torch.float8_e4m3fn).cuda()
    sa = torch.from_numpy(qa.block_scales.to_numpy(client).reshape(M, K // 128).copy()).cuda()
    b8 = torch.from_numpy(codes.reshape(N, K).copy()).view(torch.float8_e4m3fn).cuda()
    sbt = torch.from_numpy(s2.copy()).cuda()
    try:
        # torch's block-wise recipes: 1 x 128 activation scales outer-dim-major, 128 x 128 weight scales, B column-major
        ref = F.scaled_mm(a8, b8.t(), sa.t().contiguous().t(), F.ScalingType.BlockWise1x128, sbt, F.ScalingType.BlockWise128x128,
                          output_dtype=torch.float32)
        torch.cuda.synchronize()
    except Exception as e:   # noqa: BLE001 -- an unsupported recipe is reported, not failed
        pytest.skip(f"this torch does not accept F.scaled_mm(BlockWise1x128, BlockWise128x128) on this GPU: {type(e).__name__}: {e}")
    t = ref.cpu().numpy().astype(np.float64)
    da, db = ha.dequantized()[0], hb.dequantized()[0]
    mag = np.abs(da) @ np.abs(db).T
    assert np.all(np.abs(got - t) <= 2.0 * 2.0 ** -10 * mag + 2.0 ** -22 * np.abs(t))


def test_non_finite_codes_and_scales_touch_only_their_outputs(client):
    K = 256
    rng = np.random.default_rng(60)
    qa_vals = rng.integers(-4, 5, size=(1, 64, K)).astype(np.float32)
    qb_vals = rng.integers(-4, 5, size=(1, 40, K)).astype(np.float32)
    qb_vals[0, 3, 17] = np.inf                                    # e5m2 +inf
    qb_vals[0, 9, 200] = -np.inf                                  # e5m2 -inf
    qa, ha = make(client, scheme_of("e4m3", 32, "f32"), 1, 64, K, 61, scale_values=np.ones((1, 64, K // 32), np.float32), q=qa_vals)
    codes = ha.values.copy()
    codes[0, 11, 5] = 0x7F                                        # e4m3 NaN
    qa.values = TensorHandle.from_numpy(client, codes, "f8e4m3")
    ha.values = codes
    sa = np.ones((1, 64, K // 32), np.float32)
    sa[0, 5, 2] = np.nan
    sb = np.ones((1, 40, K // 32), np.float32)
    sb[0, 7, 1] = np.inf
    qa.block_scales = TensorHandle.from_numpy(client, qo.scale_store("f32", sa), "f32")
    ha.scales = qo.scale_store("f32", sa)
    qb, hb = make(client, scheme_of("e5m2", 32, "f32"), 1, 40, K, 62, scale_values=sb, q=qb_vals)
    got = run(client, qa, qb, "f32").to_numpy(client)[0]
    bad = ~np.isfinite(got)
    mask = np.ones_like(bad)
    for r in (5, 11):
        mask[r, :] = False
    for c in (3, 7, 9):
        mask[:, c] = False
    assert bad[5].all() and bad[11].all() and bad[:, 7].all()
    assert not bad[mask].any()
    exp = qf8.matmul(ha, hb)[0]
    assert np.array_equal(got[mask].view(np.uint32), exp[mask].view(np.uint32))


def test_stream_order_pool_and_determinism(client):
    qa, ha = make(client, scheme_of("e4m3", 32, "bf16", tensor=True), 2, 256, 1024, 41)
    qb, hb = make(client, scheme_of("e5m2", 128, "f32"), 2, 384, 1024, 42)
    a = TensorHandle.empty_contiguous(client, [2, 256, 384], "bf16")
    b = TensorHandle.empty_contiguous(client, [2, 256, 384], "bf16")
    client.sync()
    base = client.memory_usage().bytes_in_use
    s = client.create_stream()
    try:
        matmul.launch_quantized_fp8(client, qa, qb, a, s)
        matmul.launch_quantized_fp8(client, qa, qb, b, s)
        client.sync_stream(s)
        assert client.memory_usage().bytes_in_use == base   # the pooled temporaries went back after the launches
        ga, gb = a.to_numpy(client), b.to_numpy(client)
    finally:
        client.destroy_stream(s)
    assert np.array_equal(ga.view(np.uint16), gb.view(np.uint16))
    assert np.array_equal(ga.view(np.uint16), qmo.to_out(qf8.matmul(ha, hb), "bf16").view(np.uint16))


def test_full_size_e4m3_128_bf16(client):
    M = N = K = 8192
    qa, ha = make(client, scheme_of("e4m3", 128, "f32"), 1, M, K, 51)
    qb, hb = make(client, scheme_of("e4m3", 128, "f32"), 1, N, K, 52)
    got = run(client, qa, qb, "bf16").to_numpy(client).view(np.uint16).reshape(M, N)
    rows = np.random.default_rng(53).choice(M, 128, replace=False)
    exp = qmo.to_out(qf8.matmul(ha, hb, rows=rows), "bf16").view(np.uint16)[0]
    assert np.array_equal(got[rows], exp)
