"""GPU: b200_matmul_quantized bit for bit against the numpy oracle of its contract (tests/qmatmul_oracle.py), end to end from
b200_quantize, its bound against an f64 matmul of the dequantized operands, non-finite scales, ordering, pool use and
determinism, and the full-size 8192^3 Q8S/128 case."""
import numpy as np
import pytest

import qmatmul_oracle as qmo
import quant_oracle as qo
from cubecl_b200 import TensorHandle, matmul, quant, synth
from cubecl_b200.quant import QuantScheme, QuantizedTensor

pytestmark = pytest.mark.gpu

INT_VALUES = ["q8s", "q8f", "q4s", "q4f", "q2s", "q2f"]


def scheme_of(value, block=0, dt=None, tensor=False):
    return QuantScheme(value=value, block=block, block_scale=dt if block else None, tensor=tensor or block == 0)


def make(client, scheme, batch, rows, K, seed, scale_values=None):
    """Random codes over the value's whole range and random scales on the scale dtype's grid: (device tensor, host copy)."""
    rng = np.random.default_rng(seed)
    lo, hi = qo.RANGE[scheme.value]
    bits = qo.BITS[scheme.value]
    fields = (rng.integers(int(lo), int(hi) + 1, size=(batch, rows, K)) & ((1 << bits) - 1)).astype(np.uint8)
    values = qo.pack(fields, bits)
    raw = None
    if scheme.block:
        s = scale_values if scale_values is not None else \
            (rng.uniform(0.5, 2.0, size=(batch, rows, K // scheme.block)) * np.exp2(rng.integers(-4, 4, size=(batch, rows, K // scheme.block))))
        raw = qo.scale_store(scheme.block_scale, qo.round_up(scheme.block_scale, np.asarray(s, np.float32)))
    g = np.float32(rng.uniform(0.001, 0.01)) if scheme.has_tensor else None
    vt = TensorHandle.from_numpy(client, values, quant.VALUE_DTYPES.get(scheme.value, "u8"))
    st = TensorHandle.from_numpy(client, np.ascontiguousarray(raw), quant.SCALE_DTYPES[scheme.block_scale]) if raw is not None else None
    tt = TensorHandle.from_numpy(client, np.array([g], np.float32), "f32") if g is not None else None
    return QuantizedTensor(vt, st, tt, scheme, [batch, rows, K]), qmo.Operand(scheme, values, raw, g, batch, rows, K)


def run(client, qa, qb, out_dtype, stream=None):
    batch, M, N = qa.shape[0], qa.shape[1], qb.shape[1]
    out = TensorHandle.empty_contiguous(client, [batch, M, N], out_dtype)
    matmul.launch_quantized(client, qa, qb, out, stream)
    return out


def check(client, qa, ha, qb, hb, out_dtype="f32"):
    got = run(client, qa, qb, out_dtype).to_numpy(client)
    exp = qmo.to_out(qmo.matmul(ha, hb), out_dtype)
    assert np.array_equal(got.view(np.uint8), np.ascontiguousarray(exp).view(np.uint8)), \
        np.argwhere(got.view(np.uint8).reshape(exp.shape + (-1,)) != np.ascontiguousarray(exp).view(np.uint8).reshape(exp.shape + (-1,)))[:4]


@pytest.mark.parametrize("va", INT_VALUES)
@pytest.mark.parametrize("vb", ["q8s", "q4f", "q2s"])
def test_every_value_on_each_side(client, va, vb):
    qa, ha = make(client, scheme_of(va, 32, "f32"), 1, 130, 256, 1)
    qb, hb = make(client, scheme_of(vb, 64, "ue8m0"), 1, 72, 256, 2)
    check(client, qa, ha, qb, hb)
    qa, ha = make(client, scheme_of(va), 1, 130, 256, 3)
    qb, hb = make(client, scheme_of(vb), 1, 72, 256, 4)
    check(client, qa, ha, qb, hb)


@pytest.mark.parametrize("dt", ["f32", "f16", "bf16", "ue8m0", "ue4m3"])
@pytest.mark.parametrize("block", [32, 64, 128])
def test_block_sizes_and_scale_dtypes(client, block, dt):
    qa, ha = make(client, scheme_of("q8s", block, dt), 1, 200, 512, 5)
    qb, hb = make(client, scheme_of("q8s", block, dt), 1, 136, 512, 6)
    check(client, qa, ha, qb, hb)
    # two levels on both sides
    qa, ha = make(client, scheme_of("q8s", block, dt, tensor=True), 1, 200, 512, 7)
    qb, hb = make(client, scheme_of("q4s", block, dt, tensor=True), 1, 136, 512, 8)
    check(client, qa, ha, qb, hb, "bf16")


@pytest.mark.parametrize("out_dtype", ["f32", "bf16", "f16"])
@pytest.mark.parametrize("sa,sb", [(("q8s", 0), ("q8s", 128)), (("q8s", 128), ("q8s", 0)), (("q8s", 32), ("q4s", 128)),
                                   (("q8f", 128), ("q8s", 64)), (("q8s", 0), ("q8s", 0))])
def test_mixed_levels_outputs_ragged_batch(client, sa, sb, out_dtype):
    qa, ha = make(client, scheme_of(sa[0], sa[1], "f16"), 3, 77, 384, 9)
    qb, hb = make(client, scheme_of(sb[0], sb[1], "bf16"), 3, 45, 384, 10)
    check(client, qa, ha, qb, hb, out_dtype)


@pytest.mark.parametrize("variant", ["2sm_n256", "2sm_n128", "1sm_n128"])
def test_each_tile_variant(client, variant):
    client.set_option("gemm.variant", variant)
    try:
        qa, ha = make(client, scheme_of("q8s"), 1, 300, 640, 11)
        qb, hb = make(client, scheme_of("q8s"), 1, 520, 640, 12)
        check(client, qa, ha, qb, hb, "bf16")
        if variant != "2sm_n256":   # the per-block fold has 128-wide tiles only
            qa, ha = make(client, scheme_of("q8s", 32, "f32"), 1, 300, 640, 13)
            qb, hb = make(client, scheme_of("q8s", 64, "f16", tensor=True), 1, 520, 640, 14)
            check(client, qa, ha, qb, hb, "f32")
    finally:
        client.set_option("gemm.variant", "auto")


def test_staged_and_unaligned_codes(client):
    # K % 16 != 0 (per-tensor, Q8): the staging pass; Q2 rows of K = 100 need the widening pass with a padded pitch
    qa, ha = make(client, scheme_of("q8s"), 2, 70, 100, 15)
    qb, hb = make(client, scheme_of("q2f"), 2, 33, 100, 16)
    check(client, qa, ha, qb, hb, "f32")


def test_end_to_end_from_quantize_and_bound(client):
    M, N, K = 192, 160, 1024
    x = synth.uniform_f32(21, M * K, -2.0, 2.0).reshape(M, K)
    w = synth.uniform_f32(22, N * K, -1.0, 1.0).reshape(N, K)
    xd = TensorHandle.from_numpy(client, synth.to_device_dtype(x, "bf16"), "bf16")
    wd = TensorHandle.from_numpy(client, w, "f32")
    for sa, sb in ((QuantScheme().with_value("q8s").per_block(128, "f32"), QuantScheme().with_value("q8s").per_block(128, "f32")),
                   (QuantScheme().with_value("q8s").per_tensor(), QuantScheme().with_value("q4s").per_block(32, "f16").per_tensor()),
                   (QuantScheme().with_value("q8s").per_tensor(), QuantScheme().with_value("q8s").per_tensor())):
        qa, qb = quant.quantize(client, xd, sa), quant.quantize(client, wd, sb)
        out = TensorHandle.empty_contiguous(client, [M, N], "f32")
        matmul.launch_quantized(client, qa, qb, out)          # no sync between quantize and the matmul
        got = out.to_numpy(client)
        ops = []
        for q, rows in ((qa, M), (qb, N)):
            v = q.values.to_numpy(client).view(np.uint8)
            s = q.block_scales.to_numpy(client) if q.block_scales is not None else None
            if s is not None and q.scheme.block_scale in ("ue4m3", "ue8m0"):
                s = s.view(np.uint8)
            t = np.float32(q.tensor_scale.to_numpy(client)[0]) if q.tensor_scale is not None else None
            ops.append(qmo.Operand(q.scheme, v, s, t, 1, rows, K))
        exp = qmo.matmul(*ops)[0]
        assert np.array_equal(got.view(np.uint32), exp.view(np.uint32)), (sa, sb)
        da, db = ops[0].dequantized()[0], ops[1].dequantized()[0]
        ref = da @ db.T
        bk = qmo.kernel_block(*ops) or K
        bound = (K // bk + 2) * 2.0 ** -24 * (np.abs(da) @ np.abs(db).T) + np.abs(ref) * 2.0 ** -24
        assert np.all(np.abs(got - ref) <= bound), (sa, sb, np.max(np.abs(got - ref) - bound))


def test_non_finite_scales_touch_only_their_outputs(client):
    K = 256
    qa, ha = make(client, scheme_of("q8s", 32, "ue8m0"), 1, 64, K, 31, scale_values=np.ones((1, 64, K // 32), np.float32))
    raw = ha.scales.copy()
    raw[0, 5, 2] = 255   # ue8m0 code 255: NaN
    qa.block_scales = TensorHandle.from_numpy(client, raw, "ue8m0")
    ha.scales = raw
    sb = np.ones((1, 40, K // 32), np.float32)
    sb[0, 7, 1] = np.inf
    qb, hb = make(client, scheme_of("q8s", 32, "f32"), 1, 40, K, 32, scale_values=sb)
    got = run(client, qa, qb, "f32").to_numpy(client)
    exp = qmo.matmul(ha, hb)
    # IEEE does not fix a NaN's payload: NaN where the oracle has NaN, the same bits everywhere else
    assert np.array_equal(np.isnan(got), np.isnan(exp))
    ok = ~np.isnan(exp)
    assert np.array_equal(got[ok].view(np.uint32), exp[ok].view(np.uint32))
    bad = ~np.isfinite(got[0])
    assert bad[5].all() and bad[:, 7].all()
    mask = np.ones_like(bad)
    mask[5, :] = False
    mask[:, 7] = False
    assert not bad[mask].any()


def test_stream_order_pool_and_determinism(client):
    qa, ha = make(client, scheme_of("q4s", 32, "bf16", tensor=True), 2, 256, 1024, 41)
    qb, hb = make(client, scheme_of("q8s", 128, "f32"), 2, 384, 1024, 42)
    a = TensorHandle.empty_contiguous(client, [2, 256, 384], "bf16")
    b = TensorHandle.empty_contiguous(client, [2, 256, 384], "bf16")
    client.sync()
    base = client.memory_usage().bytes_in_use
    s = client.create_stream()
    try:
        matmul.launch_quantized(client, qa, qb, a, s)
        matmul.launch_quantized(client, qa, qb, b, s)
        client.sync_stream(s)
        assert client.memory_usage().bytes_in_use == base   # the pooled temporaries went back after the launches
        ga, gb = a.to_numpy(client), b.to_numpy(client)
    finally:
        client.destroy_stream(s)
    assert np.array_equal(ga.view(np.uint16), gb.view(np.uint16))
    assert np.array_equal(ga.view(np.uint16), qmo.to_out(qmo.matmul(ha, hb), "bf16").view(np.uint16))


def test_full_size_q8s_128_bf16(client):
    M = N = K = 8192
    qa, ha = make(client, scheme_of("q8s", 128, "f32"), 1, M, K, 51)
    qb, hb = make(client, scheme_of("q8s", 128, "f32"), 1, N, K, 52)
    out = run(client, qa, qb, "bf16")
    got = out.to_numpy(client).view(np.uint16).reshape(M, N)
    rows = np.random.default_rng(53).choice(M, 256, replace=False)
    exp = qmo.to_out(qmo.matmul(ha, hb, rows=rows), "bf16").view(np.uint16)[0]
    assert np.array_equal(got[rows], exp)
    # every 128 x 128 block: the f64 sum of the outputs against the f64 product of the dequantized operands, from row-group sums
    da, db = ha.dequantized()[0], hb.dequantized()[0]
    grp = lambda x: x.reshape(x.shape[0] // 128, 128, K).sum(axis=1)
    ref = grp(da) @ grp(db).T
    mag = grp(np.abs(da)) @ grp(np.abs(db)).T
    gf = synth.from_device_dtype(got, "bf16").astype(np.float64).reshape(M // 128, 128, N // 128, 128).sum(axis=(1, 3))
    assert np.all(np.abs(gf - ref) <= mag * ((K // 128 + 2) * 2.0 ** -24 + 2.0 ** -8))
