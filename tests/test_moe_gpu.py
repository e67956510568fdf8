"""GPU: mixture-of-experts routing against tests/moe_oracle.py -- plan and permute bit for bit (up to 2^18 slots, 1 to 1024
experts, empty / first-only / all-in-one experts, dropped ids, untouched sentinel rows), route ids exactly and weights within
the bound of moe_oracle.weight_bound, DeepSeek-V3 group-limited routing, combine and its backward bit for bit on
integer-valued data, an end-to-end bf16 layer and its backward against torch autograd, the fp8 recipe (quantize, then
permute codes and scales) against quantize-after-permute, layers that follow inputs rewritten on the stream, enqueue without
a host sync, and run-to-run determinism."""
import ctypes as C
import time

import numpy as np
import pytest
import torch

import moe_oracle as mo
from cubecl_b200 import TensorHandle, _ffi, matmul, moe, quant, synth
from cubecl_b200.quant import QuantizedTensor, QuantScheme

pytestmark = pytest.mark.gpu


def up(c, arr, dtype):
    return TensorHandle.from_numpy(c, synth.to_device_dtype(np.asarray(arr, np.float32), dtype) if dtype in ("f32", "bf16", "f16")
                                   else np.ascontiguousarray(arr), dtype)


def down(c, t):
    return synth.from_device_dtype(t.to_numpy(c), t.dtype) if t.dtype in ("f32", "bf16", "f16") else t.to_numpy(c)


def filled(c, shape, dtype, byte=0x5A):
    """A device tensor whose bytes are all `byte` (the sentinel of rows a call must not write)."""
    np_dt = {"i32": np.int32, "f32": np.float32, "u8": np.uint8, "bf16": np.uint16, "f16": np.uint16}[dtype]
    host = np.full(int(np.prod(shape)) * np.dtype(np_dt).itemsize, byte, np.uint8).view(np_dt).reshape(shape)
    return TensorHandle.from_numpy(c, host, dtype), host


# ---------------------------------------------------------------------------------------------- plan
def ids_for(kind, T, k, E, seed):
    rng = np.random.default_rng(seed)
    if kind == "random":
        return rng.integers(0, E, (T, k)).astype(np.int32)
    if kind == "empty_experts":        # only every third expert is used
        return (rng.integers(0, (E + 2) // 3, (T, k)) * 3 % E).astype(np.int32)
    if kind == "first_only":
        return np.zeros((T, k), np.int32)
    if kind == "all_in_one":
        return np.full((T, k), E - 1, np.int32)
    if kind == "dropped":              # expert parallelism: non-local experts marked outside [0, E)
        ids = rng.integers(0, E, (T, k)).astype(np.int32)
        m = rng.uniform(size=(T, k))
        ids[m < 0.2] = -1
        ids[(m >= 0.2) & (m < 0.3)] = E + 7
        return ids
    raise ValueError(kind)


PLAN_CASES = [("random", 65536, 4, 256), ("random", 1000, 1, 1), ("random", 5000, 2, 8), ("random", 4096, 8, 128),
              ("random", 8192, 8, 1024), ("random", 3, 2, 8), ("empty_experts", 3000, 8, 128), ("first_only", 2500, 2, 8),
              ("all_in_one", 2049, 8, 256), ("dropped", 10000, 8, 256), ("dropped", 777, 6, 1024), ("dropped", 1, 1, 1),
              ("dropped", 300001, 8, 256)]       # 2.4M slots: 512 per warp, so the [E][CTAs] table stays within 1024 CTAs


@pytest.mark.parametrize("kind,T,k,E", PLAN_CASES)
def test_plan_matches_oracle(client, kind, T, k, E):
    ids = ids_for(kind, T, k, E, T + E)
    offs, o_h = filled(client, [E], "i32")
    row_of, _ = filled(client, [T, k], "i32")
    slot_of, _ = filled(client, [T * k], "i32")
    moe.plan(client, up(client, ids, "i32"), E, offs, row_of, slot_of)
    client.sync()
    w_offs, w_row, w_slot = mo.plan(ids, E)
    np.testing.assert_array_equal(offs.to_numpy(client), w_offs)
    np.testing.assert_array_equal(row_of.to_numpy(client), w_row)
    np.testing.assert_array_equal(slot_of.to_numpy(client), w_slot)


def test_plan_with_no_slots_zeroes_offs(client):
    offs, _ = filled(client, [16], "i32")
    dummy = TensorHandle.empty_contiguous(client, [0, 4], "i32")
    moe.plan(client, dummy, 16, offs, TensorHandle.empty_contiguous(client, [0, 4], "i32"),
             TensorHandle.empty_contiguous(client, [0], "i32"))
    client.sync()
    assert not offs.to_numpy(client).any()


# ---------------------------------------------------------------------------------------------- permute
@pytest.mark.parametrize("row_bytes,src_pitch,dst_pitch", [(8192, 8192, 8192), (7168, 7168, 7168), (224, 224, 224), (56, 56, 56),
                                                           (14, 14, 14), (8192, 8208, 8224), (12, 20, 16)])
def test_permute_matches_oracle(client, row_bytes, src_pitch, dst_pitch):
    T, k, E = 1500, 8, 64
    ids = ids_for("dropped", T, k, E, row_bytes)
    _, _, slot_of = mo.plan(ids, E)
    rng = np.random.default_rng(row_bytes)
    src_full = rng.integers(0, 256, (T, src_pitch), dtype=np.uint8)
    src = TensorHandle(TensorHandle.from_numpy(client, src_full, "u8").handle, [T, row_bytes], [src_pitch, 1], "u8")
    dst_dev, dst_init = filled(client, [T * k, dst_pitch], "u8", 0xA7)
    dst = TensorHandle(dst_dev.handle, [T * k, row_bytes], [dst_pitch, 1], "u8")
    moe.permute(client, src, up(client, slot_of, "i32"), k, dst)
    client.sync()
    want = dst_init.copy()
    want[:, :row_bytes] = mo.permute(src_full[:, :row_bytes], slot_of, k, dst_init[:, :row_bytes])
    np.testing.assert_array_equal(dst_dev.to_numpy(client), want)     # rows without a slot and the pitch padding untouched


def test_permute_bf16_rows_through_the_api(client):
    T, k, E, K = 300, 2, 8, 96
    ids = ids_for("random", T, k, E, 1)
    _, _, slot_of = mo.plan(ids, E)
    x = np.random.default_rng(2).standard_normal((T, K)).astype(np.float32)
    xs = moe.permute_alloc(client, up(client, x, "bf16"), up(client, slot_of, "i32"), k)
    client.sync()
    xb = synth.bf16_bits_to_f32(synth.f32_to_bf16_bits(x))
    np.testing.assert_array_equal(down(client, xs), mo.permute(xb, slot_of, k, np.zeros((T * k, K), np.float32)))


# ---------------------------------------------------------------------------------------------- route
def run_route(c, logits, dtype, k, stride=None, bias=None, **kw):
    T, E = logits.shape
    if stride:
        pad = np.zeros((T, stride), np.float32)
        pad[:, :E] = logits
        full = up(c, pad, dtype)
        lt = TensorHandle(full.handle, [T, E], [stride, 1], dtype)
    else:
        lt = up(c, logits, dtype)
    ids, w = moe.route_alloc(c, lt, k, bias=up(c, bias, "f32") if bias is not None else None, **kw)
    c.sync()
    return ids.to_numpy(c), w.to_numpy(c)


def separated(rng, T, E, dtype):
    """Distinct logits exactly representable in `dtype` (integers / 16 within +-128 / 16 for the 16-bit types)."""
    span = min(E, 256) if dtype != "f32" else E
    return np.stack([rng.choice(span, E, replace=E > span) for _ in range(T)]).astype(np.float32) / 16 - span / 32


@pytest.mark.parametrize("dtype", ["f32", "bf16", "f16"])
@pytest.mark.parametrize("score,renorm,E,k", [("softmax", True, 8, 2), ("softmax", True, 128, 8), ("sigmoid", False, 256, 8),
                                              ("softmax", False, 1024, 32), ("sigmoid", True, 64, 1)])
def test_route_ids_exact_and_weights_bounded(client, dtype, score, renorm, E, k):
    rng = np.random.default_rng(E + k)
    logits = separated(rng, 777, E, dtype)
    ids, w = run_route(client, logits, dtype, k, score=score, renormalize=renorm, scale=1.5, stride=E + 24 if E == 128 else None)
    want_ids, want_w = mo.route(logits, k, score, renorm, scale=1.5)
    np.testing.assert_array_equal(ids, want_ids)
    bound = mo.weight_bound(logits, k, score)[:, None]
    rel = np.abs(w.astype(np.float64) - want_w) / np.abs(want_w)
    assert (rel <= bound).all(), (rel.max(), bound.min())


def test_route_ties_go_to_the_lower_index(client):
    rng = np.random.default_rng(7)
    T, E, k = 500, 64, 8
    logits = rng.integers(0, 3, (T, E)).astype(np.float32)            # every row full of ties
    logits[0, :8] = [np.nan, -np.inf, -0.0, 0.0, np.nan, 5.0, 5.0, -np.inf]
    logits[1] = np.nan
    logits[2] = -0.0
    logits[2, 5] = 0.0
    ids, _ = run_route(client, logits, "f32", k, score="sigmoid", renormalize=False)
    want, _ = mo.route(logits, k, "sigmoid", False)
    np.testing.assert_array_equal(ids, want)
    assert ids[1].tolist() == list(range(8)) and ids[2].tolist() == list(range(8))


def deepseek_inputs(T, seed):
    """Sigmoid logits and a bias whose keys rn(s + b), and the 4th / 5th group scores, are more than 1e-4 apart (far more than
    expf's error): rows are drawn on a 1/400 grid with a continuous jitter below 1/1000, and rows too close are skipped."""
    rng = np.random.default_rng(seed)
    E, G, n = 256, 8, 4 * T
    key = (np.stack([rng.permutation(E) for _ in range(n)]) + 40) / 400.0 + rng.uniform(0, 1e-3, (n, E))   # in (0.1, 0.74)
    bias = (rng.integers(-20, 21, E) / 1024.0).astype(np.float32)
    s = key - bias[None, :]
    logits = np.log(s / (1 - s)).astype(np.float32)
    kf = mo.keys(logits, "sigmoid", bias).astype(np.float64)
    gs = np.sort(np.sort(kf.reshape(n, G, E // G), axis=2)[:, :, -2:].sum(2), axis=1)
    ok = (np.diff(np.sort(kf, axis=1), axis=1).min(1) > 1e-4) & (gs[:, G - 4] - gs[:, G - 5] > 1e-4)
    assert ok.sum() >= T
    return logits[ok][:T], bias


def test_route_deepseek_group_limited(client):
    logits, bias = deepseek_inputs(300, 11)
    for dt in ("f32",):
        ids, w = run_route(client, logits, dt, 8, bias=bias, score="sigmoid", renormalize=True, n_group=8, topk_group=4, scale=2.5)
        want_ids, want_w = mo.route(logits, 8, "sigmoid", True, 8, 4, 2.5, bias)
        np.testing.assert_array_equal(ids, want_ids)
        assert (np.abs(w - want_w) / want_w <= mo.weight_bound(logits, 8, "sigmoid")[:, None]).all()
        # only experts of 4 groups were chosen
        assert max(len(set((row // 32).tolist())) for row in ids) <= 4


def test_route_softmax_with_bias(client):
    rng = np.random.default_rng(5)
    logits = separated(rng, 200, 64, "f32")
    bias = np.zeros(64, np.float32)
    bias[::2] = 0.5                                       # selection moves towards even experts; the weights stay s_e
    ids, w = run_route(client, logits, "f32", 4, bias=bias, renormalize=False)
    want_ids, want_w = mo.route(logits, 4, "softmax", False, bias=bias)
    kf = mo.keys(logits, "softmax", bias)
    ks = np.sort(kf, axis=1)
    assert (ks[:, -4] - ks[:, -5] > 1e-5).all()            # the cut is far from expf's error
    np.testing.assert_array_equal(ids, want_ids)
    assert (np.abs(w - want_w) / want_w <= mo.weight_bound(logits, 4, "softmax")[:, None]).all()


# ---------------------------------------------------------------------------------------------- combine
DTS = ["f32", "bf16", "f16"]


def combine_case(T, k, R, N, seed, drop=True):
    rng = np.random.default_rng(seed)
    row_of = rng.permutation(R)[: T * k].reshape(T, k).astype(np.int32) if R >= T * k else rng.integers(0, R, (T, k)).astype(np.int32)
    if drop:
        row_of[rng.uniform(size=(T, k)) < 0.15] = -1
    ys = rng.integers(-8, 9, (R, N)).astype(np.float32)
    w = rng.integers(-3, 4, (T, k)).astype(np.float32)
    dy = rng.integers(-8, 9, (T, N)).astype(np.float32)
    return row_of, ys, w, dy


@pytest.mark.parametrize("a", DTS)
@pytest.mark.parametrize("b", DTS)
@pytest.mark.parametrize("N", [256, 100])
def test_combine_and_backward_exact(client, a, b, N):
    T, k, R = 300, 4, 1300
    row_of, ys, w, dy = combine_case(T, k, R, N, N)
    ro, wt, yt = up(client, row_of, "i32"), up(client, w, "f32"), up(client, ys, a)
    y = moe.combine_alloc(client, yt, ro, wt, out_dtype=b)
    y0 = moe.combine_alloc(client, yt, ro, None, out_dtype=b)
    d_ys, d_ys_init = filled(client, [R, N], b, 0x3C)
    d_w = TensorHandle.empty_contiguous(client, [T, k], "f32")
    moe.combine_backward(client, up(client, dy, b), yt, wt, ro, d_ys, d_w)
    client.sync()
    np.testing.assert_array_equal(down(client, y), mo.combine(ys, row_of, w))
    np.testing.assert_array_equal(down(client, y0), mo.combine(ys, row_of))
    want_dys, want_dw = mo.combine_backward(dy, ys, w, row_of)
    np.testing.assert_array_equal(d_w.to_numpy(client), want_dw.astype(np.float32))
    got = d_ys.to_numpy(client)
    used = np.isin(np.arange(R), row_of)
    np.testing.assert_array_equal(synth.from_device_dtype(got[used], b), want_dys[used])
    raw = lambda a: a.view(np.uint8).reshape(R, -1)[~used]  # noqa: E731
    np.testing.assert_array_equal(raw(got), raw(d_ys_init))              # rows no slot references are not written


def test_combine_pitched_rows_and_out_of_range_rows(client):
    T, k, R, N = 64, 3, 200, 64
    row_of, ys, w, dy = combine_case(T, k, R, N, 9)
    row_of[0, 0], row_of[1, 2] = R, R + 100                # outside [0, rows): dropped
    full = np.zeros((R, N + 8), np.float32)
    full[:, :N] = ys
    yt = TensorHandle(up(client, full, "bf16").handle, [R, N], [N + 8, 1], "bf16")
    yfull, _ = filled(client, [T, N + 16], "f32")
    y = TensorHandle(yfull.handle, [T, N], [N + 16, 1], "f32")
    moe.combine(client, yt, up(client, row_of, "i32"), y, up(client, w, "f32"))
    client.sync()
    np.testing.assert_array_equal(y.to_numpy(client), mo.combine(ys, row_of, w))


# ---------------------------------------------------------------------------------------------- end to end
def layer_buffers(c, T, K, F, N, E, k):
    """Every output of one layer, allocated up front."""
    shapes = dict(logits=([T, E], "f32"), ids=([T, k], "i32"), weights=([T, k], "f32"), offs=([E], "i32"), row_of=([T, k], "i32"),
                  slot_of=([T * k], "i32"), xs=([T * k, K], "bf16"), h=([T * k, F], "bf16"), ys=([T * k, N], "bf16"), y=([T, N], "bf16"))
    return {n: TensorHandle.empty_contiguous(c, shape, dt) for n, (shape, dt) in shapes.items()}


def enqueue_layer(c, x, wr, w1, w2, k, b, stream=None):
    """route -> plan -> permute -> grouped GEMM (relu epilogue) -> grouped GEMM -> combine into the buffers `b`, all enqueued on
    `stream` with the non-allocating forms."""
    matmul.launch(c, x, wr, b["logits"], stream)
    moe.route(c, b["logits"], b["ids"], b["weights"], k, score="softmax", renormalize=True, stream=stream)
    moe.plan(c, b["ids"], w1.shape[0], b["offs"], b["row_of"], b["slot_of"], stream=stream)
    moe.permute(c, x, b["slot_of"], k, b["xs"], stream=stream)
    matmul.launch_grouped(c, b["xs"], w1, b["offs"], b["h"], activation="relu", stream=stream)
    matmul.launch_grouped(c, b["h"], w2, b["offs"], b["ys"], stream=stream)
    moe.combine(c, b["ys"], b["row_of"], b["y"], b["weights"], stream=stream)


def layer(c, x, wr, w1, w2, k):
    (T, K), (E, _, F), N = x.shape, w1.shape, w2.shape[2]
    b = layer_buffers(c, T, K, F, N, E, k)
    enqueue_layer(c, x, wr, w1, w2, k, b)
    return b


def layer_inputs(c, T, K, F, N, E, seed):
    rng = np.random.default_rng(seed)
    host = dict(x=rng.standard_normal((T, K)) * 0.5, wr=rng.standard_normal((K, E)) * 0.3, w1=rng.standard_normal((E, K, F)) / np.sqrt(K),
                w2=rng.standard_normal((E, F, N)) / np.sqrt(F))
    host = {n: synth.bf16_bits_to_f32(synth.f32_to_bf16_bits(v.astype(np.float32))) for n, v in host.items()}
    return host, {n: up(c, v, "bf16") for n, v in host.items()}


def test_end_to_end_bf16_layer_and_backward(client):
    T, K, F, N, E, k = 512, 256, 384, 256, 8, 2
    host, dev = layer_inputs(client, T, K, F, N, E, 1)
    out = layer(client, dev["x"], dev["wr"], dev["w1"], dev["w2"], k)
    client.sync()
    ids, weights = out["ids"].to_numpy(client), out["weights"].to_numpy(client)
    # forward: torch f32 per token with the device's routing
    x, w1, w2 = (torch.tensor(host[n], requires_grad=True) for n in ("x", "w1", "w2"))
    wt = torch.tensor(weights, requires_grad=True)
    ys_ref = torch.stack([torch.einsum("tf,tfn->tn", torch.relu(torch.einsum("tk,tkf->tf", x, w1[ids[:, j]])), w2[ids[:, j]])
                          for j in range(k)], 1)
    y_ref = (wt[:, :, None] * ys_ref).sum(1)
    y = down(client, out["y"])
    scale = float(y_ref.detach().abs().max())
    assert np.abs(y - y_ref.detach().numpy()).max() <= 2e-2 * scale
    # backward pieces against autograd
    dy = np.random.default_rng(3).standard_normal((T, N)).astype(np.float32)
    dy = synth.bf16_bits_to_f32(synth.f32_to_bf16_bits(dy))
    y_ref.backward(torch.tensor(dy))
    row_of = out["row_of"].to_numpy(client)
    d_ys, d_w = moe.combine_backward_alloc(client, up(client, dy, "bf16"), out["ys"], out["weights"], out["row_of"])
    dh = matmul.launch_grouped_alloc(client, d_ys, dev["w2"].transposed(), out["offs"])                # dgrad: d_ys @ W2_e^T
    dw2 = matmul.launch_grouped_alloc(client, out["h"].transposed(), d_ys, out["offs"], out_dtype="f32")  # wgrad: h^T @ d_ys
    client.sync()
    tol = lambda ref: 3e-2 * float(np.abs(ref).max())  # noqa: E731
    ysd = down(client, out["ys"])
    d_w_ref = np.einsum("tn,tkn->tk", dy, ysd[row_of])
    assert np.abs(d_w.to_numpy(client) - d_w_ref).max() <= 1e-3 * float(np.abs(d_w_ref).max())
    np.testing.assert_allclose(d_w.to_numpy(client), wt.grad.numpy(), atol=tol(wt.grad.numpy()))
    assert np.abs(dw2.to_numpy(client) - w2.grad.numpy()).max() <= tol(w2.grad.numpy())
    # dx: relu' from the device's h, the grouped dgrad through W1, then the permute's backward (combine without weights)
    hd = down(client, out["h"])
    dhd = down(client, dh) * (hd > 0)
    dxs = matmul.launch_grouped_alloc(client, up(client, dhd, "bf16"), dev["w1"].transposed(), out["offs"])
    dx = moe.combine_alloc(client, dxs, out["row_of"], None, out_dtype="f32")
    client.sync()
    assert np.abs(dx.to_numpy(client) - x.grad.numpy()).max() <= tol(x.grad.numpy())


def test_fp8_recipe_equals_quantize_after_permute(client):
    T, K, N, E, k = 640, 512, 256, 8, 2
    host, dev = layer_inputs(client, T, K, 128, N, E, 4)
    rng = np.random.default_rng(5)
    ids = rng.integers(0, E, (T, k)).astype(np.int32)
    offs, row_of, slot_of = moe.plan_alloc(client, up(client, ids, "i32"), E)
    s = QuantScheme().with_value("e4m3").per_block(128, "f32")
    qx = quant.quantize(client, dev["x"], s)
    codes = moe.permute_alloc(client, qx.values, slot_of, k)
    scales = moe.permute_alloc(client, qx.block_scales, slot_of, k)
    q_sorted = quant.quantize(client, moe.permute_alloc(client, dev["x"], slot_of, k), s)
    wq = quant.quantize(client, up(client, rng.standard_normal((E, N, K)).astype(np.float32), "bf16"), s)
    o1 = TensorHandle.empty_contiguous(client, [T * k, N], "bf16")
    o2 = TensorHandle.empty_contiguous(client, [T * k, N], "bf16")
    matmul.launch_grouped_quantized_fp8(client, QuantizedTensor(codes, scales, None, s, [T * k, K]), wq, offs, o1)
    matmul.launch_grouped_quantized_fp8(client, q_sorted, wq, offs, o2)
    client.sync()
    np.testing.assert_array_equal(codes.to_numpy(client), q_sorted.values.to_numpy(client))
    np.testing.assert_array_equal(scales.to_numpy(client), q_sorted.block_scales.to_numpy(client))
    np.testing.assert_array_equal(o1.to_numpy(client), o2.to_numpy(client))


LAYER_FIELDS = ("ids", "weights", "offs", "row_of", "slot_of", "xs", "h", "ys", "y")


def test_pipeline_repeats_bitwise(client):
    T, K, F, N, E, k = 4096, 1024, 1024, 1024, 64, 4
    _, dev = layer_inputs(client, T, K, F, N, E, 8)
    runs = [layer(client, dev["x"], dev["wr"], dev["w1"], dev["w2"], k) for _ in range(4)]
    client.sync()
    for r in runs[1:]:
        for name in LAYER_FIELDS:
            np.testing.assert_array_equal(r[name].to_numpy(client), runs[0][name].to_numpy(client), err_msg=name)


def test_layers_follow_inputs_rewritten_on_the_stream(client):
    """Two layers enqueued back to back, their input rewritten on the stream between them: each follows its own input, so
    every routing decision (ids, offs, row_of, slot_of) is read on the device when the kernels run."""
    T, K, F, N, E, k = 2048, 512, 512, 512, 32, 4
    _, dev = layer_inputs(client, T, K, F, N, E, 21)
    _, other = layer_inputs(client, T, K, F, N, E, 22)
    xin = TensorHandle.empty_contiguous(client, [T, K], "bf16")
    b1, b2 = layer_buffers(client, T, K, F, N, E, k), layer_buffers(client, T, K, F, N, E, k)
    lib, nbytes = client._lib, T * K * 2
    _ffi.check(lib.b200_copy(client._ctx, None, C.c_uint64(xin.handle.ptr), C.c_uint64(dev["x"].handle.ptr), nbytes))
    enqueue_layer(client, xin, dev["wr"], dev["w1"], dev["w2"], k, b1)
    _ffi.check(lib.b200_copy(client._ctx, None, C.c_uint64(xin.handle.ptr), C.c_uint64(other["x"].handle.ptr), nbytes))
    enqueue_layer(client, xin, dev["wr"], dev["w1"], dev["w2"], k, b2)
    client.sync()
    for got, x in ((b1, dev["x"]), (b2, other["x"])):
        want = layer(client, x, dev["wr"], dev["w1"], dev["w2"], k)
        client.sync()
        for name in LAYER_FIELDS:
            np.testing.assert_array_equal(got[name].to_numpy(client), want[name].to_numpy(client), err_msg=name)
    assert not np.array_equal(b1["offs"].to_numpy(client), b2["offs"].to_numpy(client))     # the two inputs route differently


def test_pipeline_enqueues_without_host_sync(client):
    """The stream is held behind a ~2 s spin kernel on a torch stream.  Three whole layers (outputs allocated up front, warmed up
    on the same stream so every pooled temporary is already there) must enqueue while it still waits: a host sync anywhere in
    them would block until the spin ends."""
    T, K, F, N, E, k = 4096, 1024, 1024, 1024, 64, 4
    _, dev = layer_inputs(client, T, K, F, N, E, 8)
    s = client.create_stream()
    bufs = [layer_buffers(client, T, K, F, N, E, k) for _ in range(3)]
    for b in bufs:
        enqueue_layer(client, dev["x"], dev["wr"], dev["w1"], dev["w2"], k, b, stream=s)
    client.sync_stream(s)
    hold = torch.cuda.Stream()
    with torch.cuda.stream(hold):
        torch.cuda._sleep(4_000_000_000)                 # ~2 s at 1.98 GHz, longer at lower clocks
    held = torch.cuda.Event()
    held.record(hold)
    client.stream_wait_event(s, C.c_void_p(held.cuda_event))
    t0 = time.perf_counter()
    for b in bufs:
        enqueue_layer(client, dev["x"], dev["wr"], dev["w1"], dev["w2"], k, b, stream=s)
    enqueue_ms = (time.perf_counter() - t0) * 1e3
    done = torch.cuda.Event()
    done.record(torch.cuda.ExternalStream(s.value))
    still_waiting = not done.query()
    client.sync_stream(s)
    torch.cuda.synchronize()
    client.destroy_stream(s)
    assert still_waiting, f"the layers had finished when their enqueue returned ({enqueue_ms:.1f} ms)"
    assert enqueue_ms < 500, enqueue_ms
