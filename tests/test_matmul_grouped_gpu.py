"""GPU: b200_matmul_grouped against its exact contract and against b200_matmul.

- Integer-valued operands with sum |a||b| < 2^24 give rne(f64 result) bit for bit, in both modes, on both tiles, both store
  paths, both out dtypes and all four ragged-M layouts, with group sizes at every tile edge, one group of all rows and 256
  small groups.  Rows past the last group keep their sentinels; in ragged K, NaN and inf in a neighbouring group's rows and
  past the last group change no other group's bits, and empty groups are +0.
- On random data each group's result equals b200_matmul on that group's slices bit for bit (same tile, no stream-K), and
  balanced groups equal the batched b200_matmul on the same bytes.
- A dyadic epilogue is exact; offsets rewritten on the stream between two calls are followed by each call; a malformed table is
  clamped; repeats are bitwise equal; torch's GPU grouped_mm agrees within bf16 rounding.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import gemm_exact_oracle as ge
import grouped_mm_oracle as gmo
from cubecl_b200 import TensorHandle, _ffi, matmul, synth

pytestmark = pytest.mark.gpu

SENT = {"bf16": 0x7FA1, "f16": 0x7E01, "f32": 0x7FC0_1234}
EDGES = [0, 1, 63, 64, 65, 127, 128, 129, 255, 256, 257, 0]
SIZES = {"edges": (EDGES, 40), "one_group": ([0, 700, 0], 0), "many_small": (list(np.random.default_rng(3).integers(0, 7, 256)), 9)}
OPTIONS = {"gemm.variant": "auto", "gemm.epilogue": "tma", "gemm.split_k": "auto"}


@pytest.fixture(autouse=True)
def _reset_options(client):
    yield
    for k, v in OPTIONS.items():
        client.set_option(k, v)


def up(client, vals, dtype):
    if dtype == "i32":
        return TensorHandle.from_numpy(client, np.ascontiguousarray(vals, np.int32), "i32")
    return TensorHandle.from_numpy(client, synth.to_device_dtype(np.ascontiguousarray(vals, np.float32), dtype), dtype)


def bits(client, t):
    return np.asarray(t.to_numpy(client)).view(np.uint32 if t.dtype == "f32" else np.uint16).reshape(t.shape)


def sentinel(client, shape, dtype):
    return TensorHandle.from_numpy(client, np.full(shape, SENT[dtype], np.uint32 if dtype == "f32" else np.uint16), dtype)


def lhs_m(client, a, dtype, layout):
    """[T, K]: compact (k), or the transposed view of a compact [K, T] (m)"""
    return up(client, a, dtype) if layout[0] == "k" else up(client, a.T, dtype).transposed()


def rhs_m(client, b, dtype, layout):
    """[G, K, N]: compact (n), or the transposed view of compact [G, N, K] weights (k)"""
    return up(client, b, dtype) if layout[1] == "n" else up(client, b.transpose(0, 2, 1), dtype).transposed()


def run_m(client, a, b, offs, dtype="bf16", odt="bf16", layout="kn", **kw):
    T, N = a.shape[0], b.shape[2]
    out = sentinel(client, [T, N], odt)
    matmul.launch_grouped(client, lhs_m(client, a, dtype, layout), rhs_m(client, b, dtype, layout), up(client, offs, "i32"), out, **kw)
    client.sync()
    return out


def run_k(client, x, dy, offs, dtype="bf16", odt="bf16"):
    """lhs = x.t() (the [M, T] view of x [T, M]), rhs = dy [T, N]"""
    out = sentinel(client, [len(offs), x.shape[1], dy.shape[1]], odt)
    matmul.launch_grouped(client, up(client, x, dtype).transposed(), up(client, dy, dtype), up(client, offs, "i32"), out)
    client.sync()
    return out


def ints(rng, shape, bound=16):
    return rng.integers(-bound, bound + 1, shape).astype(np.float64)


# ---------------------------------------------------------------------------------------------- exact contract
@pytest.mark.parametrize("sizes", sorted(SIZES))
@pytest.mark.parametrize("tile", ["2sm_n128", "1sm_n128"])
@pytest.mark.parametrize("store", ["tma", "direct"])
@pytest.mark.parametrize("odt", ["bf16", "f32"])
@pytest.mark.parametrize("layout", ["kn", "kk", "mn", "mk"])
def test_ragged_m_is_exact(client, sizes, tile, store, odt, layout):
    client.set_option("gemm.variant", tile)
    client.set_option("gemm.epilogue", store)
    sz, extra = SIZES[sizes]
    offs = gmo.offsets(sz)
    T, K, N, G = int(sum(sz)) + extra, 200, 200, len(sz)
    rng = np.random.default_rng(hash((sizes, layout)) % 1000)
    a, b = ints(rng, (T, K)), ints(rng, (G, K, N))
    want, written = gmo.ragged_m(a, b, offs)
    ge.assert_exact_bound(gmo.ragged_m(np.abs(a), np.abs(b), offs)[0][written])
    got = bits(client, run_m(client, a, b, offs, odt=odt, layout=layout))
    assert client.last_kernel() == f"gemm_grouped_m_bf16_{odt}_{tile}_{layout}"
    ge.assert_exact(got[written], want[written], odt, f"{sizes} {tile} {store} {layout}")
    assert (got[~written] == SENT[odt]).all(), "a row past the last group was written"


@pytest.mark.parametrize("dtype,odt", [("f16", "f16"), ("f16", "f32")])
def test_ragged_m_f16_inputs_are_exact(client, dtype, odt):
    sz = EDGES
    offs = gmo.offsets(sz)
    rng = np.random.default_rng(8)
    a, b = ints(rng, (sum(sz) + 5, 136)), ints(rng, (len(sz), 136, 72))
    want, written = gmo.ragged_m(a, b, offs)
    got = bits(client, run_m(client, a, b, offs, dtype, odt))
    ge.assert_exact(got[written], want[written], odt, dtype)
    assert (got[~written] == SENT[odt]).all()


@pytest.mark.parametrize("sizes", sorted(SIZES))
@pytest.mark.parametrize("tile", ["2sm_n128", "1sm_n128"])
@pytest.mark.parametrize("store", ["tma", "direct"])
@pytest.mark.parametrize("dtype,odt", [("bf16", "bf16"), ("bf16", "f32"), ("f16", "f16")])
def test_ragged_k_is_exact(client, sizes, tile, store, dtype, odt):
    client.set_option("gemm.variant", tile)
    client.set_option("gemm.epilogue", store)
    sz, extra = SIZES[sizes]
    offs = gmo.offsets(sz)
    T, M, N = int(sum(sz)) + extra, 200, 136
    rng = np.random.default_rng(len(sz) + M)
    x, dy = ints(rng, (T, M)), ints(rng, (T, N))
    want = gmo.ragged_k(x.T, dy, offs)
    ge.assert_exact_bound(gmo.ragged_k(np.abs(x).T, np.abs(dy), offs))
    got = bits(client, run_k(client, x, dy, offs, dtype, odt))
    assert client.last_kernel() == f"gemm_grouped_k_{dtype}_{odt}_{tile}"
    ge.assert_exact(got, want, odt, f"{sizes} {tile} {store}")
    empty = np.asarray(sz) == 0
    assert (got[empty] == 0).all(), "an empty group is not +0"


@pytest.mark.parametrize("tile", ["2sm_n128", "1sm_n128"])
def test_ragged_k_nan_and_inf_in_neighbouring_rows_change_no_other_bit(client, tile):
    """group 3's positions and the positions past the last group hold NaN and inf: every other group stays exact (its last
    k-block reads those rows and must clear them), and empty groups are +0"""
    client.set_option("gemm.variant", tile)
    sz = [65, 0, 127, 70, 1, 0, 200]
    offs = gmo.offsets(sz)
    T, M, N = sum(sz) + 30, 136, 200
    rng = np.random.default_rng(11)
    x, dy = ints(rng, (T, M)), ints(rng, (T, N))
    lo, hi = int(offs[2]), int(offs[3])
    x[lo:hi:2] = np.nan
    dy[lo + 1:hi:2] = np.inf
    x[offs[-1]:] = np.inf
    dy[offs[-1]:] = np.nan
    got = bits(client, run_k(client, x, dy, offs, odt="f32"))
    xs, dys = np.nan_to_num(x, nan=0, posinf=0), np.nan_to_num(dy, nan=0, posinf=0)
    want = gmo.ragged_k(xs.T, dys, offs)
    keep = [g for g in range(len(sz)) if g != 3]
    ge.assert_exact(got[keep], want[keep], "f32", "neighbours of NaN / inf rows")
    assert (got[[1, 5]] == 0).all()


# ---------------------------------------------------------------------------------------------- identity with b200_matmul
def _view(t, start_elems, shape, strides):
    return TensorHandle(t.handle.offset(start_elems * 2), shape, strides, t.dtype)


@pytest.mark.parametrize("tile", ["2sm_n128", "1sm_n128"])
@pytest.mark.parametrize("dtype", ["bf16", "f16"])
@pytest.mark.parametrize("layout", ["kn", "kk", "mn", "mk"])
def test_each_group_equals_b200_matmul_on_its_slices(client, tile, dtype, layout):
    client.set_option("gemm.variant", tile)
    client.set_option("gemm.split_k", "off")
    # an M-contiguous lhs slice is read in place (not staged) by b200_matmul when its first row is 16-byte aligned
    sz = [0, 1, 63, 64, 65, 127, 128, 129, 255, 256, 257, 300] if layout[0] == "k" else [0, 8, 64, 72, 128, 136, 256, 264, 512]
    offs = gmo.offsets(sz)
    T, K, N, G = sum(sz), 320, 256, len(sz)
    rng = np.random.default_rng(21)
    a, b = rng.uniform(-1, 1, (T, K)), rng.uniform(-1, 1, (G, K, N))
    lhs, rhs = lhs_m(client, a, dtype, layout), rhs_m(client, b, dtype, layout)
    out = sentinel(client, [T, N], dtype)
    matmul.launch_grouped(client, lhs, rhs, up(client, offs, "i32"), out)
    client.sync()
    got = bits(client, out)
    for g, (lo, hi) in enumerate(gmo.bounds(offs, T)):
        if hi == lo:
            continue
        sl = _view(lhs, lo * lhs.strides[0], [hi - lo, K], lhs.strides)
        wg = _view(rhs, g * rhs.strides[0], [K, N], rhs.strides[1:])
        ref = TensorHandle.empty_contiguous(client, [hi - lo, N], dtype)
        matmul.launch(client, sl, wg, ref)
        client.sync()
        np.testing.assert_array_equal(got[lo:hi], bits(client, ref), err_msg=f"group {g}")


@pytest.mark.parametrize("tile", ["2sm_n128", "1sm_n128"])
def test_each_ragged_k_group_equals_b200_matmul_on_its_slices(client, tile):
    client.set_option("gemm.variant", tile)
    client.set_option("gemm.split_k", "off")
    sz = [1, 63, 64, 65, 0, 200, 512]
    offs = gmo.offsets(sz)
    T, M, N = sum(sz), 256, 192
    rng = np.random.default_rng(22)
    x, dy = rng.uniform(-1, 1, (T, M)), rng.uniform(-1, 1, (T, N))
    xt, dyt = up(client, x, "bf16"), up(client, dy, "bf16")
    out = TensorHandle.empty_contiguous(client, [len(sz), M, N], "f32")
    matmul.launch_grouped(client, xt.transposed(), dyt, up(client, offs, "i32"), out)
    client.sync()
    got = bits(client, out)
    for g, (lo, hi) in enumerate(gmo.bounds(offs, T)):
        if hi == lo:
            continue
        ref = TensorHandle.empty_contiguous(client, [M, N], "f32")
        matmul.launch(client, _view(xt, lo * M, [M, hi - lo], [1, M]), _view(dyt, lo * N, [hi - lo, N], [N, 1]), ref)
        client.sync()
        np.testing.assert_array_equal(got[g], bits(client, ref), err_msg=f"group {g}")


@pytest.mark.parametrize("tile", ["2sm_n128", "1sm_n128"])
def test_balanced_groups_equal_the_batched_matmul(client, tile):
    client.set_option("gemm.variant", tile)
    client.set_option("gemm.split_k", "off")
    G, Mg, K, N = 6, 512, 384, 256
    rng = np.random.default_rng(23)
    a, b = rng.uniform(-1, 1, (G * Mg, K)), rng.uniform(-1, 1, (G, K, N))
    lhs, rhs = up(client, a, "bf16"), up(client, b, "bf16")
    out = TensorHandle.empty_contiguous(client, [G * Mg, N], "bf16")
    matmul.launch_grouped(client, lhs, rhs, up(client, gmo.offsets([Mg] * G), "i32"), out)
    ref = TensorHandle.empty_contiguous(client, [G, Mg, N], "bf16")
    matmul.launch(client, TensorHandle(lhs.handle, [G, Mg, K], [Mg * K, K, 1], "bf16"), rhs, ref)
    client.sync()
    np.testing.assert_array_equal(bits(client, out).reshape(G, Mg, N), bits(client, ref))
    # ragged K with groups of whole k-blocks: the batched product of the [G, M, n] and [G, n, N] views
    n, M = 320, 256
    x, dy = rng.uniform(-1, 1, (G * n, M)), rng.uniform(-1, 1, (G * n, N))
    xt, dyt = up(client, x, "bf16"), up(client, dy, "bf16")
    out = TensorHandle.empty_contiguous(client, [G, M, N], "f32")
    matmul.launch_grouped(client, xt.transposed(), dyt, up(client, gmo.offsets([n] * G), "i32"), out)
    ref = TensorHandle.empty_contiguous(client, [G, M, N], "f32")
    matmul.launch(client, TensorHandle(xt.handle, [G, M, n], [n * M, 1, M], "bf16"), TensorHandle(dyt.handle, [G, n, N], [n * N, N, 1], "bf16"), ref)
    client.sync()
    np.testing.assert_array_equal(bits(client, out), bits(client, ref))


# ---------------------------------------------------------------------------------------------- epilogue, offsets, repeats
@pytest.mark.parametrize("tile", ["2sm_n128", "1sm_n128"])
@pytest.mark.parametrize("odt", ["bf16", "f32"])
def test_dyadic_epilogue_is_exact(client, tile, odt):
    client.set_option("gemm.variant", tile)
    sz = [100, 0, 300, 257, 1]
    offs = gmo.offsets(sz)
    T, K, N, G = sum(sz) + 20, 192, 160, len(sz)
    rng = np.random.default_rng(31)
    a, b = ints(rng, (T, K)), ints(rng, (G, K, N))
    bias = rng.integers(-400, 400, (G, N)) / 4.0
    want, written = gmo.ragged_m(a, b, offs, bias=bias, alpha=0.5, activation="relu")
    out = run_m(client, a, b, offs, odt=odt, bias=up(client, bias, "f32"), alpha=0.5, activation="relu")
    got = bits(client, out)
    ge.assert_exact(got[written], want[written], odt, "epilogue")
    assert (got[~written] == SENT[odt]).all()


def test_offsets_rewritten_on_the_stream_are_followed(client):
    """two calls enqueued back to back, the offsets rewritten on the stream between them (no host sync): each result follows
    its own offsets"""
    rng = np.random.default_rng(41)
    T, K, N, G = 1500, 128, 128, 5
    a, b = ints(rng, (T, K), 8), ints(rng, (G, K, N), 8)
    first, second = gmo.offsets([300, 0, 500, 200, 100]), gmo.offsets([10, 700, 1, 300, 489])
    src1, src2, offs = up(client, first, "i32"), up(client, second, "i32"), up(client, np.zeros(G), "i32")
    lhs, rhs = up(client, a, "bf16"), up(client, b, "bf16")
    o1, o2 = sentinel(client, [T, N], "f32"), sentinel(client, [T, N], "f32")
    lib = client._lib
    _ffi.check(lib.b200_copy(client._ctx, None, C.c_uint64(offs.handle.ptr), C.c_uint64(src1.handle.ptr), 4 * G))
    matmul.launch_grouped(client, lhs, rhs, offs, o1)
    _ffi.check(lib.b200_copy(client._ctx, None, C.c_uint64(offs.handle.ptr), C.c_uint64(src2.handle.ptr), 4 * G))
    matmul.launch_grouped(client, lhs, rhs, offs, o2)
    client.sync()
    for o, table in ((o1, first), (o2, second)):
        want, written = gmo.ragged_m(a, b, table)
        got = bits(client, o)
        ge.assert_exact(got[written], want[written], "f32", "rewritten offsets")
        assert (got[~written] == SENT["f32"]).all()


@pytest.mark.parametrize("table", [[50, 30, 400, 10000, -5], [100, 90, 80], [-7, -1, 2000, 3]])
def test_malformed_offsets_are_clamped(client, table):
    rng = np.random.default_rng(42)
    T, K, N, G = 600, 96, 136, len(table)
    a, b = ints(rng, (T, K), 8), ints(rng, (G, K, N), 8)
    offs = np.asarray(table, np.int32)
    want, written = gmo.ragged_m(a, b, offs)
    got = bits(client, run_m(client, a, b, offs, odt="f32"))
    ge.assert_exact(got[written], want[written], "f32", "clamped")
    assert (got[~written] == SENT["f32"]).all()
    x, dy = ints(rng, (T, 72), 8), ints(rng, (T, 64), 8)
    got_k = bits(client, run_k(client, x, dy, offs, odt="f32"))
    ge.assert_exact(got_k, gmo.ragged_k(x.T, dy, offs), "f32", "clamped ragged K")


def test_repeats_give_the_same_bits(client):
    rng = np.random.default_rng(51)
    sz = list(rng.integers(0, 700, 64))
    offs = gmo.offsets(sz)
    T, K, N = sum(sz), 512, 384
    a, b = rng.uniform(-1, 1, (T, K)), rng.uniform(-1, 1, (64, K, N))
    r1, r2 = (bits(client, run_m(client, a, b, offs)) for _ in range(2))
    np.testing.assert_array_equal(r1, r2)
    x, dy = rng.uniform(-1, 1, (T, 256)), rng.uniform(-1, 1, (T, 192))
    k1, k2 = (bits(client, run_k(client, x, dy, offs, odt="f32")) for _ in range(2))
    np.testing.assert_array_equal(k1, k2)


def test_agrees_with_torch_grouped_mm(client):
    rng = np.random.default_rng(61)
    sz = [128, 0, 256, 64, 512, 16]
    offs = gmo.offsets(sz)
    T, K, N = sum(sz), 256, 256
    a, b = rng.uniform(-1, 1, (T, K)), rng.uniform(-1, 1, (len(sz), K, N))
    ta = torch.tensor(a, dtype=torch.bfloat16, device="cuda")
    tb = torch.tensor(b, dtype=torch.bfloat16, device="cuda")
    to = torch.tensor(offs, device="cuda")
    want = torch.nn.functional.grouped_mm(ta, tb, offs=to).float().cpu().numpy()
    got = synth.from_device_dtype(run_m(client, ta.float().cpu().numpy(), tb.float().cpu().numpy(), offs).to_numpy(client), "bf16")
    got = got.reshape(T, N)
    scale = gmo.ragged_m(np.abs(ta.float().cpu().numpy()), np.abs(tb.float().cpu().numpy()), offs)[0]
    assert np.max(np.abs(got - want) / scale) <= 2.0 ** -7
    x, dy = rng.uniform(-1, 1, (T, 128)), rng.uniform(-1, 1, (T, 192))
    tx = torch.tensor(x, dtype=torch.bfloat16, device="cuda")
    tdy = torch.tensor(dy, dtype=torch.bfloat16, device="cuda")
    want_k = torch.nn.functional.grouped_mm(tx.t(), tdy, offs=to).float().cpu().numpy()
    got_k = synth.from_device_dtype(run_k(client, tx.float().cpu().numpy(), tdy.float().cpu().numpy(), offs).to_numpy(client), "bf16")
    got_k = got_k.reshape(want_k.shape)
    scale_k = np.maximum(gmo.ragged_k(np.abs(tx.float().cpu().numpy()).T, np.abs(tdy.float().cpu().numpy()), offs), 1e-30)
    assert np.max(np.abs(got_k - want_k) / scale_k) <= 2.0 ** -7
    torch.cuda.synchronize()
