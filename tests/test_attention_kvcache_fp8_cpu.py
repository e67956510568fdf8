"""CPU: the fp8 KV-cache oracles (attention pinned to torch SDPA with causal_lower_right on the cache torch dequantizes; the
quantizing write pinned to torch's float8 casts, saturation and NaN included), and the dry-run plans of
b200_attention_kvcache_fp8 and b200_kvcache_write_fp8: kernel names, the esz=1 maps and their boxes, shared memory, splits
and the combine equal to the 16-bit plan's, gathers of q and of new tokens, every new refusal and the zero-extent no-ops, and
the attention_kv_fp8 cubin's kernels (no spills, no stack or local memory)."""
import ctypes as C
import math
import re
import subprocess

import numpy as np
import pytest
import torch

import attention_kvcache_fp8_oracle as fo
import attention_kvcache_oracle as ko
from cubecl_b200 import _ffi
from test_attention_kvcache_cpu import Planner, _launches, _paged, _tmaps
from test_conv_cpu import ROOT, _tool

F32, F16, BF16, I8, E4M3, E5M2 = _ffi.F32, _ffi.F16, _ffi.BF16, _ffi.I8, _ffi.F8E4M3, _ffi.F8E5M2
Q, KC, VC, BT, SL, OUT, KS, VS = 0x10000000, 0x20000000, 0x30000000, 0x40000000, 0x50000000, 0x60000000, 0x70000000, 0x71000000
INVALID, UNSUPPORTED = 6, 7
TORCH = {"f8e4m3": torch.float8_e4m3fn, "f8e5m2": torch.float8_e5m2}


# ---------------------------------------------------------------------------------------------- oracles
@pytest.mark.parametrize("fmt", fo.FORMATS)
def test_decode_matches_torch_on_every_code(fmt):
    codes = np.arange(256, dtype=np.uint8)
    ref = torch.from_numpy(codes).view(TORCH[fmt]).to(torch.float64).numpy()
    got = fo.decode(codes, fmt)
    assert np.array_equal(np.isnan(got), np.isnan(ref))
    assert np.array_equal(got[~np.isnan(got)], ref[~np.isnan(ref)])


@pytest.mark.parametrize("fmt", fo.FORMATS)
def test_quantize_matches_torch_casts(fmt):
    rng = np.random.default_rng(1)
    Hkv, D = 4, 64
    mx = fo.MAX[fmt]
    x = np.concatenate([rng.standard_normal((500, Hkv, D)) * 10.0 ** rng.uniform(-4, 5, (500, Hkv, 1)),
                        np.full((1, Hkv, D), np.nan), np.full((1, Hkv, D), np.inf), np.full((1, Hkv, D), -np.inf),
                        np.full((1, Hkv, D), 2 * mx), np.full((1, Hkv, D), -mx * 1.0001)]).astype(np.float32)
    # midpoints between neighbouring values (ties to even), and the values themselves
    vals = np.sort(fo.decode(np.arange(0x7F, dtype=np.uint8), fmt))
    vals = vals[np.isfinite(vals)]
    mids = ((vals[1:] + vals[:-1]) / 2).astype(np.float32)
    extra = np.resize(np.concatenate([mids, vals.astype(np.float32), -mids]), (4, Hkv, D))
    x = np.concatenate([x, extra])
    scale = np.array([1.0, 0.37, 2.0 ** -5, 3.3], dtype=np.float32)
    got = fo.quantize(x, scale, fmt)
    q = torch.from_numpy(x) / torch.from_numpy(scale)[:, None]
    ref = q.clamp(-mx, mx).to(TORCH[fmt]).view(torch.uint8).numpy()
    nan = np.isnan(q.numpy())
    assert np.array_equal(got[~nan], ref[~nan])
    assert np.all(np.isnan(fo.decode(got[nan], fmt))) and nan.any()
    assert np.all(np.abs(fo.decode(got, fmt)[~nan]) <= mx)


@pytest.mark.parametrize("fmt", fo.FORMATS)
@pytest.mark.parametrize("causal", [False, True])
def test_oracle_matches_torch_sdpa_on_the_dequantized_cache(fmt, causal):
    from torch.nn.attention.bias import causal_lower_right
    B, Hq, Hkv, Sq, D, cap = 3, 4, 2, 5, 32, 64
    rng = np.random.default_rng(5)
    q = rng.standard_normal((B, Hq, Sq, D))
    ks, vs = np.array([0.5, 3.0], np.float32), np.array([0.125, 1.7], np.float32)
    k8, v8 = (fo.quantize(rng.standard_normal((B * cap, Hkv, D)).astype(np.float32) * 4, s, fmt).reshape(B, cap, Hkv, D)
              for s in (np.ones(Hkv, np.float32),) * 2)
    lens = [37, 5, 64]
    k8p, table = _paged(k8.transpose(0, 2, 1, 3), 16, np.random.default_rng(2))
    v8p, _ = _paged(v8.transpose(0, 2, 1, 3), 16, np.random.default_rng(2))
    k8p, v8p = k8p.astype(np.uint8), v8p.astype(np.uint8)
    out, lse = fo.attention_kvcache_fp8_f64(q, k8p, v8p, ks, vs, fmt, lens, table, 0.3, causal)
    for b, L in enumerate(lens):
        kt, vt = (torch.from_numpy(np.ascontiguousarray(t[b, :L])).view(TORCH[fmt]).to(torch.float64) * torch.from_numpy(s).double()[:, None]
                  for t, s in ((k8, ks), (v8, vs)))
        kt, vt = (t.permute(1, 0, 2)[None].repeat_interleave(Hq // Hkv, dim=1) for t in (kt, vt))
        qt = torch.from_numpy(q[b:b + 1])
        mask = causal_lower_right(Sq, L) if causal else None
        ref = torch.nn.functional.scaled_dot_product_attention(qt, kt, vt, attn_mask=mask, scale=0.3)
        np.testing.assert_allclose(out[b:b + 1], ref.numpy(), rtol=0, atol=1e-12)
        s = 0.3 * torch.einsum("bhid,bhjd->bhij", qt, kt)
        if causal:
            s = s.masked_fill(~torch.ones(Sq, L, dtype=torch.bool).tril(L - Sq), -math.inf)
        np.testing.assert_allclose(lse[b], torch.logsumexp(s, dim=-1)[0].numpy(), rtol=1e-13, atol=1e-13)


def test_power_of_two_scales_equal_the_dequantized_16_bit_problem():
    """the contract the GPU tests build on, in f64: scaling the fp8 values by powers of two is the 16-bit oracle's input"""
    rng = np.random.default_rng(9)
    k8 = fo.quantize(rng.standard_normal((4, 16, 2, 16)).reshape(64, 2, 16).astype(np.float32), np.ones(2, np.float32), "f8e4m3")
    k8 = k8.reshape(4, 16, 2, 16)
    s = np.array([0.25, 8.0], np.float32)
    deq = fo.dequantize(k8, s, "f8e4m3")
    assert np.array_equal(deq.astype(np.float16).astype(np.float64), deq)   # exact in f16
    q = rng.standard_normal((4, 4, 1, 16))
    a = fo.attention_kvcache_fp8_f64(q, k8, k8, s, s, "f8e4m3", [16, 3, 0, 9])
    b = ko.attention_kvcache_f64(q, deq, deq, [16, 3, 0, 9])
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


# ---------------------------------------------------------------------------------------------- dry-run plans
class Planner8(Planner):
    def run8(self, qs, kcs, vcs=None, bts=None, outs=None, idt=BF16, cdt=E4M3, odt=None, strides=(None, None, None, None, None),
             ptrs=(Q, KC, VC, BT, SL, OUT), scales=(KS, VS), lse=0, scale=0.125, causal=0, null_args=False):
        vcs = kcs if vcs is None else vcs
        outs = qs if outs is None else outs
        odt = idt if odt is None else odt
        arr = lambda v: _ffi.u64_array(v) if v is not None else None  # noqa: E731
        args = _ffi.AttentionArgs(scale, causal)
        bt = ptrs[3] if bts is not None else 0
        rc = self.lib.b200_attention_kvcache_fp8(self.ctx, None, idt, cdt, odt, ptrs[0], arr(qs), arr(strides[0]), ptrs[1], arr(kcs),
                                                 arr(strides[1]), ptrs[2], arr(vcs), arr(strides[2]), bt, arr(bts), arr(strides[3]),
                                                 ptrs[4], scales[0], scales[1], ptrs[5], arr(outs), arr(strides[4]), lse,
                                                 None if null_args else C.byref(args))
        return rc, self.text()

    def write8(self, kns, kcs, dt=BF16, cdt=E4M3, strides=(None, None, None, None), ptrs=(Q, KC, VC, BT, SL), scales=(KS, VS)):
        arr = lambda v: _ffi.u64_array(v) if v is not None else None  # noqa: E731
        rc = self.lib.b200_kvcache_write_fp8(self.ctx, None, dt, cdt, ptrs[0], arr(kns), arr(strides[0]), ptrs[3], arr(kns),
                                             arr(strides[1]), ptrs[1], arr(kcs), arr(strides[2]), ptrs[2], arr(kcs), arr(strides[3]),
                                             ptrs[4], scales[0], scales[1])
        return rc, self.text()


@pytest.fixture
def plan():
    p = Planner8()
    yield p
    p.close()


def _smem8(bucket):
    return 1024 + bucket // 64 * (64 + 3 * 64) * 128 + 8 * 2 * 64 * 128 + 256


@pytest.mark.parametrize("idt,tag", [(BF16, "bf16"), (F16, "f16")])
@pytest.mark.parametrize("cdt,fmt", [(E4M3, "e4m3"), (E5M2, "e5m2")])
@pytest.mark.parametrize("D,bucket", [(16, 64), (48, 64), (64, 64), (80, 128), (112, 128), (128, 128)])
@pytest.mark.parametrize("out_f32", [False, True])
def test_kernel_per_dtype_format_bucket_and_out(plan, idt, tag, cdt, fmt, D, bucket, out_f32):
    rc, t = plan.run8([32, 32, 1, D], [32, 128, 8, D], idt=idt, cdt=cdt, odt=F32 if out_f32 else idt)
    assert rc == 0, _ffi.load().b200_last_error()
    (name, grid, block, smem), = _launches(t)
    assert name == f"attn_kv_{tag}_{fmt}_d{bucket}_{'f32' if out_f32 else tag}"
    assert (int(grid), int(block), int(smem)) == (32 * 8, 160, _smem8(bucket))
    assert _smem8(128) <= 227 * 1024
    assert "alloc" not in t and "gather" not in t


def test_maps_of_a_paged_fp8_cache(plan):
    B, Hq, Hkv, D, P, page, mp = 4, 32, 8, 128, 100, 16, 40
    rc, t = plan.run8([B, Hq, 1, D], [P, page, Hkv, D], bts=[B, mp])
    assert rc == 0, _ffi.load().b200_last_error()
    mq, mk, mv = _tmaps(t)
    assert mq == (2, (D, 1, Hq, B), (2 * D, 2 * D, 2 * D * Hq), (64, 1, 4, 1))   # q: the 16-bit map of b200_attention_kvcache
    assert mk == mv == (1, (D, page, Hkv, P), (Hkv * D, D, page * Hkv * D), (128, 16, 1, 1))


def test_maps_of_a_head_major_fp8_cache(plan):
    B, Hq, Hkv, Sq, D, P, page = 2, 8, 2, 3, 64, 10, 64
    hm = [Hkv * page * D, D, page * D, 1]
    rc, t = plan.run8([B, Hq, Sq, D], [P, page, Hkv, D], bts=[B, 5], strides=(None, hm, hm, None, None))
    assert rc == 0, _ffi.load().b200_last_error()
    assert "gather" not in t
    _, mk, mv = _tmaps(t)
    assert mk == mv == (1, (D, page, Hkv, P), (D, page * D, Hkv * page * D), (128, 64, 1, 1))


@pytest.mark.parametrize("page,rows", [(16, 16), (32, 32), (64, 64), (128, 64), (256, 64)])
def test_load_rows_per_page_size(plan, page, rows):
    rc, t = plan.run8([2, 8, 1, 128], [64, page, 2, 128], bts=[2, 4])
    assert rc == 0 and _tmaps(t)[1][3] == (128, rows, 1, 1) and _tmaps(t)[2][3] == (128, rows, 1, 1)


@pytest.mark.parametrize("sms", [132, 8])
def test_splits_and_combine_equal_the_16_bit_plan(sms):
    p = Planner8(sms)
    try:
        seen = set()
        for B in (1, 8, 128):
            for Hq, Hkv in ((32, 8), (32, 32)):
                for Sq in (1, 4):
                    for cap in (64, 2048, 65536):
                        rc, t16 = p.run([B, Hq, Sq, 128], [B, cap, Hkv, 128])
                        assert rc == 0
                        rc, t8 = p.run8([B, Hq, Sq, 128], [B, cap, Hkv, 128], odt=F32)
                        assert rc == 0, _ffi.load().b200_last_error()
                        l16, l8 = _launches(t16), _launches(t8)
                        assert [g for _, g, _, _ in l8] == [g for _, g, _, _ in l16]
                        assert re.findall(r"alloc (\d+)", t8) == re.findall(r"alloc (\d+)", t16)
                        if len(l8) == 2:
                            assert l8[1][0] == "attn_kv_combine_fp8_f32"
                        gt, st = ko.kv_tile(Hq // Hkv, Sq)
                        units = B * Hkv * -(-(Hq // Hkv) // gt) * -(-Sq // st)
                        assert int(l8[0][1]) == units * ko.kv_splits(units, -(-cap // 64), sms)
                        seen.add(len(l8))
        assert seen == ({1, 2} if sms == 132 else {1})   # 8 SMs: every shape here has >= 8 CTAs per split
    finally:
        p.close()


def test_misaligned_query_is_gathered(plan):
    rc, t = plan.run8([64, 4, 1, 64], [64, 128, 2, 64], ptrs=(Q + 2, KC, VC, BT, SL, OUT))
    assert rc == 0
    assert [x[0] for x in _launches(t)] == ["gather_strided", "attn_kv_bf16_e4m3_d64_bf16"]
    assert _tmaps(t)[0][2] == (2 * 64, 2 * 64, 2 * 64 * 4)


def test_16_bit_plans_keep_their_maps(plan):
    """the fp8 map rule (UINT8, 128-byte box) leaves the 16-bit cache maps as they were"""
    rc, t = plan.run([2, 8, 1, 128], [64, 16, 2, 128], bts=[2, 4])
    assert rc == 0 and _tmaps(t)[1] == (2, (128, 16, 2, 64), (512, 256, 8192), (64, 16, 1, 1))


# ---------------------------------------------------------------------------------------------- refusals
@pytest.mark.parametrize("case,status,words", [
    ("cache_bf16", UNSUPPORTED, "cache dtype"), ("cache_i8", UNSUPPORTED, "cache dtype"), ("cache_f32", UNSUPPORTED, "cache dtype"),
    ("null_k_scale", INVALID, "k_scale"), ("null_v_scale", INVALID, "v_scale"), ("k_scale_align", INVALID, "aligned"),
    ("v_scale_align", INVALID, "aligned"), ("compact_d8", UNSUPPORTED, "cache"), ("compact_d40", UNSUPPORTED, "cache"),
    ("cache_misaligned", UNSUPPORTED, "cache"), ("in_f32", UNSUPPORTED, "input dtype"), ("in_fp8", UNSUPPORTED, "input dtype"),
    ("out_other", UNSUPPORTED, "output dtype"), ("d136", UNSUPPORTED, "head dim"), ("gqa", INVALID, "multiple of Hkv"),
    ("null_seqlens", INVALID, "null"), ("page24", UNSUPPORTED, "multiple of 16"),
])
def test_refusals(plan, case, status, words):
    qs, kcs, bts = [2, 4, 1, 64], [8, 16, 2, 64], [2, 4]
    kw, ptrs, scales = {}, [Q, KC, VC, BT, SL, OUT], [KS, VS]
    if case == "cache_bf16":
        kw["cdt"] = BF16
    elif case == "cache_i8":
        kw["cdt"] = I8
    elif case == "cache_f32":
        kw["cdt"] = F32
    elif case == "null_k_scale":
        scales[0] = 0
    elif case == "null_v_scale":
        scales[1] = 0
    elif case == "k_scale_align":
        scales[0] = KS + 2
    elif case == "v_scale_align":
        scales[1] = VS + 1
    elif case == "compact_d8":            # a compact fp8 row of 8 bytes is not a 16-byte multiple
        qs, kcs = [2, 4, 1, 8], [8, 16, 2, 8]
    elif case == "compact_d40":
        qs, kcs = [2, 4, 1, 40], [8, 16, 2, 40]
    elif case == "cache_misaligned":
        ptrs[2] = VC + 8
    elif case == "in_f32":
        kw["idt"], kw["odt"] = F32, F32
    elif case == "in_fp8":
        kw["idt"], kw["odt"] = E4M3, F32
    elif case == "out_other":
        kw["idt"], kw["odt"] = BF16, F16
    elif case == "d136":
        qs, kcs = [2, 4, 1, 136], [8, 16, 2, 136]
    elif case == "gqa":
        kcs = [8, 16, 3, 64]
    elif case == "null_seqlens":
        ptrs[4] = 0
    elif case == "page24":
        kcs = [8, 24, 2, 64]
    rc, t = plan.run8(qs, kcs, bts=bts, ptrs=tuple(ptrs), scales=tuple(scales), **kw)
    msg = _ffi.load().b200_last_error().decode()
    assert rc == status, (case, rc, msg)
    assert words in msg and msg.startswith("attention_kvcache_fp8"), msg
    assert _launches(t) == [] and "gather" not in t


def test_padded_fp8_cache_rows_are_read_in_place(plan):
    """D = 40 with rows padded to 48 bytes: the maps read the view"""
    st = [16 * 2 * 48, 2 * 48, 48, 1]
    rc, t = plan.run8([2, 4, 1, 40], [8, 16, 2, 40], bts=[2, 4], strides=(None, st, st, None, None))
    assert rc == 0, _ffi.load().b200_last_error()
    assert _tmaps(t)[1] == (1, (40, 16, 2, 8), (96, 48, 1536), (128, 16, 1, 1))


def test_zero_extents_plan_no_launch(plan):
    for qs in ([0, 4, 1, 64], [2, 0, 1, 64], [2, 4, 0, 64]):
        rc, t = plan.run8(qs, [8, 16, 2, 64], bts=[qs[0], 4], scales=(0, 0))
        assert rc == 0 and t == "", (qs, t)
    rc, t = plan.write8([0, 3, 2, 64], [10, 16, 2, 64], scales=(0, 0))
    assert rc == 0 and t == ""


# ---------------------------------------------------------------------------------------------- kvcache_write_fp8
@pytest.mark.parametrize("dt", [BF16, F16])
@pytest.mark.parametrize("cdt", [E4M3, E5M2])
def test_write_plan_and_gathered_views(plan, dt, cdt):
    rc, t = plan.write8([2, 3, 4, 128], [10, 16, 4, 128], dt=dt, cdt=cdt)
    assert rc == 0, _ffi.load().b200_last_error()
    assert _launches(t) == [("attn_kv_write_fp8", str(-(-2 * 3 * 4 * 16 // 256)), "256", "0")]
    rc, t = plan.write8([2, 3, 4, 128], [10, 16, 4, 128], ptrs=(Q + 2, KC, VC, BT, SL))
    assert rc == 0 and [x[0] for x in _launches(t)] == ["gather_strided", "attn_kv_write_fp8"]
    st = [3 * 4 * 136, 4 * 136, 136, 1]
    rc, t = plan.write8([2, 3, 4, 128], [10, 16, 4, 128], strides=(st, st, None, None))
    assert rc == 0 and "gather" not in t


@pytest.mark.parametrize("case,status,words", [
    ("cache_bf16", UNSUPPORTED, "cache dtype"), ("in_f32", UNSUPPORTED, "dtype"), ("null_k_scale", INVALID, "k_scale"),
    ("v_scale_align", INVALID, "aligned"), ("compact_d8", UNSUPPORTED, "cache"), ("heads", INVALID, "heads or head dim"),
    ("null", INVALID, "null"),
])
def test_write_refusals(plan, case, status, words):
    kns, kcs = [2, 3, 4, 64], [10, 16, 4, 64]
    kw, ptrs, scales = {}, [Q, KC, VC, BT, SL], [KS, VS]
    if case == "cache_bf16":
        kw["cdt"] = BF16
    elif case == "in_f32":
        kw["dt"] = F32
    elif case == "null_k_scale":
        scales[0] = 0
    elif case == "v_scale_align":
        scales[1] = VS + 2
    elif case == "compact_d8":
        kns, kcs = [2, 3, 4, 8], [10, 16, 4, 8]
    elif case == "heads":
        kcs = [10, 16, 2, 64]
    elif case == "null":
        ptrs[4] = 0
    rc, t = plan.write8(kns, kcs, ptrs=tuple(ptrs), scales=tuple(scales), **kw)
    msg = _ffi.load().b200_last_error().decode()
    assert rc == status, (case, rc, msg)
    assert words in msg and msg.startswith("kvcache_write_fp8") and _launches(t) == []


def test_python_entry_points_defer_errors():
    from cubecl_b200 import attention

    class _Stub:
        def __init__(self):
            self.errors = []

        def _defer(self, e):
            self.errors.append(e)

    class _T:
        def __init__(self, shape, dtype="bf16"):
            self.shape, self.dtype = shape, dtype

        def is_contiguous(self):
            return True

    stub = _Stub()
    kc8, sc = _T([8, 16, 2, 64], "f8e4m3"), _T([2], "f32")
    attention.launch_kvcache_fp8(stub, _T([2, 4, 1]), kc8, kc8, _T([2], "i32"), sc, sc, _T([2, 4, 1, 64]))
    attention.launch_kvcache_fp8(stub, _T([2, 4, 1, 64]), kc8, _T([8, 16, 2, 64], "f8e5m2"), _T([2], "i32"), sc, sc, _T([2, 4, 1, 64]))
    attention.launch_kvcache_fp8(stub, _T([2, 4, 1, 64]), kc8, kc8, _T([2], "i32"), _T([3], "f32"), sc, _T([2, 4, 1, 64]))
    attention.kvcache_write_fp8(stub, _T([2, 1, 2, 64]), _T([2, 1, 2, 64]), _T([8, 16, 2, 64]), _T([8, 16, 2, 64]), _T([2], "i32"), sc, sc)
    assert [e.status for e in stub.errors] == [INVALID, UNSUPPORTED, INVALID, UNSUPPORTED]
    assert "rank 4" in str(stub.errors[0]) and "dtypes differ" in str(stub.errors[1])
    assert "k_scale" in str(stub.errors[2]) and "cache dtype" in str(stub.errors[3])


# ---------------------------------------------------------------------------------------------- kernels
def test_fp8_kernels_widen_on_chip_and_do_not_spill():
    tool = _tool("cuobjdump")
    _ffi.load()
    cubin = ROOT / "cubecl_b200" / "build" / "attention_kv_fp8.cubin"
    out = subprocess.run([tool, "-res-usage", str(cubin)], capture_output=True, text=True, check=True).stdout
    funcs = re.findall(r"Function (\w+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)
    want = {f"attn_kv_{i}_{f}_d{d}_{o}" for i in ("bf16", "f16") for f in ("e4m3", "e5m2") for d in (64, 128) for o in (i, "f32")}
    want |= {f"attn_kv_combine_fp8_{o}" for o in ("bf16", "f16", "f32")} | {"attn_kv_write_fp8"}
    assert {f for f, *_ in funcs} == want
    for name, reg, stack, local in funcs:
        assert int(stack) == 0 and int(local) == 0, (name, stack, local)
    sass = subprocess.run([tool, "-sass", str(cubin)], capture_output=True, text=True, check=True).stdout
    for body in re.split(r"\n\s*Function : ", sass)[1:]:
        name = body.split()[0]
        if "combine" in name or "write" in name:
            continue
        n = 64 if "_d64_" in name else 128
        assert re.search(rf"HGMMA\.64x{n}x16\.F32\S* R\d+, R\d+, gdesc\[UR\d+\]\.tnspB", body), name
        assert re.search(r"HGMMA\.64x64x16\.F32\S* R\d+, gdesc\[UR\d+\]", body), name
        assert "UTMALDG.4D" in body and "F2FP" in body, name
