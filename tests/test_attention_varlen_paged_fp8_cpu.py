"""CPU: paged variable-length attention against fp8 caches (b200_attention_varlen_paged_fp8).

- The f64 oracle (the fp8 dequantization, then the paged varlen oracle) is pinned to torch's SDPA on torch's dequantized
  float8 cache; with power-of-two scales it equals the 16-bit problem on the dequantized cache rounded to q's dtype.
- Dry-run plans: kernel names per q dtype, format, bucket and out dtype, grids and shared memory; the map order, dims, esz=1
  and boxes for every page size and one page per sequence; a head-major fp8 cache is read in place and a misaligned q is
  gathered; every refusal of b200_attention_varlen_paged and the fp8 ones; zero extents.
- The Python entry points defer errors to sync(); the attention_paged_fp8 kernels use register-A wgmma and TMA and do not spill."""
import ctypes as C
import re
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from torch.nn.attention.bias import causal_lower_right

import attention_kvcache_fp8_oracle as fo
from cubecl_b200 import _ffi, synth
from test_attention_varlen_paged_cpu import (BT, CUQ, KC, LSE, OUT, Q, SEQ, VC, Planner, _launches, _only_alloc_tmap_launch,
                                             _tmaps, attention_varlen_paged_f64)
from test_conv_cpu import ROOT, _tool

F32, F16, BF16, E4M3, E5M2 = _ffi.F32, _ffi.F16, _ffi.BF16, _ffi.F8E4M3, _ffi.F8E5M2
KS, VS = 0x90000000, 0xA0000000
INVALID, UNSUPPORTED = 6, 7
TORCH_F8 = {"f8e4m3": torch.float8_e4m3fn, "f8e5m2": torch.float8_e5m2}


# ---------------------------------------------------------------------------------------------- oracle
def attention_varlen_paged_fp8_f64(q, k8, v8, k_scale, v_scale, fmt, table, seqlens, cu_q, max_k, scale=None, window=(-1, -1)):
    """-> (out [Tq, Hq, D], lse [Hq, Tq]) in float64: the paged varlen oracle on the dequantized cache"""
    return attention_varlen_paged_f64(q, fo.dequantize(k8, k_scale, fmt), fo.dequantize(v8, v_scale, fmt), table, seqlens, cu_q,
                                      max_k, scale, window)


def _problem(rng, lens_q, lens_k, Hq, Hkv, D, page, fmt, stale):
    """fp8 codes of normal keys in shuffled pages plus two unowned pages; other slots hold the stale bytes"""
    B = len(lens_q)
    mp = -(-max(lens_k) // page) + 1
    P = B * mp + 2
    k8 = np.resize(np.asarray(stale, np.uint8), (P, page, Hkv, D)).copy()
    v8 = k8.copy()
    table = rng.permutation(P)[:B * mp].reshape(B, mp).astype(np.int32)
    one = np.ones(Hkv, np.float32)
    for b, L in enumerate(lens_k):
        for j in range(L):
            k8[table[b, j // page], j % page] = fo.quantize(rng.standard_normal((Hkv, D)), one, fmt)
            v8[table[b, j // page], j % page] = fo.quantize(rng.standard_normal((Hkv, D)), one, fmt)
    cu_q = np.concatenate([[0], np.cumsum(lens_q)]).astype(np.int64)
    return rng.standard_normal((int(cu_q[-1]), Hq, D)), k8, v8, table, cu_q


def _sdpa_fp8(q, k8, v8, ks, vs, fmt, table, lens, cu_q, scale, window):
    """torch SDPA per sequence on torch's float8 dequantization of the gathered pages"""
    page, g = k8.shape[1], q.shape[1] // k8.shape[2]
    deq = lambda c, s: torch.from_numpy(c).view(TORCH_F8[fmt]).to(torch.float64) * torch.from_numpy(s).double()[:, None]  # noqa: E731
    out = np.full(q.shape, np.nan)
    for b, Lk in enumerate(lens):
        qa, qb = int(cu_q[b]), int(cu_q[b + 1])
        Lq = qb - qa
        if Lq == 0 or Lk == 0:
            continue
        rows = [(table[b, j // page], j % page) for j in range(Lk)]
        kk = deq(np.stack([k8[p, r] for p, r in rows]), ks)
        vv = deq(np.stack([v8[p, r] for p, r in rows]), vs)
        qs = torch.tensor(q[qa:qb]).transpose(0, 1)[None]
        kt, vt = (t.transpose(0, 1).repeat_interleave(g, dim=0)[None] for t in (kk, vv))
        if window == (-1, 0):
            mask = causal_lower_right(Lq, Lk)
        else:
            i, j = torch.arange(Lq)[:, None], torch.arange(Lk)[None, :]
            mask = torch.ones(Lq, Lk, dtype=torch.bool)
            if window[0] >= 0:
                mask &= j >= i + (Lk - Lq) - window[0]
            if window[1] >= 0:
                mask &= j <= i + (Lk - Lq) + window[1]
        out[qa:qb] = F.scaled_dot_product_attention(qs, kt, vt, attn_mask=mask, scale=scale)[0].transpose(0, 1).numpy()
    return out


@pytest.mark.parametrize("fmt", ["f8e4m3", "f8e5m2"])
@pytest.mark.parametrize("lens_q,lens_k,page,window", [
    ([5, 0, 9, 3], [12, 0, 9, 20], 4, (-1, 0)), ([9, 12], [17, 15], 4, (3, 0)), ([9, 0, 12], [17, 3, 15], 8, (2, 2)),
])
def test_oracle_matches_torch_sdpa_on_the_dequantized_cache(fmt, lens_q, lens_k, page, window):
    rng = np.random.default_rng(sum(lens_q) + page)
    Hq, Hkv, D, scale = 4, 2, 16, 0.3
    stale = (0x7F, 0xFF) if fmt == "f8e4m3" else (0x7F, 0x7C, 0xFC)
    q, k8, v8, table, cu_q = _problem(rng, lens_q, lens_k, Hq, Hkv, D, page, fmt, stale)
    ks, vs = np.array([0.37, 1.9], np.float32), np.array([2.5, 0.11], np.float32)
    out, lse = attention_varlen_paged_fp8_f64(q, k8, v8, ks, vs, fmt, table, lens_k, cu_q, max(lens_k), scale, window)
    ref = _sdpa_fp8(q, k8, v8, ks, vs, fmt, table, lens_k, cu_q, scale, window)
    seen = np.isfinite(lse).T
    assert np.all(np.isfinite(out)), "stale bytes reached the oracle's output"
    np.testing.assert_allclose(out[seen], ref[seen], rtol=0, atol=1e-12)
    assert np.all(out[~seen] == 0)


@pytest.mark.parametrize("fmt", ["f8e4m3", "f8e5m2"])
@pytest.mark.parametrize("dtype", ["bf16", "f16"])
def test_power_of_two_scales_give_the_16_bit_problem(fmt, dtype):
    rng = np.random.default_rng(5)
    lens_q, lens_k = [6, 4], [30, 9]
    q, k8, v8, table, cu_q = _problem(rng, lens_q, lens_k, 4, 2, 16, 8, fmt, 0)
    ks, vs = np.array([0.125, 4.0], np.float32), np.array([0.5, 2.0], np.float32)
    kd, vd = fo.dequantize(k8, ks, fmt), fo.dequantize(v8, vs, fmt)
    k16, v16 = (synth.from_device_dtype(synth.to_device_dtype(a.astype(np.float32), dtype), dtype).astype(np.float64) for a in (kd, vd))
    np.testing.assert_array_equal(k16, kd)   # scale * code is exact in q's dtype
    np.testing.assert_array_equal(v16, vd)
    got = attention_varlen_paged_fp8_f64(q, k8, v8, ks, vs, fmt, table, lens_k, cu_q, 64, None, (-1, 0))
    want = attention_varlen_paged_f64(q, k16, v16, table, lens_k, cu_q, 64, None, (-1, 0))
    for a, b in zip(got, want):
        np.testing.assert_array_equal(a, b)


# ---------------------------------------------------------------------------------------------- dry-run plans
class Planner8(Planner):
    def fwd(self, qs, kcs, B, maxq, maxk, bts=None, vcs=None, outs=None, idt=BF16, odt=None, strides=(None, None, None, None),
            bt_strides=None, ptrs=(Q, KC, VC, BT, CUQ, SEQ, OUT), lse=0, scale=0.125, window=(-1, -1), null_args=False, table=True,
            cdt=E4M3, scales=(KS, VS)):
        vcs = kcs if vcs is None else vcs
        outs = qs if outs is None else outs
        odt = idt if odt is None else odt
        bts = [B, 4] if bts is None else bts
        arr = lambda v: _ffi.u64_array(v) if v is not None else None  # noqa: E731
        args = _ffi.AttentionVarlenArgs(scale, window[0], window[1], maxq, maxk)
        bt = (ptrs[3], arr(bts), arr(bt_strides)) if table else (0, None, None)
        rc = self.lib.b200_attention_varlen_paged_fp8(
            self.ctx, None, idt, cdt, odt, ptrs[0], arr(qs), arr(strides[0]), ptrs[1], arr(kcs), arr(strides[1]), ptrs[2], arr(vcs),
            arr(strides[2]), *bt, ptrs[4], ptrs[5], B, scales[0], scales[1], ptrs[6], arr(outs), arr(strides[3]), lse,
            None if null_args else C.byref(args))
        return rc, self.text()


@pytest.fixture
def plan():
    p = Planner8()
    yield p
    p.close()


@pytest.mark.parametrize("idt,tag", [(BF16, "bf16"), (F16, "f16")])
@pytest.mark.parametrize("cdt,fmt", [(E4M3, "e4m3"), (E5M2, "e5m2")])
@pytest.mark.parametrize("D,bucket", [(16, 64), (48, 64), (64, 64), (80, 128), (128, 128)])
@pytest.mark.parametrize("f32", [False, True])
def test_kernel_names_grids_and_shared_memory(plan, idt, tag, cdt, fmt, D, bucket, f32):
    B, Hq, Hkv, Tq, maxq, maxk = 5, 8, 2, 3000, 1000, 700
    rc, t = plan.fwd([Tq, Hq, D], [40, 64, Hkv, D], B, maxq, maxk, bts=[B, 16], idt=idt, odt=F32 if f32 else idt, cdt=cdt)
    assert rc == 0, _ffi.load().b200_last_error()
    o = "f32" if f32 else tag
    smem = 1024 + 5 * 128 * bucket * 2 + 2 * 2 * 128 * 128 + 1024
    assert _launches(t) == [(f"attn_fwd_paged_{tag}_{fmt}_d{bucket}_{o}", str(8 * Hq * B), "384", str(smem))]
    assert smem <= 232448   # the per-block opt-in limit
    _only_alloc_tmap_launch(t)


def test_shared_memory_at_d128_is_231424_bytes(plan):
    rc, t = plan.fwd([300, 8, 128], [40, 64, 2, 128], 2, 128, 256)
    assert rc == 0 and _launches(t)[0][3] == "231424"


@pytest.mark.parametrize("page,rows", [(16, 16), (32, 32), (64, 64), (128, 128), (192, 64), (256, 128)])
def test_maps_of_paged_fp8_caches(plan, page, rows):
    Tq, Hq, Hkv, D, B, P = 300, 8, 2, 128, 3, 40
    rc, t = plan.fwd([Tq, Hq, D], [P, page, Hkv, D], B, 128, 4096, bts=[B, 8], odt=F32)
    assert rc == 0, _ffi.load().b200_last_error()
    assert "gather" not in t
    mq, mk, mv, mo = _tmaps(t)
    assert mq == (2, (D, Tq, Hq, 1), (2 * Hq * D, 2 * D, 2 * Tq * Hq * D), (64, 128, 1, 1))
    assert mk == mv == (1, (D, page, Hkv, P), (Hkv * D, D, page * Hkv * D), (128, rows, 1, 1))
    assert mo[:2] == (4, (D, Tq, Hq, 1)) and mo[3] == (32, 64, 1, 1)
    _only_alloc_tmap_launch(t)


@pytest.mark.parametrize("page", [40, 100, 1000])
def test_one_page_per_sequence_loads_128_rows(plan, page):
    Hkv, D, B = 2, 64, 3
    rc, t = plan.fwd([300, 4, D], [B, page, Hkv, D], B, 128, 4096, table=False)
    assert rc == 0, _ffi.load().b200_last_error()
    assert [m[3] for m in _tmaps(t)[1:3]] == [(128, 128, 1, 1)] * 2 and _tmaps(t)[1][:2] == (1, (D, page, Hkv, B))
    rc, t = plan.fwd([300, 4, D], [7, page, Hkv, D], B, 128, 4096, bts=[B, 1])
    assert rc == 0 and [m[3] for m in _tmaps(t)[1:3]] == [(128, 128, 1, 1)] * 2


def test_head_major_fp8_cache_is_read_in_place(plan):
    P, page, Hkv, D, B = 30, 64, 4, 128, 3
    head_major = [Hkv * page * D, D, page * D, 1]
    rc, t = plan.fwd([300, 8, D], [P, page, Hkv, D], B, 128, 1024, strides=(None, head_major, head_major, None))
    assert rc == 0, _ffi.load().b200_last_error()
    assert "gather" not in t
    mk = _tmaps(t)[1]
    assert mk == (1, (D, page, Hkv, P), (D, page * D, Hkv * page * D), (128, 64, 1, 1))


def test_misaligned_q_is_gathered(plan):
    T, H, D = 256, 4, 64
    rc, t = plan.fwd([T, H, D], [10, 32, 2, D], 2, 128, 256, ptrs=(Q + 2, KC, VC, BT, CUQ, SEQ, OUT), cdt=E5M2)
    assert rc == 0, _ffi.load().b200_last_error()
    assert [n for n, *_ in _launches(t)] == ["gather_strided", "attn_fwd_paged_bf16_e5m2_d64_bf16"]
    assert _tmaps(t)[0][2][:2] == (2 * H * D, 2 * D)
    _only_alloc_tmap_launch(t)


# every refusal of b200_attention_varlen_paged (its test's cases), then the fp8 ones
CASES = [
    ("head_dim", INVALID, "k_cache head dim"), ("v_shape", INVALID, "does not match"), ("gqa", INVALID, "multiple of Hkv"),
    ("hkv0", INVALID, "multiple of Hkv"), ("out_shape", INVALID, "out is"), ("window_left", INVALID, "window"),
    ("window_right", INVALID, "window"), ("max_neg", INVALID, "max_seqlen"), ("scale_inf", INVALID, "finite"),
    ("null_args", INVALID, "null shape or args"), ("null_bt_shape", INVALID, "block-table shape"), ("null_q", INVALID, "null device"),
    ("null_cu", INVALID, "null device"), ("null_seqlens", INVALID, "null device"), ("cu_align", INVALID, "aligned"),
    ("seqlens_align", INVALID, "aligned"), ("bt_align", INVALID, "aligned"), ("lse_align", INVALID, "aligned"),
    ("empty_pages", INVALID, "empty cache"), ("empty_page", INVALID, "empty cache"), ("bt_rows", INVALID, "block_table is"),
    ("bt_zero", INVALID, "block_table is"), ("no_table_p", INVALID, "one page per sequence"), ("in_f32", UNSUPPORTED, "input dtype"),
    ("out_other", UNSUPPORTED, "output dtype"), ("d136", UNSUPPORTED, "head dim"), ("dv", UNSUPPORTED, "v_cache's head dim"),
    ("page_24", UNSUPPORTED, "a page of 24 keys"), ("page_96", UNSUPPORTED, "a page of 96 keys"),
    ("cache_misaligned", UNSUPPORTED, "never gathered"), ("cache_stride", UNSUPPORTED, "never gathered"),
    ("out_misaligned", UNSUPPORTED, "out needs"), ("huge", UNSUPPORTED, "2^31"), ("capacity", UNSUPPORTED, "capacity"),
    ("max_huge", UNSUPPORTED, "2^30"), ("ctas", UNSUPPORTED, "CTAs"),
    ("cache_bf16", UNSUPPORTED, "cache dtype"), ("cache_f32", UNSUPPORTED, "cache dtype"), ("null_k_scale", INVALID, "null k_scale"),
    ("null_v_scale", INVALID, "null k_scale or v_scale"), ("k_scale_align", INVALID, "4-byte aligned"),
    ("v_scale_align", INVALID, "4-byte aligned"), ("d40_compact", UNSUPPORTED, "never gathered"),
    ("d8_compact", UNSUPPORTED, "never gathered"),
]
_PTR = {"null_q": (0, 0), "null_cu": (4, 0), "null_seqlens": (5, 0), "cu_align": (4, CUQ + 2), "seqlens_align": (5, SEQ + 2),
        "bt_align": (3, BT + 2), "cache_misaligned": (1, KC + 2), "out_misaligned": (6, OUT + 2)}
_KW = {"v_shape": {"vcs": [10, 16, 2, 64]}, "out_shape": {"outs": [300, 2, 64]}, "window_left": {"window": (-2, 0)},
       "window_right": {"window": (4, -5)}, "scale_inf": {"scale": float("inf")}, "null_args": {"null_args": True},
       "lse_align": {"lse": LSE + 2}, "bt_rows": {"bts": [3, 4]}, "bt_zero": {"bts": [2, 0]}, "no_table_p": {"table": False},
       "in_f32": {"idt": F32, "odt": F32}, "out_other": {"idt": BF16, "odt": F16}, "dv": {"vcs": [10, 32, 2, 32]},
       "cache_stride": {"strides": (None, None, [32 * 2 * 72, 2 * 72, 72, 1], None)},   # v_cache rows of 72 bytes at D = 64
       "capacity": {"bts": [2, 1 << 27]}, "cache_bf16": {"cdt": BF16}, "cache_f32": {"cdt": F32},
       "null_k_scale": {"scales": (0, VS)}, "null_v_scale": {"scales": (KS, 0)}, "k_scale_align": {"scales": (KS + 2, VS)},
       "v_scale_align": {"scales": (KS, VS + 6)}}
_KCS = {"head_dim": [10, 32, 2, 32], "gqa": [10, 32, 3, 64], "hkv0": [10, 32, 0, 64], "empty_pages": [0, 32, 2, 64],
        "empty_page": [10, 0, 2, 64], "page_24": [10, 24, 2, 64], "page_96": [10, 96, 2, 64]}


@pytest.mark.parametrize("case,status,words", CASES)
def test_refusals(plan, case, status, words):
    qs, kcs, B, maxq, maxk = [300, 4, 64], _KCS.get(case, [10, 32, 2, 64]), 2, 128, 256
    kw, ptrs = dict(_KW.get(case, {})), [Q, KC, VC, BT, CUQ, SEQ, OUT]
    if case in _PTR:
        ptrs[_PTR[case][0]] = _PTR[case][1]
    if case == "null_bt_shape":
        lib, arr = _ffi.load(), _ffi.u64_array
        args = _ffi.AttentionVarlenArgs(0.125, -1, -1, maxq, maxk)
        rc = lib.b200_attention_varlen_paged_fp8(plan.ctx, None, BF16, E4M3, BF16, Q, arr(qs), None, KC, arr(kcs), None, VC, arr(kcs),
                                                 None, BT, None, None, CUQ, SEQ, B, KS, VS, OUT, arr(qs), None, 0, C.byref(args))
        msg = lib.b200_last_error().decode()
        assert rc == status and words in msg and plan.text() == "", msg
        return
    if case == "max_neg":
        maxk = -1
    elif case == "d136":
        qs, kcs = [300, 4, 136], [10, 32, 2, 136]
    elif case == "d40_compact":   # 40-byte rows: a compact fp8 cache needs D % 16 == 0
        qs, kcs = [300, 4, 40], [10, 32, 2, 40]
    elif case == "d8_compact":
        qs, kcs = [300, 4, 8], [10, 32, 2, 8]
    elif case == "huge":
        qs = [1 << 31, 4, 64]
    elif case == "max_huge":
        maxq = 1 << 30
    elif case == "ctas":
        qs, B, maxq = [300, 1 << 16, 64], 1 << 13, (1 << 30) - 1
        kcs, kw["outs"], kw["bts"] = [1 << 13, 32, 1 << 16, 64], [300, 1 << 16, 64], [1 << 13, 4]
    if "bts" not in kw and case not in ("no_table_p",):
        kw["bts"] = [B, 4]
    rc, t = plan.fwd(qs, kcs, B, maxq, maxk, ptrs=tuple(ptrs), **kw)
    msg = _ffi.load().b200_last_error().decode()
    assert rc == status, (case, rc, msg)
    assert words in msg, msg
    assert msg.startswith("attention_varlen_paged_fp8: "), msg
    assert _launches(t) == [] and "gather" not in t


def test_16_bit_views_of_the_same_d40_cache_are_accepted(plan):
    """the D % 16 rule is the fp8 cache's byte strides, not the entry's: a 16-bit D = 40 cache has 80-byte rows"""
    rc, _ = Planner.fwd(plan, [300, 4, 40], [10, 32, 2, 40], 2, 128, 256)
    assert rc == 0, _ffi.load().b200_last_error()


def test_zero_extents_launch_nothing(plan):
    for qs, B, maxq in (([300, 4, 64], 0, 128), ([0, 4, 64], 2, 128), ([300, 0, 64], 2, 128), ([300, 4, 64], 2, 0)):
        kcs = [10, 32, 2 if qs[1] else 1, 64]
        rc, t = plan.fwd(qs, kcs, B, maxq, 256, bts=[B, 4])
        assert rc == 0 and t == "", (qs, B, maxq, t, _ffi.load().b200_last_error())


def test_python_entry_points_defer_errors():
    from cubecl_b200 import attention

    class _Stub:
        def __init__(self):
            self.errors = []

        def _defer(self, e):
            self.errors.append(e)

    class _T:
        def __init__(self, shape, dtype="bf16", contiguous=True):
            self.shape, self.dtype, self._c = shape, dtype, contiguous

        def is_contiguous(self):
            return self._c

    stub = _Stub()
    q, kc, cq, sl, s = _T([30, 4, 64]), _T([8, 16, 2, 64], "f8e4m3"), _T([3], "i32"), _T([2], "i32"), _T([2], "f32")
    f = attention.launch_varlen_paged_fp8
    f(stub, _T([30, 4]), kc, kc, cq, sl, s, s, 16, 16, q)                                     # q rank
    f(stub, q, _T([8, 16, 64], "f8e4m3"), kc, cq, sl, s, s, 16, 16, q)                         # cache rank
    f(stub, q, _T([8, 16, 2, 64]), _T([8, 16, 2, 64]), cq, sl, s, s, 16, 16, q)                # 16-bit caches
    f(stub, q, kc, _T([8, 16, 2, 64], "f8e5m2"), cq, sl, s, s, 16, 16, q)                      # cache dtypes differ
    f(stub, q, kc, kc, cq, sl, _T([3], "f32"), s, 16, 16, q)                                   # k_scale not [Hkv]
    f(stub, q, kc, kc, cq, sl, s, _T([2], "f16"), 16, 16, q)                                   # v_scale not f32
    f(stub, q, kc, kc, _T([3], "i64"), sl, s, s, 16, 16, q)                                    # cu not i32
    f(stub, q, kc, kc, cq, _T([3], "i32"), s, s, 16, 16, q)                                    # seqlens not [B]
    f(stub, q, kc, kc, cq, sl, s, s, 16, 16, q, block_table=_T([2, 4], "i64"))                 # table not i32
    f(stub, q, kc, kc, cq, sl, s, s, 16, 16, q, lse=_T([30, 4], "f32"))                        # lse shape
    assert [e.status for e in stub.errors] == [INVALID, INVALID, UNSUPPORTED, UNSUPPORTED] + [INVALID] * 6
    msgs = [str(e) for e in stub.errors]
    assert all("attention_varlen_paged_fp8" in m for m in msgs)
    assert "rank 3" in msgs[0] and "rank 4" in msgs[1] and "unsupported" in msgs[2] and "differ" in msgs[3]
    assert "k_scale" in msgs[4] and "v_scale" in msgs[5] and "cu_seqlens_q" in msgs[6] and "cache_seqlens" in msgs[7]
    assert "block_table" in msgs[8] and "lse" in msgs[9]


# ---------------------------------------------------------------------------------------------- kernels
def test_paged_fp8_kernels_use_register_a_wgmma_and_tma_and_do_not_spill():
    tool = _tool("cuobjdump")
    _ffi.load()
    path = ROOT / "cubecl_b200" / "build" / "attention_paged_fp8.cubin"
    out = subprocess.run([tool, "-res-usage", str(path)], capture_output=True, text=True, check=True).stdout
    funcs = re.findall(r"Function (\w+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)
    want = {f"attn_fwd_paged_{i}_{f}_d{d}_{o}" for i in ("bf16", "f16") for f in ("e4m3", "e5m2") for d in (64, 128) for o in (i, "f32")}
    assert {f for f, *_ in funcs} == want and len(want) == 16
    for name, reg, stack, local in funcs:
        assert int(stack) == 0 and int(local) == 0, (name, stack, local)
        assert int(reg) <= 168, (name, reg)
    sass = subprocess.run([tool, "-sass", str(path)], capture_output=True, text=True, check=True).stdout
    for body in re.split(r"\n\s*Function : ", sass)[1:]:
        name = body.split()[0]
        n = 64 if "_d64_" in name else 128
        assert re.search(rf"HGMMA\.64x{n}x16\.F32\S* R\d+, R\d+, gdesc\[UR\d+\]\.tnspB", body), name   # register-A product
        assert "UTMALDG.4D" in body and "UTMASTG.4D" in body, name
        assert "F2FP" in body or "F2F" in body, name   # the fp8 widening
