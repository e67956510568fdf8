"""CPU: the f64 KV-cache attention oracle (pinned to the dense oracle and to torch's SDPA with causal_lower_right), and the
dry-run plans of b200_attention_kvcache and b200_kvcache_write: kernel names, the split count over a grid of shapes, one
launch at nsplit = 1 and alloc + kernel + combine otherwise, the maps of paged and head-major caches, the (gt, st) m-tile,
every refusal with its status, and the new cubin's kernels (no spills, no local memory)."""
import ctypes as C
import math
import re
import subprocess

import numpy as np
import pytest
import torch

import attention_kvcache_oracle as ko
import attention_oracle as ao
from cubecl_b200 import _ffi
from plan_context import PlanContext
from test_conv_cpu import ROOT, _tool

F32, F16, BF16, I8 = _ffi.F32, _ffi.F16, _ffi.BF16, _ffi.I8
Q, KC, VC, BT, SL, OUT, LSE = 0x10000000, 0x20000000, 0x30000000, 0x40000000, 0x50000000, 0x60000000, 0x70000000
INVALID, UNSUPPORTED = 6, 7


# ---------------------------------------------------------------------------------------------- oracle
def _paged(k, page, rng):
    """k [B, Hkv, cap, D] -> a [P, page, Hkv, D] cache with shuffled pages and its block table"""
    B, Hkv, cap, D = k.shape
    mp = cap // page
    perm = rng.permutation(B * mp)
    cache = np.full((B * mp, page, Hkv, D), np.nan)
    table = perm.reshape(B, mp)
    for b in range(B):
        for p in range(mp):
            cache[table[b, p]] = k[b, :, p * page:(p + 1) * page].transpose(1, 0, 2)
    return cache, table


@pytest.mark.parametrize("B,Hq,Hkv,S,D,causal", [(2, 4, 2, 32, 16, False), (1, 6, 3, 48, 8, True), (3, 2, 2, 16, 24, True)])
def test_oracle_equals_the_dense_oracle_when_every_length_is_sq(B, Hq, Hkv, S, D, causal):
    rng = np.random.default_rng(S + D)
    q, k, v = rng.standard_normal((B, Hq, S, D)), rng.standard_normal((B, Hkv, S, D)), rng.standard_normal((B, Hkv, S, D))
    kc, table = _paged(k, 16, np.random.default_rng(1))
    vc, _ = _paged(v, 16, np.random.default_rng(1))
    out, lse = ko.attention_kvcache_f64(q, kc, vc, [S] * B, table, None, causal)
    ref, ref_lse = ao.attention_f64(q, k, v, None, causal)
    np.testing.assert_allclose(out, ref, rtol=0, atol=1e-12)
    np.testing.assert_allclose(lse, ref_lse, rtol=0, atol=1e-12)


@pytest.mark.parametrize("causal", [False, True])
def test_oracle_matches_torch_causal_lower_right(causal):
    from torch.nn.attention.bias import causal_lower_right
    B, Hq, Hkv, Sq, D, cap = 3, 4, 2, 5, 16, 64
    rng = np.random.default_rng(7)
    q, k, v = rng.standard_normal((B, Hq, Sq, D)), rng.standard_normal((B, Hkv, cap, D)), rng.standard_normal((B, Hkv, cap, D))
    lens = [37, 5, 64]
    kc, table = _paged(k, 16, np.random.default_rng(2))
    vc, _ = _paged(v, 16, np.random.default_rng(2))
    out, lse = ko.attention_kvcache_f64(q, kc, vc, lens, table, 0.3, causal)
    for b, L in enumerate(lens):
        qt = torch.from_numpy(q[b:b + 1])
        kt, vt = (torch.from_numpy(t[b:b + 1, :, :L]).repeat_interleave(Hq // Hkv, dim=1) for t in (k, v))
        mask = causal_lower_right(Sq, L) if causal else None
        ref = torch.nn.functional.scaled_dot_product_attention(qt, kt, vt, attn_mask=mask, scale=0.3)
        np.testing.assert_allclose(out[b:b + 1], ref.numpy(), rtol=0, atol=1e-12)
        s = 0.3 * torch.einsum("bhid,bhjd->bhij", qt, kt)
        if causal:
            s = s.masked_fill(~torch.ones(Sq, L, dtype=torch.bool).tril(L - Sq), -math.inf)
        np.testing.assert_allclose(lse[b], torch.logsumexp(s, dim=-1)[0].numpy(), rtol=1e-13, atol=1e-13)


def test_oracle_rows_without_keys_and_clamped_lengths():
    rng = np.random.default_rng(3)
    q, kc = rng.standard_normal((2, 2, 4, 8)), rng.standard_normal((2, 16, 1, 8))
    out, lse = ko.attention_kvcache_f64(q, kc, kc, [2, 99], None, 1.0, True)   # L = 2 < Sq: rows 0, 1 see nothing
    assert np.all(out[0, :, :2] == 0) and np.all(lse[0, :, :2] == -np.inf) and np.isfinite(lse[0, :, 2:]).all()
    full, _ = ko.attention_kvcache_f64(q, kc, kc, [16, 16], None, 1.0, True)
    np.testing.assert_array_equal(out[1], full[1])   # 99 is clamped to the capacity 16


# ---------------------------------------------------------------------------------------------- dry-run plans
class Planner(PlanContext):
    def run(self, qs, kcs, vcs=None, bts=None, outs=None, idt=BF16, odt=None, strides=(None, None, None, None, None),
            ptrs=(Q, KC, VC, BT, SL, OUT), lse=0, scale=0.125, causal=0, null_args=False):
        vcs = kcs if vcs is None else vcs
        outs = qs if outs is None else outs
        odt = idt if odt is None else odt
        arr = lambda v: _ffi.u64_array(v) if v is not None else None  # noqa: E731
        args = _ffi.AttentionArgs(scale, causal)
        bt = ptrs[3] if bts is not None else 0
        rc = self.lib.b200_attention_kvcache(self.ctx, None, idt, odt, ptrs[0], arr(qs), arr(strides[0]), ptrs[1], arr(kcs), arr(strides[1]),
                                             ptrs[2], arr(vcs), arr(strides[2]), bt, arr(bts), arr(strides[3]), ptrs[4], ptrs[5], arr(outs),
                                             arr(strides[4]), lse, None if null_args else C.byref(args))
        return rc, self.text()

    def write(self, kns, kcs, vns=None, vcs=None, dt=BF16, strides=(None, None, None, None), ptrs=(Q, KC, VC, BT, SL)):
        vns = kns if vns is None else vns
        vcs = kcs if vcs is None else vcs
        arr = lambda v: _ffi.u64_array(v) if v is not None else None  # noqa: E731
        rc = self.lib.b200_kvcache_write(self.ctx, None, dt, ptrs[0], arr(kns), arr(strides[0]), ptrs[3], arr(vns), arr(strides[1]),
                                         ptrs[1], arr(kcs), arr(strides[2]), ptrs[2], arr(vcs), arr(strides[3]), ptrs[4])
        return rc, self.text()


@pytest.fixture
def plan():
    with Planner() as p:
        yield p


def _launches(t):
    return re.findall(r"launch (\S+) grid=\((\d+),1,1\) block=(\d+) smem=(\d+) cluster=1", t)


_TMAP = re.compile(r"tmap4d esz=(\d+) dims=\(([\d,]+)\) strides=\(([\d,]+)\) box=\(([\d,]+)\) swizzle=3")


def _tmaps(t):
    ints = lambda g: tuple(int(v) for v in g.split(","))  # noqa: E731
    return [(int(m.group(1)), ints(m.group(2)), ints(m.group(3)), ints(m.group(4))) for m in _TMAP.finditer(t)]


def _smem(bucket):
    return 1024 + bucket // 64 * (64 + 2 * 4 * 64) * 128 + 128


@pytest.mark.parametrize("idt,tag", [(BF16, "bf16"), (F16, "f16")])
@pytest.mark.parametrize("D,bucket", [(8, 64), (64, 64), (72, 128), (128, 128)])
@pytest.mark.parametrize("out_f32", [False, True])
def test_kernel_per_dtype_bucket_and_out(plan, idt, tag, D, bucket, out_f32):
    # B * Hkv = 256 CTAs with 2 key blocks each: one split
    rc, t = plan.run([32, 32, 1, D], [32, 128, 8, D], idt=idt, odt=F32 if out_f32 else idt)
    assert rc == 0, _ffi.load().b200_last_error()
    (name, grid, block, smem), = _launches(t)
    assert name == f"attn_kv_{tag}_d{bucket}_{'f32' if out_f32 else tag}"
    assert (int(grid), int(block), int(smem)) == (32 * 8, 160, _smem(bucket))
    assert "alloc" not in t and "gather" not in t


@pytest.mark.parametrize("sms", [132, 8])
def test_split_count_over_a_grid_of_shapes(sms):
    p = Planner(sms)
    try:
        seen = set()
        for B in (1, 2, 8, 64, 128):
            for Hq, Hkv in ((32, 8), (32, 32), (8, 1)):
                for Sq in (1, 4):
                    for cap in (64, 1000, 2048, 16384, 65536):
                        rc, t = p.run([B, Hq, Sq, 128], [B, cap, Hkv, 128])
                        assert rc == 0, _ffi.load().b200_last_error()
                        gt, st = ko.kv_tile(Hq // Hkv, Sq)
                        units = B * Hkv * -(-(Hq // Hkv) // gt) * -(-Sq // st)
                        n = ko.kv_splits(units, -(-cap // 64), sms)
                        names = [x[0] for x in _launches(t)]
                        assert int(_launches(t)[0][1]) == units * n, (B, Hq, Hkv, Sq, cap)
                        if n == 1:
                            assert names == ["attn_kv_bf16_d128_bf16"] and "alloc" not in t
                        else:
                            assert names == ["attn_kv_bf16_d128_bf16", "attn_kv_combine_bf16"]
                            (alloc,) = re.findall(r"alloc (\d+)", t)
                            assert int(alloc) >= n * B * Hq * Sq * 130 * 4
                            assert int(_launches(t)[1][1]) == -(-B * Hq * Sq * 32 // 256)
                        seen.add(n > 1)
        assert seen == {False, True}
    finally:
        p.close()


def test_splits_of_long_decodes_fill_the_gpu(plan):
    """B = 1, L = 65536, Hq = 32, Hkv = 8: 8 CTAs without splits; the plan splits each into 16 ranges of 64 blocks"""
    rc, t = plan.run([1, 32, 1, 128], [1, 65536, 8, 128])
    assert rc == 0 and int(_launches(t)[0][1]) == 8 * 16 and len(_launches(t)) == 2


def test_split_count_ignores_the_page_layout(plan):
    """equal capacity, equal plan: identity, 16-token pages, 256-token pages"""
    grids = []
    for kcs, bts in (([4, 4096, 8, 128], None), ([4 * 256, 16, 8, 128], [4, 256]), ([4 * 16, 256, 8, 128], [4, 16])):
        rc, t = plan.run([4, 32, 1, 128], kcs, bts=bts)
        assert rc == 0, _ffi.load().b200_last_error()
        grids.append([g for _, g, _, _ in _launches(t)])
    assert grids[0] == grids[1] == grids[2]


def test_maps_of_a_paged_cache(plan):
    B, Hq, Hkv, D, P, page, mp = 4, 32, 8, 128, 100, 16, 40
    rc, t = plan.run([B, Hq, 1, D], [P, page, Hkv, D], bts=[B, mp])
    assert rc == 0, _ffi.load().b200_last_error()
    mq, mk, mv = _tmaps(t)
    assert mq == (2, (D, 1, Hq, B), (2 * D, 2 * D, 2 * D * Hq), (64, 1, 4, 1))
    row, head, pg = 2 * Hkv * D, 2 * D, 2 * page * Hkv * D
    assert mk == mv == (2, (D, page, Hkv, P), (row, head, pg), (64, 16, 1, 1))


def test_maps_of_a_head_major_cache_and_a_bshd_query(plan):
    """a [P, Hkv, page, D] cache and a [B, Sq, Hq, D] q are views: the strides go into the maps, nothing is gathered"""
    B, Hq, Hkv, Sq, D, P, page = 2, 8, 2, 3, 64, 10, 64
    hm = [Hkv * page * D, D, page * D, 1]
    qv = [Sq * Hq * D, D, Hq * D, 1]
    rc, t = plan.run([B, Hq, Sq, D], [P, page, Hkv, D], bts=[B, 5], strides=(qv, hm, hm, None, None))
    assert rc == 0, _ffi.load().b200_last_error()
    assert "gather" not in t
    mq, mk, mv = _tmaps(t)
    assert mq[1:3] == ((D, Sq, Hq, B), (2 * Hq * D, 2 * D, 2 * Sq * Hq * D)) and mq[3] == (64, 3, 4, 1)
    assert mk == mv == (2, (D, page, Hkv, P), (2 * D, 2 * page * D, 2 * Hkv * page * D), (64, 64, 1, 1))


@pytest.mark.parametrize("page,rows", [(16, 16), (32, 32), (64, 64), (128, 64), (256, 64)])
def test_load_rows_per_page_size(plan, page, rows):
    rc, t = plan.run([2, 8, 1, 128], [64, page, 2, 128], bts=[2, 4])
    assert rc == 0 and _tmaps(t)[1][3] == (64, rows, 1, 1)


def test_one_page_per_sequence_takes_any_size(plan):
    for kcs, bts in (([3, 1000, 2, 64], None), ([7, 1000, 2, 64], [3, 1]), ([3, 20, 2, 64], None)):
        rc, t = plan.run([3, 4, 1, 64], kcs, bts=bts)
        assert rc == 0, _ffi.load().b200_last_error()
        assert _tmaps(t)[1][3] == (64, 64, 1, 1)


@pytest.mark.parametrize("G,Sq,gt,st", [
    (1, 1, 1, 1), (1, 4, 1, 4), (1, 33, 1, 33), (4, 1, 4, 1), (4, 4, 4, 4), (4, 33, 4, 16), (8, 1, 8, 1), (8, 4, 8, 4),
    (8, 33, 8, 8), (64, 1, 64, 1), (64, 4, 16, 4), (64, 33, 64, 1), (128, 1, 64, 1), (128, 4, 16, 4), (128, 33, 64, 1),
])
def test_m_tile_of_heads_and_queries(plan, G, Sq, gt, st):
    assert ko.kv_tile(G, Sq) == (gt, st)
    B, Hkv = 2, 2
    rc, t = plan.run([B, G * Hkv, Sq, 64], [B, 640, Hkv, 64])
    assert rc == 0, _ffi.load().b200_last_error()
    assert _tmaps(t)[0][3] == (64, st, gt, 1)
    mtiles = -(-G // gt) * -(-Sq // st)
    assert gt * st <= 64 and int(_launches(t)[0][1]) == B * Hkv * mtiles * ko.kv_splits(B * Hkv * mtiles, 10, 132)


def test_misaligned_query_is_gathered(plan):
    rc, t = plan.run([64, 4, 1, 64], [64, 128, 2, 64], ptrs=(Q + 2, KC, VC, BT, SL, OUT))   # 128 CTAs: one split
    assert rc == 0
    assert [x[0] for x in _launches(t)] == ["gather_strided", "attn_kv_bf16_d64_bf16"]
    assert _tmaps(t)[0][2] == (2 * 64, 2 * 64, 2 * 64 * 4)   # the q map reads the compact copy


# ---------------------------------------------------------------------------------------------- refusals
@pytest.mark.parametrize("case,status,words", [
    ("head_dim", INVALID, "head dim"), ("v_shape", INVALID, "does not match"), ("gqa", INVALID, "multiple of Hkv"),
    ("hkv0", INVALID, "multiple of Hkv"), ("out_shape", INVALID, "out is"), ("page0", INVALID, "empty cache"),
    ("bt_batch", INVALID, "block_table"), ("bt_empty", INVALID, "block_table"), ("no_table_p", INVALID, "one page per sequence"),
    ("scale_inf", INVALID, "finite"), ("null_args", INVALID, "null"), ("null_seqlens", INVALID, "null"), ("null_q", INVALID, "null"),
    ("lse_align", INVALID, "aligned"), ("seqlens_align", INVALID, "aligned"), ("bt_align", INVALID, "aligned"),
    ("in_f32", UNSUPPORTED, "input dtype"), ("in_i8", UNSUPPORTED, "input dtype"), ("out_other", UNSUPPORTED, "output dtype"),
    ("d136", UNSUPPORTED, "head dim"), ("d12", UNSUPPORTED, "head dim"), ("dv", UNSUPPORTED, "v_cache's head dim"),
    ("page24", UNSUPPORTED, "multiple of 16"), ("page96", UNSUPPORTED, "multiple of 16"),
    ("cache_misaligned", UNSUPPORTED, "cache"), ("cache_d_stride", UNSUPPORTED, "cache"), ("cache_odd_stride", UNSUPPORTED, "cache"),
    ("out_misaligned", UNSUPPORTED, "out"), ("huge", UNSUPPORTED, "2^31"),
])
def test_refusals(plan, case, status, words):
    qs, kcs, bts = [2, 4, 1, 64], [8, 16, 2, 64], [2, 4]
    kw = {}
    ptrs = [Q, KC, VC, BT, SL, OUT]
    if case == "head_dim":
        kcs = [8, 16, 2, 32]
    elif case == "v_shape":
        kw["vcs"] = [8, 32, 2, 64]
    elif case == "gqa":
        kcs = [8, 16, 3, 64]
    elif case == "hkv0":
        kcs = [8, 16, 0, 64]
    elif case == "out_shape":
        kw["outs"] = [2, 4, 2, 64]
    elif case == "page0":
        kcs = [8, 0, 2, 64]
    elif case == "bt_batch":
        bts = [3, 4]
    elif case == "bt_empty":
        bts = [2, 0]
    elif case == "no_table_p":
        bts = None
    elif case == "scale_inf":
        kw["scale"] = math.inf
    elif case == "null_args":
        kw["null_args"] = True
    elif case == "null_seqlens":
        ptrs[4] = 0
    elif case == "null_q":
        ptrs[0] = 0
    elif case == "lse_align":
        kw["lse"] = LSE + 2
    elif case == "seqlens_align":
        ptrs[4] = SL + 2
    elif case == "bt_align":
        ptrs[3] = BT + 2
    elif case == "in_f32":
        kw["idt"], kw["odt"] = F32, F32
    elif case == "in_i8":
        kw["idt"], kw["odt"] = I8, F32
    elif case == "out_other":
        kw["idt"], kw["odt"] = BF16, F16
    elif case == "d136":
        qs, kcs = [2, 4, 1, 136], [8, 16, 2, 136]
    elif case == "d12":
        qs, kcs = [2, 4, 1, 12], [8, 16, 2, 12]
    elif case == "dv":
        kw["vcs"] = [8, 16, 2, 32]
    elif case == "page24":
        kcs = [8, 24, 2, 64]
    elif case == "page96":
        kcs = [8, 96, 2, 64]
    elif case == "cache_misaligned":      # a gather of the whole cache per step is refused, not performed
        ptrs[1] = KC + 2
    elif case == "cache_d_stride":
        kw["strides"] = (None, [16 * 2 * 64, 1, 64 * 16, 16], None, None, None)
    elif case == "cache_odd_stride":      # a row stride of 136 bytes is not a 16-byte multiple
        kw["strides"] = (None, None, [16 * 2 * 68, 2 * 68, 68, 1], None, None)
    elif case == "out_misaligned":
        ptrs[5] = OUT + 2
    elif case == "huge":
        kcs, bts = [8, 1 << 16, 2, 64], [2, 1 << 15]
    rc, t = plan.run(qs, kcs, bts=bts, ptrs=tuple(ptrs), **kw)
    msg = _ffi.load().b200_last_error().decode()
    assert rc == status, (case, rc, msg)
    assert words in msg, msg
    assert _launches(t) == [] and "gather" not in t


def test_zero_extents_plan_no_launch(plan):
    for qs in ([0, 4, 1, 64], [2, 0, 1, 64], [2, 4, 0, 64]):
        rc, t = plan.run(qs, [8, 16, 2, 64], bts=[qs[0], 4])
        assert rc == 0 and t == "", (qs, t)


# ---------------------------------------------------------------------------------------------- kvcache_write
def test_write_plan_and_gathered_views(plan):
    rc, t = plan.write([2, 3, 4, 128], [10, 16, 4, 128])
    assert rc == 0, _ffi.load().b200_last_error()
    assert _launches(t) == [("attn_kv_write", str(-(-2 * 3 * 4 * 16 // 256)), "256", "0")]
    st = [3 * 4 * 136, 4 * 136, 136, 1]   # a padded row of 136 elements is 16-byte aligned: read in place
    rc, t = plan.write([2, 3, 4, 128], [10, 16, 4, 128], strides=(st, None, None, None))
    assert rc == 0 and "gather" not in t
    rc, t = plan.write([2, 3, 4, 128], [10, 16, 4, 128], ptrs=(Q + 2, KC, VC, BT, SL))
    assert rc == 0 and [x[0] for x in _launches(t)] == ["gather_strided", "attn_kv_write"]


@pytest.mark.parametrize("case,status,words", [
    ("v_new", INVALID, "v_new"), ("v_cache", INVALID, "v_cache"), ("heads", INVALID, "heads or head dim"), ("null", INVALID, "null"),
    ("slots_align", INVALID, "aligned"), ("dtype", UNSUPPORTED, "dtype"), ("d12", UNSUPPORTED, "multiple of 8"),
    ("cache_misaligned", UNSUPPORTED, "cache"),
])
def test_write_refusals(plan, case, status, words):
    kns, kcs = [2, 3, 4, 64], [10, 16, 4, 64]
    kw, ptrs = {}, [Q, KC, VC, BT, SL]
    if case == "v_new":
        kw["vns"] = [2, 4, 4, 64]
    elif case == "v_cache":
        kw["vcs"] = [10, 32, 4, 64]
    elif case == "heads":
        kcs = [10, 16, 2, 64]
    elif case == "null":
        ptrs[4] = 0
    elif case == "slots_align":
        ptrs[4] = SL + 2
    elif case == "dtype":
        kw["dt"] = F32
    elif case == "d12":
        kns, kcs = [2, 3, 4, 12], [10, 16, 4, 12]
    elif case == "cache_misaligned":
        ptrs[1] = KC + 2
    rc, t = plan.write(kns, kcs, ptrs=tuple(ptrs), **kw)
    msg = _ffi.load().b200_last_error().decode()
    assert rc == status, (case, rc, msg)
    assert words in msg and _launches(t) == []


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

    stub = _Stub()
    attention.launch_kvcache(stub, _T([2, 4, 1]), _T([8, 16, 2, 64]), _T([8, 16, 2, 64]), _T([2], "i32"), _T([2, 4, 1, 64]))
    attention.kvcache_write(stub, _T([2, 1, 2, 64]), _T([2, 1, 2, 64]), _T([8, 16, 2]), _T([8, 16, 2, 64]), _T([2], "i32"))
    assert [e.status for e in stub.errors] == [INVALID, INVALID] and all("rank 4" in str(e) for e in stub.errors)


# ---------------------------------------------------------------------------------------------- kernels
def test_kvcache_kernels_use_wgmma_and_tma_and_do_not_spill():
    tool = _tool("cuobjdump")
    _ffi.load()
    cubin = ROOT / "cubecl_b200" / "build" / "attention_kv.cubin"
    out = subprocess.run([tool, "-res-usage", str(cubin)], capture_output=True, text=True, check=True).stdout
    funcs = re.findall(r"Function (\w+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)
    want = {f"attn_kv_{i}_d{d}_{o}" for i in ("bf16", "f16") for d in (64, 128) for o in (i, "f32")}
    want |= {f"attn_kv_combine_{o}" for o in ("bf16", "f16", "f32")} | {"attn_kv_write"}
    assert {f for f, *_ in funcs} == want
    for name, reg, stack, local in funcs:
        assert int(stack) == 0 and int(local) == 0, (name, stack, local)
    sass = subprocess.run([tool, "-sass", str(cubin)], capture_output=True, text=True, check=True).stdout
    for body in re.split(r"\n\s*Function : ", sass)[1:]:
        name = body.split()[0]
        if "combine" in name or "write" in name:
            continue
        n = 64 if "_d64_" in name else 128
        assert re.search(rf"HGMMA\.64x{n}x16\.F32\S* R\d+, R\d+, gdesc\[UR\d+\]\.tnspB", body), name   # O += P V, P in registers
        assert re.search(r"HGMMA\.64x64x16\.F32\S* R\d+, gdesc\[UR\d+\]", body), name                   # S = Q K^T
        assert "UTMALDG.4D" in body, name
