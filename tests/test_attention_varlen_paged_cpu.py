"""CPU: paged variable-length attention (b200_attention_varlen_paged).

- The f64 oracle is a gather of each sequence's pages followed by the varlen oracle; it is pinned to torch's SDPA with explicit
  per-sequence masks (causal_lower_right and window masks), with stale NaN and inf in unused slots and pages, and empty
  sequences (Lq = 0 and Lk = 0).
- Dry-run plans: kernel names, grids and shared memory; the map order, dims and boxes for every page size, no table and a
  head-major cache; a misaligned q is gathered while a misaligned cache or out is refused; every refusal; zero extents; the
  host reads no device array (a plan holds only alloc, tmap and launch lines).
- The Python entry points defer errors to sync(); the attention_paged kernels do not spill."""
import ctypes as C
import math
import re
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from torch.nn.attention.bias import causal_lower_right

import attention_varlen_oracle as vo
from cubecl_b200 import _ffi
from plan_context import PlanContext
from test_conv_cpu import ROOT, _tool

F32, F16, BF16 = _ffi.F32, _ffi.F16, _ffi.BF16
Q, KC, VC, BT, CUQ, SEQ, OUT, LSE = (0x10000000 * (i + 1) for i in range(8))
INVALID, UNSUPPORTED = 6, 7


# ---------------------------------------------------------------------------------------------- oracle
def cache_lengths(seqlens, max_k, cap):
    """Lk_b = clamp(cache_seqlens[b], 0, min(max_seqlen_k, capacity))"""
    return [int(min(max(int(s), 0), max_k, cap)) for s in seqlens]


def gather_pages(k_cache, v_cache, table, lens):
    """The keys and values of every sequence packed contiguously: k_cache, v_cache [P, page, Hkv, D], table [B, max_pages] (None:
    page b), lens the Lk_b -> (k [sum Lk, Hkv, D], v, cu_k)"""
    page = k_cache.shape[1]
    ks, vs = [], []
    for b, L in enumerate(lens):
        rows = [(table[b, j // page] if table is not None else b, j % page) for j in range(L)]
        ks.append(np.stack([k_cache[p, r] for p, r in rows]) if rows else k_cache[:0, 0])
        vs.append(np.stack([v_cache[p, r] for p, r in rows]) if rows else v_cache[:0, 0])
    cu_k = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    return np.concatenate(ks), np.concatenate(vs), cu_k


def attention_varlen_paged_f64(q, k_cache, v_cache, table, seqlens, cu_q, max_k, scale=None, window=(-1, -1), fill=0.0):
    """-> (out [Tq, Hq, D], lse [Hq, Tq]) in float64: the varlen oracle on the gathered keys"""
    cap = k_cache.shape[1] * (table.shape[1] if table is not None else 1)
    k, v, cu_k = gather_pages(np.asarray(k_cache, np.float64), np.asarray(v_cache, np.float64), table, cache_lengths(seqlens, max_k, cap))
    return vo.attention_varlen_f64(q, k, v, cu_q, cu_k, scale, window, fill)


def _sdpa_ref(q, k_cache, v_cache, table, lens, cu_q, scale, window):
    """torch SDPA per sequence with an explicit mask built from page lookups; rows that see no key are left NaN"""
    page, g = k_cache.shape[1], q.shape[1] // k_cache.shape[2]
    out = np.full(q.shape, np.nan)
    for b, Lk in enumerate(lens):
        qa, qb = int(cu_q[b]), int(cu_q[b + 1])
        Lq = qb - qa
        if Lq == 0:
            continue
        idx = [(table[b, j // page] if table is not None else b, j % page) for j in range(Lk)]
        kk = torch.tensor(np.stack([k_cache[p, r] for p, r in idx]) if idx else np.zeros((0,) + k_cache.shape[2:]))
        vv = torch.tensor(np.stack([v_cache[p, r] for p, r in idx]) if idx else np.zeros((0,) + v_cache.shape[2:]))
        qs = torch.tensor(q[qa:qb]).transpose(0, 1)[None]
        ks, vs = (t.transpose(0, 1).repeat_interleave(g, dim=0)[None] for t in (kk, vv))
        if window == (-1, 0):
            mask = causal_lower_right(Lq, Lk)
        else:
            i, j = torch.arange(Lq)[:, None], torch.arange(Lk)[None, :]
            mask = torch.ones(Lq, Lk, dtype=torch.bool)
            if window[0] >= 0:
                mask &= j >= i + (Lk - Lq) - window[0]
            if window[1] >= 0:
                mask &= j <= i + (Lk - Lq) + window[1]
        if Lk == 0:
            continue
        o = F.scaled_dot_product_attention(qs, ks, vs, attn_mask=mask, scale=scale)
        out[qa:qb] = o[0].transpose(0, 1).numpy()
    return out


def _paged_problem(rng, lens_q, lens_k, Hq, Hkv, D, page, max_pages, table=True, stale="nan"):
    """Shuffled pages plus two pages no sequence owns; slots at or past Lk and unused pages hold NaN / +-inf"""
    B = len(lens_q)
    P = B * max_pages + 2 if table else B
    def stale_fill(shape):
        return np.full(shape, np.nan) if stale == "nan" else np.where(rng.random(shape) < 0.5, np.inf, -np.inf)
    k_cache, v_cache = stale_fill((P, page, Hkv, D)), stale_fill((P, page, Hkv, D))
    perm = rng.permutation(P)
    tbl = perm[:B * max_pages].reshape(B, max_pages).astype(np.int32) if table else None
    for b, L in enumerate(lens_k):
        for j in range(L):
            p = tbl[b, j // page] if table else b
            k_cache[p, j % page] = rng.standard_normal((Hkv, D))
            v_cache[p, j % page] = rng.standard_normal((Hkv, D))
    cu_q = np.concatenate([[0], np.cumsum(lens_q)]).astype(np.int64)
    q = rng.standard_normal((int(cu_q[-1]), Hq, D))
    return q, k_cache, v_cache, tbl, cu_q


@pytest.mark.parametrize("lens_q,lens_k,page,window", [
    ([5, 0, 9, 3], [12, 0, 9, 20], 4, (-1, 0)),       # chunked prefill; an empty sequence
    ([6, 3, 4], [2, 8, 0], 8, (-1, 0)),               # Lq > Lk: rows that see nothing; Lk = 0 with queries
    ([9, 12], [17, 15], 4, (3, 0)), ([9, 12], [17, 15], 8, (2, 2)), ([9, 0, 12], [17, 3, 15], 4, (-1, -1)),
])
@pytest.mark.parametrize("stale", ["nan", "inf"])
@pytest.mark.filterwarnings("ignore:Lower right causal bias")   # torch's warning for Lq > Lk rows: those are compared apart
def test_oracle_matches_torch_sdpa(lens_q, lens_k, page, window, stale):
    rng = np.random.default_rng(sum(lens_q) + 7 * sum(lens_k) + page)
    Hq, Hkv, D, scale = 4, 2, 8, 0.3
    max_pages = -(-max(lens_k) // page) + 1
    q, kc, vc, tbl, cu_q = _paged_problem(rng, lens_q, lens_k, Hq, Hkv, D, page, max_pages, stale=stale)
    seqlens = np.array(lens_k)
    out, lse = attention_varlen_paged_f64(q, kc, vc, tbl, seqlens, cu_q, max(lens_k), scale, window)
    ref = _sdpa_ref(q, kc, vc, tbl, lens_k, cu_q, scale, window)
    seen = np.isfinite(lse).T        # [Tq, Hq]: rows with a visible key
    assert np.all(np.isfinite(out)), "stale slots reached the oracle's output"
    np.testing.assert_allclose(out[seen], ref[seen], rtol=0, atol=1e-12)
    assert np.all(out[~seen] == 0)
    if window == (-1, 0) and lens_q[0] > lens_k[0]:   # bottom-right: the first Lq - Lk rows of sequence 0 see nothing
        assert np.all(np.isneginf(lse[:, :lens_q[0] - lens_k[0]]))


def test_lengths_clamp_to_max_seqlen_k_and_capacity():
    assert cache_lengths([-3, 5, 70, 40], 50, 64) == [0, 5, 50, 40]
    assert cache_lengths([100], 1000, 64) == [64]


def test_oracle_is_the_varlen_oracle_on_gathered_keys():
    rng = np.random.default_rng(3)
    lens_q, lens_k, page = [3, 5], [7, 13], 4
    q, kc, vc, tbl, cu_q = _paged_problem(rng, lens_q, lens_k, 2, 1, 8, page, 4, stale="inf")
    k, v, cu_k = gather_pages(kc, vc, tbl, lens_k)
    assert k.shape == (20, 1, 8) and list(cu_k) == [0, 7, 20] and np.all(np.isfinite(k))
    got = attention_varlen_paged_f64(q, kc, vc, tbl, lens_k, cu_q, 100, None, (-1, 0))
    want = vo.attention_varlen_f64(q, k, v, cu_q, cu_k, None, (-1, 0))
    for a, b in zip(got, want):
        np.testing.assert_array_equal(a, b)


# ---------------------------------------------------------------------------------------------- dry-run plans
class Planner(PlanContext):
    def fwd(self, qs, kcs, B, maxq, maxk, bts=None, vcs=None, outs=None, idt=BF16, odt=None, strides=(None, None, None, None),
            bt_strides=None, ptrs=(Q, KC, VC, BT, CUQ, SEQ, OUT), lse=0, scale=0.125, window=(-1, -1), null_args=False, table=True):
        vcs = kcs if vcs is None else vcs
        outs = qs if outs is None else outs
        odt = idt if odt is None else odt
        bts = [B, 4] if bts is None else bts
        arr = lambda v: _ffi.u64_array(v) if v is not None else None  # noqa: E731
        args = _ffi.AttentionVarlenArgs(scale, window[0], window[1], maxq, maxk)
        bt = (ptrs[3], arr(bts), arr(bt_strides)) if table else (0, None, None)
        rc = self.lib.b200_attention_varlen_paged(
            self.ctx, None, idt, odt, ptrs[0], arr(qs), arr(strides[0]), ptrs[1], arr(kcs), arr(strides[1]), ptrs[2], arr(vcs),
            arr(strides[2]), *bt, ptrs[4], ptrs[5], B, ptrs[6], arr(outs), arr(strides[3]), lse, None if null_args else C.byref(args))
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


def _only_alloc_tmap_launch(t):
    """The host reads no device array (no copy, no sync): a plan is allocations, tensor maps and launches only"""
    assert all(re.match(r"(alloc|tmap4d|launch) ", line) for line in t.splitlines()), t


@pytest.mark.parametrize("idt,tag", [(BF16, "bf16"), (F16, "f16")])
@pytest.mark.parametrize("D,bucket", [(8, 64), (40, 64), (64, 64), (72, 128), (128, 128)])
@pytest.mark.parametrize("f32", [False, True])
def test_kernel_names_grids_and_shared_memory(plan, idt, tag, D, bucket, f32):
    B, Hq, Hkv, Tq, maxq, maxk = 5, 8, 2, 3000, 1000, 700
    rc, t = plan.fwd([Tq, Hq, D], [40, 64, Hkv, D], B, maxq, maxk, bts=[B, 16], idt=idt, odt=F32 if f32 else idt)
    assert rc == 0, _ffi.load().b200_last_error()
    o = "f32" if f32 else tag
    assert _launches(t) == [(f"attn_fwd_paged_{tag}_d{bucket}_{o}", str(8 * Hq * B), "384", str(1024 + 5 * 128 * bucket * 2 + 1024))]
    _only_alloc_tmap_launch(t)


@pytest.mark.parametrize("page,rows", [(16, 16), (32, 32), (64, 64), (128, 128), (192, 64), (256, 128)])
def test_maps_of_paged_caches(plan, page, rows):
    Tq, Hq, Hkv, D, B, P = 300, 8, 2, 128, 3, 40
    rc, t = plan.fwd([Tq, Hq, D], [P, page, Hkv, D], B, 128, 4096, bts=[B, 8], odt=F32)
    assert rc == 0, _ffi.load().b200_last_error()
    assert "gather" not in t
    mq, mk, mv, mo = _tmaps(t)
    assert mq == (2, (D, Tq, Hq, 1), (2 * Hq * D, 2 * D, 2 * Tq * Hq * D), (64, 128, 1, 1))
    assert mk == mv == (2, (D, page, Hkv, P), (2 * Hkv * D, 2 * D, 2 * page * Hkv * D), (64, rows, 1, 1))
    assert mo[:2] == (4, (D, Tq, Hq, 1)) and mo[3] == (32, 64, 1, 1)
    _only_alloc_tmap_launch(t)


@pytest.mark.parametrize("page", [40, 100, 1000])
def test_one_page_per_sequence_loads_128_rows(plan, page):
    Hkv, D, B = 2, 64, 3
    rc, t = plan.fwd([300, 4, D], [B, page, Hkv, D], B, 128, 4096, table=False)   # no table: page b is sequence b
    assert rc == 0, _ffi.load().b200_last_error()
    assert [m[3] for m in _tmaps(t)[1:3]] == [(64, 128, 1, 1)] * 2 and _tmaps(t)[1][1] == (D, page, Hkv, B)
    rc, t = plan.fwd([300, 4, D], [7, page, Hkv, D], B, 128, 4096, bts=[B, 1])    # a table of one page per sequence
    assert rc == 0 and [m[3] for m in _tmaps(t)[1:3]] == [(64, 128, 1, 1)] * 2


def test_head_major_cache_is_read_in_place(plan):
    P, page, Hkv, D, B = 30, 64, 4, 128, 3
    head_major = [Hkv * page * D, D, page * D, 1]   # a [P, Hkv, page, D] cache seen as [P, page, Hkv, D]
    rc, t = plan.fwd([300, 8, D], [P, page, Hkv, D], B, 128, 1024, strides=(None, head_major, head_major, None))
    assert rc == 0, _ffi.load().b200_last_error()
    assert "gather" not in t
    mk = _tmaps(t)[1]
    assert mk[1] == (D, page, Hkv, P) and mk[2] == (2 * D, 2 * page * D, 2 * Hkv * page * D) and mk[3] == (64, 64, 1, 1)


def test_misaligned_q_is_gathered(plan):
    T, H, D = 256, 4, 64
    rc, t = plan.fwd([T, H, D], [10, 32, 2, D], 2, 128, 256, ptrs=(Q + 2, KC, VC, BT, CUQ, SEQ, OUT))
    assert rc == 0, _ffi.load().b200_last_error()
    assert [n for n, *_ in _launches(t)] == ["gather_strided", "attn_fwd_paged_bf16_d64_bf16"]
    assert len(re.findall(r"^alloc ", t, re.M)) == 1
    assert _tmaps(t)[0][2][:2] == (2 * H * D, 2 * D)   # the q map reads the compact copy
    _only_alloc_tmap_launch(t)


@pytest.mark.parametrize("case,status,words", [
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
])
def test_refusals(plan, case, status, words):
    qs, kcs, B, maxq, maxk = [300, 4, 64], [10, 32, 2, 64], 2, 128, 256
    kw, ptrs = {}, [Q, KC, VC, BT, CUQ, SEQ, OUT]
    if case == "head_dim":
        kcs = [10, 32, 2, 32]
    elif case == "v_shape":
        kw["vcs"] = [10, 16, 2, 64]
    elif case == "gqa":
        kcs = [10, 32, 3, 64]
    elif case == "hkv0":
        kcs = [10, 32, 0, 64]
    elif case == "out_shape":
        kw["outs"] = [300, 2, 64]
    elif case == "window_left":
        kw["window"] = (-2, 0)
    elif case == "window_right":
        kw["window"] = (4, -5)
    elif case == "max_neg":
        maxk = -1
    elif case == "scale_inf":
        kw["scale"] = math.inf
    elif case == "null_args":
        kw["null_args"] = True
    elif case == "null_bt_shape":
        lib = _ffi.load()
        args = _ffi.AttentionVarlenArgs(0.125, -1, -1, maxq, maxk)
        arr = _ffi.u64_array
        rc = lib.b200_attention_varlen_paged(plan.ctx, None, BF16, BF16, Q, arr(qs), None, KC, arr(kcs), None, VC, arr(kcs), None, BT,
                                             None, None, CUQ, SEQ, B, OUT, arr(qs), None, 0, C.byref(args))
        msg = _ffi.load().b200_last_error().decode()
        assert rc == status and words in msg and plan.text() == "", msg
        return
    elif case == "null_q":
        ptrs[0] = 0
    elif case == "null_cu":
        ptrs[4] = 0
    elif case == "null_seqlens":
        ptrs[5] = 0
    elif case == "cu_align":
        ptrs[4] = CUQ + 2
    elif case == "seqlens_align":
        ptrs[5] = SEQ + 2
    elif case == "bt_align":
        ptrs[3] = BT + 2
    elif case == "lse_align":
        kw["lse"] = LSE + 2
    elif case == "empty_pages":
        kcs = [0, 32, 2, 64]
    elif case == "empty_page":
        kcs = [10, 0, 2, 64]
    elif case == "bt_rows":
        kw["bts"] = [3, 4]
    elif case == "bt_zero":
        kw["bts"] = [B, 0]
    elif case == "no_table_p":
        kw["table"] = False
    elif case == "in_f32":
        kw["idt"], kw["odt"] = F32, F32
    elif case == "out_other":
        kw["idt"], kw["odt"] = BF16, F16
    elif case == "d136":
        qs, kcs = [300, 4, 136], [10, 32, 2, 136]
    elif case == "dv":
        kw["vcs"] = [10, 32, 2, 32]
    elif case == "page_24":
        kcs = [10, 24, 2, 64]
    elif case == "page_96":
        kcs = [10, 96, 2, 64]
    elif case == "cache_misaligned":
        ptrs[1] = KC + 2
    elif case == "cache_stride":
        kw["strides"] = (None, None, [32 * 2 * 68, 2 * 68, 68, 1], None)   # v_cache rows of 68 elements: 136-byte strides
    elif case == "out_misaligned":
        ptrs[6] = OUT + 2
    elif case == "huge":
        qs = [1 << 31, 4, 64]
    elif case == "capacity":
        kw["bts"] = [B, 1 << 27]   # 2^27 pages of 32 keys
    elif case == "max_huge":
        maxq = 1 << 30
    elif case == "ctas":
        qs, B, maxq = [300, 1 << 16, 64], 1 << 13, (1 << 30) - 1   # 2^23 query blocks * 2^16 heads * 2^13 sequences
        kcs, kw["outs"] = [1 << 13, 32, 1 << 16, 64], [300, 1 << 16, 64]
        kw["bts"] = [B, 4]
    rc, t = plan.fwd(qs, kcs, B, maxq, maxk, ptrs=tuple(ptrs), **kw)
    msg = _ffi.load().b200_last_error().decode()
    assert rc == status, (case, rc, msg)
    assert words in msg, msg
    assert msg.startswith("attention_varlen_paged: "), msg
    assert _launches(t) == [] and "gather" not in t


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
    q, kc, cq, sl = _T([30, 4, 64]), _T([8, 16, 2, 64]), _T([3], "i32"), _T([2], "i32")
    attention.launch_varlen_paged(stub, _T([30, 4]), kc, kc, cq, sl, 16, 16, q)                                  # q rank
    attention.launch_varlen_paged(stub, q, _T([8, 16, 64]), kc, cq, sl, 16, 16, q)                               # cache rank
    attention.launch_varlen_paged(stub, q, _T([8, 16, 2, 64], "f8e4m3"), _T([8, 16, 2, 64], "f8e4m3"), cq, sl, 16, 16, q)   # fp8
    attention.launch_varlen_paged(stub, q, _T([8, 16, 2, 64], "f16"), kc, cq, sl, 16, 16, q)                      # dtypes differ
    attention.launch_varlen_paged(stub, q, kc, kc, _T([3], "i64"), sl, 16, 16, q)                                 # cu not i32
    attention.launch_varlen_paged(stub, q, kc, kc, _T([3], "i32", contiguous=False), sl, 16, 16, q)               # cu not compact
    attention.launch_varlen_paged(stub, q, kc, kc, _T([3, 1], "i32"), sl, 16, 16, q)                              # cu not 1-D
    attention.launch_varlen_paged(stub, q, kc, kc, cq, _T([3], "i32"), 16, 16, q)                                 # seqlens not [B]
    attention.launch_varlen_paged(stub, q, kc, kc, cq, _T([2], "i64"), 16, 16, q)                                 # seqlens not i32
    attention.launch_varlen_paged(stub, q, kc, kc, cq, _T([2], "i32", contiguous=False), 16, 16, q)               # not compact
    attention.launch_varlen_paged(stub, q, kc, kc, cq, sl, 16, 16, q, block_table=_T([2, 4], "i64"))              # table not i32
    attention.launch_varlen_paged(stub, q, kc, kc, cq, sl, 16, 16, q, lse=_T([30, 4], "f32"))                     # lse shape
    assert [e.status for e in stub.errors] == [INVALID, INVALID, UNSUPPORTED] + [INVALID] * 9
    msgs = [str(e) for e in stub.errors]
    assert all("attention_varlen_paged" in m for m in msgs)
    assert "rank 3" in msgs[0] and "rank 4" in msgs[1] and "fp8" in msgs[2] and "dtypes differ" in msgs[3]
    assert all("cu_seqlens_q" in m for m in msgs[4:7]) and all("cache_seqlens" in m for m in msgs[7:10])
    assert "block_table" in msgs[10] and "lse" in msgs[11]


# ---------------------------------------------------------------------------------------------- kernels
def test_paged_kernels_use_register_a_wgmma_and_tma_and_do_not_spill():
    tool = _tool("cuobjdump")
    _ffi.load()
    path = ROOT / "cubecl_b200" / "build" / "attention_paged.cubin"
    out = subprocess.run([tool, "-res-usage", str(path)], capture_output=True, text=True, check=True).stdout
    funcs = re.findall(r"Function (\w+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)
    want = {f"attn_fwd_paged_{i}_d{d}_{o}" for i in ("bf16", "f16") for d in (64, 128) for o in (i, "f32")}
    assert {f for f, *_ in funcs} == want
    for name, reg, stack, local in funcs:
        assert int(stack) == 0 and int(local) == 0, (name, stack, local)
        assert int(reg) <= 168, (name, reg)
    sass = subprocess.run([tool, "-sass", str(path)], capture_output=True, text=True, check=True).stdout
    for body in re.split(r"\n\s*Function : ", sass)[1:]:
        name = body.split()[0]
        n = 64 if "_d64_" in name else 128
        assert re.search(rf"HGMMA\.64x{n}x16\.F32\S* R\d+, R\d+, gdesc\[UR\d+\]\.tnspB", body), name   # register-A product
        assert "UTMALDG.4D" in body and "UTMASTG.4D" in body, name
