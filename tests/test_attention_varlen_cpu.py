"""CPU: the f64 varlen oracle (pinned to torch's CPU SDPA and autograd with explicit per-sequence boolean masks), and the
dry-run plans of b200_attention_varlen and b200_attention_varlen_backward: kernel names, the grids of all four launches, the
workspace, the maps of compact, fused-QKV and strided views, gathers, every refusal, zero extents, deferred Python errors, and
the varlen cubins' kernels (register-A wgmma, TMA, no spills)."""
import ctypes as C
import math
import re
import subprocess

import numpy as np
import pytest
import torch

import attention_varlen_oracle as vo
from cubecl_b200 import _ffi
from plan_context import PlanContext
from test_conv_cpu import ROOT, _tool

F32, F16, BF16, I8 = _ffi.F32, _ffi.F16, _ffi.BF16, _ffi.I8
Q, K, V, OUT, LSE, CUQ, CUK, DOUT, DQ, DK, DV = (0x10000000 * (i + 1) for i in range(11))
INVALID, UNSUPPORTED = 6, 7


# ---------------------------------------------------------------------------------------------- oracle
def _torch_ref(q, k, v, dout, cu_q, cu_k, scale, window):
    qt, kt, vt = (torch.tensor(t, requires_grad=True) for t in (q, k, v))
    g = q.shape[1] // k.shape[1]
    outs, lses = torch.zeros(q.shape, dtype=torch.float64), torch.full((q.shape[1], q.shape[0]), -math.inf, dtype=torch.float64)
    pieces = []
    for b in range(len(cu_q) - 1):
        qa, qb, ka, kb = cu_q[b], cu_q[b + 1], cu_k[b], cu_k[b + 1]
        mask = torch.from_numpy(vo.band_mask(qb - qa, kb - ka, window))
        qs = qt[qa:qb].transpose(0, 1)[None]
        ks, vs = (t[ka:kb].transpose(0, 1).repeat_interleave(g, dim=0)[None] for t in (kt, vt))
        s = scale * qs @ ks.transpose(-1, -2)
        s = s.masked_fill(~mask, -math.inf)
        lse = torch.logsumexp(s, dim=-1)
        p = torch.where(torch.isfinite(lse)[..., None], torch.exp(s - torch.where(torch.isfinite(lse), lse, 0)[..., None]), 0)
        o = (p @ vs)[0].transpose(0, 1)
        pieces.append((qa, qb, o, lse[0]))
    total = sum((o * torch.from_numpy(dout[qa:qb])).sum() for qa, qb, o, _ in pieces)
    total.backward()
    for qa, qb, o, lse in pieces:
        outs[qa:qb], lses[:, qa:qb] = o.detach(), lse.detach()
    return outs.numpy(), lses.numpy(), qt.grad.numpy(), kt.grad.numpy(), vt.grad.numpy()


@pytest.mark.parametrize("lens_q,lens_k,Hq,Hkv,window", [
    ([5, 0, 9, 3], [5, 0, 9, 3], 2, 2, (-1, -1)), ([5, 7, 9], [5, 7, 9], 4, 2, (-1, 0)),
    ([6, 3, 4], [2, 8, 4], 2, 1, (-1, 0)),     # Lq != Lk, bottom-right: rows that see nothing
    ([9, 12], [9, 15], 2, 2, (3, 0)), ([9, 12], [9, 15], 2, 2, (2, 2)), ([9, 12], [9, 15], 2, 2, (0, 3)),
])
def test_oracle_matches_torch_sdpa_and_autograd(lens_q, lens_k, Hq, Hkv, window):
    rng = np.random.default_rng(sum(lens_q) + 7 * sum(lens_k))
    cu_q, cu_k = np.concatenate([[0], np.cumsum(lens_q)]), np.concatenate([[0], np.cumsum(lens_k)])
    D, scale = 8, 0.4
    q, k, v = rng.standard_normal((cu_q[-1], Hq, D)), rng.standard_normal((cu_k[-1], Hkv, D)), rng.standard_normal((cu_k[-1], Hkv, D))
    dout = rng.standard_normal(q.shape)
    out, lse = vo.attention_varlen_f64(q, k, v, cu_q, cu_k, scale, window)
    dq, dk, dv = vo.attention_varlen_backward_f64(q, k, v, dout, cu_q, cu_k, scale, window)
    r_out, r_lse, r_dq, r_dk, r_dv = _torch_ref(q, k, v, dout, cu_q, cu_k, scale, window)
    for a, b in ((out, r_out), (dq, r_dq), (dk, r_dk), (dv, r_dv)):
        np.testing.assert_allclose(a, b, rtol=0, atol=1e-12)
    np.testing.assert_array_equal(np.isinf(lse), np.isinf(r_lse))
    np.testing.assert_allclose(lse[np.isfinite(lse)], r_lse[np.isfinite(r_lse)], rtol=1e-13, atol=1e-13)
    if lens_q[0] > lens_k[0]:   # bottom-right: the first Lq - Lk rows of sequence 0 see nothing
        assert np.all(np.isneginf(lse[:, :lens_q[0] - lens_k[0]])) and np.all(out[:lens_q[0] - lens_k[0]] == 0)


def test_band_mask_rules():
    assert (vo.band_mask(4, 4, (-1, 0)) == np.tril(np.ones((4, 4), bool))).all()
    assert (vo.band_mask(2, 5, (-1, 0)) == np.tril(np.ones((2, 5), bool), 3)).all()   # bottom-right
    assert vo.band_mask(6, 6, (1, 0)).sum() == 6 + 5
    assert vo.visible_pairs([4, 3], [4, 3], (-1, -1)) == 16 + 9


# ---------------------------------------------------------------------------------------------- dry-run plans
class Planner(PlanContext):
    def fwd(self, qs, ks, B, maxq, maxk, vs=None, outs=None, idt=BF16, odt=None, strides=(None, None, None, None),
            ptrs=(Q, K, V, CUQ, CUK, OUT), lse=0, scale=0.125, window=(-1, -1), null_args=False):
        vs = ks if vs is None else vs
        outs = qs if outs is None else outs
        odt = idt if odt is None else odt
        arr = lambda v: _ffi.u64_array(v) if v is not None else None  # noqa: E731
        args = _ffi.AttentionVarlenArgs(scale, window[0], window[1], maxq, maxk)
        rc = self.lib.b200_attention_varlen(self.ctx, None, idt, odt, ptrs[0], arr(qs), arr(strides[0]), ptrs[1], arr(ks), arr(strides[1]),
                                            ptrs[2], arr(vs), arr(strides[2]), ptrs[3], ptrs[4], B, ptrs[5], arr(outs), arr(strides[3]),
                                            lse, None if null_args else C.byref(args))
        return rc, self.text()

    def bwd(self, qs, ks, B, maxq, maxk, idt=BF16, odt=None, gdt=None, strides=None, window=(-1, -1), scale=0.125,
            ptrs=(Q, K, V, OUT, DOUT, LSE, CUQ, CUK, DQ, DK, DV)):
        odt = idt if odt is None else odt
        gdt = idt if gdt is None else gdt
        strides = strides or [None] * 8
        arr = lambda v: _ffi.u64_array(v) if v is not None else None  # noqa: E731
        args = _ffi.AttentionVarlenArgs(scale, window[0], window[1], maxq, maxk)
        ops = []
        for p, sh, st in zip(ptrs[:5], (qs, ks, ks, qs, qs), strides[:5]):
            ops += [p, arr(sh), arr(st)]
        ops += [ptrs[5], ptrs[6], ptrs[7], B]
        for p, sh, st in zip(ptrs[8:], (qs, ks, ks), strides[5:]):
            ops += [p, arr(sh), arr(st)]
        rc = self.lib.b200_attention_varlen_backward(self.ctx, None, idt, odt, gdt, *ops, C.byref(args))
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


@pytest.mark.parametrize("idt,tag", [(BF16, "bf16"), (F16, "f16")])
@pytest.mark.parametrize("D,bucket", [(8, 64), (40, 64), (64, 64), (72, 128), (128, 128)])
@pytest.mark.parametrize("f32", [False, True])
def test_kernel_names_and_grids(plan, idt, tag, D, bucket, f32):
    B, Hq, Hkv, Tq, Tk, maxq, maxk = 5, 8, 2, 3000, 2500, 1000, 700
    rc, t = plan.fwd([Tq, Hq, D], [Tk, Hkv, D], B, maxq, maxk, idt=idt, odt=F32 if f32 else idt)
    assert rc == 0, _ffi.load().b200_last_error()
    o = "f32" if f32 else tag
    assert _launches(t) == [(f"attn_fwd_varlen_{tag}_d{bucket}_{o}", str(8 * Hq * B), "384", str(1024 + 5 * 128 * bucket * 2 + 1024))]
    plan.text()
    rc, t = plan.bwd([Tq, Hq, D], [Tk, Hkv, D], B, maxq, maxk, idt=idt, odt=F32 if f32 else idt, gdt=F32 if f32 else idt)
    assert rc == 0, _ffi.load().b200_last_error()
    names = [(n, int(g), int(b)) for n, g, b, _ in _launches(t)]
    assert names == [(f"attn_bwd_varlen_delta_{tag}_{o}", 8 * 8 * Hq * B, 256), (f"attn_bwd_varlen_dq_{tag}_d{bucket}_{o}", 8 * Hq * B, 384),
                     (f"attn_bwd_varlen_dkdv_{tag}_d{bucket}_{o}", 6 * Hkv * B, 384)]
    (alloc,) = re.findall(r"alloc (\d+)", t)
    assert int(alloc) >= 2 * Hq * ((-(-Tq // 128) + B) * 128) * 4


def test_maps_of_compact_views(plan):
    Tq, Tk, Hq, Hkv, D = 300, 200, 8, 2, 128
    rc, t = plan.fwd([Tq, Hq, D], [Tk, Hkv, D], 3, 128, 128, odt=F32)
    assert rc == 0 and "gather" not in t
    mq, mk, mv, mo = _tmaps(t)
    assert mq[:2] == (2, (D, Tq, Hq, 1)) and mq[2][:2] == (2 * Hq * D, 2 * D) and mq[3] == (64, 128, 1, 1)
    assert mk[:2] == mv[:2] == (2, (D, Tk, Hkv, 1)) and mk[2][:2] == (2 * Hkv * D, 2 * D)
    assert mo[:2] == (4, (D, Tq, Hq, 1)) and mo[2][:2] == (4 * Hq * D, 4 * D) and mo[3] == (32, 64, 1, 1)


def test_fused_qkv_slices_and_strided_views_are_read_in_place(plan):
    T, H, D = 256, 4, 64
    fused = [3 * H * D, D, 1]          # q, k, v slices of a [T, 3, H, D] projection
    rc, t = plan.fwd([T, H, D], [T, H, D], 2, 128, 128, strides=(fused, fused, fused, None), ptrs=(Q, Q + 2 * H * D, Q + 4 * H * D, CUQ, CUK, OUT))
    assert rc == 0 and "gather" not in t
    assert [m[2][:2] for m in _tmaps(t)[:3]] == [(2 * 3 * H * D, 2 * D)] * 3
    head_major = [D, T * D, 1]         # a [H, T, D] tensor seen as [T, H, D]
    rc, t = plan.fwd([T, H, D], [T, H, D], 2, 128, 128, strides=(head_major, None, None, None))
    assert rc == 0 and "gather" not in t and _tmaps(t)[0][2][:2] == (2 * D, 2 * T * D)


@pytest.mark.parametrize("case", ["misaligned", "d_stride", "odd_stride"])
def test_views_a_map_cannot_read_are_gathered(plan, case):
    T, H, D = 256, 4, 64
    st, ptrs = [None] * 4, [Q, K, V, CUQ, CUK, OUT]
    if case == "misaligned":
        ptrs[0] = Q + 2
    elif case == "d_stride":
        st[0] = [H * D * 2, D * 2, 2]
    else:
        st[0] = [H * 68, 68, 1]
    rc, t = plan.fwd([T, H, D], [T, H, D], 2, 128, 128, strides=tuple(st), ptrs=tuple(ptrs))
    assert rc == 0, _ffi.load().b200_last_error()
    assert [n for n, *_ in _launches(t)] == ["gather_strided", "attn_fwd_varlen_bf16_d64_bf16"]
    assert _tmaps(t)[0][2][:2] == (2 * H * D, 2 * D)   # the q map reads the compact copy


@pytest.mark.parametrize("case,status,words", [
    ("head_dim", INVALID, "head dim"), ("v_shape", INVALID, "does not match"), ("gqa", INVALID, "multiple of Hkv"),
    ("hkv0", INVALID, "multiple of Hkv"), ("out_shape", INVALID, "out is"), ("window_left", INVALID, "window"),
    ("window_right", INVALID, "window"), ("max_neg", INVALID, "max_seqlen"), ("scale_inf", INVALID, "finite"),
    ("scale_nan", INVALID, "finite"), ("null_args", INVALID, "null"), ("null_q", INVALID, "null"), ("null_cu", INVALID, "null"),
    ("cu_align", INVALID, "aligned"), ("lse_align", INVALID, "aligned"), ("in_f32", UNSUPPORTED, "input dtype"),
    ("in_i8", UNSUPPORTED, "input dtype"), ("out_other", UNSUPPORTED, "output dtype"), ("d136", UNSUPPORTED, "head dim"),
    ("d12", UNSUPPORTED, "head dim"), ("dv", UNSUPPORTED, "v's head dim"), ("out_misaligned", UNSUPPORTED, "out"),
    ("huge", UNSUPPORTED, "2^31"), ("max_huge", UNSUPPORTED, "2^30"),
])
def test_forward_refusals(plan, case, status, words):
    qs, ks, B, maxq, maxk = [300, 4, 64], [200, 2, 64], 3, 128, 128
    kw, ptrs = {}, [Q, K, V, CUQ, CUK, OUT]
    if case == "head_dim":
        ks = [200, 2, 32]
    elif case == "v_shape":
        kw["vs"] = [100, 2, 64]
    elif case == "gqa":
        ks = [200, 3, 64]
    elif case == "hkv0":
        ks = [200, 0, 64]
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
    elif case == "scale_nan":
        kw["scale"] = math.nan
    elif case == "null_args":
        kw["null_args"] = True
    elif case == "null_q":
        ptrs[0] = 0
    elif case == "null_cu":
        ptrs[4] = 0
    elif case == "cu_align":
        ptrs[3] = CUQ + 2
    elif case == "lse_align":
        kw["lse"] = LSE + 2
    elif case == "in_f32":
        kw["idt"], kw["odt"] = F32, F32
    elif case == "in_i8":
        kw["idt"], kw["odt"] = I8, F32
    elif case == "out_other":
        kw["idt"], kw["odt"] = BF16, F16
    elif case == "d136":
        qs, ks = [300, 4, 136], [200, 2, 136]
    elif case == "d12":
        qs, ks = [300, 4, 12], [200, 2, 12]
    elif case == "dv":
        kw["vs"] = [200, 2, 32]
    elif case == "out_misaligned":
        ptrs[5] = OUT + 2
    elif case == "huge":
        qs = [1 << 31, 4, 64]
    elif case == "max_huge":
        maxq = 1 << 30
    rc, t = plan.fwd(qs, ks, B, maxq, maxk, ptrs=tuple(ptrs), **kw)
    msg = _ffi.load().b200_last_error().decode()
    assert rc == status, (case, rc, msg)
    assert words in msg, msg
    assert _launches(t) == [] and "gather" not in t


@pytest.mark.parametrize("case,status,words", [
    ("dq_shape", INVALID, "dq is"), ("null_lse", INVALID, "null"), ("grad_other", UNSUPPORTED, "grad dtype"),
    ("dk_misaligned", UNSUPPORTED, "dk needs"), ("window", INVALID, "window"),
])
def test_backward_refusals(plan, case, status, words):
    qs, ks = [300, 4, 64], [200, 2, 64]
    ptrs = [Q, K, V, OUT, DOUT, LSE, CUQ, CUK, DQ, DK, DV]
    kw = {}
    strides = [None] * 8
    if case == "dq_shape":
        lib = _ffi.load()
        arr = _ffi.u64_array
        args = _ffi.AttentionVarlenArgs(0.125, -1, -1, 128, 128)
        ops = []
        for p, sh in zip(ptrs[:5], (qs, ks, ks, qs, qs)):
            ops += [p, arr(sh), None]
        ops += [LSE, CUQ, CUK, 3, DQ, arr([300, 4, 32]), None, DK, arr(ks), None, DV, arr(ks), None]
        rc = lib.b200_attention_varlen_backward(plan.ctx, None, BF16, BF16, BF16, *ops, C.byref(args))
        t = plan.text()
    else:
        if case == "null_lse":
            ptrs[5] = 0
        elif case == "grad_other":
            kw["gdt"] = F16
        elif case == "dk_misaligned":
            ptrs[9] = DK + 2
        elif case == "window":
            kw["window"] = (-3, -1)
        rc, t = plan.bwd(qs, ks, 3, 128, 128, strides=strides, ptrs=tuple(ptrs), **kw)
    msg = _ffi.load().b200_last_error().decode()
    assert rc == status, (case, rc, msg)
    assert words in msg and _launches(t) == []


def test_zero_extents_launch_nothing(plan):
    for qs, B, maxq in (([300, 4, 64], 0, 128), ([0, 4, 64], 3, 128), ([300, 0, 64], 3, 128), ([300, 4, 64], 3, 0)):
        rc, t = plan.fwd(qs, [200, 2, 64], B, maxq, 128)
        assert rc == 0 and t == "", (qs, B, maxq, t)
    rc, t = plan.bwd([0, 4, 64], [0, 2, 64], 3, 0, 0)
    assert rc == 0 and t == ""
    # no query rows but keys: only dk / dv run (every key row of a sequence gets +0)
    rc, t = plan.bwd([0, 4, 64], [200, 2, 64], 3, 0, 128)
    assert rc == 0 and [n for n, *_ in _launches(t)] == ["attn_bwd_varlen_dkdv_bf16_d64_bf16"]
    # queries but no keys: delta and dq run (every row +0)
    rc, t = plan.bwd([300, 4, 64], [200, 2, 64], 3, 128, 0)
    assert rc == 0 and [n for n, *_ in _launches(t)] == ["attn_bwd_varlen_delta_bf16_bf16", "attn_bwd_varlen_dq_bf16_d64_bf16"]


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
    q, k = _T([30, 4, 64]), _T([20, 2, 64])
    attention.launch_varlen(stub, _T([30, 4]), k, k, _T([3], "i32"), _T([3], "i32"), 16, 16, q)
    attention.launch_varlen(stub, q, k, k, _T([3], "i64"), _T([3], "i32"), 16, 16, q)                      # not i32
    attention.launch_varlen(stub, q, k, k, _T([3], "i32"), _T([4], "i32"), 16, 16, q)                      # lengths differ
    attention.launch_varlen(stub, q, k, k, _T([3], "i32", contiguous=False), _T([3], "i32"), 16, 16, q)   # not compact
    attention.launch_varlen(stub, q, k, k, _T([3, 1], "i32"), _T([3, 1], "i32"), 16, 16, q)                # not 1-D
    attention.launch_varlen_backward(stub, q, k, k, q, q, _T([4, 30], "f32"), _T([3], "i32"), _T([3], "i32"), 16, 16, _T([30, 4]), k, k)
    assert [e.status for e in stub.errors] == [INVALID] * 6
    assert "rank 3" in str(stub.errors[0]) and all("cu_seqlens" in str(e) for e in stub.errors[1:5]) and "rank 3" in str(stub.errors[5])


# ---------------------------------------------------------------------------------------------- kernels
@pytest.mark.parametrize("cubin,kinds", [("attention_varlen", ("fwd",)), ("attention_varlen_bwd", ("dq", "dkdv", "delta"))])
def test_varlen_kernels_use_register_a_wgmma_and_tma_and_do_not_spill(cubin, kinds):
    tool = _tool("cuobjdump")
    _ffi.load()
    path = ROOT / "cubecl_b200" / "build" / f"{cubin}.cubin"
    out = subprocess.run([tool, "-res-usage", str(path)], capture_output=True, text=True, check=True).stdout
    funcs = re.findall(r"Function (\w+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)
    want = set()
    for kind in kinds:
        if kind == "delta":
            want |= {f"attn_bwd_varlen_delta_{i}_{o}" for i in ("bf16", "f16") for o in (i, "f32")}
        else:
            pfx = "attn_fwd_varlen" if kind == "fwd" else f"attn_bwd_varlen_{kind}"
            want |= {f"{pfx}_{i}_d{d}_{o}" for i in ("bf16", "f16") for d in (64, 128) for o in (i, "f32")}
    assert {f for f, *_ in funcs} == want
    for name, reg, stack, local in funcs:
        assert int(stack) == 0 and int(local) == 0, (name, stack, local)
    sass = subprocess.run([tool, "-sass", str(path)], capture_output=True, text=True, check=True).stdout
    for body in re.split(r"\n\s*Function : ", sass)[1:]:
        name = body.split()[0]
        if "delta" in name:
            continue
        n = 64 if "_d64_" in name else 128
        assert re.search(rf"HGMMA\.64x{n}x16\.F32\S* R\d+, R\d+, gdesc\[UR\d+\]\.tnspB", body), name   # register-A product
        assert "UTMALDG.4D" in body and "UTMASTG.4D" in body, name
