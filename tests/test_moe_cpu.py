"""CPU: the mixture-of-experts oracle (pinned to torch's CPU topk, stable argsort + bincount + cumsum, index_select and
weighted sums), the dry-run plans of the five b200_moe_* entry points (kernel names, grids, shared memory, launch counts)
for every dtype, every refusal and zero extent, the Python layer's deferred errors, and the moe cubin's resources and SASS."""
import ctypes as C
import re
import subprocess

import numpy as np
import pytest
import torch

import moe_oracle as mo
from cubecl_b200 import _ffi, moe
from plan_context import PlanContext
from qmatmul_oracle import fma_f32
from test_conv_cpu import ROOT, _tool

F32, F16, BF16, I32 = _ffi.F32, _ffi.F16, _ffi.BF16, _ffi.I32
DT = {F32: "f32", BF16: "bf16", F16: "f16"}
SRC, IDS, W, OFFS, ROW, SLOT, DST, BIAS = (0x10000000 * i for i in range(1, 9))
INVALID, UNSUPPORTED = 6, 7


# ---------------------------------------------------------------------------------------------- oracle vs torch
def _separated_logits(rng, T, E, step=1.0 / 64):
    """Every row a random permutation of distinct values: no two keys tie, in any dtype."""
    return np.stack([rng.permutation(E) for _ in range(T)]).astype(np.float32) * np.float32(step) - np.float32(E * step / 2)


@pytest.mark.parametrize("score", ["softmax", "sigmoid"])
@pytest.mark.parametrize("E,k", [(8, 2), (128, 8), (256, 8), (1024, 32)])
def test_route_oracle_matches_torch_topk(score, E, k):
    rng = np.random.default_rng(E + k)
    logits = _separated_logits(rng, 33, E)
    ids, w = mo.route(logits, k, score, renormalize=True)
    tl = torch.tensor(logits, dtype=torch.float64)
    s = torch.softmax(tl, dim=-1) if score == "softmax" else torch.sigmoid(tl)
    tw, tid = torch.topk(s, k, dim=-1)
    np.testing.assert_array_equal(ids, tid.numpy())
    np.testing.assert_allclose(w, (tw / tw.sum(-1, keepdim=True)).numpy(), rtol=1e-12)


def test_route_oracle_group_limited_matches_deepseek_recipe():
    # DeepSeek-V3: sigmoid scores, a correction bias on the selection only, 8 groups scored by their top-2 sum, top-4 groups
    rng = np.random.default_rng(3)
    T, E, k = 40, 256, 8
    logits = _separated_logits(rng, T, E, 1.0 / 32)
    bias = (rng.permutation(E).astype(np.float32) / np.float32(4096)).astype(np.float32)
    ids, w = mo.route(logits, k, "sigmoid", True, 8, 4, 2.5, bias)
    s = torch.sigmoid(torch.tensor(logits, dtype=torch.float64))
    choice = torch.tensor(mo.keys(logits, "sigmoid", bias), dtype=torch.float64)
    g = choice.view(T, 8, -1).topk(2, dim=-1)[0].sum(-1)
    gidx = g.topk(4, dim=-1)[1]
    mask = torch.zeros_like(g).scatter_(1, gidx, 1).unsqueeze(-1).expand(T, 8, E // 8).reshape(T, E)
    tid = choice.masked_fill(mask == 0, float("-inf")).topk(k, dim=-1)[1]
    tw = s.gather(1, tid)
    np.testing.assert_array_equal(ids, tid.numpy())
    np.testing.assert_allclose(w, (tw / tw.sum(-1, keepdim=True) * 2.5).numpy(), rtol=1e-12)


def test_route_oracle_ties_and_nan():
    logits = np.array([[1.0, 3.0, 3.0, np.nan, -np.inf, 0.0, -0.0, 3.0]], np.float32)
    ids, _ = mo.route(logits, 8, renormalize=False)
    assert ids[0].tolist() == [1, 2, 7, 0, 5, 6, 4, 3]      # ties to the lower index, -0 ties +0, NaN below -inf


@pytest.mark.parametrize("E", [1, 8, 128, 1024])
def test_plan_oracle_matches_torch_argsort(E):
    rng = np.random.default_rng(E)
    ids = rng.integers(-2, E + 2, (300, 4)).astype(np.int32)     # includes dropped ids on both sides
    offs, row_of, slot_of = mo.plan(ids, E)
    flat = torch.tensor(ids).reshape(-1)
    keep = (flat >= 0) & (flat < E)
    order = torch.argsort(torch.where(keep, flat, E), stable=True)[: int(keep.sum())]
    np.testing.assert_array_equal(offs, torch.cumsum(torch.bincount(flat[keep], minlength=E), 0).numpy())
    np.testing.assert_array_equal(slot_of[: len(order)], order.numpy())
    assert (slot_of[len(order):] == -1).all()
    np.testing.assert_array_equal(row_of.reshape(-1)[order.numpy()], np.arange(len(order)))
    assert (row_of.reshape(-1)[~keep.numpy()] == -1).all()


def test_permute_and_combine_oracles_match_torch():
    rng = np.random.default_rng(1)
    T, k, E, N = 50, 3, 6, 24
    ids = rng.integers(-1, E, (T, k)).astype(np.int32)
    offs, row_of, slot_of = mo.plan(ids, E)
    x = rng.standard_normal((T, N)).astype(np.float32)
    xs = mo.permute(x, slot_of, k, np.zeros((T * k, N), np.float32))
    kept = int(offs[-1])
    np.testing.assert_array_equal(xs[:kept], torch.index_select(torch.tensor(x), 0, torch.tensor(slot_of[:kept] // k)).numpy())
    assert not xs[kept:].any()
    w = rng.uniform(0, 1, (T, k)).astype(np.float32)
    y = mo.combine(xs, row_of, w)
    acc = np.zeros((T, N), np.float32)
    for j in range(k):
        live = row_of[:, j] >= 0
        acc = np.where(live[:, None], fma_f32(w[:, j:j + 1], xs[np.maximum(row_of[:, j], 0)], acc), acc)
    np.testing.assert_array_equal(y, acc)
    want = (torch.tensor(w, dtype=torch.float64)[:, :, None] * torch.tensor(x, dtype=torch.float64)[:, None, :]
            * torch.tensor(row_of >= 0)[:, :, None]).sum(1).numpy()
    np.testing.assert_allclose(y, want, rtol=1e-5, atol=1e-5)
    # without weights it is the permute's backward: every kept copy of x[t] summed
    np.testing.assert_allclose(mo.combine(xs, row_of), x * (row_of >= 0).sum(1, keepdims=True), rtol=1e-6)


def test_combine_backward_oracle_matches_autograd():
    rng = np.random.default_rng(2)
    T, k, R, N = 20, 2, 40, 16
    row_of = rng.permutation(R)[: T * k].reshape(T, k).astype(np.int32)
    row_of[3, 1] = -1
    ys = rng.integers(-4, 5, (R, N)).astype(np.float32)
    w = rng.integers(-3, 4, (T, k)).astype(np.float32)
    dy = rng.integers(-4, 5, (T, N)).astype(np.float32)
    tys = torch.tensor(ys, dtype=torch.float64, requires_grad=True)
    tw = torch.tensor(w, dtype=torch.float64, requires_grad=True)
    live = torch.tensor(row_of >= 0)
    y = (tw[:, :, None] * tys[torch.tensor(np.maximum(row_of, 0))] * live[:, :, None]).sum(1)
    y.backward(torch.tensor(dy, dtype=torch.float64))
    d_ys, d_w = mo.combine_backward(dy, ys, w, row_of)
    np.testing.assert_array_equal(d_w, tw.grad.numpy())
    used = np.isin(np.arange(R), row_of)
    np.testing.assert_array_equal(d_ys[used], tys.grad.numpy()[used])
    assert np.isnan(d_ys[~used]).all()


# ---------------------------------------------------------------------------------------------- dry-run plans
class Planner(PlanContext):
    def route(self, T, E, k, dt=F32, stride=None, bias=0, score=_ffi.MOE_SOFTMAX, renorm=1, n_group=0, topk_group=0, args=True,
              ptrs=(SRC, IDS, W)):
        a = _ffi.MoeRouteArgs(k, score, renorm, n_group, topk_group, 1.0)
        rc = self.lib.b200_moe_route(self.ctx, None, dt, ptrs[0], T, E, E if stride is None else stride, bias,
                                     C.byref(a) if args else None, ptrs[1], ptrs[2])
        return rc, self.text()

    def plan(self, T, k, E, ptrs=(IDS, OFFS, ROW, SLOT)):
        rc = self.lib.b200_moe_plan(self.ctx, None, ptrs[0], T, k, E, ptrs[1], ptrs[2], ptrs[3])
        return rc, self.text()

    def permute(self, T, k, row_bytes, src_pitch=None, dst_pitch=None, ptrs=(SRC, SLOT, DST)):
        rc = self.lib.b200_moe_permute(self.ctx, None, ptrs[0], row_bytes if src_pitch is None else src_pitch, ptrs[1], T, k,
                                       ptrs[2], row_bytes if dst_pitch is None else dst_pitch, row_bytes)
        return rc, self.text()

    def combine(self, T, k, N, R, a=BF16, b=BF16, w=W, strides=None, ptrs=(SRC, ROW, DST)):
        s = strides or (N, N)
        rc = self.lib.b200_moe_combine(self.ctx, None, a, b, ptrs[0], R, s[0], w, ptrs[1], T, k, N, ptrs[2], s[1])
        return rc, self.text()

    def backward(self, T, k, N, R, g=BF16, y=BF16, strides=None, ptrs=(SRC, 0x18000000, W, ROW, DST, 0x90000000)):
        s = strides or (N, N, N)
        rc = self.lib.b200_moe_combine_backward(self.ctx, None, g, y, ptrs[0], s[0], ptrs[1], R, s[1], ptrs[2], ptrs[3], T, k, N,
                                                ptrs[4], s[2], ptrs[5])
        return rc, self.text()


@pytest.fixture
def plan():
    with Planner() as p:
        yield p


def _launches(text):
    return re.findall(r"^launch (\S+) grid=\((\d+),(\d+),(\d+)\) block=(\d+) smem=(\d+) cluster=(\d+)$", text, flags=re.M)


@pytest.mark.parametrize("dt", [F32, BF16, F16])
@pytest.mark.parametrize("T,E,k,groups", [(1, 8, 2, 0), (4096, 128, 8, 0), (1001, 256, 8, 8), (3, 1024, 32, 0)])
def test_route_plan(plan, dt, T, E, k, groups):
    rc, t = plan.route(T, E, k, dt, bias=BIAS if groups else 0, score=_ffi.MOE_SIGMOID if groups else _ffi.MOE_SOFTMAX,
                       n_group=groups, topk_group=4 if groups else 0)
    assert rc == 0, _ffi.load().b200_last_error()
    score = "sigmoid" if groups else "softmax"
    assert t.splitlines()[0] == f"moe route t={T} e={E} k={k} score={score} bias={1 if groups else 0} groups={4 if groups else 0}/{groups}"
    assert _launches(t) == [(f"moe_route_{DT[dt]}", str((T + 3) // 4), "1", "1", "128", str(4 * (E + E // 2) * 4), "1")]


@pytest.mark.parametrize("T,k,E,ctas,warp_slots", [
    (1, 1, 1, 1, 256), (1000, 8, 128, 4, 256), (32768, 8, 256, 128, 256), (4096, 2, 1024, 4, 256), (2048, 1, 8, 1, 256),
    (262144, 8, 1024, 1024, 256),                 # 2^21 slots: the last size with 2048 slots per CTA
    (262144 * 8 + 1, 1, 256, 513, 512),           # one more slot: each warp takes 512, and the CTA count halves
    (1 << 20, 8, 1024, 1024, 1024), ((1 << 31) - 1, 1, 1024, 1024, 262144)])   # the table stays at <= 1024 CTAs (4 MiB)
def test_plan_plan(plan, T, k, E, ctas, warp_slots):
    rc, t = plan.plan(T, k, E)
    assert rc == 0, _ffi.load().b200_last_error()
    n = T * k
    assert ctas == -(-n // (8 * warp_slots))
    lines = t.splitlines()
    assert lines[0] == f"moe plan slots={n} e={E} ctas={ctas} warp_slots={warp_slots}"
    assert lines[1].startswith("alloc ") and E * ctas * 4 <= int(lines[1].split()[1]) <= 4 << 20
    smem = str(8 * E * 4)
    assert _launches(t) == [("moe_plan_histogram", str(ctas), "1", "1", "256", smem, "1"), ("moe_plan_scan", "1", "1", "1", "1024", "0", "1"),
                            ("moe_plan_scatter", str(ctas), "1", "1", "256", smem, "1")]


def test_plan_with_no_slots_writes_offs_only(plan):
    for T, k in ((0, 8), (16, 0)):
        rc, t = plan.plan(T, k, 64)
        assert rc == 0
        assert t.splitlines()[0] == "moe plan slots=0 e=64 ctas=0 warp_slots=256" and "alloc" not in t
        assert _launches(t) == [("moe_plan_scan", "1", "1", "1", "1024", "0", "1")]


@pytest.mark.parametrize("row_bytes,src_pitch,dst_pitch,src,vec", [
    (8192, 8192, 8192, SRC, 16),            # bf16 activations, K = 4096
    (7168, 7168, 7168, SRC, 16),            # fp8 codes, K = 7168
    (224, 224, 224, SRC, 16),               # f32 block scales of K = 7168 / 128
    (56, 56, 56, SRC, 4),                   # ue8m0 scales of K = 1792 / 32
    (8192, 8200, 8192, SRC, 4),             # pitched source
    (8192, 8192, 8192, SRC + 2, 1),         # a misaligned base
    (30, 30, 30, SRC, 1),
])
def test_permute_plan(plan, row_bytes, src_pitch, dst_pitch, src, vec):
    rc, t = plan.permute(1000, 4, row_bytes, src_pitch, dst_pitch, ptrs=(src, SLOT, DST))
    assert rc == 0, _ffi.load().b200_last_error()
    assert t.splitlines()[0] == f"moe permute rows=4000 row_bytes={row_bytes} vec={vec}"
    assert _launches(t) == [(f"moe_permute_v{vec}", "500", "1", "1", "256", "0", "1")]


@pytest.mark.parametrize("a", [F32, BF16, F16])
@pytest.mark.parametrize("b", [F32, BF16, F16])
def test_combine_plans(plan, a, b):
    T, k, N, R = 3000, 8, 4096, 24000
    rc, t = plan.combine(T, k, N, R, a, b)
    assert rc == 0, _ffi.load().b200_last_error()
    assert t.splitlines()[0] == f"moe combine t={T} k={k} n={N} rows={R} weights=1 vec=1"
    assert _launches(t) == [(f"moe_combine_{DT[a]}_{DT[b]}", str(T), "2", "1", "256", "0", "1")]
    rc, t = plan.backward(T, k, N, R, a, b)
    assert rc == 0, _ffi.load().b200_last_error()
    assert t.splitlines()[0] == f"moe combine_backward t={T} k={k} n={N} rows={R} vec=1"
    assert _launches(t) == [(f"moe_combine_bwd_{DT[a]}_{DT[b]}", str(T), "1", "1", "256", str(N * 4), "1")]


def test_combine_vector_rule(plan):
    assert "vec=1" in plan.combine(10, 2, 7168, 20, w=0)[1] and "weights=0" in plan.combine(10, 2, 64, 20, w=0)[1]
    assert "vec=0" in plan.combine(10, 2, 100, 20)[1]                          # n % 8 != 0
    assert "vec=0" in plan.combine(10, 2, 64, 20, strides=(68, 64))[1]         # a row stride of 136 bytes
    assert "vec=0" in plan.combine(10, 2, 64, 20, ptrs=(SRC + 2, ROW, DST))[1]
    assert "vec=1" in plan.combine(10, 2, 64, 20, strides=(72, 64))[1]         # 144-byte rows stay 16-byte aligned
    assert "vec=0" in plan.backward(10, 2, 64, 20, strides=(64, 64, 68))[1]
    assert _launches(plan.combine(10, 2, 6000, 20)[1])[0][2] == "3"            # column chunks of 2048


def test_zero_extents_are_no_ops(plan):
    for rc, t in (plan.route(0, 8, 2), plan.permute(0, 4, 64), plan.permute(10, 0, 64), plan.permute(10, 4, 0),
                  plan.combine(0, 2, 64, 8), plan.combine(4, 2, 0, 8), plan.backward(0, 2, 64, 8), plan.backward(4, 2, 0, 8),
                  plan.backward(4, 0, 64, 8)):
        assert rc == 0 and "launch" not in t, t
    rc, t = plan.combine(4, 0, 64, 8)                       # k = 0: y = +0 is still written
    assert rc == 0 and _launches(t)[0][0] == "moe_combine_bf16_bf16"
    rc, t = plan.combine(4, 2, 64, 0)                       # no rows: every slot is dropped, y = +0
    assert rc == 0 and len(_launches(t)) == 1


REFUSALS = [
    ("route", dict(T=8, E=8, k=2, args=False), INVALID, "null args"),
    ("route", dict(T=8, E=8, k=2, dt=I32), UNSUPPORTED, "dtype"),
    ("route", dict(T=8, E=0, k=1), INVALID, "no experts"),
    ("route", dict(T=8, E=1025, k=2), UNSUPPORTED, "limit of 1024"),
    ("route", dict(T=1 << 31, E=8, k=2), UNSUPPORTED, "2^31"),
    ("route", dict(T=8, E=8, k=0), INVALID, "k = 0"),
    ("route", dict(T=8, E=8, k=9), INVALID, "k = 9"),
    ("route", dict(T=8, E=64, k=33), INVALID, "k = 33"),
    ("route", dict(T=8, E=8, k=2, score=2), INVALID, "unknown score"),
    ("route", dict(T=8, E=12, k=2, n_group=8, topk_group=4), INVALID, "groups of at least 2"),
    ("route", dict(T=8, E=8, k=2, n_group=8, topk_group=4), INVALID, "groups of at least 2"),
    ("route", dict(T=8, E=64, k=8, n_group=8, topk_group=0), INVALID, "topk_group"),
    ("route", dict(T=8, E=64, k=8, n_group=8, topk_group=9), INVALID, "topk_group"),
    ("route", dict(T=8, E=64, k=17, n_group=8, topk_group=2), INVALID, "topk_group"),
    ("route", dict(T=8, E=64, k=2, n_group=-1), INVALID, "negative"),
    ("route", dict(T=8, E=64, k=2, stride=63), INVALID, "stride"),
    ("route", dict(T=8, E=64, k=2, ptrs=(0, IDS, W)), INVALID, "null device pointer"),
    ("route", dict(T=8, E=64, k=2, ptrs=(SRC, IDS, 0)), INVALID, "null device pointer"),
    ("route", dict(T=8, E=64, k=2, ptrs=(SRC, IDS + 2, W)), INVALID, "misaligned"),
    ("route", dict(T=8, E=64, k=2, dt=BF16, ptrs=(SRC + 1, IDS, W)), INVALID, "misaligned"),
    ("route", dict(T=8, E=64, k=2, bias=BIAS + 2), INVALID, "misaligned"),
    ("plan", dict(T=8, k=2, E=0), INVALID, "no experts"),
    ("plan", dict(T=8, k=2, E=1025), UNSUPPORTED, "limit of 1024"),
    ("plan", dict(T=1 << 28, k=8, E=8), UNSUPPORTED, "2^31"),
    ("plan", dict(T=8, k=2, E=8, ptrs=(IDS, 0, ROW, SLOT)), INVALID, "null device pointer"),
    ("plan", dict(T=8, k=2, E=8, ptrs=(0, OFFS, ROW, SLOT)), INVALID, "null device pointer"),
    ("plan", dict(T=8, k=2, E=8, ptrs=(IDS, OFFS, ROW, 0)), INVALID, "null device pointer"),
    ("plan", dict(T=8, k=2, E=8, ptrs=(IDS, OFFS + 2, ROW, SLOT)), INVALID, "misaligned"),
    ("permute", dict(T=1 << 28, k=8, row_bytes=16), UNSUPPORTED, "2^31"),
    ("permute", dict(T=8, k=2, row_bytes=1 << 31), UNSUPPORTED, "row_bytes must be below 2^31"),
    ("permute", dict(T=8, k=2, row_bytes=64, src_pitch=32), INVALID, "pitches"),
    ("permute", dict(T=8, k=2, row_bytes=64, dst_pitch=32), INVALID, "pitches"),
    ("permute", dict(T=8, k=2, row_bytes=64, ptrs=(0, SLOT, DST)), INVALID, "null device pointer"),
    ("permute", dict(T=8, k=2, row_bytes=64, ptrs=(SRC, SLOT + 1, DST)), INVALID, "misaligned"),
    ("combine", dict(T=8, k=2, N=64, R=16, a=I32), UNSUPPORTED, "dtypes"),
    ("combine", dict(T=8, k=2, N=64, R=16, b=_ffi.F8E4M3), UNSUPPORTED, "dtypes"),
    ("combine", dict(T=1 << 31, k=1, N=64, R=16), UNSUPPORTED, "2^31"),
    ("combine", dict(T=8, k=2, N=65535 * 2048 + 1, R=16), UNSUPPORTED, "exceeds 134215680"),
    ("combine", dict(T=8, k=2, N=64, R=16, strides=(63, 64)), INVALID, "row stride"),
    ("combine", dict(T=8, k=2, N=64, R=16, strides=(64, 32)), INVALID, "row stride"),
    ("combine", dict(T=8, k=2, N=64, R=16, ptrs=(SRC, 0, DST)), INVALID, "null device pointer"),
    ("combine", dict(T=8, k=2, N=64, R=16, ptrs=(SRC + 1, ROW, DST)), INVALID, "misaligned"),
    ("combine", dict(T=8, k=2, N=64, R=16, w=W + 2), INVALID, "misaligned"),
    ("backward", dict(T=8, k=2, N=64, R=16, g=I32), UNSUPPORTED, "dtypes"),
    ("backward", dict(T=8, k=2, N=32769, R=16), UNSUPPORTED, "exceeds 32768"),
    ("backward", dict(T=8, k=2, N=64, R=16, strides=(64, 64, 63)), INVALID, "row stride"),
    ("backward", dict(T=8, k=2, N=64, R=16, ptrs=(SRC, 0x18000000, 0, ROW, DST, 0x90000000)), INVALID, "null device pointer"),
    ("backward", dict(T=8, k=2, N=64, R=16, ptrs=(SRC, 0x18000000, W, ROW, DST, 0)), INVALID, "null device pointer"),
    ("backward", dict(T=8, k=2, N=64, R=16, ptrs=(SRC, 0x18000000, W, ROW, DST + 1, 0x90000000)), INVALID, "misaligned"),
]


@pytest.mark.parametrize("case", range(len(REFUSALS)))
def test_refusals(plan, case):
    entry, kw, status, words = REFUSALS[case]
    rc, t = getattr(plan, entry)(**kw)
    msg = _ffi.load().b200_last_error().decode()
    assert rc == status, (case, rc, msg)
    assert words in msg and "launch" not in t, (case, msg, t)


# ---------------------------------------------------------------------------------------------- Python layer
def test_python_layer_defers_errors():
    class _Stub:
        def __init__(self):
            self.errors = []

        def _defer(self, e):
            self.errors.append(e)

    class _T:
        def __init__(self, shape, dtype="bf16", strides=None):
            self.shape, self.dtype = list(shape), dtype
            self.strides = strides or [int(np.prod(shape[i + 1:])) for i in range(len(shape))]

        def is_contiguous(self):
            return self.strides == [int(np.prod(self.shape[i + 1:])) for i in range(len(self.shape))]

    s = _Stub()
    logits, ids, w = _T([16, 8], "f32"), _T([16, 2], "i32"), _T([16, 2], "f32")
    moe.route(s, _T([16, 8, 1], "f32"), ids, w, 2)                         # logits not 2-D
    moe.route(s, logits, ids, w, 2, score="relu")                           # unknown score
    moe.route(s, logits, _T([16, 3], "i32"), w, 2)                          # ids not [T, k]
    moe.route(s, logits, ids, _T([16, 2], "bf16"), 2)                       # weights not f32
    moe.route(s, logits, ids, w, 2, bias=_T([7], "f32"))                    # bias not [E]
    moe.plan(s, _T([16, 2], "i64"), 8, _T([8], "i32"), ids, _T([32], "i32"))    # ids not i32
    moe.plan(s, ids, 8, _T([7], "i32"), ids, _T([32], "i32"))               # offs not [E]
    moe.plan(s, ids, 8, _T([8], "i32"), ids, _T([31], "i32"))               # slot_of not [T * k]
    x, slot = _T([16, 64]), _T([32], "i32")
    moe.permute(s, x, slot, 2, _T([32, 64], "f16"))                         # dst dtype
    moe.permute(s, x, slot, 2, _T([31, 64]))                                # dst rows
    moe.permute(s, _T([16, 64], strides=[64, 2]), slot, 2, _T([32, 64]))   # column stride
    ys, row_of, y = _T([32, 64]), _T([16, 2], "i32"), _T([16, 64])
    moe.combine(s, ys, row_of, _T([16, 32]))                                # y not [T, N]
    moe.combine(s, ys, _T([16, 2], "i64"), y)                               # row_of not i32
    moe.combine(s, ys, row_of, y, weights=_T([16, 2], "bf16"))              # weights not f32
    moe.combine_backward(s, y, ys, w, row_of, _T([32, 64], "f32"), w)       # d_ys not in dy's dtype
    moe.combine_backward(s, y, ys, w, row_of, ys, _T([16, 3], "f32"))       # d_w not [T, k]
    assert [e.status for e in s.errors] == [INVALID] * 16
    msgs = [str(e) for e in s.errors]
    for i, word in enumerate(["logits", "score", "ids", "weights", "bias", "ids", "offs", "slot_of", "dst", "dst", "src", "y",
                              "row_of", "weights", "d_ys", "d_w"]):
        assert word in msgs[i], (i, msgs[i])


# ---------------------------------------------------------------------------------------------- kernels
KERNELS = ({f"moe_route_{d}" for d in ("f32", "bf16", "f16")} | {"moe_plan_histogram", "moe_plan_scan", "moe_plan_scatter"}
           | {f"moe_permute_v{v}" for v in (1, 4, 16)}
           | {f"moe_combine_{a}_{b}" for a in ("f32", "bf16", "f16") for b in ("f32", "bf16", "f16")}
           | {f"moe_combine_bwd_{a}_{b}" for a in ("f32", "bf16", "f16") for b in ("f32", "bf16", "f16")})


def test_moe_kernels_do_not_spill_and_use_no_atomics():
    tool = _tool("cuobjdump")
    _ffi.load()
    cubin = ROOT / "cubecl_b200" / "build" / "moe.cubin"
    out = subprocess.run([tool, "-res-usage", str(cubin)], capture_output=True, text=True, check=True).stdout
    funcs = re.findall(r"Function (\w+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)
    assert {f for f, *_ in funcs} == KERNELS and len(KERNELS) == 27
    for name, reg, stack, local in funcs:
        assert int(stack) == 0 and int(local) == 0, (name, stack, local)
    sass = subprocess.run([tool, "-sass", str(cubin)], capture_output=True, text=True, check=True).stdout
    bodies = {b.split()[0]: b for b in re.split(r"\n\s*Function : ", sass)[1:]}
    assert set(bodies) == KERNELS
    for name, body in bodies.items():
        assert not re.search(r"\b(ATOM|ATOMS|ATOMG|RED|REDG)\b", body), name          # no atomics of any kind
        assert not re.search(r"\b(LDL|STL)\b", body), name                              # no local memory
    assert "MATCH.ANY" in bodies["moe_plan_scatter"] and "MATCH.ANY" in bodies["moe_plan_histogram"]
    assert "LDG.E.128" in bodies["moe_permute_v16"] and "STG.E.128" in bodies["moe_permute_v16"]
    assert "LDG.E.128" in bodies["moe_combine_bf16_bf16"] and "STG.E.128" in bodies["moe_combine_bf16_bf16"]
