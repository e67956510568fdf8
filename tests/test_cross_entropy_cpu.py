"""CPU: the cross-entropy oracle (tests/cross_entropy_oracle.py) pinned to torch's F.cross_entropy and autograd in f64, the
exact cases' power to catch a wrong contract, the dry-run plans of b200_cross_entropy and b200_cross_entropy_backward (row
class, cluster size and access path, the same for any t; the count pre-launch and the total launch), every refusal and zero
extent, the in-place / partial-overlap rule, the Python layer's deferred errors, and the xent cubin's resources and SASS."""
import ctypes as C
import re
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import cross_entropy_oracle as xo
from cubecl_b200 import _ffi, cross_entropy as xent
from plan_context import PlanContext
from test_conv_cpu import ROOT, _tool

F32, F16, BF16, I32, I64 = _ffi.F32, _ffi.F16, _ffi.BF16, _ffi.I32, _ffi.I64
DT = {F32: "f32", BF16: "bf16", F16: "f16"}
X, Y, L, S, DL, G = ((1 << 40) * i for i in range(1, 7))   # far apart: no [t, v] extent overlaps another
INVALID, UNSUPPORTED = 6, 7


# ---------------------------------------------------------------------------------------------- oracle vs torch
@pytest.mark.parametrize("reduction", xo.REDUCTIONS)
@pytest.mark.parametrize("eps", [0.0, 0.1, 1.0])
@pytest.mark.parametrize("v", [1, 7, 1000, 5000])
def test_oracle_matches_torch_cross_entropy(v, eps, reduction):
    rng = np.random.default_rng(v)
    T = 37
    x = (rng.standard_normal((T, v)) * 3).astype(np.float32)
    y = rng.integers(0, v, size=T)
    y[::5] = -100
    out = xo.forward(x, y, reduction, -100, eps)[0]
    ref = F.cross_entropy(torch.tensor(x, dtype=torch.float64), torch.tensor(y), reduction=reduction, label_smoothing=eps).numpy()
    np.testing.assert_allclose(out, ref, rtol=1e-5, atol=2e-5 * max(1, np.log(v)))


@pytest.mark.parametrize("reduction", xo.REDUCTIONS)
@pytest.mark.parametrize("eps,z", [(0.0, 0.0), (0.1, 0.0), (0.0, 1e-3), (0.2, 1e-2)])
def test_oracle_gradient_matches_autograd_with_z_loss(eps, z, reduction):
    rng = np.random.default_rng(int(eps * 10 + z * 1000))
    T, v = 29, 3000
    x = (rng.standard_normal((T, v)) * 2).astype(np.float32)
    y = rng.integers(0, v, size=T)
    y[::4] = -100
    xt = torch.tensor(x, dtype=torch.float64, requires_grad=True)
    yt = torch.tensor(y)
    keep = (yt != -100).to(torch.float64)
    rows = F.cross_entropy(xt, yt, reduction="none", label_smoothing=eps) + z * torch.logsumexp(xt, 1) ** 2 * keep
    loss = rows if reduction == "none" else rows.sum() if reduction == "sum" else rows.sum() / keep.sum()
    dloss = (rng.random(T if reduction == "none" else 1) + 0.5).astype(np.float32)
    loss.backward(torch.tensor(dloss, dtype=torch.float64) if reduction == "none" else torch.tensor(float(dloss[0]), dtype=torch.float64))
    out, lse, _, _ = xo.forward(x, y, reduction, -100, eps, z)
    np.testing.assert_allclose(out, loss.detach().numpy(), rtol=1e-5, atol=1e-5)
    d = xo.backward(x, y, lse, dloss, reduction, -100, eps, z)
    ref = xt.grad.numpy()
    assert np.max(np.abs(d - ref)) <= 1e-6 * np.abs(ref).max() * np.log2(v) + 1e-9


def test_oracle_total_is_the_kernel_order():
    rng = np.random.default_rng(3)
    for t in (1, 31, 1024, 1025, 5000):
        rows = (rng.integers(-64, 65, size=t) / 8).astype(np.float32)
        assert xo.total(rows, "sum", t) == np.float32(rows.astype(np.float64).sum())
        assert xo.total(rows, "mean", t) == np.float32(np.float32(rows.astype(np.float64).sum()) / np.float32(t))
    assert np.isnan(xo.total(np.zeros(4, np.float32), "mean", 0))


@pytest.mark.parametrize("v", [1, 2, 7, 1000, 32000, 50257, 128256, 151936, 262144])
def test_exact_rows_are_exact(v):
    rng = np.random.default_rng(v)
    x, k = xo.exact_rows(rng, 6, v, "bf16")
    m, s, sx, lse = xo.row_stats(x)
    np.testing.assert_array_equal(s, np.exp2(k).astype(np.float32))
    np.testing.assert_array_equal(sx, x.astype(np.float64).sum(1).astype(np.float32))
    for r in range(6):
        assert xo.exact_k_ok(m[r], k[r])
        a = ((x[r] - lse[r]).astype(np.float32) * xo.LOG2E).astype(np.float32)
        hi = x[r] == m[r]
        assert np.all(a[hi] == -k[r]) and np.all(a[~hi] <= -150 * 1.44)


MUTANTS = ["eps_over_v_minus_1", "mean_over_all_rows", "ignored_rows_grad", "z_grad_without_2", "lse_without_shift",
           "g_not_divided"]


@pytest.mark.parametrize("v", [1024, 32768, 262144])
def test_exact_cases_catch_each_wrong_contract(v):
    rng = np.random.default_rng(v)
    T = 12
    x, _ = xo.exact_rows(rng, T, v, "bf16")
    x[0] = np.where(x[0] == x[0].max(), 304, 304 - 160).astype(np.float32)    # a large max: exp without the shift overflows
    y = xo.exact_targets(rng, x)
    eps, z = 0.25, 2.0 ** -6
    caught = set()
    for reduction in xo.REDUCTIONS:
        dloss = (rng.integers(1, 8, size=T if reduction == "none" else 1) / 4.0).astype(np.float32)
        ok_out, ok_lse, _, _ = xo.forward(x, y, reduction, -100, eps, z)
        ok_dx = xo.backward(x, y, ok_lse, dloss, reduction, -100, eps, z, "bf16")
        for m in MUTANTS:
            out, lse, _, _ = xo.forward(x, y, reduction, -100, eps, z, _mutant=m)
            dx = xo.backward(x, y, lse, dloss, reduction, -100, eps, z, "bf16", _mutant=m)
            if not (np.array_equal(out, ok_out, equal_nan=True) and np.array_equal(lse, ok_lse, equal_nan=True)
                    and np.array_equal(dx, ok_dx, equal_nan=True)):
                caught.add(m)
    assert caught == set(MUTANTS), set(MUTANTS) - caught


# ---------------------------------------------------------------------------------------------- dry-run plans
class Planner(PlanContext):
    def _run(self, fn, *a):
        before = self.text()
        rc = fn(self.ctx, None, *a)
        return rc, self.text()[len(before):]

    def fwd(self, t=64, v=128256, x=BF16, tg=I64, g=BF16, reduction=2, eps=0.0, z=0.0, ignore=-100, ls=None, gs=None,
            ptrs=(X, Y, L, S, DL, G), args=True):
        a = _ffi.XentArgs(reduction, ignore, eps, z)
        return self._run(self.lib.b200_cross_entropy, C.byref(a) if args else None, x, tg, t, v, C.c_uint64(ptrs[0]), ls or v,
                         C.c_uint64(ptrs[1]), C.c_uint64(ptrs[2]), C.c_uint64(ptrs[3]), C.c_uint64(ptrs[4]), g,
                         C.c_uint64(ptrs[5]), gs or v)

    def bwd(self, t=64, v=128256, x=BF16, tg=I64, g=BF16, reduction=2, eps=0.0, z=0.0, ls=None, gs=None, ptrs=(X, Y, S, DL, G)):
        a = _ffi.XentArgs(reduction, -100, eps, z)
        return self._run(self.lib.b200_cross_entropy_backward, C.byref(a), x, tg, g, t, v, C.c_uint64(ptrs[0]), ls or v,
                         C.c_uint64(ptrs[1]), C.c_uint64(ptrs[2]), C.c_uint64(ptrs[3]), C.c_uint64(ptrs[4]), gs or v)


@pytest.fixture
def plan():
    with Planner() as p:
        yield p


def _launches(text):
    return re.findall(r"launch (\w+) grid=\((\d+),(\d+),1\) block=(\d+) smem=(\d+) cluster=(\d+)", text)


def _without_t(text):
    return re.sub(r"grid=\(\d+,", "grid=(*,", re.sub(r"alloc \d+", "alloc *", text))


ROWS = [(1, "warp", 32, 1), (10, "warp", 32, 1), (1024, "warp", 32, 1), (1025, "cta", 64, 1), (2048, "cta", 64, 1),
        (4096, "cta", 128, 1), (4097, "cta", 256, 1), (16384, "cta", 256, 1), (16385, "cta", 256, 2), (32000, "cta", 256, 2),
        (50257, "cta", 256, 4), (128256, "cta", 256, 8), (151936, "cta", 256, 8), (1 << 20, "cta", 256, 8)]


@pytest.mark.parametrize("v,cls,nt,ranks", ROWS)
def test_plans_name_kernel_row_class_and_launches(plan, v, cls, nt, ranks):
    rows = 256 // nt
    for x in (F32, BF16, F16):
        for red, pre, post in ((0, [], []), (1, [], ["xent_total"]), (2, ["xent_count"], ["xent_total"])):
            rc, t = plan.fwd(t=100, v=v, x=x, reduction=red, ptrs=(X, Y, L, S, 0, 0))
            assert rc == 0, _ffi.load().b200_last_error()
            assert f"xent fwd x={DT[x]} target=i64 grad=none v={v} class={cls} threads={nt} ranks={ranks}" in t
            ls = _launches(t)
            assert [k[0] for k in ls] == pre + [f"xent_fwd_{DT[x]}_{cls}"] + post
            k = ls[len(pre)]
            assert int(k[1]) == -(-100 // rows) * ranks and k[5] == str(ranks)
            for g in (F32, BF16, F16):
                rc, t = plan.fwd(t=100, v=v, x=x, g=g, reduction=red)
                assert rc == 0 and [k[0] for k in _launches(t)] == pre + [f"xent_fused_{DT[x]}_{DT[g]}_{cls}"] + post
                rc, t = plan.bwd(t=100, v=v, x=x, g=g, reduction=red)
                ls = _launches(t)
                assert rc == 0 and [k[0] for k in ls] == pre + [f"xent_bwd_{DT[x]}_{DT[g]}_{cls}"]
                assert ls[-1][5] == "1"        # the backward merges nothing: plain CTAs


@pytest.mark.parametrize("v", [7, 1000, 4000, 32000, 50257, 128256, 262144])
def test_plan_for_v_is_the_same_for_any_t(plan, v):
    for entry in (plan.fwd, plan.bwd):
        texts = {_without_t(entry(t=t, v=v)[1]) for t in (1, 3, 64, 4096, 65537)}
        assert len(texts) == 1, texts


def test_grid_is_capped(plan):
    rc, t = plan.fwd(t=(1 << 31) - 1, v=128256, reduction=0, ptrs=(X, Y, L, S, 0, 0))
    ((_, gx, *_),) = _launches(t)
    assert rc == 0 and int(gx) == (1 << 20) * 8


def test_vector_path_needs_aligned_rows(plan):
    assert "vec=1" in plan.fwd(v=128256)[1]
    assert "vec=0" in plan.fwd(v=50257)[1]                                        # v % 8
    assert "vec=0" in plan.fwd(v=128256, ls=128257)[1]                            # logits pitch
    assert "vec=0" in plan.fwd(v=128256, gs=128260)[1]                            # dlogits pitch (8 bytes)
    assert "vec=0" in plan.fwd(v=128256, ptrs=(X + 2, Y, L, S, DL, G))[1]
    assert "vec=0" in plan.bwd(v=128256, ptrs=(X, Y, S, DL, G + 8))[1]
    assert "vec=1" in plan.fwd(v=128256, x=F32, g=F32, ls=128260, gs=128264)[1]   # 16-byte pitches


def test_in_place_and_partial_overlap(plan):
    rc, t = plan.fwd(ptrs=(X, Y, L, S, DL, X))
    assert rc == 0 and "in_place=1" in t
    rc, t = plan.bwd(ptrs=(X, Y, S, DL, X))
    assert rc == 0 and "in_place=1" in t
    for kw in (dict(ptrs=(X, Y, L, S, DL, X + 2)), dict(ptrs=(X, Y, L, S, DL, X), g=F16), dict(ptrs=(X, Y, L, S, DL, X), gs=128264),
               dict(ptrs=(X, Y, L, S, DL, X), g=F32), dict(ptrs=(X, Y, L, S, DL, X - 64))):
        rc, t = plan.fwd(**kw)
        assert rc == INVALID and "overlaps" in _ffi.load().b200_last_error().decode() and "launch" not in t, kw
    rc, t = plan.bwd(ptrs=(X, Y, S, DL, X + 1024))
    assert rc == INVALID
    # adjacent but disjoint extents are out of place
    assert plan.fwd(t=4, v=1000, ptrs=(X, Y, L, S, DL, X + 4 * 1000 * 2))[0] == 0
    assert plan.fwd(t=4, v=1000, ptrs=(X + 4 * 1000 * 2, Y, L, S, DL, X))[0] == 0


REFUSALS = [
    ("fwd", dict(args=False), INVALID, "null args"),
    ("fwd", dict(reduction=3), INVALID, "reduction"),
    ("fwd", dict(reduction=-1), INVALID, "reduction"),
    ("fwd", dict(eps=-0.1), INVALID, "label_smoothing"),
    ("fwd", dict(eps=1.5), INVALID, "label_smoothing"),
    ("fwd", dict(eps=float("nan")), INVALID, "label_smoothing"),
    ("fwd", dict(z=-1.0), INVALID, "z_loss"),
    ("fwd", dict(z=float("nan")), INVALID, "z_loss"),
    ("fwd", dict(z=float("inf")), INVALID, "z_loss"),
    ("fwd", dict(x=_ffi.F64), INVALID, "logits dtype"),
    ("fwd", dict(tg=_ffi.U32), INVALID, "target dtype"),
    ("fwd", dict(g=_ffi.I32), INVALID, "grad dtype"),
    ("fwd", dict(v=0), INVALID, "v = 0"),
    ("fwd", dict(v=(1 << 20) + 1), UNSUPPORTED, "exceeds"),
    ("fwd", dict(t=1 << 31), UNSUPPORTED, "2^31"),
    ("fwd", dict(ls=128255), INVALID, "row stride"),
    ("fwd", dict(gs=128255), INVALID, "row stride"),
    ("fwd", dict(ptrs=(X, Y, L, S, DL, 0)), INVALID, "dloss needs dlogits"),
    ("fwd", dict(ptrs=(X, Y, L, S, 0, G)), INVALID, "dloss needs dlogits"),
    ("fwd", dict(ptrs=(0, Y, L, S, DL, G)), INVALID, "null device pointer"),
    ("fwd", dict(ptrs=(X, 0, L, S, DL, G)), INVALID, "null device pointer"),
    ("fwd", dict(ptrs=(X, Y, 0, S, DL, G)), INVALID, "null device pointer"),
    ("fwd", dict(ptrs=(X + 1, Y, L, S, DL, G)), INVALID, "misaligned"),
    ("fwd", dict(ptrs=(X, Y + 4, L, S, DL, G)), INVALID, "misaligned"),
    ("fwd", dict(ptrs=(X, Y, L + 2, S, DL, G)), INVALID, "misaligned"),
    ("fwd", dict(ptrs=(X, Y, L, S + 1, DL, G)), INVALID, "misaligned"),
    ("fwd", dict(ptrs=(X, Y, L, S, DL + 2, G)), INVALID, "misaligned"),
    ("fwd", dict(ptrs=(X, Y, L, S, DL, G + 1)), INVALID, "misaligned"),
    ("bwd", dict(ptrs=(X, Y, 0, DL, G)), INVALID, "null device pointer"),
    ("bwd", dict(ptrs=(X, Y, S, 0, G)), INVALID, "null device pointer"),
    ("bwd", dict(ptrs=(X, Y, S, DL, 0)), INVALID, "null device pointer"),
    ("bwd", dict(ptrs=(0, Y, S, DL, G)), INVALID, "null device pointer"),
    ("bwd", dict(ptrs=(X, Y, S + 2, DL, G)), INVALID, "misaligned"),
    ("bwd", dict(g=_ffi.F64), INVALID, "grad dtype"),
    ("bwd", dict(v=(1 << 21)), UNSUPPORTED, "exceeds"),
    ("bwd", dict(gs=5), INVALID, "row stride"),
]


@pytest.mark.parametrize("case", range(len(REFUSALS)))
def test_refusals(plan, case):
    entry, kw, status, words = REFUSALS[case]
    rc, t = getattr(plan, entry)(**kw)
    msg = _ffi.load().b200_last_error().decode()
    assert rc == status, (case, rc, msg)
    assert words in msg and "launch" not in t, (case, msg, t)


def test_zero_rows_are_a_no_op_even_without_pointers(plan):
    for entry, n in (("fwd", 6), ("bwd", 5)):
        rc, t = getattr(plan, entry)(t=0, ptrs=(0,) * n)
        assert rc == 0 and t == "", (entry, t)
    # the argument checks still run
    assert plan.fwd(t=0, v=0)[0] == INVALID and plan.fwd(t=0, v=1 << 21)[0] == UNSUPPORTED and plan.bwd(t=0, eps=2.0)[0] == INVALID


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
    x, y, one = _T([16, 256]), _T([16], "i64"), _T([1], "f32")
    xent.forward(s, _T([16, 256, 1]), y, one)                                # logits not 2-D
    xent.forward(s, x, _T([16], "f32"), one)                                 # targets not i32 / i64
    xent.forward(s, x, y, _T([16], "f32"))                                   # loss not [1] for mean
    xent.forward(s, x, y, one, reduction="avg")                              # unknown reduction
    xent.forward(s, x, y, one, lse=_T([15], "f32"))                          # lse not [T]
    xent.forward(s, _T([16, 256], strides=[512, 2]), y, one)                 # column stride
    xent.forward(s, x, y, one, dloss=one, dlogits=_T([16, 128]))             # dlogits not [T, V]
    xent.backward(s, x, y, _T([16], "f32"), _T([16], "f32"), x)              # dloss not [1] for mean
    xent.backward(s, x, y, _T([16], "bf16"), one, x)                         # lse not f32
    assert [e.status for e in s.errors] == [INVALID] * 9
    for i, word in enumerate(["logits", "targets", "loss", "reduction", "lse", "logits", "dlogits", "dloss", "lse"]):
        assert word in str(s.errors[i]), (i, str(s.errors[i]))


# ---------------------------------------------------------------------------------------------- kernels
KERNELS = ({f"xent_fwd_{x}_{c}" for x in ("f32", "bf16", "f16") for c in ("warp", "cta")}
           | {f"xent_{m}_{x}_{g}_{c}" for m in ("fused", "bwd") for x in ("f32", "bf16", "f16") for g in ("f32", "bf16", "f16")
              for c in ("warp", "cta")}
           | {"xent_count", "xent_total"})


def test_xent_kernels_do_not_spill_and_use_no_atomics():
    tool = _tool("cuobjdump")
    _ffi.load()
    cubin = ROOT / "cubecl_b200" / "build" / "xent.cubin"
    out = subprocess.run([tool, "-res-usage", str(cubin)], capture_output=True, text=True, check=True).stdout
    funcs = re.findall(r"Function (\w+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)
    assert {f for f, *_ in funcs} == KERNELS and len(KERNELS) == 44
    for name, reg, stack, local in funcs:
        assert int(stack) == 0 and int(local) == 0, (name, stack, local)
        assert int(reg) <= (128 if "_fused_" in name else 80), (name, reg)   # 2 (fused) or 3 resident 256-thread CTAs per SM
    sass = subprocess.run([tool, "-sass", str(cubin)], capture_output=True, text=True, check=True).stdout
    bodies = {b.split()[0]: b for b in re.split(r"\n\s*Function : ", sass)[1:]}
    assert set(bodies) == KERNELS
    for name, body in bodies.items():
        assert not re.search(r"\b(ATOM|ATOMS|ATOMG|RED|REDG)\b", body), name
        assert not re.search(r"\b(LDL|STL)\b", body), name
    for name in ("xent_fused_bf16_bf16_cta", "xent_bwd_f32_bf16_warp", "xent_fwd_bf16_cta"):
        assert "LDG.E.128" in bodies[name], name
    assert "STG.E.128" in bodies["xent_fused_bf16_bf16_cta"] and "STG.E.128" in bodies["xent_bwd_bf16_f32_cta"]
    assert "MUFU.EX2" in bodies["xent_fwd_bf16_cta"] and "MUFU.LG2" in bodies["xent_fwd_bf16_cta"]
    assert "UCGABAR" in bodies["xent_fwd_bf16_cta"] or "CGABAR" in bodies["xent_fwd_bf16_cta"]   # cluster barrier
