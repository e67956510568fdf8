"""CPU: the normalization oracle (tests/norm_oracle.py) pinned to torch's rms_norm / layer_norm and autograd within the
oracle's bound, the exact cases' power to catch a wrong contract, the dry-run plans of b200_norm, b200_norm_quantized_fp8
and b200_norm_backward for every dtype cell and row class (the same for any t), every refusal and zero extent, the Python
layer's deferred errors, and the norm cubin's resources and SASS."""
import ctypes as C
import re
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import norm_oracle as no
from cubecl_b200 import _ffi, norm
from cubecl_b200.quant import QuantScheme
from plan_context import PlanContext
from test_conv_cpu import ROOT, _tool

F32, F16, BF16 = _ffi.F32, _ffi.F16, _ffi.BF16
DT = {F32: "f32", BF16: "bf16", F16: "f16"}
X, R, H, W, B, Y, MEAN, RSTD, DY, DH, DX, DW, DB, SC = (0x10000000 * i for i in range(1, 15))
INVALID, UNSUPPORTED = 6, 7


# ---------------------------------------------------------------------------------------------- oracle vs torch
@pytest.mark.parametrize("kind", ["rms", "layer"])
@pytest.mark.parametrize("n", [1, 7, 100, 1000, 4096, 9000, 20000])
def test_oracle_forward_matches_torch(kind, n):
    rng = np.random.default_rng(n)
    x = (rng.standard_normal((9, n)) * 2 + 0.7).astype(np.float32)
    w = rng.standard_normal(n).astype(np.float32)
    b = rng.standard_normal(n).astype(np.float32) if kind == "layer" else None
    _, y, mu, rstd = no.forward(kind, x, 1e-5, w, b)
    xt = torch.tensor(x, dtype=torch.float64)
    wt, bt = torch.tensor(w, dtype=torch.float64), (torch.tensor(b, dtype=torch.float64) if b is not None else None)
    yt = F.rms_norm(xt, (n,), wt, 1e-5) if kind == "rms" else F.layer_norm(xt, (n,), wt, bt, 1e-5)
    ref, bound = no.reference_f64(kind, x, 1e-5, w, b)
    np.testing.assert_allclose(ref, yt.numpy(), rtol=1e-12, atol=1e-12)
    assert np.all(np.abs(y - yt.numpy()) <= bound)


@pytest.mark.parametrize("kind", ["rms", "layer"])
@pytest.mark.parametrize("n,T", [(7, 40), (1000, 40), (4096, 40), (20000, 40), (1000, 3001), (4096, 3001)])
def test_oracle_backward_with_fused_residual_matches_autograd(kind, n, T):
    # T = 3001: several rows per dweight / dbias unit, and a short last unit
    rng = np.random.default_rng(n + 3)
    x = no.rnd(rng.standard_normal((T, n)).astype(np.float32), "bf16")
    r = no.rnd(rng.standard_normal((T, n)).astype(np.float32) * 0.5, "bf16")
    w = rng.standard_normal(n).astype(np.float32)
    b = rng.standard_normal(n).astype(np.float32) if kind == "layer" else None
    dy = rng.standard_normal((T, n)).astype(np.float32)
    dh = rng.standard_normal((T, n)).astype(np.float32)
    h, _, mu, rstd = no.forward(kind, x, 1e-5, w, b, r, "bf16")
    dx, dw, db = no.backward(kind, dy, h, rstd, w, mu, dh, "f32")
    # autograd through h = x + r: the gradient of x and of r is dL/dh + d_h (the residual stream's own gradient)
    xt = torch.tensor(x, dtype=torch.float64, requires_grad=True)
    rt = torch.tensor(r, dtype=torch.float64, requires_grad=True)
    wt = torch.tensor(w, dtype=torch.float64, requires_grad=True)
    bt = torch.tensor(b, dtype=torch.float64, requires_grad=True) if b is not None else None
    s = xt + rt
    ht = torch.tensor(h, dtype=torch.float64) + (s - s.detach())    # h is rounded; its gradient flows to x and r
    yt = F.rms_norm(ht, (n,), wt, 1e-5) if kind == "rms" else F.layer_norm(ht, (n,), wt, bt, 1e-5)
    (yt * torch.tensor(dy, dtype=torch.float64)).sum().backward()
    gx = xt.grad.numpy() + dh
    scale = np.abs(gx).max(1, keepdims=True) + 1
    assert np.max(np.abs(dx - gx) / scale) <= (8 * n + 64) * 2.0 ** -24
    assert np.max(np.abs(dx - (rt.grad.numpy() + dh)) / scale) <= (8 * n + 64) * 2.0 ** -24
    wref = wt.grad.numpy()
    assert np.max(np.abs(dw - wref)) <= (4 * T + 4 * n + 64) * 2.0 ** -24 * (np.abs(dy).sum(0).max() * 8 + 1)
    if b is not None:
        np.testing.assert_allclose(db, bt.grad.numpy(), atol=(4 * T + 16) * 2.0 ** -24 * np.abs(dy).sum(0).max())


@pytest.mark.parametrize("n", [1, 7, 31, 1024, 1025, 8192, 8193, 16384, 16385, 32768])
def test_kernel_order_sum_is_the_sum_on_exact_terms(n):
    rng = np.random.default_rng(n)
    t = (rng.integers(-64, 65, size=(5, n)) / 16.0).astype(np.float32)
    np.testing.assert_array_equal(no.ksum(t, n), t.astype(np.float64).sum(1).astype(np.float32))


@pytest.mark.parametrize("n", [7, 128, 1000, 4096, 7168, 16384, 32768])
def test_exact_cases_catch_each_wrong_contract(n):
    rng = np.random.default_rng(n)
    T = 16
    # a residual whose f32 sum is not on bf16's grid: statistics from the unrounded sum differ
    h = no.exact_rms_rows(rng, T, n)
    eps = np.float32(2.0 ** -10)
    r = (np.where(rng.random((T, n)) < 0.5, 1, -1) * eps * np.abs(h)).astype(np.float32)
    x = h
    ok = no.forward("rms", x, 0.0, residual=r, x_dtype="bf16")
    bad = no.forward("rms", x, 0.0, residual=r, x_dtype="bf16", _mutant="unrounded_residual")
    assert np.array_equal(ok[0], h) and not np.array_equal(ok[3], bad[3])
    # Layer: one-pass variance (f32 rows with a large mean), n - 1, dropped c2, d_h added after the rounding
    hl = no.exact_layer_rows(rng, T, n, "f32")
    no.assert_exact("layer", hl)
    _, _, mu, rstd = no.forward("layer", hl, 0.0)
    # (at n >= 16384 the mean fits so few bits that n * (mu^2 + var) stays exact and a one-pass variance goes unnoticed)
    for m in ("one_pass_var", "n_minus_1") if n < 16384 else ("n_minus_1",):
        assert not np.array_equal(rstd, no.forward("layer", hl, 0.0, _mutant=m)[3]), m
    w, dy, dh = no.exact_weight(rng, n), no.exact_grad(rng, T, n), no.exact_grad(rng, T, n)
    no.assert_exact("layer", hl, 0.0, w, dy)
    dx = no.backward("layer", dy, hl, rstd, w, mu, dh, "bf16")[0]
    for m in ("no_c2", "d_h_after_round"):
        assert not np.array_equal(dx, no.backward("layer", dy, hl, rstd, w, mu, dh, "bf16", _mutant=m)[0]), m


def test_units_depend_on_t_and_n_only_and_cover_every_row():
    for n in (1, 1000, 4096, 32768):
        for t in (1, 7, 64, 1000, 4096, 65537, (1 << 31) - 1):
            u, per = no.units(t, n)
            assert (u - 1) * per < t <= u * per and u <= 1024
    assert no.units(3001, 4096) == (501, 6) and no.units(3001, 1000) == (1001, 3) and no.units(1001, 16384) == (126, 8)


# ---------------------------------------------------------------------------------------------- dry-run plans
class Planner(PlanContext):
    def args(self, kind="rms", x=BF16, w=F32, eps=1e-6):
        return _ffi.NormArgs(_ffi.NORM_RMS if kind == "rms" else _ffi.NORM_LAYER, x, w, eps)

    def _run(self, fn, *a):
        before = self.text()
        rc = fn(self.ctx, None, *a)
        return rc, self.text()[len(before):]

    def fwd(self, t=64, n=4096, kind="rms", x=BF16, w=F32, y=BF16, eps=1e-6, strides=None, ptrs=None, args=True):
        s = strides or (n, n, n, n)
        p = ptrs or (X, 0, 0, W, 0, Y, 0, RSTD)
        a = self.args(kind, x, w, eps)
        return self._run(self.lib.b200_norm, C.byref(a) if args else None, y, t, n, C.c_uint64(p[0]), s[0], C.c_uint64(p[1]),
                         s[1], C.c_uint64(p[2]), s[2], C.c_uint64(p[3]), C.c_uint64(p[4]), C.c_uint64(p[5]), s[3],
                         C.c_uint64(p[6]), C.c_uint64(p[7]))

    def fp8(self, t=64, n=4096, kind="rms", x=BF16, w=F32, scheme=(2, 128, F32, 0), ptrs=None):
        p = ptrs or (X, 0, 0, W, 0, Y, SC, 0, RSTD)
        a, q = self.args(kind, x, w), _ffi.QuantScheme(*scheme)
        return self._run(self.lib.b200_norm_quantized_fp8, C.byref(a), C.byref(q), t, n, C.c_uint64(p[0]), n, C.c_uint64(p[1]), n,
                         C.c_uint64(p[2]), n, C.c_uint64(p[3]), C.c_uint64(p[4]), C.c_uint64(p[5]), C.c_uint64(p[6]),
                         C.c_uint64(p[7]), C.c_uint64(p[8]))

    def bwd(self, t=64, n=4096, kind="rms", x=BF16, w=F32, g=BF16, strides=None, ptrs=None):
        s = strides or (n, n, n, n)
        p = ptrs or (DY, H, W, MEAN if kind == "layer" else 0, RSTD, 0, DX, DW, 0)
        a = self.args(kind, x, w)
        return self._run(self.lib.b200_norm_backward, C.byref(a), g, t, n, C.c_uint64(p[0]), s[0], C.c_uint64(p[1]), s[1],
                         C.c_uint64(p[2]), C.c_uint64(p[3]), C.c_uint64(p[4]), C.c_uint64(p[5]), s[2], C.c_uint64(p[6]), s[3],
                         C.c_uint64(p[7]), C.c_uint64(p[8]))


@pytest.fixture
def plan():
    with Planner() as p:
        yield p


def _launches(text):
    return re.findall(r"launch (\w+) grid=\((\d+),(\d+),1\) block=(\d+) smem=(\d+) cluster=(\d+)", text)


def _without_t(text):
    """the plan with what depends on t (grids and the partials' size) left out"""
    return re.sub(r"grid=\(\d+,", "grid=(*,", re.sub(r"alloc \d+", "alloc *", text))


ROWS = [(1, "warp", 32, 1), (1024, "warp", 32, 1), (1025, "cta", 64, 1), (2048, "cta", 64, 1), (2049, "cta", 128, 1),
        (4096, "cta", 128, 1), (4097, "cta", 256, 1), (8192, "cta", 256, 1), (8193, "cta", 256, 2), (16384, "cta", 256, 2),
        (16385, "cta", 256, 4), (32768, "cta", 256, 4)]
CELLS = [(x, w, y) for x in (F32, BF16, F16) for w in (F32, x) for y in (F32, BF16, F16)]


@pytest.mark.parametrize("n,cls,nt,ranks", ROWS)
def test_forward_plan_names_kernel_and_row_class(plan, n, cls, nt, ranks):
    for x, w, y in CELLS:
        rc, t = plan.fwd(t=100, n=n, x=x, w=w, y=y)
        assert rc == 0, _ffi.load().b200_last_error()
        assert f"class={cls} threads={nt} ranks={ranks}" in t
        ((name, gx, gy, block, smem, cluster),) = _launches(t)
        assert name == f"norm_fwd_{DT[x]}_{DT[y]}_{cls}" and block == "256" and smem == "0" and cluster == str(ranks)
        assert int(gx) == -(-100 // (256 // nt)) * ranks       # 256 // nt rows per CTA, a cluster of `ranks` per row
    rc, t = plan.fp8(t=100, n=n - n % 128 or 128)
    assert rc == 0 and _launches(t)[0][0].startswith("norm_fwd_bf16_fp8_")


@pytest.mark.parametrize("n,cls,nt,ranks", ROWS)
def test_backward_plan_names_kernel_partials_and_reduce(plan, n, cls, nt, ranks):
    for x in (F32, BF16, F16):
        for g in (F32, BF16, F16):
            rc, t = plan.bwd(t=5000, n=n, x=x, g=g, kind="layer", ptrs=(DY, H, W, MEAN, RSTD, DH, DX, DW, DB))
            assert rc == 0, _ffi.load().b200_last_error()
            u, per = no.units(5000, n)
            (size,) = map(int, re.findall(r"alloc (\d+)", t))     # the pool's size class of the [2][units][n] f32 partials
            assert 2 * u * n * 4 <= size < 2 * u * n * 4 + (2 << 20)
            (k1, k2) = _launches(t)
            assert k1[0] == f"norm_bwd_{DT[x]}_{DT[g]}_{cls}" and k1[4] == "65536" and k1[5] == str(ranks)
            assert int(k1[1]) == -(-u // (256 // nt)) * ranks
            assert k2[:3] == ("norm_bwd_reduce", str(-(-n // 256)), "2")
    rc, t = plan.bwd(t=5000, n=n, ptrs=(DY, H, W, 0, RSTD, 0, DX, 0, 0))   # no dweight / dbias: one launch, no temporary
    assert rc == 0 and "alloc" not in t and len(_launches(t)) == 1


@pytest.mark.parametrize("n", [1, 7, 1000, 4096, 7168, 20000, 32768])
def test_plan_for_n_is_the_same_for_any_t(plan, n):
    for entry in (plan.fwd, plan.bwd):
        texts = {_without_t(entry(t=t, n=n)[1]) for t in (1, 7, 4096)}
        assert len(texts) == 1, texts


def test_vector_path_needs_aligned_rows(plan):
    assert "vec=1" in plan.fwd(n=4096)[1]
    assert "vec=0" in plan.fwd(n=4100)[1]                                   # n % 8
    assert "vec=0" in plan.fwd(n=4096, strides=(4097, 4096, 4096, 4096))[1]  # pitch not 16-byte aligned
    assert "vec=0" in plan.fwd(n=4096, ptrs=(X + 2, 0, 0, W, 0, Y, 0, RSTD))[1]
    assert "vec=0" in plan.bwd(n=4096, ptrs=(DY, H + 2, W, 0, RSTD, 0, DX, DW, 0))[1]


REFUSALS = [
    ("fwd", dict(args=False), INVALID, "null args"),
    ("fwd", dict(kind="rms", x=_ffi.F64), INVALID, "x dtype"),
    ("fwd", dict(w=F16), INVALID, "weight dtype"),
    ("fwd", dict(y=_ffi.I32), INVALID, "y dtype"),
    ("fwd", dict(eps=-1.0), INVALID, "eps"),
    ("fwd", dict(eps=float("nan")), INVALID, "eps"),
    ("fwd", dict(n=0), INVALID, "n = 0"),
    ("fwd", dict(n=32769), UNSUPPORTED, "exceeds"),
    ("fwd", dict(t=1 << 31), UNSUPPORTED, "2^31"),
    ("fwd", dict(strides=(4095, 4096, 4096, 4096)), INVALID, "row stride"),
    ("fwd", dict(strides=(4096, 4096, 4096, 100)), INVALID, "row stride"),
    ("fwd", dict(ptrs=(X, R, 0, W, 0, Y, 0, RSTD)), INVALID, "residual"),
    ("fwd", dict(ptrs=(X, 0, H, W, 0, Y, 0, RSTD)), INVALID, "residual"),
    ("fwd", dict(ptrs=(X, 0, 0, W, B, Y, 0, RSTD)), INVALID, "no bias"),
    ("fwd", dict(ptrs=(X, 0, 0, W, 0, Y, MEAN, RSTD)), INVALID, "no bias"),
    ("fwd", dict(ptrs=(0, 0, 0, W, 0, Y, 0, RSTD)), INVALID, "null device pointer"),
    ("fwd", dict(ptrs=(X, 0, 0, W, 0, 0, 0, RSTD)), INVALID, "null device pointer"),
    ("fwd", dict(ptrs=(X + 1, 0, 0, W, 0, Y, 0, RSTD)), INVALID, "misaligned"),
    ("fwd", dict(ptrs=(X, 0, 0, W + 2, 0, Y, 0, RSTD)), INVALID, "misaligned"),
    ("fwd", dict(ptrs=(X, 0, 0, W, 0, Y, 0, RSTD + 2)), INVALID, "misaligned"),
    ("fp8", dict(scheme=(2, 128, F32, 1)), UNSUPPORTED, "tensor-level"),
    ("fp8", dict(scheme=(0, 128, F32, 0)), INVALID, "value"),
    ("fp8", dict(scheme=(4, 32, _ffi.UE8M0, 0)), INVALID, "value"),
    ("fp8", dict(scheme=(2, 16, F32, 0)), INVALID, "block"),
    ("fp8", dict(scheme=(2, 0, F32, 0)), INVALID, "block"),
    ("fp8", dict(scheme=(2, 128, F16, 0)), INVALID, "block scale dtype"),
    ("fp8", dict(scheme=(2, 128, _ffi.F8E4M3, 0)), INVALID, "block scale dtype"),
    ("fp8", dict(n=4000), INVALID, "multiple of the block"),
    ("fp8", dict(ptrs=(X, 0, 0, W, 0, Y, 0, 0, RSTD)), INVALID, "null device pointer"),
    ("fp8", dict(scheme=(2, 32, F32, 0), ptrs=(X, 0, 0, W, 0, Y, SC + 2, 0, RSTD)), INVALID, "misaligned"),
    ("bwd", dict(g=_ffi.I32), INVALID, "grad dtype"),
    ("bwd", dict(kind="rms", ptrs=(DY, H, W, 0, RSTD, 0, DX, DW, DB)), INVALID, "bias gradient"),
    ("bwd", dict(kind="layer", ptrs=(DY, H, W, 0, RSTD, 0, DX, DW, DB)), INVALID, "null device pointer"),
    ("bwd", dict(ptrs=(DY, H, W, 0, 0, 0, DX, DW, 0)), INVALID, "null device pointer"),
    ("bwd", dict(ptrs=(0, H, W, 0, RSTD, 0, DX, DW, 0)), INVALID, "null device pointer"),
    ("bwd", dict(ptrs=(DY, H, W, 0, RSTD, 0, 0, DW, 0)), INVALID, "null device pointer"),
    ("bwd", dict(ptrs=(DY, H, W, 0, RSTD, DH + 1, DX, DW, 0)), INVALID, "misaligned"),
    ("bwd", dict(ptrs=(DY, H, W, 0, RSTD, 0, DX, DW + 2, 0)), INVALID, "misaligned"),
    ("bwd", dict(strides=(4096, 4095, 4096, 4096)), INVALID, "row stride"),
    ("bwd", dict(n=40000), UNSUPPORTED, "exceeds"),
    ("bwd", dict(n=0), INVALID, "n = 0"),
]


@pytest.mark.parametrize("case", range(len(REFUSALS)))
def test_refusals(plan, case):
    entry, kw, status, words = REFUSALS[case]
    rc, t = getattr(plan, entry)(**kw)
    msg = _ffi.load().b200_last_error().decode()
    assert rc == status, (case, rc, msg)
    assert words in msg and "launch" not in t, (case, msg, t)


def test_zero_rows_are_a_no_op_even_without_pointers(plan):
    for entry, kw in (("fwd", dict(ptrs=(0,) * 8)), ("fp8", dict(ptrs=(0,) * 9)), ("bwd", dict(ptrs=(0,) * 9))):
        rc, t = getattr(plan, entry)(t=0, **kw)
        assert rc == 0 and t == "", (entry, t)
    # the argument checks still run
    assert plan.fwd(t=0, n=0)[0] == INVALID and plan.fwd(t=0, n=40000)[0] == UNSUPPORTED


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

    class _Q:
        def __init__(self, shape, scales=True):
            self.shape, self.scheme = list(shape), QuantScheme().with_value("e4m3").per_block(128, "f32")
            self.block_scales = _T([shape[0], shape[1] // 128], "f32") if scales else None

    s = _Stub()
    x, y = _T([16, 256]), _T([16, 256])
    norm.forward(s, _T([16, 256, 1]), y)                                    # x not 2-D
    norm.forward(s, x, _T([16, 128]))                                       # y not [T, n]
    norm.forward(s, x, y, kind="group")                                     # unknown kind
    norm.forward(s, x, y, residual=_T([16, 256], "f16"))                    # residual not in x's dtype
    norm.forward(s, x, y, weight=_T([255], "f32"))                          # weight not [n]
    norm.forward(s, x, y, rstd=_T([16], "bf16"))                            # rstd not f32
    norm.forward(s, _T([16, 256], strides=[512, 2]), y)                     # column stride
    norm.forward_quantized(s, x, _Q([16, 128]))                             # q not [T, n]
    norm.backward(s, _T([16, 128]), x, _T([16], "f32"), x)                  # dy not [T, n]
    norm.backward(s, x, x, _T([16], "f32"), _T([16, 256], "f16"))           # dx not in dy's dtype
    norm.backward(s, x, x, _T([16], "f32"), x, dweight=_T([256], "bf16"))   # dweight not f32
    assert [e.status for e in s.errors] == [INVALID] * 11
    for i, word in enumerate(["x", "y", "kind", "residual", "weight", "rstd", "x", "q", "dy", "dx", "dweight"]):
        assert word in str(s.errors[i]), (i, str(s.errors[i]))


# ---------------------------------------------------------------------------------------------- kernels
KERNELS = ({f"norm_fwd_{x}_{y}_{c}" for x in ("f32", "bf16", "f16") for y in ("f32", "bf16", "f16", "fp8") for c in ("warp", "cta")}
           | {f"norm_bwd_{x}_{g}_{c}" for x in ("f32", "bf16", "f16") for g in ("f32", "bf16", "f16") for c in ("warp", "cta")}
           | {"norm_bwd_reduce"})


def test_norm_kernels_do_not_spill_and_use_no_atomics():
    tool = _tool("cuobjdump")
    _ffi.load()
    cubin = ROOT / "cubecl_b200" / "build" / "norm.cubin"
    out = subprocess.run([tool, "-res-usage", str(cubin)], capture_output=True, text=True, check=True).stdout
    funcs = re.findall(r"Function (\w+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)
    assert {f for f, *_ in funcs} == KERNELS and len(KERNELS) == 43
    for name, reg, stack, local in funcs:
        assert int(stack) == 0 and int(local) == 0, (name, stack, local)
        assert int(reg) <= 128, (name, reg)     # two 256-thread CTAs per SM
    sass = subprocess.run([tool, "-sass", str(cubin)], capture_output=True, text=True, check=True).stdout
    bodies = {b.split()[0]: b for b in re.split(r"\n\s*Function : ", sass)[1:]}
    assert set(bodies) == KERNELS
    for name, body in bodies.items():
        assert not re.search(r"\b(ATOM|ATOMS|ATOMG|RED|REDG)\b", body), name
        assert not re.search(r"\b(LDL|STL)\b", body), name
    for name in ("norm_fwd_bf16_bf16_cta", "norm_fwd_f32_f32_warp", "norm_bwd_bf16_bf16_cta", "norm_bwd_f16_f32_warp"):
        assert "LDG.E.128" in bodies[name] and "STG.E.128" in bodies[name], name
    assert "LDG.E.128" in bodies["norm_fwd_bf16_fp8_cta"] and "STG.E.64" in bodies["norm_fwd_bf16_fp8_cta"]
    assert "F2FP.SATFINITE.E4M3.F32" in bodies["norm_fwd_bf16_fp8_cta"] or "E4M3" in bodies["norm_fwd_bf16_fp8_cta"]
    assert "UCGABAR" in bodies["norm_fwd_bf16_bf16_cta"] or "CGABAR" in bodies["norm_fwd_bf16_bf16_cta"]   # cluster barrier


@pytest.mark.parametrize("n,rows,ranks", [(8, 8, 1), (4104, 1, 1), (8200, 1, 2)])
def test_forward_grid_is_capped_and_groups_loop_over_the_rest(plan, n, rows, ranks):
    t = (1 << 20) * rows + 1001
    rc, text = plan.fwd(t=t, n=n)
    ((_, gx, _, _, _, cluster),) = _launches(text)
    assert rc == 0 and int(gx) == (1 << 20) * ranks and cluster == str(ranks)
