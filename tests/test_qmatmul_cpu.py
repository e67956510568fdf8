"""CPU: the quantized-matmul oracle (exact fma emulation against fractions, the bound against an f64 matmul of the dequantized
operands), the host plans of b200_matmul_quantized through a dry-run planning context, every validation code, and the SASS
and register report of the new kernels."""
import ctypes as C
import re
import shutil
import subprocess
from fractions import Fraction
from pathlib import Path

import numpy as np
import pytest

import qmatmul_oracle as qmo
import quant_oracle as qo
from cubecl_b200 import _ffi
from cubecl_b200.quant import QuantScheme

ROOT = Path(__file__).resolve().parent.parent
F32, F16, BF16, U32, F8E4M3, UE8M0 = _ffi.F32, _ffi.F16, _ffi.BF16, _ffi.U32, _ffi.F8E4M3, _ffi.UE8M0
VA, VB, SA, SB, TA, TB, OUT = 0x10000000, 0x20000000, 0x30000000, 0x40000000, 0x50000000, 0x50000100, 0x60000000
INVALID, UNSUPPORTED = 6, 7


# ---------------------------------------------------------------------------------------------- oracle
def _exact_fma(a, b, c):
    return np.float32(float(Fraction(int(a)) * Fraction(float(b)) + Fraction(float(c))))


def _rn_f32(fr: Fraction) -> np.float32:
    """Round a rational to the nearest f32 (ties to even) by bisection on the f32 grid."""
    x = np.float32(float(fr))   # float(fr) is correctly rounded to f64; refine at the f32 level
    lo = np.nextafter(x, np.float32(-np.inf)) if Fraction(float(x)) > fr else x
    hi = np.nextafter(lo, np.float32(np.inf))
    dl, dh = fr - Fraction(float(lo)), Fraction(float(hi)) - fr
    if dl < dh:
        return lo
    if dh < dl:
        return hi
    return lo if (lo.view(np.uint32) & 1) == 0 else hi


def test_fma_emulation_is_exact():
    rng = np.random.default_rng(0)
    a = rng.integers(-(1 << 21), 1 << 21, size=4000)
    b = (rng.standard_normal(4000) * np.exp2(rng.integers(-30, 30, size=4000))).astype(np.float32)
    c = (rng.standard_normal(4000) * np.exp2(rng.integers(-30, 30, size=4000))).astype(np.float32)
    # adversarial ties: c sits half an f32 ulp of a*b away, so a double rounding through f64 would pick the wrong side
    for i in range(0, 4000, 4):
        p = np.float32(a[i] * np.float64(b[i]))
        if np.isfinite(p) and p != 0:
            c[i] = np.float32(np.spacing(p) / 2) if i % 8 else np.float32(-np.spacing(p) / 2)
            a[i + 1], b[i + 1], c[i + 1] = 3, np.float32(1 + 2.0 ** -23), np.float32(2.0 ** -45 * (1 + i % 3))
    got = qmo.fma_f32(a, b, c)
    exp = np.array([_rn_f32(Fraction(int(x)) * Fraction(float(y)) + Fraction(float(z))) for x, y, z in zip(a, b, c)], np.float32)
    assert np.array_equal(got.view(np.uint32), exp.view(np.uint32))


def _operand(scheme, batch, rows, K, seed):
    rng = np.random.default_rng(seed)
    lo, hi = qo.RANGE[scheme.value]
    bits = qo.BITS[scheme.value]
    fields = (rng.integers(int(lo), int(hi) + 1, size=(batch, rows, K)) & ((1 << bits) - 1)).astype(np.uint8)
    raw = None
    if scheme.block:
        s = rng.uniform(0.5, 2.0, size=(batch, rows, K // scheme.block)).astype(np.float32)
        raw = qo.scale_store(scheme.block_scale, qo.round_up(scheme.block_scale, s))
    g = np.float32(rng.uniform(0.001, 0.01)) if scheme.has_tensor else None
    return qmo.Operand(scheme, qo.pack(fields, bits), raw, g, batch, rows, K)


@pytest.mark.parametrize("sa,sb", [(QuantScheme().with_value("q8s").per_block(128, "f32"), QuantScheme().with_value("q8s").per_block(128, "f32")),
                                   (QuantScheme().with_value("q8s").per_block(32, "f16").per_tensor(), QuantScheme().with_value("q4s").per_block(64, "ue8m0")),
                                   (QuantScheme().with_value("q8f").per_tensor(), QuantScheme().with_value("q2s").per_tensor())])
def test_oracle_within_the_bound_of_an_f64_matmul(sa, sb):
    a, b = _operand(sa, 2, 24, 512, 1), _operand(sb, 2, 20, 512, 2)
    got = qmo.matmul(a, b).astype(np.float64)
    da, db = a.dequantized(), b.dequantized()
    ref = np.einsum("bmk,bnk->bmn", da, db)
    J = 512 // (qmo.kernel_block(a, b) or 512)
    bound = (J + 2) * 2.0 ** -24 * np.einsum("bmk,bnk->bmn", np.abs(da), np.abs(db))
    assert np.all(np.abs(got - ref) <= bound)


def test_oracle_fold_order_matches_a_scalar_loop():
    a = _operand(QuantScheme().with_value("q8s").per_block(32, "bf16"), 1, 3, 128, 3)
    b = _operand(QuantScheme().with_value("q4f").per_block(64, "f32").per_tensor(), 1, 2, 128, 4)
    got = qmo.matmul(a, b)
    A, B = a.codes(), b.codes()
    ea, eb = qmo.block_scales(a.scheme, a.scales, a.tensor, 1, 3, 128, 32), qmo.block_scales(b.scheme, b.scales, b.tensor, 1, 2, 128, 32)
    for m in range(3):
        for n in range(2):
            acc = np.float32(0)
            for j in range(4):
                d = int(np.dot(A[0, m, 32 * j:32 * j + 32], B[0, n, 32 * j:32 * j + 32]))
                acc = _exact_fma(d, np.float32(ea[0, m, j] * eb[0, n, j]), acc)
            assert got[0, m, n].view(np.uint32) == acc.view(np.uint32)


# ---------------------------------------------------------------------------------------------- dry-run plans
class Planner:
    def __init__(self, sms=132):   # H100 SXM
        self.lib = _ffi.load()
        self.ctx = C.c_void_p()
        _ffi.check(self.lib.b200_plan_begin(sms, C.byref(self.ctx)))

    def close(self):
        self.lib.b200_destroy(self.ctx)

    def text(self):
        need = C.c_size_t()
        _ffi.check(self.lib.b200_plan_text(self.ctx, None, 0, C.byref(need)))
        buf = C.create_string_buffer(need.value)
        _ffi.check(self.lib.b200_plan_text(self.ctx, buf, need.value, None))
        return buf.value.decode()

    def run(self, sa, sb, batch, m, n, k, odt=BF16, va=VA, vb=VB, out=OUT, ptrs=None):
        ca = sa if isinstance(sa, _ffi.QuantScheme) else sa.to_c()
        cb = sb if isinstance(sb, _ffi.QuantScheme) else sb.to_c()
        pa = ptrs[0] if ptrs else (SA if ca.block else 0, TA if ca.tensor_scale else 0)
        pb = ptrs[1] if ptrs else (SB if cb.block else 0, TB if cb.tensor_scale else 0)
        a, b = _ffi.QuantOperand(ca, va, *pa), _ffi.QuantOperand(cb, vb, *pb)
        rc = self.lib.b200_matmul_quantized(self.ctx, None, C.byref(a), C.byref(b), odt, out, batch, m, n, k)
        return rc, self.text()


@pytest.fixture
def plan():
    p = Planner()
    yield p
    p.close()


def launches(text):
    return [ln.split()[1] for ln in text.splitlines() if ln.startswith("launch")]


Q8T = QuantScheme().with_value("q8s").per_tensor()
Q8B128 = QuantScheme().with_value("q8s").per_block(128, "f32")


def test_plans(plan):
    # per-tensor x per-tensor: one launch, the s8 mainloop with the scales in the epilogue
    rc, t = plan.run(Q8T, Q8T, 1, 8192, 8192, 8192)
    assert rc == 0 and t == ("tmap esz=1 dims=(8192,8192,1) strides=(8192,67108864) box=(128,128) swizzle=3\n"
                             "tmap esz=1 dims=(8192,8192,1) strides=(8192,67108864) box=(128,128) swizzle=3\n"
                             "tmap esz=2 dims=(8192,8192,1) strides=(16384,134217728) box=(64,64) swizzle=3\n"
                             "launch gemm_q8t_bf16_2sm_n256_kk grid=(132,1,1) block=384 smem=215040 cluster=2\n")
    # per-block: two scale passes into pooled block-major f32 buffers, then the GEMM reading them through two more maps
    rc, t = plan.run(Q8B128, Q8B128, 1, 8192, 8192, 8192)
    assert rc == 0 and t == ("alloc 2097152\n"
                             "launch quant_scales_f32_f32 grid=(2048,1,1) block=256 smem=0 cluster=1\n"
                             "alloc 2097152\n"
                             "launch quant_scales_f32_f32 grid=(2048,1,1) block=256 smem=0 cluster=1\n"
                             "tmap esz=1 dims=(8192,8192,1) strides=(8192,67108864) box=(128,128) swizzle=3\n"
                             "tmap esz=1 dims=(8192,8192,1) strides=(8192,67108864) box=(128,64) swizzle=3\n"
                             "tmap esz=4 dims=(8192,64,1) strides=(32768,2097152) box=(128,1) swizzle=0\n"
                             "tmap esz=4 dims=(8192,64,1) strides=(32768,2097152) box=(128,1) swizzle=0\n"
                             "tmap esz=2 dims=(8192,8192,1) strides=(16384,134217728) box=(64,64) swizzle=3\n"
                             "launch gemm_q8_bf16_2sm_n128_kk grid=(132,1,1) block=384 smem=202752 cluster=2\n")
    # two-level Q8S / 32 / f16 x Q4S / 64 / ue8m0: Bk = 32, the Q4 operand is widened first
    rc, t = plan.run(QuantScheme().with_value("q8s").per_block(32, "f16").per_tensor(), QuantScheme().with_value("q4s").per_block(64, "ue8m0"),
                     1, 256, 256, 1024, odt=F32)
    assert rc == 0 and launches(t) == ["quant_widen_s8", "quant_scales_f32_f16", "quant_scales_f32_ue8m0", "gemm_q8_f32_2sm_n128_kk"]
    assert "box=(128,4) swizzle=0" in t
    # K = 200 (a multiple of 8 but not of 16): the Q8 operands are staged
    rc, t = plan.run(Q8T, Q8T, 2, 100, 64, 200, odt=F16)
    assert rc == 0 and launches(t) == ["repitch_rows", "repitch_rows", "gemm_q8t_f16_1sm_n128_kk"]
    # an unaligned code base
    rc, t = plan.run(Q8T, Q8T, 1, 512, 512, 256, va=VA + 8)
    assert rc == 0 and launches(t) == ["repitch_rows", "gemm_q8t_bf16_2sm_n128_kk"]
    # zero extents: no-op
    for shape in ((0, 4, 4, 64), (1, 0, 4, 64), (1, 4, 0, 64)):
        assert plan.run(Q8B128, Q8B128, *shape[:3], 128) == (0, "")
    assert plan.run(Q8T, Q8T, 1, 0, 4, 64, va=0, vb=0, out=0) == (0, "")


def test_variants_and_no_stream_k(plan):
    # the per-block fold has 128-wide tiles only; a forced 2sm_n256 is refused, no stream-K head for either kind
    plan.lib.b200_set_option(plan.ctx, b"gemm.variant", b"2sm_n256")
    assert plan.run(Q8B128, Q8B128, 1, 1024, 1024, 1024)[0] == INVALID
    rc, t = plan.run(Q8T, Q8T, 1, 1024, 1024, 1024)
    assert rc == 0 and launches(t) == ["gemm_q8t_bf16_2sm_n256_kk"]
    plan.lib.b200_set_option(plan.ctx, b"gemm.variant", b"1sm_n128")
    rc, t = plan.run(Q8B128, Q8B128, 1, 1024, 1024, 1024)
    assert rc == 0 and launches(t)[-1] == "gemm_q8_bf16_1sm_n128_kk" and "smem=202752" in t
    plan.lib.b200_set_option(plan.ctx, b"gemm.variant", b"auto")
    for sa in (Q8T, Q8B128):
        rc, t = plan.run(sa, sa, 1, 8192 + 128, 8192, 4096)
        assert rc == 0 and "stream-k" not in t


def _sc(value=_ffi.QV_Q8S, block=32, block_scale=F32, tensor=0):
    return _ffi.QuantScheme(value, block, block_scale, tensor)


def test_validation(plan):
    r = plan.run
    assert r(_sc(), _sc(), 1, 4, 4, 64)[0] == 0
    assert r(_sc(value=9), _sc(), 1, 4, 4, 64)[0] == INVALID                        # unknown value
    assert r(_sc(), _sc(block_scale=U32), 1, 4, 4, 64)[0] == INVALID                # unknown block-scale dtype
    assert r(_sc(), _sc(), 1, 4, 4, 64, odt=U32)[0] == INVALID                      # unknown output dtype
    assert r(_sc(block=64), _sc(), 1, 4, 4, 96)[0] == INVALID                       # K not divisible by a block
    assert r(_sc(), _sc(block=0, tensor=0), 1, 4, 4, 64)[0] == INVALID              # no level
    assert r(_sc(), _sc(), 1, 4, 4, 64, ptrs=((0, 0), (SB, 0)))[0] == INVALID       # null pointer for a present level
    assert r(_sc(), _sc(), 1, 4, 4, 64, ptrs=((SA, TA), (SB, 0)))[0] == INVALID     # non-null pointer for an absent level
    assert r(_sc(block=0, tensor=1), _sc(), 1, 4, 4, 64, ptrs=((0, 0), (SB, 0)))[0] == INVALID
    assert r(_sc(), _sc(), 1, 4, 4, 64, va=0)[0] == INVALID
    assert r(_sc(), _sc(), 1, 4, 4, 64, out=0)[0] == INVALID
    assert r(_sc(), _sc(), 1, 4, 4, 0)[0] == INVALID                                # K = 0 with a non-empty output
    for v in (_ffi.QV_E4M3, _ffi.QV_E5M2, _ffi.QV_E2M1):                           # minifloats: b200_matmul_scaled
        assert r(_sc(value=v), _sc(), 1, 4, 4, 64)[0] == UNSUPPORTED
        assert "b200_matmul_scaled" in plan.lib.b200_last_error().decode()
    for blk in (8, 16):
        assert r(_sc(block=blk), _sc(), 1, 4, 4, 64)[0] == UNSUPPORTED
    # per-tensor x per-tensor: exact s32 dot products need K < 131072; any block level lifts the limit
    assert r(_sc(block=0, tensor=1), _sc(block=0, tensor=1), 1, 4, 4, 131072)[0] == UNSUPPORTED
    assert r(_sc(block=0, tensor=1), _sc(block=0, tensor=1), 1, 4, 4, 131056)[0] == 0
    assert r(_sc(block=0, tensor=1), _sc(), 1, 4, 4, 131072)[0] == 0
    # every block-scale dtype b200_dequantize reads, on a two-level side
    for dt in (F32, F16, BF16, UE8M0, F8E4M3):
        rc, t = r(_sc(block_scale=dt, tensor=1), _sc(), 1, 4, 4, 64)
        assert rc == 0, dt
    assert plan.lib.b200_matmul_quantized(plan.ctx, None, None, None, F32, OUT, 1, 4, 4, 64) == INVALID


# ---------------------------------------------------------------------------------------------- kernels
def _tool(name):
    t = shutil.which(name) or (f"/usr/local/cuda/bin/{name}" if Path(f"/usr/local/cuda/bin/{name}").exists() else None)
    if t is None:
        pytest.skip(f"{name} is not installed")
    return t


def test_new_kernels_use_s8_wgmma_and_tma_and_do_not_spill():
    tool = _tool("cuobjdump")
    _ffi.load()   # builds the cubins when they are missing
    build = ROOT / "cubecl_b200" / "build"
    out = "".join(subprocess.run([tool, "-res-usage", str(build / f)], capture_output=True, text=True, check=True).stdout
                  for f in ("gemm_q.cubin", "quant_mm.cubin"))
    funcs = re.findall(r"Function (\w+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)
    names = {f for f, *_ in funcs}
    tiles = ("2sm_n256", "2sm_n128", "1sm_n128")
    assert names == ({f"gemm_q8t_{o}_{t}_kk" for o in ("bf16", "f16", "f32") for t in tiles}
                     | {f"gemm_q8_{o}_{t}_kk" for o in ("bf16", "f16", "f32") for t in tiles[1:]}
                     | {f"quant_scales_f32_{d}" for d in ("f32", "f16", "bf16", "ue8m0", "ue4m3", "tensor")} | {"quant_widen_s8"})
    for name, reg, stack, local in funcs:
        assert int(stack) == 0 and int(local) == 0, (name, stack, local)
    sass = subprocess.run([tool, "-sass", str(build / "gemm_q.cubin")], capture_output=True, text=True, check=True).stdout
    for body in re.split(r"\n\s*Function : ", sass)[1:]:
        name = body.split()[0]
        assert re.search(r"IGMMA\.64x(64|128|256)x32\.S8\.S8", body), name
        assert "UTMALDG" in body, name
