"""CPU: b200_matmul_quantized_fp8 -- the exact-input oracle against a scalar loop, the host plans through a dry-run planning
context, every validation code, the Python deferral of shape errors, and the SASS and register report of gemm_qf8.cubin."""
import ctypes as C
import re
import shutil
import subprocess
from fractions import Fraction
from pathlib import Path

import numpy as np
import pytest

import qmatmul_fp8_oracle as qf8
import qmatmul_oracle as qmo
import quant_oracle as qo
from cubecl_b200 import _ffi
from cubecl_b200.quant import QuantScheme

ROOT = Path(__file__).resolve().parent.parent
F32, F16, BF16, U32, F8E4M3, UE8M0 = _ffi.F32, _ffi.F16, _ffi.BF16, _ffi.U32, _ffi.F8E4M3, _ffi.UE8M0
VA, VB, SA, SB, TA, TB, OUT = 0x10000000, 0x20000000, 0x30000000, 0x40000000, 0x50000000, 0x50000100, 0x60000000
INVALID, UNSUPPORTED = 6, 7


# ---------------------------------------------------------------------------------------------- oracle
def _operand(scheme, batch, rows, K, seed):
    """Integer-valued fp8 codes in [-4, 4] (exact in e4m3 and e5m2) and scales on the block-scale dtype's grid."""
    rng = np.random.default_rng(seed)
    q = rng.integers(-4, 5, size=(batch, rows, K)).astype(np.float32)
    fields = qo.fp8_codes(q, scheme.value)
    raw = None
    if scheme.block:
        s = rng.uniform(0.5, 2.0, size=(batch, rows, K // scheme.block)).astype(np.float32)
        raw = qo.scale_store(scheme.block_scale, qo.round_up(scheme.block_scale, s))
    g = np.float32(rng.uniform(0.001, 0.01)) if scheme.has_tensor else None
    return qmo.Operand(scheme, fields, raw, g, batch, rows, K)


def _rn(fr):
    # nearest f32 of a rational, ties to even (the scalar loop's reference rounding)
    x = np.float32(float(fr))
    lo = np.nextafter(x, np.float32(-np.inf)) if Fraction(float(x)) > fr else x
    hi = np.nextafter(lo, np.float32(np.inf))
    dl, dh = fr - Fraction(float(lo)), Fraction(float(hi)) - fr
    return lo if dl < dh or (dl == dh and (lo.view(np.uint32) & 1) == 0) else hi


@pytest.mark.parametrize("sa,sb,K", [
    (QuantScheme().with_value("e4m3").per_block(32, "bf16"), QuantScheme().with_value("e5m2").per_block(64, "f32").per_tensor(), 128),
    (QuantScheme().with_value("e5m2").per_tensor(), QuantScheme().with_value("e4m3").per_tensor(), 200),   # short last block
    (QuantScheme().with_value("e4m3").per_block(128, "ue8m0"), QuantScheme().with_value("e4m3").per_tensor(), 256)])
def test_oracle_fold_order_matches_a_scalar_loop(sa, sb, K):
    a, b = _operand(sa, 1, 3, K, 3), _operand(sb, 1, 2, K, 4)
    got = qf8.matmul(a, b)
    A, B = a.codes(), b.codes()
    bk = qf8.kernel_block(a, b)
    ea, eb = qf8.effective(a, bk), qf8.effective(b, bk)
    for m in range(3):
        for n in range(2):
            acc = np.float32(0)
            for j in range(-(-K // bk)):
                d = sum(int(A[0, m, k]) * int(B[0, n, k]) for k in range(j * bk, min((j + 1) * bk, K)))
                p = np.float32(ea[0, m, j] * eb[0, n, j])
                acc = _rn(Fraction(d) * Fraction(float(p)) + Fraction(float(acc)))
            assert got[0, m, n].view(np.uint32) == acc.view(np.uint32), (m, n)


def test_oracle_equals_the_integer_contract_on_exact_inputs():
    # integer-valued fp8 codes: the fp8 oracle is b200_matmul_quantized's per-block fold on the same numbers
    sa, sb = QuantScheme().with_value("e4m3").per_block(64, "f16"), QuantScheme().with_value("e5m2").per_block(32, "f32")
    a, b = _operand(sa, 2, 5, 256, 5), _operand(sb, 2, 7, 256, 6)
    ia = qmo.Operand(QuantScheme().with_value("q8s").per_block(64, "f16"), qo.pack(a.codes().astype(np.int64) & 0xFF, 8), a.scales,
                     None, 2, 5, 256)
    ib = qmo.Operand(QuantScheme().with_value("q8s").per_block(32, "f32"), qo.pack(b.codes().astype(np.int64) & 0xFF, 8), b.scales,
                     None, 2, 7, 256)
    assert np.array_equal(qf8.matmul(a, b).view(np.uint32), qmo.matmul(ia, ib).view(np.uint32))


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
        rc = self.lib.b200_matmul_quantized_fp8(self.ctx, None, C.byref(a), C.byref(b), odt, out, batch, m, n, k)
        return rc, self.text()


@pytest.fixture
def plan():
    p = Planner()
    yield p
    p.close()


def launches(text):
    return [ln.split()[1] for ln in text.splitlines() if ln.startswith("launch")]


E4B128 = QuantScheme().with_value("e4m3").per_block(128, "f32")
E5B128 = QuantScheme().with_value("e5m2").per_block(128, "f32")
E4T = QuantScheme().with_value("e4m3").per_tensor()


def test_plans(plan):
    # per-block 128 on both sides: two scale passes into pooled block-major f32 buffers, the five maps, one GEMM launch
    rc, t = plan.run(E4B128, E4B128, 1, 8192, 8192, 8192)
    assert rc == 0 and t == ("alloc 2097152\n"
                             "launch quant_scales_f32_f32 grid=(2048,1,1) block=256 smem=0 cluster=1\n"
                             "alloc 2097152\n"
                             "launch quant_scales_f32_f32 grid=(2048,1,1) block=256 smem=0 cluster=1\n"
                             "tmap esz=1 dims=(8192,8192,1) strides=(8192,67108864) box=(128,128) swizzle=3\n"
                             "tmap esz=1 dims=(8192,8192,1) strides=(8192,67108864) box=(128,64) swizzle=3\n"
                             "tmap esz=4 dims=(8192,64,1) strides=(32768,2097152) box=(128,1) swizzle=0\n"
                             "tmap esz=4 dims=(8192,64,1) strides=(32768,2097152) box=(128,1) swizzle=0\n"
                             "tmap esz=2 dims=(8192,8192,1) strides=(16384,134217728) box=(64,64) swizzle=3\n"
                             "launch gemm_qf8_e4m3_bf16_2sm_n128_kk grid=(132,1,1) block=384 smem=202752 cluster=2\n")
    # two-level e4m3 / 32 / f16 x e4m3 / 128 / ue8m0: Bk = 32, four scale blocks per stage
    rc, t = plan.run(QuantScheme().with_value("e4m3").per_block(32, "f16").per_tensor(), QuantScheme().with_value("e4m3").per_block(128, "ue8m0"),
                     1, 256, 256, 1024, odt=F32)
    assert rc == 0 and launches(t) == ["quant_scales_f32_f16", "quant_scales_f32_ue8m0", "gemm_qf8_e4m3_f32_2sm_n128_kk"]
    assert "tmap esz=4 dims=(256,32,1) strides=(1024,32768) box=(128,4) swizzle=0" in t
    # per-tensor x per-tensor, K = 8192 + 64: Bk = 128 and the scale buffers cover the short 65th block
    rc, t = plan.run(E4T, E4T, 1, 4096, 4096, 8192 + 64)
    assert rc == 0 and launches(t) == ["quant_scales_f32_tensor", "quant_scales_f32_tensor", "gemm_qf8_e4m3_bf16_2sm_n128_kk"]
    assert t.count("launch quant_scales_f32_tensor grid=(1040,1,1)") == 2   # 65 blocks x 4096 rows, 256 per CTA
    assert t.count("tmap esz=4 dims=(4096,65,1) strides=(16384,1064960) box=(128,1) swizzle=0") == 2
    # e5m2 x e4m3: the lhs format names the kernel, the rhs format is chosen at run time
    rc, t = plan.run(E5B128, E4B128, 1, 1024, 1024, 1024)
    assert rc == 0 and launches(t)[-1] == "gemm_qf8_e5m2_bf16_2sm_n128_kk"
    # K = 200 (not a multiple of 16): the codes are staged
    rc, t = plan.run(E4T, E4T, 2, 100, 64, 200, odt=F16)
    assert rc == 0 and launches(t) == ["repitch_rows", "repitch_rows", "quant_scales_f32_tensor", "quant_scales_f32_tensor",
                                       "gemm_qf8_e4m3_f16_1sm_n128_kk"]
    # an unaligned code base
    rc, t = plan.run(E4B128, E4B128, 1, 512, 512, 256, va=VA + 8)
    assert rc == 0 and launches(t) == ["repitch_rows", "quant_scales_f32_f32", "quant_scales_f32_f32", "gemm_qf8_e4m3_bf16_2sm_n128_kk"]
    # M <= 128: one CTA per tile
    rc, t = plan.run(E4B128, E4B128, 1, 128, 4096, 4096)
    assert rc == 0 and launches(t)[-1] == "gemm_qf8_e4m3_bf16_1sm_n128_kk"
    # zero extents: no-op
    for shape in ((0, 4, 4, 128), (1, 0, 4, 128), (1, 4, 0, 128)):
        assert plan.run(E4B128, E4B128, *shape[:3], shape[3]) == (0, "")
    assert plan.run(E4T, E4T, 1, 0, 4, 64, va=0, vb=0, out=0) == (0, "")


def test_variants_and_no_stream_k(plan):
    plan.lib.b200_set_option(plan.ctx, b"gemm.variant", b"2sm_n256")
    assert plan.run(E4B128, E4B128, 1, 1024, 1024, 1024)[0] == INVALID
    plan.lib.b200_set_option(plan.ctx, b"gemm.variant", b"1sm_n128")
    rc, t = plan.run(E4B128, E4B128, 1, 1024, 1024, 1024)
    assert rc == 0 and launches(t)[-1] == "gemm_qf8_e4m3_bf16_1sm_n128_kk" and "smem=202752" in t
    plan.lib.b200_set_option(plan.ctx, b"gemm.variant", b"2sm_n128")
    rc, t = plan.run(E4B128, E4B128, 1, 128, 1024, 1024)
    assert rc == 0 and launches(t)[-1] == "gemm_qf8_e4m3_bf16_2sm_n128_kk"
    plan.lib.b200_set_option(plan.ctx, b"gemm.variant", b"auto")
    plan.lib.b200_set_option(plan.ctx, b"gemm.split_k", b"on")
    for sa in (E4T, E4B128):
        for shape in ((1, 8192 + 128, 8192, 4096), (1, 8192, 8192, 8192), (3, 300, 200, 256)):
            rc, t = plan.run(sa, sa, *shape)
            assert rc == 0 and "stream-k" not in t


def _sc(value=_ffi.QV_E4M3, block=32, block_scale=F32, tensor=0):
    return _ffi.QuantScheme(value, block, block_scale, tensor)


def test_validation(plan):
    r = plan.run
    assert r(_sc(), _sc(), 1, 4, 4, 64)[0] == 0
    assert r(_sc(value=_ffi.QV_E5M2), _sc(), 1, 4, 4, 64)[0] == 0
    assert r(_sc(value=9), _sc(), 1, 4, 4, 64)[0] == INVALID                        # unknown value
    assert r(_sc(), _sc(block_scale=U32), 1, 4, 4, 64)[0] == INVALID                # unknown block-scale dtype
    assert r(_sc(), _sc(), 1, 4, 4, 64, odt=U32)[0] == INVALID                      # unknown output dtype
    assert r(_sc(block=64), _sc(), 1, 4, 4, 96)[0] == INVALID                       # K not divisible by a block
    assert "not a multiple of the block" in plan.lib.b200_last_error().decode()
    assert r(_sc(), _sc(block=0, tensor=0), 1, 4, 4, 64)[0] == INVALID              # no level
    assert r(_sc(), _sc(), 1, 4, 4, 64, ptrs=((0, 0), (SB, 0)))[0] == INVALID       # null pointer for a present level
    assert r(_sc(), _sc(), 1, 4, 4, 64, ptrs=((SA, TA), (SB, 0)))[0] == INVALID     # non-null pointer for an absent level
    assert r(_sc(block=0, tensor=1), _sc(), 1, 4, 4, 64, ptrs=((0, 0), (SB, 0)))[0] == INVALID
    assert r(_sc(), _sc(), 1, 4, 4, 64, va=0)[0] == INVALID
    assert r(_sc(), _sc(), 1, 4, 4, 64, vb=0)[0] == INVALID
    assert r(_sc(), _sc(), 1, 4, 4, 64, out=0)[0] == INVALID
    assert r(_sc(), _sc(), 1, 4, 4, 64, out=OUT + 1)[0] == INVALID                  # misaligned output
    assert r(_sc(), _sc(), 1, 4, 4, 0)[0] == INVALID                                # K = 0 with a non-empty output
    for v in (_ffi.QV_Q8S, _ffi.QV_Q8F, _ffi.QV_Q4S, _ffi.QV_Q2F):                 # integers: b200_matmul_quantized
        for side in ((_sc(value=v), _sc()), (_sc(), _sc(value=v))):
            assert r(*side, 1, 4, 4, 64)[0] == UNSUPPORTED
            assert "b200_matmul_quantized" in plan.lib.b200_last_error().decode()
    assert r(_sc(value=_ffi.QV_E2M1), _sc(), 1, 4, 4, 64)[0] == UNSUPPORTED         # e2m1: b200_matmul_scaled
    assert "b200_matmul_scaled" in plan.lib.b200_last_error().decode()
    for blk in (8, 16):
        assert r(_sc(block=blk), _sc(), 1, 4, 4, 64)[0] == UNSUPPORTED
        assert "steps of 32" in plan.lib.b200_last_error().decode()
    # per-tensor x per-tensor has no K limit (f32 partials per 128-element block)
    assert r(_sc(block=0, tensor=1), _sc(block=0, tensor=1), 1, 4, 4, 131072)[0] == 0
    # every block-scale dtype b200_dequantize reads, on a one- and a two-level side
    for dt in (F32, F16, BF16, UE8M0, F8E4M3):
        for tensor in (0, 1):
            rc, t = r(_sc(block_scale=dt, tensor=tensor), _sc(), 1, 4, 4, 64)
            assert rc == 0, (dt, tensor)
    assert plan.lib.b200_matmul_quantized_fp8(plan.ctx, None, None, None, F32, OUT, 1, 4, 4, 64) == INVALID


def test_python_entry_point_defers_errors():
    from cubecl_b200 import matmul

    class _Stub:
        def __init__(self):
            self.errors = []

        def _defer(self, e):
            self.errors.append(e)

    class _T:
        def __init__(self, shape):
            self.shape = shape

        def is_contiguous(self):
            return True

    stub = _Stub()
    matmul.launch_quantized_fp8(stub, _T([4, 64]), _T([2, 4, 64]), _T([4, 4]))
    matmul.launch_quantized_fp8(stub, _T([4, 64]), _T([4, 32]), _T([4, 4]))
    matmul.launch_quantized_fp8(stub, _T([4, 64]), _T([8, 64]), _T([4, 4]))
    assert [e.status for e in stub.errors] == [INVALID] * 3
    assert all(str(e).startswith("matmul_quantized_fp8") or "matmul_quantized_fp8" in str(e) for e in stub.errors)
    assert "K mismatch" in str(stub.errors[1]) and "out must be contiguous" in str(stub.errors[2])


# ---------------------------------------------------------------------------------------------- kernels
def _tool(name):
    t = shutil.which(name) or (f"/usr/local/cuda/bin/{name}" if Path(f"/usr/local/cuda/bin/{name}").exists() else None)
    if t is None:
        pytest.skip(f"{name} is not installed")
    return t


def test_fp8_kernels_use_fp8_wgmma_and_tma_and_do_not_spill():
    tool = _tool("cuobjdump")
    _ffi.load()   # builds the cubins when they are missing
    cubin = ROOT / "cubecl_b200" / "build" / "gemm_qf8.cubin"
    out = subprocess.run([tool, "-res-usage", str(cubin)], capture_output=True, text=True, check=True).stdout
    funcs = re.findall(r"Function (\w+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)
    assert {f for f, *_ in funcs} == {f"gemm_qf8_{v}_{o}_{t}_kk" for v in ("e4m3", "e5m2") for o in ("bf16", "f16", "f32")
                                      for t in ("2sm_n128", "1sm_n128")}
    for name, reg, stack, local in funcs:
        assert int(stack) == 0 and int(local) == 0, (name, stack, local)
    sass = subprocess.run([tool, "-sass", str(cubin)], capture_output=True, text=True, check=True).stdout
    for body in re.split(r"\n\s*Function : ", sass)[1:]:
        name = body.split()[0]
        lhs = "E4M3" if "_e4m3_" in name else "E5M2"
        for rhs in ("E4M3", "E5M2"):   # the rhs format of a mixed pair is chosen at run time
            assert re.search(rf"QGMMA\.64x(64|128)x32\.F32\.{lhs}\.{rhs}", body), (name, rhs)
        assert "UTMALDG" in body, name
        assert not re.search(r"\b[IH]GMMA\b", body), name
