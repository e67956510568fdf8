"""CPU: b200_matmul_grouped_quantized_fp8 -- the host plans through a dry-run planning context, every validation code, the
Python deferral of shape errors, and the register and SASS report of gemm_grouped_qf8.cubin."""
import ctypes as C
import re
import shutil
import subprocess
from pathlib import Path

import pytest

from cubecl_b200 import _ffi
from cubecl_b200.quant import QuantScheme
from plan_context import PlanContext

ROOT = Path(__file__).resolve().parent.parent
F32, F16, BF16, U32, F8E4M3, UE8M0 = _ffi.F32, _ffi.F16, _ffi.BF16, _ffi.U32, _ffi.F8E4M3, _ffi.UE8M0
VA, VB, SA, SB, TA, TB, OFFS, OUT = 0x10000000, 0x20000000, 0x30000000, 0x40000000, 0x50000000, 0x50000100, 0x58000000, 0x60000000
INVALID, UNSUPPORTED = 6, 7
QF8_SMEM = 202752                 # gemm_qf8_*: 5 stages of 32 KB codes + 4 KB scale tiles, barriers, TMA-store staging
GRP_SMEM = QF8_SMEM + 8208        # + the group table (kGroupedTableBytes)


class Planner(PlanContext):
    def run(self, sa, sb, groups, t, n, k, odt=BF16, va=VA, vb=VB, out=OUT, offs=OFFS, ptrs=None):
        ca = sa if isinstance(sa, _ffi.QuantScheme) else sa.to_c()
        cb = sb if isinstance(sb, _ffi.QuantScheme) else sb.to_c()
        pa = ptrs[0] if ptrs else (SA if ca.block else 0, TA if ca.tensor_scale else 0)
        pb = ptrs[1] if ptrs else (SB if cb.block else 0, TB if cb.tensor_scale else 0)
        a, b = _ffi.QuantOperand(ca, va, *pa), _ffi.QuantOperand(cb, vb, *pb)
        rc = self.lib.b200_matmul_grouped_quantized_fp8(self.ctx, None, C.byref(a), C.byref(b), offs, groups, odt, out, t, n, k)
        return rc, self.text()


@pytest.fixture
def plan():
    with Planner() as p:
        yield p


def launches(text):
    return [ln.split()[1] for ln in text.splitlines() if ln.startswith("launch")]


E4B128 = QuantScheme().with_value("e4m3").per_block(128, "f32")
E5B128 = QuantScheme().with_value("e5m2").per_block(128, "f32")
E4T = QuantScheme().with_value("e4m3").per_tensor()


def test_plan_of_a_deepseek_like_layer(plan):
    # G = 32, 7168 -> 4096, T = 32768: the bound first, two scale passes, the lhs maps at batch 1, the rhs code and scale maps
    # batched over the 32 groups, one launch with the group table after the qf8 kernels' shared memory
    rc, t = plan.run(E4B128, E4B128, 32, 32768, 4096, 7168)
    assert rc == 0 and t == ("gemm grouped ragged_m groups=32 T=32768 tile_rows<=161 tiles<=5152\n"
                             "alloc 7340032\n"
                             "launch quant_scales_f32_f32 grid=(2112,1,1) block=256 smem=0 cluster=1\n"
                             "alloc 29360128\n"
                             "launch quant_scales_f32_f32 grid=(2112,1,1) block=256 smem=0 cluster=1\n"
                             "tmap esz=1 dims=(7168,32768,1) strides=(7168,234881024) box=(128,128) swizzle=3\n"
                             "tmap esz=1 dims=(7168,4096,32) strides=(7168,29360128) box=(128,64) swizzle=3\n"
                             "tmap esz=4 dims=(32768,56,1) strides=(131072,7340032) box=(128,1) swizzle=0\n"
                             "tmap esz=4 dims=(4096,56,32) strides=(16384,917504) box=(128,1) swizzle=0\n"
                             "tmap esz=2 dims=(4096,32768,1) strides=(8192,268435456) box=(64,64) swizzle=3\n"
                             f"launch gemm_grouped_qf8_e4m3_bf16_2sm_n128_kk grid=(132,1,1) block=384 smem={GRP_SMEM} cluster=2\n")


@pytest.mark.parametrize("tile", ["2sm_n128", "1sm_n128"])
@pytest.mark.parametrize("lhs,fmt", [(E4B128, "e4m3"), (E5B128, "e5m2")])
@pytest.mark.parametrize("odt,otag", [(BF16, "bf16"), (F16, "f16"), (F32, "f32")])
def test_kernel_names(plan, tile, lhs, fmt, odt, otag):
    plan.option("gemm.variant", tile)
    for rhs in (E4B128, E5B128):   # the lhs format names the kernel; the rhs format is chosen at run time
        rc, t = plan.run(lhs, rhs, 4, 1000, 256, 512, odt=odt)
        assert rc == 0 and launches(t)[-1] == f"gemm_grouped_qf8_{fmt}_{otag}_{tile}_kk"
        assert f"smem={GRP_SMEM} cluster={2 if tile == '2sm_n128' else 1}" in t


@pytest.mark.parametrize("G,T,N", [(1, 1, 1), (8, 1000, 256), (128, 32768, 1536), (3, 100000, 700), (1024, 4096, 128)])
def test_grid_bound(plan, G, T, N):
    # every group may add one partial tile-row, and its tile-rows start up to 3 rows early (a 16-byte aligned row coordinate
    # for the f32 scale-tile loads): ceil((T + 3 G) / (128 CG)) + G tile-rows, each of ceil(N / 128) tiles
    rc, t = plan.run(E4B128, E4B128, G, T, N, 256)
    assert rc == 0
    cg = 2 if T >= 1024 * G else 1   # the 2sm / 1sm threshold: 1024 rows per group
    rows = -(-(T + 3 * G) // (128 * cg)) + G
    assert f"gemm grouped ragged_m groups={G} T={T} tile_rows<={rows} tiles<={rows * -(-N // 128)}\n" in t
    assert launches(t)[-1].endswith(f"_{cg}sm_n128_kk")
    grid = min(rows * -(-N // 128), 132 // cg) * cg
    assert f"grid=({grid},1,1) block=384 smem={GRP_SMEM} cluster={cg}" in t


def test_tile_threshold(plan):
    assert launches(plan.run(E4B128, E4B128, 8, 8 * 1024, 256, 256)[1])[-1].endswith("_2sm_n128_kk")
    assert launches(plan.run(E4B128, E4B128, 8, 8 * 1024 - 1, 256, 256)[1])[-1].endswith("_1sm_n128_kk")


def test_scale_maps_and_staging(plan):
    # two-level e4m3 / 32 / f16 x e5m2 / 64 / ue8m0: Bk = 32, four blocks per stage; the rhs maps batched over G = 6
    rc, t = plan.run(QuantScheme().with_value("e4m3").per_block(32, "f16").per_tensor(),
                     QuantScheme().with_value("e5m2").per_block(64, "ue8m0"), 6, 300, 200, 256, odt=F32)
    assert rc == 0 and launches(t) == ["quant_scales_f32_f16", "quant_scales_f32_ue8m0", "gemm_grouped_qf8_e4m3_f32_1sm_n128_kk"]
    assert "tmap esz=4 dims=(300,8,1) strides=(1200,9600) box=(128,4) swizzle=0" in t
    assert "tmap esz=4 dims=(200,8,6) strides=(800,6400) box=(128,4) swizzle=0" in t
    assert "tmap esz=1 dims=(256,200,6) strides=(256,51200) box=(128,128) swizzle=3" in t
    # per-tensor x per-tensor, K = 200: Bk = 128 with a short second block; K % 16 != 0 stages both code operands
    rc, t = plan.run(E4T, E4T, 3, 100, 64, 200)
    assert rc == 0 and launches(t) == ["repitch_rows", "repitch_rows", "quant_scales_f32_tensor", "quant_scales_f32_tensor",
                                       "gemm_grouped_qf8_e4m3_bf16_1sm_n128_kk"]
    assert "tmap esz=1 dims=(200,64,3) strides=(208,13312) box=(128,128) swizzle=3" in t
    assert "tmap esz=4 dims=(64,2,3) strides=(256,512) box=(128,1) swizzle=0" in t
    # an unaligned lhs base: the lhs alone is staged
    rc, t = plan.run(E4B128, E4B128, 4, 512, 256, 256, va=VA + 8)
    assert rc == 0 and launches(t) == ["repitch_rows", "quant_scales_f32_f32", "quant_scales_f32_f32",
                                       "gemm_grouped_qf8_e4m3_bf16_1sm_n128_kk"]


def test_one_group_reads_the_rhs_as_one_batch(plan):
    rc, t = plan.run(E4B128, E4B128, 1, 4096, 256, 256)
    assert rc == 0 and "tmap esz=1 dims=(256,256,1)" in t and "tmap esz=4 dims=(256,2,1)" in t


def test_store_path_and_no_stream_k(plan):
    rc, t = plan.run(E4B128, E4B128, 4, 8192, 1024, 1024)
    assert rc == 0 and "box=(64,64) swizzle=3" in t        # the TMA-store map of whole tiles
    plan.option("gemm.epilogue", "direct")
    rc, t = plan.run(E4B128, E4B128, 4, 8192, 1024, 1024)
    assert rc == 0 and "box=(64,64)" not in t
    plan.option("gemm.epilogue", "tma")
    for opt in ("on", "8", "auto"):
        plan.option("gemm.split_k", opt)
        for shape in ((4, 8192 + 128, 8192, 4096), (128, 32768, 1536, 2048), (3, 300, 200, 256)):
            rc, t = plan.run(E4B128, E4B128, *shape)
            assert rc == 0 and "stream-k" not in t and "alloc" in t


def _sc(value=_ffi.QV_E4M3, block=32, block_scale=F32, tensor=0):
    return _ffi.QuantScheme(value, block, block_scale, tensor)


def test_validation(plan):
    r = plan.run
    err = lambda: plan.lib.b200_last_error().decode()   # noqa: E731
    assert r(_sc(), _sc(), 2, 4, 4, 64)[0] == 0
    assert r(_sc(value=_ffi.QV_E5M2), _sc(), 2, 4, 4, 64)[0] == 0
    # everything quant_check rejects
    assert r(_sc(value=9), _sc(), 2, 4, 4, 64)[0] == INVALID                        # unknown value
    assert r(_sc(), _sc(block_scale=U32), 2, 4, 4, 64)[0] == INVALID                # unknown block-scale dtype
    assert r(_sc(block=64), _sc(), 2, 4, 4, 96)[0] == INVALID                       # K not divisible by a block
    assert "not a multiple of the block" in err()
    assert r(_sc(), _sc(block=0, tensor=0), 2, 4, 4, 64)[0] == INVALID              # no level
    assert r(_sc(), _sc(), 2, 4, 4, 64, ptrs=((0, 0), (SB, 0)))[0] == INVALID       # null pointer for a present level
    assert r(_sc(), _sc(), 2, 4, 4, 64, ptrs=((SA, TA), (SB, 0)))[0] == INVALID     # non-null pointer for an absent level
    assert r(_sc(), _sc(), 2, 4, 4, 64, ptrs=((SA + 2, 0), (SB, 0)))[0] == INVALID  # misaligned scales
    assert r(_sc(), _sc(), 2, 4, 4, 64, odt=U32)[0] == INVALID                      # unknown output dtype
    # offsets, pointers, K
    assert r(_sc(), _sc(), 2, 4, 4, 64, offs=0)[0] == INVALID and "null offs" in err()
    assert r(_sc(), _sc(), 2, 4, 4, 64, offs=OFFS + 2)[0] == INVALID and "offs is misaligned" in err()
    assert r(_sc(), _sc(), 2, 4, 4, 64, va=0)[0] == INVALID
    assert r(_sc(), _sc(), 2, 4, 4, 64, vb=0)[0] == INVALID
    assert r(_sc(), _sc(), 2, 4, 4, 64, out=0)[0] == INVALID
    assert r(_sc(), _sc(), 2, 4, 4, 64, out=OUT + 1)[0] == INVALID                  # misaligned output
    assert r(_sc(), _sc(), 2, 4, 4, 0)[0] == INVALID and "K must be positive" in err()
    # formats that run elsewhere
    for v in (_ffi.QV_Q8S, _ffi.QV_Q8F, _ffi.QV_Q4S, _ffi.QV_Q2F):
        for side in ((_sc(value=v), _sc()), (_sc(), _sc(value=v))):
            assert r(*side, 2, 4, 4, 64)[0] == UNSUPPORTED and "b200_matmul_quantized" in err()
    assert r(_sc(value=_ffi.QV_E2M1), _sc(), 2, 4, 4, 64)[0] == UNSUPPORTED
    for blk in (8, 16):
        assert r(_sc(block=blk), _sc(), 2, 4, 4, 64)[0] == UNSUPPORTED and "steps of 32" in err()
    # limits
    assert r(_sc(), _sc(), 1025, 4, 4, 64)[0] == UNSUPPORTED and "1025 groups" in err()
    assert r(_sc(), _sc(), 1024, 4, 4, 64)[0] == 0
    for t, n, k in ((1 << 31, 4, 64), (4, 1 << 31, 64), (4, 4, 1 << 31)):
        assert r(_sc(), _sc(), 2, t, n, k)[0] == UNSUPPORTED and "2^31" in err()
    assert r(_sc(), _sc(), 2, (1 << 31) - 1, (1 << 31) - 1, 64)[0] == UNSUPPORTED and "too many tiles" in err()
    plan.option("gemm.variant", "2sm_n256")
    assert r(_sc(), _sc(), 2, 4, 4, 64)[0] == INVALID and "not a grouped matmul tile" in err()
    plan.option("gemm.variant", "auto")
    plan.option("gemm.epilogue", "stmatrix")
    assert r(_sc(), _sc(), 2, 4, 4, 64)[0] == INVALID
    plan.option("gemm.epilogue", "tma")
    # every block-scale dtype b200_dequantize reads, on a one- and a two-level side
    for dt in (F32, F16, BF16, UE8M0, F8E4M3):
        for tensor in (0, 1):
            assert r(_sc(block_scale=dt, tensor=tensor), _sc(), 2, 4, 4, 64)[0] == 0, (dt, tensor)
    assert plan.lib.b200_matmul_grouped_quantized_fp8(plan.ctx, None, None, None, OFFS, 2, F32, OUT, 4, 4, 64) == INVALID


def test_empty_calls_are_no_ops(plan):
    for shape in ((0, 4, 4, 128), (2, 0, 4, 128), (2, 4, 0, 128)):
        assert plan.run(E4B128, E4B128, *shape) == (0, "")
    # nothing is read or written: null pointers pass
    assert plan.run(E4T, E4T, 0, 4, 4, 64, va=0, vb=0, out=0, offs=0) == (0, "")
    assert plan.run(E4T, E4T, 2, 0, 4, 64, va=0, vb=0, out=0, offs=0) == (0, "")


def test_python_entry_point_defers_errors():
    from cubecl_b200 import matmul

    class _Stub:
        def __init__(self):
            self.errors = []

        def _defer(self, e):
            self.errors.append(e)

    class _T:
        def __init__(self, shape, dtype="i32"):
            self.shape, self.dtype = shape, dtype

        def is_contiguous(self):
            return True

    stub = _Stub()
    offs = _T([4])
    matmul.launch_grouped_quantized_fp8(stub, _T([16, 64]), _T([4, 8, 64, 1]), offs, _T([16, 8]))    # rank of qw
    matmul.launch_grouped_quantized_fp8(stub, _T([16, 64]), _T([4, 8, 32]), offs, _T([16, 8]))       # K mismatch
    matmul.launch_grouped_quantized_fp8(stub, _T([16, 64]), _T([4, 8, 64]), _T([4], "i64"), _T([16, 8]))
    matmul.launch_grouped_quantized_fp8(stub, _T([16, 64]), _T([3, 8, 64]), offs, _T([16, 8]))       # groups
    matmul.launch_grouped_quantized_fp8(stub, _T([16, 64]), _T([4, 8, 64]), offs, _T([16, 9]))       # out shape
    assert [e.status for e in stub.errors] == [INVALID] * 5
    assert all("matmul_grouped_quantized_fp8" in str(e) for e in stub.errors)
    assert "K mismatch" in str(stub.errors[1]) and "i32" in str(stub.errors[2]) and "out must be contiguous" in str(stub.errors[4])


# ---------------------------------------------------------------------------------------------- kernels
def _tool(name):
    t = shutil.which(name) or (f"/usr/local/cuda/bin/{name}" if Path(f"/usr/local/cuda/bin/{name}").exists() else None)
    if t is None:
        pytest.skip(f"{name} is not installed")
    return t


def test_grouped_fp8_kernels_use_fp8_wgmma_and_tma_and_do_not_spill():
    tool = _tool("cuobjdump")
    _ffi.load()   # builds the cubins when they are missing
    cubin = ROOT / "cubecl_b200" / "build" / "gemm_grouped_qf8.cubin"
    out = subprocess.run([tool, "-res-usage", str(cubin)], capture_output=True, text=True, check=True).stdout
    funcs = re.findall(r"Function (\w+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)
    assert {f for f, *_ in funcs} == {f"gemm_grouped_qf8_{v}_{o}_{t}_kk" for v in ("e4m3", "e5m2") for o in ("bf16", "f16", "f32")
                                      for t in ("2sm_n128", "1sm_n128")}
    for name, reg, stack, local in funcs:
        assert int(reg) <= 168 and int(stack) == 0 and int(local) == 0, (name, reg, stack, local)
    sass = subprocess.run([tool, "-sass", str(cubin)], capture_output=True, text=True, check=True).stdout
    bodies = re.split(r"\n\s*Function : ", sass)[1:]
    assert len(bodies) == 12
    for body in bodies:
        name = body.split()[0]
        lhs = "E4M3" if "_e4m3_" in name else "E5M2"
        for rhs in ("E4M3", "E5M2"):   # the rhs format of a mixed pair is chosen at run time
            assert re.search(rf"QGMMA\.64x(64|128)x32\.F32\.{lhs}\.{rhs}", body), (name, rhs)
        assert "UTMALDG" in body, name
        assert not re.search(r"\b[IH]GMMA\b", body), name
        assert not re.search(r"\bSTL\b|\bLDL\b", body), name   # no spill stores or loads
