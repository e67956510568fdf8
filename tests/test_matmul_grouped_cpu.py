"""CPU: the grouped-matmul oracle (pinned to torch's CPU grouped_mm in both offset modes), the dry-run plans of
b200_matmul_grouped (kernel names, grid bounds, clusters, shared memory and tensor maps for both modes, all four ragged-M
layouts, both tiles and both out dtypes), the tile policy and the gemm.variant override, every refusal, zero extents, the
Python layer's deferred errors and the SASS of the grouped kernels."""
import ctypes as C
import re
import subprocess

import numpy as np
import pytest
import torch

import grouped_mm_oracle as gmo
from cubecl_b200 import _ffi, matmul
from plan_context import PlanContext
from test_conv_cpu import ROOT, _tool

F32, F16, BF16, F8E4M3 = _ffi.F32, _ffi.F16, _ffi.BF16, _ffi.F8E4M3
LHS, RHS, OFFS, OUT, BIAS = 0x10000000, 0x20000000, 0x30000000, 0x40000000, 0x50000000
INVALID, UNSUPPORTED = 6, 7
SMS = 132                                               # H100 SXM
SMEM = 1024 + 6 * (16384 + 128 * 128) + 1024 + 16384 + (2 * 1024 + 4) * 4   # GEMM ring + staging + the offset table


# ---------------------------------------------------------------------------------------------- oracle
SIZE_LISTS = {
    "empty_groups": [0, 5, 0, 0, 17, 3, 0],
    "one_group": [37],
    "all_rows_in_one": [0, 0, 40, 0],
    "rows_past_the_end": [4, 9, 2],     # T is larger than the sum: the last rows belong to no group
    "edges": [1, 63, 64, 65, 0, 2],
}


@pytest.mark.parametrize("case", sorted(SIZE_LISTS))
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_oracle_matches_torch_grouped_mm(case, dtype):
    sizes = SIZE_LISTS[case]
    G, K, N, M = len(sizes), 24, 16, 16   # torch wants 16-byte strides
    T = sum(sizes) + (7 if case == "rows_past_the_end" else 0)
    offs = gmo.offsets(sizes)
    rng = np.random.default_rng(len(case))
    # integer values: every product and sum is exact, so torch and the oracle agree bit for bit
    a = rng.integers(-4, 5, (T, K)).astype(np.float64)
    b = rng.integers(-4, 5, (G, K, N)).astype(np.float64)
    ot = torch.tensor(offs)
    got = torch.nn.functional.grouped_mm(torch.tensor(a).to(dtype), torch.tensor(b).to(dtype), offs=ot).double().numpy()
    want, written = gmo.ragged_m(a, b, offs)
    assert written.sum() == sum(sizes)
    np.testing.assert_array_equal(got[written], want[written])
    x = rng.integers(-4, 5, (T, M)).astype(np.float64)
    dy = rng.integers(-4, 5, (T, N)).astype(np.float64)
    got_k = torch.nn.functional.grouped_mm(torch.tensor(x).to(dtype).t(), torch.tensor(dy).to(dtype), offs=ot).double().numpy()
    want_k = gmo.ragged_k(x.T, dy, offs)
    np.testing.assert_array_equal(got_k, want_k)
    for g, n in enumerate(sizes):
        if n == 0:
            assert not want_k[g].any()


def test_oracle_matches_torch_on_random_data():
    rng = np.random.default_rng(5)
    sizes = [30, 0, 71, 12]
    offs, T, K, N = gmo.offsets(sizes), sum(sizes), 40, 24
    a, b = rng.uniform(-1, 1, (T, K)), rng.uniform(-1, 1, (4, K, N))
    ta, tb = torch.tensor(a).bfloat16(), torch.tensor(b).bfloat16()
    got = torch.nn.functional.grouped_mm(ta, tb, offs=torch.tensor(offs)).double().numpy()
    want, _ = gmo.ragged_m(ta.double().numpy(), tb.double().numpy(), offs)
    np.testing.assert_allclose(got, want, rtol=1e-2, atol=1e-2)


def test_clamping_rule():
    assert gmo.clamp_offsets([5, 3, 9, -2, 100], 50).tolist() == [5, 5, 9, 9, 50]
    assert gmo.bounds([-4, 3, 2], 10) == [(0, 0), (0, 3), (3, 3)]


# ---------------------------------------------------------------------------------------------- dry-run plans
class Planner(PlanContext):
    def run(self, ls, rs, os_, groups=None, lst=None, rst=None, ost=None, idt=BF16, odt=BF16, ptrs=(LHS, RHS, OFFS, OUT), ep=None):
        arr = lambda v: _ffi.u64_array(v) if v is not None else None  # noqa: E731
        if groups is None:
            groups = rs[0] if len(rs) == 3 else os_[0]
        rc = self.lib.b200_matmul_grouped(self.ctx, None, idt, odt, ptrs[0], len(ls), arr(ls), arr(lst), ptrs[1], len(rs), arr(rs),
                                          arr(rst), ptrs[2], groups, ptrs[3], len(os_), arr(os_), arr(ost),
                                          C.byref(ep) if ep is not None else None)
        return rc, self.text()


@pytest.fixture
def plan():
    with Planner() as p:
        yield p


def _launches(t):
    return re.findall(r"^launch (\S+) grid=\((\d+),1,1\) block=(\d+) smem=(\d+) cluster=(\d+)$", t, re.M)


def _tmaps(t):
    return re.findall(r"^tmap esz=(\d+) dims=\(([\d,]+)\) strides=\(([\d,]+)\) box=\(([\d,]+)\)", t, re.M)


def _ints(s):
    return tuple(int(v) for v in s.split(","))


# ragged-M layouts: (lhs strides of [T, K], rhs strides of [G, K, N]) for a = k (K-major) / m, b = n (N-contiguous) / k
def _rm_strides(layout, T, K, N, G):
    lst = [K, 1] if layout[0] == "k" else [1, T]
    rst = [K * N, N, 1] if layout[1] == "n" else [N * K, 1, K]
    return lst, rst


@pytest.mark.parametrize("tile", ["2sm_n128", "1sm_n128"])
@pytest.mark.parametrize("odt", ["bf16", "f32"])
@pytest.mark.parametrize("layout", ["kn", "kk", "mn", "mk"])
def test_ragged_m_plan(plan, tile, odt, layout):
    T, K, N, G = 8192, 1024, 768, 8
    plan.option("gemm.variant", tile)
    lst, rst = _rm_strides(layout, T, K, N, G)
    rc, t = plan.run([T, K], [G, K, N], [T, N], lst=lst, rst=rst, odt=F32 if odt == "f32" else BF16)
    assert rc == 0, (t, _ffi.load().b200_last_error())
    cg = 2 if tile.startswith("2sm") else 1
    rows, tiles_n = 128 * cg, (N + 127) // 128
    span = T + (63 * G if layout[0] == "m" else 0)    # an M-contiguous lhs: tile-rows start at 64-row boundaries
    bound = ((span + rows - 1) // rows + G) * tiles_n
    assert f"gemm grouped ragged_m groups={G} T={T} tile_rows<={bound // tiles_n} tiles<={bound}" in t, t
    [(name, grid, block, smem, cluster)] = _launches(t)
    assert name == f"gemm_grouped_m_bf16_{odt}_{tile}_{layout}"
    assert int(grid) == min(bound, SMS // cg) * cg and block == "384" and int(smem) == SMEM and int(cluster) == cg
    maps = _tmaps(t)
    assert len(maps) == 3, t
    a_map = ("2", (K, T, 1), (K * 2, K * T * 2), (64, 128)) if layout[0] == "k" else ("2", (T, K, 1), (T * 2, T * K * 2), (64, 64))
    b_map = (("2", (N, K, G), (N * 2, K * N * 2), (64, 64)) if layout[1] == "n"
             else ("2", (K, N, G), (K * 2, N * K * 2), (64, 128 // cg)))
    osz = 4 if odt == "f32" else 2
    o_map = (str(osz), (N, T, 1), (N * osz, N * T * osz), (128 // osz, 64))
    got = [(e, _ints(d), _ints(s), _ints(b)) for e, d, s, b in maps]
    assert got == [a_map, b_map, o_map], got


@pytest.mark.parametrize("tile", ["2sm_n128", "1sm_n128"])
@pytest.mark.parametrize("odt", ["bf16", "f32"])
def test_ragged_k_plan(plan, tile, odt):
    M, T, N, G = 1024, 16384, 768, 8
    plan.option("gemm.variant", tile)
    rc, t = plan.run([M, T], [T, N], [G, M, N], lst=[1, M], odt=F32 if odt == "f32" else BF16)
    assert rc == 0, (t, _ffi.load().b200_last_error())
    cg = 2 if tile.startswith("2sm") else 1
    bound = G * ((M + 128 * cg - 1) // (128 * cg)) * ((N + 127) // 128)
    assert f"gemm grouped ragged_k groups={G} T={T} tile_rows<={bound // 6} tiles<={bound}" in t, t
    [(name, grid, block, smem, cluster)] = _launches(t)
    assert name == f"gemm_grouped_k_bf16_{odt}_{tile}"
    assert int(grid) == min(bound, SMS // cg) * cg and int(smem) == SMEM and int(cluster) == cg
    osz = 4 if odt == "f32" else 2
    got = [(e, _ints(d), _ints(s), _ints(b)) for e, d, s, b in _tmaps(t)]
    assert got == [("2", (M, T, 1), (M * 2, M * T * 2), (64, 64)), ("2", (N, T, 1), (N * 2, N * T * 2), (64, 64)),
                   (str(osz), (N, M, G), (N * osz, M * N * osz), (128 // osz, 64))], got


def test_plans_never_depend_on_offsets(plan):
    """the host reads no offset: two calls with different offs pointers plan the same launch"""
    _, t1 = plan.run([4096, 512], [8, 512, 512], [4096, 512])
    _, t2 = plan.run([4096, 512], [8, 512, 512], [4096, 512], ptrs=(LHS, RHS, OFFS + 4096, OUT))
    assert t1 == t2 and len(_launches(t1)) == 1


@pytest.mark.parametrize("T,G,M,want", [
    (32768, 32, None, "2sm_n128"), (32768, 8, None, "2sm_n128"), (32768, 128, None, "1sm_n128"), (1024, 1, None, "2sm_n128"),
    (1023, 1, None, "1sm_n128"), (16384, 256, None, "1sm_n128"),
    (32768, 32, 7168, "2sm_n128"), (32768, 128, 2048, "1sm_n128"), (32768, 8, 128, "1sm_n128"),
])
def test_tile_policy(plan, T, G, M, want):
    """fewer than 1024 rows per group on average: the 128-row tile (less padding at each group's end); ragged K with M <= 128
    would idle half of a pair"""
    if M is None:
        rc, t = plan.run([T, 256], [G, 256, 256], [T, 256])
    else:
        rc, t = plan.run([M, T], [T, 256], [G, M, 256], lst=[1, M])
    assert rc == 0 and want in _launches(t)[0][0], t


def test_variant_override(plan):
    for v in ("2sm_n128", "1sm_n128"):
        plan.option("gemm.variant", v)
        rc, t = plan.run([32768, 256], [128, 256, 256], [32768, 256])
        assert rc == 0 and v in _launches(t)[0][0], t
    for v in ("2sm_n256", "simt", "bogus"):
        plan.option("gemm.variant", v)
        rc, _ = plan.run([32768, 256], [128, 256, 256], [32768, 256])
        assert rc == INVALID and "grouped matmul tile" in _ffi.load().b200_last_error().decode()
    plan.option("gemm.variant", "auto")
    plan.option("gemm.epilogue", "direct")
    rc, t = plan.run([4096, 256], [4, 256, 256], [4096, 256])
    assert rc == 0 and len(_tmaps(t)) == 2, t       # no out map: every tile stores directly
    plan.option("gemm.epilogue", "bogus")
    assert plan.run([4096, 256], [4, 256, 256], [4096, 256])[0] == INVALID


def test_split_k_option_does_not_apply(plan):
    _, t0 = plan.run([4096, 512], [8, 512, 512], [4096, 512])
    plan.option("gemm.split_k", "on")
    _, t1 = plan.run([4096, 512], [8, 512, 512], [4096, 512])
    assert t0 == t1 and "stream-k" not in t1


def test_views_tma_cannot_read_are_staged_and_out_is_not(plan):
    # lhs rows of 1000 bf16 elements in a 1001-element pitch: staged once, then the grouped kernel
    rc, t = plan.run([4096, 1000], [4, 1000, 512], [4096, 512], lst=[1001, 1])
    assert rc == 0 and [n for n, *_ in _launches(t)] == ["repitch_rows", "gemm_grouped_m_bf16_bf16_2sm_n128_kn"], t
    # a ragged-K rhs with a misaligned pitch is staged N-contiguous
    rc, t = plan.run([512, 4096], [4096, 500], [4, 512, 500], lst=[1, 512], rst=[501, 1])
    assert rc == 0 and [n for n, *_ in _launches(t)] == ["repitch_rows", "gemm_grouped_k_bf16_bf16_2sm_n128"], t
    # out is written in place whatever its pitch: 16-byte aligned rows also leave through the TMA store, others do not
    rc, t = plan.run([4096, 512], [4, 512, 504], [4096, 504], ost=[512, 1])
    assert rc == 0 and len(_launches(t)) == 1 and len(_tmaps(t)) == 3, t
    rc, t = plan.run([4096, 512], [4, 512, 504], [4096, 504], ost=[505, 1])
    assert rc == 0 and len(_launches(t)) == 1 and len(_tmaps(t)) == 2, t   # rows not 16-byte aligned: no TMA store


def test_broadcast_rhs_is_one_map_batch(plan):
    rc, t = plan.run([4096, 512], [4, 512, 256], [4096, 256], rst=[0, 256, 1])
    assert rc == 0, t
    assert _ints(_tmaps(t)[1][1]) == (256, 512, 1), t


def test_zero_extents(plan):
    for args in (([0, 64], [0, 64, 64], [0, 64]),          # no groups
                 ([0, 64], [4, 64, 64], [0, 64]),          # no rows
                 ([128, 64], [4, 64, 0], [128, 0]),        # no columns
                 ([0, 256], [256, 64], [4, 0, 64], dict(lst=[1, 1]))):   # ragged K, M = 0
        kw = args[3] if len(args) > 3 else {}
        rc, t = plan.run(*args[:3], **kw)
        assert rc == 0 and t == "", (args, t, _ffi.load().b200_last_error())
    # K = 0 (ragged M) or T = 0 (ragged K): one launch that stores act(bias) or +0, with no operand map
    rc, t = plan.run([256, 0], [4, 0, 64], [256, 64], ptrs=(0, 0, OFFS, OUT))
    assert rc == 0 and len(_launches(t)) == 1 and len(_tmaps(t)) == 1, t
    rc, t = plan.run([64, 0], [0, 64], [4, 64, 64], lst=[1, 64], ptrs=(0, 0, OFFS, OUT))
    assert rc == 0 and len(_launches(t)) == 1 and len(_tmaps(t)) == 1, t


# every refusal: (case, status, words of the message)
REFUSALS = [
    ("rank_1_lhs", INVALID, "ranks"), ("rank_out", INVALID, "ranks"), ("3x3", UNSUPPORTED, "b200_matmul"),
    ("3x2", UNSUPPORTED, "ragged N"), ("f32_inputs", UNSUPPORTED, "input dtype"), ("fp8_inputs", UNSUPPORTED, "input dtype"),
    ("f16_out_of_bf16", UNSUPPORTED, "output dtype"), ("offs_null", INVALID, "null offs"),
    ("offs_misaligned", INVALID, "offs is misaligned"), ("groups_mismatch_m", INVALID, "groups in offs"),
    ("groups_mismatch_k", INVALID, "groups in offs"), ("groups_over_cap", UNSUPPORTED, "limit of 1024"),
    ("k_mismatch", INVALID, "inner dimensions differ"), ("n_mismatch", INVALID, "output is"), ("t_mismatch", INVALID, "output is"),
    ("rk_t_mismatch", INVALID, "inner dimensions differ"), ("rk_out_shape", INVALID, "output is"),
    ("rk_k_major_lhs", UNSUPPORTED, "K-major"), ("rk_k_major_rhs", UNSUPPORTED, "K-major"), ("rk_epilogue", UNSUPPORTED, "epilogue"),
    ("activation", INVALID, "activation"), ("null_lhs", INVALID, "null device pointer"), ("misaligned_out", INVALID, "misaligned"),
    ("misaligned_lhs", INVALID, "misaligned"), ("misaligned_bias", INVALID, "misaligned bias"),
    ("out_column_stride", UNSUPPORTED, "unit column stride"), ("extent", UNSUPPORTED, "2^31"), ("cta_bound", UNSUPPORTED, "too many tiles"),
]


@pytest.mark.parametrize("case,status,words", REFUSALS, ids=[r[0] for r in REFUSALS])
def test_refusals(plan, case, status, words):
    T, K, N, G, M = 4096, 256, 512, 4, 384
    rm = dict(ls=[T, K], rs=[G, K, N], os_=[T, N])
    rk = dict(ls=[M, T], rs=[T, N], os_=[G, M, N], lst=[1, M])
    kw = dict(rm)
    if case == "rank_1_lhs":
        kw["ls"] = [T]
    elif case == "rank_out":
        kw["os_"] = [1, T, N]
    elif case == "3x3":
        kw.update(ls=[G, T, K])
    elif case == "3x2":
        kw.update(ls=[G, T, K], rs=[K, N], groups=G)
    elif case == "f32_inputs":
        kw.update(idt=F32, odt=F32)
    elif case == "fp8_inputs":
        kw.update(idt=F8E4M3, odt=F32)
    elif case == "f16_out_of_bf16":
        kw["odt"] = F16
    elif case == "offs_null":
        kw["ptrs"] = (LHS, RHS, 0, OUT)
    elif case == "offs_misaligned":
        kw["ptrs"] = (LHS, RHS, OFFS + 2, OUT)
    elif case == "groups_mismatch_m":
        kw["groups"] = G + 1
    elif case == "groups_mismatch_k":
        kw = dict(rk, groups=G - 1)
    elif case == "groups_over_cap":
        kw.update(rs=[1025, K, N])
    elif case == "k_mismatch":
        kw["rs"] = [G, K + 8, N]
    elif case == "n_mismatch":
        kw["os_"] = [T, N + 8]
    elif case == "t_mismatch":
        kw["os_"] = [T - 1, N]
    elif case == "rk_t_mismatch":
        kw = dict(rk, rs=[T + 1, N])
    elif case == "rk_out_shape":
        kw = dict(rk, os_=[G, M + 1, N])
    elif case == "rk_k_major_lhs":
        kw = dict(rk, lst=[T, 1])
    elif case == "rk_k_major_rhs":
        kw = dict(rk, rst=[1, T])
    elif case == "rk_epilogue":
        kw = dict(rk, ep=_ffi.Epilogue(2.0, 0, 0))
    elif case == "activation":
        kw["ep"] = _ffi.Epilogue(1.0, 5, 0)
    elif case == "null_lhs":
        kw["ptrs"] = (0, RHS, OFFS, OUT)
    elif case == "misaligned_out":
        kw["ptrs"] = (LHS, RHS, OFFS, OUT + 1)
    elif case == "misaligned_lhs":
        kw["ptrs"] = (LHS + 1, RHS, OFFS, OUT)
    elif case == "misaligned_bias":
        kw["ep"] = _ffi.Epilogue(1.0, 0, BIAS + 2)
    elif case == "out_column_stride":
        kw["ost"] = [1, T]
    elif case == "extent":
        kw.update(ls=[1 << 31, K], os_=[1 << 31, N])
    elif case == "cta_bound":       # (2^31 / 128 + 1024) tile-rows x 2^24 column tiles
        n = (1 << 31) - 8
        kw.update(ls=[(1 << 31) - 1, 64], rs=[1024, 64, n], os_=[(1 << 31) - 1, n])
    rc, t = plan.run(**kw)
    msg = _ffi.load().b200_last_error().decode()
    assert rc == status, (case, rc, msg, t)
    assert words in msg and "launch" not in t, (case, msg, t)


def test_python_layer_defers_errors():
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
    a, b, o, offs = _T([64, 32]), _T([4, 32, 16]), _T([64, 16]), _T([4], "i32")
    matmul.launch_grouped(stub, a, _T([4, 32, 16], "f16"), offs, o)                   # dtype mismatch
    matmul.launch_grouped(stub, a, b, _T([4], "i64"), o)                              # offs not i32
    matmul.launch_grouped(stub, a, b, _T([4], "i32", contiguous=False), o)            # offs not compact
    matmul.launch_grouped(stub, a, b, _T([2, 2], "i32"), o)                           # offs not 1-D
    matmul.launch_grouped(stub, a, b, offs, o, bias=_T([16], "f32"))                  # bias not [G, N]
    matmul.launch_grouped(stub, a, b, offs, o, activation="tanh")                     # unknown activation
    assert [e.status for e in stub.errors] == [INVALID] * 6
    msgs = [str(e) for e in stub.errors]
    assert "dtype" in msgs[0] and all("offs" in m for m in msgs[1:4]) and "bias" in msgs[4] and "activation" in msgs[5]


def test_output_shape_rule():
    assert matmul.calculate_grouped_output([100, 64], [8, 64, 32], 8) == [100, 32]
    assert matmul.calculate_grouped_output([48, 100], [100, 32], 8) == [8, 48, 32]
    for args in (([100, 64], [8, 63, 32], 8), ([100, 64], [8, 64, 32], 7), ([48, 100], [99, 32], 8), ([2, 3, 4], [2, 4, 5], 2)):
        with pytest.raises(matmul.MatmulShapeError):
            matmul.calculate_grouped_output(*args)


# ---------------------------------------------------------------------------------------------- kernels
def test_grouped_kernels_use_wgmma_and_tma_and_do_not_spill():
    tool = _tool("cuobjdump")
    _ffi.load()
    cubin = ROOT / "cubecl_b200" / "build" / "gemm_grouped.cubin"
    out = subprocess.run([tool, "-res-usage", str(cubin)], capture_output=True, text=True, check=True).stdout
    funcs = re.findall(r"Function (\w+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)
    io = (("bf16", "bf16"), ("bf16", "f32"), ("f16", "f16"), ("f16", "f32"))
    tiles = ("2sm_n128", "1sm_n128")
    want = {f"gemm_grouped_m_{i}_{o}_{t}_{ab}" for i, o in io for t in tiles for ab in ("kn", "kk", "mn", "mk")}
    want |= {f"gemm_grouped_k_{i}_{o}_{t}" for i, o in io for t in tiles}
    assert {f for f, *_ in funcs} == want and len(want) == 40
    for name, reg, stack, local in funcs:
        assert int(stack) == 0 and int(local) == 0, (name, stack, local)
    sass = subprocess.run([tool, "-sass", str(cubin)], capture_output=True, text=True, check=True).stdout
    for body in re.split(r"\n\s*Function : ", sass)[1:]:
        name = body.split()[0]
        assert "HGMMA.64x128x16.F32" in body and "UTMALDG.3D" in body and "UTMASTG.3D" in body, name
