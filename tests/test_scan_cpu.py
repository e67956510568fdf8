"""CPU: the axis scans' oracle against the reference's plane-scan vectors, and the host plans of b200_scan (validation,
view handling, single-pass vs three-pass choice, tile geometry) through a dry-run planning context."""
import json
from pathlib import Path

import numpy as np
import pytest

from cubecl_b200 import _ffi
from plan_context import PlanContext
from scan_oracle import scan_axis_f32, scan_axis_f64

F32, F16, BF16, U32 = _ffi.F32, _ffi.F16, _ffi.BF16, _ffi.U32
SUM, PROD, MAX, MIN, ARGMAX, MEAN = _ffi.REDUCE_SUM, _ffi.REDUCE_PROD, _ffi.REDUCE_MAX, _ffi.REDUCE_MIN, _ffi.REDUCE_ARGMAX, _ffi.REDUCE_MEAN
A, O = 0x10000000, 0x30000000


@pytest.fixture(scope="module")
def scan_golden():
    """The reference's plane-scan vectors (tests/golden/make_scan_golden.py)."""
    return json.loads((Path(__file__).resolve().parent / "golden" / "scan_golden.json").read_text())


class Planner(PlanContext):
    def scan(self, op, dt, shape, axis, strides=None, odt=F32, exclusive=False, a=A, o=O):
        rc = self.lib.b200_scan(self.ctx, None, op, int(exclusive), dt, odt, a, o, len(shape), _ffi.u64_array(shape),
                                _ffi.u64_array(strides) if strides else None, axis)
        return rc, self.text()


@pytest.fixture
def plan():
    with Planner() as p:
        yield p


def launches(text):
    return [ln.split()[1] for ln in text.splitlines() if ln.startswith("launch")]


# ---------------------------------------------------------------------------------------------- oracle vs the reference
@pytest.mark.parametrize("kind", ["inclusive_sum", "exclusive_sum", "inclusive_prod", "exclusive_prod"])
@pytest.mark.parametrize("vec", [1, 2, 4])
def test_oracle_matches_the_reference_plane_scans(scan_golden, kind, vec):
    g = scan_golden[f"plane_{kind}"]
    assert vec in g["vec_sizes"] and g["epsilon"] == 1e-5
    n = 32 * vec
    if g["generator"] == "index":
        x = np.arange(n, dtype=np.float32)
    else:
        x = np.array([(0.5, 1.25, 1.75)[i % 3] for i in range(n)], dtype=np.float32)
    got = scan_axis_f32(x.reshape(32, vec), 0, g["op"], g["exclusive"]).ravel()
    exp = np.array(g["expected"][str(vec)], dtype=np.float32)
    # assert_equals_approx (runtime_tests/binary.rs:15-53) at the stored epsilon, f32
    assert np.all(np.abs(got - exp) < np.maximum(g["epsilon"] * np.abs(exp), g["epsilon"]))
    if g["op"] == "sum":
        assert got.tolist() == exp.tolist()     # integer prefixes: exact in any order
    if kind == "exclusive_sum" and vec == 1:
        assert got[:4].tolist() == [0, 0, 1, 3] and got[-1] == 465


def test_serial_scan_agrees_with_f64_on_integers():
    x = (np.arange(3 * 1000) % 8).astype(np.float32).reshape(3, 1000)
    for axis in (0, 1):
        for exclusive in (False, True):
            f32 = scan_axis_f32(x, axis, "sum", exclusive)
            f64, fabs = scan_axis_f64(x, axis, "sum", exclusive)
            assert np.array_equal(f32.astype(np.float64), f64) and np.array_equal(fabs, f64)
    assert scan_axis_f32(np.array([3, np.nan, 1, 5], np.float32), 0, "max").tolist()[:1] == [3.0]
    assert np.isnan(scan_axis_f32(np.array([3, np.nan, 1, 5], np.float32), 0, "max")[1:]).all()
    assert scan_axis_f32(np.array([3, 1, 5], np.float32), 0, "min", exclusive=True).tolist() == [np.inf, 3.0, 1.0]


# ---------------------------------------------------------------------------------------------- dry-run plans
def test_single_pass_plans(plan):
    # rows: 8192 elements per row = 512 chunks of 16 -> 128 threads per row (four tiles each), a block per row
    rc, t = plan.scan(SUM, F32, [8192, 8192], 1)
    assert rc == 0 and t == "launch scan_rows_sum_f32 grid=(8192,1,1) block=128 smem=0 cluster=1\n"
    # columns: 2^22 / 4 vector units in 256-unit blocks, each thread walks the 64 rows of its unit
    rc, t = plan.scan(SUM, F32, [64, 1 << 22], 0)
    assert rc == 0 and t == "launch scan_cols_sum_f32 grid=(4096,1,1) block=256 smem=0 cluster=1\n"
    # short rows: one thread per row, 256 rows per block
    rc, t = plan.scan(SUM, F32, [1000, 3], 1)
    assert rc == 0 and t == "launch scan_rows_sum_f32 grid=(4,1,1) block=256 smem=0 cluster=1\n"
    rc, t = plan.scan(SUM, F32, [1 << 26, 4], 1)
    assert rc == 0 and t == "launch scan_rows_sum_f32 grid=(262144,1,1) block=256 smem=0 cluster=1\n"
    # dtype suffixes: f32 output has none, a 16-bit output names its dtype
    rc, t = plan.scan(MAX, BF16, [8192, 8192], 1, odt=BF16)
    assert rc == 0 and launches(t) == ["scan_rows_max_bf16_bf16"]
    rc, t = plan.scan(MIN, F16, [64, 1 << 22], 0)
    assert rc == 0 and launches(t) == ["scan_cols_min_f16"]


def test_three_pass_plans(plan):
    # [8192, 8192] along axis 0: 2048 vector units = 8 column blocks; the axis is cut into 128 segments of 64 rows:
    # reduce first pass -> exclusive scan of the [128, 8192] partials -> the segments from their carries
    rc, t = plan.scan(SUM, F32, [8192, 8192], 0)
    assert rc == 0
    assert t == ("alloc 4194304\nalloc 4194304\n"
                 "launch reduce_cols_sum_f32_n8 grid=(1056,1,1) block=256 smem=0 cluster=1\n"
                 "launch scan_cols_sum_f32 grid=(8,1,1) block=256 smem=0 cluster=1 pdl\n"
                 "launch scan_cols_sum_f32 grid=(1024,1,1) block=256 smem=0 cluster=1 pdl\n")
    # rank 1, 2^28: 2106 segments of 127488 elements (16 per SM, 512-aligned); the partials fit one 64-thread item
    rc, t = plan.scan(SUM, F32, [1 << 28], 0)
    assert rc == 0
    assert t == ("alloc 8704\nalloc 8704\n"
                 "launch reduce_rows_sum_f32 grid=(2106,1,1) block=512 smem=0 cluster=1\n"
                 "launch scan_rows_sum_f32 grid=(1,1,1) block=64 smem=0 cluster=1 pdl\n"
                 "launch scan_rows_sum_f32 grid=(2106,1,1) block=512 smem=0 cluster=1 pdl\n")
    # few long rows: 4 x 521 segments
    rc, t = plan.scan(PROD, F32, [4, 1 << 24], 1, exclusive=True)
    assert rc == 0 and launches(t) == ["reduce_rows_prod_f32", "scan_rows_prod_f32", "scan_rows_prod_f32"]
    assert "scan_rows_prod_f32 grid=(2084,1,1) block=512" in t and t.count("alloc") == 2 and t.count(" pdl") == 2
    # few outputs on a long column axis: one 32-unit block, 1056 segments
    rc, t = plan.scan(SUM, F32, [1 << 20, 4], 0)
    assert rc == 0 and launches(t) == ["reduce_cols_sum_f32_n8", "scan_cols_sum_f32", "scan_cols_sum_f32"]
    assert "scan_cols_sum_f32 grid=(1056,1,1) block=32 smem=0 cluster=1 pdl" in t
    # 16-bit input: the partials and carries are f32, only the last launch reads the input and writes its dtype
    rc, t = plan.scan(SUM, BF16, [1 << 28], 0, odt=BF16)
    assert rc == 0 and launches(t) == ["reduce_rows_sum_bf16", "scan_rows_sum_f32", "scan_rows_sum_bf16_bf16"]


def test_views(plan):
    # pitched rows (TensorHandle::empty) are scanned in place along both axes
    rc, t = plan.scan(SUM, F32, [100, 72], 0, strides=[128, 1])
    assert rc == 0 and t == "launch scan_cols_sum_f32 grid=(1,1,1) block=32 smem=0 cluster=1\n"
    rc, t = plan.scan(SUM, F32, [100, 72], 1, strides=[128, 1])
    assert rc == 0 and t == "launch scan_rows_sum_f32 grid=(1,1,1) block=256 smem=0 cluster=1\n"
    # the output is logical row-major: a transposed or permuted view is gathered first
    rc, t = plan.scan(SUM, F32, [72, 100], 0, strides=[1, 72])
    assert rc == 0 and t.splitlines()[0] == "alloc 29184" and launches(t) == ["gather_strided", "scan_cols_sum_f32"]
    rc, t = plan.scan(SUM, F32, [3, 5, 7], 1, strides=[35, 1, 5])
    assert rc == 0 and launches(t) == ["gather_strided", "scan_cols_sum_f32"]
    rc, t = plan.scan(SUM, F32, [3, 5, 7], 2, strides=[35, 1, 5])
    assert rc == 0 and launches(t) == ["gather_strided", "scan_rows_sum_f32"]
    # contiguous strides spelled out are the contiguous plan
    rc, t = plan.scan(SUM, F32, [3, 5, 7], 1, strides=[35, 7, 1])
    assert rc == 0 and launches(t) == ["scan_cols_sum_f32"]


def test_validation(plan):
    assert plan.scan(ARGMAX, F32, [4], 0)[0] == 7
    assert plan.scan(MEAN, F32, [4], 0)[0] == 7
    assert plan.scan(SUM, F32, [4], 0, odt=U32)[0] == 6
    assert plan.scan(SUM, F32, [4], 0, odt=F16)[0] == 6          # f32 input: f32 output only
    assert plan.scan(SUM, F16, [4], 0, odt=BF16)[0] == 6
    assert plan.scan(SUM, F32, [4, 4], -1)[0] == 6
    assert plan.scan(SUM, F32, [4, 4], 2)[0] == 6
    assert plan.scan(SUM, U32, [4], 0)[0] == 7
    assert plan.scan(SUM, F32, [4], 0, a=0)[0] == 6
    assert plan.scan(SUM, F32, [4], 0, a=A + 2)[0] == 6          # not element aligned
    assert plan.scan(SUM, F32, [4] * 9, 0)[0] == 6
    for shape in ([4, 0], [0, 4], [0]):
        rc, t = plan.scan(SUM, F32, shape, 0)
        assert rc == 0 and t == ""
    assert plan.scan(SUM, F32, [4, 0], 1, a=0, o=0) == (0, "")      # an empty scan touches no pointer
    # an element-aligned (not 16-byte aligned) base is planned like an aligned one: the kernel peels the head
    rc, t = plan.scan(SUM, F32, [8192, 8192], 1, a=A + 4)
    assert rc == 0 and launches(t) == ["scan_rows_sum_f32"]
