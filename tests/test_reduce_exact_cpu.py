"""CPU: the path coverage of tests/test_reduce_exact_gpu.py, read off dry-run plans of its case lists on an H100's 132 SMs, and
the teeth of its data: each wrong kernel of reduce_exact_oracle.mutants changes at least one expected output of every case."""
import re

import numpy as np
import pytest

import reduce_exact_oracle as ro
import test_reduce_exact_gpu as gpu
from cubecl_b200 import build

CASES = gpu.CASES + gpu.LOADS_CASES

ALL_PATHS = ("all-plain", "all-bulk", "all-bulk-forced", "allp-vec", "allp-scalar")
TUNING_PATHS = tuple(f"all-{v}" for v in ("u2", "u4", "u16", "b4", "b8", "w2", "w4"))
ROW_PATHS = ("rows-1vec", "rows-subwarp", "rows-multiwarp", "rows-block", "rows-big", "rows-misaligned", "rows-2pass")
COL_PATHS = ("cols-vec", "cols-scalar", "cols-vec-walk", "cols-vec-perblock", "cols-strided", "cols-pitched",
             "cols-2pass-wide", "cols-2pass-narrow", "cols-fused")
OTHER_PATHS = ("unit-axis", "gather", "rank8")


def _required():
    cells = set()
    for dt in ro.DTYPES:
        for path in ALL_PATHS + ROW_PATHS + COL_PATHS + OTHER_PATHS:
            ops = ro.VALUE_OPS if path.startswith(("all-bulk",)) else ro.ALL_OPS
            cells |= {(op, dt, path) for op in ops}
        cells |= {(op, dt, "cols-vec-loads4") for op in ro.VALUE_OPS}
        cells |= {(op, dt, "cols-vec-loads8") for op in ro.ARG_OPS}
    cells |= {(op, "f32", path) for path in TUNING_PATHS for op in ("sum", "mean")}
    return cells


@pytest.fixture(scope="module")
def planned():
    """{case: {op: (plan, path)}} for every case of the GPU file."""
    out = {}
    for case in CASES:
        out[case] = {}
        for op in case.ops:
            plan = ro.probe(case, op)
            out[case][op] = (plan, ro.path_of(case, op, plan))
    return out


def _cells(planned, cases):
    return {(op, case.dtype, path) for case in cases for op, (_, path) in planned[case].items()}


def test_every_case_takes_its_path(planned):
    for case, per_op in planned.items():
        paths = {path for _, path in per_op.values()}
        assert case.path in paths, (case.id, paths)


def test_every_op_dtype_path_cell_is_covered(planned):
    missing = _required() - _cells(planned, CASES)
    assert not missing, sorted(missing)


def test_no_case_is_redundant(planned):
    # deleting any one case from the GPU lists loses a required cell
    required = _required()
    for case in CASES:
        rest = _cells(planned, [c for c in CASES if c is not case])
        assert required - rest, f"{case.id} covers no cell the other cases miss"


def _reduce_image_kernels():
    table = (build.BUILD / "cubin_table.inc").read_text()
    images = re.findall(r'^\s*\{"(\w+)", b200_cubin_', table, re.M)
    home = images.index("reduce")
    return {name for name, i in re.findall(r'^\s*\{"(\w+)", (\d+)\},$', table, re.M) if int(i) == home and name.startswith("reduce_")}


def test_every_reduce_kernel_is_reached(planned):
    kernels = _reduce_image_kernels()
    assert "reduce_all_argmax_f32_u8" not in kernels
    reached = {k for per_op in planned.values() for plan, _ in per_op.values() for k in plan.kernels}
    unreached = sorted(k for k in kernels - reached if not k.endswith("_xgpu"))
    assert not unreached, unreached
    assert sorted(k for k in kernels if k.endswith("_xgpu")) == ["reduce_all_argmax_f32_xgpu", "reduce_all_argmin_f32_xgpu",
                                                                  "reduce_all_sum_f32_xgpu"]
    assert reached <= kernels


def test_two_pass_plans_and_segments(planned):
    for case, per_op in planned.items():
        for op, (plan, path) in per_op.items():
            if path == "rows-2pass" or path.startswith("cols-2pass"):
                assert plan.nseg > 1 and len(plan.kernels) == 2, (case.id, op)
                if op in ro.ARG_OPS:
                    assert plan.kernels[1] == "reduce_argcombine"
                else:
                    assert plan.launches[1][3], "the second pass waits on the first through programmatic dependent launch"
            if path == "cols-fused":
                assert plan.fused and len(plan.kernels) == 1
    wide = planned[next(c for c in CASES if c.path == "cols-2pass-wide")]["argmax"][0]
    narrow = planned[next(c for c in CASES if c.path == "cols-2pass-narrow")]["argmax"][0]
    assert wide.nseg >= 8 > narrow.nseg


# ------------------------------------------------------------------------------------------------ teeth
def _needed(case, op, flat, seg_len):
    """The wrong kernels that must change at least one expected output of `op` on the case."""
    L = case.length()
    if op in ro.ARG_OPS and L == 1:                 # the index over a unit axis is 0 whatever the kernel reads
        return {"padding read"} if case.pitch else set()
    need = {f"drop {p}" for p in flat}
    if op in ("sum", "mean", "prod"):
        need |= {f"double {p}" for p in flat}
    if op == "mean" and L > 1:                      # a unit axis has scale 1
        need.add("scale twice")
        if seg_len < L:
            need.add("scale per segment")
    if op in ro.ARG_OPS and L > 1:                  # ... and no ties
        need.add("ties to the higher index")
        if seg_len < L:
            need.add("index not offset by its segment")
    if case.outputs() > 1:
        need.add("outputs shifted by one")
    if case.pitch:
        need.add("padding read")
    return need


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.id)
def test_wrong_kernels_change_an_expected_output(planned, case):
    # checked per op: each op's own expected outputs must catch each wrong kernel of that op
    plan = planned[case][case.ops[0]][0]
    positions = ro.named_positions(case, plan)
    seg_len = ro.seg_len_from_plan(case, max(p.nseg for p, _ in planned[case].values()))
    x0 = ro.base_values(case, 7)
    launches = []
    for r, tie, nan in ro.runs(case, positions):
        xr = ro.plant(x0, positions, r, tie, nan)
        if not nan:
            ro.assert_exact_bound(xr)
            assert np.all(xr != 0)
        launches.append((nan, xr[:64]))   # the first 64 outputs hold an extreme at every named position
    flat = sorted({p for pos in positions for p in pos})
    missed = []
    for op in case.ops:
        caught = {}
        for nan, xr in launches:
            if nan and op not in ("max", "min") + ro.ARG_OPS:
                continue
            want = ro.expected(xr, op)
            for name, wrong in ro.mutants(xr, op, positions, seg_len, padding=bool(case.pitch)):
                caught[name] = caught.get(name, False) or bool((~ro.outputs_equal(wrong, want)).any())
        need = _needed(case, op, flat, seg_len)
        assert need <= set(caught), (op, sorted(need - set(caught)))
        missed += [f"{op}: {n}" for n in sorted(need) if not caught[n]]
    assert not missed, f"{case.id}: these wrong kernels would pass: {missed}"


def test_every_output_has_its_own_extremes():
    # max and min are not constants: outputs differ from each other, and one launch per rotation has no tie
    case = next(c for c in gpu.COL_CASES if c.path == "cols-vec" and c.dtype == "bf16")
    positions = ro.named_positions(case, ro.probe(case, "max"))
    rs = ro.runs(case, positions)
    assert any(not tie for _, tie, _ in rs) and any(nan for *_, nan in rs)
    x0 = ro.base_values(case, 7)
    for r, tie, nan in rs:
        xr = ro.plant(x0, positions, r, tie, nan)
        for op in ("max", "min"):
            vals = ro.expected(xr, op)
            assert len(np.unique(vals[~np.isnan(vals)])) == (4 if nan else 8), (op, r, tie, nan)
            assert np.isnan(vals).any() == nan and not np.isnan(vals).all()
    unit = next(c for c in gpu.OTHER_CASES if c.path == "unit-axis")
    xr = ro.plant(ro.base_values(unit, 7), ro.named_positions(unit, ro.probe(unit, "sum")), 0)
    assert len(np.unique(xr)) > 3                     # a unit axis keeps its varied base values


def test_named_positions_include_the_seams():
    case = next(c for c in gpu.ROW_CASES if c.path == "rows-2pass" and c.dtype == "f32")
    plan = ro.probe(case, "sum")
    seg = ro.seg_len_from_plan(case, plan.nseg)
    assert seg % 512 == 0 and seg == ro.host_seg_len(case)
    pos = ro.named_positions(case, plan)[0]
    mid = plan.nseg // 2
    assert {0, case.length() - 1, mid * seg, (mid + 1) * seg - 1} <= set(pos)
    bulk = next(c for c in gpu.ALL_CASES if c.path == "all-bulk" and c.dtype == "bf16")
    pos = ro.named_positions(bulk, ro.probe(bulk, "sum"))[0]
    head = (16 - bulk.offset * 2) // 2
    assert {head - 1, head + 8192} <= set(pos)       # the last head element and the first element of the second tile
