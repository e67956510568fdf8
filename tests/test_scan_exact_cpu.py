"""CPU: the path coverage of tests/test_scan_exact_gpu.py, read off dry-run plans of its case lists on an H100's 132 SMs, the
preconditions and correctness of its oracle, and the teeth of its data: each wrong kernel of scan_exact_oracle.mutants
changes at least one expected output of every case it applies to."""
import re

import numpy as np
import pytest

import scan_exact_oracle as so
import test_scan_exact_gpu as gpu
from cubecl_b200 import build
from scan_oracle import scan_axis_f64

CASES = gpu.CASES + gpu.LOADS_CASES

ROW_PATHS = ("rows-thread", "rows-subwarp", "rows-warp", "rows-multiwarp", "rows-block", "rows-misaligned", "rows-3pass",
             "rows-3pass-misaligned")
COL_PATHS = ("cols-vec", "cols-scalar", "cols-pitched", "cols-3pass-pitched", "cols-3pass-wide", "cols-3pass-narrow",
             "cols-3pass-scalar", "cols-3pass-loads4")
OTHER_PATHS = ("gather", "rank8", "unit-axis")


def _required():
    return {(op, dt, odt, path) for dt in so.DTYPES for odt in {"f32", dt} for op in so.OPS
            for path in ROW_PATHS + COL_PATHS + OTHER_PATHS}


@pytest.fixture(scope="module")
def planned():
    """{case: {(op, exclusive, out dtype): (plan, path)}} for every case of the GPU file."""
    out = {}
    for case in CASES:
        out[case] = {}
        for op in case.ops:
            for ex in (False, True):
                for odt in case.out_dtypes():
                    plan = so.probe(case, op, ex, odt)
                    out[case][(op, ex, odt)] = (plan, so.path_of(case, plan))
    return out


def _cells(planned, cases):
    return {(op, case.dtype, odt, path) for case in cases for (op, _, odt), (_, path) in planned[case].items()}


def test_every_case_takes_its_path(planned):
    for case, per_call in planned.items():
        assert {path for _, path in per_call.values()} == {case.path}, case.id


def test_every_op_dtype_path_cell_is_covered(planned):
    missing = _required() - _cells(planned, CASES)
    assert not missing, sorted(missing)


def test_no_case_is_redundant(planned):
    required = _required()
    for case in CASES:
        rest = _cells(planned, [c for c in CASES if c is not case])
        assert required - rest, f"{case.id} covers no cell the other cases miss"


def _image_kernels(image):
    table = (build.BUILD / "cubin_table.inc").read_text()
    images = re.findall(r'^\s*\{"(\w+)", b200_cubin_', table, re.M)
    home = images.index(image)
    return {name for name, i in re.findall(r'^\s*\{"(\w+)", (\d+)\},$', table, re.M) if int(i) == home}


def test_every_scan_kernel_is_reached(planned):
    kernels = _image_kernels("reduce")
    scans = {k for k in kernels if k.startswith("scan_")}
    assert len(scans) == 40
    reached = {k for per_call in planned.values() for plan, _ in per_call.values() for k in plan.kernels}
    assert not sorted(scans - reached), sorted(scans - reached)
    # every value-op first pass of the reduce image: rows, and columns with eight and with four loads in flight
    first = {k for k in kernels if re.fullmatch(r"reduce_(rows|cols)_(sum|prod|max|min)_(f32|f16|bf16)(_n8)?", k)}
    assert len(first) == 36
    firsts = {plan.kernels[0] for per_call in planned.values() for plan, _ in per_call.values() if plan.nseg > 1}
    assert not sorted(first - firsts), sorted(first - firsts)
    assert reached <= kernels | {"gather_strided"}


def test_three_pass_plans(planned):
    for case, per_call in planned.items():
        for (op, ex, odt), (plan, path) in per_call.items():
            if plan.nseg == 1:
                assert len(plan.launches) == 1 and not plan.launches[0][3], (case.id, op)
                continue
            fam = "rows" if so.ro.view_geometry(case)[2] == 1 else "cols"
            n8 = "" if fam == "rows" or case.options.get("reduce.cols_loads") == "4" else "_n8"
            sfx = case.dtype + ("" if odt == "f32" else "_" + odt)
            assert plan.kernels == [f"reduce_{fam}_{op}_{case.dtype}{n8}", f"scan_{fam}_{op}_f32", f"scan_{fam}_{op}_{sfx}"], \
                (case.id, op, ex, odt, plan.kernels)
            assert [ln[3] for ln in plan.launches] == [False, True, True], "launches 2 and 3 wait through programmatic dependent launch"


def test_three_pass_rows_have_a_short_last_segment_and_misaligned_heads(planned):
    for case in (c for c in CASES if c.path.startswith("rows-3pass")):
        plan = planned[case][("sum", False, "f32")][0]
        seg, L = so.host_seg_len(case), case.length()
        assert seg % 512 == 0 and plan.nseg == -(-L // seg) > 8
        assert L % seg and (L % seg) % 512, "the last segment is short, and not a whole number of 512-element blocks"
        heads = so.row_heads(case, seg)
        # aligned: no head anywhere; misaligned: every row (and so every segment of it) starts at another alignment
        assert len(np.unique(heads)) == (4 if case.path.endswith("misaligned") else 1) and heads.any() == case.path.endswith("misaligned")
        pos = so.named_positions(case, plan)
        mid = plan.nseg // 2
        for o, p in enumerate(pos):
            assert {0, L - 1, mid * seg, (mid + 1) * seg - 1, (plan.nseg - 1) * seg} <= set(p)
            h = int(heads[o, 0])
            assert set(range(h)) | {h, h + so.rows_tpr(case, seg) * so.SCAN_ELEMS} <= set(p)


def test_pitched_rank3_three_pass_uses_logical_columns():
    case = next(c for c in CASES if c.path == "cols-3pass-pitched")
    outer, L, inner, s_outer, s_len, row_len, row_pitch, _ = so.ro.view_geometry(case)
    assert (row_len, row_pitch) == (72, 128) and inner == 40 * 72 != s_len and so.probe(case, "sum").nseg > 1


# ------------------------------------------------------------------------------------------------ the oracle
def _launch_sets(case, planned):
    plan = planned[case][(case.ops[0], False, "f32")][0]
    positions = so.named_positions(case, plan)
    return plan, positions, {op: list(so.launches(case, op, positions)) for op in case.ops}


def _logical(case, xr):
    shape = case.shape
    rest = [n for i, n in enumerate(shape) if i != case.axis]
    return np.moveaxis(xr.reshape(rest + [shape[case.axis]]), -1, case.axis)


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.id)
def test_data_preconditions_and_oracle_vs_f64(planned, case):
    _, positions, sets = _launch_sets(case, planned)
    for op, runs in sets.items():
        assert runs[0][0] == "finite"
        so.assert_preconditions(case, op, runs[0][1])
        if op == "sum" and case.length() >= 64:
            big = np.abs(so.expected(runs[0][1], "sum", False)).max()
            assert big > 2048, f"no prefix beyond 2048 (max {big}): 16-bit stores would not have to round"
        if op in ("max", "min"):
            assert (np.abs(runs[0][1]) > so.BASE_RANGE).sum() == sum(len(so.line_positions(positions, o)) for o in range(case.lines()))
        for label, xr in runs:
            for ex in (False, True):
                want = so.expected(xr, op, ex)
                if label != "finite" and not (ex and case.length() == 1):     # the planted values show in the outputs
                    assert not so.outputs_equal(want, so.expected(runs[0][1], op, ex)).all(), (op, label, ex)
                if label != "finite" and xr.size > 1 << 22:
                    continue                                  # the long lines' non-finite launches change a few elements
                f64, _ = scan_axis_f64(xr, 1, op, ex)
                assert so.outputs_equal(want, f64.astype(np.float32)).all(), (op, label, ex)
    full = so.expected(sets["sum"][0][1], "sum", False)
    assert np.array_equal(so.expected(sets["sum"][0][1], "sum", False, case.dtype), so.rne16(full, case.dtype))


def test_oracle_agrees_with_f64_in_logical_order(planned):
    # the [lines, len] order of the oracle is the logical tensor scanned along its axis
    for case in (c for c in CASES if c.path in ("cols-3pass-narrow", "gather", "rank8") and c.dtype == "f32"):
        _, _, sets = _launch_sets(case, planned)
        xr = sets["sum"][0][1]
        f64, _ = scan_axis_f64(_logical(case, xr), case.axis, "sum", True)
        assert np.array_equal(gpu.DeviceView.lines(type("V", (), {"case": case})(), f64).astype(np.float32),
                              so.expected(xr, "sum", True))


def test_non_finite_onsets():
    x = np.array([[1, 2, 3, 4, 5]], np.float32)
    s = so.plant_nonfinite(x, "sum", [[1, 3]], 0, 1)
    assert so.expected(s, "sum", False).tolist()[0][:3] == [1, np.inf, np.inf] and np.isnan(so.expected(s, "sum", False)[0, 3:]).all()
    p = so.plant_nonfinite(-x, "prod", [[1, 3]], 0, 1)
    got = so.expected(p, "prod", True)[0]
    assert got[0] == 1 and got[1] == -1 and got[2] == 0 and np.signbit(got[2]) and got[3] == 0 and np.isnan(got[4])
    m = so.plant_nonfinite(x, "max", [[3]], 0, 1)
    assert np.isnan(so.expected(m, "max", False)[0, 3:]).all() and not np.isnan(so.expected(m, "max", True)[0, 3])


# ------------------------------------------------------------------------------------------------ teeth
def _needed(case, op, ex, odt, flat, seg_len, heads):
    """The wrong kernels that must change at least one expected output of (op, exclusive, out dtype) on the case."""
    L, n = case.length(), case.lines()
    need = set()
    if L > 1:
        reach = [p for p in flat if not ex or p < L - 1]   # an exclusive scan never shows its last element
        need |= {f"drop {p}" for p in reach}
        if op in ("sum", "prod"):
            need |= {f"double {p}" for p in reach}
        need |= {"inclusive and exclusive swapped", "outputs shifted by one position"}
    else:   # a unit axis: inclusive copies the element, exclusive writes the identity everywhere
        need.add("inclusive and exclusive swapped")
        if not ex:
            need.add("drop 0")
    # (the unit axis's prod lines all hold the same planted -2)
    if n > 1 and (L > 1 or not ex and op != "prod"):
        need.add("outputs shifted by one line")
    if seg_len < L:
        need |= {"carry missing", "carry of the neighbouring segment"}
        if op in ("sum", "prod"):
            need.add("carry applied twice")
    if heads is not None and heads.any():
        need |= {"head-tile outputs lost", "head-tile outputs shifted"}
    if ex and op != "sum":
        need.add("exclusive identity 0")
    if odt != "f32" and op == "sum" and L >= 64:
        need.add("16-bit store truncates")
    if op in ("max", "min") and (L > 1 or not ex):
        need.add(("fmaxf" if op == "max" else "fminf") + " drops the NaN")
    if case.pitch:
        need.add("padding read")
    return need


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.id)
def test_wrong_kernels_change_an_expected_output(planned, case):
    # each (op, exclusive) on its f32 output, and the 16-bit store on the 16-bit output (whose other results are the f32
    # ones rounded).  The finite data must catch every wrong kernel but one: only a NaN shows fmaxf / fminf semantics.
    plan, positions, sets = _launch_sets(case, planned)
    seg_len = so.host_seg_len(case)
    heads = so.row_heads(case, seg_len) if so.ro.view_geometry(case)[2] == 1 and case.length() > 1 else None
    flat = sorted({p for pos in positions for p in pos})
    missed = []
    for op in case.ops:
        for ex in (False, True):
            caught = {}
            for label, xr in sets[op]:
                want = so.expected(xr, op, ex)
                for name, wrong in so.mutants(xr, op, ex, "f32", positions, seg_len, heads, padding=bool(case.pitch),
                                              nan_only=label != "finite"):
                    caught[name] = caught.get(name, False) or bool((~so.outputs_equal(wrong, want)).any())
                for odt in case.out_dtypes()[1:]:
                    if label == "finite":
                        wrong = so.mutant_truncating_store(want, odt)
                        caught["16-bit store truncates"] = bool((~so.outputs_equal(wrong, so.rne16(want, odt))).any())
            need = set()
            for odt in case.out_dtypes():
                need |= _needed(case, op, ex, odt, flat, seg_len, heads)
            assert need <= set(caught), (op, ex, sorted(need - set(caught)))
            missed += [f"{op} {'excl' if ex else 'incl'}: {m}" for m in sorted(need) if not caught[m]]
    assert not missed, f"{case.id}: these wrong kernels would pass: {missed}"
