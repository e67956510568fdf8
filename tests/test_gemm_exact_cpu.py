"""CPU: the exact-oracle helpers of tests/gemm_exact_oracle.py (rounding against hand-written bit patterns, the generators'
exactness bound, checks that fail when they should) and the path coverage of tests/test_gemm_exact_gpu.py, read off dry-run
plans of its case lists on an H100's 132 SMs."""
import re

import numpy as np
import pytest

import gemm_exact_oracle as ge
import test_gemm_exact_gpu as gpu
from cubecl_b200 import TensorHandle, matmul

SMS = 132


# ------------------------------------------------------------------------------------------------ rne
@pytest.mark.parametrize("x,bits", [
    (1.0, 0x3F80), (-2.0, 0xC000), (256.0, 0x4380), (257.0, 0x4380), (259.0, 0x4382), (385.0, 0x43C0), (387.0, 0x43C2),
    (1.0 + 2.0 ** -8, 0x3F80), (1.0 + 3 * 2.0 ** -8, 0x3F82),     # ties to even, both directions
    (3.4028234663852886e38, 0x7F80), (-np.inf, 0xFF80),           # f32 max rounds up to inf
    (2.0 ** -130, 0x0008), (-0.0, 0x8000), (1.5 * 2.0 ** -133, 0x0002), (2.5 * 2.0 ** -133, 0x0002),
])
def test_rne_bf16_bit_patterns(x, bits):
    assert int(ge.rne(np.array([x]), "bf16")[0]) == bits


@pytest.mark.parametrize("x,bits", [
    (1.0, 0x3C00), (2049.0, 0x6800), (2051.0, 0x6802), (65504.0, 0x7BFF), (65519.0, 0x7BFF), (65520.0, 0x7C00),
    (70000.0, 0x7C00), (-70000.0, 0xFC00), (2.0 ** -20, 0x0010), (2.0 ** -24, 0x0001), (2.0 ** -25, 0x0000),
    (3 * 2.0 ** -26, 0x0001), (-(2.0 ** -25), 0x8000), (1.5 * 2.0 ** -24, 0x0002),
])
def test_rne_f16_bit_patterns(x, bits):
    assert int(ge.rne(np.array([x]), "f16")[0]) == bits


def test_rne_rounds_through_f32_first_and_keeps_nan():
    # 1 + 2^-8 + 2^-40: f64 -> f32 drops 2^-40, leaving a bf16 tie that rounds to even (a direct f64 rounding would go up)
    assert int(ge.rne(np.array([1.0 + 2.0 ** -8 + 2.0 ** -40]), "bf16")[0]) == 0x3F80
    for dt in ("bf16", "f16", "f32"):
        assert np.isnan(ge.bits_to_f64(ge.rne(np.array([np.nan]), dt), dt)[0])


def test_rz_truncates_toward_zero():
    assert list(ge.rz(np.array([259.0, -259.0, 257.0, 65520.0]), "bf16")) == [0x4381, 0xC381, 0x4380, 0x477F]
    assert list(ge.rz(np.array([65520.0, -2051.0, 3 * 2.0 ** -26]), "f16")) == [0x7BFF, 0xE801, 0x0000]


# ------------------------------------------------------------------------------------------------ the checks fail when they should
def test_exact_check_catches_one_ulp_rz_and_accepts_signed_zero_and_nan_positions():
    exact = np.array([[257.0, 259.0, 0.0, np.nan], [385.0, -3.0, 1.0, 2.0]])
    good = ge.rne(exact, "bf16")
    ge.assert_exact(good, exact, "bf16")
    signed = good.copy()
    signed[0, 2] = 0x8000            # -0 where +0 is expected
    ge.assert_exact(signed, exact, "bf16")
    for bad in (good.copy(), ge.rz(exact, "bf16")):
        if bad is not None and np.array_equal(bad, good):
            bad[1, 1] += 1           # one ulp on one element
        with pytest.raises(AssertionError):
            ge.assert_exact(bad, exact, "bf16")
    moved = good.copy()
    moved[0, 3], moved[1, 3] = good[1, 3], good[0, 3]   # the NaN at another position
    with pytest.raises(AssertionError):
        ge.assert_exact(moved, exact, "bf16")
    f32 = ge.rne(exact, "f32")
    f32[1, 0] += 1
    with pytest.raises(AssertionError):
        ge.assert_exact(f32, exact, "f32")


# ------------------------------------------------------------------------------------------------ generators
def test_matmul_generator_enforces_the_2_24_bound_and_real_rounding():
    a, b, exact = ge.matmul_operands((300, 200), (200, 264), 16, seed=1, out_dtype="f16")
    assert np.array_equal(exact, a @ b) and np.max(np.abs(a) @ np.abs(b)) < 2 ** 24
    assert np.mean(np.abs(exact) > ge.ROUNDING_ABOVE["f16"]) > 0.01
    with pytest.raises(AssertionError, match="2\\^24"):
        ge.matmul_operands((2, 300000), (300000, 2), 16, seed=1, out_dtype="f32")
    with pytest.raises(AssertionError, match="too small"):
        ge.matmul_operands((64, 8), (8, 64), 2, seed=1, out_dtype="bf16")


@pytest.mark.parametrize("kind", ["e4m3", "e5m2", "e2m1", "nvfp4"])
def test_block_scaled_generator_gives_integer_products(kind):
    a_dev, b_dev, sa, sb, a, b = ge.block_scaled_operands(64, 48, 256, kind, seed=3)
    assert np.array_equal(a, np.round(a)) and np.array_equal(b, np.round(b))
    assert np.max(np.abs(a) @ np.abs(b).T) < 2 ** 24
    # the scale bytes decode to 2^1 .. 2^4
    from cubecl_b200 import synth
    dec = synth.fp8_bits_to_f32(sa, "f8e4m3") if kind == "nvfp4" else synth.ue8m0_to_f32(sa)
    assert set(np.unique(dec)) <= {2.0, 4.0, 8.0, 16.0}


def test_edge_operands_hit_their_targets_exactly():
    targets = [65504, 65519, 65520, 70000, -70000, 2.0 ** -12]
    a, b, exact = ge.edge_operands(targets, "f16", col_signs=(1.0, -1.0, 2.0 ** -13))
    assert np.array_equal(a @ b, exact)
    assert exact[5, 2] == 2.0 ** -25
    a, b, exact = ge.edge_operands([257, 259, 385], "bf16")
    assert np.array_equal(a @ b, exact)


def test_ieee_matmul_propagates_inf_times_zero():
    a = np.array([[np.inf, 1.0]])
    b = np.array([[0.0], [1.0]])
    assert np.isnan(ge.matmul_f64_ieee(a, b)[0, 0])


# ------------------------------------------------------------------------------------------------ coverage from dry-run plans
def _variant(kernel):
    if kernel == "gemm_simt_strided":
        return "simt"
    m = re.search(r"_(2sm_n256|2sm_n224|2sm_n128|1sm_n128|2sm_m512)(_|$)", kernel)
    return m.group(1) if m else kernel


def _cell(case, plan):
    store = "tma" if plan.tma_store and (not plan.head or plan.whole_tiles > 0) else "direct"
    return _variant(plan.kernel), store, "head" if plan.head else "nohead", case.out_dtype


def _required_cells():
    cells = set()
    for v in gpu.VARIANT_SHAPES:
        for od in ("f32", "bf16", "f16"):
            if v == "simt":
                cells.add((v, "direct", "nohead", od))
                continue
            for store in ("tma", "direct"):
                for head in (("head", "nohead") if v in gpu.HEAD_VARIANTS else ("nohead",)):
                    cells.add((v, store, head, od))
    return cells


@pytest.fixture(scope="module")
def gemm_plans():
    return [(c, ge.plan_gemm_case(c, SMS)) for c in gpu.GEMM_CASES]


def test_gemm_case_lists_cover_every_variant_store_head_and_output(gemm_plans):
    covered = {_cell(c, p) for c, p in gemm_plans}
    missing = _required_cells() - covered
    assert not missing, f"no case runs {sorted(missing)}"
    # and the fused-epilogue and one-rounding lists see every wgmma path with a 16-bit output too
    for subset in (gpu.EPILOGUE_CASES, gpu.ONE_ROUNDING):
        cells = {_cell(c, p) for c, p in gemm_plans if c in subset}
        want = {cell for cell in _required_cells() if cell[3] != "f32" and cell[0] != "2sm_m512"}
        assert not (want - cells), sorted(want - cells)


def test_gemm_cases_take_the_paths_their_names_say(gemm_plans):
    for c, p in gemm_plans:
        assert p.kernel, (c.name, p.text)
        gpu._expect_path(c, p)
        if c.name.startswith("n2mod8"):
            assert not p.tma_store and "simt" not in p.kernel        # scalar direct stores of the wgmma kernel
        if c.name == "skauto-bf16":
            assert p.head
        if c.in_dtype == "f32":
            assert "tf32" in p.kernel


def test_224_tile_runs_with_16bit_outputs():
    for od in ("bf16", "f16"):
        def issue(pc, od=od):
            fake = ge.FakeAlloc()
            t = lambda shape, dt: TensorHandle.new_contiguous(shape, fake(np.zeros(int(np.prod(shape)), np.uint8)), dt)  # noqa: E731
            matmul.launch_scaled(pc, t([300, 256], "f8e4m3"), t([520, 256], "f8e4m3"), t([300, 8], "ue8m0"), t([520, 8], "ue8m0"),
                                 t([300, 520], od))
        p = ge.probe(SMS, {"gemm.variant": "2sm_n224"}, issue)
        assert p.kernel == f"gemm_mx_{od}_2sm_n224_kk" and p.tma_store, p.text


def _conv_plans():
    plans = []
    geoms = [(w, g, od, {}) for g in gpu.CONV_CASES for od in ("bf16", "f16") for w in ("fwd", "dgrad", "wgrad")]
    geoms += [(w, g, od, dict([o])) for w, g, od, o in gpu.CONV_PATH_CASES]
    geoms += [(w, g, "bf16", {}) for w, g in gpu.ROUNDING_CONV]
    for which, geom, od, opts in geoms:
        issue, _, _ = gpu.conv_issue(which, *geom, "f16" if od == "f16" else "bf16", od, ge.FakeAlloc())
        plans.append((which, geom, od, opts, ge.probe(SMS, {**gpu.GEMM_OPTIONS, **opts}, issue)))
    return plans


def test_conv_case_lists_cover_multi_phase_dgrad_and_the_wgrad_head():
    plans = _conv_plans()
    assert all(p.kernels for *_, p in plans)
    assert any(w == "dgrad" and p.phases > 1 and od != "f32" for w, _, od, _, p in plans)
    assert any(w == "dgrad" and p.phases > 1 and not p.tma_store for w, _, _, _, p in plans)   # the direct-store epilogue
    assert any(w == "wgrad" and p.head and od != "f32" for w, _, od, _, p in plans)
    assert any(w == "wgrad" and p.tma_store and od != "f32" for w, _, od, _, p in plans)        # the channel-clipping TMA store
    for variant in ("2sm_n128", "1sm_n128"):
        assert any(variant in p.kernel for *_, p in plans)
    # the one-rounding list holds a multi-phase dgrad and a wgrad with a head
    rounding = [p for w, g, od, o, p in plans if (w, g) in gpu.ROUNDING_CONV and not o]
    assert any(p.phases > 1 for p in rounding) and any(p.head and "wgrad" in p.kernel for p in rounding)
