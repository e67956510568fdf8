"""GPU: f32 matmuls whose operands have nonzero low parts, checked exactly (tests/gemm_exact_oracle.py, lowpart_operands).

Integer f32 operands have zero low parts, so on them the low-part segments of the 3xTF32 and hybrid schedules only add exact
zeros.  Here every operand is x = hi + lo with lo below half the tf32 ulp of hi: both schedules must return
sum(a b - a_lo b_lo) and the tf32 schedule sum(a_hi b_hi), exactly in f32, on every tile, store path, stream-K plan, batch
stride, broadcast, transposed (staged) operand and unaligned K.  A low plane read at the wrong k, batch or transpose, a cross
term with the wrong sign or a wrongly built pair buffer changes these results (tests/test_gemm_exact_cpu.py shows each such
kernel would fail), where the bounded-error tests could not tell.  Each case asserts through a dry-run plan which GEMM kernel,
split kernel, store path and stream-K head it took; tests/test_gemm_exact_cpu.py checks that the list covers every cell."""
import re

import pytest

import gemm_exact_oracle as ge
from test_gemm_exact_gpu import GEMM_OPTIONS, HEAD_VARIANTS, _opts, run_gemm

pytestmark = pytest.mark.gpu

# Per tile a ragged shape with more tiles than clusters, as in test_gemm_exact_gpu: split_k "2" gives a head and whole tiles.
TILE_SHAPES = {"2sm_n256": (2300, 2056, 200), "2sm_n128": (1300, 1544, 200), "1sm_n128": (1400, 1672, 200)}
SPLIT_KERNEL = {"hybrid": "split_f32_bf16_pair", "3xtf32": "split_tf32_lo", "tf32": None}


def _plan_grid():
    cases = []
    for sched in ("3xtf32", "hybrid"):
        for variant, (M, N, K) in TILE_SHAPES.items():
            for epi in ("tma", "direct"):
                for split in ("off", "2"):
                    cases.append(ge.GemmCase(f"{sched}-{variant}-{epi}-sk{split}", "f32", "f32", M, N, K,
                                             opts=_opts(f32=sched, variant=variant, epilogue=epi, split_k=split)))
    return cases


def _layout_cases():
    cases = []
    for sched in ("3xtf32", "hybrid"):
        o = dict(f32=sched)
        cases += [
            ge.GemmCase(f"{sched}-batched", "f32", "f32", 300, 264, 136, batch=3, opts=_opts(**o)),
            ge.GemmCase(f"{sched}-bcast", "f32", "f32", 300, 264, 136, batch=3, bcast=True, opts=_opts(**o)),
            ge.GemmCase(f"{sched}-lhs_t", "f32", "f32", 264, 200, 136, lhs_t=True, opts=_opts(**o)),
            ge.GemmCase(f"{sched}-rhs_t", "f32", "f32", 264, 200, 136, rhs_t=True, opts=_opts(**o)),
            ge.GemmCase(f"{sched}-both_t-batched", "f32", "f32", 264, 200, 136, batch=2, lhs_t=True, rhs_t=True, opts=_opts(**o)),
            # K = 201: rows are not 16-byte multiples, so the operands are re-pitched before the split and the K tail is 9 wide
            ge.GemmCase(f"{sched}-k201", "f32", "f32", 300, 264, 201, opts=_opts(**o)),
            ge.GemmCase(f"{sched}-k201-bcast-sk2", "f32", "f32", 300, 264, 201, batch=2, bcast=True, opts=_opts(split_k=2, **o)),
            ge.GemmCase(f"{sched}-window", "f32", "f32", 300, 264, 136, window=True, opts=_opts(**o)),
            ge.GemmCase(f"{sched}-sk3-1sm", "f32", "f32", 520, 392, 1000, opts=_opts(split_k=3, variant="1sm_n128", **o)),
        ]
    cases += [ge.GemmCase(f"tf32-{v}-sk2", "f32", "f32", M, N, K, opts=_opts(f32="tf32", variant=v, split_k=2))
              for v, (M, N, K) in TILE_SHAPES.items()]
    cases.append(ge.GemmCase("tf32-batched-both_t", "f32", "f32", 264, 200, 136, batch=2, lhs_t=True, rhs_t=True, opts=_opts(f32="tf32")))
    return cases


LOWPART_CASES = _plan_grid() + _layout_cases()


def density(case):
    return 0.35 if case.K > 400 else 1.0   # sparser high parts keep sum |terms| below 2^24 grains at K = 1000


def schedule(case):
    return case.options["gemm.f32"]


def operands(case):
    ls, rs = ge.gemm_shapes(case)
    return ge.lowpart_operands(ls, rs, seed=case.M + case.K, schedule=schedule(case), density=density(case))


def expect_lowpart_path(case, plan):
    """The plan runs the tf32 kernel of the forced tile, the schedule's split kernel once per operand, and the forced split."""
    o = {**GEMM_OPTIONS, **case.options}
    assert "tf32" in plan.kernel, (case.name, plan.kernel)
    if o["gemm.variant"] != "auto":
        assert o["gemm.variant"] in plan.kernel, (case.name, plan.kernel)
    splits = re.findall(r"^launch (split_\S+)", plan.text, re.M)
    want = SPLIT_KERNEL[schedule(case)]
    assert splits == ([want, want] if want else []), (case.name, splits)
    if o["gemm.split_k"] == "2" and o["gemm.variant"] in HEAD_VARIANTS:
        assert plan.head and plan.whole_tiles > 0, (case.name, plan.text)
    if o["gemm.split_k"] == "3":
        assert plan.head
    if o["gemm.split_k"] == "off":
        assert not plan.head
    # tf32 reads K-major operands only: an MN-major operand (lhs_t, or an rhs that is not rhs_t) or rows that are not 16-byte
    # multiples are re-pitched K-major first, and the split then reads the staged copy
    staged = int(case.lhs_t or case.K % 4 != 0) + int(not case.rhs_t or case.K % 4 != 0)
    assert plan.text.count("launch repitch_rows") == staged, (case.name, plan.text)


@pytest.fixture(autouse=True)
def _reset_options(client):
    yield
    for k, v in GEMM_OPTIONS.items():
        client.set_option(k, v)


@pytest.mark.parametrize("case", LOWPART_CASES, ids=[c.name for c in LOWPART_CASES])
def test_f32_low_parts_are_exact_on_every_plan(client, case):
    a, b, exact, _ = operands(case)
    bits, plan = run_gemm(client, case, a, b)
    expect_lowpart_path(case, plan)
    ge.assert_exact(bits, exact, "f32", f"{case.name} on {plan.kernel}")
