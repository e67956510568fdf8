"""CPU: numerics model of the f32 matmul schedules (csrc/gemm_wgmma.cu, run_gemm in capi.cpp) -- what each split leaves out, in
exact arithmetic (numpy f64 sums of the exactly representable partial products), so the accuracy claims in DESIGN.md are pinned:

  tf32     : hi(a) . hi(b)                                        hi = the top 19 bits of the f32 (what the tf32 datapath reads)
  3xtf32   : hi.hi + hi(a).hi(b_lo) + hi(a_lo).hi(b)              lo = x - hi (exact in f32), read through the tf32 datapath again
  hybrid   : hi.hi + bf16(a).bf16(b_lo) + bf16(a_lo).bf16(b)      the cross terms on bf16 operands at twice the tensor rate

The hardware adds its own accumulation error on top (f32 accumulator, truncating adds); this model isolates the SPLIT."""
import numpy as np
import pytest


def trunc19(x):
    return (x.view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def bf16_rn(x):
    u = x.view(np.uint32).astype(np.uint64)
    return (((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16).astype(np.uint32).view(np.float32)


def schedules(a, b):
    d = lambda x: x.astype(np.float64)
    ah, bh = trunc19(a), trunc19(b)
    al, bl = (a - ah).astype(np.float32), (b - bh).astype(np.float32)   # exact: the low 13 bits
    assert np.array_equal(d(ah) + d(al), d(a)) and np.array_equal(d(bh) + d(bl), d(b))
    main = d(ah) @ d(bh)
    return {"tf32": main,
            "3xtf32": main + d(ah) @ d(trunc19(bl)) + d(trunc19(al)) @ d(bh),
            "hybrid": main + d(bf16_rn(a)) @ d(bf16_rn(bl)) + d(bf16_rn(al)) @ d(bf16_rn(b))}


def scaled_errors(a, b):
    exact = a.astype(np.float64) @ b.astype(np.float64)
    scale = np.abs(a).astype(np.float64) @ np.abs(b).astype(np.float64)
    return {k: float(np.max(np.abs(v - exact) / scale)) for k, v in schedules(a, b).items()}


@pytest.mark.parametrize("K", [64, 1024, 4096])
@pytest.mark.parametrize("dist", ["uniform_pm1", "uniform_01", "normal"])
def test_split_error_of_each_schedule(K, dist):
    rng = np.random.default_rng(K + len(dist))
    M = N = 64
    gen = {"uniform_pm1": lambda s: rng.uniform(-1, 1, s), "uniform_01": lambda s: rng.uniform(0, 1, s), "normal": rng.standard_normal}[dist]
    a, b = gen((M, K)).astype(np.float32), gen((K, N)).astype(np.float32)
    e = scaled_errors(a, b)
    assert e["tf32"] <= 1.0e-3                       # the north star's f32 tolerance, single pass
    assert e["3xtf32"] <= 5.0e-7                     # the dropped lo.lo term: <= 2^-20 per product, ~2^-22 typical
    assert e["hybrid"] <= 1.5e-6                     # cross terms rounded to bf16: 2^-9 of a 2^-11 term
    assert e["hybrid"] <= 8.0 * e["3xtf32"] + 1e-9   # a small constant factor above 3xTF32 ...
    assert e["hybrid"] <= e["tf32"] / 100.0          # ... and two orders of magnitude below the single pass


def test_wide_dynamic_range_keeps_the_ordering():
    rng = np.random.default_rng(7)
    a = (rng.standard_normal((48, 512)) * np.exp(rng.uniform(-8, 8, (48, 512)))).astype(np.float32)
    b = (rng.standard_normal((512, 48)) * np.exp(rng.uniform(-8, 8, (512, 48)))).astype(np.float32)
    e = scaled_errors(a, b)
    assert e["3xtf32"] < e["hybrid"] < 1e-5 < e["tf32"] < 2e-3


def test_exactly_representable_operands_are_exact_in_every_schedule():
    # small integers (the reference's cmma goldens): hi = x, lo = 0, bf16(x) = x -- all three schedules return the exact product
    a = np.arange(128, dtype=np.float32).reshape(16, 8)
    b = (np.arange(128) % 8).astype(np.float32).reshape(8, 16)
    exact = a.astype(np.float64) @ b.astype(np.float64)
    for v in schedules(a, b).values():
        assert np.array_equal(v, exact)
