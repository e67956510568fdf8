"""CPU: the sampling oracle (tests/sample_oracle.py) -- Philox4x32-10 against Random123's known-answer vectors, the kept sets
against HF's Temperature -> TopK -> MinP -> TopP warpers on tie-free rows, the drawn distribution against an f64 softmax over
the kept set, and the exact cases' power to catch six wrong contracts -- then b200_sample's dry-run plans (one launch, the
same for any b, the row class, cluster size and access path), every refusal, b = 0 without pointers, the Python layer's
deferred errors, and the sample cubin's resources and SASS (no spills or local memory; shared-memory atomics only)."""
import ctypes as C
import re
import subprocess

import numpy as np
import pytest
import torch

import sample_oracle as so
from cubecl_b200 import _ffi, sample as smp
from plan_context import PlanContext
from test_conv_cpu import ROOT, _tool

F32, F16, BF16, I32, I64 = _ffi.F32, _ffi.F16, _ffi.BF16, _ffi.I32, _ffi.I64
DT = {F32: "f32", BF16: "bf16", F16: "f16"}
X, Y, A = 1 << 40, 2 << 40, 3 << 40
INVALID, UNSUPPORTED = 6, 7


# ---------------------------------------------------------------------------------------------- oracle
@pytest.mark.parametrize("ctr,key,out", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0), (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_matches_random123_known_answers(ctr, key, out):
    assert so.philox4x32(ctr, key) == out


def test_draw_bits_take_seed_as_key_and_offset_as_counter():
    seed, off = 0x299f31d0a4093822, 0x85a308d3243f6a88
    r = so.philox4x32((off & 0xFFFFFFFF, off >> 32, 0, 0), (seed & 0xFFFFFFFF, seed >> 32))
    assert so.draw_bits(seed, off)[0] == r[0] + (r[1] << 32)


def test_ceil_mul_is_exact():
    rng = np.random.default_rng(1)
    for _ in range(200):
        p = np.float32(rng.random()) or np.float32(0.5)
        S = int(rng.integers(1 << 40, 1 << 58))
        from fractions import Fraction
        want = -(-Fraction(float(p)) * S // 1)
        assert so.ceil_mul(p, S) == want
    assert so.ceil_mul(np.float32(1.0), 12345) == 12345 and so.ceil_mul(np.float32(2.0 ** -149), 1 << 58) == 1


def _tie_free_rows(rng, b, v):
    while True:
        x = (rng.standard_normal((b, v)) * 2.5).astype(np.float32)
        if all(len(np.unique(r)) == v for r in x):
            return x


HF_CONF = [(1.0, 50, 0.9, 0.05), (0.7, 0, 0.8, 0.0), (1.3, 20, 1.0, 0.0), (1.0, 0, 1.0, 0.1), (0.9, 100, 0.95, 0.02),
           (1.0, 5, 0.5, 0.3)]


@pytest.mark.parametrize("conf", HF_CONF, ids=str)
def test_kept_sets_match_hf_warpers_on_tie_free_rows(conf):
    lp = pytest.importorskip("transformers.generation.logits_process")
    T, k, p, mp = conf
    rng = np.random.default_rng(int(T * 100) + k)
    b, v = 24, 5000
    x = _tie_free_rows(rng, b, v)
    scores = torch.tensor(x, dtype=torch.float64)
    warpers = [lp.TemperatureLogitsWarper(T)]
    if k:
        warpers.append(lp.TopKLogitsWarper(k))
    if mp:
        warpers.append(lp.MinPLogitsWarper(mp))
    if p < 1:
        warpers.append(lp.TopPLogitsWarper(p))
    for w in warpers:
        scores = w(None, scores)
    compared = 0
    for r in range(b):
        keep = []
        _, margin, _ = so.sample_row(x[r], T, k, p, mp, 1, 2, _keep=keep)
        S = int(keep[1].sum())
        if margin <= 1e-6 * S:          # too near a boundary for HF's float arithmetic to agree
            continue
        hf = torch.isfinite(scores[r]).numpy()
        np.testing.assert_array_equal(keep[0], hf)
        # the drawn distribution, q / S', is within the mass truncation and ex2's error of the f64 softmax over the kept set
        z = torch.tensor(x[r], dtype=torch.float64) / T
        ref = torch.softmax(z[torch.tensor(hf)], 0).numpy()
        got = keep[1][hf].astype(np.float64) / S
        assert np.max(np.abs(got - ref)) <= 4 * so.EX2_REL + v * 2.0 ** -40
        compared += 1
    assert compared >= b * 3 // 4, compared


def test_every_mutant_changes_an_exact_case():
    caught = set()
    for v in (7, 1000, 16385, 50257, 128256):
        for dtype in ("f32", "bf16", "f16"):
            rng = np.random.default_rng(v * 7 + len(dtype))
            x, params = so.exact_batch(rng, v, dtype)
            ok = so.sample(x, **params)[0]
            for m in so.MUTANTS:
                if m not in caught and not np.array_equal(so.sample(x, **params, _mutant=m)[0], ok):
                    caught.add(m)
    assert caught == set(so.MUTANTS), set(so.MUTANTS) - caught


def test_exact_rows_have_power_of_two_masses():
    rng = np.random.default_rng(3)
    steps = so.exact_steps()
    assert {-13, -15, -26, -27, -30, -31}.isdisjoint(steps) and len(steps) == 46 - 6
    for dtype in ("f32", "bf16", "f16"):
        for T in (0.5, 1.0, 2.0):
            x = so.exact_rows(rng, 3, 4000, dtype, T)
            z = (x / np.float32(T)).astype(np.float32)
            with np.errstate(invalid="ignore"):
                a = ((z - z.max(1, keepdims=True)).astype(np.float32) * so.LOG2E).astype(np.float32)
            fin = np.isfinite(a) & (a >= -149)                              # below that ex2 flushes to +0
            assert np.all(a[fin] == np.round(a[fin]))
            w = so.ex2(np.where(fin, a, -np.inf))
            q = so.masses(w)
            assert np.all((q == 0) | ((q & (q - np.uint64(1))) == 0))       # every mass 0 or a power of two


# ---------------------------------------------------------------------------------------------- dry-run plans
class Planner(PlanContext):
    def run(self, b=64, v=128256, x=BF16, ids=I64, ls=None, ptrs=(X, Y), args=True, **kw):
        a = _ffi.SampleArgs()
        a.temperature, a.top_k, a.top_p, a.min_p = 1.0, 50, 0.9, 0.0
        for k, val in kw.items():
            setattr(a, k, val)
        before = self.text()
        rc = self.lib.b200_sample(self.ctx, None, C.byref(a) if args else None, x, ids, b, v, C.c_uint64(ptrs[0]), ls or v,
                                  C.c_uint64(ptrs[1]))
        return rc, self.text()[len(before):]


@pytest.fixture
def plan():
    with Planner() as p:
        yield p


def _launches(text):
    return re.findall(r"launch (\w+) grid=\((\d+),(\d+),1\) block=(\d+) smem=(\d+) cluster=(\d+)", text)


ROWS = [(1, "cta", 1, 8), (1000, "cta", 1, 1000), (16384, "cta", 1, 16384), (16385, "cluster", 2, 8200),
        (32000, "cluster", 2, 16000), (50257, "cluster", 4, 12568), (128256, "cluster", 8, 16032),
        (151936, "cluster", 8, 18992), (262144, "cluster", 8, 32768)]


@pytest.mark.parametrize("v,cls,ranks,slice_", ROWS)
def test_plan_names_class_ranks_and_one_launch(plan, v, cls, ranks, slice_):
    for x in (F32, BF16, F16):
        for ids in (I32, I64):
            rc, t = plan.run(b=100, v=v, x=x, ids=ids)
            assert rc == 0, _ffi.load().b200_last_error()
            assert (f"sample x={DT[x]} ids={'i64' if ids == I64 else 'i32'} v={v} class={cls} threads=256 ranks={ranks}"
                    in t), t
            assert "greedy_only=0" in t
            (k,) = _launches(t)
            assert k[0] == f"sample_{DT[x]}" and int(k[1]) == 100 * ranks and k[3] == "256"
            assert int(k[4]) == slice_ * 4 + 2 * 3 * 2048 * 4 and k[5] == str(ranks)     # the slice, two histograms
            rc, t = plan.run(b=100, v=v, x=x, ids=ids, temperature=0.0)
            (k,) = _launches(t)
            assert rc == 0 and "greedy_only=1" in t and k[0] == f"sample_greedy_{DT[x]}" and k[4] == "0"


def test_per_row_temperatures_are_never_greedy_only(plan):
    rc, t = plan.run(temperature=0.0, temperatures=A)
    assert rc == 0 and "greedy_only=0" in t and _launches(t)[0][0] == "sample_bf16"


@pytest.mark.parametrize("v", [1, 1000, 32000, 50257, 128256, 151936, 262144])
def test_plan_for_v_is_the_same_for_any_b(plan, v):
    texts = {re.sub(r"grid=\(\d+,", "grid=(*,", plan.run(b=b, v=v)[1]) for b in (1, 3, 64, 4096, 65537)}
    assert len(texts) == 1, texts


def test_grid_is_capped(plan):
    rc, t = plan.run(b=(1 << 31) - 1, v=262144)
    ((_, gx, *_),) = _launches(t)
    assert rc == 0 and int(gx) == (1 << 20) * 8


def test_vector_path_needs_aligned_rows(plan):
    assert "vec=1" in plan.run(v=128256)[1]
    assert "vec=0" in plan.run(v=50257)[1]                        # v % 8
    assert "vec=0" in plan.run(v=128256, ls=128257)[1]            # row pitch
    assert "vec=0" in plan.run(v=128256, ls=128260)[1]            # 8-byte pitch in bf16
    assert "vec=1" in plan.run(v=128256, x=F32, ls=128260)[1]     # 16 bytes in f32
    assert "vec=0" in plan.run(v=128256, ptrs=(X + 2, Y))[1]


REFUSALS = [
    (dict(args=False), INVALID, "null args"),
    (dict(x=_ffi.F64), INVALID, "logits dtype"),
    (dict(ids=_ffi.U32), INVALID, "ids dtype"),
    (dict(v=0), INVALID, "v = 0"),
    (dict(v=(1 << 18) + 1), UNSUPPORTED, "exceeds"),
    (dict(b=1 << 31), UNSUPPORTED, "2^31"),
    (dict(ls=128255), INVALID, "row stride"),
    (dict(temperature=-1.0), INVALID, "temperature"),
    (dict(temperature=float("nan")), INVALID, "temperature"),
    (dict(temperature=float("inf")), INVALID, "temperature"),
    (dict(top_p=0.0), INVALID, "top_p"),
    (dict(top_p=1.5), INVALID, "top_p"),
    (dict(top_p=float("nan")), INVALID, "top_p"),
    (dict(min_p=-0.5), INVALID, "min_p"),
    (dict(min_p=1.5), INVALID, "min_p"),
    (dict(min_p=float("nan")), INVALID, "min_p"),
    (dict(advance_offsets=1), INVALID, "advance_offsets"),
    (dict(ptrs=(0, Y)), INVALID, "null device pointer"),
    (dict(ptrs=(X, 0)), INVALID, "null device pointer"),
    (dict(ptrs=(X + 1, Y)), INVALID, "misaligned"),
    (dict(ptrs=(X, Y + 4)), INVALID, "misaligned"),
    (dict(ids=I32, ptrs=(X, Y + 2)), INVALID, "misaligned"),
    (dict(temperatures=A + 2), INVALID, "misaligned"),
    (dict(top_ks=A + 1), INVALID, "misaligned"),
    (dict(top_ps=A + 2), INVALID, "misaligned"),
    (dict(min_ps=A + 2), INVALID, "misaligned"),
    (dict(seeds=A + 4), INVALID, "misaligned"),
    (dict(offsets=A + 4), INVALID, "misaligned"),
]


@pytest.mark.parametrize("case", range(len(REFUSALS)))
def test_refusals(plan, case):
    kw, status, words = REFUSALS[case]
    rc, t = plan.run(**kw)
    msg = _ffi.load().b200_last_error().decode()
    assert rc == status, (case, rc, msg)
    assert words in msg and "launch" not in t, (case, msg, t)


def test_zero_rows_are_a_no_op_even_without_pointers(plan):
    rc, t = plan.run(b=0, ptrs=(0, 0))
    assert rc == 0 and t == ""
    # the argument checks still run
    assert plan.run(b=0, v=0)[0] == INVALID and plan.run(b=0, v=1 << 19)[0] == UNSUPPORTED
    assert plan.run(b=0, top_p=2.0)[0] == INVALID


def test_accepted_edges(plan):
    for kw in (dict(top_p=1.0), dict(top_p=2.0 ** -149), dict(min_p=0.0), dict(min_p=1.0), dict(temperature=-0.0),
               dict(top_k=-5), dict(top_k=1 << 30), dict(advance_offsets=1, offsets=A), dict(v=1 << 18)):
        rc, t = plan.run(**kw)
        assert rc == 0, (kw, _ffi.load().b200_last_error())


# ---------------------------------------------------------------------------------------------- Python layer
def test_python_layer_defers_errors():
    class _Stub:
        def __init__(self):
            self.errors = []

        def _defer(self, e):
            self.errors.append(e)

    class _T:
        def __init__(self, shape, dtype="bf16", strides=None):
            self.shape, self.dtype = list(shape), dtype
            self.strides = strides or [int(np.prod(shape[i + 1:])) for i in range(len(shape))]

        def is_contiguous(self):
            return self.strides == [int(np.prod(self.shape[i + 1:])) for i in range(len(self.shape))]

    s = _Stub()
    x, ids = _T([16, 256]), _T([16], "i64")
    smp.sample(s, _T([16, 256, 1]), ids)                                  # logits not 2-D
    smp.sample(s, _T([16, 256], strides=[512, 2]), ids)                   # column stride
    smp.sample(s, x, _T([16], "f32"))                                     # ids not i32 / i64
    smp.sample(s, x, _T([15], "i64"))                                     # ids not [B]
    smp.sample(s, x, ids, temperature=_T([16], "bf16"))                   # per-row temperature not f32
    smp.sample(s, x, ids, top_k=_T([16], "i64"))                          # per-row top_k not i32
    smp.sample(s, x, ids, seed=_T([8], "u64"))                            # per-row seed not [B]
    smp.sample(s, x, ids, offset=3, advance_offsets=True)                 # advance without per-row offsets
    assert [e.status for e in s.errors] == [INVALID] * 8
    for i, word in enumerate(["logits", "logits", "ids", "ids", "temperature", "top_k", "seed", "advance_offsets"]):
        assert word in str(s.errors[i]), (i, str(s.errors[i]))


# ---------------------------------------------------------------------------------------------- kernels
KERNELS = {f"sample{g}_{x}" for g in ("", "_greedy") for x in ("f32", "bf16", "f16")}


def test_sample_kernels_do_not_spill_and_use_shared_atomics_only():
    tool = _tool("cuobjdump")
    _ffi.load()
    cubin = ROOT / "cubecl_b200" / "build" / "sample.cubin"
    out = subprocess.run([tool, "-res-usage", str(cubin)], capture_output=True, text=True, check=True).stdout
    funcs = re.findall(r"Function (\w+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", out)
    assert {f for f, *_ in funcs} == KERNELS
    for name, reg, stack, shared, local in funcs:
        assert int(stack) == 0 and int(local) == 0, (name, stack, local)
        # 2 resident 256-thread CTAs per SM (4 for the greedy-only kernels)
        assert int(reg) <= (64 if "greedy" in name else 128), (name, reg)
        # the 128 KB slice of v = 2^18 and the two 24 KB histograms fit beside the static state
        assert int(shared) + 4 * 32768 + 2 * 3 * 2048 * 4 <= 227 * 1024, (name, shared)
    sass = subprocess.run([tool, "-sass", str(cubin)], capture_output=True, text=True, check=True).stdout
    bodies = {b.split()[0]: b for b in re.split(r"\n\s*Function : ", sass)[1:]}
    assert set(bodies) == KERNELS
    for name, body in bodies.items():
        assert not re.search(r"\b(ATOM|ATOMG|RED|REDG)\b", body), name        # no global (or generic) atomics
        assert not re.search(r"\b(LDL|STL)\b", body), name
        assert "LDG.E.128" in body, name
        assert ("ATOMS.ADD" in body) == ("greedy" not in name), name           # histograms: shared-memory atomics,
        assert "ATOMS.CAS" not in body, name                                   # 32-bit and native, not a CAS loop
    assert "MUFU.EX2" in bodies["sample_bf16"] and "MATCH" in bodies["sample_bf16"]
    assert "UCGABAR" in bodies["sample_bf16"] or "CGABAR" in bodies["sample_bf16"]   # cluster barrier
