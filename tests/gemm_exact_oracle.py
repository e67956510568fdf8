"""Exact oracles for the GEMM and convolution outputs, shared by tests/test_gemm_exact_cpu.py and tests/test_gemm_exact_gpu.py.

Two contracts make every output checkable bit for bit:
  * integer-valued operands with sum_k |a||b| < 2^24: every f32 partial sum is exact in any association, so every tile, store
    path and stream-K reduction order must give exactly rne(exact result);
  * one rounding: a 16-bit output is the round-to-nearest-even of the f32 output of the same plan.
The plan probe replays a call in a dry-run planning context and reports which kernel, store path and stream-K head it takes, so
a test can assert the path it meant to exercise really ran.
"""
from __future__ import annotations

import re
from dataclasses import dataclass, field

import numpy as np

from cubecl_b200 import synth
from cubecl_b200.client import DTYPE_SIZE, Handle, TensorHandle
from plan_context import PlanContext

EXACT_LIMIT = 2.0 ** 24
# smallest |output| at which a 16-bit result is rounded (integers above it are not all representable)
ROUNDING_ABOVE = {"bf16": 256.0, "f16": 2048.0}
OUT_BITS_VIEW = {"f32": np.uint32, "bf16": np.uint16, "f16": np.uint16}


# ------------------------------------------------------------------------------------------------ rounding
def rne(x, dtype: str) -> np.ndarray:
    """Bit patterns of x rounded once to f32 (RNE), then once to `dtype` (RNE): uint32 for f32, uint16 for bf16 / f16.
    Overflow gives inf, subnormals are kept, NaN stays NaN."""
    f = np.asarray(x, dtype=np.float64).astype(np.float32)
    if dtype == "f32":
        return f.view(np.uint32)
    if dtype == "bf16":
        return synth.f32_to_bf16_bits(f)
    if dtype == "f16":
        with np.errstate(over="ignore"):
            return f.astype(np.float16).view(np.uint16)
    raise ValueError(dtype)


def rz(x, dtype: str) -> np.ndarray:
    """Bit patterns of x rounded toward zero to `dtype` (from its f32 value): the conversion bug the exact checks must catch."""
    x = np.asarray(x, dtype=np.float64).astype(np.float32).astype(np.float64)
    bits = rne(x, dtype)
    with np.errstate(invalid="ignore"):
        away = np.isfinite(x) & (np.abs(bits_to_f64(bits, dtype)) > np.abs(x))
    return np.where(away, bits - 1, bits).astype(bits.dtype)   # sign-magnitude: one step toward zero


def bits_to_f64(bits, dtype: str) -> np.ndarray:
    bits = np.asarray(bits)
    if dtype == "f32":
        return bits.astype(np.uint32).view(np.float32).astype(np.float64)
    if dtype == "bf16":
        return synth.bf16_bits_to_f32(bits).astype(np.float64)
    return bits.astype(np.uint16).view(np.float16).astype(np.float64)


def bit_mismatches(got_bits, want_bits, dtype: str) -> np.ndarray:
    """Mask of elements whose values differ: +0 and -0 are equal, a NaN matches a NaN at the same position."""
    g, w = bits_to_f64(got_bits, dtype), bits_to_f64(want_bits, dtype)
    both_nan = np.isnan(g) & np.isnan(w)
    same = (np.asarray(got_bits) == np.asarray(want_bits)) | ((g == 0) & (w == 0)) | both_nan
    return ~same


def assert_bits_equal(got_bits, want_bits, dtype: str, what: str = "") -> None:
    bad = bit_mismatches(got_bits, want_bits, dtype)
    if bad.any():
        idx = tuple(int(i) for i in np.argwhere(bad)[0])
        g, w = bits_to_f64(got_bits, dtype)[idx], bits_to_f64(want_bits, dtype)[idx]
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.size} {dtype} outputs differ from the single rounding; "
                             f"first at {idx}: got {g!r}, want {w!r}")


def assert_exact(got_bits, exact, dtype: str, what: str = "") -> None:
    """got_bits == rne(exact) bit for bit, and the check has teeth: a one-ulp change of one element fails it, and so does the
    round-toward-zero conversion of the same values wherever that differs from round-to-nearest-even."""
    want = rne(exact, dtype)
    assert_bits_equal(got_bits, want, dtype, what)
    flat = np.asarray(got_bits).reshape(-1)
    finite = np.flatnonzero(np.isfinite(bits_to_f64(flat, dtype)))
    if finite.size:
        bumped = flat.copy()
        bumped[finite[finite.size // 2]] += 1
        assert bit_mismatches(bumped, want.reshape(-1), dtype).any(), "a one-ulp change went unnoticed"
    if dtype != "f32":
        truncated = rz(exact, dtype)
        if bit_mismatches(truncated, want, dtype).any():
            assert bit_mismatches(truncated, got_bits, dtype).any(), "round-toward-zero results would pass"


def f32_run_rounded(f32_out, dtype: str) -> np.ndarray:
    """The 16-bit bits a one-rounding kernel must produce from its own f32 result."""
    return rne(np.asarray(f32_out, dtype=np.float32), dtype)


# ------------------------------------------------------------------------------------------------ integer operands
def int_values(shape, bound: int, seed: int) -> np.ndarray:
    rng = np.random.default_rng(seed)
    return rng.integers(-bound, bound + 1, size=shape).astype(np.float64)


def assert_exact_bound(abs_sum: np.ndarray) -> None:
    """Every output's sum_k |a||b| stays below 2^24, so no f32 partial sum of it is ever rounded."""
    worst = float(np.max(abs_sum)) if abs_sum.size else 0.0
    assert worst < EXACT_LIMIT, f"sum |a||b| reaches {worst:.0f} >= 2^24: f32 partial sums could round"


def matmul_operands(lhs_shape, rhs_shape, bound: int, seed: int, out_dtype: str):
    """Integer lhs [.., M, K] and rhs [.., K, N] in [-bound, bound] (exact in bf16 / f16 / e4m3 / tf32 for bound <= 16), their f64
    product, and the check that (a) the product is exact in f32 and (b) 16-bit outputs really get rounded."""
    a, b = int_values(lhs_shape, bound, seed), int_values(rhs_shape, bound, seed + 1)
    exact = np.matmul(a, b)
    assert_exact_bound(np.matmul(np.abs(a), np.abs(b)))
    if out_dtype in ROUNDING_ABOVE and exact.size >= 64:
        assert np.max(np.abs(exact)) > 2 * ROUNDING_ABOVE[out_dtype], "outputs too small to exercise the 16-bit rounding"
    return a, b, exact


def block_scaled_operands(M, N, K, kind: str, seed: int, batch=()):
    """Integer-product block-scaled operands.  kind:
      "e4m3" / "e5m2"  integer fp8 values |v| <= 8 with ue8m0 scales 2^1 .. 2^4 per 32 elements;
      "e2m1"           e2m1 codes (0 .. 6 in halves) with ue8m0 scales 2^1 .. 2^4 per 32 elements;
      "nvfp4"          e2m1 codes with power-of-two e4m3 scales 2, 4, 8, 16 per 16 elements.
    Every scaled element is an integer, so every product and partial sum is exact.  Returns (a_dev, b_dev, sa, sb, a_scaled,
    b_scaled) with a_scaled [.., M, K] and b_scaled [.., N, K] the f64 values the GEMM multiplies."""
    rng = np.random.default_rng(seed)
    block = 16 if kind == "nvfp4" else 32

    def side(rows):
        if kind in ("e4m3", "e5m2"):
            dt = "f8" + kind
            vals = rng.integers(-8, 9, size=batch + (rows, K)).astype(np.float32)
            dev = synth.f32_to_fp8_bits(vals, dt)
            v = synth.fp8_bits_to_f32(dev, dt).astype(np.float64)
        else:
            codes = rng.integers(0, 16, size=batch + (rows, K)).astype(np.uint8)
            dev = synth.pack_e2m1x2(codes)
            v = synth.e2m1_codes_to_f32(codes).astype(np.float64)
        e = rng.integers(1, 5, size=batch + (rows, K // block))
        if kind == "nvfp4":
            sbits = (0x38 + 8 * e).astype(np.uint8)          # e4m3 2^e: exponent field 7 + e, mantissa 0
        else:
            sbits = (127 + e).astype(np.uint8)
        scaled = v * np.repeat(np.ldexp(1.0, e), block, axis=-1)
        assert np.array_equal(scaled, np.round(scaled))
        return dev, sbits, scaled

    a_dev, sa, a = side(M)
    b_dev, sb, b = side(N)
    assert_exact_bound(np.matmul(np.abs(a), np.swapaxes(np.abs(b), -1, -2)))
    return a_dev, b_dev, sa, sb, a, b


# ------------------------------------------------------------------------------------------------ f32 operands with low parts
# x = hi + lo with hi an integer of at most 2 bits and lo a multiple of LOW_GRAIN of the same sign and below half the tf32 ulp of
# hi: the tf32 datapath reads hi whether it truncates or rounds, x - trunc_tf32(x) = lo exactly, bf16(x) = hi, and lo is exact in
# tf32 and bf16.  So the 3xTF32 and hybrid schedules both compute sum(a b - a_lo b_lo) and tf32 alone sum(a_hi b_hi), and with
# every partial sum a multiple of LOW_GRAIN below 2^24 LOW_GRAIN, each of them is exact in f32.
LOW_GRAIN = 2.0 ** -14
F32_SCHEDULES = ("3xtf32", "hybrid", "tf32")
# kernels that compute the wrong low-part arithmetic, each of which the exact checks must catch
LOWPART_MUTANTS = ("tf32_only", "lo_lo_added", "a_lo_shifted_k", "b_lo_shifted_k", "a_lo_b_hi_negated", "a_hi_b_lo_negated")


def tf32_trunc(x) -> np.ndarray:
    return (np.asarray(x, np.float32).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def tf32_rn(x) -> np.ndarray:
    u = np.asarray(x, np.float32).view(np.uint32).astype(np.uint64)
    return (((u + 0xFFF + ((u >> 13) & 1)) >> 13) << 13).astype(np.uint32).view(np.float32)


def lowpart_values(shape, seed: int, hi_max: int = 3, lo_max: int = 7, density: float = 1.0):
    """(x, hi, lo) in f64: hi integers in [-hi_max, hi_max] (zero with probability 1 - density), lo = sign(hi) * j * LOW_GRAIN
    with j in [0, lo_max].  Asserts what the schedules read from x."""
    assert hi_max <= 3 and (lo_max + 1) * LOW_GRAIN <= 2.0 ** -11, "lo must stay below half the tf32 ulp of hi"
    rng = np.random.default_rng(seed)
    hi = rng.integers(1, hi_max + 1, size=shape) * rng.choice([-1.0, 1.0], size=shape)
    hi[rng.random(size=shape) >= density] = 0.0
    lo = np.sign(hi) * rng.integers(0, lo_max + 1, size=shape) * LOW_GRAIN
    x = hi + lo
    x32 = x.astype(np.float32)
    assert np.array_equal(x32.astype(np.float64), x)
    assert np.array_equal(tf32_trunc(x32), hi) and np.array_equal(tf32_rn(x32), hi), "the tf32 datapath must read hi"
    assert np.array_equal((x32 - tf32_trunc(x32)).astype(np.float64), lo), "the split must leave lo"
    assert np.array_equal(synth.bf16_bits_to_f32(synth.f32_to_bf16_bits(x32)), hi), "bf16(x) must be hi"
    lo32 = lo.astype(np.float32)
    assert np.array_equal(tf32_trunc(lo32), lo32) and np.array_equal(synth.bf16_bits_to_f32(synth.f32_to_bf16_bits(lo32)), lo32)
    return x, hi, lo


def lowpart_products(parts, schedule: str, mutant: str | None = None) -> np.ndarray:
    """f64 result of a schedule on lowpart_values operands parts = (a_hi, a_lo, b_hi, b_lo) ([.., M, K] and [.., K, N]), or of
    one of LOWPART_MUTANTS of it."""
    ah, al, bh, bl = parts
    if schedule == "tf32" or mutant == "tf32_only":
        return np.matmul(ah, bh)
    if mutant == "a_lo_shifted_k":     # the low plane of a read one k further on
        al = np.concatenate([al[..., 1:], np.zeros_like(al[..., :1])], axis=-1)
    if mutant == "b_lo_shifted_k":
        bl = np.concatenate([bl[..., 1:, :], np.zeros_like(bl[..., :1, :])], axis=-2)
    hl, lh = np.matmul(ah, bl), np.matmul(al, bh)
    if mutant == "a_hi_b_lo_negated":
        hl = -hl
    if mutant == "a_lo_b_hi_negated":
        lh = -lh
    out = np.matmul(ah, bh) + hl + lh
    if mutant == "lo_lo_added":
        out = out + np.matmul(al, bl)
    return out


def lowpart_operands(lhs_shape, rhs_shape, seed: int, schedule: str, density: float = 1.0):
    """Low-part f32 operands a [.., M, K] and b [.., K, N], the exact result of `schedule`, and the (a_hi, a_lo, b_hi, b_lo)
    parts.  Asserts that every partial sum of every schedule's terms is exact in f32 (sum |terms| < 2^24 LOW_GRAIN) and that the
    low parts really change the result."""
    a, ah, al = lowpart_values(lhs_shape, seed, density=density)
    b, bh, bl = lowpart_values(rhs_shape, seed + 1, density=density)
    parts = (ah, al, bh, bl)
    assert_exact_bound((np.matmul(np.abs(ah), np.abs(bh)) + np.matmul(np.abs(ah), np.abs(bl)) + np.matmul(np.abs(al), np.abs(bh)))
                       / LOW_GRAIN)
    exact = lowpart_products(parts, schedule)
    if schedule != "tf32":
        assert np.mean(exact != lowpart_products(parts, "tf32")) > 0.5, "the low parts must change most outputs"
    return a, b, exact, parts


def matmul_f64_ieee(a, b) -> np.ndarray:
    """a [M, K] @ b [K, N] in f64 one k at a time, so inf * 0 and inf - inf give NaN as IEEE arithmetic does (an optimised BLAS
    may skip zero terms)."""
    out = np.zeros((a.shape[0], b.shape[1]))
    with np.errstate(invalid="ignore", over="ignore"):
        for k in range(a.shape[1]):
            out = out + a[:, k:k + 1] * b[k:k + 1, :]
    return out


def edge_operands(targets, in_dtype: str, K: int = 256, col_signs=(1.0, -1.0, 0.5)):
    """Rank-1-style operands whose products hit chosen values exactly: row m of A holds target m split into parts exactly
    representable in `in_dtype` (one part every 64 elements of K, so a stream-K cut separates them), and column n of B is
    col_signs[n] at those positions.  out[m, n] = col_signs[n] * targets[m] in exact arithmetic."""
    targets = np.asarray(targets, dtype=np.float64)
    M, N = len(targets), len(col_signs)
    a = np.zeros((M, K))
    for m, t in enumerate(targets):
        rest, slot = t, 0
        while rest != 0:
            with np.errstate(over="ignore"):
                part = float(synth.from_device_dtype(synth.to_device_dtype(np.array([rest], np.float32), in_dtype), in_dtype)[0])
            if not np.isfinite(part):   # f16 rounds 65520 and up to inf: take the largest finite value instead
                part = float(np.copysign(65504.0, rest))
            assert part != 0, f"{t} is below the input dtype's resolution"
            a[m, 64 * slot] = part
            rest -= part
            slot += 1
            assert slot * 64 <= K, f"{t} needs more than {K // 64} parts"
    b = np.zeros((K, N))
    for n, s in enumerate(col_signs):
        b[::64, n] = s
    for arr in (a, b):
        back = synth.from_device_dtype(synth.to_device_dtype(arr.astype(np.float32), in_dtype), in_dtype)
        assert np.array_equal(back, arr), "an edge operand is not representable in the input dtype"
    return a, b, np.outer(targets, np.asarray(col_signs, dtype=np.float64))


# ------------------------------------------------------------------------------------------------ plan probe
@dataclass
class Plan:
    text: str
    kernels: list = field(default_factory=list)   # GEMM / conv kernel launches, in order
    head: bool = False                            # a stream-K head was planned
    whole_tiles: int = 0                          # whole tiles of the launch with the head (when head)
    tma_store: bool = False                       # whole tiles leave through TMA stores
    phases: int = 0                               # data-gradient output phases

    @property
    def kernel(self) -> str:
        return self.kernels[-1] if self.kernels else ""


_KERNEL = re.compile(r"^launch ((?:gemm|conv2d)_\S+)", re.M)
_HEAD = re.compile(r"gemm stream-k head: (\d+) whole tiles")


class PlanClient(PlanContext):
    """Stands in for a ComputeClient with a dry-run planning context (b200_plan_begin): the library's launch functions take it
    as they take a client, and launch errors raise instead of being deferred."""

    def __init__(self, sms: int, options: dict):
        super().__init__(sms, options)
        self._lib, self._ctx = self.lib, self.ctx

    def _defer(self, err):
        raise err


def _plan_text(sms, options, issue) -> str:
    with PlanClient(sms, options) as pc:
        issue(pc)
        return pc.text()


def probe(sms: int, options: dict, issue) -> Plan:
    """Plan of issue(client) under `options` on a GPU with `sms` SMs.  The store path is read off the plan by planning once more
    with direct stores forced: a TMA-store plan encodes one more tensor map."""
    text = _plan_text(sms, options, issue)
    direct = _plan_text(sms, {**options, "gemm.epilogue": "direct"}, issue)
    head = _HEAD.search(text)
    return Plan(text=text, kernels=_KERNEL.findall(text), head=head is not None, whole_tiles=int(head.group(1)) if head else 0,
                tma_store=text.count("tmap ") > direct.count("tmap "), phases=text.count("conv dgrad phase"))


def out_tag_free(kernel: str) -> str:
    """Kernel name with its output tag removed: plans that differ only in the output dtype give the same string."""
    return re.sub(r"^(gemm_mx|gemm_\w+?|conv2d(?:_dgrad|_wgrad)?_\w+?)_(f32|bf16|f16)_", r"\1_", kernel)


# ------------------------------------------------------------------------------------------------ tensor layouts
FAKE_BASE = 0x10000000


class FakeAlloc:
    """Addresses for planning without a device: every buffer 512-byte aligned, never dereferenced."""

    def __init__(self):
        self.next = FAKE_BASE

    def __call__(self, host: np.ndarray) -> Handle:
        ptr, self.next = self.next, self.next + (host.nbytes + 511) // 512 * 512 + 512
        return Handle(None, ptr, host.nbytes, owner=False)


def device_alloc(client):
    return lambda host: client.create_from_slice(host)


@dataclass(frozen=True)
class GemmCase:
    """One matmul: lhs [batch.., M, K] @ rhs [batch.. or 1, K, N] -> out [batch.., M, N] under plan options."""
    name: str
    in_dtype: str            # bf16, f16, f8e4m3, mixed (e4m3 x e5m2), f32
    out_dtype: str
    M: int
    N: int
    K: int
    batch: int = 0           # 0: rank 2
    bcast: bool = False      # rhs has batch extent 1
    lhs_t: bool = False      # lhs is a transposed view of a [.., K, M] buffer
    rhs_t: bool = False      # rhs is a transposed view of a [.., N, K] buffer
    window: bool = False     # out is a pitched window inside a sentinel-filled buffer
    opts: tuple = ()         # plan options, (key, value) pairs

    @property
    def options(self) -> dict:
        return dict(self.opts)

    def dtypes(self):
        if self.in_dtype == "mixed":
            return "f8e4m3", "f8e5m2"
        return self.in_dtype, self.in_dtype


SENTINEL = {"f32": 0x7F8A5A5A, "bf16": 0x7FA5, "f16": 0x7E5A}   # NaN payloads no conversion produces
WINDOW_COL0, WINDOW_PAD = 8, 24


def gemm_tensors(case: GemmCase, a, b, alloc):
    """(lhs, rhs, out, out buffer) TensorHandles of the case, with a [.., M, K] and b [.., K or 1, K, N] logical values."""
    ld, rd = case.dtypes()

    def operand(vals, dtype, transposed):
        host = np.swapaxes(vals, -1, -2) if transposed else vals
        dev = synth.to_device_dtype(np.ascontiguousarray(host, dtype=np.float32), dtype)
        t = TensorHandle.new_contiguous(list(dev.shape), alloc(dev), dtype)
        return t.transposed() if transposed else t

    lhs = operand(a, ld, case.lhs_t)
    rhs = operand(b, rd, case.rhs_t)
    batch = [case.batch] if case.batch else []
    shape = batch + [case.M, case.N]
    od = case.out_dtype
    if case.window:
        pitch = case.N + WINDOW_PAD
        host = np.full(batch + [case.M, pitch], SENTINEL[od], dtype=OUT_BITS_VIEW[od])
        buf = alloc(host)
        strides = ([case.M * pitch] if batch else []) + [pitch, 1]
        out = TensorHandle(buf.offset(WINDOW_COL0 * DTYPE_SIZE[od]), shape, strides, od)
        return lhs, rhs, out, (buf, host)
    host = np.zeros(shape, dtype=OUT_BITS_VIEW[od])
    return lhs, rhs, TensorHandle.new_contiguous(shape, alloc(host), od), None


def gemm_shapes(case: GemmCase):
    batch = (case.batch,) if case.batch else ()
    rb = (1,) if (case.batch and case.bcast) else batch
    return batch + (case.M, case.K), rb + (case.K, case.N)


def plan_gemm_case(case: GemmCase, sms: int = 132, epilogue=None) -> Plan:
    """Dry-run plan of a case without a device (operand values do not matter to the plan)."""
    from cubecl_b200 import matmul
    ls, rs = gemm_shapes(case)
    a, b = np.zeros(ls), np.zeros(rs)

    def issue(pc):
        lhs, rhs, out, _ = gemm_tensors(case, a, b, FakeAlloc())
        if epilogue:
            matmul.launch(pc, lhs, rhs, out, **epilogue)
        else:
            matmul.launch(pc, lhs, rhs, out)
    return probe(sms, case.options, issue)
