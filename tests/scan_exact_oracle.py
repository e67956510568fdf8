"""Exact oracles for the axis scans, shared by tests/test_scan_exact_cpu.py and tests/test_scan_exact_gpu.py.

Every input value is exact in f32, f16 and bf16, and every prefix is the same in any association, so the expected outputs are
exact on every kernel path and plan:
  * sum: nonzero integers +-A per line (A from 1 to 255) with random signs, leaning positive in the first half of the line and
    negative in the second.  Sum |x| < 2^24 per line, so every partial sum is exact in any order; the prefixes of long enough
    lines pass 256 and 2048 in magnitude, so a 16-bit output has to round (rne16 of the exact prefix).  A zero prefix is +0.
  * prod: +-1 with +-2 / +-1/2 steps whose running exponent walks a triangle inside [-12, 12]: every prefix is exactly
    +-2^k and representable in f16 too, and its sign depends only on the count of negative factors.
  * max / min: nonzero integers in [-8, 8] with strictly new extremes planted at the named positions, so the running
    extreme steps exactly there (min data is the negated max data).
  * non-finite launches at the named positions: sum +inf then -inf later (prefixes +inf, then NaN), prod 0 then inf later
    (a signed zero, then NaN), max / min a NaN.  Each is order-independent; the exclusive forms move every onset one element
    later, so a NaN as the last element of a segment reaches the next segment only through its carry.
The named positions along the scanned axis are element 0 and the last element, the first and last element of a middle
segment and of the short last segment, the scalar head elements of a misaligned rows item (in every segment) and the first
element of the tiles after the head.  `probe` replays a call in a dry-run planning context on 132 SMs; its partials
allocation gives the plan's segment count, and the segment length follows the host's rule, restated here.
"""
from __future__ import annotations

import math
import re
from dataclasses import dataclass, field

import numpy as np

import reduce_exact_oracle as ro
from cubecl_b200 import scan, synth
from cubecl_b200.client import DTYPE_SIZE, Handle, TensorHandle, contiguous_strides
from gemm_exact_oracle import FAKE_BASE, PlanClient

SMS = 132
OPS = ("sum", "prod", "max", "min")
DTYPES = ro.DTYPES
VEC = ro.VEC
SCAN_ELEMS = 16                 # kScanElems: elements per thread per rows tile
COL_UNITS = 256                 # kScanColUnits
AMPLITUDES = (1, 3, 37, 255)    # sum data: |x| of line o is AMPLITUDES[o % 4], capped (see amplitudes)
EXP_LIMIT = 12                  # prod data: every prefix is +-2^k with |k| <= EXP_LIMIT
BASE_RANGE = 8                  # max / min data: base values in [-8, -1] u [1, 8]
IDENTITY = {"sum": 0.0, "prod": 1.0, "max": -np.inf, "min": np.inf}
UFUNC = {"sum": np.add, "prod": np.multiply, "max": np.maximum, "min": np.minimum}   # maximum / minimum propagate NaN
# written over every output before its launch: values no exact case produces (f32 -1.0e30, a negative 16-bit subnormal)
SENTINEL = {"f32": 0xF149F2CA, "f16": 0x8001, "bf16": 0x8001}


@dataclass(frozen=True)
class ScanCase(ro.ReduceCase):
    """One input view, scanned along `axis` by each of `ops`, inclusive and exclusive, into f32 and its own 16-bit dtype."""
    ops: tuple = OPS

    def out_dtypes(self) -> tuple:
        return ("f32",) if self.dtype == "f32" else ("f32", self.dtype)

    def lines(self) -> int:
        return self.outputs()


def sentinel_f32(out_dtype: str) -> np.float32:
    """The sentinel as the f32 value a readback of an unwritten output gives."""
    if out_dtype == "f32":
        return np.array([SENTINEL["f32"]], np.uint32).view(np.float32)[0]
    return synth.from_device_dtype(np.array([SENTINEL[out_dtype]], np.uint16).view(np.float16 if out_dtype == "f16" else np.uint16),
                                   out_dtype)[0]


# ------------------------------------------------------------------------------------------------ host geometry (restated)
def _pow2_ceil(x):
    p = 1
    while p < x:
        p <<= 1
    return p


def cols_vector(case: ScanCase) -> bool:
    _, _, inner, s_outer, s_len, row_len, row_pitch, off = ro.view_geometry(case)
    esz, vec = case.esz, VEC[case.dtype]
    return (inner % vec == 0 and row_len % vec == 0 and (off * esz) % 16 == 0 and (s_len * esz) % 16 == 0
            and (s_outer * esz) % 16 == 0 and (row_pitch * esz) % 16 == 0)


def cols_units(case: ScanCase) -> int:
    inner = ro.view_geometry(case)[2]
    return inner // VEC[case.dtype] if cols_vector(case) else inner


def cols_ctu(units: int) -> int:
    return min(COL_UNITS, max(32, _pow2_ceil(units)))


def host_seg_len(case: ScanCase, sms: int = SMS) -> int:
    """Segment length of the scanned axis by the host's rule (scan_axis_view)."""
    outer, L, inner, *_ = ro.view_geometry(case)
    if inner == 1:
        if outer < sms * 4 and L >= 16384 and outer * L * case.esz >= (32 << 20):
            nseg = min(-(-sms * 16 // outer), L // 4096)
            if nseg > 1:
                return -(-(-(-L // nseg)) // 512) * 512
        return L
    units = cols_units(case)
    blocks = outer * -(-units // cols_ctu(units))
    if blocks < sms * 4 and L >= 256:
        nseg = min(-(-sms * 8 // blocks), L // 64)
        if nseg > 1:
            return -(-L // nseg)
    return L


def rows_tpr(case: ScanCase, seg_len: int) -> int:
    L = ro.view_geometry(case)[1]
    chunks = -(-min(seg_len, L) // SCAN_ELEMS)
    return min(512, _pow2_ceil(-(-chunks // 4)))


def rows_geometry(case: ScanCase, seg_len: int):
    """(tpr, threads, grid) of the final rows launch."""
    outer, L, *_ = ro.view_geometry(case)
    tpr = rows_tpr(case, seg_len)
    threads = tpr if tpr > 32 else 256
    return tpr, threads, max(1, -(-(outer * -(-L // seg_len)) // (threads // tpr)))


def cols_geometry(case: ScanCase, seg_len: int):
    """(ctu, grid) of the final column launch."""
    outer, L, *_ = ro.view_geometry(case)
    units = cols_units(case)
    ctu = cols_ctu(units)
    return ctu, max(1, outer * -(-L // seg_len) * -(-units // ctu))


def row_misaligned(case: ScanCase) -> bool:
    _, _, _, s_outer, _, _, _, off = ro.view_geometry(case)
    return bool((off * case.esz) % 16 or (s_outer * case.esz) % 16)


def row_heads(case: ScanCase, seg_len: int) -> np.ndarray:
    """Scalar head length of every rows item [lines, nseg]: elements up to the next 16-byte boundary of its input."""
    outer, L, _, s_outer, _, _, _, off = ro.view_geometry(case)
    esz = case.esz
    nseg = -(-L // seg_len)
    l0 = np.arange(nseg, dtype=np.int64) * seg_len
    start = (off + np.arange(outer, dtype=np.int64)[:, None] * s_outer + l0[None, :]) * esz
    head = ((16 - start % 16) % 16) // esz
    return np.minimum(head, np.minimum(seg_len, L - l0)[None, :])


# ------------------------------------------------------------------------------------------------ plan probe
@dataclass
class ScanPlan:
    text: str
    launches: list = field(default_factory=list)    # (kernel, grid, block, pdl) of every reduce / scan launch, in order
    gather: bool = False                            # the view went through into_contiguous first
    nseg: int = 1                                   # segments of the scanned axis (from the partials allocation)

    @property
    def kernels(self) -> list:
        return [k for k, *_ in self.launches]

    @property
    def kernel(self) -> str:
        return self.kernels[-1] if self.launches else ""


_LAUNCH = re.compile(r"^launch (\S+) grid=\((\d+),1,1\) block=(\d+) smem=\d+ cluster=1( pdl)?$", re.M)
_ALLOC = re.compile(r"^alloc (\d+)$", re.M)


def probe(case: ScanCase, op: str, exclusive: bool = False, out_dtype: str = "f32", sms: int = SMS) -> ScanPlan:
    """Dry-run plan of scanning the case's view with `op` on a GPU with `sms` SMs."""
    n = math.prod(case.shape)
    with PlanClient(sms, case.options) as pc:
        out = TensorHandle(Handle(None, FAKE_BASE + (1 << 34), n * DTYPE_SIZE[out_dtype], owner=False), list(case.shape),
                           contiguous_strides(case.shape), out_dtype)
        scan.launch(pc, ro.fake_tensor(case), out, case.axis, op, exclusive)
        text = pc.text()
    launches = [(m.group(1), int(m.group(2)), int(m.group(3)), bool(m.group(4))) for m in _LAUNCH.finditer(text)]
    gather = any(k == "gather_strided" for k, *_ in launches)
    allocs = [int(a) for a in _ALLOC.findall(text)]
    if gather:
        allocs = allocs[1:]                          # the compact copy of the view
    outer, L, inner, *_ = ro.view_geometry(case)
    nseg = -(-L // host_seg_len(case, sms))
    # the pool hands out whole 512-byte granules: partials and carries are outer x nseg x inner f32 each
    want = [-(-outer * nseg * inner * 4 // 512) * 512] * 2 if nseg > 1 else []
    assert allocs == want, f"allocations {allocs} are not the partials and carries of {nseg} segments ({want})"
    return ScanPlan(text=text, launches=[ln for ln in launches if ln[0].startswith(("scan_", "reduce_"))], gather=gather, nseg=nseg)


def path_of(case: ScanCase, plan: ScanPlan) -> str:
    """The path label of a planned call, read off the plan and checked against the host's geometry rules."""
    if len(case.shape) == 8:
        return "rank8"
    if plan.gather:
        return "gather"
    outer, L, inner, s_outer, s_len, row_len, row_pitch, off = ro.view_geometry(case)
    if L == 1:
        return "unit-axis"
    seg_len = host_seg_len(case)
    final = plan.launches[-1]
    if inner == 1:
        tpr, threads, grid = rows_geometry(case, seg_len)
        assert final[1:3] == (grid, threads), f"rows launch {final} != restated geometry {(grid, threads)}"
        if plan.nseg > 1:
            return "rows-3pass" + ("-misaligned" if row_misaligned(case) else "")
        if row_misaligned(case):
            return "rows-misaligned"
        return ("rows-thread" if tpr == 1 else "rows-subwarp" if tpr < 32 else "rows-warp" if tpr == 32
                else "rows-multiwarp" if tpr < 512 else "rows-block")
    ctu, grid = cols_geometry(case, seg_len)
    assert final[1:3] == (grid, ctu), f"column launch {final} != restated geometry {(grid, ctu)}"
    if plan.nseg > 1:
        if row_len != inner:
            return "cols-3pass-pitched"
        loads = case.options.get("reduce.cols_loads")
        if loads:
            return "cols-3pass-loads" + loads
        return "cols-3pass-" + ("scalar" if not cols_vector(case) else "wide" if plan.nseg >= 8 else "narrow")
    if row_len != inner or s_len != inner:
        return "cols-pitched"
    return "cols-vec" if cols_vector(case) else "cols-scalar"


# ------------------------------------------------------------------------------------------------ named positions
def named_positions(case: ScanCase, plan: ScanPlan) -> list:
    """Named positions along the scanned axis: one ascending list shared by every line, or one per line when rows start at
    different alignments."""
    outer, L, inner, *_ = ro.view_geometry(case)
    seg = host_seg_len(case)
    nseg = -(-L // seg)
    base = {0, L - 1}
    starts = [0]
    if nseg > 1:
        mid = nseg // 2
        base |= {mid * seg, min(L, (mid + 1) * seg) - 1, (nseg - 1) * seg}
        starts += [mid * seg, (nseg - 1) * seg]
    else:
        base.add(L // 2)
    if inner != 1 or L == 1:
        return [sorted(p for p in base if 0 <= p < L)]
    tile = rows_tpr(case, seg) * SCAN_ELEMS
    heads = row_heads(case, seg)
    out = []
    for o in range(outer if row_misaligned(case) else 1):
        pos = set(base)
        for l0 in starts:
            end = min(L, l0 + seg)
            h = int(heads[o, l0 // seg])
            pos |= {l0 + j for j in range(h)}                # the scalar head tile
            pos |= {p for p in (l0 + h, l0 + h + tile) if p < end}   # the first element of each of the next two tiles
        out.append(sorted(p for p in pos if 0 <= p < L))
    return out


def line_positions(positions: list, o: int) -> list:
    return positions[o % len(positions)]


# ------------------------------------------------------------------------------------------------ data
def amplitudes(case: ScanCase) -> np.ndarray:
    """|x| of every line: within the exactness bound A * len < 2^24, and small enough on long lines that the random walk
    (about A * sqrt(len)) stays well inside f16's range."""
    L = case.length()
    cap = max(1, min((2 ** 24 - 1) // L, int(16384 / math.sqrt(L))))
    return np.array([min(AMPLITUDES[o % len(AMPLITUDES)], cap) for o in range(case.lines())], np.float32)


def sum_values(case: ScanCase, seed: int) -> np.ndarray:
    """[lines, len] f32: +-A per line, leaning positive in the first half and negative in the second, so long lines reach
    prefixes beyond 2048 while sum |x| = A * len stays below 2^24."""
    n, L = case.lines(), case.length()
    rng = np.random.default_rng(seed)
    A = amplitudes(case)[:, None]
    delta = np.minimum(0.1, 8000.0 / (L * A))
    lean = np.where(np.arange(L)[None, :] < L // 2, 0.5 + delta, 0.5 - delta)
    return (np.where(rng.random((n, L)) < lean, 1.0, -1.0) * A).astype(np.float32)


def _triangle(k: np.ndarray) -> np.ndarray:
    """Running exponent after step k (k = -1: before any step): 0, 1, .., 12, 11, .., -12, -11, .., 0, ... (period 48)."""
    t = (k + 1) % (4 * EXP_LIMIT)
    return np.where(t <= EXP_LIMIT, t, np.where(t <= 3 * EXP_LIMIT, 2 * EXP_LIMIT - t, t - 4 * EXP_LIMIT))


def prod_values(case: ScanCase, positions: list, seed: int) -> np.ndarray:
    """[lines, len] f32: +-1 with +-2 / +-1/2 steps (about one in 16, and every named position, each negative there) along a
    triangle of exponents within [-12, 12]."""
    n, L = case.lines(), case.length()
    rng = np.random.default_rng(seed)
    x = np.where(rng.random((n, L)) < 0.5, 1.0, -1.0).astype(np.float32)
    step = rng.random((n, L)) < 1.0 / 16
    for o in range(n):
        pos = line_positions(positions, o)
        step[o, pos] = True
        x[o, pos] = -1.0
    k = np.cumsum(step, axis=1, dtype=np.int64) - 1
    e = _triangle(k) - _triangle(k - 1)
    return np.where(step, x * np.exp2(e.astype(np.float32)), x).astype(np.float32)


def max_values(case: ScanCase, positions: list, seed: int) -> np.ndarray:
    """[lines, len] f32: integers in [-8, 8] without 0, and strictly rising maxima 9 + 2i + 50 (o mod 4) at the line's named
    positions, so cummax steps exactly at each of them and neighbouring lines differ."""
    n, L = case.lines(), case.length()
    rng = np.random.default_rng(seed)
    x = (rng.integers(1, BASE_RANGE + 1, (n, L)) * rng.choice([-1, 1], (n, L))).astype(np.float32)
    for o in range(n):
        pos = line_positions(positions, o)
        x[o, pos] = BASE_RANGE + 1 + 2 * np.arange(len(pos)) + 50 * (o % 4)
    return x


def finite_values(case: ScanCase, op: str, positions: list, seed: int) -> np.ndarray:
    if op == "sum":
        return sum_values(case, seed)
    if op == "prod":
        return prod_values(case, positions, seed)
    x = max_values(case, positions, seed)
    return x if op == "max" else -x


def nonfinite_rounds(case: ScanCase, positions: list) -> int:
    """Rounds R of non-finite launches: line o takes the named positions o * R .. o * R + R - 1 in turn, so every index into
    the named positions is some line's first non-finite value."""
    return max(1, -(-max(len(p) for p in positions) // case.lines()))


def plant_nonfinite(x0: np.ndarray, op: str, positions: list, r: int, rounds: int) -> np.ndarray:
    """Round r's non-finite input: line o gets its first non-finite value at its named position (o * rounds + r) mod n
    (sum +inf, prod 0, max / min NaN) and, for sum and prod, the second one (sum -inf, prod inf) at the next one."""
    x = x0.copy()
    for o in range(x.shape[0]):
        pos = line_positions(positions, o)
        i = (o * rounds + r) % len(pos)
        a, b = pos[i], pos[i + 1] if i + 1 < len(pos) else None
        first, second = {"sum": (np.inf, -np.inf), "prod": (0.0, np.inf)}.get(op, (np.nan, None))
        x[o, a] = first
        if b is not None and second is not None:
            x[o, b] = second
    return x


def launches(case: ScanCase, op: str, positions: list, seed: int = 7):
    """(label, input [lines, len]) of every launch of `op` on the case: the finite data, then the non-finite rounds."""
    x0 = finite_values(case, op, positions, seed)
    yield "finite", x0
    rounds = nonfinite_rounds(case, positions)
    for r in range(rounds):
        yield f"non-finite {r}", plant_nonfinite(x0, op, positions, r, rounds)


# ------------------------------------------------------------------------------------------------ expected values
def _scan(x: np.ndarray, op: str, exclusive: bool, init: float | None = None) -> np.ndarray:
    """Serial f32 scan of every line of [lines, len] (exact here), starting from `init` (the identity by default)."""
    x = np.asarray(x, np.float32)
    pad = np.full((x.shape[0], 1), IDENTITY[op] if init is None else init, np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        acc = UFUNC[op].accumulate(np.concatenate([pad, x], axis=1), axis=1, dtype=np.float32)
    return acc[:, :-1] if exclusive else acc[:, 1:]


def rne16(v: np.ndarray, out_dtype: str) -> np.ndarray:
    """f32 values as the out dtype stores them (rounded to nearest-even once), widened back to f32."""
    if out_dtype == "f32":
        return np.asarray(v, np.float32)
    return synth.from_device_dtype(synth.to_device_dtype(np.asarray(v, np.float32), out_dtype), out_dtype).reshape(np.shape(v))


def expected(xr: np.ndarray, op: str, exclusive: bool, out_dtype: str = "f32") -> np.ndarray:
    """Exact scan of every line of [lines, len], as stored in out_dtype (f32 values)."""
    return rne16(_scan(xr, op, exclusive), out_dtype)


def outputs_equal(got: np.ndarray, want: np.ndarray) -> np.ndarray:
    """Elementwise: f32 bits equal (so -0 != +0), or both NaN (any payload)."""
    g, w = np.asarray(got, np.float32), np.asarray(want, np.float32)
    return (g.view(np.uint32) == w.view(np.uint32)) | (np.isnan(g) & np.isnan(w))


def assert_preconditions(case: ScanCase, op: str, xr: np.ndarray) -> None:
    """The finite data is what the exact contracts need."""
    assert np.isfinite(xr).all() and (xr != 0).all(), "finite data holds no zero and no non-finite value"
    for dt in DTYPES:
        assert np.array_equal(rne16(xr, dt), xr), f"a value is not exact in {dt}"
    if op == "sum":
        assert float(np.abs(xr.astype(np.float64)).sum(axis=1).max()) < 2.0 ** 24, "sum |x| >= 2^24: partial sums could round"
        assert (xr == np.round(xr)).all()
    if op == "prod":
        m, e = np.frexp(np.abs(_scan(xr, "prod", False)).astype(np.float64))
        assert (m == 0.5).all() and (np.abs(e - 1) <= EXP_LIMIT).all(), "a prefix product is not +-2^k with |k| <= 12"


# ------------------------------------------------------------------------------------------------ wrong kernels the data must catch
def _trunc16(v: np.ndarray, out_dtype: str) -> np.ndarray:
    v = np.asarray(v, np.float32)
    if out_dtype == "bf16":
        return (v.view(np.uint32) & np.uint32(0xFFFF0000)).view(np.float32)
    h = v.astype(np.float16)
    with np.errstate(invalid="ignore"):
        over = np.abs(h.astype(np.float32)) > np.abs(v)
    return np.where(over, np.nextafter(h, np.float16(0)), h).astype(np.float32)


def _segmented(xr, op, exclusive, seg_len, carry_of):
    """Every segment scanned from the identity, then combined with carry_of(s, start, end) (or left alone for None)."""
    L = xr.shape[1]
    out = np.empty_like(xr, dtype=np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        for s in range(-(-L // seg_len)):
            a, b = s * seg_len, min(L, (s + 1) * seg_len)
            local = _scan(xr[:, a:b], op, exclusive)
            c = carry_of(s, a, b)
            out[:, a:b] = local if c is None else UFUNC[op](c[:, None], local)
    return out


def mutant_truncating_store(want: np.ndarray, out_dtype: str) -> np.ndarray:
    """A 16-bit store that truncates the exact f32 results `want` instead of rounding them to nearest-even."""
    return _trunc16(want, out_dtype)


def mutants(xr: np.ndarray, op: str, exclusive: bool, out_dtype: str, positions: list, seg_len: int, heads, padding: bool,
            nan_only: bool = False):
    """(name, result as stored in out_dtype) of kernels that are subtly wrong.  `heads` is row_heads() of a rows view, else
    None; `padding` marks a view whose row padding a wrong kernel could read; `nan_only` yields only the kernels whose fault
    only a NaN shows."""
    n, L = xr.shape
    want = expected(xr, op, exclusive)                     # f32
    ident = IDENTITY[op]
    sent = sentinel_f32(out_dtype)

    def done(v):
        return rne16(v, out_dtype)

    if op in ("max", "min"):
        with np.errstate(invalid="ignore"):
            f = (np.fmax if op == "max" else np.fmin).accumulate(np.concatenate([np.full((n, 1), ident, np.float32), xr], axis=1),
                                                                 axis=1, dtype=np.float32)
        yield f"{'fmaxf' if op == 'max' else 'fminf'} drops the NaN", done(f[:, :-1] if exclusive else f[:, 1:])
    if nan_only:
        return
    incl = _scan(xr, op, False)

    base = done(want)
    for p in sorted({p for pos in positions for p in pos}):
        # the element at p is lost or read twice in the lines that name p (every line when they share their positions)
        rows = [o for o in range(n) if p in line_positions(positions, o)]
        y = xr[rows].copy()
        y[:, p] = ident
        res = base.copy()
        res[rows] = done(_scan(y, op, exclusive))
        yield f"drop {p}", res
        if op in ("sum", "prod"):
            y[:, p] = xr[rows, p] * xr[rows, p] if op == "prod" else xr[rows, p] * 2
            res = base.copy()
            res[rows] = done(_scan(y, op, exclusive))
            yield f"double {p}", res
    yield "inclusive and exclusive swapped", done(_scan(xr, op, not exclusive))
    yield "outputs shifted by one position", done(np.roll(want, 1, axis=1))
    if n > 1:
        yield "outputs shifted by one line", done(np.roll(want, 1, axis=0))
    nseg = -(-L // seg_len)
    if nseg > 1:
        yield "carry missing", done(_segmented(xr, op, exclusive, seg_len, lambda s, a, b: None))
        yield "carry of the neighbouring segment", done(_segmented(xr, op, exclusive, seg_len, lambda s, a, b: incl[:, b - 1]))
        if op in ("sum", "prod"):                           # max / min are idempotent
            yield "carry applied twice", done(_segmented(
                xr, op, exclusive, seg_len,
                lambda s, a, b: None if s == 0 else UFUNC[op](incl[:, a - 1], incl[:, a - 1])))
    if heads is not None and heads.any():
        lost, shifted = done(want), done(want)
        for o in range(n):
            for s in range(heads.shape[1]):
                a, h = s * seg_len, int(heads[o, s])
                if h:
                    lost[o, a:a + h] = sent
                    shifted[o, a + 1:a + h] = done(want[o, a:a + h - 1])
                    shifted[o, a] = sent
        yield "head-tile outputs lost", lost
        yield "head-tile outputs shifted", shifted
    if exclusive and op != "sum":
        yield "exclusive identity 0", done(_scan(xr, op, True, init=0.0))
    if out_dtype != "f32":
        yield "16-bit store truncates", mutant_truncating_store(want, out_dtype)
    if padding:
        v = np.full((n, L), np.nan, np.float32)
        if exclusive:
            v[:, 0] = ident
        yield "padding read", done(v)
