"""Exact oracles for the reductions, shared by tests/test_reduce_exact_cpu.py and tests/test_reduce_exact_gpu.py.

Every value used is exact in f32, f16 and bf16, and each contract holds on every kernel path and plan:
  * sum: nonzero values that are integers or halves with sum |x| < 2^24 (2^23 with halves) per output: every f32 partial sum
    is exact in any association, so the result is exactly S.  Dropping or re-reading any element changes S.
  * mean: rne_f32(S * f32(1 / len)), the scale applied once, to the whole sum.
  * prod: mostly +-1 with a few +-2, +-1/2 and the planted extremes +-4 * 2^j per output, so every partial product stays
    normal and the result is exactly +-2^k; dropping or doubling an element flips the sign or moves the exponent.
  * max / min / argmax / argmin: many ties.  In each output o the unique first extremes +-4 * 2^(o mod 8) sit at named
    positions, with a tie later in the same output in one set of launches (the lowest index wins) and without one in another
    (a skipped extreme changes max and min).  In the NaN launch the even outputs hold a NaN at the named position and another
    one later: NaN propagates through max / min and the first NaN wins the arg ops.
The named positions along the reduced axis are element 0 and the last element, the first and last element of a middle
segment of the plan, the scalar head and tail elements of a misaligned view, and the first element after a 16 KB bulk-tile
edge.  `probe` replays a case in a dry-run planning context on 132 SMs; its partials allocation gives the plan's segment
count, and the segment length follows the host's rule (rows: multiples of 512 elements; columns: ceil(len / nseg)).
"""
from __future__ import annotations

import math
import re
from dataclasses import dataclass, field

import numpy as np

from cubecl_b200 import reduce
from cubecl_b200.client import DTYPE_SIZE, Handle, TensorHandle, contiguous_strides
from gemm_exact_oracle import FAKE_BASE, PlanClient

SMS = 132
VALUE_OPS = ("sum", "mean", "prod", "max", "min")
ARG_OPS = ("argmax", "argmin")
ALL_OPS = VALUE_OPS + ARG_OPS
DTYPES = ("f32", "f16", "bf16")
VEC = {"f32": 4, "f16": 8, "bf16": 8}                   # elements per 128-bit load
BULK_TILE_BYTES = 16384                                  # kBulkStageBytes
COLS_THREADS = 256                                       # kColsThreads
BIG_ROWS_BYTES = 128 << 20                               # rows plans switch to 16 vectors per thread at this input size
EXTREME = 4.0                                            # extremes are +-EXTREME * 2^(output mod 8)


@dataclass(frozen=True)
class ReduceCase:
    """One input view, reduced by each of `ops` under plan options `opts`."""
    path: str                # the path label the case exists for (see path_of)
    dtype: str
    shape: tuple
    axis: int | None
    ops: tuple = ALL_OPS
    offset: int = 0          # view base = a 512-byte aligned address + offset elements
    pitch: int = 0           # row pitch (elements) of the last-but-one axis; the padding holds NaN
    permuted: bool = False   # the view is the reversed-axes transpose of a contiguous buffer (only a gather describes it)
    opts: tuple = ()

    @property
    def id(self) -> str:
        return f"{self.path}-{self.dtype}"

    @property
    def options(self) -> dict:
        return dict(self.opts)

    @property
    def esz(self) -> int:
        return DTYPE_SIZE[self.dtype]

    def strides(self) -> list:
        if self.permuted:
            return contiguous_strides(self.shape[::-1])[::-1]
        if self.pitch:
            st = [1] * len(self.shape)
            st[-2] = self.pitch
            for i in range(len(self.shape) - 3, -1, -1):
                st[i] = st[i + 1] * self.shape[i + 1]
            return st
        return contiguous_strides(self.shape)

    def offsets(self) -> np.ndarray:
        """Buffer element offset of every logical element."""
        idx = np.full(self.shape, self.offset, dtype=np.int64)
        for d, (n, s) in enumerate(zip(self.shape, self.strides())):
            sh = [1] * len(self.shape)
            sh[d] = n
            idx += (np.arange(n, dtype=np.int64) * s).reshape(sh)
        return idx

    def buffer_elems(self) -> int:
        st = self.strides()
        return self.offset + sum((n - 1) * s for n, s in zip(self.shape, st)) + 1 + (self.pitch - self.shape[-1] if self.pitch else 0)

    def length(self) -> int:
        return math.prod(self.shape) if self.axis is None else self.shape[self.axis]

    def outputs(self) -> int:
        return math.prod(reduce.output_shape(self.shape, self.axis))


# ------------------------------------------------------------------------------------------------ plan probe
@dataclass
class ReducePlan:
    text: str
    kernels: list = field(default_factory=list)     # reduce kernel launches, in order
    gather: bool = False                            # the view went through into_contiguous first
    nseg: int = 1                                   # segments of the reduced axis (from the partials allocation)
    fused: bool = False                             # a split column reduction finished inside its one launch
    launches: list = field(default_factory=list)    # (kernel, grid, block, pdl) of every reduce launch

    @property
    def kernel(self) -> str:
        return self.kernels[-1] if self.kernels else ""


_LAUNCH = re.compile(r"^launch (\S+) grid=\((\d+),1,1\) block=(\d+) smem=\d+ cluster=1( pdl)?$", re.M)
_ALLOC = re.compile(r"^alloc (\d+)$", re.M)


def fake_tensor(case: ReduceCase) -> TensorHandle:
    h = Handle(None, FAKE_BASE + case.offset * case.esz, case.buffer_elems() * case.esz, owner=False)
    return TensorHandle(h, list(case.shape), case.strides(), case.dtype)


def probe(case: ReduceCase, op: str, sms: int = SMS) -> ReducePlan:
    """Dry-run plan of reducing the case's view with `op` on a GPU with `sms` SMs."""
    with PlanClient(sms, case.options) as pc:
        out = TensorHandle(Handle(None, FAKE_BASE + (1 << 34), 1 << 30, owner=False), reduce.output_shape(case.shape, case.axis),
                           contiguous_strides(reduce.output_shape(case.shape, case.axis)), reduce.output_dtype(op))
        reduce.launch(pc, fake_tensor(case), out, case.axis, op)
        text = pc.text()
    launches = [(m.group(1), int(m.group(2)), int(m.group(3)), bool(m.group(4))) for m in _LAUNCH.finditer(text)]
    gather = any(k == "gather_strided" for k, *_ in launches)
    red = [ln for ln in launches if ln[0].startswith("reduce_")]
    allocs = [int(a) for a in _ALLOC.findall(text)]
    if gather:
        allocs = allocs[1:]                          # the compact copy of the view
    nseg = 1
    if allocs:
        # the pool hands out whole 512-byte granules: the allocation is outputs x nseg x 4 bytes rounded up to one
        L = view_geometry(case)[1]
        nseg = -(-L // host_seg_len(case, sms))
        assert allocs[0] == -(-case.outputs() * nseg * 4 // 512) * 512, \
            f"partials allocation {allocs[0]} is not {case.outputs()} outputs x {nseg} segments x 4 bytes"
    fused = nseg > 1 and len(red) == 1
    return ReducePlan(text=text, kernels=[k for k, *_ in red], gather=gather, nseg=nseg, fused=fused, launches=red)


# ------------------------------------------------------------------------------------------------ host geometry (restated)
def view_geometry(case: ReduceCase):
    """The [outer, len, inner] view the host reduces in place (contiguous, pitched or rank-8 cases; a permuted case is gathered
    into a contiguous copy first): (outer, len, inner, s_outer, s_len, row_len, row_pitch, base_offset_elements)."""
    shape = [n for n in case.shape]
    strides = contiguous_strides(shape) if case.permuted else case.strides()
    off = 0 if case.permuted else case.offset
    if case.axis is None:
        n = math.prod(shape)
        if case.pitch and not case.permuted:
            return 1, n, 1, 0, 1, shape[-1], case.pitch, off
        return 1, n, 1, 0, 1, n, n, off
    a = case.axis
    outer = math.prod(shape[:a])
    inner = math.prod(shape[a + 1:])
    if shape[a] == 1:
        return 1, 1, math.prod(shape), 0, 0, math.prod(shape), math.prod(shape), off
    kept_outer = [i for i in range(a) if shape[i] > 1]
    s_outer = strides[kept_outer[-1]] if kept_outer else 0
    row_len = row_pitch = inner
    if case.pitch and not case.permuted and a <= len(shape) - 3:
        row_len, row_pitch = shape[-1], case.pitch
    return outer, shape[a], inner, s_outer, strides[a], row_len, row_pitch, off


def _pow2_ceil(x):
    p = 1
    while p < x:
        p <<= 1
    return p


def _pow2_floor(x):
    p = 1
    while p * 2 <= x:
        p <<= 1
    return p


def host_seg_len(case: ReduceCase, sms: int = SMS) -> int:
    """Segment length of the reduced axis by the host's rule."""
    outer, L, inner, *_ = view_geometry(case)
    esz, vec = case.esz, VEC[case.dtype]
    if case.axis is None or L == 1:
        return L
    if inner == 1:
        if outer < sms * 4 and L >= 16384 and outer * L * esz >= (32 << 20):
            nseg = min(-(-sms * 16 // outer), L // 4096)
            if nseg > 1:
                return -(-(-(-L // nseg)) // 512) * 512
        return L
    units = inner // vec if inner % vec == 0 else inner
    tiles = -(-units // min(units, 32))
    if outer * tiles < sms * 4 and L >= 256:
        nseg = min(-(-sms * 8 // (outer * tiles)), L // 64)
        if nseg > 1:
            return -(-L // nseg)
    return L


def seg_len_from_plan(case: ReduceCase, nseg: int) -> int:
    L = view_geometry(case)[1]
    if nseg <= 1:
        return L
    inner = view_geometry(case)[2]
    return -(-(-(-L // nseg)) // 512) * 512 if inner == 1 else -(-L // nseg)


def rows_geometry(case: ReduceCase, seg_len: int):
    """(tpr, threads, grid, four_rows_in_flight, big) of a rows launch, by the host's rule."""
    outer, L, _, s_outer, _, _, _, off = view_geometry(case)
    esz, vec = case.esz, VEC[case.dtype]
    nseg = -(-L // seg_len)
    big = outer * L * esz >= BIG_ROWS_BYTES
    vpt = 16 if big else 8
    nv = -(-min(seg_len, L) // vec)
    tpr = min(512, _pow2_ceil(-(-nv // vpt)))
    threads = max(tpr, 256)
    blocks = -(-(outer * nseg) // (threads // tpr))
    uniform = (off * esz) % 16 == 0 and (s_outer * esz) % 16 == 0 and L % vec == 0
    four = tpr <= 32 and uniform and nseg == 1 and L // vec <= tpr
    if four:
        blocks = -(-blocks // 4)
    return tpr, threads, max(1, blocks), four, big


def cols_geometry(case: ReduceCase, seg_len: int, sms: int = SMS):
    """(vector, ctu, grid, walks, per_block) of a column launch, by the host's rule: `walks` when a persistent grid has more
    items than blocks, `per_block` when every item gets its own block."""
    outer, L, inner, s_outer, s_len, row_len, row_pitch, off = view_geometry(case)
    esz, vec = case.esz, VEC[case.dtype]
    vector = (inner % vec == 0 and row_len % vec == 0 and (off * esz) % 16 == 0 and (s_len * esz) % 16 == 0
              and (s_outer * esz) % 16 == 0 and (row_pitch * esz) % 16 == 0)
    units = inner // vec if vector else inner
    nseg = -(-L // seg_len)
    seg = min(seg_len, L)
    ctu_min = min(units, 32)
    rl = min(COLS_THREADS // ctu_min, max(1, _pow2_floor(max(1, seg // 4))))
    ctu = min(units, COLS_THREADS // rl)
    items = outer * nseg * (-(-units // ctu))
    per_block = seg * ctu * (16 if vector else esz) >= (64 << 10)
    cap = 0x7FFFFFFF if per_block else sms * 8
    return vector, ctu, max(1, min(items, cap)), items > cap, per_block


def allp_vector(case: ReduceCase) -> bool:
    _, _, _, _, _, row_len, row_pitch, off = view_geometry(case)
    return row_len % VEC[case.dtype] == 0 and (row_pitch * case.esz) % 16 == 0 and (off * case.esz) % 16 == 0


def path_of(case: ReduceCase, op: str, plan: ReducePlan) -> str:
    """The path label of a planned call, read off the plan and checked against the host's geometry rules."""
    k = plan.kernel
    if len(case.shape) == 8:
        return "rank8"
    if plan.gather:
        return "gather"
    if k.startswith("reduce_allp_"):
        return "allp-vec" if allp_vector(case) else "allp-scalar"
    if k.startswith("reduce_all_"):
        tail = k.split("_")[-1]
        if tail == "tma":
            return "all-bulk-forced" if case.options.get("reduce.variant") == "tma" else "all-bulk"
        return f"all-{tail}" if tail in ("u2", "u4", "u16", "b4", "b8", "w2", "w4") else "all-plain"
    outer, L, inner, *_ = view_geometry(case)
    if L == 1:
        return "unit-axis"
    seg_len = seg_len_from_plan(case, plan.nseg)
    assert seg_len == host_seg_len(case), "the plan's segment count disagrees with the host's segmentation rule"
    first = plan.launches[0]
    if inner == 1:
        tpr, threads, grid, four, big = rows_geometry(case, seg_len)
        assert (first[1], first[2]) == (grid, threads), f"rows launch {first} != restated geometry {(grid, threads)}"
        if plan.nseg > 1:
            return "rows-2pass"
        _, _, _, s_outer, _, _, _, off = view_geometry(case)
        if four:
            return "rows-1vec"
        if big:
            return "rows-big"
        if (off * case.esz) % 16 or (s_outer * case.esz) % 16:
            return "rows-misaligned"
        return "rows-subwarp" if tpr < 32 else "rows-multiwarp" if tpr < 512 else "rows-block"
    vector, ctu, grid, walks, per_block = cols_geometry(case, seg_len)
    assert first[1] == grid, f"column launch grid {first[1]} != restated geometry {grid}"
    if plan.fused:
        return "cols-fused"
    if plan.nseg > 1:
        return "cols-2pass-" + ("wide" if plan.nseg >= 8 else "narrow")
    _, _, _, _, s_len, row_len, _, _ = view_geometry(case)
    if row_len != inner:
        return "cols-pitched"
    if s_len != inner:
        return "cols-strided"
    loads = case.options.get("reduce.cols_loads")
    label = "cols-" + ("vec" if vector else "scalar")
    if walks:
        label += "-walk"
    if per_block:
        label += "-perblock"
    if loads:
        label += "-loads" + loads
    return label


# ------------------------------------------------------------------------------------------------ data
def named_positions(case: ReduceCase, plan: ReducePlan) -> list:
    """Named positions along the reduced axis for each output (lists of distinct indices, ascending)."""
    outer, L, inner, s_outer, s_len, row_len, row_pitch, off = view_geometry(case)
    esz, vec = case.esz, VEC[case.dtype]
    seg_len = seg_len_from_plan(case, plan.nseg)
    nseg = -(-L // seg_len)
    base = [0, L - 1]
    if nseg > 1:
        mid = nseg // 2
        base += [mid * seg_len, min(L, (mid + 1) * seg_len) - 1]
    else:
        base += [L // 2]
    tile = BULK_TILE_BYTES // esz
    out = []
    per_row = inner == 1 and case.axis is not None and (s_outer * esz) % 16 != 0   # rows start at different alignments
    for o in range(case.outputs() if per_row else 1):
        pos = list(base)
        # scalar head and tail of the view (a row o of a rows view, or the whole contiguous run)
        start = (off + (o * s_outer if case.axis is not None and inner == 1 else 0)) * esz
        head = ((16 - start % 16) % 16) // esz
        head = min(head, L)
        if head:
            pos.append(head - 1)
        contiguous_run = case.axis is None and row_len == L or inner == 1
        if contiguous_run:
            run_tile = tile if plan.kernel.endswith("_tma") else vec
            t0 = head + (L - head) // run_tile * run_tile
            if t0 < L:
                pos.append(t0)
            if head + tile < L:
                pos.append(head + tile)
        out.append(sorted({p for p in pos if 0 <= p < L}))
    return out


def base_values(case: ReduceCase, seed: int) -> np.ndarray:
    """Logical input values [outputs, len] (f64), every one nonzero and exact in every dtype: +-1 with a few +-2 and, where the
    exactness bound allows, +-1/2 in every output.  The first half of each output leans positive and the second half negative,
    so the segment sums of a split plan are large next to the output's sum, and a mean scaled per segment rounds differently
    from one scaled once."""
    n_out, L = case.outputs(), case.length()
    rng = np.random.default_rng(seed)
    lean = np.where(np.arange(L) < L // 2, 0.6, 0.4)
    x = np.where(rng.random((n_out, L)) < lean, 1.0, -1.0)
    k = min(40, max(1, L // 16))
    rows = np.repeat(np.arange(n_out), k)
    x[rows, rng.integers(0, L, n_out * k)] *= rng.choice([1.0, 2.0], n_out * k)
    if L <= (1 << 22):
        x[rows, rng.integers(0, L, n_out * k)] *= rng.choice([1.0, 0.5], n_out * k)
    return x


def plant(x0: np.ndarray, positions: list, r: int, tie: bool = True, nan: bool = False) -> np.ndarray:
    """Launch r's input: per output o, the unique first maximum +4 * 2^(o mod 8) at positions[(o + r) % n] and the unique
    first minimum -4 * 2^(o mod 8) at positions[(o + r + 1) % n], each with a tie at a later position when `tie`, so every
    output has its own extremes.  In the NaN launch the even outputs get a NaN at the maximum's position (and, with `tie`, a
    later one) instead of both extremes.  A unit axis keeps its base values outside the NaN launch: there is nothing to order."""
    x = x0.copy()
    L = x.shape[1]
    for o in range(x.shape[0]):
        nan_here = nan and o % 2 == 0
        if L == 1 and not nan_here:
            continue
        pos = positions[o % len(positions)]
        hi = pos[(o + r) % len(pos)]
        lo = pos[(o + r + 1) % len(pos)] if len(pos) > 1 else None
        taken = {hi} | ({lo} if lo is not None else set())

        def later(p):
            for q in list(pos) + [p + 1, p + 2, L - 1]:
                if p < q < L and q not in taken:
                    return q
            return None
        t_hi = later(hi) if tie else None
        taken.add(t_hi)
        t_lo = later(lo) if tie and lo is not None else None
        v = EXTREME * 2.0 ** (o % 8)
        v_hi = np.nan if nan_here else v
        x[o, hi] = v_hi
        if t_hi is not None:
            x[o, t_hi] = v_hi
        if lo is not None and not nan_here:
            x[o, lo] = -v
            if t_lo is not None:
                x[o, t_lo] = -v
    return x


def runs(case: ReduceCase, positions: list) -> list:
    """(r, tie, nan) of every launch of a case: enough rotations that every named position holds an extreme of some output,
    once with ties (the arg ops must keep the first) and once without (a skipped extreme changes max and min), then NaNs."""
    n = max(len(p) for p in positions)
    # positions shared by all outputs: the outputs rotate through them; per-row positions: every row takes each in turn
    rot = range(n if len(positions) > 1 else max(1, -(-n // case.outputs())))
    no_tie = [(r, False, False) for r in rot] if case.length() > 1 else []
    return [(r, True, False) for r in rot] + no_tie + [(0, True, True)]


def assert_exact_bound(xr: np.ndarray) -> None:
    ok = np.isfinite(xr).all(axis=1)
    halves = (xr[ok] != np.round(xr[ok])).any()
    worst = float(np.abs(xr[ok]).sum(axis=1).max()) if ok.any() else 0.0
    assert worst < (2.0 ** 23 if halves else 2.0 ** 24), f"sum |x| = {worst}: f32 partial sums could round"


# ------------------------------------------------------------------------------------------------ expected values
def expected(xr: np.ndarray, op: str) -> np.ndarray:
    """Exact result of op over the last axis of [outputs, len] values: f32 values or u32 indices."""
    L = xr.shape[1]
    with np.errstate(invalid="ignore", over="ignore"):
        if op == "sum":
            return xr.sum(axis=1).astype(np.float32)
        if op == "mean":
            return xr.sum(axis=1).astype(np.float32) * np.float32(1.0 / L)
        if op == "prod":
            return np.prod(xr, axis=1).astype(np.float32)
        if op == "max":
            return xr.max(axis=1).astype(np.float32)
        if op == "min":
            return xr.min(axis=1).astype(np.float32)
        if op == "argmax":
            return np.argmax(xr, axis=1).astype(np.uint32)
        if op == "argmin":
            return np.argmin(xr, axis=1).astype(np.uint32)
    raise ValueError(op)


def outputs_equal(got: np.ndarray, want: np.ndarray) -> np.ndarray:
    """Per-output equality: f32 values bit for bit (a NaN matches a NaN), u32 indices exactly."""
    got, want = np.asarray(got).reshape(-1), np.asarray(want).reshape(-1)
    if want.dtype == np.uint32:
        return got.astype(np.uint32) == want
    g, w = got.astype(np.float32), want.astype(np.float32)
    return (g.view(np.uint32) == w.view(np.uint32)) | (np.isnan(g) & np.isnan(w))


# ------------------------------------------------------------------------------------------------ wrong kernels the data must catch
def mutants(xr: np.ndarray, op: str, positions: list, seg_len: int, padding: bool):
    """(name, result) of kernels that are subtly wrong, each of which must change at least one expected output of the case."""
    L = xr.shape[1]
    flat = sorted({p for pos in positions for p in pos})
    total = xr.sum(axis=1) if op in ("sum", "mean") else np.prod(xr, axis=1) if op == "prod" else None
    s32 = np.float32(1.0 / L)
    for p in flat:
        xp = xr[:, p]
        if op in ("sum", "mean"):
            for name, v in (("drop", total - xp), ("double", total + xp)):
                yield f"{name} {p}", v.astype(np.float32) * (s32 if op == "mean" else np.float32(1))
        elif op == "prod":
            yield f"drop {p}", (total / xp).astype(np.float32)
            yield f"double {p}", (total * xp).astype(np.float32)
        else:   # the element is skipped: only outputs whose result (or a NaN) sits there can change
            ref = expected(xr, op)
            hit = (ref == p) if op in ARG_OPS else (xp == ref) | np.isnan(xp)
            res = ref.copy()
            if hit.any():
                sub = xr[hit].copy()
                sub[:, p] = {"max": -np.inf, "argmax": -np.inf, "min": np.inf, "argmin": np.inf}[op]
                res[hit] = expected(sub, op)
            yield f"drop {p}", res
    nseg = -(-L // seg_len)
    if op == "mean":
        yield "scale twice", expected(xr, "mean") * s32
        if nseg > 1:
            parts = [xr[:, s * seg_len:(s + 1) * seg_len].sum(axis=1).astype(np.float32) * s32 for s in range(nseg)]
            yield "scale per segment", np.sum(np.stack(parts).astype(np.float64), axis=0).astype(np.float32)
    if op in ARG_OPS:
        idx = expected(xr, op).astype(np.int64)
        if nseg > 1:
            yield "index not offset by its segment", (idx - idx // seg_len * seg_len).astype(np.uint32)
        rev = expected(xr[:, ::-1], op).astype(np.int64)
        yield "ties to the higher index", (L - 1 - rev).astype(np.uint32)
    if xr.shape[0] > 1:
        yield "outputs shifted by one", np.roll(expected(xr, op), 1)
    if padding:
        if op in ARG_OPS:
            yield "padding read", np.full(xr.shape[0], L, np.uint32)   # a NaN in the padding would win
        else:
            yield "padding read", np.full(xr.shape[0], np.nan, np.float32)

