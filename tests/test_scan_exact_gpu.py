"""GPU: axis scans checked exactly on every kernel path (tests/scan_exact_oracle.py).

Integer sums, +-2^k products and planted extremes make every prefix exact in any association, so each case compares every
output bit for bit (NaN as NaN): all four ops, inclusive and exclusive, into f32 and into the input's own 16-bit dtype (the
exact prefix rounded to nearest-even once).  Each op runs on its finite data and then on launches with non-finite values at
the named positions (segment seams, scalar heads, tile starts, ends).  The input buffer holds NaN everywhere outside the
view, and every output is overwritten with a sentinel before its launch.  Each case also asserts, through a dry-run plan of
the same call, the path and kernel it ran; tests/test_scan_exact_cpu.py checks that the case lists below reach every path and
every scan kernel.  A second test checks that an unsegmented column scan is bit-equal to the serial f32 scan on random data."""
import numpy as np
import pytest

import scan_exact_oracle as so
from cubecl_b200 import ComputeClient, TensorHandle, _ffi, scan, synth
from cubecl_b200.client import DTYPE_SIZE
from scan_oracle import scan_axis_f32

pytestmark = pytest.mark.gpu

C = so.ScanCase


def _per_dtype(path, shapes, axis, **kw):
    """One case per dtype; `shapes` is one shape or a {dtype: shape} map."""
    return [C(path, dt, tuple(shapes[dt] if isinstance(shapes, dict) else shapes), axis, **kw) for dt in so.DTYPES]


# >= 32 MB, so the rows are cut into segments; the last segment is short and not a whole number of 512-element blocks.  The
# aligned rows are a whole number of 128-bit vectors long; the misaligned view starts one element in and its odd rows start
# every row at another alignment
THREE_PASS_ROWS = {"f32": (4, 2_100_016), "f16": (4, 4_200_016), "bf16": (4, 4_200_016)}
THREE_PASS_ROWS_ODD = {dt: (4, n + 1) for dt, (_, n) in THREE_PASS_ROWS.items()}

# ------------------------------------------------------------------------------------------------ case lists
ROW_CASES = (
    _per_dtype("rows-thread", (4001, 64), 1)
    + _per_dtype("rows-subwarp", (300, 1000), 1)
    + _per_dtype("rows-warp", (500, 2000), 1)
    + _per_dtype("rows-multiwarp", (200, 8000), 1)
    + _per_dtype("rows-block", (64, 40000), 1)
    + _per_dtype("rows-misaligned", (257, 2041), 1, offset=1)
    + _per_dtype("rows-3pass", THREE_PASS_ROWS, 1)
    + _per_dtype("rows-3pass-misaligned", THREE_PASS_ROWS_ODD, 1, offset=1)
)

COL_CASES = (
    _per_dtype("cols-vec", (200, 64), 0)
    + _per_dtype("cols-scalar", (200, 63), 0)
    + _per_dtype("cols-pitched", (100, 72), 0, pitch=128)
    + _per_dtype("cols-3pass-pitched", (300, 40, 72), 0, pitch=128)
    + _per_dtype("cols-3pass-wide", (200_000, 8), 0)
    + _per_dtype("cols-3pass-narrow", (160, 300, 8), 1)
    + _per_dtype("cols-3pass-scalar", (5000, 63), 0)
)

OTHER_CASES = (
    _per_dtype("gather", (40, 30, 20), 1, permuted=True)
    + _per_dtype("rank8", (1, 3, 1, 5, 1, 700, 1, 2), 5)
    + _per_dtype("unit-axis", (37, 1, 45), 1)
)

# the first pass of a three-pass column scan is the reduce column kernel its context's reduce.cols_loads names; that choice
# cannot be undone on a context, so these run on their own
LOADS_CASES = _per_dtype("cols-3pass-loads4", (200_000, 8), 0, opts=(("reduce.cols_loads", "4"),))

CASES = ROW_CASES + COL_CASES + OTHER_CASES

# the single-pass column cases: a thread walks its column serially, so they equal the serial f32 scan on any data
SERIAL_CASES = [c for c in CASES if c.path in ("cols-vec", "cols-scalar", "cols-pitched", "gather", "unit-axis")]


@pytest.fixture(scope="module")
def loads_client(client):
    c = ComputeClient(0)          # a second context on the same device, dropped at the end of the module
    for k, v in LOADS_CASES[0].opts:
        c.set_option(k, v)
    yield c
    c.sync()
    # destroyed directly: ComputeClient.close() would also drop the session's shared client for device 0 from the cache
    c._lib.b200_destroy(c._ctx)
    c._ctx = None


# ------------------------------------------------------------------------------------------------ running a case
class DeviceView:
    """The case's input buffer on the device: a 512-byte aligned base, the view `offset` elements in, NaN everywhere else.
    A load rewrites the whole buffer when most of the view changes, else only the changed elements."""

    def __init__(self, client, case: so.ScanCase):
        self.client, self.case = client, case
        self.raw = client.empty(case.buffer_elems() * case.esz + 512)
        self.base = self.raw.offset((-self.raw.ptr) % 512)
        self.offs = self.lines(case.offsets())
        self.host = synth.to_device_dtype(np.full(case.buffer_elems(), np.nan, np.float32), case.dtype)
        self.tensor = TensorHandle(self.base.offset(case.offset * case.esz), list(case.shape), case.strides(), case.dtype)
        self.xr = None

    def lines(self, a: np.ndarray) -> np.ndarray:
        """Logical tensor -> [lines, len], the oracle's order."""
        return np.moveaxis(a, self.case.axis, -1).reshape(-1, self.case.shape[self.case.axis])

    def load(self, xr: np.ndarray) -> None:
        changed = None
        if self.xr is not None:
            changed = np.argwhere(~so.outputs_equal(xr, self.xr))
        if changed is None or len(changed) > 4096:
            self.host[self.offs.reshape(-1)] = synth.to_device_dtype(xr.reshape(-1), self.case.dtype)
            self.client.write(self.base, self.host)
        else:
            esz = self.case.esz
            for o, l in changed:
                off = int(self.offs[o, l])
                self.host[off] = synth.to_device_dtype(xr[o, l:l + 1], self.case.dtype)[0]
                self.client.write(self.base.offset(off * esz, esz), self.host[off:off + 1])
        self.xr = xr.copy()


class Outputs:
    """One compact output buffer per out dtype, reused across launches and overwritten with the sentinel before each."""

    def __init__(self, client, case: so.ScanCase):
        self.client, self.n = client, int(np.prod(case.shape))
        self.t = {}
        for dt in case.out_dtypes():
            words = -(-self.n * DTYPE_SIZE[dt] // 4)
            self.t[dt] = TensorHandle.new_contiguous(list(case.shape), client.empty(words * 4), dt)

    def fresh(self, dt: str) -> TensorHandle:
        t = self.t[dt]
        word = so.SENTINEL[dt] if dt == "f32" else so.SENTINEL[dt] * 0x10001
        _ffi.check(self.client._lib.b200_memset32(self.client._ctx, None, t.handle.ptr, word, -(-self.n * DTYPE_SIZE[dt] // 4)))
        return t


def read_lines(client, dv: DeviceView, out: TensorHandle) -> np.ndarray:
    return dv.lines(synth.from_device_dtype(out.to_numpy(client), out.dtype).reshape(dv.case.shape))


def check_case(client, case: so.ScanCase, seed: int = 7) -> None:
    plans = {(op, ex, dt): so.probe(case, op, ex, dt) for op in case.ops for ex in (False, True) for dt in case.out_dtypes()}
    for key, plan in plans.items():
        assert so.path_of(case, plan) == case.path, (case.id, key)
    positions = so.named_positions(case, plans[(case.ops[0], False, "f32")])
    dv, outs = DeviceView(client, case), Outputs(client, case)
    for op in case.ops:
        for label, xr in so.launches(case, op, positions, seed):
            if label == "finite":
                so.assert_preconditions(case, op, xr)
            dv.load(xr)
            for ex in (False, True):
                for dt in case.out_dtypes():
                    out = outs.fresh(dt)
                    scan.launch(client, dv.tensor, out, case.axis, op, ex)
                    assert client.last_kernel() == plans[(op, ex, dt)].kernel, (case.id, op, ex, dt)
                    got = read_lines(client, dv, out)
                    want = so.expected(xr, op, ex, dt)
                    ok = so.outputs_equal(got, want)
                    if not ok.all():
                        o, l = (int(i) for i in np.argwhere(~ok)[0])
                        raise AssertionError(f"{case.id} {op} {'exclusive' if ex else 'inclusive'} -> {dt}, {label}: "
                                             f"{int((~ok).sum())} of {ok.size} outputs differ; first at line {o}, element {l}: "
                                             f"got {got[o, l]!r}, want {want[o, l]!r} ({plans[(op, ex, dt)].kernels})")


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.id)
def test_scan_exact(client, case):
    check_case(client, case)


@pytest.mark.parametrize("case", LOADS_CASES, ids=lambda c: c.id)
def test_scan_exact_cols_loads(loads_client, case):
    check_case(loads_client, case)


# ------------------------------------------------------------------------------------------------ the serial-order contract
@pytest.mark.parametrize("case", SERIAL_CASES, ids=lambda c: c.id)
def test_unsegmented_columns_are_the_serial_f32_scan(client, case):
    # DESIGN 3.2.1: per column the kernel runs the serial f32 order, so on random data (where the order shows) every op is
    # bit-equal to scan_axis_f32, and a 16-bit output is that serial result rounded once
    rng = np.random.default_rng(31)
    dv, outs = DeviceView(client, case), Outputs(client, case)
    shape = case.shape
    for op in case.ops:
        x = rng.uniform(-1.0, 1.0, (case.lines(), case.length())).astype(np.float32)
        if op == "prod":                                   # magnitudes near 1: no product underflows over 300 factors
            x = np.sign(x) * (0.9 + 0.2 * np.abs(x)).astype(np.float32)
        x = so.rne16(x, case.dtype)                        # the values the device holds
        dv.load(x)
        logical = np.moveaxis(x.reshape([n for i, n in enumerate(shape) if i != case.axis] + [shape[case.axis]]), -1, case.axis)
        for ex in (False, True):
            serial = dv.lines(scan_axis_f32(logical, case.axis, op, ex))
            for dt in case.out_dtypes():
                plan = so.probe(case, op, ex, dt)
                assert plan.nseg == 1 and so.path_of(case, plan) == case.path
                out = outs.fresh(dt)
                scan.launch(client, dv.tensor, out, case.axis, op, ex)
                got = read_lines(client, dv, out)
                ok = so.outputs_equal(got, so.rne16(serial, dt))
                assert ok.all(), (case.id, op, ex, dt, int((~ok).sum()))
