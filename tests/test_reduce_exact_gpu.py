"""GPU: reductions checked exactly on every kernel path (tests/reduce_exact_oracle.py).

Nonzero integer / half sums, +-2^k products and planted extremes with ties make every output of every op exact: each case
compares f32 values and u32 indices bit for bit, over launches that move each output's own extremes through the named
positions (ends, segment seams, misaligned head and tail, bulk-tile edge) with and without a later tie, plus one launch with
NaNs there.  Every output is overwritten with a sentinel before its launch.  Each case also
asserts, through a dry-run plan of the same call, which kernel it ran; tests/test_reduce_exact_cpu.py checks that the case
lists below reach every path and every kernel of the reduce image."""
import numpy as np
import pytest

import reduce_exact_oracle as ro
from cubecl_b200 import ComputeClient, TensorHandle, _ffi, reduce, synth

pytestmark = pytest.mark.gpu

RESTORE = {"reduce.variant": "auto", "reduce.cols_fused": "off"}
C = ro.ReduceCase
VAL, ARG = ro.VALUE_OPS, ro.ARG_OPS
SUM_MEAN = ("sum", "mean")


def _per_dtype(path, shapes, axis, **kw):
    """One case per dtype; `shapes` is one shape or a {dtype: shape} map."""
    return [C(path, dt, tuple(shapes[dt] if isinstance(shapes, dict) else shapes), axis, **kw) for dt in ro.DTYPES]


def _v(v):
    return (("reduce.variant", v),)


# ------------------------------------------------------------------------------------------------ case lists
ALL_CASES = (
    _per_dtype("all-plain", (1_000_003,), None, offset=1)
    + _per_dtype("all-bulk", (9_000_011,), None, ops=VAL + ARG, offset=1)          # >= 132 x 8 x 16 KB for every dtype
    + _per_dtype("all-bulk-forced", (600_007,), None, ops=VAL, offset=3, opts=_v("tma"))
    + [C(f"all-{v}", "f32", ((1 << 20) + 4099,), None, ops=SUM_MEAN, offset=3, opts=_v(v))
       for v in ("u2", "u4", "u16", "b4", "b8", "w2", "w4")]
    + _per_dtype("allp-vec", (100, 72), None, pitch=128)
    + _per_dtype("allp-scalar", (100, 70), None, pitch=75)
)

ROW_CASES = (
    _per_dtype("rows-1vec", {"f32": (4001, 4), "f16": (4001, 8), "bf16": (4001, 8)}, 1)
    + _per_dtype("rows-subwarp", (3000, 104), 1)
    + _per_dtype("rows-multiwarp", (300, 4000), 1)
    + _per_dtype("rows-block", (64, 40000), 1)
    + _per_dtype("rows-big", {"f32": (2800, 12000), "f16": (2800, 24000), "bf16": (2800, 24000)}, 1)   # >= 128 MB
    + _per_dtype("rows-misaligned", (257, 2041), 1, offset=1)
    + _per_dtype("rows-2pass", {"f32": (4, 2_100_017), "f16": (4, 4_200_017), "bf16": (4, 4_200_017)}, 1)   # >= 32 MB
)

COL_CASES = (
    _per_dtype("cols-vec", (200, 64), 0)
    + _per_dtype("cols-scalar", (200, 63), 0)
    + _per_dtype("cols-vec-walk", (1100, 100, 8), 1)
    + _per_dtype("cols-vec-perblock", (2, 255, 512), 1)
    + _per_dtype("cols-strided", (6, 50, 72), 1, pitch=128)
    + _per_dtype("cols-pitched", (6, 50, 72), 0, pitch=128)
    + _per_dtype("cols-2pass-wide", (200_000, 8), 0)
    + _per_dtype("cols-2pass-narrow", (160, 300, 8), 1)
    + _per_dtype("cols-fused", (200_000, 8), 0, opts=(("reduce.cols_fused", "on"),))
)

OTHER_CASES = (
    _per_dtype("unit-axis", (37, 1, 45), 1)
    + _per_dtype("gather", (40, 30, 20), 1, permuted=True)
    + _per_dtype("rank8", (1, 3, 1, 5, 1, 700, 1, 2), 5)
)

# a cols_loads choice cannot be undone on a context (its default differs for value and arg ops): these run on their own
LOADS_CASES = (
    _per_dtype("cols-vec-loads4", (200, 64), 0, ops=VAL, opts=(("reduce.cols_loads", "4"),))
    + _per_dtype("cols-vec-loads8", (200, 64), 0, ops=ARG, opts=(("reduce.cols_loads", "8"),))
)

CASES = ALL_CASES + ROW_CASES + COL_CASES + OTHER_CASES


@pytest.fixture(autouse=True)
def _reset_options(client):
    yield
    for k, v in RESTORE.items():
        client.set_option(k, v)


@pytest.fixture(scope="module")
def loads_client(client):
    c = ComputeClient(0)          # a second context on the same device, dropped at the end of the module
    yield c
    c.sync()
    # destroyed directly: ComputeClient.close() would also drop the session's shared client for device 0 from the cache
    c._lib.b200_destroy(c._ctx)
    c._ctx = None


# ------------------------------------------------------------------------------------------------ running a case
class DeviceView:
    """The case's input buffer on the device: a 512-byte aligned base, the view `offset` elements in, NaN everywhere else."""

    def __init__(self, client, case: ro.ReduceCase):
        self.client, self.case = client, case
        esz = case.esz
        self.raw = client.empty(case.buffer_elems() * esz + 512)
        self.base = self.raw.offset((-self.raw.ptr) % 512)
        self.offs = case.offsets()
        self.host = np.full(case.buffer_elems(), synth.to_device_dtype(np.array([np.nan], np.float32), case.dtype)[0])
        view = self.base.offset(case.offset * esz)
        self.tensor = TensorHandle(view, list(case.shape), case.strides(), case.dtype)
        self.xr = None

    def _dev(self, v):
        return synth.to_device_dtype(np.asarray(v, np.float32), self.case.dtype)

    def load(self, xr: np.ndarray) -> None:
        """Make the device hold xr ([outputs, len] values): a whole upload the first time, then only the changed elements."""
        offs_r = self._rows(self.offs)
        if self.xr is None:
            self.host[offs_r.reshape(-1)] = self._dev(xr.reshape(-1))
            self.client.write(self.base, self.host)
        else:
            changed = np.argwhere(~((xr == self.xr) | (np.isnan(xr) & np.isnan(self.xr))))
            esz = self.case.esz
            for o, l in changed:
                off = int(offs_r[o, l])
                self.host[off] = self._dev([xr[o, l]])[0]
                self.client.write(self.base.offset(off * esz, esz), self.host[off:off + 1])
        self.xr = xr.copy()

    def _rows(self, a: np.ndarray) -> np.ndarray:
        """Logical tensor -> [outputs, len] in the order the oracle uses."""
        if self.case.axis is None:
            return a.reshape(1, -1)
        return np.moveaxis(a, self.case.axis, -1).reshape(-1, self.case.shape[self.case.axis])


# written over every output before its launch, in stream order: a finite f32 (-1.0e30) no exact case produces and a u32 far
# beyond any index, so an output the kernel never stores cannot pass with a pooled buffer's earlier result
SENTINEL = 0xF149F2CA


def run_reduce(client, dv: DeviceView, op: str, stream=None) -> TensorHandle:
    out = TensorHandle.empty_contiguous(client, reduce.output_shape(dv.case.shape, dv.case.axis), reduce.output_dtype(op))
    out.handle.used_on(stream)
    _ffi.check(client._lib.b200_memset32(client._ctx, stream, out.handle.ptr, SENTINEL, out.size()))
    reduce.launch(client, dv.tensor, out, dv.case.axis, op, stream=stream)
    return out


def check_case(client, case: ro.ReduceCase, seed: int = 7) -> None:
    for k, v in case.opts:
        client.set_option(k, v)
    plans = {op: ro.probe(case, op) for op in case.ops}
    positions = ro.named_positions(case, plans[case.ops[0]])
    x0 = ro.base_values(case, seed)
    dv = DeviceView(client, case)
    for r, tie, nan in ro.runs(case, positions):
        xr = ro.plant(x0, positions, r, tie, nan)
        if not nan:
            ro.assert_exact_bound(xr)
        dv.load(xr)
        for op in case.ops:
            if nan and op not in ("max", "min") + ARG:
                continue
            out = run_reduce(client, dv, op)
            assert client.last_kernel() == plans[op].kernel, (case.id, op)
            got = out.to_numpy(client).reshape(-1)
            want = ro.expected(xr, op)
            ok = ro.outputs_equal(got, want)
            if not ok.all():
                o = int(np.flatnonzero(~ok)[0])
                raise AssertionError(f"{case.id} {op} launch {r}{'' if tie else ' no tie'}{' NaN' if nan else ''}: {int((~ok).sum())} of {ok.size} outputs "
                                     f"differ; first at {o}: got {got[o]!r}, want {want[o]!r} ({plans[op].kernels})")


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.id)
def test_reduce_exact(client, case):
    check_case(client, case)


@pytest.mark.parametrize("case", LOADS_CASES, ids=lambda c: c.id)
def test_reduce_exact_cols_loads(loads_client, case):
    check_case(loads_client, case)


# ------------------------------------------------------------------------------------------------ state across launches
FUSED = C("cols-fused", "f32", (200_000, 8), 0, opts=(("reduce.cols_fused", "on"),))


def test_fused_column_tickets_reset_across_launches_and_streams(client):
    # every fused launch leaves its per-tile tickets at zero for the next one on the same stream's workspace: three inputs
    # back to back on the client's stream with no host sync between, then again on a second stream
    client.set_option("reduce.cols_fused", "on")
    plan = {op: ro.probe(FUSED, op) for op in ("sum", "mean", "argmax")}
    assert all(p.fused for p in plan.values())
    views, inputs = [], []
    for seed in (11, 12, 13):
        dv = DeviceView(client, FUSED)
        xr = ro.plant(ro.base_values(FUSED, seed), ro.named_positions(FUSED, plan["sum"]), seed)
        dv.load(xr)
        views.append(dv)
        inputs.append(xr)
    stream = client.create_stream()
    try:
        for s in (None, stream):
            outs = []
            for _ in range(2):
                for dv in views:
                    for op in plan:
                        outs.append((dv, op, run_reduce(client, dv, op, stream=s)))
            if s is not None:
                client.sync_stream(s)
            for dv, op, out in outs:
                got = out.to_numpy(client).reshape(-1)
                assert ro.outputs_equal(got, ro.expected(dv.xr, op)).all(), (s is not None, op)
    finally:
        client.destroy_stream(stream)


def test_all_reduction_sees_input_rewritten_on_the_stream(client):
    # reduce, rewrite the input on the same stream (a copy, then a memset), reduce again -- no host sync between: the second
    # result must be the new input's exact value, for the plain and the bulk-copy kernels alike
    for n, kernel in (((1 << 20) + 5, "reduce_all_sum_f32"), (9_000_011, "reduce_all_sum_f32_tma")):
        case = C("all", "f32", (n,), None)
        assert ro.probe(case, "sum").kernel == kernel
        dv = DeviceView(client, case)
        x1 = ro.base_values(case, 21)
        dv.load(x1)
        x2 = -x1[:, ::-1].copy()
        sums = [float(ro.expected(x1, "sum")[0]), float(ro.expected(x2, "sum")[0]), -float(n)]
        assert len(set(sums)) == 3, "a stale read of the earlier input must change the result"
        host2 = synth.to_device_dtype(x2.reshape(-1).astype(np.float32), "f32")
        first = run_reduce(client, dv, "sum")
        client.write_async(dv.base, host2)
        second = run_reduce(client, dv, "sum")
        assert client.last_kernel() == kernel
        _ffi.check(client._lib.b200_memset32(client._ctx, None, dv.base.ptr, int(np.float32(-1.0).view(np.uint32)), n))
        third = run_reduce(client, dv, "sum")
        assert client.last_kernel() == kernel
        client.sync()
        assert float(first.to_numpy(client)[0]) == float(ro.expected(x1, "sum")[0])
        assert float(second.to_numpy(client)[0]) == float(ro.expected(x2, "sum")[0])
        assert float(third.to_numpy(client)[0]) == -float(n)
