"""CPU: the quantization oracle against the reference's known answers and scale-storage properties, the host plans of
b200_quantize / b200_dequantize through a dry-run planning context (launches, view handling, validation), and the
register report of the quant kernels."""
import ctypes as C
import json
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

from plan_context import PlanContext
import quant_oracle as qo
from cubecl_b200 import _ffi, synth
from cubecl_b200.quant import QuantScheme

ROOT = Path(__file__).resolve().parent.parent
F32, F16, BF16, U32, F8E4M3, UE8M0 = _ffi.F32, _ffi.F16, _ffi.BF16, _ffi.U32, _ffi.F8E4M3, _ffi.UE8M0
A, V, S, T = 0x10000000, 0x30000000, 0x50000000, 0x60000000
REF_DTYPES = {"F32": "f32", "F16": "f16", "BF16": "bf16", "UE4M3": "ue4m3", "UE8M0": "ue8m0"}


@pytest.fixture(scope="module")
def golden():
    """Numbers extracted from the reference (tests/golden/make_quant_golden.py)."""
    return json.loads((Path(__file__).resolve().parent / "golden" / "quant_golden.json").read_text())


def kat_inputs(kat):
    """(scheme, values bytes, stored block scales or None, tensor scale, expected f32 values) of one reference KAT."""
    value = kat["value"].lower()
    values = qo.words_to_bytes(kat["words"])
    i = np.arange(kat["len"])
    if kat["block"] == 0:
        scheme = QuantScheme().with_value(value).per_tensor()
        ts = np.float32(kat["tensor_scale"])
        if kat["formula"] == "int_range_times_scale":
            exp = (np.arange(-8, 8).astype(np.float32) * ts).astype(np.float32)
        else:
            exp = (synth.e2m1_codes_to_f32(i.astype(np.uint8)) * ts).astype(np.float32)
        return scheme, values, None, ts, exp
    dt = REF_DTYPES[kat["block_scale"]]
    scheme = QuantScheme().per_block(kat["block"], dt).per_tensor().with_value(value)
    g = np.float32(np.ldexp(1.0, kat["global_scale_pow2"]))
    bs = np.array(kat["block_scales"], dtype=np.float32)
    assert np.array_equal(qo.scale_load(dt, qo.scale_store(dt, bs)), bs)   # the literals are exact in their dtype
    exp = ((g * bs[i // kat["block"]]).astype(np.float32) * (i - 8).astype(np.float32)).astype(np.float32)
    return scheme, values, qo.scale_store(dt, bs), g, exp


def probe_grid(g, dt):
    spec = g["round_up_grid"]
    grid = [np.float32(step / spec["step_div"]) * np.float32(2.0 ** e)
            for e in range(*spec["exp"]) for step in range(*spec["step"])]
    mx = np.float32(g["scale_dtypes"][dt]["max"])
    with np.errstate(over="ignore"):
        grid += [np.float32(mx * np.float32(m)) for m in spec["max_multipliers"]] + [np.float32(np.finfo(np.float32).max)]
    return np.array(grid, dtype=np.float32)


# ---------------------------------------------------------------------------------------------- oracle vs the reference
@pytest.mark.parametrize("out_dtype", ["f32", "f16", "bf16"])
@pytest.mark.parametrize("name", ["test_quantized_per_tensor_int", "test_quantized_per_tensor_fp4", "test_quantized_global_scale",
                                  "test_quantized_two_level_int", "test_quantized_two_level_ue4m3"])
def test_oracle_reproduces_the_reference_kats(golden, name, out_dtype):
    scheme, values, scales, ts, exp = kat_inputs(golden["kats"][name])
    got = qo.dequantize(values, scheme, [16], scales, ts, out_dtype)
    assert np.array_equal(got, synth.to_device_dtype(exp, out_dtype))


def test_packed_words_are_the_byte_stream():
    b = qo.words_to_bytes([0xFEDCBA98, 0x76543210])
    assert b.tolist() == [0x98, 0xBA, 0xDC, 0xFE, 0x10, 0x32, 0x54, 0x76]
    fields = qo.unpack(b, 4, 16)
    assert fields.tolist() == [(i + 8) % 16 for i in range(16)]   # field i = nibble i of the words, low bits first
    assert np.array_equal(qo.pack(fields, 4), b)
    assert np.array_equal(qo.pack(qo.unpack(b, 2, 32), 2), b) and np.array_equal(qo.pack(qo.unpack(b, 8, 8), 8), b)
    # e2m1: the existing two-per-byte convention (element 2i in the low nibble)
    codes = np.arange(16, dtype=np.uint8)
    assert np.array_equal(qo.pack(codes, 4), synth.pack_e2m1x2(codes))


def test_constants_match_the_reference(golden):
    for ref, dt in REF_DTYPES.items():
        assert np.float32(golden["scale_dtypes"][ref]["max"]) == qo.MAX_REPR[dt], ref
    for ref, dt in (("F16", "f16"), ("BF16", "bf16"), ("UE4M3", "ue4m3")):
        assert golden["scale_dtypes"][ref]["bit_step"] == qo.BIT_STEP[dt]
    for ref, dt in (("F16", "f16"), ("UE4M3", "ue4m3")):
        c = golden["scale_dtypes"][ref]
        assert (np.float32(c["min_normal"]), np.float32(c["spacing"])) == qo.SUBNORMALS[dt]
    assert {k.lower(): tuple(v) for k, v in golden["range"].items()} == qo.RANGE


def _step(dt, v, off):
    """`off` representable steps from v, counted on the storage type's own bits (scheme.rs:859-875)."""
    if dt == "f16":
        return np.float32((np.float16(v).view(np.uint16) + np.uint16(off) if off > 0 else np.float16(v).view(np.uint16) - np.uint16(-off)).view(np.float16))
    if dt == "bf16":
        b = int(synth.f32_to_bf16_bits(np.array([v], np.float32))[0]) + off
        return synth.bf16_bits_to_f32(np.array([b], np.uint16))[0]
    b = int(synth.f32_to_fp8_bits(np.array([v], np.float32), "f8e4m3")[0]) + off
    return synth.fp8_bits_to_f32(np.array([b], np.uint8), "f8e4m3")[0]


@pytest.mark.parametrize("dt", ["f16", "bf16", "ue4m3"])
def test_round_up_has_the_reference_properties(golden, dt):
    grid = probe_grid(golden, {"f16": "F16", "bf16": "BF16", "ue4m3": "UE4M3"}[dt])
    up = qo.round_up(dt, grid)
    assert np.all(up >= np.minimum(grid, qo.MAX_REPR[dt]))                 # never below (or the maximum)
    assert np.all(np.isfinite(up)) and up.max() == qo.MAX_REPR[dt]          # saturates rather than stepping off the top
    assert np.array_equal(qo.round_up(dt, up), up)                          # idempotent
    assert np.array_equal(qo.round_up(dt, qo.MAX_REPR[dt]), np.float32(qo.MAX_REPR[dt]))
    # nearest not below: one step down from the answer lands below the scale (positive answers in the normal range)
    for s, u in zip(grid, up):
        if 0 < s < qo.MAX_REPR[dt] and u > 0:
            assert _step(dt, u, -1) < s, (dt, s, u)
    # the reference's own probes (scheme.rs:776-793): 1.7 * 2^exp
    for e in range(-8, 6):
        s = np.float32(np.float32(1.7) * np.float32(2.0 ** e))
        u = qo.round_up(dt, s)
        assert u == qo.round_up(dt, u) and _step(dt, u, -1) < s


def test_round_up_f32_and_ue8m0(golden):
    for s in (1.0e-30, 0.1, 1.0, 12345.678, float(np.finfo(np.float32).max)):
        assert qo.round_up("f32", np.float32(s)) == np.float32(s)
    grid = probe_grid(golden, "UE8M0")
    grid = grid[np.isfinite(grid)]
    up = qo.round_up("ue8m0", grid)
    e = np.log2(up.astype(np.float64))
    assert np.array_equal(e, np.round(e))                                   # powers of two
    below = grid <= np.float32(2.0 ** 127)
    assert np.all(up[below] >= grid[below]) and np.all(up[below] / 2 < grid[below])   # the smallest one not below
    assert np.all(up[~below] == np.float32(2.0 ** 127))                    # clamped to code 254
    assert qo.ue8m0_code(np.float32(0)) == 0 and qo.ue8m0_code(np.float32(2.0 ** -127)) == 0
    assert qo.ue8m0_code(np.float32(2.0 ** -127) * np.float32(1.5)) == 1


def test_synth_encoders_agree_with_the_oracle():
    # every e4m3 / e5m2 / e2m1 value, the midpoints between neighbours (ties), their f32 neighbours, saturation and non-finites
    xs = []
    for kind in ("f8e4m3", "f8e5m2"):
        t = synth.fp8_bits_to_f32(np.arange(256, dtype=np.uint8), kind).astype(np.float64)
        t = np.unique(t[np.isfinite(t)])
        xs += [t, (t[1:] + t[:-1]) / 2]
    t = np.unique(np.concatenate([synth.E2M1_VALUES, -synth.E2M1_VALUES]).astype(np.float64))
    xs += [t, (t[1:] + t[:-1]) / 2]
    x = np.concatenate(xs).astype(np.float32)
    x = np.concatenate([x, np.nextafter(x, np.float32(np.inf)), np.nextafter(x, np.float32(-np.inf)), -x,
                        np.array([np.inf, -np.inf, np.nan, -np.nan, 1e30, -1e30, 0.0, -0.0, 7.0, 1e-45], np.float32)])
    for value in ("e4m3", "e5m2"):
        assert np.array_equal(synth.f32_to_fp8_bits(x, "f8" + value), qo.fp8_codes(x, value)), value
    assert np.array_equal(synth.f32_to_e2m1_codes(x), qo.e2m1_codes(x))
    # the three edge cases: a zero scale gives 0, +-inf saturates with its sign, NaN gives 0 (integers, e2m1) / 0x7F (fp8)
    edge = np.array([np.inf, -np.inf, np.nan, 1.0], np.float32)
    assert qo.encode(edge, np.float32(1), "e4m3").tolist() == [0x7E, 0xFE, 0x7F, 0x38]
    assert qo.encode(edge, np.float32(1), "e5m2").tolist() == [0x7B, 0xFB, 0x7F, 0x3C]
    assert qo.encode(edge, np.float32(1), "e2m1").tolist() == [0x7, 0xF, 0x0, 0x2]
    assert qo.encode(edge, np.float32(1), "q4f").tolist() == [7, 8, 0, 1]           # -8 as a 4-bit field
    assert qo.encode(edge, np.float32(0), "e4m3").tolist() == [0, 0, 0, 0]
    assert qo.encode(np.array([0.5, 1.5, 2.5, -0.5], np.float32), np.float32(1), "q8s").tolist() == [0, 2, 2, 0]


def test_quantize_oracle_round_trip():
    x = synth.uniform_f32(5, 4 * 64, -3.0, 3.0).reshape(4, 64)
    for scheme in (QuantScheme().with_value("q8s").per_block(32, "f16"), QuantScheme().with_value("q4s").per_tensor(),
                   QuantScheme().with_value("q8f").per_block(16, "ue4m3").per_tensor()):
        v, s, t = qo.quantize(x, scheme)
        back = qo.dequantize(v, scheme, x.shape, s, t)
        eff = qo.effective_scale(scheme, 64, (4,), s, t)
        assert np.all(np.abs(back - x) <= eff / 2), scheme
    v, s, t = qo.quantize(x, QuantScheme.mxfp8())
    assert s.dtype == np.uint8 and s.shape == (4, 2) and t is None and v.shape == (4, 64)


# ---------------------------------------------------------------------------------------------- dry-run plans
class Planner(PlanContext):
    def quantize(self, scheme, dt, shape, strides=None, a=A, v=V, s=S, t=T):
        sc = scheme if isinstance(scheme, _ffi.QuantScheme) else scheme.to_c()
        s = s if sc.block else 0
        t = t if sc.tensor_scale else 0
        rc = self.lib.b200_quantize(self.ctx, None, C.byref(sc), dt, a, v, s, t, len(shape), _ffi.u64_array(shape),
                                    _ffi.u64_array(strides) if strides else None)
        return rc, self.text()

    def dequantize(self, scheme, odt, shape, v=V, s=S, t=T, o=A):
        sc = scheme if isinstance(scheme, _ffi.QuantScheme) else scheme.to_c()
        s = s if sc.block else 0
        t = t if sc.tensor_scale else 0
        rc = self.lib.b200_dequantize(self.ctx, None, C.byref(sc), odt, v, s, t, o, len(shape), _ffi.u64_array(shape))
        return rc, self.text()


@pytest.fixture
def plan():
    with Planner() as p:
        yield p


def launches(text):
    return [ln.split()[1] for ln in text.splitlines() if ln.startswith("launch")]


def test_plans(plan):
    # per-block: one launch; 8192 x 1024 chunks of eight bf16, 256 threads (eight MX blocks of four lanes) per CTA
    rc, t = plan.quantize(QuantScheme.mxfp8(), BF16, [8192, 8192])
    assert rc == 0 and t == "launch quant_encode_bf16 grid=(32768,1,1) block=256 smem=0 cluster=1\n"
    rc, t = plan.quantize(QuantScheme.mxfp4(), F32, [3, 5, 64])
    assert rc == 0 and t == "launch quant_encode_f32 grid=(1,1,1) block=256 smem=0 cluster=1\n"
    # a tensor level: the pooled absmax word is reset, the absmax pass runs, then the encode pass
    rc, t = plan.quantize(QuantScheme().with_value("q8s").per_tensor(), F32, [1 << 28])
    assert rc == 0 and t == ("alloc 512\nmemset32 1\n"
                             "launch quant_absmax_f32 grid=(1056,1,1) block=256 smem=0 cluster=1\n"
                             "launch quant_encode_f32 grid=(262144,1,1) block=256 smem=0 cluster=1\n")
    rc, t = plan.quantize(QuantScheme.nvfp4(), BF16, [8192, 8192])
    assert rc == 0 and t == ("alloc 512\nmemset32 1\n"
                             "launch quant_absmax_bf16 grid=(1056,1,1) block=256 smem=0 cluster=1\n"
                             "launch quant_encode_bf16 grid=(32768,1,1) block=256 smem=0 cluster=1\n")
    # a level-less scheme resolves to per-tensor f32 (scheme.rs:94-104)
    assert QuantScheme().to_c().tensor_scale == 1
    rc, t = plan.quantize(QuantScheme(), F16, [10, 6])
    assert rc == 0 and launches(t) == ["quant_absmax_f16", "quant_encode_f16"]
    # dequantize: one launch, 16 bytes of codes per thread
    rc, t = plan.dequantize(QuantScheme.mxfp8(), BF16, [8192, 8192])
    assert rc == 0 and t == "launch quant_decode_bf16 grid=(16384,1,1) block=256 smem=0 cluster=1\n"
    rc, t = plan.dequantize(QuantScheme.nvfp4(), F32, [4, 32])
    assert rc == 0 and t == "launch quant_decode_f32 grid=(1,1,1) block=256 smem=0 cluster=1\n"


def test_views(plan):
    # pitched rows with 16-byte aligned rows are read in place
    rc, t = plan.quantize(QuantScheme.mxfp8(), BF16, [100, 64], strides=[128, 1])
    assert rc == 0 and launches(t) == ["quant_encode_bf16"]
    rc, t = plan.quantize(QuantScheme.mxfp8(), F32, [2, 3, 64], strides=[3 * 72, 72, 1])
    assert rc == 0 and launches(t) == ["quant_encode_f32"]
    rc, t = plan.quantize(QuantScheme().with_value("q4s").per_tensor(), F32, [3, 6], strides=[8, 1])
    assert rc == 0 and launches(t) == ["quant_absmax_f32", "quant_encode_f32"]
    # contiguous strides spelled out are the contiguous plan
    rc, t = plan.quantize(QuantScheme.mxfp8(), F16, [4, 64], strides=[64, 1])
    assert rc == 0 and launches(t) == ["quant_encode_f16"]
    # a transposed view, rows that are not 16-byte aligned, or an unaligned base: one gather first
    rc, t = plan.quantize(QuantScheme.mxfp8(), F32, [64, 96], strides=[1, 64])
    assert rc == 0 and t.splitlines()[0] == "alloc 24576" and launches(t) == ["gather_strided", "quant_encode_f32"]
    rc, t = plan.quantize(QuantScheme.mxfp8(), BF16, [4, 32], strides=[36, 1])
    assert rc == 0 and launches(t) == ["gather_strided", "quant_encode_bf16"]
    rc, t = plan.quantize(QuantScheme.mxfp8(), BF16, [4, 32], a=A + 2)
    assert rc == 0 and launches(t) == ["gather_strided", "quant_encode_bf16"]
    rc, t = plan.quantize(QuantScheme.nvfp4(), BF16, [4, 32], a=A + 2)
    assert rc == 0 and launches(t) == ["gather_strided", "quant_absmax_bf16", "quant_encode_bf16"]
    assert "memset32 1" in t


def _sc(value=_ffi.QV_Q8S, block=32, block_scale=UE8M0, tensor=0):
    return _ffi.QuantScheme(value, block, block_scale, tensor)


def test_validation(plan):
    INVALID, UNSUPPORTED = 6, 7
    q = plan.quantize
    assert q(_sc(), F32, [4, 64])[0] == 0
    assert q(_sc(value=9), F32, [4, 64])[0] == INVALID                       # value outside the enum
    assert q(_sc(value=-1), F32, [4, 64])[0] == INVALID
    assert q(_sc(block_scale=U32), F32, [4, 64])[0] == INVALID               # block-scale dtype outside the list
    assert q(_sc(tensor=2), F32, [4, 64])[0] == INVALID
    assert q(_sc(block=0, tensor=0), F32, [4, 64])[0] == INVALID             # no level at all
    assert q(_sc(block=-8), F32, [4, 64])[0] == INVALID
    assert q(_sc(block=4), F32, [4, 64])[0] == UNSUPPORTED                   # block sizes outside the list
    assert q(_sc(block=256), F32, [4, 256])[0] == UNSUPPORTED
    assert q(_sc(), F32, [4, 48])[0] == INVALID                              # K not divisible by the block
    assert q(_sc(value=_ffi.QV_Q4S, block=0, tensor=1), F32, [4, 3])[0] == INVALID   # a sub-byte row
    assert q(_sc(value=_ffi.QV_Q2S, block=0, tensor=1), F32, [4, 6])[0] == INVALID
    assert q(_sc(value=_ffi.QV_Q2S, block=0, tensor=1), F32, [4, 8])[0] == 0
    assert q(_sc(), U32, [4, 64])[0] == INVALID                              # input dtype outside the list
    # two-level quantize: F16 and ue4m3 block scales only
    for dt, rc in ((F16, 0), (F8E4M3, 0), (F32, UNSUPPORTED), (UE8M0, UNSUPPORTED), (BF16, UNSUPPORTED)):
        assert q(_sc(block_scale=dt, tensor=1), F32, [4, 64])[0] == rc, dt
    # pointers: null for a present level, non-null for an absent one, null input / values
    sc = _sc()
    assert plan.lib.b200_quantize(plan.ctx, None, C.byref(sc), F32, A, V, 0, 0, 2, _ffi.u64_array([4, 64]), None) == INVALID
    assert plan.lib.b200_quantize(plan.ctx, None, C.byref(sc), F32, A, V, S, T, 2, _ffi.u64_array([4, 64]), None) == INVALID
    assert plan.lib.b200_quantize(plan.ctx, None, None, F32, A, V, S, 0, 2, _ffi.u64_array([4, 64]), None) == INVALID
    assert q(_sc(), F32, [4, 64], a=0)[0] == INVALID
    assert q(_sc(), F32, [4, 64], v=0)[0] == INVALID
    assert q(_sc(), F32, [4, 64], a=A + 2)[0] == INVALID                     # not element aligned
    assert q(_sc(block_scale=F16), F32, [4, 64], s=S + 1)[0] == INVALID
    assert q(_sc(), F32, [4] * 9)[0] == INVALID
    # a zero extent is a no-op and touches no pointer
    for shape in ([4, 0], [0, 64], [0]):
        assert q(_sc(), F32, shape) == (0, "")
    assert q(_sc(), F32, [0, 64], a=0, v=0) == (0, "")
    # dequantize: every block-scale dtype under a tensor level; the output dtype list
    d = plan.dequantize
    for dt in (F32, F16, BF16, UE8M0, F8E4M3):
        assert d(_sc(block_scale=dt, tensor=1), F32, [4, 64])[0] == 0, dt
    assert d(_sc(), U32, [4, 64])[0] == INVALID
    assert d(_sc(), F32, [4, 48])[0] == INVALID
    assert d(_sc(block=4), F32, [4, 64])[0] == UNSUPPORTED
    assert d(_sc(), F32, [4, 64], o=0)[0] == INVALID
    assert d(_sc(), F32, [4, 64], o=A + 2)[0] == INVALID
    assert d(_sc(), F16, [4, 0]) == (0, "")
    # without a block level the block-scale field is ignored, whatever it holds
    for dt in (U32, _ffi.U8, -1, 1000):
        rc, t = q(_sc(block=0, tensor=1, block_scale=dt), F32, [4, 64])
        assert rc == 0 and launches(t) == ["quant_absmax_f32", "quant_encode_f32"], dt
        rc, t = d(_sc(block=0, tensor=1, block_scale=dt), F32, [4, 64])
        assert rc == 0 and launches(t) == ["quant_decode_f32"], dt
    assert q(_sc(block=32, tensor=1, block_scale=U32), F32, [4, 64])[0] == INVALID
    assert d(_sc(block=32, tensor=1, block_scale=U32), F32, [4, 64])[0] == INVALID


def test_quant_kernels_do_not_spill():
    tool = shutil.which("cuobjdump") or ("/usr/local/cuda/bin/cuobjdump" if Path("/usr/local/cuda/bin/cuobjdump").exists() else None)
    if tool is None:
        pytest.skip("cuobjdump is not installed")
    _ffi.load()   # builds the cubins when they are missing
    out = subprocess.run([tool, "-res-usage", str(ROOT / "cubecl_b200" / "build" / "quant.cubin")], capture_output=True,
                         text=True, check=True).stdout
    funcs = re.findall(r"Function (quant_\w+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)
    assert {f for f, *_ in funcs} == {f"quant_{k}_{d}" for k in ("absmax", "encode", "decode") for d in ("f32", "f16", "bf16")}
    for name, reg, stack, local in funcs:
        assert int(stack) == 0 and int(local) == 0, (name, stack, local)
        assert int(reg) <= 64, (name, reg)   # at least four 256-thread CTAs per SM
