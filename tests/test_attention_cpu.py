"""CPU: the f64 attention oracle (pinned to torch.nn.functional.scaled_dot_product_attention and torch.logsumexp), the dry-run
plans of b200_attention (kernel per dtype / head-dim bucket / out dtype, grid, the 4-D tensor maps of compact, [B,S,H,D] and
fused-QKV views, gathers, D = 40), every refusal with its status, zero extents, and the attention cubin's kernels."""
import ctypes as C
import math
import re
import subprocess

import numpy as np
import pytest
import torch

import attention_oracle as ao
from cubecl_b200 import _ffi
from cubecl_b200.attention import AttentionShapeError, calculate_attention_output
from test_conv_cpu import ROOT, _tool

F32, F16, BF16, I8 = _ffi.F32, _ffi.F16, _ffi.BF16, _ffi.I8
Q, K, V, OUT, LSE = 0x10000000, 0x20000000, 0x30000000, 0x40000000, 0x50000000
INVALID, UNSUPPORTED = 6, 7


# ---------------------------------------------------------------------------------------------- oracle
@pytest.mark.parametrize("B,Hq,Hkv,Sq,Sk,D,causal,scale", [
    (2, 4, 4, 33, 33, 16, False, None), (1, 2, 2, 17, 40, 8, True, None),    # causal, Sq < Sk
    (1, 2, 2, 50, 19, 24, True, None),                                        # causal, Sq > Sk
    (2, 8, 2, 9, 31, 16, False, None), (1, 6, 3, 21, 21, 32, True, None),     # GQA
    (1, 4, 1, 12, 27, 40, False, 0.37), (1, 2, 2, 7, 11, 8, True, 1.5),       # MQA, non-default scale
])
def test_oracle_matches_torch(B, Hq, Hkv, Sq, Sk, D, causal, scale):
    rng = np.random.default_rng(B * 1000 + Sq * 10 + Sk)
    q, k, v = rng.standard_normal((B, Hq, Sq, D)), rng.standard_normal((B, Hkv, Sk, D)), rng.standard_normal((B, Hkv, Sk, D))
    out, lse = ao.attention_f64(q, k, v, scale, causal)
    qt, kt, vt = (torch.from_numpy(t) for t in (q, k, v))
    ref = torch.nn.functional.scaled_dot_product_attention(qt, kt, vt, is_causal=causal, scale=scale, enable_gqa=Hq != Hkv).numpy()
    np.testing.assert_allclose(out, ref, rtol=0, atol=1e-12)
    sc = 1 / math.sqrt(D) if scale is None else scale
    s = sc * torch.einsum("bhid,bhjd->bhij", qt, kt.repeat_interleave(Hq // Hkv, dim=1))
    if causal:
        s = s.masked_fill(torch.ones(Sq, Sk, dtype=torch.bool).triu(1), -math.inf)
    np.testing.assert_allclose(lse, torch.logsumexp(s, dim=-1).numpy(), rtol=1e-13, atol=1e-13)


def test_visible_pairs():
    for Sq, Sk in ((5, 5), (3, 7), (9, 4), (1, 1)):
        mask = np.arange(Sk)[None, :] <= np.arange(Sq)[:, None]
        assert ao.visible_pairs(Sq, Sk, True) == int(mask.sum())
        assert ao.visible_pairs(Sq, Sk, False) == Sq * Sk


def test_output_rule():
    assert calculate_attention_output([2, 8, 100, 64], [2, 2, 70, 64], [2, 2, 70, 64]) == [2, 8, 100, 64]
    for qs, ks, vs in (([2, 8, 10, 64], [2, 3, 7, 64], [2, 3, 7, 64]), ([2, 8, 10, 64], [1, 2, 7, 64], [1, 2, 7, 64]),
                       ([2, 8, 10, 64], [2, 2, 7, 64], [2, 2, 8, 64]), ([2, 8, 10], [2, 2, 7], [2, 2, 7])):
        with pytest.raises(AttentionShapeError):
            calculate_attention_output(qs, ks, vs)


# ---------------------------------------------------------------------------------------------- dry-run plans
class Planner:
    def __init__(self, sms=132):   # H100 SXM
        self.lib = _ffi.load()
        self.ctx = C.c_void_p()
        _ffi.check(self.lib.b200_plan_begin(sms, C.byref(self.ctx)))

    def text(self):
        need = C.c_size_t()
        _ffi.check(self.lib.b200_plan_text(self.ctx, None, 0, C.byref(need)))
        buf = C.create_string_buffer(need.value)
        _ffi.check(self.lib.b200_plan_text(self.ctx, buf, need.value, None))
        return buf.value.decode()

    def run(self, qs, ks, vs=None, outs=None, idt=BF16, odt=None, strides=(None, None, None, None), ptrs=(Q, K, V, OUT), lse=0,
            scale=0.125, causal=0, null_args=False):
        vs = ks if vs is None else vs
        outs = qs if outs is None else outs
        odt = idt if odt is None else odt
        arr = lambda v: _ffi.u64_array(v) if v is not None else None  # noqa: E731
        args = _ffi.AttentionArgs(scale, causal)
        ops = []
        for p, sh, st in zip(ptrs, (qs, ks, vs, outs), strides):
            ops += [p, arr(sh), arr(st)]
        rc = self.lib.b200_attention(self.ctx, None, idt, odt, *ops, lse, None if null_args else C.byref(args))
        return rc, self.text()

    def close(self):
        self.lib.b200_destroy(self.ctx)


@pytest.fixture
def plan():
    p = Planner()
    yield p
    p.close()


def _launches(t):
    return re.findall(r"launch (\S+) grid=\((\d+),1,1\) block=384 smem=(\d+) cluster=1", t)


_TMAP = re.compile(r"tmap4d esz=(\d+) dims=\(([\d,]+)\) strides=\(([\d,]+)\) box=\(([\d,]+)\) swizzle=3")


def _tmaps(t):
    ints = lambda g: tuple(int(v) for v in g.split(","))  # noqa: E731
    return [(int(m.group(1)), ints(m.group(2)), ints(m.group(3)), ints(m.group(4))) for m in _TMAP.finditer(t)]


@pytest.mark.parametrize("idt,tag", [(BF16, "bf16"), (F16, "f16")])
@pytest.mark.parametrize("D,bucket", [(8, 64), (40, 64), (64, 64), (72, 128), (128, 128)])
@pytest.mark.parametrize("out_f32", [False, True])
def test_kernel_per_dtype_bucket_and_out(plan, idt, tag, D, bucket, out_f32):
    rc, t = plan.run([2, 4, 300, D], [2, 4, 200, D], idt=idt, odt=F32 if out_f32 else idt)
    assert rc == 0, _ffi.load().b200_last_error()
    (name, grid, smem), = _launches(t)
    assert name == f"attn_fwd_{tag}_d{bucket}_{'f32' if out_f32 else tag}"
    assert int(grid) == math.ceil(300 / 128) * 4 * 2
    assert int(smem) == 1024 + 5 * 128 * bucket * 2 + 1024
    assert "gather" not in t


def test_grid_counts_query_blocks_heads_and_batches(plan):
    for (B, H, Sq), grid in (((1, 1, 1), 1), ((3, 5, 128), 15), ((3, 5, 129), 30), ((2, 32, 8192), 2 * 32 * 64)):
        rc, t = plan.run([B, H, Sq, 64], [B, H, 100, 64], causal=1)
        assert rc == 0 and int(_launches(t)[-1][1]) == grid


def test_maps_of_compact_views(plan):
    B, Hq, Hkv, Sq, Sk, D = 2, 8, 2, 300, 200, 128
    rc, t = plan.run([B, Hq, Sq, D], [B, Hkv, Sk, D], odt=F32)
    assert rc == 0
    assert _tmaps(t) == [(2, (D, Sq, Hq, B), (2 * D, 2 * D * Sq, 2 * D * Sq * Hq), (64, 128, 1, 1)),
                         (2, (D, Sk, Hkv, B), (2 * D, 2 * D * Sk, 2 * D * Sk * Hkv), (64, 128, 1, 1)),
                         (2, (D, Sk, Hkv, B), (2 * D, 2 * D * Sk, 2 * D * Sk * Hkv), (64, 128, 1, 1)),
                         (4, (D, Sq, Hq, B), (4 * D, 4 * D * Sq, 4 * D * Sq * Hq), (32, 64, 1, 1))]


def test_maps_of_bshd_views(plan):
    """[B, S, H, D] tensors as [B, H, S, D] views: the strides go straight into the maps, no gather"""
    B, H, S, D = 2, 4, 100, 64
    st = [S * H * D, D, H * D, 1]
    rc, t = plan.run([B, H, S, D], [B, H, S, D], strides=(st, st, st, st))
    assert rc == 0 and "gather" not in t and len(_launches(t)) == 1
    for esz, dims, strides, box in _tmaps(t):
        assert dims == (D, S, H, B) and strides == (2 * H * D, 2 * D, 2 * S * H * D)


def test_maps_of_fused_qkv_slices(plan):
    """q / k / v as slices of one [B, S, 3, H, D] projection: base offsets H * D elements apart, no gather"""
    B, H, S, D = 2, 4, 100, 64
    st = [S * 3 * H * D, D, 3 * H * D, 1]
    rc, t = plan.run([B, H, S, D], [B, H, S, D], strides=(st, st, st, None), ptrs=(Q, Q + 2 * H * D, Q + 4 * H * D, OUT))
    assert rc == 0 and "gather" not in t and len(_launches(t)) == 1
    for esz, dims, strides, box in _tmaps(t)[:3]:
        assert dims == (D, S, H, B) and strides == (2 * 3 * H * D, 2 * D, 2 * S * 3 * H * D)


@pytest.mark.parametrize("case", ["d_stride", "misaligned_base", "odd_stride"])
def test_views_tma_cannot_read_are_gathered(plan, case):
    B, H, S, D = 1, 2, 50, 64
    strides, ptrs = [None] * 4, [Q, K, V, OUT]
    if case == "d_stride":          # k stored [B, H, D, S]: D is not the unit stride
        strides[1] = [H * D * S, D * S, 1, S]
    elif case == "misaligned_base":
        ptrs[1] = K + 2
    else:                           # an S stride of 68 elements (136 bytes) is not a 16-byte multiple
        strides[1] = [H * S * 68, S * 68, 68, 1]
    rc, t = plan.run([B, H, S, D], [B, H, S, D], strides=tuple(strides), ptrs=tuple(ptrs))
    assert rc == 0, _ffi.load().b200_last_error()
    names = [ln.split()[1] for ln in t.splitlines() if ln.startswith("launch ")]
    assert names == ["gather_strided", "attn_fwd_bf16_d64_bf16"]
    assert _tmaps(t)[1][2] == (2 * D, 2 * D * S, 2 * D * S * H)   # the map reads the compact copy


def test_head_dim_40_reads_a_64_box(plan):
    rc, t = plan.run([1, 2, 130, 40], [1, 2, 77, 40], odt=F32)
    assert rc == 0
    maps = _tmaps(t)
    assert [m[1][0] for m in maps] == [40] * 4
    assert [m[3][0] for m in maps] == [64, 64, 64, 32]


# ---------------------------------------------------------------------------------------------- refusals
@pytest.mark.parametrize("case,status,words", [
    ("batch", INVALID, "batch or head dim"), ("head_dim", INVALID, "batch or head dim"), ("gqa", INVALID, "multiple of Hkv"),
    ("hkv0", INVALID, "multiple of Hkv"), ("v_shape", INVALID, "does not match k"), ("out_shape", INVALID, "out is"),
    ("sk0", INVALID, "Sk = 0"), ("scale_inf", INVALID, "finite"), ("scale_nan", INVALID, "finite"), ("null_ptr", INVALID, "null"),
    ("null_args", INVALID, "null"), ("lse_align", INVALID, "lse"),
    ("in_f32", UNSUPPORTED, "input dtype"), ("in_i8", UNSUPPORTED, "input dtype"), ("out_other", UNSUPPORTED, "output dtype"),
    ("d136", UNSUPPORTED, "head dim"), ("d12", UNSUPPORTED, "head dim"), ("dv", UNSUPPORTED, "v's head dim"),
    ("out_d_stride", UNSUPPORTED, "out"), ("out_misaligned", UNSUPPORTED, "out"), ("huge", UNSUPPORTED, "2^31"),
])
def test_refusals(plan, case, status, words):
    qs, ks = [2, 4, 100, 64], [2, 2, 80, 64]
    kw = {}
    if case == "batch":
        ks = [1, 2, 80, 64]
    elif case == "head_dim":
        ks = [2, 2, 80, 32]
    elif case == "gqa":
        ks = [2, 3, 80, 64]
    elif case == "hkv0":
        ks = [2, 0, 80, 64]
    elif case == "v_shape":
        kw["vs"] = [2, 2, 81, 64]
    elif case == "out_shape":
        kw["outs"] = [2, 4, 100, 32]
    elif case == "sk0":
        ks = [2, 2, 0, 64]
    elif case == "scale_inf":
        kw["scale"] = math.inf
    elif case == "scale_nan":
        kw["scale"] = math.nan
    elif case == "null_ptr":
        kw["ptrs"] = (Q, 0, V, OUT)
    elif case == "null_args":
        kw["null_args"] = True
    elif case == "lse_align":
        kw["lse"] = LSE + 2
    elif case == "in_f32":
        kw["idt"], kw["odt"] = F32, F32
    elif case == "in_i8":
        kw["idt"], kw["odt"] = I8, F32
    elif case == "out_other":
        kw["idt"], kw["odt"] = BF16, F16
    elif case == "d136":
        qs, ks = [2, 4, 100, 136], [2, 2, 80, 136]
    elif case == "d12":
        qs, ks = [2, 4, 100, 12], [2, 2, 80, 12]
    elif case == "dv":
        kw["vs"] = [2, 2, 80, 32]
    elif case == "out_d_stride":
        kw["strides"] = (None, None, None, [4 * 100 * 64, 1, 4 * 64, 4])
    elif case == "out_misaligned":
        kw["ptrs"] = (Q, K, V, OUT + 2)
    elif case == "huge":
        qs, ks = [2, 1 << 31, 100, 64], [2, 1, 80, 64]
    rc, t = plan.run(qs, ks, **kw)
    msg = _ffi.load().b200_last_error().decode()
    assert rc == status, (case, rc, msg)
    assert words in msg, msg
    assert _launches(t) == []


def test_zero_extents_plan_no_launch(plan):
    for qs, ks in (([0, 4, 100, 64], [0, 2, 80, 64]), ([2, 0, 100, 64], [2, 1, 80, 64]), ([2, 4, 0, 64], [2, 2, 80, 64]),
                   ([2, 4, 0, 64], [2, 2, 0, 64])):
        rc, t = plan.run(qs, ks)
        assert rc == 0 and t == "", (qs, ks, t)


def test_python_launch_defers_rank_errors():
    """the rank check of the Python surface raises nothing at launch; the error waits for sync"""
    from cubecl_b200 import attention

    class _Stub:
        def __init__(self):
            self.errors = []

        def _defer(self, e):
            self.errors.append(e)

    class _T:
        def __init__(self, shape, dtype="bf16"):
            self.shape, self.dtype = shape, dtype

    stub = _Stub()
    attention.launch(stub, _T([2, 4, 10]), _T([2, 4, 10, 8]), _T([2, 4, 10, 8]), _T([2, 4, 10, 8]))
    assert len(stub.errors) == 1 and stub.errors[0].status == INVALID and "rank 4" in str(stub.errors[0])


# ---------------------------------------------------------------------------------------------- kernels
def test_attention_kernels_use_register_a_wgmma_and_tma_and_do_not_spill():
    tool = _tool("cuobjdump")
    _ffi.load()
    cubin = ROOT / "cubecl_b200" / "build" / "attention.cubin"
    out = subprocess.run([tool, "-res-usage", str(cubin)], capture_output=True, text=True, check=True).stdout
    funcs = re.findall(r"Function (\w+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)
    assert {f for f, *_ in funcs} == {f"attn_fwd_{i}_d{d}_{o}" for i in ("bf16", "f16") for d in (64, 128) for o in (i, "f32")}
    for name, reg, stack, local in funcs:
        assert int(stack) == 0 and int(local) == 0, (name, stack, local)
    sass = subprocess.run([tool, "-sass", str(cubin)], capture_output=True, text=True, check=True).stdout
    for body in re.split(r"\n\s*Function : ", sass)[1:]:
        name = body.split()[0]
        n = 64 if "_d64_" in name else 128
        assert re.search(rf"HGMMA\.64x{n}x16\.F32\S* R\d+, R\d+, gdesc\[UR\d+\]\.tnspB", body), name   # O += P V, P in registers
        assert re.search(r"HGMMA\.64x128x16\.F32\S* R\d+, gdesc\[UR\d+\]", body), name                  # S = Q K^T
        assert "UTMALDG.4D" in body and "UTMASTG.4D" in body, name
