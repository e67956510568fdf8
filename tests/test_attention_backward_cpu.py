"""CPU: the f64 attention backward oracle (pinned to torch.autograd through scaled_dot_product_attention in f64), the dry-run
plans of b200_attention_backward (kernels per dtype / head-dim bucket / out dtype / grad dtype, the grids of the three
launches, the workspace, the 4-D tensor maps of compact, [B,S,H,D] and fused-QKV views, gathers), every refusal with its
status, zero extents, deferred rank errors, and the attention_bwd cubin's kernels."""
import ctypes as C
import math
import re
import subprocess

import numpy as np
import pytest
import torch

import attention_backward_oracle as abo
from cubecl_b200 import _ffi
from test_conv_cpu import ROOT, _tool

F32, F16, BF16, I8 = _ffi.F32, _ffi.F16, _ffi.BF16, _ffi.I8
Q, K, V, OUT, DOUT, LSE, DQ, DK, DV = (0x10000000 * i for i in range(1, 10))
INVALID, UNSUPPORTED = 6, 7


# ---------------------------------------------------------------------------------------------- oracle
@pytest.mark.parametrize("B,Hq,Hkv,Sq,Sk,D,causal,scale", [
    (2, 4, 4, 23, 23, 16, False, None), (1, 2, 2, 17, 40, 8, True, None),    # causal, Sq < Sk
    (1, 2, 2, 50, 19, 24, True, None),                                        # causal, Sq > Sk
    (2, 8, 2, 9, 31, 16, False, None), (1, 6, 3, 21, 21, 32, True, None),     # GQA
    (1, 4, 1, 12, 27, 40, False, 0.37), (1, 2, 2, 7, 11, 8, True, 1.5),       # MQA, non-default scale
])
def test_backward_oracle_matches_torch_autograd(B, Hq, Hkv, Sq, Sk, D, causal, scale):
    rng = np.random.default_rng(B * 1000 + Sq * 10 + Sk)
    q, k, v = rng.standard_normal((B, Hq, Sq, D)), rng.standard_normal((B, Hkv, Sk, D)), rng.standard_normal((B, Hkv, Sk, D))
    dout = rng.standard_normal((B, Hq, Sq, D))
    dq, dk, dv = abo.attention_backward_f64(q, k, v, dout, scale, causal)
    qt, kt, vt = (torch.from_numpy(t).requires_grad_() for t in (q, k, v))
    o = torch.nn.functional.scaled_dot_product_attention(qt, kt, vt, is_causal=causal, scale=scale, enable_gqa=Hq != Hkv)
    gq, gk, gv = torch.autograd.grad(o, (qt, kt, vt), torch.from_numpy(dout))
    for got, ref in ((dq, gq), (dk, gk), (dv, gv)):
        np.testing.assert_allclose(got, ref.numpy(), rtol=0, atol=1e-12)


def test_backward_oracle_writes_zero_for_keys_no_query_sees():
    rng = np.random.default_rng(1)
    q, k, v, dout = rng.standard_normal((1, 2, 5, 8)), rng.standard_normal((1, 1, 9, 8)), rng.standard_normal((1, 1, 9, 8)), \
        rng.standard_normal((1, 2, 5, 8))
    _, dk, dv = abo.attention_backward_f64(q, k, v, dout, None, True)
    assert not dk[:, :, 5:].any() and not dv[:, :, 5:].any()


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

    def run(self, qs, ks, idt=BF16, odt=None, gdt=None, shapes=None, strides=None, ptrs=None, lse=LSE, scale=0.125, causal=0,
            null_args=False):
        """shapes / strides / ptrs: dicts over q, k, v, out, dout, dq, dk, dv overriding the compact defaults"""
        odt = idt if odt is None else odt
        gdt = idt if gdt is None else gdt
        sh = {"q": qs, "k": ks, "v": ks, "out": qs, "dout": qs, "dq": qs, "dk": ks, "dv": ks}
        sh.update(shapes or {})
        st = dict.fromkeys(sh)
        st.update(strides or {})
        pt = {"q": Q, "k": K, "v": V, "out": OUT, "dout": DOUT, "dq": DQ, "dk": DK, "dv": DV}
        pt.update(ptrs or {})
        arr = lambda v: _ffi.u64_array(v) if v is not None else None  # noqa: E731
        ops = []
        for n in ("q", "k", "v", "out", "dout"):
            ops += [pt[n], arr(sh[n]), arr(st[n])]
        ops.append(lse)
        for n in ("dq", "dk", "dv"):
            ops += [pt[n], arr(sh[n]), arr(st[n])]
        args = _ffi.AttentionArgs(scale, causal)
        rc = self.lib.b200_attention_backward(self.ctx, None, idt, odt, gdt, *ops, None if null_args else C.byref(args))
        return rc, self.text()

    def close(self):
        self.lib.b200_destroy(self.ctx)


@pytest.fixture
def plan():
    p = Planner()
    yield p
    p.close()


_LAUNCH = re.compile(r"launch (\S+) grid=\((\d+),1,1\) block=(\d+) smem=(\d+) cluster=1")


def _launches(t):
    return [(m.group(1), int(m.group(2)), int(m.group(3)), int(m.group(4))) for m in _LAUNCH.finditer(t)]


_TMAP = re.compile(r"tmap4d esz=(\d+) dims=\(([\d,]+)\) strides=\(([\d,]+)\) box=\(([\d,]+)\) swizzle=3")


def _tmaps(t):
    ints = lambda g: tuple(int(v) for v in g.split(","))  # noqa: E731
    return [(int(m.group(1)), ints(m.group(2)), ints(m.group(3)), ints(m.group(4))) for m in _TMAP.finditer(t)]


def _smem_dq(db):
    return 1024 + 2 * 128 * db * 2 + 2 * 2 * 64 * db * 2 + 1024


def _smem_dkdv(db):
    return 1024 + 2 * 128 * db * 2 + 2 * 2 * 64 * db * 2 + 2 * 2 * 64 * 4 + 1024


@pytest.mark.parametrize("idt,tag", [(BF16, "bf16"), (F16, "f16")])
@pytest.mark.parametrize("D,bucket", [(8, 64), (40, 64), (64, 64), (72, 128), (128, 128)])
@pytest.mark.parametrize("out_f32", [False, True])
@pytest.mark.parametrize("grad_f32", [False, True])
def test_kernels_per_dtype_bucket_out_and_grad(plan, idt, tag, D, bucket, out_f32, grad_f32):
    rc, t = plan.run([2, 4, 300, D], [2, 2, 200, D], idt=idt, odt=F32 if out_f32 else idt, gdt=F32 if grad_f32 else idt)
    assert rc == 0, _ffi.load().b200_last_error()
    g = "f32" if grad_f32 else tag
    assert _launches(t) == [
        (f"attn_bwd_delta_{tag}_{'f32' if out_f32 else tag}", math.ceil(2 * 4 * 384 / 16), 256, 0),
        (f"attn_bwd_dq_{tag}_d{bucket}_{g}", 3 * 4 * 2, 384, _smem_dq(bucket)),
        (f"attn_bwd_dkdv_{tag}_d{bucket}_{g}", 2 * 2 * 2, 384, _smem_dkdv(bucket)),
    ]
    assert "gather" not in t


@pytest.mark.parametrize("causal", [0, 1])
def test_grids_of_the_three_launches(plan, causal):
    for (B, Hq, Hkv, Sq, Sk) in ((1, 1, 1, 1, 1), (3, 6, 2, 128, 129), (3, 5, 5, 129, 1000), (2, 32, 8, 8192, 8192)):
        rc, t = plan.run([B, Hq, Sq, 64], [B, Hkv, Sk, 64], causal=causal)
        assert rc == 0
        nqb, nkb = math.ceil(Sq / 128), math.ceil(Sk / 128)
        assert [(n.split("_")[2], g) for n, g, _, _ in _launches(t)] == [
            ("delta", math.ceil(B * Hq * nqb * 128 / 16)), ("dq", nqb * Hq * B), ("dkdv", nkb * Hkv * B)]


def test_workspace_holds_l_and_delta_of_padded_rows(plan):
    B, Hq, Sq = 2, 6, 300
    rc, t = plan.run([B, Hq, Sq, 64], [B, 3, 77, 64])
    assert rc == 0
    allocs = [int(x) for x in re.findall(r"^alloc (\d+)$", t, re.M)]
    want = 2 * B * Hq * 384 * 4
    assert allocs == [(want + 511) // 512 * 512]
    lines = t.splitlines()
    first_launch = next(i for i, ln in enumerate(lines) if ln.startswith("launch "))
    assert next(i for i, ln in enumerate(lines) if ln.startswith("alloc ")) < first_launch


def test_maps_of_compact_views(plan):
    B, Hq, Hkv, Sq, Sk, D = 2, 8, 2, 300, 200, 128
    rc, t = plan.run([B, Hq, Sq, D], [B, Hkv, Sk, D], gdt=F32)
    assert rc == 0
    qst, kst = (2 * D, 2 * D * Sq, 2 * D * Sq * Hq), (2 * D, 2 * D * Sk, 2 * D * Sk * Hkv)
    qd, kd = (D, Sq, Hq, B), (D, Sk, Hkv, B)
    b128, b64, bg = (64, 128, 1, 1), (64, 64, 1, 1), (32, 64, 1, 1)
    assert _tmaps(t) == [
        # dq kernel: q, k, v, dout, dq
        (2, qd, qst, b128), (2, kd, kst, b64), (2, kd, kst, b64), (2, qd, qst, b128), (4, qd, tuple(2 * s for s in qst), bg),
        # dk / dv kernel: q, k, v, dout, dk, dv
        (2, qd, qst, b64), (2, kd, kst, b128), (2, kd, kst, b128), (2, qd, qst, b64), (4, kd, tuple(2 * s for s in kst), bg),
        (4, kd, tuple(2 * s for s in kst), bg)]


def test_maps_of_bshd_views(plan):
    """[B, S, H, D] tensors and gradients as [B, H, S, D] views: the strides go straight into the maps, no gather"""
    B, H, S, D = 2, 4, 100, 64
    st = [S * H * D, D, H * D, 1]
    rc, t = plan.run([B, H, S, D], [B, H, S, D], strides=dict.fromkeys(("q", "k", "v", "out", "dout", "dq", "dk", "dv"), st))
    assert rc == 0 and "gather" not in t and len(_launches(t)) == 3
    maps = _tmaps(t)
    assert len(maps) == 11
    for esz, dims, strides, box in maps:
        assert dims == (D, S, H, B) and strides == (2 * H * D, 2 * D, 2 * S * H * D)


def test_maps_of_fused_qkv_slices(plan):
    """q / k / v and dq / dk / dv as slices of fused [B, S, 3, H, D] buffers: base offsets H * D elements apart, no gather"""
    B, H, S, D = 2, 4, 100, 64
    st = [S * 3 * H * D, D, 3 * H * D, 1]
    G = 0x90000000
    rc, t = plan.run([B, H, S, D], [B, H, S, D], strides={n: st for n in ("q", "k", "v", "dq", "dk", "dv")},
                     ptrs={"q": Q, "k": Q + 2 * H * D, "v": Q + 4 * H * D, "dq": G, "dk": G + 2 * H * D, "dv": G + 4 * H * D})
    assert rc == 0 and "gather" not in t and len(_launches(t)) == 3
    maps = _tmaps(t)
    fused = (2 * 3 * H * D, 2 * D, 2 * S * 3 * H * D)
    for i in (0, 1, 2, 4, 5, 6, 7, 9, 10):   # every map but dout's
        assert maps[i][1] == (D, S, H, B) and maps[i][2] == fused, i


@pytest.mark.parametrize("case", ["d_stride", "misaligned_base", "odd_stride", "out_f32_odd_stride", "dout_d_stride"])
def test_views_tma_cannot_read_are_gathered(plan, case):
    B, H, S, D = 1, 2, 50, 64
    strides, ptrs, odt = {}, {}, None
    if case == "d_stride":          # k stored [B, H, D, S]: D is not the unit stride
        strides["k"] = [H * D * S, D * S, 1, S]
    elif case == "misaligned_base":
        ptrs["k"] = K + 2
    elif case == "odd_stride":      # an S stride of 68 elements (136 bytes) is not a 16-byte multiple
        strides["k"] = [H * S * 68, S * 68, 68, 1]
    elif case == "out_f32_odd_stride":   # f32 out with an S stride of 66 elements (264 bytes)
        strides["out"], odt = [H * S * 66, S * 66, 66, 1], F32
    else:
        strides["dout"] = [H * D * S, D * S, 1, S]
    rc, t = plan.run([B, H, S, D], [B, H, S, D], strides=strides, ptrs=ptrs, odt=odt)
    assert rc == 0, _ffi.load().b200_last_error()
    names = [n for n, *_ in _launches(t)]
    f32 = odt is not None
    assert names == ["gather_strided", "attn_bwd_delta_bf16_" + ("f32" if f32 else "bf16"), "attn_bwd_dq_bf16_d64_bf16",
                     "attn_bwd_dkdv_bf16_d64_bf16"]
    allocs = re.findall(r"^alloc (\d+)$", t, re.M)
    assert len(allocs) == 2 and int(allocs[0]) == math.ceil(B * H * S * D * (4 if f32 else 2) / 512) * 512
    if case in ("d_stride", "misaligned_base", "odd_stride"):
        assert _tmaps(t)[1][2] == (2 * D, 2 * D * S, 2 * D * S * H)   # the map reads the compact copy


# ---------------------------------------------------------------------------------------------- refusals
@pytest.mark.parametrize("case,status,words", [
    ("batch", INVALID, "batch or head dim"), ("head_dim", INVALID, "batch or head dim"), ("gqa", INVALID, "multiple of Hkv"),
    ("hkv0", INVALID, "multiple of Hkv"), ("v_shape", INVALID, "does not match k"), ("out_shape", INVALID, "out is"),
    ("dout_shape", INVALID, "dout is"), ("dq_shape", INVALID, "dq is"), ("dk_shape", INVALID, "dk is"), ("dv_shape", INVALID, "dv is"),
    ("sk0", INVALID, "Sk = 0"), ("scale_inf", INVALID, "finite"), ("scale_nan", INVALID, "finite"), ("null_ptr", INVALID, "null"),
    ("null_dv", INVALID, "null"), ("null_args", INVALID, "null"), ("null_lse", INVALID, "null"), ("lse_align", INVALID, "lse"),
    ("in_f32", UNSUPPORTED, "input dtype"), ("in_i8", UNSUPPORTED, "input dtype"), ("out_other", UNSUPPORTED, "output dtype"),
    ("grad_other", UNSUPPORTED, "grad dtype"), ("d136", UNSUPPORTED, "head dim"), ("d12", UNSUPPORTED, "head dim"),
    ("dv_dim", UNSUPPORTED, "v's head dim"), ("dq_d_stride", UNSUPPORTED, "dq needs"), ("dk_misaligned", UNSUPPORTED, "dk needs"),
    ("dv_odd_stride", UNSUPPORTED, "dv needs"), ("huge", UNSUPPORTED, "2^31"),
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
        kw["shapes"] = {"v": [2, 2, 81, 64]}
    elif case in ("out_shape", "dout_shape", "dq_shape"):
        kw["shapes"] = {case[:-6]: [2, 4, 101, 64]}
    elif case in ("dk_shape", "dv_shape"):
        kw["shapes"] = {case[:2]: [2, 2, 80, 32]}
    elif case == "sk0":
        ks = [2, 2, 0, 64]
    elif case == "scale_inf":
        kw["scale"] = math.inf
    elif case == "scale_nan":
        kw["scale"] = math.nan
    elif case == "null_ptr":
        kw["ptrs"] = {"dout": 0}
    elif case == "null_dv":
        kw["ptrs"] = {"dv": 0}
    elif case == "null_args":
        kw["null_args"] = True
    elif case == "null_lse":
        kw["lse"] = 0
    elif case == "lse_align":
        kw["lse"] = LSE + 2
    elif case == "in_f32":
        kw["idt"], kw["odt"], kw["gdt"] = F32, F32, F32
    elif case == "in_i8":
        kw["idt"], kw["odt"], kw["gdt"] = I8, F32, F32
    elif case == "out_other":
        kw["idt"], kw["odt"] = BF16, F16
    elif case == "grad_other":
        kw["idt"], kw["gdt"] = BF16, F16
    elif case == "d136":
        qs, ks = [2, 4, 100, 136], [2, 2, 80, 136]
    elif case == "d12":
        qs, ks = [2, 4, 100, 12], [2, 2, 80, 12]
    elif case == "dv_dim":
        kw["shapes"] = {"v": [2, 2, 80, 32]}
    elif case == "dq_d_stride":
        kw["strides"] = {"dq": [4 * 100 * 64, 1, 4 * 64, 4]}
    elif case == "dk_misaligned":
        kw["ptrs"] = {"dk": DK + 2}
    elif case == "dv_odd_stride":
        kw["strides"] = {"dv": [2 * 80 * 68, 80 * 68, 68, 1]}
    elif case == "huge":
        qs, ks = [2, 1 << 31, 100, 64], [2, 1, 80, 64]
    rc, t = plan.run(qs, ks, **kw)
    msg = _ffi.load().b200_last_error().decode()
    assert rc == status, (case, rc, msg)
    assert words in msg, msg
    assert _launches(t) == []


def test_zero_batch_or_no_rows_and_no_keys_plan_nothing(plan):
    for qs, ks in (([0, 4, 100, 64], [0, 2, 80, 64]), ([2, 4, 0, 64], [2, 2, 0, 64]), ([0, 4, 0, 64], [0, 2, 0, 64])):
        rc, t = plan.run(qs, ks)
        assert rc == 0 and t == "", (qs, ks, t)


@pytest.mark.parametrize("qs,ks", [([2, 4, 0, 64], [2, 2, 80, 64]), ([2, 0, 100, 64], [2, 1, 80, 64]),
                                   ([1, 0, 0, 128], [1, 3, 300, 128])])
def test_no_query_rows_still_write_zero_dk_and_dv(plan, qs, ks):
    """Sq = 0 or Hq = 0 with keys: no workspace, no delta or dq launch, and one dk / dv launch that writes every key's +0"""
    rc, t = plan.run(qs, ks, ptrs={"q": 0, "out": 0, "dout": 0, "dq": 0}, lse=0)
    assert rc == 0, _ffi.load().b200_last_error()
    assert "alloc" not in t
    B, Hkv, Sk, D = ks
    assert _launches(t) == [(f"attn_bwd_dkdv_bf16_d{64 if D <= 64 else 128}_bf16", math.ceil(Sk / 128) * Hkv * B, 384,
                             _smem_dkdv(64 if D <= 64 else 128))]
    maps = _tmaps(t)
    assert len(maps) == 6 and maps[4][1] == maps[5][1] == (D, Sk, Hkv, B)


def test_python_launch_backward_defers_rank_errors():
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
    ok = [2, 4, 10, 8]
    attention.launch_backward(stub, _T(ok), _T(ok), _T(ok), _T(ok), _T([2, 4, 10]), _T([2, 4, 10], "f32"), _T(ok), _T(ok), _T(ok))
    assert len(stub.errors) == 1 and stub.errors[0].status == INVALID and "dout must have rank 4" in str(stub.errors[0])
    attention.launch_backward(stub, _T(ok), _T(ok), _T(ok), _T(ok), _T(ok), _T([2, 4, 10], "f32"), _T(ok), _T(ok, "f32"), _T(ok))
    assert len(stub.errors) == 2 and "dq, dk and dv dtypes differ" in str(stub.errors[1])


# ---------------------------------------------------------------------------------------------- kernels
def test_backward_kernels_use_register_a_wgmma_and_tma_and_do_not_spill():
    tool = _tool("cuobjdump")
    _ffi.load()
    cubin = ROOT / "cubecl_b200" / "build" / "attention_bwd.cubin"
    out = subprocess.run([tool, "-res-usage", str(cubin)], capture_output=True, text=True, check=True).stdout
    funcs = re.findall(r"Function (\w+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)
    want = {f"attn_bwd_{k}_{i}_d{d}_{g}" for k in ("dq", "dkdv") for i in ("bf16", "f16") for d in (64, 128) for g in (i, "f32")}
    want |= {f"attn_bwd_delta_{i}_{o}" for i in ("bf16", "f16") for o in (i, "f32")}
    assert {f for f, *_ in funcs} == want
    for name, reg, stack, local in funcs:
        assert int(stack) == 0 and int(local) == 0, (name, stack, local)
    sass = subprocess.run([tool, "-sass", str(cubin)], capture_output=True, text=True, check=True).stdout
    for body in re.split(r"\n\s*Function : ", sass)[1:]:
        name = body.split()[0]
        if "_delta_" in name:
            assert "HGMMA" not in body, name
            continue
        n = 64 if "_d64_" in name else 128
        # dQ += dS K, or dV += P^T dO and dK += dS^T Q: P and dS in registers, the B operand MN-major
        assert re.search(rf"HGMMA\.64x{n}x16\.F32\S* R\d+, R\d+, gdesc\[UR\d+\]\.tnspB", body), name
        assert re.search(r"HGMMA\.64x64x16\.F32\S* R\d+, gdesc\[UR\d+\]", body), name   # the 64-wide score tiles
        assert "UTMALDG.4D" in body and "UTMASTG.4D" in body, name
