"""CPU: the rope oracle (tests/rope_oracle.py) pinned to HF's apply_rotary_pos_emb, flash-attn's apply_rotary_emb_torch and
autograd in f64, its tables to transformers' ROPE_INIT_FUNCTIONS; the exact cases' power to catch a wrong contract; the
dry-run plans of b200_rope, b200_rope_kvcache_write and b200_rope_cos_sin; every refusal and zero extent; the Python layer's
deferred errors; and the rope cubin's resources."""
import ctypes as C
import re
import subprocess
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import rope_oracle as ro
from cubecl_b200 import _ffi, rope
from plan_context import PlanContext
from test_conv_cpu import ROOT, _tool

F32, F16, BF16 = _ffi.F32, _ffi.F16, _ffi.BF16
DT = {F32: "f32", BF16: "bf16", F16: "f16"}
INVALID, UNSUPPORTED = 6, 7
Q, K, QO, KO, POS, CS, V, KC, VC, SL, KS, VS = (0x10000000 * i for i in range(1, 13))


# ---------------------------------------------------------------------------------------------- oracle vs torch (f64)
def _hf_neox(x, cos, sin):
    rot = cos.shape[-1] * 2
    c = torch.cat([cos, cos], -1)[:, :, None]
    s = torch.cat([sin, sin], -1)[:, :, None]
    xr = x[..., :rot]
    rh = torch.cat([-xr[..., rot // 2:], xr[..., :rot // 2]], -1)
    return torch.cat([xr * c + rh * s, x[..., rot:]], -1)


@pytest.mark.parametrize("style", ["neox", "gptj"])
@pytest.mark.parametrize("D,rot", [(64, 64), (96, 24), (80, 32), (128, 64)])
def test_oracle_matches_torch_in_f64(style, D, rot):
    rng = np.random.default_rng(D + rot)
    B, S, H, P = 2, 12, 3, 50
    tab = ro.table(P, ro.inv_freq(rot, 10000.0), 1.0)
    x = rng.standard_normal((B, S, H, D)).astype(np.float32)
    pos = rng.integers(0, P, (B, S))
    got = ro.apply(x, tab, pos, style, rot, "f32")
    xt = torch.tensor(x, dtype=torch.float64)
    cos = torch.tensor(tab[:, :rot // 2], dtype=torch.float64)[pos]
    sin = torch.tensor(tab[:, rot // 2:], dtype=torch.float64)[pos]
    if style == "neox":
        tf = pytest.importorskip("transformers.models.llama.modeling_llama")
        c2, s2 = torch.cat([cos, cos], -1), torch.cat([sin, sin], -1)
        qx = xt.transpose(1, 2)[..., :rot]
        ref, _ = tf.apply_rotary_pos_emb(qx, qx, c2, s2)
        ref = torch.cat([ref.transpose(1, 2), xt[..., rot:]], -1)
        assert torch.allclose(ref, _hf_neox(xt, cos, sin))
    else:
        fa = pytest.importorskip("flash_attn.layers.rotary")
        ref = torch.stack([fa.apply_rotary_emb_torch(xt[b:b + 1], cos[b], sin[b], interleaved=True)[0] for b in range(B)])
    bound = 3 * 2.0 ** -24 * (np.abs(x).max() * 2)
    assert np.max(np.abs(got - ref.numpy())) <= bound
    # inverse: the gradient of the f64 forward
    xg = torch.tensor(x, dtype=torch.float64, requires_grad=True)
    dy = rng.standard_normal(x.shape).astype(np.float32)
    fwd = _hf_neox(xg, cos, sin) if style == "neox" else torch.stack(
        [pytest.importorskip("flash_attn.layers.rotary").apply_rotary_emb_torch(xg[b:b + 1], cos[b], sin[b], interleaved=True)[0]
         for b in range(B)])
    (g,) = torch.autograd.grad((fwd * torch.tensor(dy, dtype=torch.float64)).sum(), xg)
    assert np.max(np.abs(ro.apply(dy, tab, pos, style, rot, "f32", inverse=True) - g.numpy())) <= 3 * 2.0 ** -24 * np.abs(dy).max() * 2


HF_TABLES = [
    ("default", {}, 128, 1.0),
    ("linear", {"factor": 4.0}, 128, 1.0),
    ("llama3", {"factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0, "original_max_position_embeddings": 8192}, 128, 1.0),
    ("yarn", {"factor": 4.0, "original_max_position_embeddings": 32768}, 128, 1.0),
    ("yarn", {"factor": 4.0, "original_max_position_embeddings": 32768, "truncate": False}, 128, 1.0),
    ("yarn", {"factor": 40.0, "original_max_position_embeddings": 4096, "beta_fast": 32, "beta_slow": 1, "mscale": 1.0,
              "mscale_all_dim": 1.0}, 64, 1.0),                            # DeepSeek-V3
    ("yarn", {"factor": 40.0, "original_max_position_embeddings": 4096, "mscale": 0.707, "mscale_all_dim": 1.0}, 64, 1.0),
    ("linear", {"factor": 1.0}, 128, 0.25),                              # partial_rotary_factor: rot = 32 of 128
]


@pytest.mark.parametrize("case", range(len(HF_TABLES)))
def test_table_rules_match_transformers(case):
    mru = pytest.importorskip("transformers.modeling_rope_utils")
    kind, keys, head_dim, prf = HF_TABLES[case]
    base = 10000.0 if kind != "llama3" else 500000.0
    params = {"rope_type": kind, "rope_theta": base, **keys}
    if prf != 1.0:
        params["partial_rotary_factor"] = prf
    cfg = SimpleNamespace(rope_parameters=params, head_dim=head_dim, hidden_size=head_dim * 8, num_attention_heads=8,
                          max_position_embeddings=163840, standardize_rope_params=lambda: None)
    if kind == "default":   # transformers 5 keeps the default rule on the rotary embedding class
        fn = pytest.importorskip("transformers.models.llama.modeling_llama").LlamaRotaryEmbedding.compute_default_rope_parameters
    else:
        fn = mru.ROPE_INIT_FUNCTIONS[kind]
    inv_hf, af_hf = fn(cfg, "cpu")
    rot = int(head_dim * prf)
    a = rope.table_args(rot, base, params)
    inv = ro.inv_freq(rot, a.base, kind, a.factor, a.low_freq_factor, a.high_freq_factor, a.original_max_position_embeddings,
                      a.beta_fast, a.beta_slow, bool(a.truncate))
    af = ro.attention_factor(kind, a.factor, a.mscale, a.mscale_all_dim, a.attention_factor)
    # HF forms inv_freq in f32: within a few f32 ulps of the f64 rule
    np.testing.assert_allclose(inv, inv_hf.double().numpy(), rtol=8 * 2.0 ** -24)
    assert abs(af - af_hf) <= 1e-6 * af_hf


def test_exact_cases_catch_each_wrong_contract():
    rng = np.random.default_rng(1)
    B, S, H, D, rot, P = 2, 32, 4, 96, 64, 40
    tab = ro.table(P, ro.inv_freq(rot), 1.0)
    x = ro.rnd(rng.standard_normal((B, S, H, D)).astype(np.float32) * 3, "bf16")
    pos = rng.integers(0, P, (B, S))
    pos[0, :3] = [-1, P, P + 7]
    x[0, :3, :, 0] = -0.0
    x[0, :3, :, 1] = np.inf
    ok = ro.apply(x, tab, pos, "neox", rot, "f32")
    for mutant in ("fma", "swapped_pairs", "rotate_pass_through", "angle_zero_out_of_range"):
        bad = ro.apply(x, tab, pos, "neox", rot, "f32", _mutant=mutant)
        assert not np.array_equal(ro.to_bits(ok, "f32"), ro.to_bits(bad, "f32")), mutant
    okinv = ro.apply(x, tab, pos, "gptj", rot, "bf16", inverse=True)
    assert not np.array_equal(okinv, ro.apply(x, tab, pos, "gptj", rot, "bf16", inverse=True, _mutant="inverse_sign"))
    # fp8 K from the f32 rotation instead of the bf16-rounded one
    k32 = ro.apply(x, tab, pos, "neox", rot, "f32")
    kr = ro.rnd(k32, "bf16")
    scale = np.ones(H, np.float32) * np.float32(0.37)
    a = np.stack([ro.fp8_bytes(kr[b, s], scale, "f8e4m3") for b in range(B) for s in range(S)])
    b_ = np.stack([ro.fp8_bytes(k32[b, s], scale, "f8e4m3") for b in range(B) for s in range(S)])
    assert not np.array_equal(a, b_)


# ---------------------------------------------------------------------------------------------- dry-run plans
def _u64(v):
    return _ffi.u64_array(v) if v is not None else None


class Planner(PlanContext):
    def _run(self, fn, *a):
        before = self.text()
        rc = fn(self.ctx, None, *a)
        return rc, self.text()[len(before):]

    def rope(self, dt=BF16, B=1, S=100, Hq=32, Hk=8, D=128, style=0, rot=None, inverse=0, ptrs=None, qo=False, ko=False,
             q_strides=None, shapes=None, P=4096, args=True):
        q, k, qop, kop, pos, cs = ptrs or (Q, K, QO if qo else 0, KO if ko else 0, POS, CS)
        qs, ks = (shapes or ([B, S, Hq, D], [B, S, Hk, D]))
        a = _ffi.RopeArgs(style, D if rot is None else rot, inverse)
        return self._run(self.lib.b200_rope, C.byref(a) if args else None, dt, C.c_uint64(q), _u64(qs), _u64(q_strides), C.c_uint64(k),
                         _u64(ks), None, C.c_uint64(qop), _u64(qs), None, C.c_uint64(kop), _u64(ks), None, C.c_uint64(pos),
                         C.c_uint64(cs), P)

    def kv(self, dt=BF16, cache=None, B=64, S=1, Hq=32, Hk=8, D=128, style=0, rot=None, page=16, pages=4096, ptrs=None, P=4096,
           kc_strides=None):
        q, kn, vn, kc, vc, sl, ks, vs = ptrs or (Q, K, V, KC, VC, SL, KS, VS)
        a = _ffi.RopeArgs(style, D if rot is None else rot, 0)
        cd = dt if cache is None else cache
        return self._run(self.lib.b200_rope_kvcache_write, C.byref(a), dt, cd, C.c_uint64(q), _u64([B, S, Hq, D]), None, C.c_uint64(0),
                         None, None, C.c_uint64(kn), _u64([B, S, Hk, D]), None, C.c_uint64(vn), _u64([B, S, Hk, D]), None,
                         C.c_uint64(kc), _u64([pages, page, Hk, D]), _u64(kc_strides), C.c_uint64(vc), _u64([pages, page, Hk, D]), None,
                         C.c_uint64(sl), C.c_uint64(POS), C.c_uint64(CS), P, C.c_uint64(ks), C.c_uint64(vs))

    def table(self, P=4096, rot=128, kind="default", out=CS, inv_freq=None, **keys):
        a = rope.table_args(rot, keys.pop("base", 10000.0), {"rope_type": kind, **keys} if kind != "inv_freq" else None,
                            inv_freq=SimpleNamespace(handle=SimpleNamespace(ptr=inv_freq)) if inv_freq is not None else None)
        return self._run(self.lib.b200_rope_cos_sin, C.byref(a), P, C.c_uint64(out))


@pytest.fixture
def plan():
    with Planner() as p:
        yield p


def _launches(text):
    return re.findall(r"launch (\w+) grid=\((\d+),1,1\) block=(\d+) smem=(\d+) cluster=1", text)


@pytest.mark.parametrize("dt", [F32, BF16, F16])
@pytest.mark.parametrize("style", [0, 1])
def test_rope_plan_names_kernel_groups_and_grid(plan, dt, style):
    tag = "gptj" if style else "neox"
    for D, rot, qo, gr, gp in ((128, 128, False, 8, 0), (128, 64, False, 4, 0), (128, 64, True, 4, 8), (96, 24, True, 2, 9),
                               (512, 512, False, 32, 0), (80, 2, True, 1, 10)):
        rc, t = plan.rope(dt=dt, D=D, rot=rot, style=style, qo=qo, S=100)
        assert rc == 0, _ffi.load().b200_last_error()
        assert f"groups={gr}+{gp} " in t and "vec=" in t
        ((name, gx, block, smem),) = _launches(t)
        assert name == f"rope_{DT[dt]}_{tag}" and block == "256" and smem == "0"
        assert int(gx) == min(-(-100 * (gr + gp) // 256), 132 * 4)
    # the same plan for any T but the grid, capped at 4 CTAs per SM
    texts = {re.sub(r"grid=\(\d+", "grid=(*", plan.rope(dt=dt, style=style, S=s)[1]) for s in (1, 77, 100000)}
    assert len(texts) == 1
    assert _launches(plan.rope(dt=dt, style=style, S=1 << 30)[1])[0][1] == str(132 * 4)


def test_vector_path_needs_aligned_views(plan):
    assert "vec=1" in plan.rope()[1]
    assert "vec=0" in plan.rope(ptrs=(Q + 2, K, 0, 0, POS, CS))[1]
    assert "vec=0" in plan.rope(q_strides=[100 * 32 * 129, 32 * 129, 129, 1])[1]
    assert "vec=0" in plan.rope(rot=100)[1]                       # rot / 2 % 8
    assert "vec=0" in plan.rope(ptrs=(Q, K, 0, 0, POS, CS + 4))[1]


@pytest.mark.parametrize("dt", [BF16, F16])
@pytest.mark.parametrize("style", [0, 1])
def test_kvcache_plan(plan, dt, style):
    tag = "gptj" if style else "neox"
    for cache, kname, ctag in ((None, "rope_kv_", DT[dt]), (_ffi.F8E4M3, "rope_kv_fp8_", "e4m3"), (_ffi.F8E5M2, "rope_kv_fp8_", "e5m2")):
        for rot, gp in ((128, 0), (64, 8)):
            rc, t = plan.kv(dt=dt, cache=cache, style=style, rot=rot)
            assert rc == 0, _ffi.load().b200_last_error()
            assert f"groups={rot // 16}+{gp}+16 cache={ctag}" in t
            ((name, gx, _, _),) = _launches(t)
            assert name == f"{kname}{DT[dt]}_{tag}" and int(gx) == -(-64 * (rot // 16 + gp + 16) // 256)
    assert _launches(plan.kv(dt=dt, B=1 << 20, S=8)[1])[0][1] == str(132 * 3)


def test_table_plan(plan):
    for kind, keys in (("default", {}), ("linear", {"factor": 2.0}), ("yarn", {"factor": 4.0, "original_max_position_embeddings": 4096})):
        rc, t = plan.table(P=131072, kind=kind, **keys)
        assert rc == 0 and _launches(t) == [("rope_cos_sin", str(132 * 4), "256", "0")]
    assert _launches(plan.table(P=10)[1])[0][1] == "3"


REFUSALS = [
    ("rope", dict(args=False), INVALID, "null args"),
    ("rope", dict(dt=_ffi.F64), UNSUPPORTED, "dtype"),
    ("rope", dict(ptrs=(0, 0, 0, 0, POS, CS)), INVALID, "both null"),
    ("rope", dict(shapes=([1, 100, 32, 128], [2, 100, 8, 128])), INVALID, "differ in B, S or D"),
    ("rope", dict(shapes=([1, 100, 32, 128], [1, 100, 8, 64])), INVALID, "differ in B, S or D"),
    ("rope", dict(rot=3), INVALID, "rot_dim"),
    ("rope", dict(rot=0), INVALID, "rot_dim"),
    ("rope", dict(rot=130), INVALID, "rot_dim"),
    ("rope", dict(style=2), INVALID, "style"),
    ("rope", dict(P=0), INVALID, "P = 0"),
    ("rope", dict(ptrs=(Q, K, 0, 0, POS, 0)), INVALID, "cos_sin"),
    ("rope", dict(ptrs=(Q, K, 0, 0, POS, CS + 2)), INVALID, "cos_sin"),
    ("rope", dict(ptrs=(Q, K, 0, 0, POS + 2, CS)), INVALID, "positions"),
    ("rope", dict(ptrs=(Q + 1, K, 0, 0, POS, CS)), INVALID, "element size"),
    ("rope", dict(q_strides=[100 * 32 * 256, 32 * 256, 256, 2]), UNSUPPORTED, "unit D stride"),
    ("rope", dict(D=520, rot=512), UNSUPPORTED, "exceeds"),
    ("rope", dict(S=1 << 31), UNSUPPORTED, "2^31"),
    ("kv", dict(dt=F32), UNSUPPORTED, "dtype"),
    ("kv", dict(cache=_ffi.U8), UNSUPPORTED, "cache dtype"),
    ("kv", dict(D=100, rot=100), UNSUPPORTED, "multiple of 8"),
    ("kv", dict(ptrs=(Q, K, V, KC, VC, 0, KS, VS)), INVALID, "null device pointer"),
    ("kv", dict(ptrs=(Q, K, V, KC, VC, SL + 2, KS, VS)), INVALID, "slot_mapping"),
    ("kv", dict(cache=_ffi.F8E4M3, ptrs=(Q, K, V, KC, VC, SL, 0, VS)), INVALID, "k_scale"),
    ("kv", dict(kc_strides=[16 * 8 * 136, 8 * 136, 136, 1]), 0, ""),
    ("kv", dict(kc_strides=[16 * 8 * 132, 8 * 132, 132, 1]), UNSUPPORTED, "cache"),
    ("kv", dict(rot=7), INVALID, "rot_dim"),
    ("table", dict(kind="linear", factor=0.5), INVALID, "factor"),
    ("table", dict(base=-1.0), INVALID, "base"),
    ("table", dict(base=float("inf")), INVALID, "base"),
    ("table", dict(rot=7), INVALID, "rot_dim"),
    ("table", dict(kind="llama3", factor=8.0, low_freq_factor=4.0, high_freq_factor=1.0, original_max_position_embeddings=8192), INVALID, "llama3"),
    ("table", dict(kind="yarn", factor=4.0), INVALID, "original_max_position_embeddings"),
    ("table", dict(kind="inv_freq", inv_freq=0), INVALID, "inv_freq"),
    ("table", dict(out=0), INVALID, "cos_sin"),
    ("table", dict(P=1 << 31), UNSUPPORTED, "2^31"),
]


@pytest.mark.parametrize("case", range(len(REFUSALS)))
def test_refusals(plan, case):
    entry, kw, status, words = REFUSALS[case]
    rc, t = getattr(plan, entry)(**kw)
    msg = _ffi.load().b200_last_error().decode()
    assert rc == status, (case, rc, msg)
    if status:
        assert words in msg and "launch" not in t, (case, msg, t)


def test_unknown_table_kind_and_zero_extents(plan):
    a = rope.table_args(128)
    a.kind = 9
    assert plan.lib.b200_rope_cos_sin(plan.ctx, None, C.byref(a), 16, C.c_uint64(CS)) == INVALID
    for kw in (dict(S=0), dict(B=0), dict(Hq=0, Hk=0)):
        rc, t = plan.rope(ptrs=(Q, K, 0, 0, 0, 0), P=0, **kw)
        assert rc == 0 and t == "", kw
    rc, t = plan.table(P=0, out=0)
    assert rc == 0 and t == ""
    assert plan.rope(S=0, rot=3)[0] == INVALID            # the argument checks still run


def test_python_layer_defers_errors():
    class _Stub:
        def __init__(self):
            self.errors = []

        def _defer(self, e):
            self.errors.append(e)

    class _T:
        def __init__(self, shape, dtype="bf16"):
            self.shape, self.dtype = list(shape), dtype
            self.strides = [int(np.prod(shape[i + 1:])) for i in range(len(shape))]

        def is_contiguous(self):
            return True

        def size(self):
            return int(np.prod(self.shape))

    s = _Stub()
    cs, q = _T([64, 128], "f32"), _T([1, 8, 4, 128])
    rope.apply(s, cs)                                                   # q and k None
    rope.apply(s, _T([64, 128], "bf16"), q)                             # table not f32
    rope.apply(s, cs, _T([8, 4, 128]))                                  # q not 4-D
    rope.apply(s, cs, q, positions=_T([1, 7], "i32"))                   # positions not [B, S]
    rope.apply(s, cs, q, style="rotate")                                # unknown style
    rope.apply(s, cs, q, k=_T([1, 8, 2, 128], "f16"))                   # dtypes differ
    rope.kvcache_write(s, cs, q, _T([1, 8, 2, 128]), _T([1, 8, 2, 128]), _T([4, 16, 2, 128], "f8e4m3"),
                       _T([4, 16, 2, 128], "f8e4m3"), _T([8], "i32"), None)   # fp8 without scales
    rope.cos_sin(s, _T([64, 128], "bf16"))                              # table not f32
    assert [e.status for e in s.errors] == [INVALID] * 8
    with pytest.raises(_ffi.B200Error):
        rope.table_args(128, scaling={"rope_type": "longrope"})


# ---------------------------------------------------------------------------------------------- kernels
KERNELS = ({f"rope_{d}_{s}" for d in ("f32", "bf16", "f16") for s in ("neox", "gptj")}
           | {f"rope_kv_{f}{d}_{s}" for f in ("", "fp8_") for d in ("bf16", "f16") for s in ("neox", "gptj")} | {"rope_cos_sin"})


def test_rope_kernels_do_not_spill_and_use_no_atomics():
    tool = _tool("cuobjdump")
    _ffi.load()
    cubin = ROOT / "cubecl_b200" / "build" / "rope.cubin"
    out = subprocess.run([tool, "-res-usage", str(cubin)], capture_output=True, text=True, check=True).stdout
    funcs = re.findall(r"Function (\w+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", out)
    assert {f for f, *_ in funcs} == KERNELS and len(KERNELS) == 15
    for name, reg, stack, shared, local in funcs:
        assert int(stack) == 0 and int(local) == 0 and int(shared) == 0, (name, stack, local, shared)
        # every CTA of the capped grid resident at once: 4 (rope, table) or 3 (cache writes) 256-thread CTAs per SM
        assert int(reg) <= (85 if name.startswith("rope_kv_") else 64), (name, reg)
    sass = subprocess.run([tool, "-sass", str(cubin)], capture_output=True, text=True, check=True).stdout
    bodies = {b.split()[0]: b for b in re.split(r"\n\s*Function : ", sass)[1:]}
    assert set(bodies) == KERNELS
    for name, body in bodies.items():
        assert not re.search(r"\b(ATOM|ATOMS|ATOMG|RED|REDG)\b", body), name
        assert not re.search(r"\b(LDL|STL)\b", body), name
    for name in ("rope_bf16_neox", "rope_f16_gptj", "rope_f32_neox", "rope_kv_bf16_neox"):
        assert "LDG.E.128" in bodies[name] and "STG.E.128" in bodies[name], name
    assert "STG.E.64" in bodies["rope_kv_fp8_bf16_neox"]
    for name in ("rope_bf16_neox", "rope_f32_gptj"):       # separately rounded products: no fused multiply-add
        assert not re.search(r"\bFFMA\b", bodies[name]), name
