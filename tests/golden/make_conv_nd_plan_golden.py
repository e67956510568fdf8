"""Record the dry-run plans of the 3-D and transposed convolution entry points, and the full error messages of the 2-D ones,
into conv_nd_plan_golden.json.gz (read by tests/test_conv_nd_plan_golden_cpu.py).

    python tests/golden/make_conv_nd_plan_golden.py

Each case is one call in a fresh planning context (b200_plan_begin, 132 SMs); the fixture stores the call, the returned
status, the full error message and the full plan text.  The cases cover b200_conv3d and both of its gradients, and
b200_conv_transpose2d / 3d: a geometry grid (kernels of one and of several taps per dimension, mixed strides 1..3, paddings,
dilations, 3 / 16 / 64 / 130 channels, both output dtype rules), strided and misaligned views, output channel slices, a
pitched dx and a padded dw, the gemm.variant / split_k / epilogue options, stride phases no tap reaches, no input channels,
empty kernels, one case per refusal and the cases where two checks fail at once.  Every failing call of conv_plan_golden.json.gz
(the 2-D plain and grouped entry points) is replayed as well, for its full message.  Plans hold no pointer bases, so phase and
weight-block offsets are left to the GPU tests.
"""
from __future__ import annotations

import ctypes as C
import gzip
import json
import sys
from pathlib import Path

TESTS = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(TESTS.parent), str(TESTS)]

from cubecl_b200 import _ffi  # noqa: E402
from plan_context import PlanContext  # noqa: E402

GOLDEN = Path(__file__).resolve().parent / "conv_nd_plan_golden.json.gz"
GOLDEN_2D = Path(__file__).resolve().parent / "conv_plan_golden.json.gz"
DTYPES = {"f32": _ffi.F32, "f16": _ffi.F16, "bf16": _ffi.BF16, "i8": _ffi.I8}
WITH_EP = {"b200_conv2d", "b200_conv2d_grouped", "b200_conv3d", "b200_conv_transpose2d", "b200_conv_transpose3d"}

X, W, O = 0x10000000, 0x20000000, 0x30000000
BIG = 1 << 31
DT = (("bf16", "bf16"), ("f16", "f32"))


def replay(call: dict) -> dict:
    """One recorded call in a fresh dry-run context (132 SMs): {status, error (the full message, "" on success), plan}."""
    with PlanContext(132, call["options"]) as p:
        fn = call["fn"]
        arr = lambda v: _ffi.u64_array(v) if v is not None else None  # noqa: E731
        args = None
        if call["args"] is not None:
            args = C.byref((_ffi.Conv3dArgs if "3d" in fn else _ffi.Conv2dArgs)(*call["args"]))
        extra = (C.c_uint32(call["groups"]),) if call["groups"] is not None else ()
        if fn in WITH_EP:
            extra += (C.byref(_ffi.Epilogue(*call["ep"])) if call["ep"] is not None else None,)
        rc = getattr(p.lib, fn)(p.ctx, None, DTYPES[call["idt"]], DTYPES[call["odt"]], call["a"], arr(call["a_shape"]),
                                arr(call["a_strides"]), call["b"], arr(call["b_shape"]), arr(call["b_strides"]), call["o"],
                                arr(call["o_shape"]), arr(call["o_strides"]), args, *extra)
        err = ""
        if rc:
            msg = p.lib.b200_last_error()
            err = msg.decode() if msg else ""
        return {"status": rc, "error": err, "plan": p.text()}


def _vec(v, n):
    return list(v) if isinstance(v, (list, tuple)) else [v] * n


def conv_out(xs, ws, s, p, d):
    """The convolution's output extents (spatial only); a negative extent stays negative."""
    n = len(xs) - 2
    s, p, d = _vec(s, n), _vec(p, n), _vec(d, n)
    return [(xs[1 + i] + 2 * p[i] - d[i] * (ws[1 + i] - 1) - 1) // max(1, s[i]) + 1 for i in range(n)]


def tconv_out(xs, ws, s, p, op, d):
    n = len(xs) - 2
    s, p, op, d = _vec(s, n), _vec(p, n), _vec(op, n), _vec(d, n)
    return [(xs[1 + i] - 1) * s[i] - 2 * p[i] + d[i] * (ws[1 + i] - 1) + op[i] + 1 for i in range(n)]


ENTRY = {"fwd3": "b200_conv3d", "dgrad3": "b200_conv3d_backward_data", "wgrad3": "b200_conv3d_backward_weight",
         "tconv2": "b200_conv_transpose2d", "tconv3": "b200_conv_transpose3d"}


def call(fn, xs, ws, stride=1, pad=0, dil=1, dt=DT[0], ys=None, op=0, a_strides=None, b_strides=None, o_strides=None, a=X, b=W, o=O,
         ep=None, options=None, shapes=None, args="auto"):
    """The recorded arguments of one call.  Convolutions: xs / ws are the forward's input and weights, ys (dy, or the forward's
    out) defaults to the output rule, and the operands are (x, w, out), (dy, w, dx) or (x, dy, dw).  Transposed: xs is x
    [N, *X, Cin], ws is w [Cin, *K, C], ys is out (defaults to the transposed output rule with output padding op)."""
    n = len(ws) - 2
    if ys is None:
        if fn.startswith("tconv"):
            ys = [xs[0], *(max(0, e) for e in tconv_out(xs, ws, stride, pad, op, dil)), ws[-1]]
        else:
            ys = [xs[0], *(max(0, e) for e in conv_out(xs, ws, stride, pad, dil)), ws[0]]
    ops = shapes or {"fwd3": (xs, ws, ys), "dgrad3": (ys, ws, xs), "wgrad3": (xs, ys, ws), "tconv2": (xs, ws, ys), "tconv3": (xs, ws, ys)}[fn]
    if args == "auto":
        args = _vec(stride, n) + _vec(pad, n) + _vec(dil, n)
    return {"fn": ENTRY[fn], "groups": None, "a_shape": ops[0], "b_shape": ops[1], "o_shape": ops[2], "a_strides": a_strides,
            "b_strides": b_strides, "o_strides": o_strides, "idt": dt[0], "odt": dt[1], "args": args, "a": a, "b": b, "o": o,
            "ep": ep, "options": options or {}}


def from_2d(c: dict) -> dict:
    """A call of conv_plan_golden.json.gz in this fixture's form."""
    fn = {"fwd": "b200_conv2d", "dgrad": "b200_conv2d_backward_data", "wgrad": "b200_conv2d_backward_weight"}[c["fn"]]
    if c["groups"] is not None:
        fn = fn.replace("b200_conv2d", "b200_conv2d_grouped")
    (sh, sw), (ph, pw), (dh, dw) = c["stride"], c["pad"], c["dil"]
    return {"fn": fn, "groups": c["groups"], "a_shape": c["a_shape"], "b_shape": c["b_shape"], "o_shape": c["o_shape"],
            "a_strides": c["a_strides"], "b_strides": c["b_strides"], "o_strides": c["o_strides"], "idt": c["idt"], "odt": c["odt"],
            "args": [sh, sw, ph, pw, dh, dw], "a": c["a"], "b": c["b"], "o": c["o"], "ep": c["ep"], "options": c["options"]}


def compact(s):
    """Compact strides of an NHWC / NDHWC shape."""
    out, inner = [], 1
    for e in reversed(s):
        out.append(inner)
        inner *= e
    return out[::-1]


def channels_first(s):
    """Strides of an N*C-indexed view of a compact channels-first tensor (NCHW / NCDHW x and dy, OIHW / OIDHW weights)."""
    n, *sp, c = s
    inner = 1
    for e in sp:
        inner *= e
    st, acc = [], 1
    for e in reversed(sp):
        st.append(acc)
        acc *= e
    return [c * inner, *st[::-1], inner]


def pitched(s, extra):
    """Strides of an NHWC / NDHWC view whose pixels are `extra` elements wider than its channels."""
    st = compact([*s[:-1], s[-1] + extra])
    return st


def cases():
    out = []

    def add(name, fn, *args, **kw):
        out.append((f"{fn}-{name}", call(fn, *args, **kw)))

    # ---- geometry grid
    kernels3 = ((1, 1, 1), (3, 3, 3), (2, 3, 1), (1, 2, 4))
    strides3 = (1, 2, (1, 2, 3), (3, 1, 2))
    pads3 = (0, 1, (1, 0, 2))
    dils3 = (1, (2, 1, 1), (1, 1, 2))
    i = 0
    for c in (3, 16, 64, 130):
        cout = 24 if c < 64 else 80
        for k in kernels3:
            for s in strides3:
                pad, dil, dt = pads3[i % 3], dils3[(i // 3) % 3], DT[(i + i // 4) % 2]
                for fn in ("fwd3", "dgrad3", "wgrad3"):
                    add(f"c{c}-k{k}-s{s}-p{pad}-d{dil}-{dt[0]}{dt[1]}", fn, [2, 5, 9, 7, c], [cout, *k, c], s, pad, dil, dt)
                i += 1
    kernels2 = ((1, 1), (3, 3), (2, 4), (5, 1))
    strides2 = (1, 2, (1, 3), (3, 2))
    pads2 = (0, 1, (2, 0))
    dils2 = (1, (2, 1), (1, 3))
    i = 0
    for cin in (3, 16, 64, 130):
        cout = 24 if cin < 64 else 72
        for k in kernels2:
            for s in strides2:
                pad, dil, dt = pads2[i % 3], dils2[(i // 3) % 3], DT[(i + i // 4) % 2]
                op = [(sv - 1) if (i % 2) else 0 for sv in _vec(s, 2)]
                add(f"c{cin}-k{k}-s{s}-p{pad}-op{op}-d{dil}-{dt[0]}{dt[1]}", "tconv2", [2, 9, 7, cin], [cin, *k, cout], s, pad, dil, dt, op=op)
                i += 1
    i = 0
    for cin in (3, 16, 64, 130):
        cout = 24 if cin < 64 else 72
        for k in kernels3:
            for s in strides3:
                pad, dil, dt = pads3[i % 3], dils3[(i // 3) % 3], DT[(i + i // 4) % 2]
                op = [(sv - 1) if (i % 2) else 0 for sv in _vec(s, 3)]
                add(f"c{cin}-k{k}-s{s}-p{pad}-op{op}-d{dil}-{dt[0]}{dt[1]}", "tconv3", [1, 4, 6, 5, cin], [cin, *k, cout], s, pad, dil, dt, op=op)
                i += 1
    # fused epilogues: (alpha, activation, bias)
    for name, ep in (("ep-relu-bias", [1.0, 1, 0x40000000]), ("ep-gelu-alpha", [0.25, 2, 0]), ("ep-identity", [1.0, 0, 0])):
        add(name, "fwd3", [2, 5, 9, 7, 64], [80, 3, 3, 3, 64], 1, 1, ep=ep)
        add(name + "-c3", "fwd3", [2, 5, 9, 7, 3], [24, 3, 1, 3, 3], 2, 1, dt=DT[1], ep=ep)
        for s in (1, 2, 3):
            add(f"{name}-s{s}", "tconv2", [2, 9, 7, 64], [64, 3, 3, 32], s, 1, ep=ep)
            add(f"{name}-s{s}", "tconv3", [1, 4, 6, 5, 16], [16, 3, 3, 3, 24], s, 1, dt=DT[1], ep=ep)

    # ---- views
    for c in (3, 16, 64):
        xs, ws = [2, 4, 6, 5, c], [24, 3, 3, 3, c]
        ys = [2, 4, 6, 5, 24]
        add(f"ncdhw-x-c{c}", "fwd3", xs, ws, 1, 1, a_strides=channels_first(xs))
        add(f"oidhw-w-c{c}", "fwd3", xs, ws, 1, 1, b_strides=channels_first(ws))
        add(f"misaligned-x-c{c}", "fwd3", xs, ws, 1, 1, a=X + 2)
        add(f"misaligned-w-c{c}", "fwd3", xs, ws, 1, 1, b=W + 2)
        add(f"x-pitch-c{c}", "fwd3", xs, ws, 1, 1, a_strides=pitched(xs, 8))
        add(f"out-slice-c{c}", "fwd3", xs, ws, 1, 1, o=O + 48, o_strides=pitched(ys, 24))
        add(f"ncdhw-x-c{c}", "wgrad3", xs, ws, 1, 1, a_strides=channels_first(xs))
        add(f"misaligned-x-c{c}", "wgrad3", xs, ws, 1, 1, a=X + 2)
        add(f"oidhw-w-c{c}", "dgrad3", xs, ws, 1, 1, b_strides=channels_first(ws))
        add(f"pitched-dx-c{c}", "dgrad3", xs, ws, 1, 1, o_strides=pitched(xs, 8))
        add(f"dx-slice-c{c}", "dgrad3", xs, ws, 2, 1, o=O + 2 * c, o_strides=pitched(xs, c))
        add(f"dw-cout-stride-c{c}", "wgrad3", xs, ws, 1, 1, o_strides=[27 * c + 64, 9 * c, 3 * c, c, 1])
        add(f"dw-cout-stride-s2-c{c}", "wgrad3", xs, ws, 2, 1, dt=DT[1], o_strides=[27 * c + 8, 9 * c, 3 * c, c, 1])
        for fn, xt, wt in (("tconv2", [2, 6, 5, c], [c, 3, 3, 24]), ("tconv3", [1, 4, 6, 5, c], [c, 3, 3, 3, 24])):
            for s in (1, 2):
                outs = [xt[0], *tconv_out(xt, wt, s, 1, 0, 1), 24]
                add(f"nc-x-c{c}-s{s}", fn, xt, wt, s, 1, a_strides=channels_first(xt))
                add(f"io-w-c{c}-s{s}", fn, xt, wt, s, 1, b_strides=channels_first(wt))
                add(f"misaligned-x-c{c}-s{s}", fn, xt, wt, s, 1, a=X + 2)
                add(f"misaligned-w-c{c}-s{s}", fn, xt, wt, s, 1, b=W + 2)
                add(f"x-pitch-c{c}-s{s}", fn, xt, wt, s, 1, a_strides=pitched(xt, 8))
                add(f"out-slice-c{c}-s{s}", fn, xt, wt, s, 1, o=O + 48, o_strides=pitched(outs, 24))
                add(f"out-pitch-f32-c{c}-s{s}", fn, xt, wt, s, 1, dt=DT[1], o_strides=pitched(outs, 4))
                add(f"out-misaligned-c{c}-s{s}", fn, xt, wt, s, 1, o=O + 2)
    for fn in ("dgrad3", "wgrad3"):
        xs, ws = [2, 4, 6, 5, 16], [24, 3, 3, 3, 16]
        for s in (1, 2):
            ys = [2, *conv_out(xs, ws, s, 1, 1), 24]
            key = "a_strides" if fn == "dgrad3" else "b_strides"
            add(f"ncdhw-dy-s{s}", fn, xs, ws, s, 1, ys=ys, **{key: channels_first(ys)})
            add(f"misaligned-dy-s{s}", fn, xs, ws, s, 1, ys=ys, **({"a": X + 2} if fn == "dgrad3" else {"b": W + 2}))
            add(f"dy-pitch-s{s}", fn, xs, ws, s, 1, ys=ys, **{key: pitched(ys, 16)})

    # ---- options
    for opts in ({"gemm.variant": "1sm_n128"}, {"gemm.variant": "2sm_n128"}, {"gemm.split_k": "on"}, {"gemm.split_k": "3"},
                 {"gemm.epilogue": "direct"}, {"gemm.variant": "1sm_n128", "gemm.split_k": "on", "gemm.epilogue": "direct"},
                 {"gemm.variant": "2sm_n256"}, {"gemm.split_k": "9"}, {"gemm.epilogue": "bogus"}):
        tag = "-".join(f"{k.split('.')[1]}={v}" for k, v in opts.items())
        for fn in ("fwd3", "dgrad3", "wgrad3"):
            add(f"opt-{tag}", fn, [2, 8, 14, 14, 64], [128, 3, 3, 3, 64], 1, 1, options=opts)
            add(f"opt-{tag}-s2-c3", fn, [2, 8, 14, 14, 3], [64, 3, 3, 3, 3], 2, 1, dt=DT[1], options=opts)
        for s in (1, 2, 3):
            add(f"opt-{tag}-s{s}", "tconv2", [2, 14, 14, 64], [64, 3, 3, 128], s, 1, options=opts)
            add(f"opt-{tag}-s{s}", "tconv3", [1, 4, 8, 8, 64], [64, 3, 3, 3, 128], s, 1, options=opts)

    # ---- stride phases that no tap reaches, no input channels, empty kernels, empty extents
    for s in (2, (1, 2, 3), 3):
        add(f"notap-k1-s{s}", "dgrad3", [1, 6, 7, 8, 16], [24, 1, 1, 1, 16], s)
        add(f"notap-k2-d2-s{s}", "dgrad3", [1, 6, 7, 8, 16], [24, 2, 1, 2, 16], s, 0, 2)
        add(f"notap-k1-s{s}", "tconv3", [1, 3, 3, 3, 16], [16, 1, 1, 1, 24], s)
        add(f"notap-k2-d2-s{s}", "tconv3", [1, 3, 3, 3, 16], [16, 2, 1, 2, 24], s, 0, 2)
        s2 = s[1:] if isinstance(s, tuple) else s
        add(f"notap-k1-s{s2}", "tconv2", [1, 5, 4, 16], [16, 1, 1, 24], s2)
        add(f"notap-k2-d2-s{s2}", "tconv2", [1, 5, 4, 16], [16, 2, 2, 24], s2, 0, 2)
    for s in (1, 2, 3):
        add(f"cin0-s{s}", "tconv2", [1, 5, 4, 0], [0, 3, 3, 24], s, 1, ep=[1.0, 1, 0x40000000])
        add(f"cin0-s{s}", "tconv3", [1, 3, 4, 5, 0], [0, 3, 3, 3, 24], s, 1)
        add(f"cout0-s{s}", "dgrad3", [1, 4, 5, 6, 16], [0, 3, 3, 3, 16], s, 1)
        for j in range(2):
            k2 = [3, 3]
            k2[j] = 0
            add(f"empty-kernel{j}-s{s}", "tconv2", [1, 5, 4, 16], [16, *k2, 24], s, 0, ep=[0.5, 2, 0x40000000])
            add(f"empty-kernel{j}-s{s}-bad-out", "tconv2", [1, 5, 4, 16], [16, *k2, 24], s, 1, ys=[1, 30, 30, 24])
        for j in range(3):
            k3 = [3, 3, 3]
            k3[j] = 0
            add(f"empty-kernel{j}-s{s}", "tconv3", [1, 3, 4, 5, 16], [16, *k3, 24], s, 0)
            add(f"empty-kernel{j}-s{s}-bad-out", "tconv3", [1, 3, 4, 5, 16], [16, *k3, 24], s, 1, ys=[1, 9, 9, 9, 24])
            add(f"empty-kernel{j}-s{s}", "fwd3", [1, 4, 5, 6, 16], [24, *k3, 16], s, 1, ys=[1, 2, 2, 2, 24])
            add(f"empty-kernel{j}-s{s}", "dgrad3", [1, 4, 5, 6, 16], [24, *k3, 16], s, 1, ys=[1, 2, 2, 2, 24])
            add(f"empty-kernel{j}-s{s}", "wgrad3", [1, 4, 5, 6, 16], [24, *k3, 16], s, 1, ys=[1, 2, 2, 2, 24])
    add("empty-kernel-s9", "tconv2", [1, 5, 4, 16], [16, 0, 3, 24], 9, 0, ys=[1, 37, 28, 24])
    add("empty-kernel-s9", "tconv3", [1, 3, 4, 5, 16], [16, 3, 0, 3, 24], 9, 0, ys=[1, 21, 28, 35, 24])
    for fn in ("fwd3", "dgrad3", "wgrad3"):
        for name, xs, ws in (("n0", [0, 4, 5, 6, 16], [24, 3, 3, 3, 16]), ("d0", [1, 0, 5, 6, 16], [24, 3, 3, 3, 16]),
                             ("w0", [1, 4, 5, 0, 16], [24, 3, 3, 3, 16]), ("c0", [1, 4, 5, 6, 0], [24, 3, 3, 3, 0]),
                             ("cout0", [1, 4, 5, 6, 16], [0, 3, 3, 3, 16])):
            add(f"empty-{name}", fn, xs, ws, 2, 1)
        add("empty-n0-wrong-out", fn, [0, 4, 5, 6, 16], [24, 3, 3, 3, 16], ys=[0, 1, 1, 1, 24])
        add("empty-n0-dw-cout-stride", fn, [0, 4, 5, 6, 16], [24, 3, 3, 3, 16], 1, 1, o_strides=[27 * 16 + 8, 9 * 16, 3 * 16, 16, 1])
        add("no-pixels-dw-cout-stride", fn, [0, 4, 5, 6, 16], [24, 3, 3, 3, 16], 1, 1, ys=[0, 4, 5, 6, 24],
            o_strides=[27 * 16 + 8, 9 * 16, 3 * 16, 16, 1] if fn == "wgrad3" else None)
    for fn, xs, ws in (("tconv2", [1, 5, 4, 16], [16, 3, 3, 24]), ("tconv3", [1, 3, 4, 5, 16], [16, 3, 3, 3, 24])):
        n = len(ws) - 2
        for j, name in enumerate(("n0", "x0", "cout0")):
            xe, we = list(xs), list(ws)
            if j == 0:
                xe[0] = 0
            elif j == 1:
                xe[1] = 0
            else:
                we[-1] = 0
            add(f"empty-{name}", fn, xe, we, 2, 1)

    # ---- one case per refusal
    def refusals(fn, xs, ws, stride, pad, dil):
        def bad(name, **kw):
            base = dict(xs=xs, ws=ws, stride=stride, pad=pad, dil=dil)
            base.update(kw)
            add(f"err-{name}", fn, base.pop("xs"), base.pop("ws"), **base)
        n = len(ws) - 2
        base_call = call(fn, xs, ws, stride, pad, dil)
        for j in range(3):
            sh = [base_call[k] for k in ("a_shape", "b_shape", "o_shape")]
            sh[j] = None
            bad(f"null-shape{j}", shapes=sh)
        bad("null-args", args=None)
        bad("f32-input", dt=("f32", "f32"))
        bad("i8-input", dt=("i8", "f32"))
        bad("bf16-to-f16", dt=("bf16", "f16"))
        bad("f16-to-bf16", dt=("f16", "bf16"))
        for j in range(n):
            z = [1] * n
            z[j] = 0
            bad(f"stride0-{j}", stride=z)
            bad(f"dil0-{j}", dil=z)
            m = [1] * n
            m[j] = -1
            bad(f"pad-neg-{j}", pad=m)
            nine = [1] * n
            nine[j] = 9
            bad(f"stride9-{j}", xs=[1, *([20] * n), xs[-1]], stride=nine)
        bad("null-a", a=0)
        bad("null-b", b=0)
        bad("null-out", o=0)
        bad("misaligned-out", o=O + 1)
        bad("misaligned-out-f32", o=O + 2, dt=DT[1])
        bad("extent-2^31", xs=[1, BIG, *xs[2:]])
        bad("channels-2^31", xs=[*xs[:-1], BIG], ws=[*ws[:-1], BIG] if not fn.startswith("tconv") else [BIG, *ws[1:]])
        return bad

    for fn in ("fwd3", "dgrad3", "wgrad3"):
        bad = refusals(fn, [1, 6, 8, 8, 16], [32, 3, 3, 3, 16], 1, 1, 1)
        bad("weight-channels", ws=[32, 3, 3, 3, 17])
        bad("kernel-too-large", ws=[32, 9, 3, 3, 16], ys=[1, 1, 8, 8, 32])
        bad("kernel-too-large-w", ws=[32, 3, 3, 11, 16], ys=[1, 6, 8, 1, 32])
        for j in range(3):
            p = [0, 0, 0]
            p[j] = 16
            bad(f"pad16-{j}", xs=[1, 40, 40, 40, 16], pad=p)
            p[j] = 17
            bad(f"corner-pad-{j}", xs=[1, 40, 40, 40, 16], pad=p)
            k = [1, 1, 1]
            k[j] = 17
            bad(f"upper-corner-k17-{j}", xs=[1, 40, 40, 40, 16], ws=[16, *k, 16])
            k[j] = 18
            bad(f"upper-corner-k18-{j}", xs=[1, 40, 40, 40, 16], ws=[16, *k, 16])
            d = [1, 1, 1]
            d[j] = 16
            p = [0, 0, 0]
            p[j] = 16
            k = [1, 1, 1]
            k[j] = 3
            bad(f"offset-{j}", xs=[1, 40, 40, 40, 16], ws=[16, *k, 16], pad=p, dil=d)
        bad("pixels-2^31", xs=[1 << 13, 64, 64, 64, 16], ws=[32, 1, 1, 1, 16], pad=0)
        bad("kpos-2^31", xs=[1, 8, 8, 8, 1 << 26], ws=[32, 3, 3, 3, 1 << 26])
        if fn == "fwd3":
            bad("bad-out-shape", ys=[1, 5, 8, 8, 32])
            bad("bad-out-cout", ys=[1, 6, 8, 8, 31])
            bad("bad-out-n", ys=[2, 6, 8, 8, 32])
            bad("activation", ep=[1.0, 3, 0])
            bad("activation-neg", ep=[1.0, -1, 0])
            bad("out-channel-stride", o_strides=[6 * 8 * 8 * 64, 8 * 8 * 64, 8 * 64, 64, 2])
            bad("out-pitch-small", o_strides=[6 * 8 * 8 * 16, 8 * 8 * 16, 8 * 16, 16, 1])
            bad("out-rows-gap", o_strides=[6 * 8 * 8 * 40 + 8, 8 * 8 * 40 + 8, 8 * 40, 40, 1])
        else:
            bad("bad-dy-shape", ys=[1, 5, 8, 8, 32])
            bad("bad-dy-n", ys=[2, 6, 8, 8, 32])
            bad("bad-dy-cout", ys=[1, 6, 8, 8, 31])
            bad("dy-extent-2^31", ys=[1, 6, 8, 8, BIG])
        if fn == "dgrad3":
            bad("dx-channel-stride", o_strides=[6 * 8 * 8 * 32, 8 * 8 * 32, 8 * 32, 32, 2])
            bad("dx-pitch-small", o_strides=[6 * 8 * 8 * 8, 8 * 8 * 8, 8 * 8, 8, 1])
            bad("dx-plane-gap", o_strides=[6 * 8 * 8 * 16 + 8, 8 * 8 * 16 + 8, 8 * 16, 16, 1])
            bad("kpos-cout-2^31", ws=[1 << 26, 3, 3, 3, 16], ys=[1, 6, 8, 8, 1 << 26])
            bad("phase-corner", xs=[1, 8, 8, 40, 16], ws=[16, 1, 1, 18, 16], pad=0)
            bad("phase-corner-ok", xs=[1, 8, 8, 40, 16], ws=[16, 1, 1, 17, 16], pad=0)
            bad("phase-offset", xs=[1, 8, 40, 8, 16], ws=[16, 1, 5, 1, 16], stride=(1, 2, 1), pad=(0, 16, 0), dil=(1, 16, 1))
            bad("dx-pixels-2^31", xs=[1 << 13, 64, 64, 64, 16], ws=[32, 1, 1, 1, 16], pad=0)
        if fn == "wgrad3":
            bad("dw-channel-stride", o_strides=[27 * 32, 9 * 32, 3 * 32, 32, 2])
            bad("dw-kpos-not-flat", o_strides=[27 * 80, 9 * 80, 3 * 80, 24, 1])
            bad("dw-kpos-not-flat-d", o_strides=[27 * 80, 9 * 40, 3 * 16, 16, 1])
            bad("dw-stride-2^40", o_strides=[1 << 40, 9 * 16, 3 * 16, 16, 1])
            bad("dw-kpos-2^40", o_strides=[1 << 41, 1 << 40, 3 * 16, 16, 1], ws=[32, 2, 3, 3, 16])

    for fn, xs, ws in (("tconv2", [1, 8, 8, 16], [16, 3, 3, 32]), ("tconv3", [1, 4, 6, 6, 16], [16, 3, 3, 3, 32])):
        n = len(ws) - 2
        bad = refusals(fn, xs, ws, 2, 1, 1)
        outs = [xs[0], *tconv_out(xs, ws, 2, 1, 1, 1), ws[-1]]
        bad("weight-channels", xs=[*xs[:-1], 17])
        bad("activation", ep=[1.0, 7, 0])
        bad("out-channel-stride", o_strides=[*compact([*outs[:-1], 64])[:-1], 2])
        bad("out-pitch-small", o_strides=compact([*outs[:-1], 16]))
        bad("channel-mismatch", ys=[*outs[:-1], 16])
        bad("bad-out-n", ys=[2, *outs[1:]])
        bad("pixels-2^31", xs=[1 << (31 - 7 * n), *([128] * n), 16], ws=[16, *([1] * n), 32], stride=1, pad=0)
        bad("kpos-2^31", xs=[*xs[:-1], 1 << 26], ws=[1 << 26, *ws[1:]])
        for j in range(n):
            op = [0] * n
            op[j] = 2
            bad(f"output-padding-ge-stride-{j}", dil=3, ys=[xs[0], *tconv_out(xs, ws, 2, 1, op, 3), ws[-1]])
            op[j] = 5
            bad(f"output-padding-too-large-{j}", ys=[xs[0], *tconv_out(xs, ws, 2, 1, op, 1), ws[-1]])
            k = [1] * n
            k[j] = 150 if n == 2 else 33
            xe = [1] * n
            xe[j] = k[j] + 1
            bad(f"corner-{j}", xs=[1, *[e + 3 for e in xe], 16], ws=[16, *k, 32], stride=1, pad=0)
            d = [1] * n
            d[j] = 16
            p = [0] * n
            p[j] = 16
            k = [1] * n
            k[j] = 3
            bad(f"dil16-{j}", xs=[1, *([8] * n), 16], ws=[16, *k, 32], stride=1, pad=p, dil=d)
            s = [1] * n
            s[j] = 9
            bad(f"stride9-k1-{j}", ws=[16, *([1] * n), 32], stride=s, pad=0)

    # ---- two checks failing at once: the first check in each entry point's order names the fault
    for fn in ("fwd3", "dgrad3", "wgrad3"):
        xs, ws = [1, 6, 8, 8, 16], [32, 3, 3, 3, 16]
        add("err2-f32-stride-d0", fn, xs, ws, (0, 1, 1), 1, dt=("f32", "f32"), ys=[1, 6, 8, 8, 32])
        add("err2-f32-stride-h0", fn, xs, ws, (1, 0, 1), 1, dt=("f32", "f32"), ys=[1, 6, 8, 8, 32])
        add("err2-f32-dil-d0", fn, xs, ws, 1, 1, (0, 1, 1), dt=("f32", "f32"), ys=[1, 6, 8, 8, 32])
        add("err2-f16-to-bf16-pad-d-neg", fn, xs, ws, 1, (-1, 1, 1), dt=("f16", "bf16"), ys=[1, 6, 8, 8, 32])
        add("err2-bf16-to-f16-dil-w0", fn, xs, ws, 1, 1, (1, 1, 0), dt=("bf16", "f16"), ys=[1, 6, 8, 8, 32])
        # corners: (lo, up) per dimension in (D, H, W) order, then the offsets
        add("err2-lo-h-up-d", fn, [1, 40, 40, 40, 16], [16, 20, 1, 1, 16], 1, (0, 17, 0))
        add("err2-up-d-lo-w", fn, [1, 40, 40, 40, 16], [16, 19, 1, 1, 16], 1, (0, 0, 20))
        add("err2-lo-w-up-w", fn, [1, 40, 40, 40, 16], [16, 1, 1, 40, 16], 1, (0, 0, 17))
        add("err2-offset-h-corner-w", fn, [1, 40, 40, 40, 16], [16, 1, 3, 1, 16], 1, (0, 16, 17), (1, 16, 1))
        add("err2-offset-d-offset-w", fn, [1, 40, 40, 40, 16], [16, 3, 1, 3, 16], 1, (15, 0, 15), (16, 1, 16))
    for fn, xs, ws, args in (("tconv2", [1, 8, 8, 16], [16, 3, 3, 32], ((0, 1), 1, 1)), ("tconv3", [1, 4, 6, 6, 16], [16, 3, 3, 3, 32], ((0, 1, 1), 1, 1))):
        n = len(ws) - 2
        outs = [xs[0], *tconv_out(xs, ws, 1, 1, 0, 1), ws[-1]]
        add("err2-f32-stride0", fn, xs, ws, *args, dt=("f32", "f32"), ys=outs)
        add("err2-f32-dil0", fn, xs, ws, 1, 1, [1] * (n - 1) + [0], dt=("f32", "f32"), ys=outs)
        add("err2-f16-to-bf16-pad-neg", fn, xs, ws, 1, [-1] + [1] * (n - 1), dt=("f16", "bf16"), ys=outs)
        add("err2-output-padding-shape", fn, xs, ws, 2, 1, 3, ys=[xs[0], *tconv_out(xs, ws, 2, 1, 2, 3)[:-1], 99, ws[-1]])
        add("err2-stride9-shape", fn, xs, ws, 9, 1, ys=[*outs[:-1], 7])
        add("err2-stride9-corner", fn, [1, *([200] * n), 16], [16, 150, *([1] * (n - 1)), 32], 9, 0)
    # 3-D transposed: corners per dimension as in the data gradient (lo, up), then offsets
    add("err2-lo-h-up-d", "tconv3", [1, 40, 40, 40, 16], [16, 20, 1, 1, 32], 1, (0, 17, 0))
    add("err2-up-d-lo-w", "tconv3", [1, 40, 40, 40, 16], [16, 19, 1, 1, 32], 1, (0, 0, 20))
    # 2-D: corners in the order (lo_h, lo_w, up_h, up_w); a data-gradient phase's corners in the same order
    for fn2 in ("fwd", "dgrad", "wgrad"):
        for g in (None, 4):
            gt = "plain" if g is None else "g4"
            c2 = {"fn": fn2, "groups": g, "idt": "bf16", "odt": "bf16", "a": X, "b": W, "o": O, "ep": None, "options": {},
                  "a_strides": None, "b_strides": None, "o_strides": None}
            for name, xs, ws, st, pd, dl, dt in (
                    ("err2-f32-stride-h0", [1, 8, 8, 16], [32, 3, 3, 16 // (g or 1)], [0, 1], [1, 1], [1, 1], ("f32", "f32")),
                    ("err2-f32-dil-w0", [1, 8, 8, 16], [32, 3, 3, 16 // (g or 1)], [1, 1], [1, 1], [1, 0], ("f32", "f32")),
                    ("err2-lo-w-up-h", [1, 300, 300, 16], [32, 140, 1, 16 // (g or 1)], [1, 1], [0, 200], [1, 1], DT[0]),
                    ("err2-up-h-up-w", [1, 300, 300, 16], [32, 140, 150, 16 // (g or 1)], [1, 1], [0, 0], [1, 1], DT[0]),
                    ("err2-lo-h-lo-w", [1, 300, 300, 16], [32, 1, 1, 16 // (g or 1)], [1, 1], [130, 200], [1, 1], DT[0]),
                    ("err2-phase-lo-w-up-h", [1, 600, 600, 16], [32, 140, 3, 16 // (g or 1)], [2, 2], [0, 1], [1, 100], DT[0])):
                oh, ow = conv_out(xs, ws, [max(1, e) for e in st], pd, [max(1, e) for e in dl])
                ys = [xs[0], max(0, oh), max(0, ow), 32]
                ops = {"fwd": (xs, ws, ys), "dgrad": (ys, ws, xs), "wgrad": (xs, ys, ws)}[fn2]
                c = dict(c2, a_shape=ops[0], b_shape=ops[1], o_shape=ops[2], idt=dt[0], odt=dt[1], stride=st, pad=pd, dil=dl)
                out.append((f"2d-{fn2}-{gt}-{name}", from_2d(c)))
    # 2-D transposed corners, in the order (lo_h, lo_w, up_h, up_w)
    add("err2-lo-w-up-h", "tconv2", [1, 300, 300, 16], [16, 140, 160, 32], 1, 0)
    add("err2-phase-up-w-lo-h", "tconv2", [1, 300, 300, 16], [16, 140, 3, 32], 2, (0, 1), (1, 100))
    return out


def cases_2d_failing():
    """Every failing call of the 2-D fixture."""
    rows = json.loads(gzip.decompress(GOLDEN_2D.read_bytes()))["cases"]
    return [(f"2d-{r['id']}", from_2d(r["call"])) for r in rows if r["status"]]


def main() -> None:
    rows = []
    seen = set()
    for cid, c in cases() + cases_2d_failing():
        assert cid not in seen, cid
        seen.add(cid)
        rows.append({"id": cid, "call": c, **replay(c)})
    # gzip without a timestamp: the same cases always give the same bytes
    text = json.dumps({"_generated_by": "tests/golden/make_conv_nd_plan_golden.py", "cases": rows}, indent=0) + "\n"
    GOLDEN.write_bytes(gzip.compress(text.encode(), mtime=0))
    fails = sum(1 for r in rows if r["status"])
    print(f"wrote {GOLDEN}: {len(rows)} cases, {fails} failing, {GOLDEN.stat().st_size // 1024} KB")


if __name__ == "__main__":
    main()
