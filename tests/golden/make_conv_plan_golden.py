"""Record the dry-run plans of the six convolution entry points into conv_plan_golden.json.gz (read by
tests/test_conv_plan_golden_cpu.py).

    python tests/golden/make_conv_plan_golden.py

Each case is one call of b200_conv2d[_grouped][_backward_data / _weight] in a fresh planning context (b200_plan_begin, 132
SMs); the fixture stores the call, the returned status, the entry-point prefix of the error message and the full plan text.
The grid covers channel counts 3 / 16 / 64 / 256, kernels 1 / 3 / 7, strides, paddings and dilations, both output dtype
rules, strided views (NCHW x, OIHW w, NCHW dy, a misaligned base, an output channel slice, a pitched dx, a padded dw), the
GEMM variant and split-K options, groups None / 1 / wide / narrow / depthwise with and without an epilogue, one case per
failing check of every entry point, and the empty-extent rules.  Plans hold no pointer bases, so the pointer offsets of group
slices, dgrad phases and the bias are left to the GPU tests.
"""
from __future__ import annotations

import gzip
import json
import sys
from pathlib import Path

TESTS = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(TESTS.parent), str(TESTS)]

from conv_oracle import out_hw, pair  # noqa: E402
from cubecl_b200 import _ffi  # noqa: E402
from test_conv_grouped_cpu import Planner  # noqa: E402

GOLDEN = Path(__file__).resolve().parent / "conv_plan_golden.json.gz"
DTYPES = {"f32": _ffi.F32, "f16": _ffi.F16, "bf16": _ffi.BF16}
ENTRY = {"fwd": "b200_conv2d", "dgrad": "b200_conv2d_backward_data", "wgrad": "b200_conv2d_backward_weight"}

X, W, O = 0x10000000, 0x20000000, 0x30000000
BIG = 1 << 31
PADS, DILS = (0, 1, (1, 4)), (1, 2)
DT = (("bf16", "bf16"), ("f16", "f32"))


def replay(call: dict) -> dict:
    """One recorded call in a fresh dry-run context (132 SMs): {status, error (the message up to its first ':'), plan}."""
    with Planner(132, call["options"]) as p:
        ep = _ffi.Epilogue(*call["ep"]) if call["ep"] is not None else None
        rc, text = p.call(ENTRY[call["fn"]], call["a_shape"], call["b_shape"], call["o_shape"], call["groups"],
                          idt=DTYPES[call["idt"]], odt=DTYPES[call["odt"]], stride=call["stride"], pad=call["pad"], dil=call["dil"],
                          a_strides=call["a_strides"], b_strides=call["b_strides"], o_strides=call["o_strides"],
                          a=call["a"], b=call["b"], o=call["o"], ep=ep, forward=call["fn"] == "fwd")
        err = ""
        if rc:
            msg = p.lib.b200_last_error()
            err = msg.decode().split(":")[0] if msg else ""
        return {"status": rc, "error": err, "plan": text}


def call(fn, xs, ws, groups=None, stride=1, pad=0, dil=1, dt=DT[0], ys=None, a_strides=None, b_strides=None, o_strides=None,
         a=X, b=W, o=O, ep=None, options=None, shapes=None):
    """The recorded arguments of one call.  xs / ws: the forward's input and weights; ys (dy, or the forward's out) defaults to
    the output rule.  The operands are (x, w, out), (dy, w, dx) or (x, dy, dw) by entry point; shapes overrides them."""
    if ys is None and xs is not None and ws is not None:
        # a zero stride or an empty result (cases that fail their argument checks) still gets a shape of valid extents
        hw = out_hw(xs[1], xs[2], ws[1], ws[2], [max(1, e) for e in pair(stride)], pad, dil)
        ys = [xs[0], *(max(0, e) for e in hw), ws[0]]
    ops = shapes or {"fwd": (xs, ws, ys), "dgrad": (ys, ws, xs), "wgrad": (xs, ys, ws)}[fn]
    return {"fn": fn, "groups": groups, "a_shape": ops[0], "b_shape": ops[1], "o_shape": ops[2], "a_strides": a_strides,
            "b_strides": b_strides, "o_strides": o_strides, "idt": dt[0], "odt": dt[1], "stride": list(pair(stride)),
            "pad": list(pair(pad)), "dil": list(pair(dil)), "a": a, "b": b, "o": o, "ep": ep, "options": options or {}}


def nchw(s):
    """Strides of an NHWC-indexed [n, h, w, c] view of a compact NCHW tensor (also OIHW weights and NCHW dy)."""
    n, h, w, c = s
    return [c * h * w, w, 1, h * w]


def cases():
    out = []

    def add(name, fn, *args, **kw):
        out.append((f"{fn}-{name}", call(fn, *args, **kw)))

    # geometry grid, plain entry points: every (kernel, stride) per channel count; padding, dilation and dtypes in a rotation
    i = 0
    for c in (3, 16, 64, 256):
        cout = 32 if c < 64 else 96
        for k in (1, 3, 7):
            for s in (1, 2, (2, 3)):
                pad, dil, dt = PADS[(i + i // 3) % 3], DILS[(i + i // 9) % 2], DT[(i + i // 3) % 2]
                for fn in ("fwd", "dgrad", "wgrad"):
                    add(f"c{c}-k{k}-s{s}-p{pad}-d{dil}-{dt[0]}{dt[1]}", fn, [2, 17, 15, c], [cout, k, k, c], None, s, pad, dil, dt)
                i += 1
    # grouped entry points: groups 1 (the plain route), wide (Cg = 64), narrow (Cg = 8) and depthwise (multiplier 2)
    grp = {"g1": (64, 64, 1), "wide": (128, 192, 2), "narrow": (32, 48, 4), "dw": (32, 64, 32)}
    for tag, (c, cout, g) in grp.items():
        i = 0
        for k in (1, 3, 7):
            for s in (1, 2, (2, 3)):
                pad, dil, dt = PADS[(i + i // 3) % 3], DILS[i % 2], DT[(i // 2) % 2]
                for fn in ("fwd", "dgrad", "wgrad"):
                    add(f"grp-{tag}-k{k}-s{s}-p{pad}-d{dil}-{dt[0]}{dt[1]}", fn, [2, 13, 11, c], [cout, k, k, c // g], g, s, pad, dil, dt)
                i += 1
        # fused epilogue (alpha, gelu, bias) and alpha alone
        add(f"grp-{tag}-ep-gelu", "fwd", [2, 13, 11, c], [cout, 3, 3, c // g], g, 1, 1, ep=[0.5, 2, 0x40000000])
        add(f"grp-{tag}-ep-alpha-f32", "fwd", [2, 13, 11, c], [cout, 3, 3, c // g], g, 2, 1, dt=DT[1], ep=[2.0, 0, 0])
    for name, ep in (("ep-relu-bias", [1.0, 1, 0x40000000]), ("ep-gelu-alpha", [0.25, 2, 0]), ("ep-identity", [1.0, 0, 0])):
        add(name, "fwd", [2, 17, 15, 64], [96, 3, 3, 64], None, 1, 1, ep=ep)
        add(name + "-c3", "fwd", [2, 17, 15, 3], [32, 7, 7, 3], None, 2, 3, dt=DT[1], ep=ep)

    # views
    for c in (3, 16, 64):
        xs, ws = [2, 12, 10, c], [32, 3, 3, c]
        ys = [2, 12, 10, 32]
        add(f"nchw-x-c{c}", "fwd", xs, ws, None, 1, 1, a_strides=nchw(xs))
        add(f"oihw-w-c{c}", "fwd", xs, ws, None, 1, 1, b_strides=nchw(ws))
        add(f"misaligned-x-c{c}", "fwd", xs, ws, None, 1, 1, a=X + 2)
        add(f"misaligned-w-c{c}", "fwd", xs, ws, None, 1, 1, b=W + 2)
        add(f"x-pitch-c{c}", "fwd", xs, ws, None, 1, 1, a_strides=[12 * 10 * (c + 8), 10 * (c + 8), c + 8, 1])
        add(f"out-slice-c{c}", "fwd", xs, ws, None, 1, 1, o=O + 64, o_strides=[12 * 10 * 64, 10 * 64, 64, 1])
        add(f"nchw-x-c{c}", "wgrad", xs, ws, None, 1, 1, a_strides=nchw(xs))
        add(f"misaligned-x-c{c}", "wgrad", xs, ws, None, 1, 1, a=X + 2)
        add(f"oihw-w-c{c}", "dgrad", xs, ws, None, 1, 1, b_strides=nchw(ws))
        add(f"pitched-dx-c{c}", "dgrad", xs, ws, None, 1, 1, o_strides=[12 * 10 * (c + 8), 10 * (c + 8), c + 8, 1])
        add(f"dx-slice-c{c}", "dgrad", xs, ws, None, 2, 1, o=O + 2 * c, o_strides=[12 * 10 * 2 * c, 10 * 2 * c, 2 * c, 1])
        add(f"dw-cout-stride-c{c}", "wgrad", xs, ws, None, 1, 1, o_strides=[9 * c + 64, 3 * c, c, 1])
        add(f"dw-cout-stride-s2-c{c}", "wgrad", xs, ws, None, 2, 1, dt=DT[1], o_strides=[9 * c + 8, 3 * c, c, 1])
    for fn in ("dgrad", "wgrad"):
        xs, ws = [2, 12, 10, 16], [32, 3, 3, 16]
        for s in (1, 2):
            ys = [2, *out_hw(12, 10, 3, 3, s, 1, 1), 32]
            add(f"nchw-dy-s{s}", fn, xs, ws, None, s, 1, ys=ys, **{("a_strides" if fn == "dgrad" else "b_strides"): nchw(ys)})
            add(f"misaligned-dy-s{s}", fn, xs, ws, None, s, 1, ys=ys, **{("a" if fn == "dgrad" else "b"): (X if fn == "dgrad" else W) + 2})
            add(f"dy-pitch-s{s}", fn, xs, ws, None, s, 1, ys=ys,
                **{("a_strides" if fn == "dgrad" else "b_strides"): [ys[1] * ys[2] * 40, ys[2] * 40, 40, 1]})
    for tag, (c, cout, g) in grp.items():
        xs, ws = [2, 12, 10, c], [cout, 3, 3, c // g]
        ys = [2, 12, 10, cout]
        add(f"grp-{tag}-nchw-x", "fwd", xs, ws, g, 1, 1, a_strides=nchw(xs))
        add(f"grp-{tag}-oihw-w", "fwd", xs, ws, g, 1, 1, b_strides=nchw(ws))
        add(f"grp-{tag}-misaligned-x", "fwd", xs, ws, g, 1, 1, a=X + 2)
        add(f"grp-{tag}-out-slice", "fwd", xs, ws, g, 1, 1, o=O + 2 * cout, o_strides=[12 * 10 * 2 * cout, 10 * 2 * cout, 2 * cout, 1])
        add(f"grp-{tag}-nchw-dy", "dgrad", xs, ws, g, 1, 1, a_strides=nchw(ys))
        add(f"grp-{tag}-oihw-w", "dgrad", xs, ws, g, 1, 1, b_strides=nchw(ws))
        add(f"grp-{tag}-pitched-dx", "dgrad", xs, ws, g, 2, 1, o_strides=[12 * 10 * (c + 8), 10 * (c + 8), c + 8, 1])
        add(f"grp-{tag}-nchw-x", "wgrad", xs, ws, g, 1, 1, a_strides=nchw(xs))
        add(f"grp-{tag}-nchw-dy", "wgrad", xs, ws, g, 1, 1, b_strides=nchw(ys))
        add(f"grp-{tag}-dw-cout-stride", "wgrad", xs, ws, g, 1, 1, o_strides=[9 * (c // g) + 8, 3 * (c // g), c // g, 1])

    # options
    for opts in ({"gemm.variant": "1sm_n128"}, {"gemm.split_k": "on"}, {"gemm.variant": "1sm_n128", "gemm.split_k": "on"}):
        tag = "-".join(f"{k.split('.')[1]}={v}" for k, v in opts.items())
        for fn in ("fwd", "dgrad", "wgrad"):
            add(f"opt-{tag}", fn, [4, 28, 28, 64], [128, 3, 3, 64], None, 1, 1, options=opts)
            add(f"opt-{tag}-s2-c3", fn, [4, 28, 28, 3], [64, 7, 7, 3], None, 2, 3, dt=DT[1], options=opts)
            add(f"opt-{tag}-grp-wide", fn, [2, 14, 14, 128], [128, 3, 3, 64], 2, 1, 1, options=opts)

    # one case per failing check: plain, narrow (Cg = 2) and wide (Cg = 64) groups
    for g, c, wc in ((None, 16, 16), (8, 16, 2), (2, 128, 64)):
        gt = "plain" if g is None else f"g{g}"
        xs, gws = [1, 8, 8, c], [32, 3, 3, wc]
        for fn in ("fwd", "dgrad", "wgrad"):
            def bad(name, **kw):
                base = dict(xs=xs, ws=gws, groups=g, stride=1, pad=1, dil=1)
                base.update(kw)
                xs_, ws_ = base.pop("xs"), base.pop("ws")
                add(f"err-{gt}-{name}", fn, xs_, ws_, **base)
            for j in range(3):
                sh = [call(fn, xs, gws, g, 1, 1)[k] for k in ("a_shape", "b_shape", "o_shape")]
                sh[j] = None
                bad(f"null-shape{j}", shapes=sh)
            bad("f32-input", dt=("f32", "f32"))
            bad("bf16-to-f16", dt=("bf16", "f16"))
            bad("f16-to-bf16", dt=("f16", "bf16"))
            bad("stride0", stride=(0, 1))
            bad("dil0", dil=(1, 0))
            bad("pad-neg", pad=(1, -1))
            bad("weight-channels", ws=[32, 3, 3, wc + 1])
            bad("extent-2^31", xs=[1, BIG, 8, c])
            bad("kernel-too-large", ws=[32, 11, 3, wc], ys=[1, 1, 8, 32])
            bad("stride9", xs=[1, 20, 20, c], stride=9)
            bad("corner-pad", xs=[1, 300, 8, c], pad=(129, 0))
            bad("corner-dil", xs=[1, 300, 8, c], pad=(0, 1), dil=(100, 1))
            bad("pixels-2^31", xs=[1 << 16, 200, 200, c])
            bad("null-a", a=0)
            bad("null-b", b=0)
            bad("null-out", o=0)
            bad("misaligned-out", o=O + 1)
            bad("misaligned-out-f32", o=O + 2, dt=DT[1])
            bad("kpos-2^31", xs=[1, 8, 8, 1 << 28], ws=[32, 3, 3, (1 << 28) // (g or 1)])
            if fn == "fwd":
                bad("bad-out-shape", ys=[1, 7, 6, 32])
                bad("bad-out-cout", ys=[1, 8, 8, 31])
                bad("activation", ep=[1.0, 3, 0])
                bad("activation-neg", ep=[1.0, -1, 0])
                bad("out-channel-stride", o_strides=[8 * 8 * 64, 8 * 64, 64, 2])
                bad("out-pitch-small", o_strides=[8 * 8 * 16, 8 * 16, 16, 1])
                bad("out-rows-gap", o_strides=[8 * 8 * 40 + 8, 8 * 40 + 8, 40, 1])
            else:
                bad("bad-dy-shape", ys=[1, 5, 6, 32])
                bad("bad-dy-n", ys=[2, 8, 8, 32])
                bad("bad-dy-cout", ys=[1, 8, 8, 31])
                bad("dy-extent-2^31", ys=[1, 8, 8, BIG])
            if fn == "dgrad":
                bad("dx-channel-stride", o_strides=[8 * 8 * c * 2, 8 * c * 2, c * 2, 2])
                bad("dx-pitch-small", o_strides=[8 * 8 * 8, 8 * 8, 8, 1])
                bad("kpos-cout-2^31", ws=[1 << 28, 3, 3, wc], ys=[1, 8, 8, 1 << 28])
                bad("phase-corner", xs=[1, 600, 8, c], stride=(2, 1), pad=(0, 1), dil=(200, 1))
                bad("dx-pixels-2^31", xs=[1 << 16, 200, 200, c], ws=[32, 201, 3, wc], pad=(0, 1))
            if fn == "wgrad":
                bad("dw-channel-stride", o_strides=[9 * wc * 2, wc * 2, 2, wc * 2])
                bad("dw-kpos-not-flat", o_strides=[9 * 80, 3 * 80, wc + 8, 1])
                bad("dw-stride-2^40", o_strides=[1 << 40, 3 * wc, wc, 1])
        if g is not None:
            for fn in ("fwd", "dgrad", "wgrad"):
                add(f"err-{gt}-groups0", fn, xs, gws, 0, 1, 1)
                add(f"err-{gt}-c-not-divisible", fn, [1, 8, 8, c + 2], gws, g, 1, 1)
                add(f"err-{gt}-cout-not-divisible", fn, xs, [33, 3, 3, wc], g, 1, 1)
    # the direct kernels' own limits (depthwise)
    add("err-dw-too-many-chunks", "fwd", [1, 4, 4, 1 << 22], [1 << 22, 1, 1, 1], 1 << 22)
    add("err-dw-too-many-chunks", "dgrad", [1, 4, 4, 1 << 22], [1 << 22, 1, 1, 1], 1 << 22)
    add("err-dw-elems-2^31", "wgrad", [1, 8, 8, 1 << 26], [1 << 26, 7, 7, 1], 1 << 26, 1, 3)

    # empty extents, and an empty extent together with a wrong output shape
    for g, gws in ((None, [32, 3, 3, 16]), (8, [32, 3, 3, 2]), (16, [32, 3, 3, 1])):
        gt = "plain" if g is None else f"g{g}"
        for fn in ("fwd", "dgrad", "wgrad"):
            for name, xs, ws in (("n0", [0, 8, 8, 16], gws), ("h0", [1, 0, 8, 16], gws), ("c0", [1, 8, 8, 0], [32, 3, 3, 0]),
                                 ("cout0", [1, 8, 8, 16], [0, 3, 3, gws[3]]), ("kh0", [1, 8, 8, 16], [32, 0, 3, gws[3]]),
                                 ("kw0", [1, 8, 8, 16], [32, 3, 0, gws[3]])):
                add(f"empty-{gt}-{name}", fn, xs, ws, g, 2, 1)
            add(f"empty-{gt}-n0-dw-cout-stride", fn, [0, 8, 8, 16], gws, g, 1, 1, o_strides=[9 * gws[3] + 8, 3 * gws[3], gws[3], 1])
            ys = [0, 7, 6, 32]
            add(f"empty-{gt}-n0-wrong-out", fn, [0, 8, 8, 16], gws, g, ys=ys)
            add(f"empty-{gt}-n0-wrong-out-nullptr", fn, [0, 8, 8, 16], gws, g, ys=ys, a=0, b=0, o=0)
    return out


def main() -> None:
    rows = []
    seen = set()
    for cid, c in cases():
        assert cid not in seen, cid
        seen.add(cid)
        rows.append({"id": cid, "call": c, **replay(c)})
    # gzip without a timestamp: the same cases always give the same bytes
    text = json.dumps({"_generated_by": "tests/golden/make_conv_plan_golden.py", "cases": rows}, indent=0) + "\n"
    GOLDEN.write_bytes(gzip.compress(text.encode(), mtime=0))
    fails = sum(1 for r in rows if r["status"])
    print(f"wrote {GOLDEN}: {len(rows)} cases, {fails} failing, {GOLDEN.stat().st_size // 1024} KB")


if __name__ == "__main__":
    main()
