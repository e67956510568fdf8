"""Record the dry-run plans of the six attention entry points into attention_plan_golden.json.gz (read by
tests/test_attention_plan_golden_cpu.py).

    python tests/golden/make_attention_plan_golden.py

Each case is one call of b200_attention[_backward], b200_attention_kvcache, b200_kvcache_write or
b200_attention_varlen[_backward] in a fresh planning context (b200_plan_begin with 132 SMs, or 114 for some KV-cache cases,
whose split count depends on it), made through the Planner classes of the four attention CPU test files.  The fixture stores the
call, the returned status, the entry-point prefix of the error message and the full plan text.  The cases cover both input
dtypes with out and grads in the input dtype or f32, head dims 8 to 128, GQA, causal and window masks, extents around the
128-row blocks, in-place views ([B, S, H, D], fused-QKV slices, head-major caches and varlen tensors), every gather trigger on
every operand, page sizes and decode tiles, one case per failing check of every entry point, the empty-extent rules and a few
double faults whose status the check order decides.  Plans hold no pointer bases and no kernel parameter blocks, so which
buffer and which stride reaches which kernel field is left to the GPU tests.
"""
from __future__ import annotations

import ctypes as C
import gzip
import json
import math
import sys
from pathlib import Path

TESTS = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(TESTS.parent), str(TESTS)]

import test_attention_backward_cpu as tb  # noqa: E402
import test_attention_cpu as tf  # noqa: E402
import test_attention_kvcache_cpu as tk  # noqa: E402
import test_attention_varlen_cpu as tv  # noqa: E402
from cubecl_b200 import _ffi  # noqa: E402

GOLDEN = Path(__file__).resolve().parent / "attention_plan_golden.json.gz"
DTYPES = {"f32": _ffi.F32, "f16": _ffi.F16, "bf16": _ffi.BF16, "i8": _ffi.I8}
BIG = 1 << 31


def _varlen_bwd(p, qs, ks, B, maxq, maxk, shapes, idt="bf16", odt=None, gdt=None, window=(-1, -1)):
    """b200_attention_varlen_backward with every operand's shape given (shapes over q, k, v, out, dout, dq, dk, dv), for the
    shape refusals the Planner's bwd cannot express"""
    sh = {"q": qs, "k": ks, "v": ks, "out": qs, "dout": qs, "dq": qs, "dk": ks, "dv": ks}
    sh.update(shapes)
    pt = dict(zip(("q", "k", "v", "out", "dout", "dq", "dk", "dv"), (tv.Q, tv.K, tv.V, tv.OUT, tv.DOUT, tv.DQ, tv.DK, tv.DV)))
    ops = []
    for n in ("q", "k", "v", "out", "dout"):
        ops += [pt[n], _ffi.u64_array(sh[n]), None]
    ops += [tv.LSE, tv.CUQ, tv.CUK, B]
    for n in ("dq", "dk", "dv"):
        ops += [pt[n], _ffi.u64_array(sh[n]), None]
    args = _ffi.AttentionVarlenArgs(0.125, window[0], window[1], maxq, maxk)
    rc = p.lib.b200_attention_varlen_backward(p.ctx, None, DTYPES[idt], DTYPES[odt or idt], DTYPES[gdt or idt], *ops, C.byref(args))
    return rc, p.text()


PLANNERS = {
    "fwd": (tf.Planner, "run"), "bwd": (tb.Planner, "run"), "kv": (tk.Planner, "run"), "kvwrite": (tk.Planner, "write"),
    "varlen": (tv.Planner, "fwd"), "varlen_bwd": (tv.Planner, "bwd"),
}


def replay(call: dict) -> dict:
    """One recorded call in a fresh dry-run context: {status, error (the message up to its first ':'), plan}."""
    cls, method = PLANNERS[call["fn"]]
    p = cls(call["sms"])
    try:
        kw = dict(call["kw"])
        if "shapes" in kw and call["fn"] == "varlen_bwd":
            rc, text = _varlen_bwd(p, *call["args"], **kw)
        else:
            for key in ("idt", "odt", "gdt", "dt"):
                if kw.get(key) is not None:
                    kw[key] = DTYPES[kw[key]]
            rc, text = getattr(p, method)(*call["args"], **kw)
        err = ""
        if rc:
            msg = p.lib.b200_last_error()
            err = msg.decode().split(":")[0] if msg else ""
        return {"status": rc, "error": err, "plan": text}
    finally:
        p.close()


def cases():
    out = []

    def add(name, fn, *args, sms=132, **kw):
        out.append((f"{fn}-{name}", {"fn": fn, "sms": sms, "args": list(args), "kw": kw}))

    dts = [(i, o, g) for i in ("bf16", "f16") for o in (i, "f32") for g in (i, "f32")]
    Ds = (8, 40, 64, 72, 128)

    # ------------------------------------------------------------------------------------------------ b200_attention
    fwd = lambda name, qs, ks, **kw: add(name, "fwd", qs, ks, **kw)  # noqa: E731
    for i, o, _ in dts[::2]:
        for D in Ds:
            fwd(f"{i}-{o}-d{D}", [2, 4, 300, D], [2, 2, 200, D], idt=i, odt=o, causal=D % 16 == 8)
    for Sq, Sk in ((1, 1), (127, 128), (128, 129), (129, 127), (256, 257), (257, 256), (1000, 3)):
        for causal in (0, 1):
            fwd(f"edges-{Sq}x{Sk}-c{causal}", [2, 3, Sq, 64], [2, 3, Sk, 64], causal=causal)
    fwd("gqa-8-1", [1, 8, 200, 128], [1, 1, 333, 128], odt="f32", causal=1)
    fwd("scale-2", [1, 2, 64, 64], [1, 2, 64, 64], scale=2.0)
    B, H, S, D = 2, 4, 100, 64
    bshd = [S * H * D, D, H * D, 1]
    fwd("bshd", [B, H, S, D], [B, H, S, D], strides=[bshd] * 4)
    fused = [S * 3 * H * D, D, 3 * H * D, 1]
    fwd("fused-qkv", [B, H, S, D], [B, H, S, D], strides=[fused, fused, fused, None],
        ptrs=[tf.Q, tf.Q + 2 * H * D, tf.Q + 4 * H * D, tf.OUT])
    fwd("out-pitched-f32", [B, H, S, D], [B, H, S, D], odt="f32", strides=[None, None, None, [H * S * 72, S * 72, 72, 1]])
    for j, n in enumerate("qkv"):
        base = [tf.Q, tf.K, tf.V, tf.OUT]
        mis = list(base)
        mis[j] += 2
        fwd(f"gather-{n}-misaligned", [B, H, S, D], [B, H, S, D], ptrs=mis)
        st = [None] * 4
        st[j] = [H * D * S, D * S, 1, S]
        fwd(f"gather-{n}-d-stride", [B, H, S, D], [B, H, S, D], strides=st)
        st = [None] * 4
        st[j] = [H * S * 68, S * 68, 68, 1]
        fwd(f"gather-{n}-odd-stride", [B, H, S, D], [B, H, S, D], strides=st)
    fwd("gather-all-f16-f32", [B, H, S, 40], [B, 2, 77, 40], idt="f16", odt="f32", ptrs=[tf.Q + 2, tf.K + 2, tf.V + 2, tf.OUT])
    # refusals (test_attention_cpu.py's table) and a few more
    qs, ks = [2, 4, 100, 64], [2, 2, 80, 64]
    fwd("err-batch", qs, [1, 2, 80, 64])
    fwd("err-head-dim", qs, [2, 2, 80, 32])
    fwd("err-gqa", qs, [2, 3, 80, 64])
    fwd("err-hkv0", qs, [2, 0, 80, 64])
    fwd("err-v-shape", qs, ks, vs=[2, 2, 81, 64])
    fwd("err-out-shape", qs, ks, outs=[2, 4, 100, 32])
    fwd("err-sk0", qs, [2, 2, 0, 64])
    fwd("err-scale-inf", qs, ks, scale=math.inf)
    fwd("err-scale-nan", qs, ks, scale=math.nan)
    for j, n in enumerate(("q", "k", "v", "out")):
        ptrs = [tf.Q, tf.K, tf.V, tf.OUT]
        ptrs[j] = 0
        fwd(f"err-null-{n}", qs, ks, ptrs=ptrs)
    fwd("err-null-args", qs, ks, null_args=True)
    fwd("err-lse-align", qs, ks, lse=tf.LSE + 2)
    fwd("err-in-f32", qs, ks, idt="f32", odt="f32")
    fwd("err-in-i8", qs, ks, idt="i8", odt="f32")
    fwd("err-out-other", qs, ks, idt="bf16", odt="f16")
    fwd("err-d136", [2, 4, 100, 136], [2, 2, 80, 136])
    fwd("err-d12", [2, 4, 100, 12], [2, 2, 80, 12])
    fwd("err-d0", [2, 4, 100, 0], [2, 2, 80, 0])
    fwd("err-dv", qs, ks, vs=[2, 2, 80, 32])
    fwd("err-out-d-stride", qs, ks, strides=[None, None, None, [4 * 100 * 64, 1, 4 * 64, 4]])
    fwd("err-out-misaligned", qs, ks, ptrs=[tf.Q, tf.K, tf.V, tf.OUT + 2])
    fwd("err-out-misaligned-f32", qs, ks, odt="f32", ptrs=[tf.Q, tf.K, tf.V, tf.OUT + 8])
    fwd("err-out-stride-2^40", qs, ks, strides=[None, None, None, [1 << 40, 100 * 64, 64, 1]])
    fwd("err-huge", [2, BIG, 100, 64], [2, 1, 80, 64])
    fwd("err-huge-sk", [2, 4, 100, 64], [2, 2, BIG, 64])
    fwd("err-ctas", [1 << 16, 1 << 16, 1 << 10, 64], [1 << 16, 1 << 16, 8, 64])
    # empty extents, and double faults
    for name, q_, k_ in (("b0", [0, 4, 100, 64], [0, 2, 80, 64]), ("hq0", [2, 0, 100, 64], [2, 1, 80, 64]),
                         ("sq0", [2, 4, 0, 64], [2, 2, 80, 64]), ("sq0-sk0", [2, 4, 0, 64], [2, 2, 0, 64])):
        fwd(f"empty-{name}", q_, k_)
        fwd(f"empty-{name}-null", q_, k_, ptrs=[0, 0, 0, 0], lse=3)
    fwd("double-out-dtype-and-shape", qs, [1, 2, 80, 64], idt="bf16", odt="f16")
    fwd("double-in-dtype-and-d", [2, 4, 100, 12], [2, 2, 80, 12], idt="f32", odt="f32")
    fwd("double-sk0-and-scale", qs, [2, 2, 0, 64], scale=math.inf)
    fwd("double-null-and-out-view", qs, ks, ptrs=[0, tf.K, tf.V, tf.OUT + 2])
    fwd("double-lse-and-out-view", qs, ks, lse=tf.LSE + 2, ptrs=[tf.Q, tf.K, tf.V, tf.OUT + 2])

    # ------------------------------------------------------------------------------------------------ b200_attention_backward
    bwd = lambda name, qs, ks, **kw: add(name, "bwd", qs, ks, **kw)  # noqa: E731
    for i, o, g in dts:
        for D in Ds:
            bwd(f"{i}-{o}-{g}-d{D}", [2, 4, 300, D], [2, 2, 200, D], idt=i, odt=o, gdt=g, causal=D % 16 == 8)
    for Sq, Sk in ((1, 1), (127, 128), (128, 129), (129, 127), (256, 257), (257, 1000)):
        for causal in (0, 1):
            bwd(f"edges-{Sq}x{Sk}-c{causal}", [3, 6, Sq, 64], [3, 2, Sk, 64], causal=causal)
    names = ("q", "k", "v", "out", "dout", "dq", "dk", "dv")
    bwd("bshd", [B, H, S, D], [B, H, S, D], strides=dict.fromkeys(names, bshd))
    G = 0x90000000
    bwd("fused-qkv", [B, H, S, D], [B, H, S, D], strides={n: fused for n in ("q", "k", "v", "dq", "dk", "dv")},
        ptrs={"q": tb.Q, "k": tb.Q + 2 * H * D, "v": tb.Q + 4 * H * D, "dq": G, "dk": G + 2 * H * D, "dv": G + 4 * H * D})
    bwd("grads-pitched-f32", [B, H, S, D], [B, 2, 70, D], gdt="f32",
        strides={"dq": [H * S * 72, S * 72, 72, 1], "dk": [2 * 70 * 80, 70 * 80, 80, 1], "dv": [70 * 2 * D, D, 2 * D, 1]})
    ptr0 = {"q": tb.Q, "k": tb.K, "v": tb.V, "out": tb.OUT, "dout": tb.DOUT}
    for n in ("q", "k", "v", "out", "dout"):
        for odt in (None, "f32") if n == "out" else (None,):
            tag = f"gather-{n}" + ("-f32" if odt else "")
            bwd(f"{tag}-misaligned", [B, H, S, D], [B, H, S, D], odt=odt, ptrs={n: ptr0[n] + (8 if odt else 2)})
            bwd(f"{tag}-d-stride", [B, H, S, D], [B, H, S, D], odt=odt, strides={n: [H * D * S, D * S, 1, S]})
            bwd(f"{tag}-odd-stride", [B, H, S, D], [B, H, S, D], odt=odt, strides={n: [H * S * (66 if odt else 68), S * (66 if odt else 68),
                                                                                         66 if odt else 68, 1]})
    bwd("gather-all-f16", [B, H, S, 40], [B, 2, 77, 40], idt="f16", odt="f32", gdt="f32",
        ptrs={"q": tb.Q + 2, "k": tb.K + 2, "v": tb.V + 2, "out": tb.OUT + 4, "dout": tb.DOUT + 2})
    qs, ks = [2, 4, 100, 64], [2, 2, 80, 64]
    bwd("err-batch", qs, [1, 2, 80, 64])
    bwd("err-head-dim", qs, [2, 2, 80, 32])
    bwd("err-gqa", qs, [2, 3, 80, 64])
    bwd("err-hkv0", qs, [2, 0, 80, 64])
    bwd("err-v-shape", qs, ks, shapes={"v": [2, 2, 81, 64]})
    for n in ("out", "dout", "dq"):
        bwd(f"err-{n}-shape", qs, ks, shapes={n: [2, 4, 101, 64]})
    for n in ("dk", "dv"):
        bwd(f"err-{n}-shape", qs, ks, shapes={n: [2, 2, 80, 32]})
    bwd("err-sk0", qs, [2, 2, 0, 64])
    bwd("err-scale-inf", qs, ks, scale=math.inf)
    bwd("err-scale-nan", qs, ks, scale=math.nan)
    for n in names:
        bwd(f"err-null-{n}", qs, ks, ptrs={n: 0})
    bwd("err-null-args", qs, ks, null_args=True)
    bwd("err-null-lse", qs, ks, lse=0)
    bwd("err-lse-align", qs, ks, lse=tb.LSE + 2)
    bwd("err-in-f32", qs, ks, idt="f32", odt="f32", gdt="f32")
    bwd("err-in-i8", qs, ks, idt="i8", odt="f32", gdt="f32")
    bwd("err-out-other", qs, ks, odt="f16")
    bwd("err-grad-other", qs, ks, gdt="f16")
    bwd("err-d136", [2, 4, 100, 136], [2, 2, 80, 136])
    bwd("err-d12", [2, 4, 100, 12], [2, 2, 80, 12])
    bwd("err-dv-dim", qs, ks, shapes={"v": [2, 2, 80, 32]})
    bwd("err-dq-d-stride", qs, ks, strides={"dq": [4 * 100 * 64, 1, 4 * 64, 4]})
    bwd("err-dk-misaligned", qs, ks, ptrs={"dk": tb.DK + 2})
    bwd("err-dv-odd-stride", qs, ks, strides={"dv": [2 * 80 * 68, 80 * 68, 68, 1]})
    bwd("err-dq-misaligned-f32", qs, ks, gdt="f32", ptrs={"dq": tb.DQ + 8})
    bwd("err-huge", [2, BIG, 100, 64], [2, 1, 80, 64])
    bwd("err-ctas", [1 << 16, 1 << 16, 1 << 10, 64], [1 << 16, 1 << 16, 8, 64])
    for name, q_, k_ in (("b0", [0, 4, 100, 64], [0, 2, 80, 64]), ("sq0-sk0", [2, 4, 0, 64], [2, 2, 0, 64]),
                         ("b0-sq0-sk0", [0, 4, 0, 64], [0, 2, 0, 64]), ("sq0", [2, 4, 0, 64], [2, 2, 80, 64]),
                         ("hq0", [2, 0, 100, 64], [2, 1, 80, 64]), ("hq0-sq0-d128", [1, 0, 0, 128], [1, 3, 300, 128])):
        bwd(f"empty-{name}", q_, k_)
        bwd(f"empty-{name}-null-q-side", q_, k_, ptrs={"q": 0, "out": 0, "dout": 0, "dq": 0}, lse=0)
    bwd("empty-sq0-null-k", [2, 4, 0, 64], [2, 2, 80, 64], ptrs={"k": 0})
    bwd("empty-sq0-dk-misaligned", [2, 4, 0, 64], [2, 2, 80, 64], ptrs={"dk": tb.DK + 2})
    bwd("empty-sq0-dq-misaligned", [2, 4, 0, 64], [2, 2, 80, 64], ptrs={"dq": tb.DQ + 2})
    bwd("empty-sq0-q-gathered-not", [2, 4, 0, 64], [2, 2, 80, 64], ptrs={"q": tb.Q + 2, "out": tb.OUT + 2})
    bwd("double-grad-dtype-and-shape", qs, ks, gdt="f16", shapes={"dq": [2, 4, 101, 64]})
    bwd("double-shape-and-sk0", qs, [2, 2, 0, 64], shapes={"dout": [2, 4, 101, 64]})
    bwd("double-null-and-grad-view", qs, ks, ptrs={"q": 0, "dk": tb.DK + 2})
    bwd("double-grad-views", qs, ks, ptrs={"dv": tb.DV + 2}, strides={"dq": [4 * 100 * 64, 1, 4 * 64, 4]})

    # ------------------------------------------------------------------------------------------------ b200_attention_kvcache
    kv = lambda name, qs, kcs, **kw: add(name, "kv", qs, kcs, **kw)  # noqa: E731
    for i, o, _ in dts[::2]:
        for D in Ds:
            kv(f"{i}-{o}-d{D}", [4, 8, 1, D], [40, 16, 2, D], bts=[4, 10], idt=i, odt=o, causal=D % 16 == 8)
    for sms in (132, 114):
        for Bq, Hq, Hkv, Sq, cap in ((1, 32, 8, 1, 65536), (8, 32, 8, 1, 16384), (64, 32, 32, 1, 2048), (128, 32, 8, 1, 1000),
                                     (2, 8, 1, 4, 16384), (1, 32, 32, 1, 64), (4, 16, 4, 33, 8192)):
            kv(f"splits-sms{sms}-b{Bq}-h{Hq}x{Hkv}-sq{Sq}-cap{cap}", [Bq, Hq, Sq, 128], [Bq, cap, Hkv, 128], sms=sms)
    for page in (16, 64, 128, 256):
        for Sq in (1, 4):
            kv(f"page{page}-sq{Sq}", [3, 8, Sq, 128], [3 * 4096 // page + 5, page, 2, 128], bts=[3, 4096 // page], causal=Sq > 1)
    for G, Sq in ((1, 1), (1, 33), (4, 4), (4, 33), (8, 33), (64, 4), (128, 33)):
        kv(f"mtile-g{G}-sq{Sq}", [2, G * 2, Sq, 64], [2, 640, 2, 64], causal=1)
    Bq, Hq, Hkv, Sq, D, P, page = 2, 8, 2, 3, 64, 10, 64
    hm = [Hkv * page * D, D, page * D, 1]
    qv = [Sq * Hq * D, D, Hq * D, 1]
    base = [tk.Q, tk.KC, tk.VC, tk.BT, tk.SL, tk.OUT]
    kv("head-major-cache-bshd-q", [Bq, Hq, Sq, D], [P, page, Hkv, D], bts=[Bq, 5], strides=[qv, hm, hm, None, None])
    kv("bt-strided", [Bq, Hq, 1, D], [P, page, Hkv, D], bts=[Bq, 5], strides=[None, None, None, [8, 1], None])
    kv("out-pitched-f32", [Bq, Hq, Sq, D], [P, page, Hkv, D], bts=[Bq, 5], odt="f32",
       strides=[None, None, None, None, [Hq * Sq * 72, Sq * 72, 72, 1]])
    kv("gather-q-misaligned", [64, 4, 1, 64], [64, 128, 2, 64], ptrs=[tk.Q + 2] + base[1:])
    kv("gather-q-d-stride", [4, 4, 3, 64], [4, 128, 2, 64], strides=[[4 * 3 * 64, 3 * 64, 1, 3], None, None, None, None])
    kv("gather-q-odd-stride", [4, 4, 3, 64], [4, 128, 2, 64], strides=[[4 * 3 * 68, 3 * 68, 68, 1], None, None, None, None], idt="f16")
    kv("one-page-any-size", [3, 4, 1, 64], [7, 1000, 2, 64], bts=[3, 1])
    kv("no-table-any-size", [3, 4, 1, 64], [3, 20, 2, 64])
    qs, kcs, bts = [2, 4, 1, 64], [8, 16, 2, 64], [2, 4]
    kv("err-head-dim", qs, [8, 16, 2, 32], bts=bts)
    kv("err-v-shape", qs, kcs, bts=bts, vcs=[8, 32, 2, 64])
    kv("err-gqa", qs, [8, 16, 3, 64], bts=bts)
    kv("err-hkv0", qs, [8, 16, 0, 64], bts=bts)
    kv("err-out-shape", qs, kcs, bts=bts, outs=[2, 4, 2, 64])
    kv("err-page0", qs, [8, 0, 2, 64], bts=bts)
    kv("err-bt-batch", qs, kcs, bts=[3, 4])
    kv("err-bt-empty", qs, kcs, bts=[2, 0])
    kv("err-no-table-p", qs, kcs)
    kv("err-scale-inf", qs, kcs, bts=bts, scale=math.inf)
    kv("err-null-args", qs, kcs, bts=bts, null_args=True)
    for j, n in ((0, "q"), (1, "k-cache"), (2, "v-cache"), (4, "seqlens"), (5, "out")):
        ptrs = list(base)
        ptrs[j] = 0
        kv(f"err-null-{n}", qs, kcs, bts=bts, ptrs=ptrs)
    kv("err-lse-align", qs, kcs, bts=bts, lse=tk.LSE + 2)
    kv("err-seqlens-align", qs, kcs, bts=bts, ptrs=base[:4] + [tk.SL + 2, tk.OUT])
    kv("err-bt-align", qs, kcs, bts=bts, ptrs=base[:3] + [tk.BT + 2] + base[4:])
    kv("err-in-f32", qs, kcs, bts=bts, idt="f32", odt="f32")
    kv("err-in-i8", qs, kcs, bts=bts, idt="i8", odt="f32")
    kv("err-out-other", qs, kcs, bts=bts, idt="bf16", odt="f16")
    kv("err-d136", [2, 4, 1, 136], [8, 16, 2, 136], bts=bts)
    kv("err-d12", [2, 4, 1, 12], [8, 16, 2, 12], bts=bts)
    kv("err-dv", qs, kcs, bts=bts, vcs=[8, 16, 2, 32])
    kv("err-page24", qs, [8, 24, 2, 64], bts=bts)
    kv("err-page96", qs, [8, 96, 2, 64], bts=bts)
    kv("err-k-cache-misaligned", qs, kcs, bts=bts, ptrs=[tk.Q, tk.KC + 2] + base[2:])
    kv("err-v-cache-misaligned", qs, kcs, bts=bts, ptrs=[tk.Q, tk.KC, tk.VC + 2] + base[3:])
    kv("err-cache-d-stride", qs, kcs, bts=bts, strides=[None, [16 * 2 * 64, 1, 64 * 16, 16], None, None, None])
    kv("err-cache-odd-stride", qs, kcs, bts=bts, strides=[None, None, [16 * 2 * 68, 2 * 68, 68, 1], None, None])
    kv("err-out-misaligned", qs, kcs, bts=bts, ptrs=base[:5] + [tk.OUT + 2])
    kv("err-out-d-stride", qs, kcs, bts=bts, strides=[None, None, None, None, [4 * 64, 1, 4 * 64, 4]])
    kv("err-huge", qs, [8, 1 << 16, 2, 64], bts=[2, 1 << 15])
    for name, q_ in (("b0", [0, 4, 1, 64]), ("hq0", [2, 0, 1, 64]), ("sq0", [2, 4, 0, 64])):
        kv(f"empty-{name}", q_, kcs, bts=[q_[0], 4])
        kv(f"empty-{name}-null", q_, kcs, bts=[q_[0], 4], ptrs=[0, 0, 0, tk.BT, 0, 0], lse=2)
    kv("double-out-dtype-and-shape", qs, [8, 16, 3, 64], bts=bts, odt="f16")
    kv("double-empty-and-bt", [0, 4, 1, 64], kcs, bts=[2, 4])
    kv("double-null-and-cache-view", qs, kcs, bts=bts, ptrs=[0, tk.KC + 2] + base[2:])
    kv("double-out-and-cache-view", qs, kcs, bts=bts, ptrs=[tk.Q, tk.KC + 2] + base[2:5] + [tk.OUT + 2])

    # ------------------------------------------------------------------------------------------------ b200_kvcache_write
    kw_ = lambda name, kns, kcs, **kw: add(name, "kvwrite", kns, kcs, **kw)  # noqa: E731
    wbase = [tk.Q, tk.KC, tk.VC, tk.BT, tk.SL]   # k_new, k_cache, v_cache, v_new, slots
    for dt in ("bf16", "f16"):
        for D in (8, 64, 128):
            kw_(f"{dt}-d{D}", [2, 3, 4, D], [10, 16, 4, D], dt=dt)
    kw_("many", [64, 1, 8, 128], [4096, 16, 8, 128])
    st = [3 * 4 * 136, 4 * 136, 136, 1]
    kw_("padded-rows", [2, 3, 4, 128], [10, 16, 4, 128], strides=[st, st, None, None])
    hmc = [4 * 16 * 64, 64, 16 * 64, 1]
    kw_("head-major-cache", [2, 3, 4, 64], [10, 16, 4, 64], strides=[None, None, hmc, hmc])
    kw_("gather-k-new-misaligned", [2, 3, 4, 128], [10, 16, 4, 128], ptrs=[tk.Q + 2] + wbase[1:])
    kw_("gather-v-new-misaligned", [2, 3, 4, 128], [10, 16, 4, 128], ptrs=wbase[:3] + [tk.BT + 2, tk.SL])
    kw_("gather-k-new-d-stride", [2, 3, 4, 64], [10, 16, 4, 64], strides=[[3 * 4 * 64, 1, 3 * 64, 3], None, None, None])
    kw_("gather-v-new-odd-stride", [2, 3, 4, 64], [10, 16, 4, 64], strides=[None, [3 * 4 * 68, 4 * 68, 68, 1], None, None])
    kw_("gather-both-f16", [2, 3, 4, 64], [10, 16, 4, 64], dt="f16", ptrs=[tk.Q + 2, tk.KC, tk.VC, tk.BT + 2, tk.SL])
    kns, kcs = [2, 3, 4, 64], [10, 16, 4, 64]
    kw_("err-v-new", kns, kcs, vns=[2, 4, 4, 64])
    kw_("err-v-cache", kns, kcs, vcs=[10, 32, 4, 64])
    kw_("err-heads", kns, [10, 16, 2, 64])
    kw_("err-head-dim", kns, [10, 16, 4, 32])
    for j, n in enumerate(("k-new", "k-cache", "v-cache", "v-new", "slots")):
        ptrs = list(wbase)
        ptrs[j] = 0
        kw_(f"err-null-{n}", kns, kcs, ptrs=ptrs)
    kw_("err-slots-align", kns, kcs, ptrs=wbase[:4] + [tk.SL + 2])
    kw_("err-dtype", kns, kcs, dt="f32")
    kw_("err-d12", [2, 3, 4, 12], [10, 16, 4, 12])
    kw_("err-k-cache-misaligned", kns, kcs, ptrs=[tk.Q, tk.KC + 2] + wbase[2:])
    kw_("err-v-cache-d-stride", kns, kcs, strides=[None, None, None, [16 * 4 * 64, 1, 64 * 16, 16]])
    kw_("empty-b0", [0, 3, 4, 64], kcs)
    kw_("empty-snew0-null", [2, 0, 4, 64], kcs, ptrs=[0, 0, 0, 0, 0])
    kw_("double-dtype-and-shape", kns, kcs, dt="f32", vns=[2, 4, 4, 64])
    kw_("double-empty-and-d12", [0, 3, 4, 12], [10, 16, 4, 12])

    # ------------------------------------------------------------------------------------------------ varlen forward
    vf = lambda name, qs, ks, B, mq, mk, **kw: add(name, "varlen", qs, ks, B, mq, mk, **kw)  # noqa: E731
    vbase = [tv.Q, tv.K, tv.V, tv.CUQ, tv.CUK, tv.OUT]
    for i, o, _ in dts[::2]:
        for D in Ds:
            vf(f"{i}-{o}-d{D}", [3000, 8, D], [2500, 2, D], 5, 1000, 700, idt=i, odt=o, window=[-1, 0] if D % 16 == 8 else [-1, -1])
    for mq, mk in ((1, 1), (127, 128), (128, 129), (129, 127), (256, 257)):
        for window in ([-1, -1], [-1, 0], [64, 0], [3, 5]):
            vf(f"edges-{mq}x{mk}-w{window[0]}_{window[1]}", [1000, 4, 64], [1100, 2, 64], 4, mq, mk, window=window)
    T, H, D = 256, 4, 64
    vfused = [3 * H * D, D, 1]
    vf("fused-qkv", [T, H, D], [T, H, D], 2, 128, 128, strides=[vfused, vfused, vfused, None],
       ptrs=[tv.Q, tv.Q + 2 * H * D, tv.Q + 4 * H * D, tv.CUQ, tv.CUK, tv.OUT])
    vf("head-major", [T, H, D], [T, H, D], 2, 128, 128, strides=[[D, T * D, 1], [D, T * D, 1], [D, T * D, 1], [D, T * D, 1]])
    vf("out-pitched-f32", [T, H, D], [T, H, D], 2, 128, 128, odt="f32", strides=[None, None, None, [H * 72, 72, 1]])
    for j, n in enumerate("qkv"):
        mis = list(vbase)
        mis[j] += 2
        vf(f"gather-{n}-misaligned", [T, H, D], [T, H, D], 2, 128, 128, ptrs=mis)
        st = [None] * 4
        st[j] = [H * D * 2, D * 2, 2]
        vf(f"gather-{n}-d-stride", [T, H, D], [T, H, D], 2, 128, 128, strides=st)
        st = [None] * 4
        st[j] = [H * 68, 68, 1]
        vf(f"gather-{n}-odd-stride", [T, H, D], [T, H, D], 2, 128, 128, strides=st)
    qs, ks, Bv = [300, 4, 64], [200, 2, 64], 3
    vf("err-head-dim", qs, [200, 2, 32], Bv, 128, 128)
    vf("err-v-shape", qs, ks, Bv, 128, 128, vs=[100, 2, 64])
    vf("err-gqa", qs, [200, 3, 64], Bv, 128, 128)
    vf("err-hkv0", qs, [200, 0, 64], Bv, 128, 128)
    vf("err-out-shape", qs, ks, Bv, 128, 128, outs=[300, 2, 64])
    vf("err-window-left", qs, ks, Bv, 128, 128, window=[-2, 0])
    vf("err-window-right", qs, ks, Bv, 128, 128, window=[4, -5])
    vf("err-max-neg", qs, ks, Bv, 128, -1)
    vf("err-scale-inf", qs, ks, Bv, 128, 128, scale=math.inf)
    vf("err-scale-nan", qs, ks, Bv, 128, 128, scale=math.nan)
    vf("err-null-args", qs, ks, Bv, 128, 128, null_args=True)
    for j, n in enumerate(("q", "k", "v", "cu-q", "cu-k", "out")):
        ptrs = list(vbase)
        ptrs[j] = 0
        vf(f"err-null-{n}", qs, ks, Bv, 128, 128, ptrs=ptrs)
    vf("err-cu-align", qs, ks, Bv, 128, 128, ptrs=vbase[:3] + [tv.CUQ + 2] + vbase[4:])
    vf("err-lse-align", qs, ks, Bv, 128, 128, lse=tv.LSE + 2)
    vf("err-in-f32", qs, ks, Bv, 128, 128, idt="f32", odt="f32")
    vf("err-in-i8", qs, ks, Bv, 128, 128, idt="i8", odt="f32")
    vf("err-out-other", qs, ks, Bv, 128, 128, idt="bf16", odt="f16")
    vf("err-d136", [300, 4, 136], [200, 2, 136], Bv, 128, 128)
    vf("err-d12", [300, 4, 12], [200, 2, 12], Bv, 128, 128)
    vf("err-dv", qs, ks, Bv, 128, 128, vs=[200, 2, 32])
    vf("err-out-misaligned", qs, ks, Bv, 128, 128, ptrs=vbase[:5] + [tv.OUT + 2])
    vf("err-out-d-stride", qs, ks, Bv, 128, 128, strides=[None, None, None, [4 * 64 * 2, 2, 4 * 64]])
    vf("err-huge", [BIG, 4, 64], ks, Bv, 128, 128)
    vf("err-huge-batch", qs, ks, BIG, 128, 128)
    vf("err-max-huge", qs, ks, Bv, 1 << 30, 128)
    vf("err-ctas", [1 << 20, 1 << 20, 64], [1 << 20, 1 << 20, 64], 1 << 20, 1 << 20, 128)
    for name, q_, b_, mq in (("b0", qs, 0, 128), ("tq0", [0, 4, 64], Bv, 128), ("hq0", [300, 0, 64], Bv, 128), ("maxq0", qs, Bv, 0)):
        vf(f"empty-{name}", q_, ks, b_, mq, 128)
        vf(f"empty-{name}-null", q_, ks, b_, mq, 128, ptrs=[0] * 6, lse=3)
    vf("double-out-dtype-and-shape", qs, ks, Bv, 128, 128, odt="f16", outs=[300, 2, 64])
    vf("double-out-dtype-and-head-dim", [300, 4, 12], [200, 2, 12], Bv, 128, 128, odt="f16")
    vf("double-in-dtype-and-shape", qs, [200, 3, 64], Bv, 128, 128, idt="f32", odt="f32")
    vf("double-window-and-scale", qs, ks, Bv, 128, 128, window=[-2, 0], scale=math.nan)
    vf("double-null-and-out-view", qs, ks, Bv, 128, 128, ptrs=[0] + vbase[1:5] + [tv.OUT + 2])

    # ------------------------------------------------------------------------------------------------ varlen backward
    vb = lambda name, qs, ks, B, mq, mk, **kw: add(name, "varlen_bwd", qs, ks, B, mq, mk, **kw)  # noqa: E731
    bb = [tv.Q, tv.K, tv.V, tv.OUT, tv.DOUT, tv.LSE, tv.CUQ, tv.CUK, tv.DQ, tv.DK, tv.DV]
    for i, o, g in dts:
        for D in Ds:
            vb(f"{i}-{o}-{g}-d{D}", [3000, 8, D], [2500, 2, D], 5, 1000, 700, idt=i, odt=o, gdt=g,
               window=[-1, 0] if D % 16 == 8 else [-1, -1])
    for mq, mk in ((1, 1), (127, 128), (128, 129), (129, 127), (256, 257)):
        for window in ([-1, -1], [-1, 0], [3, 5]):
            vb(f"edges-{mq}x{mk}-w{window[0]}_{window[1]}", [1000, 4, 64], [1100, 2, 64], 4, mq, mk, window=window)
    vb("fused-qkv", [T, H, D], [T, H, D], 2, 128, 128, strides=[vfused, vfused, vfused, None, None, vfused, vfused, vfused],
       ptrs=[tv.Q, tv.Q + 2 * H * D, tv.Q + 4 * H * D] + bb[3:8] + [tv.DQ, tv.DQ + 2 * H * D, tv.DQ + 4 * H * D])
    vb("head-major", [T, H, D], [T, H, D], 2, 128, 128, strides=[[D, T * D, 1]] * 8)
    vb("pitched-f32", [T, H, D], [T, H, D], 2, 128, 128, odt="f32", gdt="f32", strides=[None, None, None, [H * 72, 72, 1],
                                                                                       [H * 72, 72, 1], [H * 72, 72, 1],
                                                                                       [H * 80, 80, 1], [H * 80, 80, 1]])
    for j, n in enumerate(("q", "k", "v", "out", "dout")):
        for odt in (None, "f32") if n == "out" else (None,):
            tag = f"gather-{n}" + ("-f32" if odt else "")
            mis = list(bb)
            mis[j] += 8 if odt else 2
            vb(f"{tag}-misaligned", [T, H, D], [T, H, D], 2, 128, 128, odt=odt, ptrs=mis)
            st = [None] * 8
            st[j] = [H * D * 2, D * 2, 2]
            vb(f"{tag}-d-stride", [T, H, D], [T, H, D], 2, 128, 128, odt=odt, strides=st)
            st = [None] * 8
            st[j] = [H * (66 if odt else 68), 66 if odt else 68, 1]
            vb(f"{tag}-odd-stride", [T, H, D], [T, H, D], 2, 128, 128, odt=odt, strides=st)
    vb("gather-all-f16", [T, H, 40], [200, 2, 40], 2, 128, 128, idt="f16", odt="f32", gdt="f32",
       ptrs=[tv.Q + 2, tv.K + 2, tv.V + 2, tv.OUT + 4, tv.DOUT + 2] + bb[5:])
    qs, ks = [300, 4, 64], [200, 2, 64]
    vb("err-head-dim", qs, [200, 2, 32], Bv, 128, 128)
    vb("err-v-shape", qs, ks, Bv, 128, 128, shapes={"v": [100, 2, 64]})
    vb("err-gqa", qs, [200, 3, 64], Bv, 128, 128)
    vb("err-hkv0", qs, [200, 0, 64], Bv, 128, 128)
    for n in ("out", "dout", "dq"):
        vb(f"err-{n}-shape", qs, ks, Bv, 128, 128, shapes={n: [300, 4, 32]})
    for n in ("dk", "dv"):
        vb(f"err-{n}-shape", qs, ks, Bv, 128, 128, shapes={n: [201, 2, 64]})
    vb("err-window", qs, ks, Bv, 128, 128, window=[-3, -1])
    vb("err-max-neg", qs, ks, Bv, -1, 128)
    vb("err-scale-inf", qs, ks, Bv, 128, 128, scale=math.inf)
    for j, n in enumerate(("q", "k", "v", "out", "dout", "lse", "cu-q", "cu-k", "dq", "dk", "dv")):
        ptrs = list(bb)
        ptrs[j] = 0
        vb(f"err-null-{n}", qs, ks, Bv, 128, 128, ptrs=ptrs)
    vb("err-lse-align", qs, ks, Bv, 128, 128, ptrs=bb[:5] + [tv.LSE + 2] + bb[6:])
    vb("err-cu-k-align", qs, ks, Bv, 128, 128, ptrs=bb[:7] + [tv.CUK + 2] + bb[8:])
    vb("err-in-f32", qs, ks, Bv, 128, 128, idt="f32", odt="f32", gdt="f32")
    vb("err-out-other", qs, ks, Bv, 128, 128, odt="f16")
    vb("err-grad-other", qs, ks, Bv, 128, 128, gdt="f16")
    vb("err-d136", [300, 4, 136], [200, 2, 136], Bv, 128, 128)
    vb("err-dv-dim", qs, ks, Bv, 128, 128, shapes={"v": [200, 2, 32]})
    vb("err-dq-d-stride", qs, ks, Bv, 128, 128, strides=[None] * 5 + [[4 * 64 * 2, 2, 4 * 64], None, None])
    vb("err-dk-misaligned", qs, ks, Bv, 128, 128, ptrs=bb[:9] + [tv.DK + 2, tv.DV])
    vb("err-dv-odd-stride", qs, ks, Bv, 128, 128, strides=[None] * 7 + [[2 * 68, 68, 1]])
    vb("err-huge", [BIG, 4, 64], ks, Bv, 128, 128)
    vb("err-max-huge", qs, ks, Bv, 128, 1 << 30)
    vb("err-ctas", [1 << 20, 1 << 20, 64], [1 << 20, 1 << 20, 64], 1 << 20, 1 << 20, 128)
    vb("err-ctas-k", [1 << 20, 1 << 20, 64], [1 << 20, 1 << 20, 64], 1 << 20, 0, 1 << 20)
    for name, q_, k_, b_, mq, mk in (("b0", qs, ks, 0, 128, 128), ("tq0-tk0", [0, 4, 64], [0, 2, 64], Bv, 0, 0),
                                     ("maxq0-maxk0", qs, ks, Bv, 0, 0), ("tq0", [0, 4, 64], ks, Bv, 0, 128),
                                     ("maxq0", qs, ks, Bv, 0, 128), ("hq0", [300, 0, 64], ks, Bv, 128, 128),
                                     ("tk0", qs, [0, 2, 64], Bv, 128, 0), ("maxk0", qs, ks, Bv, 128, 0)):
        vb(f"empty-{name}", q_, k_, b_, mq, mk)
        vb(f"empty-{name}-null-q-side", q_, k_, b_, mq, mk, ptrs=[0, tv.K, tv.V, 0, 0, 0, tv.CUQ, tv.CUK, 0, tv.DK, tv.DV])
        vb(f"empty-{name}-null-k-side", q_, k_, b_, mq, mk, ptrs=[tv.Q, 0, 0, tv.OUT, tv.DOUT, tv.LSE, tv.CUQ, tv.CUK, tv.DQ, 0, 0])
    vb("empty-tk0-dk-misaligned", qs, [0, 2, 64], Bv, 128, 0, ptrs=bb[:9] + [tv.DK + 2, tv.DV])
    vb("empty-tq0-dq-misaligned", [0, 4, 64], ks, Bv, 0, 128, ptrs=bb[:8] + [tv.DQ + 2, tv.DK, tv.DV])
    vb("empty-tk0-k-gathered-not", qs, [0, 2, 64], Bv, 128, 0, ptrs=[tv.Q, tv.K + 2, tv.V + 2] + bb[3:])
    vb("empty-tq0-q-gathered-not", [0, 4, 64], ks, Bv, 0, 128, ptrs=[tv.Q + 2, tv.K, tv.V, tv.OUT + 2, tv.DOUT + 2] + bb[5:])
    vb("empty-both-null-cu", [0, 4, 64], [0, 2, 64], Bv, 0, 0, ptrs=[0] * 11)
    vb("double-shape-and-out-dtype", qs, ks, Bv, 128, 128, odt="f16", shapes={"dq": [300, 4, 32]})
    vb("double-head-dim-and-grad-dtype", qs, [200, 2, 32], Bv, 128, 128, gdt="f16", shapes={})
    vb("double-null-and-grad-view", qs, ks, Bv, 128, 128, ptrs=[0] + bb[1:9] + [tv.DK + 2, tv.DV])
    vb("double-tk0-null-and-lse", qs, [0, 2, 64], Bv, 128, 0, ptrs=[tv.Q, 0, 0, tv.OUT, tv.DOUT, tv.LSE + 2] + bb[6:])
    return out


def main() -> None:
    rows = []
    seen = set()
    for cid, c in cases():
        assert cid not in seen, cid
        seen.add(cid)
        rows.append({"id": cid, "call": c, **replay(c)})
    # gzip without a timestamp: the same cases always give the same bytes
    text = json.dumps({"_generated_by": "tests/golden/make_attention_plan_golden.py", "cases": rows}, indent=0) + "\n"
    GOLDEN.write_bytes(gzip.compress(text.encode(), mtime=0))
    fails = sum(1 for r in rows if r["status"])
    print(f"wrote {GOLDEN}: {len(rows)} cases, {fails} failing, {GOLDEN.stat().st_size // 1024} KB")


if __name__ == "__main__":
    main()
