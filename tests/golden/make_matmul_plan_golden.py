"""Record the dry-run plans of the matmul entry points into matmul_plan_golden.json.gz (read by
tests/test_matmul_plan_golden_cpu.py).

    python tests/golden/make_matmul_plan_golden.py

Each case is one call of b200_matmul, b200_matmul_fused, b200_matmul_mixed, b200_matmul_scaled, b200_matmul_quantized,
b200_matmul_quantized_fp8, b200_matmul_grouped or b200_matmul_grouped_quantized_fp8 in a fresh planning context
(b200_plan_begin, 132 SMs); the fixture stores the call, the returned status, the full error message and the full plan text.
The cases cover every input dtype with every output dtype, the f32 modes, all four operand majors, batch broadcasts that
collapse and that peel, unit and empty extents, pitched and misaligned operands on the staging and the SIMT paths, every
gemm.variant / split_k / epilogue value, output strides with and without TMA stores, the epilogue fields, block-scaled,
integer-quantized and fp8-quantized operands (e4m3 / e5m2 per side, every block size, block-scale dtype and level, staged
codes), both grouped modes with all operand layouts, the fp8 grouped matmul's group counts, tile threshold and empty extents,
and one case per refusal, with a few calls where two checks fail at once.  Plans hold no pointer bases and no kernel parameter blocks, so those
are left to the GPU tests.
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

GOLDEN = Path(__file__).resolve().parent / "matmul_plan_golden.json.gz"
DT = {"f32": _ffi.F32, "f16": _ffi.F16, "bf16": _ffi.BF16, "i32": _ffi.I32, "u8": _ffi.U8, "i8": _ffi.I8, "e4m3": _ffi.F8E4M3,
      "e5m2": _ffi.F8E5M2, "e2m1x2": _ffi.F4E2M1X2, "ue8m0": _ffi.UE8M0}
QV = {"q8f": _ffi.QV_Q8F, "q8s": _ffi.QV_Q8S, "q4f": _ffi.QV_Q4F, "q4s": _ffi.QV_Q4S, "q2f": _ffi.QV_Q2F, "q2s": _ffi.QV_Q2S,
      "e4m3": _ffi.QV_E4M3, "e5m2": _ffi.QV_E5M2, "e2m1": _ffi.QV_E2M1, "bogus": 99}

A, B, O, S1, S2, OFFS, BIAS = 0x10000000, 0x20000000, 0x30000000, 0x40000000, 0x48000000, 0x50000000, 0x60000000
BIG = 1 << 31


def _arg(v):
    """A recorded argument: an int, None, a dtype name, {"u64": [...]}, {"ep": [alpha, activation, bias]} or
    {"q": [value, block, block_scale, tensor_scale, values, block_scales, tensor_scale ptr]}."""
    if isinstance(v, str):
        return DT[v]
    if isinstance(v, dict) and "u64" in v:
        return _ffi.u64_array(v["u64"])
    if isinstance(v, dict) and "ep" in v:
        return C.byref(_ffi.Epilogue(*v["ep"]))
    if isinstance(v, dict) and "q" in v:
        q = v["q"]
        return C.byref(_ffi.QuantOperand(_ffi.QuantScheme(QV[q[0]], q[1], DT.get(q[2], 0) if isinstance(q[2], str) else q[2], q[3]),
                                         q[4], q[5], q[6]))
    return v


def replay(call: dict) -> dict:
    """One recorded call in a fresh dry-run context (132 SMs): {status, error (the full message, "" on success), plan}."""
    with PlanContext(132, call["options"]) as p:
        rc = getattr(p.lib, call["fn"])(p.ctx, None, *[_arg(a) for a in call["args"]])
        err = ""
        if rc:
            msg = p.lib.b200_last_error()
            err = msg.decode() if msg else ""
        return {"status": rc, "error": err, "plan": p.text()}


def u64(v):
    return None if v is None else {"u64": list(v)}


def compact(s):
    out, inner = [], 1
    for e in reversed(s):
        out.append(inner)
        inner *= e
    return out[::-1]


# ---------------------------------------------------------------------------------------------------- b200_matmul family
def mm(M, N, K, idt="bf16", odt="f32", batch=(), lb=None, rb=None, a_major="k", b_major="n", a_pitch=0, b_pitch=0, o_pitch=0,
       a=A, b=B, o=O, ls=None, rs=None, os_=None, ep=None, rdt=None, options=None, fn=None):
    """The recorded arguments of one b200_matmul-family call: lhs [*lb, M, K], rhs [*rb, K, N], out [*batch, M, N].  a_major
    "k" = rows of K (K-contiguous), "m" = M-contiguous; b_major "n" = N-contiguous, "k" = K-contiguous.  *_pitch widens the
    leading dimension of the contiguous layout; ls / rs / os_ override the strides."""
    batch = list(batch)
    lb = batch if lb is None else list(lb)
    rb = batch if rb is None else list(rb)

    def full(bshape, rows, cols, row_major, pitch):
        inner = (cols if row_major else rows) + pitch
        plane = (rows if row_major else cols) * inner
        bs = compact(list(bshape) + [1])[:-1]
        return [x * plane for x in bs] + ([inner, 1] if row_major else [1, inner])

    lsh, rsh, osh = lb + [M, K], rb + [K, N], batch + [M, N]
    ls = ls or full(lb, M, K, a_major == "k", a_pitch)
    rs = rs or full(rb, K, N, b_major == "n", b_pitch)
    os_ = os_ or full(batch, M, N, True, o_pitch)
    rank = len(osh)
    tail = [o, rank, u64(lsh), u64(ls), u64(rsh), u64(rs), u64(osh), u64(os_)]
    if fn is None:
        fn = "b200_matmul_fused" if ep is not None else "b200_matmul_mixed" if rdt is not None else "b200_matmul"
    if fn == "b200_matmul_mixed":
        args = [idt, rdt, odt, a, b] + tail
    else:
        args = [idt, odt, a, b] + tail + ([ep] if fn == "b200_matmul_fused" else [])
    return {"fn": fn, "args": args, "options": options or {}}


def scaled(M, N, K, ldt="e4m3", rdt="e4m3", odt="f32", batch=1, block=32, packed=0, a=A, b=B, sa=S1, sb=S2, o=O, options=None):
    return {"fn": "b200_matmul_scaled", "args": [ldt, rdt, odt, a, b, sa, sb, o, batch, M, N, K, block, packed], "options": options or {}}


def qop(value="q8s", block=32, block_scale="f32", tensor=0, values=A, bs=S1, ts=0):
    return {"q": [value, block, block_scale, tensor, values, bs, ts]}


def qmm(lhs, rhs, M, N, K, odt="f32", batch=1, o=O, options=None):
    return {"fn": "b200_matmul_quantized", "args": [lhs, rhs, odt, o, batch, M, N, K], "options": options or {}}


def qf8(lhs, rhs, M, N, K, odt="bf16", batch=1, o=O, options=None):
    return {"fn": "b200_matmul_quantized_fp8", "args": [lhs, rhs, odt, o, batch, M, N, K], "options": options or {}}


def gqf8(lhs, rhs, G, T, N, K, odt="bf16", o=O, offs=OFFS, options=None):
    """b200_matmul_grouped_quantized_fp8: lhs codes [T, K] x rhs codes [G, N, K] -> out [T, N]."""
    return {"fn": "b200_matmul_grouped_quantized_fp8", "args": [lhs, rhs, offs, G, odt, o, T, N, K], "options": options or {}}


def grouped(mode, T, G, K=None, N=64, M=None, idt="bf16", odt="bf16", a_major=None, b_major=None, a_pitch=0, b_pitch=0, o_pitch=0,
            a=A, b=B, o=O, offs=OFFS, ep=None, options=None, shapes=None, strides=None, ranks=None):
    """b200_matmul_grouped.  Ragged M ("m"): lhs [T, K] x rhs [G, K, N] -> out [T, N]; a_major "k" (rows of K) or "m"
    (T-contiguous), b_major "n" (N-contiguous) or "k".  Ragged K ("k"): lhs [M, T] x rhs [T, N] -> out [G, M, N]; a_major "m"
    (M-contiguous) or "k", b_major "n" or "k"."""
    if mode == "m":
        a_major, b_major = a_major or "k", b_major or "n"
        lsh, rsh, osh = [T, K], [G, K, N], [T, N]
        ls = [K + a_pitch, 1] if a_major == "k" else [1, T + a_pitch]
        rs = [K * (N + b_pitch), N + b_pitch, 1] if b_major == "n" else [N * (K + b_pitch), 1, K + b_pitch]
        os_ = [N + o_pitch, 1]
    else:
        a_major, b_major = a_major or "m", b_major or "n"
        lsh, rsh, osh = [M, T], [T, N], [G, M, N]
        ls = [1, M + a_pitch] if a_major == "m" else [T + a_pitch, 1]
        rs = [N + b_pitch, 1] if b_major == "n" else [1, T + b_pitch]
        os_ = [M * (N + o_pitch), N + o_pitch, 1]
    if shapes:
        lsh, rsh, osh = shapes
    if strides:
        ls, rs, os_ = strides
    lr, rr, orr = ranks or (len(lsh), len(rsh), len(osh))
    args = [idt, odt, a, lr, u64(lsh), u64(ls), b, rr, u64(rsh), u64(rs), offs, G, o, orr, u64(osh), u64(os_), ep]
    return {"fn": "b200_matmul_grouped", "args": args, "options": options or {}}


def cases():
    out = []

    def add(name, c):
        out.append((name, c))

    # ---- b200_matmul: every input dtype x every output dtype, at a tensor-core shape and a SIMT-sized one
    outs = ("f32", "f16", "bf16", "i32", "u8")
    for idt in ("f32", "f16", "bf16", "e4m3", "e5m2", "u8", "i8"):
        for odt in outs:
            for shp in ((256, 256, 256), (512, 384, 192), (20, 24, 40)):
                if idt == "f32":
                    for mode in ("hybrid", "3xtf32", "tf32", "bogus"):
                        add(f"mm-{idt}-{odt}-{shp}-f32={mode}", mm(*shp, idt, odt, options={"gemm.f32": mode}))
                else:
                    add(f"mm-{idt}-{odt}-{shp}", mm(*shp, idt, odt))
    # ---- majors, per dtype class
    for idt, odt in (("bf16", "bf16"), ("f16", "f32"), ("f32", "f32"), ("e4m3", "bf16"), ("i8", "i32"), ("u8", "i32")):
        for am in ("k", "m"):
            for bm in ("n", "k"):
                for shp in ((1024, 768, 512), (384, 130, 72)):
                    add(f"major-{idt}-{am}{bm}-{shp}", mm(*shp, idt, odt, a_major=am, b_major=bm))
                    if idt == "f32":
                        add(f"major-{idt}-{am}{bm}-{shp}-3xtf32", mm(*shp, idt, odt, a_major=am, b_major=bm, options={"gemm.f32": "3xtf32"}))
    # ---- batches: collapse, broadcast, peel
    for idt, odt in (("bf16", "f32"), ("f32", "f32"), ("i8", "i32")):
        add(f"batch-collapse-{idt}", mm(256, 256, 128, idt, odt, batch=(2, 3)))
        add(f"batch-bcast-lhs-{idt}", mm(256, 256, 128, idt, odt, batch=(4,), lb=(1,)))
        add(f"batch-bcast-rhs-{idt}", mm(256, 256, 128, idt, odt, batch=(4,), rb=(1,)))
        add(f"batch-bcast-both-{idt}", mm(256, 256, 128, idt, odt, batch=(2, 3), lb=(2, 1), rb=(1, 3)))
        add(f"batch-bcast-inner-{idt}", mm(256, 256, 128, idt, odt, batch=(2, 3), lb=(1, 3), rb=(2, 1)))
        add(f"batch-unit-{idt}", mm(256, 256, 128, idt, odt, batch=(1, 1)))
        add(f"batch-rank8-{idt}", mm(64, 64, 64, idt, odt, batch=(1, 2, 1, 2, 1, 2)))
        # peel: lhs batch dims permuted, so its offsets are not linear in the flat batch index
        add(f"batch-peel-{idt}", mm(256, 128, 128, idt, odt, batch=(2, 3), ls=[256 * 128, 2 * 256 * 128, 128, 1]))
        add(f"batch-peel-out-{idt}", mm(256, 256, 128, idt, odt, batch=(2, 3), os_=[256 * 256, 2 * 256 * 256, 256, 1]))
        add(f"batch-peel-3-{idt}", mm(128, 128, 64, idt, odt, batch=(2, 2, 2), ls=[64 * 128, 4 * 64 * 128, 2 * 64 * 128, 64, 1]))
        add(f"batch-0-{idt}", mm(256, 256, 128, idt, odt, batch=(0, 3)))
        add(f"batch-0-bcast-{idt}", mm(256, 256, 128, idt, odt, batch=(0,), lb=(0,), rb=(1,)))
    for mode in ("3xtf32", "tf32"):
        opts = {"gemm.f32": mode}
        add(f"batch-collapse-f32-{mode}", mm(256, 256, 128, "f32", "f32", batch=(2, 3), options=opts))
        add(f"batch-bcast-lhs-f32-{mode}", mm(256, 256, 128, "f32", "f32", batch=(4,), lb=(1,), options=opts))
        add(f"batch-bcast-rhs-f32-{mode}", mm(256, 256, 128, "f32", "f32", batch=(4,), rb=(1,), options=opts))
        add(f"batch-m1-f32-{mode}", mm(1, 256, 130, "f32", "f32", batch=(3,), options=opts))
        add(f"batch-n1-f32-{mode}", mm(256, 1, 130, "f32", "f32", batch=(3,), rb=(1,), options=opts))
    # ---- unit and empty extents
    for idt, odt in (("bf16", "f32"), ("f16", "f16"), ("f32", "f32"), ("e5m2", "f32"), ("u8", "i32")):
        for shp in ((1, 512, 256), (512, 1, 256), (512, 384, 1), (1, 1, 1), (512, 384, 0), (0, 384, 64), (512, 0, 64), (1, 1, 4096),
                    (4096, 1, 4096), (1, 4096, 4096)):
            add(f"extent-{idt}-{shp}", mm(*shp, idt, odt))
            if shp[2] == 1 or shp[0] == 1:
                add(f"extent-{idt}-{shp}-mn", mm(*shp, idt, odt, a_major="m", b_major="k"))
        add(f"extent-{idt}-nullptr-empty", mm(0, 384, 64, idt, odt, a=0))
        add(f"extent-{idt}-nullptr", mm(16, 384, 64, idt, odt, a=0))
        add(f"extent-{idt}-nullptr-out", mm(16, 384, 64, idt, odt, o=0))
    # ---- pitched and misaligned operands: staging (big) and SIMT (small), gemm.stage on / off
    for idt, odt in (("bf16", "f32"), ("f16", "f16"), ("f32", "f32"), ("e4m3", "f32"), ("i8", "i32")):
        for stage in ("on", "off"):
            opts = {"gemm.stage": stage}
            for shp in ((1024, 512, 513), (64, 48, 40)):
                tag = f"{idt}-{shp}-stage={stage}"
                add(f"pitch-a-{tag}", mm(*shp, idt, odt, a_pitch=3, options=opts))
                add(f"pitch-b-{tag}", mm(*shp, idt, odt, b_pitch=1, options=opts))
                add(f"pitch-a-m-{tag}", mm(*shp, idt, odt, a_major="m", a_pitch=5, options=opts))
                add(f"pitch-b-k-{tag}", mm(*shp, idt, odt, b_major="k", b_pitch=7, options=opts))
                add(f"misaligned-a-{tag}", mm(*shp, idt, odt, a=A + 2, options=opts))
                add(f"misaligned-b-{tag}", mm(*shp, idt, odt, b=B + 4, options=opts))
                add(f"strided-k-{tag}", mm(*shp, idt, odt, ls=[2 * shp[2], 2], options=opts))
                add(f"batch-pitch-{tag}", mm(*shp, idt, odt, batch=(3,), ls=[shp[0] * shp[2] + 8, shp[2], 1], options=opts))
    # ---- gemm.variant
    for tag in ("auto", "2sm_n256", "2sm_n128", "1sm_n128", "2sm_m512", "2sm_n224", "simt", "bogus"):
        opts = {"gemm.variant": tag}
        for idt, odt in (("bf16", "bf16"), ("f16", "f32"), ("f32", "f32"), ("e4m3", "f32"), ("i8", "i32")):
            add(f"variant-{tag}-{idt}", mm(2048, 1536, 1024, idt, odt, options=opts))
            add(f"variant-{tag}-{idt}-small", mm(100, 72, 40, idt, odt, options=opts))
            add(f"variant-{tag}-{idt}-pitched", mm(1024, 512, 513, idt, odt, a_pitch=3, options=opts))
        add(f"variant-{tag}-bf16-mn", mm(2048, 1536, 1024, "bf16", "f32", a_major="m", b_major="k", options=opts))
        add(f"variant-{tag}-bf16-m128", mm(128, 4096, 1024, "bf16", "f32", options=opts))
        add(f"variant-{tag}-bf16-batch", mm(512, 512, 256, "bf16", "f32", batch=(5,), options=opts))
        add(f"variant-{tag}-ep", mm(2048, 1536, 1024, "bf16", "bf16", ep={"ep": [0.5, 1, BIAS]}, options=opts))
    # ---- gemm.split_k on shapes with and without a stream-K head
    for val in ("auto", "off", "on", "1", "2", "3", "4", "5", "6", "7", "8", "0", "9", "bogus"):
        opts = {"gemm.split_k": val}
        for name, shp, idt, odt in (("rem", (4096, 4096, 4096), "bf16", "bf16"), ("full", (8448, 4096, 1024), "bf16", "f32"),
                                    ("few", (512, 512, 8192), "bf16", "f32"), ("one-kb", (4096, 4096, 64), "bf16", "bf16"),
                                    ("f32", (2048, 2048, 2048), "f32", "f32"), ("int", (4096, 4096, 4096), "i8", "i32"),
                                    ("m512", (4096, 4096, 4096), "bf16", "bf16")):
            o2 = dict(opts, **({"gemm.variant": "2sm_m512"} if name == "m512" else {}))
            add(f"splitk-{val}-{name}", mm(*shp, idt, odt, options=o2))
        add(f"splitk-{val}-n128", mm(3000, 3000, 4096, "f16", "f32", options=dict(opts, **{"gemm.variant": "1sm_n128"})))
    # ---- gemm.epilogue and output strides
    for epi in ("tma", "direct", "bogus"):
        opts = {"gemm.epilogue": epi}
        for idt, odt in (("bf16", "bf16"), ("bf16", "f32"), ("f32", "f32"), ("i8", "i32")):
            add(f"epi-{epi}-{idt}-{odt}", mm(1024, 1024, 512, idt, odt, options=opts))
            add(f"epi-{epi}-{idt}-{odt}-opitch8", mm(1024, 1024, 512, idt, odt, o_pitch=8, options=opts))
            add(f"epi-{epi}-{idt}-{odt}-opitch1", mm(1024, 1000, 512, idt, odt, o_pitch=1, options=opts))
            add(f"epi-{epi}-{idt}-{odt}-omisaligned", mm(1024, 1024, 512, idt, odt, o=O + 4, options=opts))
            add(f"epi-{epi}-{idt}-{odt}-m1", mm(1, 1024, 512, idt, odt, options=opts))
            add(f"epi-{epi}-{idt}-{odt}-n1", mm(1024, 1, 512, idt, odt, options=opts))
            add(f"epi-{epi}-{idt}-{odt}-batch", mm(512, 512, 256, idt, odt, batch=(3,), options=opts))
            add(f"epi-{epi}-{idt}-{odt}-batch-gap", mm(512, 512, 256, idt, odt, batch=(3,), os_=[512 * 512 + 8, 512, 1], options=opts))
            add(f"epi-{epi}-{idt}-{odt}-transposed-out", mm(1024, 1024, 512, idt, odt, os_=[1, 1024], options=opts))
            add(f"epi-{epi}-{idt}-{odt}-overlap-rows", mm(1024, 1024, 512, idt, odt, os_=[512, 1], options=opts))
            add(f"epi-{epi}-{idt}-{odt}-row-2^40", mm(4, 1024, 512, idt, odt, os_=[1 << 40, 1], options=opts))
            add(f"epi-{epi}-{idt}-{odt}-batch-2^40", mm(512, 512, 256, idt, odt, batch=(2,), os_=[1 << 40, 512, 1], options=opts))
    # ---- too many tiles, extent refusals
    for idt, odt in (("bf16", "f32"), ("f32", "f32"), ("i8", "i32")):
        add(f"tiles-2^32-{idt}", mm(1 << 30, 1 << 30, 64, idt, odt))
        add(f"tiles-2^32-batch-{idt}", mm(1 << 20, 1 << 20, 64, idt, odt, batch=(1 << 10,)))
        add(f"extent-m-2^31-{idt}", mm(BIG, 64, 64, idt, odt))
        add(f"extent-m-2^32-{idt}", mm(1 << 32, 64, 64, idt, odt))
        add(f"extent-k-2^32-{idt}", mm(64, 64, 1 << 32, idt, odt))
        add(f"extent-batch-65536-{idt}", mm(16, 16, 16, idt, odt, batch=(65536,), os_=[256, 1, 16]))
        add(f"extent-batch-2^31-{idt}", mm(64, 64, 64, idt, odt, batch=(BIG,)))
        add(f"extent-batch-2^31-simt-{idt}", mm(64, 64, 64, idt, odt, batch=(BIG,), options={"gemm.variant": "simt"}))
    # ---- b200_matmul refusals and double faults
    add("err-rank1", {"fn": "b200_matmul", "args": ["bf16", "f32", A, B, O, 1, u64([4]), u64([1]), u64([4]), u64([1]), u64([4]), u64([1])], "options": {}})
    add("err-rank9", mm(4, 4, 4, batch=(1,) * 7))
    add("err-null-shape", {"fn": "b200_matmul", "args": ["bf16", "f32", A, B, O, 2, None, u64([4, 1]), u64([4, 4]), u64([4, 1]), u64([4, 4]), u64([4, 1])], "options": {}})
    add("err-null-strides", {"fn": "b200_matmul", "args": ["bf16", "f32", A, B, O, 2, u64([4, 4]), u64([4, 1]), u64([4, 4]), u64([4, 1]), u64([4, 4]), None], "options": {}})
    add("err-idt-f64", {"fn": "b200_matmul", "args": [_ffi.F64, _ffi.F64] + mm(4, 4, 4)["args"][2:], "options": {}})
    add("err-idt-e2m1", mm(64, 64, 64, "e2m1x2", "f32"))
    def with_arg(c, i, v):
        c["args"][i] = v
        return c

    add("err-inner", with_arg(mm(64, 64, 64), 8, u64([65, 64])))
    add("err-out-shape", with_arg(mm(64, 64, 64), 10, u64([64, 63])))
    add("err-batch-mismatch", mm(64, 64, 64, batch=(3,), lb=(2,)))
    add("err-batch-out", mm(64, 64, 64, batch=(3,), lb=(1,), rb=(1,)))
    add("err-batch-0-vs-2", mm(64, 64, 64, batch=(0,), lb=(0,), rb=(2,)))
    add("err2-inner-and-dtype", with_arg(mm(64, 64, 64, "bf16", "f16"), 8, u64([65, 64])))
    add("err2-dtype-and-rank", mm(4, 4, 4, "e2m1x2", "f32", batch=(1,) * 7))
    add("err2-null-ptr-and-batch", mm(64, 64, 64, batch=(3,), lb=(2,), a=0))
    add("err2-variant-and-epilogue", mm(1024, 1024, 512, options={"gemm.variant": "bogus", "gemm.epilogue": "bogus"}))
    add("err2-splitk-and-epilogue", mm(4096, 4096, 4096, options={"gemm.split_k": "bogus", "gemm.epilogue": "bogus"}))
    add("err2-f32-and-variant", mm(1024, 1024, 512, "f32", "f32", options={"gemm.f32": "bogus", "gemm.variant": "bogus"}))
    add("err2-f32-and-splitk", mm(1024, 1024, 512, "f32", "f32", options={"gemm.f32": "bogus", "gemm.split_k": "bogus"}))
    add("err2-variant-simt-misaligned", mm(1024, 512, 513, a_pitch=3, options={"gemm.variant": "2sm_n128", "gemm.epilogue": "bogus"}))

    # ---- b200_matmul_fused: each epilogue field, each refusal
    for idt, odt in (("bf16", "bf16"), ("f16", "f32"), ("f32", "f32"), ("e4m3", "bf16"), ("e5m2", "f16")):
        for ep in ([1.0, 0, 0], [0.5, 0, 0], [1.0, 1, 0], [1.0, 2, 0], [1.0, 0, BIAS], [-2.0, 2, BIAS]):
            add(f"fused-{idt}-{odt}-{ep}", mm(1024, 768, 512, idt, odt, ep={"ep": ep}))
            add(f"fused-{idt}-{odt}-{ep}-simt", mm(40, 24, 16, idt, odt, ep={"ep": ep}))
        add(f"fused-{idt}-{odt}-batch", mm(512, 512, 256, idt, odt, batch=(2,), ep={"ep": [0.25, 1, BIAS]}))
        add(f"fused-{idt}-{odt}-splitk", mm(4096, 4096, 4096, idt, odt, ep={"ep": [1.0, 2, BIAS]}, options={"gemm.split_k": "on"}))
    add("fused-err-null-ep", with_arg(mm(64, 64, 64, ep={"ep": [1.0, 0, 0]}), -1, None))
    add("fused-err-act3", mm(64, 64, 64, ep={"ep": [1.0, 3, 0]}))
    add("fused-err-act-neg", mm(64, 64, 64, ep={"ep": [1.0, -1, 0]}))
    add("fused-err-u8", mm(64, 64, 64, "u8", "i32", ep={"ep": [1.0, 0, 0]}))
    add("fused-err-i8", mm(64, 64, 64, "i8", "i32", ep={"ep": [1.0, 0, 0]}))
    add("fused-err2-act-and-int", mm(64, 64, 64, "i8", "i32", ep={"ep": [1.0, 5, 0]}))
    add("fused-err2-int-and-shape", mm(64, 64, 64, "i8", "i32", ep={"ep": [1.0, 0, 0]}, batch=(3,), lb=(2,)))
    add("fused-err-dtype", mm(64, 64, 64, "bf16", "f16", ep={"ep": [1.0, 0, 0]}))

    # ---- b200_matmul_mixed
    for ldt, rdt, odt in (("e4m3", "e5m2", "f32"), ("e5m2", "e4m3", "bf16"), ("e4m3", "e4m3", "f16"), ("u8", "i8", "i32"),
                          ("i8", "u8", "i32"), ("u8", "u8", "i32"), ("bf16", "bf16", "f32"), ("e4m3", "i8", "f32"),
                          ("u8", "e5m2", "i32"), ("bf16", "f16", "f32"), ("u8", "i8", "f32"), ("e4m3", "e5m2", "i32")):
        for shp in ((1024, 768, 512), (40, 24, 16)):
            add(f"mixed-{ldt}-{rdt}-{odt}-{shp}", mm(*shp, ldt, odt, rdt=rdt, fn="b200_matmul_mixed"))
        add(f"mixed-{ldt}-{rdt}-{odt}-mn", mm(1024, 768, 512, ldt, odt, rdt=rdt, a_major="m", b_major="k", fn="b200_matmul_mixed"))
        add(f"mixed-{ldt}-{rdt}-{odt}-pitched", mm(1024, 768, 513, ldt, odt, rdt=rdt, a_pitch=3, fn="b200_matmul_mixed"))

    # ---- b200_matmul_scaled
    for ldt, rdt, block in (("e4m3", "e4m3", 32), ("e4m3", "e5m2", 32), ("e5m2", "e4m3", 32), ("e5m2", "e5m2", 32),
                            ("e2m1x2", "e2m1x2", 32), ("e2m1x2", "e2m1x2", 16)):
        for odt in ("f32", "bf16", "f16"):
            for packed in (0, 1):
                add(f"scaled-{ldt}-{rdt}-b{block}-{odt}-p{packed}", scaled(1024, 768, 512, ldt, rdt, odt, block=block, packed=packed))
        for packed in (0, 1):
            tag = f"{ldt}-{rdt}-b{block}-p{packed}"
            add(f"scaled-{tag}-batch", scaled(256, 256, 256, ldt, rdt, batch=3, block=block, packed=packed))
            add(f"scaled-{tag}-small", scaled(16, 8, 32, ldt, rdt, block=block, packed=packed))
            add(f"scaled-{tag}-misaligned-a", scaled(256, 256, 256, ldt, rdt, block=block, packed=packed, a=A + 1))
            add(f"scaled-{tag}-misaligned-scales", scaled(256, 256, 256, ldt, rdt, block=block, packed=packed, sa=S1 + 1))
            add(f"scaled-{tag}-k48", scaled(256, 256, 96 if ldt == "e2m1x2" else 48, ldt, rdt, block=block, packed=packed))
            for tag2 in ("2sm_n224", "2sm_n256", "2sm_n128", "1sm_n128", "2sm_m512", "simt", "bogus"):
                add(f"scaled-{tag}-variant={tag2}", scaled(2048, 1792, 1024, ldt, rdt, block=block, packed=packed, options={"gemm.variant": tag2}))
            add(f"scaled-{tag}-splitk-on", scaled(4096, 4096, 4096, ldt, rdt, block=block, packed=packed, options={"gemm.split_k": "on"}))
            add(f"scaled-{tag}-epi-direct", scaled(1024, 768, 512, ldt, rdt, block=block, packed=packed, options={"gemm.epilogue": "direct"}))
            add(f"scaled-{tag}-epi-bogus", scaled(1024, 768, 512, ldt, rdt, block=block, packed=packed, options={"gemm.epilogue": "bogus"}))
    add("scaled-err-e4m3-e2m1", scaled(64, 64, 64, "e4m3", "e2m1x2"))
    add("scaled-err-bf16", scaled(64, 64, 64, "bf16", "bf16"))
    add("scaled-err-out-i32", scaled(64, 64, 64, odt="i32"))
    add("scaled-err-block16-fp8", scaled(64, 64, 64, block=16))
    add("scaled-err-block64", scaled(64, 64, 64, block=64))
    add("scaled-err-k0", scaled(64, 64, 0))
    add("scaled-err-k40", scaled(64, 64, 40))
    add("scaled-empty-m", scaled(0, 64, 64))
    add("scaled-empty-batch", scaled(64, 64, 64, batch=0))
    add("scaled-err-null-a", scaled(64, 64, 64, a=0))
    add("scaled-err-null-scales", scaled(64, 64, 64, sb=0))
    add("scaled-err-null-out", scaled(64, 64, 64, o=0))
    add("scaled-err-m-2^31", scaled(BIG, 64, 64))
    add("scaled-err-batch-2^20", scaled(64, 64, 64, batch=1 << 20))
    add("scaled-err-packed-misaligned", scaled(64, 64, 64, packed=1, a=A + 1))
    add("scaled-err-packed-simt", scaled(64, 64, 64, packed=1, options={"gemm.variant": "simt"}))
    add("scaled-err2-dtype-block", scaled(64, 64, 40, "bf16", "bf16", block=64))
    add("scaled-err2-block-k", scaled(64, 64, 40, block=64))
    add("scaled-err2-k-null", scaled(64, 64, 40, a=0))

    # ---- b200_matmul_quantized
    values = ("q8f", "q8s", "q4f", "q4s", "q2f", "q2s")
    for lv in values:
        for rv in values:
            add(f"qmm-tensor-{lv}-{rv}", qmm(qop(lv, 0, 0, 1, bs=0, ts=S2), qop(rv, 0, 0, 1, bs=0, ts=S2 + 4), 1024, 768, 512))
    for v in values:
        for blk in (32, 64, 128):
            for bsd in ("f32", "f16", "bf16", "ue8m0", "e4m3"):
                add(f"qmm-block-{v}-{blk}-{bsd}", qmm(qop(v, blk, bsd), qop(v, blk, bsd, bs=S2), 1024, 768, 512))
            add(f"qmm-twolevel-{v}-{blk}", qmm(qop(v, blk, "f16", 1, ts=S2), qop(v, blk, "e4m3", 1, bs=S2, ts=S2 + 4), 512, 512, 512))
    for lb, rb in ((32, 64), (128, 32), (64, 128), (0, 32), (128, 0), (0, 64)):
        for odt in ("f32", "bf16", "f16"):
            lq = qop("q8s", lb, "f32", 0 if lb else 1, bs=S1 if lb else 0, ts=0 if lb else S2)
            rq = qop("q4s", rb, "bf16", 0 if rb else 1, bs=S2 if rb else 0, ts=0 if rb else S2 + 4)
            add(f"qmm-mixed-{lb}-{rb}-{odt}", qmm(lq, rq, 1024, 768, 512, odt))
            add(f"qmm-mixed-{lb}-{rb}-{odt}-batch", qmm(lq, rq, 256, 256, 256, odt, batch=3))
    for opts in ({"gemm.variant": "2sm_n256"}, {"gemm.variant": "2sm_n128"}, {"gemm.variant": "1sm_n128"}, {"gemm.variant": "2sm_m512"},
                 {"gemm.variant": "simt"}, {"gemm.variant": "bogus"}, {"gemm.split_k": "on"}, {"gemm.split_k": "bogus"},
                 {"gemm.epilogue": "direct"}, {"gemm.epilogue": "bogus"}):
        tag = "-".join(f"{k.split('.')[1]}={v}" for k, v in opts.items())
        add(f"qmm-opt-{tag}-block", qmm(qop("q8s", 32), qop("q8s", 32, bs=S2), 4096, 4096, 4096, options=opts))
        add(f"qmm-opt-{tag}-tensor", qmm(qop("q8s", 0, 0, 1, bs=0, ts=S2), qop("q8s", 0, 0, 1, bs=0, ts=S2 + 4), 4096, 4096, 4096, options=opts))
    add("qmm-q8-misaligned", qmm(qop("q8s", 32, values=A + 8), qop("q8s", 32, bs=S2), 1024, 768, 512))
    add("qmm-q8-k-not-16", qmm(qop("q8s", 0, 0, 1, bs=0, ts=S2), qop("q8s", 0, 0, 1, bs=0, ts=S2 + 4), 256, 256, 200))
    add("qmm-small", qmm(qop("q8s", 32), qop("q2f", 32, bs=S2), 16, 8, 64))
    add("qmm-m1", qmm(qop("q4s", 64), qop("q4s", 64, bs=S2), 1, 4096, 4096))
    add("qmm-empty", qmm(qop("q8s", 32), qop("q8s", 32, bs=S2), 0, 64, 64))
    add("qmm-empty-batch", qmm(qop("q8s", 32), qop("q8s", 32, bs=S2), 64, 64, 64, batch=0))
    add("qmm-err-null-lhs", qmm(None, qop("q8s", 32, bs=S2), 64, 64, 64))
    add("qmm-err-e4m3", qmm(qop("e4m3", 32, "ue8m0"), qop("q8s", 32, bs=S2), 64, 64, 64))
    add("qmm-err-e2m1", qmm(qop("q8s", 32), qop("e2m1", 32, "ue8m0", bs=S2), 64, 64, 64))
    add("qmm-err-block16", qmm(qop("q8s", 16), qop("q8s", 16, bs=S2), 64, 64, 64))
    add("qmm-err-block8", qmm(qop("q8s", 32), qop("q8s", 8, bs=S2), 64, 64, 64))
    add("qmm-err-block256", qmm(qop("q8s", 256), qop("q8s", 32, bs=S2), 64, 64, 256))
    add("qmm-err-bad-value", qmm(qop("bogus", 32), qop("q8s", 32, bs=S2), 64, 64, 64))
    add("qmm-err-tensor-flag", qmm(qop("q8s", 32, tensor=2), qop("q8s", 32, bs=S2), 64, 64, 64))
    add("qmm-err-no-level", qmm(qop("q8s", 0, 0, 0, bs=0), qop("q8s", 32, bs=S2), 64, 64, 64))
    add("qmm-err-bad-scale-dtype", qmm(qop("q8s", 32, "i32"), qop("q8s", 32, bs=S2), 64, 64, 64))
    add("qmm-err-k-block", qmm(qop("q8s", 32), qop("q8s", 32, bs=S2), 64, 64, 48))
    add("qmm-err-null-block-scales", qmm(qop("q8s", 32, bs=0), qop("q8s", 32, bs=S2), 64, 64, 64))
    add("qmm-err-misaligned-scales", qmm(qop("q8s", 32, bs=S1 + 1), qop("q8s", 32, bs=S2), 64, 64, 64))
    add("qmm-err-out-i32", qmm(qop("q8s", 32), qop("q8s", 32, bs=S2), 64, 64, 64, "i32"))
    add("qmm-err-k0", qmm(qop("q8s", 32), qop("q8s", 32, bs=S2), 64, 64, 0))
    add("qmm-err-tensor-k-2^17", qmm(qop("q8s", 0, 0, 1, bs=0, ts=S2), qop("q8s", 0, 0, 1, bs=0, ts=S2 + 4), 64, 64, 1 << 17))
    add("qmm-block-k-2^17", qmm(qop("q8s", 128), qop("q8s", 128, bs=S2), 64, 64, 1 << 17))
    add("qmm-err-null-values", qmm(qop("q8s", 32, values=0), qop("q8s", 32, bs=S2), 64, 64, 64))
    add("qmm-err-null-out", qmm(qop("q8s", 32), qop("q8s", 32, bs=S2), 64, 64, 64, o=0))
    add("qmm-err-misaligned-out", qmm(qop("q8s", 32), qop("q8s", 32, bs=S2), 64, 64, 64, o=O + 2))
    add("qmm-err-m-2^31", qmm(qop("q8s", 32), qop("q8s", 32, bs=S2), BIG, 64, 64))
    add("qmm-err-batch-2^20", qmm(qop("q8s", 32), qop("q8s", 32, bs=S2), 64, 64, 64, batch=1 << 20))
    add("qmm-err2-lhs-and-rhs", qmm(qop("e4m3", 32, "ue8m0"), qop("q8s", 16, bs=S2), 64, 64, 64))
    add("qmm-err2-out-and-k0", qmm(qop("q8s", 32), qop("q8s", 32, bs=S2), 64, 64, 0, "i32"))
    add("qmm-err2-null-and-misaligned", qmm(qop("q8s", 32, values=0), qop("q8s", 32, bs=S2), 64, 64, 64, o=O + 2))

    # ---- b200_matmul_grouped
    for idt in ("bf16", "f16"):
        for odt in (idt, "f32"):
            for am in ("k", "m"):
                for bm in ("n", "k"):
                    for T, G in ((32768, 128), (4096, 8), (1000, 3)):
                        add(f"grp-m-{idt}-{odt}-{am}{bm}-T{T}-G{G}", grouped("m", T, G, 512, 768, idt=idt, odt=odt, a_major=am, b_major=bm))
                    add(f"grp-m-{idt}-{odt}-{am}{bm}-ep", grouped("m", 4096, 8, 512, 768, idt=idt, odt=odt, a_major=am, b_major=bm,
                                                                 ep={"ep": [0.5, 1, BIAS]}))
            for T, G, M in ((32768, 128, 768), (4096, 8, 128), (1000, 3, 100), (4096, 8, 129)):
                add(f"grp-k-{idt}-{odt}-T{T}-G{G}-M{M}", grouped("k", T, G, N=512, M=M, idt=idt, odt=odt))
    for am in ("k", "m"):
        for bm in ("n", "k"):
            tag = f"{am}{bm}"
            add(f"grp-m-pitch-a-{tag}", grouped("m", 4096, 8, 520, 768, a_major=am, b_major=bm, a_pitch=3))
            add(f"grp-m-pitch-b-{tag}", grouped("m", 4096, 8, 520, 768, a_major=am, b_major=bm, b_pitch=5))
            add(f"grp-m-misaligned-a-{tag}", grouped("m", 4096, 8, 512, 768, a_major=am, b_major=bm, a=A + 2))
            add(f"grp-m-misaligned-b-{tag}", grouped("m", 4096, 8, 512, 768, a_major=am, b_major=bm, b=B + 2))
            add(f"grp-m-G1-{tag}", grouped("m", 4096, 1, 512, 768, a_major=am, b_major=bm))
            add(f"grp-m-G1-pitch-b-{tag}", grouped("m", 4096, 1, 520, 768, a_major=am, b_major=bm, b_pitch=5))
            add(f"grp-m-G1024-{tag}", grouped("m", 65536, 1024, 256, 256, a_major=am, b_major=bm))
            add(f"grp-m-K1-{tag}", grouped("m", 4096, 8, 1, 768, a_major=am, b_major=bm))
            add(f"grp-m-T1-{tag}", grouped("m", 1, 8, 512, 768, a_major=am, b_major=bm))
            add(f"grp-m-N1-{tag}", grouped("m", 4096, 8, 512, 1, a_major=am, b_major=bm))
        add(f"grp-k-pitch-a-{am}", grouped("k", 4096, 8, N=512, M=256, a_major="m", a_pitch=3))
    add("grp-m-bcast-rhs", grouped("m", 4096, 8, 512, 768, strides=([512, 1], [0, 768, 1], [768, 1])))
    add("grp-m-K0", grouped("m", 4096, 8, 0, 768))
    add("grp-m-T0", grouped("m", 0, 8, 512, 768))
    add("grp-m-N0", grouped("m", 4096, 8, 512, 0))
    add("grp-m-G0", grouped("m", 4096, 0, 512, 768))
    add("grp-k-T0", grouped("k", 0, 8, N=512, M=256))
    add("grp-k-M0", grouped("k", 4096, 8, N=512, M=0))
    add("grp-k-T1", grouped("k", 1, 8, N=512, M=256))
    add("grp-k-M1", grouped("k", 4096, 8, N=512, M=1))
    add("grp-k-N1", grouped("k", 4096, 8, N=1, M=256))
    add("grp-k-staged-a", grouped("k", 4096, 8, N=512, M=256, a=A + 2))
    add("grp-k-staged-b", grouped("k", 4096, 8, N=512, M=256, b_pitch=3))
    add("grp-k-G1024", grouped("k", 65536, 1024, N=128, M=128))
    add("grp-m-opitch8", grouped("m", 4096, 8, 512, 768, o_pitch=8))
    add("grp-m-opitch1", grouped("m", 4096, 8, 512, 760, o_pitch=1))
    add("grp-m-omisaligned", grouped("m", 4096, 8, 512, 768, o=O + 2))
    add("grp-m-omisaligned-f32", grouped("m", 4096, 8, 512, 768, odt="f32", o=O + 4))
    add("grp-k-opitch8", grouped("k", 4096, 8, N=512, M=256, o_pitch=8))
    add("grp-k-opitch1", grouped("k", 4096, 8, N=512, M=256, o_pitch=1))
    add("grp-m-overlap-rows", grouped("m", 4096, 8, 512, 768, strides=([512, 1], [512 * 768, 768, 1], [512, 1])))
    for tag in ("auto", "2sm_n256", "2sm_n128", "1sm_n128", "2sm_m512", "2sm_n224", "simt", "bogus"):
        for epi in ("tma", "direct", "bogus"):
            opts = {"gemm.variant": tag, "gemm.epilogue": epi}
            add(f"grp-m-variant={tag}-epi={epi}", grouped("m", 32768, 64, 512, 768, options=opts))
            add(f"grp-k-variant={tag}-epi={epi}", grouped("k", 32768, 64, N=512, M=768, options=opts))
        add(f"grp-m-variant={tag}-ep", grouped("m", 4096, 8, 512, 768, ep={"ep": [1.0, 2, BIAS]}, options={"gemm.variant": tag}))
    for val in ("on", "3", "bogus"):
        add(f"grp-m-splitk={val}", grouped("m", 32768, 64, 512, 768, options={"gemm.split_k": val}))
    add("grp-m-groupm=1", grouped("m", 32768, 64, 512, 768, options={"gemm.group_m": "1"}))
    add("grp-m-l2promo=64", grouped("m", 32768, 64, 512, 768, options={"gemm.l2_promotion": "64"}))
    # refusals
    add("grp-err-null-shape", grouped("m", 4096, 8, 512, 768, shapes=(None, [8, 512, 768], [4096, 768]), ranks=(2, 3, 2)))
    add("grp-err-3x3", grouped("m", 4096, 8, 512, 768, shapes=([8, 4096, 512], [8, 512, 768], [8, 4096, 768]),
                               strides=([4096 * 512, 512, 1], [512 * 768, 768, 1], [4096 * 768, 768, 1])))
    add("grp-err-3x2", grouped("m", 4096, 8, 512, 768, shapes=([8, 4096, 512], [512, 768], [4096, 768]),
                               strides=([4096 * 512, 512, 1], [768, 1], [768, 1])))
    add("grp-err-ranks", grouped("m", 4096, 8, 512, 768, shapes=([4096, 512], [8, 512, 768], [8, 4096, 768]),
                                 strides=([512, 1], [512 * 768, 768, 1], [4096 * 768, 768, 1])))
    add("grp-err-rank1", grouped("m", 4096, 8, 512, 768, ranks=(1, 3, 2)))
    add("grp-err-rank4", grouped("m", 4096, 8, 512, 768, ranks=(2, 4, 2)))
    add("grp-err-f32", grouped("m", 4096, 8, 512, 768, idt="f32", odt="f32"))
    add("grp-err-e4m3", grouped("m", 4096, 8, 512, 768, idt="e4m3", odt="f32"))
    add("grp-err-bf16-to-f16", grouped("m", 4096, 8, 512, 768, idt="bf16", odt="f16"))
    add("grp-err-inner", grouped("m", 4096, 8, 512, 768, shapes=([4096, 512], [8, 256, 768], [4096, 768])))
    add("grp-err-groups", grouped("m", 4096, 8, 512, 768, shapes=([4096, 512], [7, 512, 768], [4096, 768])))
    add("grp-err-out", grouped("m", 4096, 8, 512, 768, shapes=([4096, 512], [8, 512, 768], [4096, 767])))
    add("grp-k-err-inner", grouped("k", 4096, 8, N=512, M=256, shapes=([256, 4096], [4095, 512], [8, 256, 512])))
    add("grp-k-err-groups", grouped("k", 4096, 8, N=512, M=256, shapes=([256, 4096], [4096, 512], [9, 256, 512])))
    add("grp-k-err-out", grouped("k", 4096, 8, N=512, M=256, shapes=([256, 4096], [4096, 512], [8, 256, 511])))
    add("grp-k-err-ep", grouped("k", 4096, 8, N=512, M=256, ep={"ep": [1.0, 0, 0]}))
    add("grp-err-act", grouped("m", 4096, 8, 512, 768, ep={"ep": [1.0, 3, 0]}))
    add("grp-err-act-neg", grouped("m", 4096, 8, 512, 768, ep={"ep": [1.0, -1, 0]}))
    add("grp-err-G1025", grouped("m", 65536, 1025, 256, 256))
    add("grp-err-T-2^31", grouped("m", BIG, 8, 512, 768))
    add("grp-k-err-M-2^31", grouped("k", 4096, 8, N=512, M=BIG))
    add("grp-err-null-offs", grouped("m", 4096, 8, 512, 768, offs=0))
    add("grp-err-misaligned-offs", grouped("m", 4096, 8, 512, 768, offs=OFFS + 2))
    add("grp-err-null-out", grouped("m", 4096, 8, 512, 768, o=0))
    add("grp-err-null-lhs", grouped("m", 4096, 8, 512, 768, a=0))
    add("grp-m-K0-null-lhs", grouped("m", 4096, 8, 0, 768, a=0, b=0))
    add("grp-err-misaligned-lhs", grouped("m", 4096, 8, 512, 768, a=A + 1))
    add("grp-err-misaligned-out", grouped("m", 4096, 8, 512, 768, odt="f32", o=O + 2))
    add("grp-err-misaligned-bias", grouped("m", 4096, 8, 512, 768, ep={"ep": [1.0, 0, BIAS + 2]}))
    add("grp-err-out-col-stride", grouped("m", 4096, 8, 512, 768, strides=([512, 1], [512 * 768, 768, 1], [1, 4096])))
    add("grp-err-out-2^40", grouped("m", 4096, 8, 512, 768, strides=([512, 1], [512 * 768, 768, 1], [1 << 40, 1])))
    add("grp-k-err-out-2^40", grouped("k", 4096, 8, N=512, M=256, strides=([1, 256], [512, 1], [1 << 40, 512, 1])))
    add("grp-k-err-k-major-a", grouped("k", 4096, 8, N=512, M=256, a_major="k"))
    add("grp-k-err-k-major-b", grouped("k", 4096, 8, N=512, M=256, b_major="k"))
    add("grp-err-tiles", grouped("m", (1 << 31) - 1, 1024, 64, (1 << 31) - 1))
    # two checks failing at once
    add("grp-err2-dtype-and-ranks", grouped("m", 4096, 8, 512, 768, idt="f32", ranks=(1, 3, 2)))
    add("grp-err2-dtype-and-inner", grouped("m", 4096, 8, 512, 768, idt="f32", odt="f32", shapes=([4096, 512], [8, 256, 768], [4096, 768])))
    add("grp-err2-groups-and-act", grouped("m", 4096, 1025, 512, 768, ep={"ep": [1.0, 9, 0]}, shapes=([4096, 512], [1025, 512, 768], [4096, 768])))
    add("grp-err2-ep-rk-and-G", grouped("k", 4096, 2000, N=512, M=256, ep={"ep": [1.0, 0, 0]}))
    add("grp-err2-offs-and-ptr", grouped("m", 4096, 8, 512, 768, offs=0, o=0))
    add("grp-err2-variant-and-epilogue", grouped("m", 4096, 8, 512, 768, options={"gemm.variant": "bogus", "gemm.epilogue": "bogus"}))
    add("grp-err2-staged-and-variant", grouped("m", 4096, 8, 520, 768, a_pitch=3, b=B + 2, options={"gemm.variant": "bogus"}))
    add("grp-err2-staged-and-epilogue", grouped("m", 4096, 8, 520, 768, a_pitch=3, b=B + 2, options={"gemm.epilogue": "bogus"}))
    add("grp-err2-tiles-and-epilogue", grouped("m", (1 << 31) - 1, 1024, 64, (1 << 31) - 1, options={"gemm.epilogue": "bogus"}))
    add("grp-err2-kmajor-and-staged", grouped("k", 4096, 8, N=512, M=256, a_major="k", a=A + 2))
    add("grp-err2-col-stride-and-misaligned", grouped("m", 4096, 8, 512, 768, a=A + 1, strides=([512, 1], [512 * 768, 768, 1], [1, 4096])))

    # ---- b200_matmul_quantized_fp8
    fp8s, bsds = ("e4m3", "e5m2"), ("f32", "f16", "bf16", "ue8m0", "e4m3")

    def tens(v, ts=S2):
        return qop(v, 0, 0, 1, bs=0, ts=ts)

    for lv in fp8s:
        for rv in fp8s:
            add(f"qf8-tensor-{lv}-{rv}", qf8(tens(lv), tens(rv, S2 + 4), 1024, 768, 512))
            add(f"qf8-block-{lv}-{rv}", qf8(qop(lv, 128), qop(rv, 128, bs=S2), 1024, 768, 512))
    for v in fp8s:
        for blk in (32, 64, 128):
            for bsd in bsds:
                add(f"qf8-block-{v}-{blk}-{bsd}", qf8(qop(v, blk, bsd), qop(v, blk, bsd, bs=S2), 1024, 768, 512))
            add(f"qf8-twolevel-{v}-{blk}", qf8(qop(v, blk, "f16", 1, ts=S2), qop(v, blk, "e4m3", 1, bs=S2, ts=S2 + 4), 512, 512, 512))
    for lb, rb in ((32, 64), (128, 32), (64, 128), (0, 32), (128, 0), (0, 0)):
        for odt in ("f32", "bf16", "f16"):
            lq = qop("e4m3", lb, "f32", 0 if lb else 1, bs=S1 if lb else 0, ts=0 if lb else S2)
            rq = qop("e5m2", rb, "ue8m0", 0 if rb else 1, bs=S2 if rb else 0, ts=0 if rb else S2 + 4)
            add(f"qf8-mixed-{lb}-{rb}-{odt}", qf8(lq, rq, 1024, 768, 512, odt))
            add(f"qf8-mixed-{lb}-{rb}-{odt}-batch", qf8(lq, rq, 256, 256, 256, odt, batch=3))
    for opts in ({"gemm.variant": "2sm_n256"}, {"gemm.variant": "2sm_n128"}, {"gemm.variant": "1sm_n128"}, {"gemm.variant": "2sm_m512"},
                 {"gemm.variant": "2sm_n224"}, {"gemm.variant": "simt"}, {"gemm.variant": "bogus"}, {"gemm.split_k": "on"},
                 {"gemm.split_k": "3"}, {"gemm.split_k": "bogus"}, {"gemm.epilogue": "tma"}, {"gemm.epilogue": "direct"},
                 {"gemm.epilogue": "bogus"}):
        tag = "-".join(f"{k.split('.')[1]}={v}" for k, v in opts.items())
        add(f"qf8-opt-{tag}-block", qf8(qop("e4m3", 128), qop("e4m3", 128, bs=S2), 4096, 4096, 4096, options=opts))
        add(f"qf8-opt-{tag}-tensor", qf8(tens("e4m3"), tens("e5m2", S2 + 4), 4096, 4096, 4096, options=opts))
    add("qf8-misaligned-lhs", qf8(qop("e4m3", 32, values=A + 8), qop("e4m3", 32, bs=S2), 1024, 768, 512))
    add("qf8-misaligned-rhs", qf8(qop("e4m3", 32), qop("e5m2", 32, values=B + 1, bs=S2), 1024, 768, 512))
    add("qf8-k-not-16", qf8(tens("e4m3"), tens("e4m3", S2 + 4), 256, 256, 200))
    add("qf8-k-not-16-batch", qf8(tens("e5m2"), tens("e4m3", S2 + 4), 256, 256, 200, batch=3))
    add("qf8-k-short-block", qf8(tens("e4m3"), tens("e4m3", S2 + 4), 256, 256, 320))
    add("qf8-small", qf8(qop("e4m3", 32), qop("e5m2", 32, bs=S2), 16, 8, 64))
    add("qf8-m1", qf8(qop("e4m3", 64), qop("e4m3", 64, bs=S2), 1, 4096, 4096))
    add("qf8-n1", qf8(qop("e4m3", 64), qop("e4m3", 64, bs=S2), 4096, 1, 4096))
    add("qf8-k-2^17", qf8(tens("e4m3"), tens("e4m3", S2 + 4), 64, 64, 1 << 17))
    add("qf8-empty-m", qf8(qop("e4m3", 32), qop("e4m3", 32, bs=S2), 0, 64, 64))
    add("qf8-empty-n", qf8(qop("e4m3", 32), qop("e4m3", 32, bs=S2), 64, 0, 64))
    add("qf8-empty-batch", qf8(qop("e4m3", 32), qop("e4m3", 32, bs=S2), 64, 64, 64, batch=0))
    add("qf8-empty-null", qf8(qop("e4m3", 32, values=0), qop("e4m3", 32, bs=S2), 0, 64, 64, o=0))
    add("qf8-err-null-lhs", qf8(None, qop("e4m3", 32, bs=S2), 64, 64, 64))
    add("qf8-err-null-rhs", qf8(qop("e4m3", 32), None, 64, 64, 64))
    for v in ("q8s", "q8f", "q4s", "q2f"):
        add(f"qf8-err-int-{v}-lhs", qf8(qop(v, 32), qop("e4m3", 32, bs=S2), 64, 64, 64))
        add(f"qf8-err-int-{v}-rhs", qf8(qop("e4m3", 32), qop(v, 32, bs=S2), 64, 64, 64))
    add("qf8-err-e2m1", qf8(qop("e4m3", 32), qop("e2m1", 32, "ue8m0", bs=S2), 64, 64, 64))
    add("qf8-err-e2m1-lhs", qf8(qop("e2m1", 32, "ue8m0"), qop("e4m3", 32, bs=S2), 64, 64, 64))
    add("qf8-err-block16", qf8(qop("e4m3", 16), qop("e4m3", 16, bs=S2), 64, 64, 64))
    add("qf8-err-block8", qf8(qop("e4m3", 32), qop("e4m3", 8, bs=S2), 64, 64, 64))
    add("qf8-err-block256", qf8(qop("e4m3", 256), qop("e4m3", 32, bs=S2), 64, 64, 256))
    add("qf8-err-bad-value", qf8(qop("bogus", 32), qop("e4m3", 32, bs=S2), 64, 64, 64))
    add("qf8-err-tensor-flag", qf8(qop("e4m3", 32, tensor=2), qop("e4m3", 32, bs=S2), 64, 64, 64))
    add("qf8-err-no-level", qf8(qop("e4m3", 0, 0, 0, bs=0), qop("e4m3", 32, bs=S2), 64, 64, 64))
    add("qf8-err-bad-scale-dtype", qf8(qop("e4m3", 32, "i32"), qop("e4m3", 32, bs=S2), 64, 64, 64))
    add("qf8-err-k-block", qf8(qop("e4m3", 32), qop("e4m3", 32, bs=S2), 64, 64, 48))
    add("qf8-err-null-block-scales", qf8(qop("e4m3", 32, bs=0), qop("e4m3", 32, bs=S2), 64, 64, 64))
    add("qf8-err-null-tensor-scale", qf8(tens("e4m3", 0), tens("e4m3", S2 + 4), 64, 64, 64))
    add("qf8-err-misaligned-scales", qf8(qop("e4m3", 32, bs=S1 + 1), qop("e4m3", 32, bs=S2), 64, 64, 64))
    add("qf8-err-out-i32", qf8(qop("e4m3", 32), qop("e4m3", 32, bs=S2), 64, 64, 64, "i32"))
    add("qf8-err-out-e4m3", qf8(qop("e4m3", 32), qop("e4m3", 32, bs=S2), 64, 64, 64, "e4m3"))
    add("qf8-err-k0", qf8(qop("e4m3", 32), qop("e4m3", 32, bs=S2), 64, 64, 0))
    add("qf8-err-k0-tensor", qf8(tens("e4m3"), tens("e4m3", S2 + 4), 64, 64, 0))
    add("qf8-err-null-values", qf8(qop("e4m3", 32, values=0), qop("e4m3", 32, bs=S2), 64, 64, 64))
    add("qf8-err-null-rhs-values", qf8(qop("e4m3", 32), qop("e4m3", 32, values=0, bs=S2), 64, 64, 64))
    add("qf8-err-null-out", qf8(qop("e4m3", 32), qop("e4m3", 32, bs=S2), 64, 64, 64, o=0))
    add("qf8-err-misaligned-out", qf8(qop("e4m3", 32), qop("e4m3", 32, bs=S2), 64, 64, 64, "f32", o=O + 2))
    add("qf8-err-m-2^31", qf8(qop("e4m3", 32), qop("e4m3", 32, bs=S2), BIG, 64, 64))
    add("qf8-err-n-2^31", qf8(qop("e4m3", 32), qop("e4m3", 32, bs=S2), 64, BIG, 64))
    add("qf8-err-k-2^31", qf8(tens("e4m3"), tens("e4m3", S2 + 4), 64, 64, BIG))
    add("qf8-err-batch-2^20", qf8(qop("e4m3", 32), qop("e4m3", 32, bs=S2), 64, 64, 64, batch=1 << 20))
    add("qf8-err-tiles", qf8(qop("e4m3", 32), qop("e4m3", 32, bs=S2), (1 << 31) - 1, (1 << 31) - 1, 64, batch=(1 << 20) - 1))
    add("qf8-err2-lhs-and-rhs", qf8(qop("q8s", 32), qop("e4m3", 16, bs=S2), 64, 64, 64))
    add("qf8-err2-e2m1-and-block", qf8(qop("e2m1", 16, "ue8m0"), qop("e4m3", 32, bs=S2), 64, 64, 64))
    add("qf8-err2-out-and-k0", qf8(qop("e4m3", 32), qop("e4m3", 32, bs=S2), 64, 64, 0, "i32"))
    add("qf8-err2-null-and-misaligned", qf8(qop("e4m3", 32, values=0), qop("e4m3", 32, bs=S2), 64, 64, 64, o=O + 2))
    add("qf8-err2-misaligned-and-extent", qf8(qop("e4m3", 32), qop("e4m3", 32, bs=S2), BIG, 64, 64, o=O + 2))
    add("qf8-err2-staged-and-variant", qf8(qop("e4m3", 32, values=A + 8), qop("e4m3", 32, bs=S2), 1024, 768, 512,
                                            options={"gemm.variant": "bogus"}))
    add("qf8-err2-staged-and-epilogue", qf8(tens("e4m3"), tens("e4m3", S2 + 4), 1024, 768, 200, options={"gemm.epilogue": "bogus"}))
    add("qf8-err2-variant-and-epilogue", qf8(qop("e4m3", 128), qop("e4m3", 128, bs=S2), 4096, 4096, 4096,
                                             options={"gemm.variant": "bogus", "gemm.epilogue": "bogus"}))

    # ---- b200_matmul_grouped_quantized_fp8
    for lv in fp8s:
        for rv in fp8s:
            add(f"gqf8-tensor-{lv}-{rv}", gqf8(tens(lv), tens(rv, S2 + 4), 8, 4096, 768, 512))
            add(f"gqf8-block-{lv}-{rv}", gqf8(qop(lv, 128), qop(rv, 128, bs=S2), 8, 4096, 768, 512))
    for v in fp8s:
        for blk in (32, 64, 128):
            for bsd in bsds:
                add(f"gqf8-block-{v}-{blk}-{bsd}", gqf8(qop(v, blk, bsd), qop(v, blk, bsd, bs=S2), 8, 4096, 768, 512))
            add(f"gqf8-twolevel-{v}-{blk}", gqf8(qop(v, blk, "f16", 1, ts=S2), qop(v, blk, "e4m3", 1, bs=S2, ts=S2 + 4), 6, 3000, 512, 512))
    for lb, rb in ((32, 64), (128, 32), (0, 128), (128, 0), (0, 0)):
        for odt in ("f32", "bf16", "f16"):
            lq = qop("e5m2", lb, "bf16", 0 if lb else 1, bs=S1 if lb else 0, ts=0 if lb else S2)
            rq = qop("e4m3", rb, "f32", 0 if rb else 1, bs=S2 if rb else 0, ts=0 if rb else S2 + 4)
            add(f"gqf8-mixed-{lb}-{rb}-{odt}", gqf8(lq, rq, 8, 4096, 768, 512, odt))
    blk = (qop("e4m3", 128), qop("e4m3", 128, bs=S2))
    for G, T, N, K in ((1, 4096, 768, 512), (128, 32768, 1536, 1024), (1024, 65536, 256, 256), (8, 8 * 1024, 256, 256),
                       (8, 8 * 1024 - 1, 256, 256), (8, 100, 256, 256), (8, 1, 256, 256), (3, 1000, 700, 384), (32, 32768, 4096, 7168)):
        add(f"gqf8-shape-G{G}-T{T}-N{N}-K{K}", gqf8(*blk, G, T, N, K))
    add("gqf8-G1-tensor", gqf8(tens("e4m3"), tens("e4m3", S2 + 4), 1, 4096, 768, 512))
    add("gqf8-G1024-tensor", gqf8(tens("e4m3"), tens("e4m3", S2 + 4), 1024, 65536, 256, 256))
    add("gqf8-T0", gqf8(*blk, 8, 0, 768, 512))
    add("gqf8-N0", gqf8(*blk, 8, 4096, 0, 512))
    add("gqf8-G0", gqf8(*blk, 0, 4096, 768, 512))
    add("gqf8-T0-null", gqf8(qop("e4m3", 128, values=0), qop("e4m3", 128, values=0, bs=S2), 8, 0, 768, 512, o=0, offs=0))
    add("gqf8-err-K0", gqf8(*blk, 8, 4096, 768, 0))
    add("gqf8-err-K0-tensor", gqf8(tens("e4m3"), tens("e4m3", S2 + 4), 8, 4096, 768, 0))
    for tag in ("auto", "2sm_n256", "2sm_n128", "1sm_n128", "2sm_m512", "2sm_n224", "simt", "bogus"):
        for epi in ("tma", "direct", "bogus"):
            opts = {"gemm.variant": tag, "gemm.epilogue": epi}
            add(f"gqf8-variant={tag}-epi={epi}", gqf8(*blk, 64, 32768, 768, 512, options=opts))
    for val in ("on", "3", "bogus"):
        add(f"gqf8-splitk={val}", gqf8(*blk, 64, 32768, 768, 512, options={"gemm.split_k": val}))
    add("gqf8-misaligned-lhs", gqf8(qop("e4m3", 128, values=A + 8), qop("e4m3", 128, bs=S2), 8, 4096, 768, 512))
    add("gqf8-misaligned-rhs", gqf8(qop("e4m3", 128), qop("e4m3", 128, values=B + 1, bs=S2), 8, 4096, 768, 512))
    add("gqf8-k-not-16", gqf8(tens("e4m3"), tens("e5m2", S2 + 4), 8, 4096, 768, 200))
    add("gqf8-k-not-16-G1", gqf8(tens("e4m3"), tens("e5m2", S2 + 4), 1, 4096, 768, 200))
    add("gqf8-err-null-lhs", gqf8(None, qop("e4m3", 128, bs=S2), 8, 4096, 768, 512))
    add("gqf8-err-null-rhs", gqf8(qop("e4m3", 128), None, 8, 4096, 768, 512))
    add("gqf8-err-G1025", gqf8(*blk, 1025, 65536, 256, 256))
    add("gqf8-err-G1025-empty", gqf8(*blk, 1025, 0, 256, 256))
    add("gqf8-err-T-2^31", gqf8(*blk, 8, BIG, 768, 512))
    add("gqf8-err-N-2^31", gqf8(*blk, 8, 4096, BIG, 512))
    add("gqf8-err-K-2^31", gqf8(tens("e4m3"), tens("e4m3", S2 + 4), 8, 4096, 768, BIG))
    for v in ("q8s", "q4f"):
        add(f"gqf8-err-int-{v}-lhs", gqf8(qop(v, 128), qop("e4m3", 128, bs=S2), 8, 4096, 768, 512))
        add(f"gqf8-err-int-{v}-rhs", gqf8(qop("e4m3", 128), qop(v, 128, bs=S2), 8, 4096, 768, 512))
    add("gqf8-err-e2m1", gqf8(qop("e2m1", 32, "ue8m0"), qop("e4m3", 32, bs=S2), 8, 4096, 768, 512))
    add("gqf8-err-e2m1-rhs", gqf8(qop("e4m3", 32), qop("e2m1", 32, "ue8m0", bs=S2), 8, 4096, 768, 512))
    add("gqf8-err-block16", gqf8(qop("e4m3", 16), qop("e4m3", 16, bs=S2), 8, 4096, 768, 512))
    add("gqf8-err-k-block", gqf8(qop("e4m3", 128), qop("e4m3", 128, bs=S2), 8, 4096, 768, 96))
    add("gqf8-err-null-block-scales", gqf8(qop("e4m3", 128, bs=0), qop("e4m3", 128, bs=S2), 8, 4096, 768, 512))
    add("gqf8-err-out-i32", gqf8(*blk, 8, 4096, 768, 512, "i32"))
    add("gqf8-err-null-offs", gqf8(*blk, 8, 4096, 768, 512, offs=0))
    add("gqf8-err-misaligned-offs", gqf8(*blk, 8, 4096, 768, 512, offs=OFFS + 2))
    add("gqf8-err-null-out", gqf8(*blk, 8, 4096, 768, 512, o=0))
    add("gqf8-err-null-values", gqf8(qop("e4m3", 128, values=0), qop("e4m3", 128, bs=S2), 8, 4096, 768, 512))
    add("gqf8-err-misaligned-out", gqf8(*blk, 8, 4096, 768, 512, "f32", o=O + 2))
    add("gqf8-err-tiles", gqf8(*blk, 1024, (1 << 31) - 1, (1 << 31) - 1, 128))
    add("gqf8-err2-groups-and-dtype", gqf8(qop("q8s", 128), qop("e4m3", 128, bs=S2), 1025, 4096, 768, 512))
    add("gqf8-err2-extent-and-dtype", gqf8(qop("q8s", 128), qop("e4m3", 128, bs=S2), 8, BIG, 768, 512))
    add("gqf8-err2-offs-and-ptr", gqf8(*blk, 8, 4096, 768, 512, offs=0, o=0))
    add("gqf8-err2-misaligned-offs-and-out", gqf8(*blk, 8, 4096, 768, 512, offs=OFFS + 2, o=O + 2))
    add("gqf8-err2-out-and-k0", gqf8(*blk, 8, 4096, 768, 0, "i32"))
    add("gqf8-err2-staged-and-variant", gqf8(qop("e4m3", 128, values=A + 8), qop("e4m3", 128, bs=S2), 8, 4096, 768, 512,
                                             options={"gemm.variant": "bogus"}))
    add("gqf8-err2-staged-and-epilogue", gqf8(tens("e4m3"), tens("e4m3", S2 + 4), 8, 4096, 768, 200, options={"gemm.epilogue": "bogus"}))
    add("gqf8-err2-tiles-and-epilogue", gqf8(*blk, 1024, (1 << 31) - 1, (1 << 31) - 1, 128, options={"gemm.epilogue": "bogus"}))
    return out


def main() -> None:
    rows = []
    seen = set()
    for cid, c in cases():
        assert cid not in seen, cid
        seen.add(cid)
        rows.append({"id": cid, "call": c, **replay(c)})
    # gzip without a timestamp: the same cases always give the same bytes
    text = json.dumps({"_generated_by": "tests/golden/make_matmul_plan_golden.py", "cases": rows}, indent=0) + "\n"
    GOLDEN.write_bytes(gzip.compress(text.encode(), mtime=0))
    fails = sum(1 for r in rows if r["status"])
    print(f"wrote {GOLDEN}: {len(rows)} cases, {fails} failing, {GOLDEN.stat().st_size // 1024} KB")


if __name__ == "__main__":
    main()
