"""Time of mixture-of-experts routing (b200_moe_route / _plan / _permute / _combine / _combine_backward) on three models'
shapes, next to the same-run b200_probe_memcopy and torch's equivalent GPU sequence, and its share of a whole layer.

    python tools/moe_bench.py [--iters 20] [--warmup 3] [--rows mixtral,qwen3,deepseek]

Rows (T tokens chosen so that permute and combine each take well over 50 us):
  mixtral   E 8,   k 2, K 4096, F 14336, softmax + renormalize,              T 32768
  qwen3     E 128, k 8, K 2048, F 768,   softmax + renormalize,              T 16384
  deepseek  E 256, k 8, K 7168, F 2048,  sigmoid + bias, 8 groups / top 4, x2.5, T 8192
Logits f32 [T, E]; activations, expert outputs and y bf16.  Bytes are algorithmic: permute moves each kept row once in and
once out (2 * T * k * K * 2), combine reads T * k rows of ys and writes T rows of y ((T * k + T) * K * 2), combine_backward
reads dy and the T * k rows of ys and writes T * k rows of d_ys ((T + 2 * T * k) * K * 2); index arrays are not counted.
route + plan are timed a second time at 8 T ("large"), where they are bound by their work rather than by launch latency.
memcopy: b200_probe_memcopy of 1 GiB, counted as 2 GiB moved.  torch: route = softmax (or sigmoid + bias + group top-2 /
top-k masking) + topk + renormalize; plan = argsort(stable) + bincount + cumsum; permute = index_select; combine = index +
weighted sum in f32 over k; combine_backward = the scattered w * dy rows and an einsum for d_w.  Layer = route + plan +
permute + grouped GEMM [K -> F] with a relu epilogue + grouped GEMM [F -> K] + combine.  Each time is the CUDA-event mean of `--iters` back-to-back calls after `--warmup`.
Goals, stated before measuring:
  (a) permute and combine at >= 0.7 of the same-run copy rate, in algorithmic bytes, at K, N >= 2048;
  (b) route + plan in <= 0.5x torch's softmax / topk + stable argsort + bincount + cumsum;
  (c) the share of route + plan + permute + combine in a whole layer, recorded without a goal.
combine_backward's rate and its ratio to torch are recorded without a goal.
The card name and power limit are read (nvidia-smi --query-gpu, read-only) in the same run.  Prints one JSON line.
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from cubecl_b200 import ComputeClient, TensorHandle, matmul, moe, synth  # noqa: E402
from matmul_grouped_bench import torch_timed  # noqa: E402
from scan_bench import gpu_info, timed  # noqa: E402

MODELS = {
    "mixtral": dict(E=8, k=2, K=4096, F=14336, T=32768, route=dict(score="softmax", renormalize=True)),
    "qwen3": dict(E=128, k=8, K=2048, F=768, T=16384, route=dict(score="softmax", renormalize=True)),
    "deepseek": dict(E=256, k=8, K=7168, F=2048, T=8192, route=dict(score="sigmoid", renormalize=True, n_group=8, topk_group=4, scale=2.5)),
}


def torch_route(logits, bias, k, score, renormalize=True, n_group=0, topk_group=0, scale=1.0):
    import torch
    s = torch.softmax(logits, -1) if score == "softmax" else torch.sigmoid(logits)
    key = s + bias if bias is not None else s
    if n_group > 1:
        T, E = key.shape
        g = key.view(T, n_group, -1).topk(2, dim=-1)[0].sum(-1)
        mask = torch.zeros_like(g).scatter_(1, g.topk(topk_group, dim=-1)[1], 1)
        key = key.masked_fill(mask.unsqueeze(-1).expand(T, n_group, E // n_group).reshape(T, E) == 0, float("-inf"))
    ids = key.topk(k, dim=-1)[1]
    w = s.gather(1, ids)
    if renormalize:
        w = w / w.sum(-1, keepdim=True)
    return ids, w * scale


def torch_plan(ids, E):
    import torch
    flat = ids.flatten()
    order = torch.argsort(flat, stable=True)
    offs = torch.cumsum(torch.bincount(flat, minlength=E), 0)
    return order, offs


def torch_combine_backward(dy, ys, w, row_of):
    import torch
    T, k = row_of.shape
    d_ys = torch.empty_like(ys)
    d_ys[row_of.flatten()] = (w[:, :, None] * dy[:, None, :].float()).reshape(T * k, -1).to(ys.dtype)
    d_w = torch.einsum("tn,tkn->tk", dy.float(), ys[row_of].float())
    return d_ys, d_w


def run_row(c, name, m, iters, warmup, copy_gbps):
    import torch
    E, k, K, F, T = m["E"], m["k"], m["K"], m["F"], m["T"]
    rng = np.random.default_rng(1)
    logits_h = rng.standard_normal((T, E)).astype(np.float32)
    bias_h = (rng.standard_normal(E) * 0.01).astype(np.float32) if name == "deepseek" else None
    logits = TensorHandle.from_numpy(c, logits_h, "f32")
    bias = TensorHandle.from_numpy(c, bias_h, "f32") if bias_h is not None else None
    x = TensorHandle.empty_contiguous(c, [T, K], "bf16")
    c.fill_uniform(x.handle, "bf16", T * K, 3, -1.0, 1.0)
    w1 = TensorHandle.empty_contiguous(c, [E, K, F], "bf16")
    c.fill_uniform(w1.handle, "bf16", E * K * F, 4, -0.02, 0.02)
    w2 = TensorHandle.empty_contiguous(c, [E, F, K], "bf16")
    c.fill_uniform(w2.handle, "bf16", E * F * K, 5, -0.02, 0.02)
    ids = TensorHandle.empty_contiguous(c, [T, k], "i32")
    wts = TensorHandle.empty_contiguous(c, [T, k], "f32")
    offs = TensorHandle.empty_contiguous(c, [E], "i32")
    row_of = TensorHandle.empty_contiguous(c, [T, k], "i32")
    slot_of = TensorHandle.empty_contiguous(c, [T * k], "i32")
    xs = TensorHandle.empty_contiguous(c, [T * k, K], "bf16")
    h = TensorHandle.empty_contiguous(c, [T * k, F], "bf16")
    ys = TensorHandle.empty_contiguous(c, [T * k, K], "bf16")
    y = TensorHandle.empty_contiguous(c, [T, K], "bf16")
    route = lambda: moe.route(c, logits, ids, wts, k, bias=bias, **m["route"])  # noqa: E731
    plan = lambda: moe.plan(c, ids, E, offs, row_of, slot_of)  # noqa: E731
    permute = lambda: moe.permute(c, x, slot_of, k, xs)  # noqa: E731
    combine = lambda: moe.combine(c, ys, row_of, y, wts)  # noqa: E731
    dy = TensorHandle.empty_contiguous(c, [T, K], "bf16")
    c.fill_uniform(dy.handle, "bf16", T * K, 6, -1.0, 1.0)
    d_ys = TensorHandle.empty_contiguous(c, [T * k, K], "bf16")
    d_w = TensorHandle.empty_contiguous(c, [T, k], "f32")
    combine_bwd = lambda: moe.combine_backward(c, dy, ys, wts, row_of, d_ys, d_w)  # noqa: E731
    gemm1 = lambda: matmul.launch_grouped(c, xs, w1, offs, h, activation="relu")  # noqa: E731
    gemm2 = lambda: matmul.launch_grouped(c, h, w2, offs, ys)  # noqa: E731

    def layer():
        route(); plan(); permute(); gemm1(); gemm2(); combine()  # noqa: E702

    layer()
    c.sync()
    t = {n: timed(c, f, iters, warmup) for n, f in (("route", route), ("plan", plan), ("permute", permute), ("combine", combine),
                                                     ("combine_backward", combine_bwd), ("layer", layer))}
    # torch's GPU sequence on its own copies
    tl = torch.tensor(logits_h, device="cuda")
    tb = torch.tensor(bias_h, device="cuda") if bias_h is not None else None
    tx = torch.randn(T, K, device="cuda", dtype=torch.bfloat16)
    tids, tw = torch_route(tl, tb, k, **m["route"])
    order, _ = torch_plan(tids, E)
    tys = torch.randn(T * k, K, device="cuda", dtype=torch.bfloat16)
    tdy = torch.randn(T, K, device="cuda", dtype=torch.bfloat16)
    trow = torch.empty_like(order)
    trow[order] = torch.arange(T * k, device="cuda")
    trow = trow.view(T, k)
    tt = {
        "route": torch_timed(lambda: torch_route(tl, tb, k, **m["route"]), iters, warmup),
        "plan": torch_timed(lambda: torch_plan(tids, E), iters, warmup),
        "permute": torch_timed(lambda: tx.index_select(0, order // k), iters, warmup),
        "combine": torch_timed(lambda: (tys[trow].float() * tw[:, :, None]).sum(1).bfloat16(), iters, warmup),
        "combine_backward": torch_timed(lambda: torch_combine_backward(tdy, tys, tw, trow), iters, warmup),
    }
    # route + plan at 8 T, on their own
    TL = 8 * T
    big_logits_h = np.random.default_rng(2).standard_normal((TL, E)).astype(np.float32)
    big_logits = TensorHandle.from_numpy(c, big_logits_h, "f32")
    big_ids = TensorHandle.empty_contiguous(c, [TL, k], "i32")
    big_w = TensorHandle.empty_contiguous(c, [TL, k], "f32")
    big_offs = TensorHandle.empty_contiguous(c, [E], "i32")
    big_row = TensorHandle.empty_contiguous(c, [TL, k], "i32")
    big_slot = TensorHandle.empty_contiguous(c, [TL * k], "i32")
    t["route_large"] = timed(c, lambda: moe.route(c, big_logits, big_ids, big_w, k, bias=bias, **m["route"]), iters, warmup)
    t["plan_large"] = timed(c, lambda: moe.plan(c, big_ids, E, big_offs, big_row, big_slot), iters, warmup)
    tbl = torch.tensor(big_logits_h, device="cuda")
    tbig_ids, _ = torch_route(tbl, tb, k, **m["route"])
    tt["route_large"] = torch_timed(lambda: torch_route(tbl, tb, k, **m["route"]), iters, warmup)
    tt["plan_large"] = torch_timed(lambda: torch_plan(tbig_ids, E), iters, warmup)
    permute_bytes = 2 * T * k * K * 2
    combine_bytes = (T * k + T) * K * 2
    backward_bytes = (T + 2 * T * k) * K * 2
    routing = t["route"] + t["plan"] + t["permute"] + t["combine"]
    res = {
        "row": name, "T": T, "E": E, "k": k, "K": K, "F": F,
        "ms": {n: round(v, 4) for n, v in t.items()},
        "torch_ms": {n: round(v, 4) for n, v in tt.items()},
        "permute_gbps": round(permute_bytes / t["permute"] / 1e6, 1),
        "combine_gbps": round(combine_bytes / t["combine"] / 1e6, 1),
        "permute_of_copy": round(permute_bytes / t["permute"] / 1e6 / copy_gbps, 3),
        "combine_of_copy": round(combine_bytes / t["combine"] / 1e6 / copy_gbps, 3),
        "combine_backward_gbps": round(backward_bytes / t["combine_backward"] / 1e6, 1),
        "combine_backward_of_copy": round(backward_bytes / t["combine_backward"] / 1e6 / copy_gbps, 3),
        "combine_backward_of_torch": round(t["combine_backward"] / tt["combine_backward"], 3),
        "route_plan_of_torch": round((t["route"] + t["plan"]) / (tt["route"] + tt["plan"]), 3),
        "T_large": TL,
        "route_plan_large_of_torch": round((t["route_large"] + t["plan_large"]) / (tt["route_large"] + tt["plan_large"]), 3),
        "routing_share_of_layer": round(routing / t["layer"], 3),
    }
    res["goal_a"] = res["permute_of_copy"] >= 0.7 and res["combine_of_copy"] >= 0.7
    res["goal_b"] = res["route_plan_of_torch"] <= 0.5 and res["route_plan_large_of_torch"] <= 0.5
    del tl, tx, tys, tdy, tbl
    torch.cuda.empty_cache()
    return res


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rows", default="mixtral,qwen3,deepseek")
    args = ap.parse_args()
    c = ComputeClient.load(0)
    nbytes = 1 << 30
    src, dst = c.empty(nbytes), c.empty(nbytes)
    copy_ms = timed(c, lambda: c.probe_memcopy(dst, src, nbytes), args.iters, args.warmup)
    copy_gbps = 2 * nbytes / copy_ms / 1e6
    del src, dst
    rows = [run_row(c, n, MODELS[n], args.iters, args.warmup, copy_gbps) for n in args.rows.split(",")]
    print(json.dumps({"gpu": gpu_info(), "device": c.properties["name"], "memcopy_gbps": round(copy_gbps, 1), "rows": rows}))


if __name__ == "__main__":
    main()
