"""Time of softmax cross-entropy (b200_cross_entropy, b200_cross_entropy_backward) on bf16 logits, next to the same-run
b200_probe_memcopy rate and torch's eager F.cross_entropy.

    python tools/cross_entropy_bench.py [--iters 20] [--warmup 3] [--rounds 2] [--shapes 64x128256,4096x128256,...]

Every row: logits bf16 [t, v], i64 targets, MEAN reduction, lse written.  Bytes are algorithmic (reads plus writes from the
shapes, plus the per-row vectors):
  forward              logits read + targets, lse:                       2 t v + 12 t
  backward (in place)  logits read + gradient written + targets, lse:   4 t v + 12 t
  fused (in place)     the same as the backward:                         4 t v + 12 t
memcopy: b200_probe_memcopy of 1 GiB, counted as 2 GiB moved.  torch: F.cross_entropy on the bf16 logits, forward alone and
forward + backward (the logits' gradient through autograd).  Each time is the CUDA-event mean of `--iters` back-to-back
calls after `--warmup`; the shapes are measured in `--rounds` alternating rounds and each round is reported.
Goals, stated before measuring: forward >= 0.8x the copy rate at t v >= 2^28; in-place backward >= 0.75x; fused <= 0.75x
the time of forward + backward; fused >= 2x faster than torch's forward + backward at (8192, 128256).  The card name and
power limit are read (nvidia-smi --query-gpu, read-only) in the same run.  Prints one JSON line.
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from cubecl_b200 import ComputeClient, TensorHandle, cross_entropy as xent  # noqa: E402
from matmul_grouped_bench import torch_timed  # noqa: E402
from scan_bench import gpu_info, timed  # noqa: E402

SHAPES = "64x128256,4096x128256,8192x128256,8192x151936,4096x262144,8192x50257,16384x32000"


def logits_of(c, t, v, seed):
    """a bf16 [t, v] device tensor: a random 64-row block tiled down the rows (the values do not change the time)"""
    rng = np.random.default_rng(seed)
    block = ((rng.standard_normal((min(t, 64), v)).astype(np.float32) * 2).view(np.uint32) >> 16).astype(np.uint16)
    return TensorHandle.from_numpy(c, np.tile(block, (-(-t // block.shape[0]), 1))[:t], "bf16")


def run_row(c, t, v, iters, warmup, copy_gbps):
    import torch
    import torch.nn.functional as F
    x = logits_of(c, t, v, 1)
    y = TensorHandle.from_numpy(c, np.random.default_rng(2).integers(0, v, size=t).astype(np.int64), "i64")
    loss = TensorHandle.empty_contiguous(c, [1], "f32")
    lse = TensorHandle.empty_contiguous(c, [t], "f32")
    dloss = TensorHandle.from_numpy(c, np.ones(1, np.float32), "f32")
    fwd_ms = timed(c, lambda: xent.forward(c, x, y, loss, lse), iters, warmup)
    bwd_ms = timed(c, lambda: xent.backward(c, x, y, lse, dloss, x), iters, warmup)
    fused_ms = timed(c, lambda: xent.forward(c, x, y, loss, lse, dloss=dloss, dlogits=x), iters, warmup)
    c.sync()
    del x
    xt = (torch.randn(t, v, device="cuda") * 2).to(torch.bfloat16).requires_grad_(True)
    yt = torch.randint(0, v, (t,), device="cuda")
    t_fwd = torch_timed(lambda: F.cross_entropy(xt, yt), iters, warmup)

    def fwd_bwd():
        xt.grad = None
        F.cross_entropy(xt, yt).backward()

    t_fb = torch_timed(fwd_bwd, iters, warmup)
    del xt, yt
    torch.cuda.empty_cache()
    fb, gb = 2 * t * v + 12 * t, 4 * t * v + 12 * t
    fwd_gbps, bwd_gbps, fused_gbps = fb / fwd_ms / 1e6, gb / bwd_ms / 1e6, gb / fused_ms / 1e6
    return {"t": t, "v": v, "fwd_us": round(fwd_ms * 1e3, 1), "fwd_of_copy": round(fwd_gbps / copy_gbps, 3),
            "bwd_us": round(bwd_ms * 1e3, 1), "bwd_of_copy": round(bwd_gbps / copy_gbps, 3),
            "fused_us": round(fused_ms * 1e3, 1), "fused_of_copy": round(fused_gbps / copy_gbps, 3),
            "fused_over_fwd_plus_bwd": round(fused_ms / (fwd_ms + bwd_ms), 3),
            "torch_fwd_us": round(t_fwd * 1e3, 1), "torch_fwd_bwd_us": round(t_fb * 1e3, 1),
            "fused_vs_torch_fwd_bwd": round(t_fb / fused_ms, 2)}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--shapes", default=SHAPES)
    args = ap.parse_args()
    c = ComputeClient.load(0)
    nbytes = 1 << 30
    src, dst = c.empty(nbytes), c.empty(nbytes)
    copy_ms = timed(c, lambda: c.probe_memcopy(dst, src, nbytes), args.iters, args.warmup)
    copy_gbps = 2 * nbytes / copy_ms / 1e6
    del src, dst
    shapes = [tuple(map(int, s.split("x"))) for s in args.shapes.split(",")]
    rounds = [[run_row(c, t, v, args.iters, args.warmup, copy_gbps) for t, v in shapes] for _ in range(args.rounds)]
    every = [r for rows in rounds for r in rows]
    big = [r for r in every if r["t"] * r["v"] >= 1 << 28]
    goals = {"fwd_ge_0.8_copy": all(r["fwd_of_copy"] >= 0.8 for r in big),
             "bwd_ge_0.75_copy": all(r["bwd_of_copy"] >= 0.75 for r in big),
             "fused_le_0.75_fwd_plus_bwd": all(r["fused_over_fwd_plus_bwd"] <= 0.75 for r in every),
             "fused_ge_2x_torch_at_8192x128256": all(r["fused_vs_torch_fwd_bwd"] >= 2 for r in every
                                                     if (r["t"], r["v"]) == (8192, 128256))}
    print(json.dumps({"gpu": gpu_info(), "device": c.properties["name"], "memcopy_gbps": round(copy_gbps, 1), "goals_met": goals,
                      "rounds": rounds}))


if __name__ == "__main__":
    main()
