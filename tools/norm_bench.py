"""Time of RMSNorm (b200_norm, b200_norm_backward, b200_norm_quantized_fp8) on bf16 rows, next to the same-run
b200_probe_memcopy rate, torch's F.rms_norm forward and backward, and b200_norm + b200_quantize for the fp8 output.

    python tools/norm_bench.py [--iters 20] [--warmup 3] [--t 4096,16384,65536] [--n 2048,4096,7168,8192,16384]

Every row: x, y, dy and dx bf16 [t, n], weight bf16 [n], eps 1e-6, rstd f32 [t].  Bytes are algorithmic (reads plus writes
from the shapes):
  forward   x read + y written + rstd written:            4 t n + 4 t        (+ 2 n weight)
  backward  dy and h read + dx written + rstd read:        6 t n + 4 t        (+ 2 n weight + 4 n dweight)
  fp8       x read + e4m3 codes + f32 scales per 128:      3 t n + t n / 32   (+ 2 n + 4 t)
The unfused fp8 path (b200_norm to bf16, then b200_quantize of it) moves 3 t n more bytes.  memcopy: b200_probe_memcopy of
1 GiB, counted as 2 GiB moved.  torch: F.rms_norm forward, and the backward of that graph (dx and dweight) timed alone.
Each time is the CUDA-event mean of `--iters` back-to-back calls after `--warmup`.
Goals, stated before measuring: forward >= 0.8x and backward >= 0.7x the copy rate at t * n >= 2^26; the fused fp8 call
>= 1.5x faster than norm + quantize.  The card name and power limit are read (nvidia-smi --query-gpu, read-only) in the
same run.  Prints one JSON line.
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from cubecl_b200 import ComputeClient, TensorHandle, norm, quant  # noqa: E402
from cubecl_b200.quant import QuantScheme  # noqa: E402
from matmul_grouped_bench import torch_timed  # noqa: E402
from scan_bench import gpu_info, timed  # noqa: E402


def rows_of(c, t, n, seed):
    """a bf16 [t, n] device tensor: a random 1024-row block tiled down the rows (the values do not change the time)"""
    rng = np.random.default_rng(seed)
    block = (rng.standard_normal((min(t, 1024), n)).astype(np.float32).view(np.uint32) >> 16).astype(np.uint16)
    return TensorHandle.from_numpy(c, np.tile(block, (-(-t // block.shape[0]), 1))[:t], "bf16")


def run_row(c, t, n, iters, warmup, copy_gbps):
    import torch
    import torch.nn.functional as F
    x, dy = rows_of(c, t, n, 1), rows_of(c, t, n, 2)
    w = TensorHandle(rows_of(c, 1, n, 3).handle, [n], [1], "bf16")
    y = TensorHandle.empty_contiguous(c, [t, n], "bf16")
    dx = TensorHandle.empty_contiguous(c, [t, n], "bf16")
    rstd = TensorHandle.empty_contiguous(c, [t], "f32")
    dw = TensorHandle.empty_contiguous(c, [n], "f32")
    scheme = QuantScheme().with_value("e4m3").per_block(128, "f32")
    q = quant.alloc_quantized(c, [t, n], scheme)
    fwd_ms = timed(c, lambda: norm.forward(c, x, y, w, rstd=rstd), iters, warmup)
    bwd_ms = timed(c, lambda: norm.backward(c, dy, x, rstd, dx, w, dweight=dw), iters, warmup)
    fp8_ms = timed(c, lambda: norm.forward_quantized(c, x, q, w, rstd=rstd), iters, warmup)
    unfused_ms = timed(c, lambda: (norm.forward(c, x, y, w, rstd=rstd), quant.launch_quantize(c, y, q)), iters, warmup)
    c.sync()
    del q
    xt = torch.randn(t, n, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    wt = torch.randn(n, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    dyt = torch.randn(t, n, device="cuda", dtype=torch.bfloat16)
    t_fwd = torch_timed(lambda: F.rms_norm(xt, (n,), wt, 1e-6), iters, warmup)
    yt = F.rms_norm(xt, (n,), wt, 1e-6)
    t_bwd = torch_timed(lambda: torch.autograd.grad(yt, (xt, wt), dyt, retain_graph=True), iters, warmup)
    del xt, wt, dyt, yt
    torch.cuda.empty_cache()
    fb, bb, qb = 4 * t * n + 4 * t + 2 * n, 6 * t * n + 4 * t + 6 * n, 3 * t * n + t * n // 32 + 4 * t + 2 * n
    fwd_gbps, bwd_gbps = fb / fwd_ms / 1e6, bb / bwd_ms / 1e6
    return {"t": t, "n": n, "fwd_us": round(fwd_ms * 1e3, 1), "fwd_gbps": round(fwd_gbps, 1),
            "fwd_of_copy": round(fwd_gbps / copy_gbps, 3), "bwd_us": round(bwd_ms * 1e3, 1), "bwd_gbps": round(bwd_gbps, 1),
            "bwd_of_copy": round(bwd_gbps / copy_gbps, 3), "fp8_us": round(fp8_ms * 1e3, 1),
            "fp8_gbps": round(qb / fp8_ms / 1e6, 1), "norm_then_quantize_us": round(unfused_ms * 1e3, 1),
            "fp8_speedup": round(unfused_ms / fp8_ms, 2), "torch_fwd_us": round(t_fwd * 1e3, 1),
            "torch_bwd_us": round(t_bwd * 1e3, 1), "fwd_vs_torch": round(t_fwd / fwd_ms, 2), "bwd_vs_torch": round(t_bwd / bwd_ms, 2)}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--t", default="4096,16384,65536")
    ap.add_argument("--n", default="2048,4096,7168,8192,16384")
    args = ap.parse_args()
    c = ComputeClient.load(0)
    nbytes = 1 << 30
    src, dst = c.empty(nbytes), c.empty(nbytes)
    copy_ms = timed(c, lambda: c.probe_memcopy(dst, src, nbytes), args.iters, args.warmup)
    copy_gbps = 2 * nbytes / copy_ms / 1e6
    del src, dst
    rows = [run_row(c, t, n, args.iters, args.warmup, copy_gbps) for t in map(int, args.t.split(",")) for n in map(int, args.n.split(","))]
    big = [r for r in rows if r["t"] * r["n"] >= 1 << 26]
    goals = {"fwd_ge_0.8_copy": all(r["fwd_of_copy"] >= 0.8 for r in big), "bwd_ge_0.7_copy": all(r["bwd_of_copy"] >= 0.7 for r in big),
             "fp8_ge_1.5x_unfused": all(r["fp8_speedup"] >= 1.5 for r in rows)}
    print(json.dumps({"gpu": gpu_info(), "device": c.properties["name"], "memcopy_gbps": round(copy_gbps, 1), "goals_met": goals,
                      "rows": rows}))


if __name__ == "__main__":
    main()
