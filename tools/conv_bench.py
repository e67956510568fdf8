"""Throughput of the 2-D convolution (b200_conv2d) on one GPU, next to same-run baselines.

    python tools/conv_bench.py [--iters 20] [--warmup 3]

Layers, bf16 NHWC in and out at batch 64: ResNet-50's 3x3 layers 56^2 x 64 -> 64, 28^2 x 128 -> 128, 14^2 x 256 -> 256 and
7^2 x 512 -> 512 (stride 1, pad 1), its 7x7 / 2 stem (224^2 x 3 -> 64, pad 3) and a 32^2 x 512 -> 512 3x3 layer.  Each row is
timed with CUDA events around `--iters` back-to-back calls after `--warmup` untimed ones; TFLOP/s = the algorithmic FLOPs
2 * N * OH * OW * Cout * KH * KW * C over that time.  Baselines in the same run: the bf16 b200_matmul at the same (M, N, K) =
(N * OH * OW, Cout, KH * KW * C) with dense K-major operands (the mainloop ceiling; `ratio` = matmul time / conv time), and,
when torch has CUDA, torch's conv2d on channels_last bf16 tensors (cuDNN), reported only.  The card name and power limit are
read (nvidia-smi --query-gpu, read-only) in the same run.  Prints one JSON line.
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from cubecl_b200 import ComputeClient, TensorHandle, conv, matmul  # noqa: E402
from scan_bench import gpu_info, timed  # noqa: E402

BATCH = 64
# (name, H = W, C, Cout, kernel, stride, padding)
LAYERS = [("resnet50 56x56x64 3x3", 56, 64, 64, 3, 1, 1), ("resnet50 28x28x128 3x3", 28, 128, 128, 3, 1, 1),
          ("resnet50 14x14x256 3x3", 14, 256, 256, 3, 1, 1), ("resnet50 7x7x512 3x3", 7, 512, 512, 3, 1, 1),
          ("resnet50 stem 224x224x3 7x7/2", 224, 3, 64, 7, 2, 3), ("32x32x512 3x3", 32, 512, 512, 3, 1, 1)]


def torch_conv_ms(h, c, cout, k, s, p, iters, warmup):
    try:
        import torch
    except ImportError:
        return None
    if not torch.cuda.is_available():
        return None
    x = torch.randn(BATCH, c, h, h, device="cuda", dtype=torch.bfloat16).to(memory_format=torch.channels_last)
    w = torch.randn(cout, c, k, k, device="cuda", dtype=torch.bfloat16).to(memory_format=torch.channels_last)
    torch.backends.cudnn.benchmark = True
    for _ in range(warmup):
        torch.nn.functional.conv2d(x, w, stride=s, padding=p)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        torch.nn.functional.conv2d(x, w, stride=s, padding=p)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if args.iters < 20:
        raise SystemExit("--iters must be >= 20")
    client = ComputeClient.load(0)
    result = {"gpu": gpu_info(), "device": client.properties["name"], "iters": args.iters, "batch": BATCH, "dtype": "bf16", "rows": []}
    for name, h, c, cout, k, s, p in LAYERS:
        x = TensorHandle.empty_contiguous(client, [BATCH, h, h, c], "bf16")
        w = TensorHandle.empty_contiguous(client, [cout, k, k, c], "bf16")
        client.fill_uniform(x.handle, "bf16", x.size(), 1, -1.0, 1.0)
        client.fill_uniform(w.handle, "bf16", w.size(), 2, -1.0, 1.0)
        oshape = conv.calculate_conv2d_output(x.shape, w.shape, s, p)
        out = TensorHandle.empty_contiguous(client, oshape, "bf16")
        conv_ms = timed(client, lambda: conv.launch(client, x, w, out, stride=s, padding=p), args.iters, args.warmup)
        client.sync()
        M, N, K = BATCH * oshape[1] * oshape[2], cout, k * k * c
        flops = 2.0 * M * N * K
        a = TensorHandle.empty_contiguous(client, [M, K], "bf16")
        bt = TensorHandle.empty_contiguous(client, [N, K], "bf16")
        client.fill_uniform(a.handle, "bf16", M * K, 3, -1.0, 1.0)
        client.fill_uniform(bt.handle, "bf16", N * K, 4, -1.0, 1.0)
        b = TensorHandle(bt.handle, [K, N], [1, K], "bf16")   # [N, K] storage read as the [K, N] operand (K-major)
        mo = TensorHandle.empty_contiguous(client, [M, N], "bf16")
        mm_ms = timed(client, lambda: matmul.launch(client, a, b, mo), args.iters, args.warmup)
        client.sync()
        row = {"layer": name, "x": [BATCH, h, h, c], "w": [cout, k, k, c], "stride": s, "padding": p, "gemm_mnk": [M, N, K],
               "conv_ms": conv_ms, "conv_tflops": flops / (conv_ms * 1e-3) / 1e12, "matmul_ms": mm_ms,
               "matmul_tflops": flops / (mm_ms * 1e-3) / 1e12, "ratio": mm_ms / conv_ms,
               "bytes": 2 * (x.size() + w.size() + out.size())}
        t_ms = torch_conv_ms(h, c, cout, k, s, p, args.iters, args.warmup)
        if t_ms is not None:
            row["cudnn_ms"] = t_ms
            row["cudnn_tflops"] = flops / (t_ms * 1e-3) / 1e12
        result["rows"].append(row)
        del x, w, out, a, bt, b, mo
    print(json.dumps(result))


if __name__ == "__main__":
    main()
