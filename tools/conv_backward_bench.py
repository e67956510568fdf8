"""Throughput of the convolution gradients (b200_conv2d_backward_data / _weight) on one GPU, next to the forward b200_conv2d
and torch / cuDNN in the same run.

    python tools/conv_backward_bench.py [--iters 20] [--warmup 3]

Layers, bf16 NHWC at batch 64: ResNet-50's 3x3 stride-1 layers (56^2 x 64, 28^2 x 128, 14^2 x 256, 7^2 x 512, pad 1), a 3x3
stride-2 layer 56^2 x 128 -> 28^2 x 128 (pad 1) and a 1x1 stride-2 downsample 56^2 x 256 -> 28^2 x 512.  Each call is timed
with CUDA events around `--iters` back-to-back calls after `--warmup` untimed ones; TFLOP/s = the forward's algorithmic FLOPs
2 * N * OH * OW * Cout * KH * KW * C over that time (both gradients have the same count).  `dgrad_vs_fwd` / `wgrad_vs_fwd`
are the gradient's rate over the forward's on the same layer.  When torch has CUDA, torch.nn.grad.conv2d_input / _weight on
channels_last bf16 tensors (cuDNN) are reported as a yardstick.  The card name and power limit are read (nvidia-smi
--query-gpu, read-only) in the same run.  Prints one JSON line.
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from cubecl_b200 import ComputeClient, TensorHandle, conv  # noqa: E402
from scan_bench import gpu_info, timed  # noqa: E402

BATCH = 64
# (name, H = W, C, Cout, kernel, stride, padding)
LAYERS = [("resnet50 56x56x64 3x3", 56, 64, 64, 3, 1, 1), ("resnet50 28x28x128 3x3", 28, 128, 128, 3, 1, 1),
          ("resnet50 14x14x256 3x3", 14, 256, 256, 3, 1, 1), ("resnet50 7x7x512 3x3", 7, 512, 512, 3, 1, 1),
          ("56x56x128 3x3/2", 56, 128, 128, 3, 2, 1), ("downsample 56x56x256 1x1/2 -> 512", 56, 256, 512, 1, 2, 0)]


def torch_grad_ms(h, c, cout, k, s, p, iters, warmup):
    try:
        import torch
    except ImportError:
        return None
    if not torch.cuda.is_available():
        return None
    torch.backends.cudnn.benchmark = True
    x = torch.randn(BATCH, c, h, h, device="cuda", dtype=torch.bfloat16).to(memory_format=torch.channels_last)
    w = torch.randn(cout, c, k, k, device="cuda", dtype=torch.bfloat16).to(memory_format=torch.channels_last)
    oh = (h + 2 * p - k) // s + 1
    dy = torch.randn(BATCH, cout, oh, oh, device="cuda", dtype=torch.bfloat16).to(memory_format=torch.channels_last)

    def t(fn):
        for _ in range(warmup):
            fn()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / iters

    return (t(lambda: torch.nn.grad.conv2d_input(x.shape, w, dy, stride=s, padding=p)),
            t(lambda: torch.nn.grad.conv2d_weight(x, w.shape, dy, stride=s, padding=p)))


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
        oshape = conv.calculate_conv2d_output(x.shape, w.shape, s, p)
        dy = TensorHandle.empty_contiguous(client, oshape, "bf16")
        for i, t in enumerate((x, w, dy)):
            client.fill_uniform(t.handle, "bf16", t.size(), i + 1, -1.0, 1.0)
        out = TensorHandle.empty_contiguous(client, oshape, "bf16")
        dx = TensorHandle.empty_contiguous(client, x.shape, "bf16")
        dw = TensorHandle.empty_contiguous(client, w.shape, "bf16")
        fwd_ms = timed(client, lambda: conv.launch(client, x, w, out, stride=s, padding=p), args.iters, args.warmup)
        dgrad_ms = timed(client, lambda: conv.backward_data(client, dy, w, dx, stride=s, padding=p), args.iters, args.warmup)
        wgrad_ms = timed(client, lambda: conv.backward_weight(client, x, dy, dw, stride=s, padding=p), args.iters, args.warmup)
        client.sync()
        flops = 2.0 * BATCH * oshape[1] * oshape[2] * cout * k * k * c
        tf = lambda ms: flops / (ms * 1e-3) / 1e12  # noqa: E731
        row = {"layer": name, "x": [BATCH, h, h, c], "w": [cout, k, k, c], "stride": s, "padding": p,
               "fwd_ms": fwd_ms, "fwd_tflops": tf(fwd_ms), "dgrad_ms": dgrad_ms, "dgrad_tflops": tf(dgrad_ms),
               "wgrad_ms": wgrad_ms, "wgrad_tflops": tf(wgrad_ms), "dgrad_vs_fwd": fwd_ms / dgrad_ms, "wgrad_vs_fwd": fwd_ms / wgrad_ms}
        tg = torch_grad_ms(h, c, cout, k, s, p, args.iters, args.warmup)
        if tg is not None:
            row.update(cudnn_dgrad_ms=tg[0], cudnn_dgrad_tflops=tf(tg[0]), cudnn_wgrad_ms=tg[1], cudnn_wgrad_tflops=tf(tg[1]))
        result["rows"].append(row)
        del x, w, dy, out, dx, dw
    print(json.dumps(result))


if __name__ == "__main__":
    main()
