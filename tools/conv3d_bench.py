"""Throughput of the 3-D convolution (b200_conv3d and its gradients) on one GPU, next to the same-run b200_conv2d and
b200_matmul at the same implicit-GEMM shape, and torch / cuDNN as a yardstick.

    python tools/conv3d_bench.py [--iters 20] [--warmup 3]

Layers, bf16 NDHWC: the R3D-18 stem (3 -> 64, 3x7x7, stride (1,2,2), padding (1,3,3); the channel-padding path), the R3D-18
stage layers (3x3x3, padding 1), a stride-2 3x3x3 downsample and 3-D U-Net layers (3x3x3, padding 1); batches chosen so a
call takes >= ~50 us.  Each call is timed with CUDA events around `--iters` back-to-back calls after `--warmup` untimed ones;
TFLOP/s = 2 * N * OD * OH * OW * Cout * KD * KH * KW * C over that time (both gradients have the same count).  Columns:
  conv2d_*      the 2-D layer [N * D, H, W, C] with a 3x9 kernel and padding (1, 4) (stride-1 3x3x3 layers only): the same
                M, N, K and k-block count, so fwd_vs_conv2d isolates the cost of the 5-D walk (goal a: >= 0.9 where C >= 64);
  matmul_*      b200_matmul at (M, N, K) = (N * OD * OH * OW, Cout, KD * KH * KW * pad64(C));
  dgrad_vs_fwd  the data gradient's rate over the forward's (goal b: >= 0.9 on stride-1 layers with C >= 64);
  cudnn_*       torch's conv3d / conv_transpose gradients on channels_last_3d bf16 tensors, when torch has CUDA.
The card name, power limit and SM clock are read (nvidia-smi --query-gpu, read-only) in the same run.  Prints one JSON line.
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from cubecl_b200 import ComputeClient, TensorHandle, conv, conv3d, matmul  # noqa: E402
from conv_grouped_bench import sm_clock_mhz  # noqa: E402
from scan_bench import gpu_info, timed  # noqa: E402

# (name, N, D, H = W, C, Cout, kernel, stride, padding)
LAYERS = [("r3d18 stem 16x112^2x3 3x7x7/(1,2,2)", 4, 16, 112, 3, 64, (3, 7, 7), (1, 2, 2), (1, 3, 3)),
          ("r3d18 16x56^2x64 3x3x3", 4, 16, 56, 64, 64, (3, 3, 3), 1, 1),
          ("r3d18 8x28^2x128 3x3x3", 8, 8, 28, 128, 128, (3, 3, 3), 1, 1),
          ("r3d18 4x14^2x256 3x3x3", 16, 4, 14, 256, 256, (3, 3, 3), 1, 1),
          ("r3d18 2x7^2x512 3x3x3", 32, 2, 7, 512, 512, (3, 3, 3), 1, 1),
          ("16x56^2x64 -> 128 3x3x3/2", 4, 16, 56, 64, 128, (3, 3, 3), 2, 1),
          ("unet 64^3x32 3x3x3", 2, 64, 64, 32, 32, (3, 3, 3), 1, 1),
          ("unet 32^3x64 3x3x3", 4, 32, 32, 64, 64, (3, 3, 3), 1, 1),
          ("unet 16^3x128 3x3x3", 16, 16, 16, 128, 128, (3, 3, 3), 1, 1)]


def _t3(v):
    return (v,) * 3 if isinstance(v, int) else tuple(v)


def cudnn_ms(n, d, h, c, cout, k, s, p, iters, warmup):
    try:
        import torch
    except ImportError:
        return None
    if not torch.cuda.is_available():
        return None
    torch.backends.cudnn.benchmark = True
    cl = torch.channels_last_3d
    x = torch.randn(n, c, d, h, h, device="cuda", dtype=torch.bfloat16).to(memory_format=cl)
    w = torch.randn(cout, c, *k, device="cuda", dtype=torch.bfloat16).to(memory_format=cl)
    y = torch.nn.functional.conv3d(x, w, stride=s, padding=p)
    dy = torch.randn_like(y).to(memory_format=cl)

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

    return (t(lambda: torch.nn.functional.conv3d(x, w, stride=s, padding=p)),
            t(lambda: torch.nn.grad.conv3d_input(x.shape, w, dy, stride=s, padding=p)),
            t(lambda: torch.nn.grad.conv3d_weight(x, w.shape, dy, stride=s, padding=p)))


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if args.iters < 20:
        raise SystemExit("--iters must be >= 20")
    client = ComputeClient.load(0)
    result = {"gpu": gpu_info(), "clock": sm_clock_mhz(), "device": client.properties["name"], "iters": args.iters, "dtype": "bf16",
              "rows": []}
    tm = lambda fn: timed(client, fn, args.iters, args.warmup)  # noqa: E731
    for name, n, d, h, c, cout, k, s, p in LAYERS:
        x = TensorHandle.empty_contiguous(client, [n, d, h, h, c], "bf16")
        w = TensorHandle.empty_contiguous(client, [cout, *k, c], "bf16")
        oshape = conv3d.calculate_conv3d_output(x.shape, w.shape, s, p)
        dy = TensorHandle.empty_contiguous(client, oshape, "bf16")
        for i, t in enumerate((x, w, dy)):
            client.fill_uniform(t.handle, "bf16", t.size(), i + 1, -1.0, 1.0)
        out = TensorHandle.empty_contiguous(client, oshape, "bf16")
        dx = TensorHandle.empty_contiguous(client, x.shape, "bf16")
        dw = TensorHandle.empty_contiguous(client, w.shape, "bf16")
        fwd = tm(lambda: conv3d.launch(client, x, w, out, stride=s, padding=p))
        dgrad = tm(lambda: conv3d.backward_data(client, dy, w, dx, stride=s, padding=p))
        wgrad = tm(lambda: conv3d.backward_weight(client, x, dy, dw, stride=s, padding=p))
        M, K = oshape[0] * oshape[1] * oshape[2] * oshape[3], k[0] * k[1] * k[2] * ((c + 63) // 64 * 64)
        flops = 2.0 * M * cout * k[0] * k[1] * k[2] * c
        tf = lambda ms: flops / (ms * 1e-3) / 1e12  # noqa: E731
        row = {"layer": name, "x": x.shape, "w": w.shape, "stride": s, "padding": p, "fwd_ms": fwd, "fwd_tflops": tf(fwd),
               "dgrad_ms": dgrad, "dgrad_tflops": tf(dgrad), "wgrad_ms": wgrad, "wgrad_tflops": tf(wgrad), "dgrad_vs_fwd": fwd / dgrad}
        a = TensorHandle.empty_contiguous(client, [M, K], "bf16")
        b = TensorHandle.empty_contiguous(client, [K, cout], "bf16")
        mo = TensorHandle.empty_contiguous(client, [M, cout], "bf16")
        mm = tm(lambda: matmul.launch(client, a, b, mo))
        row.update(matmul_ms=mm, matmul_tflops=tf(mm), fwd_vs_matmul=mm / fwd)
        if _t3(s) == (1, 1, 1) and k == (3, 3, 3):
            x2 = TensorHandle(x.handle, [n * d, h, h, c], x.strides[1:], "bf16")
            w2 = TensorHandle.empty_contiguous(client, [cout, 3, 9, c], "bf16")
            o2 = TensorHandle.empty_contiguous(client, conv.calculate_conv2d_output(x2.shape, w2.shape, 1, (1, 4)), "bf16")
            c2 = tm(lambda: conv.launch(client, x2, w2, o2, padding=(1, 4)))
            row.update(conv2d_ms=c2, conv2d_tflops=tf(c2), fwd_vs_conv2d=c2 / fwd)
            if c >= 64:
                row.update(goal_a_met=c2 / fwd >= 0.9, goal_b_met=fwd / dgrad >= 0.9)
        cd = cudnn_ms(n, d, h, c, cout, k, _t3(s), _t3(p), args.iters, args.warmup)
        if cd is not None:
            row.update(cudnn_fwd_ms=cd[0], cudnn_fwd_tflops=tf(cd[0]), cudnn_dgrad_ms=cd[1], cudnn_dgrad_tflops=tf(cd[1]),
                       cudnn_wgrad_ms=cd[2], cudnn_wgrad_tflops=tf(cd[2]))
        client.sync()
        result["rows"].append(row)
        del x, w, dy, out, dx, dw, a, b, mo
    print(json.dumps(result))


if __name__ == "__main__":
    main()
