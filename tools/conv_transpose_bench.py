"""Throughput of the transposed convolution (b200_conv_transpose2d / 3d) on one GPU, next to the same-run per-phase data
gradient on the identical problem, the same-run forward convolution with the same FLOPs, and torch / cuDNN as a yardstick.

    python tools/conv_transpose_bench.py [--iters 20] [--warmup 3]

Layers, bf16 channels-last: U-Net decoder upsampling 2x2 / 2 and 3x3 / 2 (padding 1, output padding 1) at 28^2 -> 56^2 and
56^2 -> 112^2 with C = Cout in {64, 128, 256}, a DCGAN 4x4 / 2 (padding 1) generator layer, a 3-D U-Net 2x2x2 / 2 layer at
16^3 -> 32^3 x 64 and one stride-1 3x3 layer.  Each call is timed with CUDA events around `--iters` back-to-back calls after
`--warmup` untimed ones; TFLOP/s = 2 * N * H * W (* D) * Cin * KH * KW (* KD) * Cout over that time.  Columns:
  tconv_*         b200_conv_transpose2d / 3d (stride > 1: every phase in phase-batched launches; stride 1: the forward kernel);
  dgrad_*         b200_conv2d_backward_data / b200_conv3d_backward_data with x as dy: one GEMM launch per phase, plus a memset
                  when a phase receives no tap;
  fwd_*           b200_conv2d / b200_conv3d of an output-shaped input with w as its weights: the convolution whose data
                  gradient this is, with the same FLOPs;
  batched_vs_dgrad  dgrad time over tconv time (goal: >= 1.2 on the stride-2 layers with C, Cout >= 64);
  cudnn_*         torch's conv_transpose2d / 3d on channels_last bf16 tensors, when torch has CUDA.
The card name, power limit and SM clock are read (nvidia-smi --query-gpu, read-only) in the same run.  Prints one JSON line.
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from cubecl_b200 import ComputeClient, TensorHandle, conv, conv3d, conv_transpose  # noqa: E402
from conv_grouped_bench import sm_clock_mhz  # noqa: E402
from scan_bench import gpu_info, timed  # noqa: E402

# (name, N, input spatial extents, Cin, Cout, kernel, stride, padding, output padding)
LAYERS = [(f"unet {k}x{k}/2 {h}^2->{2 * h}^2 x{c}", n, (h, h), c, c, (k, k), 2, p, op)
          for k, p, op in ((2, 0, 0), (3, 1, 1)) for h, n in ((28, 32), (56, 8)) for c in (64, 128, 256)]
LAYERS += [("dcgan 4x4/2 16^2->32^2 256->128", 64, (16, 16), 256, 128, (4, 4), 2, 1, 0),
           ("unet3d 2x2x2/2 16^3->32^3 x64", 2, (16, 16, 16), 64, 64, (2, 2, 2), 2, 0, 0),
           ("stride-1 3x3 56^2 x128", 16, (56, 56), 128, 128, (3, 3), 1, 1, 0)]


def cudnn_ms(n, hw, c, cout, k, s, p, op, iters, warmup):
    try:
        import torch
    except ImportError:
        return None
    if not torch.cuda.is_available():
        return None
    torch.backends.cudnn.benchmark = True
    three = len(hw) == 3
    cl = torch.channels_last_3d if three else torch.channels_last
    x = torch.randn(n, c, *hw, device="cuda", dtype=torch.bfloat16).to(memory_format=cl)
    w = torch.randn(c, cout, *k, device="cuda", dtype=torch.bfloat16).to(memory_format=cl)
    f = torch.nn.functional.conv_transpose3d if three else torch.nn.functional.conv_transpose2d
    fn = lambda: f(x, w, stride=s, padding=p, output_padding=op)  # noqa: E731
    for _ in range(warmup):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
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
    result = {"gpu": gpu_info(), "clock": sm_clock_mhz(), "device": client.properties["name"], "iters": args.iters, "dtype": "bf16",
              "rows": []}
    tm = lambda fn: timed(client, fn, args.iters, args.warmup)  # noqa: E731
    for name, n, hw, c, cout, k, s, p, op in LAYERS:
        mod = conv3d if len(hw) == 3 else conv
        x = TensorHandle.empty_contiguous(client, [n, *hw, c], "bf16")
        w = TensorHandle.empty_contiguous(client, [c, *k, cout], "bf16")
        oshape = conv_transpose.calculate_conv_transpose_output(x.shape, w.shape, s, p, op)
        y = TensorHandle.empty_contiguous(client, oshape, "bf16")
        for i, t in enumerate((x, w, y)):
            client.fill_uniform(t.handle, "bf16", t.size(), i + 1, -1.0, 1.0)
        out = TensorHandle.empty_contiguous(client, oshape, "bf16")
        dx = TensorHandle.empty_contiguous(client, oshape, "bf16")
        fo = TensorHandle.empty_contiguous(client, x.shape, "bf16")
        tconv = tm(lambda: conv_transpose.launch(client, x, w, out, stride=s, padding=p))
        tconv_kernel = client.last_kernel()
        dgrad = tm(lambda: mod.backward_data(client, x, w, dx, stride=s, padding=p))
        fwd = tm(lambda: mod.launch(client, y, w, fo, stride=s, padding=p))
        flops = 2.0 * n * c * cout
        for e in (*hw, *k):
            flops *= e
        tf = lambda ms: flops / (ms * 1e-3) / 1e12  # noqa: E731
        row = {"layer": name, "x": x.shape, "w": w.shape, "out": oshape, "stride": s, "padding": p, "output_padding": op,
               "tconv_kernel": tconv_kernel, "tconv_ms": tconv, "tconv_tflops": tf(tconv), "dgrad_ms": dgrad, "dgrad_tflops": tf(dgrad),
               "fwd_ms": fwd, "fwd_tflops": tf(fwd), "batched_vs_dgrad": dgrad / tconv, "tconv_vs_fwd": fwd / tconv}
        if s == 2 and min(c, cout) >= 64:
            row["goal_met"] = dgrad / tconv >= 1.2
        cd = cudnn_ms(n, hw, c, cout, k, s, p, op, args.iters, args.warmup)
        if cd is not None:
            row.update(cudnn_ms=cd, cudnn_tflops=tf(cd))
        client.sync()
        result["rows"].append(row)
        del x, w, y, out, dx, fo
    print(json.dumps(result))


if __name__ == "__main__":
    main()
