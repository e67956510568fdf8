"""Throughput of grouped and depthwise 2-D convolution (b200_conv2d_grouped*) on one GPU, next to same-run baselines.

    python tools/conv_grouped_bench.py [--iters 20] [--warmup 3]

bf16 NHWC at batch 64.  Rows: depthwise 3x3 layers of MobileNetV2 (112^2 x 96 stride 2, 56^2 x 144, 14^2 x 576) and 7x7 pad 3
layers of ConvNeXt-T (56^2 x 96, 28^2 x 192, 14^2 x 384, 7^2 x 768), each forward, data gradient and weight gradient; the
grouped 3x3 layers of ResNeXt-50 32x4d (56^2 x 128, Cg 4; 28^2 x 256, Cg 8; 14^2 x 512, Cg 16; 7^2 x 1024, Cg 32), the same
three passes; for the Cg 32 row also the per-group GEMM route timed by hand through b200_conv2d on channel slices; and one
wide-group layer on the GEMM route (28^2 x 512, groups 8, Cg 64).  The narrow rows run the direct kernels and the last two
run the GEMM, so the routing threshold (Cg >= 64 goes to the GEMM) has a measured workload on each side.

Each pass is timed with CUDA events around `--iters` back-to-back calls after `--warmup` untimed ones.  GB/s = algorithmic
bytes over that time: forward 2*N*H*W*C + 2*|w| + out_esz*N*OH*OW*Cout (bf16 out: 2), the data gradient the same reads and
writes with dy and dx, the weight gradient reads x and dy and writes dw.  `of_copy` = that rate over the same-run
b200_probe_memcopy rate.  TFLOP/s = 2*N*OH*OW*Cout*KH*KW*Cg over the time.  The FP32-FMA bound of the card is
2 * SMs * 128 lanes * the SM clock read in the same run.  cuDNN (torch channels_last, groups=) is a yardstick, reported only,
when torch has CUDA.  The card name and power limit are read (nvidia-smi --query-gpu, read-only) in the same run.  Prints one
JSON line.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from cubecl_b200 import ComputeClient, TensorHandle, conv  # noqa: E402
from scan_bench import gpu_info, timed  # noqa: E402

BATCH = 64
# (name, H = W, C, groups, kernel, stride, padding); Cout = C throughout
LAYERS = [
    ("mobilenetv2 dw 112x112x96 3x3/2", 112, 96, 96, 3, 2, 1),
    ("mobilenetv2 dw 56x56x144 3x3", 56, 144, 144, 3, 1, 1),
    ("mobilenetv2 dw 14x14x576 3x3", 14, 576, 576, 3, 1, 1),
    ("convnext-t dw 56x56x96 7x7", 56, 96, 96, 7, 1, 3),
    ("convnext-t dw 28x28x192 7x7", 28, 192, 192, 7, 1, 3),
    ("convnext-t dw 14x14x384 7x7", 14, 384, 384, 7, 1, 3),
    ("convnext-t dw 7x7x768 7x7", 7, 768, 768, 7, 1, 3),
    ("resnext50 32x4d 56x56x128 3x3 (Cg 4)", 56, 128, 32, 3, 1, 1),
    ("resnext50 32x4d 28x28x256 3x3 (Cg 8)", 28, 256, 32, 3, 1, 1),
    ("resnext50 32x4d 14x14x512 3x3 (Cg 16)", 14, 512, 32, 3, 1, 1),
    ("resnext50 32x4d 7x7x1024 3x3 (Cg 32)", 7, 1024, 32, 3, 1, 1),
    ("wide groups 28x28x512 3x3 groups 8 (Cg 64)", 28, 512, 8, 3, 1, 1),
]


def sm_clock_mhz() -> dict:
    r = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits"], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        return {"query_error": r.stdout.strip()}
    cur, mx = [int(s.strip()) for s in r.stdout.splitlines()[0].split(",")]
    return {"sm_mhz": cur, "max_sm_mhz": mx}


def cudnn_ms(h, c, groups, k, s, p, iters, warmup):
    try:
        import torch
    except ImportError:
        return None
    if not torch.cuda.is_available():
        return None
    x = torch.randn(BATCH, c, h, h, device="cuda", dtype=torch.bfloat16).to(memory_format=torch.channels_last)
    w = torch.randn(c, c // groups, k, k, device="cuda", dtype=torch.bfloat16).to(memory_format=torch.channels_last)
    torch.backends.cudnn.benchmark = True
    for _ in range(warmup):
        torch.nn.functional.conv2d(x, w, stride=s, padding=p, groups=groups)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        torch.nn.functional.conv2d(x, w, stride=s, padding=p, groups=groups)
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
    n_copy = 1 << 28
    src, dst = client.empty(n_copy * 4), client.empty(n_copy * 4)
    client.fill_modulo(src, "f32", n_copy, 8)
    ms = timed(client, lambda: client.probe_memcopy(dst, src, n_copy * 4), args.iters, args.warmup)
    copy_gbps = 2 * n_copy * 4 / ms / 1e6
    result["memcopy_gbps"] = round(copy_gbps, 1)
    del src, dst
    for name, h, c, groups, k, s, p in LAYERS:
        cg = c // groups
        x = TensorHandle.empty_contiguous(client, [BATCH, h, h, c], "bf16")
        w = TensorHandle.empty_contiguous(client, [c, k, k, cg], "bf16")
        client.fill_uniform(x.handle, "bf16", x.size(), 1, -1.0, 1.0)
        client.fill_uniform(w.handle, "bf16", w.size(), 2, -1.0, 1.0)
        oshape = conv.calculate_conv2d_output(x.shape, w.shape, s, p, 1, groups)
        out = TensorHandle.empty_contiguous(client, oshape, "bf16")
        dy = TensorHandle.empty_contiguous(client, oshape, "bf16")
        client.fill_uniform(dy.handle, "bf16", dy.size(), 3, -1.0, 1.0)
        dx = TensorHandle.empty_contiguous(client, x.shape, "bf16")
        dw = TensorHandle.empty_contiguous(client, w.shape, "bf16")
        nbytes = 2 * (x.size() + w.size() + out.size())
        flops = 2.0 * out.size() * k * k * cg
        passes = {
            "fwd": lambda: conv.launch(client, x, w, out, stride=s, padding=p, groups=groups),
            "dgrad": lambda: conv.backward_data(client, dy, w, dx, stride=s, padding=p, groups=groups),
            "wgrad": lambda: conv.backward_weight(client, x, dy, dw, stride=s, padding=p, groups=groups),
        }
        row = {"layer": name, "x": x.shape, "w": w.shape, "groups": groups, "stride": s, "padding": p, "bytes": nbytes, "flops": flops}
        for key, fn in passes.items():
            fn()
            client.sync()
            row[f"{key}_kernel"] = client.last_kernel()
            t = timed(client, fn, args.iters, args.warmup)
            client.sync()
            row[f"{key}_ms"] = t
            row[f"{key}_gbps"] = nbytes / (t * 1e-3) / 1e9
            row[f"{key}_of_copy"] = row[f"{key}_gbps"] / copy_gbps
            row[f"{key}_tflops"] = flops / (t * 1e-3) / 1e12
        if cg == 32:
            # the per-group GEMM route by hand: one b200_conv2d per group on channel slices
            def by_hand():
                for g in range(groups):
                    xg = TensorHandle(x.handle.offset(g * cg * 2), [BATCH, h, h, cg], list(x.strides), "bf16")
                    wg = TensorHandle(w.handle.offset(g * cg * k * k * cg * 2), [cg, k, k, cg], list(w.strides), "bf16")
                    og = TensorHandle(out.handle.offset(g * cg * 2), [*oshape[:3], cg], list(out.strides), "bf16")
                    conv.launch(client, xg, wg, og, stride=s, padding=p)
            t = timed(client, by_hand, args.iters, args.warmup)
            client.sync()
            row["fwd_gemm_per_group_ms"] = t
            row["fwd_gemm_per_group_tflops"] = flops / (t * 1e-3) / 1e12
        t_ms = cudnn_ms(h, c, groups, k, s, p, args.iters, args.warmup)
        if t_ms is not None:
            row["cudnn_fwd_ms"] = t_ms
        result["rows"].append(row)
        del x, w, out, dy, dx, dw
    clk = sm_clock_mhz()
    result["clock"] = clk
    if "max_sm_mhz" in clk:
        sms = client.properties["num_streaming_multiprocessors"]
        result["fp32_fma_tflops_at_max_clock"] = 2 * sms * 128 * clk["max_sm_mhz"] * 1e6 / 1e12
    print(json.dumps(result))


if __name__ == "__main__":
    main()
