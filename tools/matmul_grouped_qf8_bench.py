"""Throughput of the fp8-quantized grouped matmul (b200_matmul_grouped_quantized_fp8) on mixture-of-experts layer shapes, next to
the ways a user would otherwise run an fp8 MoE checkpoint, alternating in one process.

    python tools/matmul_grouped_qf8_bench.py [--iters 20] [--warmup 3] [--rows deepseek,mixtral,qwen3]

Rows: the gate-up forward x [T, hidden] @ W_g^T of tools/matmul_grouped_bench.py's three layers (deepseek G = 32, 7168 -> 4096;
mixtral G = 8, 4096 -> 28672; qwen3 G = 128, 2048 -> 1536), T = 32768, with its balanced and seeded skewed routing
(`routing()`, imported from there).  Operands: e4m3 activations with per-block-128 f32 scales (1 x 128), e4m3 weights
[G, N, hidden] with 128 x 128 scales passed through the header's repeat recipe, i.e. as a per-block-128 f32 operand (the kernel
reads the same bytes whatever the scale values); output bf16.  TFLOP/s = 2 T N hidden / time.
Variants:
  grouped        b200_matmul_grouped_quantized_fp8
  grouped_quant  b200_quantize of x (bf16 -> e4m3 / 128) then the grouped call
  batched        b200_matmul_quantized_fp8 on [G, T / G, .] views of the same bytes (balanced routing only)
  loop           one b200_matmul_quantized_fp8 per non-empty group, sizes known on the host
  dequant_bf16   b200_dequantize of both operands to bf16, then b200_matmul_grouped
  bf16           b200_matmul_grouped on bf16 operands
  torch          torch.nn.functional.scaled_grouped_mm with row-wise scales on its own copies, or "refused"
Each time is the CUDA-event mean of `--iters` back-to-back calls after `--warmup` untimed ones; the variants of a row alternate
for two rounds, and each reports the mean of the rounds and `spread` = |r1 - r2| / min(r1, r2).  Goals, stated before measuring:
  (a) balanced rows at >= 0.9x the same-run batched b200_matmul_quantized_fp8;
  (b) G = 128 rows, balanced and skewed, at >= 1.5x the per-group loop;
  (c) balanced G = 32 and G = 128 rows at >= 1.0x dequantize-then-bf16-grouped.
The ratio to bf16 b200_matmul_grouped is recorded without a goal.  The card name, power limit and SM clock are read
(nvidia-smi --query-gpu, read-only) in the same run.  Prints one JSON line.
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from cubecl_b200 import ComputeClient, TensorHandle, matmul, quant  # noqa: E402
from cubecl_b200.quant import QuantScheme, QuantizedTensor  # noqa: E402
from conv_grouped_bench import sm_clock_mhz  # noqa: E402
from matmul_grouped_bench import MODELS, T, routing, torch_timed  # noqa: E402
from scan_bench import gpu_info, timed  # noqa: E402


def rows_of(q: QuantizedTensor, shape, row0: int, rows: int) -> QuantizedTensor:
    """`rows` rows of a per-block-128 f32 operand starting at row0, as a QuantizedTensor of `shape`."""
    K = q.shape[-1]
    nb = K // 128
    v = TensorHandle.new_contiguous(shape, q.values.handle.offset(row0 * K, rows * K), q.values.dtype)
    s = TensorHandle.new_contiguous(list(shape[:-1]) + [nb], q.block_scales.handle.offset(row0 * nb * 4, rows * nb * 4), "f32")
    return QuantizedTensor(v, s, None, q.scheme, list(shape))


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rows", default="deepseek,mixtral,qwen3")
    args = ap.parse_args()
    if args.iters < 20:
        raise SystemExit("--iters must be >= 20")
    import torch
    F = torch.nn.functional
    client = ComputeClient.load(0)
    result = {"gpu": gpu_info(), "clock": sm_clock_mhz(), "device": client.properties["name"], "iters": args.iters, "T": T, "rows": []}
    s128 = QuantScheme().with_value("e4m3").per_block(128, "f32")

    for model in args.rows.split(","):
        G, H, N = MODELS[model]
        x = TensorHandle.empty_contiguous(client, [T, H], "bf16")
        w = TensorHandle.empty_contiguous(client, [G, N, H], "bf16")
        for i, t in enumerate((x, w)):
            client.fill_uniform(t.handle, "bf16", t.size(), i + 1, -1.0, 1.0)
        qx, qw = quant.quantize(client, x, s128), quant.quantize(client, w, s128)
        xd, wd = TensorHandle.empty_contiguous(client, [T, H], "bf16"), TensorHandle.empty_contiguous(client, [G, N, H], "bf16")
        y = TensorHandle.empty_contiguous(client, [T, N], "bf16")
        wt = TensorHandle(w.handle, [G, H, N], [N * H, 1, H], "bf16")       # rhs [G, K, N]: W_g^T
        wdt = TensorHandle(wd.handle, [G, H, N], [N * H, 1, H], "bf16")
        client.sync()
        # torch's copies of the same codes with one f32 scale per row (row-wise), its scaled_grouped_mm's recipe on Hopper
        a8 = torch.from_numpy(qx.values.to_numpy(client).view(np.uint8).reshape(T, H).copy()).cuda().view(torch.float8_e4m3fn)
        b8 = torch.from_numpy(qw.values.to_numpy(client).view(np.uint8).reshape(G, N, H).copy()).cuda().view(torch.float8_e4m3fn)
        tsa, tsb = torch.ones(T, device="cuda"), torch.ones(G, N, device="cuda")
        for skewed in (False, True):
            sizes = routing(G, skewed)
            offs_np = np.cumsum(sizes).astype(np.int32)
            offs = TensorHandle.from_numpy(client, offs_np, "i32")
            toffs = torch.from_numpy(offs_np).cuda()
            bounds = [(int(o - s), int(o)) for s, o in zip(sizes, offs_np)]
            row = {"model": model, "routing": "skewed" if skewed else "balanced", "G": G, "hidden": H, "N": N, "T": T,
                   "empty_groups": sum(1 for s in sizes if s == 0), "max_group": max(sizes)}
            loop_ops = [(rows_of(qx, [hi - lo, H], lo, hi - lo), rows_of(qw, [N, H], g * N, N),
                         TensorHandle(y.handle.offset(lo * N * 2), [hi - lo, N], [N, 1], "bf16"))
                        for g, (lo, hi) in enumerate(bounds) if hi > lo]

            def loop():
                for a, b, o in loop_ops:
                    matmul.launch_quantized_fp8(client, a, b, o)

            def quant_then_grouped():
                quant.launch_quantize(client, x, qx)
                matmul.launch_grouped_quantized_fp8(client, qx, qw, offs, y)

            def dequant_then_bf16():
                quant.launch_dequantize(client, qx, xd)
                quant.launch_dequantize(client, qw, wd)
                matmul.launch_grouped(client, xd, wdt, offs, y)

            variants = {"grouped": lambda: matmul.launch_grouped_quantized_fp8(client, qx, qw, offs, y),
                        "grouped_quant": quant_then_grouped, "loop": loop, "dequant_bf16": dequant_then_bf16,
                        "bf16": lambda: matmul.launch_grouped(client, x, wt, offs, y)}
            if not skewed:
                n = T // G
                bx = QuantizedTensor(qx.values, qx.block_scales, None, s128, [G, n, H])
                yb = TensorHandle(y.handle, [G, n, N], [n * N, N, 1], "bf16")
                variants["batched"] = lambda: matmul.launch_quantized_fp8(client, bx, qw, yb)

            def torch_call():
                return F.scaled_grouped_mm(a8, b8.transpose(-2, -1), tsa, F.ScalingType.RowWise, tsb, F.ScalingType.RowWise,
                                           offs=toffs, output_dtype=torch.bfloat16)
            try:
                torch_call()
                torch.cuda.synchronize()
                timers = {**{k: ("b200", f) for k, f in variants.items()}, "torch": ("torch", torch_call)}
            except Exception as e:   # noqa: BLE001 -- a refusal is reported as such
                row["torch"] = f"refused: {type(e).__name__}: {str(e).splitlines()[0][:200]}"
                timers = {k: ("b200", f) for k, f in variants.items()}
            rounds = {name: [] for name in timers}
            for _ in range(2):
                for name, (kind, fn) in timers.items():
                    rounds[name].append(torch_timed(fn, args.iters, args.warmup) if kind == "torch" else timed(client, fn, args.iters, args.warmup))
            flops = 2.0 * T * N * H
            for name, ms in rounds.items():
                row[f"{name}_ms"] = sum(ms) / 2
                row[f"{name}_tflops"] = flops / (row[f"{name}_ms"] * 1e-3) / 1e12
                row[f"{name}_spread"] = abs(ms[0] - ms[1]) / min(ms)
            client.sync()
            row["vs_bf16"] = row["bf16_ms"] / row["grouped_ms"]
            if not skewed:
                row["vs_batched"] = row["batched_ms"] / row["grouped_ms"]
                row["goal_a_met"] = row["vs_batched"] >= 0.9
            if G == 128:
                row["vs_loop"] = row["loop_ms"] / row["grouped_ms"]
                row["goal_b_met"] = row["vs_loop"] >= 1.5
            if not skewed and G in (32, 128):
                row["vs_dequant_bf16"] = row["dequant_bf16_ms"] / row["grouped_ms"]
                row["goal_c_met"] = row["vs_dequant_bf16"] >= 1.0
            result["rows"].append(row)
            print(json.dumps(row), file=sys.stderr, flush=True)
        del x, w, qx, qw, xd, wd, y, a8, b8
        torch.cuda.empty_cache()
        client.sync()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
