"""Throughput of the quantized matmul (b200_matmul_quantized) on one GPU, next to same-run baselines.

    python tools/qmatmul_bench.py [--iters 20] [--warmup 3]

Rows at M = N = K = 8192 with bf16 output: Q8S per-tensor x per-tensor, Q8S/128/f32 x Q8S/128/f32, Q8S/32/f32 x Q8S/32/f32 and
Q8S/128/f32 x Q4S/32/f16 (the last one includes its widening pass).  Baselines in the same run: the s8 -> i32 b200_matmul
(the int8 mainloop ceiling), the bf16 b200_matmul, and what users do without this entry point: dequantize both Q8S/128
operands to bf16, then the bf16 matmul.  Each row is timed with CUDA events around `--iters` back-to-back calls after
`--warmup` untimed ones; TOPS = 2 M N K / time.  The card name and power limit are read (nvidia-smi --query-gpu, read-only)
in the same run.  Prints one JSON line.
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
from scan_bench import gpu_info, timed  # noqa: E402

M = N = K = 8192


def operand(client, scheme: QuantScheme, rows: int, seed: int) -> QuantizedTensor:
    """Random codes and scales of a [rows, K] operand (the values do not change the GEMM's work)."""
    rng = np.random.default_rng(seed)
    codes = rng.integers(0, 256, size=(rows, K * quant.BITS[scheme.value] // 8), dtype=np.uint8)
    vals = TensorHandle.from_numpy(client, codes, quant.VALUE_DTYPES.get(scheme.value, "u8"))
    scales = None
    if scheme.block:
        s = rng.uniform(0.5, 2.0, size=(rows, K // scheme.block)).astype(np.float32)
        raw = s if scheme.block_scale == "f32" else s.astype(np.float16)
        scales = TensorHandle.from_numpy(client, raw, scheme.block_scale)
    tensor = TensorHandle.from_numpy(client, np.array([0.01], np.float32), "f32") if scheme.has_tensor else None
    return QuantizedTensor(vals, scales, tensor, scheme, [rows, K])


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if args.iters < 20:
        raise SystemExit("--iters must be >= 20")
    client = ComputeClient.load(0)
    tops = lambda ms: 2.0 * M * N * K / (ms * 1e-3) / 1e12   # noqa: E731
    result = {"gpu": gpu_info(), "device": client.properties["name"], "iters": args.iters, "shape": [M, N, K], "rows": []}
    out = TensorHandle.empty_contiguous(client, [M, N], "bf16")
    q8t = QuantScheme().with_value("q8s").per_tensor()
    q8_128 = QuantScheme().with_value("q8s").per_block(128, "f32")
    q8_32 = QuantScheme().with_value("q8s").per_block(32, "f32")
    q4_32 = QuantScheme().with_value("q4s").per_block(32, "f16")
    for name, sa, sb in (("q8s_tensor x q8s_tensor", q8t, q8t), ("q8s/128/f32 x q8s/128/f32", q8_128, q8_128),
                         ("q8s/32/f32 x q8s/32/f32", q8_32, q8_32), ("q8s/128/f32 x q4s/32/f16", q8_128, q4_32)):
        a, b = operand(client, sa, M, 1), operand(client, sb, N, 2)
        ms = timed(client, lambda: matmul.launch_quantized(client, a, b, out), args.iters, args.warmup)
        result["rows"].append({"row": name, "ms": ms, "tops": tops(ms)})
    # baselines
    i8a = TensorHandle.from_numpy(client, np.random.default_rng(3).integers(-127, 128, size=(M, K), dtype=np.int8), "i8")
    i8b = TensorHandle.from_numpy(client, np.random.default_rng(4).integers(-127, 128, size=(N, K), dtype=np.int8), "i8")
    i32 = TensorHandle.empty_contiguous(client, [M, N], "i32")
    rhs_t = TensorHandle(i8b.handle, [K, N], [1, K], "i8")   # [N, K] storage read as the [K, N] operand (K-major)
    ms = timed(client, lambda: matmul.launch(client, i8a, rhs_t, i32), args.iters, args.warmup)
    result["rows"].append({"row": "s8 -> i32 b200_matmul (baseline)", "ms": ms, "tops": tops(ms)})
    bfa = TensorHandle.empty_contiguous(client, [M, K], "bf16")
    bfb = TensorHandle.empty_contiguous(client, [N, K], "bf16")
    client.fill_uniform(bfa.handle, "bf16", M * K, 5, -1.0, 1.0)
    client.fill_uniform(bfb.handle, "bf16", N * K, 6, -1.0, 1.0)
    bfb_t = TensorHandle(bfb.handle, [K, N], [1, K], "bf16")
    ms = timed(client, lambda: matmul.launch(client, bfa, bfb_t, out), args.iters, args.warmup)
    result["rows"].append({"row": "bf16 b200_matmul (baseline)", "ms": ms, "tops": tops(ms)})
    qa, qb = operand(client, q8_128, M, 1), operand(client, q8_128, N, 2)

    def deq_then_bf16():
        quant.launch_dequantize(client, qa, bfa)
        quant.launch_dequantize(client, qb, bfb)
        matmul.launch(client, bfa, bfb_t, out)
    ms = timed(client, deq_then_bf16, args.iters, args.warmup)
    result["rows"].append({"row": "dequantize q8s/128 x2 + bf16 b200_matmul (baseline)", "ms": ms, "tops": tops(ms)})
    client.sync()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
