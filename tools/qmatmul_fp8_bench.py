"""Throughput of the fp8-quantized matmul (b200_matmul_quantized_fp8) on one GPU, next to same-run baselines.

    python tools/qmatmul_fp8_bench.py [--iters 20] [--warmup 3] [--rounds 2]

Rows at M = N = K = 8192 with bf16 output: e4m3/128/f32 x e4m3/128/f32, e4m3/32/f32 x e4m3/32/f32, e4m3 per-tensor x
per-tensor, and e5m2/128/f32 x e4m3/128/f32.  Baselines in the same run: the bf16 b200_matmul, the fp8 b200_matmul on the
same codes (widened to f16 before its GEMM), dequantize both e4m3/128 operands to bf16 then the bf16 b200_matmul, and torch's
F.scaled_mm (RowWise, and BlockWise1x128 x BlockWise128x128 when this torch accepts it) as a yardstick.  Every row is timed
with CUDA events around `--iters` back-to-back calls after `--warmup` untimed ones; the rows alternate in one process for
`--rounds` rounds, and each row reports the mean over rounds, TFLOP/s = 2 M N K / time, and the spread (max - min) / mean
between rounds.  The card name and power limit are read (nvidia-smi --query-gpu, read-only) in the same run.  Prints one
JSON line.
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
    """Random finite codes and scales of a [rows, K] operand (the values do not change the GEMM's work)."""
    rng = np.random.default_rng(seed)
    codes = rng.integers(0, 0x70, size=(rows, K), dtype=np.uint8) | (rng.integers(0, 2, size=(rows, K), dtype=np.uint8) << 7)
    vals = TensorHandle.from_numpy(client, codes, quant.VALUE_DTYPES[scheme.value])
    scales = None
    if scheme.block:
        scales = TensorHandle.from_numpy(client, rng.uniform(0.5, 2.0, size=(rows, K // scheme.block)).astype(np.float32), "f32")
    tensor = TensorHandle.from_numpy(client, np.array([0.01], np.float32), "f32") if scheme.has_tensor else None
    return QuantizedTensor(vals, scales, tensor, scheme, [rows, K])


def torch_rows(qa):
    """F.scaled_mm on the e4m3/128 operands: {row name: callable}, with a note for each recipe this torch refuses."""
    try:
        import torch
        import torch.nn.functional as F
    except Exception as e:   # noqa: BLE001
        return {}, {"torch": f"not importable: {e}"}
    rows, notes = {}, {}
    rng = np.random.default_rng(7)
    a8 = torch.from_numpy(rng.integers(0, 0x70, size=(M, K), dtype=np.uint8)).view(torch.float8_e4m3fn).cuda()
    b8 = torch.from_numpy(rng.integers(0, 0x70, size=(N, K), dtype=np.uint8)).view(torch.float8_e4m3fn).cuda()
    cases = {
        "torch F.scaled_mm RowWise (yardstick)": (torch.ones(M, 1, device="cuda"), F.ScalingType.RowWise,
                                                  torch.ones(1, N, device="cuda"), F.ScalingType.RowWise),
        "torch F.scaled_mm BlockWise1x128 x BlockWise128x128 (yardstick)": (
            torch.ones(K // 128, M, device="cuda").t(), F.ScalingType.BlockWise1x128,
            torch.ones(N // 128, K // 128, device="cuda"), F.ScalingType.BlockWise128x128)}
    for name, (sa, ra, sb, rb) in cases.items():
        def fn(sa=sa, ra=ra, sb=sb, rb=rb):
            return F.scaled_mm(a8, b8.t(), sa, ra, sb, rb, output_dtype=torch.bfloat16)
        try:
            fn()
            torch.cuda.synchronize()
            rows[name] = fn
        except Exception as e:   # noqa: BLE001 -- a recipe this torch refuses is recorded, not fatal
            notes[name] = f"refused: {type(e).__name__}: {str(e).splitlines()[0][:160]}"
    return rows, notes


def torch_timed(fn, iters: int, warmup: int) -> float:
    import torch
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
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    if args.iters < 20:
        raise SystemExit("--iters must be >= 20")
    client = ComputeClient.load(0)
    tflops = lambda ms: 2.0 * M * N * K / (ms * 1e-3) / 1e12   # noqa: E731
    result = {"gpu": gpu_info(), "device": client.properties["name"], "iters": args.iters, "rounds": args.rounds,
              "shape": [M, N, K], "rows": []}
    out = TensorHandle.empty_contiguous(client, [M, N], "bf16")
    e4_128 = QuantScheme().with_value("e4m3").per_block(128, "f32")
    e5_128 = QuantScheme().with_value("e5m2").per_block(128, "f32")
    e4_32 = QuantScheme().with_value("e4m3").per_block(32, "f32")
    e4_t = QuantScheme().with_value("e4m3").per_tensor()
    runs = {}   # row name -> (timing function, callable)
    for name, sa, sb in (("e4m3/128/f32 x e4m3/128/f32", e4_128, e4_128), ("e4m3/32/f32 x e4m3/32/f32", e4_32, e4_32),
                         ("e4m3 per-tensor x e4m3 per-tensor", e4_t, e4_t), ("e5m2/128/f32 x e4m3/128/f32", e5_128, e4_128)):
        a, b = operand(client, sa, M, 1), operand(client, sb, N, 2)
        runs[name] = ("cubecl", lambda a=a, b=b: matmul.launch_quantized_fp8(client, a, b, out))
    # baselines
    bfa = TensorHandle.empty_contiguous(client, [M, K], "bf16")
    bfb = TensorHandle.empty_contiguous(client, [N, K], "bf16")
    client.fill_uniform(bfa.handle, "bf16", M * K, 5, -1.0, 1.0)
    client.fill_uniform(bfb.handle, "bf16", N * K, 6, -1.0, 1.0)
    bfb_t = TensorHandle(bfb.handle, [K, N], [1, K], "bf16")
    runs["bf16 b200_matmul (baseline)"] = ("cubecl", lambda: matmul.launch(client, bfa, bfb_t, out))
    qa, qb = operand(client, e4_128, M, 1), operand(client, e4_128, N, 2)
    f8a = TensorHandle(qa.values.handle, [M, K], [K, 1], "f8e4m3")
    f8b_t = TensorHandle(qb.values.handle, [K, N], [1, K], "f8e4m3")
    runs["fp8 b200_matmul on the same codes, f16-widened (baseline)"] = ("cubecl", lambda: matmul.launch(client, f8a, f8b_t, out))

    def deq_then_bf16():
        quant.launch_dequantize(client, qa, bfa)
        quant.launch_dequantize(client, qb, bfb)
        matmul.launch(client, bfa, bfb_t, out)
    runs["dequantize e4m3/128 x2 + bf16 b200_matmul (baseline)"] = ("cubecl", deq_then_bf16)
    trows, notes = torch_rows(qa)
    for name, fn in trows.items():
        runs[name] = ("torch", fn)
    if notes:
        result["torch_notes"] = notes
    times = {name: [] for name in runs}
    for _ in range(args.rounds):
        for name, (kind, fn) in runs.items():
            times[name].append(timed(client, fn, args.iters, args.warmup) if kind == "cubecl" else torch_timed(fn, args.iters, args.warmup))
    base = float(np.mean(times["bf16 b200_matmul (baseline)"]))
    for name, ts in times.items():
        ms = float(np.mean(ts))
        result["rows"].append({"row": name, "ms": ms, "tflops": tflops(ms), "vs_bf16": base / ms,
                               "round_spread": (max(ts) - min(ts)) / ms, "round_ms": ts})
    client.sync()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
