"""Throughput of quantize / dequantize (b200_quantize, b200_dequantize) on one GPU, next to the same-run copy bandwidth.

    python tools/quant_bench.py [--iters 50] [--warmup 5]

Rows: bf16 [8192, 8192] -> MXFP8 and -> MXFP4 (one pass), bf16 [8192, 8192] -> NVFP4 two-level (an absmax pass, then the
encode pass: the input is read twice by construction), f32 [2^28] -> Q8S per-tensor (two passes likewise), and MXFP8 ->
bf16 dequantize.  Each is timed with CUDA events around `--iters` back-to-back calls after `--warmup` untimed ones.  GB/s
counts the algorithmic bytes: one read of the input plus the writes of codes and scales (dequantize: the reads of codes and
scales plus one write of the output); the second read of the two-pass rows is not credited.  b200_probe_memcopy gives the
same-run ceiling.  The card name and power limit are read (nvidia-smi --query-gpu, read-only) in the same run.  Prints
one JSON line.
"""
from __future__ import annotations

import argparse
import json
import math
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from cubecl_b200 import ComputeClient, TensorHandle, quant  # noqa: E402
from cubecl_b200.quant import QuantScheme  # noqa: E402
from scan_bench import gpu_info, timed  # noqa: E402

ROWS = [("quantize", [8192, 8192], "bf16", "mxfp8", "one pass"), ("quantize", [8192, 8192], "bf16", "mxfp4", "one pass"),
        ("quantize", [8192, 8192], "bf16", "nvfp4", "two passes"), ("quantize", [1 << 28], "f32", "q8s_per_tensor", "two passes"),
        ("dequantize", [8192, 8192], "bf16", "mxfp8", "one pass")]
ESZ = {"f32": 4, "f16": 2, "bf16": 2}
SCALE_ESZ = {"f32": 4, "f16": 2, "bf16": 2, "ue8m0": 1, "ue4m3": 1}


def scheme_of(name: str) -> QuantScheme:
    if name == "q8s_per_tensor":
        return QuantScheme().with_value("q8s").per_tensor()
    return getattr(QuantScheme, name)()


def quant_bytes(shape, scheme: QuantScheme) -> int:
    """Codes plus scales of a quantized tensor of `shape`."""
    n = math.prod(shape)
    b = quant.values_bytes(shape, scheme)
    if scheme.block:
        b += n // scheme.block * SCALE_ESZ[scheme.block_scale]
    return b + (4 if scheme.has_tensor else 0)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if args.iters < 20:
        raise SystemExit("--iters must be >= 20")
    client = ComputeClient.load(0)
    result = {"gpu": gpu_info(), "device": client.properties["name"], "iters": args.iters, "rows": []}
    n_copy = 1 << 28
    src = client.empty(n_copy * 4)
    dst = client.empty(n_copy * 4)
    client.fill_modulo(src, "f32", n_copy, 8)
    ms = timed(client, lambda: client.probe_memcopy(dst, src, n_copy * 4), args.iters, args.warmup)
    copy_gbps = 2 * n_copy * 4 / ms / 1e6
    result["memcopy_gbps"] = round(copy_gbps, 1)
    del src, dst
    for op, shape, dtype, name, path in ROWS:
        scheme = scheme_of(name)
        n = math.prod(shape)
        x = TensorHandle.empty_contiguous(client, shape, dtype)
        client.fill_uniform(x.handle, dtype, n, 7, -4.0, 4.0)
        q = quant.alloc_quantized(client, shape, scheme)
        quant.launch_quantize(client, x, q)
        if op == "quantize":
            fn = lambda: quant.launch_quantize(client, x, q)   # noqa: E731
        else:
            y = TensorHandle.empty_contiguous(client, shape, dtype)
            fn = lambda: quant.launch_dequantize(client, q, y)   # noqa: E731
        client.sync()
        before = client.launch_count()
        fn()
        launches = client.launch_count() - before
        client.sync()
        ms = timed(client, fn, args.iters, args.warmup)
        nbytes = n * ESZ[dtype] + quant_bytes(shape, scheme)
        gbps = nbytes / ms / 1e6
        result["rows"].append({"op": op, "shape": shape, "dtype": dtype, "scheme": name, "path": path, "launches": launches,
                               "ms": round(ms, 4), "gbps": round(gbps, 1), "of_copy": round(gbps / copy_gbps, 3)})
        del x, q
    print(json.dumps(result))


if __name__ == "__main__":
    main()
