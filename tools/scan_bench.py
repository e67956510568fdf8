"""Throughput of the axis scans (b200_scan) on one GPU, next to the same-run copy bandwidth.

    python tools/scan_bench.py [--iters 50] [--warmup 5]

Shapes (f32 cumsum): [2^28] (three-pass), [8192, 8192] along axis 1 (rows, one launch), [8192, 8192] along axis 0
(three-pass) and [64, 2^22] along axis 0 (columns, one launch).  Each is timed with CUDA events around `--iters`
back-to-back scans after `--warmup` untimed ones.  GB/s counts the algorithmic bytes, one read of the input and one write
of the output (N * 4 + N * 4); the three-pass shapes read the input a second time, which this figure does not credit.
b200_probe_memcopy over the same number of bytes moves exactly what a single-pass scan moves, so its rate is the same-run
ceiling.  The card name and power limit are read (nvidia-smi --query-gpu, read-only) in the same run.  Prints one JSON line.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

from cubecl_b200 import ComputeClient, TensorHandle, scan  # noqa: E402

SHAPES = [([1 << 28], 0, "three-pass"), ([8192, 8192], 1, "rows"), ([8192, 8192], 0, "three-pass"), ([64, 1 << 22], 0, "columns")]


def gpu_info() -> dict:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        return {"query_error": r.stdout.strip()}
    name, limit = [s.strip() for s in r.stdout.splitlines()[0].split(",")]
    return {"name": name, "power_limit": limit}


def timed(client, fn, iters: int, warmup: int) -> float:
    """Mean ms per call over `iters` calls, CUDA events on the client's stream."""
    for _ in range(warmup):
        fn()
    a, b = client.event(), client.event()
    client.record(a)
    for _ in range(iters):
        fn()
    client.record(b)
    ms = client.elapsed_ms(a, b) / iters
    client.event_destroy(a)
    client.event_destroy(b)
    client.sync()
    return ms


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
    result["memcopy_gbps"] = round(2 * n_copy * 4 / ms / 1e6, 1)
    del src, dst
    for shape, axis, path in SHAPES:
        n = 1
        for s in shape:
            n *= s
        x = TensorHandle.empty_contiguous(client, shape, "f32")
        client.fill_uniform(x.handle, "f32", n, 7, -1.0, 1.0)
        y = TensorHandle.empty_contiguous(client, shape, "f32")
        before = client.launch_count()
        scan.launch(client, x, y, axis, "sum")
        launches = client.launch_count() - before
        client.sync()
        ms = timed(client, lambda: scan.launch(client, x, y, axis, "sum"), args.iters, args.warmup)
        result["rows"].append({"shape": shape, "axis": axis, "path": path, "launches": launches, "ms": round(ms, 4),
                               "gbps": round(2 * n * 4 / ms / 1e6, 1)})
        del x, y
    print(json.dumps(result))


if __name__ == "__main__":
    main()
