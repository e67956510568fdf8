#!/usr/bin/env python
"""examples/throughput (reference: examples/throughput/src/lib.rs, README.md:28-34) on the H100-native path.

Prints the reference's table -- using its own sampling protocol (ThroughputBenchmarker: warm up to a plateau, min of N
samples, host clock around launch+sync) -- for (a) the kernels CubeCL itself would JIT on this GPU (wmma probe, float_4
read probe: "reference-equivalent") and (b) the hand-written sm_90a kernels that replace them.
"""
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from cubecl_b200 import ComputeClient, TensorHandle, matmul, reduce  # noqa: E402
from cubecl_b200.throughput import ThroughputBenchmarker, device_sampler  # noqa: E402


def fmt(value: float, unit: str) -> str:
    return f"{value:.4f} {unit}"


def run(device: int = 0, clock: str = "host") -> None:
    c = ComputeClient.load(device)
    bench = ThroughputBenchmarker()
    rows = []
    scratch = c.empty(4096)

    ops = [0.0]

    def wmma():
        ops[0] = c.probe_wmma("f16", 2048, scratch)

    v = bench.measure(device_sampler(c, wmma, clock), 1)
    rows.append(("compute-cmma", "f16→f16 16×16×16 (wmma, as CubeCL JITs it)", fmt(ops[0] / v.duration_s / 1e12, "TOPS/s")))

    def umma():
        ops[0] = c.probe_umma(4096, scratch)

    v = bench.measure(device_sampler(c, umma, clock), 1)
    rows.append(("compute-wgmma", "bf16→f32 64×256×16 per warpgroup (wgmma)", fmt(ops[0] / v.duration_s / 1e12, "TOPS/s")))

    n = 8192
    a, b, o = (TensorHandle.empty_contiguous(c, [n, n], "bf16") for _ in range(3))
    c.fill_uniform(a.handle, "bf16", n * n, 3, -1, 1)
    c.fill_uniform(b.handle, "bf16", n * n, 4, -1, 1)
    v = bench.measure(device_sampler(c, lambda: matmul.launch(c, a, b, o), clock), int(2 * n ** 3))
    rows.append(("matmul", "bf16 8192×8192×8192 (wgmma + TMA)", fmt(v.ops_per_s() / 1e12, "TOPS/s")))
    del a, b, o

    nbytes = 512 << 20   # the reference's buffer size (throughput/base.rs:9)
    buf = c.empty(nbytes)
    c.fill_modulo(buf, "f32", nbytes // 4, 8)
    v = bench.measure(device_sampler(c, lambda: c.probe_memread(buf, nbytes, scratch), clock), nbytes)
    rows.append(("memory-read", "512 MiB float_4 (as CubeCL JITs it)", fmt(v.bytes_per_s() / 1e9, "Gbytes/s")))
    buf2 = c.empty(nbytes)
    v = bench.measure(device_sampler(c, lambda: c.probe_memwrite(buf2, nbytes), clock), nbytes)
    rows.append(("memory-write", "512 MiB float_4 (as CubeCL JITs it)", fmt(v.bytes_per_s() / 1e9, "Gbytes/s")))
    v = bench.measure(device_sampler(c, lambda: c.probe_memcopy(buf2, buf, nbytes), clock), 2 * nbytes)
    rows.append(("memory", "512 MiB copy, read+write counted", fmt(v.bytes_per_s() / 1e9, "Gbytes/s")))
    c.fill_modulo(buf, "f32", nbytes // 4, 8)
    t = TensorHandle.new_contiguous([nbytes // 4], buf, "f32")
    out = TensorHandle.empty_contiguous(c, [1], "f32")
    v = bench.measure(device_sampler(c, lambda: reduce.launch(c, t, out, None, "sum"), clock), nbytes)
    rows.append(("reduce-sum", "512 MiB f32 (hand-written, 1 launch)", fmt(v.bytes_per_s() / 1e9, "Gbytes/s")))

    tiny = c.empty(64)
    v = bench.measure(device_sampler(c, lambda: c.fill_modulo(tiny, "f32", 1, 2), clock), 1)
    rows.append(("launch", "", f"{v.duration_s * 1e6:.1f}µs/launch"))

    print(f"Peak throughput — cuda-b200<{c.properties['name']}>  (clock: {clock})")
    for mode, desc, value in rows:
        print(f"  {mode:<15}{desc:<46}{value:>20}")


if __name__ == "__main__":
    run(0, sys.argv[1] if len(sys.argv) > 1 else "host")
