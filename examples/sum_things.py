#!/usr/bin/env python
"""examples/sum_things (reference: examples/sum_things/src/lib.rs:178-227) on the H100-native path.

The reference launches 4 kernel kinds over input [-1, 10, 1, 5] with one unit per element, every unit computing the full
sum (15) -- or sum * input[unit] for the series kind -- and prints the output buffer after each.  Here the sum is the
device-wide reduce kernel (`reduce::launch`, warp-shuffle `plane_sum` stage inside); the per-unit output buffer is produced
ON THE DEVICE by a [4,1] x [1,1] matmul against the reduced scalar (ones for the plain kinds, the input for the series kind),
so every printed number comes from the GPU through the C ABI -- nothing is replicated on the host.
"""
import sys
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from cubecl_b200 import ComputeClient, TensorHandle, matmul, reduce  # noqa: E402


def launch(device: int = 0) -> None:
    client = ComputeClient.load(device)
    data = np.array([-1.0, 10.0, 1.0, 5.0], dtype=np.float32)
    inp = TensorHandle.from_numpy(client, data, "f32")
    name = f"cuda-b200<{client.properties['name']}>"
    ones = TensorHandle.from_numpy(client, np.ones(len(data), dtype=np.float32), "f32")
    client.set_option("gemm.f32", "tf32")                                    # small integers: exact on the tf32 pipe
    for kind in ("Basic", "Plane", "TraitSum", "SeriesSumThenMul"):
        total = reduce.launch_alloc(client, inp, None, "sum")                 # [1] f32 on the device
        per_unit = inp if kind == "SeriesSumThenMul" else ones                # output[unit] = sum * input[unit]  /  = sum
        lhs = TensorHandle(per_unit.handle, [4, 1], [1, 1], "f32")
        rhs = TensorHandle(total.handle, [1, 1], [1, 1], "f32")
        out = TensorHandle.empty_contiguous(client, [4, 1], "f32")
        matmul.launch(client, lhs, rhs, out)
        output = out.to_numpy(client).ravel()
        print(f"[{name!r} - {kind}]\n {output.tolist()}")
    client.set_option("gemm.f32", "hybrid")                                  # back to the default


if __name__ == "__main__":
    launch(int(sys.argv[1]) if len(sys.argv) > 1 else 0)
