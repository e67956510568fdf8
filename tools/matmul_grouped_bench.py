"""Throughput of the grouped matmul (b200_matmul_grouped) on mixture-of-experts layer shapes, next to a batched b200_matmul on
the same work, a per-group b200_matmul loop with host-known sizes, and torch's grouped_mm, alternating in one process.

    python tools/matmul_grouped_bench.py [--iters 20] [--warmup 3] [--rows deepseek,mixtral,qwen3]

Rows (bf16 in and out, T = 32768 routed rows; every model with balanced routing and with a seeded skewed routing that has
empty experts, group sizes rounded to multiples of 16):
  deepseek  G = 32, hidden 7168, expert width 2048: gate-up N = 4096
  mixtral   G = 8, hidden 4096, width 14336: gate-up N = 28672
  qwen3     G = 128, hidden 2048, width 768: gate-up N = 1536
  ragged M  the gate-up forward x [T, hidden] @ W_g^T with W [G, N, hidden] (rhs the transposed view);
            TFLOP/s = 2 T N hidden / time
  ragged K  its weight gradient x.t() [hidden, T] @ dy [T, N] -> [G, hidden, N]; TFLOP/s = 2 hidden N T / time
Comparators: `batched` (balanced routing only: b200_matmul on [G, T / G, .] views of the same bytes), `loop` (one b200_matmul per
non-empty group) and `torch` (torch.nn.functional.grouped_mm on its own copies).  Each time is the CUDA-event mean of
`--iters` back-to-back calls after `--warmup` untimed ones; the variants of a row alternate for two rounds, and each reports the
mean of the rounds and `spread` = |r1 - r2| / min(r1, r2).  Goals, stated before measuring:
  (a) balanced ragged M and ragged K at >= 0.95x the TFLOP/s of the batched b200_matmul on the same work;
  (b) >= 0.9x torch grouped_mm's speed on the balanced deepseek and mixtral rows;
  (c) >= 1.5x the per-group loop on the G = 128 rows.
Skewed rows have no goal.  The card name, power limit and SM clock are read (nvidia-smi --query-gpu, read-only) in the same
run.  Prints one JSON line.
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from cubecl_b200 import ComputeClient, TensorHandle, matmul  # noqa: E402
from conv_grouped_bench import sm_clock_mhz  # noqa: E402
from scan_bench import gpu_info, timed  # noqa: E402

MODELS = {"deepseek": (32, 7168, 4096), "mixtral": (8, 4096, 28672), "qwen3": (128, 2048, 1536)}
T = 32768


def routing(G: int, skewed: bool, seed: int = 7) -> list[int]:
    """group sizes summing to T, multiples of 16; skewed: Dirichlet(0.3) shares with a tenth of the experts (at least one) empty"""
    if not skewed:
        return [T // G] * G
    rng = np.random.default_rng(seed + G)
    share = rng.dirichlet(np.full(G, 0.3))
    share[rng.permutation(G)[:max(1, G // 10)]] = 0
    units = np.floor(share / share.sum() * (T // 16)).astype(np.int64)
    units[np.argmax(units)] += T // 16 - units.sum()
    return [int(u) * 16 for u in units]


def torch_timed(fn, iters, warmup):
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
    ap.add_argument("--rows", default="deepseek,mixtral,qwen3")
    args = ap.parse_args()
    if args.iters < 20:
        raise SystemExit("--iters must be >= 20")
    import torch
    client = ComputeClient.load(0)
    result = {"gpu": gpu_info(), "clock": sm_clock_mhz(), "device": client.properties["name"], "iters": args.iters, "T": T, "rows": []}

    def run(row, variants, flops):
        rounds = {name: [] for name in variants}
        for _ in range(2):
            for name, (kind, fn) in variants.items():
                rounds[name].append(torch_timed(fn, args.iters, args.warmup) if kind == "torch" else timed(client, fn, args.iters, args.warmup))
        for name, ms in rounds.items():
            row[f"{name}_ms"] = sum(ms) / 2
            row[f"{name}_tflops"] = flops / (row[f"{name}_ms"] * 1e-3) / 1e12
            row[f"{name}_spread"] = abs(ms[0] - ms[1]) / min(ms)
        client.sync()
        result["rows"].append(row)
        print(json.dumps(row), file=sys.stderr, flush=True)
        return row

    for model in args.rows.split(","):
        G, H, N = MODELS[model]
        x = TensorHandle.empty_contiguous(client, [T, H], "bf16")          # routed tokens, sorted by expert
        w = TensorHandle.empty_contiguous(client, [G, N, H], "bf16")       # gate-up weights [G, N, hidden]
        dy = TensorHandle.empty_contiguous(client, [T, N], "bf16")
        for i, t in enumerate((x, w, dy)):
            client.fill_uniform(t.handle, "bf16", t.size(), i + 1, -1.0, 1.0)
        y = TensorHandle.empty_contiguous(client, [T, N], "bf16")
        dw = TensorHandle.empty_contiguous(client, [G, H, N], "bf16")
        wt = TensorHandle(w.handle, [G, H, N], [N * H, 1, H], "bf16")       # rhs [G, K, N]: W_g^T
        xt = TensorHandle(x.handle, [H, T], [1, H], "bf16")                # x.t()
        client.sync()
        # torch's copies of the same values
        tx = torch.from_numpy(x.to_numpy(client).view(np.int16)).cuda().view(torch.bfloat16)
        tw = torch.from_numpy(w.to_numpy(client).view(np.int16)).cuda().view(torch.bfloat16)
        tdy = torch.from_numpy(dy.to_numpy(client).view(np.int16)).cuda().view(torch.bfloat16)
        for skewed in (False, True):
            sizes = routing(G, skewed)
            offs_np = np.cumsum(sizes).astype(np.int32)
            offs = TensorHandle.from_numpy(client, offs_np, "i32")
            toffs = torch.from_numpy(offs_np).cuda()
            bounds = [(int(o - s), int(o)) for s, o in zip(sizes, offs_np)]
            meta = {"model": model, "routing": "skewed" if skewed else "balanced", "G": G, "hidden": H, "N": N, "T": T,
                    "empty_groups": sum(1 for s in sizes if s == 0), "max_group": max(sizes)}

            def loop_m():
                for g, (lo, hi) in enumerate(bounds):
                    if hi > lo:
                        matmul.launch(client, TensorHandle(x.handle.offset(lo * H * 2), [hi - lo, H], [H, 1], "bf16"),
                                      TensorHandle(w.handle.offset(g * N * H * 2), [H, N], [1, H], "bf16"),
                                      TensorHandle(y.handle.offset(lo * N * 2), [hi - lo, N], [N, 1], "bf16"))

            def loop_k():
                for g, (lo, hi) in enumerate(bounds):
                    if hi > lo:
                        matmul.launch(client, TensorHandle(x.handle.offset(lo * H * 2), [H, hi - lo], [1, H], "bf16"),
                                      TensorHandle(dy.handle.offset(lo * N * 2), [hi - lo, N], [N, 1], "bf16"),
                                      TensorHandle(dw.handle.offset(g * H * N * 2), [H, N], [N, 1], "bf16"))

            vm = {"grouped": ("b200", lambda: matmul.launch_grouped(client, x, wt, offs, y)), "loop": ("b200", loop_m),
                  "torch": ("torch", lambda: torch.nn.functional.grouped_mm(tx, tw.transpose(1, 2), offs=toffs))}
            vk = {"grouped": ("b200", lambda: matmul.launch_grouped(client, xt, dy, offs, dw)), "loop": ("b200", loop_k),
                  "torch": ("torch", lambda: torch.nn.functional.grouped_mm(tx.t(), tdy, offs=toffs))}
            if not skewed:
                n = T // G
                vm["batched"] = ("b200", lambda: matmul.launch(client, TensorHandle(x.handle, [G, n, H], [n * H, H, 1], "bf16"), wt,
                                                               TensorHandle(y.handle, [G, n, N], [n * N, N, 1], "bf16")))
                vk["batched"] = ("b200", lambda: matmul.launch(client, TensorHandle(x.handle, [G, H, n], [n * H, 1, H], "bf16"),
                                                               TensorHandle(dy.handle, [G, n, N], [n * N, N, 1], "bf16"), dw))
            for mode, variants in (("ragged_m", vm), ("ragged_k", vk)):
                row = run(dict(meta, mode=mode), variants, 2.0 * T * N * H)
                if not skewed:
                    row["vs_batched"] = row["grouped_tflops"] / row["batched_tflops"]
                    row["goal_a_met"] = row["vs_batched"] >= 0.95
                    if model in ("deepseek", "mixtral"):
                        row["vs_torch"] = row["torch_ms"] / row["grouped_ms"]
                        row["goal_b_met"] = row["vs_torch"] >= 0.9
                if G == 128:
                    row["vs_loop"] = row["loop_ms"] / row["grouped_ms"]
                    row["goal_c_met"] = row["vs_loop"] >= 1.5
        del x, w, dy, y, dw, tx, tw, tdy
        torch.cuda.empty_cache()
        client.sync()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
