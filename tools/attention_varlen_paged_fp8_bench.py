"""Throughput of paged variable-length attention against an e4m3 cache (b200_attention_varlen_paged_fp8) next to the same call
against a 16-bit cache (b200_attention_varlen_paged), alternating in one process for two rounds.

    python tools/attention_varlen_paged_fp8_bench.py [--iters 20] [--warmup 3]

Rows (bf16 q, D = 128 unless stated; the pages of every cache are in a seeded shuffled order, and the 16-bit and the e4m3 cache
are filled from the same packed keys with b200_kvcache_write and b200_kvcache_write_fp8, per-head scales of 1):
  prefill   B = 8 chunks of Lq = 2048 queries on 6144 cached keys (Lk = 8192), (Hq, Hkv) = (32, 8), window (-1, 0), pages of 16
            and of 256 keys.
  ragged    16 seeded sequences with Lq in [1, 4096] and prefixes in [0, 16384], 16-key pages, causal.
  prefill   the first row with f16 q and caches.
  prefill   (Hq, Hkv) = (32, 32) and D = 64 (recorded only).
Each time is the CUDA-event mean of `--iters` back-to-back calls after `--warmup` untimed ones.  A row's e4m3 / 16-bit ratio is
the mean of the two rounds' ratios, and `spread` is the relative difference between the rounds' ratios.  TFLOP/s counts
visible (i, j) pairs: 4 * Hq * D * pairs.  Goals:
  (a) prefill row, 256-key pages: e4m3 <= 1.10x the bf16-cache time;
  (b) prefill and ragged rows, 16-key pages: e4m3 <= 1.10x the bf16-cache time at the same page size.
The card name, power limit and SM clock are read (nvidia-smi --query-gpu, read-only) in the same run.  Prints one JSON line.
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tests"))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from attention_varlen_oracle import visible_pairs  # noqa: E402
from attention_varlen_paged_bench import cu, i32, ragged  # noqa: E402
from cubecl_b200 import ComputeClient, TensorHandle, attention  # noqa: E402
from conv_grouped_bench import sm_clock_mhz  # noqa: E402
from scan_bench import gpu_info, timed  # noqa: E402


class Problem:
    """Packed q [Tq, Hq, D] and keys / values [Tk, Hkv, D] (uniform random in dtype), and for every page size asked for a 16-bit
    and an e4m3 paged cache holding the same keys in the same shuffled pages, with their block table."""

    def __init__(self, client, lens_q, lens_k, Hq, Hkv, D, pages, dtype="bf16", seed=0):
        self.client, self.lens_q, self.lens_k, self.dtype = client, lens_q, lens_k, dtype
        rng = np.random.default_rng(seed)
        Tq, Tk = sum(lens_q), sum(lens_k)
        self.q = TensorHandle.empty_contiguous(client, [Tq, Hq, D], dtype)
        k = TensorHandle.empty_contiguous(client, [Tk, Hkv, D], dtype)
        v = TensorHandle.empty_contiguous(client, [Tk, Hkv, D], dtype)
        for i, t in enumerate((self.q, k, v)):
            client.fill_uniform(t.handle, dtype, t.size(), i + 1 + seed, -1.0, 1.0)
        self.out = TensorHandle.empty_contiguous(client, [Tq, Hq, D], dtype)
        self.lse = TensorHandle.empty_contiguous(client, [Hq, Tq], "f32")
        self.cuq, self.seqlens = i32(client, cu(lens_q)), i32(client, lens_k)
        ones = TensorHandle.from_numpy(client, np.ones(Hkv, np.float32), "f32")
        self.ks = self.vs = ones
        packed = lambda t: TensorHandle(t.handle, [1, Tk, Hkv, D], [Tk * Hkv * D, Hkv * D, D, 1], dtype)  # noqa: E731
        self.caches = {}
        for page in pages:
            mp = -(-max(lens_k) // page)
            P = len(lens_k) * mp
            table = rng.permutation(P).reshape(len(lens_k), mp).astype(np.int32)
            slots = i32(client, np.concatenate([table[b, np.arange(L) // page] * page + np.arange(L) % page
                                                for b, L in enumerate(lens_k)]))
            c16 = [TensorHandle.empty_contiguous(client, [P, page, Hkv, D], dtype) for _ in range(2)]
            c8 = [TensorHandle.empty_contiguous(client, [P, page, Hkv, D], "f8e4m3") for _ in range(2)]
            attention.kvcache_write(client, packed(k), packed(v), c16[0], c16[1], slots)
            attention.kvcache_write_fp8(client, packed(k), packed(v), c8[0], c8[1], slots, ones, ones)
            self.caches[page] = (c16, c8, i32(client, table))
        client.sync()

    def paged(self, page, window):
        (kc, vc), _, bt = self.caches[page]
        return lambda: attention.launch_varlen_paged(self.client, self.q, kc, vc, self.cuq, self.seqlens, max(self.lens_q),
                                                     max(self.lens_k), self.out, block_table=bt, window_size=window, lse=self.lse)

    def paged_fp8(self, page, window):
        _, (kc, vc), bt = self.caches[page]
        return lambda: attention.launch_varlen_paged_fp8(self.client, self.q, kc, vc, self.cuq, self.seqlens, self.ks, self.vs,
                                                         max(self.lens_q), max(self.lens_k), self.out, block_table=bt,
                                                         window_size=window, lse=self.lse)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if args.iters < 20:
        raise SystemExit("--iters must be >= 20")
    client = ComputeClient.load(0)
    result = {"gpu": gpu_info(), "clock": sm_clock_mhz(), "device": client.properties["name"], "iters": args.iters, "rows": []}
    tm = lambda fn: timed(client, fn, args.iters, args.warmup)  # noqa: E731
    causal = (-1, 0)

    def run(row, p, pages, pairs, Hq, D):
        """for every page size: the 16-bit and the e4m3 cache, alternating for two rounds; ms (mean of rounds), TFLOP/s, and the
        e4m3 / 16-bit ratio (mean of the rounds' ratios) with its spread"""
        variants = {}
        for page in pages:
            variants[f"p{page}_16"] = p.paged(page, causal)
            variants[f"p{page}_e4m3"] = p.paged_fp8(page, causal)
        rounds = {name: [] for name in variants}
        for _ in range(2):
            for name, fn in variants.items():
                rounds[name].append(tm(fn))
        for name, ms in rounds.items():
            mean = sum(ms) / 2
            row[f"{name}_ms"] = mean
            row[f"{name}_tflops"] = 4.0 * Hq * D * pairs / (mean * 1e-3) / 1e12
        for page in pages:
            r = [a / b for a, b in zip(rounds[f"p{page}_e4m3"], rounds[f"p{page}_16"])]
            row[f"p{page}_ratio"] = sum(r) / 2
            row[f"p{page}_ratio_spread"] = abs(r[0] - r[1]) / min(r)
        client.sync()
        result["rows"].append(row)
        print(json.dumps(row), file=sys.stderr, flush=True)
        return row

    lq, lk = [2048] * 8, [8192] * 8
    p = Problem(client, lq, lk, 32, 8, 128, (16, 256))
    row = run({"row": "prefill", "q": "bf16", "B": 8, "Lq": 2048, "Lk": 8192, "Hq": 32, "Hkv": 8, "D": 128}, p, (16, 256),
              visible_pairs(lq, lk, causal), 32, 128)
    row["goal_a_met"] = row["p256_ratio"] <= 1.10
    row["goal_b_met"] = row["p16_ratio"] <= 1.10
    del p

    rq, rk = ragged()
    p = Problem(client, rq, rk, 32, 8, 128, (16,))
    row = run({"row": "ragged", "q": "bf16", "B": len(rq), "Tq": sum(rq), "Tk": sum(rk), "max_q": max(rq), "max_k": max(rk), "Hq": 32,
               "Hkv": 8, "D": 128}, p, (16,), visible_pairs(rq, rk, causal), 32, 128)
    row["goal_b_met"] = row["p16_ratio"] <= 1.10
    del p

    p = Problem(client, lq, lk, 32, 8, 128, (16, 256), dtype="f16")
    run({"row": "prefill", "q": "f16", "B": 8, "Lq": 2048, "Lk": 8192, "Hq": 32, "Hkv": 8, "D": 128}, p, (16, 256),
        visible_pairs(lq, lk, causal), 32, 128)
    del p

    p = Problem(client, lq, lk, 32, 32, 64, (16, 256))
    run({"row": "prefill", "q": "bf16", "B": 8, "Lq": 2048, "Lk": 8192, "Hq": 32, "Hkv": 32, "D": 64}, p, (16, 256),
        visible_pairs(lq, lk, causal), 32, 64)
    del p
    print(json.dumps(result))


if __name__ == "__main__":
    main()
