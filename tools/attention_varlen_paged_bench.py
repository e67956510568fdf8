"""Throughput of paged variable-length attention (b200_attention_varlen_paged) next to b200_attention_varlen on the same keys
packed contiguously and next to b200_attention_kvcache on the same cache, alternating in one process for two rounds.

    python tools/attention_varlen_paged_bench.py [--iters 20] [--warmup 3]

Rows (bf16, D = 128 unless stated; the pages of every cache are in a seeded shuffled order and filled from the packed keys with
b200_kvcache_write, so both calls read the same keys):
  prefill   B = 8 chunks of Lq = 2048 queries on 6144 cached keys (Lk = 8192), (Hq, Hkv) = (32, 8), window (-1, 0): pages of
            16 keys, pages of 256 keys, and varlen on the packed keys.
  prefill   the same with (Hq, Hkv) = (32, 32) and D = 64 (recorded only).
  ragged    16 seeded sequences with Lq in [1, 4096] and prefixes in [0, 16384], 16-key pages, causal, against varlen.
  uniform   B = 8, Sq = 2048, L = 8192, 16-key pages, (32, 8), causal: the paged call against b200_attention_kvcache.
  decode    B = 64, Lq = 1, L = 2048, 16-key pages, (32, 8): the paged call against b200_attention_kvcache (recorded only).
Each time is the CUDA-event mean of `--iters` back-to-back calls after `--warmup` untimed ones; a row's ratios use the mean
of its two rounds, and `spread` is the largest relative difference between a variant's two rounds.  TFLOP/s counts visible
(i, j) pairs: 4 * Hq * D * pairs.  Goals:
  (a) prefill and ragged rows: 16-key pages <= 1.10x the varlen time on the same keys, 256-key pages <= 1.05x;
  (b) uniform row: <= 0.6x the b200_attention_kvcache time.
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
from cubecl_b200 import ComputeClient, TensorHandle, attention  # noqa: E402
from conv_grouped_bench import sm_clock_mhz  # noqa: E402
from scan_bench import gpu_info, timed  # noqa: E402


def i32(client, a):
    return TensorHandle.from_numpy(client, np.ascontiguousarray(a, dtype=np.int32), "i32")


def cu(lens):
    return np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)


class Problem:
    """Packed q [Tq, Hq, D], packed keys and values [Tk, Hkv, D] (uniform random), and for every page size asked for a paged
    cache holding the same keys in shuffled pages, with its block table."""

    def __init__(self, client, lens_q, lens_k, Hq, Hkv, D, pages, seed=0):
        self.client, self.lens_q, self.lens_k, self.Hq, self.Hkv, self.D = client, lens_q, lens_k, Hq, Hkv, D
        rng = np.random.default_rng(seed)
        Tq, Tk = sum(lens_q), sum(lens_k)
        self.q = TensorHandle.empty_contiguous(client, [Tq, Hq, D], "bf16")
        self.k = TensorHandle.empty_contiguous(client, [Tk, Hkv, D], "bf16")
        self.v = TensorHandle.empty_contiguous(client, [Tk, Hkv, D], "bf16")
        for i, t in enumerate((self.q, self.k, self.v)):
            client.fill_uniform(t.handle, "bf16", t.size(), i + 1 + seed, -1.0, 1.0)
        self.out = TensorHandle.empty_contiguous(client, [Tq, Hq, D], "bf16")
        self.lse = TensorHandle.empty_contiguous(client, [Hq, Tq], "f32")
        self.cuq, self.cuk = i32(client, cu(lens_q)), i32(client, cu(lens_k))
        self.seqlens = i32(client, lens_k)
        self.caches = {}
        for page in pages:
            mp = -(-max(lens_k) // page)
            P = len(lens_k) * mp
            table = rng.permutation(P).reshape(len(lens_k), mp).astype(np.int32)
            slots = np.concatenate([table[b, np.arange(L) // page] * page + np.arange(L) % page for b, L in enumerate(lens_k)])
            kc = TensorHandle.empty_contiguous(client, [P, page, Hkv, D], "bf16")
            vc = TensorHandle.empty_contiguous(client, [P, page, Hkv, D], "bf16")
            packed = lambda t: TensorHandle(t.handle, [1, Tk, Hkv, D], [Tk * Hkv * D, Hkv * D, D, 1], "bf16")  # noqa: E731
            attention.kvcache_write(client, packed(self.k), packed(self.v), kc, vc, i32(client, slots))
            self.caches[page] = (kc, vc, i32(client, table))
        client.sync()

    def paged(self, page, window):
        kc, vc, bt = self.caches[page]
        return lambda: attention.launch_varlen_paged(self.client, self.q, kc, vc, self.cuq, self.seqlens, max(self.lens_q),
                                                     max(self.lens_k), self.out, block_table=bt, window_size=window, lse=self.lse)

    def varlen(self, window):
        return lambda: attention.launch_varlen(self.client, self.q, self.k, self.v, self.cuq, self.cuk, max(self.lens_q), max(self.lens_k),
                                               self.out, window_size=window, lse=self.lse)

    def kvcache(self, page, causal):
        """b200_attention_kvcache on the same cache: needs one Lq for every sequence (q viewed as [B, Hq, Sq, D])"""
        Sq, B = self.lens_q[0], len(self.lens_q)
        assert all(L == Sq for L in self.lens_q)
        kc, vc, bt = self.caches[page]
        q = TensorHandle(self.q.handle, [B, self.Hq, Sq, self.D], [Sq * self.Hq * self.D, self.D, self.Hq * self.D, 1], "bf16")
        out = TensorHandle(self.out.handle, list(q.shape), list(q.strides), "bf16")
        return lambda: attention.launch_kvcache(self.client, q, kc, vc, self.seqlens, out, block_table=bt, causal=causal)


def ragged(seed=1, n=16):
    rng = np.random.default_rng(seed)
    lq = [int(x) for x in rng.integers(1, 4097, n)]
    pre = [int(x) for x in rng.integers(0, 16385, n)]
    return lq, [a + b for a, b in zip(lq, pre)]


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if args.iters < 20:
        raise SystemExit("--iters must be >= 20")
    client = ComputeClient.load(0)
    result = {"gpu": gpu_info(), "clock": sm_clock_mhz(), "device": client.properties["name"], "iters": args.iters, "dtype": "bf16",
              "rows": []}
    tm = lambda fn: timed(client, fn, args.iters, args.warmup)  # noqa: E731

    def run(row, variants, pairs, Hq, D):
        """variants: name -> launch; two alternating rounds; per variant ms (mean of rounds), spread and TFLOP/s"""
        rounds = {name: [] for name in variants}
        for _ in range(2):
            for name, fn in variants.items():
                rounds[name].append(tm(fn))
        for name, ms in rounds.items():
            mean = sum(ms) / 2
            row[f"{name}_ms"] = mean
            row[f"{name}_spread"] = abs(ms[0] - ms[1]) / min(ms)
            row[f"{name}_tflops"] = 4.0 * Hq * D * pairs / (mean * 1e-3) / 1e12
        client.sync()
        result["rows"].append(row)
        print(json.dumps(row), file=sys.stderr, flush=True)
        return row

    causal = (-1, 0)
    # prefill chunks on a cached prefix, against varlen on the packed keys
    for Hq, Hkv, D, goal in ((32, 8, 128, True), (32, 32, 64, False)):
        lq, lk = [2048] * 8, [8192] * 8
        p = Problem(client, lq, lk, Hq, Hkv, D, (16, 256))
        row = run({"row": "prefill", "B": 8, "Lq": 2048, "Lk": 8192, "Hq": Hq, "Hkv": Hkv, "D": D},
                  {"paged16": p.paged(16, causal), "paged256": p.paged(256, causal), "varlen": p.varlen(causal)},
                  visible_pairs(lq, lk, causal), Hq, D)
        row["paged16_vs_varlen"] = row["paged16_ms"] / row["varlen_ms"]
        row["paged256_vs_varlen"] = row["paged256_ms"] / row["varlen_ms"]
        if goal:
            row["goal_a_met"] = row["paged16_vs_varlen"] <= 1.10 and row["paged256_vs_varlen"] <= 1.05
        del p

    # ragged mix of chunks and prefixes
    lq, lk = ragged()
    p = Problem(client, lq, lk, 32, 8, 128, (16,))
    row = run({"row": "ragged", "B": len(lq), "Tq": sum(lq), "Tk": sum(lk), "max_q": max(lq), "max_k": max(lk), "Hq": 32, "Hkv": 8, "D": 128},
              {"paged16": p.paged(16, causal), "varlen": p.varlen(causal)}, visible_pairs(lq, lk, causal), 32, 128)
    row["paged16_vs_varlen"] = row["paged16_ms"] / row["varlen_ms"]
    row["goal_a_met"] = row["paged16_vs_varlen"] <= 1.10
    del p

    # uniform chunks: against the decode kernel on the same cache
    lq, lk = [2048] * 8, [8192] * 8
    p = Problem(client, lq, lk, 32, 8, 128, (16,))
    row = run({"row": "uniform", "B": 8, "Sq": 2048, "L": 8192, "Hq": 32, "Hkv": 8, "D": 128},
              {"paged16": p.paged(16, causal), "kvcache": p.kvcache(16, True)}, visible_pairs(lq, lk, causal), 32, 128)
    row["paged16_vs_kvcache"] = row["paged16_ms"] / row["kvcache_ms"]
    row["goal_b_met"] = row["paged16_vs_kvcache"] <= 0.6
    del p

    # decode: recorded only (decode stays on the kvcache kernel)
    lq, lk = [1] * 64, [2048] * 64
    p = Problem(client, lq, lk, 32, 8, 128, (16,))
    row = run({"row": "decode", "B": 64, "Lq": 1, "L": 2048, "Hq": 32, "Hkv": 8, "D": 128},
              {"paged16": p.paged(16, (-1, -1)), "kvcache": p.kvcache(16, False)}, visible_pairs(lq, lk, (-1, -1)), 32, 128)
    row["paged16_vs_kvcache"] = row["paged16_ms"] / row["kvcache_ms"]
    del p
    print(json.dumps(result))


if __name__ == "__main__":
    main()
