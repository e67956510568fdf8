"""Throughput of attention against an fp8 KV cache (b200_attention_kvcache_fp8, e4m3) next to the same rows on a bf16 cache
(b200_attention_kvcache), alternating in one process for two rounds, and of the quantizing cache write next to the 16-bit one.

    python tools/attention_kvcache_fp8_bench.py [--iters 20] [--warmup 3]

Rows: those of tools/attention_kvcache_bench.py (Sq = 1, q bf16, D = 128, (Hq, Hkv) in {(32, 8), (32, 32)}, B x L from 1 x 65536
to 128 x 1024, the ragged batch and the Sq = 4 causal row), each with the identity table and with shuffled 16-token pages;
one prefill-sized write (B = 8, Snew = 4096, Hkv = 8, D = 128).  Each time is the CUDA-event mean of `--iters` back-to-back
calls after `--warmup` untimed ones; a row's ratio uses the mean of its two rounds.  bytes count the cache at its own element
size (1 byte for fp8, 2 for bf16) plus q and out.  Goals:
  (a) Sq = 1 identity rows with B * L >= 2^16: e4m3 time <= 0.6x the same-run bf16-cache time;
  (b) the same rows with 16-token pages: <= 0.7x the same-run bf16 paged time.
The card name, power limit and SM clock are read (nvidia-smi --query-gpu, read-only) in the same run.  Prints one JSON line.
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from attention_kvcache_bench import D, ROWS, i32  # noqa: E402
from cubecl_b200 import ComputeClient, TensorHandle, attention  # noqa: E402
from conv_grouped_bench import sm_clock_mhz  # noqa: E402
from scan_bench import gpu_info, timed  # noqa: E402


def fp8_codes(rng, n):
    """finite e4m3 codes of magnitude <= 2"""
    return (rng.integers(0, 0x41, n, dtype=np.uint8) | (rng.integers(0, 2, n, dtype=np.uint8) << 7)).astype(np.uint8)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if args.iters < 20:
        raise SystemExit("--iters must be >= 20")
    client = ComputeClient.load(0)
    result = {"gpu": gpu_info(), "clock": sm_clock_mhz(), "device": client.properties["name"], "iters": args.iters, "q_dtype": "bf16",
              "cache_dtypes": ["bf16", "f8e4m3"], "D": D, "rounds": 2, "rows": []}
    tm = lambda fn: timed(client, fn, args.iters, args.warmup)  # noqa: E731
    rng = np.random.default_rng(0)
    for B, L, Hq, Hkv, Sq, causal, is_ragged in ROWS:
        lens = rng.integers(1, L + 1, B) if is_ragged else np.full(B, L)
        q = TensorHandle.empty_contiguous(client, [B, Hq, Sq, D], "bf16")
        kc, vc = (TensorHandle.empty_contiguous(client, [B, L, Hkv, D], "bf16") for _ in range(2))
        for i, t in enumerate((q, kc, vc)):
            client.fill_uniform(t.handle, "bf16", t.size(), i + 1, -1.0, 1.0)
        k8, v8 = (TensorHandle.from_numpy(client, fp8_codes(rng, B * L * Hkv * D).reshape(B, L, Hkv, D), "f8e4m3") for _ in range(2))
        ks, vs = (TensorHandle.from_numpy(client, np.full(Hkv, s, np.float32), "f32") for s in (0.02, 0.03))
        out = TensorHandle.empty_contiguous(client, [B, Hq, Sq, D], "bf16")
        sl = i32(client, lens)
        page, mp = 16, L // 16
        table = rng.permutation(B * mp).astype(np.int32).reshape(B, mp)
        bt = i32(client, table)
        pv = lambda t, dt: TensorHandle(t.handle, [B * mp, page, Hkv, D], [page * Hkv * D, Hkv * D, D, 1], dt)  # noqa: E731
        kp, vp, kp8, vp8 = pv(kc, "bf16"), pv(vc, "bf16"), pv(k8, "f8e4m3"), pv(v8, "f8e4m3")
        calls = {
            "bf16_identity": lambda: attention.launch_kvcache(client, q, kc, vc, sl, out, causal=causal),
            "e4m3_identity": lambda: attention.launch_kvcache_fp8(client, q, k8, v8, sl, ks, vs, out, causal=causal),
            "bf16_paged16": lambda: attention.launch_kvcache(client, q, kp, vp, sl, out, block_table=bt, causal=causal),
            "e4m3_paged16": lambda: attention.launch_kvcache_fp8(client, q, kp8, vp8, sl, ks, vs, out, block_table=bt, causal=causal),
        }
        row = {"B": B, "L": L, "Hq": Hq, "Hkv": Hkv, "Sq": Sq, "causal": causal, "ragged": is_ragged}
        times = {name: [] for name in calls}
        for _ in range(2):
            for name, fn in calls.items():
                times[name].append(tm(fn))
                if name == "e4m3_identity":
                    row["kernel_e4m3"] = client.last_kernel()
        keys = int(lens.sum()) * Hkv * D
        for name, ts in times.items():
            t = sum(ts) / len(ts)
            nbytes = 2 * keys * (1 if name.startswith("e4m3") else 2) + 2 * B * Hq * Sq * D * 2
            row[f"{name}_ms"] = [round(x, 5) for x in ts]
            row[f"{name}_gbps"] = round(nbytes / t / 1e6, 1)
        mean = {name: sum(ts) / len(ts) for name, ts in times.items()}
        row["e4m3_vs_bf16_identity"] = round(mean["e4m3_identity"] / mean["bf16_identity"], 3)
        row["e4m3_vs_bf16_paged16"] = round(mean["e4m3_paged16"] / mean["bf16_paged16"], 3)
        if Sq == 1 and B * L >= 1 << 16 and not is_ragged:
            row["goal_a_met"] = row["e4m3_vs_bf16_identity"] <= 0.6
            row["goal_b_met"] = row["e4m3_vs_bf16_paged16"] <= 0.7
        client.sync()
        result["rows"].append(row)
        del q, kc, vc, k8, v8, out, kp, vp, kp8, vp8

    # one prefill-sized write: B = 8, Snew = 4096, Hkv = 8, D = 128 into identity-order slots
    B, Snew, Hkv = 8, 4096, 8
    kn, vn = (TensorHandle.empty_contiguous(client, [B, Snew, Hkv, D], "bf16") for _ in range(2))
    for i, t in enumerate((kn, vn)):
        client.fill_uniform(t.handle, "bf16", t.size(), i + 7, -1.0, 1.0)
    kc, vc = (TensorHandle.empty_contiguous(client, [B * Snew // 16, 16, Hkv, D], "bf16") for _ in range(2))
    k8, v8 = (TensorHandle.empty_contiguous(client, [B * Snew // 16, 16, Hkv, D], "f8e4m3") for _ in range(2))
    ks, vs = (TensorHandle.from_numpy(client, np.full(Hkv, 0.02, np.float32), "f32") for _ in range(2))
    slots = i32(client, np.arange(B * Snew))
    n = B * Snew * Hkv * D
    w = {"bf16": [], "e4m3": []}
    for _ in range(2):
        w["bf16"].append(tm(lambda: attention.kvcache_write(client, kn, vn, kc, vc, slots)))
        w["e4m3"].append(tm(lambda: attention.kvcache_write_fp8(client, kn, vn, k8, v8, slots, ks, vs)))
    client.sync()
    wm = {k: sum(v) / len(v) for k, v in w.items()}
    result["write"] = {"B": B, "Snew": Snew, "Hkv": Hkv, "bf16_ms": [round(x, 5) for x in w["bf16"]],
                       "e4m3_ms": [round(x, 5) for x in w["e4m3"]], "bf16_gbps": round(2 * n * 4 / wm["bf16"] / 1e6, 1),
                       "e4m3_gbps": round(2 * n * 3 / wm["e4m3"] / 1e6, 1), "e4m3_vs_bf16": round(wm["e4m3"] / wm["bf16"], 3)}
    goal_rows = [r for r in result["rows"] if "goal_a_met" in r]
    result["goal_a_met"] = all(r["goal_a_met"] for r in goal_rows)
    result["goal_b_met"] = all(r["goal_b_met"] for r in goal_rows)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
