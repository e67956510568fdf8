"""Throughput of attention against a KV cache (b200_attention_kvcache) on one GPU: decoding rows, each with the identity table
(the contiguous [B, L, Hkv, D] cache) and with 16-token pages in shuffled order, next to b200_attention and torch's
scaled_dot_product_attention on the equal-length contiguous cache, and the same-run b200_probe_memcopy rate.

    python tools/attention_kvcache_bench.py [--iters 20] [--warmup 3]

Rows: Sq = 1, bf16, D = 128, (Hq, Hkv) in {(32, 8), (32, 32)}, B x L in {1 x 65536, 8 x 16384, 64 x 2048, 128 x 1024}; one
ragged batch (B = 32, lengths uniform in [1, 8192], capacity 8192); one Sq = 4 causal row (B = 8, L = 8192).  bytes = the K and
V bytes of the visible keys plus q and out; GB/s over the CUDA-event time of `--iters` back-to-back calls after `--warmup`
untimed ones.  b200_attention and torch run on the same keys as a dense [B, Hkv, L, D] view of the identity cache (equal
lengths, Sq = 1 only); torch's row names the SDPA backend that ran.  Goals:
  (a) Sq = 1 rows with B * L >= 2^16 reach >= 0.6 of the copy rate (frac_of_copy);
  (b) B = 1, L = 65536, (32, 8) runs >= 4x faster than b200_attention (speedup_vs_attention);
  (c) 16-token pages cost <= 1.15x the identity-table time on the same row (paged_vs_identity).
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

from cubecl_b200 import ComputeClient, TensorHandle, attention  # noqa: E402
from conv_grouped_bench import sm_clock_mhz  # noqa: E402
from scan_bench import gpu_info, timed  # noqa: E402

D = 128
ROWS = [(B, L, hq, hkv, 1, False, False) for hq, hkv in ((32, 8), (32, 32))
        for B, L in ((1, 65536), (8, 16384), (64, 2048), (128, 1024))]
ROWS += [(32, 8192, 32, 8, 1, False, True), (8, 8192, 32, 8, 4, True, False)]   # ragged; Sq = 4 causal


def i32(client, a):
    return TensorHandle.from_numpy(client, np.ascontiguousarray(a, dtype=np.int32), "i32")


def torch_ms(B, Hq, Hkv, L, iters, warmup):
    """torch SDPA on a dense [B, H, L, D] cache; the first backend that accepts the call, with its name"""
    try:
        import torch
        from torch.nn.attention import SDPBackend, sdpa_kernel
    except ImportError:
        return None, None
    if not torch.cuda.is_available():
        return None, None
    q = torch.randn(B, Hq, 1, D, device="cuda", dtype=torch.bfloat16)
    k, v = (torch.randn(B, Hkv, L, D, device="cuda", dtype=torch.bfloat16) for _ in range(2))
    for name, be in (("flash", SDPBackend.FLASH_ATTENTION), ("cudnn", SDPBackend.CUDNN_ATTENTION),
                     ("efficient", SDPBackend.EFFICIENT_ATTENTION), ("math", SDPBackend.MATH)):
        try:
            with sdpa_kernel(be):
                fn = lambda: torch.nn.functional.scaled_dot_product_attention(q, k, v, enable_gqa=Hq != Hkv)  # noqa: E731
                for _ in range(warmup):
                    fn()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(iters):
                    fn()
                b.record()
                torch.cuda.synchronize()
                return a.elapsed_time(b) / iters, name
        except RuntimeError:
            continue
    return None, None


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if args.iters < 20:
        raise SystemExit("--iters must be >= 20")
    client = ComputeClient.load(0)
    result = {"gpu": gpu_info(), "clock": sm_clock_mhz(), "device": client.properties["name"], "iters": args.iters, "dtype": "bf16",
              "D": D, "rows": []}
    tm = lambda fn: timed(client, fn, args.iters, args.warmup)  # noqa: E731
    n_copy = 1 << 28
    src, dst = client.empty(n_copy * 4), client.empty(n_copy * 4)
    ms = tm(lambda: client.probe_memcopy(dst, src, n_copy * 4))
    copy_gbps = 2 * n_copy * 4 / ms / 1e6
    result["memcopy_gbps"] = round(copy_gbps, 1)
    del src, dst
    rng = np.random.default_rng(0)
    for B, L, Hq, Hkv, Sq, causal, is_ragged in ROWS:
        lens = rng.integers(1, L + 1, B) if is_ragged else np.full(B, L)
        q = TensorHandle.empty_contiguous(client, [B, Hq, Sq, D], "bf16")
        kc, vc = (TensorHandle.empty_contiguous(client, [B, L, Hkv, D], "bf16") for _ in range(2))
        for i, t in enumerate((q, kc, vc)):
            client.fill_uniform(t.handle, "bf16", t.size(), i + 1, -1.0, 1.0)
        out = TensorHandle.empty_contiguous(client, [B, Hq, Sq, D], "bf16")
        sl = i32(client, lens)
        nbytes = 2 * int(lens.sum()) * Hkv * D * 2 + 2 * B * Hq * Sq * D * 2
        row = {"B": B, "L": L, "Hq": Hq, "Hkv": Hkv, "Sq": Sq, "causal": causal, "ragged": is_ragged, "bytes": nbytes}
        ident = tm(lambda: attention.launch_kvcache(client, q, kc, vc, sl, out, causal=causal))
        row["kernel"] = client.last_kernel()
        # the same keys in shuffled 16-token pages
        page, mp = 16, L // 16
        table = rng.permutation(B * mp).astype(np.int32).reshape(B, mp)
        kp, vp = (TensorHandle(t.handle, [B * mp, page, Hkv, D], [page * Hkv * D, Hkv * D, D, 1], "bf16") for t in (kc, vc))
        bt = i32(client, table)
        paged = tm(lambda: attention.launch_kvcache(client, q, kp, vp, sl, out, block_table=bt, causal=causal))
        for name, t in (("identity", ident), ("paged16", paged)):
            row[f"{name}_ms"] = t
            row[f"{name}_gbps"] = nbytes / t / 1e6
            row[f"{name}_frac_of_copy"] = nbytes / t / 1e6 / copy_gbps
        row["paged_vs_identity"] = paged / ident
        row["goal_c_met"] = row["paged_vs_identity"] <= 1.15
        if Sq == 1 and B * L >= 1 << 16 and not is_ragged:
            row["goal_a_met"] = row["identity_frac_of_copy"] >= 0.6 and row["paged16_frac_of_copy"] >= 0.6
        if Sq == 1 and not is_ragged:
            kd, vd = (TensorHandle(t.handle, [B, Hkv, L, D], [L * Hkv * D, D, Hkv * D, 1], "bf16") for t in (kc, vc))
            dense = tm(lambda: attention.launch(client, q, kd, vd, out))
            row["attention_ms"] = dense
            row["speedup_vs_attention"] = dense / ident
            if B == 1 and L == 65536 and Hkv == 8:
                row["goal_b_met"] = row["speedup_vs_attention"] >= 4.0
            t, backend = torch_ms(B, Hq, Hkv, L, args.iters, args.warmup)
            if t is not None:
                row.update({"torch_ms": t, "torch_backend": backend, "speedup_vs_torch": t / ident})
        client.sync()
        result["rows"].append(row)
        del q, kc, vc, out, kp, vp
    print(json.dumps(result))


if __name__ == "__main__":
    main()
