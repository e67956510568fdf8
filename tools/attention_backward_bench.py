"""Throughput of the fused attention backward (b200_attention_backward: delta, dq and dk / dv) on one GPU, next to torch's
backward through scaled_dot_product_attention on the same shapes in the same run (FlashAttention and cuDNN backends, when
torch has CUDA), and the library's forward on the same shape.

    python tools/attention_backward_bench.py [--iters 20] [--warmup 3]

Shapes are tools/attention_bench.py's: 32,768 tokens per call (B = 32768 / S) at S in {1024, 2048, 4096, 8192, 16384},
model width 2,048 (Hq = 32 at D = 64, Hq = 16 at D = 128), causal off and on, bf16, plus one GQA row (Hq = 32, Hkv = 8,
D = 128, S = 4096).  Each call is timed with CUDA events around `--iters` back-to-back calls after `--warmup` untimed ones;
torch's is torch.autograd.grad of an SDPA output made under sdpa_kernel, with retain_graph.  TFLOP/s = 10 * B * Hq * D *
(visible (i, j) pairs) over that time (2.5x the forward's count, the usual convention).  Goals:
  (a) non-causal, D = 128, S >= 4096, Hq = Hkv: b200 time <= 1.25x the same-run torch flash time (flash_vs_b200 >= 0.8);
  (b) causal at S = 8192: <= 0.6x the time of the non-causal call on the same shape (causal_vs_full <= 0.6).
The card name, power limit and SM clock are read (nvidia-smi --query-gpu, read-only) in the same run.  Prints one JSON line.
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tests"))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from attention_bench import SHAPES  # noqa: E402
from attention_oracle import visible_pairs  # noqa: E402
from cubecl_b200 import ComputeClient, TensorHandle, attention  # noqa: E402
from conv_grouped_bench import sm_clock_mhz  # noqa: E402
from scan_bench import gpu_info, timed  # noqa: E402


def torch_bwd_ms(B, Hq, Hkv, S, D, causal, backend, iters, warmup):
    try:
        import torch
        from torch.nn.attention import SDPBackend, sdpa_kernel
    except ImportError:
        return None
    if not torch.cuda.is_available():
        return None
    q = torch.randn(B, Hq, S, D, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    k, v = (torch.randn(B, Hkv, S, D, device="cuda", dtype=torch.bfloat16) for _ in range(2))
    if Hq != Hkv:   # the fused backends take GQA as repeated kv heads
        k, v = k.repeat_interleave(Hq // Hkv, dim=1), v.repeat_interleave(Hq // Hkv, dim=1)
    k.requires_grad_()
    v.requires_grad_()
    be = {"flash": SDPBackend.FLASH_ATTENTION, "cudnn": SDPBackend.CUDNN_ATTENTION}[backend]
    try:
        with sdpa_kernel(be):
            o = torch.nn.functional.scaled_dot_product_attention(q, k, v, is_causal=causal)
            do = torch.randn_like(o)
            fn = lambda: torch.autograd.grad(o, (q, k, v), do, retain_graph=True)  # noqa: E731
            for _ in range(warmup):
                fn()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(iters):
                fn()
            b.record()
            torch.cuda.synchronize()
            return a.elapsed_time(b) / iters
    except RuntimeError:
        return None
    finally:
        del q, k, v
        torch.cuda.empty_cache()


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
    full_ms = {}
    for B, Hq, Hkv, S, D, causal in SHAPES:
        q = TensorHandle.empty_contiguous(client, [B, Hq, S, D], "bf16")
        k = TensorHandle.empty_contiguous(client, [B, Hkv, S, D], "bf16")
        v = TensorHandle.empty_contiguous(client, [B, Hkv, S, D], "bf16")
        do = TensorHandle.empty_contiguous(client, [B, Hq, S, D], "bf16")
        for i, t in enumerate((q, k, v, do)):
            client.fill_uniform(t.handle, "bf16", t.size(), i + 1, -1.0, 1.0)
        out = TensorHandle.empty_contiguous(client, [B, Hq, S, D], "bf16")
        lse = TensorHandle.empty_contiguous(client, [B, Hq, S], "f32")
        grads = [TensorHandle.empty_contiguous(client, t.shape, "bf16") for t in (q, k, v)]
        fwd = tm(lambda: attention.launch(client, q, k, v, out, causal=causal, lse=lse))
        ours = tm(lambda: attention.launch_backward(client, q, k, v, out, do, lse, *grads, causal=causal))
        flops = 10.0 * B * Hq * D * visible_pairs(S, S, causal)
        tf = lambda ms: flops / (ms * 1e-3) / 1e12  # noqa: E731
        row = {"B": B, "Hq": Hq, "Hkv": Hkv, "S": S, "D": D, "causal": causal, "ms": ours, "tflops": tf(ours), "fwd_ms": fwd,
               "bwd_vs_fwd": ours / fwd}
        for be in ("flash", "cudnn"):
            t = torch_bwd_ms(B, Hq, Hkv, S, D, causal, be, args.iters, args.warmup)
            if t is not None:
                row.update({f"{be}_ms": t, f"{be}_tflops": tf(t), f"{be}_vs_b200": t / ours})
        if not causal and D == 128 and S >= 4096 and Hq == Hkv and "flash_ms" in row:
            row["goal_a_met"] = ours <= 1.25 * row["flash_ms"]
        if Hq == Hkv and not causal:
            full_ms[(S, D)] = ours
        elif Hq == Hkv:   # the non-causal call on the same shape ran just before
            row["causal_vs_full"] = ours / full_ms[(S, D)]
            if S == 8192:
                row["goal_b_met"] = row["causal_vs_full"] <= 0.6
        client.sync()
        result["rows"].append(row)
        print(json.dumps(row), file=sys.stderr, flush=True)
        del q, k, v, do, out, lse, grads
    print(json.dumps(result))


if __name__ == "__main__":
    main()
