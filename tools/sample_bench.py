"""Time of token sampling (b200_sample) on bf16 logits, next to the same-run b200_probe_memcopy rate and torch's eager
sort-based pipeline.

    python tools/sample_bench.py [--iters 50] [--warmup 5] [--rounds 2] [--v 128256] [--batches 1,16,64,256]

Every row: logits bf16 [b, v], i64 ids, per-row u64 seeds and offsets.  Two configurations:
  greedy    temperature 0 (the greedy-only launch, one argmax pass);
  filtered  temperature 0.8, top-k 50, top-p 0.9, min-p 0.05.
Bytes are algorithmic: the logits read once, 2 b v (ids, seeds and offsets are noise).  memcopy: b200_probe_memcopy of 1 GiB,
counted as 2 GiB moved.  torch: the eager pipeline a framework without a fused sampler runs on the same bf16 logits --
temperature, sort descending, softmax, cumsum, the top-k / top-p / min-p masks, renormalise, torch.multinomial.
FlashInfer's top_k_top_p_sampling_from_logits is timed when it imports.  Each time is the CUDA-event mean of `--iters`
back-to-back calls after `--warmup`; the shapes are measured in `--rounds` alternating rounds and each round is reported.
Goals, stated before measuring: greedy >= 0.6x the copy rate at b = 256; filtered <= 2x the greedy time of the same shape;
filtered >= 10x faster than torch's pipeline at b = 64 and 256; the b = 1 latency is reported with no goal.  The card name
and power limit are read (nvidia-smi --query-gpu, read-only) in the same run.  Prints one JSON line.
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from cubecl_b200 import ComputeClient, TensorHandle, sample as smp  # noqa: E402
from matmul_grouped_bench import torch_timed  # noqa: E402
from scan_bench import gpu_info, timed  # noqa: E402

FILTERED = dict(temperature=0.8, top_k=50, top_p=0.9, min_p=0.05)


def logits_of(c, b, v, seed):
    """a bf16 [b, v] device tensor: a random 64-row block tiled down the rows, scale 3 (a peaked, LM-like row)"""
    rng = np.random.default_rng(seed)
    block = ((rng.standard_normal((min(b, 64), v)).astype(np.float32) * 3).view(np.uint32) >> 16).astype(np.uint16)
    return TensorHandle.from_numpy(c, np.tile(block, (-(-b // block.shape[0]), 1))[:b], "bf16")


def torch_pipeline(x, T, k, p, mp, gen):
    """eager temperature / top-k / top-p / min-p sampling over sorted rows (HF's and vLLM's fallback shape)"""
    import torch
    z = x.float() / T
    s, idx = torch.sort(z, dim=-1, descending=True)
    probs = torch.softmax(s, dim=-1)
    cum = torch.cumsum(probs, dim=-1)
    pos = torch.arange(s.shape[1], device=x.device)
    drop = (pos >= k) | ((cum - probs) >= p) | (probs < mp * probs[:, :1])
    probs = probs.masked_fill(drop, 0.0)
    choice = torch.multinomial(probs / probs.sum(-1, keepdim=True), 1, generator=gen)
    return idx.gather(1, choice)[:, 0]


def run_row(c, b, v, iters, warmup, copy_gbps):
    import torch
    x = logits_of(c, b, v, 1)
    ids = TensorHandle.empty_contiguous(c, [b], "i64")
    seeds = TensorHandle.from_numpy(c, np.arange(b, dtype=np.uint64) * 7919 + 1, "u64")
    offs = TensorHandle.from_numpy(c, np.zeros(b, np.uint64), "u64")
    greedy_ms = timed(c, lambda: smp.sample(c, x, ids, temperature=0.0), iters, warmup)
    filt_ms = timed(c, lambda: smp.sample(c, x, ids, seed=seeds, offset=offs, advance_offsets=True, **FILTERED), iters, warmup)
    c.sync()
    xt = torch.from_numpy((x.to_numpy(c).astype(np.uint32) << 16).view(np.float32)).to(torch.bfloat16).cuda()
    gen = torch.Generator(device="cuda").manual_seed(0)
    t_torch = torch_timed(lambda: torch_pipeline(xt, 0.8, 50, 0.9, 0.05, gen), iters, warmup)
    row = {"b": b, "v": v, "greedy_us": round(greedy_ms * 1e3, 1),
           "greedy_of_copy": round(2 * b * v / greedy_ms / 1e6 / copy_gbps, 3),
           "filtered_us": round(filt_ms * 1e3, 1), "filtered_of_copy": round(2 * b * v / filt_ms / 1e6 / copy_gbps, 3),
           "filtered_over_greedy": round(filt_ms / greedy_ms, 2), "torch_pipeline_us": round(t_torch * 1e3, 1),
           "vs_torch": round(t_torch / filt_ms, 1)}
    try:
        import flashinfer
        row["flashinfer_us"] = round(torch_timed(lambda: flashinfer.sampling.top_k_top_p_sampling_from_logits(
            xt.float() / 0.8, 50, 0.9), iters, warmup) * 1e3, 1)
    except Exception:  # noqa: BLE001  -- reported only when it imports and runs
        pass
    del xt
    torch.cuda.empty_cache()
    return row


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--v", type=int, default=128256)
    ap.add_argument("--batches", default="1,16,64,256")
    args = ap.parse_args()
    c = ComputeClient.load(0)
    nbytes = 1 << 30
    src, dst = c.empty(nbytes), c.empty(nbytes)
    copy_ms = timed(c, lambda: c.probe_memcopy(dst, src, nbytes), args.iters, args.warmup)
    copy_gbps = 2 * nbytes / copy_ms / 1e6
    del src, dst
    batches = [int(b) for b in args.batches.split(",")]
    rounds = [[run_row(c, b, args.v, args.iters, args.warmup, copy_gbps) for b in batches] for _ in range(args.rounds)]
    every = [r for rows in rounds for r in rows]
    goals = {"greedy_ge_0.6_copy_at_b256": all(r["greedy_of_copy"] >= 0.6 for r in every if r["b"] == 256),
             "filtered_le_2x_greedy": all(r["filtered_over_greedy"] <= 2 for r in every),
             "ge_10x_torch_at_b64_b256": all(r["vs_torch"] >= 10 for r in every if r["b"] in (64, 256))}
    print(json.dumps({"gpu": gpu_info(), "device": c.properties["name"], "memcopy_gbps": round(copy_gbps, 1), "goals_met": goals,
                      "rounds": rounds}))


if __name__ == "__main__":
    main()
