"""Time of rotary position embeddings (b200_rope, b200_rope_kvcache_write, b200_rope_cos_sin) next to the same-run
b200_probe_memcopy rate, the unfused b200_rope + b200_kvcache_write(_fp8) pair, and torch / flash-attn / vLLM rotary ops.

    python tools/rope_bench.py [--iters 50] [--warmup 5]

Shapes: Hq / Hk = 32 / 8, D = 128, bf16 unless stated, positions random in [0, 131072), a [131072, rot] f32 table.
Bytes are algorithmic (reads plus writes from the shapes):
  b200_rope in place   q and k read and written on the rotated columns, plus the table row and the position per token:
                       2 T (Hq + Hk) rot esize + T (rot * 4 + 4)
  fused cache write    q read + written, k and v read, k and v written to the cache (16-bit or fp8), table, position, slot
  unfused pair         b200_rope of q and k in place, then b200_kvcache_write of the rotated k and of v (k written and read
                       back once more)
memcopy: b200_probe_memcopy of 1 GiB, counted as 2 GiB moved.  Each time is the CUDA-event mean of `--iters` back-to-back
calls after `--warmup`, measured in two alternating rounds; both rounds are printed so the spread is visible.
Goals, stated before measuring: (a) in-place b200_rope at T = 16384, NeoX, full rotary >= 0.8x the copy rate; (b) the fused
decode step (B = 64, 256, one token each, 16-token pages) <= 0.75x the unfused pair's time, and the prefill chunk (T = 8192)
<= 0.9x, against the bf16 and the e4m3 pair.  The card name and power limit are read (nvidia-smi --query-gpu, read-only) in
the same run.  Prints one JSON line.
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from cubecl_b200 import ComputeClient, TensorHandle, attention, rope  # noqa: E402
from scan_bench import gpu_info, timed  # noqa: E402

HQ, HK, D, PMAX = 32, 8, 128, 131072
ESZ = {"bf16": 2, "f32": 4}


def rand_dev(c, shape, dt, seed):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal(shape).astype(np.float32)
    return TensorHandle.from_numpy(c, x if dt == "f32" else (x.view(np.uint32) >> 16).astype(np.uint16), dt)


def rounds(c, fns, iters, warmup):
    """[[ms of fn for round 0, round 1] for fn in fns], the fns alternating within each round"""
    out = [[] for _ in fns]
    for _ in range(2):
        for i, fn in enumerate(fns):
            out[i].append(timed(c, fn, iters, warmup))
    return out


def us(ms):
    return [round(m * 1e3, 2) for m in ms]


def apply_rows(c, tables, iters, warmup, copy_gbps):
    rows = []
    for name, T, style, rot, dt in (("neox", 16384, "neox", 128, "bf16"), ("gptj", 16384, "gptj", 128, "bf16"),
                                    ("partial 64 of 128", 16384, "neox", 64, "bf16"), ("f32", 16384, "neox", 128, "f32"),
                                    ("T = 131072", 131072, "neox", 128, "bf16")):
        q, k = rand_dev(c, [1, T, HQ, D], dt, 1), rand_dev(c, [1, T, HK, D], dt, 2)
        pos = TensorHandle.from_numpy(c, np.random.default_rng(3).integers(0, PMAX, (1, T)).astype(np.int32), "i32")
        (ms,) = rounds(c, [lambda: rope.apply(c, tables[rot], q, k, pos, style=style)], iters, warmup)
        nbytes = 2 * T * (HQ + HK) * rot * ESZ[dt] + T * (rot * 4 + 4)
        gbps = nbytes / min(ms) / 1e6
        rows.append({"case": name, "T": T, "dtype": dt, "us": us(ms), "gbps": round(gbps, 1), "of_copy": round(gbps / copy_gbps, 3)})
    return rows


def kv_rows(c, table, iters, warmup):
    rows = []
    page = 16
    for label, B, S in (("decode B=64", 64, 1), ("decode B=256", 256, 1), ("prefill T=8192", 1, 8192)):
        pages = max(B * S // page + 64, 4096)
        rng = np.random.default_rng(B + S)
        slots = TensorHandle.from_numpy(c, rng.permutation(pages * page)[:B * S].astype(np.int32), "i32")
        pos = TensorHandle.from_numpy(c, rng.integers(0, PMAX, (B, S)).astype(np.int32), "i32")
        q, kn, vn = rand_dev(c, [B, S, HQ, D], "bf16", 4), rand_dev(c, [B, S, HK, D], "bf16", 5), rand_dev(c, [B, S, HK, D], "bf16", 6)
        ks = TensorHandle.from_numpy(c, np.ones(HK, np.float32), "f32")
        for cache in ("bf16", "f8e4m3"):
            kc = TensorHandle.empty_contiguous(c, [pages, page, HK, D], cache)
            vc = TensorHandle.empty_contiguous(c, [pages, page, HK, D], cache)
            f8 = cache != "bf16"
            fused = lambda: rope.kvcache_write(c, table, q, kn, vn, kc, vc, slots, pos, k_scale=ks if f8 else None,   # noqa: E731
                                               v_scale=ks if f8 else None)
            if f8:
                unfused = lambda: (rope.apply(c, table, q, kn, pos),   # noqa: E731
                                   attention.kvcache_write_fp8(c, kn, vn, kc, vc, slots, ks, ks))
            else:
                unfused = lambda: (rope.apply(c, table, q, kn, pos), attention.kvcache_write(c, kn, vn, kc, vc, slots))   # noqa: E731
            f_ms, u_ms = rounds(c, [fused, unfused], iters, warmup)
            goal = 0.9 if S > 1 else 0.75
            ratio = min(f_ms) / min(u_ms)
            rows.append({"case": label, "cache": cache, "fused_us": us(f_ms), "unfused_us": us(u_ms), "ratio": round(ratio, 3),
                         "goal": goal, "met": ratio <= goal})
    return rows


def yardsticks(iters, warmup):
    """torch eager HF rotate_half, flash-attn's apply_rotary_emb, vLLM's rotary op on the (a) shape; "not available" when the
    import fails"""
    import torch
    T, out = 16384, {}
    q = torch.randn(1, HQ, T, D, device="cuda", dtype=torch.bfloat16)
    k = torch.randn(1, HK, T, D, device="cuda", dtype=torch.bfloat16)
    cos = torch.randn(1, T, D, device="cuda", dtype=torch.bfloat16)
    sin = torch.randn(1, T, D, device="cuda", dtype=torch.bfloat16)

    def ev(fn):
        for _ in range(warmup):
            fn()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        torch.cuda.synchronize()
        return round(a.elapsed_time(b) / iters * 1e3, 2)
    try:
        from transformers.models.llama.modeling_llama import apply_rotary_pos_emb
        out["hf_eager_us"] = ev(lambda: apply_rotary_pos_emb(q, k, cos, sin))
    except Exception as e:  # noqa: BLE001
        out["hf_eager_us"] = f"not available ({type(e).__name__})"
    try:
        from flash_attn.layers.rotary import apply_rotary_emb
        qf, kf = q.transpose(1, 2).contiguous(), k.transpose(1, 2).contiguous()
        cf, sf = cos[0, :, :D // 2].float().contiguous(), sin[0, :, :D // 2].float().contiguous()
        out["flash_attn_us"] = ev(lambda: (apply_rotary_emb(qf, cf, sf, inplace=True), apply_rotary_emb(kf, cf, sf, inplace=True)))
    except Exception as e:  # noqa: BLE001
        out["flash_attn_us"] = f"not available ({type(e).__name__})"
    try:
        from vllm import _custom_ops as ops
        pos = torch.randint(0, PMAX, (T,), device="cuda")
        cache = torch.randn(PMAX, D, device="cuda", dtype=torch.bfloat16)
        qv, kv = q.transpose(1, 2).reshape(T, HQ * D).contiguous(), k.transpose(1, 2).reshape(T, HK * D).contiguous()
        out["vllm_us"] = ev(lambda: ops.rotary_embedding(pos, qv, kv, D, cache, True))
    except Exception as e:  # noqa: BLE001
        out["vllm_us"] = f"not available ({type(e).__name__})"
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    c = ComputeClient.load(0)
    nbytes = 1 << 30
    src, dst = c.empty(nbytes), c.empty(nbytes)
    copy_ms = rounds(c, [lambda: c.probe_memcopy(dst, src, nbytes)], args.iters, args.warmup)[0]
    copy_gbps = 2 * nbytes / min(copy_ms) / 1e6
    del src, dst
    tables = {rot: rope.cos_sin_alloc(c, PMAX, rot, 500000.0) for rot in (64, 128)}
    (table_ms,) = rounds(c, [lambda: rope.cos_sin(c, tables[128], 500000.0)], 5, 1)
    apply = apply_rows(c, tables, args.iters, args.warmup, copy_gbps)
    kv = kv_rows(c, tables[128], args.iters, args.warmup)
    c.sync()
    goals = {"a_neox_ge_0.8_copy": apply[0]["of_copy"] >= 0.8, "b_all": all(r["met"] for r in kv)}
    print(json.dumps({"gpu": gpu_info(), "device": c.properties["name"], "memcopy_gbps": round(copy_gbps, 1), "goals_met": goals,
                      "apply": apply, "kvcache_write": kv, "table_P131072_rot128_us": us(table_ms),
                      "yardsticks": yardsticks(args.iters, args.warmup)}))


if __name__ == "__main__":
    main()
