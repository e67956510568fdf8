"""Throughput of variable-length (packed) attention (b200_attention_varlen and its backward) on one GPU, next to the dense
kernels and torch's varlen attention in the same run.

    python tools/attention_varlen_bench.py [--iters 20] [--warmup 3]

Rows (bf16; each call timed with CUDA events around `--iters` back-to-back calls after `--warmup` untimed ones):
  uniform  8 x 4096 tokens, Hq = Hkv = 16, D = 128, windows (-1, -1) and (-1, 0): varlen against the dense forward and backward
           on the same bytes (the [T, H, D] buffers viewed as [8, 16, 4096, 128] with strides); the dense kernels on compact
           [B, H, S, D] tensors are reported beside them (dense_bhsd_*), since the token-major layout alone changes the time.
  ragged   32,768 tokens in a seeded fixed list of lengths from 64 to 8192, causal; D = 128 with (Hq, Hkv) = (16, 16) and
           (32, 8), and D = 64 with (32, 32): varlen against torch.nn.attention.varlen.varlen_attn (kv heads repeated to Hq
           when torch refuses GQA) and against the dense kernels on the zero-padded [B, max, H, D] batch.
  window   B = 4, L = 8192, D = 128, Hq = Hkv = 16, windows (1024, 0), (4096, 0) and (-1, 0).
TFLOP/s counts visible (i, j) pairs: 4 * Hq * D * pairs for the forward, 2.5x that for the backward.  Goals:
  (a) uniform rows: varlen time <= 1.05x the dense time, forward and backward;
  (b) ragged D = 128 rows: >= 0.9x the speed of torch's varlen attention, forward and backward;
  (c) window (1024, 0): time <= 0.35x the (-1, 0) time, forward and backward.
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


def ragged_lengths(total=32768, seed=0):
    """a fixed list of lengths in [64, 8192] summing to `total`"""
    rng = np.random.default_rng(seed)
    lens = []
    while sum(lens) < total:
        lens.append(int(min(total - sum(lens), rng.integers(64, 8193))))
    if lens[-1] < 64:
        lens[-2] += lens.pop()
    return lens


class Problem:
    def __init__(self, client, lens, Hq, Hkv, D):
        self.client, self.lens, self.Hq, self.Hkv, self.D = client, lens, Hq, Hkv, D
        T = sum(lens)
        cu = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
        self.cu = TensorHandle.from_numpy(client, cu, "i32")
        self.t = {n: TensorHandle.empty_contiguous(client, [T, h, D], "bf16") for n, h in (("q", Hq), ("k", Hkv), ("v", Hkv), ("do", Hq))}
        for i, t in enumerate(self.t.values()):
            client.fill_uniform(t.handle, "bf16", t.size(), i + 1, -1.0, 1.0)
        self.out = TensorHandle.empty_contiguous(client, [T, Hq, D], "bf16")
        self.lse = TensorHandle.empty_contiguous(client, [Hq, T], "f32")
        self.grads = [TensorHandle.empty_contiguous(client, self.t[n].shape, "bf16") for n in ("q", "k", "v")]

    def fwd(self, window):
        L = max(self.lens)
        t = self.t
        return lambda: attention.launch_varlen(self.client, t["q"], t["k"], t["v"], self.cu, self.cu, L, L, self.out, window_size=window,
                                               lse=self.lse)

    def bwd(self, window):
        L = max(self.lens)
        t = self.t
        return lambda: attention.launch_varlen_backward(self.client, t["q"], t["k"], t["v"], self.out, t["do"], self.lse, self.cu, self.cu,
                                                        L, L, *self.grads, window_size=window)


def bshd(x, B, S):
    """a [B * S, H, D] tensor as the [B, H, S, D] view of the same bytes"""
    _, H, D = x.shape
    return TensorHandle(x.handle, [B, H, S, D], [S * H * D, D, H * D, 1], x.dtype)


def dense_ms(client, B, Hq, Hkv, S, D, causal, tm, same=None):
    """forward and backward ms of the dense kernels on compact [B, H, S, D] tensors, or with `same` (a Problem of B equal
    sequences of S tokens) on its own [T, H, D] buffers viewed as [B, H, S, D]"""
    if same is None:
        t = {n: TensorHandle.empty_contiguous(client, [B, h, S, D], "bf16") for n, h in (("q", Hq), ("k", Hkv), ("v", Hkv), ("do", Hq))}
        for i, x in enumerate(t.values()):
            client.fill_uniform(x.handle, "bf16", x.size(), i + 1, -1.0, 1.0)
        out = TensorHandle.empty_contiguous(client, [B, Hq, S, D], "bf16")
        grads = [TensorHandle.empty_contiguous(client, t[n].shape, "bf16") for n in ("q", "k", "v")]
    else:
        t = {n: bshd(x, B, S) for n, x in same.t.items()}
        out = bshd(same.out, B, S)
        grads = [bshd(g, B, S) for g in same.grads]
    lse = TensorHandle.empty_contiguous(client, [B, Hq, S], "f32")
    f = tm(lambda: attention.launch(client, t["q"], t["k"], t["v"], out, causal=causal, lse=lse))
    b = tm(lambda: attention.launch_backward(client, t["q"], t["k"], t["v"], out, t["do"], lse, *grads, causal=causal))
    return f, b


def torch_varlen_ms(lens, Hq, Hkv, D, iters, warmup):
    """(forward ms, backward ms, backend) of torch's varlen attention, causal; None when torch has no CUDA or refuses"""
    try:
        import torch
        from torch.nn.attention.varlen import varlen_attn
    except ImportError:
        return None
    if not torch.cuda.is_available():
        return None
    T, L = sum(lens), max(lens)
    cu = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int32, device="cuda")
    q = torch.randn(T, Hq, D, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    k, v = (torch.randn(T, Hkv, D, device="cuda", dtype=torch.bfloat16) for _ in range(2))

    def run(kk, vv):
        kk, vv = kk.detach().requires_grad_(), vv.detach().requires_grad_()
        o = varlen_attn(q, kk, vv, cu, cu, L, L, window_size=(-1, 0))
        do = torch.randn_like(o)

        def time(fn):
            for _ in range(warmup):
                fn()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(iters):
                fn()
            b.record()
            torch.cuda.synchronize()
            return a.elapsed_time(b) / iters
        f = time(lambda: varlen_attn(q, kk, vv, cu, cu, L, L, window_size=(-1, 0)))
        b = time(lambda: torch.autograd.grad(o, (q, kk, vv), do, retain_graph=True))
        return f, b

    try:
        try:
            return (*run(k, v), "varlen_attn")
        except RuntimeError:
            if Hq == Hkv:
                raise
            return (*run(k.repeat_interleave(Hq // Hkv, dim=1), v.repeat_interleave(Hq // Hkv, dim=1)), "varlen_attn, kv repeated")
    except RuntimeError:
        return None
    finally:
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

    def emit(row):
        client.sync()
        result["rows"].append(row)
        print(json.dumps(row), file=sys.stderr, flush=True)

    def rates(row, lens, Hq, D, window, f, b):
        pairs = visible_pairs(lens, lens, window)
        row.update({"fwd_ms": f, "bwd_ms": b, "fwd_tflops": 4.0 * Hq * D * pairs / (f * 1e-3) / 1e12,
                    "bwd_tflops": 10.0 * Hq * D * pairs / (b * 1e-3) / 1e12})

    # uniform: varlen against dense on the same shape
    for window in ((-1, -1), (-1, 0)):
        lens, Hq, D = [4096] * 8, 16, 128
        p = Problem(client, lens, Hq, Hq, D)
        f, b = tm(p.fwd(window)), tm(p.bwd(window))
        df, db = dense_ms(client, 8, Hq, Hq, 4096, D, window == (-1, 0), tm, same=p)
        cf, cb = dense_ms(client, 8, Hq, Hq, 4096, D, window == (-1, 0), tm)
        row = {"row": "uniform", "window": window, "dense_fwd_ms": df, "dense_bwd_ms": db, "fwd_vs_dense": f / df, "bwd_vs_dense": b / db,
               "dense_bhsd_fwd_ms": cf, "dense_bhsd_bwd_ms": cb}
        rates(row, lens, Hq, D, window, f, b)
        row["goal_a_met"] = f <= 1.05 * df and b <= 1.05 * db
        emit(row)
        del p

    # ragged: varlen against torch's varlen attention and the dense kernels on the padded batch
    lens = ragged_lengths()
    for Hq, Hkv, D in ((16, 16, 128), (32, 8, 128), (32, 32, 64)):
        p = Problem(client, lens, Hq, Hkv, D)
        f, b = tm(p.fwd((-1, 0))), tm(p.bwd((-1, 0)))
        row = {"row": "ragged", "B": len(lens), "max_len": max(lens), "Hq": Hq, "Hkv": Hkv, "D": D}
        rates(row, lens, Hq, D, (-1, 0), f, b)
        pf, pb = dense_ms(client, len(lens), Hq, Hkv, max(lens), D, True, tm)
        row.update({"padded_fwd_ms": pf, "padded_bwd_ms": pb})
        tv = torch_varlen_ms(lens, Hq, Hkv, D, args.iters, args.warmup)
        if tv is not None:
            row.update({"torch_fwd_ms": tv[0], "torch_bwd_ms": tv[1], "torch_backend": tv[2], "fwd_speed_vs_torch": tv[0] / f,
                        "bwd_speed_vs_torch": tv[1] / b})
            if D == 128:
                row["goal_b_met"] = tv[0] / f >= 0.9 and tv[1] / b >= 0.9
        emit(row)
        del p

    # window: hidden blocks are skipped
    lens, Hq, D = [8192] * 4, 16, 128
    p = Problem(client, lens, Hq, Hq, D)
    causal = None
    for window in ((-1, 0), (4096, 0), (1024, 0)):
        f, b = tm(p.fwd(window)), tm(p.bwd(window))
        row = {"row": "window", "window": window}
        rates(row, lens, Hq, D, window, f, b)
        if window == (-1, 0):
            causal = (f, b)
        else:
            row.update({"fwd_vs_causal": f / causal[0], "bwd_vs_causal": b / causal[1]})
            if window == (1024, 0):
                row["goal_c_met"] = f <= 0.35 * causal[0] and b <= 0.35 * causal[1]
        emit(row)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
