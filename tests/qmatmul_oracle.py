"""numpy oracle of b200_matmul_quantized: the bit-exact contract stated in include/cubecl_b200.h.

Codes and effective scales are read as tests/quant_oracle.py reads them for b200_dequantize.  Per-block products are exact in
f64 BLAS (|D_j| <= 2^21 < 2^53), scale products are f32 multiplies, and the fold acc = fma(f32(D_j), P, acc) is an exact fma
emulation: the f64 sum of the exact product and acc rounded to odd (TwoSum), then rounded to f32.  Rounding to odd at 53 bits
and then to nearest at 24 bits is the single rounding of the exact value (53 >= 24 + 2).
"""
from __future__ import annotations

import numpy as np

import quant_oracle as qo
from cubecl_b200 import synth

F32, F64 = np.float32, np.float64


def fma_f32(a, b, c) -> np.ndarray:
    """rn_f32(a * b + c) for f32 b, c and integer-valued a with |a| < 2^29 (a * b is then exact in f64)."""
    p = np.asarray(a, F64) * np.asarray(b, F32).astype(F64)
    c = np.asarray(c, F32).astype(F64)
    with np.errstate(invalid="ignore", over="ignore"):
        s = p + c
        bb = s - p
        err = (p - (s - bb)) + (c - bb)
        even = (s.view(np.int64) & 1) == 0
        need = np.isfinite(s) & (err != 0) & even
        s = np.where(need, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)), s)
        return s.astype(F32)


def codes(values, scheme, batch: int, rows: int, K: int) -> np.ndarray:
    """Sign-extended integer codes [batch, rows, K] as f64."""
    v = np.asarray(values).view(np.uint8).reshape(batch, rows, -1)
    return qo.decode(qo.unpack(v, qo.BITS[scheme.value], K), scheme.value).astype(F64)


def block_scales(scheme, raw, tensor_scale, batch: int, rows: int, K: int, bk: int) -> np.ndarray:
    """eff[b, r, j] per kernel block of bk elements: f32(s), rn(g * f32(s)) with two levels, or g."""
    if scheme.block:
        s = qo.scale_load(scheme.block_scale, np.asarray(raw).reshape(-1)).reshape(batch, rows, K // scheme.block)
        if scheme.has_tensor:
            with np.errstate(over="ignore", invalid="ignore"):
                s = (F32(tensor_scale) * s).astype(F32)
        return np.repeat(s, scheme.block // bk, axis=-1)
    return np.full((batch, rows, K // bk), F32(tensor_scale), dtype=F32)


class Operand:
    """Host copy of one quantized operand: scheme, code bytes, stored block scales (or None), f32 tensor scale (or None)."""

    def __init__(self, scheme, values, scales, tensor, batch: int, rows: int, K: int):
        self.scheme, self.values, self.scales, self.tensor = scheme, values, scales, tensor
        self.batch, self.rows, self.K = batch, rows, K

    def codes(self):
        return codes(self.values, self.scheme, self.batch, self.rows, self.K)

    def dequantized(self) -> np.ndarray:
        """f64 values deq = f32(q) * eff (the f32 product b200_dequantize computes)."""
        bk = self.scheme.block or self.K
        eff = np.repeat(block_scales(self.scheme, self.scales, self.tensor, self.batch, self.rows, self.K, bk), bk, axis=-1)
        with np.errstate(over="ignore", invalid="ignore"):
            return (self.codes().astype(F32) * eff).astype(F32).astype(F64)


def kernel_block(a: Operand, b: Operand) -> int:
    present = [s.scheme.block for s in (a, b) if s.scheme.block]
    return min(present) if present else 0


def matmul(a: Operand, b: Operand, rows=None) -> np.ndarray:
    """f32 result [batch, M', N] of the contract (before the output rounding); `rows` selects lhs rows (default all)."""
    rows = np.arange(a.rows) if rows is None else np.asarray(rows)
    A, B = a.codes()[:, rows], b.codes()
    bk = kernel_block(a, b)
    with np.errstate(over="ignore", invalid="ignore"):
        if bk == 0:
            D = np.einsum("bmk,bnk->bmn", A, B)
            gab = F32(F32(a.tensor) * F32(b.tensor))
            return (D.astype(F32) * gab).astype(F32)
        ea = block_scales(a.scheme, a.scales, a.tensor, a.batch, a.rows, a.K, bk)[:, rows]
        eb = block_scales(b.scheme, b.scales, b.tensor, b.batch, b.rows, b.K, bk)
        acc = np.zeros((a.batch, len(rows), b.rows), dtype=F32)
        for j in range(a.K // bk):
            D = np.matmul(A[:, :, j * bk:(j + 1) * bk], B[:, :, j * bk:(j + 1) * bk].transpose(0, 2, 1))
            P = (ea[:, :, j, None] * eb[:, None, :, j]).astype(F32)
            acc = fma_f32(D, P, acc)
        return acc


def to_out(acc, out_dtype: str) -> np.ndarray:
    """Device representation in the output dtype (bf16 / f16 as their bits)."""
    return synth.to_device_dtype(np.asarray(acc, F32), out_dtype)
