"""numpy oracle of b200_matmul_quantized_fp8 for exact inputs: the contract of include/cubecl_b200.h with P_j = D_j.

fp8 codes are decoded as tests/quant_oracle.py decodes them for b200_dequantize, effective scales are read as
tests/qmatmul_oracle.py reads them, and blocks fold with its exact fma emulation.  Bk is the finer present block level, or 128
with a short last block when neither side has one.  P_j = D_j holds when every partial sum inside a block is an integer of
magnitude <= 2^11 (the fp8 tensor cores then make no rounding); D_j is then exact in f64 and the fma emulation applies.
"""
from __future__ import annotations

import numpy as np

import qmatmul_oracle as qmo

F32 = np.float32


def kernel_block(a: qmo.Operand, b: qmo.Operand) -> int:
    present = [s.scheme.block for s in (a, b) if s.scheme.block]
    return min(present) if present else 128


def effective(op: qmo.Operand, bk: int) -> np.ndarray:
    """eff[b, r, j] over the ceil(K / bk) kernel blocks."""
    if op.scheme.block:
        return qmo.block_scales(op.scheme, op.scales, op.tensor, op.batch, op.rows, op.K, bk)
    return np.full((op.batch, op.rows, -(-op.K // bk)), F32(op.tensor), dtype=F32)


def matmul(a: qmo.Operand, b: qmo.Operand, rows=None) -> np.ndarray:
    """f32 result [batch, M', N] before the output rounding; `rows` selects lhs rows (default all)."""
    rows = np.arange(a.rows) if rows is None else np.asarray(rows)
    A, B = a.codes()[:, rows], b.codes()
    bk = kernel_block(a, b)
    ea, eb = effective(a, bk)[:, rows], effective(b, bk)
    acc = np.zeros((a.batch, len(rows), b.rows), dtype=F32)
    with np.errstate(over="ignore", invalid="ignore"):
        for j in range(-(-a.K // bk)):
            ks = slice(j * bk, min((j + 1) * bk, a.K))
            D = np.matmul(A[:, :, ks], B[:, :, ks].transpose(0, 2, 1))
            P = (ea[:, :, j, None] * eb[:, None, :, j]).astype(F32)
            acc = qmo.fma_f32(D, P, acc)
    return acc
