"""`matmul::launch` surface (cubek's tiled matmul is out of tree; in-tree contract: shape rule
crates/cubecl-zspace/src/shape.rs:489-517, std-lib op convention `op::launch(client, &TensorHandle...)`
crates/cubecl-std/src/tensor/identity.rs:39-83).

out[..., m, n] = sum_k lhs[..., m, k] * rhs[..., k, n], f32 accumulation, batch dims broadcast.
The kernel behind it is the hand-written wgmma/TMA GEMM in csrc/gemm_wgmma.cu.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _ffi
from ._ffi import B200Error
from .client import ComputeClient, DTYPES, TensorHandle


class MatmulShapeError(ValueError):
    """calculate_matmul_output's error (shape.rs:489-517): rank mismatch or incompatible dims."""


def calculate_matmul_output(shape_lhs, shape_rhs) -> list[int]:
    """Batch-broadcast matmul shape rule, restated from crates/cubecl-zspace/src/shape.rs:489-517:
    equal rank >= 2; leading dims must be equal or one of them 1; inner dims must agree."""
    shape_lhs, shape_rhs = list(shape_lhs), list(shape_rhs)
    rank = len(shape_lhs)
    if rank != len(shape_rhs):
        raise MatmulShapeError(f"rank mismatch: lhs {rank}, rhs {len(shape_rhs)}")
    if rank < 2:
        raise MatmulShapeError("matmul needs rank >= 2")
    out = []
    for l, r in zip(shape_lhs[:-2], shape_rhs[:-2]):
        if l == r or r == 1:
            out.append(l)
        elif l == 1:
            out.append(r)
        else:
            raise MatmulShapeError(f"batch dims {l} and {r} cannot broadcast")
    if shape_lhs[-1] != shape_rhs[-2]:
        raise MatmulShapeError(f"inner dims differ: lhs k={shape_lhs[-1]}, rhs k={shape_rhs[-2]}")
    return out + [shape_lhs[-2], shape_rhs[-1]]


ACTIVATIONS = {None: 0, "none": 0, "relu": 1, "gelu": 2}


def launch(client: ComputeClient, lhs: TensorHandle, rhs: TensorHandle, out: TensorHandle, stream=None,
           alpha: float = 1.0, bias: TensorHandle | None = None, activation: str | None = None) -> None:
    """Enqueue the matmul on the client's stream.  Never raises for launch problems: errors are deferred to
    client.sync()/read_one() like the reference's launch path.
    Optional fused epilogue: out = activation(alpha * (lhs @ rhs) + bias[n]) with `bias` an f32 [N] tensor."""
    if alpha != 1.0 or bias is not None or activation not in (None, "none"):
        return _launch_fused(client, lhs, rhs, out, stream, alpha, bias, activation)
    try:
        for th in (lhs, rhs, out):
            th.handle.used_on(stream)
        rank = len(lhs.shape)
        if len(rhs.shape) != rank or len(out.shape) != rank:
            raise B200Error(6, "matmul: lhs, rhs and out must have equal rank")
        if lhs.dtype != rhs.dtype:
            # mixed 8-bit formats (the reference's manual-MMA pairs: i8 x u8, e4m3 x e5m2 ...); anything else is refused by the library
            _ffi.check(client._lib.b200_matmul_mixed(
                client._ctx, stream, DTYPES[lhs.dtype], DTYPES[rhs.dtype], DTYPES[out.dtype],
                C.c_uint64(lhs.handle.ptr), C.c_uint64(rhs.handle.ptr), C.c_uint64(out.handle.ptr), rank,
                _ffi.u64_array(lhs.shape), _ffi.u64_array(lhs.strides), _ffi.u64_array(rhs.shape), _ffi.u64_array(rhs.strides),
                _ffi.u64_array(out.shape), _ffi.u64_array(out.strides)))
            return
        _ffi.check(client._lib.b200_matmul(
            client._ctx, stream, DTYPES[lhs.dtype], DTYPES[out.dtype],
            C.c_uint64(lhs.handle.ptr), C.c_uint64(rhs.handle.ptr), C.c_uint64(out.handle.ptr), rank,
            _ffi.u64_array(lhs.shape), _ffi.u64_array(lhs.strides), _ffi.u64_array(rhs.shape), _ffi.u64_array(rhs.strides),
            _ffi.u64_array(out.shape), _ffi.u64_array(out.strides)))
    except B200Error as e:
        client._defer(e)


def _launch_fused(client, lhs, rhs, out, stream, alpha, bias, activation) -> None:
    try:
        if activation not in ACTIVATIONS:
            raise B200Error(6, f"unknown activation {activation!r}")
        if bias is not None and (bias.dtype != "f32" or not bias.is_contiguous() or bias.size() != out.shape[-1]):
            raise B200Error(6, "bias must be a contiguous f32 tensor with N elements")
        if lhs.dtype != rhs.dtype:
            raise B200Error(6, f"lhs dtype {lhs.dtype} != rhs dtype {rhs.dtype}")
        rank = len(lhs.shape)
        if len(rhs.shape) != rank or len(out.shape) != rank:
            raise B200Error(6, "matmul: lhs, rhs and out must have equal rank")
        ep = _ffi.Epilogue(float(alpha), ACTIVATIONS[activation], bias.handle.ptr if bias is not None else 0)
        _ffi.check(client._lib.b200_matmul_fused(
            client._ctx, stream, DTYPES[lhs.dtype], DTYPES[out.dtype],
            C.c_uint64(lhs.handle.ptr), C.c_uint64(rhs.handle.ptr), C.c_uint64(out.handle.ptr), rank,
            _ffi.u64_array(lhs.shape), _ffi.u64_array(lhs.strides), _ffi.u64_array(rhs.shape), _ffi.u64_array(rhs.strides),
            _ffi.u64_array(out.shape), _ffi.u64_array(out.strides), C.byref(ep)))
    except B200Error as e:
        client._defer(e)


def launch_scaled(client: ComputeClient, lhs: TensorHandle, rhs: TensorHandle, lhs_scales: TensorHandle, rhs_scales: TensorHandle,
                  out: TensorHandle, stream=None, scale_block: int = 32, scales_packed: bool = False) -> None:
    """Block-scaled (MX) matmul -- the GEMM-level form of MmaDefinition::new_scaled / execute_scaled (frontend/cmma.rs:438-460,
    798-840) with the operand layout of test_cmma_scaled (runtime_tests/cmma.rs:1476-1593):
      lhs [.., M, K] and rhs [.., N, K], both K-contiguous, dtype f8e4m3 / f8e5m2 (mixable) or both f4e2m1x2 (shape [.., rows, K/2]
      bytes); scales ue8m0 [.., rows, K/32]; out [.., M, N] = sum_k (lhs * lhs_scale) * (rhs * rhs_scale), f32 accumulate.
      scale_block=16 selects NVFP4: f4e2m1x2 operands with f8e4m3 scale bytes [.., rows, K/16] (sign ignored).
    Errors are deferred to client.sync() like every launch."""
    try:
        fp4 = lhs.dtype == "f4e2m1x2"
        for t in (lhs, rhs, lhs_scales, rhs_scales, out):
            if not t.is_contiguous():
                raise B200Error(6, "matmul_scaled: tensors must be contiguous (K-major operands)")
        if len(lhs.shape) < 2 or len(lhs.shape) != len(rhs.shape) or lhs.shape[:-2] != rhs.shape[:-2]:
            raise B200Error(6, "matmul_scaled: lhs [..,M,K] and rhs [..,N,K] need equal batch dims")
        if lhs.shape[-1] != rhs.shape[-1]:
            raise B200Error(6, "matmul_scaled: K mismatch")
        M, N = lhs.shape[-2], rhs.shape[-2]
        K = lhs.shape[-1] * (2 if fp4 else 1)
        batch = int(np.prod(lhs.shape[:-2])) if len(lhs.shape) > 2 else 1
        if K % scale_block:
            raise B200Error(6, "matmul_scaled: K must be a multiple of the scale block")
        if list(out.shape) != list(lhs.shape[:-2]) + [M, N]:
            raise B200Error(6, f"matmul_scaled: out shape {out.shape} != {list(lhs.shape[:-2]) + [M, N]}")
        if not scales_packed:
            for t, rows in ((lhs_scales, M), (rhs_scales, N)):
                want = "f8e4m3" if scale_block == 16 else "ue8m0"      # NVFP4 scales are e4m3 bytes (sign ignored)
                if list(t.shape) != list(lhs.shape[:-2]) + [rows, K // scale_block] or t.dtype != want:
                    raise B200Error(6, f"matmul_scaled: scales must be {want} [.., rows, K / scale_block]")
        _ffi.check(client._lib.b200_matmul_scaled(
            client._ctx, stream, DTYPES[lhs.dtype], DTYPES[rhs.dtype], DTYPES[out.dtype],
            C.c_uint64(lhs.handle.ptr), C.c_uint64(rhs.handle.ptr), C.c_uint64(lhs_scales.handle.ptr),
            C.c_uint64(rhs_scales.handle.ptr), C.c_uint64(out.handle.ptr), batch, M, N, K, int(scale_block), int(bool(scales_packed))))
    except B200Error as e:
        client._defer(e)


def launch_quantized(client: ComputeClient, lhs, rhs, out: TensorHandle, stream=None) -> None:
    """Matmul of two integer-quantized tensors (cubecl_b200.quant.QuantizedTensor) on the s8 tensor cores, scales applied
    inside the GEMM: lhs [..., M, K] (activations) and rhs [..., N, K] (weights), both quantized along K with equal leading
    dims (flattened into one batch); out [..., M, N] contiguous f32 / bf16 / f16 = sum_k deq(lhs)[.., m, k] * deq(rhs)[.., n, k].
    Values q8f / q8s / q4f / q4s / q2f / q2s; per-tensor, per-block (32, 64, 128) or two-level scales on either side.  The
    bit-exact arithmetic is stated in include/cubecl_b200.h (b200_matmul_quantized).  Errors are deferred to client.sync()."""
    _launch_q(client, lhs, rhs, out, stream, "matmul_quantized")


def launch_quantized_fp8(client: ComputeClient, lhs, rhs, out: TensorHandle, stream=None) -> None:
    """Matmul of two fp8-quantized tensors (cubecl_b200.quant.QuantizedTensor, values e4m3 or e5m2 on either side) on the fp8
    tensor cores, block scales folded in f32 inside the GEMM: lhs [..., M, K] and rhs [..., N, K] quantized along K with equal
    leading dims (flattened into one batch); out [..., M, N] contiguous f32 / bf16 / f16.  Per-tensor, per-block (32, 64, 128)
    or two-level scales on either side.  The arithmetic is stated in include/cubecl_b200.h (b200_matmul_quantized_fp8).
    Errors are deferred to client.sync()."""
    _launch_q(client, lhs, rhs, out, stream, "matmul_quantized_fp8")


def _launch_q(client, lhs, rhs, out, stream, what: str) -> None:
    """The shared body of launch_quantized / launch_quantized_fp8: b200_<what> on two QuantizedTensors."""
    try:
        ls, rs = list(lhs.shape), list(rhs.shape)
        if len(ls) < 2 or len(ls) != len(rs) or ls[:-2] != rs[:-2]:
            raise B200Error(6, f"{what}: lhs {ls} and rhs {rs} need rank >= 2 and equal leading dims")
        if ls[-1] != rs[-1]:
            raise B200Error(6, f"{what}: K mismatch (lhs {ls[-1]}, rhs {rs[-1]})")
        M, N, K = ls[-2], rs[-2], ls[-1]
        if list(out.shape) != ls[:-2] + [M, N] or not out.is_contiguous():
            raise B200Error(6, f"{what}: out must be contiguous with shape {ls[:-2] + [M, N]}")
        batch = int(np.prod(ls[:-2])) if len(ls) > 2 else 1
        ops = []
        for q in (lhs, rhs):
            for t in (q.values, q.block_scales, q.tensor_scale):
                if t is not None:
                    t.handle.used_on(stream)
            ops.append(_ffi.QuantOperand(q.scheme.to_c(), *(t.handle.ptr if t is not None else 0
                                                              for t in (q.values, q.block_scales, q.tensor_scale))))
        out.handle.used_on(stream)
        fn = getattr(client._lib, "b200_" + what)
        _ffi.check(fn(client._ctx, stream, C.byref(ops[0]), C.byref(ops[1]), DTYPES[out.dtype], C.c_uint64(out.handle.ptr),
                      batch, M, N, K))
    except B200Error as e:
        client._defer(e)


def calculate_grouped_output(shape_lhs, shape_rhs, groups: int) -> list[int]:
    """Output shape of a grouped matmul (torch.nn.functional.grouped_mm with offs): lhs [T, K] x rhs [G, K, N] -> [T, N]
    (ragged M), or lhs [M, T] x rhs [T, N] -> [G, M, N] (ragged K); `groups` is the length of offs."""
    shape_lhs, shape_rhs = list(shape_lhs), list(shape_rhs)
    if len(shape_lhs) == 2 and len(shape_rhs) == 3:
        if shape_lhs[1] != shape_rhs[1]:
            raise MatmulShapeError(f"inner dims differ: lhs k={shape_lhs[1]}, rhs k={shape_rhs[1]}")
        if shape_rhs[0] != groups:
            raise MatmulShapeError(f"{groups} groups in offs, but rhs has {shape_rhs[0]}")
        return [shape_lhs[0], shape_rhs[2]]
    if len(shape_lhs) == 2 and len(shape_rhs) == 2:
        if shape_lhs[1] != shape_rhs[0]:
            raise MatmulShapeError(f"inner dims differ: lhs k={shape_lhs[1]}, rhs k={shape_rhs[0]}")
        return [groups, shape_lhs[0], shape_rhs[1]]
    raise MatmulShapeError(f"grouped matmul takes 2-D x 3-D (ragged M) or 2-D x 2-D (ragged K), not {len(shape_lhs)}-D x "
                           f"{len(shape_rhs)}-D")


def launch_grouped(client: ComputeClient, lhs: TensorHandle, rhs: TensorHandle, offs: TensorHandle, out: TensorHandle,
                   bias: TensorHandle | None = None, alpha: float = 1.0, activation: str | None = None, stream=None) -> None:
    """Grouped matmul for mixture-of-experts layers, the interface of torch.nn.functional.grouped_mm(lhs, rhs, offs=offs):
      ragged M: lhs [T, K] x rhs [G, K, N] -> out [T, N]; rows of group g use rhs[g]; rows >= offs[-1] are not written.
      ragged K: lhs [M, T] (M-contiguous, x.t()) x rhs [T, N] (N-contiguous) -> out [G, M, N], out[g] sums group g's positions.
    offs is a compact i32 [G] device tensor of cumulative ends, read on the device only (no host sync); see b200_matmul_grouped
    in include/cubecl_b200.h for the clamping rule.  Ragged M takes the fused epilogue out = act(alpha * acc + bias[g, n]) with
    an f32 [G, N] bias.  Errors are deferred to client.sync() like every launch."""
    try:
        if activation not in ACTIVATIONS:
            raise B200Error(6, f"unknown activation {activation!r}")
        if lhs.dtype != rhs.dtype:
            raise B200Error(6, f"matmul_grouped: lhs dtype {lhs.dtype} != rhs dtype {rhs.dtype}")
        if offs.dtype != "i32" or len(offs.shape) != 1 or not offs.is_contiguous():
            raise B200Error(6, "matmul_grouped: offs must be a compact i32 [groups] tensor")
        groups = offs.shape[0]
        if bias is not None:
            if bias.dtype != "f32" or not bias.is_contiguous() or list(bias.shape) != [groups, out.shape[-1]]:
                raise B200Error(6, "matmul_grouped: bias must be a contiguous f32 [groups, N] tensor")
        fused = alpha != 1.0 or bias is not None or activation not in (None, "none")
        ep = _ffi.Epilogue(float(alpha), ACTIVATIONS[activation], bias.handle.ptr if bias is not None else 0) if fused else None
        for th in (lhs, rhs, offs, out) + ((bias,) if bias is not None else ()):
            th.handle.used_on(stream)
        _ffi.check(client._lib.b200_matmul_grouped(
            client._ctx, stream, DTYPES[lhs.dtype], DTYPES[out.dtype],
            C.c_uint64(lhs.handle.ptr), len(lhs.shape), _ffi.u64_array(lhs.shape), _ffi.u64_array(lhs.strides),
            C.c_uint64(rhs.handle.ptr), len(rhs.shape), _ffi.u64_array(rhs.shape), _ffi.u64_array(rhs.strides),
            C.c_uint64(offs.handle.ptr), groups,
            C.c_uint64(out.handle.ptr), len(out.shape), _ffi.u64_array(out.shape), _ffi.u64_array(out.strides),
            C.byref(ep) if ep is not None else None))
    except B200Error as e:
        client._defer(e)


def launch_grouped_alloc(client: ComputeClient, lhs: TensorHandle, rhs: TensorHandle, offs: TensorHandle,
                         out_dtype: str | None = None, **kw) -> TensorHandle:
    """Convenience: allocate a contiguous `out` by calculate_grouped_output, then launch_grouped (ragged M leaves the rows
    past the last group uninitialised, as torch does)."""
    shape = calculate_grouped_output(lhs.shape, rhs.shape, offs.shape[0] if len(offs.shape) == 1 else 0)
    out = TensorHandle.empty_contiguous(client, shape, out_dtype or lhs.dtype)
    launch_grouped(client, lhs, rhs, offs, out, **kw)
    return out


def launch_alloc(client: ComputeClient, lhs: TensorHandle, rhs: TensorHandle, out_dtype: str | None = None) -> TensorHandle:
    """Convenience: allocate `out` with the reference's shape rule, then launch."""
    shape = calculate_matmul_output(lhs.shape, rhs.shape)
    out = TensorHandle.empty_contiguous(client, shape, out_dtype or lhs.dtype)
    launch(client, lhs, rhs, out)
    return out
