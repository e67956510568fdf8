"""GPU: every pooled temporary an entry point stages goes back to the pool when the call returns -- after a call that
succeeds and after one that fails on a host check made once its staging had allocated (a bogus gemm.epilogue or
gemm.variant is refused only when the GEMM is launched).  bytes_in_use must come back to its value before the call."""
import ctypes as C

import numpy as np
import pytest

from cubecl_b200 import TensorHandle, _ffi, conv, quant, reduce, scan
from cubecl_b200.quant import QuantScheme

pytestmark = pytest.mark.gpu

INVALID = 6
_live = []   # the buffers of the running test: a dropped handle would go back to the pool


@pytest.fixture(autouse=True)
def _release_buffers():
    yield
    _live.clear()


def buf(client, nbytes):
    """A zero-filled device buffer (zero codes and scales make every call well defined)."""
    _live.append(TensorHandle.from_numpy(client, np.zeros(nbytes, np.uint8), "u8"))
    return _live[-1].handle.ptr


def u64(v):
    return _ffi.u64_array(list(v))


@pytest.fixture
def in_use(client):
    """Runs a C call and checks its status and that bytes_in_use is back at its starting value."""
    def run(want, fn, *args, options=None):
        client.sync()
        base = client.memory_usage().bytes_in_use
        for k, v in (options or {}).items():
            client.set_option(k, v)
        try:
            rc = fn(client._ctx, None, *args)
        finally:
            for k in options or {}:
                client.set_option(k, {"gemm.epilogue": "tma", "gemm.variant": "auto"}[k])
        assert rc == want, _ffi.load().b200_last_error()
        assert client.memory_usage().bytes_in_use == base
        client.sync()
    return run


def matmul_args(client, idt, odt, esz, M, N, K, lda):
    """lhs [M, K] with row pitch lda (a pitch TMA cannot read is staged), rhs [K, N], out [M, N]."""
    a, b, o = buf(client, M * lda * esz), buf(client, K * N * esz), buf(client, M * N * 4)
    return (idt, odt, a, b, o, 2, u64([M, K]), u64([lda, 1]), u64([K, N]), u64([N, 1]), u64([M, N]), u64([N, 1]))


@pytest.mark.parametrize("options,want", [({}, 0), ({"gemm.epilogue": "bogus"}, INVALID)])
def test_matmul_staged_and_widened(client, in_use, options, want):
    lib = client._lib
    in_use(want, lib.b200_matmul, *matmul_args(client, _ffi.BF16, _ffi.F32, 2, 1024, 512, 513, 516), options=options)
    in_use(want, lib.b200_matmul, *matmul_args(client, _ffi.F8E4M3, _ffi.F32, 1, 1024, 512, 512, 512), options=options)


@pytest.mark.parametrize("mode", ["hybrid", "3xtf32"])
@pytest.mark.parametrize("options,want", [({}, 0), ({"gemm.variant": "bogus"}, INVALID)])
def test_matmul_f32_split(client, in_use, mode, options, want):
    client.set_option("gemm.f32", mode)
    try:
        in_use(want, client._lib.b200_matmul, *matmul_args(client, _ffi.F32, _ffi.F32, 4, 1024, 512, 512, 512), options=options)
    finally:
        client.set_option("gemm.f32", "hybrid")


@pytest.mark.parametrize("options,want", [({}, 0), ({"gemm.epilogue": "bogus"}, INVALID)])
def test_matmul_scaled(client, in_use, options, want):
    M, N, K = 1024, 768, 512
    args = (_ffi.F8E4M3, _ffi.F8E4M3, _ffi.F32, buf(client, M * K), buf(client, N * K), buf(client, M * K // 32),
            buf(client, N * K // 32), buf(client, M * N * 4), 1, M, N, K, 32, 0)
    in_use(want, client._lib.b200_matmul_scaled, *args, options=options)


def qop(client, value, block, rows, K, offset=0):
    s = QuantScheme(value=value, block=block, block_scale="f32" if block else None, tensor=block == 0).to_c()
    scales = buf(client, rows * (K // block) * 4) if block else 0
    return _ffi.QuantOperand(s, buf(client, rows * K + 16) + offset, scales, 0 if block else buf(client, 4))


@pytest.mark.parametrize("fn,value", [("b200_matmul_quantized", "q8s"), ("b200_matmul_quantized", "q4s"),
                                      ("b200_matmul_quantized_fp8", "e4m3")])
@pytest.mark.parametrize("options,want", [({}, 0), ({"gemm.variant": "bogus"}, INVALID)])
def test_matmul_quantized(client, in_use, fn, value, options, want):
    # misaligned codes take the staging pass, then both effective-scale passes; then the GEMM
    M, N, K = 1024, 768, 512
    a, b = qop(client, value, 32, M, K, offset=8), qop(client, value, 32, N, K)
    in_use(want, getattr(client._lib, fn), C.byref(a), C.byref(b), _ffi.F32, buf(client, M * N * 4), 1, M, N, K, options=options)


def test_matmul_quantized_per_tensor_staged(client, in_use):
    M, N, K = 256, 256, 200   # K % 16 != 0: both sides staged
    for fn, value in (("b200_matmul_quantized", "q8s"), ("b200_matmul_quantized_fp8", "e5m2")):
        a, b = qop(client, value, 0, M, K), qop(client, value, 0, N, K)
        in_use(0, getattr(client._lib, fn), C.byref(a), C.byref(b), _ffi.BF16, buf(client, M * N * 2), 1, M, N, K)


def offsets(client, T, G):
    return TensorHandle.from_numpy(client, (np.arange(1, G + 1) * (T // G)).astype(np.int32), "i32").handle.ptr


@pytest.mark.parametrize("options,want", [({}, 0), ({"gemm.epilogue": "bogus"}, INVALID)])
def test_matmul_grouped_staged(client, in_use, options, want):
    # ragged M, lhs [T, K] with a row pitch TMA cannot read and a misaligned rhs: both staged before the launch is planned
    T, G, K, N = 4096, 8, 520, 768
    a, b = buf(client, T * (K + 3) * 2), buf(client, G * K * N * 2 + 16) + 2
    args = (_ffi.BF16, _ffi.BF16, a, 2, u64([T, K]), u64([K + 3, 1]), b, 3, u64([G, K, N]), u64([K * N, N, 1]),
            offsets(client, T, G), G, buf(client, T * N * 2), 2, u64([T, N]), u64([N, 1]), None)
    in_use(want, client._lib.b200_matmul_grouped, *args, options=options)


def test_matmul_grouped_ragged_k_staged(client, in_use):
    T, G, M, N = 4096, 8, 256, 512
    a = buf(client, T * M * 2 + 16) + 2   # misaligned M-contiguous lhs [M, T]
    args = (_ffi.BF16, _ffi.F32, a, 2, u64([M, T]), u64([1, M]), buf(client, T * N * 2), 2, u64([T, N]), u64([N, 1]),
            offsets(client, T, G), G, buf(client, G * M * N * 4), 3, u64([G, M, N]), u64([M * N, N, 1]), None)
    in_use(0, client._lib.b200_matmul_grouped, *args)


@pytest.mark.parametrize("block,K", [(128, 512), (0, 200)])
def test_matmul_grouped_quantized_fp8(client, in_use, block, K):
    T, G, N = 4096, 8, 768
    a, b = qop(client, "e4m3", block, T, K, offset=8), qop(client, "e5m2", block, G * N, K)
    in_use(0, client._lib.b200_matmul_grouped_quantized_fp8, C.byref(a), C.byref(b), offsets(client, T, G), G, _ffi.BF16,
           buf(client, T * N * 2), T, N, K)


@pytest.mark.parametrize("op", ["quantize", "reduce", "scan", "conv"])
def test_gathered_inputs(client, op):
    # a quantize input gathered first, with a tensor level (the amax word); a reduce and a scan of a broadcast view, gathered
    # first; a convolution whose 3 channels are padded to 8
    row = TensorHandle.from_numpy(client, np.ones(2048, np.float32), "f32")
    bcast = TensorHandle(row.handle, [256, 2048], [0, 1], "f32")
    if op == "quantize":
        x = TensorHandle.from_numpy(client, np.ones((64, 96), np.float32), "f32").transposed()
        q = quant.alloc_quantized(client, [96, 64], QuantScheme(value="q8s", block=32, block_scale="f16", tensor=True))
        call = lambda: quant.launch_quantize(client, x, q)   # noqa: E731
    elif op == "reduce":
        out = TensorHandle.empty_contiguous(client, [2048], "f32")
        call = lambda: reduce.launch(client, bcast, out, 0, "sum")   # noqa: E731
    elif op == "scan":
        out = TensorHandle.empty_contiguous(client, [256, 2048], "f32")
        call = lambda: scan.launch(client, bcast, out, 0, "sum")   # noqa: E731
    else:
        x = TensorHandle.from_numpy(client, np.ones((2, 16, 16, 3), np.float16), "f16")
        w = TensorHandle.from_numpy(client, np.ones((8, 3, 3, 3), np.float16), "f16")
        out = TensorHandle.empty_contiguous(client, [2, 14, 14, 8], "f32")
        call = lambda: conv.launch(client, x, w, out)   # noqa: E731
    client.sync()
    base = client.memory_usage().bytes_in_use
    call()
    assert client.memory_usage().bytes_in_use == base
    client.sync()
