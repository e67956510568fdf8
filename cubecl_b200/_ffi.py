"""ctypes binding of include/cubecl_b200.h.

Loading this module never needs a GPU (the library dlopen's libcuda lazily), so the CPU test-suite can check that the
library loads and exports every declared symbol.  Any compute call without a GPU fails loudly with B200Error -- there is
no CPU fallback on the product path.
"""
from __future__ import annotations

import ctypes as C
import re
from pathlib import Path

PKG = Path(__file__).resolve().parent
LIB_PATH = PKG / "lib" / "libcubecl_b200.so"
HEADER_PATH = PKG.parent / "include" / "cubecl_b200.h"

# enums (must match the header)
F32, F16, BF16, U32, I32, F64, I64, U64, U8, I8, F8E4M3, F8E5M2, F4E2M1X2, UE8M0 = range(14)
REDUCE_SUM, REDUCE_PROD, REDUCE_MAX, REDUCE_MIN, REDUCE_ARGMAX, REDUCE_ARGMIN, REDUCE_MEAN = range(7)
COMM_SUM, COMM_MEAN = 0, 1
QV_Q8F, QV_E5M2, QV_E4M3, QV_Q4F, QV_E2M1, QV_Q2F, QV_Q8S, QV_Q4S, QV_Q2S = range(9)
UNIQUE_ID_BYTES = 128
IPC_HANDLE_BYTES = 64

STATUS_NAMES = {
    0: "Ok", 1: "CompilationError", 2: "OutOfMemory", 3: "TooManyResources", 4: "Unknown", 5: "IoError",
    6: "InvalidArgument", 7: "Unsupported", 8: "NoDevice", 9: "Communication", 10: "ServerUnhealthy",
}


class B200Error(RuntimeError):
    """Mirrors LaunchError / ServerError (crates/cubecl-runtime/src/server/base.rs:177-272)."""

    def __init__(self, status: int, message: str):
        super().__init__(f"{STATUS_NAMES.get(status, status)}: {message}")
        self.status = status
        self.kind = STATUS_NAMES.get(status, str(status))


class Epilogue(C.Structure):
    _fields_ = [("alpha", C.c_float), ("activation", C.c_int32), ("bias", C.c_uint64)]


class Conv2dArgs(C.Structure):
    """b200_conv2d_args: stride, padding and dilation per spatial axis (h, w)."""
    _fields_ = [("stride_h", C.c_int32), ("stride_w", C.c_int32), ("pad_h", C.c_int32), ("pad_w", C.c_int32),
                ("dilation_h", C.c_int32), ("dilation_w", C.c_int32)]


class Conv3dArgs(C.Structure):
    """b200_conv3d_args: stride, padding and dilation per spatial axis (d, h, w)."""
    _fields_ = [("stride_d", C.c_int32), ("stride_h", C.c_int32), ("stride_w", C.c_int32), ("pad_d", C.c_int32),
                ("pad_h", C.c_int32), ("pad_w", C.c_int32), ("dilation_d", C.c_int32), ("dilation_h", C.c_int32),
                ("dilation_w", C.c_int32)]


class AttentionArgs(C.Structure):
    """b200_attention_args: the score scale and the causal flag (1: key j visible to query i iff j <= i)."""
    _fields_ = [("scale", C.c_float), ("causal", C.c_int32)]


class AttentionVarlenArgs(C.Structure):
    """b200_attention_varlen_args: the score scale, the window (-1: unbounded on that side; (-1, 0) is bottom-right causal)
    and the host bounds on the sequence lengths."""
    _fields_ = [("scale", C.c_float), ("window_left", C.c_int32), ("window_right", C.c_int32), ("max_seqlen_q", C.c_int32),
                ("max_seqlen_k", C.c_int32)]


class QuantScheme(C.Structure):
    """b200_quant_scheme: value (b200_quant_value), block, block_scale (b200_dtype), tensor_scale (0 / 1)."""
    _fields_ = [("value", C.c_int32), ("block", C.c_int32), ("block_scale", C.c_int32), ("tensor_scale", C.c_int32)]


class Props(C.Structure):
    _fields_ = [
        ("device", C.c_int32), ("cc_major", C.c_int32), ("cc_minor", C.c_int32), ("num_sms", C.c_int32),
        ("max_shared_per_block", C.c_int32), ("clock_khz", C.c_int32), ("mem_clock_khz", C.c_int32),
        ("plane_size", C.c_int32), ("total_mem", C.c_uint64), ("name", C.c_char * 128),
    ]


class QuantOperand(C.Structure):
    """b200_quant_operand: a quantized matmul operand (scheme, codes, block scales, device tensor scale)."""
    _fields_ = [("scheme", QuantScheme), ("values", C.c_uint64), ("block_scales", C.c_uint64), ("tensor_scale", C.c_uint64)]


_u64p = C.POINTER(C.c_uint64)
_intp = C.POINTER(C.c_int)
_vp = C.c_void_p

# name -> (restype, argtypes); the CPU tests compare this table with the header.
SIGNATURES = {
    "b200_abi_version": (C.c_int, []),
    "b200_device_count": (C.c_int, [_intp]),
    "b200_get_cubin": (C.c_int, [C.c_char_p, C.POINTER(_vp), C.POINTER(C.c_size_t)]),
    "b200_init": (C.c_int, [C.c_int, C.POINTER(_vp)]),
    "b200_destroy": (C.c_int, [_vp]),
    "b200_plan_begin": (C.c_int, [C.c_int, C.POINTER(_vp)]),
    "b200_plan_text": (C.c_int, [_vp, C.c_char_p, C.c_size_t, C.POINTER(C.c_size_t)]),
    "b200_get_props": (C.c_int, [_vp, C.POINTER(Props)]),
    "b200_set_option": (C.c_int, [_vp, C.c_char_p, C.c_char_p]),
    "b200_launch_count": (C.c_int, [_vp, _u64p]),
    "b200_last_kernel": (C.c_int, [_vp, C.c_char_p, C.c_size_t]),
    "b200_alloc": (C.c_int, [_vp, C.c_size_t, _u64p]),
    "b200_free": (C.c_int, [_vp, C.c_uint64]),
    "b200_free_async": (C.c_int, [_vp, C.c_uint64, _vp]),
    "b200_memory_usage": (C.c_int, [_vp, _u64p, _u64p]),
    "b200_memory_cleanup": (C.c_int, [_vp]),
    "b200_host_alloc": (C.c_int, [_vp, C.c_size_t, C.POINTER(_vp)]),
    "b200_host_free": (C.c_int, [_vp, _vp]),
    "b200_write": (C.c_int, [_vp, _vp, C.c_uint64, _vp, C.c_size_t]),
    "b200_read": (C.c_int, [_vp, _vp, _vp, C.c_uint64, C.c_size_t]),
    "b200_copy": (C.c_int, [_vp, _vp, C.c_uint64, C.c_uint64, C.c_size_t]),
    "b200_memset32": (C.c_int, [_vp, _vp, C.c_uint64, C.c_uint32, C.c_size_t]),
    "b200_stream_create": (C.c_int, [_vp, C.POINTER(_vp)]),
    "b200_stream_destroy": (C.c_int, [_vp, _vp]),
    "b200_sync": (C.c_int, [_vp, _vp]),
    "b200_event_create": (C.c_int, [_vp, C.POINTER(_vp)]),
    "b200_event_record": (C.c_int, [_vp, _vp, _vp]),
    "b200_stream_wait_event": (C.c_int, [_vp, _vp, _vp]),
    "b200_event_elapsed_ms": (C.c_int, [_vp, _vp, _vp, C.POINTER(C.c_float)]),
    "b200_event_destroy": (C.c_int, [_vp, _vp]),
    "b200_matmul": (C.c_int, [_vp, _vp, C.c_int, C.c_int, C.c_uint64, C.c_uint64, C.c_uint64, C.c_int,
                              _u64p, _u64p, _u64p, _u64p, _u64p, _u64p]),
    "b200_matmul_mixed": (C.c_int, [_vp, _vp, C.c_int, C.c_int, C.c_int, C.c_uint64, C.c_uint64, C.c_uint64, C.c_int,
                                    _u64p, _u64p, _u64p, _u64p, _u64p, _u64p]),
    "b200_matmul_fused": (C.c_int, [_vp, _vp, C.c_int, C.c_int, C.c_uint64, C.c_uint64, C.c_uint64, C.c_int,
                                    _u64p, _u64p, _u64p, _u64p, _u64p, _u64p, C.POINTER(Epilogue)]),
    "b200_matmul_scaled": (C.c_int, [_vp, _vp, C.c_int, C.c_int, C.c_int, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64,
                                     C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64, C.c_int, C.c_int]),
    "b200_matmul_quantized": (C.c_int, [_vp, _vp, C.POINTER(QuantOperand), C.POINTER(QuantOperand), C.c_int, C.c_uint64,
                                        C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64]),
    "b200_conv2d": (C.c_int, [_vp, _vp, C.c_int, C.c_int, C.c_uint64, _u64p, _u64p, C.c_uint64, _u64p, _u64p, C.c_uint64, _u64p,
                              _u64p, C.POINTER(Conv2dArgs), C.POINTER(Epilogue)]),
    "b200_conv2d_backward_data": (C.c_int, [_vp, _vp, C.c_int, C.c_int, C.c_uint64, _u64p, _u64p, C.c_uint64, _u64p, _u64p,
                                            C.c_uint64, _u64p, _u64p, C.POINTER(Conv2dArgs)]),
    "b200_conv2d_backward_weight": (C.c_int, [_vp, _vp, C.c_int, C.c_int, C.c_uint64, _u64p, _u64p, C.c_uint64, _u64p, _u64p,
                                              C.c_uint64, _u64p, _u64p, C.POINTER(Conv2dArgs)]),
    "b200_conv2d_grouped": (C.c_int, [_vp, _vp, C.c_int, C.c_int, C.c_uint64, _u64p, _u64p, C.c_uint64, _u64p, _u64p, C.c_uint64,
                                      _u64p, _u64p, C.POINTER(Conv2dArgs), C.c_uint32, C.POINTER(Epilogue)]),
    "b200_conv2d_grouped_backward_data": (C.c_int, [_vp, _vp, C.c_int, C.c_int, C.c_uint64, _u64p, _u64p, C.c_uint64, _u64p, _u64p,
                                                    C.c_uint64, _u64p, _u64p, C.POINTER(Conv2dArgs), C.c_uint32]),
    "b200_conv2d_grouped_backward_weight": (C.c_int, [_vp, _vp, C.c_int, C.c_int, C.c_uint64, _u64p, _u64p, C.c_uint64, _u64p, _u64p,
                                                      C.c_uint64, _u64p, _u64p, C.POINTER(Conv2dArgs), C.c_uint32]),
    "b200_conv3d": (C.c_int, [_vp, _vp, C.c_int, C.c_int, C.c_uint64, _u64p, _u64p, C.c_uint64, _u64p, _u64p, C.c_uint64, _u64p,
                              _u64p, C.POINTER(Conv3dArgs), C.POINTER(Epilogue)]),
    "b200_conv3d_backward_data": (C.c_int, [_vp, _vp, C.c_int, C.c_int, C.c_uint64, _u64p, _u64p, C.c_uint64, _u64p, _u64p,
                                            C.c_uint64, _u64p, _u64p, C.POINTER(Conv3dArgs)]),
    "b200_conv3d_backward_weight": (C.c_int, [_vp, _vp, C.c_int, C.c_int, C.c_uint64, _u64p, _u64p, C.c_uint64, _u64p, _u64p,
                                              C.c_uint64, _u64p, _u64p, C.POINTER(Conv3dArgs)]),
    "b200_conv_transpose2d": (C.c_int, [_vp, _vp, C.c_int, C.c_int, C.c_uint64, _u64p, _u64p, C.c_uint64, _u64p, _u64p, C.c_uint64,
                                        _u64p, _u64p, C.POINTER(Conv2dArgs), C.POINTER(Epilogue)]),
    "b200_conv_transpose3d": (C.c_int, [_vp, _vp, C.c_int, C.c_int, C.c_uint64, _u64p, _u64p, C.c_uint64, _u64p, _u64p, C.c_uint64,
                                        _u64p, _u64p, C.POINTER(Conv3dArgs), C.POINTER(Epilogue)]),
    "b200_attention": (C.c_int, [_vp, _vp, C.c_int, C.c_int, C.c_uint64, _u64p, _u64p, C.c_uint64, _u64p, _u64p, C.c_uint64, _u64p,
                                 _u64p, C.c_uint64, _u64p, _u64p, C.c_uint64, C.POINTER(AttentionArgs)]),
    "b200_attention_backward": (C.c_int, [_vp, _vp, C.c_int, C.c_int, C.c_int] + [C.c_uint64, _u64p, _u64p] * 5 + [C.c_uint64]
                                + [C.c_uint64, _u64p, _u64p] * 3 + [C.POINTER(AttentionArgs)]),
    "b200_attention_varlen": (C.c_int, [_vp, _vp, C.c_int, C.c_int] + [C.c_uint64, _u64p, _u64p] * 3 + [C.c_uint64] * 3
                              + [C.c_uint64, _u64p, _u64p] + [C.c_uint64, C.POINTER(AttentionVarlenArgs)]),
    "b200_attention_varlen_backward": (C.c_int, [_vp, _vp, C.c_int, C.c_int, C.c_int] + [C.c_uint64, _u64p, _u64p] * 5
                                       + [C.c_uint64] * 4 + [C.c_uint64, _u64p, _u64p] * 3 + [C.POINTER(AttentionVarlenArgs)]),
    "b200_attention_kvcache": (C.c_int, [_vp, _vp, C.c_int, C.c_int] + [C.c_uint64, _u64p, _u64p] * 4 + [C.c_uint64]
                               + [C.c_uint64, _u64p, _u64p] + [C.c_uint64, C.POINTER(AttentionArgs)]),
    "b200_kvcache_write": (C.c_int, [_vp, _vp, C.c_int] + [C.c_uint64, _u64p, _u64p] * 4 + [C.c_uint64]),
    "b200_attention_kvcache_fp8": (C.c_int, [_vp, _vp, C.c_int, C.c_int, C.c_int] + [C.c_uint64, _u64p, _u64p] * 4 + [C.c_uint64] * 3
                                   + [C.c_uint64, _u64p, _u64p] + [C.c_uint64, C.POINTER(AttentionArgs)]),
    "b200_kvcache_write_fp8": (C.c_int, [_vp, _vp, C.c_int, C.c_int] + [C.c_uint64, _u64p, _u64p] * 4 + [C.c_uint64] * 3),
    "b200_reduce": (C.c_int, [_vp, _vp, C.c_int, C.c_int, C.c_uint64, C.c_uint64, C.c_int, _u64p, C.c_int]),
    "b200_reduce_strided": (C.c_int, [_vp, _vp, C.c_int, C.c_int, C.c_uint64, C.c_uint64, C.c_int, _u64p, _u64p, C.c_int]),
    "b200_reduce_debug": (C.c_int, [_vp, _vp, _u64p]),
    "b200_into_contiguous": (C.c_int, [_vp, _vp, C.c_int, C.c_uint64, C.c_uint64, C.c_int, _u64p, _u64p]),
    "b200_scan": (C.c_int, [_vp, _vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_uint64, C.c_uint64, C.c_int, _u64p, _u64p, C.c_int]),
    "b200_quantize": (C.c_int, [_vp, _vp, C.POINTER(QuantScheme), C.c_int, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64,
                                C.c_int, _u64p, _u64p]),
    "b200_dequantize": (C.c_int, [_vp, _vp, C.POINTER(QuantScheme), C.c_int, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64,
                                  C.c_int, _u64p]),
    "b200_comm_get_unique_id": (C.c_int, [_vp, _vp]),
    "b200_comm_init": (C.c_int, [_vp, _intp, C.c_int, _vp]),
    "b200_all_reduce": (C.c_int, [_vp, _vp, C.c_uint64, C.c_uint64, C.c_size_t, C.c_int, C.c_int, _intp, C.c_int]),
    "b200_sync_collective": (C.c_int, [_vp, _vp]),
    "b200_p2p_export": (C.c_int, [_vp, _vp, _u64p, C.POINTER(C.c_int64)]),
    "b200_p2p_connect": (C.c_int, [_vp, _intp, C.c_int, _vp, _u64p, C.POINTER(C.c_int64)]),
    "b200_reduce_all_reduce": (C.c_int, [_vp, _vp, C.c_int, C.c_int, C.c_uint64, C.c_uint64, C.c_uint64, _intp, C.c_int]),
    "b200_argreduce_all_reduce": (C.c_int, [_vp, _vp, C.c_int, C.c_int, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64, _intp, C.c_int]),
    "b200_fill_uniform": (C.c_int, [_vp, _vp, C.c_int, C.c_uint64, C.c_uint64, C.c_uint64, C.c_float, C.c_float]),
    "b200_fill_modulo": (C.c_int, [_vp, _vp, C.c_int, C.c_uint64, C.c_uint64, C.c_uint32]),
    "b200_probe_wmma": (C.c_int, [_vp, _vp, C.c_int, C.c_uint32, C.c_uint64, C.POINTER(C.c_double)]),
    "b200_probe_umma": (C.c_int, [_vp, _vp, C.c_uint32, C.c_uint64, C.POINTER(C.c_double)]),
    "b200_probe_umma_kind": (C.c_int, [_vp, _vp, C.c_int, C.c_int, C.c_uint32, C.c_uint64, C.POINTER(C.c_double)]),
    "b200_probe_memread": (C.c_int, [_vp, _vp, C.c_uint64, C.c_uint64, C.c_uint64]),
    "b200_probe_memwrite": (C.c_int, [_vp, _vp, C.c_uint64, C.c_uint64]),
    "b200_probe_memcopy": (C.c_int, [_vp, _vp, C.c_uint64, C.c_uint64, C.c_uint64]),
    "b200_last_error": (C.c_char_p, []),
}

_lib = None


def header_symbols() -> list[str]:
    """Every function the header declares (used by the CPU tests and by load())."""
    text = HEADER_PATH.read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(b200_[a-z0-9_]+)\s*\(", text)))


def load() -> C.CDLL:
    """dlopen the in-tree library; raise if it is missing (the product path never degrades to a CPU implementation)."""
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        # a fresh checkout (built artefacts are git-ignored): build in-tree once; nvcc cross-compiles without a GPU
        try:
            from . import build as _build
            _build.build()
        except Exception as e:  # noqa: BLE001
            raise B200Error(1, f"{LIB_PATH} is missing and could not be built ({e}). There is no CPU fallback.") from e
    lib = C.CDLL(str(LIB_PATH))
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the .so does not export what the header declares
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(status: int) -> None:
    if status != 0:
        msg = load().b200_last_error()
        raise B200Error(status, msg.decode() if msg else "")


def u64_array(values) -> C.Array:
    values = [int(v) for v in values]
    return (C.c_uint64 * len(values))(*values)


def int_array(values) -> C.Array:
    values = [int(v) for v in values]
    return (C.c_int * len(values))(*values)
