"""cubecl_b200: H100-native (sm_90a) implementation of CubeCL's dense linear-algebra hot path.

  matmul.launch / conv.launch / conv3d.launch / conv_transpose.launch / attention.launch / attention.launch_kvcache / reduce.launch / scan.launch / quant.quantize over ComputeClient + TensorHandle  ->  C ABI (include/cubecl_b200.h)
  ->  prebuilt sm_90a cubins: wgmma/TMA GEMM (csrc/gemm_wgmma.cu), fused attention (csrc/attention.cu, attention_bwd.cu), split-KV decoding
      against a paged KV cache (csrc/attention_kv.cu), HBM-bound reductions
      (csrc/reduce.cu), quantization (csrc/quant.cu).

There is no CPU implementation in this package; the CPU oracle lives in /oracle and is test infrastructure only.
"""
from . import attention, conv, conv3d, conv_transpose, matmul, quant, reduce, scan, synth  # noqa: F401
from ._ffi import B200Error  # noqa: F401
from .client import ComputeClient, Handle, ServerError, TensorHandle  # noqa: F401

__all__ = ["ComputeClient", "Handle", "TensorHandle", "ServerError", "B200Error", "attention", "conv", "conv3d", "conv_transpose", "matmul",
           "quant", "reduce", "scan", "synth"]
