"""Host-side mirror of the reference launch surface for the dense-LA path.

Mirrors (same names / argument meaning / error behaviour):
  ComputeClient        crates/cubecl-runtime/src/client.rs:44-48   (create_from_slice:452, empty:654, read_one:256,
                       sync:1013, all_reduce:790, sync_collective:770, memory_usage:1048, memory_cleanup:1115)
  Handle               crates/cubecl-runtime/src/server/handle.rs:10-21 (ref-counted pool slice; freed when dropped)
  TensorHandle         crates/cubecl-std/src/tensor/handle.rs:13-150  (handle + shape + strides in ELEMENTS + dtype)

Error behaviour: like the reference, a launch never raises synchronously -- validation/launch failures are queued on the
client and surface at the next sync()/read_one() (cubecl-cuda/src/compute/server.rs:269-284,981-1002).

Everything here is plumbing over the C ABI (ctypes); no torch, no numpy compute on the product path.
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass
from typing import Iterable, Sequence

import numpy as np

from . import _ffi
from ._ffi import B200Error

DTYPES = {"f32": _ffi.F32, "f16": _ffi.F16, "bf16": _ffi.BF16, "u32": _ffi.U32, "i32": _ffi.I32, "f64": _ffi.F64,
          "i64": _ffi.I64, "u64": _ffi.U64, "u8": _ffi.U8, "i8": _ffi.I8, "f8e4m3": _ffi.F8E4M3, "f8e5m2": _ffi.F8E5M2,
          "f4e2m1x2": _ffi.F4E2M1X2, "ue8m0": _ffi.UE8M0}   # f4e2m1x2: one ELEMENT of this dtype is a byte holding two e2m1
DTYPE_SIZE = {"f32": 4, "f16": 2, "bf16": 2, "u32": 4, "i32": 4, "f64": 8, "i64": 8, "u64": 8, "u8": 1, "i8": 1,
              "f8e4m3": 1, "f8e5m2": 1, "f4e2m1x2": 1, "ue8m0": 1}
# numpy view used when bytes come back to the host (bf16 has no numpy type: raw uint16 bit patterns)
NP_VIEW = {"f32": np.float32, "f16": np.float16, "bf16": np.uint16, "u32": np.uint32, "i32": np.int32, "f64": np.float64,
           "i64": np.int64, "u64": np.uint64, "u8": np.uint8, "i8": np.int8, "f8e4m3": np.uint8, "f8e5m2": np.uint8,
           "f4e2m1x2": np.uint8, "ue8m0": np.uint8}


class ServerError(RuntimeError):
    """ServerError::ServerUnhealthy -- deferred launch errors re-raised at sync/read."""

    def __init__(self, errors):
        super().__init__("ServerUnhealthy: " + "; ".join(str(e) for e in errors))
        self.errors = list(errors)


class Handle:
    """A pooled device buffer. Dropping the last reference returns it to the pool (Handle ref-count semantics)."""

    def __init__(self, client: "ComputeClient", ptr: int, size: int, owner: bool = True):
        self.client, self.ptr, self.size, self._owner = client, ptr, size, owner
        self.last_stream = None   # a non-default stream that was handed this buffer (copies / launches): freed in that stream's order

    def offset(self, start_bytes: int, size: int | None = None) -> "Handle":
        """Sub-slice view (Handle::offset_start); does not own the allocation."""
        h = Handle(self.client, self.ptr + start_bytes, self.size - start_bytes if size is None else size, owner=False)
        h._keep = self  # keep the parent alive
        return h

    def used_on(self, stream) -> None:
        """Remember that work on `stream` touches this buffer (and its parent allocation)."""
        if stream is not None:
            self.last_stream = stream
            parent = getattr(self, "_keep", None)
            if parent is not None:
                parent.used_on(stream)

    def __del__(self):
        if getattr(self, "_owner", False) and self.ptr and self.client is not None and self.client._ctx:
            try:
                if self.last_stream is not None:
                    self.client._lib.b200_free_async(self.client._ctx, C.c_uint64(self.ptr), self.last_stream)
                else:
                    self.client._lib.b200_free(self.client._ctx, C.c_uint64(self.ptr))
            except Exception:
                pass


@dataclass
class MemoryUsage:
    """crates/cubecl-runtime/src/memory_management/base.rs:7-28"""
    bytes_in_use: int
    bytes_reserved: int


class ComputeClient:
    """One client per device; owns the C context, its compute stream and its NCCL communicators."""

    _clients: dict[int, "ComputeClient"] = {}

    def __init__(self, device: int = 0):
        self._lib = _ffi.load()
        ctx = C.c_void_p()
        _ffi.check(self._lib.b200_init(int(device), C.byref(ctx)))
        self._ctx = ctx
        self.device = int(device)
        self._errors: list[Exception] = []
        self._collective_sets: set[tuple[int, ...]] = set()
        props = _ffi.Props()
        _ffi.check(self._lib.b200_get_props(self._ctx, C.byref(props)))
        self._props = props

    # -- R::client(device): one shared client per device (DeviceHandle, cubecl-common/src/device/handle/mod.rs)
    @classmethod
    def load(cls, device: int = 0) -> "ComputeClient":
        if device not in cls._clients:
            cls._clients[device] = cls(device)
        return cls._clients[device]

    @staticmethod
    def device_count() -> int:
        n = C.c_int()
        _ffi.check(_ffi.load().b200_device_count(C.byref(n)))
        return n.value

    def close(self):
        if self._ctx:
            self._lib.b200_destroy(self._ctx)
            self._ctx = None
            ComputeClient._clients.pop(self.device, None)

    # -- properties (client.properties(), HardwareProperties)
    @property
    def properties(self) -> dict:
        p = self._props
        return {"device": p.device, "name": p.name.decode(), "cc": (p.cc_major, p.cc_minor),
                "num_streaming_multiprocessors": p.num_sms, "max_shared_memory_size": p.max_shared_per_block,
                "plane_size_min": p.plane_size, "plane_size_max": p.plane_size, "total_mem": p.total_mem,
                "clock_khz": p.clock_khz, "mem_clock_khz": p.mem_clock_khz, "load_width": 128}

    def set_option(self, key: str, value) -> None:
        _ffi.check(self._lib.b200_set_option(self._ctx, key.encode(), str(value).encode()))

    def last_kernel(self) -> str:
        """Entry-point name of the most recently launched kernel (what a harness reports as the kernel it timed)."""
        buf = C.create_string_buffer(256)
        _ffi.check(self._lib.b200_last_kernel(self._ctx, buf, 256))
        return buf.value.decode()

    def reduce_debug(self, stream=None) -> list[int]:
        """[exchange ns, grid-stage ns, 0, 0] of the last fused reduce + exchange launched with reduce.debug=1."""
        words = (C.c_uint64 * 4)()
        _ffi.check(self._lib.b200_reduce_debug(self._ctx, stream, words))
        return [int(w) for w in words]

    def launch_count(self) -> int:
        n = C.c_uint64()
        _ffi.check(self._lib.b200_launch_count(self._ctx, C.byref(n)))
        return n.value

    # -- memory
    def empty(self, size: int) -> Handle:
        ptr = C.c_uint64()
        _ffi.check(self._lib.b200_alloc(self._ctx, int(size), C.byref(ptr)))
        return Handle(self, ptr.value, int(size))

    def create_from_slice(self, data) -> Handle:
        """Upload host bytes (any buffer / numpy array) into a new pooled buffer."""
        arr = np.ascontiguousarray(data)
        h = self.empty(arr.nbytes)
        if arr.nbytes:
            _ffi.check(self._lib.b200_write(self._ctx, None, C.c_uint64(h.ptr), arr.ctypes.data_as(C.c_void_p), arr.nbytes))
            _ffi.check(self._lib.b200_sync(self._ctx, None))  # pageable source: make the copy complete before returning
        return h

    create = create_from_slice

    def write(self, handle: Handle, data) -> None:
        arr = np.ascontiguousarray(data)
        if arr.nbytes > handle.size:
            raise ValueError("write larger than the buffer")
        _ffi.check(self._lib.b200_write(self._ctx, None, C.c_uint64(handle.ptr), arr.ctypes.data_as(C.c_void_p), arr.nbytes))
        _ffi.check(self._lib.b200_sync(self._ctx, None))

    def read_one(self, handle: Handle) -> bytes:
        """Blocking D2H of the whole buffer; surfaces any deferred error first (Result<Bytes, ServerError>)."""
        out = np.empty(handle.size, dtype=np.uint8)
        if handle.size:
            _ffi.check(self._lib.b200_read(self._ctx, None, out.ctypes.data_as(C.c_void_p), C.c_uint64(handle.ptr), handle.size))
        self.sync()
        return out.tobytes()

    def read_one_array(self, handle: Handle, dtype: str, shape: Sequence[int] | None = None) -> np.ndarray:
        a = np.frombuffer(self.read_one(handle), dtype=NP_VIEW[dtype])
        return a.reshape(shape) if shape is not None else a

    def empty_tensor(self, shape: Sequence[int], elem_size: int):
        """(handle, strides) with the CUDA runtime's pitched layout (client.empty_tensor -> PitchedMemoryLayoutPolicy)."""
        strides, size = pitched_layout(shape, elem_size)
        return self.empty(max(size, 1)), strides

    def memory_usage(self) -> MemoryUsage:
        a, b = C.c_uint64(), C.c_uint64()
        _ffi.check(self._lib.b200_memory_usage(self._ctx, C.byref(a), C.byref(b)))
        return MemoryUsage(a.value, b.value)

    def memory_cleanup(self) -> None:
        _ffi.check(self._lib.b200_memory_cleanup(self._ctx))

    # -- pinned staging + async copies (used by bench.py's end-to-end arm)
    def host_alloc(self, nbytes: int) -> np.ndarray:
        p = C.c_void_p()
        _ffi.check(self._lib.b200_host_alloc(self._ctx, int(nbytes), C.byref(p)))
        buf = (C.c_uint8 * int(nbytes)).from_address(p.value)
        arr = np.frombuffer(buf, dtype=np.uint8)
        self._pinned = getattr(self, "_pinned", {})  # numpy arrays take no attributes: address side table
        self._pinned[arr.ctypes.data] = p.value
        return arr

    def host_free(self, arr: np.ndarray) -> None:
        addr = self._pinned.pop(arr.ctypes.data)
        _ffi.check(self._lib.b200_host_free(self._ctx, C.c_void_p(addr)))

    def write_async(self, handle: Handle, host: np.ndarray, nbytes: int | None = None, stream=None) -> None:
        n = host.nbytes if nbytes is None else nbytes
        handle.used_on(stream)
        _ffi.check(self._lib.b200_write(self._ctx, stream, C.c_uint64(handle.ptr), host.ctypes.data_as(C.c_void_p), n))

    def read_async(self, host: np.ndarray, handle: Handle, nbytes: int | None = None, stream=None) -> None:
        n = host.nbytes if nbytes is None else nbytes
        handle.used_on(stream)
        _ffi.check(self._lib.b200_read(self._ctx, stream, host.ctypes.data_as(C.c_void_p), C.c_uint64(handle.ptr), n))

    # -- extra streams (StreamId -> CUstream, cubecl-cuda/src/compute/stream.rs:24-44); None = the client's compute stream
    def create_stream(self):
        s = C.c_void_p()
        _ffi.check(self._lib.b200_stream_create(self._ctx, C.byref(s)))
        return s

    def destroy_stream(self, stream) -> None:
        _ffi.check(self._lib.b200_stream_destroy(self._ctx, stream))

    def stream_wait_event(self, stream, event) -> None:
        """Cross-stream dependency: work queued on `stream` after this call waits for `event` (MultiStream::resolve)."""
        _ffi.check(self._lib.b200_stream_wait_event(self._ctx, stream, event))

    def sync_stream(self, stream) -> None:
        _ffi.check(self._lib.b200_sync(self._ctx, stream))

    # -- sync / deferred errors
    def _defer(self, err: Exception) -> None:
        self._errors.append(err)

    def flush(self) -> None:
        if self._errors:
            errs, self._errors = self._errors, []
            raise ServerError(errs)

    def sync(self) -> None:
        try:
            _ffi.check(self._lib.b200_sync(self._ctx, None))
        except B200Error as e:
            self._errors.append(e)
        self.flush()

    # -- timing (CUDA events on the launching stream)
    def event(self):
        e = C.c_void_p()
        _ffi.check(self._lib.b200_event_create(self._ctx, C.byref(e)))
        return e

    def record(self, e, stream=None) -> None:
        _ffi.check(self._lib.b200_event_record(self._ctx, e, stream))

    def elapsed_ms(self, a, b) -> float:
        ms = C.c_float()
        _ffi.check(self._lib.b200_event_elapsed_ms(self._ctx, a, b, C.byref(ms)))
        return ms.value

    def event_destroy(self, e) -> None:
        _ffi.check(self._lib.b200_event_destroy(self._ctx, e))

    # -- collectives (ServerCommunication)
    def get_unique_id(self) -> bytes:
        buf = (C.c_uint8 * _ffi.UNIQUE_ID_BYTES)()
        _ffi.check(self._lib.b200_comm_get_unique_id(self._ctx, buf))
        return bytes(buf)

    def ensure_init_collective(self, device_ids: Iterable[int], unique_id: bytes) -> None:
        """client.rs:755-767.  The reference shares the ncclUniqueId through a process-global map
        (communication.rs:11-25); with one process per GPU the caller passes the id it exchanged (see distributed.py)."""
        ids = tuple(sorted(int(d) for d in device_ids))
        if ids in self._collective_sets:
            return
        arr = _ffi.int_array(ids)
        buf = (C.c_uint8 * _ffi.UNIQUE_ID_BYTES).from_buffer_copy(unique_id)
        _ffi.check(self._lib.b200_comm_init(self._ctx, arr, len(ids), buf))
        self._collective_sets.add(ids)

    def all_reduce(self, src: Handle, dst: Handle, dtype: str, device_ids: Iterable[int], op: str = "sum") -> None:
        ids = sorted(int(d) for d in device_ids)
        try:
            _ffi.check(self._lib.b200_all_reduce(self._ctx, None, C.c_uint64(src.ptr), C.c_uint64(dst.ptr), src.size,
                                                 DTYPES[dtype], _ffi.COMM_MEAN if op == "mean" else _ffi.COMM_SUM,
                                                 _ffi.int_array(ids), len(ids)))
        except B200Error as e:
            self._defer(e)

    def sync_collective(self) -> None:
        try:
            _ffi.check(self._lib.b200_sync_collective(self._ctx, None))
        except B200Error as e:
            self._defer(e)

    # -- peer-memory exchange (fused reduce + all-reduce over NVLink)
    def p2p_export(self) -> tuple[int, bytes, int, int]:
        """(device, ipc handle, mailbox pointer, pid) to be exchanged with the other ranks."""
        h = (C.c_uint8 * _ffi.IPC_HANDLE_BYTES)()
        ptr, pid = C.c_uint64(), C.c_int64()
        _ffi.check(self._lib.b200_p2p_export(self._ctx, h, C.byref(ptr), C.byref(pid)))
        return self.device, bytes(h), ptr.value, pid.value

    def p2p_connect(self, exports) -> None:
        """exports: list of p2p_export() tuples of every rank of the device set (any order)."""
        exports = sorted(exports, key=lambda e: e[0])
        ids = _ffi.int_array([e[0] for e in exports])
        handles = (C.c_uint8 * (len(exports) * _ffi.IPC_HANDLE_BYTES)).from_buffer_copy(b"".join(e[1] for e in exports))
        ptrs = _ffi.u64_array([e[2] for e in exports])
        pids = (C.c_int64 * len(exports))(*[int(e[3]) for e in exports])
        _ffi.check(self._lib.b200_p2p_connect(self._ctx, ids, len(exports), handles, ptrs, pids))

    # -- synthetic operands / probes
    def fill_uniform(self, handle: Handle, dtype: str, n: int, seed: int, lo: float, hi: float) -> None:
        _ffi.check(self._lib.b200_fill_uniform(self._ctx, None, DTYPES[dtype], C.c_uint64(handle.ptr), int(n), int(seed), float(lo), float(hi)))

    def fill_modulo(self, handle: Handle, dtype: str, n: int, modulus: int) -> None:
        _ffi.check(self._lib.b200_fill_modulo(self._ctx, None, DTYPES[dtype], C.c_uint64(handle.ptr), int(n), int(modulus)))

    def probe_wmma(self, dtype: str, n_iter: int, scratch: Handle) -> float:
        ops = C.c_double()
        _ffi.check(self._lib.b200_probe_wmma(self._ctx, None, DTYPES[dtype], int(n_iter), C.c_uint64(scratch.ptr), C.byref(ops)))
        return ops.value

    def probe_umma(self, n_iter: int, scratch: Handle) -> float:
        ops = C.c_double()
        _ffi.check(self._lib.b200_probe_umma(self._ctx, None, int(n_iter), C.c_uint64(scratch.ptr), C.byref(ops)))
        return ops.value

    def probe_umma_kind(self, dtype: str, block_scaled: bool, n_iter: int, scratch: Handle) -> float:
        """wgmma peak probe for bf16 or fp8 e4m3 operands (block-scaled kinds raise: sm_90 has no block-scaled MMA); returns the op count of the launch."""
        ops = C.c_double()
        _ffi.check(self._lib.b200_probe_umma_kind(self._ctx, None, DTYPES[dtype], int(bool(block_scaled)), int(n_iter),
                                                  C.c_uint64(scratch.ptr), C.byref(ops)))
        return ops.value

    def probe_memread(self, buf: Handle, nbytes: int, scratch: Handle) -> None:
        _ffi.check(self._lib.b200_probe_memread(self._ctx, None, C.c_uint64(buf.ptr), int(nbytes), C.c_uint64(scratch.ptr)))


    def probe_memwrite(self, dst: Handle, nbytes: int) -> None:
        _ffi.check(self._lib.b200_probe_memwrite(self._ctx, None, C.c_uint64(dst.ptr), int(nbytes)))

    def probe_memcopy(self, dst: Handle, src: Handle, nbytes: int) -> None:
        _ffi.check(self._lib.b200_probe_memcopy(self._ctx, None, C.c_uint64(dst.ptr), C.c_uint64(src.ptr), int(nbytes)))


def optimal_align(last_dim: int, elem_size: int, buffer_align: int = 512) -> int:
    """crates/cubecl-runtime/src/memory_management/memory_pool/handle.rs:255-263: unit rows stay contiguous, otherwise the
    row byte size rounded up to a power of two, clamped to [16, buffer_align] (mem_alignment = 512 on CUDA, runtime.rs:81)."""
    if last_dim == 1:
        return elem_size
    row = last_dim * elem_size
    return min(max(1 << max(0, (row - 1).bit_length()), 16), buffer_align)


def pitched_layout(shape: Sequence[int], elem_size: int, mem_alignment: int = 512) -> tuple[list[int], int]:
    """(strides in elements, allocation bytes) of PitchedMemoryLayoutPolicy::apply with MemoryLayoutStrategy::Optimized
    (crates/cubecl-runtime/src/allocator.rs:21-72): pitch = row bytes rounded up to optimal_align; strides[rank-2] =
    pitch / elem_size; outer strides compact over that."""
    shape = [int(s) for s in shape]
    rank = len(shape)
    width = shape[-1] if rank else 1
    height = 1
    for s in shape[:-1]:
        height *= s
    height = max(height, 1)
    align = optimal_align(width, elem_size, mem_alignment)
    width_bytes = width * elem_size
    pitch = (width_bytes + align - 1) // align * align
    strides = [1] * rank
    if rank > 1:
        strides[rank - 2] = pitch // elem_size
    for i in range(rank - 3, -1, -1):
        strides[i] = strides[i + 1] * shape[i + 1]
    return strides, height * pitch


def contiguous_strides(shape: Sequence[int]) -> list[int]:
    strides, acc = [], 1
    for s in reversed(shape):
        strides.append(acc)
        acc *= int(s)
    return strides[::-1]


class TensorHandle:
    """crates/cubecl-std/src/tensor/handle.rs:13-23: {handle, shape, strides (elements), dtype}."""

    def __init__(self, handle: Handle, shape: Sequence[int], strides: Sequence[int], dtype: str):
        if dtype not in DTYPES:
            raise ValueError(f"unknown dtype {dtype}")
        self.handle, self.shape, self.strides, self.dtype = handle, [int(s) for s in shape], [int(s) for s in strides], dtype

    @classmethod
    def new_contiguous(cls, shape, handle: Handle, dtype: str) -> "TensorHandle":
        return cls(handle, shape, contiguous_strides(shape), dtype)

    @classmethod
    def empty(cls, client: ComputeClient, shape, dtype: str) -> "TensorHandle":
        """Pitched layout, like TensorHandle::empty -> client.empty_tensor (handle.rs:72-86)."""
        h, strides = client.empty_tensor(shape, DTYPE_SIZE[dtype])
        return cls(h, shape, strides, dtype)

    @classmethod
    def empty_contiguous(cls, client: ComputeClient, shape, dtype: str) -> "TensorHandle":
        n = math.prod(int(s) for s in shape)
        return cls.new_contiguous(shape, client.empty(max(1, n * DTYPE_SIZE[dtype])), dtype)

    @classmethod
    def zeros(cls, client: ComputeClient, shape, dtype: str) -> "TensorHandle":
        t = cls.empty(client, shape, dtype)
        words = (t.handle.size + 3) // 4
        _ffi.check(client._lib.b200_memset32(client._ctx, None, C.c_uint64(t.handle.ptr), 0, words))
        return t

    @classmethod
    def from_numpy(cls, client: ComputeClient, array: np.ndarray, dtype: str) -> "TensorHandle":
        """Contiguous upload. For bf16 pass uint16 bit patterns (see synth.f32_to_bf16_bits)."""
        arr = np.ascontiguousarray(array)
        if arr.dtype.itemsize != DTYPE_SIZE[dtype]:
            raise ValueError(f"array itemsize {arr.dtype.itemsize} does not match {dtype}")
        return cls.new_contiguous(arr.shape, client.create_from_slice(arr), dtype)

    def size(self) -> int:
        return math.prod(self.shape)

    def is_contiguous(self) -> bool:
        return self.strides == contiguous_strides(self.shape)

    def transposed(self) -> "TensorHandle":
        """Swap the last two dims without moving data (MatrixBatchLayout::MildlyPermuted{transposed})."""
        sh, st = list(self.shape), list(self.strides)
        sh[-1], sh[-2] = sh[-2], sh[-1]
        st[-1], st[-2] = st[-2], st[-1]
        return TensorHandle(self.handle, sh, st, self.dtype)

    def to_numpy(self, client: ComputeClient) -> np.ndarray:
        """Download honouring strides (pitched rows are compacted on the host)."""
        raw = np.frombuffer(client.read_one(self.handle), dtype=NP_VIEW[self.dtype])
        if not self.shape:
            return raw[:1].reshape(())
        return np.lib.stride_tricks.as_strided(raw, shape=self.shape,
                                               strides=[s * raw.itemsize for s in self.strides]).copy()
