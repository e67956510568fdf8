"""GPU: runtime plumbing behind the C ABI -- pool, generators == host mirror, probes, collectives."""
import threading

import numpy as np
import pytest

from cubecl_b200 import ComputeClient, TensorHandle, reduce, synth

pytestmark = pytest.mark.gpu


def test_props_and_pool(client):
    p = client.properties
    assert p["cc"] == (9, 0) and p["num_streaming_multiprocessors"] >= 100 and p["plane_size_min"] == 32
    before = client.memory_usage()
    h = client.empty(1 << 20)
    mid = client.memory_usage()
    assert mid.bytes_in_use >= before.bytes_in_use + (1 << 20)
    ptr = h.ptr
    del h
    after = client.memory_usage()
    assert after.bytes_in_use == before.bytes_in_use
    client.sync()               # a freed page is reusable by anyone once its last stream has drained
    h2 = client.empty(1 << 20)  # exclusive-page pool: same page comes back
    assert h2.ptr == ptr
    data = np.arange(1000, dtype=np.float32)
    h3 = client.create_from_slice(data)
    assert np.array_equal(np.frombuffer(client.read_one(h3), dtype=np.float32), data)


def test_error_paths_are_loud(client):
    from cubecl_b200 import B200Error, _ffi
    import ctypes as C
    with pytest.raises(B200Error) as ei:
        client.set_option("no.such.option", 1)
    assert ei.value.kind == "InvalidArgument"
    assert client._lib.b200_free(client._ctx, C.c_uint64(0xdead000)) == 6          # pointer not owned by the pool
    h = client.empty(64)
    assert client._lib.b200_free(client._ctx, C.c_uint64(h.ptr)) == 0
    assert client._lib.b200_free(client._ctx, C.c_uint64(h.ptr)) == 6          # double free
    h._owner = False
    bad = C.c_void_p()
    assert client._lib.b200_init(99, C.byref(bad)) == 8                            # no such device
    with pytest.raises(B200Error):
        client.set_option("gemm.variant", "2sm_n512")
        try:
            a = TensorHandle.empty_contiguous(client, [64, 128], "f8e4m3")
            b = TensorHandle.empty_contiguous(client, [128, 64], "f8e4m3")
            o = TensorHandle.empty_contiguous(client, [64, 64], "f32")
            _ffi.check(client._lib.b200_matmul(client._ctx, None, 10, 0, C.c_uint64(a.handle.ptr), C.c_uint64(b.handle.ptr),
                                               C.c_uint64(o.handle.ptr), 2, _ffi.u64_array([64, 128]), _ffi.u64_array([128, 1]),
                                               _ffi.u64_array([128, 64]), _ffi.u64_array([64, 1]), _ffi.u64_array([64, 64]),
                                               _ffi.u64_array([64, 1])))       # no 2sm_n512 variant exists
        finally:
            client.set_option("gemm.variant", "auto")


def test_pool_holds_back_pages_that_are_still_in_flight(client):
    # stream-ordered reuse: a page freed while its last stream still has ~1 ms of queued work must not be handed to a
    # requester without stream affinity until that work has finished; afterwards it is recycled
    n = 1 << 28
    big = client.empty(n * 4)
    for _ in range(8):
        client.fill_uniform(big, "f32", n, 1, 0.0, 1.0)
    ptr = big.ptr
    del big                                      # back to the pool while the fills are still queued
    other = client.empty(n * 4)                  # b200_alloc: no stream affinity -> needs the page's event to be complete
    held_back = other.ptr != ptr
    other_ptr = other.ptr
    client.sync()
    del other
    client.sync()
    again = client.empty(n * 4)
    assert again.ptr in (ptr, other_ptr)         # once drained, cached pages are recycled (no third allocation)
    # 8 fills of 1 GiB take > 1 ms and the host gets here in microseconds, so the page really was in flight
    assert held_back
    del again
    client.memory_cleanup()


def test_buffer_freed_after_its_stream_was_destroyed(client):
    # a handle remembers the non-default stream it was used on and is freed in that stream's order (b200_free_async); if the
    # stream is gone by then (destroyed = drained), the free must fall back to the context's stream, not touch the dead handle
    s = client.create_stream()
    h = client.empty(1 << 20)
    host = client.host_alloc(1 << 20)
    client.write_async(h, host, stream=s)
    assert h.last_stream is s
    client.destroy_stream(s)
    ptr = h.ptr
    del h                                           # used to record an event on the destroyed stream (a host-side fault)
    client.sync()
    again = client.empty(1 << 20)
    assert again.ptr == ptr                         # and the page is immediately reusable: the destroy drained the stream
    client.host_free(host)
    s2 = client.create_stream()                     # a live stream: the page is held back until that stream's event completes
    big = client.empty(1 << 28)
    for _ in range(4):
        client._lib.b200_fill_uniform(client._ctx, s2, 0, __import__("ctypes").c_uint64(big.ptr), 1 << 26, 1, 0.0, 1.0)
    big.used_on(s2)
    p2 = big.ptr
    del big
    other = client.empty(1 << 28)
    assert other.ptr != p2                          # still in flight on s2
    client.sync_stream(s2)
    client.destroy_stream(s2)
    del other
    client.memory_cleanup()


def test_pooled_handles_are_recycled_per_size_class(client):
    before = client.memory_usage()
    hs = [client.empty(3 << 20) for _ in range(4)]
    ptrs = sorted(h.ptr for h in hs)
    del hs
    client.sync()
    again = [client.empty(3 << 20) for _ in range(4)]
    assert sorted(h.ptr for h in again) == ptrs                                    # exclusive pages come back
    del again
    assert client.memory_usage().bytes_in_use == before.bytes_in_use
    client.memory_cleanup()
    assert client.memory_usage().bytes_reserved <= before.bytes_reserved


@pytest.mark.parametrize("dtype", ["f32", "f16", "bf16", "f8e4m3", "f8e5m2"])
def test_device_generator_matches_host_mirror(client, dtype):
    n = 100003
    t = TensorHandle.empty_contiguous(client, [n], dtype)
    client.fill_uniform(t.handle, dtype, n, 77, -1.0, 1.0)
    got = t.to_numpy(client)
    exp = synth.to_device_dtype(synth.uniform_f32(77, n, -1.0, 1.0), dtype)
    assert np.array_equal(got.view(np.uint8), exp.view(np.uint8))
    client.fill_modulo(t.handle, dtype, n, 8)
    assert np.array_equal(synth.from_device_dtype(t.to_numpy(client), dtype), (np.arange(n) % 8).astype(np.float32))


def test_reference_probes_run(client):
    # compute_cmma.rs: A,B = 1, acc = 0, n_iter x mma -> every acc element = 16 * n_iter
    scratch = client.empty(1024)
    ops = client.probe_wmma("f16", 4, scratch)
    client.sync()
    assert ops == client.properties["num_streaming_multiprocessors"] * 32 * 8 * 2 * 16 ** 3 * 4
    assert np.all(np.frombuffer(client.read_one(scratch), dtype=np.float16)[:256] == 64.0)
    # the same accounting on wgmma: per CTA two warpgroups x 4 m64n256k16 per iteration on all-ones operands -> acc = 64 * n_iter
    from cubecl_b200 import B200Error
    ops = client.probe_umma(16, scratch)
    client.sync()
    ctas = client.properties["num_streaming_multiprocessors"]
    assert ops == ctas * 2 * 16 * 4 * 2 * 64 * 256 * 16
    assert np.all(np.frombuffer(client.read_one(scratch), dtype=np.float32)[:ctas] == 1024.0)
    # fp8 peak: K = 32 per wgmma -> acc = 4 * K * n_iter; sm_90 has no block-scaled MMA to probe
    ops = client.probe_umma_kind("f8e4m3", False, 16, scratch)
    client.sync()
    assert ops == ctas * 2 * 16 * 4 * 2 * 64 * 256 * 32
    assert np.all(np.frombuffer(client.read_one(scratch), dtype=np.float32)[:ctas] == 4.0 * 32 * 16)
    for dtype in ("f8e4m3", "f4e2m1x2"):
        with pytest.raises(B200Error):
            client.probe_umma_kind(dtype, True, 16, scratch)
    buf = client.empty(1 << 24)
    client.fill_modulo(buf, "f32", 1 << 22, 2)
    client.probe_memread(buf, 1 << 24, scratch)
    dst = client.empty(1 << 24)
    client.probe_memcopy(dst, buf, 1 << 24)
    assert np.array_equal(np.frombuffer(client.read_one(dst), dtype=np.float32), (np.arange(1 << 22) % 2).astype(np.float32))
    client.probe_memwrite(dst, 1 << 24)
    assert np.array_equal(np.frombuffer(client.read_one(dst), dtype=np.float32)[:8], np.array([1, 2, 3, 4, 1, 2, 3, 4], dtype=np.float32))
    client.sync()


def test_all_reduce_sync_collective(golden):
    # runtime_tests/all_reduce.rs:5-62 -- one client per device in one process, like the reference; needs >= 2 GPUs
    n = ComputeClient.device_count()
    if n < 2:
        pytest.skip("needs at least 2 devices (the reference test returns early too)")
    g = golden["all_reduce"]
    clients = [ComputeClient.load(d) for d in range(n)]
    uid = clients[0].get_unique_id()
    ids = list(range(n))
    threads = [threading.Thread(target=c.ensure_init_collective, args=(ids, uid)) for c in clients]
    [t.start() for t in threads]
    [t.join() for t in threads]
    jobs = []
    for i, c in enumerate(clients):
        handles = [c.create_from_slice(np.full(g["size"], i + j, dtype=np.float32)) for j in range(g["num_handles"])]
        jobs.append((c, handles))

    def issue(c, handles):
        for h in handles:
            c.all_reduce(h, h, "f32", ids, "sum")
        c.sync_collective()

    threads = [threading.Thread(target=issue, args=job) for job in jobs]
    [t.start() for t in threads]
    [t.join() for t in threads]
    base = float(sum(ids))
    for c, handles in jobs:
        for j, h in enumerate(handles):
            got = np.frombuffer(c.read_one(h), dtype=np.float32)
            assert np.all(got == base + j * n)


def test_fused_reduce_all_reduce_over_peer_memory():
    # reduce::launch + client.all_reduce(Sum) as ONE kernel: the last block exchanges the scalar through NVLink mailboxes.
    # Same single-process, one-client-per-device shape as runtime_tests/all_reduce.rs; exact-integer data so the float
    # summation order cannot matter (sum over ranks of sum(i % 8) + rank offsets).
    n_dev = ComputeClient.device_count()
    if n_dev < 2:
        pytest.skip("needs at least 2 devices")
    clients = [ComputeClient.load(d) for d in range(n_dev)]
    exports = [c.p2p_export() for c in clients]
    for c in clients:
        c.p2p_connect(exports)
    ids = list(range(n_dev))
    n = (1 << 22) + 4
    ins, outs, expect = [], [], 0.0
    for r, c in enumerate(clients):
        x = ((np.arange(n) + r) % 8).astype(np.float32)
        expect += float(x.astype(np.float64).sum())
        ins.append(TensorHandle.from_numpy(c, x, "f32"))
        outs.append(TensorHandle.empty_contiguous(c, [1], "f32"))
    for rounds in range(3):  # epochs advance in lockstep; parity double-buffering of the mailbox is exercised
        threads = [threading.Thread(target=reduce.launch_all_reduce, args=(c, ins[r], outs[r], ids)) for r, c in enumerate(clients)]
        [t.start() for t in threads]
        [t.join() for t in threads]
        for r, c in enumerate(clients):
            assert float(outs[r].to_numpy(c)[0]) == expect


def test_fused_argmax_all_reduce_over_peer_memory():
    # outer-axis shards of one logical vector; ties across ranks resolve to the lowest GLOBAL index; first NaN wins
    n_dev = ComputeClient.device_count()
    if n_dev < 2:
        pytest.skip("needs at least 2 devices")
    clients = [ComputeClient.load(d) for d in range(n_dev)]
    exports = [c.p2p_export() for c in clients]
    for c in clients:
        c.p2p_connect(exports)
    ids = list(range(n_dev))
    per = (1 << 20) + 8
    full = synth.uniform_f32(33, per * n_dev, -1.0, 1.0)
    full[[5, per + 17, per * n_dev - 3]] = 7.0          # three equal maxima: global index 5 must win
    cases = [("argmax", full.copy(), 5)]
    mn = full.copy(); mn[per * (n_dev - 1) + 11] = -9.0
    cases.append(("argmin", mn, per * (n_dev - 1) + 11))
    nan = full.copy(); nan[per + 100] = np.nan; nan[per * (n_dev - 1) + 3] = np.nan
    cases.append(("argmax", nan, min(per + 100, per * (n_dev - 1) + 3)))   # with 2 devices both NaNs sit in rank 1's shard
    for op, data, expect in cases:
        ins = [TensorHandle.from_numpy(c, data[r * per:(r + 1) * per], "f32") for r, c in enumerate(clients)]
        outs = [TensorHandle.empty_contiguous(c, [1], "u32") for c in clients]
        threads = [threading.Thread(target=reduce.launch_arg_all_reduce, args=(c, ins[r], outs[r], ids, r * per, op)) for r, c in enumerate(clients)]
        [t.start() for t in threads]
        [t.join() for t in threads]
        for r, c in enumerate(clients):
            assert int(outs[r].to_numpy(c)[0]) == expect
