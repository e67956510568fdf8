"""CPU: the C++ host logic of the library (validation, batch collapse, variant choice, TMA descriptor geometry, 3xTF32 and
reduce split plans) exercised through a dry-run planning context -- no driver, no device (DryRun, dry_run.rs)."""
import ctypes as C

import pytest

from cubecl_b200 import _ffi

F32, F16, BF16, U32, I32, E4M3 = _ffi.F32, _ffi.F16, _ffi.BF16, _ffi.U32, _ffi.I32, _ffi.F8E4M3
A, B, O = 0x10000000, 0x20000000, 0x30000000


class Planner:
    def __init__(self, sms=132):   # H100 SXM
        self.lib = _ffi.load()
        self.ctx = C.c_void_p()
        _ffi.check(self.lib.b200_plan_begin(sms, C.byref(self.ctx)))

    def close(self):
        self.lib.b200_destroy(self.ctx)

    def text(self):
        need = C.c_size_t()
        _ffi.check(self.lib.b200_plan_text(self.ctx, None, 0, C.byref(need)))
        buf = C.create_string_buffer(need.value)
        _ffi.check(self.lib.b200_plan_text(self.ctx, buf, need.value, None))
        return buf.value.decode()

    def option(self, k, v):
        _ffi.check(self.lib.b200_set_option(self.ctx, k.encode(), str(v).encode()))

    def matmul(self, idt, odt, ls, lst, rs, rst, os_, ost, a=A, b=B, o=O):
        rc = self.lib.b200_matmul(self.ctx, None, idt, odt, a, b, o, len(ls), _ffi.u64_array(ls), _ffi.u64_array(lst),
                                  _ffi.u64_array(rs), _ffi.u64_array(rst), _ffi.u64_array(os_), _ffi.u64_array(ost))
        return rc, self.text()

    def matmul_scaled(self, ldt, rdt, odt, batch, m, n, k, block=32, packed=0, a=A, b=B, o=O, sa=0x40000000, sb=0x50000000):
        rc = self.lib.b200_matmul_scaled(self.ctx, None, ldt, rdt, odt, a, b, sa, sb, o, batch, m, n, k, block, packed)
        return rc, self.text()

    def reduce(self, op, dt, shape, axis, strides=None):
        rc = self.lib.b200_reduce_strided(self.ctx, None, op, dt, A, O, len(shape), _ffi.u64_array(shape),
                                          _ffi.u64_array(strides) if strides else None, axis)
        return rc, self.text()


@pytest.fixture
def plan():
    p = Planner()
    yield p
    p.close()


def cs(shape):
    out, acc = [], 1
    for s in reversed(shape):
        out.append(acc)
        acc *= s
    return out[::-1]


def test_headline_plan_is_one_persistent_2sm_launch(plan):
    n = 8192
    rc, t = plan.matmul(BF16, BF16, [n, n], [n, 1], [n, n], [n, 1], [n, n], [n, 1])
    assert rc == 0
    lines = t.strip().splitlines()
    # 256 x 256 tiles on 66 two-CTA clusters, 384 threads (producer + two wgmma warpgroups)
    # smem: 1 KB alignment slack + 4 x (16 KB of A + 32 KB of B) + 1 KB barriers + 2 x 8 KB epilogue staging
    assert lines[-1] == "launch gemm_bf16_bf16_2sm_n256_kn grid=(132,1,1) block=384 smem=215040 cluster=2"
    # an f32 result runs the same tile
    rc, t32 = plan.matmul(BF16, F32, [n, n], [n, 1], [n, n], [n, 1], [n, n], [n, 1])
    assert rc == 0 and t32.strip().splitlines()[-1] == "launch gemm_bf16_f32_2sm_n256_kn grid=(132,1,1) block=384 smem=215040 cluster=2"
    # A: K-major box [64 k x 128 m]; B (row-major [K,N]): MN-major box [64 n x 64 k]; both SWIZZLE_128B (enum 3)
    assert "tmap esz=2 dims=(8192,8192,1) strides=(16384,134217728) box=(64,128) swizzle=3" in lines[0]
    assert "box=(64,64) swizzle=3" in lines[1]
    # C leaves through TMA stores: (N, M, batch) in [64 col x 64 row] = 128-byte-wide swizzled boxes
    assert "tmap esz=2 dims=(8192,8192,1) strides=(16384,134217728) box=(64,64) swizzle=3" in lines[2]
    assert len(lines) == 4
    plan.option("gemm.epilogue", "direct")
    rc, t = plan.matmul(BF16, BF16, [n, n], [n, 1], [n, n], [n, 1], [n, n], [n, 1])
    assert rc == 0 and t.count("tmap ") == 2
    plan.option("gemm.epilogue", "bogus")
    assert plan.matmul(BF16, BF16, [n, n], [n, 1], [n, n], [n, 1], [n, n], [n, 1])[0] != 0


def test_operand_major_combinations_pick_the_right_kernel(plan):
    n = 1024
    for lhs_t, rhs_t, suffix in ((False, False, "_kn"), (False, True, "_kk"), (True, False, "_mn"), (True, True, "_mk")):
        rc, t = plan.matmul(F16, F32, [n, n], [1, n] if lhs_t else [n, 1], [n, n], [1, n] if rhs_t else [n, 1], [n, n], [n, 1])
        assert rc == 0 and f"launch gemm_f16_f32_" in t and t.strip().endswith("cluster=2") and suffix + " grid" in t


def test_f32_defaults_to_the_hybrid_schedule_with_two_split_passes(plan):
    n = 4096
    rc, t = plan.matmul(F32, F32, [n, n], [n, 1], [n, n], [n, 1], [n, n], [n, 1])
    assert rc == 0
    launches = [ln.split()[1] for ln in t.splitlines() if ln.startswith("launch")]
    # default: tf32 product of the originals + two bf16 cross terms, ONE gemm launch behind two pair-split passes; tf32 wgmma
    # reads K-major operands only, so the row-major [K, N] rhs is first copied K-major
    assert launches == ["repitch_rows", "split_f32_bf16_pair", "split_f32_bf16_pair", "gemm_tf32_f32_2sm_n256_kk"]
    assert t.count("tmap ") == 5                                         # A, B (originals = hi) + bf16 pair buffers + C
    assert t.count("box=(32,128) swizzle=3") == 2                        # f32 K-major operands: [32 k x 128 rows] boxes
    # pair buffers: (K, rows, 2 planes) K-major, box [64 k x 128 rows]; plain 128-byte swizzle
    assert t.count(f"tmap esz=2 dims=({n},{n},2) strides=({2 * n},{2 * n * n}) box=(64,128) swizzle=3") == 2
    assert t.count(f"alloc {n * n * 4}") == 3                            # the K-major rhs copy + two bf16 planes per operand
    # 256 tiles on 66 clusters = 3.88 waves: a stream-K head would gain < 4 %
    assert "stream-k" not in t
    plan.option("gemm.f32", "3xtf32")
    rc, t = plan.matmul(F32, F32, [n, n], [n, 1], [n, n], [n, 1], [n, n], [n, 1])
    assert rc == 0
    launches = [ln.split()[1] for ln in t.splitlines() if ln.startswith("launch")]
    assert launches == ["repitch_rows", "split_tf32_lo", "split_tf32_lo", "gemm_tf32_f32_2sm_n256_kk"]   # lo parts only, ONE gemm launch
    assert t.count("tmap ") == 5                                         # A, B (originals = hi) + A_lo, B_lo + C
    assert t.count(f"alloc {n * n * 4}") == 3                            # the K-major rhs copy + 1x temporaries (lo parts), not 3x
    plan.option("gemm.f32", "tf32")
    rc, t = plan.matmul(F32, F32, [n, n], [n, 1], [n, n], [n, 1], [n, n], [n, 1])
    assert [ln.split()[1] for ln in t.splitlines() if ln.startswith("launch")] == ["repitch_rows", "gemm_tf32_f32_2sm_n256_kk"]
    rc, t = plan.matmul(F32, F32, [n, n], [n, 1], [n, n], [1, n], [n, n], [n, 1])   # K-major rhs: no copy
    assert [ln.split()[1] for ln in t.splitlines() if ln.startswith("launch")] == ["gemm_tf32_f32_2sm_n256_kk"]
    plan.option("gemm.f32", "bogus")
    rc, t = plan.matmul(F32, F32, [n, n], [n, 1], [n, n], [n, 1], [n, n], [n, 1])
    assert rc != 0


def test_hybrid_f32_pair_buffers_follow_operand_major_and_batch(plan):
    """pair buffers [2 planes][entries][rows][pitch]: one entry per batch element, a single one for a broadcast operand; rows of
    K (the tf32 wgmma reads K-major operands, MN-major f32 operands are copied K-major first), pitched to 8 bf16 elements"""
    M, N, K, Bt = 256, 384, 200, 3
    rc, t = plan.matmul(F32, F32, [Bt, M, K], cs([Bt, M, K]), [1, K, N], cs([1, K, N]), [Bt, M, N], cs([Bt, M, N]))
    assert rc == 0
    launches = [ln.split()[1] for ln in t.splitlines() if ln.startswith("launch")]
    assert launches[:3] == ["repitch_rows", "split_f32_bf16_pair", "split_f32_bf16_pair"] and launches[3].startswith("gemm_tf32_f32_") and len(launches) == 4
    assert f"alloc {N * K * 4}" in t                        # rhs broadcast, copied once K-major: [N, K] f32
    assert f"alloc {2 * Bt * M * 200 * 2}" in t            # lhs: 2 planes x 3 entries x [M, pad8(K) = 200] bf16
    assert f"alloc {2 * 1 * N * K * 2}" in t                # rhs broadcast: 2 planes x ONE entry x [N, K] bf16
    assert f"tmap esz=2 dims=({K},{M},{2 * Bt}) strides=({2 * 200},{2 * 200 * M}) box=(64,128) swizzle=3" in t
    assert f"tmap esz=2 dims=({K},{N},2) strides=({2 * 200},{2 * 200 * N}) box=(64,64) swizzle=3" in t
    # transposed views on both sides: lhs MN-major ([K, M] buffer) is copied K-major, rhs K-major ([N, K] buffer) is read in place
    rc, t = plan.matmul(F32, F32, [M, K], [1, M], [K, N], [1, K], [M, N], [N, 1])
    assert rc == 0 and "gemm_tf32_f32_" in t and "_kk grid" in t and t.count("launch repitch_rows") == 1
    assert f"tmap esz=2 dims=({K},{M},2) strides=({2 * 200},{2 * 200 * M}) box=(64,128) swizzle=3" in t
    # K not a multiple of 8: rows pitched to pad8(K)
    rc, t = plan.matmul(F32, F32, [M, 100], [100, 1], [100, N], [N, 1], [M, N], [N, 1])
    assert rc == 0 and f"alloc {2 * M * 104 * 2}" in t and f"dims=(100,{M},2) strides=({2 * 104},{2 * 104 * M})" in t


def test_stream_k_head_policy(plan):
    """Deterministic stream-K head instead of a partial last wave (launch_wgmma / sk_plan): only when the model gains,
    never for integer accumulators; it also feeds the tile choice."""
    def mm(n, k, dt=BF16, out=BF16):
        return plan.matmul(dt, out, [n, k], [k, 1], [k, n], [n, 1], [n, n], [n, 1])
    rc, t = mm(8192, 8192)                     # 1024 tiles = 15.5 waves on 66 clusters: nothing to gain
    assert rc == 0 and "stream-k" not in t and "2sm_n256" in t
    rc, t = mm(4096, 4096)                     # 256 tiles = 3.88 waves: the head would gain < 4 %
    assert rc == 0 and "stream-k" not in t and "2sm_n256" in t
    rc, t = mm(3072, 3072)                     # 144 tiles = 2.18 waves: the 12 tiles of the last wave become the head
    assert rc == 0 and "132 whole tiles + 12 tiles in 60 k-ranges (<= 2 slabs per range)" in t and "2sm_n256" in t
    assert f"alloc {60 * 2 * 256 * 256 * 4}" in t and "grid=(132,1,1)" in t
    rc, t = mm(5120, 5120)                     # 400 tiles: 4 left over after 6 whole waves, 8 ranges each
    assert rc == 0 and "396 whole tiles + 4 tiles in 32 k-ranges" in t
    rc, t = mm(1024, 8192)                     # fewer tiles than clusters: the head is the whole problem
    assert rc == 0 and "0 whole tiles + 32 tiles in 64 k-ranges" in t and "2sm_n128" in t and "grid=(128,1,1)" in t
    rc, t = mm(512, 16384)                     # 8 tiles, 256 k-blocks each: equal parts, the count the model likes best (7)
    assert rc == 0 and "0 whole tiles + 8 tiles in 56 k-ranges" in t
    rc, t = mm(1024, 256)                      # 4 k-blocks: too short to cut
    assert rc == 0 and "stream-k" not in t
    rc, t = mm(2048, 2048)                     # 64 of 66 clusters busy for one wave: an exposed exchange would cost more
    assert rc == 0 and "stream-k" not in t
    rc, t = mm(3072, 3072, dt=8, out=4)        # u8 -> i32: exact integer accumulation stays in one cluster
    assert rc == 0 and "stream-k" not in t
    plan.option("gemm.split_k", "off")
    rc, t = mm(512, 16384)
    assert rc == 0 and "stream-k" not in t
    plan.option("gemm.split_k", "3")           # N = ranges per tile of the head (test knob)
    rc, t = mm(4096, 4096, out=F32)
    assert rc == 0 and "58 tiles in 174 k-ranges" in t
    plan.option("gemm.split_k", "on")
    rc, t = mm(4096, 4096, out=F32)            # 3.88 waves: not worth it under auto, forced here
    assert rc == 0 and "198 whole tiles + 58 tiles in" in t
    plan.option("gemm.split_k", "9")
    rc, t = mm(4096, 4096, out=F32)
    assert rc != 0


def test_block_scaled_plans(plan):
    """b200_matmul_scaled: each operand expanded once to bf16 x * scale, then the bf16 wgmma GEMM with promoted accumulation
    (gemm_mx_*); fallbacks, validation."""
    E5M2, FP4 = _ffi.F8E5M2, _ffi.F4E2M1X2
    rc, t = plan.matmul_scaled(E4M3, E5M2, BF16, 1, 8192, 8192, 8192)
    assert rc == 0
    launches = [ln.split()[1] for ln in t.splitlines() if ln.startswith("launch")]
    assert launches == ["dequant_scaled_bf16", "dequant_scaled_bf16", "gemm_mx_bf16_2sm_n256_kk"]
    assert t.count(f"alloc {8192 * 8192 * 2}") == 2                         # one bf16 [rows, K] copy per operand
    assert t.count("tmap esz=2 dims=(8192,8192,1) strides=(16384,134217728) box=(64,128) swizzle=3") == 2
    assert "block=384 smem=215040 cluster=2" in t
    plan.option("gemm.variant", "2sm_n224")                                 # opt-in 256 x 224 tile for block-scaled kinds
    rc, t = plan.matmul_scaled(E4M3, E5M2, BF16, 1, 8192, 8192, 8192)       # 1 KB + 4 x (16 KB + 28 KB) + 1 KB + 16 KB
    assert rc == 0 and "launch gemm_mx_bf16_2sm_n224_kk grid=(132,1,1) block=384 smem=198656 cluster=2" in t
    assert "tmap esz=2 dims=(8192,8192,1) strides=(16384,134217728) box=(64,112) swizzle=3" in t   # 112 B rows per CTA, multicast
    assert plan.matmul(BF16, BF16, [256, 256], [256, 1], [256, 256], [256, 1], [256, 256], [256, 1])[0] != 0   # block-scaled only
    plan.option("gemm.variant", "auto")
    rc, t = plan.matmul_scaled(FP4, FP4, F32, 2, 4096, 4096, 8192)          # packed e2m1: 8192 elements of K per row
    assert rc == 0 and "gemm_mx_f32_2sm_n256_kk" in t
    assert t.count("tmap esz=2 dims=(8192,4096,2) strides=(16384,67108864) box=(64,128) swizzle=3") == 2
    assert t.count(f"alloc {2 * 4096 * 8192 * 2}") == 2
    rc, t = plan.matmul_scaled(FP4, FP4, BF16, 1, 8192, 8192, 8192, block=16)   # NVFP4
    assert rc == 0 and "gemm_mx_bf16_2sm_n256_kk" in t and t.count("launch dequant_scaled_bf16") == 2
    rc, t = plan.matmul_scaled(E4M3, E4M3, F32, 1, 16, 8, 32)               # the reference's m16 n8 k32 test shape
    assert rc == 0 and "gemm_mx_f32_1sm_n128_kk" in t and "cluster=1" in t
    rc, t = plan.matmul_scaled(E4M3, E4M3, F16, 1, 64, 64, 128, packed=1)   # caller-packed scales are read in place
    assert rc == 0 and "pack_scales" not in t and "gemm_mx_f16_1sm_n128_kk" in t
    rc, t = plan.matmul_scaled(E4M3, E4M3, F32, 1, 64, 64, 128, a=A + 4)    # misaligned operand: reference-order SIMT path
    assert rc == 0 and t.strip().startswith("launch gemm_scaled_simt")
    plan.option("gemm.variant", "simt")
    rc, t = plan.matmul_scaled(E4M3, E4M3, F32, 1, 64, 64, 128)
    assert rc == 0 and "gemm_scaled_simt" in t
    plan.option("gemm.variant", "2sm_n128")
    rc, t = plan.matmul_scaled(E4M3, E4M3, F32, 1, 512, 512, 128)
    assert rc == 0 and "gemm_mx_f32_2sm_n128_kk" in t
    plan.option("gemm.variant", "auto")
    assert plan.matmul_scaled(E4M3, E4M3, F32, 1, 64, 64, 100)[0] != 0      # K not a multiple of the scale block
    assert plan.matmul_scaled(E4M3, E4M3, F32, 1, 64, 64, 128, block=16)[0] != 0
    assert plan.matmul_scaled(E4M3, FP4, F32, 1, 64, 64, 128)[0] != 0       # fp4 cannot mix with fp8
    assert plan.matmul_scaled(BF16, BF16, F32, 1, 64, 64, 128)[0] != 0
    assert plan.matmul_scaled(E4M3, E4M3, I32, 1, 64, 64, 128)[0] != 0
    assert plan.matmul_scaled(E4M3, E4M3, F32, 0, 64, 64, 128) == (0, "")   # empty batch: nothing to do


def test_small_and_unaligned_problems(plan):
    rc, t = plan.matmul(BF16, F32, [100, 64], [64, 1], [64, 72], [72, 1], [100, 72], [72, 1])
    assert rc == 0 and "1sm_n128" in t and "cluster=1" in t               # M <= 128: one CTA per tile
    rc, t = plan.matmul(BF16, F32, [9, 5], [5, 1], [5, 3], [3, 1], [9, 3], [3, 1])
    assert rc == 0 and t.strip() == "launch gemm_simt_strided grid=(1,1,1) block=256 smem=0 cluster=1"   # 10-byte rows: no TMA
    rc, t = plan.matmul(BF16, BF16, [0, 16], [16, 1], [16, 8], [8, 1], [0, 8], [8, 1])
    assert rc == 0 and t == ""                                            # empty output: no launch


def test_batch_broadcast_collapses_or_peels(plan):
    M, N, K = 256, 256, 128
    # fully batched: one launch over 5 batches (3-D descriptors)
    rc, t = plan.matmul(BF16, BF16, [5, M, K], cs([5, M, K]), [5, K, N], cs([5, K, N]), [5, M, N], cs([5, M, N]))
    assert rc == 0 and t.count("launch") == 1 and f"dims=({K},{M},5)" in t
    # rhs broadcast over the batch: descriptor batch extent 1, still one launch
    rc, t = plan.matmul(BF16, BF16, [5, M, K], cs([5, M, K]), [1, K, N], cs([1, K, N]), [5, M, N], cs([5, M, N]))
    assert rc == 0 and t.count("launch") == 1 and f"dims=({N},{K},1)" in t
    # shape.rs:1030-1036: [1,3,M,K] x [2,1,K,N] -> [2,3,M,N]: offsets are not linear in a flat batch index -> peeled into 2 launches
    rc, t = plan.matmul(BF16, BF16, [1, 3, M, K], cs([1, 3, M, K]), [2, 1, K, N], cs([2, 1, K, N]), [2, 3, M, N], cs([2, 3, M, N]))
    assert rc == 0 and t.count("launch") == 2


def test_shape_errors_match_the_reference_rule(plan):
    # shape.rs:1046-1063
    rc, _ = plan.matmul(BF16, BF16, [1, 3, 2, 4], cs([1, 3, 2, 4]), [2, 1, 3, 2], cs([2, 1, 3, 2]), [2, 3, 2, 2], cs([2, 3, 2, 2]))
    assert rc == 6 and b"inner dimensions differ" in plan.lib.b200_last_error()
    rc, _ = plan.matmul(BF16, BF16, [1, 3, 2, 4], cs([1, 3, 2, 4]), [2, 2, 4, 2], cs([2, 2, 4, 2]), [2, 3, 2, 2], cs([2, 3, 2, 2]))
    assert rc == 6 and b"cannot broadcast" in plan.lib.b200_last_error()
    rc, _ = plan.matmul(BF16, F16, [8, 8], [8, 1], [8, 8], [8, 1], [8, 8], [8, 1])
    assert rc == 7                                                         # bf16 in, f16 out: unsupported pair
    rc, t = plan.matmul(E4M3, BF16, [256, 256], [256, 1], [256, 256], [256, 1], [256, 256], [256, 1])
    assert rc == 0                                                         # fp8: both operands widened to f16, f16 kernel
    assert [ln.split()[1] for ln in t.splitlines() if ln.startswith("launch")] == ["convert_fp8_f16", "convert_fp8_f16", "gemm_f16_bf16_2sm_n128_kn"]
    rc, _ = plan.matmul(_ffi.I8, F32, [256, 256], [256, 1], [256, 256], [256, 1], [256, 256], [256, 1])
    assert rc == 7                                                         # int8 accumulates to i32 only


def test_wave_model_prefers_big_tiles(plan):
    # 4096^3: 256 tiles of 256x256 = 3.88 waves on 66 clusters; the 256x128 tile would be 7.76 half-cost waves at an assumed
    # 0.9 of the m64n256 efficiency -> 2sm_n256, for an f32 and a 16-bit result alike
    n = 4096
    rc, t = plan.matmul(BF16, F32, [n, n], [n, 1], [n, n], [n, 1], [n, n], [n, 1])
    assert "gemm_bf16_f32_2sm_n256_kn grid=(132,1,1)" in t
    rc, t = plan.matmul(BF16, BF16, [n, n], [n, 1], [n, n], [n, 1], [n, n], [n, 1])
    assert "gemm_bf16_bf16_2sm_n256_kn grid=(132,1,1)" in t
    # 2048^2 outputs: 64 tiles of 256x256, one wave on 64 of the 66 clusters
    rc, t = plan.matmul(BF16, BF16, [2048, n], [n, 1], [n, 2048], [2048, 1], [2048, 2048], [2048, 1])
    assert "gemm_bf16_bf16_2sm_n256_kn grid=(128,1,1)" in t
    # 1024 x 256 outputs of K = 256: 4 tiles of 256x256 (4 clusters) lose to 8 tiles of 256x128 (8 clusters)
    rc, t = plan.matmul(BF16, BF16, [1024, 256], [256, 1], [256, 1024], [1024, 1], [1024, 1024], [1024, 1])
    assert "gemm_bf16_bf16_2sm_n128_kn grid=(64,1,1)" in t
    plan.option("gemm.variant", "2sm_n128")
    rc, t = plan.matmul(BF16, BF16, [n, n], [n, 1], [n, n], [n, 1], [n, n], [n, 1])
    assert "gemm_bf16_bf16_2sm_n128_kn" in t and "smem=215040" in t           # 1 KB + 6 x (16 KB + 16 KB) + 1 KB
    # a GPU with fewer SMs gets a smaller persistent grid
    small = Planner(sms=64)
    rc, t = small.matmul(BF16, BF16, [n, n], [n, 1], [n, n], [n, 1], [n, n], [n, 1])
    assert "grid=(64,1,1)" in t
    small.close()


def test_reduce_plans(plan):
    SUM, ARGMAX, MEAN = _ffi.REDUCE_SUM, _ffi.REDUCE_ARGMAX, _ffi.REDUCE_MEAN
    rc, t = plan.reduce(SUM, F32, [1 << 28], -1)                          # big value reductions: bulk-copy staged, one CTA per SM
    assert rc == 0 and t.strip() == "launch reduce_all_sum_f32_tma grid=(132,1,1) block=288 smem=98432 cluster=1"
    plan.option("reduce.variant", "u8")                                    # the plain 128-bit streaming form
    rc, t = plan.reduce(SUM, F32, [1 << 28], -1)
    assert rc == 0 and t.strip() == "launch reduce_all_sum_f32 grid=(528,1,1) block=512 smem=0 cluster=1"
    plan.option("reduce.variant", "auto")
    rc, t = plan.reduce(ARGMAX, F32, [1 << 28], -1)
    assert t.strip() == "launch reduce_all_argmax_f32 grid=(528,1,1) block=512 smem=0 cluster=1"
    rc, t = plan.reduce(SUM, F32, [1 << 20], -1)                          # 4 MB: plain loads
    assert "launch reduce_all_sum_f32 grid=(512,1,1) block=512" in t
    rc, t = plan.reduce(SUM, F32, [4], -1)
    assert "grid=(1,1,1)" in t
    rc, t = plan.reduce(SUM, F32, [512, 8192], 1)                          # the book's shape: a 256-thread block per 32 KB row
    assert t.strip() == "launch reduce_rows_sum_f32 grid=(512,1,1) block=256 smem=0 cluster=1"
    rc, t = plan.reduce(SUM, F32, [8192, 8192], 1)                         # 256 MB: 16 vectors per thread, two rows per block
    assert t.strip() == "launch reduce_rows_sum_f32 grid=(4096,1,1) block=256 smem=0 cluster=1"
    rc, t = plan.reduce(SUM, F32, [2048, 8192], 1)                         # 64 MB: 8 vectors per thread, a block per row
    assert t.strip() == "launch reduce_rows_sum_f32 grid=(2048,1,1) block=256 smem=0 cluster=1"
    rc, t = plan.reduce(SUM, F32, [20000, 2048], 1)                        # 8 KB rows: a warp per row, eight rows per block
    assert t.strip() == "launch reduce_rows_sum_f32 grid=(2500,1,1) block=256 smem=0 cluster=1"
    plan.option("reduce.rows_vpt", 8)                                      # tuning knob: vectors per thread
    rc, t = plan.reduce(SUM, F32, [8192, 8192], 1)
    assert t.strip() == "launch reduce_rows_sum_f32 grid=(8192,1,1) block=256 smem=0 cluster=1"
    plan.option("reduce.rows_vpt", "")
    rc, t = plan.reduce(SUM, F32, [1000, 3], 1)                            # short rows: one thread per row
    assert "reduce_rows_sum_f32 grid=(4,1,1) block=256" in t
    rc, t = plan.reduce(SUM, F32, [1 << 26, 4], 1)                         # one vector per row: four rows in flight per thread
    assert "reduce_rows_sum_f32 grid=(65536,1,1) block=256" in t
    rc, t = plan.reduce(SUM, F32, [4, 1 << 24], 1)                         # few long rows: two passes over pooled partials
    assert [ln.split()[1] for ln in t.splitlines() if ln.startswith("launch")] == ["reduce_rows_sum_f32", "reduce_rows_sum_f32"] and "alloc" in t
    assert "grid=(2084,1,1) block=512" in t                                # 521 segments per row
    rc, t = plan.reduce(ARGMAX, BF16, [4, 1 << 24], 1)                     # arg ops split too: (key, index) partials + combine
    assert [ln.split()[1] for ln in t.splitlines() if ln.startswith("launch")] == ["reduce_rows_argmax_bf16", "reduce_argcombine"]
    assert t.count("alloc") == 2
    rc, t = plan.reduce(MEAN, F16, [64, 256, 1024], 1)                     # middle axis -> columns kernel
    assert "reduce_cols_sum_f16" in t
    rc, t = plan.reduce(SUM, F32, [8192, 8192], 0)                         # outer axis, few outputs: 19 segments of the axis (8 blocks
    lines = [ln for ln in t.splitlines() if ln.startswith("launch")]      # per SM), then the partials -- a dependent launch (PDL)
    assert len(lines) == 2 and "reduce_cols_sum_f32_n8 grid=(1088,1,1)" in lines[0] and lines[1].endswith(" pdl")
    plan.option("reduce.cols_fused", "on")                                 # alternative: the last block of a column tile finishes it
    rc, t = plan.reduce(SUM, F32, [8192, 8192], 0)
    assert t.count("launch") == 1
    plan.option("reduce.cols_fused", "off")
    rc, t = plan.reduce(ARGMAX, F32, [1 << 20, 8], 0)                      # arg ops too: (key, index) partials + combine, four loads in flight
    assert [ln.split()[1] for ln in t.splitlines() if ln.startswith("launch")] == ["reduce_cols_argmax_f32", "reduce_argcombine"] and t.count("alloc") == 2
    rc, t = plan.reduce(SUM, F32, [4, 1 << 26], 0)                         # short axis, many columns: persistent grid, one launch
    assert t.strip() == "launch reduce_cols_sum_f32_n8 grid=(1056,1,1) block=256 smem=0 cluster=1"
    # views reduced in place (1x the logical bytes): pitched rows on every axis, transposed views, a permuted rank-3 view
    for axis, kernel in ((1, "reduce_rows_sum_f32"), (0, "reduce_cols_sum_f32_n8"), (-1, "reduce_allp_sum_f32")):
        rc, t = plan.reduce(SUM, F32, [100, 72], axis, strides=[128, 1])
        assert rc == 0 and [ln.split()[1] for ln in t.splitlines()] == [kernel], (axis, t)
    rc, t = plan.reduce(ARGMAX, F32, [100, 72], -1, strides=[128, 1])
    assert [ln.split()[1] for ln in t.splitlines()] == ["reduce_allp_argmax_f32"]
    rc, t = plan.reduce(SUM, F32, [72, 100], 1, strides=[1, 72])           # x.T over its last axis = x over axis 0
    assert [ln.split()[1] for ln in t.splitlines()] == ["reduce_cols_sum_f32_n8"]
    rc, t = plan.reduce(SUM, F32, [72, 100], 0, strides=[1, 72])
    assert [ln.split()[1] for ln in t.splitlines()] == ["reduce_rows_sum_f32"]
    rc, t = plan.reduce(SUM, F32, [3, 5, 7], 1, strides=[35, 1, 5])        # reduced axis innermost in memory, kept axes in order
    assert [ln.split()[1] for ln in t.splitlines()] == ["reduce_rows_sum_f32"]
    # what no (outer stride, axis stride, row pitch) description fits is gathered first: a flat argmax of a transposed view
    # (the index is logical), gaps between outer dimensions
    rc, t = plan.reduce(ARGMAX, F32, [72, 100], -1, strides=[1, 72])
    assert [ln.split()[1] for ln in t.splitlines() if ln.startswith("launch")] == ["gather_strided", "reduce_all_argmax_f32"]
    rc, t = plan.reduce(SUM, F32, [3, 5, 7], 0, strides=[70, 14, 2])
    assert [ln.split()[1] for ln in t.splitlines() if ln.startswith("launch")] == ["gather_strided", "reduce_cols_sum_f32_n8"]
    plan.option("reduce.variant", "tma")                                   # forced: used from 1 MB up
    rc, t = plan.reduce(SUM, BF16, [1 << 20], -1)
    assert t.strip() == "launch reduce_all_sum_bf16_tma grid=(128,1,1) block=288 smem=98432 cluster=1"
    rc, t = plan.reduce(SUM, F32, [1000], -1)                              # too small for a ring: plain loads
    assert "reduce_all_sum_f32 " in t
    plan.option("reduce.variant", "auto")
    rc, _ = plan.reduce(SUM, F32, [4, 0], 1)
    assert rc == 6                                                         # empty reduced extent
    rc, t = plan.reduce(SUM, F32, [0, 4], 1)
    assert rc == 0 and t == ""
    rc, _ = plan.reduce(SUM, U32, [4], -1)
    assert rc == 7


def test_device_only_entry_points_refuse_a_planning_context(plan):
    ev = C.c_void_p()
    assert plan.lib.b200_event_create(plan.ctx, C.byref(ev)) == 7
    assert plan.lib.b200_write(plan.ctx, None, A, None, 16) == 7
    assert plan.lib.b200_sync(plan.ctx, None) == 0


def test_pair_tile_512_plan_has_384_threads_and_no_tail_split(plan):
    n = 8192
    plan.option("gemm.variant", "2sm_m512")
    rc, t = plan.matmul(BF16, BF16, [n, n], [n, 1], [n, n], [n, 1], [n, n], [n, 1])
    assert rc == 0
    lines = t.strip().splitlines()
    # smem: 1 KB slack + 4 x (32 KB of A + 16 KB of B) + 1 KB barriers + 2 x 8 KB epilogue staging = 210 KB
    assert lines[-1] == "launch gemm_bf16_bf16_2sm_m512_kn grid=(132,1,1) block=384 smem=215040 cluster=2"
    assert 215040 <= 232448                                              # sm_90 opt-in maximum per block (227 KB)
    assert "box=(64,128) swizzle=3" in lines[0]                           # A still moves as 128-row boxes (two per stage)
    # 4096^3 on 512 x 128 tiles: 8 x 32 = 256 tiles on 66 pairs; a partial last wave is NOT cut into K-ranges for this tile
    plan.option("gemm.split_k", "4")
    m = 4096
    rc, t = plan.matmul(BF16, BF16, [m, m], [m, 1], [m, m], [m, 1], [m, m], [m, 1])
    assert rc == 0 and "stream-k" not in t and "grid=(132,1,1) block=384" in t
    # small M: 2 tiles of 512 rows x 2 tiles of 128 columns -> 4 pairs
    rc, t = plan.matmul(BF16, F32, [600, 256], [256, 1], [256, 256], [256, 1], [600, 256], [256, 1])
    assert rc == 0 and "gemm_bf16_f32_2sm_m512_kn grid=(8,1,1) block=384" in t
    # fp8 runs the same tile on its exact f16 widening
    rc, t = plan.matmul(E4M3, BF16, [n, n], [n, 1], [n, n], [n, 1], [n, n], [n, 1])
    assert rc == 0 and "launch gemm_f16_bf16_2sm_m512_kn grid=(132,1,1) block=384 smem=215040 cluster=2" in t
    plan.option("gemm.variant", "auto")
    rc, t = plan.matmul(BF16, BF16, [n, n], [n, 1], [n, n], [n, 1], [n, n], [n, 1])
    assert rc == 0 and "2sm_m512" not in t                                # opt-in: never chosen automatically until measured
    plan.option("gemm.variant", "2sm_m512")
    # dtypes without an instantiation are refused, not silently re-routed
    plan.option("gemm.f32", "tf32")
    rc, t = plan.matmul(F32, F32, [n, n], [n, 1], [n, n], [n, 1], [n, n], [n, 1])
    assert rc != 0
