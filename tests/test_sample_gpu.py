"""GPU: b200_sample against tests/sample_oracle.py, ids compared bit for bit -- exact rows (every w a power of two or +0) for
every logits dtype and ids dtype at vocabularies from 1 to 262144 under greedy, top-k, top-p, min-p and all combined, with
per-row parameter arrays; random bf16 rows wherever the oracle's margin exceeds ex2's error bound (the skipped fraction is
printed and must stay below 1%); a chi-square test of 2^16 draws of one row against the oracle's probabilities; a mixed batch
with every invalid per-row value; batch invariance; pitched and misaligned views; advance_offsets; and a decode step through
b200_matmul and b200_cross_entropy."""
import numpy as np
import pytest
import torch

import sample_oracle as so
from cross_entropy_oracle import rnd
from cubecl_b200 import TensorHandle, cross_entropy as xent, sample as smp, synth

pytestmark = pytest.mark.gpu

VS = [1, 7, 1000, 16384, 16385, 32000, 50257, 128256, 151936, 262144]
CELLS = [("f32", "i64"), ("f32", "i32"), ("bf16", "i64"), ("bf16", "i32"), ("f16", "i64"), ("f16", "i32")]
NAN, INF = float("nan"), float("inf")


def up(c, arr, dtype):
    return TensorHandle.from_numpy(c, synth.to_device_dtype(np.asarray(arr, np.float32), dtype), dtype)


def arr(c, a, dtype):
    npdt = {"f32": np.float32, "i32": np.int32, "u64": np.uint64, "i64": np.int64}[dtype]
    return TensorHandle.from_numpy(c, np.asarray(a).astype(npdt).reshape(-1), dtype)


def run(c, x, dtype, ids_dtype="i64", per_row=True, **params):
    """ids of one call on rows x, each parameter passed as a per-row array when per_row and it is a sequence"""
    X = up(c, x, dtype)
    kw = {}
    for name, val in params.items():
        if per_row and np.ndim(val):
            kw[name] = arr(c, val, {"temperature": "f32", "top_k": "i32", "top_p": "f32", "min_p": "f32", "seed": "u64",
                                    "offset": "u64"}[name])
        else:
            kw[name] = val
    ids = smp.sample_alloc(c, X, ids_dtype=ids_dtype, **kw)
    c.sync()
    return ids.to_numpy(c).astype(np.int64)


# ---------------------------------------------------------------------------------------------- exact rows
@pytest.mark.parametrize("cell", CELLS, ids=lambda c: "-".join(c))
@pytest.mark.parametrize("v", VS)
def test_exact_rows_match_oracle_bitwise(client, v, cell):
    dtype, ids_dtype = cell
    rng = np.random.default_rng(v * 7 + len(dtype))
    x, params = so.exact_batch(rng, v, dtype)
    ref, margin, _ = so.sample(x, **params)
    got = run(client, x, dtype, ids_dtype, **params)
    np.testing.assert_array_equal(got, ref)
    # the same rows with each configuration as the call's scalars
    for r in (1, 6, 9, 12, 13):
        one = {k: (val[r] if np.ndim(val) else val) for k, val in params.items()}
        got1 = run(client, x[r:r + 1], dtype, ids_dtype, **{k: (int(a) if k in ("top_k", "seed", "offset") else float(a))
                                                             for k, a in one.items()})
        assert got1[0] == ref[r], (r, got1, ref[r])


# ---------------------------------------------------------------------------------------------- random rows
RANDOM_CONF = [(1.0, 50, 0.9, 0.05), (0.7, 0, 0.9, 0.0), (1.0, 200, 1.0, 0.0), (1.2, 0, 1.0, 0.1), (0.8, 1000, 0.95, 0.02),
               (1.0, 20, 1.0, 0.0)]


@pytest.mark.parametrize("v", [32000, 128256, 151936])
def test_random_rows_match_oracle_within_margin(client, v):
    rng = np.random.default_rng(v + 11)
    b = 96
    x = rnd(rng.standard_normal((b, v)).astype(np.float32) * 3, "bf16")
    conf = [RANDOM_CONF[r % len(RANDOM_CONF)] for r in range(b)]
    params = dict(temperature=np.array([c[0] for c in conf], np.float32), top_k=np.array([c[1] for c in conf]),
                  top_p=np.array([c[2] for c in conf], np.float32), min_p=np.array([c[3] for c in conf], np.float32),
                  seed=rng.integers(0, 2 ** 63, size=b, dtype=np.int64).astype(np.uint64),
                  offset=rng.integers(0, 2 ** 40, size=b, dtype=np.int64).astype(np.uint64))
    ref, margin, bound = so.sample(x, **params)
    got = run(client, x, "bf16", **params)
    safe = margin > bound
    print(f"v={v}: {np.count_nonzero(~safe)} of {b} rows skipped (margin within the ex2 bound)")
    assert np.mean(~safe) < 0.01
    np.testing.assert_array_equal(got[safe], ref[safe])
    assert np.all(got >= 0)


# ---------------------------------------------------------------------------------------------- distribution
def test_distribution_of_one_row_chi_square(client):
    from scipy.stats import chisquare
    rng = np.random.default_rng(12)
    v, n = 1000, 1 << 16
    row = so.exact_rows(rng, 1, v, "f32")[0]
    x = np.broadcast_to(row, (n, v))
    params = dict(temperature=1.0, top_k=300, top_p=0.95, min_p=2.0 ** -12, seed=0x5EED, offset=np.arange(n, dtype=np.uint64))
    got = run(client, x, "f32", **params)
    # the oracle's ids for every offset (its masses are exact on this row), and its probabilities
    ref = np.array([so.sample_row(row, 1.0, 300, 0.95, 2.0 ** -12, 0x5EED, o)[0] for o in range(0, n, 257)])
    np.testing.assert_array_equal(got[::257], ref)
    z = row
    w = so.ex2(((z - z.max()).astype(np.float32) * so.LOG2E).astype(np.float32))
    q = so.masses(w).astype(np.float64)
    keep = (z >= np.sort(z)[v - 300]) & (w >= np.float32(2.0 ** -12))
    tau = so._nucleus(so.masses(w), keep, np.float32(0.95))[0]
    keep &= so.masses(w) >= np.uint64(tau)
    p = np.where(keep, q, 0) / q[keep].sum()
    assert np.all(keep[got]), "drew a token outside the nucleus"
    counts = np.bincount(got, minlength=v).astype(np.float64)
    exp = p * n
    big = exp >= 5
    obs = np.append(counts[big], counts[~big].sum())
    ex = np.append(exp[big], exp[~big].sum())
    if ex[-1] == 0:
        obs, ex = obs[:-1], ex[:-1]
    stat, pval = chisquare(obs, ex)
    print(f"chi-square over {len(obs)} bins: {stat:.1f}, p = {pval:.3f}")
    assert pval > 1e-3


# ---------------------------------------------------------------------------------------------- mixed batch and invalid rows
def test_mixed_batch_and_invalid_rows(client):
    rng = np.random.default_rng(13)
    v = 32000
    conf = [(0.0, 0, 1.0, 0.0), (1.0, 40, 1.0, 0.0), (1.0, 0, 0.8, 0.0), (1.0, 0, 1.0, 0.2), (0.8, 30, 0.9, 0.05),
            (-1.0, 0, 1.0, 0.0), (NAN, 0, 1.0, 0.0), (INF, 0, 1.0, 0.0), (1.0, 0, 0.0, 0.0), (1.0, 0, 1.5, 0.0),
            (1.0, 0, NAN, 0.0), (1.0, 0, 1.0, -0.1), (1.0, 0, 1.0, 1.5), (1.0, 0, 1.0, NAN), (0.0, 5, 0.0, 0.0),
            (0.0, 0, 1.0, 0.0), (0.0, 0, 1.0, 0.0), (0.0, 0, 1.0, 0.0), (1.0, 0, 1.0, 0.0), (1.0, 0, 1.0, 0.0),
            (1.0, 0, 1.0, 0.0), (1e-30, 0, 1.0, 0.0), (-0.0, 0, 1.0, 0.0)]
    b = len(conf)
    x = rnd(rng.standard_normal((b, v)).astype(np.float32) * 3, "bf16")
    x[15, 100] = NAN                    # greedy row with a NaN
    x[16, 200] = INF                    # greedy row with +inf
    x[17, :] = -INF                     # greedy row all -inf
    x[18, 300] = NAN                    # sampled rows: NaN, +inf, all -inf
    x[19, 400] = INF
    x[20, :] = -INF
    x[:, 5:9] = -INF                    # -inf columns are fine elsewhere
    x[0, 7000] = x[0, 7001] = x[0].max() + 1   # a greedy tie: the lower index wins
    x = rnd(x, "bf16")
    cols = list(zip(*conf))
    params = dict(temperature=np.array(cols[0], np.float32), top_k=np.array(cols[1]), top_p=np.array(cols[2], np.float32),
                  min_p=np.array(cols[3], np.float32), seed=np.arange(b, dtype=np.uint64) + 99, offset=np.uint64(5) + np.zeros(b, np.uint64))
    ref, margin, bound = so.sample(x, **params)
    got = run(client, x, "bf16", **params)
    assert np.all(margin > bound)
    np.testing.assert_array_equal(got, ref)
    assert np.all(got[5:21] == -1) and np.all(got[:5] >= 0)
    assert got[0] == 7000 and got[21] >= 0 and got[22] == int(np.argmax(x[22]))
    xt = torch.tensor(x, dtype=torch.float32)
    for r in (0, 22):
        assert got[r] == int(torch.argmax(xt[r]))


def test_greedy_only_launch_matches_argmax(client):
    rng = np.random.default_rng(14)
    for v in (1, 1000, 50257, 128256, 262144):
        x = rnd(rng.standard_normal((33, v)).astype(np.float32) * 2, "bf16")
        x[3, :] = x[3, 0]               # every value tied
        if v > 1:
            x[4, v // 2:] = -INF
        got = run(client, x, "bf16", temperature=0.0)
        np.testing.assert_array_equal(got, torch.argmax(torch.tensor(x), 1).numpy())


# ---------------------------------------------------------------------------------------------- invariants
@pytest.mark.parametrize("v", [1000, 50257, 128256])
def test_planted_row_is_batch_invariant(client, v):
    rng = np.random.default_rng(v + 15)
    row = rnd(rng.standard_normal(v).astype(np.float32) * 3, "bf16")
    conf = dict(temperature=0.9, top_k=64, top_p=0.92, min_p=0.01, seed=1234, offset=77)
    ref = None
    for b, pos in ((1, 0), (4096, 0), (4096, 4095)):
        x = rnd(rng.standard_normal((b, v)).astype(np.float32) * 3, "bf16")
        x[pos] = row
        got = run(client, x, "bf16", **conf)[pos]
        ref = got if ref is None else ref
        assert got == ref, (b, pos)
    assert ref == so.sample_row(row, 0.9, 64, 0.92, 0.01, 1234, 77)[0]


@pytest.mark.parametrize("dtype", ["f32", "bf16"])
@pytest.mark.parametrize("v", [1000, 32000, 128256])
def test_pitched_misaligned_views_match_compact(client, v, dtype):
    rng = np.random.default_rng(v + 16)
    b, pad, lead = 9, 3, 1
    x = rnd(rng.standard_normal((b, v)).astype(np.float32) * 3, dtype)
    conf = dict(temperature=1.0, top_k=100, top_p=0.9, min_p=0.0, seed=np.arange(b, dtype=np.uint64) + 1,
                offset=np.zeros(b, np.uint64))
    compact = run(client, x, dtype, **conf)
    buf = np.zeros(b * (v + pad) + lead, np.float32)
    buf[lead:].reshape(b, v + pad)[:, :v] = x
    H = up(client, buf, dtype)
    esz = 4 if dtype == "f32" else 2
    X = TensorHandle(H.handle.offset(lead * esz), [b, v], [v + pad, 1], dtype)
    ibuf = TensorHandle.from_numpy(client, np.full(b + 2, -7, np.int64), "i64")
    ids = TensorHandle(ibuf.handle.offset(8), [b], [1], "i64")
    smp.sample(client, X, ids, 1.0, 100, 0.9, 0.0, arr(client, conf["seed"], "u64"), arr(client, conf["offset"], "u64"))
    client.sync()
    full = ibuf.to_numpy(client)
    np.testing.assert_array_equal(full[1:-1], compact)
    assert full[0] == -7 and full[-1] == -7
    np.testing.assert_array_equal(run(client, x, dtype, **conf), compact)   # repeat: the same bits


def test_advance_offsets_steps_each_row_once(client):
    rng = np.random.default_rng(17)
    b, v = 40, 50257
    x = rnd(rng.standard_normal((b, v)).astype(np.float32) * 3, "bf16")
    X = up(client, x, "bf16")
    seeds = arr(client, rng.integers(0, 2 ** 63, size=b, dtype=np.int64).astype(np.uint64), "u64")
    o0 = rng.integers(0, 2 ** 40, size=b, dtype=np.int64).astype(np.uint64)
    o0[3] = np.uint64(0xFFFFFFFF)                                           # the carry into the counter's high word
    temps = np.ones(b, np.float32)
    temps[5] = 0.0                                                          # a greedy row advances too
    temps[6] = -1.0                                                         # and an invalid one
    T = arr(client, temps, "f32")
    offs = arr(client, o0, "u64")
    a = smp.sample_alloc(client, X, T, 50, 0.9, 0.0, seeds, offs, advance_offsets=True)
    b_ = smp.sample_alloc(client, X, T, 50, 0.9, 0.0, seeds, offs, advance_offsets=True)
    client.sync()
    np.testing.assert_array_equal(offs.to_numpy(client), o0 + np.uint64(2))
    for k, ids in ((0, a), (1, b_)):
        ref = smp.sample_alloc(client, X, T, 50, 0.9, 0.0, seeds, arr(client, o0 + np.uint64(k), "u64"))
        client.sync()
        np.testing.assert_array_equal(ids.to_numpy(client), ref.to_numpy(client))
    assert a.to_numpy(client)[6] == -1


def test_decode_step_lm_head_sample_logprob(client):
    from cubecl_b200 import matmul
    rng = np.random.default_rng(18)
    B, H, V = 64, 512, 32000
    h = rnd(rng.standard_normal((B, H)).astype(np.float32) * 0.5, "bf16")
    W = rnd(rng.standard_normal((V, H)).astype(np.float32) * 0.05, "bf16")
    Hd, Wd = up(client, h, "bf16"), up(client, W, "bf16")
    logits = TensorHandle.empty_contiguous(client, [B, V], "bf16")
    matmul.launch(client, Hd, TensorHandle(Wd.handle, [H, V], [1, H], "bf16"), logits)
    seeds = arr(client, np.arange(B, dtype=np.uint64) * 1000003, "u64")
    ids = smp.sample_alloc(client, logits, 0.8, 50, 0.9, 0.0, seeds, 0)
    loss, _, _ = xent.forward_alloc(client, logits, ids, "none", want_lse=False)
    client.sync()
    got_ids = ids.to_numpy(client)
    assert np.all((got_ids >= 0) & (got_ids < V))
    # the ids are the oracle's on the logits the GEMM wrote
    lx = synth.from_device_dtype(logits.to_numpy(client), "bf16").reshape(B, V)
    ref, margin, bound = so.sample(lx, 0.8, 50, 0.9, 0.0, np.arange(B, dtype=np.uint64) * 1000003, 0)
    safe = margin > bound
    np.testing.assert_array_equal(got_ids[safe], ref[safe])
    lp = torch.log_softmax(torch.tensor(lx, dtype=torch.float64), 1).gather(1, torch.tensor(got_ids)[:, None])[:, 0].numpy()
    got_lp = -loss.to_numpy(client).astype(np.float64)
    assert np.max(np.abs(got_lp - lp)) <= (V * 2.0 + 64) * 2.0 ** -24 * (np.abs(lx).max() + np.abs(lp).max() + 1)
