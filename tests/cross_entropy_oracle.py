"""A numpy restatement of b200_cross_entropy / b200_cross_entropy_backward (include/cubecl_b200.h) in f32, in the header's
order of operations.

ex2 and lg2 stand for PTX's ex2.approx.ftz and lg2.approx: here they are exp2 / log2 rounded once to f32, with results below
2^-126 flushed to +0.  They agree with the hardware on integer arguments of ex2 and power-of-two arguments of lg2, which is
what the exact rows are built to use (an assumption about the hardware that PTX does not promise; attention's exact tests
make the same one).  The sum S() of a row is taken here in numpy's order, not the kernel's: the exact rows are built so that
every such sum is exact in any order (ex2 terms that are 1 or +0, logits that are multiples of 8 with every partial sum below
2^27).  The SUM / MEAN total, whose terms are arbitrary f32 values, follows the kernel's order exactly.

Mutants (the `_mutant` argument) are wrong contracts the exact GPU cases must be able to tell apart:
  eps_over_v_minus_1  smoothing mass eps / (V - 1) in place of eps / V
  mean_over_all_rows  MEAN divides by t instead of the counted rows
  ignored_rows_grad   ignored rows get the gradient of a row with target 0 instead of +0
  z_grad_without_2    the z-loss gradient factor 1 + z * lse instead of 1 + 2 z * lse
  lse_without_shift   lse = log(sum exp(x)) without subtracting the max first (overflows where the max is large)
  g_not_divided       MEAN's gradient scale dloss instead of dloss / count
"""
import numpy as np
import torch

F32 = np.float32
LOG2E = F32(1.4426950408889634)
LN2 = F32(0.6931471805599453)
TOTAL_THREADS = 1024
REDUCTIONS = ("none", "sum", "mean")


def rnd(a, dtype):
    """a rounded to nearest-even in dtype and read back as f32"""
    a = np.asarray(a, F32)
    if dtype == "f32":
        return a.copy()
    tdt = {"bf16": torch.bfloat16, "f16": torch.float16}[dtype]
    return torch.from_numpy(np.ascontiguousarray(a)).to(tdt).to(torch.float32).numpy()


def ex2(a):
    r = np.exp2(np.asarray(a, np.float64)).astype(F32)
    return np.where(np.abs(r) < F32(2.0 ** -126), F32(0), r).astype(F32)


def lg2(a):
    with np.errstate(divide="ignore"):
        return np.log2(np.asarray(a, np.float64)).astype(F32)


def scalars(eps, z, V, _mutant=None):
    """(omega, eps_v, z2): rn(1 - eps), rn(eps / V), rn(2 z), as the library forms them in f32"""
    omega = F32(F32(1) - F32(eps))
    eps_v = F32(F32(eps) / F32(V - 1 if _mutant == "eps_over_v_minus_1" else V))
    z2 = F32(z) if _mutant == "z_grad_without_2" else F32(F32(2) * F32(z))
    return omega, eps_v, z2


def row_stats(x, _mutant=None):
    """(m, s, sx, lse) of f32 rows x [T, V]"""
    x = np.asarray(x, F32)
    with np.errstate(invalid="ignore", over="ignore"):
        m = x.max(1)
        if _mutant == "lse_without_shift":
            m = np.zeros_like(m)
        sh = np.where(m == -np.inf, F32(0), m).astype(F32)
        s = ex2((x - sh[:, None]).astype(F32) * LOG2E).sum(1, dtype=F32)
        sx = x.sum(1, dtype=F32)
        lse = (m + (lg2(s) * LN2).astype(F32)).astype(F32)
    return m, s, sx, lse


def counted(y, V, ignore_index):
    y = np.asarray(y, np.int64)
    c = y != ignore_index
    bad = c & ((y < 0) | (y >= V))
    return c, bad


def total(rows, reduction, count):
    """the SUM / MEAN value of the row losses, in the kernel's order: thread i of 1024 adds rows i, i + 1024, ... from +0;
    an xor butterfly over each warp (16, 8, 4, 2, 1); the warps in order; MEAN divides once by f32(count)"""
    rows = np.asarray(rows, F32)
    acc = np.zeros(TOTAL_THREADS, F32)
    for start in range(0, len(rows), TOTAL_THREADS):
        chunk = rows[start:start + TOTAL_THREADS]
        acc[:len(chunk)] = (acc[:len(chunk)] + chunk).astype(F32)
    lanes = acc.reshape(-1, 32)
    for o in (16, 8, 4, 2, 1):
        lanes = (lanes + lanes[:, np.arange(32) ^ o]).astype(F32)
    a = lanes[0, 0]
    for w in range(1, lanes.shape[0]):
        a = F32(a + lanes[w, 0])
    if reduction == "mean":
        with np.errstate(invalid="ignore", divide="ignore"):
            a = F32(a / F32(count))
    return a


def forward(x, y, reduction="mean", ignore_index=-100, eps=0.0, z=0.0, _mutant=None):
    """(loss, lse, row losses, count): loss f32 [T] for none, a 0-d f32 otherwise"""
    x = np.asarray(x, F32)
    T, V = x.shape
    omega, eps_v, _ = scalars(eps, z, V, _mutant)
    _, _, sx, lse = row_stats(x, _mutant)
    c, bad = counted(y, V, ignore_index)
    yy = np.where(c & ~bad, np.asarray(y, np.int64), 0)
    xy = x[np.arange(T), yy]
    with np.errstate(invalid="ignore", over="ignore"):
        loss = (lse - (omega * xy).astype(F32)).astype(F32)
        if eps_v != 0:
            loss = (loss - (eps_v * sx).astype(F32)).astype(F32)
        if F32(z) != 0:
            loss = (loss + (F32(z) * (lse * lse).astype(F32)).astype(F32)).astype(F32)
    loss = np.where(bad, F32(np.nan), np.where(c, loss, F32(0))).astype(F32)
    count = T if _mutant == "mean_over_all_rows" else int(c.sum())
    out = loss if reduction == "none" else total(loss, reduction, count)
    return out, lse, loss, count


def backward(x, y, lse, dloss, reduction="mean", ignore_index=-100, eps=0.0, z=0.0, grad_dtype="f32", _mutant=None):
    """dlogits [T, V] as f32 values of grad_dtype"""
    x = np.asarray(x, F32)
    T, V = x.shape
    omega, eps_v, z2 = scalars(eps, z, V, _mutant)
    c, bad = counted(y, V, ignore_index)
    dloss = np.asarray(dloss, F32).reshape(-1)
    if reduction == "none":
        g = dloss.copy()
    else:
        g = np.full(T, dloss[0], F32)
        if reduction == "mean" and _mutant != "g_not_divided":
            count = T if _mutant == "mean_over_all_rows" else int(c.sum())
            with np.errstate(invalid="ignore", divide="ignore"):
                g[:] = F32(dloss[0] / F32(count))
    lse = np.asarray(lse, F32)
    with np.errstate(invalid="ignore", over="ignore"):
        d = ex2(((x - lse[:, None]).astype(F32) * LOG2E).astype(F32))
        if F32(z) != 0:
            zf = (F32(1) + (z2 * lse).astype(F32)).astype(F32)
            d = (d * zf[:, None]).astype(F32)
        ok = c & ~bad
        rows = np.nonzero(ok)[0]
        yy = np.asarray(y, np.int64)[rows]
        d[rows, yy] = (d[rows, yy] - omega).astype(F32)
        if _mutant == "ignored_rows_grad":
            ign = np.nonzero(~c)[0]
            d[ign, 0] = (d[ign, 0] - omega).astype(F32)
        if eps_v != 0:
            d = (d - eps_v).astype(F32)
        dx = (g[:, None] * d).astype(F32)
    keep = ok | (~c if _mutant == "ignored_rows_grad" else np.zeros_like(c))
    dx = np.where(bad[:, None], F32(np.nan), np.where(keep[:, None], dx, F32(0))).astype(F32)
    return rnd(dx, grad_dtype)


# ---------------------------------------------------------------------------------------------- exact rows
def exact_k_ok(m, k):
    """whether a row with max m (a multiple of 8) and 2^k tied maxima keeps rn(rn(m - lse) * log2e) an integer >= -126"""
    lse = F32(F32(m) + F32(F32(k) * LN2))
    a = F32(F32(F32(m) - lse) * LOG2E)
    return bool(a == np.round(a) and a >= -126)


def exact_rows(rng, T, V, dtype, ms=(0, 8, -16, 96, 200, 304)):
    """(x, k): rows with 2^k tied maxima m (a multiple of 8, chosen so that exact_k_ok holds) and every other logit a multiple
    of 8 at least 152 below m, exactly representable in dtype.  The sum of exponentials is then 2^k, lse = rn(m + rn(k ln2)),
    p is 2^(integer) or +0, and every partial sum of the logits is a multiple of 8 below 2^27 in magnitude."""
    x = np.empty((T, V), F32)
    ks = np.empty(T, np.int64)
    kmax = int(np.log2(V))
    for r in range(T):
        for _ in range(100):
            m, k = int(rng.choice(ms)), int(rng.integers(0, min(kmax, 10) + 1))
            if exact_k_ok(m, k):
                break
        else:
            raise AssertionError("no exact (m, k)")
        row = (m - 8 * rng.integers(19, 26, size=V)).astype(F32)
        row[rng.choice(V, size=1 << k, replace=False)] = m
        x[r] = row
        ks[r] = k
    assert np.array_equal(rnd(x, dtype), x)
    assert np.abs(x).sum(1).max() < 2 ** 27
    return x, ks


def exact_targets(rng, x, ignore_index=-100, ignore_every=5):
    """targets on a maximum or a low logit at random, every ignore_every-th row ignored"""
    T, V = x.shape
    y = rng.integers(0, V, size=T)
    for r in range(0, T, 2):
        y[r] = int(rng.choice(np.nonzero(x[r] == x[r].max())[0]))
    y[::ignore_every] = ignore_index
    return y


def reference_f64(x, y, reduction="mean", ignore_index=-100, eps=0.0, z=0.0):
    """(loss, lse, dlogits for dloss = 1) in f64 through torch autograd, and per-row bounds of the f32 contract's error"""
    xt = torch.tensor(np.asarray(x, np.float64), requires_grad=True)
    yt = torch.tensor(np.asarray(y, np.int64))
    lse = torch.logsumexp(xt, 1)
    rows = torch.nn.functional.cross_entropy(xt, yt, reduction="none", ignore_index=ignore_index, label_smoothing=eps)
    keep = (yt != ignore_index).to(torch.float64)
    rows = rows + z * lse * lse * keep
    loss = rows if reduction == "none" else rows.sum() if reduction == "sum" else rows.sum() / keep.sum()
    loss.backward(torch.ones_like(loss))
    V = x.shape[1]
    # ex2 / lg2 approximations (about 2 ulp each), the row sum's rounding (V ulp of s), the loss's few roundings of |lse|,
    # |x_y| and eps * mean|x|
    xa = np.abs(np.asarray(x, np.float64))
    scale = np.abs(lse.detach().numpy()) + xa.max(1) + eps * xa.mean(1) + 1
    bound = (V * 2.0 + 64) * 2.0 ** -24 * scale * (1 + 2 * z * np.abs(lse.detach().numpy()))
    return loss.detach().numpy(), lse.detach().numpy(), xt.grad.numpy(), bound
