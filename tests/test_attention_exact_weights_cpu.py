"""CPU: the exact power-of-two-weight attention model (tests/attention_exact_oracle.py) and the case lists of
tests/test_attention_exact_weights_gpu.py.  Each generator meets the model's preconditions, the model agrees with the f64
oracles, the kernels' own key order (128-key blocks, KV-cache splits) gives the same bits as the closed form, the cases really
meet rescale and merge factors 2^-1 .. 2^-8, and every case's expected bits change under each wrong kernel the exact tests
exist to catch."""
import numpy as np
import pytest

import attention_backward_oracle as abo
import attention_exact_oracle as xo
import attention_kvcache_oracle as ko
import attention_oracle as ao
import attention_varlen_oracle as vo
import gemm_exact_oracle as ge
import test_attention_exact_weights_gpu as gpu


def _values(bits, dtype):
    return ge.bits_to_f64(bits, dtype)


def _scores(q, k):
    return xo.scores(q, np.repeat(k, q.shape[1] // k.shape[1], axis=1))


def _differs(a, b, dtype):
    return ge.bit_mismatches(a, b, dtype).any()


def test_scale_ln2_makes_scale_log2_one():
    assert xo.scale_log2() == np.float32(1.0)


def test_model_refuses_scores_between_the_bands_and_non_power_of_two_backward_rows():
    q = np.zeros((1, 1, 1, 4))
    k = np.zeros((1, 1, 3, 4))
    k[0, 0, :, 0] = [0, -9, -200]
    q[0, 0, 0, 0] = 1
    v = np.ones((1, 1, 3, 4))
    with pytest.raises(AssertionError, match="between NEAR and FAR"):
        xo.forward(q, k, v, np.ones((1, 3), bool), "f32")
    k[0, 0, :, 0] = [0, -1, -200]
    with pytest.raises(AssertionError, match="l = 2\\^n"):
        xo.backward(q, k, v, np.ones((1, 1, 1, 4)), np.ones((1, 3), bool), "bf16", "bf16", "bf16")


# ---------------------------------------------------------------------------------------------- dense forward
@pytest.mark.parametrize("case", gpu.FORWARD_CASES, ids=gpu.FORWARD_IDS)
def test_dense_forward_model_cases(case):
    B, Hq, Hkv, Sq, Sk, D, causal = case
    q, k, v = gpu.dense_problem(*case, seed=Sq + Sk + D)
    vis = gpu.dense_vis(Sq, Sk, causal)
    for t in (q, k, v):   # exact in both 16-bit input dtypes
        for dt in ("bf16", "f16"):
            assert xo.rounds_exactly(t, dt)
    want32, w, l = xo.forward(q, k, v, vis, "f32")
    ref, _ = ao.attention_f64(q, k, v, xo.LN2, causal)
    np.testing.assert_allclose(_values(want32, "f32"), ref, rtol=2.0 ** -22, atol=2.0 ** -20)
    assert np.mean((l != np.exp2(np.round(np.log2(l))))) > 0.5   # most rows divide by an l that is not a power of two
    s = _scores(q, k)
    vv = np.repeat(v, Hq // Hkv, axis=1)
    for od in ("f32", "bf16", "f16"):
        want = xo.forward(q, k, v, vis, od)[0]
        assert np.array_equal(xo.online_forward(s, vv, vis, 128, od), want)
        assert _differs(xo.online_forward(s, vv, vis, 128, od, rescale=False), want, od), "a skipped rescale would pass"
    assert xo.rescale_exponents(s, vis, 128) >= set(range(1, 7))
    # the weighted keys reach the first block, a middle block, the tail past Sk % 128 and, when causal, the diagonal block
    wk = (w > 0).any(axis=(0, 1, 2))
    tail = 128 * (Sk // 128)
    assert wk[:128].any() and wk[128:tail].any() and (Sk % 128 == 0 or wk[tail:].any())
    if causal:
        diag = [(w[..., i, 128 * (i // 128):i + 1] > 0).any() for i in range(Sq)]
        assert np.mean(diag) > 0.9
        for shift in (-1, 1):   # the causal alignment moved by one key either way
            bad = np.arange(Sk)[None, :] <= np.arange(Sq)[:, None] + shift
            assert _differs(xo.online_forward(s, vv, bad, 128, "bf16"), xo.forward(q, k, v, vis, "bf16")[0], "bf16"), shift


def test_forward_cases_cover_every_head_dim_gqa_and_both_masks():
    seen = set()
    for case in gpu.FORWARD_CASES:   # each case meets 2^-1 .. 2^-6, and the list together every rescale factor 2^-1 .. 2^-8
        q, k, _ = gpu.dense_problem(*case, seed=case[3] + case[4] + case[5])
        seen |= xo.rescale_exponents(_scores(q, k), gpu.dense_vis(case[3], case[4], case[6]), 128)
    assert seen == set(range(1, xo.NEAR + 1))
    assert {c[5] for c in gpu.FORWARD_CASES} == {40, 64, 96, 128}
    assert any(c[1] > c[2] for c in gpu.FORWARD_CASES if c[6]) and any(c[1] > c[2] for c in gpu.FORWARD_CASES if not c[6])
    assert all(c[4] % 128 for c in gpu.FORWARD_CASES)


# ---------------------------------------------------------------------------------------------- dense backward
@pytest.mark.parametrize("case", gpu.BACKWARD_CASES, ids=gpu.BACKWARD_IDS)
def test_dense_backward_model_cases(case):
    B, Hq, Hkv, Sq, Sk, D, causal = case
    q, k, v, dout = gpu.dense_problem(*case, seed=Sq + Sk + D, backward=True)
    vis = gpu.dense_vis(Sq, Sk, causal)
    assert Sq % 64 and Sk % 64 or Sq % 64 == Sk % 64 != 0
    for dt in ("bf16", "f16"):
        want = xo.backward(q, k, v, dout, vis, dt, "f32", "f32")
        ref = abo.attention_backward_f64(q, k, v, dout, xo.LN2, causal)
        for name, got, r in zip(("dq", "dk", "dv"), want, ref):
            np.testing.assert_allclose(_values(got, "f32"), r, rtol=2.0 ** -20, atol=2.0 ** -30, err_msg=name)
        assert all((_values(x, "f32") != 0).mean() > 0.02 for x in want)   # dS is not zero: dq and dk are not
        for od, gd in ((dt, dt), ("f32", "f32"), (dt, "f32")):
            good = xo.backward(q, k, v, dout, vis, dt, od, gd)
            for mutant in xo.BACKWARD_MUTANTS:
                if mutant == "dk_missing_a_group_head" and Hq == Hkv:
                    continue
                bad = xo.backward(q, k, v, dout, vis, dt, od, gd, mutant=mutant)
                assert any(_differs(b, g, gd) for b, g in zip(bad, good)), (mutant, od, gd)
    assert any(c[1] > c[2] for c in gpu.BACKWARD_CASES if c[6]) and any(c[1] > c[2] for c in gpu.BACKWARD_CASES if not c[6])


# ---------------------------------------------------------------------------------------------- KV cache splits
@pytest.mark.parametrize("case", gpu.KV_CASES)
def test_kvcache_model_cases_merge_several_splits(case):
    B, Hq, Hkv, Sq, D, page, mp, causal, dtype = case
    cap = page * mp
    lens = gpu.kv_lens(B, cap)
    q, k, v, vis = gpu.kv_problem(B, Hq, Hkv, Sq, D, cap, lens, causal, seed=cap + Sq)
    splits = gpu.kv_splits(B, Hq, Hkv, Sq, cap)
    assert len(splits) > 1
    want32, _, _ = xo.forward(q, k, v, vis, "f32")
    cache = lambda t: t.transpose(0, 2, 1, 3)   # noqa: E731  identity layout [B, cap, Hkv, D]: page b of `cap` keys
    ref, _ = ko.attention_kvcache_f64(q, cache(k), cache(v), lens, None, xo.LN2, causal)
    np.testing.assert_allclose(_values(want32, "f32"), ref, rtol=2.0 ** -22, atol=2.0 ** -20)
    s = _scores(q, k)
    vv = np.repeat(v, Hq // Hkv, axis=1)
    for od in ("f32", dtype):
        want = xo.forward(q, k, v, vis, od)[0]
        assert np.array_equal(xo.split_forward(s, vv, vis, splits, od), want)
        assert _differs(xo.split_forward(s, vv, vis, splits, od, merge=False), want, od), "merge weights of 1 would pass"
    assert xo.merge_exponents(s, vis, splits) >= set(range(0, 7))
    if causal:   # bottom-right alignment moved by one key either way (with Sq = 1 the length mask hides a +1 shift)
        for shift in ((-1, 1) if Sq > 1 else (-1,)):
            L = np.asarray(lens)[:, None, None, None]
            bad = (np.arange(cap) < L) & (np.arange(cap) <= L - Sq + np.arange(Sq)[:, None] + shift)
            assert _differs(xo.split_forward(s, vv, bad, splits, dtype), xo.forward(q, k, v, vis, dtype)[0], dtype), shift


def test_kv_cases_cover_both_sq_and_dtypes():
    assert {c[3] for c in gpu.KV_CASES if c[7]} == {1, 3} and {c[8] for c in gpu.KV_CASES} == {"bf16", "f16"}


def _shifted_causal(Sq, Sk, shift):
    return np.arange(Sk)[None, :] <= np.arange(Sq)[:, None] + shift


@pytest.mark.parametrize("case", [c for c in gpu.BACKWARD_CASES if c[6]], ids=[i for c, i in zip(gpu.BACKWARD_CASES, gpu.BACKWARD_IDS) if c[6]])
def test_dense_backward_cases_catch_a_causal_mask_off_by_one_in_either_kernel(case):
    B, Hq, Hkv, Sq, Sk, D, causal = case
    q, k, v, dout = gpu.dense_problem(*case, seed=Sq + Sk + D, backward=True)
    vis = gpu.dense_vis(Sq, Sk, causal)
    good = xo.backward(q, k, v, dout, vis, "bf16", "bf16", "bf16")
    for shift in (-1, 1):
        bad = _shifted_causal(Sq, Sk, shift)
        dq = xo.backward(q, k, v, dout, vis, "bf16", "bf16", "bf16", vis_dq=bad)
        assert _differs(dq[0], good[0], "bf16") and not _differs(dq[1], good[1], "bf16"), shift
        dkdv = xo.backward(q, k, v, dout, vis, "bf16", "bf16", "bf16", vis_dkdv=bad)
        assert _differs(dkdv[1], good[1], "bf16") and _differs(dkdv[2], good[2], "bf16"), shift


# ---------------------------------------------------------------------------------------------- varlen windows
def _edge_moved(window, side, d):
    """(Lq, Lk) -> the band of `window` with its left or right edge moved by d keys (the (-1, 0) causal edge is the right one)"""
    left, right = window

    def mask(Lq, Lk):
        i, j = np.arange(Lq)[:, None], np.arange(Lk)[None, :]
        off = Lk - Lq
        m = np.ones((Lq, Lk), bool)
        if left >= 0:
            m &= j >= i + off - left + (d if side == "left" else 0)
        if right >= 0:
            m &= j <= i + off + right + (d if side == "right" else 0)
        return m
    return mask


def _varlen_forward_with(q, k, v, lens_q, lens_k, mask_fn, od):
    """the forward in the kernels' key order under any mask (no band checks: a let-through decoy breaks them)"""
    out = np.zeros(q.shape, ge.OUT_BITS_VIEW[od])
    g = q.shape[1] // k.shape[1]
    for (sq, sk), Lq, Lk in zip(gpu.varlen_seqs(lens_q, lens_k), lens_q, lens_k):
        if Lq and Lk:
            qq, kk, vv = gpu._bhsd(q[sq]), np.repeat(gpu._bhsd(k[sk]), g, axis=1), np.repeat(gpu._bhsd(v[sk]), g, axis=1)
            out[sq] = xo.online_forward(xo.scores(qq, kk), vv, mask_fn(Lq, Lk), 128, od)[0].transpose(1, 0, 2)
    return out


def test_varlen_cases_cover_every_window_kind_and_sequence_shape():
    kinds = {("causal" if w == (-1, 0) else "left" if w[1] == 0 else "right" if w[0] == 0 else "both") for w in gpu.VARLEN_WINDOWS}
    assert kinds == {"causal", "left", "both", "right"}
    lq, lk = gpu.VARLEN_LENS
    pairs = list(zip(lq, lk))
    assert any(a > b > 0 for a, b in pairs) and any(0 < a < b for a, b in pairs)
    assert (0, 0) in pairs and any(a == 1 for a, _ in pairs) and any(b == 1 for _, b in pairs)


@pytest.mark.parametrize("window", gpu.VARLEN_WINDOWS, ids=gpu.VARLEN_IDS)
def test_varlen_model_cases_and_every_window_edge_off_by_one(window):
    lq, lk = gpu.VARLEN_LENS
    Hq, Hkv, D = gpu.VARLEN_SHAPE["Hq"], gpu.VARLEN_SHAPE["Hkv"], gpu.VARLEN_SHAPE["D"]
    cq, ck = np.cumsum([0] + lq), np.cumsum([0] + lk)
    sides = [s for s, b in (("left", window[0]), ("right", window[1])) if b >= 0]
    # forward: the model against the f64 oracle and the kernels' key order, and each edge moved by one key either way
    q, k, v = gpu.varlen_problem(lq, lk, Hq, Hkv, D, window, seed=sum(window) + 11)
    want32 = gpu.varlen_forward(q, k, v, lq, lk, window, "f32")
    ref, _ = vo.attention_varlen_f64(q, k, v, cq, ck, xo.LN2, window)
    np.testing.assert_allclose(_values(want32, "f32"), ref, rtol=2.0 ** -22, atol=2.0 ** -20)
    for od in ("bf16", "f16", "f32"):
        want = gpu.varlen_forward(q, k, v, lq, lk, window, od)
        assert np.array_equal(_varlen_forward_with(q, k, v, lq, lk, lambda a, b: vo.band_mask(a, b, window), od), want)
        for side in sides:
            for d in (-1, 1):
                bad = _varlen_forward_with(q, k, v, lq, lk, _edge_moved(window, side, d), od)
                assert _differs(bad, want, od), (od, side, d)
    # backward: the model against the f64 oracle, and each edge moved in the dq kernel alone and in the dk / dv kernel alone
    q, k, v, dout = gpu.varlen_problem(lq, lk, Hq, Hkv, D, window, seed=sum(window) + 12, backward=True)
    ref = vo.attention_varlen_backward_f64(q, k, v, dout, cq, ck, xo.LN2, window)
    for dt in ("bf16", "f16"):
        got = gpu.varlen_backward(q, k, v, dout, lq, lk, window, dt, "f32", "f32")
        for name, g, r in zip(("dq", "dk", "dv"), got, ref):
            np.testing.assert_allclose(_values(g, "f32"), r, rtol=2.0 ** -20, atol=2.0 ** -30, err_msg=name)
        assert all((_values(x, "f32") != 0).mean() > 0.02 for x in got)
    good = gpu.varlen_backward(q, k, v, dout, lq, lk, window, "bf16", "bf16", "bf16")
    for side in sides:
        for d in (-1, 1):
            f = _edge_moved(window, side, d)
            dq = gpu.varlen_backward(q, k, v, dout, lq, lk, window, "bf16", "bf16", "bf16", mask_dq=f)
            assert _differs(dq[0], good[0], "bf16"), ("dq", side, d)
            dkdv = gpu.varlen_backward(q, k, v, dout, lq, lk, window, "bf16", "bf16", "bf16", mask_dkdv=f)
            assert _differs(dkdv[1], good[1], "bf16") and _differs(dkdv[2], good[2], "bf16"), ("dkdv", side, d)
