"""f64 3-D convolution in numpy: forward, input gradient and weight gradient with their sum|a||b| scales (NDHWC
activations, [Cout, KD, KH, KW, C] weights).  The ground truth of the conv3d tests."""
from __future__ import annotations

import itertools
import re

import numpy as np


def triple(v):
    return (int(v),) * 3 if isinstance(v, int) else tuple(int(e) for e in v)


def out_dhw(dhw, k, stride=1, padding=0, dilation=1):
    """PyTorch's output rule per dimension: floor((I + 2p - d(K-1) - 1) / s) + 1"""
    s, p, d = triple(stride), triple(padding), triple(dilation)
    return tuple((dhw[i] + 2 * p[i] - d[i] * (k[i] - 1) - 1) // s[i] + 1 for i in range(3))


def _window(size, osize, k, s, p, d):
    """(output slice, input slice) of the outputs whose input index o*s - p + k*d lies inside [0, size), or None"""
    lo = max(0, -((k * d - p) // s))
    hi = min(osize, (size - 1 + p - k * d) // s + 1)
    if hi <= lo:
        return None
    start = lo * s - p + k * d
    return slice(lo, hi), slice(start, start + (hi - lo - 1) * s + 1, s)


def _taps(in_dhw, o_dhw, k_dhw, stride, padding, dilation):
    """every kernel position (kz, ky, kx) with its (output slices, input slices), positions that read nothing skipped"""
    s, p, d = triple(stride), triple(padding), triple(dilation)
    for kk in itertools.product(*(range(k) for k in k_dhw)):
        w = [_window(in_dhw[i], o_dhw[i], kk[i], s[i], p[i], d[i]) for i in range(3)]
        if any(v is None for v in w):
            continue
        yield kk, tuple(v[0] for v in w), tuple(v[1] for v in w)


def conv3d_f64(x, w, stride=1, padding=0, dilation=1):
    """(out, abs_out): out[n, od, oh, ow, co] = sum x[n, od*sd - pd + kz*dd, ..., c] * w[co, kz, ky, kx, c]; abs_out the same
    sum of |x||w| (the scale of the error bounds)."""
    x, w = np.asarray(x, np.float64), np.asarray(w, np.float64)
    n, c = x.shape[0], x.shape[4]
    cout = w.shape[0]
    o = out_dhw(x.shape[1:4], w.shape[1:4], stride, padding, dilation)
    out, aout = np.zeros((n, *o, cout)), np.zeros((n, *o, cout))
    for kk, os_, is_ in _taps(x.shape[1:4], o, w.shape[1:4], stride, padding, dilation):
        xi = x[(slice(None), *is_, slice(None))]
        wk = w[(slice(None), *kk, slice(None))]
        out[(slice(None), *os_, slice(None))] += xi @ wk.T
        aout[(slice(None), *os_, slice(None))] += np.abs(xi) @ np.abs(wk).T
    return out, aout


def conv3d_input_grad_f64(dy, w, input_dhw, stride=1, padding=0, dilation=1):
    """(dx, abs_dx) for dy [N, OD, OH, OW, Cout] and w [Cout, KD, KH, KW, C]."""
    dy, w = np.asarray(dy, np.float64), np.asarray(w, np.float64)
    n, c = dy.shape[0], w.shape[4]
    assert tuple(dy.shape[1:4]) == out_dhw(input_dhw, w.shape[1:4], stride, padding, dilation)
    dx, adx = np.zeros((n, *input_dhw, c)), np.zeros((n, *input_dhw, c))
    for kk, os_, is_ in _taps(input_dhw, dy.shape[1:4], w.shape[1:4], stride, padding, dilation):
        g = dy[(slice(None), *os_, slice(None))]
        wk = w[(slice(None), *kk, slice(None))]
        dx[(slice(None), *is_, slice(None))] += g @ wk
        adx[(slice(None), *is_, slice(None))] += np.abs(g) @ np.abs(wk)
    return dx, adx


def conv3d_weight_grad_f64(x, dy, kernel_dhw, stride=1, padding=0, dilation=1):
    """(dw, abs_dw) for x [N, D, H, W, C] and dy [N, OD, OH, OW, Cout]."""
    x, dy = np.asarray(x, np.float64), np.asarray(dy, np.float64)
    c, cout = x.shape[4], dy.shape[4]
    assert tuple(dy.shape[1:4]) == out_dhw(x.shape[1:4], kernel_dhw, stride, padding, dilation)
    dw, adw = np.zeros((cout, *kernel_dhw, c)), np.zeros((cout, *kernel_dhw, c))
    for kk, os_, is_ in _taps(x.shape[1:4], dy.shape[1:4], kernel_dhw, stride, padding, dilation):
        g = dy[(slice(None), *os_, slice(None))].reshape(-1, cout)
        xi = x[(slice(None), *is_, slice(None))].reshape(-1, c)
        dw[(slice(None), *kk, slice(None))] = g.T @ xi
        adw[(slice(None), *kk, slice(None))] = np.abs(g).T @ np.abs(xi)
    return dw, adw


_PHASE = re.compile(r"conv3d dgrad phase r=\((\d+),(\d+),(\d+)\) taps_d=([\d,]*) taps_h=([\d,]*) taps_w=([\d,]*) "
                    r"dil=\((\d+),(\d+),(\d+)\) lower=\((-?\d+),(-?\d+),(-?\d+)\) upper=\((-?\d+),(-?\d+),(-?\d+)\) "
                    r"extent=\((\d+),(\d+),(\d+)\)")


def rebuild_dx_from_plan(plan_text, dy, w, input_dhw, stride):
    """dx rebuilt from the `conv3d dgrad phase` lines of a b200_conv3d_backward_data dry-run plan alone: each names its
    residue, the taps per dimension in walk order, the walk's dilation, its lower corner (the dy offset of the first tap),
    upper corner and extent.  Pixels of phases the plan does not list stay zero.  Returns (dx, listed residues)."""
    dy, w = np.asarray(dy, np.float64), np.asarray(w, np.float64)
    n, o = dy.shape[0], dy.shape[1:4]
    s = triple(stride)
    dx = np.zeros((n, *input_dhw, w.shape[4]))
    phases = []
    for m in _PHASE.finditer(plan_text):
        g = [int(v) if i not in (3, 4, 5) else v for i, v in enumerate(m.groups())]
        r = tuple(g[0:3])
        taps = [[int(v) for v in g[3 + i].split(",") if v] for i in range(3)]
        dil, lo, up, ext = g[6:9], g[9:12], g[12:15], g[15:18]
        assert all(up[i] == lo[i] + ext[i] - o[i] for i in range(3))   # the walk covers exactly the phase extent
        phases.append(r)
        ph = np.zeros((n, *ext, w.shape[4]))
        for t in itertools.product(*(range(len(v)) for v in taps)):
            kk = tuple(taps[i][t[i]] for i in range(3))
            # phase pixel e reads dy at e + lo + t * dil in each dimension
            sl_o, sl_i = [], []
            for i in range(3):
                off = lo[i] + t[i] * dil[i]
                a, b = max(0, -off), min(ext[i], o[i] - off)
                if b <= a:
                    break
                sl_o.append(slice(a, b))
                sl_i.append(slice(a + off, b + off))
            else:
                ph[(slice(None), *sl_o, slice(None))] += dy[(slice(None), *sl_i, slice(None))] @ w[(slice(None), *kk, slice(None))]
        dx[:, r[0]::s[0], r[1]::s[1], r[2]::s[2], :][:, :ext[0], :ext[1], :ext[2], :] = ph
    return dx, phases
