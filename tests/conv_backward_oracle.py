"""f64 gradients of the 2-D convolution in numpy: the ground truth of the conv backward tests (NHWC activations,
[Cout, KH, KW, C] weights, the forward of tests/conv_oracle.py)."""
from __future__ import annotations

import numpy as np

from conv_oracle import out_hw, pair


def _windows(h, oh, k, s, p, d):
    """per kernel tap: (output slice, input slice) of the outputs whose input index oh*s - p + k*d lies inside [0, h)"""
    lo = max(0, -((k * d - p) // s))                  # ceil((p - k*d) / s)
    hi = min(oh, (h - 1 + p - k * d) // s + 1)
    if hi <= lo:
        return None
    start = lo * s - p + k * d
    return slice(lo, hi), slice(start, start + (hi - lo - 1) * s + 1, s)


def conv2d_input_grad_f64(dy, w, input_hw, stride=1, padding=0, dilation=1):
    """(dx, abs_dx): dx[n, h, w, c] = sum over the (oh, ow, ky, kx) whose window reads input pixel (h, w) of
    dy[n, oh, ow, co] * w[co, ky, kx, c]; abs_dx is the same sum of |dy||w|."""
    dy = np.asarray(dy, dtype=np.float64)
    w = np.asarray(w, dtype=np.float64)
    n, oh, ow, cout = dy.shape
    cout2, kh, kw, c = w.shape
    assert cout == cout2
    (sh, sw), (ph, pw), (dh, dw) = pair(stride), pair(padding), pair(dilation)
    h, wd = input_hw
    assert (oh, ow) == out_hw(h, wd, kh, kw, stride, padding, dilation)
    dx = np.zeros((n, h, wd, c))
    adx = np.zeros((n, h, wd, c))
    for ky in range(kh):
        wy = _windows(h, oh, ky, sh, ph, dh)
        if wy is None:
            continue
        for kx in range(kw):
            wx = _windows(wd, ow, kx, sw, pw, dw)
            if wx is None:
                continue
            g = dy[:, wy[0], wx[0], :]
            dx[:, wy[1], wx[1], :] += g @ w[:, ky, kx, :]
            adx[:, wy[1], wx[1], :] += np.abs(g) @ np.abs(w[:, ky, kx, :])
    return dx, adx


def conv2d_weight_grad_f64(x, dy, kernel_hw, stride=1, padding=0, dilation=1):
    """(dw, abs_dw): dw[co, ky, kx, c] = sum_{n, oh, ow} dy[n, oh, ow, co] * x[n, oh*sh - ph + ky*dh, ow*sw - pw + kx*dw, c]
    (input outside x is zero); abs_dw is the same sum of |dy||x|."""
    x = np.asarray(x, dtype=np.float64)
    dy = np.asarray(dy, dtype=np.float64)
    n, h, wd, c = x.shape
    _, oh, ow, cout = dy.shape
    kh, kw = kernel_hw
    (sh, sw), (ph, pw), (dh, dw_) = pair(stride), pair(padding), pair(dilation)
    assert (oh, ow) == out_hw(h, wd, kh, kw, stride, padding, dilation)
    dw = np.zeros((cout, kh, kw, c))
    adw = np.zeros((cout, kh, kw, c))
    for ky in range(kh):
        wy = _windows(h, oh, ky, sh, ph, dh)
        if wy is None:
            continue
        for kx in range(kw):
            wx = _windows(wd, ow, kx, sw, pw, dw_)
            if wx is None:
                continue
            g = dy[:, wy[0], wx[0], :].reshape(-1, cout)
            xi = x[:, wy[1], wx[1], :].reshape(-1, c)
            dw[:, ky, kx, :] = g.T @ xi
            adw[:, ky, kx, :] = np.abs(g).T @ np.abs(xi)
    return dw, adw


def rebuild_dx_from_plan(plan_text, dy, w, input_hw, stride):
    """dx rebuilt from the dry-run plan of b200_conv2d_backward_data: every `conv dgrad phase` line names its residue (rh, rw),
    the kernel taps in the order the phase's stride-1 convolution walks them, the dilation of that walk, its lower pixel-box
    corner (the dy offset of the first tap) and its extent.  Pixels of phases the plan does not list stay zero."""
    import re

    dy = np.asarray(dy, dtype=np.float64)
    w = np.asarray(w, dtype=np.float64)
    n, oh, ow, _ = dy.shape
    h, wd = input_hw
    sh, sw = pair(stride)
    dx = np.zeros((n, h, wd, w.shape[3]))
    pat = re.compile(r"conv dgrad phase r=\((\d+),(\d+)\) taps_h=([\d,]*) taps_w=([\d,]*) dil=\((\d+),(\d+)\) "
                     r"lower=\((-?\d+),(-?\d+)\) upper=\((-?\d+),(-?\d+)\) extent=\((\d+),(\d+)\)")
    phases = []
    for m in pat.finditer(plan_text):
        rh, rw = int(m.group(1)), int(m.group(2))
        th = [int(v) for v in m.group(3).split(",") if v]
        tw = [int(v) for v in m.group(4).split(",") if v]
        dlh, dlw, eh0, ew0 = int(m.group(5)), int(m.group(6)), int(m.group(7)), int(m.group(8))
        uh, uw, exh, exw = int(m.group(9)), int(m.group(10)), int(m.group(11)), int(m.group(12))
        assert (uh, uw) == (eh0 + exh - oh, ew0 + exw - ow)   # the walk covers exactly the phase extent
        phases.append((rh, rw))
        ph = np.zeros((n, exh, exw, w.shape[3]))
        for t, ky in enumerate(th):
            for u, kx in enumerate(tw):
                for i in range(exh):
                    yi = i + eh0 + t * dlh
                    if not 0 <= yi < oh:
                        continue
                    for j in range(exw):
                        xj = j + ew0 + u * dlw
                        if 0 <= xj < ow:
                            ph[:, i, j, :] += dy[:, yi, xj, :] @ w[:, ky, kx, :]
        dx[:, rh::sh, rw::sw, :][:, :exh, :exw, :] = ph
    return dx, phases
