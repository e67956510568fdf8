"""f64 direct 2-D convolution in numpy: the ground truth of the conv tests (NHWC input, [Cout, KH, KW, C] weights)."""
from __future__ import annotations

import json
from pathlib import Path

import numpy as np

GOLDEN = Path(__file__).resolve().parent / "golden" / "conv_golden.json"


def pair(v):
    return (int(v), int(v)) if isinstance(v, int) else tuple(int(e) for e in v)


def out_hw(h, w, kh, kw, stride=1, padding=0, dilation=1):
    (sh, sw), (ph, pw), (dh, dw) = pair(stride), pair(padding), pair(dilation)
    return (h + 2 * ph - dh * (kh - 1) - 1) // sh + 1, (w + 2 * pw - dw * (kw - 1) - 1) // sw + 1


def conv2d_f64(x, w, stride=1, padding=0, dilation=1):
    """(out, abs_out): out[n, oh, ow, co] = sum_{ky, kx, c} x[n, oh*sh - ph + ky*dh, ow*sw - pw + kx*dw, c] * w[co, ky, kx, c]
    in f64 (input outside x is zero); abs_out is the same sum of |x||w|, the scale of the error bounds."""
    x = np.asarray(x, dtype=np.float64)
    w = np.asarray(w, dtype=np.float64)
    n, h, wd, c = x.shape
    cout, kh, kw, c2 = w.shape
    assert c == c2
    (sh, sw), (ph, pw), (dh, dw) = pair(stride), pair(padding), pair(dilation)
    oh, ow = out_hw(h, wd, kh, kw, stride, padding, dilation)
    xp = np.zeros((n, h + 2 * ph, wd + 2 * pw, c))
    xp[:, ph:ph + h, pw:pw + wd, :] = x
    out = np.zeros((n, oh, ow, cout))
    aout = np.zeros((n, oh, ow, cout))
    for ky in range(kh):
        for kx in range(kw):
            win = xp[:, ky * dh: ky * dh + sh * (oh - 1) + 1: sh, kx * dw: kx * dw + sw * (ow - 1) + 1: sw, :]
            out += win @ w[:, ky, kx, :].T
            aout += np.abs(win) @ np.abs(w[:, ky, kx, :]).T
    return out, aout


def im2col_kat():
    """The reference's im2col known-answer test as a convolution: x = 1..72 as [1, 3, 3, 8], a 2 x 2 kernel, pad 1, and one-hot
    weights [32, 2, 2, 8] so output channel (ky * 2 + kx) * 8 + c is the im2col column of kernel position (ky, kx), channel c.
    Returns (x, w, expected [1, 4, 4, 32], kat dict)."""
    kat = json.loads(GOLDEN.read_text())["im2col_kat"]
    n, h, wd, c, kh, kw = kat["n"], kat["h"], kat["w"], kat["c"], kat["kernel_h"], kat["kernel_w"]
    x = np.arange(1, n * h * wd * c + 1, dtype=np.float64).reshape(n, h, wd, c)
    cout = kh * kw * c
    w = np.zeros((cout, kh, kw, c))
    for ky in range(kh):
        for kx in range(kw):
            for ci in range(c):
                w[(ky * kw + kx) * c + ci, ky, kx, ci] = 1.0
    oh, ow = kat["out_h"], kat["out_w"]
    exp = np.zeros((n, oh, ow, cout))
    for kpos, row in enumerate(kat["expected_pixels"]):
        for m, pix in enumerate(row):
            if pix:
                b, r = divmod(m, oh * ow)
                exp[b, r // ow, r % ow, kpos * c: (kpos + 1) * c] = (pix - 1) * c + 1 + np.arange(c)
    return x, w, exp, kat
