"""Grouped 2-D convolution in numpy: an f64 reference of the forward and both gradients (per-group calls of the dense
oracles, pinned to torch by tests/test_conv_grouped_cpu.py), and a serial-f32 restatement of the direct kernels' summation
orders (csrc/conv_grouped.cu), which the GPU tests compare bit for bit.

Layouts: x NHWC [N, H, W, C], w [Cout, KH, KW, C / groups], out / dy [N, OH, OW, Cout].

Restriction of the f32 restatement: every product of two operands must be exact in f32, so that `float32(a * b)` followed
by one float32 add equals the kernel's fma.  Products of two f16 values are (22 significant bits, exponents well inside
f32's normal range); products of two bf16 values are when they stay in f32's normal range, which data drawn from [-8, 8]
(or integers) does.
"""
from __future__ import annotations

import numpy as np

from conv_backward_oracle import conv2d_input_grad_f64, conv2d_weight_grad_f64
from conv_oracle import conv2d_f64, out_hw, pair

F32 = np.float32


def _split(c, cout, groups):
    assert c % groups == 0 and cout % groups == 0
    return c // groups, cout // groups


# ------------------------------------------------------------------------------------------------ f64 reference
def grouped_f64(x, w, groups, stride=1, padding=0, dilation=1):
    """(out, abs_out) of the grouped convolution, one dense f64 convolution per group."""
    cg, coutg = _split(x.shape[3], w.shape[0], groups)
    assert w.shape[3] == cg
    parts = [conv2d_f64(x[..., g * cg:(g + 1) * cg], w[g * coutg:(g + 1) * coutg], stride, padding, dilation) for g in range(groups)]
    return np.concatenate([p[0] for p in parts], axis=3), np.concatenate([p[1] for p in parts], axis=3)


def grouped_input_grad_f64(dy, w, input_hw, groups, stride=1, padding=0, dilation=1):
    cg, coutg = _split(w.shape[3] * groups, dy.shape[3], groups)
    parts = [conv2d_input_grad_f64(dy[..., g * coutg:(g + 1) * coutg], w[g * coutg:(g + 1) * coutg], input_hw, stride, padding, dilation)
             for g in range(groups)]
    return np.concatenate([p[0] for p in parts], axis=3), np.concatenate([p[1] for p in parts], axis=3)


def grouped_weight_grad_f64(x, dy, kernel_hw, groups, stride=1, padding=0, dilation=1):
    cg, coutg = _split(x.shape[3], dy.shape[3], groups)
    parts = [conv2d_weight_grad_f64(x[..., g * cg:(g + 1) * cg], dy[..., g * coutg:(g + 1) * coutg], kernel_hw, stride, padding, dilation)
             for g in range(groups)]
    return np.concatenate([p[0] for p in parts], axis=0), np.concatenate([p[1] for p in parts], axis=0)


# ------------------------------------------------------------------------------------------------ serial f32 orders
def forward_f32(x, w, groups, stride=1, padding=0, dilation=1, alpha=None, bias=None, relu=False):
    """conv2d_grp_*: acc = +0; for ky, kx, ci ascending: acc = fma(x, w, acc); then out = act(alpha * acc + bias) in f32
    (alpha / bias / relu as the fused epilogue; None = absent)."""
    x, w = np.asarray(x, F32), np.asarray(w, F32)
    n, h, wd, c = x.shape
    cout, kh, kw, cg = w.shape
    _, coutg = _split(c, cout, groups)
    (sh, sw), (ph, pw), (dh, dw) = pair(stride), pair(padding), pair(dilation)
    oh, ow = out_hw(h, wd, kh, kw, stride, padding, dilation)
    xp = np.zeros((n, h + 2 * ph, wd + 2 * pw, c), F32)
    xp[:, ph:ph + h, pw:pw + wd, :] = x
    cbase = (np.arange(cout) // coutg) * cg
    acc = np.zeros((n, oh, ow, cout), F32)
    with np.errstate(invalid="ignore", over="ignore"):
        for ky in range(kh):
            for kx in range(kw):
                win = xp[:, ky * dh: ky * dh + sh * (oh - 1) + 1: sh, kx * dw: kx * dw + sw * (ow - 1) + 1: sw, :]
                for ci in range(cg):
                    acc = (acc + win[..., cbase + ci] * w[:, ky, kx, ci]).astype(F32)
        if alpha is not None:
            acc = (acc * F32(alpha)).astype(F32)
        if bias is not None:
            acc = (acc + np.asarray(bias, F32)).astype(F32)
        if relu:
            acc = np.where(acc > 0, acc, F32(0)).astype(F32)
    return acc


def dgrad_f32(dy, w, input_hw, groups, stride=1, padding=0, dilation=1):
    """conv2d_grp_dgrad_*: acc = +0; for ky, kx ascending over the taps with (h + ph - ky dh) % sh == 0 and likewise for w;
    for co in the group ascending: acc = fma(dy, w, acc), dy reading +0 outside [0, OH) x [0, OW)."""
    dy, w = np.asarray(dy, F32), np.asarray(w, F32)
    n, oh, ow, cout = dy.shape
    _, kh, kw, cg = w.shape
    c = cg * groups
    _, coutg = _split(c, cout, groups)
    (sh, sw), (ph, pw), (dh, dw) = pair(stride), pair(padding), pair(dilation)
    h, wd = input_hw
    chan = np.arange(c)
    grp, ci = chan // cg, chan % cg
    acc = np.zeros((n, h, wd, c), F32)
    with np.errstate(invalid="ignore", over="ignore"):
        for ky in range(kh):
            nh = np.arange(h) + ph - ky * dh
            div_h, oy = nh % sh == 0, nh // sh
            in_h = div_h & (oy >= 0) & (oy < oh)
            for kx in range(kw):
                nw = np.arange(wd) + pw - kx * dw
                div_w, ox = nw % sw == 0, nw // sw
                in_w = div_w & (ox >= 0) & (ox < ow)
                tap = (div_h[:, None] & div_w[None, :])[None, :, :, None]
                inside = (in_h[:, None] & in_w[None, :])[None, :, :, None]
                rows = dy[:, np.clip(oy, 0, oh - 1)][:, :, np.clip(ox, 0, ow - 1)]   # [n, h, w, Cout]
                for j in range(coutg):
                    co = grp * coutg + j
                    dv = np.where(inside, rows[..., co], F32(0))
                    acc = np.where(tap, (acc + dv * w[co, ky, kx, ci]).astype(F32), acc)
    return acc


def wgrad_segments(pixels: int, elems: int) -> tuple[int, int]:
    """(segment length L, segments S) of conv2d_grp_wgrad_*: S' = min(4096, max(1, ceil(2^18 / E))), L = max(64,
    ceil(P / S')), S = ceil(P / L) (1 when P = 0)."""
    want = min(4096, max(1, -(-(1 << 18) // elems)))
    seg = max(64, -(-pixels // want))
    return seg, (-(-pixels // seg) if pixels else 1)


def wgrad_f32(x, dy, kernel_hw, groups, stride=1, padding=0, dilation=1):
    """conv2d_grp_wgrad_* and its combine: per segment of L pixels, acc = +0; for pixels ascending: acc = fma(dy, x, acc);
    dw = ((p_0 + p_1) + p_2) + ... in f32.  Returns (dw [Cout, KH, KW, Cg], (L, S))."""
    x, dy = np.asarray(x, F32), np.asarray(dy, F32)
    n, h, wd, c = x.shape
    _, oh, ow, cout = dy.shape
    kh, kw = kernel_hw
    cg, coutg = _split(c, cout, groups)
    (sh, sw), (ph, pw), (dh, dw) = pair(stride), pair(padding), pair(dilation)
    P = n * oh * ow
    seg, nseg = wgrad_segments(P, cout * kh * kw * cg)
    chan = ((np.arange(cout) // coutg) * cg)[:, None] + np.arange(cg)[None, :]   # [Cout, Cg] input channel
    ky = np.arange(kh)[:, None, None, None]
    kx = np.arange(kw)[None, :, None, None]
    part = np.zeros((nseg, kh, kw, cout, cg), F32)
    with np.errstate(invalid="ignore", over="ignore"):
        for i in range(seg):
            for s in range(nseg):
                q = s * seg + i
                if q >= P:
                    continue
                b, r = divmod(q, oh * ow)
                y, xo = divmod(r, ow)
                iy = y * sh - ph + ky * dh
                ix = xo * sw - pw + kx * dw
                ok = (iy >= 0) & (iy < h) & (ix >= 0) & (ix < wd)
                xv = np.where(ok, x[b, np.clip(iy, 0, h - 1), np.clip(ix, 0, wd - 1), chan[None, None]], F32(0))
                part[s] = (part[s] + dy[b, y, xo, :][None, None, :, None] * xv).astype(F32)
        out = part[0]
        for s in range(1, nseg):
            out = (out + part[s]).astype(F32)
    return np.ascontiguousarray(out.transpose(2, 0, 1, 3)), (seg, nseg)
