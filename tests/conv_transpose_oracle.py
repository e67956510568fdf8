"""f64 transposed convolution in numpy, 2-D and 3-D, straight from its definition: every input pixel i and kernel tap k
scatter x[n, i, :] @ w[:, k, :] onto output pixel o = i * s - p + k * d (per dimension) when o lies inside the output.
Channels-last activations, weights [Cin, *kernel, Cout]; the ground truth of the conv_transpose tests."""
from __future__ import annotations

import itertools

import numpy as np


def _tuple(v, n):
    return (int(v),) * n if isinstance(v, (int, np.integer)) else tuple(int(e) for e in v)


def output_shape(x_shape, w_shape, stride=1, padding=0, output_padding=0, dilation=1):
    """[N, *O, Cout]: O = (I - 1) * s - 2 * p + d * (K - 1) + op + 1 per spatial dimension"""
    n = len(x_shape) - 2
    s, p, op, d = (_tuple(v, n) for v in (stride, padding, output_padding, dilation))
    return [x_shape[0]] + [(x_shape[1 + i] - 1) * s[i] - 2 * p[i] + d[i] * (w_shape[1 + i] - 1) + op[i] + 1 for i in range(n)] + [w_shape[-1]]


def conv_transpose_f64(x, w, stride=1, padding=0, output_padding=0, dilation=1, bias=None):
    """(out, abs_out): out = sum of the scattered products (+ bias[co]), abs_out the same sum of |x||w| (+ |bias|)"""
    x = np.asarray(x, dtype=np.float64)
    w = np.asarray(w, dtype=np.float64)
    n = x.ndim - 2
    s, p, d = (_tuple(v, n) for v in (stride, padding, dilation))
    shape = output_shape(x.shape, w.shape, stride, padding, output_padding, dilation)
    out = np.zeros(shape)
    aout = np.zeros(shape)
    for k in itertools.product(*(range(w.shape[1 + i]) for i in range(n))):
        src, dst = [slice(None)], [slice(None)]
        for i in range(n):
            # input pixels j with 0 <= j * s - p + k * d < O
            off = -p[i] + k[i] * d[i]
            lo = max(0, -(off // s[i]))
            hi = min(x.shape[1 + i] - 1, (shape[1 + i] - 1 - off) // s[i])
            if hi < lo:
                break
            src.append(slice(lo, hi + 1))
            dst.append(slice(lo * s[i] + off, hi * s[i] + off + 1, s[i]))
        else:
            wk = w[(slice(None),) + k + (slice(None),)]
            xs = x[tuple(src)]
            out[tuple(dst)] += xs @ wk
            aout[tuple(dst)] += np.abs(xs) @ np.abs(wk)
    if bias is not None:
        out += np.asarray(bias, dtype=np.float64)
        aout += np.abs(np.asarray(bias, dtype=np.float64))
    return out, aout
