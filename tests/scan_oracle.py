"""CPU restatement of the axis scans for the scan tests (test infrastructure only).

scan_axis_f32 is the serial left-to-right f32 scan: the running value starts at the identity and takes one element at a
time (numpy's ufunc.accumulate is sequential in the output dtype), the order of plane.rs's expected loops
(crates/cubecl-core/src/runtime_tests/plane.rs:191-405) for a whole axis.  scan_axis_f64 gives the f64 truth and the
prefix sums of |x|, the scale of the error bounds.
"""
from __future__ import annotations

import numpy as np

IDENTITY = {"sum": 0.0, "prod": 1.0, "max": -np.inf, "min": np.inf}
UFUNC = {"sum": np.add, "prod": np.multiply, "max": np.maximum, "min": np.minimum}   # maximum / minimum propagate NaN


def _scan(x, axis: int, op: str, exclusive: bool, dtype) -> np.ndarray:
    x = np.moveaxis(np.asarray(x, dtype=dtype), axis, 0)
    pad = np.full((1,) + x.shape[1:], IDENTITY[op], dtype=dtype)
    acc = UFUNC[op].accumulate(np.concatenate([pad, x]), axis=0, dtype=dtype)
    out = acc[:-1] if exclusive else acc[1:]
    return np.ascontiguousarray(np.moveaxis(out, 0, axis))


def scan_axis_f32(x, axis: int, op: str = "sum", exclusive: bool = False) -> np.ndarray:
    """Reference-order f32 scan of `axis`: out[l] = (((id op x0) op x1) ... op x_l) (exclusive: up to x_{l-1})."""
    return _scan(x, axis, op, exclusive, np.float32)


def scan_axis_f64(x, axis: int, op: str = "sum", exclusive: bool = False):
    """(f64 scan, f64 prefix sum of |x| along the same positions)."""
    x = np.asarray(x, dtype=np.float64)
    return _scan(x, axis, op, exclusive, np.float64), _scan(np.abs(x), axis, "sum", exclusive, np.float64)

