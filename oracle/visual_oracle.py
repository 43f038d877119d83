"""The embedding visualiser's map of one frame, restated in NumPy fp32: visualize_warp (utils/visualization.py:24-52) with
``sort: False`` followed by to8b (utils/__init__.py:47), each step rounded on its own as the reference's fp32 tensor ops
round it.  The device path (hr_render_visuals) must equal this bit for bit on its own fp32 field values."""
from __future__ import annotations

import numpy as np


def visualize_to8b(x, use_abs: bool = False, bounds=None, normalize: bool = False) -> np.ndarray:
    """One frame's field ``x`` fp32 [P, dim] (P pixels) -> uint8 [P, dim].

    1. ``use_abs``: |x|.
    2. ``bounds`` [lo, hi]: (x - lo) / (hi - lo), lo and hi rounded to fp32 and hi - lo rounded once.
    3. ``normalize``: (x - min) / (max - min) per channel over the frame's pixels (a NaN anywhere makes min / max NaN).
    4. clamp to [0, 1] (a NaN stays NaN), then (255 * x).astype(uint8): fp32 multiply, truncation, NaN -> 0."""
    v = np.array(x, dtype=np.float32, copy=True)
    if v.ndim != 2:
        raise ValueError(f"visualize_to8b: x must be [P, dim], got {v.shape}")
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        if use_abs:
            v = np.abs(v)
        if bounds is not None and len(bounds) > 0:
            lo, hi = np.float32(bounds[0]), np.float32(bounds[1])
            v = (v - lo) / np.float32(hi - lo)
        if normalize:
            mn, mx = v.min(0, keepdims=True), v.max(0, keepdims=True)
            v = (v - mn) / (mx - mn)
        v = np.clip(v, np.float32(0), np.float32(1))
        v = np.float32(255) * v
    # NumPy's float -> uint8 cast of NaN is platform-defined; the reference's x86 result is 0
    return np.where(np.isnan(v), np.float32(0), v).astype(np.uint8)


def visualize_frames_to8b(x, use_abs: bool = False, bounds=None, normalize: bool = False) -> np.ndarray:
    """Frames [F, P, dim] fp32 -> uint8 [F, P, dim], each frame on its own (``normalize`` is per frame)."""
    x = np.asarray(x, dtype=np.float32)
    return np.stack([visualize_to8b(f, use_abs, bounds, normalize) for f in x], 0)
