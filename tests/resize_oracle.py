"""CPU oracle of the datasets' image resizes (DESIGN.md section 4.4e).  TEST INFRASTRUCTURE.

Restates, in NumPy integer arithmetic, the two resamplers the reference's ``get_rgb``s call on uint8 RGB frames:

* Pillow's 8-bit convolution resampler (``Image.resize`` with LANCZOS, BICUBIC or BOX; libImaging/Resample.c): tap
  bounds and coefficients in double, normalised, converted to fixed point with ``PRECISION_BITS`` = 22, the horizontal pass
  over the rows the vertical pass reads into a clipped uint8 intermediate, then the vertical pass.
* OpenCV's ``cv2.resize`` for CV_8UC3 (imgproc/src/resize.cpp): the INTER_LINEAR fixed-point path (11-bit coefficients)
  and the INTER_AREA fast path for integer factors, with OpenCV's rule that sends INTER_LINEAR at exactly 2x to it.

The coefficient tables are built in the same precision and order as the libraries build them (``math.sin`` is the C
library's ``sin``, as Pillow's is); the library's ``csrc/hr_resize.cu`` builds the same tables on the host.  Pinned against
cv2 and Pillow themselves and against tests/golden/resize.npz (tests/test_resize_oracle.py).
"""
from __future__ import annotations

import math

import numpy as np

PRECISION_BITS = 22  # Pillow, 8 bits per channel: 32 - 8 - 2
COEF_BITS = 11       # OpenCV INTER_RESIZE_COEF_BITS

PIL_METHODS = ("pil_lanczos", "pil_bicubic", "pil_box")
CV2_METHODS = ("cv2_linear", "cv2_area")
METHODS = PIL_METHODS + CV2_METHODS


# ---------------------------------------------------------------------------------------------------------------- Pillow
def _box(x):
    return 1.0 if -0.5 < x <= 0.5 else 0.0


def _bicubic(x):
    a = -0.5
    x = -x if x < 0.0 else x
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


def _sinc(x):
    if x == 0.0:
        return 1.0
    x = x * math.pi
    return math.sin(x) / x


def _lanczos(x):
    return _sinc(x) * _sinc(x / 3) if -3.0 <= x < 3.0 else 0.0


PIL_FILTERS = {"pil_lanczos": (_lanczos, 3.0), "pil_bicubic": (_bicubic, 2.0), "pil_box": (_box, 0.5)}


def _c_int(x: float) -> int:
    """C's (int) cast of a double: truncation toward zero."""
    return int(math.trunc(x))


def pil_coeffs(in_size: int, out_size: int, method: str):
    """precompute_coeffs + normalize_coeffs_8bpc for the box (0, in_size): (bounds [out, 2] int32 = (xmin, count),
    coefficients [out, ksize] int32)."""
    fn, fsupport = PIL_FILTERS[method]
    in0, in1 = float(np.float32(0.0)), float(np.float32(in_size))  # the box is float in Pillow
    scale = filterscale = (in1 - in0) / out_size
    if filterscale < 1.0:
        filterscale = 1.0
    support = fsupport * filterscale
    ksize = _c_int(math.ceil(support)) * 2 + 1
    bounds = np.zeros((out_size, 2), np.int32)
    kk = np.zeros((out_size, ksize), np.int32)
    for xx in range(out_size):
        center = in0 + (xx + 0.5) * scale
        ww = 0.0
        ss = 1.0 / filterscale
        xmin = _c_int(center - support + 0.5)
        if xmin < 0:
            xmin = 0
        xmax = _c_int(center + support + 0.5)
        if xmax > in_size:
            xmax = in_size
        xmax -= xmin
        k = []
        for x in range(xmax):
            w = fn((x + xmin - center + 0.5) * ss)
            k.append(w)
            ww += w
        for x in range(xmax):
            if ww != 0.0:
                k[x] /= ww
            v = k[x] * (1 << PRECISION_BITS)
            kk[xx, x] = _c_int(-0.5 + v) if k[x] < 0 else _c_int(0.5 + v)
        bounds[xx] = (xmin, xmax)
    return bounds, kk


def _clip8(acc: np.ndarray) -> np.ndarray:
    return np.clip(acc >> PRECISION_BITS, 0, 255).astype(np.uint8)  # arithmetic shift, as Pillow's lookup index


def pil_resize(img: np.ndarray, size, method: str) -> np.ndarray:
    """Image.fromarray(img).resize(size, filter) as uint8 [H, W, 3], size = (W, H)."""
    img = np.asarray(img, np.uint8)
    H0, W0 = img.shape[:2]
    W, H = int(size[0]), int(size[1])
    if (W, H) == (W0, H0):
        return img.copy()
    hb, hk = pil_coeffs(W0, W, method)
    vb, vk = pil_coeffs(H0, H, method)
    src = img.astype(np.int64)
    if W != W0:  # the horizontal pass, over the rows the vertical pass reads
        y0, y1 = int(vb[0, 0]), int(vb[-1, 0] + vb[-1, 1])
        rows = src[y0:y1]
        acc = np.full((y1 - y0, W, 3), 1 << (PRECISION_BITS - 1), np.int64)
        for t in range(hk.shape[1]):
            idx = np.minimum(hb[:, 0] + t, W0 - 1)
            acc += rows[:, idx, :] * np.where(t < hb[:, 1], hk[:, t], 0)[None, :, None]
        src = _clip8(acc).astype(np.int64)
        vb = vb.copy()
        vb[:, 0] -= y0
    if H != H0:
        acc = np.full((H, src.shape[1], 3), 1 << (PRECISION_BITS - 1), np.int64)
        for t in range(vk.shape[1]):
            idx = np.minimum(vb[:, 0] + t, src.shape[0] - 1)
            acc += src[idx, :, :] * np.where(t < vb[:, 1], vk[:, t], 0)[:, None, None]
        src = _clip8(acc).astype(np.int64)
    return src.astype(np.uint8)


# ---------------------------------------------------------------------------------------------------------------- OpenCV
def cv2_scales(in_wh, out_wh):
    """resize()'s scale factors and its fast-area test, in double as OpenCV computes them."""
    sx = 1.0 / (out_wh[0] / in_wh[0])
    sy = 1.0 / (out_wh[1] / in_wh[1])
    ix, iy = int(round(sx)), int(round(sy))  # saturate_cast<int>(double) rounds to nearest
    fast = abs(sx - ix) < np.finfo(np.float64).eps and abs(sy - iy) < np.finfo(np.float64).eps
    return sx, sy, ix, iy, fast


def cv2_path(in_wh, out_wh, method: str) -> str:
    """Which code path cv2.resize takes for uint8 3-channel frames: 'copy', 'area2' (the 2 x 2 vector path),
    'area' (integer factors), 'linear', or a refusal."""
    if tuple(in_wh) == tuple(out_wh):
        return "copy"
    if out_wh[0] > in_wh[0] or out_wh[1] > in_wh[1]:
        raise ValueError(f"{method}: upscaling {tuple(in_wh)} -> {tuple(out_wh)} is not supported")
    sx, sy, ix, iy, fast = cv2_scales(in_wh, out_wh)
    if method == "cv2_linear" and not (fast and ix == 2 and iy == 2):
        return "linear"
    if method not in ("cv2_linear", "cv2_area"):
        raise ValueError(f"unknown OpenCV method {method!r}")
    if not fast:
        raise ValueError(f"cv2_area: {tuple(in_wh)} -> {tuple(out_wh)} is not an integer reduction (OpenCV's float "
                         "INTER_AREA path is not supported)")
    return "area2" if ix == 2 and iy == 2 else "area"


def cv2_linear_coeffs(in_size: int, out_size: int, is_x: bool):
    """INTER_LINEAR along one axis: (first tap [out] int32, weights [out, 2] int32); the second tap is the first + 1,
    clamped to the last pixel.  Along x a first tap before the first or at the last pixel resets the weights to (2048, 0)
    (resizeGeneric_'s xofs loop); along y the row loop does not clamp the weight, only the row indices are clamped."""
    scale = 1.0 / (out_size / in_size)
    ofs = np.zeros(out_size, np.int32)
    w = np.zeros((out_size, 2), np.int32)
    one, unit = np.float32(1.0), np.float32(1 << COEF_BITS)
    for d in range(out_size):
        f = np.float32((d + 0.5) * scale - 0.5)
        s = math.floor(f)
        f = np.float32(f - np.float32(s))
        if is_x and s < 0:
            f, s = np.float32(0.0), 0
        if is_x and s >= in_size - 1:
            f, s = np.float32(0.0), in_size - 1
        # saturate_cast<short>(float): round half to even
        w[d] = (int(np.rint(np.float32((one - f) * unit))), int(np.rint(np.float32(f * unit))))
        ofs[d] = s
    return ofs, w


def cv2_resize(img: np.ndarray, size, method: str) -> np.ndarray:
    """cv2.resize(img, size, interpolation=INTER_LINEAR / INTER_AREA) as uint8 [H, W, 3] for downscales (and the
    identity), size = (W, H)."""
    img = np.asarray(img, np.uint8)
    H0, W0 = img.shape[:2]
    W, H = int(size[0]), int(size[1])
    path = cv2_path((W0, H0), (W, H), method)
    if path == "copy":
        return img.copy()
    src = img.astype(np.int64)
    if path in ("area", "area2"):
        _, _, ix, iy, _ = cv2_scales((W0, H0), (W, H))
        s = src[:H * iy, :W * ix].reshape(H, iy, W, ix, 3).sum(axis=(1, 3))
        if path == "area2":  # ResizeAreaFastVec: (sum + 2) >> 2
            return ((s + 2) >> 2).astype(np.uint8)
        # resizeAreaFast_Invoker: saturate_cast<uchar>(sum * (1.f / area)) in float, rounded half to even
        v =s.astype(np.float32) * np.float32(np.float32(1.0) / np.float32(ix * iy))
        return np.clip(np.rint(v), 0, 255).astype(np.uint8)
    xo, a = cv2_linear_coeffs(W0, W, True)
    yo, b = cv2_linear_coeffs(H0, H, False)
    x1 = np.minimum(xo + 1, W0 - 1)
    rows = src[:, xo, :] * a[None, :, 0, None] + src[:, x1, :] * a[None, :, 1, None]  # HResizeLinear: int sums
    r0 = rows[np.clip(yo, 0, H0 - 1)]
    r1 = rows[np.clip(yo + 1, 0, H0 - 1)]
    b0, b1 = b[:, 0, None, None], b[:, 1, None, None]
    # VResizeLinear<uchar, int, short, FixedPtCast<int, uchar, 22>>, scalar and vector code alike:
    # ((b0 * (S0 >> 4)) >> 16) + ((b1 * (S1 >> 4)) >> 16) + 2) >> 2
    v = (((b0 * (r0 >> 4)) >> 16) + ((b1 * (r1 >> 4)) >> 16) + 2) >> 2
    return np.clip(v, 0, 255).astype(np.uint8)


def resize(img: np.ndarray, size, method: str) -> np.ndarray:
    """One frame [H0, W0, 3] uint8 -> [H, W, 3] uint8 with one of METHODS; size = (W, H)."""
    if method in PIL_METHODS:
        H0, W0 = np.asarray(img).shape[:2]
        if int(size[0]) > W0 or int(size[1]) > H0:
            raise ValueError(f"{method}: upscaling {(W0, H0)} -> {tuple(size)} is not supported")
        return pil_resize(img, size, method)
    return cv2_resize(img, size, method)
