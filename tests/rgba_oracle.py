"""CPU oracle of the RGBA datasets' frames (DESIGN.md section 4.4e).  TEST INFRASTRUCTURE.

DoNeRF and Catacaustics load their frames as RGBA and return ``rgb * a + (1 - a)`` from ``get_rgb``
(datasets/donerf.py, datasets/catacaustics.py).  This restates, in NumPy, what happens to such a frame:

* ``cv2.resize(.., INTER_AREA)`` on the 4-channel array (DoNeRF): the four channels resampled independently, with the
  resamplers of tests/resize_oracle.py;
* ``Image.resize`` on an RGBA image (Catacaustics: Pillow's default BICUBIC, then BOX): Pillow converts to premultiplied
  ``RGBa``, resamples that with its 8-bit convolution and converts back, on every call that changes the size;
* ``T.ToTensor()`` then the composite over white, each fp32 operation rounded on its own.

Pinned against Pillow, OpenCV and tests/golden/rgba.npz by tests/test_rgba_oracle.py.
"""
from __future__ import annotations

import numpy as np

from tests import resize_oracle as ro

# dataset name -> (first step to _img_wh, second step to img_wh when scale() reduced it), as hyperreel_b200.resize.RGBA_RESIZE
STEPS = {"donerf": ("cv2_area", "cv2_area"), "catacaustics": ("pil_bicubic", "pil_box")}


def premultiply(c, a):
    """Pillow's RGBA -> RGBa (rgbA2rgba): MULDIV255(c, a) = ((t >> 8) + t) >> 8 with t = c * a + 128."""
    t = np.asarray(c, np.int64) * np.asarray(a, np.int64) + 128
    return ((t >> 8) + t) >> 8


def unpremultiply(c, a):
    """Pillow's RGBa -> RGBA (rgba2rgbA): c for a of 0 or 255, else min(255, 255 * c // a)."""
    c, a = np.asarray(c, np.int64), np.asarray(a, np.int64)
    return np.where((a == 0) | (a == 255), c, np.minimum(255, (255 * c) // np.maximum(a, 1)))


def _pil_passes(src: np.ndarray, W: int, H: int, method: str) -> np.ndarray:
    """Pillow's two 8-bit passes over an int64 [H0, W0, C] image of any channel count (ImagingResampleInner)."""
    H0, W0, C = src.shape
    hb, hk = ro.pil_coeffs(W0, W, method)
    vb, vk = ro.pil_coeffs(H0, H, method)
    if W != W0:
        y0, y1 = int(vb[0, 0]), int(vb[-1, 0] + vb[-1, 1])
        rows = src[y0:y1]
        acc = np.full((y1 - y0, W, C), 1 << (ro.PRECISION_BITS - 1), np.int64)
        for t in range(hk.shape[1]):
            idx = np.minimum(hb[:, 0] + t, W0 - 1)
            acc += rows[:, idx, :] * np.where(t < hb[:, 1], hk[:, t], 0)[None, :, None]
        src = ro._clip8(acc).astype(np.int64)
        vb = vb.copy()
        vb[:, 0] -= y0
    if H != H0:
        acc = np.full((H, src.shape[1], C), 1 << (ro.PRECISION_BITS - 1), np.int64)
        for t in range(vk.shape[1]):
            idx = np.minimum(vb[:, 0] + t, src.shape[0] - 1)
            acc += src[idx, :, :] * np.where(t < vb[:, 1], vk[:, t], 0)[:, None, None]
        src = ro._clip8(acc).astype(np.int64)
    return src


def pil_resize_rgba(img: np.ndarray, size, method: str) -> np.ndarray:
    """Image.fromarray(img, "RGBA").resize(size, filter) as uint8 [H, W, 4], size = (W, H): premultiply, resample,
    unpremultiply; a frame of the same size is copied."""
    img = np.asarray(img, np.uint8)
    H0, W0 = img.shape[:2]
    W, H = int(size[0]), int(size[1])
    if (W, H) == (W0, H0):
        return img.copy()
    if W > W0 or H > H0:
        raise ValueError(f"{method}: upscaling {(W0, H0)} -> {(W, H)} is not supported")
    src = img.astype(np.int64)
    src[..., :3] = premultiply(src[..., :3], src[..., 3:])
    out = _pil_passes(src, W, H, method)
    out[..., :3] = unpremultiply(out[..., :3], out[..., 3:])
    return out.astype(np.uint8)


def cv2_area_rgba(img: np.ndarray, size) -> np.ndarray:
    """cv2.resize(img, size, interpolation=INTER_AREA) of a uint8 [H0, W0, 4] array at integer factors (and the identity)."""
    img = np.asarray(img, np.uint8)
    H0, W0, C = img.shape
    W, H = int(size[0]), int(size[1])
    path = ro.cv2_path((W0, H0), (W, H), "cv2_area")
    if path == "copy":
        return img.copy()
    _, _, ix, iy, _ = ro.cv2_scales((W0, H0), (W, H))
    s = img.astype(np.int64)[:H * iy, :W * ix].reshape(H, iy, W, ix, C).sum(axis=(1, 3))
    if path == "area2":
        return ((s + 2) >> 2).astype(np.uint8)
    v = s.astype(np.float32) * np.float32(np.float32(1.0) / np.float32(ix * iy))
    return np.clip(np.rint(v), 0, 255).astype(np.uint8)


def resize(img: np.ndarray, size, method: str) -> np.ndarray:
    """One RGBA frame [H0, W0, 4] uint8 -> [H, W, 4] uint8 with pil_lanczos / pil_bicubic / pil_box (premultiplied) or
    cv2_area (per channel)."""
    if method in ro.PIL_METHODS:
        return pil_resize_rgba(img, size, method)
    if method == "cv2_area":
        return cv2_area_rgba(img, size)
    raise ValueError(f"no RGBA resize restated for {method!r}")


def composite(rgba: np.ndarray) -> np.ndarray:
    """uint8 [..., 4] -> fp32 [..., 3]: T.ToTensor() (u8 / 255, correctly rounded) then rgb * a + (1 - a), each operation
    rounded to fp32 on its own (NumPy does not contract)."""
    x = np.asarray(rgba, np.uint8).astype(np.float32) / np.float32(255)
    a = x[..., 3:]
    return (x[..., :3] * a + (np.float32(1) - a)).astype(np.float32)


def dataset_steps(name: str, capture_wh, img_wh, scale: int):
    """The resizes of get_rgb of dataset ``name`` for a frame of ``capture_wh`` with ``_img_wh = img_wh``."""
    first, second = STEPS[name]
    wh0 = (int(img_wh[0]), int(img_wh[1]))
    wh = (wh0[0] // scale, wh0[1] // scale)
    steps = []
    if tuple(int(v) for v in capture_wh) != wh0:
        steps.append((first, wh0))
    if wh != wh0:
        steps.append((second, wh))
    return steps


def get_rgb(name: str, frame: np.ndarray, img_wh, scale: int = 1) -> np.ndarray:
    """get_rgb's fp32 [H * W, 3] of one RGBA frame, restated."""
    img = np.asarray(frame, np.uint8)
    for method, wh in dataset_steps(name, (img.shape[1], img.shape[0]), img_wh, scale):
        img = resize(img, wh, method)
    return composite(img).reshape(-1, 3)
