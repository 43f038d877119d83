"""CPU restatement of the reference's validation metrics, the yardstick of ``hyperreel_b200.metrics``.

The reference scores held-out views with ``metrics.psnr`` / ``metrics.ssim`` (metrics.py:25-34), called from
``INRSystem.validation_image`` (nlf/__init__.py:976-980):

  * ``peak_signal_noise_ratio(pred, gt, data_range=1.0)``;
  * ``structural_similarity(gt, pred, win_size=11, multichannel=True, gaussian_weights=True, data_range=1.0)``.

scikit-image is restated here with NumPy / SciPy, only with those arguments: the filter is
``scipy.ndimage.gaussian_filter(sigma=1.5, truncate=3.5, mode='reflect')`` -- what scikit-image calls for
``gaussian_weights=True`` -- and the SSIM map, the sample-covariance factor and the 5-pixel crop follow its definition.

``fp64=True`` filters and evaluates in float64 (scikit-image before 0.19 converts every input to float64); it is the pin the
device kernel is tested against.  ``fp64=False`` keeps float32 images in float32 through the filter and the map, as
scikit-image 0.19 and later do.  The reference does not pin a scikit-image version, so both are "the reference".
"""
from __future__ import annotations

import numpy as np
from scipy.ndimage import gaussian_filter

SIGMA, TRUNCATE = 1.5, 3.5
WIN_SIZE = 2 * int(TRUNCATE * SIGMA + 0.5) + 1  # 11
PAD = (WIN_SIZE - 1) // 2
K1, K2, DATA_RANGE = 0.01, 0.03, 1.0


def mse(image_pred, image_gt) -> float:
    """scikit-image's mean_squared_error: difference and square in the images' dtype, mean accumulated in float64."""
    a, b = np.asarray(image_pred), np.asarray(image_gt)
    return float(np.mean((a - b) ** 2, dtype=np.float64))


def psnr(image_pred, image_gt) -> float:
    """metrics.psnr: 10 log10(data_range^2 / mse), +inf for identical images."""
    err = np.float64(mse(image_pred, image_gt))
    with np.errstate(divide="ignore"):
        return float(10 * np.log10((DATA_RANGE ** 2) / err))


def ssim_map(X: np.ndarray, Y: np.ndarray) -> np.ndarray:
    """The full SSIM map of one channel pair, in the arrays' dtype."""
    def filt(a):
        return gaussian_filter(a, sigma=SIGMA, truncate=TRUNCATE, mode="reflect")

    NP = WIN_SIZE ** 2
    cov_norm = NP / (NP - 1)
    ux, uy = filt(X), filt(Y)
    uxx, uyy, uxy = filt(X * X), filt(Y * Y), filt(X * Y)
    vx = cov_norm * (uxx - ux * ux)
    vy = cov_norm * (uyy - uy * uy)
    vxy = cov_norm * (uxy - ux * uy)
    C1, C2 = (K1 * DATA_RANGE) ** 2, (K2 * DATA_RANGE) ** 2
    A1, A2 = 2 * ux * uy + C1, 2 * vxy + C2
    B1, B2 = ux ** 2 + uy ** 2 + C1, vx + vy + C2
    return (A1 * A2) / (B1 * B2)


def structural_similarity(im1, im2, fp64: bool = True) -> float:
    """structural_similarity(im1, im2, win_size=11, multichannel=True, gaussian_weights=True, data_range=1.0) of two
    [H, W, C] images: the mean of each channel's cropped SSIM map, averaged over the channels."""
    im1, im2 = np.asarray(im1), np.asarray(im2)
    if im1.shape != im2.shape or im1.ndim != 3:
        raise ValueError(f"expected two [H, W, C] images of one shape, got {im1.shape} and {im2.shape}")
    if min(im1.shape[:2]) < WIN_SIZE:
        raise ValueError("win_size exceeds image extent")
    ft = np.float64 if fp64 else np.float32
    per_channel = np.empty(im1.shape[-1], dtype=np.float64)
    for ch in range(im1.shape[-1]):
        S = ssim_map(im1[..., ch].astype(ft), im2[..., ch].astype(ft))
        per_channel[ch] = S[PAD:-PAD, PAD:-PAD].mean(dtype=np.float64)
    return float(per_channel.mean())


def ssim(image0, image1, fp64: bool = True) -> float:
    """metrics.ssim(image0, image1) = structural_similarity(image1, image0, ...)."""
    return structural_similarity(image1, image0, fp64=fp64)


def smooth_noisy_pair(h: int, w: int, seed: int):
    """Seeded test frames (pred, gt), fp32 [h, w, 3]: a smooth 'scene' in [0, 1] and a slightly blurred, noisy render of it."""
    rng = np.random.default_rng(seed)
    gt = gaussian_filter(rng.random((h, w, 3)), sigma=(12, 12, 0))
    gt = (gt - gt.min()) / (gt.max() - gt.min())
    pred = gaussian_filter(gt, sigma=(0.7, 0.7, 0)) + 0.03 * rng.standard_normal((h, w, 3))
    return np.clip(pred, 0, 1).astype(np.float32), gt.astype(np.float32)
