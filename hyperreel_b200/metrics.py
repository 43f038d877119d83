"""Held-out view scoring on the device: the reference's validation PSNR and SSIM (metrics.py:25-34).

The reference copies every validation / test frame to the host and scores it with scikit-image
(``INRSystem.validation_image``, nlf/__init__.py:976-980).  ``image_metrics`` computes the same two quantities with one call
of ``hr_image_metrics`` (csrc/hr_metrics.cu), in fp64:

  * mse:  mean of ``(pred - gt)**2`` over all ``H*W*3`` values (difference and square in fp32, as scikit-image takes them for
    float32 images), the quantity behind ``peak_signal_noise_ratio(pred, gt, data_range=1.0)``;
  * ssim: ``structural_similarity(gt, pred, win_size=11, multichannel=True, gaussian_weights=True, data_range=1.0)``: per
    channel, Gaussian-filtered moments (sigma 1.5, truncate 3.5), sample covariance, C1 = 0.01**2, C2 = 0.03**2, the SSIM map
    averaged over ``[5, H-5) x [5, W-5)``, then over the channels.

There is no CPU path: a CPU tensor raises ``RuntimeError``.  Malformed arguments raise ``ValueError`` before any device work.
"""
from __future__ import annotations

from typing import Tuple

import torch

from . import lib as L

WIN_SIZE = 11  # scikit-image's window for sigma 1.5, truncate 3.5: 2 * int(3.5 * 1.5 + 0.5) + 1


def _validate(pred: torch.Tensor, gt: torch.Tensor) -> Tuple[int, int, int]:
    for name, t in (("pred", pred), ("gt", gt)):
        if not isinstance(t, torch.Tensor):
            raise ValueError(f"{name} must be a torch.Tensor, got {type(t).__name__}")
        if t.dtype != torch.float32:
            raise ValueError(f"{name} must be float32, got {t.dtype}")
        if t.dim() not in (3, 4) or t.shape[-1] != 3:
            raise ValueError(f"{name} must be [H, W, 3] or [n, H, W, 3], got {tuple(t.shape)}")
        if not t.is_contiguous():
            raise ValueError(f"{name} must be contiguous")
    if pred.shape != gt.shape:
        raise ValueError(f"pred and gt shapes differ: {tuple(pred.shape)} vs {tuple(gt.shape)}")
    n = pred.shape[0] if pred.dim() == 4 else 1
    H, W = pred.shape[-3], pred.shape[-2]
    if n < 1:
        raise ValueError("no images to score")
    if H < WIN_SIZE or W < WIN_SIZE:
        raise ValueError(f"win_size exceeds image extent: SSIM needs H and W >= {WIN_SIZE}, got {H} x {W}")
    for name, t in (("pred", pred), ("gt", gt)):
        if t.device.type != "cuda":
            raise RuntimeError(f"hyperreel_b200.metrics: {name} is on {t.device}; image metrics run on the GPU only "
                               "(no CPU fallback)")
    if pred.device != gt.device:
        raise ValueError(f"pred and gt are on different devices: {pred.device} vs {gt.device}")
    return n, H, W


def image_metrics(pred: torch.Tensor, gt: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """(mse, ssim) of each image pair, fp64 device tensors of shape ``[n]``.  ``pred`` / ``gt``: ``[H, W, 3]`` or
    ``[n, H, W, 3]`` fp32 contiguous CUDA tensors on one device.  Enqueued on the current stream, no host synchronisation;
    bit-reproducible, and an image scores the same alone or in a batch."""
    n, H, W = _validate(pred, gt)
    lib = L.load_library()
    dev = pred.device
    out = torch.empty((n, 2), dtype=torch.float64, device=dev)
    ws = torch.empty((int(lib.hr_image_metrics_workspace_bytes(n, H, W)),), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        L.check(lib.hr_image_metrics(pred.data_ptr(), gt.data_ptr(), n, H, W, out.data_ptr(), ws.data_ptr(), ws.numel(),
                                     torch.cuda.current_stream(dev).cuda_stream))
    return out[:, 0], out[:, 1]


def _unbatch(x: torch.Tensor, like: torch.Tensor) -> torch.Tensor:
    return x[0] if like.dim() == 3 else x


def psnr(image_pred: torch.Tensor, image_gt: torch.Tensor) -> torch.Tensor:
    """metrics.psnr: ``peak_signal_noise_ratio(pred, gt, data_range=1.0)`` = ``10 * log10(1 / mse)`` (``+inf`` when the images
    are equal).  A 0-d fp64 device tensor for ``[H, W, 3]`` inputs, ``[n]`` for a batch."""
    mse, _ = image_metrics(image_pred, image_gt)
    return _unbatch(10.0 * torch.log10(1.0 / mse), image_pred)


def ssim(image0: torch.Tensor, image1: torch.Tensor) -> torch.Tensor:
    """metrics.ssim: ``structural_similarity(image1, image0, win_size=11, multichannel=True, gaussian_weights=True,
    data_range=1.0)``.  A 0-d fp64 device tensor for ``[H, W, 3]`` inputs, ``[n]`` for a batch."""
    _, s = image_metrics(image1, image0)
    return _unbatch(s, image0)
