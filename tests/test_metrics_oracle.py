"""The CPU restatement of the reference's validation metrics (tests/metrics_oracle.py) and the device entry points' argument
checks that need no GPU."""
import numpy as np
import pytest
import torch
from numpy.lib.stride_tricks import sliding_window_view

from hyperreel_b200 import metrics as M
from tests import metrics_oracle as O


def brute_force_ssim(im1, im2):
    """SSIM from explicit 11x11 weighted window sums at every interior pixel (outer product of the normalised 1-D Gaussian):
    independent of gaussian_filter and its border mode."""
    x = np.arange(-5, 6, dtype=np.float64)
    g = np.exp(-x ** 2 / (2 * 1.5 ** 2))
    g /= g.sum()
    w2 = np.outer(g, g)
    vals = []
    for ch in range(im1.shape[-1]):
        X, Y = im1[..., ch].astype(np.float64), im2[..., ch].astype(np.float64)

        def win(a):
            return np.einsum("ijkl,kl->ij", sliding_window_view(a, (11, 11)), w2)

        ux, uy, uxx, uyy, uxy = win(X), win(Y), win(X * X), win(Y * Y), win(X * Y)
        cn = 121.0 / 120.0
        vx, vy, vxy = cn * (uxx - ux * ux), cn * (uyy - uy * uy), cn * (uxy - ux * uy)
        C1, C2 = 0.01 ** 2, 0.03 ** 2
        S = (2 * ux * uy + C1) * (2 * vxy + C2) / ((ux ** 2 + uy ** 2 + C1) * (vx + vy + C2))
        vals.append(S.mean())
    return float(np.mean(vals))


@pytest.mark.parametrize("shape", [(11, 11), (13, 17), (24, 31)])
def test_oracle_ssim_equals_brute_force_window_sums(shape):
    rng = np.random.default_rng(sum(shape))
    a = rng.random(shape + (3,), dtype=np.float32)
    b = np.clip(a + 0.2 * rng.standard_normal(shape + (3,)).astype(np.float32), 0, 1).astype(np.float32)
    assert abs(O.ssim(a, b) - brute_force_ssim(b, a)) <= 1e-12


def test_oracle_identities():
    rng = np.random.default_rng(1)
    a = rng.random((20, 23, 3), dtype=np.float32)
    assert O.ssim(a, a) == 1.0
    assert O.psnr(a, a) == float("inf")
    q = (rng.integers(0, 128, (20, 23, 3)) / 256).astype(np.float32)  # q + d and its difference are exact in fp32
    d = 0.125
    assert O.psnr(q + np.float32(d), q) == pytest.approx(-10 * np.log10(d ** 2), abs=1e-12)
    b = rng.random((20, 23, 3), dtype=np.float32)
    assert O.ssim(a, b) == O.ssim(b, a)
    assert O.psnr(a, b) == O.psnr(b, a)
    c0, c1 = np.full((16, 16, 3), 0.25, np.float32), np.full((16, 16, 3), 0.75, np.float32)
    for v in (O.ssim(c0, c1), O.psnr(c0, c1), O.ssim(c0, c0)):
        assert np.isfinite(v) or v == float("inf")
    assert np.isfinite(O.ssim(c0, c1)) and np.isfinite(O.psnr(c0, c1))


def test_oracle_fp32_and_fp64_modes_agree_on_a_full_frame():
    """scikit-image >= 0.19 filters float32 images in float32, older versions in float64; on a 1088 x 2048 frame the two
    SSIMs (about 0.584) differed by 6.3e-9 when this test was written; the bound leaves a wide margin."""
    pred, gt = O.smooth_noisy_pair(1088, 2048, seed=7)
    s64, s32 = O.ssim(pred, gt, fp64=True), O.ssim(pred, gt, fp64=False)
    assert 0.0 < s64 < 1.0
    assert abs(s64 - s32) <= 1e-6, abs(s64 - s32)


def test_python_entry_points_refuse_bad_arguments_before_the_device():
    good = torch.zeros((16, 16, 3))
    with pytest.raises(RuntimeError, match="GPU only"):
        M.image_metrics(good, good)
    with pytest.raises(RuntimeError, match="GPU only"):
        M.psnr(good, good)
    with pytest.raises(RuntimeError, match="GPU only"):
        M.ssim(good, good)
    bad = [
        (good.double(), good.double(), "float32"),
        (torch.zeros((16, 16, 4)), torch.zeros((16, 16, 4)), r"\[H, W, 3\]"),
        (torch.zeros((16, 48)), torch.zeros((16, 48)), r"\[H, W, 3\]"),
        (torch.zeros((1, 1, 16, 16, 3)), torch.zeros((1, 1, 16, 16, 3)), r"\[H, W, 3\]"),
        (good, torch.zeros((16, 17, 3)), "shapes differ"),
        (torch.zeros((10, 16, 3)), torch.zeros((10, 16, 3)), "win_size"),
        (torch.zeros((16, 10, 3)), torch.zeros((16, 10, 3)), "win_size"),
        (torch.zeros((0, 16, 16, 3)), torch.zeros((0, 16, 16, 3)), "no images"),
        (torch.zeros((16, 3, 16)).transpose(1, 2), good, "contiguous"),
    ]
    for a, b, msg in bad:
        with pytest.raises(ValueError, match=msg):
            M.image_metrics(a, b)
