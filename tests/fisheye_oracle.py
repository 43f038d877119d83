"""CPU oracle of the Immersive dataset's fisheye cameras (DESIGN.md section 4.4).  TEST INFRASTRUCTURE.

Restates the fisheye branch of ``ImmersiveDataset.get_coords`` (datasets/immersive.py:494-573): OpenCV 4.x's
``cv2.fisheye.undistortPoints`` in NumPy fp64, then the reference's fp32 tail (``F.normalize``, ``get_rays``) through
oracle/rays_oracle.py.  Pinned against cv2 itself and against tests/golden/rays_fisheye_*.npz (tests/test_fisheye_oracle.py).
"""
from __future__ import annotations

import numpy as np
import torch

from oracle.rays_oracle import get_rays, ndc_rays, ray_directions


def fisheye_undistort(points, k1, k2) -> np.ndarray:
    """cv2.fisheye.undistortPoints(points[:, None], I, [k1, k2, 0, 0])[:, 0] of OpenCV 4.x (default criteria COUNT + EPS,
    10 iterations, 1e-8) for float32 points [n, 2]: the fp64 Newton solve in OpenCV's operation order, vectorised (NumPy's
    elementwise double arithmetic is IEEE without contraction).  A point that does not converge, or whose angle flips sign,
    gives OpenCV's (-1e6, -1e6).  k1, k2 are widened from float32 like the reference's coefficient array."""
    p = np.asarray(points, dtype=np.float32).astype(np.float64)
    k1, k2 = float(np.float32(k1)), float(np.float32(k2))
    x, y = p[:, 0], p[:, 1]
    with np.errstate(all="ignore"):
        theta_d = np.minimum(np.maximum(-np.pi / 2, np.sqrt(x * x + y * y)), np.pi / 2)
        solve = np.abs(theta_d) > 1e-8
        theta = theta_d.copy()
        converged = ~solve
        active = solve.copy()
        for _ in range(10):
            t2 = theta * theta
            t4 = t2 * t2
            a, b = k1 * t2, k2 * t4
            fix = (theta * ((1.0 + a) + b) - theta_d) / ((1.0 + 3.0 * a) + 5.0 * b)
            theta = np.where(active, theta - fix, theta)
            done = active & (np.abs(fix) < 1e-8)
            converged |= done
            active &= ~done
        scale = np.where(solve, np.tan(theta) / np.where(solve, theta_d, 1.0), 0.0)
        flipped = ((theta_d < 0) & (theta > 0)) | ((theta_d > 0) & (theta < 0))
        ok = converged & ~flipped
        u = np.where(ok, x * scale, -1000000.0)
        v = np.where(ok, y * scale, -1000000.0)
    return np.stack([u, v], -1).astype(np.float32)


def fisheye_coords_from_camera(pose, K, W, H, distortion, time=0.0, cam_idx=0.0, use_ndc=False, near=1.0, c_in=8,
                               pixels=None):
    """The fisheye branch of ImmersiveDataset.get_coords (datasets/immersive.py:494-573): centred pinhole directions, their
    (x, y) undistorted (fisheye_undistort), F.normalize of (u, v, -1), then get_rays (+ NDC) and the cam_idx / time
    channels.  ``pixels``: row-major pixel ids to keep (all by default)."""
    K = torch.as_tensor(K, dtype=torch.float32)
    c2w = torch.as_tensor(pose, dtype=torch.float32)[:3, :4]
    d = ray_directions(H, W, K, centered_pixels=True).reshape(-1, 3)
    if pixels is not None:
        d = d[torch.as_tensor(pixels, dtype=torch.int64)]
    uv = torch.from_numpy(fisheye_undistort(d[:, :2].numpy(), distortion[0], distortion[1]))
    d = torch.nn.functional.normalize(torch.cat([uv, -torch.ones_like(uv[:, :1])], -1), dim=-1)
    o, d = get_rays(d, c2w)
    rays = torch.cat([o, d], -1)
    if use_ndc:
        rays = ndc_rays(H, W, K[0, 0], K[1, 1], near, rays)
    if c_in == 8:
        rays = torch.cat([rays, torch.ones_like(rays[..., :1]) * cam_idx, torch.ones_like(rays[..., :1]) * time], -1)
    return rays
