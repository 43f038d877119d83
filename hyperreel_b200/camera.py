"""Camera -> rays on the device, and whole-frame rendering to 8-bit pixels (SURVEY.md section 8(f) rows f2 and f4).

Mirrors ``get_coords_from_camera`` of the reference datasets (datasets/base.py:485-518: pixel grid ->
``get_ray_directions_K`` -> ``get_rays`` -> optional ``to_ndc`` -> append camera id and time), the fisheye cameras of
``ImmersiveDataset.get_coords`` (``Camera(distortion=(k1, k2))``, datasets/immersive.py:494-573) and ``to8b``
(utils/__init__.py:47).  The reference builds the rays on the CPU and uploads 32 B per ray for every frame
(nlf/__init__.py:828-834); here only the pose and intrinsics cross PCIe and 3 B per pixel come back.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional, Sequence, Tuple

import numpy as np
import torch

from . import lib as L


@dataclass
class Camera:
    pose: Sequence[Sequence[float]]  # camera-to-world, at least 3x4
    K: Sequence[Sequence[float]]     # 3x3 intrinsics
    width: int
    height: int
    time: float = 0.0
    cam_idx: float = 0.0
    centered_pixels: bool = True     # datasets/technicolor.py:377
    flipped: bool = False
    normalize: bool = True
    use_ndc: bool = False
    ndc_near: float = 1.0
    # (k1, k2): the Immersive dataset's fisheye camera (ImmersiveDataset.get_coords, datasets/immersive.py:494-573), the
    # first two radial_distortion coefficients of models.json, rounded to float32 as the reference's .astype(np.float32).
    # None is the pinhole.  (0, 0) is not: the fisheye model maps the radius r -> tan(r).
    distortion: Optional[Sequence[float]] = None

    def __post_init__(self):
        self._distortion_f32()

    def _distortion_f32(self) -> Optional[Tuple[float, float]]:
        if self.distortion is None:
            return None
        d = np.asarray(self.distortion, dtype=np.float64).reshape(-1)
        if d.shape != (2,):
            raise ValueError(f"distortion must be (k1, k2), got {self.distortion!r}")
        with np.errstate(over="ignore"):
            k = d.astype(np.float32)
        if not np.isfinite(k).all():
            raise ValueError(f"distortion coefficients must be finite in float32, got {self.distortion!r}")
        return float(k[0]), float(k[1])

    def to_c(self) -> L.hr_camera:
        c = L.hr_camera()
        pose = torch.as_tensor(self.pose, dtype=torch.float32)
        K = torch.as_tensor(self.K, dtype=torch.float32)
        for r in range(3):
            for k in range(4):
                c.c2w[r * 4 + k] = float(pose[r, k])
        c.fx, c.fy, c.cx, c.cy = float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2])
        c.width, c.height = int(self.width), int(self.height)
        c.centered_pixels, c.flipped = int(self.centered_pixels), int(self.flipped)
        c.normalize, c.use_ndc = int(self.normalize), int(self.use_ndc)
        c.ndc_near, c.cam_idx, c.time = float(self.ndc_near), float(self.cam_idx), float(self.time)
        k = self._distortion_f32()
        if k is not None:
            c.fisheye, (c.k1, c.k2) = 1, k
        return c


def generate_rays(camera: Camera, c_in: int = 8, device: Optional[torch.device] = None, first_pixel: int = 0,
                  n_pixels: Optional[int] = None) -> torch.Tensor:
    """rays [n, c_in] fp32 on the device for pixels ``first_pixel ... first_pixel + n - 1`` (row-major)."""
    import ctypes as C

    lib = L.load_library()
    if not torch.cuda.is_available():
        raise RuntimeError("hyperreel_b200.generate_rays needs a CUDA device (no CPU fallback)")
    device = device or torch.device("cuda", torch.cuda.current_device())
    n = camera.width * camera.height - first_pixel if n_pixels is None else n_pixels
    out = torch.empty((n, c_in), dtype=torch.float32, device=device)
    cam = camera.to_c()
    with torch.cuda.device(device):
        L.check(lib.hr_generate_rays(C.byref(cam), c_in, first_pixel, n, out.data_ptr(),
                                     torch.cuda.current_stream(device).cuda_stream))
    return out
