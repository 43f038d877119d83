"""Golden rays of the Immersive dataset's fisheye cameras, from the unmodified ``ImmersiveDataset.get_coords``
(datasets/immersive.py:494-573, with cv2.fisheye.undistortPoints) run on CPU through the shim on a stand-in dataset object.

    HYPERREEL_REFERENCE=<reference checkout> python tests/golden/make_golden_fisheye.py

writes ``tests/golden/rays_fisheye_<case>.npz``: ``rays`` [n, 8] fp32 (the rows of ``pixels``), ``pixels`` int64 (row-major
pixel ids; every pixel but for the full-size case, which keeps a fixed strided subset), ``pose`` [3, 4], ``K`` [3, 3],
``distortion`` [2] (float32, as the reference casts it), ``W``, ``H``, ``time``, ``cam_idx``.
"""
import contextlib
import io
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from tests.golden.make_golden_subsample import _install  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))


def _pose(rx, ry, t):
    cx, sx, cy, sy = np.cos(rx), np.sin(rx), np.cos(ry), np.sin(ry)
    R = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]]) @ np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    return np.concatenate([R, np.array(t, dtype=np.float64)[:, None]], 1)


def _K(f, cx, cy):
    return np.array([[f, 0.0, cx], [0.0, f, cy], [0.0, 0.0, 1.0]])


# name: (W, H, K, (k1, k2), pose, time, camera id, split, stride of the stored pixel subset)
CASES = {
    # every pixel converges: radius up to ~0.6
    "mild_40x30": (40, 30, _K(40.0, 19.3, 14.8), (0.05, -0.01), _pose(0.1, -0.2, [0.3, -0.1, 0.5]), 0.25, 3, "train", 1),
    # a strong negative k1: the corners do not converge and become OpenCV's (-1e6, -1e6)
    "strong_48x36": (48, 36, _K(22.0, 24.0, 18.0), (-0.4, 0.05), _pose(-0.05, 0.15, [0.0, 0.2, -0.3]), 0.5, 7, "train", 1),
    # principal point on a pixel centre: pixel (10, 7) has theta_d = 0; a validation view (camera id 1)
    "centre_21x15": (21, 15, _K(12.0, 10.5, 7.5), (0.1, -0.02), _pose(0.0, 0.0, [0.0, 0.0, 0.0]), 0.0, 5, "val", 1),
    # short focal length: the corners pass the pi/2 clamp of theta_d
    "wide_40x30": (40, 30, _K(8.0, 20.0, 15.0), (0.02, 0.001), _pose(0.3, 0.2, [1.0, 0.5, -0.2]), 1.0, 2, "train", 1),
    # Immersive's 1280x960 training shape: intrinsics scaled by W / 2560 and H / 1920 (immersive.py:95-104)
    "immersive_1280x960": (1280, 960, np.array([[1320.0 * 0.5, 0.0, 1283.7 * 0.5], [0.0, 1320.0 * 0.5, 962.2 * 0.5],
                                                [0.0, 0.0, 1.0]]),
                           (-0.12, 0.03), _pose(0.05, -0.3, [0.2, 0.0, 0.1]), 0.75, 11, "train", 97),
}


def reference_rays(W, H, K, dist, pose, time, cam_id, split):
    from datasets.immersive import ImmersiveDataset

    ds = object.__new__(ImmersiveDataset)
    ds.split = split
    ds.camera_ids = np.array([float(cam_id)])
    ds.intrinsics = np.asarray(K, dtype=np.float64)[None]
    ds.distortions = np.asarray(dist, dtype=np.float64)[None]
    ds.poses = np.asarray(pose, dtype=np.float64)[None]
    ds.times = np.array([time])
    ds.img_wh = (W, H)
    ds.num_frames = 50
    ds.use_ndc = False
    with contextlib.redirect_stdout(io.StringIO()):
        return ds.get_coords(0).float().numpy()


def main():
    _install()
    for name, (W, H, K, dist, pose, time, cam_id, split, stride) in CASES.items():
        rays = reference_rays(W, H, K, dist, pose, time, cam_id, split)
        pixels = np.arange(0, W * H, stride, dtype=np.int64)
        np.savez_compressed(os.path.join(OUT, f"rays_fisheye_{name}.npz"), rays=rays[pixels], pixels=pixels,
                            pose=np.asarray(pose, np.float32), K=np.asarray(K, np.float32),
                            distortion=np.asarray(dist, np.float32), W=W, H=H, time=np.float32(time),
                            cam_idx=np.float32(1.0 if split != "train" else cam_id))
        print(name, rays.shape, "stored", pixels.shape[0], "rows")


if __name__ == "__main__":
    main()
