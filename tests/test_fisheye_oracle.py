"""Fisheye cameras on the host: the oracle against the reference goldens (tests/golden/rays_fisheye_*.npz, from the unmodified
ImmersiveDataset.get_coords), its undistortion against cv2 itself when cv2 is installed, and Camera(distortion=...)."""
import glob
import math
import os

import numpy as np
import pytest
import torch

import hyperreel_b200 as hb
from oracle.rays_oracle import ray_directions
from tests.fisheye_oracle import fisheye_coords_from_camera, fisheye_undistort

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
FISHEYE = {os.path.basename(p)[len("rays_fisheye_"):-4]: p for p in sorted(glob.glob(os.path.join(GOLDEN, "rays_fisheye_*.npz")))}


def load_fisheye(name):
    g = np.load(FISHEYE[name])
    return {k: g[k] for k in g.files}


def oracle_rays(g):
    return fisheye_coords_from_camera(g["pose"], g["K"], int(g["W"]), int(g["H"]), g["distortion"], float(g["time"]),
                                      float(g["cam_idx"]), pixels=g["pixels"]).numpy()


def test_fisheye_goldens_cover_the_edge_cases():
    assert set(FISHEYE) == {"mild_40x30", "strong_48x36", "centre_21x15", "wide_40x30", "immersive_1280x960"}
    theta_d, sentinel = {}, {}
    for n in FISHEYE:
        g = load_fisheye(n)
        xy = ray_directions(int(g["H"]), int(g["W"]), torch.from_numpy(g["K"]), centered_pixels=True).reshape(-1, 3)[:, :2]
        xy = xy[torch.from_numpy(g["pixels"])].numpy()
        theta_d[n] = np.hypot(xy[:, 0].astype(np.float64), xy[:, 1].astype(np.float64))
        sentinel[n] = int((fisheye_undistort(xy, *g["distortion"])[:, 0] == -1e6).sum())
    assert sentinel["mild_40x30"] == 0 and sentinel["strong_48x36"] > 100  # OpenCV's (-1e6, -1e6) at the corners
    assert (theta_d["centre_21x15"] == 0).sum() == 1
    assert (theta_d["wide_40x30"] > math.pi / 2).sum() > 100
    g = load_fisheye("centre_21x15")
    assert np.array_equal(g["pose"][:, :3], np.eye(3, dtype=np.float32))
    assert np.abs(g["rays"][7 * 21 + 10, 3:6] - [0.0, 0.0, -1.0]).max() == 0.0  # theta_d = 0: straight down the axis
    g = load_fisheye("immersive_1280x960")
    assert (int(g["W"]), int(g["H"])) == (1280, 960) and g["pixels"].shape[0] == g["rays"].shape[0] > 10000


@pytest.mark.parametrize("name", list(FISHEYE))
def test_fisheye_oracle_matches_reference_golden(name):
    g = load_fisheye(name)
    r = oracle_rays(g)
    assert r.shape == g["rays"].shape
    assert np.abs(r - g["rays"]).max() <= 2e-6 * max(1.0, np.abs(g["rays"]).max())


def _edge_points():
    t = np.float32(np.pi / 2)
    return np.array([[0, 0], [-0.0, 0.0], [1e-9, 0], [1e-8, 0], [2e-8, 0], [0, -1e-8], [t, 0], [0, -t],
                     [np.nextafter(t, np.float32(3)), 0], [1.0, 1.0], [-3, 4], [100, -100], [0.5, -0.25]], dtype=np.float32)


@pytest.mark.parametrize("k", [(0.0, 0.0), (0.05, -0.01), (-0.4, 0.0), (-0.4, 0.05), (0.3, 0.2), (-0.12, 0.03),
                               (1e-3, -2.5)])
def test_fisheye_undistort_is_cv2_bit_for_bit(k):
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(abs(hash(k)) % 2 ** 32)
    pts = np.concatenate([_edge_points(), rng.uniform(-2.5, 2.5, (6000, 2)).astype(np.float32),
                          rng.normal(0.0, 0.3, (2000, 2)).astype(np.float32)])
    kk = np.array([k[0], k[1], 0.0, 0.0]).astype(np.float32)
    want = cv2.fisheye.undistortPoints(pts[:, None], np.eye(3, dtype=np.float32), kk)[:, 0]
    assert np.array_equal(fisheye_undistort(pts, k[0], k[1]), want)


def _camera(**kw):
    return hb.Camera(pose=[[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0]], K=[[50, 0, 20], [0, 50, 15], [0, 0, 1]], width=40,
                     height=30, **kw)


def test_camera_distortion_fills_the_record():
    c = _camera().to_c()
    assert c.fisheye == 0 and c.k1 == 0.0 and c.k2 == 0.0
    c = _camera(distortion=(0.1, -0.3)).to_c()
    assert c.fisheye == 1
    assert (c.k1, c.k2) == (float(np.float32(0.1)), float(np.float32(-0.3)))
    c = _camera(distortion=np.array([0.0, 0.0])).to_c()  # (0, 0) is a fisheye, not the pinhole
    assert c.fisheye == 1 and (c.k1, c.k2) == (0.0, 0.0)


@pytest.mark.parametrize("bad", [(float("nan"), 0.0), (0.0, float("inf")), (-float("inf"), 0.0), (1e300, 0.0), (0.1,),
                                 (0.1, 0.2, 0.3)])
def test_camera_distortion_refuses_bad_coefficients(bad):
    with pytest.raises(ValueError):
        _camera(distortion=bad)
    cam = _camera()
    cam.distortion = bad  # set after construction: to_c refuses it too
    with pytest.raises(ValueError):
        cam.to_c()
