"""Golden render-split camera paths (the poses and times of the reference's validation / render_only videos), from the
unmodified ``prepare_render_data`` of the Technicolor, Neural-3D, Immersive and DoNeRF datasets run on CPU through the shim on
stand-in dataset objects that hold synthetic rigs shaped like each dataset's.

    HYPERREEL_REFERENCE=<reference checkout> python tests/golden/make_golden_video_path.py

writes ``tests/golden/video_path.npz``: per case ``<case>/poses_in`` [N, 3, 4] fp64 and ``<case>/bounds`` (the dataset facts
prepare_render_data reads), ``<case>/params`` int64 (num_frames, supersample, interpolate, interpolate_time), then the video
as the reference's get_coords consumes it: ``<case>/poses`` [F, 3, 4] fp32 (torch.FloatTensor(pose)) and ``<case>/times`` [F]
fp32 (``ones * time``).
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from tests.golden.make_golden_subsample import _install  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))


def _rot(rx, ry, rz):
    cx, sx, cy, sy, cz, sz = np.cos(rx), np.sin(rx), np.cos(ry), np.sin(ry), np.cos(rz), np.sin(rz)
    return (np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]]) @ np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
            @ np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]]))


def _rig(centres, angles, num_frames, drift):
    """num_frames copies of a rig (cameras at `centres` with small rotations `angles`), frame-major, the rig moved by
    frame * drift (translation, rotation about y) as a handheld or re-calibrated rig would."""
    out = []
    for f in range(num_frames):
        R0 = _rot(0.0, drift[3] * f, 0.0)
        for c, a in zip(centres, angles):
            R = R0 @ _rot(*a)
            t = R0 @ np.asarray(c, np.float64) + f * np.asarray(drift[:3], np.float64)
            out.append(np.concatenate([R, t[:, None]], 1))
    return np.stack(out, 0)


def _cases():
    rng = np.random.default_rng(7)
    # Technicolor: a 4x4 planar rig, NDC-corrected scale (bounds after correct_poses_bounds)
    tc = [[(i - 1.5) * 0.12, (j - 1.5) * 0.12, 0.0] for j in range(4) for i in range(4)]
    tc_a = [tuple(rng.normal(0, 0.01, 3)) for _ in tc]
    # Neural-3D: ~20 cameras on a frontal arc
    n3 = [[1.5 * np.sin(a), 0.1 * np.cos(3 * a), 1.5 * (1 - np.cos(a))] for a in np.linspace(-0.6, 0.6, 19)]
    n3_a = [(0.0, -a, 0.0) for a in np.linspace(-0.6, 0.6, 19)]
    # Immersive: 46 cameras on a hemisphere cap looking outward (z back)
    im, im_a = [], []
    for k in range(46):
        az, el = 2 * np.pi * k / 46, 0.15 + 0.35 * (k % 3) / 2
        im.append([0.3 * np.sin(az) * np.cos(el), 0.3 * np.sin(el), 0.3 * np.cos(az) * np.cos(el) - 0.3])
        im_a.append((el * 0.5, az * 0.1, 0.0))
    # name: (reference class, module, poses, bounds, num_frames, supersample, interpolate, interpolate_time)
    return {
        "technicolor_video": ("TechnicolorDataset", "technicolor", _rig(tc, tc_a, 5, (0.0, 0.0, 0.0, 0.0)),
                              np.array([0.95, 12.0]), 5, 2, False, False),
        "technicolor_still": ("TechnicolorDataset", "technicolor", _rig(tc, tc_a, 1, (0.0, 0.0, 0.0, 0.0)),
                              np.array([0.95, 12.0]), 1, 2, False, False),
        "neural_3d_video": ("Neural3DVideoDataset", "neural_3d", _rig(n3, n3_a, 4, (0.01, -0.005, 0.002, 0.01)),
                            np.array([1.2, 80.0]), 4, 2, False, False),
        "immersive_video": ("ImmersiveDataset", "immersive", _rig(im, im_a, 3, (0.02, 0.0, -0.01, 0.02)),
                            np.array([0.4, 100.0]), 3, 3, False, True),
        "immersive_interpolate": ("ImmersiveDataset", "immersive", _rig(im[:5], im_a[:5], 1, (0.0, 0.0, 0.0, 0.0)),
                                  np.array([0.4, 100.0]), 1, 3, True, False),
        "donerf_path": ("DONeRFDataset", "donerf", _rig([[0.1 * k, 0.02 * k, -0.05 * k] for k in range(6)],
                                                        [(0.01 * k, 0.05 * k, 0.0) for k in range(6)], 1, (0, 0, 0, 0)),
                        np.array([0.5, 30.0]), 1, 1, False, False),
    }


def reference_path(cls_name, module, poses, bounds, num_frames, supersample, interpolate, interpolate_time):
    import importlib

    import torch

    cls = getattr(importlib.import_module(f"datasets.{module}"), cls_name)
    ds = object.__new__(cls)
    ds.split = "render"
    ds.poses = np.copy(poses)
    ds.bounds = np.copy(bounds)
    ds.num_frames = num_frames
    ds.render_supersample = supersample
    ds.render_interpolate = interpolate
    ds.render_interpolate_time = interpolate_time
    ds.times = np.zeros(len(poses))
    cls.prepare_render_data(ds)
    out_poses = np.stack([torch.FloatTensor(ds.poses[i]).numpy() for i in range(len(ds.poses))], 0)
    if cls_name == "DONeRFDataset":  # a static dataset: its rays have no time column
        out_times = np.zeros(len(ds.poses), np.float32)
    else:
        out_times = np.array([(torch.ones(1) * ds.times[i]).numpy()[0] for i in range(len(ds.poses))], np.float32)
    return out_poses, out_times


def main():
    _install()
    arrays = {}
    for name, (cls_name, module, poses, bounds, nf, ss, interp, interp_t) in _cases().items():
        p, t = reference_path(cls_name, module, poses, bounds, nf, ss, interp, interp_t)
        arrays[f"{name}/poses_in"] = poses
        arrays[f"{name}/bounds"] = bounds
        arrays[f"{name}/params"] = np.array([nf, ss, int(interp), int(interp_t)], np.int64)
        arrays[f"{name}/poses"] = p
        arrays[f"{name}/times"] = t
        print(name, poses.shape, "->", p.shape, "times", t[:4], "...")
    np.savez_compressed(os.path.join(OUT, "video_path.npz"), **arrays)


if __name__ == "__main__":
    main()
