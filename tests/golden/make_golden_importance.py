"""Golden training tables of the Immersive dataset's importance subsample, from the unmodified
``ImmersiveDataset.prepare_train_data`` / ``subsample`` / ``importance_subsample`` / ``get_rgb`` (datasets/immersive.py:295-391,
575-587) run on CPU through the shim on a stand-in dataset object.  ``cv2.VideoCapture`` is replaced by an in-memory frame
source of the seeded videos of tests/importance_oracle.py (BGR, as a decoder returns them), and ``get_coords`` returns the
unmodified fisheye rays of ``ImmersiveDataset.get_coords`` (tests/golden/make_golden_fisheye.py) with a pixel-id column
inserted before the time column, so that ``coords[mask]`` carries each kept pixel's id into ``all_coords``.

    HYPERREEL_REFERENCE=<reference checkout> python tests/golden/make_golden_importance.py

writes ``tests/golden/reference/train_importance.npz``; for each case ``<case>/params`` ``[n_videos, n_frames, H, W,
load_full_step, subsample_keyframe_step, subsample_keyframe_frac, subsample_frac]``, ``<case>/seed``, ``<case>/static`` (frames
equal to their predecessor), the cameras ``<case>/{pose, K, distortion, cam_id}`` (one per video), ``<case>/times``
(frame-major, as read_meta leaves them), ``<case>/dz`` fp32 [n_videos, H*W] (the reference rays' channel 5),
``<case>/keep`` (``np.packbits(..., bitorder="little")`` of the table's pixels over all ``n_videos*n_frames*H*W`` pixels of the
video-major views) and ``<case>/counts`` (rows per view); ``cases`` lists the case names.
"""
import contextlib
import io
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from tests.golden.make_golden_fisheye import _K, _pose, reference_rays  # noqa: E402
from tests.golden.make_golden_subsample import _install  # noqa: E402
from tests.importance_oracle import video_frames  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference", "train_importance.npz")

SHIPPED = (8, 4, 0.25, 0.125)     # conf/experiment/dataset/immersive.yaml:31-34
OTHER = (5, 3, 0.5, 1.0 / 6.0)
IMM_K = (1320.0 * 0.5, 1283.7 * 0.5, 962.2 * 0.5)  # the 1280x960 training camera of make_golden_fisheye.py


def _cams(n, f, cx, cy, dist, tilt=0.0):
    return [(_K(f, cx, cy), dist, _pose(tilt + 0.05 * v, -0.1 * v, [0.1 * v, -0.05, 0.2]), 3 + 2 * v) for v in range(n)]


# name: (H, W, n_frames, steps, seed, static frames, cameras (K, (k1, k2), pose, camera id) per video)
CASES = {
    # the shipped steps on three small videos: whole, keyframe and other frames, ties at the threshold
    "shipped_3v_18x24": (18, 24, 12, SHIPPED, 1, (), _cams(3, 20.0, 11.7, 9.2, (0.05, -0.01))),
    # a camera tilted so that the ray z crosses -0.05 inside the image
    "crossing_2v_30x40": (30, 40, 6, SHIPPED, 2, (), _cams(2, 14.0, 19.6, 15.3, (0.02, 0.001), tilt=1.2)),
    # frame 2 repeats frame 1: every diff is 0 and the frame keeps nothing
    "static_1v_12x16": (12, 16, 5, SHIPPED, 3, (2,), _cams(1, 12.0, 7.9, 6.1, (0.05, -0.01))),
    # 1x3 views: num_take = round(3 * 0.125) = 0, the reference's sorted[-0] is the minimum
    "tiny_2v_1x3": (1, 3, 10, SHIPPED, 4, (), _cams(2, 2.0, 1.5, 0.5, (0.05, -0.01))),
    # other steps: full every 5th, keyframes every 3rd at 1/2, others at 1/6
    "other_2v_15x20": (15, 20, 8, OTHER, 5, (), _cams(2, 16.0, 9.8, 7.4, (0.05, -0.01))),
    # the top-left 320x240 crop of Immersive's 1280x960 training camera (same intrinsics: the crop starts at pixel (0, 0)),
    # where the fisheye is strongest
    "immersive_crop_240x320": (240, 320, 5, SHIPPED, 6, (),
                               [(_K(*IMM_K), (-0.12, 0.03), _pose(0.05, -0.3, [0.2, 0.0, 0.1]),
                                 11)]),
}


class _Frames:
    """cv2.VideoCapture over in-memory BGR frames: read() returns (True, frame)."""
    videos = {}

    def __init__(self, path):
        self.frames = _Frames.videos[path]
        self.i = 0

    def read(self):
        f = self.frames[self.i]
        self.i += 1
        return True, f

    def release(self):
        pass


def reference_table(H, W, n_frames, steps, seed, static, cams):
    import cv2
    import torchvision.transforms as T

    import datasets.immersive as imm

    n_videos = len(cams)
    rays = [reference_rays(W, H, K, dist, pose, 0.0, cam_id, "train") for K, dist, pose, cam_id in cams]
    hw = H * W
    pid = torch.arange(hw, dtype=torch.float32)[:, None]
    frames = [video_frames(seed * 1000 + v, n_frames, H, W, static) for v in range(n_videos)]
    ds = object.__new__(imm.ImmersiveDataset)
    ds.img_wh = ds._img_wh = (W, H)
    ds.transform = T.ToTensor()
    ds.num_frames = n_frames
    ds.start_frame = 0
    ds.video_paths = [f"{v}.mp4" for v in range(n_videos)]
    ds.images_per_frame = n_videos
    ds.times = np.tile(np.linspace(0, 1, n_frames)[..., None], (1, n_videos)).reshape(-1)  # immersive.py:140-141
    ds.load_full_step, ds.subsample_keyframe_step, ds.subsample_keyframe_frac, ds.subsample_frac = steps
    ds.keyframe_offset = ds.frame_offset = 0
    # rays [x 6, cam_idx, time] -> [x 6, cam_idx, pixel id, time]; prepare_train_data replaces the last column by the time
    ds.get_coords = lambda v: torch.cat([torch.from_numpy(rays[v][:, :7]), pid, torch.from_numpy(rays[v][:, 7:])], -1)
    ds.get_weights = lambda: torch.ones_like(ds.all_coords[..., :1])
    _Frames.videos = {f"{v}.mp4": [np.ascontiguousarray(fr[..., ::-1]) for fr in frames[v]] for v in range(n_videos)}
    imm.cv2 = types.SimpleNamespace(VideoCapture=_Frames, cvtColor=cv2.cvtColor, COLOR_BGR2RGB=cv2.COLOR_BGR2RGB,
                                    resize=cv2.resize, INTER_LANCZOS4=cv2.INTER_LANCZOS4, INTER_AREA=cv2.INTER_AREA,
                                    fisheye=cv2.fisheye)
    try:
        with contextlib.redirect_stdout(io.StringIO()):
            ds.prepare_train_data()
    finally:
        imm.cv2 = cv2
    # views are video-major: view (video, frame) is view video * n_frames + frame; all_coords holds them in that order
    coords, rgb = ds.all_coords, ds.all_rgb
    ids, counts, row = [], [], 0
    for v in range(n_videos):
        for f in range(n_frames):
            # a view's rows run until the pixel ids stop increasing
            start = row
            while row < coords.shape[0] and (row == start or coords[row, 7] > coords[row - 1, 7]) and \
                    float(coords[row, 8]) == float(np.float32(ds.times[f * n_videos + v])):
                row += 1
            p = coords[start:row, 7].long().numpy()
            want = frames[v][f].reshape(-1, 3)[p].astype(np.float32) / np.float32(255.0)
            assert np.array_equal(rgb[start:row].numpy(), want)
            assert np.array_equal(coords[start:row, :7].numpy(), rays[v][p, :7])
            ids.append((v * n_frames + f) * hw + p)
            counts.append(row - start)
    assert row == coords.shape[0], (row, coords.shape)
    ids = np.concatenate(ids)
    keep = np.zeros(n_videos * n_frames * hw, dtype=bool)
    keep[ids] = True
    assert np.array_equal(np.flatnonzero(keep), ids)  # row-major within each view, views in order
    dz = np.stack([r[:, 5] for r in rays]).astype(np.float32)
    return keep, np.array(counts, dtype=np.int64), dz, ds.times


def main():
    _install()
    out = {"cases": np.array(list(CASES))}
    for name, (H, W, n_frames, steps, seed, static, cams) in CASES.items():
        keep, counts, dz, times = reference_table(H, W, n_frames, steps, seed, static, cams)
        out[f"{name}/params"] = np.array([len(cams), n_frames, H, W, *steps], dtype=np.float64)
        out[f"{name}/seed"] = np.int64(seed)
        out[f"{name}/static"] = np.array(static, dtype=np.int64)
        out[f"{name}/pose"] = np.stack([np.asarray(c[2], np.float32) for c in cams])
        out[f"{name}/K"] = np.stack([np.asarray(c[0], np.float32) for c in cams])
        out[f"{name}/distortion"] = np.stack([np.asarray(c[1], np.float32) for c in cams])
        out[f"{name}/cam_id"] = np.array([c[3] for c in cams], dtype=np.float32)
        out[f"{name}/times"] = np.asarray(times, dtype=np.float64)
        out[f"{name}/dz"] = dz
        out[f"{name}/keep"] = np.packbits(keep, bitorder="little")
        out[f"{name}/counts"] = counts
        print(name, int(counts.sum()), "rows of", keep.shape[0], "per view", counts.tolist()[:12], "dz >= -0.05:",
              int((dz >= np.float32(-0.05)).sum()), "within 4e-6:", int((np.abs(dz + 0.05) <= 4e-6).sum()))
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    np.savez_compressed(OUT, **out)


if __name__ == "__main__":
    main()
