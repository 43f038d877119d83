"""Golden table orders for the video datasets' per-frame pixel subsets: the pixel ids of the reference's ``all_coords``, in
table order, from the unmodified ``TechnicolorDataset.prepare_train_data`` / ``subsample`` (datasets/technicolor.py:211-269)
and ``Neural3DVideoDataset.prepare_train_data`` / ``regular_subsample`` (datasets/neural_3d.py:168-185,217-269), run on CPU
through the shim on a stand-in dataset object whose ``get_coords`` / ``get_rgb`` encode each pixel's id.

    HYPERREEL_REFERENCE=<reference checkout> python tests/golden/make_golden_subsample.py

writes ``tests/golden/reference/train_subsample.npz``: for each case ``<case>/ids`` (int64, the table's pixel ids
``view*H*W + y*W + x``), ``<case>/times`` (the views' times) and ``<case>/params``
``[n_cams, n_frames, H, W, load_full_step, subsample_keyframe_step, subsample_keyframe_frac, subsample_frac]``; ``cases`` lists
the case names and ``datasets`` their dataset.
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

from oracle import ref_shim  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference", "train_subsample.npz")

SHIPPED = (8, 4, 0.25, 0.125)          # conf/experiment/dataset/technicolor.yaml:31-34
SHIPPED_N3D = (4, 2, 0.25, 0.125)      # conf/experiment/dataset/neural_3d.yaml:32-35
OTHER = (5, 3, 0.5, 1.0 / 6.0)         # strides 2 and 6
# (name, dataset, n_cams (technicolor) or n_videos (neural_3d), frames, H, W, steps): H and W not multiples of the strides,
# and W < stride
CASES = [
    ("technicolor_shipped_13x11", "technicolor", 3, 50, 13, 11, SHIPPED),
    ("technicolor_shipped_9x5", "technicolor", 2, 50, 9, 5, SHIPPED),
    ("technicolor_other_7x10", "technicolor", 2, 50, 7, 10, OTHER),
    ("neural_3d_shipped_13x11", "neural_3d", 3, 50, 13, 11, SHIPPED_N3D),
    ("neural_3d_shipped_6x3", "neural_3d", 2, 50, 6, 3, SHIPPED_N3D),
    ("neural_3d_other_11x7", "neural_3d", 2, 50, 11, 7, OTHER),
]


def _install():
    ref_shim.install()

    def stub(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules.setdefault(name, m)
        return sys.modules[name]

    # import-only modules of datasets/base.py
    stub("iopath")
    stub("iopath.common")
    stub("iopath.common.file_io", PathManager=object, NativePathHandler=object)
    stub("omegaconf", OmegaConf=object)
    try:
        import torchvision.transforms  # noqa: F401
    except ImportError:
        stub("torchvision")
        stub("torchvision.transforms")
        sys.modules["torchvision"].transforms = sys.modules["torchvision.transforms"]
    # the dataset package without datasets/__init__.py, which imports every dataset and its dependencies
    pkg = types.ModuleType("datasets")
    pkg.__path__ = [os.path.join(ref_shim.REFERENCE_ROOT, "datasets")]
    sys.modules["datasets"] = pkg


def _pixel_column(H, W):
    return torch.arange(H * W, dtype=torch.float32)[:, None]


def technicolor_ids(n_cams, n_frames, H, W, steps):
    from datasets.technicolor import TechnicolorDataset

    ds = object.__new__(TechnicolorDataset)
    n = n_cams * n_frames
    ds.img_wh = (W, H)
    ds.num_frames = n_frames
    ds.image_paths = [f"{i:04d}.png" for i in range(n)]
    # frame-major training views, as read_meta leaves them (technicolor.py:117-123,205-209)
    ds.times = np.tile(np.linspace(0, 1, n_frames)[..., None], (1, n_cams)).reshape(-1)
    ds.load_full_step, ds.subsample_keyframe_step, ds.subsample_keyframe_frac, ds.subsample_frac = steps
    ds.keyframe_offset = 0
    ds.frame_offset = 0
    hw = H * W
    ds.get_coords = lambda idx: torch.cat([idx * hw + _pixel_column(H, W), torch.zeros(hw, 7)], -1)
    ds.get_rgb = lambda idx: (idx * hw + _pixel_column(H, W)).expand(hw, 3)
    with contextlib.redirect_stdout(io.StringIO()):
        ds.prepare_train_data()
    ids = ds.all_coords[:, 0].long()
    assert torch.equal(ds.all_rgb[:, 0].long(), ids)
    return ids.numpy(), ds.times


class _FakeVideo:
    """cv2.VideoCapture over a video of frame tokens: read() returns (True, (video index, frame index))."""

    def __init__(self, path):
        self.video = int(os.path.basename(path).split(".")[0])
        self.frame = 0

    def read(self):
        out = (True, (self.video, self.frame))
        self.frame += 1
        return out

    def release(self):
        pass


def neural_3d_ids(n_videos, n_frames, H, W, steps):
    import datasets.neural_3d as n3d

    ds = object.__new__(n3d.Neural3DVideoDataset)
    ds.img_wh = (W, H)
    ds.num_frames = n_frames
    ds.start_frame = 0
    ds.video_paths = [f"{v}.mp4" for v in range(n_videos)]
    ds.images_per_frame = n_videos
    # frame-major times of the training videos (neural_3d.py:115-117,141-150)
    ds.times = np.tile(np.linspace(0, 1, n_frames)[..., None], (1, n_videos)).reshape(-1)
    ds.load_full_step, ds.subsample_keyframe_step, ds.subsample_keyframe_frac, ds.subsample_frac = steps
    hw = H * W
    ds.get_coords = lambda video_idx: torch.zeros(hw, 8)
    # the table is video-major: view (video, frame) is view video * n_frames + frame
    ds.get_rgb = lambda tok: ((tok[0] * n_frames + tok[1]) * hw + _pixel_column(H, W)).expand(hw, 3)
    n3d.cv2 = types.SimpleNamespace(VideoCapture=_FakeVideo)
    with contextlib.redirect_stdout(io.StringIO()):
        ds.prepare_train_data()
    return ds.all_rgb[:, 0].long().numpy(), ds.times


def main():
    _install()
    out = {"cases": np.array([c[0] for c in CASES]), "datasets": np.array([c[1] for c in CASES])}
    for name, dataset, n_cams, n_frames, H, W, steps in CASES:
        fn = technicolor_ids if dataset == "technicolor" else neural_3d_ids
        ids, times = fn(n_cams, n_frames, H, W, steps)
        out[f"{name}/ids"] = ids.astype(np.int64)
        out[f"{name}/times"] = np.asarray(times, dtype=np.float64)
        out[f"{name}/params"] = np.array([n_cams, n_frames, H, W, *steps], dtype=np.float64)
        print(name, ids.shape[0], "rows of", n_cams * n_frames * H * W)
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    np.savez_compressed(OUT, **out)


if __name__ == "__main__":
    main()
