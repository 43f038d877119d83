"""The views of a scene directory as the reference's dataset loaders build them: the Technicolor (``name: technicolor``,
datasets/technicolor.py), Neural-3D (``neural_3d``, datasets/neural_3d.py), Immersive (``immersive``, datasets/immersive.py)
and DoNeRF (``donerf``, datasets/donerf.py) datasets.

``dataset_cameras(dataset_cfg, root, split)`` reads the dataset's pose files as its ``read_meta`` does, selects the split's
views with the config's ``val_set`` / ``val_skip`` / ``val_all`` rules, and returns them as ``Camera``s in the order the
reference's split visits them, with the ground-truth source of each view and the dataset facts the model constructors read
(``DatasetViews``).  The pose arithmetic is the reference's, in float64 numpy; each value is rounded to float32 where the
reference's ``get_coords`` makes a float32 tensor of it (``torch.FloatTensor(pose)``, ``ones * time``).  Rays are generated
from the cameras on the device (``generate_rays``, ``DeviceRayBatches``); images and videos are decoded by the caller.

The ``render`` split's path is ``spiral_path`` (camera.py).  What the restatement does not carry raises
``UnsupportedPipeline`` naming the config key; see ``dataset_cameras``.
"""
from __future__ import annotations

import csv
import dataclasses
import glob
import json
import os
from dataclasses import dataclass
from typing import List, NamedTuple, Optional, Tuple

import numpy as np

from .camera import Camera, _average_poses, spiral_path
from .signature import UnsupportedPipeline

SPLITS = ("train", "val", "test", "render")
DATASETS = ("technicolor", "neural_3d", "immersive", "donerf")


class FrameSource(NamedTuple):
    """Where a view's ground truth comes from: an image file (``frame`` None) or frame ``frame`` (0-based, counted from
    the start of the file) of a video."""
    path: str
    frame: Optional[int]


@dataclass
class DatasetViews:
    """One split of a dataset.  ``cameras`` in the reference's split order; ``frames[i]`` is the ground truth of
    ``cameras[i]`` (empty for the render split, which has none); ``facts`` the values of the reference's training dataset
    that the model constructors read (``LightfieldModel(cfg, dataset=facts)``).  ``rgba``: the frames are RGBA, composited
    over white (DoNeRF).  ``crop``: the render split's ``render_params.crop`` window ``(y0, y1, x0, x1)`` of each frame
    (``crop_batch``), or None."""
    split: str
    cameras: List[Camera]
    frames: List[FrameSource]
    facts: dict
    rgba: bool = False
    crop: Optional[Tuple[int, int, int, int]] = None

    @property
    def times(self) -> np.ndarray:
        return np.array([c.time for c in self.cameras], dtype=np.float32)


def _get(cfg, key, default=None):
    if cfg is None:
        return default
    if isinstance(cfg, dict):
        return cfg.get(key, default)
    return getattr(cfg, key, default)


def _has(cfg, key) -> bool:
    return cfg is not None and key in cfg


def _f32(v) -> float:
    return float(np.float32(v))


def _homo(p34):
    h = np.eye(4)
    h[:3] = p34
    return h


def _center_poses(poses):  # utils/pose_utils.py:48-59
    last = np.tile(np.array([0, 0, 0, 1]), (len(poses), 1, 1))
    return (np.linalg.inv(_homo(_average_poses(poses))) @ np.concatenate([poses, last], 1))[:, :3]


def _center_poses_with(poses, train_poses):  # utils/pose_utils.py:62-77
    last = np.tile(np.array([0, 0, 0, 1]), (len(poses), 1, 1))
    return (np.linalg.inv(_homo(_average_poses(train_poses))) @ np.concatenate([poses, last], 1))[:, :3]


def _center_poses_with_rotation_only(poses, train_poses):  # utils/pose_utils.py:80-91
    avg = np.eye(4)
    avg[:3, :3] = _average_poses(train_poses)[:3, :3]
    last = np.tile(np.array([0, 0, 0, 1]), (len(poses), 1, 1))
    return (np.linalg.inv(avg) @ np.concatenate([poses, last], 1))[:, :3]


def _correct_poses_bounds(poses, bounds, flip=True):
    """correct_poses_bounds(poses, bounds, flip, center=True) (utils/pose_utils.py:230-255): the "down right back" to "right
    up back" column swap with ``flip``, positions and bounds scaled by 1 / (0.75 * bounds.min()), recentred."""
    if flip:
        poses = np.concatenate([poses[..., 1:2], -poses[..., :1], poses[..., 2:4]], -1)
    poses = np.array(poses, dtype=np.float64)
    bounds = np.array(bounds, dtype=np.float64)
    scale = bounds.min() * 0.75
    bounds /= scale
    poses[..., :3, 3] /= scale
    return _center_poses(poses), bounds


def _flip_yz(pose):  # pose_pre @ pose @ pose_pre (technicolor.py:110-114, immersive.py:121-124)
    pre = np.eye(4)
    pre[1, 1] *= -1
    pre[2, 2] *= -1
    return pre @ pose @ pre


def _split_len(n: int, split: str, dcfg) -> int:
    """BaseDataset.__len__ (datasets/base.py:229-243): the validation loop visits min(val_num, n) views, the render loop
    min(render_params.max_frames, n) when max_frames > 0."""
    if split == "val":
        return min(int(_get(dcfg, "val_num")), n)
    if split == "render":
        m = int(_get(_get(dcfg, "render_params", {}), "max_frames", 0) or 0)
        return min(m, n) if m > 0 else n
    return n


def _refuse_options(dcfg, name: str, split: str) -> None:
    for s in SPLITS:
        if isinstance(_get(dcfg, s, None), dict):
            raise UnsupportedPipeline(f"dataset_cameras: a per-split '{s}' section of the dataset config is not supported")
    wh = _get(dcfg, "img_wh", None)
    if wh is None or isinstance(wh, str) or len(wh) != 2:
        raise UnsupportedPipeline(f"dataset_cameras: 'img_wh' must be [W, H], got {wh!r} (the 'downsample' path is not "
                                  "supported)")
    if split in ("val", "test") and float(_get(dcfg, "val_crop", 1.0)) < 1.0:
        raise UnsupportedPipeline("dataset_cameras: 'val_crop' < 1 scores a crop of each held-out view, which is not "
                                  "supported")
    if name in ("neural_3d", "immersive") and bool(_get(dcfg, "val_all", False)) and list(_get(dcfg, "val_set", []) or []):
        raise UnsupportedPipeline(f"dataset_cameras: {name} 'val_all' with a non-empty 'val_set' pairs the reference's "
                                  "views with the wrong videos (its video list keeps the held-out video)")


def _require_ndc_focal(cameras, K_ndc, name):
    """The device's NDC step scales by the camera's own focal lengths; the reference scales every view by the dataset's
    first camera's (self.K).  A view whose float32 fx or fy differs is refused."""
    k = np.asarray(K_ndc, dtype=np.float32)
    for i, c in enumerate(cameras):
        if c.use_ndc and (c.K[0, 0] != k[0, 0] or c.K[1, 1] != k[1, 1]):
            raise UnsupportedPipeline(f"dataset_cameras: {name} 'use_ndc' with view {i}'s focal length differing from the "
                                      "first camera's (the reference's NDC focal) is not supported")


def _camera(pose, K, W, H, time, cam_idx, use_ndc, near, distortion=None) -> Camera:
    return Camera(pose=np.asarray(pose, dtype=np.float64)[:3, :4].astype(np.float32),
                  K=np.asarray(K, dtype=np.float64).astype(np.float32), width=int(W), height=int(H), time=_f32(time),
                  cam_idx=_f32(cam_idx), centered_pixels=True, use_ndc=bool(use_ndc), ndc_near=_f32(near),
                  distortion=distortion)


def _render_views(name, template, poses, bounds, num_frames, dcfg):
    rp = _get(dcfg, "render_params", {}) or {}
    return spiral_path(name, template, poses, bounds, num_frames=num_frames, supersample=int(_get(rp, "supersample", 1)),
                       interpolate=bool(_get(rp, "interpolate", False)),
                       interpolate_time=bool(_get(rp, "interpolate_time", False)))[0]


def _crop(dcfg, W, H):
    """crop_batch's window for render_params.crop < 1 (datasets/base.py:339-360)."""
    crop = float(_get(_get(dcfg, "render_params", {}) or {}, "crop", 1.0))
    if crop >= 1.0:
        return None
    dW, dH = int(W // 2 * crop), int(H // 2 * crop)
    return (H // 2 - dH, H // 2 + dH + 1, W // 2 - dW, W // 2 + dW + 1)


def _video_frames(dcfg):
    num_frames = int(_get(dcfg, "num_frames", 1))
    start_frame = int(_get(dcfg, "start_frame", 1))
    keyframe_step = int(_get(dcfg, "keyframe_step", 1))
    num_keyframes = int(_get(dcfg, "num_keyframes", num_frames // keyframe_step))
    return num_frames, start_frame, num_keyframes


# ---------------------------------------------------------------------------------------------------------- Technicolor

# read_meta's bounds per collection (datasets/technicolor.py:125-153)
_TECHNICOLOR_BOUNDS = {"painter": (1.75, 10.0), "trains": (0.65, 10.0), "theater": (0.65, 10.0), "fabien": (0.35, 2.0),
                       "birthday": (1.75, 10.0)}


def read_technicolor_cameras(path: str, W: int, H: int):
    """cameras_parameters.txt as TechnicolorDataset.read_meta reads it (datasets/technicolor.py:87-115): one row per
    camera after a header, ``f cx cy aspect _ qw qx qy qz tx ty tz`` at 2048 x 1088; K scaled to W x H, the pose the
    inverse of the world-to-camera rotation (scipy quaternion, x y z w) and translation, flipped to y up / z back.
    Returns (intrinsics [n, 3, 3], poses [n, 3, 4]) fp64."""
    from scipy.spatial.transform import Rotation

    intrinsics, poses = [], []
    with open(path, "r") as f:
        for idx, row in enumerate(csv.reader(f, delimiter=" ")):
            if idx == 0:
                continue
            row = [float(c) for c in row if c.strip() != ""]
            if len(row) < 12:
                raise ValueError(f"{path}: row {idx} holds {len(row)} numbers, 12 are needed")
            K = np.eye(3)
            K[0, 0] = row[0] * W / 2048
            K[0, 2] = row[1] * W / 2048
            K[1, 1] = row[3] * row[0] * H / 1088
            K[1, 2] = row[2] * H / 1088
            intrinsics.append(K)
            R = Rotation.from_quat([row[6], row[7], row[8], row[5]]).as_matrix()
            pose = np.eye(4)
            pose[:3, :3] = R.T
            pose[:3, -1] = -R.T @ np.array(row[-3:]).T
            poses.append(_flip_yz(pose)[:3, :4])
    return np.stack(intrinsics), np.stack(poses)


def _technicolor(dcfg, root, split):
    W, H = (int(v) for v in _get(dcfg, "img_wh"))
    use_ndc, correct = bool(_get(dcfg, "use_ndc", False)), bool(_get(dcfg, "correct_poses", False))
    num_frames, start_frame, num_keyframes = _video_frames(dcfg)
    rows, cols = int(_get(dcfg, "lightfield_rows")), int(_get(dcfg, "lightfield_cols"))
    ipf = rows * cols
    names = sorted(os.listdir(os.path.join(root, "images")))[ipf * start_frame:ipf * (start_frame + num_frames)]
    num_frames = len(names) // ipf
    if num_frames < 1 or len(names) != num_frames * ipf:
        raise ValueError(f"dataset_cameras: {os.path.join(root, 'images')} holds {len(names)} images from frame "
                         f"{start_frame}, not whole frames of {ipf} views")
    K1, P1 = read_technicolor_cameras(os.path.join(root, "cameras_parameters.txt"), W, H)
    if len(P1) != ipf:
        raise ValueError(f"dataset_cameras: cameras_parameters.txt holds {len(P1)} cameras, lightfield_rows x "
                         f"lightfield_cols is {ipf}")
    intrinsics = np.stack([K1] * num_frames).reshape(-1, 3, 3)
    poses = np.stack([P1] * num_frames).reshape(-1, 3, 4)
    times = np.tile(np.linspace(0, 1, num_frames)[..., None], (1, ipf)).reshape(-1)
    collection = _get(dcfg, "collection")
    near, far = _TECHNICOLOR_BOUNDS.get(collection, (0.65, 10.0))
    if collection == "birthday" and len(names) > 377:  # the broken file (technicolor.py:145-150)
        names[377], poses[377], intrinsics[377], times[377] = names[361], poses[361], intrinsics[361], times[361]
    bounds = np.array([near, far])
    if use_ndc or correct:
        poses, bounds = _correct_poses_bounds(np.copy(poses), bounds, flip=False)
    near, far = bounds.min() * 0.95, bounds.max() * 1.05

    # held-out views (technicolor.py:168-209)
    val_all = bool(_get(dcfg, "val_all", False))
    val_set = _get(dcfg, "val_set", [])
    val_set = [] if val_set is None else val_set
    n = len(names)
    if isinstance(val_set, str):
        if val_set != "lightfield":
            raise UnsupportedPipeline(f"dataset_cameras: technicolor 'val_set' {val_set!r} is not a list or 'lightfield'")
        step = int(_get(dcfg, "lightfield_step"))
        val_pairs = [[int(v) for v in p] for p in (_get(dcfg, "val_pairs", []) or [])]
        val_all = (step == 1 and len(val_pairs) == 0) or val_all
        val_indices = []
        for row in range(rows):
            for col in range(cols):
                idx = row * rows + col  # as written: rows, not cols
                if (row % step != 0 or col % step != 0 or [row, col] in val_pairs) and not val_all:
                    val_indices += [frame * ipf + idx for frame in range(num_frames)]
    elif len(val_set) > 0 or val_all:
        val_indices = [int(i) for i in val_set]
    elif _get(dcfg, "val_skip") != "inf":
        val_indices = list(range(0, n, min(n, int(_get(dcfg, "val_skip")))))
    else:
        val_indices = []
    if any(not 0 <= i < n for i in val_indices):
        raise ValueError(f"dataset_cameras: technicolor held-out views {val_indices} outside the {n} views")
    train_indices = [i for i in range(n) if i not in val_indices]
    if val_all:
        val_indices = list(train_indices)
    facts = {"num_frames": num_frames, "num_keyframes": num_keyframes, "near": float(near), "far": float(far),
             "val_all": val_all}

    def cam_idx(i, held_out):  # get_coords (technicolor.py:360-364)
        return 3 if held_out and not val_all else i % ipf

    if split == "render":
        template = _camera(poses[0], intrinsics[0], W, H, 0.0, 3, use_ndc, near)
        cams = _render_views("technicolor", template, poses, bounds, num_frames, dcfg)
        cams = [dataclasses.replace(c, cam_idx=_f32(cam_idx(i, True))) for i, c in enumerate(cams)]
        return cams, [], facts
    sel = train_indices if split == "train" else val_indices
    cams = [_camera(poses[j], intrinsics[j], W, H, times[j], cam_idx(i, split != "train"), use_ndc, near)
            for i, j in enumerate(sel)]
    _require_ndc_focal(cams, intrinsics[0], "technicolor")
    frames = [FrameSource(os.path.join(root, "images", names[j]), None) for j in sel]
    return cams, frames, facts


# ------------------------------------------------------------------------------------------------ Neural-3D, Immersive

def _video_train(poses, times, camera_ids, paths, val_indices, start_frame, num_frames, make):
    """prepare_train_data's views of a multi-video dataset (neural_3d.py:217-296, immersive.py:323-402): video-major, video v
    at the pose, intrinsics and camera id of the v-th training entry, each frame's time from the frame-major time table."""
    train_indices = [i for i in range(len(poses)) if i not in val_indices]
    nv = len(paths)
    cams, frames = [], []
    for v in range(nv):
        for f in range(num_frames):
            cams.append(make(train_indices[v], times[train_indices[f * nv + v]], camera_ids[train_indices[v]]))
            frames.append(FrameSource(paths[v], start_frame + f))
    return cams, frames


def _held_out(val_indices, times, paths, start_frame, make):
    """The held-out views in order, cam_idx 1, each one's ground truth get_rgb_one's frame (neural_3d.py:426-451,
    immersive.py:589-614): video ``idx % n_videos``, frame ``idx // n_videos`` of the split's video list."""
    cams = [make(j, times[j], 1) for j in val_indices]
    return cams, [FrameSource(paths[i % len(paths)], start_frame + i // len(paths)) for i in range(len(cams))]


def _neural_3d(dcfg, root, split):
    W, H = (int(v) for v in _get(dcfg, "img_wh"))
    use_ndc = bool(_get(dcfg, "use_ndc", False))
    num_frames, start_frame, num_keyframes = _video_frames(dcfg)
    pb = np.load(os.path.join(root, "poses_bounds.npy"))
    video_paths = sorted(glob.glob(os.path.join(root, "*.mp4")))
    ipf = len(video_paths)
    if pb.ndim != 2 or pb.shape[1] != 17 or pb.shape[0] != ipf or ipf < 1:
        raise ValueError(f"dataset_cameras: poses_bounds.npy is {pb.shape}, one row of 17 per video is needed "
                         f"({ipf} videos)")
    p35 = pb[:, :15].reshape(-1, 3, 5)
    h, w, focal = p35[0, :, -1]
    K = np.eye(3)
    K[0, 0] = focal * W / w
    K[0, 2] = (w / 2.0) * W / w
    K[1, 1] = focal * H / h
    K[1, 2] = (h / 2.0) * H / h
    poses, bounds = _correct_poses_bounds(p35, pb[:, -2:], flip=True)
    near, far = bounds.min() * 0.95, bounds.max() * 1.05
    val_all = bool(_get(dcfg, "val_all", False))
    val_set = [int(i) for i in (_get(dcfg, "val_set", []) or [])]
    if any(not 0 <= i < ipf for i in val_set):
        raise ValueError(f"dataset_cameras: neural_3d 'val_set' {val_set} outside the {ipf} videos")
    if len(val_set) > 1 and num_frames > 1:
        raise UnsupportedPipeline("dataset_cameras: neural_3d 'val_set' with more than one video: the reference scores "
                                  "each held-out view against another video's frame (get_rgb_one reads them frame-major)")
    facts = {"num_frames": num_frames, "num_keyframes": num_keyframes, "near": float(near), "far": float(far),
             "depth_range": [float(near * 2.0), float(far)], "total_images_per_frame": ipf, "val_all": val_all}
    if split == "render":
        template = _camera(poses[0], K, W, H, 0.0, 1, use_ndc, near)
        cams = _render_views("neural_3d", template, np.stack([poses] * num_frames).reshape(-1, 3, 4), bounds,
                             num_frames, dcfg)
        return cams, [], facts
    poses = np.stack([poses] * num_frames).reshape(-1, 3, 4)
    times = np.tile(np.linspace(0, 1, num_frames)[..., None], (1, ipf)).reshape(-1)
    camera_ids = np.tile(np.linspace(0, ipf - 1, ipf)[None, :], (num_frames, 1)).reshape(-1)
    val_indices = [frame * ipf + i for i in val_set for frame in range(num_frames)]

    def make(j, t, cid):
        return _camera(poses[j], K, W, H, t, cid, use_ndc, near)

    if split == "train":
        paths = video_paths if val_all else [p for i, p in enumerate(video_paths) if i not in val_set]
        return (*_video_train(poses, times, camera_ids, paths, val_indices, start_frame, num_frames, make), facts)
    if val_all:
        val_indices = [i for i in range(len(poses)) if i not in val_indices]
    return (*_held_out(val_indices, times, video_paths if val_all else [video_paths[i] for i in val_set], start_frame,
                       make), facts)


# read_meta's bounds per collection (datasets/immersive.py:145-208), the last if / elif chain; 01_Welder and 02_Flames set
# theirs in separate ifs before it, which its else branch then overwrites
_IMMERSIVE_BOUNDS = {"04_Truck": (0.5, 10.0, None), "05_Horse": (0.5, 45.0, None), "07_Car": (0.5, 50.0, None),
                     "09_Alexa_Meade_Exhibit": (0.5, 30.0, None), "10_Alexa_Meade_Face_Paint_1": (0.25, 6.0, 0.5),
                     "11_Alexa_Meade_Face_Paint_2": (0.25, 6.0, 0.5), "12_Cave": (0.5, 20.0, None)}


def read_immersive_cameras(path: str, W: int, H: int):
    """models.json as ImmersiveDataset.read_meta reads it (datasets/immersive.py:81-130): K scaled from 2560 x 1920 to
    W x H, the first two radial distortion coefficients, the pose [R(orientation)^T | position] flipped to y up / z back.
    Returns (names, intrinsics [n, 3, 3], distortions [n, 2], poses [n, 3, 4]), fp64."""
    from scipy.spatial.transform import Rotation

    with open(path, "r") as f:
        meta = json.load(f)
    names, intrinsics, distortions, poses = [], [], [], []
    for camera in meta:
        wf, hf = W / 2560.0, H / 1920.0
        intrinsics.append(np.array([[camera["focal_length"] * wf, 0.0, camera["principal_point"][0] * wf],
                                    [0.0, camera["focal_length"] * hf, camera["principal_point"][1] * hf],
                                    [0.0, 0.0, 1.0]]))
        distortions.append(np.array(camera["radial_distortion"])[:2])
        pose = np.eye(4)
        pose[:3, :3] = Rotation.from_rotvec(camera["orientation"]).as_matrix().T
        pose[:3, -1] = np.array(camera["position"])
        poses.append(_flip_yz(pose)[:3, :4])
        names.append(camera["name"])
    return names, np.stack(intrinsics), np.stack(distortions), np.stack(poses)


def _immersive(dcfg, root, split):
    W, H = (int(v) for v in _get(dcfg, "img_wh"))
    use_ndc, correct = bool(_get(dcfg, "use_ndc", False)), bool(_get(dcfg, "correct_poses", False))
    num_frames, start_frame, num_keyframes = _video_frames(dcfg)
    names, K1, D1, P1 = read_immersive_cameras(os.path.join(root, "models.json"), W, H)
    video_paths = [os.path.join(root, nm + ".mp4") for nm in names]
    ipf = len(names)
    val_idx = max((i for i, nm in enumerate(names) if nm == "camera_0001"), default=None)
    val_set = list(_get(dcfg, "val_set", []) or [])
    if val_idx is None and (val_set or use_ndc or correct):
        raise ValueError("dataset_cameras: immersive 'val_set', 'use_ndc' and 'correct_poses' need the camera named "
                         "camera_0001 in models.json (the held-out view and the centre)")
    intrinsics = np.stack([K1] * num_frames).reshape(-1, 3, 3)
    distortions = np.stack([D1] * num_frames).reshape(-1, 2)
    poses = np.stack([P1] * num_frames).reshape(-1, 3, 4)
    times = np.tile(np.linspace(0, 1, num_frames)[..., None], (1, ipf)).reshape(-1)
    camera_ids = np.tile(np.linspace(0, ipf - 1, ipf)[None, :], (num_frames, 1)).reshape(-1)
    near, far, dr0 = _IMMERSIVE_BOUNDS.get(_get(dcfg, "collection"), (0.5, 10.0, None))
    depth_range = [dr0 if dr0 is not None else near * 2.0, far]
    bounds = np.array([near, far])
    if use_ndc or correct:
        poses = _center_poses_with(np.copy(poses), P1[val_idx][None])
    near, far = bounds.min() * 0.95, bounds.max() * 1.05
    val_all = bool(_get(dcfg, "val_all", False))
    facts = {"num_frames": num_frames, "num_keyframes": num_keyframes, "near": float(near), "far": float(far),
             "depth_range": [float(v) for v in depth_range], "val_all": val_all}
    if split == "render":
        K = intrinsics[0].astype(np.float32)  # torch.FloatTensor(intrinsics[0]), fx and fy * 0.75 in fp32
        K[0, 0] *= np.float32(0.75)
        K[1, 1] *= np.float32(0.75)
        template = _camera(poses[0], K, W, H, 0.0, 1, use_ndc, near)
        _require_ndc_focal([template], intrinsics[0], "immersive")  # the reference's NDC keeps the unscaled focal
        return _render_views("immersive", template, poses, bounds, num_frames, dcfg), [], facts
    val_indices = [frame * ipf + val_idx for frame in range(num_frames)] if val_set else []

    def make(j, t, cid):
        return _camera(poses[j], intrinsics[j], W, H, t, cid, use_ndc, near, distortion=tuple(distortions[j]))

    held_one = bool(val_set) and not val_all
    if split == "train":
        paths = [p for i, p in enumerate(video_paths) if i != val_idx] if held_one else video_paths
        cams, frames = _video_train(poses, times, camera_ids, paths, val_indices, start_frame, num_frames, make)
    else:
        if val_all:
            val_indices = [i for i in range(len(poses)) if i not in val_indices]
        cams, frames = _held_out(val_indices, times, [video_paths[val_idx]] if held_one else video_paths, start_frame, make)
    _require_ndc_focal(cams, intrinsics[0], "immersive")
    return cams, frames, facts


# ---------------------------------------------------------------------------------------------------------------- DoNeRF

_DONERF_FILES = {"train": "transforms_train.json", "val": "transforms_val.json", "test": "transforms_test.json",
                 "render": "cam_path_pan.json"}


def _donerf(dcfg, root, split):
    """DONeRFDataset.read_meta_for_split (datasets/donerf.py:50-150)."""
    W, H = (int(v) for v in _get(dcfg, "img_wh"))
    use_ndc, correct = bool(_get(dcfg, "use_ndc", False)), bool(_get(dcfg, "correct_poses", False))
    center = bool(_get(dcfg, "center_poses", False))

    def load(name):
        with open(os.path.join(root, name), "r") as f:
            return json.load(f)

    train_meta, meta, info = load("transforms_train.json"), load(_DONERF_FILES[split]), load("dataset_info.json")
    frames_meta = meta["frames"][:int(_get(dcfg, "val_num"))] if split == "val" else meta["frames"]
    origin = np.array(info["view_cell_center"])

    def poses_of(frames):  # load_poses_from_meta (donerf.py:62-86)
        out = []
        for fr in frames:
            pose = np.array(fr["transform_matrix"])[:3, :4]
            if center:
                pose[:3, -1] = pose[:3, -1] - origin
            out.append(pose)
        return np.stack(out, 0)

    focal = 0.5 * 800 / np.tan(0.5 * info["camera_angle_x"])
    focal *= W / 800
    K = np.eye(3)
    K[0, 0], K[0, 2], K[1, 1], K[1, 2] = focal, W / 2.0, focal, H / 2.0
    near, far = info["depth_range"][0], info["depth_range"][1]
    if not frames_meta:
        raise UnsupportedPipeline(f"dataset_cameras: donerf 'split' {split!r} holds no view")
    poses = poses_of(frames_meta)
    if use_ndc or correct:
        poses = _center_poses_with_rotation_only(poses, poses_of(train_meta["frames"]))
        if _get(dcfg, "collection") in ["pavillon"] and split == "render":
            poses[..., :3, -1] *= 0.35
    facts = {"near": near, "far": far, "depth_range": info["depth_range"], "val_all": bool(_get(dcfg, "val_all", False))}
    template = _camera(poses[0], K, W, H, 0.0, 0, use_ndc, near)
    if split == "render":
        return spiral_path("donerf", template, poses)[0], [], facts
    cams = [dataclasses.replace(template, pose=np.asarray(p, np.float64).astype(np.float32)) for p in poses]
    if any("file_path" not in fr for fr in frames_meta):
        raise ValueError(f"dataset_cameras: a frame of {_DONERF_FILES[split]} has no file_path")
    return cams, [FrameSource(os.path.join(root, f"{fr['file_path']}.png"), None) for fr in frames_meta], facts


_READERS = {"technicolor": _technicolor, "neural_3d": _neural_3d, "immersive": _immersive, "donerf": _donerf}


def dataset_cameras(dataset_cfg, root: str, split: str) -> DatasetViews:
    """The views of ``split`` (train, val, test or render) of the scene directory ``root`` for ``dataset_cfg``, a loaded
    conf/experiment/dataset/*.yaml (``name``, ``collection``, ``img_wh``, ``start_frame``, ``num_frames``, ``val_set``,
    ``val_skip``, ``val_all``, ``val_num``, ``use_ndc``, ``correct_poses``, ``render_params``, ...), as the reference's
    dataset of that split holds and visits them.

    - technicolor: ``images/`` (sorted, ``lightfield_rows * lightfield_cols`` per frame) and ``cameras_parameters.txt``;
      train frame-major without the held-out views, val / test the held-out views in the order the ``val_set`` rule lists
      them (``'lightfield'``, a list, or every ``val_skip``-th view).  cam_idx 3 on held-out views unless ``val_all``.
    - neural_3d: ``poses_bounds.npy`` and the ``*.mp4`` videos, ``val_set`` the held-out video indices.
    - immersive: ``models.json`` (fisheye ``distortion`` on the train and held-out views) and ``<name>.mp4``; a non-empty
      ``val_set`` holds out camera_0001, whatever it lists.
    - neural_3d and immersive: train is video-major (each video's frames in order), as ``DeviceRayBatches.from_config``
      takes it; held-out views have cam_idx 1.
    - donerf: ``transforms_{train,val,test}.json`` / ``cam_path_pan.json`` and ``dataset_info.json``; RGBA frames.
    - render: ``spiral_path`` of the dataset's poses (donerf: cam_path_pan.json's poses as they are).
    The val split stops at ``val_num`` views and the render split at ``render_params.max_frames`` when set, as the
    reference's ``__len__`` does.

    Raises ``UnsupportedPipeline``, naming the key, for any other dataset ``name`` or ``split``, a per-split config section,
    ``img_wh`` missing, ``val_crop`` < 1 on val / test, a split that holds no view, neural_3d / immersive ``val_all`` with a
    non-empty ``val_set``, neural_3d ``val_set`` of several videos with several frames, and technicolor / immersive
    ``use_ndc`` with views whose focal length differs from the first camera's (so every Immersive render split in NDC, whose
    focal is scaled by 0.75).  Files that do not describe a whole rig
    raise ``ValueError``.  Nothing is returned from a refused call."""
    name = _get(dataset_cfg, "name", None)
    if name not in DATASETS:
        raise UnsupportedPipeline(f"dataset_cameras: dataset 'name' {name!r} is not supported: one of {DATASETS}")
    if split not in SPLITS:
        raise UnsupportedPipeline(f"dataset_cameras: 'split' {split!r} is not defined: one of {SPLITS}")
    _refuse_options(dataset_cfg, name, split)
    cams, frames, facts = _READERS[name](dataset_cfg, root, split)
    n = _split_len(len(cams), split, dataset_cfg)
    if n < 1:
        raise UnsupportedPipeline(f"dataset_cameras: {name} 'split' {split!r} holds no view under the config's val_set / "
                                  "val_skip / val_all")
    facts.update({k: _get(dataset_cfg, k) for k in ("name", "collection") if _has(dataset_cfg, k)})
    W, H = (int(v) for v in _get(dataset_cfg, "img_wh"))
    return DatasetViews(split=split, cameras=cams[:n], frames=frames[:n], facts=facts, rgba=name == "donerf",
                        crop=_crop(dataset_cfg, W, H) if split == "render" else None)
