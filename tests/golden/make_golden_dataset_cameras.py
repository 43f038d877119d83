"""Golden dataset views: every split of synthetic Technicolor, Neural-3D, Immersive and DoNeRF scene directories as the
unmodified reference dataset classes build them (``read_meta``, the split selection, ``prepare_train_data``'s view order,
``prepare_render_data`` and ``get_coords``), run on CPU through the shim with image and video reads stubbed.

    HYPERREEL_REFERENCE=<reference checkout> python tests/golden/make_golden_dataset_cameras.py

writes ``tests/golden/dataset_cameras.npz``.  Per case: ``<case>/scene`` (JSON: the scene directory's text files, empty
image / video files and ``.npy`` arrays stored as ``<case>/npy/<name>``), ``<case>/cfg`` (JSON dataset config) and
``<case>/facts`` (JSON: the training dataset's attributes that the model constructors read).  Per case and split:
``<case>/<split>/poses`` [n, 3, 4] and ``K`` [n, 3, 3] fp32 (``torch.FloatTensor`` of the arrays ``get_coords`` indexes),
``times`` / ``cam_idx`` [n] fp32 (the time and camera columns of its rays; 0 for DoNeRF, whose rays have 6 columns),
``distortion`` [n, 2] fp32 (Immersive), ``frames`` (JSON: the file and video frame each view's ground truth is read from,
relative to the scene directory), ``ray_views`` int64 and ``rays`` [k, H*W, C] fp32: the reference's ``get_coords`` rays of
a few views.
"""
import contextlib
import io
import json
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import ref_shim  # noqa: E402
from tests.golden.make_golden_subsample import _install  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "dataset_cameras.npz")
SPLITS = ("train", "val", "test", "render")


def _rot(rx, ry, rz):
    cx, sx, cy, sy, cz, sz = np.cos(rx), np.sin(rx), np.cos(ry), np.sin(ry), np.cos(rz), np.sin(rz)
    return (np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]]) @ np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
            @ np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]]))


def _quat_wxyz(R):
    from scipy.spatial.transform import Rotation

    x, y, z, w = Rotation.from_matrix(R).as_quat()
    return w, x, y, z


def technicolor_scene(rows, cols, n_frames, same_focal, rng):
    lines = ["f cx cy ar skew qw qx qy qz tx ty tz"]
    for r in range(rows):
        for c in range(cols):
            f = 1800.0 if same_focal else 1800.0 + 37.0 * (r * cols + c)
            R = _rot(*rng.normal(0, 0.02, 3))
            t = np.array([(c - (cols - 1) / 2) * 0.08, (r - (rows - 1) / 2) * 0.08, 0.01 * r])
            w, x, y, z = _quat_wxyz(R)
            vals = [f, 1024.0 + 3 * c, 544.0 - 2 * r, 1.0 if same_focal else 1.0 + 0.001 * c, 0.0, w, x, y, z, *t]
            lines.append(" ".join(repr(float(v)) for v in vals))
    images = [f"images/{fr:04d}_{v:02d}.png" for fr in range(n_frames) for v in range(rows * cols)]
    return {"files": {"cameras_parameters.txt": "\n".join(lines) + "\n"}, "empty": images, "npy": []}


def neural_3d_scene(n_videos, rng):
    rows = []
    for k in range(n_videos):
        a = -0.4 + 0.8 * k / max(n_videos - 1, 1)
        R = _rot(0.0, a, 0.0) @ _rot(*rng.normal(0, 0.01, 3))
        # LLFF "down right back" columns, then [H, W, focal]
        c2w = np.concatenate([R[:, 1:2], R[:, 0:1], -R[:, 2:3]], 1) @ np.diag([1.0, 1.0, -1.0])
        t = np.array([1.5 * np.sin(a), 0.05 * k, 1.5 * (1 - np.cos(a))])
        p = np.concatenate([c2w, t[:, None], np.array([[2028.0], [2704.0], [1460.0]])], 1)
        rows.append(np.concatenate([p.reshape(-1), [2.2 + 0.1 * k, 90.0 - k]]))
    return {"files": {}, "empty": [f"cam{k:02d}.mp4" for k in range(n_videos)],
            "npy": [("poses_bounds.npy", np.stack(rows))]}


def immersive_scene(n_cams, same_focal, rng):
    meta = []
    for k in range(n_cams):
        az = 2 * np.pi * k / n_cams
        meta.append({"name": f"camera_{k + 1:04d}", "focal_length": 1000.0 if same_focal else 1000.0 + 11.0 * k,
                     "principal_point": [1280.0 + 5 * k, 960.0 - 3 * k], "radial_distortion": [0.05 + 0.01 * k, -0.01, 0.0],
                     "orientation": [0.1 * np.sin(az), 0.3 * np.cos(az), 0.02 * k],
                     "position": [0.3 * np.sin(az), 0.05 * k, 0.3 * np.cos(az) - 0.2]})
    return {"files": {"models.json": json.dumps(meta)}, "empty": [m["name"] + ".mp4" for m in meta], "npy": []}


def donerf_scene(rng):
    def frames(n, prefix, with_path=True):
        out = []
        for k in range(n):
            R = _rot(*rng.normal(0, 0.1, 3))
            T = np.eye(4)
            T[:3, :3], T[:3, 3] = R, rng.normal(0, 0.3, 3) + np.array([0.5, -0.2, 1.0])
            fr = {"transform_matrix": T.tolist()}
            if with_path:
                fr["file_path"] = f"{prefix}/{k:05d}"
            out.append(fr)
        return {"frames": out}

    info = {"camera_angle_x": 0.9, "depth_range": [0.4, 18.0], "view_cell_center": [0.5, -0.2, 1.0],
            "view_cell_size": [0.3, 0.2, 0.4]}
    files = {"transforms_train.json": json.dumps(frames(6, "train")), "transforms_val.json": json.dumps(frames(4, "val")),
             "transforms_test.json": json.dumps(frames(3, "test")),
             "cam_path_pan.json": json.dumps(frames(5, "pan", with_path=False)), "dataset_info.json": json.dumps(info)}
    return {"files": files, "empty": [], "npy": []}


def _render_params(**kw):
    rp = {"interpolate": False, "interpolate_time": False, "supersample": 2, "crop": 1.0}
    rp.update(kw)
    return rp


def _cases():
    rng = np.random.default_rng(11)
    tc = dict(name="technicolor", collection="painter", img_wh=[8, 6], use_ndc=False, correct_poses=False, val_num=8,
              val_skip=2, val_all=False, lightfield_step=1, lightfield_rows=3, lightfield_cols=3, start_frame=0,
              num_frames=3, keyframe_step=1, render_params=_render_params())
    n3 = dict(name="neural_3d", collection="coffee_martini", img_wh=[10, 7], use_ndc=True, correct_poses=False, val_num=8,
              val_skip=2, val_all=False, val_set=[0], start_frame=2, num_frames=3, keyframe_step=2,
              render_params=_render_params(crop=0.85))
    im = dict(name="immersive", collection="05_Horse", img_wh=[8, 6], use_ndc=False, correct_poses=True, val_num=8,
              val_skip=2, val_all=False, val_set=[0], start_frame=1, num_frames=3, keyframe_step=1,
              render_params=_render_params(supersample=1))
    dn = dict(name="donerf", collection="barbershop", img_wh=[8, 8], use_ndc=False, correct_poses=False, center_poses=True,
              val_num=3, val_skip=1, val_all=False, render_params=_render_params(interpolate=False, supersample=4))
    return {
        # the shipped rule (val_set 'lightfield', step 1, one val pair) in NDC, from frame 1
        "technicolor_lightfield": (dict(tc, use_ndc=True, val_set="lightfield", val_pairs=[[1, 1]], start_frame=1),
                                   technicolor_scene(3, 3, 5, True, rng)),
        "technicolor_skip": (dict(tc, correct_poses=True, val_set=[], lightfield_rows=2, lightfield_cols=2, num_frames=2,
                                  collection="trains"), technicolor_scene(2, 2, 2, False, rng)),
        "technicolor_val_all": (dict(tc, val_set=[], val_all=True, collection="fabien", lightfield_rows=2,
                                     lightfield_cols=2, num_frames=2, render_params=_render_params(interpolate=True)),
                                technicolor_scene(2, 2, 2, False, rng)),
        # 4 x 4 x 25 = 400 views: read_meta replaces view 377 by view 361
        "technicolor_birthday": (dict(tc, collection="birthday", val_set="lightfield", val_pairs=[[1, 2]],
                                      lightfield_rows=4, lightfield_cols=4, num_frames=25, val_num=4,
                                      render_params=_render_params(supersample=1, max_frames=7)),
                                 technicolor_scene(4, 4, 25, False, rng)),
        "neural_3d_ndc": (n3, neural_3d_scene(5, rng)),
        "neural_3d_val_all": (dict(n3, use_ndc=False, val_all=True, val_set=[], start_frame=0, num_frames=2,
                                   render_params=_render_params(interpolate_time=True)), neural_3d_scene(4, rng)),
        "immersive_ndc": (dict(im, use_ndc=True, correct_poses=False), immersive_scene(5, True, rng)),
        "immersive_correct": (im, immersive_scene(6, False, rng)),
        "immersive_val_all": (dict(im, collection="01_Welder", correct_poses=False, val_set=[], val_all=True,
                                   num_frames=2, start_frame=0), immersive_scene(4, False, rng)),
        "donerf_center": (dn, donerf_scene(rng)),
        "donerf_ndc": (dict(dn, use_ndc=True, collection="pavillon"), donerf_scene(rng)),
        "donerf_correct": (dict(dn, correct_poses=True, center_poses=False, val_num=8, val_all=True), donerf_scene(rng)),
    }


def write_scene(root, scene):
    for rel, text in scene["files"].items():
        with open(os.path.join(root, rel), "w") as f:
            f.write(text)
    for rel in scene["empty"]:
        os.makedirs(os.path.dirname(os.path.join(root, rel)), exist_ok=True)
        open(os.path.join(root, rel), "wb").close()
    for rel, arr in scene["npy"]:
        np.save(os.path.join(root, rel), arr)


class _Paths:
    """iopath's PathManager on the local file system."""

    def register_handler(self, handler):
        pass

    def ls(self, path):
        return os.listdir(path)

    def open(self, path, mode="r"):
        return open(path, mode)


class _Video:
    """cv2.VideoCapture stand-in: each read() returns the file and the frame's position in it."""

    def __init__(self, path):
        self.path, self.pos = path, 0

    def read(self):
        self.pos += 1
        return True, (self.path, self.pos - 1)

    def release(self):
        pass


_CLASSES = {"technicolor": ("technicolor", "TechnicolorDataset"), "neural_3d": ("neural_3d", "Neural3DVideoDataset"),
            "immersive": ("immersive", "ImmersiveDataset"), "donerf": ("donerf", "DONeRFDataset")}
_FACT_KEYS = ("num_keyframes", "num_frames", "near", "far", "depth_range", "bbox_min", "bbox_max", "total_images_per_frame",
              "val_all")


def _plain(v):
    if isinstance(v, np.ndarray):
        return v.tolist()
    if isinstance(v, (np.floating, np.integer, np.bool_)):
        return v.item()
    return v


def reference_split(dcfg, root, split):
    """(poses, K, times, cam_idx, distortion, frames, rays per view, facts) of one split of the reference's dataset."""
    import importlib

    module, cls_name = _CLASSES[dcfg["name"]]
    mod = importlib.import_module(f"datasets.{module}")
    cls = getattr(mod, cls_name)
    cfg = ref_shim.to_attr({"dataset": dict(dcfg, root_dir=root), "params": {"render_only": True, "test_only": False}})
    with contextlib.redirect_stdout(io.StringIO()):
        ds = cls(cfg, split=split)
    facts = {k: _plain(getattr(ds, k)) for k in _FACT_KEYS if hasattr(ds, k)}
    name = dcfg["name"]
    W, H = dcfg["img_wh"]
    read = []
    views = []  # (pose array, K array, distortion or None, rays)
    with contextlib.redirect_stdout(io.StringIO()):
        if split == "train" and name in ("neural_3d", "immersive"):
            # prepare_train_data's loop with the decoded frames stubbed: every (video, frame) view's rays and source
            mod.cv2.VideoCapture = _Video
            ds.get_rgb = lambda frame: (read.append(frame), torch.zeros(W * H, 3))[1]
            ds.prepare_train_data()
            coords = ds.all_coords.view(-1, W * H, ds.all_coords.shape[-1])
            nv = len(ds.video_paths)
            for i in range(coords.shape[0]):
                v = i // ds.num_frames
                K = ds.K if name == "neural_3d" else ds.intrinsics[v]
                dist = ds.distortions[v] if name == "immersive" else None
                views.append((ds.poses[v], K, dist, coords[i]))
            assert nv * ds.num_frames == coords.shape[0]
            frames = [[os.path.relpath(p, root), f] for p, f in read]
        else:
            n = len(ds.image_paths) if split == "train" else len(ds)
            frames = []
            for idx in range(n):
                rays = ds.get_coords(idx)
                if name == "technicolor":
                    K = ds.intrinsics[idx] if split != "render" else ds.intrinsics[0]
                    dist = None
                elif name == "neural_3d" or name == "donerf":
                    K, dist = ds.K, None
                else:
                    K = torch.FloatTensor(ds.intrinsics[idx] if split != "render" else ds.intrinsics[0])
                    if split == "render":
                        K[0, 0] *= 0.75
                        K[1, 1] *= 0.75
                    dist = ds.distortions[idx] if split != "render" else None
                views.append((ds.poses[idx], K, dist, rays))
                if split == "render":
                    continue
                if name in ("neural_3d", "immersive"):
                    mod.cv2.VideoCapture = _Video
                    ds.get_rgb = lambda frame: frame
                    p, f = ds.get_rgb_one(idx)
                    frames.append([os.path.relpath(p, root), f])
                elif name == "technicolor":
                    frames.append([os.path.join("images", ds.image_paths[idx]), None])
                else:
                    frames.append([f"{ds.image_paths[idx]}.png", None])
    poses = np.stack([torch.FloatTensor(np.asarray(p)[:3, :4]).numpy() for p, _, _, _ in views])
    Ks = np.stack([torch.FloatTensor(np.asarray(K)).numpy() for _, K, _, _ in views])
    rays = [r.reshape(W * H, -1).numpy() for _, _, _, r in views]
    C = rays[0].shape[-1]
    times = np.array([r[0, 7] if C == 8 else 0.0 for r in rays], np.float32)
    cam_idx = np.array([r[0, 6] if C == 8 else 0.0 for r in rays], np.float32)
    assert all(np.all(r[:, 6:] == r[0:1, 6:]) for r in rays)
    dist = (np.stack([np.asarray(d).astype(np.float32) for _, _, d, _ in views]) if views[0][2] is not None
            else np.zeros((len(views), 2), np.float32))
    return poses, Ks, times, cam_idx, dist, frames, rays, facts


def _ray_views(n, extra=()):
    return sorted({0, n // 2, n - 1, *[e for e in extra if e < n]})


def main():
    _install()
    import sys as _sys

    _sys.modules["iopath.common.file_io"].PathManager = _Paths
    arrays = {}
    for case, (dcfg, scene) in _cases().items():
        with tempfile.TemporaryDirectory() as root:
            root = os.path.join(root, "scene")
            os.makedirs(root)
            write_scene(root, scene)
            spec = {"files": scene["files"], "empty": scene["empty"], "npy": [rel for rel, _ in scene["npy"]]}
            for rel, arr in scene["npy"]:
                arrays[f"{case}/npy/{rel}"] = arr
            arrays[f"{case}/scene"] = np.array(json.dumps(spec))
            arrays[f"{case}/cfg"] = np.array(json.dumps(dcfg))
            for split in SPLITS:
                poses, Ks, times, cam_idx, dist, frames, rays, facts = reference_split(dcfg, root, split)
                if split == "train":
                    arrays[f"{case}/facts"] = np.array(json.dumps(facts))
                idx = _ray_views(len(rays), extra=(361, 377) if "birthday" in case else ())
                for k, v in (("poses", poses), ("K", Ks), ("times", times), ("cam_idx", cam_idx), ("distortion", dist),
                             ("ray_views", np.array(idx, np.int64)), ("rays", np.stack([rays[i] for i in idx]))):
                    arrays[f"{case}/{split}/{k}"] = v
                arrays[f"{case}/{split}/frames"] = np.array(json.dumps(frames))
                print(case, split, len(poses), "views")
    np.savez_compressed(OUT, **arrays)


if __name__ == "__main__":
    main()
