"""Camera -> rays on the device, and whole-frame rendering to 8-bit pixels (SURVEY.md section 8(f) rows f2 and f4).

Mirrors ``get_coords_from_camera`` of the reference datasets (datasets/base.py:485-518: pixel grid ->
``get_ray_directions_K`` -> ``get_rays`` -> optional ``to_ndc`` -> append camera id and time), the fisheye cameras of
``ImmersiveDataset.get_coords`` (``Camera(distortion=(k1, k2))``, datasets/immersive.py:494-573), the Stanford light-field
dataset's two-plane views (``TwoPlaneCamera``, ``get_lightfield_rays``, utils/ray_utils.py:14-45) and ``to8b``
(utils/__init__.py:47).  The reference builds the rays on the CPU and uploads 32 B per ray for every frame
(nlf/__init__.py:828-834); here only the pose and intrinsics cross PCIe and 3 B per pixel come back.
"""
from __future__ import annotations

import dataclasses
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


def _f32(name: str, value) -> float:
    with np.errstate(over="ignore", invalid="ignore"):
        v = np.float32(np.float64(value))
    if not np.isfinite(v):
        raise ValueError(f"TwoPlaneCamera: {name} = {value!r} is not finite in float32")
    return float(v)


@dataclass
class TwoPlaneCamera:
    """One view of a two-plane light field: the Stanford light-field dataset's rays (``get_lightfield_rays``,
    utils/ray_utils.py:14-45), pixel (x, y) -> origin (s * st_scale, t * st_scale, near) and direction
    F.normalize(u * uv_scale - s * st_scale, v * uv_scale - t * st_scale, far - near) with u = linspace(-1, 1, width)[x]
    and v = linspace(1, -1, height)[y] / aspect.  ``aspect`` defaults to width / height; the reference passes its dataset's
    ``img_wh`` ratio, which differs from the view's when the view is cropped.  ``lightfield_cameras`` gives a split's views.

    The reference makes fp32 tensors of these Python numbers, so each is rounded to float32 (s, t, st_scale, uv_scale,
    near, aspect, and far - near, which it subtracts in double).  The device subtracts the rounded far and near in fp32, so a
    pair whose float32 difference is not the rounded double difference raises ``ValueError``, as does a non-finite value or
    an aspect that rounds to 0."""
    width: int
    height: int
    s: float
    t: float
    st_scale: float = 1.0
    uv_scale: float = 1.0
    near: float = -1.0
    far: float = 0.0
    aspect: Optional[float] = None
    time: float = 0.0
    cam_idx: float = 0.0

    def __post_init__(self):
        self._fields_f32()

    def _fields_f32(self) -> Tuple[float, ...]:
        if int(self.width) < 1 or int(self.height) < 1:
            raise ValueError(f"TwoPlaneCamera: bad size {self.width} x {self.height}")
        aspect = float(self.width) / float(self.height) if self.aspect is None else self.aspect
        f = tuple(_f32(n, v) for n, v in (("s", self.s), ("t", self.t), ("st_scale", self.st_scale),
                                          ("uv_scale", self.uv_scale), ("near", self.near), ("far", self.far),
                                          ("aspect", aspect), ("time", self.time), ("cam_idx", self.cam_idx)))
        if f[6] == 0.0:
            raise ValueError(f"TwoPlaneCamera: aspect = {aspect!r} is 0 in float32")
        dz = _f32("far - near", float(self.far) - float(self.near))
        if float(np.float32(f[5]) - np.float32(f[4])) != dz:
            raise ValueError(f"TwoPlaneCamera: far - near of far = {self.far!r}, near = {self.near!r} in float32 is not the "
                             "reference's (the difference in double, rounded): choose near and far whose float32 difference "
                             "is exact")
        return f

    def to_c(self) -> L.hr_camera:
        c = L.hr_camera()
        s, t, st, uv, near, far, aspect, time, cam_idx = self._fields_f32()
        c.width, c.height = int(self.width), int(self.height)
        c.two_plane = 1
        c.lf_s, c.lf_t, c.lf_st_scale, c.lf_uv_scale = s, t, st, uv
        c.lf_near, c.lf_far, c.lf_aspect = near, far, aspect
        c.time, c.cam_idx = time, cam_idx
        return c


# ---- the render split's camera path: the poses and times of the reference's validation / render_only videos
# (prepare_render_data of each dataset, rendered in order by validation_video, nlf/__init__.py:809-891), restated in fp64 numpy
# in the reference's operation order and rounded to float32 where its get_coords makes tensors (torch.FloatTensor(pose),
# `ones * time`).

def _normalize(v):
    return v / np.linalg.norm(v)


def _average_poses(poses):  # utils/pose_utils.py:14-37
    center = poses[..., 3].mean(0)
    z = _normalize(poses[..., 2].mean(0))
    y_ = poses[..., 1].mean(0)
    x = _normalize(np.cross(y_, z))
    y = np.cross(z, x)
    return np.concatenate([np.stack([x, y, z], 1), center[..., None]], 1)


def _viewmatrix(z, up, pos):  # utils/pose_utils.py:39-45
    vec2 = _normalize(z)
    vec0 = _normalize(np.cross(up, vec2))
    vec1 = _normalize(np.cross(vec2, vec0))
    return np.stack([vec0, vec1, vec2, pos], 1)


def _spiral_poses(poses, rads, focal, n):  # create_spiral_poses (flip=False), utils/pose_utils.py:162-183
    c2w = _average_poses(poses)
    up = _normalize(poses[:, :3, 1].sum(0))
    rads = np.array(list(rads) + [1.0])
    out = []
    for theta in np.linspace(0.0, 2.0 * np.pi * 2, n + 1)[:-1]:
        c = np.dot(c2w[:3, :4], np.array([np.cos(theta), -np.sin(theta), -np.sin(theta * 0.5), 1.0]) * rads)
        z = _normalize(c - np.dot(c2w[:3, :4], np.array([0, 0, -focal, 1.0])))
        out.append(_viewmatrix(z, up, c))
    return out


def _interpolate_poses(poses, supersample):
    """interpolate_poses (utils/pose_utils.py:269-356): `supersample` poses per gap, linear in the se(3) twist of each pose,
    with scipy's logm / expm as the reference calls them; the last pose repeated `supersample` times."""
    import scipy.linalg

    p44 = np.concatenate([poses, np.tile(np.eye(4)[-1, :].reshape(1, 1, 4), [poses.shape[0], 1, 1])], 1)
    twists = []
    for p in p44:
        M = scipy.linalg.logm(p)
        twists.append(np.stack([M[..., 2, 1], M[..., 0, 2], M[..., 1, 0], M[..., 0, 3], M[..., 1, 3], M[..., 2, 3]], -1))
    twists = np.stack(twists, 0)
    t = np.linspace(0, 1, supersample, endpoint=False).reshape(1, supersample, 1)
    tw = twists.reshape(-1, 1, twists.shape[-1])
    tw = ((1 - t) * tw[:-1] + t * tw[1:]).reshape(-1, twists.shape[-1])
    tw = np.concatenate([tw, np.tile(twists[-1:], [supersample, 1])], 0)
    out = []
    for w in tw:
        z = np.zeros_like(w[0])
        M = np.array([[z, -w[2], w[1], w[3]], [w[2], z, -w[0], w[4]], [-w[1], w[0], z, w[5]], [z, z, z, z]])
        out.append(scipy.linalg.expm(M))
    return np.stack(out, 0)[:, :3, :4]


# video datasets: (percentile of |camera centre| per axis, scale of the x and y radii, scale of the z radius, focus depth
# multiplier of a multi-frame video) of the spiral
_VIDEO_SPIRALS = {
    "technicolor": (60, 0.25, 1.0, 100.0),  # TechnicolorDataset.prepare_render_data, datasets/technicolor.py:294-353
    "neural_3d": (50, 0.5, 1.0, 2.0),       # Neural3DVideoDataset.prepare_render_data, datasets/neural_3d.py:321-380
    "immersive": (50, 1.0, 0.05, 1.0),      # ImmersiveDataset.prepare_render_data, datasets/immersive.py:427-487
}
SPIRAL_DATASETS = tuple(_VIDEO_SPIRALS) + ("donerf",)


def spiral_path(dataset: str, camera: Camera, poses, bounds=None, num_frames: int = 1, supersample: int = 1,
                interpolate: bool = False, interpolate_time: bool = False):
    """The cameras and per-frame times of the reference's render-split video, for ``render_video``.

    ``poses`` [N, 3, 4] and ``bounds`` are the dataset's ``poses`` and ``bounds`` as its read_meta leaves them for the
    render split (pose-corrected, every camera of every frame: video datasets are frame-major with N / num_frames cameras
    per frame); ``supersample``,
    ``interpolate`` and ``interpolate_time`` are the config's ``render_params`` (supersample, interpolate, interpolate_time).
    Video datasets (technicolor, neural_3d, immersive) fly a two-turn spiral around the middle frame's rig
    (create_spiral_poses, utils/pose_utils.py:162-183) carried along the rig's per-frame motion (interpolate_poses), with
    num_frames * supersample frames (120 for a one-frame dataset) and times over [0, 1] rounded to whole frames unless
    interpolate_time; with ``interpolate`` the path goes through the given poses instead.  DoNeRF renders its render split's
    poses (cam_path_pan.json) as they are (DONeRFDataset.prepare_render_data, datasets/donerf.py:216-217): pass those.
    Every frame copies ``camera`` (intrinsics, size, ray flags, camera id) with the path's pose and time.  Returns
    (list of Camera, times float32 [F])."""
    if dataset not in SPIRAL_DATASETS:
        raise ValueError(f"spiral_path: dataset must be one of {SPIRAL_DATASETS}, got {dataset!r}")
    P = np.asarray(poses, dtype=np.float64)
    if P.ndim != 3 or P.shape[1:] != (3, 4) or P.shape[0] < 1:
        raise ValueError(f"spiral_path: poses must be [N, 3, 4] with N >= 1, got {P.shape}")
    if not np.isfinite(P).all():
        raise ValueError("spiral_path: poses must be finite")
    num_frames, supersample = int(num_frames), int(supersample)
    if dataset == "donerf":
        path, times = list(P), np.zeros(P.shape[0])
    else:
        if num_frames < 1 or P.shape[0] % num_frames != 0:
            raise ValueError(f"spiral_path: {P.shape[0]} poses are not num_frames = {num_frames} frames of one rig")
        if supersample < 1:
            raise ValueError(f"spiral_path: supersample must be >= 1, got {supersample}")
        if interpolate:
            path = list(_interpolate_poses(P, supersample))
        else:
            if bounds is None:
                raise ValueError(f"spiral_path: the {dataset} spiral needs the dataset's bounds")
            b = np.asarray(bounds, dtype=np.float64)
            if b.size < 1 or not np.isfinite(b).all():
                raise ValueError("spiral_path: bounds must be finite")
            pct, s_xy, s_z, focus_mul = _VIDEO_SPIRALS[dataset]
            close_depth, inf_depth = b.min() * 0.9, b.max() * 5.0
            dt = 0.75
            focus_depth = 1.0 / (((1.0 - dt) / close_depth + dt / inf_depth))
            per_frame = P.shape[0] // num_frames
            mid = (num_frames // 2) * per_frame
            one_frame = P[mid:mid + per_frame]
            radii = np.percentile(np.abs(one_frame[..., 3]), pct, axis=0)
            radii[..., :2] *= s_xy
            if s_z != 1.0:
                radii[..., -1] *= s_z
            if num_frames > 1:
                each_frame = _interpolate_poses(P[::per_frame], supersample)
                path = _spiral_poses(one_frame, radii, focus_depth * focus_mul, num_frames * supersample)
                reference_pose = np.eye(4)
                reference_pose[:3, :4] = P[mid]
                reference_pose = np.linalg.inv(reference_pose)
                for i in range(len(path)):
                    cur = np.eye(4)
                    cur[:3, :4] = path[i]
                    path[i] = each_frame[i] @ (reference_pose @ cur)
            else:
                path = _spiral_poses(one_frame, radii, focus_depth * 100, 120)
        if num_frames - 1 > 0:
            times = np.linspace(0, num_frames - 1, len(path))
            if not interpolate_time:
                times = np.round(times)
            times = times / (num_frames - 1)
        else:
            times = np.zeros(len(path))
    poses32 = np.stack(path, 0).astype(np.float32)
    times32 = np.asarray(times, dtype=np.float64).astype(np.float32)
    cams = [dataclasses.replace(camera, pose=poses32[i], time=float(times32[i])) for i in range(len(path))]
    return cams, times32


def render_video(model_or_system, cameras: Sequence[Camera], times=None, out: Optional[torch.Tensor] = None,
                 stream=None) -> torch.Tensor:
    """uint8 video [F, H, W, 3] on the device of a LightfieldModel, RenderLightfield or INRSystem along ``cameras`` (one
    size, Camera or TwoPlaneCamera, models mixed freely) at ``times`` (default each camera's ``time``): the reference's validation_video loop
    (nlf/__init__.py:809-891) with its to8b, as one call that never synchronises (hr_render_video_to8b).  ``spiral_path``
    gives the reference's cameras and times."""
    target = model_or_system if hasattr(model_or_system, "render_video") else getattr(model_or_system, "model", None)
    if target is None or not hasattr(target, "render_video"):
        raise TypeError(f"render_video: expected a LightfieldModel, RenderLightfield or INRSystem, got {type(model_or_system)}")
    return target.render_video(cameras, times, out=out, stream=stream)


def score_views(model_or_system, cameras: Sequence[Camera], images: torch.Tensor, times=None, out: Optional[torch.Tensor] = None,
                stream=None, *, rgba: bool = False):
    """(mse, ssim), fp64 [n] device tensors, of a held-out split: view i of a LightfieldModel, RenderLightfield or INRSystem
    rendered from ``cameras[i]`` (one size, Camera or TwoPlaneCamera, models mixed freely) at ``times[i]`` (default each
    camera's ``time``) and scored against ``images[i]`` (uint8 [n, H, W, 3], contiguous, on the model's device) -- the
    reference's evaluation of a split (nlf/__init__.py:895-982) as one call that never synchronises (hr_score_views).  Each
    pair equals ``metrics.image_metrics`` of the view's eval render against ``images[i] / 255`` correctly rounded in fp32 (T.ToTensor()'s conversion), bit for bit.
    ``rgba=True``: ``images`` are uint8 RGBA [n, H, W, 4] (the DoNeRF and Catacaustics frames) and each view is scored
    against its composite over white, ``rgb * a + (1 - a)`` as their ``get_rgb`` computes it, bit for bit."""
    target = model_or_system if hasattr(model_or_system, "score_views") else getattr(model_or_system, "model", None)
    if target is None or not hasattr(target, "score_views"):
        raise TypeError(f"score_views: expected a LightfieldModel, RenderLightfield or INRSystem, got {type(model_or_system)}")
    return target.score_views(cameras, images, times, out=out, stream=stream, rgba=rgba)


@dataclass(frozen=True)
class VisualRequest:
    """One map of the embedding visualiser: field ``key`` of the colour net reduced in ``mode`` (lib.FIELD_OVER or
    FIELD_PRED_WEIGHTS) over ``channels`` channels, then visualize_warp's options: ``use_abs``, ``bounds`` (lo, hi) rounded to
    float32 or None, ``normalize``."""
    key: str
    mode: int
    channels: int
    use_abs: bool
    bounds: Optional[Tuple[float, float]]
    normalize: bool


def embedding_requests(visualizer) -> list:
    """The maps of an embedding-visualiser config (``cfg.visualizers.embedding``, or a loaded
    conf/experiment/visualizers/embedding/*.yaml) as VisualRequests, in the config's order.  Supported: every field the fused
    path carries (lib.FIELDS), reduced over the samples (``pred_weights_fields`` selects the predicted weights), with
    ``use_abs``, scalar ``bounds`` and ``normalize``, and ``sort: False``.  ``data_fields`` (raw dumps) are not maps and are
    ignored.  Anything else raises UnsupportedPipeline naming the key: another visualiser type, a field the path does not
    carry, a field in ``no_over_fields`` (per-sample channels), ``sort: True`` (data-dependent channels), or bounds that are
    not two finite float32 numbers with hi != lo."""
    from .signature import UnsupportedPipeline

    kind = visualizer.get("type", "embedding")
    if kind != "embedding":
        raise UnsupportedPipeline(f"visualiser type '{kind}' is not supported: only 'embedding' maps are rendered")
    no_over = set(visualizer.get("no_over_fields", None) or [])
    pred_w = set(visualizer.get("pred_weights_fields", None) or [])
    out = []
    for key, opts in (visualizer.get("fields", None) or {}).items():
        opts = dict(opts or {})
        if key not in L.FIELDS:
            raise UnsupportedPipeline(f"embedding visualiser: field '{key}' is not produced by the fused path")
        if key in no_over:
            raise UnsupportedPipeline(f"embedding visualiser: field '{key}' is in no_over_fields: per-sample channels are not mapped")
        if opts.get("sort", False):
            raise UnsupportedPipeline(f"embedding visualiser: field '{key}' has sort: True, which is not supported")
        bounds = opts.get("bounds", None)
        if bounds is not None and len(bounds) > 0:
            try:
                with np.errstate(over="ignore"):
                    lo, hi = (np.float32(float(b)) for b in bounds)
            except (TypeError, ValueError):
                raise UnsupportedPipeline(f"embedding visualiser: field '{key}': bounds must be [lo, hi], got {bounds!r}") from None
            if len(bounds) != 2 or not (np.isfinite(lo) and np.isfinite(hi)) or lo == hi:
                raise UnsupportedPipeline(f"embedding visualiser: field '{key}': bounds must be two finite float32 numbers "
                                          f"with hi != lo, got {bounds!r}")
            bounds = (float(lo), float(hi))
        else:
            bounds = None
        out.append(VisualRequest(key, L.FIELD_PRED_WEIGHTS if key in pred_w else L.FIELD_OVER, L.FIELD_CHANNELS[key],
                                 bool(opts.get("use_abs", False)), bounds, bool(opts.get("normalize", False))))
    return out


def render_embeddings(model_or_system, cameras: Sequence[Camera], visualizer, times=None, rgb: bool = True, stream=None):
    """The embedding visualiser's maps of every frame (EmbeddingVisualizer.validation, nlf/visualizers/embedding.py:37-90, with
    visualize_warp and to8b, utils/visualization.py:24-52, utils/__init__.py:47) of a LightfieldModel, RenderLightfield or
    INRSystem along ``cameras`` at ``times`` (default each camera's ``time``), on the device in the render pass that makes
    the RGB frame (hr_render_visuals): one call that never synchronises.  ``visualizer`` is an embedding-visualiser config
    (see embedding_requests).  Returns a dict of device uint8 stacks keyed as the reference names the maps:
    'embedding_<key>' [F, H, W] for a 1-channel field (the grayscale image it saves) or [F, H, W, 3], and, with ``rgb``,
    'rgb' [F, H, W, 3], bit for bit render_video's.  Each map equals visualize_warp + to8b applied to the fp32 field that
    ``forward(rays, {'fields': [key]})`` returns for the frame's rays."""
    target = model_or_system if hasattr(model_or_system, "render_visuals") else getattr(model_or_system, "model", None)
    if target is None or not hasattr(target, "render_visuals"):
        raise TypeError(f"render_embeddings: expected a LightfieldModel, RenderLightfield or INRSystem, got {type(model_or_system)}")
    requests = embedding_requests(visualizer)
    return keyed_maps(requests, *target.render_visuals(cameras, requests, times, rgb=rgb, stream=stream))


def keyed_maps(requests, video, maps, prefix: str = "") -> dict:
    """render_visuals' outputs under the reference's names: prefix + 'rgb' (when rendered) and prefix + 'embedding_<key>',
    a 1-channel map as [F, H, W]."""
    out = {} if video is None else {prefix + "rgb": video}
    for r in requests:
        out[f"{prefix}embedding_{r.key}"] = maps[r.key][..., 0] if r.channels == 1 else maps[r.key]
    return out


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
