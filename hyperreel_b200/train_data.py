"""Training batches generated on the device from the training images (SURVEY.md section 2 row 23).

The reference's training dataset in its default mode (datasets/base.py:111-143,202-227,254-289) concatenates the rays of every
training pixel into one host table ``all_inputs = cat([coords, rgb, weights])`` (48 B per ray with 8 ray channels),
re-permutes the whole table every epoch and hands out consecutive slices, which ``format_batch`` splits and the loop copies to
the GPU.  ``DeviceRayBatches`` keeps the images on the device as uint8 (3 B per pixel) and the cameras as ``hr_camera``
records; ``hr_sample_train_batch`` (csrc/hr_train_batch.cu) produces each batch in one launch: the batch's pixels in the
epoch's shuffled order (a keyed bijection, no permutation array), each pixel's ray with ``generate_rays``'s arithmetic (bit for
bit) and its colour ``u8 / 255`` (``T.ToTensor()``), weight 1.  ``INRSystem.training_step`` takes the batches as they are::

    batches = DeviceRayBatches(cameras, images, batch_size=16384, seed=0)
    for epoch in range(n_epochs):
        batches.set_epoch(epoch)
        for batch in batches:
            system.training_step(batch)

The shipped training configs train differently: they sample with replacement (``num_iters`` batches per epoch) from a table
in which the video datasets keep only a per-frame subset of each view's pixels.  ``DeviceRayBatches.from_config`` reads both
from a config, and ``hr_sample_train_rows`` (same file) generates those batches, again without any table in memory.  The
Immersive dataset keeps its per-frame pixels by image content; ``hr_build_importance_table`` selects them on the device into a
keep bitmask per frame and ``hr_sample_train_mask_rows`` samples from it.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import lib as L
from .camera import Camera


def _as_image_stack(images) -> torch.Tensor:
    if isinstance(images, (list, tuple)):
        views = [torch.as_tensor(im) for im in images]
        if not views:
            raise ValueError("DeviceRayBatches needs at least one training image")
        shapes = {tuple(v.shape) for v in views}
        if len(shapes) > 1:
            raise ValueError(f"DeviceRayBatches needs training views of one size (the reference's img_wh), got {sorted(shapes)}")
        dtypes = {v.dtype for v in views}
        if dtypes != {torch.uint8}:
            raise ValueError(f"DeviceRayBatches needs uint8 images, got {sorted(str(d) for d in dtypes)}")
        return torch.stack(views)
    images = torch.as_tensor(images)
    if images.dtype != torch.uint8:
        raise ValueError(f"DeviceRayBatches needs uint8 images, got {images.dtype}")
    return images


def _video_major(frames: Sequence[int], videos: Sequence[int]) -> List[bool]:
    """Whether each view is its video's first, checking that views are video-major with each video's frames consecutive."""
    if len(videos) != len(frames):
        raise ValueError(f"{len(videos)} video indices for {len(frames)} views: one per view is needed")
    first = [i == 0 or videos[i] != videos[i - 1] for i in range(len(frames))]
    seen = set()
    for i, f in enumerate(first):
        if f:
            if videos[i] in seen:
                raise ValueError(f"views must be video-major: video {videos[i]} appears again at view {i}")
            seen.add(videos[i])
        elif frames[i] != frames[i - 1] + 1:
            raise ValueError(f"views must be video-major with consecutive frames: view {i} has frame {frames[i]} "
                             f"after frame {frames[i - 1]}")
    return first


def regular_subsample_plan(frames: Sequence[int], *, load_full_step: int, subsample_keyframe_step: int,
                           subsample_keyframe_frac: float, subsample_frac: float, counters: str = "technicolor",
                           videos: Optional[Sequence[int]] = None) -> List[Tuple[int, int]]:
    """The video datasets' per-frame pixel subsets as one ``(stride, offset)`` per training view, in the table's order: the
    view keeps the pixels with ``(x + y + offset) % stride == 0`` (``stride == 1`` keeps every pixel).

    ``frames[i]`` is view ``i``'s frame.  A frame with ``frame % load_full_step == 0`` is whole; otherwise one with ``frame %
    subsample_keyframe_step == 0`` has stride ``round(1 / subsample_keyframe_frac)`` and every other frame ``round(1 /
    subsample_frac)``; the offset is a running counter, one for each of the two kinds.  ``counters`` selects how they run:

    * ``"technicolor"`` (datasets/technicolor.py:211-269): both start at 0 and advance over all views in order.
    * ``"neural_3d"`` (datasets/neural_3d.py:168-185,217-269): ``videos[i]`` is view ``i``'s video index; views are video-major
      with each video's frames consecutive.  Both counters restart at the video index, and each video's first view is whole
      and advances neither.
    """
    frames = [int(f) for f in frames]
    if any(f < 0 for f in frames):
        raise ValueError("frames must be >= 0")
    for name, step in (("load_full_step", load_full_step), ("subsample_keyframe_step", subsample_keyframe_step)):
        if int(step) < 1:
            raise ValueError(f"{name} must be >= 1, got {step}")
    strides = {}
    for name, frac in (("subsample_keyframe_frac", subsample_keyframe_frac), ("subsample_frac", subsample_frac)):
        if not float(frac) > 0.0:
            raise ValueError(f"{name} must be > 0, got {frac}")
        strides[name] = int(round(1.0 / float(frac)))  # Python's round halves to even, as np.round does
        if strides[name] < 1:
            raise ValueError(f"{name}={frac} keeps more than every pixel (stride {strides[name]})")
    if counters == "technicolor":
        if videos is not None:
            raise ValueError("videos is for counters='neural_3d'")
        first_of_video = [False] * len(frames)
        restart = [None] * len(frames)
    elif counters == "neural_3d":
        if videos is None or len(videos) != len(frames):
            raise ValueError("counters='neural_3d' needs one video index per view")
        videos = [int(v) for v in videos]
        first_of_video = _video_major(frames, videos)
        restart = [videos[i] if first else None for i, first in enumerate(first_of_video)]
    else:
        raise ValueError(f"counters must be 'technicolor' or 'neural_3d', got {counters!r}")
    plan, key_offset, frame_offset = [], 0, 0
    for i, f in enumerate(frames):
        if restart[i] is not None:
            key_offset = frame_offset = restart[i]
        if first_of_video[i] or f % load_full_step == 0:
            plan.append((1, 0))
        elif f % subsample_keyframe_step == 0:
            plan.append((strides["subsample_keyframe_frac"], key_offset))
            key_offset += 1
        else:
            plan.append((strides["subsample_frac"], frame_offset))
            frame_offset += 1
    return plan


def subset_rows(stride: int, offset: int, height: int, width: int) -> int:
    """The number of pixels of an ``height x width`` view with ``(x + y + offset) % stride == 0``: every ``stride`` consecutive
    rows hold ``width`` of them, and the rows past the last whole block are counted one by one."""
    full = height // stride
    n = full * width
    for y in range(full * stride, height):
        x0 = (stride - (y + offset) % stride) % stride
        n += (width - 1 - x0) // stride + 1 if x0 < width else 0
    return n


def importance_subsample_plan(frames: Sequence[int], videos: Sequence[int], *, load_full_step: int,
                              subsample_keyframe_step: int, subsample_keyframe_frac: float, subsample_frac: float,
                              height: int, width: int) -> List[Optional[Tuple[int, int]]]:
    """The Immersive dataset's per-frame pixel subsets (datasets/immersive.py:295-391) as one entry per training view, in the
    table's order: ``None`` for a view that keeps every pixel, or ``(num_take, prev)`` for one that keeps the pixels whose
    colour changed most since view ``prev`` (the previous frame of its video).

    ``frames[i]`` and ``videos[i]`` are view ``i``'s frame and video; views are video-major with each video's frames
    consecutive.  A video's first view is whole, as is a frame with ``frame % load_full_step == 0``.  Every other frame takes
    ``num_take = int(np.round(H*W * frac))`` with ``frac = subsample_keyframe_frac`` when ``frame % subsample_keyframe_step ==
    0`` and ``subsample_frac`` otherwise, and keeps the pixels whose mean absolute colour change exceeds that change's
    ``num_take``-th largest value (ties excluded, so often fewer than ``num_take``) and whose ray points down the camera's
    -z (direction z < -0.05).  ``DeviceRayBatches(..., importance=plan)`` builds that table on the device."""
    frames, videos = [int(f) for f in frames], [int(v) for v in videos]
    if any(f < 0 for f in frames):
        raise ValueError("frames must be >= 0")
    for name, step in (("load_full_step", load_full_step), ("subsample_keyframe_step", subsample_keyframe_step)):
        if int(step) != step or int(step) < 1:
            raise ValueError(f"{name} must be an integer >= 1, got {step}")
    n = int(height) * int(width)
    if int(height) < 1 or int(width) < 1:
        raise ValueError(f"views must hold at least one pixel, got {height}x{width}")
    take = {}
    for name, frac in (("subsample_keyframe_frac", subsample_keyframe_frac), ("subsample_frac", subsample_frac)):
        frac = float(frac)
        if not 0.0 <= frac:
            raise ValueError(f"{name} must be >= 0, got {frac}")
        take[name] = int(np.round(n * frac * 1.0))  # importance_subsample's num_take (fac = 1.0)
        if take[name] > n:
            raise ValueError(f"{name}={frac} takes {take[name]} of {n} pixels: the reference's sorted[-num_take] fails")
    first = _video_major(frames, videos)
    plan: List[Optional[Tuple[int, int]]] = []
    for i, f in enumerate(frames):
        if first[i] or f % int(load_full_step) == 0:
            plan.append(None)
        elif f % int(subsample_keyframe_step) == 0:
            plan.append((take["subsample_keyframe_frac"], i - 1))
        else:
            plan.append((take["subsample_frac"], i - 1))
    return plan


class DeviceRayBatches:
    """Shuffled training batches ``{'coords' [B, c_in], 'rgb' [B, 3], 'weight' [B, 1]}`` (fp32, on the device) over every
    pixel of the training views, generated on the device per batch.

    ``cameras``: one ``Camera`` per view, each of the images' size.  ``images``: uint8 ``[n, H, W, 3]`` (or a sequence of
    ``[H, W, 3]`` of one size), on the host or the device; uploaded once.  An epoch visits each of the ``n*H*W`` pixels exactly
    once, in an order fixed by ``(seed, epoch)``; batches are consecutive ``batch_size`` pieces of that order and the last one
    is short, like the reference's last slice.  ``set_epoch(e)`` selects the order (0 at construction); ``len()`` is the
    number of batches per epoch and iterating yields them in turn.

    Two options reproduce what the shipped training configs train on (``from_config`` sets both from a config):

    * ``subsample``: one ``(stride, offset)`` per view (``regular_subsample_plan``).  The training table then holds, view by
      view, only the pixels with ``(x + y + offset) % stride == 0``, each view's in row-major order: the order of the video
      datasets' ``all_coords``.  ``n_rows`` is the table's size (``n*H*W`` without a plan); ``gather_rows`` returns rows by
      table index.
    * ``importance``: the Immersive dataset's content-dependent subsets (``importance_subsample_plan``), built on the device
      at construction into a keep bitmask per importance view (about 0.14 B per pixel); the table is then each view's kept
      pixels in row-major order, as with ``subsample``, and ``view_rows`` gives the per-view counts.  Not combined with
      ``subsample``.
    * ``replacement=True`` with ``num_iters``: every batch is ``batch_size`` independent uniform draws from the table, keyed
      by ``(seed, epoch, position)``, and an epoch is ``num_iters`` batches, as the reference's
      ``RandomSampler(replacement=True, num_samples=num_iters * batch_size)`` (nlf/__init__.py:222-237).

    Only the reference's default training mode is provided.  The dataset options of the others (datasets/base.py:85-101)
    are accepted under the reference's names so that they can be refused: ``use_patches``, ``precrop_iters`` > 0 (crop),
    ``use_full_image`` and ``blur_radius`` > 0 raise ``ValueError``, as do views of different sizes and non-uint8 images.

    ``rgba=True``: the images are uint8 RGBA ``[n, H, W, 4]`` (4 B per pixel held), as the DoNeRF and Catacaustics datasets
    load them (``dataset_frames`` resizes them), and each row's ``'rgb'`` is the pixel's composite over white that their
    ``get_rgb`` returns, ``rgb * a + (1 - a)`` of the ``u8 / 255`` values with each operation rounded as torch rounds it on
    the CPU.  Rays, order, draws and ids are those of the same views given as RGB.  Not combined with ``importance`` (the
    Immersive dataset, whose frames are RGB)."""

    def __init__(self, cameras: Sequence[Camera], images, batch_size: int, seed: int = 0, c_in: int = 8,
                 device: Optional[torch.device] = None, *, use_patches: bool = False, precrop_iters: int = 0,
                 use_full_image: bool = False, blur_radius: int = 0, replacement: bool = False,
                 num_iters: Optional[int] = None, subsample: Optional[Sequence[Tuple[int, int]]] = None,
                 importance: Optional[Sequence[Optional[Tuple[int, int]]]] = None, rgba: bool = False):
        for name, value, default in (("use_patches", use_patches, False), ("precrop_iters", precrop_iters, 0),
                                     ("use_full_image", use_full_image, False), ("blur_radius", blur_radius, 0)):
            if value != default:
                raise ValueError(f"DeviceRayBatches generates the reference's default training batches only: "
                                 f"{name}={value!r} is not supported")
        if c_in not in (6, 8):
            raise ValueError(f"c_in must be 6 or 8, got {c_in}")
        if int(batch_size) < 1:
            raise ValueError(f"batch_size must be >= 1, got {batch_size}")
        images = _as_image_stack(images)
        ch = 4 if rgba else 3
        if images.dim() != 4 or images.shape[-1] != ch:
            raise ValueError(f"images must be [n, H, W, {ch}]{' (rgba=True)' if rgba else ''}, got {tuple(images.shape)}")
        cameras = list(cameras)
        n, H, W = int(images.shape[0]), int(images.shape[1]), int(images.shape[2])
        if n < 1 or H < 1 or W < 1:
            raise ValueError(f"images must hold at least one pixel, got {tuple(images.shape)}")
        if len(cameras) != n:
            raise ValueError(f"{len(cameras)} cameras for {n} images")
        for i, cam in enumerate(cameras):
            if (int(cam.width), int(cam.height)) != (W, H):
                raise ValueError(f"camera {i} is {cam.width}x{cam.height}, the images are {W}x{H}: every view needs the "
                                 "camera grid's size")
        if replacement:
            if num_iters is None or int(num_iters) < 1:
                raise ValueError(f"replacement=True needs num_iters >= 1 (batches per epoch), got {num_iters!r}")
        elif num_iters is not None:
            raise ValueError("num_iters sets the epoch length of replacement=True; without replacement an epoch is "
                             "ceil(n_rows / batch_size) batches")
        if importance is not None:
            if rgba:
                raise ValueError("importance tables are built from RGB frames (the Immersive dataset): rgba=True is not "
                                 "supported with importance")
            if subsample is not None:
                raise ValueError("importance and subsample are two different tables: give one of them")
            importance = self._check_importance(importance, n, H * W)
        if subsample is None:
            rule = [(1, 0)] * n
        else:
            rule = [tuple(r) for r in subsample]
            if len(rule) != n or any(len(r) != 2 for r in rule):
                raise ValueError(f"subsample needs one (stride, offset) per view: {len(rule)} entries for {n} views")
            if any(int(s) != s or int(o) != o or not 1 <= int(s) < 2 ** 31 for s, o in rule):
                raise ValueError("subsample strides must be integers in [1, 2^31) and offsets integers")
            rule = [(int(s), int(o) % int(s)) for s, o in rule]
        counts = [subset_rows(s, o, H, W) for s, o in rule]
        if sum(counts) < 1:
            raise ValueError("subsample keeps no pixel: the training table is empty")
        if not torch.cuda.is_available():
            raise RuntimeError("hyperreel_b200.DeviceRayBatches needs a CUDA device (no CPU fallback)")
        if device is None:
            device = images.device if images.is_cuda else torch.device("cuda", torch.cuda.current_device())
        self.device = torch.device(device)
        self._lib = L.load_library()
        self.images = images.to(self.device).contiguous()
        recs = (L.hr_camera * n)(*[cam.to_c() for cam in cameras])
        self.cameras = torch.frombuffer(bytearray(bytes(recs)), dtype=torch.uint8).to(self.device)
        self.n_views, self.height, self.width = n, H, W
        self.n_pixels = n * H * W
        self.batch_size = int(batch_size)
        self.seed = int(seed) & ((1 << 64) - 1)
        self.c_in = int(c_in)
        self.epoch = 0
        self.replacement = bool(replacement)
        self.num_iters = int(num_iters) if replacement else None
        self.subsample = None if subsample is None else rule
        self.importance = importance
        self.rgba = bool(rgba)
        if importance is None:
            self._n_rows = int(sum(counts))
            # the table's plan for hr_sample_train_rows: exclusive prefix of the per-view row counts, and (stride, offset) per view
            self._view_start = torch.tensor(np.concatenate([[0], np.cumsum(counts)]), dtype=torch.int64, device=self.device)
            self._view_rule = torch.tensor(rule, dtype=torch.int32, device=self.device).contiguous()
        else:
            self._n_rows = None  # read from the device on first use
            self._build_importance(importance)

    @staticmethod
    def _check_importance(plan, n: int, hw: int) -> List[Optional[Tuple[int, int]]]:
        plan = list(plan)
        if len(plan) != n:
            raise ValueError(f"importance needs one entry per view: {len(plan)} entries for {n} views")
        out = []
        for v, e in enumerate(plan):
            if e is None:
                out.append(None)
                continue
            e = tuple(e)
            if len(e) != 2 or any(int(a) != a for a in e):
                raise ValueError(f"importance entry {v} must be None or (num_take, prev), got {e!r}")
            take, prev = int(e[0]), int(e[1])
            if not 0 <= take <= hw:
                raise ValueError(f"importance entry {v} takes {take} pixels, outside [0, {hw}]")
            if prev != v - 1 or v == 0:
                raise ValueError(f"importance entry {v}'s previous frame is view {prev}: it must be view {v - 1}, the "
                                 "previous frame of the same video")
            out.append((take, prev))
        return out

    def _build_importance(self, plan) -> None:
        """Builds the keep masks of the importance views and the per-view row counts on the device (no synchronisation)."""
        dev, n = self.device, self.n_views
        n_slots = sum(e is not None for e in plan)
        blocks = -(-self.height * self.width // 256)
        host = np.array([(-1, -1) if e is None else e for e in plan], dtype=np.int64).reshape(n, 2)
        self._view_slot = torch.empty((n,), dtype=torch.int32, device=dev)
        self._block_start = torch.empty((max(n_slots, 1) * blocks,), dtype=torch.int32, device=dev)
        self._masks = torch.empty((max(n_slots, 1) * blocks * 8,), dtype=torch.int32, device=dev)
        self._view_rows = torch.empty((n,), dtype=torch.int64, device=dev)
        self._view_start = torch.empty((n + 1,), dtype=torch.int64, device=dev)
        ws_bytes = int(self._lib.hr_importance_workspace_bytes(n_slots))
        ws = torch.empty((max(ws_bytes, 1),), dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            L.check(self._lib.hr_build_importance_table(
                self.cameras.data_ptr(), n, self.images.data_ptr(), self.height, self.width,
                host.ctypes.data_as(C.c_void_p), ws.data_ptr(), ws_bytes, self._view_slot.data_ptr(),
                self._block_start.data_ptr(), self._masks.data_ptr(), self._view_rows.data_ptr(),
                self._view_start.data_ptr(), torch.cuda.current_stream(dev).cuda_stream))

    @property
    def n_rows(self) -> int:
        """The training table's size; for an ``importance`` table, reading it waits for the table's build."""
        if self._n_rows is None:
            n = int(self._view_start[-1])
            if n < 1:
                raise ValueError("importance keeps no pixel: the training table is empty")
            self._n_rows = n
        return self._n_rows

    @property
    def view_rows(self) -> torch.Tensor:
        """The number of table rows of each view, int64 [n_views] on the host."""
        return self._view_start.diff().cpu()

    @classmethod
    def from_config(cls, cfg, cameras: Sequence[Camera], images, seed: int = 0, c_in: int = 8,
                    device: Optional[torch.device] = None) -> "DeviceRayBatches":
        """The training batches a reference config trains on: ``cfg.training.batch_size``, ``sample_with_replacement`` and
        ``num_iters``, and for the ``technicolor``, ``neural_3d`` and ``immersive`` datasets the per-frame pixel subsets of
        ``cfg.dataset.{num_frames, load_full_step, subsample_keyframe_step, subsample_keyframe_frac, subsample_frac}``
        (``importance_subsample_plan`` for immersive, built on the device from the images).  For the ``donerf`` and
        ``catacaustics`` datasets the images may be their RGBA frames ``[n, H, W, 4]`` (``dataset_frames``' output), which
        are then composited over white as ``rgba=True`` does.

        ``cameras`` and ``images`` must be the training views in the reference's training order: frame-major with the
        held-out views removed for technicolor, video-major (each video's frames in order) for neural_3d and immersive.  A
        view's frame is ``int(np.round(time * (num_frames - 1)))`` of its ``Camera.time``; for neural_3d and immersive each
        run of equal ``cam_idx`` is one video, numbered 0, 1, ... in order (the reference numbers videos after removing the
        held-out one).  Any other dataset that sets subsample keys raises ``ValueError``.

        With replacement the reference runs with ``iters_per_epoch = num_iters`` (main.py:100-101), and its epoch-based
        schedules are scaled by that value: an ``INRSystem`` built from the same config must be given
        ``training.iters_per_epoch = num_iters``."""
        training, dataset = cfg["training"], cfg["dataset"]
        replacement = bool(training.get("sample_with_replacement", False))
        num_iters = int(training["num_iters"]) if replacement else None
        name = dataset.get("name", None)
        keys = ("load_full_step", "subsample_keyframe_step", "subsample_keyframe_frac", "subsample_frac")
        cameras = list(cameras)
        subsample = importance = None
        steps = dict(load_full_step=dataset.get("load_full_step", 1),
                     subsample_keyframe_step=dataset.get("subsample_keyframe_step", 1),
                     subsample_keyframe_frac=dataset.get("subsample_keyframe_frac", 1.0),
                     subsample_frac=dataset.get("subsample_frac", 1.0))
        if name in ("technicolor", "neural_3d", "immersive"):
            num_frames = int(dataset.get("num_frames", 1))
            frames = [int(np.round(float(cam.time) * (num_frames - 1))) for cam in cameras]
            videos = None
            if name != "technicolor":
                videos, seen = [], set()
                for i, cam in enumerate(cameras):
                    if i == 0 or cam.cam_idx != cameras[i - 1].cam_idx:
                        if cam.cam_idx in seen:
                            raise ValueError(f"{name} views must be video-major: cam_idx {cam.cam_idx} appears again at "
                                             f"view {i}")
                        seen.add(cam.cam_idx)
                    videos.append(len(seen) - 1)
            if name == "immersive":
                if not cameras:
                    raise ValueError("DeviceRayBatches needs at least one training view")
                try:
                    importance = importance_subsample_plan(frames, videos, height=int(cameras[0].height),
                                                           width=int(cameras[0].width), **steps)
                except ValueError as e:
                    raise ValueError(f"immersive importance_subsample: {e}") from None
            else:
                subsample = regular_subsample_plan(frames, counters=name, videos=videos, **steps)
        elif any(k in dataset for k in keys):
            raise ValueError(f"dataset {name!r} sets {[k for k in keys if k in dataset]}: only technicolor's, neural_3d's "
                             "and immersive's subsets are supported")
        images = _as_image_stack(images)
        rgba = name in ("donerf", "catacaustics") and images.dim() == 4 and images.shape[-1] == 4
        return cls(cameras, images, batch_size=int(training["batch_size"]), seed=seed, c_in=c_in, device=device,
                   replacement=replacement, num_iters=num_iters, subsample=subsample, importance=importance, rgba=rgba)

    def __len__(self) -> int:
        if self.replacement:
            return self.num_iters
        return -(-self.n_rows // self.batch_size)

    def set_epoch(self, epoch: int) -> None:
        self.epoch = int(epoch)

    def batch(self, i: int, with_pixel_ids: bool = False, with_table_ids: bool = False) -> Dict[str, torch.Tensor]:
        """Batch ``i`` of the current epoch (``0 <= i < len(self)``).  ``with_pixel_ids=True`` adds ``'pixel_ids'`` [B] int64, the
        pixel of each row (``view*H*W + y*W + x``), for callers that keep per-pixel state; ``with_table_ids=True`` adds
        ``'table_ids'`` [B] int64, the training-table row of each row."""
        i = int(i)
        if not 0 <= i < len(self):
            raise IndexError(f"batch {i} outside [0, {len(self)})")
        rows = self.batch_size if self.replacement else min(self.batch_size, self.n_rows - i * self.batch_size)
        return self._launch(rows, i, None, with_pixel_ids, with_table_ids)

    def gather_rows(self, table_ids, with_pixel_ids: bool = False) -> Dict[str, torch.Tensor]:
        """The rows of the given training-table indices, in the given order, the table in the reference's ``all_coords``
        order (views in order, each view's kept pixels row-major): for replaying the reference's own sampler indices.  An
        index outside ``[0, n_rows)`` raises ``ValueError`` (for device indices the check synchronises with the device)."""
        ids = self._check_ids(table_ids, self.n_rows, "table ids")
        return self._launch(ids.numel(), 0, ids, with_pixel_ids, False)

    def gather(self, pixel_ids, with_pixel_ids: bool = False) -> Dict[str, torch.Tensor]:
        """The rows of the given pixels, in the given order: for callers that bring their own order (the reference's
        ``np.random.permutation``, say).  An id outside ``[0, n*H*W)`` raises ``ValueError`` (for device ids the check
        synchronises with the device)."""
        ids = self._check_ids(pixel_ids, self.n_pixels, "pixel ids")
        return self._launch(ids.numel(), 0, ids, with_pixel_ids, False, ids_are_pixels=True)

    def __iter__(self):
        for i in range(len(self)):
            yield self.batch(i)

    def _check_ids(self, ids, n: int, what: str) -> torch.Tensor:
        ids = torch.as_tensor(ids)
        name = what.replace(" ", "_")
        if ids.dim() != 1 or ids.numel() < 1:
            raise ValueError(f"{name} must be a non-empty 1-D tensor, got shape {tuple(ids.shape)}")
        if ids.dtype.is_floating_point or ids.dtype == torch.bool or ids.is_complex():
            raise ValueError(f"{name} must be integers, got {ids.dtype}")
        lo, hi = int(ids.min()), int(ids.max())
        if lo < 0 or hi >= n:
            raise ValueError(f"{what} must lie in [0, {n}), got [{lo}, {hi}]")
        return ids.to(device=self.device, dtype=torch.int64).contiguous()

    def _launch(self, rows: int, index: int, ids: Optional[torch.Tensor], with_pixel_ids: bool, with_table_ids: bool,
                ids_are_pixels: bool = False) -> Dict[str, torch.Tensor]:
        """Batch ``index`` of the epoch, or the rows of the explicit ``ids`` (table rows, or pixels with ``ids_are_pixels``).
        Explicit pixels and the permuted batches without a plan go through ``hr_sample_train_batch``, everything else
        through the plan's entry (``hr_sample_train_rows`` or ``hr_sample_train_mask_rows``)."""
        dev = self.device
        whole = ids_are_pixels or (ids is None and not self.replacement and self.subsample is None and
                                   self.importance is None)
        coords = torch.empty((rows, self.c_in), dtype=torch.float32, device=dev)
        rgb = torch.empty((rows, 3), dtype=torch.float32, device=dev)
        weight = torch.empty((rows, 1), dtype=torch.float32, device=dev)
        pids = torch.empty((rows,), dtype=torch.int64, device=dev) if with_pixel_ids or (whole and with_table_ids) else None
        tids = torch.empty((rows,), dtype=torch.int64, device=dev) if with_table_ids and not whole else None
        ptr = lambda t: t.data_ptr() if t is not None else None
        n_rows = C.c_int64(0)
        head = (self.cameras.data_ptr(), self.n_views, self.images.data_ptr(), self.height, self.width, self.c_in)
        fmt = L.PIXEL_RGBA8 if self.rgba else L.PIXEL_RGB8
        head_fmt = (*head[:3], fmt, *head[3:])
        # an explicit list is the whole batch; otherwise the entry shortens the epoch's last batch
        batch = (index, rows if ids is not None else self.batch_size, ptr(ids), coords.data_ptr(), rgb.data_ptr(),
                 weight.data_ptr(), ptr(pids))
        stream = torch.cuda.current_stream(dev).cuda_stream
        with torch.cuda.device(dev):
            if whole:
                L.check(self._lib.hr_sample_train_batch(*head_fmt, self.seed, self.epoch, *batch, C.byref(n_rows), stream))
            else:
                mode = L.SAMPLE_REPLACE if self.replacement else L.SAMPLE_PERMUTE
                tail = (self.n_rows, mode, self.seed, self.epoch, *batch, ptr(tids), C.byref(n_rows), stream)
                if self.importance is None:
                    L.check(self._lib.hr_sample_train_rows(*head_fmt, self._view_start.data_ptr(),
                                                           self._view_rule.data_ptr(), *tail))
                else:
                    L.check(self._lib.hr_sample_train_mask_rows(*head, self._view_start.data_ptr(),
                                                                self._view_slot.data_ptr(), self._block_start.data_ptr(),
                                                                self._masks.data_ptr(), *tail))
        assert n_rows.value == rows, (n_rows.value, rows)
        if whole and with_table_ids:  # without a plan, table ids are pixel ids
            tids = pids.clone() if with_pixel_ids else pids
        out = {"coords": coords, "rgb": rgb, "weight": weight}
        if with_pixel_ids:
            out["pixel_ids"] = pids
        if with_table_ids:
            out["table_ids"] = tids
        return out
