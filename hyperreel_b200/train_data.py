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
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional, Sequence

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


class DeviceRayBatches:
    """Shuffled training batches ``{'coords' [B, c_in], 'rgb' [B, 3], 'weight' [B, 1]}`` (fp32, on the device) over every
    pixel of the training views, generated on the device per batch.

    ``cameras``: one ``Camera`` per view, each of the images' size.  ``images``: uint8 ``[n, H, W, 3]`` (or a sequence of
    ``[H, W, 3]`` of one size), on the host or the device; uploaded once.  An epoch visits each of the ``n*H*W`` pixels exactly
    once, in an order fixed by ``(seed, epoch)``; batches are consecutive ``batch_size`` pieces of that order and the last one
    is short, like the reference's last slice.  ``set_epoch(e)`` selects the order (0 at construction); ``len()`` is the
    number of batches per epoch and iterating yields them in turn.

    Only the reference's default training mode is provided.  The dataset options of the others (datasets/base.py:85-101)
    are accepted under the reference's names so that they can be refused: ``use_patches``, ``precrop_iters`` > 0 (crop),
    ``use_full_image`` and ``blur_radius`` > 0 raise ``ValueError``, as do views of different sizes and non-uint8 images."""

    def __init__(self, cameras: Sequence[Camera], images, batch_size: int, seed: int = 0, c_in: int = 8,
                 device: Optional[torch.device] = None, *, use_patches: bool = False, precrop_iters: int = 0,
                 use_full_image: bool = False, blur_radius: int = 0):
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
        if images.dim() != 4 or images.shape[-1] != 3:
            raise ValueError(f"images must be [n, H, W, 3], got {tuple(images.shape)}")
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

    def __len__(self) -> int:
        return -(-self.n_pixels // self.batch_size)

    def set_epoch(self, epoch: int) -> None:
        self.epoch = int(epoch)

    def batch(self, i: int, with_pixel_ids: bool = False) -> Dict[str, torch.Tensor]:
        """Batch ``i`` of the current epoch (``0 <= i < len(self)``).  ``with_pixel_ids=True`` adds ``'pixel_ids'`` [B] int64, the
        pixel of each row (``view*H*W + y*W + x``), for callers that keep per-pixel state."""
        i = int(i)
        if not 0 <= i < len(self):
            raise IndexError(f"batch {i} outside [0, {len(self)})")
        rows = min(self.batch_size, self.n_pixels - i * self.batch_size)
        return self._launch(rows, i, None, with_pixel_ids)

    def gather(self, pixel_ids, with_pixel_ids: bool = False) -> Dict[str, torch.Tensor]:
        """The rows of the given pixels, in the given order: for callers that bring their own order (the reference's
        ``np.random.permutation``, say).  An id outside ``[0, n*H*W)`` raises ``ValueError`` (for device ids the check
        synchronises with the device)."""
        ids = torch.as_tensor(pixel_ids)
        if ids.dim() != 1 or ids.numel() < 1:
            raise ValueError(f"pixel_ids must be a non-empty 1-D tensor, got shape {tuple(ids.shape)}")
        if ids.dtype.is_floating_point or ids.dtype == torch.bool or ids.is_complex():
            raise ValueError(f"pixel_ids must be integers, got {ids.dtype}")
        lo, hi = int(ids.min()), int(ids.max())
        if lo < 0 or hi >= self.n_pixels:
            raise ValueError(f"pixel ids must lie in [0, {self.n_pixels}), got [{lo}, {hi}]")
        ids = ids.to(device=self.device, dtype=torch.int64).contiguous()
        return self._launch(ids.numel(), 0, ids, with_pixel_ids)

    def __iter__(self):
        for i in range(len(self)):
            yield self.batch(i)

    def _launch(self, rows: int, index: int, order: Optional[torch.Tensor], with_ids: bool) -> Dict[str, torch.Tensor]:
        dev = self.device
        coords = torch.empty((rows, self.c_in), dtype=torch.float32, device=dev)
        rgb = torch.empty((rows, 3), dtype=torch.float32, device=dev)
        weight = torch.empty((rows, 1), dtype=torch.float32, device=dev)
        ids = torch.empty((rows,), dtype=torch.int64, device=dev) if with_ids else None
        n_rows = C.c_int64(0)
        with torch.cuda.device(dev):
            L.check(self._lib.hr_sample_train_batch(
                self.cameras.data_ptr(), self.n_views, self.images.data_ptr(), self.height, self.width, self.c_in, self.seed,
                self.epoch, index, rows if order is not None else self.batch_size,
                order.data_ptr() if order is not None else None, coords.data_ptr(), rgb.data_ptr(), weight.data_ptr(),
                ids.data_ptr() if ids is not None else None, C.byref(n_rows), torch.cuda.current_stream(dev).cuda_stream))
        assert n_rows.value == rows, (n_rows.value, rows)
        out = {"coords": coords, "rgb": rgb, "weight": weight}
        if ids is not None:
            out["pixel_ids"] = ids
        return out
