"""Capture-resolution frames to the training resolution on the device (DESIGN.md section 4.4e).

The reference's ``get_rgb`` resizes every decoded frame on the host before ``T.ToTensor()``; ``resize_frames`` does that
resize on the device (``hr_resize_frames``, csrc/hr_resize.cu) into the uint8 ``[n, H, W, 3]`` frames that
``DeviceRayBatches``, ``importance_subsample_plan`` and ``score_views`` take, bit for bit as Pillow or OpenCV computes it.
``dataset_frames`` picks the resizes a dataset's ``get_rgb`` applies::

    frames = torch.from_numpy(decoded).cuda()        # uint8 [n, H0, W0, 3] at the capture size
    train = hb.dataset_frames(cfg.dataset, frames)   # uint8 [n, H, W, 3] at img_wh, as get_rgb makes them

DoNeRF and Catacaustics load RGBA and composite it over white after the resize, in fp32.  For them ``dataset_frames`` takes
and returns uint8 RGBA ``[n, H, W, 4]``, resized as their ``get_rgb`` resizes it, and the composite is computed where the
colour is consumed: ``DeviceRayBatches(..., rgba=True)`` and ``score_views(..., rgba=True)``.
"""
from __future__ import annotations

from typing import Optional, Sequence

import torch

from . import lib as L
from .lightfield import _get

METHODS = tuple(L.RESIZE_METHODS)

# dataset name -> (first step to _img_wh, second step to img_wh when scale() made it differ), as each get_rgb resizes
_PIL = ("pil_lanczos", "pil_box")
# the cv2 datasets pass their interpolation flag in cv2.resize's `dst` slot: both steps run OpenCV's default INTER_LINEAR
_CV2 = ("cv2_linear", "cv2_linear")
DATASET_RESIZE = {"technicolor": _PIL, "llff": _PIL, "dense_llff": _PIL, "shiny": _PIL, "dense_shiny": _PIL, "spaces": _PIL,
                  "stanford": _PIL, "stanford_llff": _PIL, "stanford_epi": _PIL, "neural_3d": _CV2, "immersive": _CV2}
# the RGBA datasets: their frames stay RGBA through the resize, composited over white where the colour is consumed.
# donerf.py: cv2.resize(INTER_AREA, as a keyword) on the 4-channel array, twice; catacaustics.py: Image.resize with
# Pillow's default filter (BICUBIC), then BOX, each call on the RGBA image, so each resamples premultiplied RGBa.
RGBA_RESIZE = {"donerf": ("cv2_area", "cv2_area"), "catacaustics": ("pil_bicubic", "pil_box")}
_RGBA_NEEDED = {
    "donerf": "donerf loads RGBA frames and composites rgb * a + (1 - a) in fp32 after the resize (datasets/donerf.py)",
    "catacaustics": "catacaustics loads RGBA frames, resizes them premultiplied with Pillow's default filter (BICUBIC) and "
                    "composites rgb * a + (1 - a) in fp32 after the resize (datasets/catacaustics.py)",
}


def resize_frames(frames: torch.Tensor, size: Sequence[int], method: str, bgr: bool = False,
                  out: Optional[torch.Tensor] = None, stream=None, *, rgba: bool = False) -> torch.Tensor:
    """uint8 ``[n, H0, W0, 3]`` (or one ``[H0, W0, 3]`` frame) on the device -> uint8 ``[n, H, W, 3]`` RGB, ``size = (W, H)``
    as Pillow and OpenCV take it, in one call that never synchronises (hr_resize_frames).

    ``method``: ``pil_lanczos``, ``pil_bicubic``, ``pil_box`` (``Image.resize`` with that filter) or ``cv2_linear``,
    ``cv2_area`` (``cv2.resize`` with INTER_LINEAR / INTER_AREA), each frame bit for bit the library's result.  Reductions
    only; ``cv2_area`` at integer factors only.  A frame of the same size is copied.  ``bgr``: the frames are BGR, as OpenCV
    decodes them (the reference's ``cvtColor(BGR2RGB)``).  ``out``: a CUDA uint8 tensor of shape ``[n, H, W, 3]`` whose rows
    are contiguous and whose frames are ``H`` rows apart (a contiguous tensor or a slice of one along the frame axis, e.g.
    ``train[i:i + n]``), written in place.  The work goes on ``stream`` (default the current stream), including the copy
    that makes non-contiguous ``frames`` contiguous; as with any side stream, the caller orders ``stream`` after the work
    that wrote ``frames`` (``stream.wait_stream(torch.cuda.current_stream())``).

    ``rgba=True``: the frames are uint8 RGBA ``[n, H0, W0, 4]`` (BGRA with ``bgr``) and the result is RGBA ``[n, H, W, 4]``,
    as the RGBA datasets resize them: the Pillow methods resample the premultiplied image and convert back, as
    ``Image.resize`` does for an RGBA image; ``cv2_area`` resamples the four channels independently, as ``cv2.resize``
    does.  ``cv2_linear`` is not supported for RGBA."""
    if method not in L.RESIZE_METHODS:
        raise ValueError(f"resize_frames: unknown method {method!r}; one of {METHODS}")
    ch = 4 if rgba else 3
    if not isinstance(frames, torch.Tensor) or frames.dtype != torch.uint8 or frames.dim() not in (3, 4) \
            or frames.shape[-1] != ch:
        got = f"{frames.dtype} {tuple(frames.shape)}" if isinstance(frames, torch.Tensor) else type(frames).__name__
        raise ValueError(f"resize_frames: frames must be a uint8 tensor [n, H, W, {ch}] or [H, W, {ch}]"
                         f"{' (rgba=True)' if rgba else ''}, got {got}")
    if rgba and method == "cv2_linear":
        raise ValueError("resize_frames: cv2_linear is not supported for RGBA frames (no dataset resizes RGBA with it)")
    if not frames.is_cuda:
        raise RuntimeError("hyperreel_b200 resizes frames on an H100 only: frames must be a CUDA tensor (no CPU fallback)")
    single = frames.dim() == 3
    src = frames.unsqueeze(0) if single else frames
    n, H0, W0 = (int(v) for v in src.shape[:3])
    W, H = (int(v) for v in size)
    lib = L.load_library()
    m = L.RESIZE_METHODS[method]
    fmt = L.PIXEL_RGBA8 if rgba else L.PIXEL_RGB8
    need = int(lib.hr_resize_workspace_bytes(n, H0, W0, H, W, m, fmt))
    dev = src.device
    given = out is not None
    if given:
        row = _row_stride(out, n, H, W, ch)
        if row is None or out.device != dev:
            got = f"{out.dtype} {tuple(out.shape)} strides {out.stride()} on {out.device}" \
                if isinstance(out, torch.Tensor) else type(out).__name__
            raise ValueError(f"resize_frames: out must be a CUDA uint8 tensor of shape {(n, H, W, ch)} on {dev} with "
                             f"contiguous rows and frames H rows apart, got {got}")
    stream = stream if stream is not None else torch.cuda.current_stream(dev)
    with torch.cuda.stream(stream):  # the contiguous copy, the scratch and a new out are made on and belong to that stream
        src = src.contiguous()
        ws = torch.empty(max(need, 0), dtype=torch.uint8, device=dev)
        if out is None:
            out, row = torch.empty((n, H, W, ch), dtype=torch.uint8, device=dev), ch * W
        L.check(lib.hr_resize_frames(src.data_ptr(), n, H0, W0, out.data_ptr(), H, W, row, m, L.RESIZE_BGR if bgr else 0, fmt,
                                     ws.data_ptr() if need > 0 else None, max(need, 0), stream.cuda_stream))
    return out[0] if single and not given else out


def _row_stride(t, n: int, H: int, W: int, ch: int = 3) -> Optional[int]:
    """Bytes between the starts of rows of ``t`` (``ch`` channels) if frame f's row y starts at (f * H + y) rows, else
    None."""
    if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.uint8 and tuple(t.shape) == (n, H, W, ch)):
        return None
    if t.stride(3) != 1 or (W > 1 and t.stride(2) != ch):
        return None
    if H > 1:
        row = t.stride(1)
        if n > 1 and t.stride(0) != H * row:
            return None
    else:
        row = t.stride(0) if n > 1 else ch * W
    return int(row) if row >= ch * W else None


def dataset_steps(dataset_cfg, capture_wh: Sequence[int], scale: int = 1):
    """The resizes the ``get_rgb`` of the config's dataset (``name``, ``img_wh``) applies to a frame of ``capture_wh``
    (W, H) at the reference's ``scale()`` factor: a list of ``(method, (W, H))``, empty when the frame is kept as it is."""
    name = _get(dataset_cfg, "name", None)
    if name not in DATASET_RESIZE and name not in RGBA_RESIZE:
        raise ValueError(f"dataset_frames: no get_rgb resize restated for dataset {name!r}; supported: "
                         f"{sorted(DATASET_RESIZE) + sorted(RGBA_RESIZE)}")
    img_wh = _get(dataset_cfg, "img_wh", None)
    if img_wh is None or len(img_wh) != 2:
        raise ValueError(f"dataset_frames: the dataset config needs img_wh = [W, H], got {img_wh!r}")
    wh0 = (int(img_wh[0]), int(img_wh[1]))
    scale = int(scale)
    if scale < 1:
        raise ValueError(f"dataset_frames: scale must be a positive integer, got {scale}")
    wh = (wh0[0] // scale, wh0[1] // scale)  # BaseDataset.scale
    first, second = DATASET_RESIZE[name] if name in DATASET_RESIZE else RGBA_RESIZE[name]
    steps = []
    if tuple(int(v) for v in capture_wh) != wh0:
        steps.append((first, wh0))
    if wh != wh0:
        steps.append((second, wh))
    return steps


def dataset_frames(dataset_cfg, frames: torch.Tensor, out: Optional[torch.Tensor] = None, bgr: bool = False, scale: int = 1,
                   stream=None) -> torch.Tensor:
    """Decoded frames (uint8 ``[n, H0, W0, 3]`` on the device, RGB, or BGR with ``bgr=True``) -> the uint8 frames the
    reference's ``get_rgb`` makes of them for the config's dataset (``name``, ``img_wh``; ``scale`` is the reference's
    ``scale()`` factor, 1 unless a multi-scale schedule reduced img_wh), before ``T.ToTensor()``: ``get_rgb(...) * 255``
    exactly.

    technicolor, llff (and dense_llff, shiny, dense_shiny), spaces and the stanford datasets: Pillow LANCZOS to img_wh,
    then BOX to img_wh // scale.  neural_3d and immersive: cv2.resize to img_wh, then to img_wh // scale, both with
    OpenCV's default INTER_LINEAR (their interpolation flag is passed as cv2.resize's `dst` argument), which OpenCV runs as
    INTER_AREA at exactly 2x.  A step whose size matches is the identity.  ``out`` as in ``resize_frames``.

    donerf and catacaustics load RGBA: ``frames`` are uint8 RGBA ``[n, H0, W0, 4]`` and the result is RGBA ``[n, H, W, 4]``,
    ``get_rgb``'s frame before ``T.ToTensor()`` and the composite over white, which ``DeviceRayBatches(..., rgba=True)`` and
    ``score_views(..., rgba=True)`` compute (4 bytes per pixel held instead of 12).  donerf: ``cv2.resize`` INTER_AREA to
    img_wh, then to img_wh // scale (integer factors only).  catacaustics: Pillow BICUBIC to img_wh, then BOX to
    img_wh // scale, each on the premultiplied image as ``Image.resize`` resamples RGBA."""
    if not isinstance(frames, torch.Tensor) or frames.dim() != 4:
        raise ValueError("dataset_frames: frames must be a uint8 tensor [n, H, W, 3]")
    name = _get(dataset_cfg, "name", None)
    rgba = name in RGBA_RESIZE
    if rgba and frames.shape[-1] != 4:
        raise ValueError(f"dataset_frames: {_RGBA_NEEDED[name]}: frames must be uint8 RGBA [n, H0, W0, 4], got "
                         f"{tuple(frames.shape)}")
    steps = dataset_steps(dataset_cfg, (int(frames.shape[2]), int(frames.shape[1])), scale)
    if not steps:
        W, H = int(frames.shape[2]), int(frames.shape[1])
        steps = [("cv2_area", (W, H))]  # the copy (and the channel swap)
    x = frames
    for i, (method, wh) in enumerate(steps):
        last = i == len(steps) - 1
        x = resize_frames(x, wh, method, bgr=bgr and i == 0, out=out if last else None, stream=stream, rgba=rgba)
    return x
