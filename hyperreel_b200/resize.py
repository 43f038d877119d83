"""Capture-resolution frames to the training resolution on the device (DESIGN.md section 4.4e).

The reference's ``get_rgb`` resizes every decoded frame on the host before ``T.ToTensor()``; ``resize_frames`` does that
resize on the device (``hr_resize_frames``, csrc/hr_resize.cu) into the uint8 ``[n, H, W, 3]`` frames that
``DeviceRayBatches``, ``importance_subsample_plan`` and ``score_views`` take, bit for bit as Pillow or OpenCV computes it.
``dataset_frames`` picks the resizes a dataset's ``get_rgb`` applies::

    frames = torch.from_numpy(decoded).cuda()        # uint8 [n, H0, W0, 3] at the capture size
    train = hb.dataset_frames(cfg.dataset, frames)   # uint8 [n, H, W, 3] at img_wh, as get_rgb makes them
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
_REFUSED = {
    "donerf": "donerf loads RGBA frames and composites rgb * a + (1 - a) in fp32 after the resize (datasets/donerf.py), a "
              "ground truth no uint8 frame holds",
    "catacaustics": "catacaustics loads RGBA frames and composites rgb * a + (1 - a) in fp32 after the resize, and its "
                    "first resize is Pillow's default filter (BICUBIC), so no uint8 frame holds its ground truth",
}


def resize_frames(frames: torch.Tensor, size: Sequence[int], method: str, bgr: bool = False,
                  out: Optional[torch.Tensor] = None, stream=None) -> torch.Tensor:
    """uint8 ``[n, H0, W0, 3]`` (or one ``[H0, W0, 3]`` frame) on the device -> uint8 ``[n, H, W, 3]`` RGB, ``size = (W, H)``
    as Pillow and OpenCV take it, in one call that never synchronises (hr_resize_frames).

    ``method``: ``pil_lanczos``, ``pil_bicubic``, ``pil_box`` (``Image.resize`` with that filter) or ``cv2_linear``,
    ``cv2_area`` (``cv2.resize`` with INTER_LINEAR / INTER_AREA), each frame bit for bit the library's result.  Reductions
    only; ``cv2_area`` at integer factors only.  A frame of the same size is copied.  ``bgr``: the frames are BGR, as OpenCV
    decodes them (the reference's ``cvtColor(BGR2RGB)``).  ``out``: a CUDA uint8 tensor of shape ``[n, H, W, 3]`` whose rows
    are contiguous and whose frames are ``H`` rows apart (a contiguous tensor or a slice of one along the frame axis, e.g.
    ``train[i:i + n]``), written in place.  The work goes on ``stream`` (default the current stream), including the copy
    that makes non-contiguous ``frames`` contiguous; as with any side stream, the caller orders ``stream`` after the work
    that wrote ``frames`` (``stream.wait_stream(torch.cuda.current_stream())``)."""
    if method not in L.RESIZE_METHODS:
        raise ValueError(f"resize_frames: unknown method {method!r}; one of {METHODS}")
    if not isinstance(frames, torch.Tensor) or frames.dtype != torch.uint8 or frames.dim() not in (3, 4) \
            or frames.shape[-1] != 3:
        got = f"{frames.dtype} {tuple(frames.shape)}" if isinstance(frames, torch.Tensor) else type(frames).__name__
        raise ValueError(f"resize_frames: frames must be a uint8 tensor [n, H, W, 3] or [H, W, 3], got {got}")
    if not frames.is_cuda:
        raise RuntimeError("hyperreel_b200 resizes frames on an H100 only: frames must be a CUDA tensor (no CPU fallback)")
    single = frames.dim() == 3
    src = frames.unsqueeze(0) if single else frames
    n, H0, W0 = (int(v) for v in src.shape[:3])
    W, H = (int(v) for v in size)
    lib = L.load_library()
    m = L.RESIZE_METHODS[method]
    need = int(lib.hr_resize_workspace_bytes(n, H0, W0, H, W, m))
    dev = src.device
    given = out is not None
    if given:
        row = _row_stride(out, n, H, W)
        if row is None or out.device != dev:
            got = f"{out.dtype} {tuple(out.shape)} strides {out.stride()} on {out.device}" \
                if isinstance(out, torch.Tensor) else type(out).__name__
            raise ValueError(f"resize_frames: out must be a CUDA uint8 tensor of shape {(n, H, W, 3)} on {dev} with "
                             f"contiguous rows and frames H rows apart, got {got}")
    stream = stream if stream is not None else torch.cuda.current_stream(dev)
    with torch.cuda.stream(stream):  # the contiguous copy, the scratch and a new out are made on and belong to that stream
        src = src.contiguous()
        ws = torch.empty(max(need, 0), dtype=torch.uint8, device=dev)
        if out is None:
            out, row = torch.empty((n, H, W, 3), dtype=torch.uint8, device=dev), 3 * W
        L.check(lib.hr_resize_frames(src.data_ptr(), n, H0, W0, out.data_ptr(), H, W, row, m, L.RESIZE_BGR if bgr else 0,
                                     ws.data_ptr() if need > 0 else None, max(need, 0), stream.cuda_stream))
    return out[0] if single and not given else out


def _row_stride(t, n: int, H: int, W: int) -> Optional[int]:
    """Bytes between the starts of rows of ``t`` if frame f's row y starts at (f * H + y) rows, else None."""
    if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.uint8 and tuple(t.shape) == (n, H, W, 3)):
        return None
    if t.stride(3) != 1 or (W > 1 and t.stride(2) != 3):
        return None
    if H > 1:
        row = t.stride(1)
        if n > 1 and t.stride(0) != H * row:
            return None
    else:
        row = t.stride(0) if n > 1 else 3 * W
    return int(row) if row >= 3 * W else None


def dataset_steps(dataset_cfg, capture_wh: Sequence[int], scale: int = 1):
    """The resizes the ``get_rgb`` of the config's dataset (``name``, ``img_wh``) applies to a frame of ``capture_wh``
    (W, H) at the reference's ``scale()`` factor: a list of ``(method, (W, H))``, empty when the frame is kept as it is."""
    name = _get(dataset_cfg, "name", None)
    if name in _REFUSED:
        raise ValueError(f"dataset_frames: {_REFUSED[name]}")
    if name not in DATASET_RESIZE:
        raise ValueError(f"dataset_frames: no get_rgb resize restated for dataset {name!r}; supported: "
                         f"{sorted(DATASET_RESIZE)}")
    img_wh = _get(dataset_cfg, "img_wh", None)
    if img_wh is None or len(img_wh) != 2:
        raise ValueError(f"dataset_frames: the dataset config needs img_wh = [W, H], got {img_wh!r}")
    wh0 = (int(img_wh[0]), int(img_wh[1]))
    scale = int(scale)
    if scale < 1:
        raise ValueError(f"dataset_frames: scale must be a positive integer, got {scale}")
    wh = (wh0[0] // scale, wh0[1] // scale)  # BaseDataset.scale
    first, second = DATASET_RESIZE[name]
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
    INTER_AREA at exactly 2x.  A step whose size matches is the identity.  donerf and catacaustics are refused: their
    ground truth is an fp32 alpha composite no uint8 frame holds.  ``out`` as in ``resize_frames``."""
    if not isinstance(frames, torch.Tensor) or frames.dim() != 4:
        raise ValueError("dataset_frames: frames must be a uint8 tensor [n, H, W, 3]")
    steps = dataset_steps(dataset_cfg, (int(frames.shape[2]), int(frames.shape[1])), scale)
    if not steps:
        W, H = int(frames.shape[2]), int(frames.shape[1])
        steps = [("cv2_area", (W, H))]  # the copy (and the channel swap)
    x = frames
    for i, (method, wh) in enumerate(steps):
        last = i == len(steps) - 1
        x = resize_frames(x, wh, method, bgr=bgr and i == 0, out=out if last else None, stream=stream)
    return x
