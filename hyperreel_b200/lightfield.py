"""The Stanford light-field dataset's views as ``TwoPlaneCamera``s (``name: stanford``, StanfordLightfieldDataset,
datasets/stanford.py, on LightfieldDataset, datasets/lightfield.py).

``lightfield_cameras`` lists a split's views in the reference's order with the positions and scales its ``get_coords``
passes to ``get_lightfield_rays``; ``stanford_file_coords`` parses the camera positions out of the image file names as
``read_meta`` does when ``lightfield.use_file_coords`` is set.  Both restate the reference in Python double arithmetic, the
arithmetic it uses, and ``TwoPlaneCamera`` rounds the results to float32 as its tensors do.

The reference's training split cannot be built: ``LightfieldDataset.prepare_train_data`` stops at a debug ``exit()``
(datasets/lightfield.py:118-120) before its first view is stored.  The ``train`` order here is the loop as written above
that line (rows ``range(start_row, end_row, step)``, columns likewise, ``val_pairs`` skipped); it is not checked against a
run of the reference.  The ``val``, ``test`` and ``render`` orders are ``prepare_test_data`` and ``prepare_render_data``.
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import numpy as np

from .camera import TwoPlaneCamera

SPLITS = ("train", "val", "test", "render")

# read_meta's second file-name pattern: "<prefix>_<row>_<col>_<y>_<x>.png" with y negated (datasets/stanford.py:70-74)
_NEGATED_Y = ("beans", "knights", "tarot", "tarot_small")


def _get(cfg, key, default=None):
    if cfg is None:
        return default
    if isinstance(cfg, dict):
        return cfg.get(key, default)
    return getattr(cfg, key, default)


def stanford_file_coords(filenames: Sequence[str], collection: str) -> List[Tuple[float, float]]:
    """The camera positions (x, y) of StanfordLightfieldDataset.read_meta (datasets/stanford.py:50-80), one per image in
    sorted file-name order (the order of its ``image_paths``).  For the beans, knights, tarot and tarot_small collections
    the last two ``_`` fields are y and x with y negated; otherwise the two fields before the last are y and x."""
    coords = []
    for name in sorted(filenames):
        if collection in _NEGATED_Y:
            yx = name.split("_")[-2:]
            if len(yx) != 2:
                raise ValueError(f"stanford_file_coords: cannot read a camera position from {name!r}")
            y, x = -float(yx[0]), float(yx[1].split(".png")[0])
        else:
            yx = name.split("_")[-3:-1]
            if len(yx) != 2:
                raise ValueError(f"stanford_file_coords: cannot read a camera position from {name!r}")
            y, x = float(yx[0]), float(yx[1])
        coords.append((x, y))
    return coords


def _normalize_coord(coords, coord):
    """StanfordLightfieldDataset.normalize_coord (datasets/stanford.py:95-106) over every image's position."""
    xs, ys = [c[0] for c in coords], [c[1] for c in coords]
    x0, x1, y0, y1 = np.min(xs), np.max(xs), np.min(ys), np.max(ys)
    aspect = (x1 - x0) / (y1 - y0)
    norm_x = ((coord[0] - x0) / (x1 - x0)) * 2 - 1
    norm_y = (((coord[1] - y0) / (y1 - y0)) * 2 - 1) / aspect
    return norm_x, norm_y


def lightfield_cameras(dataset_cfg, width: int, height: int, split: str,
                       file_coords: Optional[Sequence[Tuple[float, float]]] = None) -> List[TwoPlaneCamera]:
    """The views of ``split`` (train, val, test or render) of a ``name: stanford`` dataset config, in the reference's order.

    ``dataset_cfg`` is the config's ``dataset`` section (a dict or attribute object, with the split's own section used
    when it has one, as the reference does); ``width`` x ``height`` is the views' size, the dataset's ``img_wh``, which
    also gives the aspect.  ``file_coords`` are ``stanford_file_coords`` of the dataset's image names: with
    ``lightfield.use_file_coords`` the train, val and test views sit at those positions (normalize_coord), and the render
    views always sit on the row/column grid (``__getitem__`` calls LightfieldDataset.get_coords for that split).

    - train: rows ``range(start_row, end_row, step)``, columns likewise, ``val_pairs`` skipped; see the module docstring.
    - val / test: prepare_test_data (datasets/lightfield.py:151-163), truncated as ``__len__`` counts them: val to
      ``min(val_num, num_test_images)``, test to ``num_test_images``.
    - render: prepare_render_data (:165-183), ``cols * supersample`` views along ``disp_row`` or the two-turn 120-view
      spiral of radius ``spiral_rad``, at ``vis_st_scale`` / ``vis_uv_scale``.
    ``keyframe_step != -1`` with ``keyframe_subsample != 1`` (an unseeded random subset of each training view) raises
    ``ValueError``."""
    if split not in SPLITS:
        raise ValueError(f"lightfield_cameras: split must be one of {SPLITS}, got {split!r}")
    if _get(dataset_cfg, "name", "stanford") != "stanford":
        raise ValueError(f"lightfield_cameras: expected a stanford dataset config, got name {_get(dataset_cfg, 'name')!r}")
    width, height = int(width), int(height)
    top_lf = _get(dataset_cfg, "lightfield")
    dcfg = _get(dataset_cfg, split, None) or dataset_cfg
    lf = _get(dcfg, "lightfield")
    if lf is None:
        raise ValueError("lightfield_cameras: the dataset config has no lightfield section")
    rows, cols, step = int(lf["rows"]), int(lf["cols"]), int(lf["step"])
    start_row, end_row = int(_get(lf, "start_row", 0)), int(_get(lf, "end_row", rows))
    start_col, end_col = int(_get(lf, "start_col", 0)), int(_get(lf, "end_col", cols))
    st_scale, uv_scale = _get(lf, "st_scale", 1.0), _get(lf, "uv_scale", 1.0)
    near, far = _get(lf, "near", -1.0), _get(lf, "far", 0.0)
    vis_st = _get(lf, "vis_st_scale", None)
    vis_st = st_scale if vis_st is None else vis_st
    vis_uv = _get(lf, "vis_uv_scale", None)
    vis_uv = uv_scale if vis_uv is None else vis_uv
    keyframe_step, keyframe_subsample = _get(lf, "keyframe_step", -1), _get(lf, "keyframe_subsample", 1)
    if keyframe_step != -1 and keyframe_subsample != 1:
        raise ValueError("lightfield_cameras: keyframe_step with keyframe_subsample != 1 keeps an unseeded random subset of "
                         "each non-keyframe training view (np.random.permutation), which cannot be reproduced")
    val_all = bool(_get(dcfg, "val_all", False)) or step == 1
    flat = list(_get(dcfg, "val_pairs", []) or [])
    val_pairs = list(zip(flat[::2], flat[1::2]))
    use_file_coords = bool(_get(top_lf, "use_file_coords", False))
    if file_coords is not None and not use_file_coords:
        raise ValueError("lightfield_cameras: file_coords given but the config does not set lightfield.use_file_coords")
    if use_file_coords and split != "render" and file_coords is None:
        raise ValueError("lightfield_cameras: the config sets lightfield.use_file_coords: pass file_coords "
                         "(stanford_file_coords of the dataset's image file names)")
    aspect = float(width) / height

    def grid(st_idx):  # LightfieldDataset.get_coord (datasets/lightfield.py:185-191)
        s = (st_idx[0] / (cols - 1)) * 2 - 1 if cols > 1 else 0
        t = -(((st_idx[1] / (rows - 1)) * 2 - 1) if rows > 1 else 0)
        return s, t

    def view(st_idx, render):
        if render:
            (s, t), st, uv = grid(st_idx), vis_st, vis_uv
        elif use_file_coords:
            idx = st_idx[1] * cols + st_idx[0]
            if not 0 <= idx < len(file_coords):
                raise ValueError(f"lightfield_cameras: view (s, t) = {st_idx} is image {idx}, but {len(file_coords)} file "
                                 "coordinates were given")
            (s, t), st, uv = _normalize_coord(file_coords, file_coords[idx]), st_scale, uv_scale
        else:
            (s, t), st, uv = grid(st_idx), st_scale, uv_scale
        return TwoPlaneCamera(width, height, s, t, st_scale=st, uv_scale=uv, near=near, far=far, aspect=aspect)

    if split == "train":
        idx = [(s, t) for t in range(start_row, end_row, step) for s in range(start_col, end_col, step)
               if (s, t) not in val_pairs]
        return [view(i, False) for i in idx]
    if split in ("val", "test"):
        idx = []
        for t in range(start_row, end_row):
            for s in range(start_col, end_col):
                if not val_pairs:
                    if t % step == 0 and s % step == 0 and not val_all:
                        continue
                elif (s, t) not in val_pairs:
                    continue
                idx.append((s, t))
        # __len__ (datasets/lightfield.py:230-240): val stops at min(val_num, num_test_images), test at num_test_images,
        # which undercounts the views off the step grid when the range does not end on it
        num_rows = (end_row - start_row) // step + (1 if step > 1 else 0)
        num_cols = (end_col - start_col) // step + (1 if step > 1 else 0)
        if val_pairs:
            num_test = len(val_pairs)
        elif val_all:
            num_test = (end_row - start_row) * (end_col - start_col)
        else:
            num_test = (end_row - start_row) * (end_col - start_col) - num_rows * num_cols
        n = min(int(_get(dcfg, "val_num")), num_test) if split == "val" else num_test
        idx = idx[:max(0, n)]
        return [view(i, False) for i in idx]
    # render
    rp = _get(dcfg, "render_params", {}) or {}
    disp_row, supersample = lf["disp_row"], int(lf["supersample"])
    if not _get(rp, "spiral", False):
        idx = [(s / supersample, disp_row) for s in range(cols * supersample)]
    else:
        scale = _get(rp, "spiral_rad", 0.5)
        idx = []
        for theta in np.linspace(0.0, 2.0 * np.pi * 2, 120 + 1)[:-1]:
            s = (np.cos(theta) * scale + 1) / 2.0 * (cols - 1)
            t = -np.sin(theta) * scale / 2.0 * (rows - 1) + ((rows - 1) - disp_row)
            idx.append((s, t))
    return [view(i, True) for i in idx]
