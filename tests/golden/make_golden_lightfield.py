"""Golden rays and view lists of the Stanford light-field dataset (two-plane rays), from the unmodified reference run on
CPU through the shim on stand-in dataset objects (no images are read).

    HYPERREEL_REFERENCE=<reference checkout> python tests/golden/make_golden_lightfield.py

writes ``tests/golden/lightfield_rays.npz`` and ``tests/golden/lightfield_views.npz``.

* ``lightfield_rays.npz``, per case ``<case>/...``: ``rays`` [n, 6] fp32, the rows of ``pixels`` (row-major pixel ids, every
  pixel but for the 1024 x 1024 case, which keeps a strided subset) of ``LightfieldDataset.get_coords``
  (datasets/lightfield.py:193-219, which calls ``get_lightfield_rays``, utils/ray_utils.py:14-45) on an object whose
  attributes are set directly; ``params`` [W, H, s, t, st_scale, uv_scale, near, far, aspect] float64, the numbers it passes.
* ``lightfield_views.npz``, per case ``<case>/...``: ``config`` (the dataset section as JSON), ``files`` (image names),
  ``split``, ``st_idx`` [F, 2] float64 (``all_st_idx`` in order, truncated to ``len(dataset)``), ``pos`` [F, 2] float64 (the
  s, t the reference passes to get_lightfield_rays: ``get_coord``, or ``normalize_coord`` of the file positions),
  ``scales`` [F, 2] (st_scale, uv_scale passed), ``rays`` [F, H*W, 6] fp32 as ``__getitem__`` makes them, ``file_coords``
  [N, 2] float64 (``camera_coords`` of read_meta, empty unless use_file_coords).  The dataset is built by the reference's own
  ``StanfordLightfieldDataset.__init__`` / ``LightfieldDataset.__init__`` with the base class's constructor replaced by one
  that sets the attributes they read (img_wh, aspect, val_num, the split) and calls ``prepare_data``, so ``read_meta`` parses
  the file names from a stand-in listing and ``prepare_test_data`` / ``prepare_render_data`` run unmodified.  The training
  split is not built: ``prepare_train_data`` calls ``exit()`` (datasets/lightfield.py:118-120).
"""
import contextlib
import io
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from tests.golden.make_golden_subsample import _install  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))

# name: (W, H, s, t, st_scale, uv_scale, near, far, aspect, split, stride of the stored pixel subset)
RAY_CASES = {
    "odd_37x23": (37, 23, 0.375, -0.625, 1.0, 1.0, -1.0, 0.0, 1.75, "train", 1),      # aspect != W / H
    "w1_1x9": (1, 9, -0.25, 0.5, 0.25, 1.0, -1.0, 0.0, 1.0 / 9.0, "train", 1),        # one-step linspace in u
    "h1_9x1": (9, 1, 0.75, -1.0, 0.25, 1.0, -1.0, 0.0, 9.0, "train", 1),              # and in v
    "st0125_33x17": (33, 17, -0.875, 0.125, 0.125, 1.0, -1.0, 0.0, 33.0 / 17.0, "val", 1),
    "st025_24x16": (24, 16, 1.0 / 3.0, -0.1, 0.25, 1.0, -1.0, 0.0, 1.5, "val", 1),
    "planes_20x14": (20, 14, 0.3, 0.7, 0.25, 0.7, -1.5, 0.25, 20.0 / 14.0, "val", 1),  # uv_scale, near, far
    # a render-sweep view between grid columns: (s_idx, t_idx) = (3.5, 2) of a 9 x 9 grid through get_coord
    "render_frac_16x12": (16, 12, None, None, 0.1, 1.0, -1.0, 0.0, 16.0 / 12.0, "render", 1),
    "big_1024x1024": (1024, 1024, -0.4375, 0.8125, 0.125, 1.0, -1.0, 0.0, 1.0, "train", 1009),
}


def _grid_files(rows, cols, negated):
    """Stand-in image names in the two patterns read_meta parses, positions on a jittered grid."""
    rng = np.random.default_rng(7 if negated else 3)
    files = []
    for r in range(rows):
        for c in range(cols):
            y, x = -600.0 + 300.0 * r + rng.uniform(-20, 20), -700.0 + 350.0 * c + rng.uniform(-20, 20)
            if negated:  # beans / knights / tarot / tarot_small: "<r>_<c>_<-y>_<x>.png"
                files.append(f"{r:02d}_{c:02d}_{-y:.6f}_{x:.6f}.png")
            else:        # the others: "out_<r>_<c>_<y>_<x>_.png"
                files.append(f"out_{r:02d}_{c:02d}_{y:.6f}_{x:.6f}_.png")
    return files


def _cfg(img_wh, lf, render_params=None, **top):
    d = dict(name="stanford", collection="gem", root_dir="", img_wh=list(img_wh), spherical_poses=False, use_ndc=False,
             val_pairs=[], val_num=8, val_skip=1,
             render_params=dict(interpolate=False, supersample=4, crop=1.0, **(render_params or {})), lightfield=lf)
    d.update(top)
    return d


_LF = dict(rows=5, cols=5, step=2, supersample=2, disp_row=2, st_scale=0.25)

# name: (dataset config, split, files)
VIEW_CASES = {
    # the two-turn spiral of 120 views (render_params.spiral, spiral_rad), vis_st_scale / vis_uv_scale
    "render_spiral": (_cfg((6, 4), dict(_LF, vis_st_scale=0.5, vis_uv_scale=0.75),
                           dict(spiral=True, far=False, spiral_rad=0.75)), "render", []),
    # the disp_row sweep: cols * supersample views with fractional s_idx; vis_st_scale left empty (st_scale)
    "render_sweep": (_cfg((7, 5), dict(_LF, supersample=3, disp_row=1, vis_st_scale=None)), "render", []),
    # render_far changes nothing but the branch taken; file coordinates are not used for the render split
    "render_far_files": (_cfg((6, 4), dict(_LF, use_file_coords=True), dict(far=True)), "render",
                         _grid_files(5, 5, False)),
    # val: the listed pairs, in the loop's order (not the list's)
    "val_pairs": (_cfg((6, 4), dict(_LF, uv_scale=0.9), val_pairs=[3, 1, 0, 4, 2, 2]), "val", []),
    # val_all: every view, truncated to val_num
    "val_all": (_cfg((5, 3), dict(_LF, start_row=1, end_row=4), val_all=True, val_num=6), "val", []),
    # test: every view off the step grid
    "test_grid": (_cfg((5, 4), dict(_LF, rows=4, cols=6, step=2, st_scale=0.125)), "test", []),
    # file coordinates, both name patterns
    "val_files": (_cfg((6, 4), dict(_LF, use_file_coords=True)), "val", _grid_files(5, 5, False)),
    "test_files_tarot": (_cfg((6, 4), dict(_LF, use_file_coords=True), collection="tarot"), "test",
                         _grid_files(5, 5, True)),
}


def reference_ray_case(W, H, s, t, st, uv, near, far, aspect, split):
    from datasets.lightfield import LightfieldDataset

    ds = object.__new__(LightfieldDataset)
    ds.split = split
    ds.img_wh = (W, H)
    ds.aspect = aspect
    ds.rows, ds.cols = 5, 5
    ds.st_scale = ds.vis_st_scale = st
    ds.uv_scale = ds.vis_uv_scale = uv
    ds.near_plane, ds.far_plane = near, far
    ds.render_spiral = ds.render_far = False
    ds.uv_downscale = 0.0
    if s is None:  # a fractional render view of a 9 x 9 grid
        ds.rows, ds.cols = 9, 9
        s, t = ds.get_coord((3.5, 2))
        return ds.get_coords(3.5, 2).numpy(), s, t
    # get_coords takes grid indices: the instance's get_coord returns (s, t) as given
    ds.get_coord = lambda st_idx: (s, t)
    return ds.get_coords(0, 0).numpy(), s, t


class _Listing:
    def __init__(self, files):
        self.files = list(files)

    def ls(self, _):
        return list(self.files)


def reference_views(cfg, split, files):
    from oracle.ref_shim import to_attr
    from datasets.base import Base5DDataset
    from datasets.lightfield import LightfieldDataset
    from datasets.stanford import StanfordLightfieldDataset

    def base_init(self, cfg, split="train", **kwargs):  # the attributes BaseDataset.__init__ sets that these read
        self.cfg = cfg
        self.split = getattr(cfg.dataset, "split", split)
        self.dataset_cfg = getattr(cfg.dataset, self.split, cfg.dataset)
        self.root_dir = ""
        self._img_wh = tuple(self.dataset_cfg.img_wh)
        self.img_wh = self._img_wh
        self.aspect = float(self.img_wh[0]) / self.img_wh[1]
        self.val_num = self.dataset_cfg.val_num
        self.pmgr = _Listing(files)
        self.prepare_data()

    orig = Base5DDataset.__init__
    Base5DDataset.__init__ = base_init
    try:
        ds = StanfordLightfieldDataset(to_attr(dict(dataset=cfg, params=dict(render_only=False, test_only=False))), split)
    finally:
        Base5DDataset.__init__ = orig
    n = len(ds)
    st_idx = ds.all_st_idx[:n]
    pos, scales, rays = [], [], []
    for s_idx, t_idx in st_idx:
        if split == "render":
            coords = LightfieldDataset.get_coords(ds, s_idx, t_idx)
            pos.append(ds.get_coord((s_idx, t_idx)))
            scales.append((ds.vis_st_scale, ds.vis_uv_scale))
        else:
            coords = ds.get_coords(s_idx, t_idx)
            if ds.use_file_coords:
                pos.append(ds.normalize_coord(ds.camera_coords[t_idx * ds.cols + s_idx]))
            else:
                pos.append(ds.get_coord((s_idx, t_idx)))
            scales.append((ds.st_scale, ds.uv_scale))
        rays.append(coords.numpy())
    fc = np.asarray(ds.camera_coords, np.float64).reshape(-1, 2)
    return (np.asarray(st_idx, np.float64), np.asarray(pos, np.float64), np.asarray(scales, np.float64),
            np.stack(rays, 0), fc)


def main():
    _install()
    out = {}
    for name, (W, H, s, t, st, uv, near, far, aspect, split, stride) in RAY_CASES.items():
        with contextlib.redirect_stdout(io.StringIO()):
            rays, s, t = reference_ray_case(W, H, s, t, st, uv, near, far, aspect, split)
        pixels = np.arange(0, W * H, stride, dtype=np.int64)
        out[f"{name}/rays"] = rays[pixels]
        out[f"{name}/pixels"] = pixels
        out[f"{name}/params"] = np.array([W, H, s, t, st, uv, near, far, aspect], np.float64)
        print(name, rays.shape, "stored", pixels.shape[0], "rows")
    np.savez_compressed(os.path.join(OUT, "lightfield_rays.npz"), **out)
    out = {}
    for name, (cfg, split, files) in VIEW_CASES.items():
        with contextlib.redirect_stdout(io.StringIO()):
            st_idx, pos, scales, rays, fc = reference_views(cfg, split, files)
        out[f"{name}/config"] = np.array(json.dumps(cfg))
        out[f"{name}/files"] = np.array(files if files else [""])
        out[f"{name}/split"] = np.array(split)
        out[f"{name}/st_idx"], out[f"{name}/pos"], out[f"{name}/scales"] = st_idx, pos, scales
        out[f"{name}/rays"], out[f"{name}/file_coords"] = rays, fc
        print(name, split, st_idx.shape[0], "views", rays.shape)
    np.savez_compressed(os.path.join(OUT, "lightfield_views.npz"), **out)


if __name__ == "__main__":
    main()
