"""Golden embedding maps from the unmodified reference: visualize_warp (utils/visualization.py) followed by to8b
(utils/__init__.py:47) on seeded fp32 fields, run on CPU, and the shipped embedding-visualiser configs.

    HYPERREEL_REFERENCE=<reference checkout> python tests/golden/make_golden_visuals.py

writes ``tests/golden/visuals.npz``:

* ``<case>/x`` fp32 [F, P, dim]: one field over F frames of P pixels; ``<case>/opts`` JSON: the field's visualiser options
  (use_abs, bounds, normalize); ``<case>/u8`` uint8 [F, P, dim]: what the reference saves for each frame;
* ``configs`` JSON: {name: the parsed conf/experiment/visualizers/embedding/<name>.yaml} for every shipped config.

The cases cover every option combination of the shipped configs on 1- and 3-channel fields, values exactly at the bounds,
values on either side of every truncation step of 255 * x, and constant frames (normalize: 0 / 0 = NaN, saved as 0).
"""
import glob
import importlib.util
import json
import os
import sys

import numpy as np

OUT = os.path.dirname(os.path.abspath(__file__))

# the shipped configs' option sets (default, default_time, points) and the combinations between them
OPTION_SETS = {
    "normalize": dict(use_abs=False, bounds=None, normalize=True),                 # distances
    "abs_0_025": dict(use_abs=True, bounds=[0.0, 0.25], normalize=False),          # point_offset
    "bounds_pm2": dict(use_abs=False, bounds=[-2.0, 2.0], normalize=False),        # points
    "abs_0_1": dict(use_abs=True, bounds=[0.0, 1.0], normalize=False),             # spatial_flow
    "abs_normalize": dict(use_abs=True, bounds=None, normalize=True),              # raw_flow's options, sort aside
    "bounds_normalize": dict(use_abs=False, bounds=[-2.0, 2.0], normalize=True),
    "plain": dict(use_abs=False, bounds=None, normalize=False),
}


def fields(opts, dim, seed):
    """Three frames of one field: seeded values around the bounds, exact bounds, truncation edges; the third frame of a
    normalize case is constant."""
    rng = np.random.default_rng(seed)
    lo, hi = (opts["bounds"] if opts["bounds"] else (0.0, 1.0))
    lo, hi = np.float32(lo), np.float32(hi)
    P = 600
    f0 = rng.uniform(float(lo) - 0.5 * float(hi - lo), float(hi) + 0.5 * float(hi - lo), (P, dim)).astype(np.float32)
    # at the bounds, their negatives, and 255 * x on either side of every integer step of the mapped value
    k = np.arange(256, dtype=np.float32) / np.float32(255)
    steps = np.concatenate([k, np.nextafter(k, np.float32(-1)), np.nextafter(k, np.float32(2))]).astype(np.float32)
    mapped = (lo + steps * (hi - lo)).astype(np.float32)
    edge = np.concatenate([[lo, hi, -lo, -hi, np.nextafter(lo, -np.inf), np.nextafter(hi, np.inf)], mapped])
    edge = np.resize(edge, (P, dim)).astype(np.float32)
    frames = [f0, edge]
    frames.append(np.full((P, dim), np.float32(0.3), np.float32) if opts["normalize"] else
                  rng.normal(0.0, 2.0, (P, dim)).astype(np.float32))
    return np.stack(frames, 0)


def cases():
    out = {}
    seed = 0
    for name, opts in OPTION_SETS.items():
        for dim in (1, 3):
            out[f"{name}_{dim}"] = (opts, fields(opts, dim, seed))
            seed += 1
    return out


def reference_visualiser(root):
    """(visualize_warp, to8b) of the reference checkout at ``root``, its utils package loaded under a private name."""
    spec = importlib.util.spec_from_file_location("hr_ref_utils", os.path.join(root, "utils", "__init__.py"),
                                                  submodule_search_locations=[os.path.join(root, "utils")])
    pkg = importlib.util.module_from_spec(spec)
    sys.modules["hr_ref_utils"] = pkg
    spec.loader.exec_module(pkg)
    spec = importlib.util.spec_from_file_location("hr_ref_utils.visualization", os.path.join(root, "utils", "visualization.py"))
    vis = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(vis)
    return vis, pkg.to8b


def reference_maps(root, opts, x):
    """What validation_video / validation_image save for each frame of x [F, P, dim] (sort: False)."""
    import torch

    vis, to8b = reference_visualiser(root)
    out = []
    for f in x:
        e = torch.from_numpy(f.copy())
        dims = vis.get_warp_dimensions(e, 1, f.shape[0], k=min(f.shape[-1], 3), **opts)
        with np.errstate(invalid="ignore"):
            out.append(to8b(vis.visualize_warp(e, dims, **opts).numpy()))
    return np.stack(out, 0)


def main():
    import yaml

    root = os.environ.get("HYPERREEL_REFERENCE", "")
    if not os.path.isdir(os.path.join(root, "utils")):
        sys.exit("set HYPERREEL_REFERENCE to a reference checkout")
    arrays = {}
    for name, (opts, x) in cases().items():
        arrays[f"{name}/x"] = x
        arrays[f"{name}/opts"] = np.array(json.dumps(opts))
        arrays[f"{name}/u8"] = reference_maps(root, opts, x)
    configs = {}
    for p in sorted(glob.glob(os.path.join(root, "conf", "experiment", "visualizers", "embedding", "*.yaml"))):
        with open(p) as f:
            configs[os.path.basename(p)[:-5]] = yaml.safe_load(f)
    arrays["configs"] = np.array(json.dumps(configs))
    np.savez_compressed(os.path.join(OUT, "visuals.npz"), **arrays)
    print("wrote", os.path.join(OUT, "visuals.npz"), len(configs), "configs")


if __name__ == "__main__":
    main()
