"""Golden vectors for the model YAMLs the reference SHIPS (conf/experiment/model/*.yaml) and the fused path accepts.

For each such YAML: the configuration as JSON (the tests need no reference checkout, hence no YAML files), the dataset
facts, seeded rays, and the rgb the *unmodified reference* renders for seeded parameters (grid shrunk to 24^3 so that the
fixtures stay small; parameters are regenerated from the seed by hyperreel_b200.state.seeded_state_dict).

    python tests/golden/make_golden_shipped.py
"""
from __future__ import annotations

import glob
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

import hyperreel_b200 as hb  # noqa: E402
from hyperreel_b200.config import to_plain  # noqa: E402
from hyperreel_b200.signature import UnsupportedPipeline  # noqa: E402
from hyperreel_b200.state import seeded_state_dict  # noqa: E402
from oracle import ref_shim  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "shipped")
DATASET = {"num_keyframes": 12, "num_frames": 50, "near": 0.5, "far": 10.0, "depth_range": [0.5, 10.0], "name": "x", "collection": "y"}
# dataset facts only some constructors read (voxel.py:27-29: bbox_min / bbox_max; point.py:574-575: total_images_per_frame, val_all);
# used for the fixtures added in round 2 -- the 35 older fixtures keep the dictionary above
DATASET_R2 = dict(DATASET, bbox_min=[-1.5, -1.25, -1.0], bbox_max=[1.5, 1.25, 1.0], total_images_per_frame=5, val_all=True)
PARAM_SEED, RAY_SEED, N_RAYS, GRID = 3, 9, 96, 24 ** 3


def main():
    ref_shim.install()
    from nlf.rendering import render_chunked

    os.makedirs(OUT, exist_ok=True)
    for f in sorted(glob.glob(os.path.join(ref_shim.REFERENCE_ROOT, "conf/experiment/model/*.yaml"))):
        name = os.path.basename(f)[:-5]
        cfg = hb.load_model_yaml(f)
        if cfg is None:
            continue
        cfg.color.net.N_voxel_init = GRID
        cfg.color.net.N_voxel_final = GRID
        out_path = os.path.join(OUT, f"{name}.npz")
        if os.path.exists(out_path) and "--all" not in sys.argv:
            continue  # fixtures are append-only: regenerate everything with --all
        ds_facts = DATASET_R2
        try:
            sig = hb.lower(cfg, ds_facts)
        except UnsupportedPipeline:
            continue
        sd = seeded_state_dict(sig, seed=PARAM_SEED, density_gain=30.0)
        rays = hb.rays.for_signature(sig, N_RAYS, seed=RAY_SEED)
        plain = to_plain(cfg)
        ref = ref_shim.build_reference(plain, ds_facts)
        _, unexpected = ref.load_state_dict(sd, strict=False)
        assert not unexpected, (name, unexpected)
        with torch.no_grad():
            rgb = render_chunked(rays.clone(), ref, {}, rays.shape[0])["rgb"].reshape(-1, 3)
        np.savez_compressed(out_path, config_json=np.array(json.dumps(plain)),
                            dataset_json=np.array(json.dumps(ds_facts)), rays=rays.numpy(), rgb=rgb.numpy())
        print(f"{name}: S={sig.n_samples} rgb mean {float(rgb.mean()):.4f} max {float(rgb.max()):.4f}")


if __name__ == "__main__":
    main()
