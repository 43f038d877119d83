"""Training cases for the pipelines whose backward runs on the RARE variants of the render backward: bbox / z_depth
contraction, per-ray colour heads, the per-camera colour transform and the voxel-grid / deformable-plane primitives.

Kept apart from tests/cases.py:CASES (whose tests run every case).  A case is either a built-in case of tests/cases.py as it
is, or a model YAML the reference ships (tests/golden/shipped/<name>.npz: configuration, dataset facts, rays) with parameters
re-seeded at the gains given here.  Every case is non-trivial: sum(w) > 0.5 on at least a quarter of its rays, so the table,
head and colour-transform gradients are not zero by construction (tests/test_train_rare.py asserts it).
"""
from __future__ import annotations

import json
import os

import numpy as np
import torch

import hyperreel_b200 as hb
from hyperreel_b200.state import seeded_state_dict
from tests.cases import Case, build_case

SHIPPED_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "shipped")
N_RAYS = 96

TRAIN_CASES = {
    # built-in cases (tests/cases.py)
    "technicolor_bbox": dict(builtin=True),             # bbox contraction
    "technicolor_z_depth": dict(builtin=True),          # z_depth contraction
    "technicolor_global_color": dict(builtin=True),     # per-ray colour heads
    # shipped YAMLs.  flip: the fixture's rays start at z = -1 and look along +z, away from the world-space z planes
    # (sum w = 0 on every ray); flipped, they start at z = 0 and look along -z through the planes.
    "immersive_z_plane": dict(gain=100.0, app_gain=6.0, flip=True),          # per-camera colour transform, mipnerf contraction
    "technicolor_z_plane_world": dict(gain=600.0, app_gain=6.0, flip=True),  # bbox contraction of a world-space model
    "donerf_voxel": dict(gain=30.0),                                         # voxel grid
    "shiny_z_deformable": dict(gain=30.0),                                   # deformable planes
    "catacaustics_z_plane": dict(gain=30.0),                                 # per-ray colour heads
    "catacaustics_cylinder": dict(gain=30.0),
    "catacaustics_distance": dict(gain=30.0),
}
PARAM_SEED = 3


def build_train_case(name: str) -> Case:
    spec = TRAIN_CASES[name]
    if spec.get("builtin"):
        case = build_case(name)
        case.rays = case.rays[:N_RAYS].clone()
        return case
    g = np.load(os.path.join(SHIPPED_DIR, f"{name}.npz"))
    plain = json.loads(str(g["config_json"]))
    ds = json.loads(str(g["dataset_json"]))
    cfg = hb.to_cfg(plain)
    sig = hb.lower(cfg, ds)
    sd = seeded_state_dict(sig, seed=PARAM_SEED, density_gain=spec["gain"], app_gain=spec.get("app_gain", 1.0))
    rays = torch.from_numpy(g["rays"])[:N_RAYS].clone()
    if spec.get("flip"):
        rays[:, 2] = 0.0
        rays[:, 5] = -rays[:, 5]
    return Case(name=name, model_cfg=cfg, model_cfg_plain=plain, dataset=ds, sig=sig, rays=rays, state_dict=sd,
                n_samples=sig.n_samples)
