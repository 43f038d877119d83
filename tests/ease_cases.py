"""EaseValue warm-up (nlf/activations.py:462-496) for the oracle and the tests of ``ease="reference"``.

``eased_oracle(cur_iter)`` makes oracle.hyperreel_oracle evaluate every EaseValue at ``cur_iter`` with the reference's own
expression (``w * out + (1 - w) * start_value`` with Python-scalar w, or the start value alone for an empty window), instead
of the render-iteration semantics it implements (the inner activation).  The cases, iterations and the training loop are
shared by tests/golden/make_golden_ease.py and the tests.
"""
from __future__ import annotations

import contextlib
import copy
import json
import os

import numpy as np
import torch

import hyperreel_b200 as hb
from hyperreel_b200.state import seeded_state_dict
from tests.cases import Case, build_case

ITERS_PER_EPOCH = 4000
# sigma eases over epochs 0-3, point_sigma waits one epoch and eases over epochs 1-4 (both from the start value 1.0):
# both held at the start value; sigma mid-window, point_sigma waiting; both mid-window; sigma elapsed, point_sigma
# mid-window; both elapsed
ITERS = (0, 2000, 6000, 13000, 16000)
# the five-step training loop: iterations 6000-6004 (both heads mid-window; 6000 is also an up-sampling iteration of the
# TensoRF schedules, which re-creates the tables and restarts the optimisers)
LOOP_START, LOOP_STEPS = 6000, 5
N_RAYS = 96
SHIPPED_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "shipped")

EASE_CASES = {
    "technicolor_trained": dict(builtin=True),                   # dynamic, z-plane, flow, point offset
    "immersive_sphere": dict(gain=30.0),                          # spheres, dynamic
    "llff_z_plane": dict(gain=30.0),                              # static
    "technicolor_cascaded": dict(gain=30.0, forward_only=True),  # the first stage eases sigma (pre_act_sigma)
}
PARAM_SEED = 5


def build_ease_case(name: str) -> Case:
    spec = EASE_CASES[name]
    if spec.get("builtin"):
        case = build_case(name)
        case.rays = case.rays[:N_RAYS].clone()
        return case
    g = np.load(os.path.join(SHIPPED_DIR, f"{name}.npz"))
    plain = json.loads(str(g["config_json"]))
    ds = json.loads(str(g["dataset_json"]))
    cfg = hb.to_cfg(plain)
    sig = hb.lower(cfg, ds)
    sd = seeded_state_dict(sig, seed=PARAM_SEED, density_gain=spec["gain"])
    rays = torch.from_numpy(g["rays"])[:N_RAYS].clone()
    return Case(name=name, model_cfg=cfg, model_cfg_plain=plain, dataset=ds, sig=sig, rays=rays, state_dict=sd,
                n_samples=sig.n_samples)


def ease_value_cfgs(cfg, path=""):
    """Every ``type: ease_value`` dict of a plain model config, by its path."""
    out = {}
    if isinstance(cfg, dict):
        if cfg.get("type") == "ease_value":
            out[path] = cfg
        for k, v in cfg.items():
            out.update(ease_value_cfgs(v, f"{path}/{k}"))
    elif isinstance(cfg, list):
        for i, v in enumerate(cfg):
            out.update(ease_value_cfgs(v, f"{path}/{i}"))
    return out


def in_iters(ease_cfg: dict, iters_per_epoch: int = ITERS_PER_EPOCH) -> dict:
    """An ease_value dict with its ``*_epochs`` keys converted to ``*_iters`` (as INRSystem does for the whole config)."""
    return hb.config.epochs_to_iters(copy.deepcopy(ease_cfg), iters_per_epoch)


class _Eased:
    def __init__(self, inner, cfg, cur_iter):
        self.inner = inner
        self.start_value = cfg.get("start_value", 0.0)
        self.wait_iters = cfg.get("wait_iters", 0.0)
        self.window_iters = cfg.get("window_iters", 0.0)
        self.cur_iter = cur_iter - self.wait_iters  # EaseValue.set_iter


@contextlib.contextmanager
def eased_oracle(cur_iter: int, iters_per_epoch: int = ITERS_PER_EPOCH):
    """Within the block, HyperReelOracle (constructed and evaluated there) applies EaseValue at ``cur_iter``."""
    import oracle.hyperreel_oracle as O

    resolve0, apply0 = O.resolve_activation, O.apply_activation

    def resolve(cfg):
        if isinstance(cfg, dict) and cfg.get("type") == "ease_value":
            c = in_iters(cfg, iters_per_epoch)
            return _Eased(resolve(c["activation"]), c, cur_iter)
        return resolve0(cfg)

    def apply(act, x):
        if not isinstance(act, _Eased):
            return apply0(act, x)
        out = apply(act.inner, x)
        if act.cur_iter >= act.window_iters:  # EaseValue.ease_out (activations.py:482-489)
            return out
        if act.window_iters == 0:
            return torch.ones_like(out) * act.start_value
        w = min(max(float(act.cur_iter) / act.window_iters, 0.0), 1.0)
        return w * out + (1 - w) * act.start_value

    O.resolve_activation, O.apply_activation = resolve, apply
    try:
        yield
    finally:
        O.resolve_activation, O.apply_activation = resolve0, apply0


def loop_target(n: int) -> torch.Tensor:
    return torch.rand(n, 3, generator=torch.Generator().manual_seed(0))


def loop_seed(step: int) -> int:
    """Seed of the CPU generator before step `step`: the training forward's white-background coin flip draws from it."""
    return 1000 + step


def opt_group(name: str):
    """The optimiser group of a RenderLightfield parameter (INRSystem.optimizer_groups); None for the ray params'
    `dummy_layer`s, which no forward reads."""
    if "dummy_layer" in name:
        return None
    if name.endswith("color_embedding"):
        return "embedding"
    if "embedding_model" in name:
        return "embedding_impl"
    if "basis_mat" in name:
        return "color_impl"
    assert "plane" in name or "line" in name, name
    return "color"
