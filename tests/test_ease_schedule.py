"""EaseValue warm-up on the host: the lowered eased activations against the reference's EaseValue modules, the eased oracle
against the reference's renders and gradients (goldens of tests/golden/make_golden_ease.py), the lowering's invariants and the
option checks of ease="reference"."""
import ctypes as C
import glob
import json
import os
import re

import numpy as np
import pytest
import torch

import hyperreel_b200 as hb
from hyperreel_b200 import lib as L
from hyperreel_b200.signature import lower, resolve_activation
from oracle.hyperreel_oracle import HyperReelOracle
from tests.ease_cases import EASE_CASES, ITERS, ITERS_PER_EPOCH, SHIPPED_DIR, build_ease_case, eased_oracle, ease_value_cfgs, in_iters
from tests.golden.make_golden_grads import probe_indices, target_for

GOLDEN = os.path.dirname(os.path.abspath(__file__)) + "/golden"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _apply(act, x):
    """The render kernel's apply_act in fp32 torch ops (exact sigmoid / tanh)."""
    v = x * np.float32(act.inner_fac) + np.float32(act.shift)
    v = {L.ACT_IDENTITY: v, L.ACT_SIGMOID: torch.sigmoid(v), L.ACT_TANH: torch.tanh(v)}[act.kind]
    v = v * np.float32(act.outer_fac)
    if act.eased:
        v = v * np.float32(act.ease_mul) + np.float32(act.ease_add)
    return v


def _shipped_that_lower():
    out = []
    for path in sorted(glob.glob(os.path.join(SHIPPED_DIR, "*.npz"))):
        g = np.load(path)
        plain, ds = json.loads(str(g["config_json"])), json.loads(str(g["dataset_json"]))
        try:
            lower(hb.to_cfg(plain), ds)
        except hb.UnsupportedPipeline:
            continue
        out.append((os.path.basename(path)[:-4], plain, ds))
    return out


def test_eased_activations_match_the_reference_modules():
    g = np.load(os.path.join(GOLDEN, "ease_activations.npz"))
    x = torch.from_numpy(g["input"])
    n = 0
    for yaml, plain, _ in _shipped_that_lower():
        for where, ecfg in ease_value_cfgs(plain).items():
            for it in ITERS:
                act = resolve_activation(in_iters(ecfg), it, ease=True)
                ref = torch.from_numpy(g[f"{yaml}{where}/{it}"])
                assert float((_apply(act, x) - ref).abs().max()) <= 1e-6, (yaml, where, it)
                n += 1
    assert n >= 600


@pytest.mark.parametrize("name", list(EASE_CASES))
@pytest.mark.parametrize("it", ITERS)
def test_eased_oracle_matches_the_reference(name, it):
    g = np.load(os.path.join(GOLDEN, f"ease_{name}.npz"))
    case = build_ease_case(name)
    rays = case.rays.clone()
    with eased_oracle(it):
        orc = HyperReelOracle(case.model_cfg_plain, case.dataset, case.state_dict)
        if EASE_CASES[name].get("forward_only"):
            rgb = orc.render(rays)
            assert float((rgb - torch.from_numpy(g[f"{it}/rgb"])).abs().max()) <= 2e-6
            return
        rgb, leaves = orc.render_with_grad(rays)
        assert float((rgb.detach() - torch.from_numpy(g[f"{it}/rgb"])).abs().max()) <= 2e-6
        loss = ((rgb - target_for(rays.shape[0])) ** 2).mean()
        loss.backward()
    assert abs(float(loss.detach()) - float(g[f"{it}/loss"])) <= 1e-6
    keys = [k[len(f"{it}/norm/"):] for k in g.files if k.startswith(f"{it}/norm/")]
    assert len(keys) >= 17
    for k in keys:  # the tolerances of tests/test_oracle_grads_train.py
        nrm = float(g[f"{it}/norm/{k}"])
        if nrm == 0.0:
            continue
        flat = leaves[k].grad.reshape(-1)
        scale = float(g[f"{it}/max/{k}"]) + 1e-12
        assert abs(float(flat.norm()) - nrm) <= 1e-4 * nrm + 1e-9, k
        probe = flat[probe_indices(flat.numel())].detach().numpy()
        assert np.abs(probe - g[f"{it}/probe/{k}"]).max() <= 2e-5 * scale + 1e-10, k


def test_elapsed_windows_lower_to_the_plain_config():
    """At and past the end of every window, ease=True gives the hr_config of ease=False byte for byte."""
    for yaml, plain, ds in _shipped_that_lower():
        for it in (16000, 10_000_000):
            a = lower(hb.to_cfg(plain), ds, cur_iter=it, iters_per_epoch=ITERS_PER_EPOCH, ease=True)
            b = lower(hb.to_cfg(plain), ds, cur_iter=it, iters_per_epoch=ITERS_PER_EPOCH)
            assert bytes(a.cfg) == bytes(b.cfg), (yaml, it)


def test_open_windows_lower_only_when_eased():
    case = build_ease_case("technicolor_trained")
    with pytest.raises(hb.UnsupportedPipeline):
        lower(case.model_cfg, case.dataset, cur_iter=6000, iters_per_epoch=ITERS_PER_EPOCH)
    sig = lower(case.model_cfg, case.dataset, cur_iter=6000, iters_per_epoch=ITERS_PER_EPOCH, ease=True)
    sites = {s.field: s for s in sig.ease_sites}
    assert {"act_sigma", "act_point_sigma"} <= set(sites)
    assert (sites["act_point_sigma"].wait_iters, sites["act_point_sigma"].window_iters) == (4000, 12000)
    assert (sig.cfg.act_sigma.eased, sig.cfg.act_sigma.ease_mul, sig.cfg.act_sigma.ease_add) == (1, 0.5, 0.5)
    p = sig.cfg.act_point_sigma
    assert p.eased == 1 and p.ease_mul == np.float32(2000 / 12000) and p.ease_add == np.float32(1 - 2000 / 12000)
    nested = {"type": "ease_value", "window_iters": 10, "activation": {"type": "ease_value", "activation": "sigmoid"}}
    with pytest.raises(hb.UnsupportedPipeline):
        resolve_activation(nested, 5, ease=True)


def test_ease_option_values_are_checked_on_the_cpu():
    case = build_ease_case("technicolor_trained")
    with pytest.raises(ValueError, match="ease"):
        hb.LightfieldModel(case.model_cfg, dataset=case.dataset, iters_per_epoch=ITERS_PER_EPOCH, ease="always")
    with pytest.raises(ValueError, match="iters_per_epoch"):
        hb.LightfieldModel(case.model_cfg, dataset=case.dataset, ease="reference")
    with pytest.raises(ValueError, match="ease"):
        hb.INRSystem(hb.to_cfg({"model": case.model_cfg_plain, "training": {"iters_per_epoch": 4000}}), dataset=case.dataset,
                     ease="none")


def test_ctypes_act_struct_matches_header_field_order():
    header = open(os.path.join(ROOT, "include", "hyperreel_b200.h")).read()
    body = re.search(r"typedef struct hr_act \{(.*?)\} hr_act;", header, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = []
    for decl in body.split(";"):
        decl = decl.strip()
        if decl:
            names += [n.strip() for n in decl.split(None, 1)[1].split(",")]
    assert names == [f for f, _ in L.hr_act._fields_]
    assert C.sizeof(L.hr_act) == 4 * len(names)
