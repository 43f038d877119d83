"""Golden data of tests/test_oracle_vs_reference.py and of the YAML-coverage tests of tests/test_host_logic.py: what the
*unmodified reference* builds and computes, recorded once so that the tests need no reference checkout.

    HYPERREEL_REFERENCE=<checkout of facebookresearch/hyperreel> python tests/golden/make_golden_reference.py

Writes tests/golden/reference/<test>.npz: every shipped model YAML as JSON (model_yamls.npz) and, per test, the reference's
side of each comparison (rgb, sample points and distances, regulariser terms, re-sampled and pruned tables, lowered
constants, activation values, NDC rays).  Large arrays are cut to a fixed row sample (ROWS_*) to keep every file small.
"""
from __future__ import annotations

import glob
import json
import os
import sys
import types
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

import hyperreel_b200 as hb  # noqa: E402
from hyperreel_b200.config import epochs_to_iters, to_plain  # noqa: E402
from hyperreel_b200.signature import RENDER_ITER, UnsupportedPipeline  # noqa: E402
from hyperreel_b200.state import seeded_state_dict  # noqa: E402
from oracle import ref_shim  # noqa: E402
from tests.cases import build_case  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference")

DS = {"num_keyframes": 12, "num_frames": 50, "near": 0.5, "far": 10.0, "depth_range": [0.5, 10.0], "name": "x", "collection": "y"}
DS_R2 = dict(DS, bbox_min=[-1.5, -1.25, -1.0], bbox_max=[1.5, 1.25, 1.0], total_images_per_frame=5, val_all=True)
FACTS = [DS_R2, {"num_keyframes": 7, "num_frames": 30, "near": 0.25, "far": 6.0, "depth_range": [0.75, 4.0], "name": "x",
                 "collection": "y", "bbox_min": [-0.5, -2.0, -1.5], "bbox_max": [2.5, 1.0, 0.5], "total_images_per_frame": 3,
                 "val_all": False}]
BUILTIN_NAMES = ["technicolor_z_plane", "neural_3d_z_plane", "donerf_sphere", "shiny_z_plane_tiny"]
FRESH_CASES = ["technicolor_trained", "neural3d_trained", "donerf_s16"]
FRESH_N = 777
ROWS_FRESH = np.arange(0, FRESH_N, 7)  # rays whose sample points / distances are kept
EDGE_CASES = ["technicolor_trained", "neural3d_trained", "donerf_trained", "immersive_sphere_new", "donerf_cylinder", "technicolor_bbox"]
R2_FAMILIES = ["catacaustics_voxel", "donerf_voxel", "shiny_z_deformable", "immersive_z_plane", "neural_3d_z_plane_static",
               "technicolor_z_plane_no_sample", "shiny_z_plane_cascaded", "shiny_z_plane_feedback", "shiny_z_tensorf_cascaded",
               "technicolor_cascaded"]
ROWS_R2 = np.arange(0, 40, 3)
ACT_X = torch.linspace(-6.0, 6.0, 97)


def yaml_files():
    return sorted(glob.glob(os.path.join(ref_shim.REFERENCE_ROOT, "conf/experiment/model/*.yaml")))


def model_yamls():
    """Every shipped model YAML, read the way the product reads it (hb.load_model_yaml), as JSON ("null": empty file)."""
    return {os.path.basename(f)[:-5]: json.dumps(None if (c := hb.load_model_yaml(f)) is None else to_plain(c)) for f in yaml_files()}


def import_ref_regularizers():
    ref_shim.install()
    # nlf/regularizers/__init__.py imports every regulariser (and through them the datasets): import tensorf.py alone, with
    # a stand-in for the base class it derives from
    if "nlf.regularizers" not in sys.modules:
        pkg = types.ModuleType("nlf.regularizers")
        pkg.__path__ = [f"{ref_shim.REFERENCE_ROOT}/nlf/regularizers"]
        sys.modules["nlf.regularizers"] = pkg
        base = types.ModuleType("nlf.regularizers.base")
        base.BaseRegularizer = type("BaseRegularizer", (torch.nn.Module,), {})
        sys.modules["nlf.regularizers.base"] = base
    import nlf.regularizers.tensorf as t
    return t


def tables(net, prefix=""):
    return {prefix + k: v.numpy() for k, v in net.state_dict().items() if any(t in k for t in ("plane", "line"))}


def rec_builtin_configs():
    return {n: json.dumps(ref_shim.load_reference_yaml(n)) for n in BUILTIN_NAMES}


def rec_fresh_rays():
    out = {}
    for name in FRESH_CASES:
        case = build_case(name, n=FRESH_N)
        ref = ref_shim.build_reference(case.model_cfg_plain, case.dataset)
        ref.load_state_dict(case.state_dict, strict=False)
        r = ref_shim.run_reference(ref, case.rays.clone(), chunk=200, capture=True)
        out[f"{name}/rgb"] = r["rgb"].numpy()
        out[f"{name}/points"] = r["_embed"]["points"].reshape(FRESH_N, -1)[ROWS_FRESH].numpy()
        out[f"{name}/distances"] = r["_embed"]["distances"].reshape(FRESH_N, -1)[ROWS_FRESH].numpy()
    return out


def rec_edge_rays():
    from nlf.rendering import render_chunked
    from tests.test_edge_rays_gpu import craft

    out = {}
    for name in EDGE_CASES:
        case = build_case(name)
        rays = craft(case)
        ref = ref_shim.build_reference(case.model_cfg_plain, case.dataset)
        ref.load_state_dict(case.state_dict, strict=False)
        with torch.no_grad():
            out[name] = render_chunked(rays.clone(), ref, {}, rays.shape[0])["rgb"].numpy()
    return out


def rec_every_shipped_yaml(yamls):
    from nlf.rendering import render_chunked

    out = {}
    for name, js in yamls.items():
        plain = json.loads(js)
        if plain is None:
            continue
        cfg = hb.to_cfg(plain)
        cfg.color.net.N_voxel_init = cfg.color.net.N_voxel_final = 24 ** 3
        try:
            sig = hb.lower(cfg, DS_R2)
        except UnsupportedPipeline:
            continue
        sd = seeded_state_dict(sig, seed=3, density_gain=30.0)
        rays = hb.rays.for_signature(sig, 48, seed=9)
        ref = ref_shim.build_reference(to_plain(cfg), DS_R2)
        _, unexpected = ref.load_state_dict(sd, strict=False)
        assert not unexpected, (name, unexpected)
        with torch.no_grad():
            out[name] = render_chunked(rays.clone(), ref, {}, rays.shape[0])["rgb"].numpy()
    return out


def rec_upsampling_and_regulariser_terms(yamls):
    t = import_ref_regularizers()
    out = {}
    for name in ("technicolor_z_plane", "donerf_sphere"):
        cfg = hb.to_cfg(json.loads(yamls[name]))
        cfg.color.net.N_voxel_init, cfg.color.net.N_voxel_final = 12 ** 3, 20 ** 3
        sig = hb.lower(cfg, DS)
        ref = ref_shim.build_reference(to_plain(cfg), DS)
        ref.load_state_dict(seeded_state_dict(sig, seed=4), strict=False)
        rnet = ref.model.color_model.net
        out[f"{name}/terms"] = np.array([float(rnet.density_L1()), float(rnet.TV_loss_density(t.TVLoss())),
                                         float(rnet.TV_loss_app(t.TVLoss()))], dtype=np.float64)
        out[f"{name}/N_voxel_list"] = np.array([int(v) for v in rnet.N_voxel_list])
        reso = hb.state.n_to_reso(int(rnet.N_voxel_list[0]), torch.tensor(cfg.color.net.aabb))
        rnet.upsample_volume_grid(reso)
        out[f"{name}/gridSize"] = np.array(rnet.gridSize.tolist())
        out.update(tables(rnet, f"{name}/tab/"))
    return out


def rec_regulariser_sequence(yamls):
    t = import_ref_regularizers()
    RefReg = t.TensoRF

    class Base(torch.nn.Module):  # what BaseRegularizer provides to this class: the system handle and the iteration counter
        def __init__(self, system, cfg):
            super().__init__()
            self._system, self.cur_iter = [system], 0

        def get_system(self):
            return self._system[0]

        def set_iter(self, i):
            self.cur_iter = i

    RefReg.__bases__ = (Base,)
    cfg = hb.to_cfg(json.loads(yamls["technicolor_z_plane"]))
    cfg.color.net.N_voxel_init = cfg.color.net.N_voxel_final = 14 ** 3
    sig = hb.lower(cfg, DS)
    ref = ref_shim.build_reference(to_plain(cfg), DS)
    ref.load_state_dict(seeded_state_dict(sig, seed=6), strict=False)
    rcfg = ref_shim.to_attr(REG_CFG)
    theirs = RefReg(SimpleNamespace(is_subdivided=False, render_fn=ref), rcfg)
    losses = []
    for it in range(6):
        theirs.set_iter(it)
        losses.append(float(theirs._loss(None, None, 0)))
    return {"losses": np.array(losses, dtype=np.float64), "TV_weight_density": np.array(float(theirs.TV_weight_density))}


REG_CFG = {"type": "tensorf", "update_AlphaMask_list": [2], "lr_decay_target_ratio": 0.1, "n_iters": 50,
           "L1_weight_initial": 8e-5, "L1_weight_rest": 4e-5, "TV_weight_density": 0.05, "TV_weight_app": 0.05}


def rec_round_2_stages(yamls):
    out = {}
    for name in R2_FAMILIES:
        cfg = hb.to_cfg(json.loads(yamls[name]))
        cfg.color.net.N_voxel_init = cfg.color.net.N_voxel_final = 16 ** 3
        sig = hb.lower(cfg, DS_R2)
        sd = seeded_state_dict(sig, seed=5, density_gain=30.0)
        rays = hb.rays.for_signature(sig, 40, seed=3)
        ref = ref_shim.build_reference(to_plain(cfg), DS_R2)
        ref.load_state_dict(sd, strict=False)
        r = ref_shim.run_reference(ref, rays.clone(), capture=True)
        out[f"{name}/rgb"] = r["rgb"].reshape(40, -1).numpy()
        out[f"{name}/points"] = r["_embed"]["points"].reshape(40, -1)[ROWS_R2].numpy()
        out[f"{name}/distances"] = r["_embed"]["distances"].reshape(40, -1)[ROWS_R2].numpy()
    return out


ALPHA_DS = {"num_keyframes": 4, "num_frames": 6, "near": 0.5, "far": 10.0, "depth_range": [0.5, 10.0], "name": "x", "collection": "y"}


def corner_occupancy(sd, gain):
    """Occupancy confined to a corner region, so that the box of occupied voxels is a strict subset of the grid (empty for x
    in the lower half of the box: groups 0 and 1 have x as their planes' column axis, group 2 as its line's axis)."""
    for k in list(sd):
        if "density_plane" in k and "time" not in k and sd[k].numel() > 0:
            t = sd[k].clone() * gain
            if not k.endswith(".2"):
                t[..., : t.shape[-1] // 2] = 0
            sd[k] = t
        if "density_line.2" in k and sd[k].numel() > 0:
            t = sd[k].clone()
            t[..., : t.shape[-2] // 2, :] = 0
            sd[k] = t
    return sd


def rec_alpha_mask(yamls):
    out = {}
    for name in ("technicolor_z_plane", "donerf_sphere"):
        cfg = hb.to_cfg(json.loads(yamls[name]))
        cfg.color.net.N_voxel_init = cfg.color.net.N_voxel_final = 13 ** 3
        sig = hb.lower(cfg, ALPHA_DS)
        sd = corner_occupancy(seeded_state_dict(sig, seed=8), 40000.0)
        ref = ref_shim.build_reference(to_plain(cfg), ALPHA_DS)
        ref.load_state_dict(sd, strict=False)
        rnet = ref.model.color_model.net
        reso = tuple(rnet.gridSize.tolist())
        with torch.no_grad():
            out[f"{name}/alpha"] = rnet.getDenseAlpha(reso)[0].numpy()
        box = rnet.updateAlphaMask(reso)
        out[f"{name}/box"] = box.numpy()
        out[f"{name}/alpha_volume"] = rnet.alphaMask.alpha_volume.numpy()
        rnet.shrink(box)
        out[f"{name}/gridSize"] = np.array(rnet.gridSize.tolist())
        out[f"{name}/aabb"] = rnet.aabb.numpy()
        out.update(tables(rnet, f"{name}/tab/"))
        out[f"{name}/box2"] = rnet.updateAlphaMask(tuple(rnet.gridSize.tolist())).numpy()
    return out


def rec_lowered_constants(yamls):
    from hyperreel_b200 import lib as L

    out = {}
    for name, js in yamls.items():
        plain = json.loads(js)
        if plain is None:
            continue
        cfg = hb.to_cfg(plain)
        cfg.color.net.N_voxel_init = cfg.color.net.N_voxel_final = 12 ** 3
        for fi, ds in enumerate(FACTS):
            try:
                sig = hb.lower(cfg, ds)
            except UnsupportedPipeline:
                continue
            ref = ref_shim.build_reference(to_plain(cfg), ds)
            embs = ref.model.embedding_model.embeddings
            keys = list(to_plain(cfg)["embedding"]["embeddings"].keys())
            isects = [embs[i].intersect_fn for i, k in enumerate(keys) if cfg.embedding.embeddings[k].type == "ray_intersect"]
            it = isects[-1]
            net = ref.model.color_model.net
            rec = {"samples": it.samples.reshape(-1).float().tolist(), "z_scale": torch.as_tensor(it.z_scale).reshape(-1).float().tolist(),
                   "masked": bool(it.cur_iter <= it.mask_stop_iters), "near": float(it.near), "far": float(it.far),
                   "distance_scale": float(net.distance_scale), "weight_thre": float(net.rayMarch_weight_thres),
                   "white_bg": bool(net.white_bg), "black_bg": bool(net.black_bg), "aabb": [float(v) for v in net.aabb.reshape(-1)],
                   "gridSize": net.gridSize.tolist()}
            if sig.cfg.contract_type == L.CONTRACT_MIPNERF:
                cf = it.contract_fn
                rec["contract"] = [float(cf.contract_start_radius), float(cf.contract_end_radius),
                                   float(cf.contract_start_distance), float(cf.contract_end_distance)]
            if sig.cfg.cascade:
                rec["pre_samples"] = isects[0].samples.reshape(-1).float().tolist()
                rec["pre_z_scale"] = float(torch.as_tensor(isects[0].z_scale).reshape(-1)[0])
            if sig.cfg.dynamic:
                rec["keyframes_frames"] = [int(net.num_keyframes), int(net.total_num_frames)]
            out[f"{name}/{fi}"] = json.dumps(rec)
    return out


def walk_activations(o, path=""):
    if isinstance(o, dict):
        for k, v in o.items():
            if k.endswith("activation") and (isinstance(v, (dict, str))):
                yield path + "/" + k, v
            if isinstance(v, (dict, list)):
                yield from walk_activations(v, path + "/" + k)
    elif isinstance(o, list):
        for i, v in enumerate(o):
            yield from walk_activations(v, f"{path}[{i}]")


def rec_activations(yamls):
    ref_shim.install()
    from nlf.activations import get_activation

    out = {}
    for name, js in yamls.items():
        plain = json.loads(js)
        if plain is None:
            continue
        try:
            hb.lower(hb.to_cfg(plain), DS_R2)
        except UnsupportedPipeline:
            continue
        for path, acfg in walk_activations(epochs_to_iters(plain, 1)["embedding"]):
            if isinstance(acfg, dict) and "type" not in acfg:
                continue
            mod = get_activation(ref_shim.to_attr(acfg) if isinstance(acfg, dict) else acfg)
            if hasattr(mod, "set_iter"):
                mod.set_iter(RENDER_ITER)
            out[f"{name}{path}"] = mod(ACT_X.clone()).detach().numpy()
    return out


def rec_ndc_rays():
    """get_rays + get_ndc_rays_fx_fy of the reference (utils/ray_utils.py) on the ndc_73x41 camera, 6-channel rays"""
    ref_shim.install()
    from utils.ray_utils import get_ndc_rays_fx_fy, get_ray_directions_K, get_rays

    from tests.cases_rays import RAY_CASES
    c = RAY_CASES["ndc_73x41"]
    K = torch.FloatTensor(c["K"])
    d = get_ray_directions_K(c["H"], c["W"], K, centered_pixels=True, device="cpu")
    o, d = get_rays(d, torch.FloatTensor(c["pose"])[:3, :4])
    return {"rays": get_ndc_rays_fx_fy(c["H"], c["W"], K[0, 0], K[1, 1], c["near"], torch.cat([o, d], -1)).numpy()}


def main():
    if not ref_shim.reference_available():
        raise SystemExit("set HYPERREEL_REFERENCE to a checkout of the reference")
    ref_shim.install()
    os.makedirs(OUT, exist_ok=True)
    yamls = model_yamls()
    jobs = {
        "model_yamls": lambda: yamls,
        "builtin_configs": rec_builtin_configs,
        "fresh_rays": rec_fresh_rays,
        "edge_rays": rec_edge_rays,
        "every_shipped_yaml": lambda: rec_every_shipped_yaml(yamls),
        "upsampling_and_regulariser_terms": lambda: rec_upsampling_and_regulariser_terms(yamls),
        "regulariser_sequence": lambda: rec_regulariser_sequence(yamls),
        "round_2_stages": lambda: rec_round_2_stages(yamls),
        "alpha_mask": lambda: rec_alpha_mask(yamls),
        "lowered_constants": lambda: rec_lowered_constants(yamls),
        "activations": lambda: rec_activations(yamls),
        "ndc_rays": rec_ndc_rays,
    }
    for name, fn in jobs.items():
        d = fn()
        np.savez_compressed(os.path.join(OUT, name + ".npz"), **{k: np.asarray(v) for k, v in d.items()})
        print(f"{name}: {len(d)} arrays, {os.path.getsize(os.path.join(OUT, name + '.npz')) // 1024} KB")


if __name__ == "__main__":
    main()
