"""Built-in model configs in the reference's own schema (the keys ``conf/experiment/model/*.yaml`` uses).

The package ships no copies of the reference's YAML files, so the BASELINE.json configurations are generated here from a few
parametric builders; ``tests/test_oracle_vs_reference.py`` asserts that each built-in equals ``yaml.safe_load`` of the
reference file it names.  A user of the reference passes their own YAML through
``hyperreel_b200.config.load_model_yaml`` instead.

Dataset facts the reference reads from ``system.dm.train_dataset`` (K keyframes, F frames, near/far,
depth_range: tensorf_dynamic.py:49-50, contract.py:121-125, primitive.py:371-373) travel in a small
``dataset`` dict next to the model config.
"""
from __future__ import annotations

import copy

from typing import Dict, Tuple

from .config import Cfg, to_cfg


def _ease(inner: dict, start_value: float, window_epochs: int, wait_epochs: int) -> dict:
    return {"type": "ease_value", "start_value": start_value, "window_epochs": window_epochs,
            "wait_epochs": wait_epochs, "activation": inner}


def _identity_full() -> dict:
    return {"type": "identity", "shift": 0.0, "inner_fac": 1.0, "outer_fac": 1.0}


def _windowed_pe(n_freqs: int, freq_multiplier=None) -> dict:
    pe = {"type": "windowed"}
    if freq_multiplier is not None:
        pe["freq_multiplier"] = freq_multiplier
    pe.update({"n_freqs": n_freqs, "wait_iters": 0, "max_freq_epoch": 0, "exclude_identity": False})
    return pe


def _ray_group(fn: str, n_freqs: int) -> dict:
    if fn == "two_plane":
        param = {"n_dims": 4, "fn": "two_plane"}
    else:
        param = {"n_dims": 6, "fn": "pluecker", "direction_multiplier": 1.0, "moment_multiplier": 1.0}
    return {"start": 0, "end": 6, "param": param, "pe": _windowed_pe(n_freqs, 2.0)}


def _time_group(freq_multiplier=None) -> dict:
    return {"start": 7, "end": 8, "param": {"n_dims": 1, "fn": "identity"}, "pe": _windowed_pe(2, freq_multiplier)}


def _heads(z_ch: int, flow_fac, sigma_shift: float, offset_fac: float) -> dict:
    outs = {"z_vals": {"channels": z_ch}}
    if flow_fac is not None:
        outs["spatial_flow"] = {"channels": 3, "activation": {"type": "identity", "outer_fac": flow_fac}}
    outs["sigma"] = {"channels": 1, "activation": _ease({"type": "sigmoid", "shift": sigma_shift}, 1.0, 3, 0)}
    outs["point_sigma"] = {"channels": 1, "activation": _ease({"type": "sigmoid", "shift": 4.0}, 1.0, 3, 1)}
    outs["point_offset"] = {"channels": 3, "activation": {"type": "tanh", "outer_fac": offset_fac}}
    outs["color_scale"] = {"channels": 3, "activation": _ease(_identity_full(), 0.0, 0, 0)}
    outs["color_shift"] = {"channels": 3, "activation": _ease(_identity_full(), 0.0, 0, 0)}
    return outs


def _flow_block() -> dict:
    fac = {"type": "identity", "fac": 0.25}
    return {"type": "advect_points", "use_spatial_flow": True, "use_angular_flow": False,
            "out_flow_field": "raw_flow", "flow_scale": 0.0, "spatial_flow_activation": dict(fac),
            "angular_flow_rotation_activation": dict(fac), "angular_flow_anchor_activation": dict(fac)}


_DYN_FIELDS = ["points", "distances", "base_times", "time_offset", "times", "viewdirs", "weights",
               "color_transform_global", "color_scale_global", "color_shift_global",
               "color_transform", "color_scale", "color_shift"]
_STATIC_FIELDS = ["points", "distances", "viewdirs", "weights", "color_scale", "color_shift"]


def _tensorf(net_type: str, aabb, n_init: int, n_final: int, comps, shading: str, dim: int, distance_scale: float,
             alpha_list, density_mode: bool) -> dict:
    net = {"type": net_type, "white_bg": 0, "black_bg": 0, "fea2denseAct": "relu", "distance_scale": distance_scale,
           "density_shift": 0.0, "aabb": aabb, "N_voxel_init": n_init, "N_voxel_final": n_final,
           "upsamp_list": [4000, 6000, 8000, 10000, 12000], "lr_upsample_reset": True,
           "update_AlphaMask_list": alpha_list, "rm_weight_mask_thre": 0, "alpha_mask_thre": 1e-3,
           "n_lamb_sigma": list(comps), "n_lamb_sh": list(comps), "shadingMode": shading, "data_dim_color": dim}
    if density_mode:
        net["densityMode"] = "Density"
    return net


def _model(params: dict, net_cfg: dict, S: int, outputs: dict, intersect: dict, flow: bool, offset: dict,
           extra_outputs, fields, color_net: dict) -> dict:
    embeddings = {
        "ray_prediction_0": {"type": "ray_prediction", "params": params, "net": net_cfg, "z_channels": S,
                             "outputs": outputs},
        "ray_intersect_0": {"type": "ray_intersect", "z_channels": S, "intersect": intersect},
    }
    if flow:
        embeddings["flow_0"] = _flow_block()
    embeddings["point_offset_0"] = offset
    embeddings["add_point_outputs_0"] = {"type": "add_point_outputs", "extra_outputs": list(extra_outputs)}
    embeddings["extract_fields"] = {"type": "extract_fields", "fields": list(fields)}
    return {"type": "lightfield", "render": {"type": "lightfield"}, "param": {"n_dims": 6, "fn": "identity"},
            "embedding": {"type": "ray_point", "embeddings": embeddings},
            "color": {"type": "base", "net": color_net}}


def _mlp(depth: int, width: int, skips) -> dict:
    return {"type": "base", "group": "embedding_impl", "depth": depth, "hidden_channels": width, "skips": list(skips)}


def _z_plane_intersect(contract=None) -> dict:
    it = {"type": "z_plane", "sort": True, "outward_facing": False, "use_disparity": False, "use_sigma": True,
          "out_points": "raw_points", "out_distance": "raw_distance", "initial": -1.0, "end": 1.0}
    if contract is not None:
        it["contract"] = contract
    it["activation"] = {"type": "identity", "fac": 0.5}
    return it


def technicolor_z_plane() -> Cfg:
    """conf/experiment/model/technicolor_z_plane.yaml (BASELINE config 'Technicolor-shape')."""
    return to_cfg(_model(
        params={"ray": _ray_group("two_plane", 0), "time": _time_group()},
        net_cfg=_mlp(6, 256, [3]), S=32, outputs=_heads(1, 0.25, 4.0, 0.25),
        intersect=_z_plane_intersect(), flow=True,
        offset={"type": "point_offset", "in_density_field": "point_sigma", "use_sigma": True},
        extra_outputs=["viewdirs", "times"], fields=_DYN_FIELDS,
        color_net=_tensorf("tensor_vm_split_time", [[-2.0, -2.0, -1.0], [2.0, 2.0, 1.0]], 2097152, 512000000,
                           [8, 0, 0], "SH", 27, 16.0, [4000, 8000], True)))


def neural_3d_z_plane() -> Cfg:
    """conf/experiment/model/neural_3d_z_plane.yaml (BASELINE config 'Neural-3D-shape')."""
    contract = {"type": "mipnerf", "contract_samples": True, "contract_start_radius": 1.0, "contract_end_radius": 8.0}
    return to_cfg(_model(
        params={"ray": _ray_group("pluecker", 1), "time": _time_group(2.0)},
        net_cfg=_mlp(6, 256, [3]), S=64, outputs=_heads(1, 4.0, 1.0, 0.25),
        intersect=_z_plane_intersect(contract), flow=True,
        offset={"type": "point_offset", "in_density_field": "point_sigma", "use_sigma": True},
        extra_outputs=["viewdirs", "times"], fields=_DYN_FIELDS,
        color_net=_tensorf("tensor_vm_split_time", [[-2.0, -1.5, -1.25], [2.0, 1.5, 1.25]], 2097152, 262144000,
                           [8, 4, 4], "SH", 27, 16.0, [], True)))


def donerf_sphere() -> Cfg:
    """conf/experiment/model/donerf_sphere.yaml (BASELINE config 'DoNeRF-shape')."""
    intersect = {"type": "sphere", "sort": True, "outward_facing": False, "use_disparity": False, "max_axis": False,
                 "use_sigma": True, "out_points": "raw_points", "out_distance": "raw_distance",
                 "use_dataset_bounds": True, "origin_scale_factor": 0.0,
                 "contract": {"type": "mipnerf", "contract_samples": True, "use_dataset_bounds": True},
                 "activation": {"type": "identity", "fac": 0.5}}
    return to_cfg(_model(
        params={"ray": _ray_group("pluecker", 1)},
        net_cfg=_mlp(6, 256, [3]), S=32, outputs=_heads(4, None, 4.0, 0.125),
        intersect=intersect, flow=False, offset={"type": "point_offset", "use_sigma": True},
        extra_outputs=["viewdirs"], fields=_STATIC_FIELDS,
        color_net=_tensorf("tensor_vm_split_no_sample", [[-2.0, -2.0, -2.0], [2.0, 2.0, 2.0]], 3375000, 216000000,
                           [8, 4, 4], "RGB", 3, 16.0, [4000, 8000], False)))


def shiny_z_plane_tiny() -> Cfg:
    """conf/experiment/model/shiny_z_plane_tiny.yaml (static z-plane, W=128, S=8; plumbing-size net)."""
    return to_cfg(_model(
        params={"ray": _ray_group("two_plane", 1)},
        net_cfg=_mlp(4, 128, [2]), S=8, outputs=_heads(1, None, 4.0, 0.25),
        intersect=_z_plane_intersect(), flow=False,
        offset={"type": "point_offset", "in_density_field": "point_sigma", "use_sigma": True},
        extra_outputs=["viewdirs"], fields=_STATIC_FIELDS,
        color_net=_tensorf("tensor_vm_split_no_sample", [[-2.0, -2.0, -1.0], [2.0, 2.0, 1.0]], 2097152, 262144000,
                           [8, 4, 4], "RGB", 3, 8.0, [4000, 8000], False)))


# dataset facts used with each built-in (SURVEY.md section 8(d)): reference defaults K = 50 // 4 = 12
DATASETS: Dict[str, dict] = {
    "technicolor_z_plane": {"name": "technicolor", "collection": "synthetic", "num_keyframes": 12, "num_frames": 50,
                            "near": 0.0, "far": 1.0, "depth_range": [0.0, 1.0]},
    "neural_3d_z_plane": {"name": "neural_3d", "collection": "synthetic", "num_keyframes": 12, "num_frames": 50,
                          "near": 0.0, "far": 1.0, "depth_range": [0.0, 1.0]},
    "donerf_sphere": {"name": "donerf", "collection": "synthetic", "num_keyframes": 1, "num_frames": 1,
                      "near": 0.5, "far": 10.0, "depth_range": [0.5, 10.0]},
    "shiny_z_plane_tiny": {"name": "shiny", "collection": "synthetic", "num_keyframes": 1, "num_frames": 1,
                           "near": 0.0, "far": 1.0, "depth_range": [0.0, 1.0]},
}

BUILTIN = {
    "technicolor_z_plane": technicolor_z_plane,
    "neural_3d_z_plane": neural_3d_z_plane,
    "donerf_sphere": donerf_sphere,
    "shiny_z_plane_tiny": shiny_z_plane_tiny,
}


def get(name: str, **overrides) -> Tuple[Cfg, dict]:
    """(model cfg, dataset dict) of a built-in.  Overrides: ``z_channels`` (S), ``n_voxels`` (sets
    N_voxel_init = N_voxel_final, i.e. a grid already at that size), ``num_keyframes``, ``num_frames``."""
    cfg = BUILTIN[name]()
    ds = dict(DATASETS[name])
    if "z_channels" in overrides:
        S = int(overrides["z_channels"])
        cfg.embedding.embeddings.ray_prediction_0.z_channels = S
        cfg.embedding.embeddings.ray_intersect_0.z_channels = S
    if "n_voxels" in overrides:
        cfg.color.net.N_voxel_init = int(overrides["n_voxels"])
        cfg.color.net.N_voxel_final = int(overrides["n_voxels"])
    for k in ("num_keyframes", "num_frames"):
        if k in overrides:
            ds[k] = int(overrides[k])
    for v in _as_list(overrides.get("variant")):
        _apply_variant(cfg, v)
    return cfg, ds


def _as_list(v):
    return [] if v is None else ([v] if isinstance(v, str) else list(v))


def _apply_variant(cfg: Cfg, variant: str) -> None:
    """Schema-level edits that turn a built-in into the other shipped pipeline families (SURVEY 8 f3): the result is
    still a valid reference config (the parity tests build the unmodified reference from it)."""
    emb = cfg.embedding.embeddings
    pred, it = emb.ray_prediction_0, emb.ray_intersect_0.intersect
    if variant == "basic_pe":  # technicolor_z_plane_{small,tiny,large}.yaml: `pe: {type: basic}`
        for g in pred.params.values():
            if "pe" in g and g.pe is not None:
                g.pe = to_cfg({"type": "basic", "n_freqs": int(g.pe.n_freqs), "freq_multiplier": 2.0})
    elif variant == "wide_pe":  # stanford_z_plane_mem.yaml / immersive_cylinder_pe.yaml: more PE bands -> 33..64 input features
        pred.params.ray.pe.n_freqs = 4
    elif variant == "zero_net":  # technicolor_z_plane_no_sample.yaml:55-57: `net: {type: zero}` -- samples stay on their base planes
        pred.net.type = "zero"
    elif variant == "distance":  # catacaustics_distance.yaml:113-134: samples at signed distances from the ray's closest point
        if it.type != "sphere":
            raise ValueError("the distance variant starts from a sphere pipeline")
        it.type = "euclidean_distance_unified"
        pred.outputs.z_vals.channels = 1
        for k in ("origin_scale_factor", "max_axis"):
            if k in it:
                del it[k]
    elif variant == "bbox":  # technicolor_z_plane_world.yaml:143-147
        it.contract = to_cfg({"type": "bbox", "contract_samples": True, "bbox_min": [-2.0, -2.0, 0.5],
                              "bbox_max": [2.0, 2.0, -2.5]})
    elif variant == "z_depth":
        it.contract = to_cfg({"type": "z_depth", "contract_samples": True, "contract_end_radius": 3.0})
    elif variant == "cylinder":  # donerf_cylinder.yaml / immersive_cylinder.yaml: `type: cylinder`
        if it.type != "sphere":
            raise ValueError("the cylinder variant starts from a sphere pipeline")
        it.type = "cylinder"
    elif variant == "sphere":  # immersive_sphere.yaml: a dynamic (keyframe) pipeline behind sphere primitives
        if it.type != "z_plane":
            raise ValueError("the sphere variant starts from a z_plane pipeline")
        it.type = "sphere"
        it.origin_scale_factor = 0.0
        pred.outputs.z_vals.channels = 4
        for k in ("initial", "end"):
            if k in it:
                del it[k]
        it.use_dataset_bounds = True
    elif variant == "sphere_new":  # immersive_sphere_new.yaml:153-172 / bom_sphere.yaml:149-163
        if it.type not in ("z_plane", "sphere"):
            raise ValueError("the sphere_new variant starts from a z_plane or sphere pipeline")
        it.type = "sphere_new"
        it.origin_scale_factor = 1.0
        it.resize_scale_factor = 1.0
        pred.outputs.z_vals.channels = 8
        for k in ("initial", "end"):
            if k in it:
                del it[k]
        it.use_dataset_bounds = True
    elif variant == "scale_mask":  # shiny_z_plane.yaml:143 (num_samples_for_scale), stanford_llff_z_plane.yaml:142-143 (mask)
        it.num_samples_for_scale = 2 * int(emb.ray_intersect_0.z_channels)
        it.mask = to_cfg({"stop_iters": -1})
    elif variant == "z_scale":
        it.z_scale = 0.05
    elif variant == "outward_facing":  # immersive_*.yaml / bom_*.yaml
        it.outward_facing = True
    elif variant == "global_color":  # catacaustics_z_plane.yaml:77-100,148: per-ray scale / shift after compositing
        outs = pred.outputs
        for a, b in (("color_scale", "color_scale_global"), ("color_shift", "color_shift_global")):
            items = [(b if k == a else k, v) for k, v in outs.items()]
            for k in list(outs.keys()):
                del outs[k]
            for k, v in items:
                outs[k] = v
        f = emb.extract_fields.fields
        emb.extract_fields.fields = [{"color_scale": "color_scale_global", "color_shift": "color_shift_global"}.get(k, k) for k in f]
    elif variant == "both_color":  # per-sample and per-ray heads together (immersive_*.yaml field lists)
        outs = pred.outputs
        outs["color_scale_global"] = copy.deepcopy(outs["color_scale"])
        outs["color_shift_global"] = copy.deepcopy(outs["color_shift"])
        emb.extract_fields.fields = list(emb.extract_fields.fields) + ["color_scale_global", "color_shift_global"]
    else:
        raise ValueError(f"unknown variant {variant}")
