"""The oracle, the built-in configs, the lowering and the training-schedule pieces against what the unmodified reference
builds and computes on the same inputs, recorded in tests/golden/reference/ by tests/golden/make_golden_reference.py."""
import json
import os

import numpy as np
import pytest
import torch

from oracle.hyperreel_oracle import HyperReelOracle
from tests.cases import build_case
from tests.golden import make_golden_reference as G

REF = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference")


def recorded(name):
    with np.load(os.path.join(REF, name + ".npz")) as z:
        return {k: z[k] for k in z.files}


def shipped_yamls():
    """name -> plain model config of every shipped model YAML (None: the empty bom_z_plane.yaml)"""
    return {k: json.loads(str(v)) for k, v in recorded("model_yamls").items()}


def shipped_cfg(name):
    import hyperreel_b200 as hb
    return hb.to_cfg(shipped_yamls()[name])


def _floatify(o):
    if isinstance(o, dict):
        return {k: _floatify(v) for k, v in o.items()}
    if isinstance(o, list):
        return [_floatify(v) for v in o]
    if isinstance(o, str):
        try:
            return float(o)  # PyYAML 1.1 reads `1e-3` as a string
        except ValueError:
            return o
    return o


@pytest.mark.parametrize("name", G.BUILTIN_NAMES)
def test_builtin_config_equals_reference_yaml(name):
    from hyperreel_b200 import configs
    from hyperreel_b200.config import to_plain
    ref = _floatify(json.loads(str(recorded("builtin_configs")[name])))
    mine = _floatify(to_plain(configs.BUILTIN[name]()))
    assert ref == mine
    # ordered sections: embedding order, head order and param-group order are semantic
    e_ref, e_mine = ref["embedding"]["embeddings"], mine["embedding"]["embeddings"]
    assert list(e_ref) == list(e_mine)
    assert list(e_ref["ray_prediction_0"]["outputs"]) == list(e_mine["ray_prediction_0"]["outputs"])
    assert list(e_ref["ray_prediction_0"]["params"]) == list(e_mine["ray_prediction_0"]["params"])


@pytest.mark.parametrize("name", G.FRESH_CASES)
def test_oracle_matches_live_reference_on_fresh_rays(name):
    case = build_case(name, n=G.FRESH_N)
    want = recorded("fresh_rays")
    st = {}
    rgb = HyperReelOracle(case.model_cfg_plain, case.dataset, case.state_dict).render(case.rays.clone(), st)
    assert (rgb - torch.from_numpy(want[f"{name}/rgb"])).abs().max() <= 2e-6
    n, rows = case.rays.shape[0], torch.from_numpy(G.ROWS_FRESH)
    assert (st["points"].reshape(n, -1)[rows] - torch.from_numpy(want[f"{name}/points"])).abs().max() <= 2e-6
    assert (st["distances"].reshape(n, -1)[rows] - torch.from_numpy(want[f"{name}/distances"])).abs().max() <= 2e-6


@pytest.mark.parametrize("name", G.EDGE_CASES)
def test_oracle_matches_reference_on_crafted_edge_rays(name):
    """The rays of tests/test_edge_rays_gpu.py (plane-parallel, keyframe boundaries, far / centred origins, un-normalised
    directions): the oracle must still equal the unmodified reference there before it may judge the CUDA path."""
    from tests.test_edge_rays_gpu import craft

    case = build_case(name)
    rays = craft(case)
    a = torch.from_numpy(recorded("edge_rays")[name])
    b = HyperReelOracle(case.model_cfg_plain, case.dataset, case.state_dict).render(rays.clone())
    assert torch.isfinite(a).all()
    assert float((a.reshape(b.shape) - b).abs().max()) <= 2e-6


def test_oracle_matches_reference_on_every_shipped_yaml_that_lowers():
    """Every model YAML the reference ships that the fused path accepts: the configuration as the reference ships it (grid
    shrunk to 24^3 for speed), seeded parameters, and the oracle held to the reference's rgb on seeded rays.  This pins the
    oracle's reading of the real configuration files, not only of the built-ins and their variants."""
    import hyperreel_b200 as hb
    from hyperreel_b200.config import to_plain
    from hyperreel_b200.signature import UnsupportedPipeline
    from hyperreel_b200.state import seeded_state_dict

    want = recorded("every_shipped_yaml")
    checked, nonzero = 0, 0
    for name, plain in shipped_yamls().items():
        if plain is None:  # bom_z_plane.yaml is empty
            continue
        cfg = hb.to_cfg(plain)
        cfg.color.net.N_voxel_init = 24 ** 3
        cfg.color.net.N_voxel_final = 24 ** 3
        try:
            sig = hb.lower(cfg, G.DS_R2)
        except UnsupportedPipeline:
            continue
        sd = seeded_state_dict(sig, seed=3, density_gain=30.0)
        rays = hb.rays.for_signature(sig, 48, seed=9)
        a = torch.from_numpy(want[name])
        b = HyperReelOracle(to_plain(cfg), G.DS_R2, sd).render(rays.clone())
        assert float((a.reshape(b.shape) - b).abs().max()) <= 2e-6, name
        checked += 1
        nonzero += int(float(b.abs().max()) > 0)
    assert checked == len(want) >= 45 and nonzero >= 40


@pytest.mark.parametrize("name", ["technicolor_z_plane", "donerf_sphere"])
def test_grid_upsampling_and_regulariser_terms_match_the_reference(name):
    """The training-schedule pieces mirrored on the host (SURVEY.md 8 row f1): `upsample_volume_grid` re-samples every table
    exactly like the reference's (tensorf_base.py:1151-1188, tensorf_dynamic.py:394-441), and the TensoRF regulariser's terms
    (density_L1, TV on the space planes; nlf/regularizers/tensorf.py:14-96) agree on the same parameters."""
    import hyperreel_b200 as hb
    from hyperreel_b200.state import _Color, seeded_state_dict
    from hyperreel_b200.system import TVLoss

    want = recorded("upsampling_and_regulariser_terms")
    cfg = shipped_cfg(name)
    cfg.color.net.N_voxel_init, cfg.color.net.N_voxel_final = 12 ** 3, 20 ** 3
    sig = hb.lower(cfg, G.DS)
    sd = seeded_state_dict(sig, seed=4)
    mine = _Color(sig, hb.state.default_grid(sig))
    mine.load_state_dict({k[len("model.color_model."):]: v for k, v in sd.items() if k.startswith("model.color_model.")}, strict=False)
    l1, tv_d, tv_a = (float(v) for v in want[f"{name}/terms"])
    assert abs(l1 - float(mine.net.density_L1())) <= 1e-7
    assert abs(tv_d - float(mine.net.TV_loss_density(TVLoss()))) <= 1e-9
    assert abs(tv_a - float(mine.net.TV_loss_app(TVLoss()))) <= 1e-7
    # the schedule: same voxel counts, same re-sampled tables
    assert want[f"{name}/N_voxel_list"].tolist() == [int(v) for v in mine.net.N_voxel_list]
    reso = hb.state.n_to_reso(int(mine.net.N_voxel_list[0]), torch.tensor(cfg.color.net.aabb))
    mine.net.upsample_volume_grid(reso)
    assert want[f"{name}/gridSize"].tolist() == mine.net.gridSize.tolist() == list(reso)
    got = mine.state_dict()
    prefix = f"{name}/tab/"
    tabs = {k[len(prefix):]: v for k, v in want.items() if k.startswith(prefix)}
    assert tabs
    for k, v in tabs.items():
        assert torch.equal(torch.from_numpy(v), got["net." + k]), k


def test_tensorf_regulariser_loss_sequence_matches_the_reference():
    """hyperreel_b200.system.TensoRFRegularizer against nlf/regularizers/tensorf.py:35-96 (the unmodified class, its base
    replaced by a stand-in): same loss over several calls -- including the reference's running-weight bookkeeping (the TV
    weights decay per call, the density TV term is counted again inside the appearance term) and the L1 switch at the first
    alpha-mask iteration."""
    import hyperreel_b200 as hb
    from hyperreel_b200.state import _Color, seeded_state_dict
    from hyperreel_b200.system import TensoRFRegularizer

    want = recorded("regulariser_sequence")
    cfg = shipped_cfg("technicolor_z_plane")
    cfg.color.net.N_voxel_init = cfg.color.net.N_voxel_final = 14 ** 3
    sig = hb.lower(cfg, G.DS)
    sd = seeded_state_dict(sig, seed=6)
    mine = TensoRFRegularizer(dict(G.REG_CFG))
    net = _Color(sig, hb.state.default_grid(sig))
    net.load_state_dict({k[len("model.color_model."):]: v for k, v in sd.items() if k.startswith("model.color_model.")}, strict=False)
    for it in range(6):
        mine.set_iter(it)
        a = float(want["losses"][it])
        b = float(mine.loss(net.net))
        assert abs(a - b) <= 1e-7 * max(1.0, abs(a)), (it, a, b)
    assert mine.L1_reg_weight == 4e-5 and abs(mine.TV_weight_density - float(want["TV_weight_density"])) < 1e-12


def test_oracle_stages_match_the_reference_on_the_round_2_families():
    """Beyond rgb: the sample points and distances the oracle computes for the voxel-grid, plane-grid, colour-transform, 128 /
    256-sample and cascaded (point_prediction) YAMLs equal what the unmodified reference's `render_fn.embed` returns -- the GPU
    stage tests (tests/test_widened_gpu.py) lean on exactly these oracle stages."""
    import hyperreel_b200 as hb
    from hyperreel_b200.config import to_plain
    from hyperreel_b200.state import seeded_state_dict

    want = recorded("round_2_stages")
    rows = torch.from_numpy(G.ROWS_R2)
    for name in G.R2_FAMILIES:
        cfg = shipped_cfg(name)
        cfg.color.net.N_voxel_init = cfg.color.net.N_voxel_final = 16 ** 3
        sig = hb.lower(cfg, G.DS_R2)
        sd = seeded_state_dict(sig, seed=5, density_gain=30.0)
        rays = hb.rays.for_signature(sig, 40, seed=3)
        st = {}
        rgb = HyperReelOracle(to_plain(cfg), G.DS_R2, sd).render(rays.clone(), st)
        n = rays.shape[0]
        assert float((rgb - torch.from_numpy(want[f"{name}/rgb"]).reshape(rgb.shape)).abs().max()) <= 2e-6, name
        assert float((st["points"].reshape(n, -1)[rows] - torch.from_numpy(want[f"{name}/points"])).abs().max()) <= 2e-6, name
        assert float((st["distances"].reshape(n, -1)[rows] - torch.from_numpy(want[f"{name}/distances"])).abs().max()) <= 2e-6, name


@pytest.mark.parametrize("name,gain", [("technicolor_z_plane", 40000.0), ("donerf_sphere", 40000.0)])
def test_alpha_mask_update_and_shrink_match_the_reference(name, gain):
    """The pruning step of the training schedule (tensorf_base.py:379-429,1190-1232 / tensorf_dynamic.py:443-541): dense
    occupancy, mask, bounding box, cropped tables and corrected aabb equal the unmodified reference's on the same parameters;
    a second mask update (which, in the static net, consults the first mask) as well."""
    import hyperreel_b200 as hb
    from hyperreel_b200.state import _Color, seeded_state_dict

    want = recorded("alpha_mask")
    cfg = shipped_cfg(name)
    cfg.color.net.N_voxel_init = cfg.color.net.N_voxel_final = 13 ** 3
    sig = hb.lower(cfg, G.ALPHA_DS)
    sd = G.corner_occupancy(seeded_state_dict(sig, seed=8), gain)
    mine = _Color(sig, hb.state.default_grid(sig))
    mine.load_state_dict({k[len("model.color_model."):]: v for k, v in sd.items() if k.startswith("model.color_model.")}, strict=False)
    reso = tuple(mine.net.gridSize.tolist())
    a_ref = torch.from_numpy(want[f"{name}/alpha"])
    with torch.no_grad():
        a_mine, _ = mine.net.getDenseAlpha(reso)
    # (the reference evaluates slab by slab, here in one batch: the same values up to the last bit or two)
    assert float((a_ref - a_mine).abs().max()) <= 1e-6 and float(a_ref.max()) > 0.05 > 0.001 > float(a_ref.min())
    box_ref = torch.from_numpy(want[f"{name}/box"])
    box_mine = mine.net.updateAlphaMask(reso)
    assert torch.equal(box_ref, box_mine)
    assert torch.equal(torch.from_numpy(want[f"{name}/alpha_volume"]), mine.net.alphaMask.volume)
    mine.net.shrink(box_mine)
    grid = want[f"{name}/gridSize"].tolist()
    assert grid == mine.net.gridSize.tolist() and any(g < r for g, r in zip(grid, reso))
    assert torch.equal(torch.from_numpy(want[f"{name}/aabb"]), mine.net.aabb)
    got = mine.state_dict()
    prefix = f"{name}/tab/"
    tabs = {k[len(prefix):]: v for k, v in want.items() if k.startswith(prefix)}
    assert tabs
    for k, v in tabs.items():
        assert torch.equal(torch.from_numpy(v), got["net." + k]), k
    reso2 = tuple(mine.net.gridSize.tolist())
    assert torch.equal(torch.from_numpy(want[f"{name}/box2"]), mine.net.updateAlphaMask(reso2))


def test_lowered_constants_equal_the_reference_constructors_on_every_shipped_yaml():
    """hyperreel_b200.signature.lower (product host code) against the objects the unmodified reference builds from the same YAML
    and dataset facts: base primitives (`samples`), their spacing (`z_scale`), the mask bounds, the contraction radii, and the
    colour net's scalars -- for all 45 shipped model YAMLs that run, under two sets of dataset facts."""
    import hyperreel_b200 as hb
    from hyperreel_b200 import lib as L
    from hyperreel_b200.signature import UnsupportedPipeline

    want = recorded("lowered_constants")
    checked = 0
    for name, plain in shipped_yamls().items():
        if plain is None:
            continue
        cfg = hb.to_cfg(plain)
        cfg.color.net.N_voxel_init = cfg.color.net.N_voxel_final = 12 ** 3
        for fi, ds in enumerate(G.FACTS):
            try:
                sig = hb.lower(cfg, ds)
            except UnsupportedPipeline:
                continue
            c = sig.cfg
            r = json.loads(str(want[f"{name}/{fi}"]))
            S = c.n_samples
            assert torch.equal(torch.tensor(list(c.samples)[:S]), torch.tensor(r["samples"])), name
            zs = torch.tensor(r["z_scale"])
            if c.isect_type == L.ISECT_VOXEL:
                assert torch.equal(torch.tensor(list(c.z_scale3)), zs), name
            else:
                assert abs(c.z_scale - float(zs[0])) <= 1e-7 * max(1.0, abs(float(zs[0]))), name
            f32 = lambda v: float(torch.tensor(float(v), dtype=torch.float32))  # the struct holds fp32, like the tensors they meet
            if r["masked"]:  # otherwise nothing is masked and the bounds are irrelevant
                assert c.isect_near == f32(r["near"]) and c.isect_far == f32(r["far"]), name
            if c.contract_type == L.CONTRACT_MIPNERF:
                assert (c.contract_start_radius, c.contract_end_radius, c.contract_start_distance, c.contract_end_distance) == \
                    tuple(f32(v) for v in r["contract"]), name
            if c.cascade:
                assert torch.equal(torch.tensor(list(c.pre_samples_tab)[:c.pre_samples]), torch.tensor(r["pre_samples"])), name
                assert abs(c.pre_z_scale - r["pre_z_scale"]) <= 1e-7, name
            assert c.distance_scale == f32(r["distance_scale"]) and c.weight_thre == f32(r["weight_thre"]), name
            assert bool(c.white_bg) == r["white_bg"] and bool(c.black_bg) == r["black_bg"], name
            assert [c.aabb[i] for i in range(6)] == [f32(v) for v in r["aabb"]], name
            assert hb.state.default_grid(sig) == r["gridSize"], name
            if c.dynamic:
                assert [c.num_keyframes, c.num_frames] == r["keyframes_frames"], name
            checked += 1
    assert checked == len(want) == 90


def test_lowered_activations_equal_the_reference_modules_on_every_shipped_yaml():
    """signature.resolve_activation lowers every head / intersect / flow / offset activation to y = f(x * inner + shift) * outer
    (the form the kernels evaluate): the same numbers as the reference's activation modules at render iteration, for every
    activation of all shipped YAMLs that lower."""
    import hyperreel_b200 as hb
    from hyperreel_b200 import lib as L
    from hyperreel_b200.config import epochs_to_iters
    from hyperreel_b200.signature import RENDER_ITER, UnsupportedPipeline, resolve_activation

    want = recorded("activations")
    x = G.ACT_X
    n = 0
    for name, plain in shipped_yamls().items():
        if plain is None:
            continue
        try:
            hb.lower(hb.to_cfg(plain), G.DS_R2)
        except UnsupportedPipeline:
            continue
        for path, acfg in G.walk_activations(epochs_to_iters(plain, 1)["embedding"]):
            if isinstance(acfg, dict) and "type" not in acfg:
                continue
            try:
                act = resolve_activation(hb.to_cfg(acfg) if isinstance(acfg, dict) else acfg, RENDER_ITER)
            except UnsupportedPipeline:
                continue  # an activation of an embedding the fused path does not evaluate (e.g. angular flow): never lowered
            ref = torch.from_numpy(want[f"{name}{path}"])
            v = x * act.inner_fac + act.shift
            v = torch.sigmoid(v) if act.kind == L.ACT_SIGMOID else (torch.tanh(v) if act.kind == L.ACT_TANH else v)
            got = v * act.outer_fac
            assert float((got - ref).abs().max()) <= 1e-6, (name, path)
            n += 1
    assert n > 300
