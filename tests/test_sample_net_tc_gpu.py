"""The wgmma (bf16x3 split) sample net against the reference golden vectors and the fp32 CUDA-core path."""
import os

import numpy as np
import pytest
import torch

import hyperreel_b200 as hb
from tests.cases import CASES, build_case
from tests.test_parity_gpu import GOLDEN, RGB_TOL, make_render

pytestmark = pytest.mark.gpu
TC_CASES = list(CASES)  # hidden width 128 (shiny_*) and 256, encoded inputs of one or two 32-feature chunks (*_wide_pe)


@pytest.mark.parametrize("name", TC_CASES)
def test_tc_sample_net_output_matches_reference(name):
    case = build_case(name)
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    render = make_render(case, mlp_mode="bf16x3")
    st = render.model.render_stages(case.rays.cuda())
    got = st["mlp_out"][:64].cpu().numpy()
    scale = max(1.0, float(np.abs(g["mlp_out"]).max()))
    err = np.abs(got - g["mlp_out"]).max()
    assert err <= 1e-4 * scale, f"{name}: sample-net max abs error {err}"
    assert np.abs(st["rgb"].cpu().numpy() - g["rgb"]).max() <= RGB_TOL


@pytest.mark.parametrize("name", ["technicolor_trained", "neural3d_trained", "donerf_wide_pe", "neural3d_wide_pe", "shiny_tiny"])
def test_tc_matches_fp32_path_on_many_tiles(name):
    """Several persistent tiles per CTA + a ragged last tile; compare with the fp32 CUDA-core sample net."""
    case = build_case(name, n=128 * 300 + 77)
    a = make_render(case, mlp_mode="fp32").model.render_stages(case.rays.cuda())
    b = make_render(case, mlp_mode="bf16x3").model.render_stages(case.rays.cuda())
    scale = max(1.0, float(a["mlp_out"].abs().max()))
    assert float((a["mlp_out"] - b["mlp_out"]).abs().max()) <= 1e-4 * scale
    assert float((a["rgb"] - b["rgb"]).abs().max()) <= RGB_TOL


def test_default_mode_is_the_tensor_core_net():
    """The registry path (no mlp_mode argument, like the reference constructor) must run the wgmma kernel."""
    from hyperreel_b200 import lib as L

    case = build_case("technicolor_trained")
    model = hb.LightfieldModel(case.model_cfg, dataset=case.dataset)
    assert model.sig.cfg.mlp_mode == L.MLP_BF16X3_TC
    system = hb.INRSystem(hb.to_cfg({"model": case.model_cfg, "training": {"iters_per_epoch": 4000}, "dataset": case.dataset}))
    assert system.render_fn.model.sig.cfg.mlp_mode == L.MLP_BF16X3_TC
