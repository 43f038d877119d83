"""CUDA path vs the unmodified reference for every model YAML the reference ships and the fused path accepts
(tests/golden/shipped/*.npz, see tests/test_shipped_yaml_golden.py for the fixture format and the CPU half).

A regression fails the suite.  The tensor-core
sample net covers every one of them (hidden width 128 / 256, encoded inputs up to 64 features): no skips."""
import os

import pytest
import torch

import hyperreel_b200 as hb
from tests.test_parity_gpu import RGB_TOL
from tests.test_shipped_yaml_golden import SHIPPED, load_fixture

pytestmark = pytest.mark.gpu


def _render(cfg, ds, sd, rays, mode):
    model = hb.LightfieldModel(cfg, dataset=ds, mlp_mode=mode)
    render = hb.RenderLightfield(model, None, cfg.render, net_chunk=1 << 20)
    _, unexpected = render.load_state_dict(sd, strict=False)
    assert not unexpected
    render.eval()
    return render(rays.cuda())["rgb"].cpu()


@pytest.mark.parametrize("path", SHIPPED, ids=[os.path.basename(p)[:-4] for p in SHIPPED])
def test_shipped_yaml_fp32_path_matches_reference(path):
    plain, cfg, ds, sig, sd, rays, rgb = load_fixture(path)
    out = _render(cfg, ds, sd, rays, "fp32")
    assert float((out - rgb).abs().max()) <= RGB_TOL


@pytest.mark.parametrize("path", SHIPPED, ids=[os.path.basename(p)[:-4] for p in SHIPPED])
def test_shipped_yaml_tensor_core_path_matches_reference(path):
    plain, cfg, ds, sig, sd, rays, rgb = load_fixture(path)
    out = _render(cfg, ds, sd, rays, "auto")
    assert float((out - rgb).abs().max()) <= RGB_TOL
