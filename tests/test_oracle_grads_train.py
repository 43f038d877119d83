"""Gradient oracle (HyperReelOracle.render_with_grad) against the reference's own autograd for the training cases of
tests/cases_train.py (goldens by tests/golden/make_golden_grads_train.py), to the tolerances of tests/test_oracle_grads.py;
and the check that every such case is non-trivial (sum w > 0.5 on at least a quarter of the rays)."""
import os

import numpy as np
import pytest

from oracle.hyperreel_oracle import HyperReelOracle
from tests.cases_train import TRAIN_CASES, build_train_case
from tests.golden.make_golden_grads import probe_indices, target_for

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.mark.parametrize("name", list(TRAIN_CASES))
def test_training_case_is_not_trivial(name):
    case = build_train_case(name)
    st = {}
    HyperReelOracle(case.model_cfg_plain, case.dataset, case.state_dict).render(case.rays.clone(), st)
    sw = st["weights"].sum(-1)
    assert float((sw > 0.5).float().mean()) >= 0.25, name


@pytest.mark.parametrize("name", list(TRAIN_CASES))
def test_oracle_gradients_match_reference_autograd_for_training_cases(name):
    g = np.load(os.path.join(GOLDEN, f"grads_{name}.npz"))
    case = build_train_case(name)
    rays = case.rays.clone()
    orc = HyperReelOracle(case.model_cfg_plain, case.dataset, case.state_dict)
    rgb, leaves = orc.render_with_grad(rays)
    loss = ((rgb - target_for(rays.shape[0])) ** 2).mean()
    loss.backward()
    assert abs(float(loss) - float(g["loss"])) <= 1e-6
    keys = [k[len("norm/"):] for k in g.files if k.startswith("norm/")]
    assert len(keys) >= 17
    if case.sig.cfg.n_color_views > 0:
        assert any(k.endswith("color_embedding") for k in keys)
    for k in keys:
        assert float(g[f"norm/{k}"]) > 0.0, k
        grad = leaves[k].grad
        assert grad is not None, k
        flat = grad.reshape(-1)
        scale = float(g[f"max/{k}"]) + 1e-12
        assert abs(float(flat.norm()) - float(g[f"norm/{k}"])) <= 1e-4 * float(g[f"norm/{k}"]) + 1e-9, k
        probe = flat[probe_indices(flat.numel())].detach().numpy()
        assert np.abs(probe - g[f"probe/{k}"]).max() <= 2e-5 * scale + 1e-10, k
