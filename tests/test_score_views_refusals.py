"""Host-side refusals of score_views and INRSystem.validation_views: malformed input raises ValueError before any device
work, a CPU image tensor raises RuntimeError (there is no CPU path)."""
import numpy as np
import pytest
import torch

import hyperreel_b200 as hb
from tests.cases import build_case

K = [[20.0, 0, 8], [0, 20.0, 6], [0, 0, 1]]


def _cams(n=3, w=16, h=12):
    return [hb.Camera(pose=np.eye(4)[:3], K=K, width=w, height=h) for _ in range(n)]


def _model():
    case = build_case("technicolor_trained")
    model = hb.LightfieldModel(case.model_cfg, dataset=case.dataset)
    model.eval()
    return model, case


def test_score_views_refusals():
    model, _ = _model()
    cams = _cams()
    images = torch.zeros((3, 12, 16, 3), dtype=torch.uint8)
    with pytest.raises(ValueError, match="no cameras"):
        hb.score_views(model, [], images)
    with pytest.raises(ValueError, match="3 cameras but 2 times"):
        hb.score_views(model, cams, images, [0.0, 1.0])
    with pytest.raises(ValueError, match="finite"):
        hb.score_views(model, cams, images, [0.0, float("nan"), 1.0])
    odd = cams[:2] + [hb.Camera(pose=np.eye(4)[:3], K=K, width=16, height=13)]
    with pytest.raises(ValueError, match="camera 2 is 16 x 13"):
        hb.score_views(model, odd, images)
    with pytest.raises(ValueError, match="11 x 11"):
        hb.score_views(model, _cams(w=10), torch.zeros((3, 12, 10, 3), dtype=torch.uint8))
    for bad in (torch.zeros((3, 12, 16, 3), dtype=torch.float32), torch.zeros((2, 12, 16, 3), dtype=torch.uint8),
                torch.zeros((3, 16, 12, 3), dtype=torch.uint8), torch.zeros((3, 12, 16, 6), dtype=torch.uint8)[..., ::2],
                np.zeros((3, 12, 16, 3), np.uint8)):
        with pytest.raises(ValueError, match="images must be"):
            hb.score_views(model, cams, bad)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        hb.score_views(model, cams, images)
    with pytest.raises(TypeError):
        hb.score_views(object(), cams, images)
    model.train()
    with pytest.raises(RuntimeError, match="eval"):
        hb.score_views(model, cams, images)


def test_validation_views_refusals_restore_the_mode():
    _, case = _model()
    system = hb.INRSystem(hb.to_cfg({"model": case.model_cfg_plain}), dataset=case.dataset)
    system.train()
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        system.validation_views(_cams(), torch.zeros((3, 12, 16, 3), dtype=torch.uint8))
    assert system.training
    with pytest.raises(ValueError, match="images must be"):
        system.validation_views(_cams(), torch.zeros((3, 12, 16, 3), dtype=torch.float32))
    assert system.training
    with pytest.raises(ValueError, match="no cameras"):
        hb.score_views(system, [], torch.zeros((0, 12, 16, 3), dtype=torch.uint8))
