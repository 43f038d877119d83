"""spiral_path against the reference's render-split camera paths (tests/golden/video_path.npz, made by
make_golden_video_path.py from the unmodified prepare_render_data of each dataset family), and the host-side refusals of
spiral_path and render_video."""
import os

import numpy as np
import pytest
import torch

import hyperreel_b200 as hb
from tests.cases import build_case

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "video_path.npz")
FAMILY = {"technicolor": "technicolor", "neural": "neural_3d", "immersive": "immersive", "donerf": "donerf"}


def _golden():
    z = np.load(GOLDEN)
    return z, sorted({k.split("/")[0] for k in z.files})


def _template():
    return hb.Camera(pose=np.eye(4)[:3], K=[[100.0, 0, 50.0], [0, 100.0, 40.0], [0, 0, 1]], width=100, height=80, cam_idx=3.0)


@pytest.mark.parametrize("case", _golden()[1])
def test_spiral_path_equals_the_reference(case):
    z, _ = _golden()
    nf, ss, interp, interp_t = (int(v) for v in z[f"{case}/params"])
    cams, times = hb.spiral_path(FAMILY[case.split("_")[0]], _template(), z[f"{case}/poses_in"], z[f"{case}/bounds"],
                                 num_frames=nf, supersample=ss, interpolate=bool(interp), interpolate_time=bool(interp_t))
    poses = np.stack([np.asarray(c.pose) for c in cams], 0)
    assert poses.dtype == np.float32 and times.dtype == np.float32
    assert poses.shape == z[f"{case}/poses"].shape
    assert np.array_equal(poses, z[f"{case}/poses"])
    assert np.array_equal(times, z[f"{case}/times"])
    assert all(c.time == float(t) for c, t in zip(cams, times))
    assert all(c.width == 100 and c.height == 80 and c.cam_idx == 3.0 for c in cams)


def test_the_fixture_covers_every_family():
    _, cases = _golden()
    assert {FAMILY[c.split("_")[0]] for c in cases} == set(hb.camera.SPIRAL_DATASETS)


def test_spiral_path_refusals():
    z, _ = _golden()
    P, b = z["neural_3d_video/poses_in"], z["neural_3d_video/bounds"]
    cam = _template()
    with pytest.raises(ValueError, match="dataset"):
        hb.spiral_path("llff", cam, P, b)
    with pytest.raises(ValueError, match=r"\[N, 3, 4\]"):
        hb.spiral_path("neural_3d", cam, P[:, :, :3], b)
    bad = P.copy()
    bad[3, 0, 0] = np.nan
    with pytest.raises(ValueError, match="finite"):
        hb.spiral_path("neural_3d", cam, bad, b, num_frames=4)
    with pytest.raises(ValueError, match="num_frames"):
        hb.spiral_path("neural_3d", cam, P, b, num_frames=5)
    with pytest.raises(ValueError, match="bounds"):
        hb.spiral_path("neural_3d", cam, P, None, num_frames=4)
    with pytest.raises(ValueError, match="supersample"):
        hb.spiral_path("neural_3d", cam, P, b, num_frames=4, supersample=0)


def test_render_video_refusals():
    case = build_case("technicolor_trained")
    model = hb.LightfieldModel(case.model_cfg, dataset=case.dataset)
    model.eval()
    cams = [hb.Camera(pose=np.eye(4)[:3], K=[[20.0, 0, 8], [0, 20.0, 6], [0, 0, 1]], width=16, height=12) for _ in range(3)]
    with pytest.raises(ValueError, match="no cameras"):
        hb.render_video(model, [], [])
    with pytest.raises(ValueError, match="3 cameras but 2 times"):
        hb.render_video(model, cams, [0.0, 1.0])
    with pytest.raises(ValueError, match="finite"):
        hb.render_video(model, cams, [0.0, float("inf"), 1.0])
    odd = cams[:2] + [hb.Camera(pose=np.eye(4)[:3], K=[[20.0, 0, 8], [0, 20.0, 6], [0, 0, 1]], width=16, height=13)]
    with pytest.raises(ValueError, match="camera 2 is 16 x 13"):
        hb.render_video(model, odd, [0.0, 0.5, 1.0])
    for out in (torch.zeros((3, 12, 16, 3), dtype=torch.float32), torch.zeros((3, 12, 16, 3), dtype=torch.uint8),
                torch.zeros((2, 12, 16, 3), dtype=torch.uint8)):
        with pytest.raises(ValueError, match="out must be"):
            hb.render_video(model, cams, [0.0, 0.5, 1.0], out=out)
    with pytest.raises(TypeError):
        hb.render_video(object(), cams, [0.0, 0.5, 1.0])
    model.train()
    with pytest.raises(RuntimeError, match="eval"):
        hb.render_video(model, cams, [0.0, 0.5, 1.0])
