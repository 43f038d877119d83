"""dataset_cameras' views on the device: their rays against the reference's get_coords rays (tests/golden/
dataset_cameras.npz), and training and held-out scoring end to end from a synthetic Technicolor and DoNeRF scene."""
import numpy as np
import pytest
import torch

import hyperreel_b200 as hb
from hyperreel_b200.state import seeded_state_dict
from tests.cases import build_case
from tests.test_dataset_cameras import REFUSED, SPLITS, _cases, _golden, make_scene

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("split", SPLITS)
@pytest.mark.parametrize("case", _cases())
def test_device_rays_equal_the_reference_get_coords(case, split, tmp_path):
    z = _golden()
    root, cfg = make_scene(z, case, tmp_path)
    if (case, split) in REFUSED:
        pytest.skip("refused: the reference's NDC focal differs from the view's")
    views = hb.dataset_cameras(cfg, root, split)
    want = z[f"{case}/{split}/rays"]
    for k, i in enumerate(z[f"{case}/{split}/ray_views"]):
        got = hb.generate_rays(views.cameras[int(i)], c_in=want.shape[-1]).cpu().numpy()
        assert got.shape == want[k].shape
        # the standard of test_rays_gpu.py and test_fisheye_gpu.py against the reference's rays
        assert np.abs(got - want[k]).max() <= 4e-6 * max(1.0, np.abs(want[k]).max()), (case, split, int(i))


def _system(model_case, dataset_cfg, root):
    case = build_case(model_case, n=8)
    cfg = hb.to_cfg({"model": case.model_cfg,
                     "training": {"batch_size": 256, "ray_chunk": 700, "iters_per_epoch": 4000,
                                  "optimizers": {"color": {"lr": 0.002}, "color_impl": {"lr": 0.001},
                                                 "embedding_impl": {"lr": 0.0002}}},
                     "dataset": dataset_cfg})
    system = hb.INRSystem.from_dataset(cfg, root)
    system.load_state_dict(seeded_state_dict(system.render_fn.model.sig, seed=3, density_gain=30.0))
    return cfg, system.cuda()


def _frames(n, H, W, ch, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randint(0, 256, (n, H, W, ch), generator=g, device="cuda", dtype=torch.int16).to(torch.uint8)


@pytest.mark.parametrize("case,model_case", [("technicolor_lightfield", "technicolor_trained"),
                                             ("donerf_center", "donerf_app")])
def test_train_and_score_a_scene_directory(case, model_case, tmp_path):
    z = _golden()
    root, dcfg = make_scene(z, case, tmp_path)
    dcfg = dict(dcfg, img_wh=[16, 12])  # scored views hold the 11 x 11 SSIM window
    W, H = dcfg["img_wh"]
    rgba = dcfg["name"] == "donerf"
    ch = 4 if rgba else 3
    cfg, system = _system(model_case, dcfg, root)
    assert system.render_fn.model.sig.dataset["near"] == hb.dataset_cameras(dcfg, root, "train").facts["near"]
    c_in = system.render_fn.model.sig.c_in

    train = hb.dataset_cameras(dcfg, root, "train")
    batches = hb.DeviceRayBatches.from_config(cfg, train.cameras, _frames(len(train.cameras), H, W, ch, 1), c_in=c_in)
    assert batches.rgba == rgba and batches.n_rows == len(train.cameras) * H * W
    torch.manual_seed(0)
    losses = [float(system.training_step(batches.batch(i % len(batches)))["train/loss"]) for i in range(5)]
    assert all(np.isfinite(losses)), losses

    val = hb.dataset_cameras(dcfg, root, "val")
    images = _frames(len(val.cameras), H, W, ch, 2)
    got = system.validation_views(val, images)
    assert len(got) == len(val.cameras) == len(val.frames)
    gt = images.cpu().float() / 255  # T.ToTensor() and the composite over white, on the CPU as get_rgb computes them
    if rgba:
        gt = gt[..., :3] * gt[..., 3:] + (1 - gt[..., 3:])
    gt = gt.cuda()
    for c, g, t in zip(val.cameras, got, gt):
        want = system.validation_image({"coords": hb.generate_rays(c, c_in=c_in).view(H, W, -1), "rgb": t, "W": W, "H": H})
        assert torch.equal(g["val/psnr"], want["val/psnr"]) and torch.equal(g["val/ssim"], want["val/ssim"])
        assert abs(float(g["val/loss"]) - float(want["val/loss"])) <= 1e-6 * float(want["val/loss"])


def test_render_video_of_the_render_split(tmp_path):
    z = _golden()
    root, dcfg = make_scene(z, "neural_3d_ndc", tmp_path)
    dcfg = dict(dcfg, keyframe_step=1)  # the keyframe planes need two keyframes
    W, H = dcfg["img_wh"]
    _, system = _system("neural3d_trained", dcfg, root)
    views = hb.dataset_cameras(dcfg, root, "render")
    video = system.render_video(views)
    full = system.render_video(views.cameras)
    y0, y1, x0, x1 = views.crop
    assert full.shape == (len(views.cameras), H, W, 3)
    assert torch.equal(video, full[:, y0:y1, x0:x1])
