"""hr_image_metrics / hyperreel_b200.metrics / INRSystem.validation_image against the CPU restatement of the reference's
validation metrics (tests/metrics_oracle.py)."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import hyperreel_b200 as hb
from hyperreel_b200 import lib as L
from hyperreel_b200 import metrics as M
from oracle.hyperreel_oracle import HyperReelOracle
from tests import metrics_oracle as O
from tests.cases import build_case
from tests.metrics_oracle import smooth_noisy_pair

pytestmark = pytest.mark.gpu


def noisy_pair(h, w, seed, lo=0.0, hi=1.0):
    rng = np.random.default_rng(seed)
    a = rng.uniform(lo, hi, (h, w, 3)).astype(np.float32)
    b = rng.uniform(lo, hi, (h, w, 3)).astype(np.float32)
    return a, b


def constant_pair(h, w):
    return np.full((h, w, 3), 0.25, np.float32), np.full((h, w, 3), 0.75, np.float32)


PAIRS = {
    "11x11_noisy": lambda: noisy_pair(11, 11, 1),
    "11x40_smooth": lambda: smooth_noisy_pair(11, 40, 2),
    "37x53_noisy": lambda: noisy_pair(37, 53, 3),
    "37x53_smooth": lambda: smooth_noisy_pair(37, 53, 4),
    "40x11_noisy": lambda: noisy_pair(40, 11, 5),
    "outside_unit_range": lambda: noisy_pair(45, 70, 6, lo=-1.5, hi=2.5),
    "constant": lambda: constant_pair(29, 35),
    "1088x2048_smooth": lambda: smooth_noisy_pair(1088, 2048, 7),
}


def check_against_oracle(pred, gt, mse, ssim, psnr):
    """The fp64 oracle is the pin.  The float32 map (scikit-image >= 0.19) carries rounding of order 1e-5 per pixel, which a
    full frame averages away (6e-9 at 1088 x 2048) but a tiny one does not: the 11 x 40 smooth pair averages 90 values and
    its float32 SSIM lies 1.2e-6 from the fp64 one, hence 2e-6 against that mode."""
    ref_ssim = O.ssim(pred, gt, fp64=True)
    ref_mse = O.mse(pred, gt)
    assert abs(ssim - ref_ssim) <= 1e-10, (ssim, ref_ssim)
    assert abs(mse - ref_mse) <= 1e-12 * ref_mse, (mse, ref_mse)
    assert abs(psnr - O.psnr(pred, gt)) <= 1e-9, (psnr, O.psnr(pred, gt))
    assert abs(ssim - O.ssim(pred, gt, fp64=False)) <= 2e-6


@pytest.mark.parametrize("name", list(PAIRS))
def test_kernel_matches_fp64_oracle(name):
    pred, gt = PAIRS[name]()
    p, g = torch.from_numpy(pred).cuda(), torch.from_numpy(gt).cuda()
    mse, ssim = M.image_metrics(p, g)
    assert mse.dtype == ssim.dtype == torch.float64 and mse.shape == ssim.shape == (1,)
    psnr = M.psnr(p, g)
    assert psnr.shape == () and psnr.is_cuda
    assert float(M.ssim(p, g)) == float(ssim[0])
    check_against_oracle(pred, gt, float(mse[0]), float(ssim[0]), float(psnr))


def test_batch_matches_oracle_and_single_calls_bitwise():
    pairs = [noisy_pair(64, 96, 10), smooth_noisy_pair(64, 96, 11), noisy_pair(64, 96, 12, lo=-0.5, hi=1.5),
             constant_pair(64, 96)]
    p = torch.from_numpy(np.stack([a for a, _ in pairs])).cuda()
    g = torch.from_numpy(np.stack([b for _, b in pairs])).cuda()
    mse, ssim = M.image_metrics(p, g)
    psnr = M.psnr(p, g)
    assert mse.shape == ssim.shape == psnr.shape == (4,)
    for i, (a, b) in enumerate(pairs):
        check_against_oracle(a, b, float(mse[i]), float(ssim[i]), float(psnr[i]))
        m1, s1 = M.image_metrics(p[i], g[i])
        assert torch.equal(m1[0], mse[i]) and torch.equal(s1[0], ssim[i])
    m2, s2 = M.image_metrics(p, g)
    assert torch.equal(m2, mse) and torch.equal(s2, ssim)


def test_full_frame_is_bitwise_reproducible():
    pred, gt = smooth_noisy_pair(1088, 2048, 8)
    p, g = torch.from_numpy(pred).cuda(), torch.from_numpy(gt).cuda()
    a = torch.stack(M.image_metrics(p, g))
    b = torch.stack(M.image_metrics(p, g))
    assert torch.equal(a, b)


def test_identical_images_score_one_and_infinite_psnr():
    pred, _ = smooth_noisy_pair(50, 61, 9)
    p = torch.from_numpy(pred).cuda()
    assert float(M.ssim(p, p.clone())) == 1.0
    assert float(M.psnr(p, p.clone())) == math.inf
    assert float(M.image_metrics(p, p)[0][0]) == 0.0


def make_system(case):
    cfg = hb.to_cfg({"model": case.model_cfg_plain, "training": {"ray_chunk": 1 << 20}})
    system = hb.INRSystem(cfg, dataset=case.dataset)
    system.load_state_dict(case.state_dict)
    return system.cuda()


def test_validation_image_on_a_rendered_view():
    H, W = 24, 32
    case = build_case("technicolor_trained", n=H * W)
    ref = HyperReelOracle(case.model_cfg_plain, case.dataset, case.state_dict).render(case.rays.clone())
    system = make_system(case)
    system.train()
    outs, per_view = [], []
    for view in range(3):
        gen = torch.Generator().manual_seed(40 + view)
        gt = (ref + 0.05 * (view + 1) * torch.randn(ref.shape, generator=gen)).float()
        batch = {"coords": case.rays.cuda().view(H, W, -1), "rgb": gt.cuda().view(H, W, 3), "W": W, "H": H}
        out = system.validation_image(batch, view)
        assert system.training  # the mode it was called in
        assert set(out) == {"val/loss", "val/psnr", "val/ssim"}
        assert out["val/loss"].dtype == torch.float32
        assert out["val/psnr"].dtype == out["val/ssim"].dtype == torch.float64
        for v in out.values():
            assert v.shape == () and v.is_cuda and not v.requires_grad and v.grad_fn is None
        system.eval()
        with torch.no_grad():
            rgb = system(case.rays.cuda())["rgb"]
        system.train()
        assert float((rgb.cpu() - ref).abs().max()) <= 1e-4
        img, img_gt = rgb.cpu().numpy().reshape(H, W, 3), gt.numpy().reshape(H, W, 3)
        assert abs(float(out["val/psnr"]) - O.psnr(img, img_gt)) <= 1e-10
        assert abs(float(out["val/ssim"]) - O.ssim(img, img_gt)) <= 1e-10
        assert torch.equal(out["val/loss"], torch.mean((rgb - gt.cuda()) ** 2))
        outs.append(out)
        per_view.append({k: v.cpu().numpy() for k, v in out.items()})
    mean = system.validation_epoch_end(outs)
    for k in ("val/loss", "val/psnr", "val/ssim"):
        assert isinstance(mean[k], float)
        assert mean[k] == float(np.mean(np.stack([v[k] for v in per_view])))
    system.eval()
    system.validation_image({"coords": case.rays.cuda(), "rgb": ref.cuda(), "W": W, "H": H})
    assert not system.training


def test_c_abi_refusals_leave_the_output_untouched():
    lib = L.load_library()
    p = torch.rand((2, 16, 16, 3), device="cuda")
    need = lib.hr_image_metrics_workspace_bytes(2, 16, 16)
    assert need > 0
    ws = torch.empty((need,), dtype=torch.uint8, device="cuda")
    out = torch.full((2, 2), -7.0, dtype=torch.float64, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    calls = [
        (2, 10, 16, need, "height and width"),
        (2, 16, 10, need, "height and width"),
        (0, 16, 16, need, "n_images"),
        (2, 16, 16, need - 1, "workspace"),
    ]
    for n, h, w, nbytes, msg in calls:
        rc = lib.hr_image_metrics(p.data_ptr(), p.data_ptr(), n, h, w, out.data_ptr(), ws.data_ptr(), nbytes, stream)
        assert rc != 0
        assert msg in lib.hr_last_error().decode()
    assert lib.hr_image_metrics(None, p.data_ptr(), 2, 16, 16, out.data_ptr(), ws.data_ptr(), need, stream) != 0
    assert "null" in lib.hr_last_error().decode()
    assert lib.hr_image_metrics_workspace_bytes(2, 10, 16) == -1
    torch.cuda.synchronize()
    assert bool((out == -7.0).all())
    assert lib.hr_image_metrics(p.data_ptr(), p.data_ptr(), 2, 16, 16, out.data_ptr(), ws.data_ptr(), need, stream) == 0
    torch.cuda.synchronize()
    assert out[:, 0].tolist() == [0.0, 0.0] and out[:, 1].tolist() == [1.0, 1.0]
