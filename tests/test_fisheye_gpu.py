"""Fisheye cameras on the device: generate_rays against the reference goldens of ImmersiveDataset.get_coords, training
batches over views that mix fisheye and pinhole cameras, whole-frame rendering, and the C-ABI's refusal of non-finite
coefficients."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import hyperreel_b200 as hb
from hyperreel_b200 import lib as L
from tests.test_fisheye_oracle import FISHEYE, load_fisheye
from tests.test_shipped_yaml_golden import SHIPPED, load_fixture

pytestmark = pytest.mark.gpu


def _camera(g):
    return hb.Camera(pose=g["pose"], K=g["K"], width=int(g["W"]), height=int(g["H"]), time=float(g["time"]),
                     cam_idx=float(g["cam_idx"]), distortion=tuple(float(k) for k in g["distortion"]))


@pytest.mark.parametrize("name", list(FISHEYE))
def test_fisheye_rays_match_reference_golden(name):
    g = load_fisheye(name)
    rays = hb.generate_rays(_camera(g), c_in=8)
    assert rays.shape == (int(g["W"]) * int(g["H"]), 8)
    got = rays[torch.from_numpy(g["pixels"]).cuda()].cpu().numpy()
    want = g["rays"]
    # a wrong convergence decision moves a row by O(1): the bound pins the sentinel rows too
    assert np.abs(got - want).max() <= 4e-6 * max(1.0, np.abs(want).max())
    rays6 = hb.generate_rays(_camera(g), c_in=6)
    assert torch.equal(rays6, rays[:, :6])


def test_fisheye_pixel_subrange_equals_the_full_frame():
    cam = _camera(load_fisheye("strong_48x36"))
    full = hb.generate_rays(cam, c_in=8)
    for first, n in ((0, 1), (123, 777), (1700, 28)):
        assert torch.equal(hb.generate_rays(cam, c_in=8, first_pixel=first, n_pixels=n), full[first:first + n])


def _mixed_views():
    """Three 48x36 views: two fisheye cameras (one with sentinel corners) around a pinhole."""
    strong, mild = load_fisheye("strong_48x36"), load_fisheye("mild_40x30")
    W, H = 48, 36
    cams = [_camera(strong),
            hb.Camera(pose=mild["pose"], K=[[40.0, 0, 23.5], [0, 41.0, 18.0], [0, 0, 1]], width=W, height=H, time=0.5,
                      cam_idx=4.0),
            hb.Camera(pose=mild["pose"], K=[[30.0, 0, 24.3], [0, 30.0, 17.6], [0, 0, 1]], width=W, height=H, time=1.0,
                      cam_idx=9.0, distortion=(0.05, -0.01))]
    g = torch.Generator().manual_seed(0)
    images = torch.randint(0, 256, (3, H, W, 3), generator=g, dtype=torch.uint8)
    rows = torch.cat([hb.generate_rays(c, c_in=8) for c in cams])
    return cams, images, rows


def _check(out, rows, images):
    ids = out["pixel_ids"]
    assert torch.equal(out["coords"], rows[ids])
    want = images.reshape(-1, 3).numpy()[ids.cpu().numpy()].astype(np.float32) / np.float32(255.0)  # T.ToTensor()
    assert np.array_equal(out["rgb"].cpu().numpy(), want)


def test_mixed_fisheye_and_pinhole_batches_equal_generate_rays():
    cams, images, rows = _mixed_views()
    n = rows.shape[0]
    # every pixel, permuted (train_rows_kernel<WholePlan>)
    d = hb.DeviceRayBatches(cams, images, batch_size=1000, seed=3)
    seen = []
    for i in range(len(d)):
        out = d.batch(i, with_pixel_ids=True)
        _check(out, rows, images)
        seen.append(out["pixel_ids"])
    assert torch.equal(torch.cat(seen).sort().values.cpu(), torch.arange(n))
    ids = torch.randint(0, n, (4096,), generator=torch.Generator().manual_seed(1))
    out = d.gather(ids, with_pixel_ids=True)
    _check(out, rows, images)
    # per-view subsets, permuted and with replacement (train_rows_kernel<TablePlan>)
    plan = [(1, 0), (4, 1), (2, 1)]
    for kw in ({}, {"replacement": True, "num_iters": 5}):
        d = hb.DeviceRayBatches(cams, images, batch_size=700, seed=5, subsample=plan, **kw)
        for i in range(len(d)):
            _check(d.batch(i, with_pixel_ids=True), rows, images)
        t = torch.randint(0, d.n_rows, (3000,), generator=torch.Generator().manual_seed(2))
        _check(d.gather_rows(t, with_pixel_ids=True), rows, images)


def _immersive_render():
    by_name = {os.path.basename(p)[:-4]: p for p in SHIPPED}
    plain, cfg, ds, sig, sd, rays, rgb = load_fixture(by_name["immersive_z_plane"])
    model = hb.LightfieldModel(cfg, dataset=ds)
    render = hb.RenderLightfield(model, None, cfg.render, net_chunk=1 << 20)
    _, unexpected = render.load_state_dict(sd, strict=False)
    assert not unexpected
    render.eval()
    return render, rays


def test_fisheye_frame_render_matches_the_separate_steps():
    render, fixture_rays = _immersive_render()
    o = fixture_rays[0, :3].tolist()
    W, H = 96, 72
    cam = hb.Camera(pose=[[1, 0, 0, o[0]], [0, 1, 0, o[1]], [0, 0, 1, o[2]]], K=[[45.0, 0, 47.8], [0, 45.0, 36.2], [0, 0, 1]],
                    width=W, height=H, time=0.25, cam_idx=0.0, distortion=(-0.3, 0.04))
    c_in = int(fixture_rays.shape[1])
    img = render.model.render_frame_to8b(cam, chunk=2500)  # 3 chunks
    assert img.shape == (H, W, 3) and img.dtype == torch.uint8
    rays = hb.generate_rays(cam, c_in=c_in)
    sep = render.model.render_to8b(rays).cpu().reshape(H, W, 3)
    assert torch.equal(img, sep)
    assert int(img.max()) > int(img.min())
    pinhole = render.model.render_frame_to8b(hb.Camera(pose=cam.pose, K=cam.K, width=W, height=H, time=0.25), chunk=2500)
    assert not torch.equal(img, pinhole)


@pytest.mark.parametrize("bad", [(float("nan"), 0.0), (0.0, float("inf"))])
def test_non_finite_coefficients_are_refused_and_nothing_is_written(bad):
    lib = L.load_library()
    cam = hb.Camera(pose=[[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0]], K=[[20, 0, 8], [0, 20, 6], [0, 0, 1]], width=16,
                    height=12).to_c()
    cam.fisheye, cam.k1, cam.k2 = 1, bad[0], bad[1]
    out = torch.full((16 * 12, 8), 7.0, device="cuda")
    assert lib.hr_generate_rays(C.byref(cam), 8, 0, 16 * 12, out.data_ptr(), torch.cuda.current_stream().cuda_stream) != 0
    assert b"fisheye" in lib.hr_last_error()
    torch.cuda.synchronize()
    assert bool((out == 7.0).all())
    render, _ = _immersive_render()
    host = torch.full((12, 16, 3), 7, dtype=torch.uint8).pin_memory()
    render.model.render_frame_to8b(hb.Camera(pose=[[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0]], K=[[20, 0, 8], [0, 20, 6], [0, 0, 1]],
                                             width=16, height=12), out_host=host.clone().pin_memory())  # uploads the model
    assert render.model._lib.hr_render_frame_to8b_host(render.model._handle, C.byref(cam), host.data_ptr(), 0) != 0
    assert b"fisheye" in lib.hr_last_error()
    assert bool((host == 7).all())
