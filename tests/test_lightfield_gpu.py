"""Two-plane light-field views (the Stanford dataset) on the device: generate_rays against the reference's rays, training
batches over views that mix two-plane, pinhole and fisheye cameras, whole-frame and video rendering with the shipped
stanford_z_plane model, training steps fed from those batches, and the C ABI's refusals of malformed two-plane records."""
import ctypes as C
import dataclasses
import os

import numpy as np
import pytest
import torch

import hyperreel_b200 as hb
from hyperreel_b200 import lib as L
from oracle.rays_oracle import to8b
from tests.test_fisheye_oracle import load_fisheye
from tests.test_lightfield import RAY_CASES, RAYS, cameras_of
from tests.test_shipped_yaml_golden import SHIPPED, load_fixture

pytestmark = pytest.mark.gpu


def _case_camera(name, **kw):
    W, H, s, t, st, uv, near, far, aspect = RAYS[f"{name}/params"]
    return hb.TwoPlaneCamera(int(W), int(H), s, t, st_scale=st, uv_scale=uv, near=near, far=far, aspect=aspect, **kw)


@pytest.mark.parametrize("name", RAY_CASES)
def test_rays_equal_reference_golden(name):
    cam = _case_camera(name, time=0.75, cam_idx=5)
    pixels = torch.from_numpy(RAYS[f"{name}/pixels"]).cuda()
    want = torch.from_numpy(RAYS[f"{name}/rays"]).cuda()
    rays8 = hb.generate_rays(cam, c_in=8)
    assert rays8.shape == (cam.width * cam.height, 8)
    assert torch.equal(rays8[pixels, :6], want)
    assert bool((rays8[:, 6] == 5).all()) and bool((rays8[:, 7] == 0.75).all())
    rays6 = hb.generate_rays(cam, c_in=6)
    assert torch.equal(rays6, rays8[:, :6])


def test_pixel_subranges_equal_the_full_view():
    cam = _case_camera("odd_37x23")
    full = hb.generate_rays(cam, c_in=8)
    for first, n in ((0, 1), (36, 2), (100, 555), (850, 1)):
        assert torch.equal(hb.generate_rays(cam, c_in=8, first_pixel=first, n_pixels=n), full[first:first + n])


def test_split_views_equal_reference_golden():
    from tests.test_lightfield import VIEWS

    for name in ("render_spiral", "val_files", "test_files_tarot"):
        want = torch.from_numpy(VIEWS[f"{name}/rays"]).cuda()
        for i, cam in enumerate(cameras_of(name)):
            assert torch.equal(hb.generate_rays(cam, c_in=6), want[i]), (name, i)


W, H = 40, 30


def _mixed_views():
    """Five 40x30 views: two-plane views around a pinhole and a fisheye camera."""
    mild = load_fisheye("mild_40x30")
    cams = [hb.TwoPlaneCamera(W, H, -0.5, 0.25, st_scale=0.25, time=0.0, cam_idx=1.0),
            hb.Camera(pose=mild["pose"], K=[[35.0, 0, 19.5], [0, 36.0, 15.0], [0, 0, 1]], width=W, height=H, time=0.5,
                      cam_idx=4.0),
            hb.TwoPlaneCamera(W, H, 0.75, -1.0, st_scale=0.125, uv_scale=0.9, near=-1.5, far=0.25, aspect=1.5, time=1.0),
            hb.Camera(pose=mild["pose"], K=mild["K"], width=W, height=H, time=0.25, cam_idx=3.0,
                      distortion=tuple(float(k) for k in mild["distortion"])),
            hb.TwoPlaneCamera(W, H, 1.0 / 3.0, 0.1, st_scale=0.25, time=0.5, cam_idx=2.0)]
    g = torch.Generator().manual_seed(0)
    images = torch.randint(0, 256, (len(cams), H, W, 3), generator=g, dtype=torch.uint8)
    rows = torch.cat([hb.generate_rays(c, c_in=8) for c in cams])
    return cams, images, rows


def _check(out, rows, images):
    ids = out["pixel_ids"]
    assert torch.equal(out["coords"], rows[ids])
    want = images.reshape(-1, 3).numpy()[ids.cpu().numpy()].astype(np.float32) / np.float32(255.0)
    assert np.array_equal(out["rgb"].cpu().numpy(), want)


def test_mixed_model_batches_equal_generate_rays():
    cams, images, rows = _mixed_views()
    n = rows.shape[0]
    d = hb.DeviceRayBatches(cams, images, batch_size=1100, seed=3)  # train_rows_kernel<WholePlan>
    seen = []
    for i in range(len(d)):
        out = d.batch(i, with_pixel_ids=True)
        _check(out, rows, images)
        seen.append(out["pixel_ids"])
    assert torch.equal(torch.cat(seen).sort().values.cpu(), torch.arange(n))
    _check(d.gather(torch.randint(0, n, (4096,), generator=torch.Generator().manual_seed(1)), with_pixel_ids=True),
           rows, images)
    plan = [(1, 0), (3, 1), (2, 1), (1, 0), (5, 4)]  # train_rows_kernel<TablePlan>
    for kw in ({}, {"replacement": True, "num_iters": 5}):
        d = hb.DeviceRayBatches(cams, images, batch_size=700, seed=5, subsample=plan, **kw)
        for i in range(len(d)):
            _check(d.batch(i, with_pixel_ids=True), rows, images)
        t = torch.randint(0, d.n_rows, (3000,), generator=torch.Generator().manual_seed(2))
        _check(d.gather_rows(t, with_pixel_ids=True), rows, images)
    # training views of a Stanford config, from_config as it is
    cfg = hb.to_cfg({"training": {"batch_size": 512}, "dataset": {"name": "stanford"}})
    views = hb.lightfield_cameras({"name": "stanford", "img_wh": [W, H], "val_num": 8, "render_params": {"supersample": 4},
                                   "lightfield": {"rows": 5, "cols": 5, "step": 4, "supersample": 2, "disp_row": 2,
                                                  "st_scale": 0.25}}, W, H, "train")
    imgs = torch.randint(0, 256, (len(views), H, W, 3), generator=torch.Generator().manual_seed(4), dtype=torch.uint8)
    vrows = torch.cat([hb.generate_rays(c, c_in=6) for c in views])
    d = hb.DeviceRayBatches.from_config(cfg, views, imgs, c_in=6, seed=1)
    for i in range(len(d)):
        _check(d.batch(i, with_pixel_ids=True), vrows, imgs)


def _stanford(mode="bf16x3"):
    by_name = {os.path.basename(p)[:-4]: p for p in SHIPPED}
    plain, cfg, ds, sig, sd, rays, rgb = load_fixture(by_name["stanford_z_plane"])
    model = hb.LightfieldModel(cfg, dataset=ds, mlp_mode=mode)
    render = hb.RenderLightfield(model, None, cfg.render, net_chunk=1 << 20)
    _, unexpected = render.load_state_dict(sd, strict=False)
    assert not unexpected
    render.eval()
    return render, plain, ds, sd, rays, rgb


@pytest.mark.parametrize("mode", ["bf16x3", "fp32"])
def test_frame_render_equals_to8b_of_the_float_render(mode):
    render, _, _, _, rays, rgb = _stanford(mode)
    c_in = int(rays.shape[1])
    assert c_in == 6
    # the fixture's own rays still render as the reference rendered them
    assert float((render(rays.cuda())["rgb"].cpu() - rgb).abs().max()) <= 1e-4
    cam = hb.TwoPlaneCamera(96, 64, 0.3, -0.2, st_scale=0.25, aspect=1.5)
    img = render.model.render_frame_to8b(cam, chunk=2500)  # three chunks
    assert img.shape == (64, 96, 3) and img.dtype == torch.uint8
    rays = hb.generate_rays(cam, c_in=c_in)
    with torch.no_grad():
        f = render(rays)["rgb"].cpu().numpy()
    assert np.array_equal(img.reshape(-1, 3).numpy(), to8b(f))
    assert int(img.max()) > int(img.min())
    other = render.model.render_frame_to8b(dataclasses.replace(cam, s=-0.3))
    assert not torch.equal(img, other)


def test_video_of_the_render_path_equals_the_frames():
    render, plain, ds, sd, _, _ = _stanford()
    model = render.model
    model.set_sub_batch(1000)  # sub-batches across frame boundaries
    cfg = {"name": "stanford", "img_wh": [24, 16], "val_num": 8,
           "render_params": {"spiral": True, "spiral_rad": 0.5, "supersample": 4},
           "lightfield": {"rows": 17, "cols": 17, "step": 4, "supersample": 2, "disp_row": 8, "st_scale": 0.25}}
    cams = hb.lightfield_cameras(cfg, 24, 16, "render")
    assert len(cams) == 120
    video = hb.render_video(model, cams)
    assert video.shape == (120, 16, 24, 3)
    for f in range(0, 120, 7):
        assert torch.equal(video[f].cpu(), model.render_frame_to8b(cams[f])), f
    # a video that mixes the three camera models, and the system wrapper
    mild = load_fisheye("mild_40x30")
    o = [0.0, 0.0, -1.0]
    pose = [[1, 0, 0, o[0]], [0, -1, 0, o[1]], [0, 0, -1, o[2]]]
    mixed = [cams[0],
             hb.Camera(pose=pose, K=[[20.0, 0, 11.5], [0, 20.0, 7.5], [0, 0, 1]], width=24, height=16),
             hb.Camera(pose=pose, K=[[15.0, 0, 12.0], [0, 15.0, 8.0], [0, 0, 1]], width=24, height=16,
                       distortion=tuple(float(k) for k in mild["distortion"])),
             cams[60]]
    got = hb.render_video(model, mixed)
    for f, c in enumerate(mixed):
        assert torch.equal(got[f].cpu(), model.render_frame_to8b(c)), f
    assert torch.equal(got[3], video[60])
    system = hb.INRSystem(hb.to_cfg({"model": plain}), dataset=ds)
    system.load_state_dict(sd)
    assert torch.equal(system.render_video(mixed), got)


def test_training_from_device_batches_lowers_the_loss():
    by_name = {os.path.basename(p)[:-4]: p for p in SHIPPED}
    plain, cfg, ds, sig, sd, rays, rgb = load_fixture(by_name["stanford_z_plane"])
    dataset = {"name": "stanford", "img_wh": [32, 24], "val_num": 8, "render_params": {"supersample": 4},
               "lightfield": {"rows": 5, "cols": 5, "step": 2, "supersample": 2, "disp_row": 2, "st_scale": 0.25}}
    views = hb.lightfield_cameras(dataset, 32, 24, "train")
    # a smooth target: colour a function of the ray, so that the net can move towards it
    target = []
    for c in views:
        r = hb.generate_rays(c, c_in=6)
        target.append(((torch.stack([r[:, 3], r[:, 4], r[:, 0] + r[:, 1]], -1) * 0.5 + 0.5).clamp(0, 1) * 255).to(torch.uint8))
    images = torch.stack(target).reshape(len(views), 24, 32, 3).cpu()
    n = len(views) * 24 * 32
    tcfg = hb.to_cfg({"model": plain, "training": {"ray_chunk": 1 << 20, "iters_per_epoch": 4000, "batch_size": n},
                      "dataset": ds})
    batches = hb.DeviceRayBatches.from_config(hb.to_cfg({"training": {"batch_size": n}, "dataset": dataset}), views, images,
                                              c_in=6, seed=2)
    assert len(batches) == 1
    torch.manual_seed(0)
    system = hb.INRSystem(tcfg, dataset=ds)
    system.load_state_dict(sd)
    system.cuda()
    losses = []
    for i in range(8):
        batches.set_epoch(i)
        losses.append(float(system.training_step(batches.batch(0))["train/loss"]))
    print("stanford_z_plane losses:", losses)
    assert all(np.isfinite(losses))
    assert losses[-1] < losses[0]


def _bad_records():
    good = hb.TwoPlaneCamera(16, 12, 0.1, 0.2, st_scale=0.25).to_c()
    out = []
    for field, value, msg in (("fisheye", 1, b"fisheye"), ("lf_s", float("nan"), b"not finite"),
                              ("lf_t", float("inf"), b"not finite"), ("lf_st_scale", float("nan"), b"not finite"),
                              ("lf_uv_scale", float("-inf"), b"not finite"), ("lf_near", float("nan"), b"not finite"),
                              ("lf_far", float("inf"), b"not finite"), ("lf_aspect", float("nan"), b"not finite"),
                              ("lf_aspect", 0.0, b"lf_aspect")):
        rec = L.hr_camera.from_buffer_copy(good)
        setattr(rec, field, value)
        if field == "fisheye":
            rec.k1, rec.k2 = 0.1, 0.01
        out.append((rec, msg))
    return good, out


def test_malformed_records_are_refused_and_nothing_is_written():
    lib = L.load_library()
    good, bad = _bad_records()
    stream = torch.cuda.current_stream().cuda_stream
    rays = torch.full((16 * 12, 8), 7.0, device="cuda")
    render, _, _, _, _, _ = _stanford()
    model = render.model
    model.render_frame_to8b(hb.TwoPlaneCamera(16, 12, 0.1, 0.2))  # uploads the model
    host = torch.full((12, 16, 3), 7, dtype=torch.uint8).pin_memory()
    need = int(lib.hr_video_workspace_bytes(model._handle, 2, 12, 16))
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    video = torch.full((2, 12, 16, 3), 7, dtype=torch.uint8, device="cuda")
    for rec, msg in bad:
        assert lib.hr_generate_rays(C.byref(rec), 8, 0, 16 * 12, rays.data_ptr(), stream) != 0
        assert msg in lib.hr_last_error(), lib.hr_last_error()
        assert model._lib.hr_render_frame_to8b_host(model._handle, C.byref(rec), host.data_ptr(), 0) != 0
        assert msg in lib.hr_last_error(), lib.hr_last_error()
        recs = (L.hr_camera * 2)(good, rec)
        tt = (C.c_float * 2)(0.0, 0.0)
        assert lib.hr_render_video_to8b(model._handle, recs, tt, 2, video.data_ptr(), ws.data_ptr(), need, stream) != 0
        assert msg in lib.hr_last_error() and b"frame 1" in lib.hr_last_error(), lib.hr_last_error()
    torch.cuda.synchronize()
    assert bool((rays == 7.0).all()) and bool((host == 7).all()) and bool((video == 7).all())
    # the good record draws
    assert lib.hr_generate_rays(C.byref(good), 8, 0, 16 * 12, rays.data_ptr(), stream) == 0
    torch.cuda.synchronize()
    assert torch.equal(rays, hb.generate_rays(hb.TwoPlaneCamera(16, 12, 0.1, 0.2, st_scale=0.25), c_in=8))
