"""Held-out splits scored on the device (hr_score_views): every view's (mse, ssim) is bit for bit what the per-view path
gives -- generate_rays, the model's eval forward, image_metrics against u8 / 255 -- for static and dynamic models,
both sample-net modes, sub-batches that split a frame, hold several frames or the whole split, a split that alternates
pinhole, fisheye and two-plane views, one view, and frame sizes whose metrics tiles do not divide the image.
INRSystem.validation_views against validation_image, repeated calls, a side stream with caller-owned output, and the C
ABI's refusals, which leave the output untouched."""
import ctypes as C
import dataclasses
import os

import numpy as np
import pytest
import torch

import hyperreel_b200 as hb
from hyperreel_b200 import lib as L
from hyperreel_b200.metrics import image_metrics
from tests.cases import build_case
from tests.test_fisheye_oracle import load_fisheye
from tests.test_shipped_yaml_golden import SHIPPED, load_fixture
from tests.test_video_gpu import FACING, _pose

pytestmark = pytest.mark.gpu

W, H = 48, 30  # 1440 pixels per view; neither side a multiple of the 32 x 16 metrics tile


def _render(name, mode="bf16x3"):
    case = build_case(name)
    model = hb.LightfieldModel(case.model_cfg, dataset=case.dataset, mlp_mode=mode)
    render = hb.RenderLightfield(model, None, case.model_cfg.render)
    render.load_state_dict(case.state_dict, strict=False)
    render.eval()
    return render


def _cameras(n, w=W, h=H):
    return [hb.Camera(pose=_pose(FACING[0], FACING[1], 0.03 * f, -0.05 * f),
                      K=[[40.0 * w / W, 0, 0.49 * w], [0, 40.0 * w / W, 0.51 * h], [0, 0, 1]], width=w, height=h,
                      time=f / max(n - 1, 1), cam_idx=0.0) for f in range(n)]


def to_float(u8):
    """u8 / 255 correctly rounded in fp32: the reference's ground truth (T.ToTensor(), a CPU division).  On CUDA, torch divides
    by a Python scalar as a multiply by its reciprocal, one ulp off for some values, so the divisor is a device tensor."""
    return u8.float() / torch.tensor(255.0, device=u8.device)


def test_the_conversion_is_the_correctly_rounded_quotient():
    u8 = torch.arange(256, dtype=torch.uint8)
    want = u8.float() / 255  # the CPU divides
    assert np.array_equal(want.numpy(), np.arange(256, dtype=np.float32) / np.float32(255))
    assert torch.equal(to_float(u8.cuda()).cpu(), want)


def _ground_truth(model, cams, times, seed):
    """The views' own uint8 renders with noise on top: close to the prediction, as a held-out split is."""
    video = hb.render_video(model, cams, times)
    g = torch.Generator(device="cuda").manual_seed(seed)
    noise = torch.randint(-12, 13, video.shape, generator=g, device="cuda", dtype=torch.int16)
    return (video.to(torch.int16) + noise).clamp(0, 255).to(torch.uint8).contiguous()


def _per_view(model, cams, times, images):
    """The existing path, one view at a time: rays, eval forward, image_metrics against the fp32 conversion."""
    mse, ssim = [], []
    for c, t, img in zip(cams, times, images):
        cam = dataclasses.replace(c, time=float(np.float32(t)))
        rays = hb.generate_rays(cam, c_in=model.sig.c_in)
        with torch.no_grad():
            pred = model(rays)["rgb"]
        m, s = image_metrics(pred.reshape(cam.height, cam.width, 3), to_float(img))
        mse.append(m)
        ssim.append(s)
    return torch.cat(mse), torch.cat(ssim)


def _assert_bitwise(got, want):
    for g, w in zip(got, want):
        assert g.dtype == torch.float64 and g.is_cuda
        assert torch.equal(g, w), (g, w)


@pytest.mark.parametrize("mode", ["bf16x3", "fp32"])
@pytest.mark.parametrize("name", ["technicolor_trained", "donerf_s16"])  # dynamic (c_in 8), static (c_in 6)
@pytest.mark.parametrize("sub", [1000, 2880, 0])  # splits a view; two views per sub-batch; the default (the whole split)
def test_views_equal_the_per_view_path(name, mode, sub):
    model = _render(name, mode).model
    model.set_sub_batch(sub)
    F = 5
    cams = _cameras(F)
    times = np.linspace(0.1, 0.9, F)  # not the cameras' own times: the call's times are the ones rendered
    images = _ground_truth(model, cams, times, seed=F)
    got = hb.score_views(model, cams, images, times)
    assert got[0].shape == got[1].shape == (F,)
    _assert_bitwise(got, _per_view(model, cams, times, images))
    assert bool((got[0] > 0).all()) and bool((got[1] < 1).all())
    again = hb.score_views(model, cams, images, times)
    assert torch.equal(torch.stack(again), torch.stack(got))


@pytest.mark.parametrize("size", [(11, 11), (37, 23), (70, 45)])
@pytest.mark.parametrize("sub", [500, 0])
def test_sizes_and_ring_wraps(size, sub):
    """Sub-batches of 500 rays over 7 views: the ring of whole frames wraps several times, frames straddle sub-batches."""
    model = _render("technicolor_trained").model
    model.set_sub_batch(sub)
    w, h = size
    cams = _cameras(7, w, h)
    times = [c.time for c in cams]
    images = _ground_truth(model, cams, times, seed=w)
    _assert_bitwise(hb.score_views(model, cams, images), _per_view(model, cams, times, images))


def test_one_view():
    model = _render("technicolor_trained").model
    cams = _cameras(1)
    images = _ground_truth(model, cams, [0.0], seed=1)
    _assert_bitwise(hb.score_views(model, cams, images), _per_view(model, cams, [0.0], images))


def test_split_alternating_pinhole_fisheye_and_two_plane_views():
    by_name = {os.path.basename(p)[:-4]: p for p in SHIPPED}
    plain, cfg, ds, sig, sd, rays, rgb = load_fixture(by_name["stanford_z_plane"])
    model = hb.LightfieldModel(cfg, dataset=ds)
    render = hb.RenderLightfield(model, None, cfg.render, net_chunk=1 << 20)
    render.load_state_dict(sd, strict=False)
    render.eval()
    w, h = 40, 30
    mild = load_fisheye("mild_40x30")
    pin = hb.Camera(pose=mild["pose"], K=[[35.0, 0, 19.5], [0, 36.0, 15.0], [0, 0, 1]], width=w, height=h, time=0.5)
    fish = hb.Camera(pose=mild["pose"], K=mild["K"], width=w, height=h, time=0.25,
                     distortion=tuple(float(k) for k in mild["distortion"]))
    cams = [pin, fish, hb.TwoPlaneCamera(w, h, -0.5, 0.25, st_scale=0.25),
            dataclasses.replace(pin, time=0.0), dataclasses.replace(fish, time=1.0),
            hb.TwoPlaneCamera(w, h, 0.75, -1.0, st_scale=0.125, uv_scale=0.9, near=-1.5, far=0.25, aspect=1.5)]
    times = [c.time for c in cams]
    for sub in (700, 0):
        model.set_sub_batch(sub)
        images = _ground_truth(model, cams, times, seed=sub)
        _assert_bitwise(hb.score_views(render, cams, images), _per_view(model, cams, times, images))


def _system():
    case = build_case("technicolor_trained")
    cfg = hb.to_cfg({"model": case.model_cfg_plain, "training": {"ray_chunk": 1 << 20}})
    system = hb.INRSystem(cfg, dataset=case.dataset)
    system.load_state_dict(case.state_dict)
    return system.cuda()


def test_validation_views_equal_validation_image():
    system = _system()
    model = system.render_fn.model
    model.set_sub_batch(1000)
    cams = _cameras(4)
    times = [c.time for c in cams]
    images = _ground_truth(model, cams, times, seed=7)
    system.train()
    views = system.validation_views(cams, images)
    assert system.training  # the mode it was called in
    loop = []
    for c, img in zip(cams, images):
        batch = {"coords": hb.generate_rays(c, c_in=8).view(H, W, -1), "rgb": to_float(img), "W": W, "H": H}
        loop.append(system.validation_image(batch))
    assert len(views) == len(loop)
    for got, want in zip(views, loop):
        assert set(got) == set(want) == {"val/loss", "val/psnr", "val/ssim"}
        for k in got:
            assert got[k].dtype == want[k].dtype and got[k].shape == () and got[k].is_cuda
        assert torch.equal(got["val/psnr"], want["val/psnr"]) and torch.equal(got["val/ssim"], want["val/ssim"])
        assert abs(float(got["val/loss"]) - float(want["val/loss"])) <= 1e-6 * float(want["val/loss"])
    mean, want = system.validation_epoch_end(views), system.validation_epoch_end(loop)
    assert mean["val/psnr"] == want["val/psnr"] and mean["val/ssim"] == want["val/ssim"]
    assert abs(mean["val/loss"] - want["val/loss"]) <= 1e-6 * want["val/loss"]


def test_out_on_a_side_stream():
    system = _system()
    model = system.render_fn.model
    model.set_sub_batch(1000)
    cams = _cameras(3)
    images = _ground_truth(model, cams, [c.time for c in cams], seed=3)
    want = torch.stack(hb.score_views(system, cams, images), 1)
    side = torch.cuda.Stream()
    out = torch.full((3, 2), -7.0, dtype=torch.float64, device="cuda")
    side.wait_stream(torch.cuda.current_stream())
    system.train()
    mse, ssim = system.score_views(cams, images, out=out, stream=side)
    assert system.training
    assert mse.data_ptr() == out.data_ptr()
    side.synchronize()
    assert torch.equal(out, want)


def test_refusals_leave_the_output_untouched():
    model = _render("technicolor_trained").model
    cams = _cameras(3)
    images = _ground_truth(model, cams, [0.0, 0.5, 1.0], seed=2)  # uploads the model
    lib = L.load_library()
    need = int(lib.hr_score_views_workspace_bytes(model._handle, 3, H, W))
    assert need > 0
    assert lib.hr_score_views_workspace_bytes(model._handle, 3, 10, W) == -1
    assert lib.hr_score_views_workspace_bytes(model._handle, 0, H, W) == -1
    assert lib.hr_score_views_workspace_bytes(model._handle, 3, 1 << 30, 1 << 30) == -1
    ws = torch.empty(need + 16, dtype=torch.uint8, device="cuda")
    out = torch.full((4, 2), -7.0, dtype=torch.float64, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream

    def call(recs, times, n=3, gt=images.data_ptr(), dst=out.data_ptr(), wsp=ws.data_ptr(), ws_bytes=need):
        arr = (L.hr_camera * len(recs))(*recs)
        tt = (C.c_float * len(times))(*times)
        return lib.hr_score_views(model._handle, arr, tt, n, gt, L.PIXEL_RGB8, dst, wsp, ws_bytes, stream)

    good = [c.to_c() for c in cams]
    nan_pose = [c.to_c() for c in cams]
    nan_pose[2].c2w[3] = float("nan")
    fish = [c.to_c() for c in cams]
    fish[1].fisheye, fish[1].k1 = 1, float("inf")
    two = [c.to_c() for c in cams]
    two[0].two_plane, two[0].lf_aspect = 1, 0.0
    other = [c.to_c() for c in cams]
    other[1].width = W + 1
    small = [c.to_c() for c in cams]
    for r in small:
        r.width = 10
    big = [c.to_c() for c in cams]
    for r in big:
        r.width = r.height = 1 << 30
    for args, kw, msg in (((nan_pose, [0.0] * 3), {}, b"not finite"),
                          ((fish, [0.0] * 3), {}, b"fisheye"),
                          ((two, [0.0] * 3), {}, b"lf_aspect"),
                          ((good, [0.0, float("nan"), 0.0]), {}, b"time of frame 1"),
                          ((other, [0.0] * 3), {}, b"frame 1 is"),
                          ((small, [0.0] * 3), {}, b"the SSIM window"),
                          ((big, [0.0] * 3), {}, b"overflow"),
                          ((good, [0.0] * 3), {"n": 0}, b"n_views"),
                          ((good, [0.0] * 3), {"ws_bytes": need - 1}, b"workspace too small"),
                          ((good, [0.0] * 3), {"wsp": ws.data_ptr() + 8}, b"16-byte aligned"),
                          ((good, [0.0] * 3), {"dst": out.data_ptr() + 4}, b"8-byte aligned"),
                          ((good, [0.0] * 3), {"gt": None}, b"null")):
        assert call(*args, **kw) != 0
        assert msg in lib.hr_last_error(), (msg, lib.hr_last_error())
    torch.cuda.synchronize()
    assert bool((out == -7.0).all())
    assert call(good, [0.0, 0.5, 1.0]) == 0
    torch.cuda.synchronize()
    want = torch.stack(_per_view(model, cams, [0.0, 0.5, 1.0], images), 1)
    assert torch.equal(out[:3], want) and bool((out[3] == -7.0).all())
