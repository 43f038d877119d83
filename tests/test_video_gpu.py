"""Videos on the device (hr_render_video_to8b): every frame of render_video is the uint8 frame the whole-frame path
(hr_render_frame_to8b_host) renders for the same camera and time, for static and dynamic models, both sample-net modes,
sub-batches that do and do not fall on frame boundaries, and one video that mixes fisheye and pinhole cameras."""
import ctypes as C
import dataclasses
import os

import numpy as np
import pytest
import torch

import hyperreel_b200 as hb
from hyperreel_b200 import lib as L
from tests.cases import build_case
from tests.test_shipped_yaml_golden import SHIPPED, load_fixture

pytestmark = pytest.mark.gpu

W, H = 48, 30  # 1440 pixels per frame


def _render(name, mode):
    case = build_case(name)
    model = hb.LightfieldModel(case.model_cfg, dataset=case.dataset, mlp_mode=mode)
    render = hb.RenderLightfield(model, None, case.model_cfg.render)
    render.load_state_dict(case.state_dict, strict=False)
    render.eval()
    return render, case.rays


def _pose(base, origin, rx, ry):
    cx, sx, cy, sy = np.cos(rx), np.sin(rx), np.cos(ry), np.sin(ry)
    R = base @ np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]]) @ np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    return np.concatenate([R, np.asarray(origin, np.float64)[:, None]], 1)


# the seeded cases' scenes lie ahead of z = -1 along +z: the camera (looking down its -z axis) turned around to face them
FACING = (np.diag([-1.0, 1.0, -1.0]), [0.0, 0.0, -1.0])


def _cameras(n, base=FACING, distortion=lambda f: None):
    """n cameras turning a little from frame to frame, times spread over [0, 1]."""
    return [hb.Camera(pose=_pose(base[0], base[1], 0.03 * f, -0.05 * f), K=[[40.0, 0, 23.7], [0, 40.0, 15.2], [0, 0, 1]],
                      width=W, height=H, time=f / max(n - 1, 1), cam_idx=0.0, distortion=distortion(f)) for f in range(n)]


def _frames(model, cams, times):
    out = []
    for c, t in zip(cams, times):
        out.append(model.render_frame_to8b(dataclasses.replace(c, time=float(np.float32(t)))).cuda())
    return torch.stack(out, 0)


@pytest.mark.parametrize("mode", ["bf16x3", "fp32"])
@pytest.mark.parametrize("name", ["technicolor_trained", "donerf_s16"])  # dynamic (c_in 8), static (c_in 6)
@pytest.mark.parametrize("sub", [1000, 2880, 0])  # spans frame boundaries; two frames per sub-batch; the default (one)
def test_video_frames_equal_the_whole_frame_path(name, mode, sub):
    render, _ = _render(name, mode)
    model = render.model
    model.set_sub_batch(sub)
    F = 5
    cams = _cameras(F)
    times = np.linspace(0.1, 0.9, F)  # not the cameras' own times: the call's times are the ones rendered
    video = hb.render_video(render, cams, times)
    assert video.shape == (F, H, W, 3) and video.dtype == torch.uint8 and video.is_cuda
    want = _frames(model, cams, times)
    for f in range(F):
        assert torch.equal(video[f], want[f]), f
    assert int(video.max()) > int(video.min())
    again = hb.render_video(model, cams, times)
    assert torch.equal(again, video)
    if model.sig.c_in == 8:  # the time column reaches the pixels of a dynamic model
        assert not torch.equal(hb.render_video(model, cams, times[::-1].copy()), video)


def test_one_frame_equals_the_single_frame_paths():
    render, _ = _render("technicolor_trained", "bf16x3")
    cam = _cameras(1)[0]
    video = hb.render_video(render, [cam], [cam.time])
    assert video.shape == (1, H, W, 3)
    assert torch.equal(video[0].cpu(), render.model.render_frame_to8b(cam))
    sep = render.model.render_to8b(hb.generate_rays(cam, c_in=8)).reshape(H, W, 3)
    assert torch.equal(video[0], sep)


def test_video_mixes_fisheye_and_pinhole_frames():
    by_name = {os.path.basename(p)[:-4]: p for p in SHIPPED}
    plain, cfg, ds, sig, sd, rays, rgb = load_fixture(by_name["immersive_z_plane"])
    model = hb.LightfieldModel(cfg, dataset=ds)
    render = hb.RenderLightfield(model, None, cfg.render, net_chunk=1 << 20)
    render.load_state_dict(sd, strict=False)
    render.eval()
    model.set_sub_batch(1000)
    F = 4
    # at the fixture rays' first origin, looking down -z (as test_fisheye_gpu's frame)
    cams = _cameras(F, base=(np.eye(3), rays[0, :3].tolist()), distortion=lambda f: (-0.3, 0.04) if f % 2 == 0 else None)
    times = [c.time for c in cams]
    video = hb.render_video(model, cams, times)
    want = _frames(model, cams, times)
    for f in range(F):
        assert torch.equal(video[f], want[f]), f
    # the fisheye frames are not the pinhole frames of the same pose
    pin = hb.render_video(model, [dataclasses.replace(c, distortion=None) for c in cams], times)
    assert not torch.equal(pin[0], video[0]) and torch.equal(pin[1], video[1])


def test_out_on_a_side_stream_and_the_system_wrapper():
    case = build_case("technicolor_trained")
    system = hb.INRSystem(hb.to_cfg({"model": case.model_cfg_plain}), dataset=case.dataset)
    system.load_state_dict(case.state_dict)
    cams = _cameras(3)
    times = [c.time for c in cams]
    want = hb.render_video(system, cams, times)
    side = torch.cuda.Stream()
    out = torch.full((3, H, W, 3), 7, dtype=torch.uint8, device="cuda")
    side.wait_stream(torch.cuda.current_stream())
    system.train()
    got = system.render_video(cams, times, out=out, stream=side)
    assert system.training  # the wrapper restores the mode it found
    assert got is out
    side.synchronize()
    assert torch.equal(out, want)


def test_bad_records_are_refused_and_nothing_is_written():
    render, _ = _render("technicolor_trained", "bf16x3")
    model = render.model
    cams = _cameras(3)
    hb.render_video(model, cams, [0.0, 0.5, 1.0])  # uploads the model
    lib = L.load_library()
    need = int(lib.hr_video_workspace_bytes(model._handle, 3, H, W))
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    out = torch.full((3, H, W, 3), 7, dtype=torch.uint8, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream

    def call(recs, times, n=3, ws_bytes=need):
        arr = (L.hr_camera * len(recs))(*recs)
        tt = (C.c_float * len(times))(*times)
        return lib.hr_render_video_to8b(model._handle, arr, tt, n, out.data_ptr(), ws.data_ptr(), ws_bytes, stream)

    good = [c.to_c() for c in cams]
    nan_pose = [c.to_c() for c in cams]
    nan_pose[2].c2w[3] = float("nan")
    fish = [c.to_c() for c in cams]
    fish[1].fisheye, fish[1].k1 = 1, float("inf")
    other = [c.to_c() for c in cams]
    other[1].width = W + 1
    for recs, times, n, ws_bytes, msg in ((nan_pose, [0.0] * 3, 3, need, b"not finite"),
                                          (fish, [0.0] * 3, 3, need, b"fisheye"),
                                          (good, [0.0, float("nan"), 0.0], 3, need, b"time of frame 1"),
                                          (other, [0.0] * 3, 3, need, b"frame 1 is"),
                                          (good, [0.0] * 3, 0, need, b"n_frames"),
                                          (good, [0.0] * 3, 3, need - 1, b"workspace too small")):
        assert call(recs, times, n, ws_bytes) != 0
        assert msg in lib.hr_last_error(), lib.hr_last_error()
    big = [c.to_c() for c in cams]
    for r in big:
        r.width = r.height = 1 << 30
    assert lib.hr_video_workspace_bytes(model._handle, 3, 1 << 30, 1 << 30) == -1
    assert call(big, [0.0] * 3) != 0 and b"overflow" in lib.hr_last_error()
    torch.cuda.synchronize()
    assert bool((out == 7).all())
