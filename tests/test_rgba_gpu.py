"""RGBA frames on the device (DoNeRF, Catacaustics): the RGBA resize against the CPU oracle (tests/rgba_oracle.py, itself
pinned to Pillow, OpenCV and the reference's get_rgb), training rows and held-out scores against the fp32 composite built on
the CPU, opaque RGBA against the RGB paths, a short training run, and side streams, repeats and refusals.  All torch.equal."""
import ctypes as C
import dataclasses
import json
import os

import numpy as np
import pytest
import torch

import hyperreel_b200 as hb
from hyperreel_b200 import lib as L
from hyperreel_b200.metrics import image_metrics
from tests import rgba_oracle as O
from tests.cases import build_case
from tests.test_score_views_gpu import _cameras, _ground_truth, _render, _system
from tests.test_score_views_gpu import H as SH, W as SW
from tests.test_train_data_gpu import H, W, _cameras as _train_cameras

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "rgba.npz")


def _rgba(n, W, H, seed):
    """Seeded RGBA frames with alpha 0, 255 and in between."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(0, 256, (n, H, W, 4), generator=g, dtype=torch.uint8)
    x[torch.rand((n, H, W), generator=g) < 0.15] = 255
    x[..., 3][torch.rand((n, H, W), generator=g) < 0.15] = 0
    return x


def _oracle(frames, wh, method):
    return torch.from_numpy(np.stack([O.resize(f, wh, method) for f in frames.numpy()]))


def _composite(rgba):
    """get_rgb's composite on the CPU, fp32 [..., 3] (CUDA's division by a scalar is not correctly rounded)."""
    return torch.from_numpy(O.composite(rgba.cpu().numpy()))


def _golden():
    z = np.load(GOLDEN)
    return z, sorted({k.split("/")[0] for k in z.files})


# ---- resize

def test_device_resize_equals_the_oracle():
    for i, (method, (W0, H0), wh) in enumerate((("pil_bicubic", (54, 36), (27, 18)), ("pil_bicubic", (97, 61), (41, 26)),
                                                ("pil_box", (97, 61), (20, 13)), ("pil_lanczos", (63, 45), (21, 15)),
                                                ("pil_bicubic", (48, 40), (48, 23)), ("pil_box", (48, 40), (20, 40)),
                                                ("cv2_area", (64, 48), (32, 24)), ("cv2_area", (45, 33), (15, 11)),
                                                ("cv2_area", (40, 30), (40, 30)), ("pil_bicubic", (40, 30), (40, 30)))):
        frames = _rgba(3, W0, H0, i)
        want = _oracle(frames, wh, method)
        got = hb.resize_frames(frames.cuda(), wh, method, rgba=True).cpu()
        assert torch.equal(got, want), (method, (W0, H0), wh, int((got != want).sum()))
        # BGRA input, a slice of a larger tensor, a side stream, a repeat
        bgra = frames[..., [2, 1, 0, 3]].contiguous().cuda()
        assert torch.equal(hb.resize_frames(bgra, wh, method, bgr=True, rgba=True).cpu(), want), method
        big = torch.full((5, wh[1], wh[0], 4), 77, dtype=torch.uint8, device="cuda")
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        src = frames.cuda()
        with torch.cuda.stream(s):
            hb.resize_frames(src, wh, method, out=big[1:4], stream=s, rgba=True)
            again = hb.resize_frames(src, wh, method, stream=s, rgba=True)
        s.synchronize()
        assert torch.equal(big[1:4].cpu(), want) and torch.equal(again.cpu(), want), method
        assert bool((big[0] == 77).all()) and bool((big[4] == 77).all())


@pytest.mark.parametrize("method,wh", [("cv2_area", (800, 800)), ("pil_bicubic", (1000, 666)), ("pil_box", (500, 333))])
def test_capture_sizes(method, wh):
    """DoNeRF's 2x from 1600 x 1600 and Catacaustics-sized bicubic and box reductions."""
    W0, H0 = (1600, 1600) if method == "cv2_area" else (1500, 999) if method == "pil_bicubic" else (1000, 666)
    frames = _rgba(1, W0, H0, 3)
    assert torch.equal(hb.resize_frames(frames.cuda(), wh, method, rgba=True).cpu(), _oracle(frames, wh, method))


def test_refused_resizes_write_nothing():
    src = _rgba(2, 40, 30, 9).cuda()
    out = torch.full((2, 20, 25, 4), 123, dtype=torch.uint8, device="cuda")
    with pytest.raises(RuntimeError, match="integer factors"):
        hb.resize_frames(src, (25, 20), "cv2_area", out=out, rgba=True)
    with pytest.raises(ValueError, match="out must be"):
        hb.resize_frames(src, (25, 20), "pil_box", out=out[..., :3], rgba=True)
    with pytest.raises(ValueError, match="cv2_linear"):
        hb.resize_frames(src, (25, 20), "cv2_linear", out=out, rgba=True)
    lib = L.load_library()
    need = int(lib.hr_resize_workspace_bytes(2, 30, 40, 20, 25, L.RESIZE_METHODS["pil_bicubic"], L.PIXEL_RGBA8))
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    assert lib.hr_resize_frames(src.data_ptr(), 2, 30, 40, out.data_ptr(), 20, 25, 100, L.RESIZE_METHODS["pil_bicubic"], 0,
                                L.PIXEL_RGBA8, ws.data_ptr(), need - 1, None) != 0
    assert b"needed" in lib.hr_last_error()
    torch.cuda.synchronize()
    assert bool((out == 123).all())


# ---- get_rgb, end to end

def test_batches_from_dataset_frames_carry_get_rgb():
    """For every fixture case: dataset_frames of the RGBA frames, then DeviceRayBatches(rgba=True) (the whole image and
    from_config), and every pixel's row carries the reference's get_rgb colour exactly."""
    z, cases = _golden()
    for case in cases:
        meta = json.loads(str(z[f"{case}/meta"]))
        frames = torch.from_numpy(z[f"{case}/frames"]).cuda()
        rgb = torch.from_numpy(z[f"{case}/rgb"]).cuda()
        out = hb.dataset_frames(meta, frames, scale=meta["scale"])
        W_, H_ = meta["out_wh"]
        assert tuple(out.shape) == (frames.shape[0], H_, W_, 4), case
        n = out.shape[0]
        cams = [hb.Camera(pose=np.eye(4)[:3], K=[[20.0, 0, W_ / 2], [0, 20.0, H_ / 2], [0, 0, 1]], width=W_, height=H_)
                for _ in range(n)]
        ids = torch.arange(n * H_ * W_)
        d = hb.DeviceRayBatches(cams, out, batch_size=97, c_in=6, rgba=True)
        assert torch.equal(d.gather(ids)["rgb"], rgb.reshape(-1, 3)), case
        cfg = hb.to_cfg({"training": {"batch_size": 97}, "dataset": meta})
        f = hb.DeviceRayBatches.from_config(cfg, cams, out, c_in=6)
        assert f.rgba
        b = f.batch(0, with_pixel_ids=True)
        assert torch.equal(b["rgb"], rgb.reshape(-1, 3)[b["pixel_ids"]]), case


# ---- training batches

def test_rows_equal_the_rgb_rays_and_the_composite_in_every_mode():
    cams = _train_cameras()
    rgba = _rgba(3, W, H, 11)
    want_rgb = _composite(rgba).reshape(-1, 3).cuda()
    opaque = rgba.clone()
    opaque[..., 3] = 255
    rgb_images = rgba[..., :3].contiguous()
    n = 3 * H * W
    subsample = [(1, 0), (3, 1), (2, 0)]
    perm = torch.from_numpy(np.random.RandomState(4).permutation(n))
    for kw in (dict(), dict(replacement=True, num_iters=5), dict(subsample=subsample),
               dict(subsample=subsample, replacement=True, num_iters=5)):
        a = hb.DeviceRayBatches(cams, rgba, batch_size=1000, seed=7, rgba=True, **kw)
        r = hb.DeviceRayBatches(cams, rgb_images, batch_size=1000, seed=7, **kw)
        o = hb.DeviceRayBatches(cams, opaque, batch_size=1000, seed=7, rgba=True, **kw)
        for e in (0, 3):
            for x in (a, r, o):
                x.set_epoch(e)
            for i in (0, len(a) - 1):
                ga = a.batch(i, with_pixel_ids=True, with_table_ids=True)
                gr = r.batch(i, with_pixel_ids=True, with_table_ids=True)
                go = o.batch(i, with_pixel_ids=True, with_table_ids=True)
                for k in ("coords", "weight", "pixel_ids", "table_ids"):
                    assert torch.equal(ga[k], gr[k]) and torch.equal(go[k], gr[k]), (kw, k)
                assert torch.equal(ga["rgb"], want_rgb[ga["pixel_ids"]]), kw
                assert torch.equal(go["rgb"], gr["rgb"]), kw  # opaque RGBA is the RGB path bit for bit
        if "subsample" in kw:
            tids = torch.arange(0, a.n_rows, 5)
            ga, gr = a.gather_rows(tids, with_pixel_ids=True), r.gather_rows(tids, with_pixel_ids=True)
            assert torch.equal(ga["coords"], gr["coords"]) and torch.equal(ga["pixel_ids"], gr["pixel_ids"])
            assert torch.equal(ga["rgb"], want_rgb[ga["pixel_ids"]])
    a = hb.DeviceRayBatches(cams, rgba.cuda(), batch_size=1000, rgba=True)
    ga = a.gather(perm, with_pixel_ids=True)
    assert torch.equal(ga["rgb"], want_rgb[perm.cuda()])
    # repeat calls and a side stream write the same bits
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        again = a.gather(perm, with_pixel_ids=True)
    s.synchronize()
    for k in ga:
        assert torch.equal(ga[k], again[k]), k


def test_refused_batch_calls_write_nothing():
    cams = _train_cameras()
    rgba = _rgba(3, W, H, 12).cuda()
    lib = L.load_library()
    recs = (L.hr_camera * 3)(*[c.to_c() for c in cams])
    dcams = torch.frombuffer(bytearray(bytes(recs)), dtype=torch.uint8).cuda()
    coords = torch.full((16, 8), -3.0, device="cuda")
    rgb = torch.full((16, 3), -3.0, device="cuda")
    weight = torch.full((16, 1), -3.0, device="cuda")
    n_rows = C.c_int64(0)
    unaligned = torch.empty(rgba.numel() + 4, dtype=torch.uint8, device="cuda")[1:]
    for images, fmt, msg in ((rgba.data_ptr(), 2, b"unknown pixel format"),
                             (unaligned.data_ptr(), L.PIXEL_RGBA8, b"RGBA images need 4 bytes")):
        assert lib.hr_sample_train_batch(dcams.data_ptr(), 3, images, fmt, H, W, 8, 0, 0, 0, 16, None, coords.data_ptr(),
                                         rgb.data_ptr(), weight.data_ptr(), None, C.byref(n_rows), None) != 0
        assert msg in lib.hr_last_error()
    torch.cuda.synchronize()
    assert bool((coords == -3).all()) and bool((rgb == -3).all()) and bool((weight == -3).all())


def test_donerf_training_from_rgba_batches_lowers_the_loss():
    """Five training_steps of a DoNeRF model on one batch of RGBA rows (the optimiser settings of
    tests/test_train_net_tc_gpu.py's training test): the loss goes down, and the batch's rgb is the composite."""
    case = build_case("donerf_app", n=2048)
    cfg = hb.to_cfg({"model": case.model_cfg, "training": {"ray_chunk": 700, "iters_per_epoch": 4000,
                                                          "optimizers": {"color": {"lr": 0.002}, "color_impl": {"lr": 0.001},
                                                                         "embedding_impl": {"lr": 0.0002}}},
                     "dataset": case.dataset})
    cams, rgba = _train_cameras(), _rgba(3, W, H, 13)
    batches = hb.DeviceRayBatches(cams, rgba, batch_size=2048, c_in=int(case.rays.shape[1]), seed=5, rgba=True)
    batch = batches.batch(0, with_pixel_ids=True)
    ids = batch.pop("pixel_ids")
    assert torch.equal(batch["rgb"], _composite(rgba).reshape(-1, 3).cuda()[ids])
    torch.manual_seed(0)  # the white-background coin flips
    system = hb.INRSystem(cfg, train_net="tc")
    system.load_state_dict(case.state_dict)
    system.cuda()
    losses = [float(system.training_step(batch)["train/loss"]) for _ in range(5)]
    print("donerf_app losses from RGBA batches:", losses)
    assert all(np.isfinite(losses))
    assert losses[-1] < losses[0], losses


# ---- scoring

def _rgba_truth(model, cams, times, seed):
    """The views' renders with noise as colour, and alpha 0, 255 and in between."""
    rgb = _ground_truth(model, cams, times, seed)
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    a = torch.randint(0, 256, rgb.shape[:3], generator=g, device="cuda", dtype=torch.int16)
    a = torch.where(a < 40, 0, torch.where(a > 200, 255, a)).to(torch.uint8)
    return torch.cat([rgb, a[..., None]], -1).contiguous()


@pytest.mark.parametrize("name", ["technicolor_trained", "donerf_s16"])
@pytest.mark.parametrize("sub", [1000, 0])
def test_score_views_equal_image_metrics_of_the_composite(name, sub):
    model = _render(name).model
    model.set_sub_batch(sub)
    F = 4
    cams = _cameras(F)
    times = np.linspace(0.1, 0.9, F)
    images = _rgba_truth(model, cams, times, seed=F)
    got = hb.score_views(model, cams, images, times, rgba=True)
    comp = _composite(images).cuda()
    for f, c in enumerate(cams):
        rays = hb.generate_rays(dataclasses.replace(c, time=float(np.float32(times[f]))), c_in=model.sig.c_in)
        with torch.no_grad():
            pred = model(rays)["rgb"]
        m, s = image_metrics(pred.reshape(SH, SW, 3), comp[f])
        assert torch.equal(got[0][f:f + 1], m) and torch.equal(got[1][f:f + 1], s), f
    again = hb.score_views(model, cams, images, times, rgba=True)
    assert torch.equal(torch.stack(again), torch.stack(got))
    # opaque RGBA scores as the RGB frame, bit for bit
    opaque = images.clone()
    opaque[..., 3] = 255
    rgb = images[..., :3].contiguous()
    assert torch.equal(torch.stack(hb.score_views(model, cams, opaque, times, rgba=True)),
                       torch.stack(hb.score_views(model, cams, rgb, times)))


def test_validation_views_rgba_equal_validation_image_of_the_composite():
    system = _system()
    model = system.render_fn.model
    model.set_sub_batch(1000)
    cams = _cameras(3)
    times = [c.time for c in cams]
    images = _rgba_truth(model, cams, times, seed=7)
    comp = _composite(images).cuda()
    system.train()
    views = system.validation_views(cams, images, rgba=True)
    assert system.training
    for c, got, gt in zip(cams, views, comp):
        want = system.validation_image({"coords": hb.generate_rays(c, c_in=8).view(SH, SW, -1), "rgb": gt, "W": SW, "H": SH})
        assert torch.equal(got["val/psnr"], want["val/psnr"]) and torch.equal(got["val/ssim"], want["val/ssim"])
        assert abs(float(got["val/loss"]) - float(want["val/loss"])) <= 1e-6 * float(want["val/loss"])
    # a side stream with caller-owned output
    want = torch.stack(hb.score_views(system, cams, images, rgba=True), 1)
    side = torch.cuda.Stream()
    out = torch.full((3, 2), -7.0, dtype=torch.float64, device="cuda")
    side.wait_stream(torch.cuda.current_stream())
    system.score_views(cams, images, out=out, stream=side, rgba=True)
    side.synchronize()
    assert torch.equal(out, want)


def test_refused_scores_leave_the_output_untouched():
    model = _render("technicolor_trained").model
    cams = _cameras(3)
    images = _rgba_truth(model, cams, [0.0, 0.5, 1.0], seed=2)  # uploads the model
    lib = L.load_library()
    need = int(lib.hr_score_views_workspace_bytes(model._handle, 3, SH, SW))
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    out = torch.full((3, 2), -7.0, dtype=torch.float64, device="cuda")
    recs = (L.hr_camera * 3)(*[c.to_c() for c in cams])
    tt = (C.c_float * 3)(0.0, 0.5, 1.0)
    unaligned = torch.empty(images.numel() + 4, dtype=torch.uint8, device="cuda")[2:]
    for gt, fmt, msg in ((images.data_ptr(), 5, b"unknown pixel format"),
                         (unaligned.data_ptr(), L.PIXEL_RGBA8, b"4-byte aligned")):
        assert lib.hr_score_views(model._handle, recs, tt, 3, gt, fmt, out.data_ptr(), ws.data_ptr(), need,
                                  torch.cuda.current_stream().cuda_stream) != 0
        assert msg in lib.hr_last_error()
    torch.cuda.synchronize()
    assert bool((out == -7.0).all())
