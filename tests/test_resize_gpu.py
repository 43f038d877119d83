"""hr_resize_frames on the device (csrc/hr_resize.cu) against the CPU oracle (tests/resize_oracle.py, itself pinned to Pillow,
OpenCV and the reference's get_rgb), bit for bit: every method at the fixture's sizes and at the shipped capture sizes,
batches, writes into a slice, BGR input, a side stream, repeatability, refusals, and training batches built from the
resized frames."""
import json
import os

import numpy as np
import pytest
import torch

import hyperreel_b200 as hb
from hyperreel_b200 import lib as L
from tests import resize_oracle as ro

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "resize.npz")
K = [[20.0, 0, 8], [0, 20.0, 6], [0, 0, 1]]


def _golden():
    z = np.load(GOLDEN)
    return z, sorted({k.split("/")[0] for k in z.files})


def _frames(n, W, H, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(0, 256, (n, H, W, 3), generator=g, dtype=torch.uint8)
    x[torch.rand((n, H, W), generator=g) < 0.15] = 255
    x[torch.rand((n, H, W), generator=g) < 0.15] = 0
    return x


def _oracle(frames, wh, method):
    return torch.from_numpy(np.stack([ro.resize(f, wh, method) for f in frames.numpy()]))


def _check(frames, wh, method, **kw):
    got = hb.resize_frames(frames.cuda(), wh, method, **kw).cpu()
    want = _oracle(frames, wh, method)
    assert torch.equal(got, want), (method, tuple(frames.shape), wh, int((got != want).sum()))


def test_every_method_at_the_fixture_sizes():
    z, cases = _golden()
    for case in cases:
        meta = json.loads(str(z[f"{case}/meta"]))
        frames = torch.from_numpy(z[f"{case}/frames"])
        for wh in {tuple(meta["img_wh"]), tuple(meta["out_wh"])}:
            for method in ro.METHODS:
                try:
                    want = _oracle(frames, wh, method)
                except ValueError:  # cv2_area at a non-integer factor: the device refuses it too
                    with pytest.raises(RuntimeError, match="integer factors"):
                        hb.resize_frames(frames.cuda(), wh, method)
                    continue
                assert torch.equal(hb.resize_frames(frames.cuda(), wh, method).cpu(), want), (case, wh, method)


def test_dataset_frames_equal_get_rgb():
    """dataset_frames on the fixture's frames, RGB and BGR, is the reference's get_rgb output times 255 exactly."""
    z, cases = _golden()
    for case in cases:
        meta = json.loads(str(z[f"{case}/meta"]))
        frames = torch.from_numpy(z[f"{case}/frames"]).cuda()
        rgb = torch.from_numpy(z[f"{case}/rgb"])
        for bgr in (False, True):
            x = frames.flip(-1).contiguous() if bgr else frames
            out = hb.dataset_frames(meta, x, bgr=bgr, scale=meta["scale"]).cpu()
            assert list(out.shape[1:3]) == meta["out_wh"][::-1], case
            got = out.reshape(out.shape[0], -1, 3).float().div(255)  # T.ToTensor()'s conversion, on the CPU
            assert torch.equal(got, rgb), (case, bgr)


@pytest.mark.parametrize("method,wh", [("cv2_linear", (1352, 1014)), ("cv2_area", (1352, 1014)), ("cv2_linear", (1000, 750)),
                                       ("cv2_area", (676, 507)), ("pil_lanczos", (1352, 1014)), ("pil_box", (1352, 1014)),
                                       ("pil_bicubic", (1000, 750))])
def test_neural3d_capture_size(method, wh):
    _check(_frames(1, 2704, 2028, 5), wh, method)


def test_llff_capture_size():
    _check(_frames(1, 4032, 3024, 6), (504, 378), "pil_lanczos")


def test_batch_slice_bgr_stream_repeat():
    frames = _frames(5, 97, 61, 7)
    # the last two keep one axis: Pillow's one-pass paths (the horizontal pass straight into out, the vertical pass reading
    # the BGR source)
    for method, wh in (("pil_lanczos", (43, 37)), ("cv2_linear", (43, 37)), ("cv2_area", (97, 61)), ("pil_box", (48, 30)),
                       ("pil_bicubic", (40, 61)), ("pil_lanczos", (97, 30))):
        want = _oracle(frames, wh, method)
        src = frames.cuda()
        big = torch.full((9, wh[1], wh[0], 3), 77, dtype=torch.uint8, device="cuda")
        ret = hb.resize_frames(src, wh, method, out=big[2:7])
        assert ret.data_ptr() == big[2].data_ptr()
        assert torch.equal(big[2:7].cpu(), want), method
        assert bool((big[:2] == 77).all()) and bool((big[7:] == 77).all())
        bgr = hb.resize_frames(src.flip(-1).contiguous(), wh, method, bgr=True).cpu()
        assert torch.equal(bgr, want), method
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            a = hb.resize_frames(src, wh, method, stream=s)
            b = hb.resize_frames(src, wh, method, stream=s)
        s.synchronize()
        assert torch.equal(a.cpu(), want) and torch.equal(a, b), method
        one = hb.resize_frames(src[3], wh, method)
        assert one.shape == (wh[1], wh[0], 3) and torch.equal(one.cpu(), want[3])


def test_rows_of_a_wider_tensor():
    """out may be a column window of wider frames: rows contiguous, frames H rows apart."""
    frames = _frames(3, 50, 40, 8)
    wide = torch.full((3, 20, 40, 3), 9, dtype=torch.uint8, device="cuda")
    window = wide[:, :, 5:30]
    hb.resize_frames(frames.cuda(), (25, 20), "cv2_linear", out=window)
    assert torch.equal(window.cpu(), _oracle(frames, (25, 20), "cv2_linear"))
    assert bool((wide[:, :, :5] == 9).all()) and bool((wide[:, :, 30:] == 9).all())


def test_refused_calls_write_nothing():
    src = _frames(2, 40, 30, 9).cuda()
    out = torch.full((2, 20, 25, 3), 123, dtype=torch.uint8, device="cuda")
    with pytest.raises(RuntimeError, match="integer factors"):
        hb.resize_frames(src, (25, 20), "cv2_area", out=out)
    out2 = torch.full((2, 31, 40, 3), 123, dtype=torch.uint8, device="cuda")
    with pytest.raises(RuntimeError, match="enlarges"):
        hb.resize_frames(src, (40, 31), "pil_lanczos", out=out2)
    with pytest.raises(ValueError, match="out must be"):
        hb.resize_frames(src, (25, 20), "cv2_linear", out=out[:, :, :24])
    with pytest.raises(ValueError, match="out must be"):
        hb.resize_frames(src, (20, 25), "cv2_linear", out=out.transpose(1, 2))
    lib = L.load_library()
    need = int(lib.hr_resize_workspace_bytes(2, 30, 40, 20, 25, L.RESIZE_METHODS["pil_lanczos"], L.PIXEL_RGB8))
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    assert lib.hr_resize_frames(src.data_ptr(), 2, 30, 40, out.data_ptr(), 20, 25, 75, L.RESIZE_METHODS["pil_lanczos"], 0,
                                L.PIXEL_RGB8, ws.data_ptr(), need - 1, None) != 0
    assert b"needed" in lib.hr_last_error()
    torch.cuda.synchronize()
    assert bool((out == 123).all()) and bool((out2 == 123).all())


def test_streamed_chunks_into_training_batches():
    """A Neural-3D-style load: capture-size BGR chunks resized into slices of one training tensor, then DeviceRayBatches over
    it; every pixel's rgb row is the reference's get_rgb value."""
    z, _ = _golden()
    meta = json.loads(str(z["neural3d_odd_s2/meta"]))
    frames = torch.from_numpy(z["neural3d_odd_s2/frames"])
    rgb = torch.from_numpy(z["neural3d_odd_s2/rgb"])
    W, H = meta["out_wh"]
    n = frames.shape[0]
    train = torch.empty((n, H, W, 3), dtype=torch.uint8, device="cuda")
    for i in range(n):  # one frame per chunk, decoded as BGR
        hb.dataset_frames(meta, frames[i:i + 1].flip(-1).contiguous().cuda(), out=train[i:i + 1], bgr=True,
                          scale=meta["scale"])
    cams = [hb.Camera(pose=np.eye(4)[:3], K=K, width=W, height=H, time=0.0) for _ in range(n)]
    d = hb.DeviceRayBatches(cams, train, batch_size=64)
    rows = d.gather(torch.arange(n * H * W), with_pixel_ids=True)
    assert torch.equal(rows["rgb"].cpu(), rgb.reshape(-1, 3))


def test_non_contiguous_frames_on_a_side_stream():
    """Non-contiguous frames (an NCHW decode permuted, the colour channels of a BGRA decode, a strided slice) are copied on
    the work stream, in memory of that stream: reusing the caller's stream's memory right after the call cannot touch the
    copy."""
    frames = _frames(4, 97, 61, 10)
    nchw = frames.permute(0, 3, 1, 2).contiguous().cuda()
    bgra = torch.cat([frames.flip(-1), frames[..., :1]], -1).cuda()
    pairs = torch.stack([frames, 255 - frames], 3).reshape(4, 61, 194, 3).cuda()   # every other pixel is a frame's
    cases = ((nchw.permute(0, 2, 3, 1), False), (bgra[..., :3], True), (pairs[:, :, ::2], False))
    for method, wh in (("pil_lanczos", (43, 37)), ("cv2_linear", (43, 37)), ("pil_box", (97, 30))):
        want = _oracle(frames, wh, method)
        for src, bgr in cases:
            assert not src.is_contiguous()
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            got = hb.resize_frames(src, wh, method, bgr=bgr, stream=s)
            # the caller's stream reuses its freed memory at once
            junk = torch.full((src.numel() * 2,), 255, dtype=torch.uint8, device="cuda")
            s.synchronize()
            del junk
            assert torch.equal(got.cpu(), want), (method, tuple(src.stride()), bgr)
