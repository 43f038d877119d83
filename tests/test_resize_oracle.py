"""The frame-resize oracle (tests/resize_oracle.py) against Pillow and OpenCV themselves and against the reference's get_rgb
(tests/golden/resize.npz), and the host-side refusals of resize_frames / dataset_frames and of the C entry points.  No GPU."""
import json
import os

import numpy as np
import pytest
import torch

import hyperreel_b200 as hb
from hyperreel_b200 import lib as L
from tests import resize_oracle as ro

cv2 = pytest.importorskip("cv2")
Image = pytest.importorskip("PIL.Image")

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "resize.npz")
PIL_FILTER = {"pil_lanczos": Image.LANCZOS, "pil_bicubic": Image.BICUBIC, "pil_box": Image.BOX}
CV2_FLAG = {"cv2_linear": cv2.INTER_LINEAR, "cv2_area": cv2.INTER_AREA}

# (W0, H0) -> (W, H): 1-pixel and prime sizes, exact 2x / 3x / 8x, non-integer ratios, one axis kept, the identity
SIZES = [((1, 1), (1, 1)), ((7, 1), (3, 1)), ((1, 13), (1, 5)), ((2, 2), (1, 1)), ((13, 11), (13, 11)),
         ((13, 11), (6, 5)), ((13, 11), (1, 1)), ((17, 19), (5, 7)), ((31, 29), (30, 28)), ((64, 48), (32, 24)),
         ((64, 48), (8, 6)), ((63, 45), (21, 15)), ((64, 48), (64, 24)), ((64, 48), (20, 48)), ((97, 61), (43, 37)),
         ((101, 67), (50, 33)), ((128, 96), (16, 12)), ((200, 150), (133, 100)), ((338, 254), (169, 127)),
         ((504, 378), (63, 47)), ((331, 257), (110, 85))]


def _frame(W, H, seed):
    rng = np.random.default_rng(seed)
    img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    img[rng.random((H, W)) < 0.2] = 255  # hard edges drive the Lanczos and bicubic taps past both clips
    img[rng.random((H, W)) < 0.2] = 0
    return img


def _library(img, size, method):
    if method in PIL_FILTER:
        return np.asarray(Image.fromarray(img).resize(tuple(size), PIL_FILTER[method]))
    return cv2.resize(img, tuple(size), interpolation=CV2_FLAG[method])


@pytest.mark.parametrize("method", ro.METHODS)
def test_oracle_equals_the_library(method):
    checked = 0
    for i, ((W0, H0), (W, H)) in enumerate(SIZES):
        img = _frame(W0, H0, i)
        try:
            ours = ro.resize(img, (W, H), method)
        except ValueError:  # cv2_area at a non-integer factor: refused, checked below
            assert method == "cv2_area"
            continue
        ref = _library(img, (W, H), method)
        assert ours.shape == ref.shape and np.array_equal(ours, ref), (method, (W0, H0), (W, H))
        checked += 1
    assert checked >= 10


def test_cv2_paths_and_refusals():
    assert ro.cv2_path((54, 40), (27, 20), "cv2_linear") == "area2"  # OpenCV's own rule: INTER_LINEAR at 2x is INTER_AREA
    assert ro.cv2_path((54, 40), (18, 20), "cv2_linear") == "linear"
    assert ro.cv2_path((54, 40), (18, 20), "cv2_area") == "area"
    assert ro.cv2_path((54, 40), (54, 40), "cv2_linear") == "copy"
    with pytest.raises(ValueError, match="integer reduction"):
        ro.cv2_path((54, 40), (25, 20), "cv2_area")
    with pytest.raises(ValueError, match="upscaling"):
        ro.cv2_path((54, 40), (55, 40), "cv2_linear")
    with pytest.raises(ValueError, match="upscaling"):
        ro.resize(np.zeros((4, 4, 3), np.uint8), (4, 5), "pil_lanczos")


def test_flag_in_the_dst_slot_is_inter_linear():
    """neural_3d.py / immersive.py call cv2.resize(img, wh, cv2.INTER_LANCZOS4) and cv2.resize(img, wh, cv2.INTER_AREA):
    the third positional argument is dst, so both run INTER_LINEAR.  An OpenCV that changes this fails here."""
    img = _frame(97, 61, 3)
    for wh in ((48, 30), (64, 40), (30, 20)):
        linear = cv2.resize(img, wh, interpolation=cv2.INTER_LINEAR)
        assert np.array_equal(cv2.resize(img, wh, cv2.INTER_LANCZOS4), linear)
        assert np.array_equal(cv2.resize(img, wh, cv2.INTER_AREA), linear)
    assert not np.array_equal(cv2.resize(img, (64, 40), cv2.INTER_LANCZOS4),
                              cv2.resize(img, (64, 40), interpolation=cv2.INTER_LANCZOS4))


def _golden_cases():
    z = np.load(GOLDEN)
    return z, sorted({k.split("/")[0] for k in z.files})


def test_oracle_reproduces_get_rgb():
    """dataset_steps' resizes, restated by the oracle, then u8 / 255 correctly rounded (T.ToTensor()), equal the reference's
    get_rgb output for every fixture case."""
    z, cases = _golden_cases()
    assert len(cases) >= 15
    for case in cases:
        meta = json.loads(str(z[f"{case}/meta"]))
        frames, rgb = z[f"{case}/frames"], z[f"{case}/rgb"]
        steps = hb.resize.dataset_steps(meta, (frames.shape[2], frames.shape[1]), meta["scale"])
        for f in range(frames.shape[0]):
            img = frames[f]
            for method, wh in steps:
                img = ro.resize(img, wh, method)
            assert [img.shape[1], img.shape[0]] == meta["out_wh"], case
            ours = img.reshape(-1, 3).astype(np.float32) / np.float32(255)
            assert np.array_equal(ours, rgb[f]), (case, f)


def test_dataset_steps():
    n3d = {"name": "neural_3d", "img_wh": [1352, 1014]}
    assert hb.resize.dataset_steps(n3d, (2704, 2028)) == [("cv2_linear", (1352, 1014))]
    assert hb.resize.dataset_steps(n3d, (2704, 2028), scale=2) == [("cv2_linear", (1352, 1014)), ("cv2_linear", (676, 507))]
    assert hb.resize.dataset_steps(n3d, (1352, 1014)) == []
    llff = {"name": "llff", "img_wh": [504, 378]}
    assert hb.resize.dataset_steps(llff, (4032, 3024)) == [("pil_lanczos", (504, 378))]
    assert hb.resize.dataset_steps(llff, (504, 378), scale=4) == [("pil_box", (126, 94))]


def test_dataset_frames_refusals():
    frames = torch.zeros((2, 8, 8, 3), dtype=torch.uint8)
    with pytest.raises(ValueError, match="RGBA"):
        hb.dataset_frames({"name": "donerf", "img_wh": [4, 4]}, frames)
    with pytest.raises(ValueError, match="BICUBIC"):
        hb.dataset_frames({"name": "catacaustics", "img_wh": [4, 4]}, frames)
    with pytest.raises(ValueError, match="no get_rgb resize"):
        hb.dataset_frames({"name": "blender", "img_wh": [4, 4]}, frames)
    with pytest.raises(ValueError, match="img_wh"):
        hb.dataset_frames({"name": "llff"}, frames)
    with pytest.raises(ValueError, match="scale"):
        hb.dataset_frames({"name": "llff", "img_wh": [4, 4]}, frames, scale=0)
    with pytest.raises(ValueError, match="frames must be"):
        hb.dataset_frames({"name": "llff", "img_wh": [4, 4]}, frames[0])
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        hb.dataset_frames({"name": "llff", "img_wh": [4, 4]}, frames)


def test_resize_frames_refusals():
    frames = torch.zeros((2, 8, 8, 3), dtype=torch.uint8)
    with pytest.raises(ValueError, match="unknown method"):
        hb.resize_frames(frames, (4, 4), "lanczos")
    for bad in (frames.float(), torch.zeros((2, 8, 8, 4), dtype=torch.uint8), torch.zeros((8, 3), dtype=torch.uint8),
                frames.numpy()):
        with pytest.raises(ValueError, match="frames must be"):
            hb.resize_frames(bad, (4, 4), "pil_box")
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        hb.resize_frames(frames, (4, 4), "pil_box")


def test_c_entry_points_refuse_before_touching_the_device():
    """hr_resize_frames validates on the host before anything is enqueued: these calls fail without a GPU and without
    dereferencing their (fake) pointers."""
    lib = L.load_library()
    ws = lambda *args: lib.hr_resize_workspace_bytes(*args, L.PIXEL_RGB8)
    assert ws(4, 2028, 2704, 1014, 1352, L.RESIZE_METHODS["cv2_linear"]) == 0  # the 2x INTER_AREA path needs no tables
    assert ws(4, 2028, 2704, 1014, 1352, L.RESIZE_METHODS["cv2_area"]) == 0
    assert ws(1, 30, 40, 30, 40, L.RESIZE_METHODS["pil_lanczos"]) == 0         # the copy
    assert ws(1, 30, 40, 20, 25, L.RESIZE_METHODS["cv2_linear"]) > 0
    assert ws(2, 3024, 4032, 378, 504, L.RESIZE_METHODS["pil_lanczos"]) >= 2 * 3024 * 504 * 3 // 2
    assert ws(1, 30, 40, 20, 25, L.RESIZE_METHODS["cv2_area"]) == -1          # non-integer INTER_AREA
    assert ws(1, 30, 40, 31, 40, L.RESIZE_METHODS["pil_box"]) == -1           # enlargement
    assert ws(1, 30, 40, 20, 20, 7) == -1
    fake = 1 << 40
    def call(n=1, H0=30, W0=40, H=15, W=20, row=60, method=4, flags=0, wsp=None, wsb=0, src=fake, dst=fake):
        return lib.hr_resize_frames(src, n, H0, W0, dst, H, W, row, method, flags, L.PIXEL_RGB8, wsp, wsb, None)
    # every call below is refused by the host checks (a valid call would launch; the GPU tests make those)
    cases = [(dict(src=None), "null"), (dict(method=9), "unknown method"), (dict(flags=2), "unknown flags"),
             (dict(n=0), "bad sizes"), (dict(H=31), "enlarges"), (dict(W=30, method=4), "integer factors"),
             (dict(row=59), "dst_row_stride"), (dict(H=20, W=25, row=75, method=3), "workspace"),
             (dict(H=20, W=25, row=75, method=3, wsp=fake + 8, wsb=1 << 20), "workspace"),
             (dict(H=20, W=25, row=75, method=3, wsp=fake, wsb=16), "workspace of 16 bytes"),
             (dict(row=1 << 62), "overflow a 64-bit size"),
             (dict(n=2 ** 31 - 1, H0=2 ** 31 - 1, W0=2 ** 31 - 1, H=1, W=1), "overflow a 64-bit size")]
    for kw, msg in cases:
        assert call(**kw) != 0, kw
        assert msg in lib.hr_last_error().decode(), (kw, lib.hr_last_error())


def test_size_limits():
    """Sizes whose bytes overflow int64 are refused (-1), and so are Pillow reductions that need more filter coefficients
    than Pillow itself allows (outSize > INT_MAX / (ksize * sizeof(double)): it raises MemoryError)."""
    lib = L.load_library()
    ws = lambda *args: lib.hr_resize_workspace_bytes(*args, L.PIXEL_RGB8)
    big = 2 ** 31 - 1
    assert ws(big, big, big, 1, 1, L.RESIZE_METHODS["cv2_area"]) == -1
    assert ws(big, 4096, 4096, 2048, 2047, L.RESIZE_METHODS["pil_lanczos"]) > 2 ** 50  # large, but within int64
    # Lanczos, one output pixel: ksize = ceil(3 * W0) * 2 + 1, at most INT_MAX / 8 = 268435455, so W0 <= 44739242
    last = 44739242
    assert ws(1, 1, last, 1, 1, L.RESIZE_METHODS["pil_lanczos"]) > 0
    assert ws(1, 1, last + 1, 1, 1, L.RESIZE_METHODS["pil_lanczos"]) == -1
    with pytest.raises(MemoryError):
        Image.new("RGB", (last + 1, 1)).resize((1, 1), Image.LANCZOS)
