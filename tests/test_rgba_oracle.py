"""The RGBA frame oracle (tests/rgba_oracle.py) against Pillow, OpenCV and torch themselves and against the reference's
get_rgb of DoNeRF and Catacaustics (tests/golden/rgba.npz), and the host-side refusals of the RGBA paths.  No GPU."""
import json
import os

import numpy as np
import pytest
import torch

import hyperreel_b200 as hb
from hyperreel_b200 import lib as L
from tests import rgba_oracle as O
from tests.test_resize_oracle import SIZES

cv2 = pytest.importorskip("cv2")
Image = pytest.importorskip("PIL.Image")

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "rgba.npz")
PIL_FILTER = {"pil_lanczos": Image.LANCZOS, "pil_bicubic": Image.BICUBIC, "pil_box": Image.BOX}
K = [[20.0, 0, 8], [0, 20.0, 6], [0, 0, 1]]


def _all_pairs():
    """Every (c, a) pair once: a [256, 256, 4] image with c = column in the three colour channels and a = row."""
    c, a = np.meshgrid(np.arange(256), np.arange(256))
    return np.stack([c, c, c, a], -1).astype(np.uint8)


def _frame(W, H, seed):
    rng = np.random.default_rng(seed)
    img = rng.integers(0, 256, (H, W, 4), dtype=np.uint8)
    img[rng.random((H, W)) < 0.2] = 255  # hard edges, opaque
    img[..., 3][rng.random((H, W)) < 0.2] = 0  # transparent pixels keep their colour in RGBA
    return img


def test_premultiply_equals_pillow_for_every_pair():
    img = _all_pairs()
    ref = np.asarray(Image.fromarray(img, "RGBA").convert("RGBa"))
    ours = img.astype(np.int64)
    ours[..., :3] = O.premultiply(ours[..., :3], ours[..., 3:])
    assert np.array_equal(ours, ref)


def test_unpremultiply_equals_pillow_for_every_pair():
    img = _all_pairs()
    ref = np.asarray(Image.frombytes("RGBa", (256, 256), img.tobytes()).convert("RGBA"))
    ours = img.astype(np.int64)
    ours[..., :3] = O.unpremultiply(ours[..., :3], ours[..., 3:])
    assert np.array_equal(ours, ref)


def test_composite_equals_torch_for_every_pair():
    """get_rgb's composite with torch on the CPU (T.ToTensor()'s division, then rgb * a + (1 - a)) for all 65 536 pairs, and
    an FMA-contracted composite differs, so the device must round each operation on its own."""
    img = _all_pairs()
    t = torch.from_numpy(img).permute(2, 0, 1).float().div(255).view(4, -1).permute(1, 0)
    ref = (t[:, :3] * t[:, -1:] + (1 - t[:, -1:])).numpy()
    ours = O.composite(img).reshape(-1, 3)
    assert np.array_equal(ours, ref)
    x = img.reshape(-1, 4).astype(np.float64) / 255
    x = x.astype(np.float32).astype(np.float64)
    fused = (x[:, :3] * x[:, 3:] + (1 - x[:, 3:]).astype(np.float32)).astype(np.float32)  # one rounding of c * a + b
    assert not np.array_equal(fused, ref)


@pytest.mark.parametrize("method", ["pil_lanczos", "pil_bicubic", "pil_box", "cv2_area"])
def test_oracle_equals_the_library(method):
    checked = 0
    for i, ((W0, H0), (W, H)) in enumerate(SIZES):
        img = _frame(W0, H0, i)
        try:
            ours = O.resize(img, (W, H), method)
        except ValueError:  # cv2_area at a non-integer factor
            assert method == "cv2_area"
            continue
        if method in PIL_FILTER:
            ref = np.asarray(Image.fromarray(img, "RGBA").resize((W, H), PIL_FILTER[method]))
        else:
            ref = cv2.resize(img, (W, H), interpolation=cv2.INTER_AREA)
        assert ours.shape == ref.shape and np.array_equal(ours, ref), (method, (W0, H0), (W, H))
        checked += 1
    assert checked >= 8


def test_pillow_resamples_rgba_premultiplied():
    """Image.resize of an RGBA image is not a per-channel resample, and two resizes are not one round trip: the second
    starts from the RGBA the first returned."""
    img = _frame(54, 36, 7)
    per_channel = np.asarray(Image.fromarray(img[..., :3]).resize((27, 18), Image.BICUBIC))
    ref = np.asarray(Image.fromarray(img, "RGBA").resize((27, 18), Image.BICUBIC))
    assert not np.array_equal(per_channel, ref[..., :3])
    twice = np.asarray(Image.fromarray(ref, "RGBA").resize((9, 6), Image.BOX))
    assert np.array_equal(O.resize(O.resize(img, (27, 18), "pil_bicubic"), (9, 6), "pil_box"), twice)


def test_oracle_reproduces_get_rgb():
    """The resizes dataset_steps picks for donerf and catacaustics, restated by the oracle, then the composite, equal the
    reference's get_rgb output for every fixture case."""
    z = np.load(GOLDEN)
    cases = sorted({k.split("/")[0] for k in z.files})
    assert len(cases) >= 10 and {json.loads(str(z[f"{c}/meta"]))["name"] for c in cases} == {"donerf", "catacaustics"}
    for case in cases:
        meta = json.loads(str(z[f"{case}/meta"]))
        frames, rgb = z[f"{case}/frames"], z[f"{case}/rgb"]
        steps = hb.resize.dataset_steps(meta, (frames.shape[2], frames.shape[1]), meta["scale"])
        assert steps == O.dataset_steps(meta["name"], (frames.shape[2], frames.shape[1]), meta["img_wh"], meta["scale"])
        for f in range(frames.shape[0]):
            img = frames[f]
            for method, wh in steps:
                img = O.resize(img, wh, method)
            assert [img.shape[1], img.shape[0]] == meta["out_wh"], case
            assert np.array_equal(O.composite(img).reshape(-1, 3), rgb[f]), (case, f)


def test_dataset_steps():
    don = {"name": "donerf", "img_wh": [800, 800]}
    assert hb.resize.dataset_steps(don, (800, 800)) == []
    assert hb.resize.dataset_steps(don, (1600, 1600)) == [("cv2_area", (800, 800))]
    assert hb.resize.dataset_steps(don, (800, 800), scale=2) == [("cv2_area", (400, 400))]
    cat = {"name": "catacaustics", "img_wh": [1000, 666]}
    assert hb.resize.dataset_steps(cat, (1500, 999)) == [("pil_bicubic", (1000, 666))]
    assert hb.resize.dataset_steps(cat, (1500, 999), scale=2) == [("pil_bicubic", (1000, 666)), ("pil_box", (500, 333))]


def test_rgba_host_refusals():
    rgba = torch.zeros((2, 8, 8, 4), dtype=torch.uint8)
    rgb = torch.zeros((2, 8, 8, 3), dtype=torch.uint8)
    # dataset_frames: RGBA frames pass the channel check for both datasets and reach the device check
    for name in ("donerf", "catacaustics"):
        with pytest.raises(RuntimeError, match="CUDA tensor"):
            hb.dataset_frames({"name": name, "img_wh": [4, 4]}, rgba)
    with pytest.raises(ValueError, match="frames must be"):
        hb.dataset_frames({"name": "llff", "img_wh": [4, 4]}, rgba)
    # resize_frames: the caller says the fourth channel is alpha, and 3-channel frames are refused with rgba=True
    with pytest.raises(ValueError, match=r"frames must be a uint8 tensor \[n, H, W, 4\]"):
        hb.resize_frames(rgb, (4, 4), "pil_box", rgba=True)
    with pytest.raises(ValueError, match="cv2_linear"):
        hb.resize_frames(rgba, (4, 4), "cv2_linear", rgba=True)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        hb.resize_frames(rgba, (4, 4), "pil_box", rgba=True)
    # DeviceRayBatches
    cams = [hb.Camera(pose=np.eye(4)[:3], K=K, width=8, height=8) for _ in range(2)]
    with pytest.raises(ValueError, match=r"\[n, H, W, 4\]"):
        hb.DeviceRayBatches(cams, rgb, batch_size=4, rgba=True)
    with pytest.raises(ValueError, match=r"\[n, H, W, 3\]"):
        hb.DeviceRayBatches(cams, rgba, batch_size=4)
    with pytest.raises(ValueError, match="importance"):
        hb.DeviceRayBatches(cams, rgba, batch_size=4, rgba=True, importance=[None, (4, 0)])


def test_score_views_rgba_refusals():
    from tests.cases import build_case

    case = build_case("technicolor_trained")
    model = hb.LightfieldModel(case.model_cfg, dataset=case.dataset)
    model.eval()
    cams = [hb.Camera(pose=np.eye(4)[:3], K=K, width=16, height=12) for _ in range(3)]
    with pytest.raises(ValueError, match=r"images must be .*\(3, 12, 16, 4\)"):
        hb.score_views(model, cams, torch.zeros((3, 12, 16, 3), dtype=torch.uint8), rgba=True)
    with pytest.raises(ValueError, match=r"images must be .*\(3, 12, 16, 3\)"):
        hb.score_views(model, cams, torch.zeros((3, 12, 16, 4), dtype=torch.uint8))
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        hb.score_views(model, cams, torch.zeros((3, 12, 16, 4), dtype=torch.uint8), rgba=True)
    system = hb.INRSystem(hb.to_cfg({"model": case.model_cfg_plain}), dataset=case.dataset)
    system.train()
    with pytest.raises(ValueError, match="images must be"):
        system.validation_views(cams, torch.zeros((3, 12, 16, 3), dtype=torch.uint8), rgba=True)
    assert system.training


def test_c_entry_points_refuse_before_touching_the_device():
    """The entry points validate RGBA calls on the host before anything is enqueued: these calls fail without a GPU and without
    dereferencing their (fake) pointers."""
    lib = L.load_library()
    ws = lib.hr_resize_workspace_bytes
    pil, lin, area = (L.RESIZE_METHODS[m] for m in ("pil_bicubic", "cv2_linear", "cv2_area"))
    # RGB workspaces as they were before the entry points took a pixel format
    for args, need in (((2, 3024, 4032, 378, 504, pil), 9268224), ((1, 30, 40, 20, 25, pil), 4352),
                       ((1, 30, 40, 15, 20, area), 0)):
        assert ws(*args, L.PIXEL_RGB8) == need, args
    # the tables are the same; the intermediate holds 4 bytes per pixel instead of 3
    n, H0, W0, H, W = 2, 300, 400, 150, 130
    rgb, rgba = ws(n, H0, W0, H, W, pil, L.PIXEL_RGB8), ws(n, H0, W0, H, W, pil, L.PIXEL_RGBA8)
    assert rgba > rgb and rgba - rgb >= n * H0 * W // 3 - 512
    assert ws(1, 30, 40, 15, 20, lin, L.PIXEL_RGBA8) == -1
    assert ws(1, 30, 40, 15, 20, pil, 2) == -1
    fake = 1 << 40

    def resize(H=15, W=20, row=80, method=pil, fmt=L.PIXEL_RGBA8):
        return lib.hr_resize_frames(fake, 1, 30, 40, fake, H, W, row, method, 0, fmt, None, 0, None)

    for kw, msg in ((dict(fmt=7), "unknown pixel format"), (dict(method=lin), "cv2_linear is not supported for RGBA"),
                    (dict(row=79), "dst_row_stride"), (dict(), "workspace")):
        assert resize(**kw) != 0, kw
        assert msg in lib.hr_last_error().decode(), (kw, lib.hr_last_error())
    assert resize(method=area, row=79) != 0 and "dst_row_stride 79" in lib.hr_last_error().decode()

    def batch(images=fake, fmt=L.PIXEL_RGBA8):
        return lib.hr_sample_train_batch(fake, 1, images, fmt, 4, 4, 8, 0, 0, 0, 4, None, fake, fake, fake, None, None, None)

    def rows(images=fake, fmt=L.PIXEL_RGBA8):
        return lib.hr_sample_train_rows(fake, 1, images, fmt, 4, 4, 8, fake, fake, 16, L.SAMPLE_PERMUTE, 0, 0, 0, 4, None,
                                        fake, fake, fake, None, None, None, None)

    for fn in (batch, rows):
        assert fn(fmt=2) != 0 and "unknown pixel format 2" in lib.hr_last_error().decode()
        assert fn(images=fake + 2) != 0 and "RGBA images need 4 bytes" in lib.hr_last_error().decode()
