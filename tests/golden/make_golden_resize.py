"""Golden frames of the datasets' image resize, from the unmodified reference ``get_rgb`` run on CPU through the shim on
stand-in dataset objects.

    HYPERREEL_REFERENCE=<reference checkout> python tests/golden/make_golden_resize.py

writes ``tests/golden/resize.npz``, per case ``<case>/...``:

* ``frames`` uint8 [n, H0, W0, 3]: seeded RGB frames at the stand-in capture size;
* ``rgb`` fp32 [n, H * W, 3]: what ``get_rgb`` returns for each frame (after ``T.ToTensor()``);
* ``meta`` JSON: the dataset ``name``, the class and the ``_img_wh`` / ``img_wh`` set on the object (``img_wh`` differs
  when the reference's ``scale()`` reduced it).

The Pillow datasets (technicolor, llff, spaces, and the three stanford classes) read their image through ``self.pmgr.open``:
the stand-in serves the frame as a lossless PNG, which ``Image.open(...).convert("RGB")`` decodes to the same pixels.  The
OpenCV datasets (neural_3d, immersive) take the decoded frame as an argument; it is passed as BGR, as ``cv2.VideoCapture``
returns it.  The capture sizes are small but keep the shipped ratios (exactly 2x for neural_3d and immersive, 8x for llff)
and add non-integer ratios, odd and prime sizes, and the identity.
"""
import contextlib
import io
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from tests.golden.make_golden_subsample import _install  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))

# name: (dataset name, module, class, capture (W0, H0), _img_wh, scale, frames)
CASES = {
    "technicolor_2x_s2": ("technicolor", "technicolor", "TechnicolorDataset", (64, 34), (32, 17), 2, 2),
    "technicolor_same": ("technicolor", "technicolor", "TechnicolorDataset", (40, 30), (40, 30), 1, 1),
    "technicolor_odd": ("technicolor", "technicolor", "TechnicolorDataset", (53, 37), (29, 21), 1, 2),
    "llff_8x": ("llff", "llff", "LLFFDataset", (96, 72), (12, 9), 1, 2),
    "llff_odd_s2": ("llff", "llff", "LLFFDataset", (53, 37), (29, 21), 2, 1),
    "spaces_8_3": ("spaces", "spaces", "SpacesDataset", (80, 48), (30, 18), 1, 2),
    "stanford_4x_s4": ("stanford", "stanford", "StanfordLightfieldDataset", (64, 64), (16, 16), 4, 2),
    "stanford_epi_prime": ("stanford_epi", "stanford", "StanfordEPIDataset", (61, 43), (17, 11), 1, 1),
    "stanford_llff_same_s3": ("stanford_llff", "stanford", "StanfordLLFFDataset", (48, 36), (48, 36), 3, 1),
    "neural3d_2x": ("neural_3d", "neural_3d", "Neural3DVideoDataset", (54, 40), (27, 20), 1, 2),
    "neural3d_2x_s2": ("neural_3d", "neural_3d", "Neural3DVideoDataset", (54, 40), (27, 20), 2, 2),
    "neural3d_same": ("neural_3d", "neural_3d", "Neural3DVideoDataset", (27, 20), (27, 20), 1, 1),
    "neural3d_odd_s2": ("neural_3d", "neural_3d", "Neural3DVideoDataset", (45, 31), (20, 14), 2, 2),
    "immersive_2x_s2": ("immersive", "immersive", "ImmersiveDataset", (64, 48), (32, 24), 2, 2),
    "immersive_8x_s3": ("immersive", "immersive", "ImmersiveDataset", (64, 48), (8, 6), 3, 1),
    "immersive_3x": ("immersive", "immersive", "ImmersiveDataset", (45, 33), (15, 11), 1, 1),
    "immersive_prime": ("immersive", "immersive", "ImmersiveDataset", (43, 29), (41, 23), 1, 1),
}


def frames_for(name, W0, H0, n):
    """Seeded frames with smooth gradients, edges and noise, so every filter tap and both clips are exercised."""
    rng = np.random.default_rng(sum(map(ord, name)))
    y, x = np.mgrid[0:H0, 0:W0]
    out = []
    for i in range(n):
        base = np.stack([x * 255.0 / max(W0 - 1, 1), y * 255.0 / max(H0 - 1, 1), ((x + y + 7 * i) % 9) * 31.0], -1)
        noise = rng.integers(-60, 61, (H0, W0, 3))
        edge = np.where(((x // 5 + y // 3 + i) % 2 == 0)[..., None], 255, 0)
        img = np.where(rng.random((H0, W0, 1)) < 0.3, edge, base + noise)
        out.append(np.clip(img, 0, 255).astype(np.uint8))
    return np.stack(out)


class _Files:
    """The stand-in path manager: open() serves the frame set on it as a PNG."""

    def __init__(self):
        self.png = b""

    @contextlib.contextmanager
    def open(self, path, mode="rb"):
        yield io.BytesIO(self.png)


def reference_rgb(module, cls_name, frames, img_wh0, scale):
    import importlib

    import torchvision.transforms as T
    from PIL import Image

    cls = getattr(importlib.import_module(f"datasets.{module}"), cls_name)
    ds = object.__new__(cls)
    ds._img_wh = tuple(img_wh0)
    ds.img_wh = (img_wh0[0] // scale, img_wh0[1] // scale)  # BaseDataset.scale
    ds.transform = T.ToTensor()
    ds.root_dir = ""
    ds.image_paths = ["frame.png"]
    ds.cols = 1
    ds.pmgr = _Files()
    out = []
    for f in frames:
        if module in ("neural_3d", "immersive"):
            rgb = ds.get_rgb(np.ascontiguousarray(f[..., ::-1]))  # BGR, as cv2 decodes it
        else:
            buf = io.BytesIO()
            Image.fromarray(f).save(buf, format="PNG")
            ds.pmgr.png = buf.getvalue()
            rgb = ds.get_rgb(0, 0) if cls_name == "StanfordLightfieldDataset" else \
                ds.get_rgb() if cls_name == "StanfordEPIDataset" else ds.get_rgb(0)
        out.append(rgb.numpy())
    return np.stack(out).astype(np.float32), ds.img_wh


def main():
    _install()
    out = {}
    for case, (name, module, cls_name, (W0, H0), img_wh0, scale, n) in CASES.items():
        frames = frames_for(case, W0, H0, n)
        with contextlib.redirect_stdout(io.StringIO()):
            rgb, img_wh = reference_rgb(module, cls_name, frames, img_wh0, scale)
        assert rgb.shape == (n, img_wh[0] * img_wh[1], 3), (case, rgb.shape)
        out[f"{case}/frames"] = frames
        out[f"{case}/rgb"] = rgb
        out[f"{case}/meta"] = np.array(json.dumps(dict(name=name, cls=cls_name, img_wh=list(img_wh0), scale=scale,
                                                       out_wh=list(img_wh))))
        print(case, frames.shape, "->", img_wh)
    np.savez_compressed(os.path.join(OUT, "resize.npz"), **out)


if __name__ == "__main__":
    main()
