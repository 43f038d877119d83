"""Golden frames of the RGBA datasets' get_rgb (DoNeRF, Catacaustics), from the unmodified reference ``get_rgb`` run on CPU
through the shim on stand-in dataset objects.

    HYPERREEL_REFERENCE=<reference checkout> python tests/golden/make_golden_rgba.py

writes ``tests/golden/rgba.npz``, per case ``<case>/...``:

* ``frames`` uint8 [n, H0, W0, 4]: seeded RGBA frames at the stand-in capture size, alpha 0, 255 and in between;
* ``rgb`` fp32 [n, H * W, 3]: what ``get_rgb`` returns for each frame (the resize, ``T.ToTensor()``, the composite over
  white);
* ``meta`` JSON: the dataset ``name``, the class, ``img_wh`` (the ``_img_wh`` set on the object), ``scale`` and ``out_wh``
  (``img_wh``, reduced when the reference's ``scale()`` reduced it).

Both classes read their image through ``self.pmgr.open``: the stand-in serves the frame as a lossless RGBA PNG, which
``Image.open(...).convert("RGBA")`` decodes to the same pixels.  The cases cover the identity, exact 2x and 3x reductions,
non-integer ratios, odd and prime sizes, one axis kept, and a second resize after ``scale()``.  DoNeRF's INTER_AREA runs at
integer factors only (OpenCV's float INTER_AREA path is not restated).
"""
import contextlib
import io
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from tests.golden.make_golden_resize import _Files  # noqa: E402
from tests.golden.make_golden_subsample import _install  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))

# name: (dataset name, module, class, capture (W0, H0), _img_wh, scale, frames)
CASES = {
    "donerf_same": ("donerf", "donerf", "DONeRFDataset", (40, 30), (40, 30), 1, 2),
    "donerf_2x": ("donerf", "donerf", "DONeRFDataset", (64, 48), (32, 24), 1, 2),
    "donerf_2x_s2": ("donerf", "donerf", "DONeRFDataset", (64, 48), (32, 24), 2, 1),
    "donerf_3x_odd": ("donerf", "donerf", "DONeRFDataset", (45, 33), (15, 11), 1, 2),
    "donerf_same_s2": ("donerf", "donerf", "DONeRFDataset", (50, 38), (50, 38), 2, 1),
    "catacaustics_same": ("catacaustics", "catacaustics", "CatacausticsDataset", (40, 30), (40, 30), 1, 1),
    "catacaustics_2x_s2": ("catacaustics", "catacaustics", "CatacausticsDataset", (64, 48), (32, 24), 2, 2),
    "catacaustics_odd": ("catacaustics", "catacaustics", "CatacausticsDataset", (53, 37), (29, 21), 1, 2),
    "catacaustics_prime": ("catacaustics", "catacaustics", "CatacausticsDataset", (61, 43), (17, 11), 1, 1),
    "catacaustics_one_axis": ("catacaustics", "catacaustics", "CatacausticsDataset", (48, 40), (48, 23), 1, 1),
    "catacaustics_same_s3": ("catacaustics", "catacaustics", "CatacausticsDataset", (48, 36), (48, 36), 3, 1),
    "catacaustics_3_7_s2": ("catacaustics", "catacaustics", "CatacausticsDataset", (97, 61), (41, 26), 2, 1),
}


def frames_for(name, W0, H0, n):
    """Seeded RGBA frames: colour gradients, edges and noise; alpha transparent, opaque and in between (smooth ramps,
    hard edges and noise), so premultiply, unpremultiply and both clips are exercised."""
    rng = np.random.default_rng(sum(map(ord, name)))
    y, x = np.mgrid[0:H0, 0:W0]
    out = []
    for i in range(n):
        base = np.stack([x * 255.0 / max(W0 - 1, 1), y * 255.0 / max(H0 - 1, 1), ((x + y + 7 * i) % 9) * 31.0], -1)
        noise = rng.integers(-60, 61, (H0, W0, 3))
        edge = np.where(((x // 5 + y // 3 + i) % 2 == 0)[..., None], 255, 0)
        rgb = np.where(rng.random((H0, W0, 1)) < 0.3, edge, base + noise)
        ramp = (x + 2 * y + 13 * i) * 255.0 / max(W0 + 2 * H0, 1)
        alpha = np.where(rng.random((H0, W0)) < 0.5, ramp + rng.integers(-40, 41, (H0, W0)),
                         np.where((x // 4 + y // 4 + i) % 3 == 0, 0, 255))
        img = np.concatenate([rgb, alpha[..., None]], -1)
        out.append(np.clip(img, 0, 255).astype(np.uint8))
    return np.stack(out)


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
    ds.image_paths = ["frame"]
    ds.pmgr = _Files()
    out = []
    for f in frames:
        buf = io.BytesIO()
        Image.fromarray(f, "RGBA").save(buf, format="PNG")
        ds.pmgr.png = buf.getvalue()
        out.append(ds.get_rgb(0).numpy())
    return np.stack(out).astype(np.float32), ds.img_wh


def main():
    _install()
    out = {}
    for case, (name, module, cls_name, (W0, H0), img_wh0, scale, n) in CASES.items():
        frames = frames_for(case, W0, H0, n)
        alpha = frames[..., 3]
        assert (alpha == 0).any() and (alpha == 255).any() and ((alpha > 0) & (alpha < 255)).any(), case
        with contextlib.redirect_stdout(io.StringIO()):
            rgb, img_wh = reference_rgb(module, cls_name, frames, img_wh0, scale)
        assert rgb.shape == (n, img_wh[0] * img_wh[1], 3), (case, rgb.shape)
        out[f"{case}/frames"] = frames
        out[f"{case}/rgb"] = rgb
        out[f"{case}/meta"] = np.array(json.dumps(dict(name=name, cls=cls_name, img_wh=list(img_wh0), scale=scale,
                                                       out_wh=list(img_wh))))
        print(case, frames.shape, "->", img_wh)
    np.savez_compressed(os.path.join(OUT, "rgba.npz"), **out)


if __name__ == "__main__":
    main()
