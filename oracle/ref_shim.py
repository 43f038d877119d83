"""Reference-through-shim runner (TEST INFRASTRUCTURE ONLY -- never imported by the product).

Imports the *unmodified* HyperReel hot-path modules from a reference checkout (``$HYPERREEL_REFERENCE``) on CPU so that their
outputs can pin the oracle (``oracle/hyperreel_oracle.py``) and generate the golden vectors under
``tests/golden/``.  It only works where that checkout exists; the tests read the recorded vectors and
never call into it.

What the shim does (SURVEY.md Appendix D):
  * registers an empty namespace package ``nlf`` whose ``__path__`` points at the reference, so the
    sub-modules import without running ``nlf/__init__.py`` (which needs pytorch_lightning, iopath,
    omegaconf, ... -- all absent here);
  * stubs the four third-party modules that are imported but never called on the render path
    (kornia, plyfile, skimage.measure, pytorch3d.transforms);
  * maps every hard-coded ``'cuda'`` device to ``'cpu'`` (``nlf/nets/tensorf_base.py:143``,
    ``nlf/intersect/base.py:85`` ...);
  * builds the model from an attribute-access dict standing in for OmegaConf's ``DictConfig`` after
    applying the ``*_epoch(s) -> *_iter(s)`` rewrite of ``nlf/__init__.py:306-315``.
"""
from __future__ import annotations

import contextlib
import io
import os
import sys
import types
from types import SimpleNamespace

import torch

REFERENCE_ROOT = os.environ.get("HYPERREEL_REFERENCE", "")


def reference_available() -> bool:
    return os.path.isdir(os.path.join(REFERENCE_ROOT, "nlf"))


class AttrDict(dict):
    """dict with attribute access: the subset of DictConfig behaviour the reference code uses
    (``'k' in cfg``, ``cfg.k``, ``cfg['k']``, item assignment, ``.keys()``, ``getattr(cfg, k, d)``)."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:  # pragma: no cover - mirrors DictConfig raising on a missing key
            raise AttributeError(k) from e

    def __setattr__(self, k, v):
        self[k] = v


def to_attr(o):
    if isinstance(o, dict):
        return AttrDict({k: to_attr(v) for k, v in o.items()})
    if isinstance(o, (list, tuple)):
        return [to_attr(v) for v in o]
    return o


_EPOCH_KEYS = ["max_freq", "wait", "stop", "falloff", "window", "no_bias", "window_bias",
               "window_bias_start", "decay", "warmup"]


def epochs_to_iters(cfg, iters_per_epoch: int):
    """``INRSystem.__init__`` rewrite (nlf/__init__.py:306-315, utils/config_utils.py:32-38)."""
    if isinstance(cfg, dict):
        for key in list(cfg.keys()):
            hit = False
            for base in _EPOCH_KEYS:
                if key in (f"{base}_epoch", f"{base}_epochs"):
                    v = cfg[key]
                    if isinstance(v, list):
                        cfg[key.replace("epoch", "iter")] = [[x * iters_per_epoch for x in li] for li in v]
                    else:
                        cfg[key.replace("epoch", "iter")] = v * iters_per_epoch
                    hit = True
            if not hit:
                epochs_to_iters(cfg[key], iters_per_epoch)
    elif isinstance(cfg, list):
        for v in cfg:
            epochs_to_iters(v, iters_per_epoch)
    return cfg


_INSTALLED = False


def install():
    """Idempotently install the import shim + the cuda->cpu rewrite."""
    global _INSTALLED
    if _INSTALLED:
        return
    if not reference_available():
        raise RuntimeError(f"reference checkout not found at {REFERENCE_ROOT}")
    if REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, REFERENCE_ROOT)

    nlf = types.ModuleType("nlf")
    nlf.__path__ = [os.path.join(REFERENCE_ROOT, "nlf")]
    sys.modules["nlf"] = nlf

    def stub(name, **attrs):
        m = types.ModuleType(name)
        for k, v in attrs.items():
            setattr(m, k, v)
        sys.modules[name] = m
        return m

    if "kornia" not in sys.modules:
        def create_meshgrid(height, width, normalized_coordinates=True, device="cpu", dtype=torch.float32):
            # functional stand-in for kornia.utils.create_meshgrid (pixel-coordinate form only): [1, H, W, 2] = (x, y)
            assert not normalized_coordinates
            xs = torch.linspace(0, width - 1, width, dtype=dtype)
            ys = torch.linspace(0, height - 1, height, dtype=dtype)
            gy, gx = torch.meshgrid(ys, xs, indexing="ij")
            return torch.stack([gx, gy], -1)[None]

        stub("kornia", create_meshgrid=create_meshgrid)
    if "plyfile" not in sys.modules:
        stub("plyfile", PlyData=None, PlyElement=None)
    if "skimage" not in sys.modules:
        sk = stub("skimage")
        sk.measure = stub("skimage.measure")
    if "pytorch3d" not in sys.modules:
        p3 = stub("pytorch3d")
        p3.transforms = stub("pytorch3d.transforms")

    if not torch.cuda.is_available():
        ident = lambda self, *a, **k: self
        torch.Tensor.cuda = ident
        torch.nn.Module.cuda = ident

        def fix_dev(kwargs):
            d = kwargs.get("device", None)
            if d is not None and "cuda" in str(d):
                kwargs["device"] = "cpu"
            return kwargs

        for name in ["tensor", "linspace", "zeros", "ones", "randn", "rand", "empty", "full",
                     "arange", "eye", "zeros_like", "ones_like"]:
            orig = getattr(torch, name)

            def wrapped(*a, __orig=orig, **k):
                return __orig(*a, **fix_dev(k))

            setattr(torch, name, wrapped)

        def wrap_to(orig):
            def to(self, *a, **k):
                a = tuple("cpu" if (isinstance(x, (str, torch.device)) and "cuda" in str(x)) else x for x in a)
                return orig(self, *a, **fix_dev(k))
            return to

        torch.Tensor.to = wrap_to(torch.Tensor.to)
        torch.nn.Module.to = wrap_to(torch.nn.Module.to)
    _INSTALLED = True


def make_system(dataset: dict):
    """Stand-in for the LightningModule handed to constructors as ``system=`` (they read
    ``system.dm.train_dataset.{num_keyframes,num_frames,near,far,depth_range}`` and
    ``system.cfg.dataset.{collection,name}``: tensorf_dynamic.py:49-50, tensorf_no_sample.py:41-45,
    contract.py:121-125, primitive.py:371-373)."""
    ds = SimpleNamespace(
        num_keyframes=dataset.get("num_keyframes", 1),
        num_frames=dataset.get("num_frames", 1),
        near=dataset.get("near", 0.0),
        far=dataset.get("far", 1.0),
        depth_range=dataset.get("depth_range", [dataset.get("near", 0.0), dataset.get("far", 1.0)]),
    )
    for k in ("bbox_min", "bbox_max", "total_images_per_frame", "val_all"):  # voxel.py:27-29, point.py:574-575
        if k in dataset:
            v = dataset[k]
            setattr(ds, k, torch.tensor(v) if k.startswith("bbox") else v)
    cfg = to_attr({"dataset": {"collection": dataset.get("collection", "synthetic"),
                               "name": dataset.get("name", "synthetic")}})
    return SimpleNamespace(dm=SimpleNamespace(train_dataset=ds), cfg=cfg)


def build_reference(model_cfg: dict, dataset: dict, iters_per_epoch: int = 4000, net_chunk: int = 1 << 30,
                    quiet: bool = True):
    """Build ``RenderLightfield(LightfieldModel(cfg))`` from the unmodified reference classes.

    ``model_cfg`` is a plain dict in the schema of ``conf/experiment/model/*.yaml`` (it is deep-copied:
    reference constructors mutate their cfg, e.g. nlf/embedding/ray.py:283-285)."""
    import copy

    install()
    cfg = to_attr(epochs_to_iters(copy.deepcopy(model_cfg), iters_per_epoch))
    system = make_system(dataset)
    sink = io.StringIO()
    with (contextlib.redirect_stdout(sink) if quiet else contextlib.nullcontext()):
        from nlf.models.models import model_dict
        from nlf.rendering import render_fn_dict

        model = model_dict[cfg.type](cfg, system=system)
        render = render_fn_dict[cfg.render.type](model, None, cfg.render, net_chunk=net_chunk)
    render.eval()
    model.set_iter(10_000_000)
    return render


def load_reference_yaml(name: str) -> dict:
    import yaml

    with open(os.path.join(REFERENCE_ROOT, "conf/experiment/model", name + ".yaml")) as f:
        return yaml.safe_load(f)


@torch.no_grad()
def run_reference(render, rays: torch.Tensor, chunk: int | None = None, capture: bool = False):
    """``render_chunked`` (nlf/rendering.py:100-150) on CPU.  With ``capture=True`` also returns the
    embedding dict ``x`` (points / distances / heads ...) via ``render.embed``."""
    install()
    from nlf.rendering import render_chunked

    chunk = chunk or rays.shape[0]
    out = {k: v for k, v in render_chunked(rays, render, {}, chunk).items()}
    if capture:
        emb = render.embed(rays.clone())
        out["_embed"] = {k: v for k, v in emb.items()}
    return out
