"""dataset_cameras against the reference's dataset classes (tests/golden/dataset_cameras.npz, made by
make_golden_dataset_cameras.py from the unmodified read_meta / split selection / get_coords on synthetic scene
directories): every split's cameras field by field, their ground-truth sources and the dataset facts, the facts lowering
as the reference's do, and the refusals."""
import copy
import json
import os

import numpy as np
import pytest

import hyperreel_b200 as hb
from hyperreel_b200 import configs

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dataset_cameras.npz")
SPLITS = ("train", "val", "test", "render")
# the reference projects Immersive render views to NDC with the unscaled focal, the ray record with its own (K * 0.75)
REFUSED = {("immersive_ndc", "render"): "'use_ndc'"}


def _golden():
    return np.load(GOLDEN)


def _cases():
    return sorted({k.split("/")[0] for k in _golden().files})


def make_scene(z, case, root):
    """Writes the case's synthetic scene directory under ``root``; returns (root, dataset config)."""
    spec = json.loads(str(z[f"{case}/scene"]))
    for rel, text in spec["files"].items():
        with open(os.path.join(root, rel), "w") as f:
            f.write(text)
    for rel in spec["empty"]:
        os.makedirs(os.path.dirname(os.path.join(root, rel)), exist_ok=True)
        open(os.path.join(root, rel), "wb").close()
    for rel in spec["npy"]:
        np.save(os.path.join(root, rel), z[f"{case}/npy/{rel}"])
    return str(root), json.loads(str(z[f"{case}/cfg"]))


@pytest.mark.parametrize("split", SPLITS)
@pytest.mark.parametrize("case", _cases())
def test_cameras_equal_the_reference(case, split, tmp_path):
    z = _golden()
    root, cfg = make_scene(z, case, tmp_path)
    if (case, split) in REFUSED:
        return _refused(cfg, root, split, REFUSED[case, split])
    views = hb.dataset_cameras(cfg, root, split)
    g = {k: z[f"{case}/{split}/{k}"] for k in ("poses", "K", "times", "cam_idx", "distortion")}
    cams = views.cameras
    assert len(cams) == len(g["poses"])
    W, H = cfg["img_wh"]
    for i, c in enumerate(cams):
        assert np.asarray(c.pose).dtype == np.float32 and np.asarray(c.K).dtype == np.float32
        assert np.array_equal(np.asarray(c.pose), g["poses"][i]), i
        assert np.array_equal(np.asarray(c.K), g["K"][i]), i
        assert c.time == float(g["times"][i]) and c.cam_idx == float(g["cam_idx"][i]), i
        assert (c.width, c.height) == (W, H) and c.centered_pixels and not c.flipped and c.normalize
        assert c.use_ndc == bool(cfg["use_ndc"])
        if c.use_ndc:
            assert c.ndc_near == float(np.float32(views.facts["near"]))
        if cfg["name"] == "immersive" and split != "render":
            assert c._distortion_f32() == tuple(float(v) for v in g["distortion"][i])
        else:
            assert c.distortion is None
    frames = json.loads(str(z[f"{case}/{split}/frames"]))
    assert [(os.path.relpath(f.path, root), f.frame) for f in views.frames] == [(p, f) for p, f in frames]
    assert views.rgba == (cfg["name"] == "donerf")
    assert np.array_equal(views.times, g["times"])


@pytest.mark.parametrize("case", _cases())
def test_facts_equal_the_reference_training_dataset(case, tmp_path):
    z = _golden()
    root, cfg = make_scene(z, case, tmp_path)
    ref = json.loads(str(z[f"{case}/facts"]))
    ref.update({"name": cfg["name"], "collection": cfg["collection"]})
    for split in SPLITS:
        if (case, split) not in REFUSED:
            assert hb.dataset_cameras(cfg, root, split).facts == ref


def _model(name):
    if name == "immersive":
        g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "shipped", "immersive_sphere.npz"))
        return hb.to_cfg(json.loads(str(g["config_json"])))
    return configs.get({"technicolor": "technicolor_z_plane", "neural_3d": "neural_3d_z_plane",
                        "donerf": "donerf_sphere"}[name])[0]


def _lowered(sig):
    return (bytes(sig.cfg), sig.head_names, sig.head_channels, sig.mlp_layer_shapes, sig.in_perm, sig.color_views,
            sig.cascade, sig.graph_iters)


@pytest.mark.parametrize("case", _cases())
def test_facts_lower_as_the_reference_facts(case, tmp_path):
    z = _golden()
    root, cfg = make_scene(z, case, tmp_path)
    ref = json.loads(str(z[f"{case}/facts"]))
    ref.update({"name": cfg["name"], "collection": cfg["collection"]})
    model = _model(cfg["name"])
    facts = hb.dataset_cameras(cfg, root, "train").facts
    assert _lowered(hb.lower(copy.deepcopy(model), facts)) == _lowered(hb.lower(copy.deepcopy(model), ref))


def test_birthday_substitutes_the_broken_view(tmp_path):
    z = _golden()
    root, cfg = make_scene(z, "technicolor_birthday", tmp_path)
    views = hb.dataset_cameras(cfg, root, "train")
    by_source = {os.path.basename(f.path): c for f, c in zip(views.frames, views.cameras)}
    names = sorted(os.listdir(os.path.join(root, "images")))
    assert names[377] not in by_source  # view 377 reads view 361's file, pose and time
    assert sum(os.path.basename(f.path) == names[361] for f in views.frames) == 2


def test_render_crop_window(tmp_path):
    z = _golden()
    root, cfg = make_scene(z, "neural_3d_ndc", tmp_path)
    W, H = cfg["img_wh"]
    views = hb.dataset_cameras(cfg, root, "render")
    dW, dH = int(W // 2 * 0.85), int(H // 2 * 0.85)
    assert views.crop == (H // 2 - dH, H // 2 + dH + 1, W // 2 - dW, W // 2 + dW + 1)
    assert hb.dataset_cameras(cfg, root, "val").crop is None


def _refused(cfg, root, split, key):
    with pytest.raises(hb.UnsupportedPipeline, match=key):
        hb.dataset_cameras(cfg, root, split)


def test_refusals_name_the_key(tmp_path):
    z = _golden()
    roots = {}
    for case in ("technicolor_skip", "neural_3d_ndc", "immersive_correct", "donerf_center"):
        d = tmp_path / case
        d.mkdir()
        roots[case] = make_scene(z, case, d)
    root, tc = roots["technicolor_skip"]
    for other in ("llff", "shiny", "spaces", "catacaustics", "bom", "blender", None):
        _refused(dict(tc, name=other), root, "train", "'name'")
    _refused(tc, root, "validation", "'split'")
    _refused(dict(tc, train={"val_all": True}), root, "train", "'train'")
    _refused(dict(tc, img_wh=None), root, "train", "'img_wh'")
    _refused(dict(tc, val_crop=0.5), root, "val", "'val_crop'")
    _refused(dict(tc, val_set="odd"), root, "val", "'val_set'")
    _refused(dict(tc, val_skip="inf"), root, "val", "'split'")  # nothing held out
    _refused(dict(tc, use_ndc=True), root, "train", "'use_ndc'")  # focal lengths differ per camera
    root, n3 = roots["neural_3d_ndc"]
    _refused(dict(n3, val_all=True), root, "train", "'val_all'")
    _refused(dict(n3, val_set=[0, 1]), root, "val", "'val_set'")
    _refused(dict(n3, val_set=[]), root, "test", "'split'")
    root, im = roots["immersive_correct"]
    _refused(dict(im, use_ndc=True), root, "train", "'use_ndc'")
    _refused(dict(im, val_all=True), root, "val", "'val_all'")
    root, dn = roots["donerf_center"]
    _refused(dict(dn, val_num=0), root, "val", "'split'")
    assert len(hb.dataset_cameras(dn, root, "val").cameras) == 3


def test_malformed_scene_files_raise(tmp_path):
    z = _golden()
    root, tc = make_scene(z, "technicolor_skip", tmp_path)
    os.remove(os.path.join(root, "images", sorted(os.listdir(os.path.join(root, "images")))[-1]))
    with pytest.raises(ValueError, match="whole frames"):
        hb.dataset_cameras(tc, root, "train")
    d = tmp_path / "n3"
    d.mkdir()
    root, n3 = make_scene(z, "neural_3d_ndc", d)
    open(os.path.join(root, "extra.mp4"), "wb").close()
    with pytest.raises(ValueError, match="poses_bounds"):
        hb.dataset_cameras(n3, root, "train")
