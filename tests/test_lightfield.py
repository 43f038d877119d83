"""Two-plane light-field views (the Stanford dataset) on the host: the NumPy oracle against the reference's rays, the view
lists of ``lightfield_cameras`` / ``stanford_file_coords`` against the reference's, and ``TwoPlaneCamera``'s checks.
The fixtures come from tests/golden/make_golden_lightfield.py."""
import json
import os

import numpy as np
import pytest

import hyperreel_b200 as hb
from tests.lightfield_oracle import camera_rays, lightfield_rays

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
RAYS = np.load(os.path.join(GOLDEN, "lightfield_rays.npz"))
VIEWS = np.load(os.path.join(GOLDEN, "lightfield_views.npz"))
RAY_CASES = sorted({k.split("/")[0] for k in RAYS.files})
VIEW_CASES = sorted({k.split("/")[0] for k in VIEWS.files})


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def view_case(name):
    cfg = json.loads(str(VIEWS[f"{name}/config"]))
    files = [f for f in VIEWS[f"{name}/files"].tolist() if f]
    return cfg, str(VIEWS[f"{name}/split"]), files


def cameras_of(name):
    cfg, split, files = view_case(name)
    W, H = cfg["img_wh"]
    fc = hb.stanford_file_coords(files, cfg["collection"]) if cfg["lightfield"].get("use_file_coords") else None
    return hb.lightfield_cameras(cfg, W, H, split, file_coords=fc if split != "render" else None)


@pytest.mark.parametrize("name", RAY_CASES)
def test_oracle_equals_reference_rays(name):
    W, H, s, t, st, uv, near, far, aspect = RAYS[f"{name}/params"]
    got = lightfield_rays(int(W), int(H), s, t, st, uv, near, far, aspect, RAYS[f"{name}/pixels"])
    np.testing.assert_array_equal(bits(got), bits(RAYS[f"{name}/rays"]))


@pytest.mark.parametrize("name", RAY_CASES)
def test_camera_oracle_equals_reference_rays(name):
    W, H, s, t, st, uv, near, far, aspect = RAYS[f"{name}/params"]
    cam = hb.TwoPlaneCamera(int(W), int(H), s, t, st_scale=st, uv_scale=uv, near=near, far=far, aspect=aspect,
                            time=0.5, cam_idx=3)
    got = camera_rays(cam, RAYS[f"{name}/pixels"])
    np.testing.assert_array_equal(bits(got[:, :6]), bits(RAYS[f"{name}/rays"]))
    assert (got[:, 6] == 3).all() and (got[:, 7] == 0.5).all()


@pytest.mark.parametrize("name", VIEW_CASES)
def test_views_equal_reference(name):
    cams = cameras_of(name)
    pos, scales, rays = VIEWS[f"{name}/pos"], VIEWS[f"{name}/scales"], VIEWS[f"{name}/rays"]
    assert len(cams) == pos.shape[0] == rays.shape[0]
    for i, cam in enumerate(cams):
        assert (np.float32(cam.s), np.float32(cam.t)) == (np.float32(pos[i, 0]), np.float32(pos[i, 1])), i
        assert (np.float32(cam.st_scale), np.float32(cam.uv_scale)) == tuple(np.float32(scales[i])), i
        np.testing.assert_array_equal(bits(camera_rays(cam)[:, :6]), bits(rays[i]), err_msg=f"view {i}")


def test_view_positions_are_the_references_doubles():
    """The positions are computed in double as the reference computes them, before any rounding."""
    for name in VIEW_CASES:
        cams = cameras_of(name)
        np.testing.assert_array_equal(np.array([[c.s, c.t] for c in cams], np.float64), VIEWS[f"{name}/pos"])


@pytest.mark.parametrize("name", ["render_far_files", "val_files", "test_files_tarot"])
def test_stanford_file_coords_equal_read_meta(name):
    cfg, _, files = view_case(name)
    got = np.array(hb.stanford_file_coords(list(reversed(files)), cfg["collection"]), np.float64)
    np.testing.assert_array_equal(got, VIEWS[f"{name}/file_coords"])


def test_render_split_counts():
    assert len(cameras_of("render_spiral")) == 120
    cfg, _, _ = view_case("render_sweep")
    sweep = cameras_of("render_sweep")
    assert len(sweep) == cfg["lightfield"]["cols"] * cfg["lightfield"]["supersample"]
    assert any(c.s != round(c.s, 1) for c in sweep)  # fractional s_idx between the grid columns


def test_train_order_restates_the_loop():
    """The training views: rows range(start_row, end_row, step), columns likewise, val_pairs skipped (the loop of
    prepare_train_data above its exit(), which the reference never gets past)."""
    cfg = dict(name="stanford", img_wh=[6, 4], val_num=8, val_pairs=[2, 0, 4, 4],
               render_params=dict(supersample=4), lightfield=dict(rows=5, cols=5, step=2, supersample=2, disp_row=2,
                                                                   st_scale=0.25, uv_scale=0.5, start_col=0, end_col=5))
    cams = hb.lightfield_cameras(cfg, 6, 4, "train")
    st = [(s, t) for t in range(0, 5, 2) for s in range(0, 5, 2) if (s, t) not in [(2, 0), (4, 4)]]
    assert [(c.s, c.t) for c in cams] == [((s / 4) * 2 - 1, -((t / 4) * 2 - 1)) for s, t in st]
    assert all(c.st_scale == 0.25 and c.uv_scale == 0.5 and c.aspect == 1.5 for c in cams)


def test_train_views_with_file_coords():
    files = [f"out_{r:02d}_{c:02d}_{100.0 * r:.1f}_{-50.0 * c:.1f}_.png" for r in range(3) for c in range(3)]
    fc = hb.stanford_file_coords(files, "gem")
    assert fc[4] == (-50.0, 100.0)
    cfg = dict(name="stanford", img_wh=[4, 4], val_num=8, val_pairs=[], render_params=dict(supersample=4),
               lightfield=dict(rows=3, cols=3, step=2, supersample=1, disp_row=1, use_file_coords=True))
    cams = hb.lightfield_cameras(cfg, 4, 4, "train", file_coords=fc)
    # views (0, 0), (2, 0), (0, 2), (2, 2); x in [-100, 0], y in [0, 200], aspect 0.5
    assert [(c.s, c.t) for c in cams] == [(1.0, -2.0), (-1.0, -2.0), (1.0, 2.0), (-1.0, 2.0)]
    with pytest.raises(ValueError, match="file_coords"):
        hb.lightfield_cameras(cfg, 4, 4, "train")
    cfg["lightfield"]["use_file_coords"] = False
    with pytest.raises(ValueError, match="use_file_coords"):
        hb.lightfield_cameras(cfg, 4, 4, "train", file_coords=fc)


def test_keyframe_subsample_refused():
    cfg = dict(name="stanford", img_wh=[4, 4], val_num=8, render_params=dict(supersample=4),
               lightfield=dict(rows=3, cols=3, step=1, supersample=1, disp_row=1, keyframe_step=2, keyframe_subsample=4))
    with pytest.raises(ValueError, match="keyframe_subsample"):
        hb.lightfield_cameras(cfg, 4, 4, "train")
    cfg["lightfield"]["keyframe_subsample"] = 1  # what the shipped configs set
    assert len(hb.lightfield_cameras(cfg, 4, 4, "train")) == 9


def test_bad_arguments_refused():
    cfg = dict(name="stanford", img_wh=[4, 4], val_num=8, render_params=dict(supersample=4),
               lightfield=dict(rows=3, cols=3, step=1, supersample=1, disp_row=1))
    with pytest.raises(ValueError, match="split"):
        hb.lightfield_cameras(cfg, 4, 4, "training")
    with pytest.raises(ValueError, match="stanford"):
        hb.lightfield_cameras(dict(cfg, name="stanford_epi"), 4, 4, "train")
    with pytest.raises(ValueError, match="camera position"):
        hb.stanford_file_coords(["a.png"], "gem")


@pytest.mark.parametrize("kw, match", [
    (dict(s=float("nan")), "s ="), (dict(t=float("inf")), "t ="), (dict(st_scale=1e39), "st_scale"),
    (dict(uv_scale=-float("inf")), "uv_scale"), (dict(near=float("nan")), "near"), (dict(far=1e40), "far"),
    (dict(aspect=1e-50), "aspect"), (dict(aspect=0.0), "aspect"), (dict(time=float("nan")), "time"),
    (dict(near=-1.1, far=0.3), "far - near"), (dict(width=0), "size"),
])
def test_two_plane_camera_validation(kw, match):
    args = dict(width=8, height=6, s=0.1, t=-0.2)
    args.update(kw)
    with pytest.raises(ValueError, match=match):
        hb.TwoPlaneCamera(**args)


def test_to_c_fields():
    cam = hb.TwoPlaneCamera(37, 23, s=0.1, t=-1.0 / 3.0, st_scale=0.125, uv_scale=0.7, near=-1.5, far=0.25, time=0.25,
                            cam_idx=4)
    c = cam.to_c()
    f32 = lambda v: float(np.float32(v))  # noqa: E731
    assert (c.width, c.height, c.two_plane, c.fisheye) == (37, 23, 1, 0)
    assert (c.lf_s, c.lf_t, c.lf_st_scale, c.lf_uv_scale) == (f32(0.1), f32(-1.0 / 3.0), 0.125, f32(0.7))
    assert (c.lf_near, c.lf_far, c.lf_aspect) == (-1.5, 0.25, f32(37 / 23))
    assert (c.time, c.cam_idx) == (0.25, 4.0)
    assert list(c.c2w) == [0.0] * 12 and (c.fx, c.use_ndc, c.normalize) == (0.0, 0, 0)
    assert hb.TwoPlaneCamera(8, 6, 0, 0, aspect=2.5).to_c().lf_aspect == 2.5
    # an existing zero-initialised record is not a light-field view
    assert hb.Camera(pose=np.eye(4)[:3], K=np.eye(3), width=4, height=4).to_c().two_plane == 0
