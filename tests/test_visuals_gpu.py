"""Embedding maps on the device (hr_render_visuals): every map equals the restatement of visualize_warp + to8b
(oracle/visual_oracle.py) applied to the fp32 field LightfieldModel.forward returns for the same view, the RGB video equals
render_video's, the maps are within 1 LSB of the fp32 oracle's, calls are deterministic, and every refusal leaves the
outputs untouched."""
import ctypes as C
import dataclasses
import json
import os

import numpy as np
import pytest
import torch

import hyperreel_b200 as hb
from hyperreel_b200 import lib as L
from oracle.hyperreel_oracle import HyperReelOracle
from oracle.visual_oracle import visualize_to8b
from tests.cases import build_case
from tests.test_kernel_variants_gpu import kernels_run
from tests.test_shipped_yaml_golden import SHIPPED, load_fixture

pytestmark = pytest.mark.gpu

W, H = 48, 30  # 1440 pixels per frame
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "visuals.npz")
CONFIGS = json.loads(str(np.load(GOLDEN)["configs"]))


def _pose(rx, ry):
    cx, sx, cy, sy = np.cos(rx), np.sin(rx), np.cos(ry), np.sin(ry)
    R = np.diag([-1.0, 1.0, -1.0]) @ np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]]) @ np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    return np.concatenate([R, np.array([[0.0], [0.0], [-1.0]])], 1)  # facing the seeded scenes, which lie along +z


def _cameras(n):
    """n frames cycling pinhole, fisheye and two-plane cameras, times spread over [0, 1]."""
    out = []
    for f in range(n):
        t = f / max(n - 1, 1)
        if f % 3 == 2:
            out.append(hb.TwoPlaneCamera(width=W, height=H, s=0.05 * f, t=-0.03 * f, st_scale=0.25, uv_scale=0.6, time=t))
        else:
            out.append(hb.Camera(pose=_pose(0.03 * f, -0.05 * f), K=[[40.0, 0, 23.7], [0, 40.0, 15.2], [0, 0, 1]], width=W,
                                 height=H, time=t, distortion=(0.08, 0.01) if f % 3 == 1 else None))
    return out


def _model(name):
    """(render fn, plain config, dataset, state dict) of a seeded case or a shipped-YAML fixture."""
    if name.startswith("shipped:"):
        path = next(p for p in SHIPPED if os.path.basename(p) == name[8:] + ".npz")
        plain, cfg, ds, _, sd, _, _ = load_fixture(path)
    else:
        case = build_case(name)
        plain, cfg, ds, sd = case.model_cfg_plain, case.model_cfg, case.dataset, case.state_dict
    model = hb.LightfieldModel(cfg, dataset=ds)
    render = hb.RenderLightfield(model, None, cfg.render)
    render.load_state_dict(sd, strict=False)
    render.eval()
    return render, plain, ds, sd


def _field_frames(model, cams, times, keys, pred_w=()):
    """The fp32 fields [F, H*W, dim] forward returns for each frame's rays."""
    per = {k: [] for k in keys}
    for c, t in zip(cams, times):
        rays = hb.generate_rays(dataclasses.replace(c, time=float(np.float32(t))), c_in=model.sig.c_in)
        out = model(rays, {"fields": list(keys), "pred_weights_fields": list(pred_w)})
        for k in keys:
            per[k].append(out[k].cpu().numpy())
    return {k: np.stack(v, 0) for k, v in per.items()}


def _restated(reqs, fields):
    out = {}
    for r in reqs:
        m = np.stack([visualize_to8b(f, r.use_abs, r.bounds, r.normalize) for f in fields[r.key]], 0)
        out[f"embedding_{r.key}"] = m.reshape(m.shape[0], H, W, r.channels)[..., 0] if r.channels == 1 else m.reshape(-1, H, W, 3)
    return out


MODELS = [("technicolor_trained", "default_time", 5), ("donerf_trained", "default", 4), ("shipped:shiny_z_plane", "default", 3),
          ("shipped:neural_3d_z_plane_static", "points", 3)]  # the last one: 256 samples, 8 per lane


@pytest.mark.parametrize("sub", [1000, 0])  # sub-batches straddling frames on two streams; the whole video in one
@pytest.mark.parametrize("name, config, n", MODELS)
def test_maps_equal_the_restatement_of_the_fp32_fields(name, config, n, sub):
    render, _, _, _ = _model(name)
    model = render.model
    model.set_sub_batch(sub)
    cams = _cameras(n)
    times = [c.time for c in cams]
    vcfg = hb.to_cfg(CONFIGS[config])
    reqs = hb.embedding_requests(vcfg)
    got = hb.render_embeddings(render, cams, vcfg)
    fields = _field_frames(model, cams, times, [r.key for r in reqs])
    want = _restated(reqs, fields)
    assert sorted(got) == sorted(["rgb"] + list(want))
    for k, v in want.items():
        g = got[k].cpu().numpy()
        assert g.dtype == np.uint8 and g.shape == v.shape, (k, g.shape, v.shape)
        assert np.array_equal(g, v), (k, int((g != v).sum()))
    for r in reqs:  # a normalised map spans [0, 255] unless its frame is constant
        if r.normalize:
            assert len(np.unique(got[f"embedding_{r.key}"].cpu().numpy())) > 8, r.key
    # the RGB frames of the same pass are render_video's, and so are those of a call without maps
    video = model.render_video(cams, times)
    assert torch.equal(got["rgb"], video)
    assert torch.equal(hb.render_embeddings(render, cams, hb.to_cfg({"type": "embedding", "fields": {}}))["rgb"], video)


@pytest.mark.parametrize("name, config, n", MODELS[:3])
def test_maps_are_within_one_step_of_the_fp32_oracle(name, config, n):
    render, plain, ds, sd = _model(name)
    model = render.model
    cams = _cameras(n)
    vcfg = hb.to_cfg(CONFIGS[config])
    reqs = hb.embedding_requests(vcfg)
    got = hb.render_embeddings(render, cams, vcfg, rgb=False)
    oracle = HyperReelOracle(plain, ds, sd)
    fields = {r.key: [] for r in reqs}
    for c in cams:
        rays = hb.generate_rays(c, c_in=model.sig.c_in).cpu()
        out = oracle.render_fields(rays, {"fields": [r.key for r in reqs]})
        for r in reqs:
            fields[r.key].append(out[r.key].reshape(-1, r.channels).float().numpy())
    want = _restated(reqs, {k: np.stack(v, 0) for k, v in fields.items()})
    for k, v in want.items():
        d = np.abs(got[k].cpu().numpy().astype(np.int64) - v.astype(np.int64))
        assert (d <= 1).mean() >= 0.999, (k, float((d <= 1).mean()), int(d.max()))


def test_pred_weights_mode_and_mixed_requests():
    render, _, _, _ = _model("technicolor_trained")
    model = render.model
    model.set_sub_batch(700)
    cams = _cameras(4)
    vcfg = hb.to_cfg({"type": "embedding", "pred_weights_fields": ["points"],
                      "fields": {"points": {"bounds": [-2.0, 2.0], "normalize": True}, "sigma": {"use_abs": True, "normalize": True},
                                 "distances": {"bounds": [0.0, 5.0]}, "color_scale": {"use_abs": True, "bounds": [0.0, 0.5]}}})
    reqs = hb.embedding_requests(vcfg)
    got = hb.render_embeddings(render, cams, vcfg)
    fields = _field_frames(model, cams, [c.time for c in cams], [r.key for r in reqs], pred_w=["points"])
    for k, v in _restated(reqs, fields).items():
        assert np.array_equal(got[k].cpu().numpy(), v), k


def _raw(model, cams, reqs, video, ws_delta=0, ws_offset=0):
    """hr_render_visuals called directly; returns the return code."""
    lib = model._lib
    arr = (L.hr_visual_request * max(len(reqs), 1))(*reqs)
    F = len(cams)
    need = int(lib.hr_render_visuals_workspace_bytes(model._handle, arr, len(reqs), F, H, W))
    ws = torch.empty(max(need, 0) + 256, dtype=torch.uint8, device="cuda")
    recs = (L.hr_camera * F)(*[c.to_c() for c in cams])
    tt = (C.c_float * F)(*[c.time for c in cams])
    rc = lib.hr_render_visuals(model._handle, recs, tt, F, video, arr, len(reqs), ws.data_ptr() + ws_offset, need + ws_delta,
                               torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return rc


def _req(field, out, channels=None, mode=L.FIELD_OVER, use_abs=0, bounded=1, normalize=1, lo=0.0, hi=2.0):
    ch = L.FIELD_CHANNELS[field] if channels is None else channels
    return L.hr_visual_request(L.FIELDS[field], mode, ch, use_abs, bounded, normalize, lo, hi, out)


def test_two_calls_write_the_same_bytes_and_a_short_workspace_is_refused():
    render, _, _, _ = _model("technicolor_trained")
    model = render.model
    model.set_sub_batch(1000)
    cams = _cameras(5)
    model.render_video(cams[:1])  # upload
    outs = [[torch.full((5, H, W, 3), 77, dtype=torch.uint8, device="cuda") for _ in range(3)] for _ in range(2)]
    for o in outs:
        reqs = [_req("distances", o[1].data_ptr(), normalize=1, bounded=0), _req("points", o[2].data_ptr(), normalize=0, lo=-2.0)]
        assert _raw(model, cams, reqs, o[0].data_ptr()) == 0
    for a, b in zip(*outs):
        assert torch.equal(a, b)
    short = [torch.full((5, H, W, 3), 77, dtype=torch.uint8, device="cuda") for _ in range(3)]
    reqs = [_req("distances", short[1].data_ptr(), normalize=1, bounded=0), _req("points", short[2].data_ptr(), normalize=0)]
    assert _raw(model, cams, reqs, short[0].data_ptr(), ws_delta=-1) != 0
    assert "workspace too small" in L.load_library().hr_last_error().decode()
    assert all(bool((t == 77).all()) for t in short)


def test_a_call_without_maps_runs_the_video_render_kernel():
    """render_embeddings without a map is render_video launch for launch: the same render_kernel<...>, without the extra
    fields' epilogue (EXTRA, the seventh template argument, false); a call with a map runs the EXTRA = true kernel."""
    render, _, _, _ = _model("technicolor_trained")
    model = render.model
    model.set_sub_batch(1000)
    cams = _cameras(3)
    model.render_video(cams)  # upload
    no_maps = hb.to_cfg({"type": "embedding", "fields": {}})
    one_map = hb.to_cfg({"type": "embedding", "fields": {"distances": {"bounds": [0.0, 5.0]}}})
    video = kernels_run(lambda: model.render_video(cams))[0]
    assert len(video) == 1 and not next(iter(video))[6], video
    assert kernels_run(lambda: hb.render_embeddings(render, cams, no_maps))[0] == video
    mapped = kernels_run(lambda: hb.render_embeddings(render, cams, one_map))[0]
    assert len(mapped) == 1 and next(iter(mapped))[6], mapped


def test_the_workspaces_share_one_layout():
    """Without a request the visual workspace is the video's; the video, score and visual workspaces grow with the frame
    count by the 256-byte aligned record and time tables alone (the ring, partials and slots depend on the sub-batch)."""
    render, _, _, _ = _model("technicolor_trained")
    model = render.model
    model.set_sub_batch(1000)  # a ring of 3 frames of 48 x 30: both frame counts below exceed it
    model.render_video(_cameras(1))  # upload
    lib, h = model._lib, model._handle
    m = torch.empty((40, H, W), dtype=torch.uint8, device="cuda")
    arr = (L.hr_visual_request * 1)(_req("distances", m.data_ptr(), normalize=1, bounded=0))

    def tables(F):
        return sum((b + 255) // 256 * 256 for b in (F * C.sizeof(L.hr_camera), F * 4))

    for F in (5, 40):
        assert lib.hr_video_workspace_bytes(h, F, H, W) == lib.hr_render_visuals_workspace_bytes(h, None, 0, F, H, W) > 0
    for size in (lambda F: lib.hr_video_workspace_bytes(h, F, H, W), lambda F: lib.hr_score_views_workspace_bytes(h, F, H, W),
                 lambda F: lib.hr_render_visuals_workspace_bytes(h, arr, 1, F, H, W)):
        assert size(40) - size(5) == tables(40) - tables(5)


def test_refusals_leave_the_outputs_untouched():
    render, _, _, _ = _model("donerf_trained")  # static: no keyframe times
    model = render.model
    cams = _cameras(3)
    model.render_video(cams[:1])
    video = torch.full((3, H, W, 3), 77, dtype=torch.uint8, device="cuda")
    m3 = torch.full((3, H, W, 3), 77, dtype=torch.uint8, device="cuda")
    p, v = m3.data_ptr(), video.data_ptr()
    bad_cam = _cameras(3)
    bad_cam[1] = dataclasses.replace(bad_cam[1], pose=np.full((3, 4), np.nan))
    cases = [
        ("unknown field", [L.hr_visual_request(15, 0, 1, 0, 0, 0, 0.0, 1.0, p)], cams, v, 0),
        ("mode 1", [_req("points", p, mode=L.FIELD_NO_OVER)], cams, v, 0),
        ("3 channels, not 2", [_req("points", p, channels=2)], cams, v, 0),
        ("bounds", [_req("points", p, lo=1.0, hi=1.0)], cams, v, 0),
        ("bounds", [_req("points", p, lo=float("nan"))], cams, v, 0),
        ("null output", [_req("points", None)], cams, v, 0),
        ("requested twice", [_req("points", p), _req("points", p)], cams, v, 0),
        ("no keyframe times", [_req("base_times", p)], cams, v, 0),
        ("nothing to write", [], cams, None, 0),
        ("not finite", [_req("points", p)], bad_cam, v, 0),
        ("16-byte aligned", [_req("points", p)], cams, v, 8),
    ]
    for why, reqs, cs, vid, ws_off in cases:
        assert _raw(model, cs, reqs, vid, ws_offset=ws_off) != 0, why
        assert why in L.load_library().hr_last_error().decode(), (why, L.load_library().hr_last_error())
        assert bool((video == 77).all()) and bool((m3 == 77).all()), why
    # a field this model lacks is refused in Python with the key named, before any work
    with pytest.raises(hb.UnsupportedPipeline, match="spatial_flow"):
        hb.render_embeddings(render, cams, hb.to_cfg(CONFIGS["default_time"]))


def test_system_returns_the_reference_keys_dtypes_and_shapes():
    case = build_case("technicolor_trained")
    cfg = hb.to_cfg({"model": case.model_cfg_plain, "visualizers": {"embedding": CONFIGS["default_time"]}})
    system = hb.INRSystem(cfg, dataset=case.dataset)
    system.load_state_dict(case.state_dict)
    system.train()
    cams = _cameras(4)
    vid = system.validation_video_outputs(cams)
    assert system.training  # the mode is restored
    assert {k: (v.dtype, tuple(v.shape)) for k, v in vid.items()} == {
        "videos/rgb": (torch.uint8, (4, H, W, 3)), "videos/embedding_distances": (torch.uint8, (4, H, W)),
        "videos/embedding_point_offset": (torch.uint8, (4, H, W, 3)), "videos/embedding_spatial_flow": (torch.uint8, (4, H, W, 3))}
    assert torch.equal(vid["videos/rgb"], system.render_video(cams))
    img = system.validation_image_embeddings(cams)
    assert {k: (v.dtype, tuple(v.shape)) for k, v in img.items()} == {
        "images/embedding_distances": (torch.uint8, (4, H, W)), "images/embedding_point_offset": (torch.uint8, (4, H, W, 3)),
        "images/embedding_spatial_flow": (torch.uint8, (4, H, W, 3))}
    for k in img:
        assert torch.equal(img[k], vid["videos/" + k[len("images/"):]])
    assert system.validation_image_embeddings(cams, testing=True) == {}  # run_on_test: False
    bad = hb.INRSystem(hb.to_cfg({"model": case.model_cfg_plain, "visualizers": {"e": {"type": "flow"}}}), dataset=case.dataset)
    with pytest.raises(hb.UnsupportedPipeline, match="flow"):
        bad.validation_video_outputs(cams)
