"""The Immersive dataset's importance subsample without a GPU: the NumPy restatement (tests/importance_oracle.py) against the
reference's own tables (tests/golden/reference/train_importance.npz), importance_subsample_plan's rounding and validation, and
the refusals of DeviceRayBatches(importance=...) and from_config."""
import numpy as np
import pytest
import torch

import hyperreel_b200 as hb
from tests import importance_oracle as O

CASES = O.golden_cases()


def _plan(c):
    return hb.importance_subsample_plan(c["frames"], c["videos"], height=c["H"], width=c["W"], **c["steps"])


def test_the_goldens_cover_the_edge_cases():
    by = {c["name"]: c for c in CASES}
    assert set(by) == {"shipped_3v_18x24", "crossing_2v_30x40", "static_1v_12x16", "tiny_2v_1x3", "other_2v_15x20",
                       "immersive_crop_240x320"}
    assert (by["crossing_2v_30x40"]["dz"] >= np.float32(-0.05)).any() and (by["crossing_2v_30x40"]["dz"] < -0.05).any()
    assert by["static_1v_12x16"]["counts"][2] == 0
    assert [e[0] for e in _plan(by["tiny_2v_1x3"]) if e is not None and e[0] == 0]  # num_take rounds to 0
    # ties: some frame keeps fewer than num_take pixels although every one of its rays passes the dz test
    c = by["shipped_3v_18x24"]
    assert any(e is not None and n < e[0] for e, n in zip(_plan(c), c["counts"]))
    assert (c["dz"] < -0.05).all()


@pytest.mark.parametrize("c", CASES, ids=[c["name"] for c in CASES])
def test_the_restated_table_is_the_references(c):
    plan = _plan(c)
    ids = O.table_ids(c["images"], c["dz"], plan)
    assert np.array_equal(ids, c["ids"])
    hw = c["H"] * c["W"]
    assert np.array_equal(np.bincount(ids // hw, minlength=len(plan)), c["counts"])
    assert all(n == hw for e, n in zip(plan, c["counts"]) if e is None)


def test_plan_follows_the_reference_rules_and_rounding():
    steps = dict(load_full_step=8, subsample_keyframe_step=4, subsample_keyframe_frac=0.25, subsample_frac=0.125)
    frames = list(range(10)) + list(range(10))
    videos = [0] * 10 + [1] * 10
    plan = hb.importance_subsample_plan(frames, videos, height=4, width=5, **steps)
    # 20 pixels: keyframes take round(5.0) = 5, others round(2.5) = 2 (half to even, as np.round)
    want = [None, (2, 0), (2, 1), (2, 2), (5, 3), (2, 4), (2, 5), (2, 6), None, (2, 8)]
    assert plan == want + [None if e is None else (e[0], e[1] + 10) for e in want]
    # a video's first view is whole whatever its frame; load_full_step wins over the keyframe step
    plan = hb.importance_subsample_plan([3, 4, 5], [0, 0, 0], height=2, width=3, load_full_step=4,
                                        subsample_keyframe_step=2, subsample_keyframe_frac=0.5, subsample_frac=1 / 6)
    assert plan == [None, None, (1, 1)]
    plan = hb.importance_subsample_plan([0, 1, 2], [0, 0, 0], height=2, width=3, load_full_step=1,
                                        subsample_keyframe_step=1, subsample_keyframe_frac=0.5, subsample_frac=0.5)
    assert plan == [None, None, None]
    # num_take = N and 0 are representable
    assert hb.importance_subsample_plan([0, 1, 2], [0, 0, 0], height=1, width=3, load_full_step=5, subsample_keyframe_step=2,
                                        subsample_keyframe_frac=1.0, subsample_frac=0.0) == [None, (0, 0), (3, 1)]


def test_plan_refusals():
    steps = dict(load_full_step=8, subsample_keyframe_step=4, subsample_keyframe_frac=0.25, subsample_frac=0.125)
    for kw, msg in ((dict(frames=[0, 1], videos=[0]), "video indices"),
                    (dict(frames=[0, 1, 0, 1, 2], videos=[0, 0, 1, 1, 0]), "video-major"),
                    (dict(frames=[0, 2, 3], videos=[0, 0, 0]), "consecutive"),
                    (dict(frames=[-1, 0], videos=[0, 0]), "frames"),
                    (dict(frames=[0, 1], videos=[0, 0], load_full_step=0), "load_full_step"),
                    (dict(frames=[0, 1], videos=[0, 0], subsample_keyframe_step=1.5), "subsample_keyframe_step"),
                    (dict(frames=[0, 1], videos=[0, 0], subsample_frac=1.5), "subsample_frac"),
                    (dict(frames=[0, 1], videos=[0, 0], subsample_keyframe_frac=-0.1), "subsample_keyframe_frac"),
                    (dict(frames=[0, 1], videos=[0, 0], height=0), "pixel")):
        args = dict(steps, height=3, width=4)
        args.update(kw)
        with pytest.raises(ValueError, match=msg):
            hb.importance_subsample_plan(args.pop("frames"), args.pop("videos"), **args)


def _cams(n, w=8, h=6, times=None, idx=None):
    K = [[10.0, 0.0, w / 2], [0.0, 10.0, h / 2], [0.0, 0.0, 1.0]]
    pose = [[1.0, 0.0, 0.0, 0.0], [0.0, 1.0, 0.0, 0.0], [0.0, 0.0, 1.0, 0.0]]
    return [hb.Camera(pose=pose, K=K, width=w, height=h, time=0.0 if times is None else times[i],
                      cam_idx=0.0 if idx is None else idx[i], distortion=(0.05, -0.01)) for i in range(n)]


def test_device_batches_refuse_malformed_importance_plans():
    img = torch.zeros(3, 6, 8, 3, dtype=torch.uint8)
    for kw, msg in ((dict(importance=[None, (1, 0)]), "one entry per view"),
                    (dict(importance=[None, (1, 0), (49, 1)]), "outside"),
                    (dict(importance=[None, (1, 0), (-1, 1)]), "outside"),
                    (dict(importance=[None, (1, 0), (1, 0)]), "previous frame"),
                    (dict(importance=[(1, -1), None, None]), "previous frame"),
                    (dict(importance=[None, (1, 0, 2), None]), "num_take, prev"),
                    (dict(importance=[None, (1.5, 0), None]), "num_take, prev"),
                    (dict(importance=[None, None, None], subsample=[(1, 0)] * 3), "importance and subsample")):
        with pytest.raises(ValueError, match=msg):
            hb.DeviceRayBatches(_cams(3), img, 16, **kw)


def test_from_config_refuses_immersive_views_the_plan_cannot_represent():
    training = {"batch_size": 16, "sample_with_replacement": True, "num_iters": 4000}
    imm = {"name": "immersive", "num_frames": 50, "load_full_step": 8, "subsample_keyframe_step": 4,
           "subsample_keyframe_frac": 0.25, "subsample_frac": 0.125}
    img = torch.zeros(4, 6, 8, 3, dtype=torch.uint8)
    cfg = hb.to_cfg({"training": training, "dataset": imm})
    # frame-major views: cam_idx 0 appears again after cam_idx 1
    with pytest.raises(ValueError, match="video-major"):
        hb.DeviceRayBatches.from_config(cfg, _cams(4, times=[0, 0, 1 / 49, 1 / 49], idx=[0, 1, 0, 1]), img)
    # a skipped frame inside a video
    with pytest.raises(ValueError, match="consecutive"):
        hb.DeviceRayBatches.from_config(cfg, _cams(4, times=[0, 1 / 49, 3 / 49, 4 / 49], idx=[0, 0, 0, 0]), img)
    with pytest.raises(ValueError, match="subsample_frac"):
        bad = hb.to_cfg({"training": training, "dataset": dict(imm, subsample_frac=2.0)})
        hb.DeviceRayBatches.from_config(bad, _cams(4, times=[0, 1 / 49, 2 / 49, 3 / 49], idx=[0, 0, 0, 0]), img)
