"""The training table of per-view pixel subsets and the draws with replacement (tests/train_subset_oracle.py) against the
reference's own table order (tests/golden/reference/train_subsample.npz), and the refusals of DeviceRayBatches' table
options, without a GPU."""
import os

import numpy as np
import pytest
import torch

import hyperreel_b200 as hb
from hyperreel_b200.train_data import subset_rows
from tests import train_subset_oracle as S

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference", "train_subsample.npz")


def _golden_cases():
    g = np.load(GOLDEN)
    for name, dataset in zip(g["cases"], g["datasets"]):
        n_cams, n_frames, H, W, full, kf_step, kf_frac, frac = g[f"{name}/params"]
        n_cams, n_frames, H, W = int(n_cams), int(n_frames), int(H), int(W)
        times = g[f"{name}/times"]
        if dataset == "technicolor":
            frames = [int(np.round(t * (n_frames - 1))) for t in times]  # technicolor.py:250
            videos = None
        else:  # video-major views; the times array is frame-major over the videos (neural_3d.py:246-247)
            frames = [int(np.round(times[f * n_cams + v] * (n_frames - 1))) for v in range(n_cams) for f in range(n_frames)]
            videos = [v for v in range(n_cams) for _ in range(n_frames)]
        steps = dict(load_full_step=int(full), subsample_keyframe_step=int(kf_step), subsample_keyframe_frac=float(kf_frac),
                     subsample_frac=float(frac))
        yield str(name), str(dataset), frames, videos, H, W, steps, g[f"{name}/ids"]


CASES = list(_golden_cases())


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_the_restated_table_is_the_references(case):
    name, dataset, frames, videos, H, W, steps, ids = case
    rules = S.plan(frames, counters=dataset, videos=videos, **steps)
    assert np.array_equal(S.table(rules, H, W), ids)
    assert np.array_equal(S.table_pixels(rules, H, W, np.arange(ids.size)), ids)
    # the library's plan and row counts
    assert hb.regular_subsample_plan(frames, counters=dataset, videos=videos, **steps) == rules
    assert [subset_rows(s, o, H, W) for s, o in rules] == list(S.counts(rules, H, W))
    assert {s for s, _ in rules} > {1}  # the case exercises subsets


def test_the_fixture_covers_the_shapes_and_steps_it_should():
    names = [c[0] for c in CASES]
    assert {c[1] for c in CASES} == {"technicolor", "neural_3d"}
    assert all(len(c[2]) >= 100 for c in CASES)  # 50 frames of at least 2 views or videos
    strides = {name: {s for s, _ in S.plan(f, counters=d, videos=v, **st)} for name, d, f, v, H, W, st, _ in CASES}
    assert any(c[5] < max(strides[c[0]]) for c in CASES)  # W < stride
    assert any(c[4] % max(strides[c[0]]) and c[5] % max(strides[c[0]]) for c in CASES)
    assert len({tuple(c[6].values()) for c in CASES}) >= 3, names


def test_the_closed_form_is_the_mask_order():
    for s in range(1, 9):
        for o in list(range(s)) + [s + 3, 37]:
            for H in range(1, 2 * s + 2):
                for W in range(1, 2 * s + 2):
                    want = np.nonzero(S.mask(s, o, H, W).reshape(-1))[0]
                    assert subset_rows(s, o % s, H, W) == want.size == subset_rows(s, o, H, W)
                    y, x = S.rank_to_pixel(s, o % s, H, W, np.arange(want.size))
                    assert np.array_equal(y * W + x, want), (s, o, H, W)


def test_the_shipped_technicolor_split():
    """15 training views x 50 frames of 2048x1088 (technicolor.yaml): 7 whole frames, 6 at 1/4 and 37 at 1/8."""
    frames = [f for f in range(50) for _ in range(15)]
    rules = hb.regular_subsample_plan(frames, load_full_step=8, subsample_keyframe_step=4, subsample_keyframe_frac=0.25,
                                      subsample_frac=0.125)
    per_frame = [rules[15 * f][0] for f in range(50)]
    assert (per_frame.count(1), per_frame.count(4), per_frame.count(8)) == (7, 6, 37)
    rows = [subset_rows(s, o % s, 1088, 2048) for s, o in rules]
    assert sum(rows) == 438_681_600
    whole = sum(r for r, (s, _) in zip(rows, rules) if s == 1)
    assert abs(whole / sum(rows) - 0.533) < 1e-3


def test_draws_are_in_range_reproducible_and_keyed():
    for n in (1, 2, 7, 8979, 438_681_600, 2 ** 62 + 5):
        d = S.draws(n, 3, 1, np.arange(20000))
        assert d.min() >= 0 and d.max() < n
        assert np.array_equal(d, S.draws(n, 3, 1, np.arange(20000)))
        if n > 1000:
            assert not np.array_equal(d, S.draws(n, 4, 1, np.arange(20000)))
            assert not np.array_equal(d, S.draws(n, 3, 2, np.arange(20000)))
    # positions are independent of the batch split, and the draws are uniform
    n = 1000
    d = S.draws(n, 0, 0, np.arange(200000))
    assert np.array_equal(d[5000:6000], S.draws(n, 0, 0, np.arange(5000, 6000)))
    hist = np.bincount(d, minlength=n)
    assert abs(hist.mean() - 200) < 1e-9 and hist.min() > 140 and hist.max() < 265
    # the reduction against exact integer arithmetic
    h = S.mix64(np.arange(1000, dtype=np.uint64) * np.uint64(12345))
    for n in (3, 2 ** 40 + 1, 2 ** 62):
        assert [int(v) for v in S._mulhi(h, n)] == [(int(a) * n) >> 64 for a in h]


def _cams(n, w=8, h=6):
    K = [[10.0, 0.0, w / 2], [0.0, 10.0, h / 2], [0.0, 0.0, 1.0]]
    pose = [[1.0, 0.0, 0.0, 0.0], [0.0, 1.0, 0.0, 0.0], [0.0, 0.0, 1.0, 0.0]]
    return [hb.Camera(pose=pose, K=K, width=w, height=h) for _ in range(n)]


def test_table_options_are_refused_when_malformed():
    img = torch.zeros(2, 6, 8, 3, dtype=torch.uint8)
    for kw, msg in ((dict(replacement=True), "num_iters"), (dict(replacement=True, num_iters=0), "num_iters"),
                    (dict(num_iters=10), "num_iters"), (dict(subsample=[(1, 0)]), "one \\(stride, offset\\) per view"),
                    (dict(subsample=[(1, 0), (0, 0)]), "strides"), (dict(subsample=[(1, 0), (2.5, 0)]), "strides"),
                    (dict(subsample=[(1, 0), (1, 0, 0)]), "per view")):
        with pytest.raises(ValueError, match=msg):
            hb.DeviceRayBatches(_cams(2), img, 16, **kw)
    one = torch.zeros(2, 1, 1, 3, dtype=torch.uint8)
    with pytest.raises(ValueError, match="empty"):
        hb.DeviceRayBatches(_cams(2, 1, 1), one, 16, subsample=[(2, 1), (3, 1)])


def test_plan_refusals():
    steps = dict(load_full_step=4, subsample_keyframe_step=2, subsample_keyframe_frac=0.25, subsample_frac=0.125)
    with pytest.raises(ValueError, match="counters"):
        hb.regular_subsample_plan([0, 1], counters="immersive", **steps)
    with pytest.raises(ValueError, match="one video index per view"):
        hb.regular_subsample_plan([0, 1], counters="neural_3d", **steps)
    with pytest.raises(ValueError, match="neural_3d"):
        hb.regular_subsample_plan([0, 1], videos=[0, 0], **steps)
    with pytest.raises(ValueError, match="video-major"):
        hb.regular_subsample_plan([0, 1, 0, 1, 2], counters="neural_3d", videos=[0, 0, 1, 1, 0], **steps)
    with pytest.raises(ValueError, match="consecutive"):
        hb.regular_subsample_plan([0, 2, 3], counters="neural_3d", videos=[0, 0, 0], **steps)
    with pytest.raises(ValueError, match="load_full_step"):
        hb.regular_subsample_plan([0, 1], **dict(steps, load_full_step=0))
    with pytest.raises(ValueError, match="subsample_frac"):
        hb.regular_subsample_plan([0, 1], **dict(steps, subsample_frac=0.0))
    with pytest.raises(ValueError, match="subsample_keyframe_frac"):
        hb.regular_subsample_plan([0, 1], **dict(steps, subsample_keyframe_frac=3.0))
    # strides round half to even, as the reference's np.round does
    assert hb.regular_subsample_plan([1, 2], **dict(steps, subsample_keyframe_frac=0.4, subsample_frac=1 / 3.5)) == \
        [(4, 0), (2, 0)]


def test_from_config_refuses_the_datasets_it_cannot_reproduce():
    img = torch.zeros(2, 6, 8, 3, dtype=torch.uint8)
    training = {"batch_size": 16, "sample_with_replacement": True, "num_iters": 4000}
    imm = {"name": "immersive", "load_full_step": 8, "subsample_keyframe_step": 4, "subsample_keyframe_frac": 0.25,
           "subsample_frac": 0.125}
    with pytest.raises(ValueError, match="importance_subsample"):
        hb.DeviceRayBatches.from_config(hb.to_cfg({"training": training, "dataset": imm}), _cams(2), img)
    with pytest.raises(ValueError, match="subsample_frac"):
        hb.DeviceRayBatches.from_config(hb.to_cfg({"training": training, "dataset": {"name": "video3d_time",
                                                                                      "subsample_frac": 0.5}}),
                                        _cams(2), img)
    with pytest.raises(ValueError, match="video-major"):
        cams = _cams(4)
        for c, (idx, t) in zip(cams, [(0, 0.0), (1, 0.0), (0, 1 / 49), (1, 1 / 49)]):  # frame-major: not neural_3d's order
            c.cam_idx, c.time = idx, t
        hb.DeviceRayBatches.from_config(hb.to_cfg({"training": training, "dataset": {"name": "neural_3d",
                                                                                      "num_frames": 50}}),
                                        cams, torch.zeros(4, 6, 8, 3, dtype=torch.uint8))
