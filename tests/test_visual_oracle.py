"""The embedding visualiser's maps without a GPU: the restatement (oracle/visual_oracle.py) against the reference's own
visualize_warp + to8b, through the goldens and, when a reference checkout is configured, live; and the parsing of every
shipped embedding-visualiser config."""
import json
import os

import numpy as np
import pytest

import hyperreel_b200 as hb
from hyperreel_b200 import lib as L
from oracle.ref_shim import REFERENCE_ROOT, reference_available
from oracle.visual_oracle import visualize_frames_to8b, visualize_to8b
from tests.golden import make_golden_visuals as G

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "visuals.npz")


def _golden():
    z = np.load(GOLDEN)
    names = sorted({k.split("/")[0] for k in z.files if "/" in k})
    return z, names


def test_goldens_cover_the_cases():
    z, names = _golden()
    assert names == sorted(G.cases())
    assert any(z[f"{n}/u8"].max() == 255 for n in names) and any((z[f"{n}/u8"] == 0).any() for n in names)


@pytest.mark.parametrize("name", sorted(G.cases()))
def test_oracle_equals_the_reference_goldens(name):
    z, _ = _golden()
    opts = json.loads(str(z[f"{name}/opts"]))
    got = visualize_frames_to8b(z[f"{name}/x"], **opts)
    assert got.dtype == np.uint8 and np.array_equal(got, z[f"{name}/u8"])


@pytest.mark.skipif(not reference_available(), reason="needs the reference checkout (HYPERREEL_REFERENCE)")
@pytest.mark.parametrize("name", sorted(G.cases()))
def test_oracle_equals_the_live_reference(name):
    opts, x = G.cases()[name]
    assert np.array_equal(visualize_frames_to8b(x, **opts), G.reference_maps(REFERENCE_ROOT, opts, x))


def test_constant_frame_normalises_to_zero_and_bounds_map_to_the_ends():
    assert (visualize_to8b(np.full((7, 3), 2.5, np.float32), normalize=True) == 0).all()
    x = np.array([[0.0], [0.25], [-0.25], [0.125]], np.float32)
    assert visualize_to8b(x, use_abs=True, bounds=[0.0, 0.25])[:, 0].tolist() == [0, 255, 255, 127]
    # 255 * (k / 255) truncates to k - 1 where the fp32 product falls below k
    k = np.arange(256, dtype=np.float32) / np.float32(255)
    got = visualize_to8b(k[:, None])[:, 0].astype(np.int64)
    assert np.array_equal(got, np.floor(np.float32(255) * k).astype(np.int64))


def _configs():
    return json.loads(str(np.load(GOLDEN)["configs"]))


def test_every_shipped_embedding_config_is_in_the_goldens():
    assert sorted(_configs()) == ["default", "default_cascaded", "default_cascaded_2", "default_reflect", "default_time",
                                  "default_time_cascaded", "default_time_cascaded_2", "points"]


ACCEPTED = {
    "default": [("distances", 1, False, None, True), ("point_offset", 3, True, (0.0, 0.25), False),
                ("points", 3, False, (-2.0, 2.0), False)],
    "default_time": [("distances", 1, False, None, True), ("point_offset", 3, True, (0.0, 0.25), False),
                     ("spatial_flow", 3, True, (0.0, 1.0), False)],
    "points": [("points", 3, False, (-2.0, 2.0), False)],
}
REFUSED = {"default_cascaded": "raw_distance", "default_cascaded_2": "raw_distance", "default_reflect": "'normal'",
           "default_time_cascaded": "raw_distance", "default_time_cascaded_2": "raw_distance"}


@pytest.mark.parametrize("name", sorted(ACCEPTED))
def test_shipped_config_is_parsed(name):
    reqs = hb.embedding_requests(hb.to_cfg(_configs()[name]))
    assert [(r.key, r.channels, r.use_abs, r.bounds, r.normalize) for r in reqs] == ACCEPTED[name]
    assert all(r.mode == L.FIELD_OVER for r in reqs)


@pytest.mark.parametrize("name", sorted(REFUSED))
def test_shipped_config_is_refused_naming_the_key(name):
    with pytest.raises(hb.UnsupportedPipeline, match=REFUSED[name]):
        hb.embedding_requests(hb.to_cfg(_configs()[name]))


@pytest.mark.parametrize("cfg, match", [
    (dict(type="flow"), "type 'flow'"),
    (dict(fields=dict(distances=dict(sort=True))), "'distances' has sort"),
    (dict(fields=dict(points=dict(bounds=[1.0, 1.0]))), "'points': bounds"),
    (dict(fields=dict(points=dict(bounds=[0.0, float("inf")]))), "'points': bounds"),
    (dict(fields=dict(points=dict(bounds=[0.0, 1e39]))), "'points': bounds"),
    (dict(fields=dict(points=dict(bounds=[0.0, 1.0, 2.0]))), "'points': bounds"),
    (dict(fields=dict(points=dict(bounds=[[0.0, 0.0, 0.0], [1.0, 1.0, 1.0]]))), "'points': bounds"),
    (dict(no_over_fields=["distances"], fields=dict(distances=dict(normalize=True))), "'distances' is in no_over_fields"),
    (dict(fields=dict(normal=dict(use_abs=True))), "'normal'"),
])
def test_unsupported_options_are_refused_naming_the_key(cfg, match):
    with pytest.raises(hb.UnsupportedPipeline, match=match):
        hb.embedding_requests(hb.to_cfg(cfg))


def test_pred_weights_fields_select_the_mode():
    reqs = hb.embedding_requests(hb.to_cfg(dict(pred_weights_fields=["points"], fields=dict(points={}, distances={}))))
    assert [(r.key, r.mode) for r in reqs] == [("points", L.FIELD_PRED_WEIGHTS), ("distances", L.FIELD_OVER)]
