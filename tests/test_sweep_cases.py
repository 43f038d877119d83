"""The sample-count sweep and the sample-net shape cover (tests/sweep_cases.py), lowered without a GPU: each configuration
reaches the hr_config shape its name states, and together they reach every edge the GPU tests are there for.  A later edit
to a case list that drops an edge fails here."""
import re

import pytest

import hyperreel_b200 as hb
from hyperreel_b200 import configs, lib as L
from hyperreel_b200.signature import UnsupportedPipeline, lower, tc_passes
from tests.sweep_cases import (NET_SHAPES, SAMPLE_COUNTS, SWEEP_BUILTINS, guard_ok, guard_stats, net_cfg, net_shape,
                               sweep_case)


def _shapes():
    out = {}
    for spec in NET_SHAPES:
        cfg, ds = net_cfg(*spec[1:])
        out[spec[0]] = net_shape(lower(cfg, ds))
    return out


def test_net_shapes_lower_to_their_names():
    for name, s in _shapes().items():
        m = re.fullmatch(r"w(\d+)_d(\d+)(?:_skip(\d+))?_in(\d+)_out(\d+)", name)
        assert m, name
        W, depth, skip, n_in, n_out = (int(g) if g is not None else -1 for g in m.groups())
        assert (s["W"], s["layers"], s["skip"], s["mlp_in"], s["mlp_out"]) == (W, depth, skip, n_in, n_out), (name, s)
        assert s["passes"] == depth - 1 + -(-n_out // W) <= L.HR_TC_MAX_PASSES, (name, s)


def test_net_shapes_cover_every_edge():
    shapes = list(_shapes().values())
    widths = {128, 256}
    for W in widths:
        at = [s for s in shapes if s["W"] == W]
        assert {s["layers"] for s in at} >= {2, 3, 6, 10}, W
        assert {-1, 1} <= {s["skip"] for s in at} and any(s["skip"] == s["layers"] - 2 > 1 for s in at), W
        assert {(s["mlp_in"] + 31) // 32 for s in at} == {1, 2}, W  # one and two 32-wide input chunks
        outs = {s["mlp_out"] for s in at}
        assert any(o < W for o in outs) and W in outs and W + 4 in outs, (W, outs)  # below, one pass, one group past it
    ins = {s["mlp_in"] for s in shapes}
    assert min(ins) == 4 and ins & {16, 17} and ins & {32, 33} and max(ins) == 63, ins  # smallest and largest reachable
    assert {s["mlp_out"] % 4 for s in shapes} == {0, 1, 2, 3}
    assert max(s["passes"] for s in shapes) == L.HR_TC_MAX_PASSES
    assert any(s["layers"] == 10 and s["W"] == 128 for s in shapes)


def test_the_tensor_core_net_is_refused_one_pass_past_the_table():
    """One output column more than the largest net NET_SHAPES holds: the tensor-core net is refused at lowering, naming the
    limit (it would otherwise fail at upload); the fp32 net has no such limit."""
    cfg, ds = net_cfg("technicolor_z_plane", 128, 10, "L-2", 0, 2, 189, "global")
    with pytest.raises(UnsupportedPipeline, match="HR_TC_MAX_PASSES"):
        lower(cfg, ds)
    with pytest.raises(UnsupportedPipeline, match="HR_TC_MAX_PASSES"):
        hb.LightfieldModel(cfg, dataset=ds)
    sig = lower(cfg, ds, mlp_mode=L.MLP_FP32_SIMT)
    assert tc_passes(128, 10, sig.cfg.mlp_out) == L.HR_TC_MAX_PASSES + 1


def test_sample_counts_reach_every_edge():
    counts = set(SAMPLE_COUNTS)
    assert {16, 17, 32, 33, 64, 65, 128, 129, 1, 256} <= counts  # variant edges, the smallest and largest count
    for lo, hi in ((17, 31), (33, 47), (65, 95), (129, 255)):
        assert any(lo <= S <= hi for S in counts), (lo, hi)
    assert {S % 4 for S in counts} == {0, 1, 2, 3}
    for b in SWEEP_BUILTINS:
        for S in SAMPLE_COUNTS:
            cfg, ds = configs.get(b, n_voxels=32 ** 3, z_channels=S)
            c = lower(cfg, ds).cfg
            assert c.n_samples == S and c.head_stride == 15 and c.mlp_out == 15 * S, (b, S)
            assert tc_passes(c.mlp_width, c.mlp_layers, c.mlp_out) <= L.HR_TC_MAX_PASSES, (b, S)
    # every residue of the head row mod 4 on every built-in
    assert {(15 * S) % 4 for S in counts} == {0, 1, 2, 3}


@pytest.mark.parametrize("builtin", SWEEP_BUILTINS)
def test_more_than_256_samples_are_refused(builtin):
    cfg, ds = configs.get(builtin, n_voxels=32 ** 3, z_channels=257)
    with pytest.raises(UnsupportedPipeline, match="257"):
        hb.LightfieldModel(cfg, dataset=ds)


@pytest.mark.parametrize("builtin", SWEEP_BUILTINS)
def test_sweep_cases_pass_their_guards(builtin):
    """Every sweep case, from the fp64 oracle: rays whose sort keys are out of order, masked samples, samples outside the
    AABB, a quarter of the rays opaque (sweep_cases.guard_ok)."""
    bad = [(S, guard_stats(sweep_case(builtin, S))) for S in SAMPLE_COUNTS
           if not guard_ok(guard_stats(sweep_case(builtin, S)), S)]
    assert not bad, bad
