"""The kernel-variant cases (tests/variant_cases.py), lowered without a GPU: each case reaches the render and backward kernel
instantiations it claims, together they reach every cell of CELLS, every RARE primitive and backward feature meets every
sample-count edge, the refusals are the ones listed, and every case passes its guard against the fp64 oracle.  An edit to
the case list that drops a cell fails here."""
import pytest

from hyperreel_b200.signature import UnsupportedPipeline
from tests.variant_cases import (CELLS, EDGE_RANGE, EDGES, RARE_BWD, RARE_PRIMS, REFUSALS, SPECS, backward_cell,
                                 forward_cell, guard_ok, guard_stats, lower_spec, variant_case)


def _lowered():
    return [(s, lower_spec(s.src, s.variants, s.S, s.layout, s.shade, s.eased).cfg) for s in SPECS]


def _bwd(c):
    try:
        return backward_cell(c)
    except ValueError:
        return None


def test_the_grid():
    """132 plain forward cells (lean / RARE / EASE at two rays per warp, one, and 2 samples per lane; BIG at 4 and 8; each
    x dynamic x 3 layouts x 2 shadings), 96 with extra outputs (one ray per warp), 72 backward cells."""
    fwd = [c for c in CELLS if c.kind == "fwd"]
    assert len(set(CELLS)) == len(CELLS)
    assert len([c for c in fwd if not c.extra]) == 132
    assert len([c for c in fwd if c.extra]) == 96 and all(c.rpw == 1 for c in fwd if c.extra)
    assert len([c for c in CELLS if c.kind == "bwd"]) == 72


def test_every_case_lowers_to_the_cells_it_claims():
    for s, c in _lowered():
        assert c.n_samples == s.S, s.name
        assert forward_cell(c, False) == s.fwd, (s.name, str(forward_cell(c, False)), str(s.fwd))
        assert _bwd(c) == s.bwd, (s.name, str(_bwd(c)), str(s.bwd))


def test_the_cases_cover_every_cell():
    reached = set()
    for s, c in _lowered():
        reached |= {forward_cell(c, False), forward_cell(c, True)}
        if _bwd(c) is not None:
            reached.add(_bwd(c))
    missing = [str(c) for c in CELLS if c not in reached]
    assert not missing, missing
    assert reached <= set(CELLS), [str(c) for c in reached - set(CELLS)]


def test_sample_counts_vary_across_each_edge():
    for edge in EDGES:
        lo, hi = EDGE_RANGE[edge]
        counts = {s.S for s in SPECS if lo <= s.S <= hi}
        assert hi in counts and (lo if edge != "rpw2" else 13) in counts, (edge, counts)
        assert any(S % 4 for S in counts), (edge, counts)


def _edge(S):
    return next(e for e in EDGES if EDGE_RANGE[e][0] <= S <= EDGE_RANGE[e][1])


def test_every_rare_primitive_reaches_every_edge():
    """The RARE primitives are runtime branches inside the RARE and BIG kernels: each one at two rays per warp, one, 2
    samples per lane and 4 / 8 samples per lane; each RARE backward feature at 1 and 2 samples per lane."""
    for p in RARE_PRIMS:
        for edge in EDGES:
            assert any(s.prim == p and s.fwd.family in ("rare", "big") and _edge(s.S) == edge for s in SPECS), (p, edge)
    for p in RARE_BWD:
        for spl in (1, 2):
            assert any(s.prim == p and s.bwd is not None and s.bwd.family == "rare" and s.bwd.spl == spl for s in SPECS), (p, spl)


@pytest.mark.parametrize("src,variants,S,eased,what,message", REFUSALS, ids=[f"{r[4]}-{r[0]}-s{r[2]}" for r in REFUSALS])
def test_refusals(src, variants, S, eased, what, message):
    """Eased density heads above 64 samples are refused at lowering (and by hr_create); the backward refuses more than 64
    samples and the sphere_new primitive (hr_render_backward: tests/test_sample_counts_gpu.py and
    tests/test_kernel_variants_gpu.py call it), and the restated dispatch refuses them the same way."""
    if what == "forward":
        with pytest.raises(UnsupportedPipeline, match=message):
            lower_spec(src, variants, S, eased=eased)
        return
    c = lower_spec(src, variants, S, eased=eased).cfg
    forward_cell(c, False)
    with pytest.raises(ValueError, match=message):
        backward_cell(c)


@pytest.mark.parametrize("name", [s.name for s in SPECS])
def test_every_case_passes_its_guard(name):
    """From the fp64 oracle: rays whose sort keys are out of order, masked samples, samples outside the AABB, a quarter of the
    rays opaque (variant_cases.guard_ok)."""
    spec = next(s for s in SPECS if s.name == name)
    stats = guard_stats(variant_case(name), spec.eased)
    assert guard_ok(stats), stats
