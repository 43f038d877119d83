"""Every render and render-backward kernel instantiation the host dispatch can reach, against the fp64 oracle.

The render forward and backward are template families; each cell of tests/variant_cases.py:CELLS is separate machine code
(register arrays, shared-memory layouts, shuffle patterns).  Each case of variant_cases.SPECS runs
* its plain render (`render`, both `mlp_mode`s) and its extra-output render (`render_stages`) with the model's own sample
  net, with the bounds and the admission rule of tests/test_sample_counts_gpu.py:test_full_path_matches_fp64;
* hr_render_heads on heads fixed to the fp64 oracle's net and, where the backward takes the pipeline, hr_render_backward
  against fp64 autograd (tests/test_grads_batch_gpu.py:check_render_heads), eased cases through the eased path;
* and the kernels that actually ran, read from the profiler's CUDA events, equal the cells variant_cases claims.
"""
from functools import lru_cache

import pytest
import torch

from oracle.hyperreel_oracle import HyperReelOracle
from tests.test_grads_batch_gpu import _render, _sms, check_render_heads, n_multi
from tests.test_sample_counts_gpu import check_full_path
from tests.variant_cases import SPECS, Cell, oracle_ctx, variant_case, with_rays

pytestmark = pytest.mark.gpu
NAMES = [s.name for s in SPECS]
BY_NAME = {s.name: s for s in SPECS}


@lru_cache(maxsize=4)
def _oracle(name):
    spec, case = BY_NAME[name], variant_case(name)
    st = {}
    with oracle_ctx(spec.eased):
        rgb = HyperReelOracle(case.model_cfg_plain, case.dataset, case.state_dict, dtype=torch.float64).render(case.rays.double(), st)
    return rgb, st


@pytest.mark.parametrize("mode", ["fp32", "auto"])
@pytest.mark.parametrize("name", NAMES)
def test_full_path_matches_fp64(name, mode):
    """rgb of `render` and the stages of `render_stages` with the model's own net, against the fp64 oracle on its net and on
    the kernel's own heads (check_full_path's `own_heads` rule): every stage is compared on every case, and a distance or
    point may exceed its bound only by twice the fp32 oracle's own miss on the same heads."""
    spec, case = BY_NAME[name], variant_case(name)
    want, ref = _oracle(name)
    check_full_path(case, _render(case, spec.eased, mode), want, ref, mode, f"{name} {mode}",
                    oracle_ctx=lambda: oracle_ctx(spec.eased), own_heads=True)


@pytest.mark.parametrize("name", NAMES)
def test_render_heads_and_backward_match_fp64(name):
    """hr_render_heads on the fp64 oracle's heads, and hr_render_backward where the backward takes the pipeline; where it
    does not (sphere_new, more than 64 samples), the backward refuses it."""
    spec, case = BY_NAME[name], variant_case(name)
    check_render_heads(case, False, spec.eased, name, backward=spec.bwd is not None, ties_aside=True)
    if spec.bwd is None:
        model = _render(case, spec.eased).model
        rays = case.rays[:8].cuda()
        model._ensure_uploaded(rays.device)
        refusal = "sphere_new primitive is not supported" if spec.prim == "sphere_new" else "more than 64 samples per ray"
        with pytest.raises(RuntimeError, match=refusal):
            model._render_backward(rays, torch.zeros((8, case.sig.cfg.mlp_out), device="cuda"), torch.ones((8, 3), device="cuda"),
                                   False, False)


# one case per backward family, at a batch where every warp of the backward walks several rays
MULTI = [next(s.name for s in SPECS if s.bwd is not None and s.bwd.family == fam and s.S <= 16) for fam in ("lean", "rare", "ease")]


@pytest.mark.parametrize("name", MULTI)
def test_backward_walks_several_rays_per_warp(name):
    spec = BY_NAME[name]
    n = n_multi()
    assert n > 32 * _sms()
    case = with_rays(variant_case(name), spec.src, n, seed=4000 + SPECS.index(spec))
    check_render_heads(case, False, spec.eased, f"{name} n={n}", ties_aside=True)


def _template_args(text):
    return tuple(a == "true" if a in ("true", "false") else int(a) for a in (t.strip() for t in text.split(",")))


def kernels_run(fn):
    """Template arguments of every render_kernel and render_bwd_kernel launched by fn(), from the profiler's CUDA events."""
    import re
    import time

    # The profiler now and then hands back no CUDA activity at all for a window: the kernel records of a short window can
    # still be on their way from the device when the window closes.  The window therefore stays open a moment after the
    # synchronise, and an empty window is profiled again.
    for attempt in range(8):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
            time.sleep(0.02 * (attempt + 1))
        names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
        if names:
            break
    assert names, "the profiler recorded no CUDA activity"
    fwd = {_template_args(m) for nm in names for m in re.findall(r"(?<![\w])render_kernel<([^<>]*)>", nm)}
    bwd = {_template_args(m) for nm in names for m in re.findall(r"(?<![\w])render_bwd_kernel<([^<>]*)>", nm)}
    return fwd, bwd, names


@pytest.mark.parametrize("name", NAMES)
def test_the_kernels_that_ran_are_the_claimed_cells(name):
    """The CPU restatement of the dispatch (variant_cases.forward_cell / backward_cell) against the binary: the
    render_kernel<...> of a plain render and of render_stages, and the render_bwd_kernel<...> of the backward."""
    spec, case = BY_NAME[name], variant_case(name)
    model = _render(case, spec.eased).model
    rays = case.rays.cuda()
    model._ensure_uploaded(rays.device)
    heads = torch.zeros((rays.shape[0], case.sig.cfg.mlp_out), device="cuda")
    d_rgb = torch.ones((rays.shape[0], 3), device="cuda")
    f = spec.fwd
    extra = Cell("fwd", f.family, f.spl, f.dyn, f.layout, f.shade, True, 1)
    fwd, _, names = kernels_run(lambda: model._render_heads(rays, heads, False, False))
    assert fwd == {f.template()}, (fwd, f, sorted(names))
    fwd, _, _ = kernels_run(lambda: model.render_stages(rays))
    assert fwd == {extra.template()}, (fwd, extra)
    if spec.bwd is not None:
        _, bwd, _ = kernels_run(lambda: model._render_backward(rays, heads, d_rgb, False, False))
        assert bwd == {spec.bwd.template()}, (bwd, spec.bwd)
