"""The render path at every sample-count edge the lowering admits, against the fp64 oracle.

Every other test renders a multiple of 4 samples per ray.  The render kernels pad the lanes past S (+inf sort keys, alpha = 0,
a1 = 1), may run a partly empty gather round, and change variant at S = 16/17, 32/33, 64/65 and 128/129; the backward changes
samples per lane at 32/33 and refuses S > 64.  With the built-ins' 15 head channels per sample an S that is not a multiple of 4
also gives a head row that is not a multiple of 4 wide, which the tensor-core sample net stores with its narrow store and the
training backward pads.  Cases: tests/sweep_cases.py (each one asserts that it has rays to sort, masked samples and samples
outside the AABB).
"""
import contextlib
from functools import lru_cache

import pytest
import torch

from oracle.hyperreel_oracle import HyperReelOracle
from tests.sweep_cases import BWD_MAX_SAMPLES, SAMPLE_COUNTS, SWEEP_BUILTINS, guard_ok, guard_stats, sweep_case
from tests.test_grads_batch_gpu import check_render_heads
from tests.test_parity_gpu import RGB_TOL, make_render
from tests.test_train_net_tc_sizes_gpu import check_case

pytestmark = pytest.mark.gpu
SWEEP = [(b, S) for b in SWEEP_BUILTINS for S in SAMPLE_COUNTS]
IDS = [f"{b}-s{S}" for b, S in SWEEP]
OFF_RAYS = 256


@lru_cache(maxsize=None)
def _oracle(builtin, S):
    case = sweep_case(builtin, S)
    st = {}
    rgb = HyperReelOracle(case.model_cfg_plain, case.dataset, case.state_dict, dtype=torch.float64).render(case.rays.double(), st)
    return rgb, st


@pytest.mark.parametrize("builtin,S", SWEEP, ids=IDS)
def test_render_heads_and_backward_match_fp64(builtin, S):
    """hr_render_heads on heads fixed to the fp64 oracle's net (rounded to fp32) at every S -- hr_render_heads has no 64-sample
    limit -- and hr_render_backward's d heads and table gradients up to 64 samples, with the rules of
    test_render_backward_matches_fp64_at_batch_size."""
    case = sweep_case(builtin, S)
    assert guard_ok(guard_stats(case), S), "the case no longer exercises the sort, the sample mask and the AABB"
    check_render_heads(case, False, False, f"{builtin} S={S}", backward=S <= BWD_MAX_SAMPLES,
                       few_samples=S <= 2, ties_aside=True)


@pytest.mark.parametrize("mode", ["fp32", "auto"])
@pytest.mark.parametrize("builtin,S", SWEEP, ids=IDS)
def test_full_path_matches_fp64(builtin, S, mode):
    """render and render_stages with the model's own sample net: rgb within RGB_TOL of the fp64 oracle, the stages within the
    bounds of tests/test_widened_gpu.py (the heads of the tensor-core net within its 1e-4), on every ray but those admitted
    below."""
    case = sweep_case(builtin, S)
    want, ref = _oracle(builtin, S)
    check_full_path(case, make_render(case, mlp_mode=mode).cuda(), want, ref, mode, f"{builtin} S={S} {mode}")


def check_full_path(case, render, want, ref, mode, label, oracle_ctx=contextlib.nullcontext, own_heads=False):
    """`render`'s rgb and render_stages against the fp64 oracle's rgb `want` and stages `ref` (rendered within
    `oracle_ctx()`), with the bounds and the admission rule of test_full_path_matches_fp64.

    `own_heads`: the render is also held to the fp64 oracle run on the kernel's own heads (which are held to the oracle's
    net within heads_tol), so that the render kernel is compared with nothing between them.  Its rgb must then be within
    RGB_TOL of that oracle on every ray, so the admitted rays need no cap.  The stages are compared with that oracle too.
    A sample's distance (and point) may miss the 1e-5 (2e-5) bound by twice what the fp32 oracle on the same heads misses
    it by: that is the intersection's own conditioning.  The deformable planes put distances of up to 21 000 on rays
    nearly parallel to a plane, and there the fp32 oracle misses the fp64 oracle by up to 49 times the bound.  On every
    case of tests/test_kernel_variants_gpu.py the kernel's distances equal the fp32 oracle's to the printed digits, and
    stay within 0.5 of the allowance."""
    rays = case.rays.cuda()
    n = rays.shape[0]
    rgb = render(rays)["rgb"].cpu().double()
    st = {k: v.cpu().double() for k, v in render.model.render_stages(rays).items()}
    heads_tol = 2e-5 if mode == "fp32" else 1e-4
    assert float((st["mlp_out"] - ref["mlp_out"]).abs().max()) <= heads_tol * max(1.0, float(ref["mlp_out"].abs().max()))
    own = own32 = None
    if own_heads:
        own, own32 = {}, {}
        with oracle_ctx():
            for dt, out in ((torch.float64, own), (torch.float32, own32)):
                orc = HyperReelOracle(case.model_cfg_plain, case.dataset, case.state_dict, dtype=dt)
                orc.sample_net = lambda r: st["mlp_out"].to(r.dtype)
                out["rgb"] = orc.render(case.rays.to(dt), out)
        own_err = (rgb - own["rgb"].double()).abs().max(-1).values
        assert float(own_err.max()) <= RGB_TOL, f"rays {(own_err > RGB_TOL).nonzero().flatten().tolist()} off the oracle on own heads"
    # A ray off by more than RGB_TOL is admitted only when the fp64 oracle on the kernel's own heads (held to heads_tol above)
    # renders what the kernel renders: a sample that sits on the sample mask or an AABB face within the heads' rounding is
    # in or out as a whole.  At most one per OFF_RAYS rays, unless every ray is held to the oracle on its own heads.
    off = ((rgb - want).abs().max(-1).values > RGB_TOL).nonzero().flatten().tolist()
    if off:
        with oracle_ctx():
            orc = HyperReelOracle(case.model_cfg_plain, case.dataset, case.state_dict, dtype=torch.float64)
            orc.sample_net = lambda r: st["mlp_out"][off].to(r.dtype)
            on_own = orc.render(case.rays[off].double())
        print(f"\n[{label}] rays {off} off the oracle by {float((rgb[off] - want[off]).abs().max()):.2e}, "
              f"by {float((rgb[off] - on_own).abs().max()):.2e} from the oracle on the kernel's heads")
        assert float((rgb[off] - on_own).abs().max()) <= RGB_TOL
        assert own_heads or len(off) <= max(1, n // OFF_RAYS)
    keep = torch.ones(n, dtype=torch.bool)
    keep[off] = False
    assert float((rgb[keep] - want[keep]).abs().max()) <= RGB_TOL
    assert float((st["rgb"] - rgb).abs().max()) <= RGB_TOL
    if own_heads:
        ref = own
    d = ref["distances"].reshape(n, -1)
    p = ref["points"].reshape(n, -1)
    d_tol = torch.full_like(d, 1e-5 * max(1.0, float(d.abs().max())))
    p_tol = torch.full_like(p, 2e-5 * max(1.0, float(p.abs().max())))
    if own_heads:  # the intersection's conditioning, measured by the fp32 oracle on the same heads
        d_tol += 2.0 * (own32["distances"].reshape(n, -1).double() - d).abs()
        p_tol += 2.0 * (own32["points"].reshape(n, -1).double() - p).abs()
    assert bool(((st["distances"] - d).abs() <= d_tol)[keep].all()), float(((st["distances"] - d).abs() / d_tol)[keep].max())
    assert bool(((st["points"].reshape(n, -1) - p).abs() <= p_tol)[keep].all()), \
        float(((st["points"].reshape(n, -1) - p).abs() / p_tol)[keep].max())
    assert float((st["sigma"] - ref["sigma"])[keep].abs().max()) <= 1e-4 * max(1.0, float(ref["sigma"].abs().max()))
    assert float((st["weights"] - ref["weights"])[keep].abs().max()) <= 5e-5


@pytest.mark.parametrize("builtin,S", [(b, S) for b, S in SWEEP if S <= BWD_MAX_SAMPLES],
                         ids=[i for (b, S), i in zip(SWEEP, IDS) if S <= BWD_MAX_SAMPLES])
def test_training_net_on_the_tensor_cores(builtin, S):
    """train_net="tc": the training forward's heads equal the render net's bit for bit, and every layer gradient stays within
    the magnitude bound of tests/test_train_net_tc_sizes_gpu.py -- including head rows that are not a multiple of 4 wide."""
    check_case(sweep_case(builtin, S), f"{builtin} S={S}")


@pytest.mark.parametrize("builtin", SWEEP_BUILTINS)
def test_backward_refuses_more_than_64_samples(builtin):
    case = sweep_case(builtin, BWD_MAX_SAMPLES + 1)
    model = make_render(case).cuda().model
    rays = case.rays[:8].cuda()
    model._ensure_uploaded(rays.device)
    heads = torch.zeros((8, case.sig.cfg.mlp_out), device="cuda")
    with pytest.raises(RuntimeError, match="more than 64 samples per ray"):
        model._render_backward(rays, heads, torch.ones((8, 3), device="cuda"), False, False)
