"""The render path at every sample-count edge the lowering admits, against the fp64 oracle.

Every other test renders a multiple of 4 samples per ray.  The render kernels pad the lanes past S (+inf sort keys, alpha = 0,
a1 = 1), may run a partly empty gather round, and change variant at S = 16/17, 32/33, 64/65 and 128/129; the backward changes
samples per lane at 32/33 and refuses S > 64.  With the built-ins' 15 head channels per sample an S that is not a multiple of 4
also gives a head row that is not a multiple of 4 wide, which the tensor-core sample net stores with its narrow store and the
training backward pads.  Cases: tests/sweep_cases.py (each one asserts that it has rays to sort, masked samples and samples
outside the AABB).
"""
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
    render = make_render(case, mlp_mode=mode).cuda()
    rays = case.rays.cuda()
    n = rays.shape[0]
    rgb = render(rays)["rgb"].cpu().double()
    st = {k: v.cpu().double() for k, v in render.model.render_stages(rays).items()}
    heads_tol = 2e-5 if mode == "fp32" else 1e-4
    # A ray off by more than RGB_TOL is admitted only when the fp64 oracle on the kernel's own heads (held to heads_tol below)
    # renders what the kernel renders: a sample that sits on the sample mask or an AABB face within the heads' rounding is
    # in or out as a whole.  At most one per OFF_RAYS rays.
    off = ((rgb - want).abs().max(-1).values > RGB_TOL).nonzero().flatten().tolist()
    if off:
        orc = HyperReelOracle(case.model_cfg_plain, case.dataset, case.state_dict, dtype=torch.float64)
        orc.sample_net = lambda r: st["mlp_out"][off].to(r.dtype)
        on_own = orc.render(case.rays[off].double())
        print(f"\n[{builtin} S={S} {mode}] rays {off} off the oracle by {float((rgb[off] - want[off]).abs().max()):.2e}, "
              f"by {float((rgb[off] - on_own).abs().max()):.2e} from the oracle on the kernel's heads")
        assert float((rgb[off] - on_own).abs().max()) <= RGB_TOL
        assert len(off) <= max(1, n // OFF_RAYS)
    keep = torch.ones(n, dtype=torch.bool)
    keep[off] = False
    assert float((rgb[keep] - want[keep]).abs().max()) <= RGB_TOL
    assert float((st["rgb"] - rgb).abs().max()) <= RGB_TOL
    assert float((st["mlp_out"] - ref["mlp_out"]).abs().max()) <= heads_tol * max(1.0, float(ref["mlp_out"].abs().max()))
    d = ref["distances"].reshape(n, -1)
    assert float((st["distances"] - d)[keep].abs().max()) <= 1e-5 * max(1.0, float(d.abs().max()))
    p = ref["points"].reshape(n, -1)
    assert float((st["points"].reshape(n, -1) - p)[keep].abs().max()) <= 2e-5 * max(1.0, float(p.abs().max()))
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
