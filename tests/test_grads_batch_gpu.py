"""The render backward (hr_render_backward) at training batch sizes against fp64 autograd, with the sample net taken out of
the loop.

The backward kernel walks rays grid-stride, `kBwdWarps` = 4 warps per CTA and at most 8 CTAs per SM, so a batch of more than
32 rays per SM gives each warp several rays: the per-warp shared buffers (shading matrix, SH row, sort inverse) are rewritten
for the next ray and the CTA's basis and colour-transform sums accumulate over many rays before they are flushed.  Training
runs 16 384 to 65 536 rays per step, so these tests run batches of 3 * 32 * SMs + 37 and 65 536 rays, and 1 and 5 rays (CTAs
whose warps get no ray still flush their sums).

The heads are computed once by the fp64 oracle's sample net and rounded to fp32: the GPU, the fp64 oracle and the fp32 oracle
then see bit-identical heads, and the comparison is blind to the sample net and its LeakyReLU kinks.  The fp32 oracle measures
how well conditioned each ray is: on nearly opaque rays (alpha close to 1) the reference's own fp32 arithmetic loses most of
the digits of d heads, and the kernel may be no worse than it there.
"""
import contextlib

import pytest
import torch

import hyperreel_b200 as hb
from hyperreel_b200 import rays as rays_mod
from oracle.hyperreel_oracle import HyperReelOracle
from tests.cases import build_case
from tests.cases_train import TRAIN_CASES, build_train_case
from tests.ease_cases import ITERS_PER_EPOCH, eased_oracle
from tests.test_parity_gpu import make_render

BWD_WARPS, BWD_CTAS_PER_SM = 4, 8  # hr_render_bwd_kernel.cuh: kBwdWarps, the grid cap of bwd_launch_one
EASE_ITER = 6000  # both eased density heads mid-window (tests/ease_cases.py)
TOL_RGB = 2e-5
MISMATCH_RAYS = 32768  # at most one ray straddling the sample mask per this many rays
FACE_ULPS = 4.0  # how far (fp32 ulps) mask_moved moves the AABB faces
TOL_HEADS = 1e-3  # of max |d heads| (fp64)
TOL_TABLE = 2e-3  # of max |d table| (fp64)
MAX_ILL = 0.01  # fraction of rays on which the fp32 reference itself is off by more than TOL_HEADS
TIE_ULPS = 16.0  # sort keys this close (fp32 ulps of max(|key|, 1)) have no defined order
TOL_ADD = 2e-4  # additivity over a split of the batch, of max |d table|


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def n_multi():
    """Three rays per warp and a ragged last round."""
    return 3 * 32 * _sms() + 37


def bwd_warps(n):
    """Warps of the backward grid for n rays (bwd_launch_one)."""
    ctas = min(max((n + BWD_WARPS - 1) // BWD_WARPS, 1), BWD_CTAS_PER_SM * _sms())
    return ctas * BWD_WARPS


def _case(name, n):
    """A case with n rays: tests/cases.py's rays of that count, or a shipped YAML of tests/cases_train.py with rays of the
    pipeline's layout (spread over every camera of a colour transform), flipped like the fixture's."""
    name = name[len("ease_"):] if name.startswith("ease_") else name
    spec = TRAIN_CASES.get(name, {"builtin": True})
    if spec.get("builtin"):
        return build_case(name, n=n)
    case = build_train_case(name)
    rays = rays_mod.for_signature(case.sig, n, seed=301)
    if spec.get("flip"):
        rays[:, 2] = 0.0
        rays[:, 5] = -rays[:, 5]
    case.rays = rays
    return case


def _render(case, eased, mlp_mode="fp32"):
    if not eased:
        return make_render(case, mlp_mode=mlp_mode).cuda()
    model = hb.LightfieldModel(case.model_cfg, dataset=case.dataset, iters_per_epoch=ITERS_PER_EPOCH, ease="reference",
                               mlp_mode=mlp_mode)
    render = hb.RenderLightfield(model, None, case.model_cfg.render, net_chunk=1 << 20)
    render.load_state_dict(case.state_dict, strict=False)
    render.cuda().eval()
    render.model.set_iter(EASE_ITER)
    return render


def grad_names(render):
    """Names of the tensors _render_backward returns, in its order (render_differentiable's `params`)."""
    model = render.model
    tn = model.color_model.net
    dplane, dsecond, aplane, asecond = tn.tables()
    params = [t for t in list(dplane) + list(aplane) + list(dsecond) + list(asecond) if t.numel() > 0] + [tn.basis_mat.weight]
    if model.sig.cfg.n_color_views > 0:
        params.append(model.embedding_model.embeddings[model.sig.color_embedding_index].color_embedding)
    by_id = {id(p): k for k, p in render.named_parameters()}
    return [by_id[id(p)] for p in params]


def mask_moved(case, heads, i, white, eased):
    """fp64 rgb of ray i with the AABB moved outwards and inwards by FACE_ULPS fp32 ulps of its faces: a sample that lies that
    close to a face changes sides of the colour net's `valid` mask, every other sample keeps its side."""
    key = "model.color_model.net.aabb"
    aabb = case.state_dict[key].double()
    out = []
    for sign in (1.0, -1.0):
        sd = dict(case.state_dict)
        sd[key] = (aabb + sign * torch.tensor([[-1.0], [1.0]], dtype=torch.float64) * FACE_ULPS * torch.finfo(torch.float32).eps
                   * aabb.abs().clamp(min=1.0)).to(case.state_dict[key].dtype)
        orc = HyperReelOracle(case.model_cfg_plain, case.dataset, sd, dtype=torch.float64)
        orc.sample_net = lambda rays: heads[i:i + 1].to(rays.dtype)
        with eased_oracle(EASE_ITER) if eased else contextlib.nullcontext():
            rgb, _ = orc.render_with_grad(case.rays[i:i + 1].clone(), clamp=False, white_bg=white)
        out.append(rgb.detach()[0])
    return out


def fixed_heads(case):
    """The fp64 oracle's sample-net output, rounded to fp32."""
    orc = HyperReelOracle(case.model_cfg_plain, case.dataset, case.state_dict, dtype=torch.float64)
    with torch.no_grad():
        return orc.sample_net(case.rays.double()).float()


def oracle_grads(case, heads, d_rgb, white, dtype):
    """(rgb, d heads, {name: d name}, the colour net's stages: weights, points, distances) of the oracle in `dtype` on the
    given heads: training semantics (no clamp), the loss (rgb * d_rgb).sum()."""
    orc = HyperReelOracle(case.model_cfg_plain, case.dataset, case.state_dict, dtype=dtype)
    orc.sample_net = lambda rays: heads.to(rays.dtype)
    stages = {}
    color = orc.color
    orc.color = lambda x, _stages, **kw: color(x, stages, **kw)
    rgb, leaves = orc.render_with_grad(case.rays.clone(), clamp=False, white_bg=white, heads_leaf=True)
    (rgb * d_rgb.to(dtype)).sum().backward()
    grads = {k: v.grad for k, v in leaves.items() if k != "_mlp_out" and v.grad is not None}
    return rgb.detach(), leaves["_mlp_out"].grad, grads, {k: stages[k].detach() for k in ("weights", "points", "distances",
                                                                                          "unsorted_distances") if k in stages}


def _oracles(case, heads, d_rgb, white, eased):
    if not eased:
        return [oracle_grads(case, heads, d_rgb, white, dt) for dt in (torch.float64, torch.float32)]
    with eased_oracle(EASE_ITER):
        return [oracle_grads(case, heads, d_rgb, white, dt) for dt in (torch.float64, torch.float32)]


def test_injected_heads_reproduce_the_fp64_oracle_and_agree_with_fp32():
    """The head injection itself, on a well-conditioned case: the fp64 oracle on the rounded heads renders what the plain
    fp64 oracle renders, and its d heads and table gradients agree with the fp32 oracle's on the same heads."""
    case = _case("neural3d_s16", 300)
    heads = fixed_heads(case)
    assert heads.dtype == torch.float32 and heads.shape == (300, case.sig.cfg.mlp_out)
    d_rgb = torch.randn(300, 3, generator=torch.Generator().manual_seed(1))
    (rgb64, dh64, g64, st64), (rgb32, dh32, g32, _) = _oracles(case, heads, d_rgb, False, False)
    acc = st64["weights"].sum(-1)
    plain = HyperReelOracle(case.model_cfg_plain, case.dataset, case.state_dict, dtype=torch.float64)
    plain_rgb, _ = plain.render_with_grad(case.rays.clone(), clamp=False, white_bg=False)
    assert float((rgb64 - plain_rgb.detach()).abs().max()) <= 1e-5
    assert float((acc > 0.5).float().mean()) >= 0.25
    assert dh64.dtype == torch.float64 and dh64.shape == heads.shape
    assert float((dh32.double() - dh64).abs().max()) <= 1e-4 * float(dh64.abs().max())
    assert g64.keys() == g32.keys() and len(g64) >= 7
    for k, ref in g64.items():
        scale = float(ref.abs().max())
        assert scale > 0.0, k
        assert float((g32[k].double() - ref).abs().max()) <= 1e-4 * scale, k


# (case, rays, white background); "multi" = n_multi()
BATCH_CASES = [
    ("technicolor_app", "multi", False),    # lean, RGB shading
    ("technicolor_app", 65536, True),
    ("neural3d_app", "multi", False),       # SH shading, three VM groups
    ("donerf_app", "multi", True),
    ("donerf_app", 1, False),
    ("donerf_app", 5, False),
    ("neural3d_s16", "multi", False),       # two rays per warp in the forward, one in the backward
    ("neural3d_s16", "multi", True),
    ("technicolor_s8", "multi", False),
    ("donerf_s16", "multi", False),
    ("technicolor_bbox", "multi", False),   # RARE: bbox contraction
    ("donerf_voxel", "multi", False),       # RARE: voxel grid
    ("immersive_z_plane", 65536, False),    # RARE: per-camera colour transform over every camera
    ("ease_neural3d_app", "multi", False),  # EASE: the density heads eased mid-window
]


@pytest.mark.gpu
@pytest.mark.parametrize("name,n,white", BATCH_CASES, ids=[f"{c}-{n}-{'white' if w else 'black'}" for c, n, w in BATCH_CASES])
def test_render_backward_matches_fp64_at_batch_size(name, n, white):
    n = n_multi() if n == "multi" else n
    if n == n_multi():
        assert n > 32 * _sms()  # every warp of the backward walks several rays
    check_render_heads(_case(name, n), white, name.startswith("ease_"), f"{name} n={n} white={white}")


def tied_rays(keys):
    """Rays two of whose sort keys lie within TIE_ULPS fp32 ulps of max(|key|, 1) of each other but are not equal: their order
    is decided by the last bits of the arithmetic, and with it which of the two samples each sorted slot's gradient goes back
    to.  (Equal keys -- masked samples at t = 0, samples that miss the same primitive -- are the same value on both sides.)"""
    k = torch.sort(keys, dim=-1).values
    gap = k[:, 1:] - k[:, :-1]
    tie = (gap > 0.0) & (gap <= TIE_ULPS * torch.finfo(torch.float32).eps * k[:, 1:].abs().clamp(min=1.0))
    return tie.any(-1).nonzero().flatten()


def check_render_heads(case, white, eased, label, backward=True, few_samples=False, ties_aside=False):
    """hr_render_heads on the fixed heads against the fp64 oracle and, with `backward`, hr_render_backward against fp64
    autograd, with the rules below.  `few_samples`: one or two samples per ray, where most rays may be transparent and a
    density table's gradient may vanish exactly (alpha = 1 whatever the density, on a ray's last sample).  `ties_aside`: rays
    with tied sort keys (tied_rays) are left out of the backward comparison like the rays that straddle the sample mask."""
    n = case.rays.shape[0]
    heads = fixed_heads(case)
    d_rgb = torch.randn(n, 3, generator=torch.Generator().manual_seed(n + 17))
    (rgb64, dh64, g64, st64), (rgb32, dh32, g32, _) = _oracles(case, heads, d_rgb, white, eased)

    render = _render(case, eased)
    model = render.model
    rays = case.rays.cuda()
    model._ensure_uploaded(rays.device)
    rgb = model._render_heads(rays, heads.cuda(), False, white)

    # rgb: within 2e-5, or within twice the fp32 reference's own error on the rays where that is larger.  A ray off by more
    # is admitted only when it straddles the sample mask: moving the AABB's faces by FACE_ULPS fp32 ulps in the fp64 reference
    # gives the GPU's rgb, so a sample lies on a face and a one-ulp difference in the point arithmetic flips its `valid` bit,
    # adding or dropping a whole sample.  At most one per MISMATCH_RAYS rays, each rendering the same value alone as in the
    # batch; they are listed and left out of the backward comparison (d_rgb zeroed on both sides).
    rgb_err = ((rgb.cpu().double() - rgb64).abs() - 2.0 * (rgb32.double() - rgb64).abs()).max(-1).values
    mismatch = (rgb_err > TOL_RGB).nonzero().flatten()
    for i in mismatch.tolist():
        moved = min(float((rgb[i].cpu().double() - m).abs().max()) for m in mask_moved(case, heads, i, white, eased))
        print(f"\n[{label}] ray {i} straddles the sample mask: {rgb[i].tolist()} vs {rgb64[i].tolist()}, "
              f"{moved:.2e} from the reference with the AABB moved")
        assert moved <= TOL_RGB, f"ray {i} is off the reference by {float(rgb_err[i])}, and not by a sample on an AABB face"
        alone = model._render_heads(rays[i:i + 1].contiguous(), heads[i:i + 1].cuda(), False, white)
        assert torch.equal(alone[0], rgb[i]), f"ray {i} renders differently alone"
    assert len(mismatch) <= n // MISMATCH_RAYS, f"{len(mismatch)} rays off the reference by up to {float(rgb_err.max())}"
    if not backward:
        return
    if ties_aside:
        tied = tied_rays(st64["unsorted_distances"])
        print(f"\n[{label}] {len(tied)} rays with tied sort keys left out of the backward comparison")
        assert len(tied) <= MAX_ILL * n, f"{len(tied)} of {n} rays have tied sort keys"
        mismatch = torch.cat([mismatch, tied])
    if len(mismatch):
        d_rgb[mismatch] = 0.0
        (rgb64, dh64, g64, st64), (rgb32, dh32, g32, _) = _oracles(case, heads, d_rgb, white, eased)
    acc = st64["weights"].sum(-1)
    d_heads, grads = model._render_backward(rays, heads.cuda(), d_rgb.cuda(), False, white)
    names = grad_names(render)
    assert len(names) == len(grads)
    assert few_samples or float((acc > 0.5).float().mean()) >= 0.25, "the case is nearly transparent"

    # d heads, per ray
    scale = float(dh64.abs().max())
    assert scale > 0.0
    err = (d_heads.cpu().double() - dh64).abs().max(-1).values
    cond = (dh32.double() - dh64).abs().max(-1).values
    ill = cond > TOL_HEADS * scale
    bound = torch.where(ill, 2.0 * cond, torch.zeros_like(cond)) + TOL_HEADS * scale
    bad = (err > bound).nonzero().flatten()
    nw = bwd_warps(n)
    first, later = bad[bad < nw].tolist(), bad[bad >= nw].tolist()
    well_frac = float((err[~ill] / (TOL_HEADS * scale)).max()) if bool((~ill).any()) else 0.0
    print(f"\n[{label}] ill-conditioned rays {int(ill.sum())}/{n}, "
          f"largest well-conditioned d heads error {well_frac:.3f} of the tolerance")
    assert not first and not later, (f"d heads: {len(first)} failing rays of a warp's first round (first {first[:5]}), "
                                     f"{len(later)} of later rounds (first {later[:5]})")
    assert int(ill.sum()) <= MAX_ILL * n, f"{int(ill.sum())} of {n} rays are ill-conditioned"

    # tables, basis and colour transform, per entry
    assert len(names) >= 4
    if case.sig.cfg.n_color_views > 0:
        assert names[-1].endswith("color_embedding")
    for k, g in zip(names, grads):
        assert k in g64, k
        ref, ref32 = g64[k], g32[k].double()
        tscale = float(ref.abs().max())
        if few_samples and tscale == 0.0:
            assert float(g.abs().max()) == 0.0, k
            continue
        assert tscale > 0.0, k
        assert float(g.abs().max()) > 0.0, k
        diff = (g.cpu().double() - ref).abs()
        tol = TOL_TABLE * tscale + 2.0 * (ref32 - ref).abs()
        worst = float((diff - tol).max())
        assert worst <= 0.0, f"{k}: {int((diff > tol).sum())} entries out of tolerance, worst error {float(diff.max())} vs max {tscale}"

    # additivity: the batch against [0, nwarps) and [nwarps, n), each in its own call, where every warp of the first call
    # has one ray; d heads are per ray and must be bit for bit those of the whole batch
    if n > nw:
        parts = [model._render_backward(rays[a:b].contiguous(), heads[a:b].cuda(), d_rgb[a:b].cuda(), False, white)
                 for a, b in ((0, nw), (nw, n))]
        assert torch.equal(torch.cat([parts[0][0], parts[1][0]]), d_heads)
        for i, (k, g) in enumerate(zip(names, grads)):
            s = parts[0][1][i] + parts[1][1][i]
            assert float((s - g).abs().max()) <= TOL_ADD * float(g.abs().max()), k
