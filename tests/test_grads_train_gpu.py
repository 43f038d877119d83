"""Training the pipelines whose backward runs on the RARE variants of the render backward (bbox / z_depth contraction,
per-ray colour heads, the per-camera colour transform, voxel-grid and deformable-plane primitives) on the GPU: gradients
against the reference's own autograd (tests/golden/grads_<case>.npz of tests/cases_train.py) and against the gradient oracle
with training semantics, which shipped model YAMLs train and which refuse, and INRSystem.training_step end to end."""
import os

import numpy as np
import pytest
import torch

import hyperreel_b200 as hb
from hyperreel_b200.state import seeded_state_dict
from oracle.hyperreel_oracle import HyperReelOracle
from tests.cases_train import PARAM_SEED, TRAIN_CASES, build_train_case
from tests.golden.make_golden_grads import probe_indices, target_for
from tests.test_parity_gpu import make_render
from tests.test_shipped_yaml_golden import SHIPPED, load_fixture

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
COLOR_EMB = "color_embedding"
# The sample net's LeakyReLU has a kink at 0.  A pre-activation within fp32 rounding of 0 may land on either side of it in the
# reference (CPU fp32) and on the GPU (cuBLAS fp32): both derivatives are right, and they differ by a factor of 100 for that
# (ray, unit), which moves the gradients of every layer below it.  Measured on one H100 for donerf_voxel: the GPU's
# pre-activations differ from fp64 by at most 2.2e-7, and layer 1 of ray 19 has one at +1.9e-8 (fp64) that the GPU computes as
# -1.9e-8.  So for every pre-activation within KINK of 0 (fp64), both sides are admitted: the sample-net gradients may differ
# from the reference by exactly what moving those units across the kink changes, computed in fp64 (`kink_moves`).
KINK = 1e-6
NET = "model.embedding_model.embeddings.0.net."


def kink_moves(orc, rays, d_heads):
    """Possible differences of the sample-net parameter gradients between two fp32 computations that put the pre-activations
    within KINK of 0 on different sides of the kink: {name: grad(sides a) - grad(sides b)} for every pair of side choices
    (the zero difference included)."""
    import itertools

    from oracle.hyperreel_oracle import _get, ray_param, windowed_pe

    net = orc.pred["net"]
    if net["type"] == "zero":
        return [{}]
    rays = rays.double()
    x = torch.cat([windowed_pe(_get(p, "pe"), ray_param(p["param"], rays[:, p["start"]:p["end"]])) for p in orc.pred["params"].values()], -1)
    depth, skips = net["depth"], list(_get(net, "skips", []))
    names = [f"{NET}layers.{i}" + ("" if i == depth - 1 else ".0") for i in range(depth)]
    params = {f"{n}.{t}": orc.sd[f"{n}.{t}"].double().requires_grad_(True) for n in names for t in ("weight", "bias")}

    def grads(flip):  # flip: per hidden layer, a bool mask of the units moved to the other side of the kink
        inp, h = x, x
        for i, n in enumerate(names):
            if i in skips:
                h = torch.cat([inp, h], -1)
            h = h @ params[f"{n}.weight"].t() + params[f"{n}.bias"]
            if i < depth - 1:
                h = torch.where((h > 0) != flip[i], h, 0.01 * h)
        g = torch.autograd.grad((h * d_heads.double()).sum(), list(params.values()))
        return dict(zip(params, g))

    # the units within KINK of 0
    with torch.no_grad():
        inp, h, near = x, x, []
        for i, n in enumerate(names[:-1]):
            if i in skips:
                h = torch.cat([inp, h], -1)
            h = h @ params[f"{n}.weight"].t() + params[f"{n}.bias"]
            near.append(h.abs() < KINK)
            h = torch.where(h > 0, h, 0.01 * h)
    units = [(i, int(r), int(u)) for i, m in enumerate(near) for r, u in m.nonzero()]
    assert len(units) <= 3, units
    sides = []
    for bits in itertools.product([False, True], repeat=len(units)):
        flip = [torch.zeros_like(m) for m in near]
        for (i, r, u), b in zip(units, bits):
            flip[i][r, u] = b
        sides.append(grads(flip))
    return [{k: (a[k] - b[k]).float() for k in a} for a in sides for b in sides]


def _min_err(got, ref, k, moves):
    """max |got - ref - move| for the admitted kink move that fits best."""
    return min(float((got - ref - m[k].reshape(got.shape) if k in m else got - ref).abs().max()) for m in moves)


def _loss(rgb, n):
    return ((rgb - target_for(n).to(rgb.device)) ** 2).mean()


@pytest.mark.parametrize("name", list(TRAIN_CASES))
def test_training_case_gradients_match_reference_autograd(name):
    """Same tolerances as tests/test_grads_gpu.py::test_parameter_gradients_match_reference_autograd."""
    g = np.load(os.path.join(GOLDEN, f"grads_{name}.npz"))
    case = build_train_case(name)
    rays = case.rays.clone().cuda()
    render = make_render(case).cuda()
    rgb = render.model.render_differentiable(rays, clamp_output=True)  # eval-mode forward, like the golden
    loss = _loss(rgb, rays.shape[0])
    loss.backward()
    assert abs(float(loss) - float(g["loss"])) <= 1e-5
    orc = HyperReelOracle(case.model_cfg_plain, case.dataset, case.state_dict)
    rgb_h, leaves_h = orc.render_with_grad(case.rays.clone(), heads_leaf=True)
    _loss(rgb_h, rays.shape[0]).backward()
    moves = kink_moves(orc, case.rays, leaves_h["_mlp_out"].grad)
    named = dict(render.named_parameters())
    keys = [k[len("norm/"):] for k in g.files if k.startswith("norm/")]
    assert len(keys) >= 17
    if case.sig.cfg.n_color_views > 0:
        assert any(k.endswith(COLOR_EMB) for k in keys)
    for k in keys:
        assert k in named, k
        grad = named[k].grad
        assert grad is not None, k
        assert float(g[f"norm/{k}"]) > 0.0, k
        scale = float(g[f"max/{k}"]) + 1e-12
        ok = False
        for m in moves:  # the GPU's gradient with its kink sides moved to some admitted choice
            flat = (grad.cpu() - m[k].reshape(grad.shape) if k in m else grad.cpu()).reshape(-1)
            probe = flat[probe_indices(flat.numel())].numpy()
            ok = ok or (abs(float(flat.norm()) - float(g[f"norm/{k}"])) <= 2e-3 * float(g[f"norm/{k}"]) + 1e-9
                        and np.abs(probe - g[f"probe/{k}"]).max() <= 1e-3 * scale + 1e-10)
        assert ok, k


@pytest.mark.parametrize("name", list(TRAIN_CASES))
@pytest.mark.parametrize("white", [False, True])
def test_training_case_gradients_match_the_oracle(name, white):
    """training_step semantics (no clamp, white background or not): every parameter tensor, the colour transform's table
    included, and d loss / d (sample-net output), entry by entry against the oracle's autograd, each within 2e-3 of the
    tensor's largest entry; the sample-net layers up to the admitted kink moves (KINK above)."""
    case = build_train_case(name)
    rays = case.rays.clone()
    orc = HyperReelOracle(case.model_cfg_plain, case.dataset, case.state_dict)
    rgb_h, leaves_h = orc.render_with_grad(rays, clamp=False, white_bg=white, heads_leaf=True)
    _loss(rgb_h, rays.shape[0]).backward()
    rgb_o, leaves = orc.render_with_grad(rays, clamp=False, white_bg=white)
    _loss(rgb_o, rays.shape[0]).backward()
    render = make_render(case).cuda()
    render.train()
    rgb, heads = render.model.render_differentiable(rays.cuda(), white_bg=white, return_heads=True)
    heads.retain_grad()
    assert float((rgb.detach().cpu() - rgb_o.detach()).abs().max()) <= 2e-5
    _loss(rgb, rays.shape[0]).backward()
    ref_h = leaves_h["_mlp_out"].grad
    assert float(ref_h.abs().max()) > 0.0
    err_h = float((heads.grad.cpu() - ref_h).abs().max())
    assert err_h <= 2e-3 * float(ref_h.abs().max()), f"d loss / d heads: {err_h} vs {float(ref_h.abs().max())}"
    moves = kink_moves(orc, rays, ref_h)
    compared = []
    for k, p in render.named_parameters():
        if p.numel() == 0 or k not in leaves or leaves[k].grad is None:
            continue
        ref = leaves[k].grad
        scale = float(ref.abs().max())
        assert scale > 0.0, k
        assert p.grad is not None, k
        err = _min_err(p.grad.cpu(), ref, k, moves)
        assert err <= 2e-3 * scale, f"{k}: {err} vs scale {scale}"
        compared.append(k)
    assert len(compared) >= 17
    if case.sig.cfg.n_color_views > 0:
        assert any(k.endswith(COLOR_EMB) for k in compared)


BY_NAME = {os.path.basename(p)[:-4]: p for p in SHIPPED}
REFUSED = {"bom_sphere", "immersive_sphere_new", "catacaustics_voxel", "neural_3d_z_plane_static", "technicolor_z_plane_no_sample",
           "shiny_z_plane_cascaded", "shiny_z_plane_feedback", "shiny_z_tensorf_cascaded", "technicolor_cascaded"}


def test_which_shipped_yamls_train():
    """loss.backward() runs for 36 of the 45 shipped model YAMLs; the other 9 (sphere_new, learned sphere origins, cascaded
    pipelines, more than 64 samples per ray) refuse with an error."""
    trained, refused = set(), set()
    for name, path in BY_NAME.items():
        plain, cfg, ds, sig, sd, rays, rgb = load_fixture(path)
        model = hb.LightfieldModel(cfg, dataset=ds, mlp_mode="fp32")
        render = hb.RenderLightfield(model, None, cfg.render, net_chunk=1 << 20)
        render.load_state_dict(sd, strict=False)
        render.cuda().train()
        try:
            render.model.render_differentiable(rays.cuda()).sum().backward()
            torch.cuda.synchronize()
            trained.add(name)
        except (RuntimeError, hb.UnsupportedPipeline):
            refused.add(name)
    assert len(BY_NAME) == 45
    assert refused == REFUSED, (sorted(refused - REFUSED), sorted(REFUSED - refused))
    assert len(trained) == 36


def test_colour_transform_with_more_views_than_the_backward_sums_refuses_to_train():
    """The backward sums the colour transform's gradient per CTA in shared memory, for at most 512 views; more refuse."""
    case = build_train_case("immersive_z_plane")
    for views, trains in ((512, True), (513, False)):
        ds = dict(case.dataset, total_images_per_frame=views)
        model = hb.LightfieldModel(case.model_cfg, dataset=ds, mlp_mode="fp32")
        assert model.sig.cfg.n_color_views == views
        render = hb.RenderLightfield(model, None, case.model_cfg.render, net_chunk=1 << 20).cuda().train()
        rgb = render.model.render_differentiable(case.rays.cuda(), white_bg=False)
        if trains:
            rgb.sum().backward()
            torch.cuda.synchronize()
        else:
            with pytest.raises(RuntimeError, match="512"):
                rgb.sum().backward()


@pytest.mark.parametrize("name", ["immersive_z_plane", "donerf_voxel"])
def test_system_training_step_on_rare_pipelines(name):
    """INRSystem.training_step for a few steps: the loss goes down, a colour transform's table sits alone in its own 'embedding'
    optimiser (the reference's opt_group, point.py:567) and moves, and the updated model renders what the oracle computes from
    the updated state dict."""
    torch.manual_seed(0)  # the training forward's white-background coin flip
    case = build_train_case(name)
    if name == "immersive_z_plane":
        # opaque rays (sum w -> 1), so that the coin flip leaves the target the same and a few steps must lower the loss
        case.state_dict = seeded_state_dict(case.sig, seed=PARAM_SEED, density_gain=3000.0, app_gain=6.0)
    cfg = hb.to_cfg({"model": case.model_cfg, "training": {"ray_chunk": 1 << 20, "iters_per_epoch": 4000,
                                                          "optimizers": {"color": {"lr": 0.002}, "color_impl": {"lr": 0.001},
                                                                         "embedding_impl": {"lr": 0.0002}, "embedding": {"lr": 0.001}}}})
    system = hb.INRSystem(cfg, dataset=case.dataset)
    system.load_state_dict(case.state_dict)
    system.cuda()
    opts = system.configure_optimizers()
    emb_params = [p for n, p in system.named_parameters() if n.endswith(COLOR_EMB)]
    if case.sig.cfg.n_color_views > 0:
        assert len(opts) == 4 and list(system.optimizer_groups()) == ["color", "color_impl", "embedding_impl", "embedding"]
        emb = emb_params[0]
        own = [o for o in opts if any(q is emb for q in o.param_groups[0]["params"])]
        assert len(own) == 1 and len(own[0].param_groups[0]["params"]) == 1
        assert own[0].param_groups[0]["lr"] == 0.001
        before = emb.detach().clone()
    else:
        assert len(opts) == 3 and not emb_params
    rays = case.rays.cuda()
    g = torch.Generator().manual_seed(0)
    batch = {"coords": rays, "rgb": torch.rand(rays.shape[0], 3, generator=g).cuda()}

    def loss_black():  # the training loss without the coin flip, which moves the loss of rays with sum w < 1 up and down
        with torch.no_grad():
            return float(((system.render_fn.model.render_differentiable(rays, clamp_output=False, white_bg=False) - batch["rgb"]) ** 2).mean())

    before_loss = loss_black()
    for _ in range(3):
        system.training_step(batch)
    assert loss_black() < before_loss
    if case.sig.cfg.n_color_views > 0:
        assert float((emb.detach() - before).abs().max()) > 0.0
    system.eval()
    with torch.no_grad():
        a = system(rays)["rgb"].cpu()
    sd = {k[len("render_fn."):]: v.detach().cpu() for k, v in system.state_dict().items()}
    ref = HyperReelOracle(case.model_cfg_plain, case.dataset, sd).render(case.rays.clone())
    assert float((a - ref).abs().max()) <= 1e-4
