"""The sample net's tensor-core training path (LightfieldModel(train_net="tc"): hr_train_net_forward / hr_train_net_backward):
its heads against the wgmma render net, its layer gradients against fp64 autograd with the LeakyReLU sides it chose, the
whole model's gradients and INRSystem.training_step against the torch path, determinism and the refusals."""
import numpy as np
import pytest
import torch

import hyperreel_b200 as hb
from hyperreel_b200 import configs, rays as rays_mod
from hyperreel_b200.signature import lower
from hyperreel_b200.state import seeded_state_dict
from oracle.hyperreel_oracle import HyperReelOracle
from tests.cases import build_case
from tests.cases_train import build_train_case
from tests.test_shipped_yaml_golden import SHIPPED, load_fixture

RAGGED = 128 * 40 + 77  # several tiles per CTA of the forward, several K splits of dW, a ragged last tile


def _model(case, train_net="tc", mlp_mode="bf16x3"):
    model = hb.LightfieldModel(case.model_cfg, dataset=case.dataset, mlp_mode=mlp_mode, train_net=train_net)
    render = hb.RenderLightfield(model, None, case.model_cfg.render, net_chunk=1 << 20)
    _, unexpected = render.load_state_dict(case.state_dict, strict=False)
    assert not unexpected
    return render.cuda().model


def _s64_case(n):
    """Technicolor's net with 64 samples per ray (960 outputs: 4 passes of the last layer)."""
    cfg, ds = configs.get("technicolor_z_plane", n_voxels=32 ** 3, z_channels=64)
    sig = lower(cfg, ds)
    sd = seeded_state_dict(sig, seed=31, density_gain=30.0)
    from tests.cases import Case
    from hyperreel_b200.config import to_plain
    return Case(name="technicolor_s64", model_cfg=cfg, model_cfg_plain=to_plain(cfg), dataset=ds, sig=sig,
                rays=rays_mod.for_signature(sig, n, seed=131), state_dict=sd, n_samples=sig.n_samples)


# hidden width 256 with a skip layer (Technicolor), width 128, an encoded input of more than 32 features, BasicPE, S = 64
HEAD_CASES = ["technicolor_trained", "shiny_tiny", "donerf_wide_pe", "technicolor_basic_pe", "technicolor_s64"]


def _case(name, n):
    return _s64_case(n) if name == "technicolor_s64" else build_case(name, n=n)


def _saved(model, ws, n):
    """(encoded input [n, mlp_in], [activation of hidden layer l, [n, W]]) from the workspace (hyperreel_b200.h)."""
    c = model.sig.cfg
    seg = lambda floats: (floats * 4 + 255) // 256 * 256
    ld = (c.mlp_in + 15) // 16 * 16
    f = ws.view(torch.float32)
    enc = f[: n * ld].view(n, ld)[:, : c.mlp_in]
    a0, step = seg(n * ld) // 4, seg(n * c.mlp_width) // 4
    acts = [f[a0 + l * step: a0 + l * step + n * c.mlp_width].view(n, c.mlp_width) for l in range(c.mlp_layers - 1)]
    return enc, acts


def test_bad_train_net_value_raises():
    case = build_case("technicolor_init")
    with pytest.raises(ValueError):
        hb.LightfieldModel(case.model_cfg, dataset=case.dataset, train_net="cublas")
    with pytest.raises(ValueError):
        hb.LightfieldModel(case.model_cfg, dataset=case.dataset, train_net="tc", mlp_mode="fp32")


@pytest.mark.gpu
@pytest.mark.parametrize("name", HEAD_CASES)
def test_training_forward_heads_equal_the_render_net(name):
    """Bit for bit: the same kernel arithmetic, the heads stored in the reference's column order."""
    case = _case(name, RAGGED)
    model = _model(case)
    rays = case.rays.cuda()
    model._ensure_uploaded(rays.device)
    heads, _ = model._train_net_forward(rays)
    model.eval()
    want = model.render_stages(rays)["mlp_out"]
    assert torch.equal(heads, want)


def _fp64_net_grads(model, enc_k, acts, d_heads):
    """fp64 autograd of the sample net on the tc forward's encoded input, every LeakyReLU side fixed to the one the tc forward
    chose (the sign of its saved activation), in the reference's parameter layouts."""
    c = model.sig.cfg
    perm = list(model.sig.in_perm)
    inv = torch.empty(len(perm), dtype=torch.long)
    inv[torch.tensor(perm)] = torch.arange(len(perm))
    enc = enc_k.double()[:, inv.to(enc_k.device)]  # kernel feature order -> the reference's
    params = [p.detach().double().requires_grad_(True) for p in model._net_params()]
    x = enc
    for i in range(c.mlp_layers):
        if i == c.mlp_skip:
            x = torch.cat([enc, x], -1)
        x = x @ params[2 * i].t() + params[2 * i + 1]
        if i < c.mlp_layers - 1:
            x = torch.where(acts[i] > 0, x, c.leaky_slope * x)
    return torch.autograd.grad((x * d_heads.double()).sum(), params)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["technicolor_trained", "shiny_tiny", "donerf_wide_pe", "technicolor_basic_pe"])
def test_net_gradients_match_fp64_with_fixed_sides(name):
    case = _case(name, RAGGED)
    model = _model(case)
    rays = case.rays.cuda()
    model._ensure_uploaded(rays.device)
    heads, ws = model._train_net_forward(rays)
    n = rays.shape[0]
    d_heads = torch.randn(heads.shape, generator=torch.Generator().manual_seed(5)).cuda()
    got = model._train_net_backward(ws, d_heads, n)
    enc, acts = _saved(model, ws, n)
    want = _fp64_net_grads(model, enc, acts, d_heads)
    assert len(got) == 2 * model.sig.cfg.mlp_layers
    for i, (g, w) in enumerate(zip(got, want)):
        scale = float(w.abs().max())
        assert scale > 0.0, i
        err = float((g.double() - w).abs().max())
        assert err <= 1e-3 * scale, (i, err, scale)


@pytest.mark.gpu
def test_backward_is_bitwise_deterministic():
    case = _case("technicolor_trained", 128 * 300 + 5)
    model = _model(case)
    rays = case.rays.cuda()
    model._ensure_uploaded(rays.device)
    heads, ws = model._train_net_forward(rays)
    d_heads = torch.randn(heads.shape, generator=torch.Generator().manual_seed(6)).cuda()
    a = model._train_net_backward(ws, d_heads, rays.shape[0])
    b = model._train_net_backward(ws, d_heads, rays.shape[0])
    for x, y in zip(a, b):
        assert torch.equal(x, y)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["technicolor_bbox", "immersive_z_plane", "donerf_voxel"])
def test_model_gradients_match_the_torch_path(name):
    """d heads and every table / basis / colour-transform gradient of render_differentiable, tc against torch, each within
    2e-3 of the tensor's largest entry.  (The net's own gradients are compared with fixed kink sides above: bf16x3 and fp32
    may put a pre-activation near 0 on different sides.)"""
    case = build_train_case(name)
    rays = case.rays.cuda()
    out = {}
    for mode in ("torch", "tc"):
        model = _model(case, train_net=mode)
        model.train()
        rgb, heads = model.render_differentiable(rays, clamp_output=False, white_bg=True, return_heads=True)
        heads.retain_grad()
        target = torch.rand(rgb.shape, generator=torch.Generator().manual_seed(7)).cuda()
        ((rgb - target) ** 2).mean().backward()
        net = {id(p) for p in model._net_params()}
        grads = {k: p.grad.detach().clone() for k, p in model.named_parameters() if p.grad is not None and id(p) not in net}
        grads["d_heads"] = heads.grad.detach().clone()
        out[mode] = grads
    assert out["torch"].keys() == out["tc"].keys() and len(out["tc"]) >= 4
    for k, ref in out["torch"].items():
        scale = float(ref.abs().max())
        assert scale > 0.0, k
        assert float((out["tc"][k] - ref).abs().max()) <= 2e-3 * scale, k


@pytest.mark.gpu
def test_training_step_follows_the_torch_path():
    """5 steps of INRSystem.training_step: the loss goes down, stays within 1e-3 (relative) of the torch path's, and the
    updated model renders what the oracle computes from its state dict."""
    case = build_case("donerf_app", n=2048)
    cfg = hb.to_cfg({"model": case.model_cfg, "training": {"ray_chunk": 700, "iters_per_epoch": 4000,
                                                          "optimizers": {"color": {"lr": 0.002}, "color_impl": {"lr": 0.001},
                                                                         "embedding_impl": {"lr": 0.0002}}},
                     "dataset": case.dataset})
    g = torch.Generator().manual_seed(0)
    batch = {"coords": case.rays.cuda(), "rgb": torch.rand(case.rays.shape[0], 3, generator=g).cuda(),
             "weight": torch.ones(case.rays.shape[0], 1).cuda()}
    losses = {}
    for mode in ("torch", "tc"):
        torch.manual_seed(0)  # the white-background coin flips
        system = hb.INRSystem(cfg, train_net=mode)
        system.load_state_dict(case.state_dict)
        system.cuda()
        losses[mode] = [float(system.training_step(batch)["train/loss"]) for _ in range(5)]
    assert losses["tc"][-1] < losses["tc"][0], losses
    for a, b in zip(losses["tc"], losses["torch"]):
        assert abs(a - b) <= 1e-3 * abs(b), losses
    system.eval()
    with torch.no_grad():
        a = system(case.rays.cuda())["rgb"].cpu()
    sd = {k[len("render_fn."):]: v.detach().cpu() for k, v in system.state_dict().items()}
    ref = HyperReelOracle(case.model_cfg_plain, case.dataset, sd).render(case.rays.clone())
    assert float((a - ref).abs().max()) <= 1e-4


@pytest.mark.gpu
def test_cascaded_and_zero_nets_are_refused():
    zero = build_case("technicolor_zero_net")
    model = _model(zero)
    model.train()
    with pytest.raises(RuntimeError, match="zero sample net"):
        model.render_differentiable(zero.rays.cuda())
    path = next(p for p in SHIPPED if p.endswith("technicolor_cascaded.npz"))
    plain, cfg, ds, sig, sd, rays, rgb = load_fixture(path)
    model = hb.LightfieldModel(cfg, dataset=ds, train_net="tc")
    render = hb.RenderLightfield(model, None, cfg.render, net_chunk=1 << 20)
    render.load_state_dict(sd, strict=False)
    render.cuda().train()
    with pytest.raises(Exception, match="cascaded"):
        model.render_differentiable(rays.cuda())
    model._ensure_uploaded(rays.cuda().device)
    heads = torch.empty((rays.shape[0], sig.cfg.mlp_out), device="cuda")
    ws = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
    assert model._lib.hr_train_net_forward(model._handle, rays.cuda().data_ptr(), rays.shape[0], heads.data_ptr(), ws.data_ptr(),
                                           ws.numel(), None) != 0
    assert b"cascaded" in model._lib.hr_last_error()
