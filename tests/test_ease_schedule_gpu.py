"""ease="reference" on the GPU: renders and gradients against the reference at every iteration of tests/ease_cases.py, the
in-place activation update of set_iter and its refusals, and five training steps against the reference's own loop."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import hyperreel_b200 as hb
from hyperreel_b200 import lib as L
from oracle.hyperreel_oracle import HyperReelOracle
from tests.ease_cases import (EASE_CASES, ITERS, ITERS_PER_EPOCH, LOOP_START, LOOP_STEPS, build_ease_case, eased_oracle,
                              loop_seed, loop_target)
from tests.golden.make_golden_grads import probe_indices, target_for
from tests.test_grads_train_gpu import kink_moves

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TRAINED = [n for n, s in EASE_CASES.items() if not s.get("forward_only")]


def _render(case, ease="reference", mlp_mode="auto"):
    model = hb.LightfieldModel(case.model_cfg, dataset=case.dataset, iters_per_epoch=ITERS_PER_EPOCH, ease=ease,
                               mlp_mode=mlp_mode)
    render = hb.RenderLightfield(model, None, case.model_cfg.render, net_chunk=1 << 20)
    render.load_state_dict(case.state_dict, strict=False)
    return render.cuda().eval()


@pytest.mark.parametrize("name", list(EASE_CASES))
@pytest.mark.parametrize("mlp_mode", ["fp32", "bf16x3"])
def test_rgb_matches_the_reference_at_every_iteration(name, mlp_mode):
    g = np.load(os.path.join(GOLDEN, f"ease_{name}.npz"))
    case = build_ease_case(name)
    render = _render(case, mlp_mode=mlp_mode)
    rays = case.rays.cuda()
    for it in ITERS:
        render.model.set_iter(it)
        with torch.no_grad():
            rgb = render.model(rays)["rgb"].cpu()
        assert float((rgb - torch.from_numpy(g[f"{it}/rgb"])).abs().max()) <= 1e-4, it


@pytest.mark.parametrize("name", TRAINED)
@pytest.mark.parametrize("it", ITERS)
def test_gradients_match_the_reference_at_every_iteration(name, it):
    """The tolerances and LeakyReLU-kink allowance of tests/test_grads_train_gpu.py."""
    g = np.load(os.path.join(GOLDEN, f"ease_{name}.npz"))
    case = build_ease_case(name)
    render = _render(case, mlp_mode="fp32")
    render.model.set_iter(it)
    rays = case.rays.cuda()
    rgb = render.model.render_differentiable(rays, clamp_output=True)
    loss = ((rgb - target_for(rays.shape[0]).cuda()) ** 2).mean()
    loss.backward()
    assert abs(float(loss.detach()) - float(g[f"{it}/loss"])) <= 1e-5
    with eased_oracle(it):
        orc = HyperReelOracle(case.model_cfg_plain, case.dataset, case.state_dict)
        rgb_h, leaves_h = orc.render_with_grad(case.rays.clone(), heads_leaf=True)
        ((rgb_h - target_for(rays.shape[0])) ** 2).mean().backward()
    moves = kink_moves(orc, case.rays, leaves_h["_mlp_out"].grad)
    named = dict(render.named_parameters())
    keys = [k[len(f"{it}/norm/"):] for k in g.files if k.startswith(f"{it}/norm/")]
    assert len(keys) >= 17
    for k in keys:
        nrm = float(g[f"{it}/norm/{k}"])
        grad = named[k].grad
        assert grad is not None, k
        scale = float(g[f"{it}/max/{k}"]) + 1e-12
        ok = False
        for m in moves:
            flat = (grad.cpu() - m[k].reshape(grad.shape) if k in m else grad.cpu()).reshape(-1)
            probe = flat[probe_indices(flat.numel())].numpy()
            ok = ok or (abs(float(flat.norm()) - nrm) <= 2e-3 * nrm + 1e-9
                        and np.abs(probe - g[f"{it}/probe/{k}"]).max() <= 1e-3 * scale + 1e-10)
        assert ok, k


def test_heads_held_at_their_start_value_get_no_gradient():
    """Iteration 0: sigma sits at its start value (w = 0) and point_sigma's wait has not ended: their d heads are exactly 0."""
    case = build_ease_case("technicolor_trained")
    render = _render(case)
    render.model.set_iter(0)
    c = render.model.sig.cfg
    rgb, heads = render.model.render_differentiable(case.rays.cuda(), clamp_output=True, return_heads=True)
    heads.retain_grad()
    ((rgb - target_for(rgb.shape[0]).cuda()) ** 2).mean().backward()
    d = heads.grad.reshape(heads.shape[0], c.n_samples, c.head_stride)
    assert bool(torch.isfinite(d).all())
    assert float(d.abs().max()) > 0.0
    for off in (c.off_sigma, c.off_point_sigma):
        assert float(d[:, :, off].abs().max()) == 0.0


class _CountingLib:
    def __init__(self, lib):
        self._lib, self.calls = lib, []

    def __getattr__(self, name):
        fn = getattr(self._lib, name)

        def call(*a):
            self.calls.append(name)
            return fn(*a)
        return call


def test_set_iter_inside_a_window_updates_the_handle_in_place():
    case = build_ease_case("technicolor_trained")
    model = _render(case).model
    rays = case.rays.cuda()
    model.set_iter(6000)
    with torch.no_grad():
        a = model(rays)["rgb"]
    rays_host = case.rays.clone().pin_memory()
    rgb_host = torch.empty((rays_host.shape[0], 3), pin_memory=True)
    model.render_host(rays_host, rgb_host)  # captures the host pipeline's graph at iteration 6000 for these two buffers
    handle = model._handle.value
    spy = model._lib = _CountingLib(model._lib)
    model.set_iter(13000)
    with torch.no_grad():
        b = model(rays)["rgb"]
    host = model.render_host(rays_host, rgb_host).clone()  # same buffers: the graph key is unchanged
    model._lib = spy._lib
    assert model._handle.value == handle
    assert "hr_set_activations" in spy.calls and "hr_upload" not in spy.calls and "hr_create" not in spy.calls
    assert float((a - b).abs().max()) > 1e-3
    assert torch.equal(host, b.cpu())


def test_elapsed_windows_render_like_the_default_model():
    case = build_ease_case("technicolor_trained")
    eased, plain = _render(case).model, _render(case, ease="elapsed").model
    rays = case.rays.cuda()
    eased.set_iter(6000)
    with torch.no_grad():
        eased(rays)
    for it in (16000, 20000):
        eased.set_iter(it)
        plain.set_iter(it)
        with torch.no_grad():
            assert torch.equal(eased(rays)["rgb"], plain(rays)["rgb"])


def test_default_model_refuses_an_open_window():
    case = build_ease_case("technicolor_trained")
    model = _render(case, ease="elapsed").model
    with pytest.raises(hb.UnsupportedPipeline):
        model.set_iter(6000)


def test_set_activations_refuses_anything_but_activations():
    """hr_set_activations leaves the handle as it was when the configuration differs beyond its activations, when an
    activation outside the density heads is eased, or when an activation kind is unknown."""
    case = build_ease_case("technicolor_trained")
    model = _render(case).model
    rays = case.rays.cuda()
    model.set_iter(6000)
    with torch.no_grad():
        before = model(rays)["rgb"]
    lib, h = model._lib, model._handle

    def attempt(edit):
        c = L.hr_config.from_buffer_copy(bytes(model.sig.cfg))
        edit(c)
        c.act_sigma.ease_mul = 0.25  # an activation change that would alter the render if it were applied
        assert lib.hr_set_activations(h, C.byref(c)) != 0
        assert lib.hr_last_error()

    attempt(lambda c: setattr(c, "isect_near", c.isect_near + 1.0))
    attempt(lambda c: setattr(c.act_z, "eased", 1))
    attempt(lambda c: setattr(c.act_offset, "kind", 7))
    with torch.no_grad():
        assert torch.equal(model(rays)["rgb"], before)


@pytest.mark.parametrize("name", TRAINED)
@pytest.mark.parametrize("train_net", ["torch", "tc"])
def test_training_steps_match_the_reference_loop(name, train_net):
    """Five INRSystem.training_steps from iteration 6000 against the reference's loop (tests/golden/make_golden_ease.py)."""
    g = np.load(os.path.join(GOLDEN, f"ease_{name}.npz"))
    case = build_ease_case(name)
    cfg = hb.to_cfg({"model": case.model_cfg_plain, "training": {"ray_chunk": 1 << 20, "iters_per_epoch": ITERS_PER_EPOCH}})
    system = hb.INRSystem(cfg, dataset=case.dataset, ease="reference", train_net=train_net)
    system.load_state_dict(case.state_dict)
    system.cuda()
    batch = {"coords": case.rays.cuda(), "rgb": loop_target(case.rays.shape[0]).cuda()}
    losses = []
    for step in range(LOOP_STEPS):
        torch.manual_seed(loop_seed(step))  # the training forward's white-background coin flip, drawn as in the golden loop
        losses.append(float(system.training_step(batch, train_iter=LOOP_START + step)["train/loss"]))
    ref = g["loop_losses"]
    assert np.all(np.abs(np.array(losses) - ref) <= 1e-3 * np.abs(ref)), (losses, ref)
