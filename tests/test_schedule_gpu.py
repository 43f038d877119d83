"""INRSystem(schedule="reference") training on the GPU from DeviceRayBatches.from_config: six epochs of four iterations of the
small case of tests/golden/reference/schedule.npz, with every optimiser's lr against the reference's at every step, the Adam
state around each listed restart and around an up-sampling step no group lists, the epoch means, and the trained model against
the oracle.  Then schedule="constant" against a system built without the argument."""
import numpy as np
import pytest
import torch

import hyperreel_b200 as hb
from oracle.hyperreel_oracle import HyperReelOracle
from tests import importance_oracle as O
from tests.cases_train import build_train_case
from tests.test_schedule import golden

pytestmark = pytest.mark.gpu

UPSAMPLE = 9  # inside epoch 2; the small case's 'color' group lists 4, 6, 8, 10 and 12


def _setup(variants=({"schedule": "reference"},)):
    """immersive_z_plane (all four groups) up-sampled from 192^3 to 224^3 at iteration 9, fed by from_config's replacement
    batches over two fisheye videos of six frames (the data of tests/test_train_importance_gpu.py)."""
    training, groups, want_lr, want_restarts = golden("small")
    case = build_train_case("immersive_z_plane")
    mcfg = hb.to_cfg(hb.config.to_plain(case.model_cfg))
    mcfg.color.net.grid_size.end = [224, 224, 224]
    mcfg.color.net.upsamp_list, mcfg.color.net.update_AlphaMask_list = [UPSAMPLE], []
    o = case.rays[0, :3].tolist()
    W, H, n_frames = 48, 36, 6
    cams = [hb.Camera(pose=[[1, 0, 0, o[0]], [0, 1, 0, o[1]], [0, 0, 1, o[2]]], K=[[30.0, 0, 23.7], [0, 30.0, 17.9], [0, 0, 1]],
                      width=W, height=H, time=f / (n_frames - 1), cam_idx=float(v), distortion=(-0.1, 0.02))
            for v in range(2) for f in range(n_frames)]
    images = np.concatenate([O.video_frames(40 + v, n_frames, H, W) for v in range(2)])
    cfg = hb.to_cfg({"model": mcfg, "training": dict(training, ray_chunk=1 << 20),
                     "dataset": dict(name="immersive", num_frames=n_frames, load_full_step=4, subsample_keyframe_step=2,
                                     subsample_keyframe_frac=0.25, subsample_frac=0.125)})
    batches = hb.DeviceRayBatches.from_config(cfg, cams, images, seed=5)
    assert len(batches) == training["iters_per_epoch"] == 4
    systems = []
    for kw in variants:
        system = hb.INRSystem(cfg, dataset=case.dataset, **kw)
        system.load_state_dict(case.state_dict)
        systems.append(system.cuda())
    return systems, batches, mcfg, case, groups, want_lr, want_restarts


def _steps(opt):
    return {int(s["step"]) for s in opt.state.values()}


def test_reference_schedule_trains_on_the_reference_rates_and_restarts():
    (system,), batches, mcfg, case, groups, want_lr, want_restarts = _setup()
    listed = {}
    for i, g in want_restarts.tolist():
        listed.setdefault(i, set()).add(g)
    net = system.render_fn.model.color_model.net
    grid0 = net.gridSize.tolist()
    system.configure_optimizers()
    assert list(system.optimizer_groups()) == groups
    torch.manual_seed(0)  # the white-background coin flips
    i, losses = 0, []
    for epoch in range(want_lr.shape[0] // len(batches)):
        batches.set_epoch(epoch)
        outs = []
        for batch in batches:
            before = system.optimizers()
            steps = [_steps(o) for o in before]
            system.train()
            system.set_train_iter(i)  # what training_step(batch, train_iter=i) runs first, so the restart can be seen
            after = system.optimizers()
            for g in range(4):
                if g in listed.get(i, ()):
                    assert after[g] is not before[g] and len(after[g].state) == 0, (i, g)
                elif i == UPSAMPLE and g == 0:  # the tables were re-created, no group lists this iteration
                    assert after[g] is before[g] and len(after[g].state) == 0
                    tables = [p for p in system.optimizer_groups()["color"] if p.numel() > 0]
                    assert all(a is b for a, b in zip(after[g].param_groups[0]["params"], tables))
                else:
                    assert after[g] is before[g] and _steps(after[g]) == steps[g], (i, g)
            assert [o.param_groups[0]["lr"] for o in after] == list(want_lr[i]), i
            outs.append(system.training_step(batch))
            losses.append(outs[-1]["train/loss"])
            i += 1
        means = system.training_epoch_end(outs)
        for k in ("train/loss", "train/psnr"):
            assert means[k] == float(torch.stack([o[k] for o in outs]).mean()), k
    assert net.gridSize.tolist() != grid0
    assert all(np.isfinite(float(v)) for v in losses)
    system.eval()
    rays = case.rays.cuda()
    with torch.no_grad():
        a = system(rays)["rgb"].cpu()
    sd = {k[len("render_fn."):]: v.detach().cpu() for k, v in system.state_dict().items()}
    ref = HyperReelOracle(hb.config.to_plain(mcfg), case.dataset, sd).render(case.rays.clone())
    assert float((a - ref).abs().max()) <= 1e-4


def test_constant_schedule_updates_the_parameters_bit_for_bit_like_the_default():
    """A system built without `schedule` and one with schedule="constant", across the up-sampling step.  The render
    backward sums gradients with float atomics, so two backward passes differ in the last bits: the second system is stepped
    on the gradients the first computed.  Equal parameters after every step then mean equal optimisers, rates and restarts."""
    (a, b), batches, _, _, _, _, _ = _setup(variants=({}, {"schedule": "constant"}))
    torch.manual_seed(0)
    i = 0
    for epoch in range(3):
        batches.set_epoch(epoch)
        for batch in batches:
            a.training_step(batch, train_iter=i)
            b.train()
            b.set_train_iter(i)
            if not b.optimizers():
                b.configure_optimizers()
            for opt in b.optimizers():
                opt.zero_grad(set_to_none=True)
            named_b = dict(b.named_parameters())
            for n, p in a.named_parameters():
                if p.grad is not None:
                    named_b[n].grad = p.grad.clone()
            for opt in b.optimizers():
                opt.step()
            assert [o.param_groups[0]["lr"] for o in a.optimizers()] == [o.param_groups[0]["lr"] for o in b.optimizers()]
            for n, p in a.named_parameters():
                assert torch.equal(p, named_b[n]), (i, n)
            i += 1
        a.training_epoch_end([])
        b.training_epoch_end([])
    assert i > UPSAMPLE and a.lr_schedulers() == b.lr_schedulers() == []
