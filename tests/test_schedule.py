"""The optimisers' schedule of INRSystem(schedule="reference") on the host: every group's learning rate at every iteration and
every restart against the reference's own get_scheduler / reset_optimizers (tests/golden/reference/schedule.npz, written by
tests/golden/make_golden_schedule.py), a table re-creation at an iteration no group lists, the epoch hook, and the
refusals."""
import json
import os
import warnings

import numpy as np
import pytest
import torch

import hyperreel_b200 as hb
from tests.cases_train import build_train_case

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference", "schedule.npz")


def golden(name):
    g = np.load(GOLDEN)
    return json.loads(str(g[f"{name}/training_json"])), list(g[f"{name}/groups"]), g[f"{name}/lr"], g[f"{name}/restarts"]


def make_system(training, schedule="reference", model_cfg=None):
    """immersive_z_plane: its colour transform gives it all four of the reference's groups."""
    case = build_train_case("immersive_z_plane")
    cfg = hb.to_cfg({"model": model_cfg or case.model_cfg, "training": dict(training, ray_chunk=1 << 20)})
    return hb.INRSystem(cfg, dataset=case.dataset, schedule=schedule), case


def lrs(system):
    return [o.param_groups[0]["lr"] for o in system.optimizers()]


def replay(system, groups, n_iters, ipe, each=None):
    """The reference's loop without the forward: set_train_iter(i) per iteration (training_step's first act after setting
    `training_started`), training_epoch_end after every ipe iterations.  Returns the lrs and (iteration, group) restarts."""
    system.configure_optimizers()
    assert [k for k, p in system.optimizer_groups().items() if any(q.numel() > 0 for q in p)] == groups
    lr, restarts = np.zeros((n_iters, len(groups))), []
    with warnings.catch_warnings():
        warnings.filterwarnings("ignore", message=".*lr_scheduler.step.*")  # no optimiser step runs here
        for i in range(n_iters):
            before = system.optimizers()
            system.set_train_iter(i)
            system.training_started = True
            restarts += [(i, g) for g, (a, b) in enumerate(zip(before, system.optimizers())) if a is not b]
            lr[i] = lrs(system)
            if each is not None:
                each(i)
            if (i + 1) % ipe == 0:
                system.training_epoch_end([])
    return lr, np.array(restarts, dtype=np.int64).reshape(-1, 2)


@pytest.mark.parametrize("name", ["technicolor", "neural_3d", "immersive", "shiny", "steplr", "small", "cosine_poly"])
def test_learning_rates_and_restarts_match_the_reference(name):
    training, groups, want_lr, want_restarts = golden(name)
    system, _ = make_system(training)
    lr, restarts = replay(system, groups, want_lr.shape[0], training["iters_per_epoch"])
    assert np.array_equal(lr, want_lr)
    assert np.array_equal(restarts, want_restarts)
    # exactly the listed iterations of exactly the listing groups
    listed = sorted((i, g) for g, k in enumerate(groups) for i in training["optimizers"][k].get("reset_opt_list", [])
                    if i < want_lr.shape[0])
    assert [tuple(r) for r in restarts] == listed


def test_the_shipped_decay_reaches_the_reference_final_rate():
    """technicolor_tensorf.yaml over 40 epochs: the colour tables' lr ends at 0.02 * 0.125 ** (36 / 100), 36 epochs after the
    last restart at iteration 12000 (epoch 3), where the constant schedule would still train at 0.02."""
    training, groups, lr, _ = golden("technicolor")
    assert lr[-1, 0] == 0.02 * 0.125 ** (36 / 100.0)
    assert lr[3999, 0] == 0.02 and lr[4000, 0] == 0.02 and lr[15999, 0] == 0.02
    assert lr[16000, 0] == 0.02 * 0.125 ** (1 / 100.0)


def test_a_table_recreation_no_group_lists_restarts_only_that_groups_adam():
    """Up-sampling at iteration 9, which the 'color' group of the small case does not list: the colour tables' Adam drops its
    state and holds the new Parameters, its lr stays on the reference's curve, and every other group keeps its Adam state."""
    training, groups, want_lr, _ = golden("small")
    case = build_train_case("immersive_z_plane")
    mcfg = hb.to_cfg(hb.config.to_plain(case.model_cfg))
    mcfg.color.net.grid_size.end = [224, 224, 224]
    mcfg.color.net.upsamp_list, mcfg.color.net.update_AlphaMask_list = [9], []
    system, _ = make_system(training, model_cfg=mcfg)
    system.train()
    net = system.render_fn.model.color_model.net
    seen = {}

    def each(i):
        if i == 9:
            opts = system.optimizers()
            assert opts[0] is seen["opts"][0] and len(opts[0].state) == 0
            tables = [p for p in system.optimizer_groups()["color"] if p.numel() > 0]
            assert all(a is b for a, b in zip(opts[0].param_groups[0]["params"], tables))
            assert net.gridSize.tolist() == [224, 224, 224] and tables[0].shape[-1] == 224
            for g in range(1, 4):
                assert opts[g] is seen["opts"][g]
                assert {int(s["step"]) for s in opts[g].state.values()} == seen["steps"][g]
        for o in system.optimizers():  # one Adam step on made-up gradients, so that each group has state to keep
            for p in o.param_groups[0]["params"]:
                p.grad = torch.full_like(p, 1e-3)
            o.step()
        seen["opts"] = system.optimizers()
        seen["steps"] = [{int(s["step"]) for s in o.state.values()} for o in seen["opts"]]

    lr, restarts = replay(system, groups, want_lr.shape[0], training["iters_per_epoch"], each)
    assert net.gridSize.tolist() == [224, 224, 224]
    assert np.array_equal(lr, want_lr)
    assert 9 not in restarts[:, 0]


def test_constant_schedule_keeps_the_configured_rates_and_has_no_schedulers():
    training, groups, want_lr, _ = golden("small")
    for kw in ({}, {"schedule": "constant"}):
        case = build_train_case("immersive_z_plane")
        cfg = hb.to_cfg({"model": case.model_cfg, "training": dict(training, ray_chunk=1 << 20)})
        system = hb.INRSystem(cfg, dataset=case.dataset, **kw)
        assert system.schedule == "constant"
        lr, restarts = replay(system, groups, want_lr.shape[0], training["iters_per_epoch"])
        assert system.lr_schedulers() == [] and len(restarts) == 0
        assert np.array_equal(lr, np.broadcast_to(want_lr[0], lr.shape))


def test_epoch_end_returns_the_means_and_steps_only_after_training_started():
    training, groups, want_lr, _ = golden("small")
    system, _ = make_system(training)
    system.configure_optimizers()
    system.training_epoch_end([])  # no training_step yet: the reference's training_started is False
    assert lrs(system) == list(want_lr[0])
    outs = [{"train/loss": torch.tensor(v, dtype=torch.float32), "train/psnr": torch.tensor(10.0 * v, dtype=torch.float32)}
            for v in (0.5, 0.25, 0.125)]
    system.training_started = True
    with warnings.catch_warnings():
        warnings.filterwarnings("ignore", message=".*lr_scheduler.step.*")
        means = system.training_epoch_end(outs)
    assert means == {"train/loss": float(torch.tensor([0.5, 0.25, 0.125]).mean()),
                     "train/psnr": float(torch.tensor([5.0, 2.5, 1.25]).mean())}
    assert lrs(system) == [0.02 * 0.125 ** 0.5, 0.001 * 0.5 ** (1 / 3.0), 0.00075 * 0.125 ** 0.5, 0.01]


def test_what_is_not_mirrored_is_refused():
    training, _, _, _ = golden("small")

    def attempt(exc, edit, key="color"):
        t = json.loads(json.dumps(training))
        edit(t, t["optimizers"][key])
        system, _ = make_system(t)
        with pytest.raises(exc):
            system.configure_optimizers()

    attempt(NotImplementedError, lambda t, o: o.update(warmup_epochs=2))
    attempt(NotImplementedError, lambda t, o: o.update(lr_scheduler="plateau"))
    attempt(NotImplementedError, lambda t, o: o.update(optimizer="sgd"), key="embedding")
    attempt(NotImplementedError, lambda t, o: o.update(skip_opt_list=[4]))
    attempt(NotImplementedError, lambda t, o: o.update(remove_skip_opt_list=[4]))
    attempt(NotImplementedError, lambda t, o: t.update(multiscale=True))
    attempt(ValueError, lambda t, o: o.pop("lr_scheduler"), key="embedding")
    attempt(ValueError, lambda t, o: t["optimizers"].pop("embedding"))
    with pytest.raises(ValueError, match="schedule"):
        make_system(training, schedule="exp")
