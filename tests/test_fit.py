"""hyperreel_b200.fit on the host: its epoch rules against a restatement of the reference's loop for every shipped training
config, its checkpoint layout against the reference's state_dict (tests/golden/reference/fit.npz, written by
tests/golden/make_golden_fit.py) and optimiser groups, the idempotence of the validation's set_train_iter, the default
frame reader, and the refusals."""
import copy
import json
import os
import types
import warnings

import numpy as np
import pytest
import torch

import hyperreel_b200 as hb
from hyperreel_b200.fit import (MASK_PREFIX, STATE_KEY, checkpoint, epoch_events, get_train_iter, num_iters, read_image,
                                restore)
from tests.test_dataset_cameras import _golden as _scenes
from tests.test_dataset_cameras import make_scene
from tests.test_schedule import golden as schedule_golden
from tests.test_schedule import make_system as schedule_system

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference", "fit.npz")


def _golden():
    return np.load(GOLDEN)


def _trainings():
    return sorted(k.split("/", 1)[1] for k in _golden().files if k.startswith("training/"))


def _training(name):
    return json.loads(str(_golden()[f"training/{name}"]))


def reference_loop(t, n_rows, epochs):
    """The reference's loop, restated: per epoch the train_iter of each training_step (get_train_iter, nlf/__init__.py:
    580-606, one GPU, no pre-training iterations), whether Lightning validates (check_val_every_n_epoch), which split the
    current val dataloader holds (val_dataloader, :248-275, built first at datamodule.current_epoch 0 and re-built with
    current_epoch + 1 by training_epoch_end when reset_val holds, :728-752), the train_iter validation_step sets (:990-991),
    whether it renders the video (:998-1001) and whether the checkpoint callbacks save (main.py:44-50)."""
    n = t["num_iters"] if t.get("sample_with_replacement", False) else n_rows // t["batch_size"]
    T, loader_epoch, out = t["test_every"], 0, []
    for e in range(epochs):
        validate = (e + 1) % t["val_every"] == 0
        out.append({"first_iter": n * e, "last_iter": n * e + n - 1, "validate": validate,
                    "split": "test" if (loader_epoch + 1) % T == 0 else "val", "val_iter": max(n * (e + 1), 0),
                    "render": validate and (e + 1) % t["render_every"] == 0,
                    "checkpoint": (e + 1) % t["ckpt_every"] == 0})
        if (e + 2) % T == 0 or (e + 1) % T == 0 or e % T == 0:  # reset_val (test_only is False)
            loader_epoch = e + 1
    return out


def _fit_loop(t, n_rows, epochs):
    n, out = num_iters(t, n_rows), []
    for e in range(epochs):
        ev = epoch_events(t, e)
        out.append({"first_iter": get_train_iter(t, n_rows, e, 0), "last_iter": get_train_iter(t, n_rows, e, n - 1),
                    "validate": ev["validate"], "split": ev["split"], "val_iter": max(get_train_iter(t, n_rows, e + 1, 0), 0),
                    "render": ev["render"], "checkpoint": ev["checkpoint"]})
    return out


def _validated_split(rows):
    """The split matters on validating epochs only."""
    return [dict(r, split=r["split"] if r["validate"] else None) for r in rows]


@pytest.mark.parametrize("name", _trainings())
def test_epoch_rules_equal_the_reference_loop(name):
    t = _training(name)
    assert t["sample_with_replacement"] and t["num_gpus"] == 1
    assert _validated_split(_fit_loop(t, 10 ** 6, 100)) == _validated_split(reference_loop(t, 10 ** 6, 100))
    # without replacement an epoch is len(train rows) // batch_size iterations
    t = dict(t, sample_with_replacement=False)
    assert _validated_split(_fit_loop(t, 100_001, 100)) == _validated_split(reference_loop(t, 100_001, 100))
    assert _fit_loop(t, 100_001, 2)[1]["first_iter"] == 100_001 // t["batch_size"]


def test_small_test_every_alternates_like_the_reference_dataloader():
    for T in (1, 2, 3, 5):
        t = {"sample_with_replacement": True, "num_iters": 3, "batch_size": 8, "val_every": 1, "test_every": T,
             "render_every": 2, "ckpt_every": 1}
        assert _validated_split(_fit_loop(t, 0, 40)) == _validated_split(reference_loop(t, 0, 40)), T


def _tiny_system(training=None):
    z = _golden()
    model = hb.to_cfg(json.loads(str(z["state_dict/model"])))
    cfg = hb.to_cfg({"model": model, "training": dict(training or {}, iters_per_epoch=4000, ray_chunk=1 << 20)})
    return hb.INRSystem(cfg, dataset=json.loads(str(z["state_dict/dataset"])))


def test_checkpoint_state_dict_has_the_reference_keys_and_shapes():
    """Every key of the reference's INRSystem.state_dict() for technicolor_z_plane_tiny, with its shape, but the Linear(1, 1)
    `dummy_layer` placeholders of its parameterisation and PE modules (nlf/param.py:383, nlf/pe.py:50), which no forward
    reads; the reference's load_state_dict (strict=False) keeps its own for them."""
    want = json.loads(str(_golden()["state_dict/shapes"]))
    system = _tiny_system()
    ck = checkpoint(system, types.SimpleNamespace(seed=5, epoch=2), epoch=2, global_step=12, weights_only=True)
    got = {k: list(v.shape) for k, v in ck["state_dict"].items()}
    assert set(ck) == {"epoch", "global_step", "state_dict"} and (ck["epoch"], ck["global_step"]) == (2, 12)
    assert {k for k in want if k not in got} == {k for k in want if ".dummy_layer." in k}
    assert {k: want[k] for k in got} == got
    # after pruning, the occupancy mask under the reference's AlphaGridMask buffer names (utils/tensorf_utils.py:466-467)
    net = system.render_fn.model.color_model.net
    net.alphaMask_thres = 0.0  # the fresh tables' density is below the configured threshold everywhere
    net.updateAlphaMask((6, 5, 4))
    sd = checkpoint(system, types.SimpleNamespace(seed=5, epoch=2), 2, 12, weights_only=True)["state_dict"]
    assert list(sd[MASK_PREFIX + "alpha_volume"].shape) == [1, 1, 4, 5, 6]
    assert torch.equal(sd[MASK_PREFIX + "alpha_aabb"], net.aabb)


def test_checkpoint_optimizer_states_follow_the_reference_groups():
    training, groups, want_lr, _ = schedule_golden("technicolor")
    system, _ = schedule_system(training)
    system.configure_optimizers()
    ck = checkpoint(system, types.SimpleNamespace(seed=5, epoch=0), 0, 0)
    assert len(ck["optimizer_states"]) == len(groups) == len(ck["lr_schedulers"])
    assert [s["param_groups"][0]["lr"] for s in ck["optimizer_states"]] == list(want_lr[0])
    assert list(system.optimizer_groups())[:len(groups)] == groups
    extra = ck[STATE_KEY]
    assert extra["batches"] == {"seed": 5, "epoch": 0} and (extra["ease"], extra["schedule"]) == ("elapsed", "reference")
    assert torch.equal(extra["rng_state"], torch.get_rng_state())


def _regularised(training):
    """immersive_z_plane (test_schedule.py) with the TensoRF regulariser, up-sampling and pruning at iteration 9 and a
    'color' restart there."""
    from tests.cases_train import build_train_case

    case = build_train_case("immersive_z_plane")
    mcfg = hb.to_cfg(hb.config.to_plain(case.model_cfg))
    mcfg.color.net.grid_size.start, mcfg.color.net.grid_size.end = [12, 12, 12], [20, 20, 20]
    mcfg.color.net.upsamp_list, mcfg.color.net.update_AlphaMask_list = [9], [9]
    mcfg.color.net.alpha_mask_thre = 0.0  # keep every voxel of the fresh tables
    reg = {"type": "tensorf", "update_AlphaMask_list": [9], "lr_decay_target_ratio": 0.1, "n_iters": 30000,
           "L1_weight_initial": 8e-5, "L1_weight_rest": 4e-5, "TV_weight_density": 0.0125, "TV_weight_app": 0.0125}
    cfg = hb.to_cfg({"model": mcfg, "training": dict(training, ray_chunk=1 << 20), "regularizers": {"tensorf": reg}})
    torch.manual_seed(0)
    return hb.INRSystem(cfg, dataset=case.dataset, schedule="reference")


def _state(system):
    net = system.render_fn.model.color_model.net
    reg = system.regularizers[0]
    return (net.gridSize.tolist(), net.aabb.tolist(), [p.detach().clone() for p in system.parameters()],
            net.alphaMask.volume.clone() if net.alphaMask is not None else None,
            (reg.cur_iter, reg.L1_reg_weight, reg.TV_weight_density, reg.TV_weight_app),
            [o.param_groups[0]["lr"] for o in system.optimizers()], [len(o.state) for o in system.optimizers()],
            [s.last_epoch for s in system.lr_schedulers()])


def test_validation_set_train_iter_then_the_next_step_equals_the_step_alone():
    """fit's order at an epoch boundary that is an up-sampling, pruning and restart iteration: validation_step's
    set_train_iter in eval(), training_epoch_end, then the next training_step's set_train_iter of the same iteration.  It
    leaves the state the step's call alone leaves, as the reference's does (its validation runs the net in eval, where
    TensorBase.set_iter returns before the schedule, tensorf_base.py:509-513)."""
    training = json.loads(json.dumps(schedule_golden("small")[0]))
    training["optimizers"]["color"]["reset_opt_list"] = [9]
    states = []
    for validate in (True, False):
        system = _regularised(training)
        system.configure_optimizers()
        system.train()
        system.set_train_iter(8)
        for o in system.optimizers():  # moments to keep or drop
            for p in o.param_groups[0]["params"]:
                p.grad = torch.full_like(p, 1e-3)
            o.step()
        system.training_started = True
        if validate:
            system.eval()
            system.set_train_iter(9)
            assert system.render_fn.model.color_model.net.gridSize.tolist() == [12, 12, 12]  # nothing up-sampled in eval
            system.train()
        with warnings.catch_warnings():
            warnings.filterwarnings("ignore", message=".*lr_scheduler.step.*")
            system.training_epoch_end([])
        system.set_train_iter(9)
        states.append(_state(system))
    a, b = states
    assert a[0] == b[0] == [20, 20, 20] and a[1] == b[1]
    assert len(a[2]) == len(b[2]) and all(torch.equal(x, y) for x, y in zip(a[2], b[2]))
    assert a[3] is not None and torch.equal(a[3], b[3])
    assert a[4:] == b[4:]


def test_read_image_converts_as_the_dataset_does(tmp_path):
    """get_rgb converts by the dataset, not by the file: RGB for Technicolor whatever the PNG holds (an alpha channel, a
    palette with transparency, grey), RGBA for DoNeRF (alpha 255 for a file without one)."""
    from PIL import Image

    rng = np.random.default_rng(0)
    rgb = rng.integers(0, 256, (5, 7, 3), dtype=np.uint8)
    rgba = rng.integers(0, 256, (5, 7, 4), dtype=np.uint8)
    files = {"RGB": Image.fromarray(rgb, "RGB"), "RGBA": Image.fromarray(rgba, "RGBA"),
             "L": Image.fromarray(rgb[..., 0], "L"), "P": Image.fromarray(rgb, "RGB").quantize(8)}
    files["P"].info["transparency"] = 0
    for mode, im in files.items():
        path = str(tmp_path / f"{mode}.png")
        im.save(path)
        with Image.open(path) as f:
            want_rgb, want_rgba = np.asarray(f.convert("RGB")), np.asarray(f.convert("RGBA"))
        for flag, want in ((False, want_rgb), (True, want_rgba)):
            got = read_image(hb.FrameSource(path, None), rgba=flag)
            assert got.dtype == np.uint8 and got.shape == (5, 7, 4 if flag else 3), (mode, flag)
            assert np.array_equal(got, want), (mode, flag)
    assert np.array_equal(read_image(hb.FrameSource(str(tmp_path / "RGBA.png"), None)), rgba[..., :3])
    assert np.array_equal(read_image(hb.FrameSource(str(tmp_path / "RGB.png"), None), rgba=True),
                          np.concatenate([rgb, np.full((5, 7, 1), 255, np.uint8)], -1))
    with pytest.raises(ValueError, match="read_frame"):
        read_image(hb.FrameSource(str(tmp_path / "RGB.png"), 3))


class _Batches:
    def __init__(self, seed, epoch):
        self.seed, self.epoch = seed, epoch

    def set_epoch(self, epoch):
        self.epoch = epoch


def _same(a, b, where=()):
    """Nested checkpoint values equal: tensors by torch.equal (dtype and shape included), the rest by ==."""
    if isinstance(a, torch.Tensor):
        assert isinstance(b, torch.Tensor) and a.dtype == b.dtype and torch.equal(a.cpu(), b.cpu()), where
    elif isinstance(a, dict):
        assert isinstance(b, dict) and a.keys() == b.keys(), where
        for k in a:
            _same(a[k], b[k], where + (k,))
    elif isinstance(a, (list, tuple)):
        assert type(a) is type(b) and len(a) == len(b), where
        for i, (x, y) in enumerate(zip(a, b)):
            _same(x, y, where + (i,))
    else:
        assert a == b, (where, a, b)


def test_checkpoint_restore_round_trip_is_exact(tmp_path):
    """A system past an up-sampling, a pruning (mask and shrink) and a restart, with Adam moments and stepped schedulers:
    checkpoint -> torch.save -> torch.load(weights_only=True) -> restore into a fresh system -> checkpoint gives the same
    checkpoint, every tensor and moment torch.equal, and the fresh system holds the same parameters, mask and generator."""
    training = json.loads(json.dumps(schedule_golden("small")[0]))
    training["optimizers"]["color"]["reset_opt_list"] = [9]
    system = _regularised(training)
    system.configure_optimizers()
    system.train()
    with warnings.catch_warnings():
        warnings.filterwarnings("ignore", message=".*lr_scheduler.step.*")
        for i in range(11):
            system.set_train_iter(i)
            for o in system.optimizers():
                for p in o.param_groups[0]["params"]:
                    p.grad = torch.randn_like(p) * 1e-3
                o.step()
            system.regularizers[0].loss(system.render_fn.model.color_model.net)  # the running TV weights decay per use
            system.training_started = True
            if i % 4 == 3:
                system.training_epoch_end([])
    net = system.render_fn.model.color_model.net
    assert net.gridSize.tolist() == [20, 20, 20] and net.alphaMask is not None and net.N_voxel_list == [[], [], []]
    want = checkpoint(system, _Batches(7, 2), 2, 11)
    path = str(tmp_path / "last.ckpt")
    torch.save(want, path)
    torch.rand(5)  # the generator moves on; restore puts it back
    fresh = _regularised(training)
    batches = _Batches(0, 0)
    assert restore(fresh, batches, torch.load(path, map_location="cpu", weights_only=True)) == 2
    assert (batches.seed, batches.epoch) == (7, 2)
    assert torch.equal(torch.get_rng_state(), want[STATE_KEY]["rng_state"])
    _same(checkpoint(fresh, batches, 2, 11), want)
    a, b = dict(system.named_parameters()), dict(fresh.named_parameters())
    assert a.keys() == b.keys() and all(torch.equal(a[k], b[k]) for k in a)
    fnet = fresh.render_fn.model.color_model.net
    assert torch.equal(fnet.alphaMask.volume, net.alphaMask.volume) and torch.equal(fnet.alphaMask.aabb, net.alphaMask.aabb)
    assert [o.param_groups[0]["lr"] for o in fresh.optimizers()] == [o.param_groups[0]["lr"] for o in system.optimizers()]


def _scene_cfg(case, tmp_path, **training):
    root, dcfg = make_scene(_scenes(), case, tmp_path)
    t = dict(_training("technicolor"), **training)
    return {"model": hb.configs.get("technicolor_z_plane")[0], "dataset": dcfg, "training": t, "regularizers": {}}, root


def test_a_video_split_needs_read_frame(tmp_path):
    cfg, root = _scene_cfg("neural_3d_ndc", tmp_path)
    with pytest.raises(ValueError, match="read_frame"):
        hb.fit(cfg, root, str(tmp_path / "run"))
    assert not os.path.exists(tmp_path / "run")


def test_what_fit_does_not_run_is_refused(tmp_path):
    cfg, root = _scene_cfg("technicolor_skip", tmp_path, num_gpus=2)
    with pytest.raises(hb.UnsupportedPipeline, match="num_gpus"):
        hb.fit(cfg, root, str(tmp_path / "run"))
    cfg, root = _scene_cfg("technicolor_skip", tmp_path, multiscale=True)
    with pytest.raises(hb.UnsupportedPipeline, match="multiscale"):
        hb.fit(cfg, root, str(tmp_path / "run"))
    cfg = copy.deepcopy(cfg)
    cfg["training"] = dict(cfg["training"], multiscale=False)
    cfg["dataset"]["name"] = "llff"  # dataset_cameras' own refusal surfaces unchanged
    with pytest.raises(hb.UnsupportedPipeline, match="'name'"):
        hb.fit(cfg, root, str(tmp_path / "run"))
