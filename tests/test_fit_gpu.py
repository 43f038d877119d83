"""hyperreel_b200.fit on the GPU, from a synthetic Technicolor scene directory (tests/golden/dataset_cameras.npz) and the
shipped technicolor_z_plane_tiny model, four epochs of two steps, with pruning at iterations 3 and 6, up-sampling at 4 and
7 and a 'color' restart at 6, validating every epoch, testing and rendering every second epoch and saving every epoch:

- fit against a hand-written loop of the public calls in the documented order;
- a run stopped after two epochs and resumed from last.ckpt against the uninterrupted run;
- no host synchronisation in the steps of an epoch without a schedule iteration;
- last-weights.ckpt loaded into a fresh INRSystem renders as last.ckpt restored;
- the default reader converts PNGs as get_rgb does.

The render backward sums table gradients with float atomics, so two runs of the same steps differ in the last bits (as in
tests/test_schedule_gpu.py): every discrete schedule state (grid size, aabb, occupancy
mask, up-sampling steps left, optimiser step counts, learning rates, regulariser weights, the CPU generator) and the epoch
records' keys must be equal; parameters, Adam moments, losses and metrics agree to a tolerance far below one training
step's change."""
import json
import os
import types
import warnings

import numpy as np
import pytest
import torch

import hyperreel_b200 as hb
from hyperreel_b200.fit import MASK_PREFIX, STATE_KEY, checkpoint, load_frames, restore
from tests.test_dataset_cameras import _golden as _scenes
from tests.test_dataset_cameras import make_scene

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference", "fit.npz")
KW = {"ease": "reference", "schedule": "reference"}
EPOCHS, NUM_ITERS = 4, 2


def read_frame(source):
    """A deterministic 32 x 24 capture per file (the scene's image files are empty)."""
    seed = sum(ord(c) * (i + 1) for i, c in enumerate(os.path.basename(source.path)))
    return np.random.default_rng(seed).integers(0, 256, (24, 32, 3), dtype=np.uint8)


def make_run(tmp_path, upsamp=(4, 7), prune=(3, 6), restart=(6,)):
    z = np.load(GOLDEN)
    root, dcfg = make_scene(_scenes(), "technicolor_lightfield", tmp_path)
    dcfg = dict(dcfg, img_wh=[16, 12])  # scored views hold the 11 x 11 SSIM window
    model = json.loads(str(z["state_dict/model"]))
    net = model["color"]["net"]
    net.update(N_voxel_init=8 ** 3, N_voxel_final=12 ** 3, upsamp_list=list(upsamp), update_AlphaMask_list=list(prune),
               alpha_mask_thre=0.0)  # a fresh model's density is below any positive threshold: keep every voxel
    training = json.loads(str(z["training/technicolor"]))
    training.update(batch_size=256, ray_chunk=4096, net_chunk=4096, render_ray_chunk=4096, num_iters=NUM_ITERS,
                    num_epochs=EPOCHS, val_every=1, test_every=2, render_every=2, ckpt_every=1)
    for key, oc in training["optimizers"].items():
        oc["reset_opt_list"] = list(restart) if key == "color" else []
    reg = {"type": "tensorf", "update_AlphaMask_list": list(prune), "lr_decay_target_ratio": 0.1, "n_iters": 30000,
           "total_num_tv_iters": 60000, "L1_weight_initial": 8e-5, "L1_weight_rest": 4e-5, "TV_weight_density": 0.0125,
           "TV_weight_app": 0.0125}
    return {"model": model, "dataset": dcfg, "training": training, "regularizers": {"tensorf": reg}}, root


def hand_loop(cfg, root, epochs=EPOCHS, seed=0, stop_before=None):
    """fit's documented order, written out with the public calls."""
    cfg = hb.to_cfg(json.loads(json.dumps(cfg)))
    dcfg, training = cfg.dataset, cfg.training
    views = {s: hb.dataset_cameras(dcfg, root, s) for s in ("train", "val", "test", "render")}
    torch.manual_seed(seed)
    images = {s: hb.dataset_frames(dcfg, torch.stack([torch.from_numpy(read_frame(f)) for f in views[s].frames]).cuda())
              for s in ("train", "val", "test")}
    training.iters_per_epoch = training.num_iters
    system = hb.INRSystem(cfg, dataset=views["train"].facts, **KW).cuda()
    batches = hb.DeviceRayBatches.from_config(cfg, views["train"].cameras, images["train"], seed=seed,
                                              c_in=system.render_fn.model.sig.c_in)
    records, videos, metrics = [], {}, {}
    for e in range(epochs):
        batches.set_epoch(e)
        outputs = []
        for i in range(len(batches)):
            if stop_before is not None and (e, i) == stop_before:
                return system, batches, views, images
            outputs.append(system.training_step(batches.batch(i), i, train_iter=NUM_ITERS * e + i))
        system.eval()
        system.set_train_iter(NUM_ITERS * (e + 1))
        if (e + 1) % 2 == 0:
            videos[e + 1] = system.render_video(views["render"]).cpu().numpy()
        split = "test" if (e + 1) % 2 == 0 else "val"
        metrics[e + 1] = hb.INRSystem.validation_epoch_end(system.validation_views(views[split], images[split]))
        system.train()
        records.append({"epoch": e, **system.training_epoch_end(outputs), **metrics[e + 1]})
    return system, batches, views, records, videos, metrics


def close(a, b, what, rel=1e-3):
    a, b = a.float().cpu(), b.float().cpu()
    assert a.shape == b.shape, what
    if a.numel() == 0:
        return
    scale = max(float(a.abs().max()), 1e-12)
    assert float((a - b).abs().max()) <= rel * scale, (what, float((a - b).abs().max()), scale)


def same_state(got, want, what):
    """Two full checkpoints: equal discrete state, parameters and Adam moments within `close`."""
    assert got["epoch"] == want["epoch"] and got["global_step"] == want["global_step"], what
    assert set(got["state_dict"]) == set(want["state_dict"]), what
    for k, v in want["state_dict"].items():
        if v.dtype in (torch.int64, torch.bool) or k.endswith(("aabb", "gridSize", "alpha_volume")):
            assert torch.equal(got["state_dict"][k], v), (what, k)
        else:
            close(got["state_dict"][k], v, (what, k))
    assert len(got["optimizer_states"]) == len(want["optimizer_states"]), what
    for g, (og, ow) in enumerate(zip(got["optimizer_states"], want["optimizer_states"])):
        assert og["param_groups"] == ow["param_groups"], (what, g)
        assert og["state"].keys() == ow["state"].keys(), (what, g)
        for j, s in ow["state"].items():
            assert torch.equal(og["state"][j]["step"], s["step"]), (what, g, j)
            for m in ("exp_avg", "exp_avg_sq"):
                close(og["state"][j][m], s[m], (what, g, j, m))
    assert got["lr_schedulers"] == want["lr_schedulers"], what
    eg, ew = dict(got[STATE_KEY]), dict(want[STATE_KEY])
    assert torch.equal(eg.pop("rng_state"), ew.pop("rng_state")), what
    for k in ("aabb", "gridSize"):
        assert torch.equal(eg.pop(k), ew.pop(k)), (what, k)
    assert eg == ew, what


def same_records(got, want):
    assert [sorted(r) for r in got] == [sorted(r) for r in want]
    for g, w in zip(got, want):
        assert g["epoch"] == w["epoch"]
        for k in w:
            if k != "epoch":
                assert abs(g[k] - w[k]) <= 1e-4 * max(1.0, abs(w[k])), (w["epoch"], k, g[k], w[k])


def checkpoint_of(system, batches, epoch, weights_only=False):
    return checkpoint(system, batches, epoch, NUM_ITERS * (epoch + 1), weights_only=weights_only)


@pytest.fixture(scope="module")
def uninterrupted(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("fit")
    cfg, root = make_run(tmp)
    out = str(tmp / "run")
    records = hb.fit(cfg, root, out, read_frame=read_frame, **KW)
    return cfg, root, out, records


def test_fit_equals_the_hand_written_loop(uninterrupted, tmp_path):
    cfg, root, out, records = uninterrupted
    system, batches, _, want_records, videos, metrics = hand_loop(cfg, root)
    assert [r["epoch"] for r in records] == list(range(EPOCHS))
    assert set(records[0]) == {"epoch", "train/loss", "train/psnr", "val/loss", "val/psnr", "val/ssim"}
    same_records(records, want_records)
    net = system.render_fn.model.color_model.net
    assert net.N_voxel_list == [] and net.alphaMask is not None  # both up-samplings and both prunings ran
    last = torch.load(os.path.join(out, "last.ckpt"), map_location="cpu", weights_only=True)
    same_state(last, checkpoint_of(system, batches, EPOCHS - 1), "fit vs hand loop")
    for e in range(EPOCHS):
        assert os.path.exists(os.path.join(out, f"epoch={e}.ckpt")) and os.path.exists(os.path.join(out, f"epoch={e}-weights.ckpt"))
        with open(os.path.join(out, str(e + 1), "metrics.txt")) as f:
            lines = f.read().splitlines()
        assert [ln.split(": ")[0] for ln in lines] == list(metrics[e + 1])
        for ln in lines:
            k, v = ln.split(": ")
            assert abs(float(v) - metrics[e + 1][k]) <= 1e-4 * max(1.0, abs(metrics[e + 1][k])), (e, k)
        video = os.path.join(out, str(e + 1), "video.npy")
        assert os.path.exists(video) == ((e + 1) % 2 == 0)
        if (e + 1) % 2 == 0:
            got = np.load(video)
            assert got.dtype == np.uint8 and got.shape == videos[e + 1].shape and got.shape[-1] == 3
            diff = np.abs(got.astype(np.int16) - videos[e + 1])
            assert diff.max() <= 1 and (diff == 0).mean() >= 0.99, e


def test_resume_from_last_ckpt_equals_the_uninterrupted_run(uninterrupted, tmp_path):
    cfg, root, out, records = uninterrupted
    resumed = str(tmp_path / "run")
    first = hb.fit(cfg, root, resumed, read_frame=read_frame, max_epochs=2, **KW)
    assert [r["epoch"] for r in first] == [0, 1]
    mid = torch.load(os.path.join(resumed, "last.ckpt"), map_location="cpu", weights_only=True)
    assert mid["epoch"] == 1 and MASK_PREFIX + "alpha_volume" in mid["state_dict"]  # pruned at 3; 4, 6 and 7 still to come
    rest = hb.fit(cfg, root, resumed, read_frame=read_frame, **KW)
    assert [r["epoch"] for r in rest] == [2, 3]
    same_records(first + rest, records)
    for e in range(EPOCHS):
        same_state(torch.load(os.path.join(resumed, f"epoch={e}.ckpt"), map_location="cpu", weights_only=True),
                   torch.load(os.path.join(out, f"epoch={e}.ckpt"), map_location="cpu", weights_only=True), e)
    assert hb.fit(cfg, root, resumed, read_frame=read_frame, **KW) == []  # nothing left to run


def test_the_steps_of_an_epoch_without_schedule_iterations_do_not_synchronise(tmp_path):
    """Epoch 1 of a run whose schedule lists lie past it, under torch.cuda.set_sync_debug_mode("error")."""
    cfg, root = make_run(tmp_path, upsamp=(100,), prune=(100,), restart=(100,))
    system, batches, _, _ = hand_loop(cfg, root, stop_before=(1, 0))
    batches.set_epoch(1)
    outputs = []
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for i in range(len(batches)):
            outputs.append(system.training_step(batches.batch(i), i, train_iter=NUM_ITERS + i))
    finally:
        torch.cuda.set_sync_debug_mode("default")
    with warnings.catch_warnings():
        warnings.filterwarnings("ignore", message=".*lr_scheduler.step.*")
        means = system.training_epoch_end(outputs)
    assert all(np.isfinite(v) for v in means.values())


def test_last_weights_load_into_a_fresh_system_and_render_alike(uninterrupted):
    """fit's own files: last.ckpt restored into one fresh INRSystem (the trained state, as a resume sees it) and
    last-weights.ckpt loaded into another with load_state_dict render the same rgb bit for bit."""
    cfg, root, out, _ = uninterrupted
    weights = torch.load(os.path.join(out, "last-weights.ckpt"), map_location="cpu", weights_only=True)
    full = torch.load(os.path.join(out, "last.ckpt"), map_location="cpu", weights_only=True)
    assert set(weights) == {"epoch", "global_step", "state_dict"} and weights["epoch"] == EPOCHS - 1
    c = hb.to_cfg(json.loads(json.dumps(cfg)))
    c.training.iters_per_epoch = NUM_ITERS
    train = hb.dataset_cameras(c.dataset, root, "train")
    trained = hb.INRSystem(c, dataset=train.facts, **KW).cuda()
    restore(trained, types.SimpleNamespace(seed=0, epoch=0, set_epoch=lambda e: None), full)
    fresh = hb.INRSystem(c, dataset=train.facts, **KW)
    fresh.load_state_dict(weights)
    fresh.cuda()
    rays = hb.generate_rays(hb.dataset_cameras(c.dataset, root, "test").cameras[0], c_in=fresh.render_fn.model.sig.c_in)
    rgb = []
    for s in (trained, fresh):
        s.eval()
        s.set_train_iter(NUM_ITERS * EPOCHS)  # the eased heads at the iteration the run's last validation set
        with torch.no_grad():
            rgb.append(s(rays)["rgb"])
    assert float(rgb[0].abs().sum()) > 0 and torch.equal(rgb[0], rgb[1])


@pytest.mark.parametrize("case,file_mode", [("technicolor_lightfield", "RGBA"), ("donerf_center", "RGB")])
def test_default_reader_loads_frames_as_get_rgb(case, file_mode, tmp_path):
    """load_frames without a reader on real PNG files whose mode is not the dataset's: an RGBA Technicolor capture is read
    as RGB and an RGB DoNeRF capture as RGBA, as get_rgb converts them, then resized like any frame."""
    from PIL import Image

    root, dcfg = make_scene(_scenes(), case, tmp_path)
    dcfg = dict(dcfg, img_wh=[16, 12])
    views = hb.dataset_cameras(dcfg, root, "val")
    rng = np.random.default_rng(3)
    want = []
    for f in views.frames:
        arr = rng.integers(0, 256, (24, 32, len(file_mode)), dtype=np.uint8)
        os.makedirs(os.path.dirname(f.path), exist_ok=True)  # the scene lists its image files but need not hold them
        Image.fromarray(arr, file_mode).save(f.path, format="PNG")
        with Image.open(f.path) as im:
            want.append(np.asarray(im.convert("RGBA" if views.rgba else "RGB")))
    got = load_frames(views, dcfg)
    assert got.shape == (len(views.frames), 12, 16, 4 if views.rgba else 3)
    assert torch.equal(got, hb.dataset_frames(dcfg, torch.from_numpy(np.stack(want)).cuda()))
