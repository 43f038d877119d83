"""One training run of a reference config from a scene directory: the order in which the reference's ``main.py`` and
Lightning call ``INRSystem`` (nlf/__init__.py), on one GPU, with resumable checkpoints.

``fit(cfg, root, out_dir)`` loads the train, val, test and render splits (``dataset_cameras``), reads and resizes their
frames on the device (``dataset_frames``), trains on ``DeviceRayBatches.from_config`` and, epoch by epoch, runs

    for i in range(len(batches)):                                   # Lightning's training loop
        system.training_step(batches.batch(i), i, train_iter=num_iters * epoch + i)   # get_train_iter, :580-606
    if (epoch + 1) % val_every == 0:                                # check_val_every_n_epoch
        system.set_train_iter(max(get_train_iter(epoch + 1, 0, val=True), 0))        # validation_step, :985-991
        if (epoch + 1) % render_every == 0: system.render_video(render split)      # :998-1001
        system.validation_views(test split if (epoch + 1) % test_every == 0 else val split)   # :248-275, :1004
    system.training_epoch_end(outputs)                              # the scheduler step, :711-725
    if (epoch + 1) % ckpt_every == 0: save epoch={epoch}.ckpt, last.ckpt and their -weights twins   # main.py:126-148

Validation runs at the end of the last training batch, before ``training_epoch_end`` (DESIGN §4.4h).  A run whose
``out_dir`` holds ``last.ckpt`` resumes from it at the next epoch (main.py:116-124).  Nothing between two
``training_epoch_end`` calls reads the device back, except the schedule iterations (up-sampling, occupancy pruning) and
the evaluations.
"""
from __future__ import annotations

import copy
import os
from functools import partial
from typing import Callable, List, Optional

import numpy as np
import torch

from .config import to_cfg, to_plain
from .datasets import DatasetViews, FrameSource, dataset_cameras
from .resize import dataset_frames
from .signature import UnsupportedPipeline, lower
from .state import _AlphaGrid
from .system import INRSystem
from .train_data import DeviceRayBatches

SPLITS = ("train", "val", "test", "render")
# the checkpoint key that holds what a bit-exact resume needs beyond Lightning's own keys
STATE_KEY = "hyperreel_b200"
MASK_PREFIX = "render_fn.model.color_model.net.alphaMask."
# Lightning's max_epochs when neither max_epochs nor max_steps is set (INRTrainer passes None without num_epochs, :70)
DEFAULT_EPOCHS = 1000
FRAMES_PER_UPLOAD = 8


# ---------------------------------------------------------------------------------------------------- the epoch rules

def num_iters(training, n_rows: int) -> int:
    """get_train_iter's iterations per epoch (nlf/__init__.py:587-592): ``num_iters`` with replacement, otherwise
    ``len(train_dataset) // batch_size`` (the rows of the training table, floored)."""
    if training.get("sample_with_replacement", False):
        return int(training["num_iters"])
    return int(n_rows) // int(training["batch_size"])


def get_train_iter(training, n_rows: int, epoch: int, batch_idx: int) -> int:
    """get_train_iter (nlf/__init__.py:580-606) on one GPU: rank 0, no regulariser pre-training iterations, neither
    render_only, test_only nor load_from_weights."""
    return num_iters(training, n_rows) * int(epoch) + int(batch_idx)


def epoch_events(training, epoch: int) -> dict:
    """What follows the training batches of ``epoch`` (0-based, Lightning's ``current_epoch``):

    - ``validate``: ``(epoch + 1) % val_every == 0`` (``check_val_every_n_epoch``);
    - ``split``: the split validation scores, ``'test'`` when ``(epoch + 1) % test_every == 0``, else ``'val'``
      (val_dataloader, :248-275, as training_epoch_end's ``reset_val`` re-creates it, :730-752);
    - ``render``: the render split's video, on validating epochs with ``(epoch + 1) % render_every == 0`` (:998-1001);
    - ``checkpoint``: ``(epoch + 1) % ckpt_every == 0`` (INRModelCheckpoint's every_n_epochs, main.py:44-50)."""
    e1 = int(epoch) + 1
    validate = e1 % int(training["val_every"]) == 0
    return {"validate": validate, "split": "test" if e1 % int(training["test_every"]) == 0 else "val",
            "render": validate and e1 % int(training["render_every"]) == 0,
            "checkpoint": e1 % int(training["ckpt_every"]) == 0}


def _refuse(cfg) -> None:
    training = cfg.get("training", None)
    if training is None or "dataset" not in cfg or "model" not in cfg:
        raise ValueError("fit: cfg needs the reference's 'model', 'dataset' and 'training' sections")
    if int(training.get("num_gpus", 1)) != 1:
        raise UnsupportedPipeline(f"fit: training 'num_gpus' {training.get('num_gpus')} is not supported: fit trains on one "
                                  "GPU (num_gpus: 1)")
    if training.get("multiscale", False):
        raise UnsupportedPipeline("fit: training 'multiscale' is not supported (the datamodule's per-scale frames and lr)")
    if int(training.get("num_regularizer_pretraining_iters", 0)) != 0:
        raise UnsupportedPipeline("fit: training 'num_regularizer_pretraining_iters' is not supported (negative iterations "
                                  "skip the image loss, :663)")
    for key in ("val_every", "test_every", "render_every", "ckpt_every", "batch_size"):
        if key not in training:
            raise ValueError(f"fit: cfg.training.{key} is needed")


# -------------------------------------------------------------------------------------------------------------- frames

def read_image(source: FrameSource, rgba: bool = False) -> np.ndarray:
    """The default frame reader: the image file of ``source`` with Pillow, converted as the dataset's ``get_rgb`` converts
    it whatever the file's own mode: uint8 ``[h, w, 3]`` (``.convert("RGB")``, datasets/technicolor.py:400-402), or
    ``[h, w, 4]`` with ``rgba`` (``.convert("RGBA")``, datasets/donerf.py:240).  A video frame raises ``ValueError``."""
    if source.frame is not None:
        raise ValueError(f"fit: {source.path} frame {source.frame} is a video frame: pass read_frame to decode it")
    from PIL import Image

    with Image.open(source.path) as im:
        return np.asarray(im.convert("RGBA" if rgba else "RGB"))


def load_frames(views: DatasetViews, dataset_cfg, read_frame: Optional[Callable] = None,
                device: Optional[torch.device] = None) -> torch.Tensor:
    """The ground truth of every view of ``views`` as the reference's ``get_rgb`` makes it, uint8 ``[n, H, W, 3]`` (``[n, H,
    W, 4]`` for RGBA datasets) on the device: ``read_frame`` at capture size (default ``read_image`` with the split's
    ``rgba``), a few views at a time, each group resized by ``dataset_frames`` into its slice of the one output tensor."""
    if read_frame is None:
        read_frame = partial(read_image, rgba=views.rgba)
    device = device or torch.device("cuda", torch.cuda.current_device())
    W, H = (int(v) for v in dataset_cfg["img_wh"])
    ch = 4 if views.rgba else 3
    out = torch.empty((len(views.frames), H, W, ch), dtype=torch.uint8, device=device)
    for i in range(0, len(views.frames), FRAMES_PER_UPLOAD):
        group = []
        for source in views.frames[i:i + FRAMES_PER_UPLOAD]:
            frame = torch.from_numpy(np.ascontiguousarray(read_frame(source)))
            if frame.dtype != torch.uint8 or frame.dim() != 3 or frame.shape[-1] != ch:
                raise ValueError(f"fit: read_frame({source}) gave {frame.dtype} {tuple(frame.shape)}, uint8 [h, w, {ch}] is "
                                 "needed")
            group.append(frame)
        dataset_frames(dataset_cfg, torch.stack(group).to(device), out=out[i:i + len(group)])
    return out


# ---------------------------------------------------------------------------------------------------------- checkpoints

def checkpoint(system: INRSystem, batches: DeviceRayBatches, epoch: int, global_step: int, weights_only: bool = False) -> dict:
    """Lightning's checkpoint layout of the run after ``epoch``'s ``training_epoch_end``: ``epoch``, ``global_step`` (the
    training steps run), ``state_dict`` (``INRSystem.state_dict()``: ``render_fn.model...``, as the reference's
    load_state_dict reads it, with the occupancy mask under its AlphaGridMask names once pruning has made one), and unless
    ``weights_only`` ``optimizer_states`` (one Adam state_dict per group in ``optimizer_groups()`` order),
    ``lr_schedulers`` and ``STATE_KEY``: the TensoRF regulariser's running weights, the aabb, the grid size and the
    up-sampling steps still to come, the torch CPU generator (the white-background coin flip), the batches' seed and epoch
    and the ease / schedule modes."""
    net = system.render_fn.model.color_model.net
    mask = net.alphaMask
    state_dict = {k: v.detach().cpu().clone() for k, v in system.state_dict().items()}
    if mask is not None:  # the reference's AlphaGridMask buffers (utils/tensorf_utils.py:459-467), read by its load_state_dict
        state_dict[MASK_PREFIX + "alpha_aabb"] = mask.aabb.detach().cpu().clone()
        state_dict[MASK_PREFIX + "alpha_volume"] = mask.volume.detach().cpu().clone()
    out = {"epoch": int(epoch), "global_step": int(global_step), "state_dict": state_dict}
    if weights_only:
        return out
    out["optimizer_states"] = [copy.deepcopy(o.state_dict()) for o in system.optimizers()]
    out["lr_schedulers"] = [copy.deepcopy(s.state_dict()) for s in system.lr_schedulers()]
    out[STATE_KEY] = {
        "regularizers": [{"cur_iter": r.cur_iter, "L1_reg_weight": r.L1_reg_weight, "TV_weight_density": r.TV_weight_density,
                          "TV_weight_app": r.TV_weight_app} for r in system.regularizers],
        "aabb": net.aabb.detach().cpu().clone(),
        "gridSize": net.gridSize.detach().cpu().clone(),
        "N_voxel_list": copy.deepcopy(net.N_voxel_list),
        "net_cur_iter": net.cur_iter,
        "training_started": bool(system.training_started),
        "rng_state": torch.get_rng_state(),
        "batches": {"seed": int(batches.seed), "epoch": int(batches.epoch)},
        "ease": system.ease, "schedule": system.schedule,
    }
    return out


def restore(system: INRSystem, batches: DeviceRayBatches, ckpt: dict) -> int:
    """Puts ``system`` and ``batches`` in the state ``checkpoint`` recorded; returns the checkpoint's epoch.  The CPU
    generator is restored last: loading a grown grid re-creates the tables, which draws from it."""
    state = ckpt.get(STATE_KEY)
    if state is None or "optimizer_states" not in ckpt:
        raise ValueError("fit: the checkpoint holds weights only; resuming needs a full checkpoint (last.ckpt)")
    for key, have in (("ease", system.ease), ("schedule", system.schedule)):
        if state[key] != have:
            raise ValueError(f"fit: the checkpoint was trained with {key}={state[key]!r}, this run has {key}={have!r}")
    dev = next(system.parameters()).device
    system.load_state_dict(ckpt["state_dict"])  # re-creates the tables at the checkpoint's gridSize, on the host
    system.to(dev)
    net = system.render_fn.model.color_model.net
    net.aabb.copy_(state["aabb"].to(dev))
    net.update_stepSize(state["gridSize"])
    net.gridSize = net.gridSize.to(dev)
    net.N_voxel_list = copy.deepcopy(state["N_voxel_list"])
    net.cur_iter = state["net_cur_iter"]
    sd = ckpt["state_dict"]
    net.alphaMask = None if MASK_PREFIX + "alpha_volume" not in sd else \
        _AlphaGrid(sd[MASK_PREFIX + "alpha_aabb"].to(dev), sd[MASK_PREFIX + "alpha_volume"].to(dev))
    if len(state["regularizers"]) != len(system.regularizers):
        raise ValueError("fit: the checkpoint's regularisers differ from the config's")
    for reg, s in zip(system.regularizers, state["regularizers"]):
        reg.cur_iter, reg.L1_reg_weight = s["cur_iter"], s["L1_reg_weight"]
        reg.TV_weight_density, reg.TV_weight_app = s["TV_weight_density"], s["TV_weight_app"]
    system.render_fn.model.mark_dirty()
    system.configure_optimizers()
    if len(ckpt["optimizer_states"]) != len(system.optimizers()) or \
            len(ckpt["lr_schedulers"]) != len(system.lr_schedulers()):
        raise ValueError("fit: the checkpoint's optimisers differ from the config's groups")
    for opt, s in zip(system.optimizers(), ckpt["optimizer_states"]):
        opt.load_state_dict(s)
    for sched, s in zip(system.lr_schedulers(), ckpt["lr_schedulers"]):
        sched.load_state_dict(s)
    system.training_started = state["training_started"]
    batches.seed = state["batches"]["seed"]
    batches.set_epoch(state["batches"]["epoch"])
    torch.set_rng_state(state["rng_state"])
    return int(ckpt["epoch"])


def _save(system, batches, out_dir, epoch, global_step) -> None:
    full = checkpoint(system, batches, epoch, global_step)
    weights = {k: full[k] for k in ("epoch", "global_step", "state_dict")}  # Lightning's save_weights_only keys
    for name, obj in ((f"epoch={epoch}", full), (f"epoch={epoch}-weights", weights), ("last", full),
                      ("last-weights", weights)):
        path = os.path.join(out_dir, f"{name}.ckpt")
        torch.save(obj, path + ".tmp")
        os.replace(path + ".tmp", path)  # a run stopped mid-write leaves the previous last.ckpt whole


def write_metrics(path: str, metrics: dict) -> None:
    """validation_epoch_end's metrics.txt (nlf/__init__.py:1021-1028): one ``key: value`` line per key."""
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "w") as f:
        for key, val in metrics.items():
            f.write(f"{key}: {float(val)}\n")


# ------------------------------------------------------------------------------------------------------------------ fit

def fit(cfg, root: str, out_dir: str, *, read_frame: Optional[Callable] = None, max_epochs: Optional[int] = None,
        seed: int = 0, **system_kwargs) -> List[dict]:
    """Trains ``cfg`` (a full reference config: ``model``, ``dataset``, ``training``, ``regularizers``) on the scene
    directory ``root`` in the reference's order (module docstring) and returns one record per epoch run: ``epoch``, the
    epoch means of ``training_epoch_end`` and, on validating epochs, the scored split's ``val/loss``, ``val/psnr`` and
    ``val/ssim`` (floats).

    ``read_frame(FrameSource)`` returns a view's ground truth, uint8 ``[h, w, 3]`` (``[h, w, 4]`` for DoNeRF) at capture
    size; the default reads image files with Pillow and converts them to RGB, or RGBA for DoNeRF, as ``get_rgb`` does;
    a dataset of video frames needs one.  ``seed`` seeds the CPU generator before the system is built (its initial
    weights) and the training batches.  ``system_kwargs`` go to
    ``INRSystem`` (``mlp_mode``, ``train_net``, ``ease``, ``schedule``).  ``max_epochs`` stops after that many epochs
    (default ``cfg.training.num_epochs``, Lightning's 1000 without it).

    Under ``out_dir``: ``{epoch + 1}/metrics.txt`` per validating epoch, ``{epoch + 1}/video.npy`` (uint8 ``[F, H, W, 3]``)
    per rendering epoch, and every ``ckpt_every`` epochs ``epoch={epoch}.ckpt``, ``last.ckpt`` and their ``-weights`` twins
    (``checkpoint``).  When ``out_dir/last.ckpt`` exists the run resumes from it at the next epoch."""
    cfg = to_cfg(copy.deepcopy(to_plain(cfg)))
    _refuse(cfg)
    training, dcfg = cfg.training, cfg.dataset
    views = {s: dataset_cameras(dcfg, root, s) for s in SPLITS}  # the datamodule's four datasets (:150-163)
    if read_frame is None:
        video = next((f for s in SPLITS for f in views[s].frames if f.frame is not None), None)
        if video is not None:
            raise ValueError(f"fit: {video.path} is a video: pass read_frame to decode its frames")
    torch.manual_seed(int(seed))
    device = torch.device("cuda", torch.cuda.current_device())
    images = {s: load_frames(views[s], dcfg, read_frame, device) for s in ("train", "val", "test")}
    train = views["train"]
    c_in = lower(cfg.model, train.facts).c_in
    batches = DeviceRayBatches.from_config(cfg, train.cameras, images["train"], seed=seed, c_in=c_in, device=device)
    # main.py:100-103: the epoch length that scales the configs' *_epoch(s) keys
    training.iters_per_epoch = int(training["num_iters"]) if training.get("sample_with_replacement", False) else len(batches)
    system = INRSystem(cfg, dataset=train.facts, **system_kwargs).to(device)
    n_iters = num_iters(training, batches.n_rows)

    os.makedirs(out_dir, exist_ok=True)
    start = 0
    last = os.path.join(out_dir, "last.ckpt")
    if os.path.exists(last):
        start = restore(system, batches, torch.load(last, map_location="cpu", weights_only=True)) + 1
    end = int(max_epochs if max_epochs is not None else training.get("num_epochs", DEFAULT_EPOCHS))
    records = []
    for epoch in range(start, end):
        batches.set_epoch(epoch)
        outputs = [system.training_step(batches.batch(i), i, train_iter=n_iters * epoch + i) for i in range(len(batches))]
        events = epoch_events(training, epoch)
        metrics = {}
        if events["validate"]:
            edir = os.path.join(out_dir, str(epoch + 1))
            system.eval()  # validation_step: render_fn.eval() first, so the schedule's up-sampling and pruning wait
            system.set_train_iter(max(get_train_iter(training, batches.n_rows, epoch + 1, 0), 0))
            if events["render"]:
                os.makedirs(edir, exist_ok=True)
                np.save(os.path.join(edir, "video.npy"), system.render_video(views["render"]).cpu().numpy())
            split = events["split"]
            metrics = INRSystem.validation_epoch_end(system.validation_views(views[split], images[split]))
            write_metrics(os.path.join(edir, "metrics.txt"), metrics)
            system.train()
        record = {"epoch": epoch, **system.training_epoch_end(outputs), **metrics}
        records.append(record)
        if events["checkpoint"]:
            _save(system, batches, out_dir, epoch, len(batches) * (epoch + 1))
    return records
