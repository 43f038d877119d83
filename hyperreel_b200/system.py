"""Render-path surface of the reference's ``INRSystem`` (nlf/__init__.py:278-502).

Only what sits on the hot path is kept: construction from the full config (``cfg.model``, ``cfg.training``,
``cfg.dataset``), ``forward`` / ``render`` / ``run_chunked`` with the reference's chunk selection,
``load_state_dict`` with the reference's grid-size fix-up (nlf/__init__.py:433-479), including Lightning
checkpoints whose keys carry the ``render_fn.`` prefix, and -- SURVEY.md section 8 row f1 -- ``configure_optimizers`` /
``training_step`` (nlf/__init__.py:504-523, 634-709) over the differentiable path: image loss, manual optimisation with
one Adam per optimiser group, the TensoRF regulariser (L1 + TV on the tables, nlf/regularizers/tensorf.py:35-96) and the grid
up-sampling / occupancy-pruning schedule with its optimiser reset (tensorf_base.py:379-429,509-553,1151-1232), and, with
``schedule="reference"``, the optimisers' own schedule: one learning-rate scheduler per group stepped by
``training_epoch_end`` (utils/__init__.py:78-125, nlf/__init__.py:711-725) and the per-group ``reset_opt_list`` restarts
(nlf/__init__.py:529-578).  Visualisers and datasets are out of scope (SURVEY.md section 2).
"""
from __future__ import annotations

from functools import partial
from typing import Dict, Optional

import torch
from torch import nn

from .config import Cfg, epochs_to_iters, to_cfg
from .models import model_dict
from .rendering import render_chunked, render_fn_dict


class TVLoss(nn.Module):
    """nlf/regularizers/tensorf.py:14-32: 2 * (mean squared row difference + mean squared column difference) / batch."""

    def forward(self, x):
        count_h = x[:, :, 1:, :].size(1) * x[:, :, 1:, :].size(2) * x[:, :, 1:, :].size(3)
        count_w = x[:, :, :, 1:].size(1) * x[:, :, :, 1:].size(2) * x[:, :, :, 1:].size(3)
        h_tv = torch.pow(x[:, :, 1:, :] - x[:, :, :-1, :], 2).sum()
        w_tv = torch.pow(x[:, :, :, 1:] - x[:, :, :, :-1], 2).sum()
        return 2 * (h_tv / count_h + w_tv / count_w) / x.size(0)


class TensoRFRegularizer:
    """The TensoRF regulariser of the reference (nlf/regularizers/tensorf.py:35-96; conf/experiment/regularizers/tensorf/
    *.yaml): L1 on the density tables plus total variation on the space planes, the TV weights decaying by `lr_factor` per
    use exactly like the reference (which scales the *running* weights but multiplies by the configured ones, :79-88)."""

    def __init__(self, cfg):
        import math

        self.cfg = to_cfg(cfg)
        self.tvreg = TVLoss()
        self.cur_iter = 0
        self.update_AlphaMask_list = list(self.cfg.get("update_AlphaMask_list", []))
        self.lr_factor = float(self.cfg.lr_decay_target_ratio) ** (1.0 / float(self.cfg.n_iters))
        self.total_num_tv_iters = (int(self.cfg.total_num_tv_iters) if "total_num_tv_iters" in self.cfg else
                                   int(round(math.log(1e-4) / math.log(float(self.cfg.lr_decay_target_ratio)) * float(self.cfg.n_iters))))
        self.L1_reg_weight = float(self.cfg.L1_weight_initial)
        self.TV_weight_density = float(self.cfg.TV_weight_density)
        self.TV_weight_app = float(self.cfg.TV_weight_app)

    def loss(self, tensorf):
        total = 0.0
        if self.L1_reg_weight > 0:
            total = total + self.L1_reg_weight * tensorf.density_L1()
        if self.cur_iter > self.total_num_tv_iters:
            return total
        loss_tv = 0.0
        if self.TV_weight_density > 0:
            self.TV_weight_density *= self.lr_factor
            loss_tv = tensorf.TV_loss_density(self.tvreg) * float(self.cfg.TV_weight_density)
            total = total + loss_tv
        if self.TV_weight_app > 0:
            self.TV_weight_app *= self.lr_factor
            loss_tv = loss_tv + tensorf.TV_loss_app(self.tvreg) * float(self.cfg.TV_weight_app)  # the density term is counted twice, as in :85-88
            total = total + loss_tv
        return total

    def set_iter(self, iteration):
        self.cur_iter = iteration
        if len(self.update_AlphaMask_list) > 0 and self.cur_iter == self.update_AlphaMask_list[0]:
            self.L1_reg_weight = float(self.cfg.L1_weight_rest)


def exp_decay(decay_gamma, stop_epoch, decay_epoch, epoch):
    """utils/__init__.py:78-84, the `exp` schedule's factor on the base learning rate."""
    if epoch > stop_epoch:
        return 0.0
    return decay_gamma ** (epoch / decay_epoch)


def poly_exp_decay(num_epochs, poly_exp, epoch):
    """utils/__init__.py:86-87, the `poly` schedule's factor."""
    return (1 - epoch / num_epochs) ** poly_exp


def make_scheduler(oc, optimizer):
    """get_scheduler (utils/__init__.py:89-125) for one group's config `oc` (cfg.training.optimizers.<group>): torch's own
    LambdaLR / MultiStepLR / CosineAnnealingLR, stepped once per epoch.  The GradualWarmupScheduler wrapper of
    `warmup_epochs > 0` is refused; no shipped training config sets it."""
    kind = oc.get("lr_scheduler")
    if oc.get("warmup_epochs", 0) > 0:
        raise NotImplementedError("warmup_epochs > 0 (GradualWarmupScheduler) is not mirrored")
    if kind == "exp":
        fn = partial(exp_decay, oc.decay_gamma, oc.stop_epoch if "stop_epoch" in oc else float("inf"), float(oc.decay_epoch))
        scheduler = torch.optim.lr_scheduler.LambdaLR(optimizer, fn)
    elif kind == "steplr":
        scheduler = torch.optim.lr_scheduler.MultiStepLR(optimizer, milestones=[oc.decay_epoch], gamma=oc.decay_gamma)
    elif kind == "cosine":
        scheduler = torch.optim.lr_scheduler.CosineAnnealingLR(optimizer, T_max=oc.num_epochs, eta_min=1e-8)
    elif kind == "poly":
        scheduler = torch.optim.lr_scheduler.LambdaLR(optimizer, partial(poly_exp_decay, oc.num_epochs, oc.poly_exp))
    else:
        raise NotImplementedError(f"lr_scheduler {kind!r}: only the reference's exp, steplr, cosine and poly are mirrored")
    return scheduler


class INRSystem(nn.Module):
    def __init__(self, cfg, dm=None, dataset: Optional[dict] = None, mlp_mode: str = "auto", train_net: str = "torch",
                 ease: str = "elapsed", schedule: str = "constant"):
        super().__init__()
        # "constant": every group trains at its configured lr, and every group restarts when the tables are re-created;
        # "reference": the reference's per-group lr schedulers (stepped by training_epoch_end) and reset_opt_list restarts
        if schedule not in ("constant", "reference"):
            raise ValueError(f"schedule must be 'constant' or 'reference', got {schedule!r}")
        self.schedule = schedule
        self.training_started = False
        self.cfg = to_cfg(cfg)
        self.dm = dm
        training = self.cfg.get("training", Cfg())
        ipe = training.get("iters_per_epoch", None)
        if ipe is not None:
            epochs_to_iters(self.cfg, ipe)  # nlf/__init__.py:306-315
        if dataset is None and dm is None and "dataset" in self.cfg:
            d = self.cfg.dataset
            dataset = {k: d[k] for k in ("name", "collection", "num_keyframes", "num_frames", "near", "far", "depth_range") if k in d}
        model = model_dict[self.cfg.model.type](self.cfg.model, system=self if dm is not None else None,
                                                dataset=dataset, iters_per_epoch=ipe, mlp_mode=mlp_mode,
                                                train_net=train_net, ease=ease)
        self.ease = ease
        self.rendering = False
        self.render_fn = render_fn_dict[self.cfg.model.render.type](
            model, None, self.cfg.model.render, net_chunk=training.get("net_chunk", 32768))
        # regularisers (nlf/__init__.py:396-407): only the TensoRF one touches this path's parameters
        self.regularizers = []
        for key, rcfg in (self.cfg.get("regularizers", Cfg()) or Cfg()).items():
            if rcfg.get("type") == "tensorf":
                self.regularizers.append(TensoRFRegularizer(rcfg))
            else:
                raise NotImplementedError(f"regularizer '{rcfg.get('type')}' is outside the fused path's scope")
        self.eval()

    # ---- nlf/__init__.py:481-502
    def render(self, method_name, coords, **render_kwargs):
        return self.run_chunked(coords, getattr(self.render_fn, method_name), **render_kwargs)

    def forward(self, coords, **render_kwargs):
        return self.run_chunked(coords, self.render_fn, **render_kwargs)

    def run_chunked(self, coords, fn, **render_kwargs):
        training = self.cfg.get("training", Cfg())
        if self.rendering or render_kwargs.pop("rendering", False):
            chunk = training.get("render_ray_chunk", training.get("ray_chunk", 1 << 20))
        else:
            chunk = training.get("ray_chunk", 1 << 20)
        return render_chunked(coords, fn, render_kwargs, chunk=chunk)

    # ---- nlf/__init__.py:504-523 + utils/__init__.py:49-76 (get_optimizer): one Adam(betas=(0.9, 0.99), eps=1e-8) per group
    OPT_DEFAULTS = {"color": 0.02, "color_impl": 0.001, "embedding_impl": 0.00075,  # conf/experiment/training/*_tensorf.yaml
                    "embedding": 0.01}

    def optimizer_groups(self):
        """Parameters by the reference's `opt_group` names: the VM tables ('color'), basis_mat ('color_impl'), the sample
        net ('embedding_impl') (nlf/nets/tensorf_base.py opt_group dict, nlf/embedding/ray.py net group) and, when the
        pipeline has a per-camera colour transform, its table ('embedding', ColorTransformEmbedding, point.py:567)."""
        model = self.render_fn.model
        net = model.color_model.net
        tables = [p for n, p in net.named_parameters() if "plane" in n or "line" in n]
        impl = [p for n, p in net.named_parameters() if "basis_mat" in n]
        emb = [p for n, p in model.embedding_model.named_parameters() if n.endswith("color_embedding")]
        groups = {"color": tables, "color_impl": impl,
                  "embedding_impl": [p for n, p in model.embedding_model.named_parameters() if not n.endswith("color_embedding")]}
        if emb:
            groups["embedding"] = emb
        return groups

    def _group_cfg(self, key):
        training = self.cfg.get("training", Cfg())
        oc = training.get("optimizers", Cfg()).get(key, Cfg())
        if self.schedule == "reference":
            if "lr_scheduler" not in oc:
                raise ValueError(f"schedule='reference' needs cfg.training.optimizers.{key}.lr_scheduler")
            if training.get("multiscale", False):
                raise NotImplementedError("multiscale training (the datamodule's per-scale cur_lr) is not mirrored")
            for k in ("skip_opt_list", "remove_skip_opt_list"):
                if k in oc:
                    raise NotImplementedError(f"{k} is not mirrored: no shipped training config sets it")
        return oc

    def _adam(self, key, oc, params):
        if oc.get("optimizer", "adam") != "adam":
            raise NotImplementedError("only the reference's default optimizer (adam) is mirrored")
        return torch.optim.Adam(params, lr=float(oc.get("lr", self.OPT_DEFAULTS[key])), eps=1e-8,
                                weight_decay=float(oc.get("weight_decay", 0)), betas=(0.9, 0.99))

    def configure_optimizers(self):
        """One Adam per non-empty group; with schedule="reference" also its scheduler (nlf/__init__.py:504-527: the lr times
        the datamodule's cur_lr, which is 1.0 without multiscale)."""
        self._optimizers, self._schedulers, self._opt_keys, self._reset_iters = [], [], [], []
        self._opt_struct = self.render_fn.model.color_model.net.struct_version
        for key, params in self.optimizer_groups().items():
            params = [p for p in params if p.numel() > 0]
            if not params:
                continue
            oc = self._group_cfg(key)
            self._optimizers.append(self._adam(key, oc, params))
            self._opt_keys.append(key)
            if self.schedule == "reference":
                self._schedulers.append(make_scheduler(oc, self._optimizers[-1]))
                self._reset_iters.append(frozenset(oc.get("reset_opt_list", None) or ()))
        return self._optimizers

    def optimizers(self):
        """The optimisers training_step steps, one per group in optimizer_groups() order (LightningModule.optimizers)."""
        return list(getattr(self, "_optimizers", []))

    def lr_schedulers(self):
        """Their schedulers with schedule="reference", in the same order; none with "constant"."""
        return list(getattr(self, "_schedulers", []))

    def _reference_restarts(self, train_iter: int):
        """needs_opt_reset / reset_optimizers (nlf/__init__.py:529-578): a group whose reset_opt_list holds train_iter gets a
        new Adam and a new scheduler (its lr back at the base); the others keep both.  The reference has no rule for tables
        re-created (up-sampling, shrink) at an iteration its 'color' group does not list: its Adam would go on stepping the
        stale Parameters.  Here the Adam of each group whose Parameters changed restarts on the new ones -- its moments and
        step counts dropped, as in a new Adam -- and its scheduler carries on, so the lr stays on its curve (DESIGN §7)."""
        net = self.render_fn.model.color_model.net
        groups = None
        if net.struct_version != self._opt_struct:
            groups = self.optimizer_groups()
            self._opt_struct = net.struct_version
        for idx, key in enumerate(self._opt_keys):
            listed = train_iter in self._reset_iters[idx]
            if not listed and groups is None:
                continue
            params = [p for p in (groups or self.optimizer_groups())[key] if p.numel() > 0]
            opt = self._optimizers[idx]
            if listed:
                oc = self._group_cfg(key)
                self._optimizers[idx] = self._adam(key, oc, params)
                self._schedulers[idx] = make_scheduler(oc, self._optimizers[idx])
            elif len(params) != len(opt.param_groups[0]["params"]) or any(
                    a is not b for a, b in zip(params, opt.param_groups[0]["params"])):
                opt.param_groups[0]["params"] = params
                opt.state.clear()

    def set_train_iter(self, train_iter: int):
        """The per-iteration hook of the reference's loop (nlf/__init__.py:592-632): the colour net's schedule (grid
        up-sampling, tensorf_base.py:509-553) and the regularisers' (`L1_weight_rest`), then the optimiser restarts.  With
        schedule="constant" every group restarts when the tables were re-created (`lr_upsample_reset`, nlf/__init__.py:541-578:
        Adam state of the old Parameter objects is meaningless for the new ones); with schedule="reference" the groups restart
        at their `reset_opt_list` iterations (_reference_restarts).  With ease="reference" the whole model's set_iter runs, as
        in the reference (nlf/__init__.py:608-614), so its EaseValue heads are eased at `train_iter` for this step and later
        renders."""
        model = self.render_fn.model
        if self.ease == "reference":
            model.set_iter(int(train_iter))  # includes the colour net's schedule
        else:
            model.color_model.set_iter(int(train_iter))
        for reg in self.regularizers:
            reg.set_iter(int(train_iter))
        net = model.color_model.net
        if self.schedule == "reference":
            if getattr(self, "_optimizers", None):
                self._reference_restarts(int(train_iter))
        elif getattr(net, "needs_opt_reset", False) or (getattr(self, "_opt_struct", None) not in (None, net.struct_version)):
            self.configure_optimizers()
            net.needs_opt_reset = False

    def training_step(self, batch, batch_idx: int = 0, train_iter: Optional[int] = None):
        """One iteration of nlf/__init__.py:634-709 on this path: batch {'coords' [N,C], 'rgb' [N,3], optional 'weight'};
        loss = MSE(rgb_pred * w, rgb * w) (losses.py 'mse') + regularisers, manual optimisation (zero_grad / backward / step
        per group).  `train_iter` (optional) drives the schedules like the reference's `set_train_iter`."""
        self.training_started = True
        self.train()
        if train_iter is not None:
            self.set_train_iter(train_iter)
        if not getattr(self, "_optimizers", None):
            self.configure_optimizers()
        coords, rgb = batch["coords"], batch["rgb"]
        weight = batch.get("weight", None)
        results = self(coords)
        pred = results["rgb"]
        if weight is not None:
            loss = torch.mean((pred * weight - rgb * weight) ** 2)
        else:
            loss = torch.mean((pred - rgb) ** 2)
        for reg in self.regularizers:  # nlf/__init__.py:677-683 (loss weight 1: `exponential_decay` with decay 1.0)
            loss = loss + reg.loss(self.render_fn.model.color_model.net)
        for opt in self._optimizers:
            opt.zero_grad(set_to_none=True)
        loss.backward()
        for opt in self._optimizers:
            opt.step()
        with torch.no_grad():
            psnr = -10.0 * torch.log10(torch.mean((pred.detach() - rgb) ** 2))  # metrics.py:37-45
        return {"train/loss": loss.detach(), "train/psnr": psnr}

    def training_epoch_end(self, outputs):
        """nlf/__init__.py:711-725, to be called after an epoch's training_steps with their outputs: steps every scheduler
        once if a training_step has run (the reference's `training_started`), and returns the epoch means of the outputs'
        keys ('train/loss', 'train/psnr') as Python floats -- get_mean_outputs (metrics.py:60-82), fp32 means on the device,
        read back in one copy, the epoch's one synchronisation."""
        if self.training_started:
            for scheduler in self.lr_schedulers():
                scheduler.step()
        if not outputs:
            return {}
        keys = list(outputs[0])
        means = torch.stack([torch.stack([o[k] for o in outputs]).mean() for k in keys]).tolist()
        return dict(zip(keys, means))

    # ---- nlf/__init__.py:895-982, 1015-1030
    def validation_image(self, batch, batch_idx: int = 0):
        """Scores one held-out view like the reference's validation_image, without visualisers, image files or logging.
        batch {'coords' [.., C], 'rgb' [.., 3], 'W', 'H'}: the view is rendered under no_grad in eval() (clamped output, as
        validation_step runs it, :987-1010) and the previous train / eval mode is restored.  Returns 0-d device tensors, so a
        loop over views never synchronises: 'val/loss' the unweighted MSE (MSELoss, losses.py:21-28), 'val/psnr' and
        'val/ssim' metrics.psnr / metrics.ssim of the [H, W, 3] frame (metrics.py:25-34), computed on the device in fp64."""
        from .metrics import image_metrics

        was_training = self.training
        self.eval()
        try:
            with torch.no_grad():
                coords = batch["coords"]
                rgb = batch["rgb"].reshape(-1, 3)
                W, H = int(batch["W"]), int(batch["H"])
                pred = self(coords.reshape(-1, coords.shape[-1]))["rgb"]
                loss = torch.mean((pred - rgb) ** 2)
                mse, ssim = image_metrics(pred.reshape(H, W, 3), rgb.reshape(H, W, 3))
                psnr = 10.0 * torch.log10(1.0 / mse[0])
        finally:
            self.train(was_training)
        return {"val/loss": loss, "val/psnr": psnr, "val/ssim": ssim[0]}

    @staticmethod
    def validation_epoch_end(outputs):
        """get_mean_outputs(outputs, cpu=True) (metrics.py): the NumPy mean over views of every key, as a Python float (a
        mean of per-view PSNRs, not the PSNR of the mean MSE).  One device-to-host copy per key."""
        return {k: float(torch.stack([o[k] for o in outputs]).cpu().numpy().mean()) for k in outputs[0]}

    # ---- nlf/__init__.py:433-479
    def load_state_dict(self, state_dict: Dict[str, torch.Tensor], strict: bool = False):
        if "state_dict" in state_dict and isinstance(state_dict["state_dict"], dict):
            state_dict = state_dict["state_dict"]  # a Lightning .ckpt
        net = self.render_fn.model.color_model.net
        sd = {}
        for k, v in state_dict.items():
            k2 = k if k.startswith("render_fn.") else "render_fn." + k
            sd[k2] = v
            if k2.endswith("color_model.net.gridSize"):
                net.gridSize = torch.as_tensor(v, dtype=torch.long).cpu()
                net.init_svd_volume(net.gridSize[0], net.device)
        own = self.state_dict()
        for k in list(sd.keys()):
            if k in own and any(t in k for t in ("app_plane", "density_plane", "app_line", "density_line")):
                if sd[k].shape != own[k].shape:
                    sd[k] = sd[k].view(*own[k].shape)
        missing = super().load_state_dict({k: v for k, v in sd.items() if k in own}, strict=False)
        net.update_stepSize(net.gridSize)
        self.render_fn.model.mark_dirty()
        return missing
