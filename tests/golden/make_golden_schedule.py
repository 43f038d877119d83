"""Golden learning rates of the reference's optimiser schedule: the unmodified ``get_optimizer`` / ``get_scheduler``
(utils/__init__.py:49-125) and ``INRSystem.configure_optimizers`` / ``needs_opt_reset`` / ``reset_optimizers``
(nlf/__init__.py:504-578) driven through a synthetic run of the reference's loop.  ``nlf/__init__.py`` needs Lightning,
OmegaConf and the datasets to import, so the three methods are compiled from its source on their own and bound to a
stand-in system whose ``trainer`` holds the optimisers and scheduler configs as Lightning's does.  Each iteration runs the
order of ``training_step`` (``needs_opt_reset`` then ``reset_optimizers``, :646-648) and records every group's lr, the lr
that iteration's ``opt.step()`` uses; each epoch ends with the scheduler step of ``training_epoch_end`` (:720-725).

    HYPERREEL_REFERENCE=<reference checkout> python tests/golden/make_golden_schedule.py

writes ``tests/golden/reference/schedule.npz``: for each case ``<case>/training_json`` (the training config, with
``iters_per_epoch``), ``<case>/groups`` (group names), ``<case>/lr`` float64 [iterations, groups] and ``<case>/restarts``
int64 [k, 2] (iteration, group index) of every optimiser the reference re-created; ``cases`` lists the case names.
"""
import ast
import copy
import json
import os
import sys
import types
import warnings
from collections import namedtuple

import numpy as np
import torch
import yaml

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import ref_shim  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference", "schedule.npz")
GROUPS = ["color", "color_impl", "embedding_impl", "embedding"]  # the fused path's groups (hyperreel_b200/system.py)


def _shipped(name, epochs=None):
    """conf/experiment/training/<name>_tensorf.yaml over its num_epochs (20 where it sets none) of num_iters iterations."""
    with open(os.path.join(ref_shim.REFERENCE_ROOT, "conf/experiment/training", f"{name}_tensorf.yaml")) as f:
        t = yaml.safe_load(f)
    t["iters_per_epoch"] = t["num_iters"]  # main.py:100-101 under sample_with_replacement
    return t, epochs or t.get("num_epochs", 20)


def _steplr():
    """conf/experiment/training/default.yaml, the shipped steplr schedule: its 'color' group (steplr) for the two colour
    groups and its 'embedding' group (exp) for the two embedding groups, two iterations per epoch, past the milestone."""
    with open(os.path.join(ref_shim.REFERENCE_ROOT, "conf/experiment/training/default.yaml")) as f:
        d = yaml.safe_load(f)
    opts = {"color": d["color"], "color_impl": d["color"], "embedding_impl": d["embedding"], "embedding": d["embedding"]}
    return {"optimizers": copy.deepcopy(opts), "iters_per_epoch": 2}, 2010


def _group(lr, kind="exp", **kw):
    return dict(optimizer="adam", lr=lr, momentum=0.9, weight_decay=0, lr_scheduler=kind, warmup_multiplier=1.0,
                warmup_epochs=0, **kw)


def _small():
    """Four iterations per epoch: restarts at a different set of iterations per group (some inside an epoch), a
    stop_epoch that zeroes one group's lr, and a steplr group.  Batches of 512 rows, drawn with replacement."""
    opts = {"color": _group(0.02, decay_epoch=2, decay_gamma=0.125, reset_opt_list=[4, 6, 8, 10, 12]),
            "color_impl": _group(0.001, decay_epoch=3, decay_gamma=0.5, reset_opt_list=[6, 12]),
            "embedding_impl": _group(0.00075, decay_epoch=2, decay_gamma=0.125, stop_epoch=3),
            "embedding": _group(0.01, "steplr", decay_epoch=2, decay_gamma=0.5, reset_opt_list=[8])}
    return {"batch_size": 512, "sample_with_replacement": True, "num_iters": 4, "iters_per_epoch": 4,
            "optimizers": opts}, 6


def _cosine_poly():
    opts = {"color": _group(0.02, "cosine", num_epochs=5),
            "color_impl": _group(0.001, "poly", num_epochs=8, poly_exp=0.9),
            "embedding_impl": _group(0.00075, "poly", num_epochs=6, poly_exp=2.0, reset_opt_list=[7]),
            "embedding": _group(0.01, "cosine", num_epochs=4, reset_opt_list=[5])}
    return {"iters_per_epoch": 3, "optimizers": opts}, 5


CASES = {"technicolor": lambda: _shipped("technicolor"), "neural_3d": lambda: _shipped("neural_3d"),
         "immersive": lambda: _shipped("immersive"), "shiny": lambda: _shipped("shiny"), "steplr": _steplr,
         "small": _small, "cosine_poly": _cosine_poly}


def _reference_methods():
    """configure_optimizers / needs_opt_reset / reset_optimizers compiled from the reference's nlf/__init__.py."""
    from utils import get_optimizer, get_scheduler

    path = os.path.join(ref_shim.REFERENCE_ROOT, "nlf", "__init__.py")
    tree = ast.parse(open(path).read(), path)
    cls = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == "INRSystem")
    wanted = ("configure_optimizers", "needs_opt_reset", "reset_optimizers")
    defs = [n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name in wanted]
    assert [d.name for d in defs] == list(wanted)
    ns = {"copy": copy, "namedtuple": namedtuple, "get_optimizer": get_optimizer, "get_scheduler": get_scheduler,
          "print": lambda *a, **k: None}
    exec(compile(ast.Module(body=defs, type_ignores=[]), path, "exec"), ns)
    return [ns[n] for n in wanted]


class _Trainer:
    """The parts of a Lightning Trainer the three methods touch."""

    def __init__(self):
        self.datamodule = types.SimpleNamespace(cur_lr=1.0)  # no multiscale in any shipped config
        self.strategy = types.SimpleNamespace(lr_scheduler_configs=[])
        self.optimizers = []

    @property
    def lr_scheduler_configs(self):
        return self.strategy.lr_scheduler_configs


def run(training, epochs):
    configure, needs_reset, reset = _reference_methods()
    ipe = training["iters_per_epoch"]
    t = ref_shim.to_attr(ref_shim.epochs_to_iters(copy.deepcopy(training), ipe))  # nlf/__init__.py:306-315, then :368-372
    system = types.SimpleNamespace(cfg=ref_shim.to_attr({"training": t}), trainer=_Trainer(), skip_opt_list=[],
                                   optimizer_configs={k: copy.deepcopy(t.optimizers[k]) for k in GROUPS},
                                   optimizer_groups={k: [torch.nn.Linear(2, 2)] for k in GROUPS})
    opts, scheds = configure(system)
    system.trainer.optimizers = opts
    system.trainer.strategy.lr_scheduler_configs = [namedtuple("scheduler_config", ("scheduler",))(s) for s in scheds]
    lr = np.zeros((epochs * ipe, len(GROUPS)))
    restarts = []
    training_started = False
    for epoch in range(epochs):
        for b in range(ipe):
            i = epoch * ipe + b  # get_train_iter (:580-606): one GPU, no regulariser pretraining
            training_started = True
            before = list(system.trainer.optimizers)
            if needs_reset(system, i):
                reset(system, i)
            restarts += [(i, g) for g, (a, o) in enumerate(zip(before, system.trainer.optimizers)) if a is not o]
            lr[i] = [o.param_groups[0]["lr"] for o in system.trainer.optimizers]
        if training_started:  # training_epoch_end (:720-725)
            for c in system.trainer.lr_scheduler_configs:
                c.scheduler.step()
    return lr, np.array(restarts, dtype=np.int64).reshape(-1, 2)


def main():
    ref_shim.install()
    warnings.filterwarnings("ignore", message=".*lr_scheduler.step.*")  # no opt.step() runs: only the lrs are recorded
    out = {"cases": np.array(list(CASES))}
    for name, make in CASES.items():
        training, epochs = make()
        lr, restarts = run(training, epochs)
        out[f"{name}/training_json"] = np.array(json.dumps(training))
        out[f"{name}/groups"] = np.array(GROUPS)
        out[f"{name}/lr"] = lr
        out[f"{name}/restarts"] = restarts
        print(name, lr.shape, "restarts", len(restarts), "final lr", lr[-1])
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
