"""Golden values of the EaseValue warm-up (nlf/activations.py:462-496) from the unmodified reference (through
oracle/ref_shim.py, CPU), at the iterations of tests/ease_cases.py (iters_per_epoch = 4000):

  ease_<case>.npz   per iteration i: rgb of the eval-mode forward after ``model.set_iter(i)``; unless the case is forward-only,
                    d loss / d parameter (loss = mean((rgb - target)^2), L2 norm, max |g| and 64 probes per parameter, as in
                    make_golden_grads_train.py) and the losses of a five-step training loop from iteration 6000: set_iter,
                    training-mode forward, MSE, backward, one Adam(betas=(0.9, 0.99), eps=1e-8) per optimiser group at
                    INRSystem.OPT_DEFAULTS, every optimiser restarted when the colour net re-creates its tables (as
                    INRSystem.set_train_iter does)
  ease_activations.npz   every EaseValue of every shipped model YAML that lowers, applied to a fixed input at each iteration

    python tests/golden/make_golden_ease.py
"""
from __future__ import annotations

import glob
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

import hyperreel_b200 as hb  # noqa: E402
from oracle import ref_shim  # noqa: E402
from tests.ease_cases import (EASE_CASES, ITERS, ITERS_PER_EPOCH, LOOP_START, LOOP_STEPS, SHIPPED_DIR, build_ease_case,  # noqa: E402
                              ease_value_cfgs, in_iters, loop_seed, loop_target, opt_group)
from tests.golden.make_golden_grads import probe_indices, target_for  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
ACT_INPUT = torch.linspace(-8.0, 8.0, 97)


def build(case):
    ref = ref_shim.build_reference(case.model_cfg_plain, case.dataset, iters_per_epoch=ITERS_PER_EPOCH)
    _, unexpected = ref.load_state_dict(case.state_dict, strict=False)
    assert not unexpected, unexpected
    return ref


def reference_loop(case):
    ref = build(case)
    ref.train()

    def optimizers():
        groups = {}
        for k, p in ref.named_parameters():
            p.requires_grad_(True)
            if p.numel() > 0 and opt_group(k) is not None:
                groups.setdefault(opt_group(k), []).append(p)
        return [torch.optim.Adam(ps, lr=hb.INRSystem.OPT_DEFAULTS[g], eps=1e-8, betas=(0.9, 0.99)) for g, ps in groups.items()]

    def ids():
        return [id(p) for p in ref.parameters()]

    opts, held = optimizers(), ids()
    target = loop_target(case.rays.shape[0])
    losses = []
    for step in range(LOOP_STEPS):
        ref.model.set_iter(LOOP_START + step)
        if ids() != held or getattr(ref.model.color_model.net, "needs_opt_reset", False):
            opts, held = optimizers(), ids()  # the up-sampling schedule replaced the tables: new Parameters, fresh Adam state
        torch.manual_seed(loop_seed(step))
        loss = ((ref(case.rays.clone())["rgb"].reshape(-1, 3) - target) ** 2).mean()
        for o in opts:
            o.zero_grad(set_to_none=True)
        loss.backward()
        for o in opts:
            o.step()
        losses.append(float(loss.detach()))
    return np.array(losses)


def main():
    ref_shim.install()
    for name, spec in EASE_CASES.items():
        case = build_ease_case(name)
        rec = {}
        for it in ITERS:
            ref = build(case)
            ref.eval()
            ref.model.set_iter(it)
            for p in ref.parameters():
                p.requires_grad_(not spec.get("forward_only"))
            rays = case.rays.clone()
            out = ref(rays)["rgb"].reshape(-1, 3)
            rec[f"{it}/rgb"] = out.detach().numpy()
            if spec.get("forward_only"):
                continue
            loss = ((out - target_for(rays.shape[0])) ** 2).mean()
            loss.backward()
            rec[f"{it}/loss"] = np.array(float(loss))
            for k, p in ref.named_parameters():
                if p.grad is None or p.numel() == 0:
                    continue
                g = p.grad.detach().reshape(-1)
                rec[f"{it}/norm/{k}"] = np.array(float(g.norm()))
                rec[f"{it}/max/{k}"] = np.array(float(g.abs().max()))
                rec[f"{it}/probe/{k}"] = g[probe_indices(g.numel())].numpy()
        if not spec.get("forward_only"):
            rec["loop_losses"] = reference_loop(case)
        np.savez_compressed(os.path.join(OUT, f"ease_{name}.npz"), **rec)
        print(name, {it: float(np.abs(rec[f"{it}/rgb"]).mean()) for it in ITERS}, rec.get("loop_losses"))

    from nlf.activations import get_activation

    acts = {"input": ACT_INPUT.numpy()}
    for path in sorted(glob.glob(os.path.join(SHIPPED_DIR, "*.npz"))):
        yaml = os.path.basename(path)[:-4]
        g = np.load(path)
        plain = json.loads(str(g["config_json"]))
        try:
            hb.lower(hb.to_cfg(plain), json.loads(str(g["dataset_json"])))
        except hb.UnsupportedPipeline:
            continue
        for where, ecfg in ease_value_cfgs(plain).items():
            mod = get_activation(ref_shim.to_attr(in_iters(ecfg)))
            for it in ITERS:
                mod.set_iter(it)
                with torch.no_grad():
                    acts[f"{yaml}{where}/{it}"] = mod(ACT_INPUT.clone()).numpy()
    np.savez_compressed(os.path.join(OUT, "ease_activations.npz"), **acts)
    print("activations", len(acts) - 1)


if __name__ == "__main__":
    main()
