"""Golden GRADIENTS for the training cases of tests/cases_train.py (bbox / z_depth contraction, per-ray colour heads, the
per-camera colour transform, voxel-grid and deformable-plane primitives): d loss / d parameter from the reference's own
autograd, exactly as tests/golden/make_golden_grads.py does for its cases (unmodified modules through oracle/ref_shim.py,
CPU, eval-mode forward, loss = mean((rgb - target)^2) with its seeded target; per parameter: L2 norm, max |g|, 64 probes).

    python tests/golden/make_golden_grads_train.py
"""
from __future__ import annotations

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import ref_shim  # noqa: E402
from tests.cases_train import TRAIN_CASES, build_train_case  # noqa: E402
from tests.golden.make_golden_grads import probe_indices, target_for  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))


def main():
    ref_shim.install()
    for name in TRAIN_CASES:
        case = build_train_case(name)
        rays = case.rays.clone()
        ref = ref_shim.build_reference(case.model_cfg_plain, case.dataset)
        _, unexpected = ref.load_state_dict(case.state_dict, strict=False)
        assert not unexpected, (name, unexpected)
        ref.eval()
        for p in ref.parameters():
            p.requires_grad_(True)
        out = ref(rays.clone())["rgb"].reshape(-1, 3)
        loss = ((out - target_for(rays.shape[0])) ** 2).mean()
        loss.backward()
        rec = {"loss": np.array(float(loss))}
        for k, p in ref.named_parameters():
            if p.grad is None or p.numel() == 0:
                continue
            g = p.grad.detach().reshape(-1)
            rec[f"norm/{k}"] = np.array(float(g.norm()))
            rec[f"max/{k}"] = np.array(float(g.abs().max()))
            rec[f"probe/{k}"] = g[probe_indices(g.numel())].numpy()
        np.savez_compressed(os.path.join(OUT, f"grads_{name}.npz"), **rec)
        print(name, "loss", float(loss), "params with grad", sum(1 for k in rec if k.startswith("norm/")),
              "zero grads", [k[5:] for k in rec if k.startswith("norm/") and float(rec[k]) == 0.0])


if __name__ == "__main__":
    main()
