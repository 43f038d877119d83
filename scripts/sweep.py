#!/usr/bin/env python
"""Throughput sweep over the BASELINE.json configurations (device-resident inputs, CUDA events, L2 flushed):

    python scripts/sweep.py --out sweep.json

For each workload x rays-per-batch it reports Mrays/s of the whole path and the two kernel times.  Rays are
rendered in one hr_render call (no chunking).  Single GPU; the multi-GPU numbers come from bench.py --gpus N.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import hyperreel_b200 as hb  # noqa: E402
from hyperreel_b200.state import seeded_state_dict  # noqa: E402

WORKLOADS = {
    # name: (builtin, overrides, note)
    "technicolor_S32_K12": ("technicolor_z_plane", dict(n_voxels=512000000), "2048x1088-shape video model, grid 1007x1007x503"),
    "technicolor_S32_K50": ("technicolor_z_plane", dict(n_voxels=512000000, num_keyframes=50), "same, 50 keyframes"),
    "donerf_sphere_S16": ("donerf_sphere", dict(n_voxels=216000000, z_channels=16), "800x800-shape static model, grid 600^3, 16 samples"),
    "donerf_sphere_S32": ("donerf_sphere", dict(n_voxels=216000000), "same, 32 samples (YAML default)"),
    "neural3d_S64": ("neural_3d_z_plane", dict(n_voxels=262144000), "2704x2028-shape video model, grid 823x617x514, 64 samples"),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--rays", default="65536,262144,1048576,4194304")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--mlp", default="bf16x3")
    ap.add_argument("--only", default="", help="comma-separated workload names (default: all)")
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    flush = torch.empty((512 << 20) // 4, dtype=torch.float32, device=dev)
    rows = []
    only = [w for w in args.only.split(",") if w]
    for wname, (builtin, over, note) in WORKLOADS.items():
        if only and wname not in only:
            continue
        cfg, ds = hb.configs.get(builtin, **over)
        sig = hb.lower(cfg, ds)
        sd = seeded_state_dict(sig, seed=11, density_gain=30.0)
        model = hb.LightfieldModel(cfg, dataset=ds, mlp_mode=args.mlp)
        render = hb.RenderLightfield(model, None, cfg.render)
        render.load_state_dict(sd, strict=False)
        render.eval()
        for n in [int(x) for x in args.rays.split(",")]:
            if n * sig.cfg.mlp_out * 4 > 20e9:
                continue
            rays = hb.rays.for_signature(sig, n, seed=5).to(dev)
            for _ in range(3):
                render(rays)
            torch.cuda.synchronize()
            model.timing(True)
            evs = []
            for _ in range(args.steps):
                flush.zero_()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                render(rays)
                b.record()
                evs.append((a, b))
            torch.cuda.synchronize()
            tm = model.timing_read()
            model.timing(False)
            ms = sum(a.elapsed_time(b) for a, b in evs) / len(evs)
            row = {"workload": wname, "note": note, "rays": n, "samples": sig.n_samples, "ms": ms, "mrays_s": n / ms / 1e3,
                   "render_kernel_ms": tm["render_ms"], "sample_net_ms": tm["mlp_ms"], "sample_net": args.mlp}
            rows.append(row)
            print(json.dumps(row), flush=True)
            del rays
        del model, render
        torch.cuda.empty_cache()
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
