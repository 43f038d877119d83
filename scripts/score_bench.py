#!/usr/bin/env python
"""Evaluating a held-out split: every view rendered and scored (loss, PSNR, SSIM), three ways, on synthetic trained-like
parameters.

  score_views     INRSystem.validation_views: one hr_score_views call for the whole split (rays generated on the device,
                  frames rendered into a ring of fp32 frames and scored against the uint8 frames), then PSNR per view
  resident_loop   INRSystem.validation_image per view, fed from fp32 rays [H*W, c_in] and fp32 ground truth [H, W, 3] of every
                  view built before the timed loop and kept on the device
  per_view_loop   the same loop, each view's rays (generate_rays) and fp32 ground truth (u8 / 255) built from its
                  camera and uint8 frame inside the loop

Per workload: ms per view (CUDA events around the whole split on the current stream, then a synchronise; the three methods
alternated `--rounds` times, the median reported), the peak of torch's device allocations during the timed split over what
was allocated when it started, and what each method keeps resident (the uint8 frames; the fp32 rays and ground truth of the
resident loop).  The script asserts that the three give the same per-view metrics: PSNR and SSIM bit for bit, the loss to
1e-6 relative (validation_image takes an fp32 mean, score_views rounds its fp64 mean).  The card's name, power limit and SM
clocks are read in the same run.

    python scripts/score_bench.py --out score.json
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import hyperreel_b200 as hb  # noqa: E402
from hyperreel_b200.state import seeded_state_dict  # noqa: E402

WORKLOADS = {
    # name: (builtin, overrides, W, H, views, note)
    "technicolor_2048x1088": ("technicolor_z_plane", dict(n_voxels=512000000), 2048, 1088, 50,
                              "Technicolor shape: 2048x1088 views, 32 samples/ray, K=12"),
    "neural3d_1352x1014_s64": ("neural_3d_z_plane", dict(n_voxels=262144000), 1352, 1014, 50,
                               "Neural-3D shape: 1352x1014 views, 64 samples/ray, K=12"),
}


def _gpu_facts():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        q = ""
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi name, power.limit, clocks.max.sm, clocks.sm": q}


def _cameras(W, H, F):
    """One held-out camera over F frames: the bench's forward-facing camera (frame_bench.py), turning slightly."""
    f = 0.9 * W
    cams = []
    for i in range(F):
        a = 0.02 * np.sin(2 * np.pi * i / max(F, 2))
        pose = [[-np.cos(a), 0, np.sin(a), 0.05 * np.sin(a)], [0, 1, 0, 0.0], [-np.sin(a), 0, -np.cos(a), -1.0]]
        cams.append(hb.Camera(pose=pose, K=[[f, 0, W / 2], [0, f, H / 2], [0, 0, 1]], width=W, height=H,
                              time=float(np.float32(i / max(F - 1, 1))), flipped=True))
    return cams


def to_float(u8):
    """u8 / 255 correctly rounded in fp32, as T.ToTensor() converts the reference's ground truth: a device-tensor divisor,
    since torch on CUDA divides by a Python scalar as a multiply by its reciprocal (one ulp off for some values)."""
    return u8.float() / torch.tensor(255.0, device=u8.device)


def _timed(fn):
    torch.cuda.synchronize()
    start = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    res = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), torch.cuda.max_memory_allocated() - start, res


def _stack(outs):
    return {k: torch.stack([o[k] for o in outs]) for k in outs[0]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--views", type=int, default=None, help="views per split (default: each workload's)")
    ap.add_argument("--only", default=None, help="run one workload")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("score_bench needs a CUDA device")
    facts = _gpu_facts()
    print(json.dumps(facts), flush=True)
    rows = []
    for name, (builtin, over, W, H, F, note) in WORKLOADS.items():
        if args.only and name != args.only:
            continue
        F = args.views or F
        cfg, ds = hb.configs.get(builtin, **over)
        sig = hb.lower(cfg, ds)
        system = hb.INRSystem(hb.to_cfg({"model": cfg, "training": {"ray_chunk": 1 << 22}}), dataset=ds)
        system.load_state_dict(seeded_state_dict(sig, seed=11, density_gain=30.0))
        system.cuda()
        cams = _cameras(W, H, F)
        # ground truth: the views' own 8-bit renders with noise on top, resident as uint8 [F, H, W, 3]
        video = system.render_video(cams)
        noise = torch.randint(-12, 13, video.shape, generator=torch.Generator(device="cuda").manual_seed(3), device="cuda",
                              dtype=torch.int16)
        images = (video.to(torch.int16) + noise).clamp(0, 255).to(torch.uint8).contiguous()
        del video, noise
        rays = [hb.generate_rays(c, c_in=sig.c_in) for c in cams]
        gts = [to_float(img) for img in images]
        resident_bytes = sum(r.numel() * 4 for r in rays) + sum(g.numel() * 4 for g in gts)

        def resident_loop():
            return [system.validation_image({"coords": r, "rgb": g, "W": W, "H": H}) for r, g in zip(rays, gts)]

        def per_view_loop():
            return [system.validation_image({"coords": hb.generate_rays(c, c_in=sig.c_in), "rgb": to_float(img),
                                             "W": W, "H": H}) for c, img in zip(cams, images)]

        runs = {"score_views": lambda: system.validation_views(cams, images), "resident_loop": resident_loop,
                "per_view_loop": per_view_loop}
        for fn in runs.values():  # warm-up: module loads, handle scratch, allocator pools
            fn()
        torch.cuda.synchronize()
        res = {k: [] for k in runs}
        outs = {}
        for _ in range(args.rounds):
            for k, fn in runs.items():
                ms, peak, out = _timed(fn)
                res[k].append((ms, peak))
                outs[k] = _stack(out)
        ref = outs["score_views"]
        same = {}
        for k in ("resident_loop", "per_view_loop"):
            rel = float(((outs[k]["val/loss"].double() - ref["val/loss"].double()).abs() / ref["val/loss"].double()).max())
            same[k] = {"psnr_bitwise": torch.equal(outs[k]["val/psnr"], ref["val/psnr"]),
                       "ssim_bitwise": torch.equal(outs[k]["val/ssim"], ref["val/ssim"]), "loss_max_rel": rel}
        row = {"workload": name, "note": note, "views": F, "W": W, "H": H, "samples": sig.n_samples, "c_in": sig.c_in,
               "metrics_vs_score_views": same,
               "mean_psnr": float(ref["val/psnr"].mean()), "mean_ssim": float(ref["val/ssim"].mean()), **facts}
        resident = {"score_views": images.numel(), "resident_loop": images.numel() + resident_bytes,
                    "per_view_loop": images.numel()}
        for k, v in res.items():
            ms = sorted(t for t, _ in v)[len(v) // 2]
            row[k] = {"ms_per_view": ms / F, "ms_split": ms, "ms_all": [t for t, _ in v],
                      "torch_peak_over_start_mb": max(p for _, p in v) / 2 ** 20, "resident_mb": resident[k] / 2 ** 20}
        rows.append(row)
        print(json.dumps(row), flush=True)
        for k, v in same.items():
            assert v["psnr_bitwise"] and v["ssim_bitwise"] and v["loss_max_rel"] <= 1e-6, (name, k, v)
        del system, rays, gts, images
        torch.cuda.empty_cache()
    facts_after = _gpu_facts()
    print(json.dumps({"after": facts_after}), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump({"gpu": facts, "gpu_after": facts_after, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
