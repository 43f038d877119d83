#!/usr/bin/env python
"""Embedding maps of a video: the per-frame cost of the visualiser's maps, three ways, on synthetic trained-like parameters
at the Technicolor shape (2048x1088 frames, 32 samples per ray) with the shipped ``default_time`` embedding config
(distances normalised, point_offset and spatial_flow bounded).

  visuals    hr_render_visuals (hb.render_embeddings): the RGB frames and the three maps from one render pass per frame,
             one call, no host synchronisation
  video      hr_render_video_to8b (hb.render_video) alone: the RGB frames without maps
  two_pass   the reference's order on this path: render_video, then per frame a forward(rays, {'fields': ...}) of the
             frame's rays and the maps in torch, visualize_warp + to8b of the fp32 fields (fp32 tensor ops, as the
             reference runs them, the to8b on the device)

Each variant is warmed up, then the three are run alternately `--reps` times (CUDA events around each call, then a
synchronise); the median per frame is reported with the card's name and power limit, read in the same run.  The maps of
`visuals` and `two_pass` are compared byte for byte, and the RGB of `visuals` and `video`.

    python scripts/visual_bench.py --out visuals.json
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

DEFAULT_TIME = {"type": "embedding", "run_on_test": False, "save_data": False, "no_over_fields": ["raw_distance", "raw_flow"],
                "fields": {"distances": {"use_abs": False, "normalize": True},
                           "point_offset": {"use_abs": True, "bounds": [0.0, 0.25]},
                           "spatial_flow": {"use_abs": True, "bounds": [0.0, 1.0]}}}


def _gpu_facts():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        q = ""
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q}


def _cameras(W, H, F):
    f = 0.9 * W
    cams = []
    for i in range(F):
        a = 0.02 * np.sin(2 * np.pi * i / max(F, 2))
        pose = [[-np.cos(a), 0, np.sin(a), 0.05 * np.sin(a)], [0, 1, 0, 0.0], [-np.sin(a), 0, -np.cos(a), -1.0]]
        cams.append(hb.Camera(pose=pose, K=[[f, 0, W / 2], [0, f, H / 2], [0, 0, 1]], width=W, height=H,
                              time=(i % 50) / 49.0, flipped=True))
    return cams


def _torch_maps(x, r):
    """visualize_warp (sort: False) + to8b of one frame's fp32 field [P, dim], as fp32 torch ops."""
    if r.use_abs:
        x = torch.abs(x)
    if r.bounds is not None:
        lo, hi = torch.tensor(r.bounds[0], device=x.device), torch.tensor(r.bounds[1], device=x.device)
        x = (x - lo) / (hi - lo)
    if r.normalize:
        mn, mx = torch.min(x, dim=0)[0].view(1, -1), torch.max(x, dim=0)[0].view(1, -1)
        x = (x - mn) / (mx - mn)
    x = (255 * x.clamp(0, 1)).nan_to_num(0.0)
    return x.to(torch.uint8)


def _two_pass(render, cams, reqs, c_in, maps):
    hb.render_video(render, cams)
    keys = [r.key for r in reqs]
    for f, c in enumerate(cams):
        out = render.model(hb.generate_rays(c, c_in=c_in), {"fields": keys})
        for r in reqs:
            maps[r.key][f].view(-1, r.channels).copy_(_torch_maps(out[r.key], r))


def _timed(fn):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("visual_bench needs a CUDA device")
    facts = _gpu_facts()
    print(json.dumps(facts), flush=True)
    W, H, F = 2048, 1088, args.frames
    cfg, ds = hb.configs.get("technicolor_z_plane", n_voxels=512000000)
    sig = hb.lower(cfg, ds)
    model = hb.LightfieldModel(cfg, dataset=ds, mlp_mode="bf16x3")
    render = hb.RenderLightfield(model, None, cfg.render)
    render.load_state_dict(seeded_state_dict(sig, seed=11, density_gain=30.0), strict=False)
    render.eval()
    cams = _cameras(W, H, F)
    vcfg = hb.to_cfg(DEFAULT_TIME)
    reqs = hb.embedding_requests(vcfg)
    maps2 = {r.key: torch.empty((F, H, W, r.channels), dtype=torch.uint8, device="cuda") for r in reqs}
    runs = {"visuals": lambda: hb.render_embeddings(render, cams, vcfg),
            "video": lambda: hb.render_video(render, cams),
            "two_pass": lambda: _two_pass(render, cams, reqs, sig.c_in, maps2)}
    outs = {k: fn() for k, fn in runs.items()}  # warm-up
    times = {k: [] for k in runs}
    for _ in range(args.reps):
        for k, fn in runs.items():
            ms, outs[k] = _timed(fn)
            times[k].append(ms)
    vis = outs["visuals"]
    row = {"workload": "technicolor_2048x1088_default_time", "frames": F, "W": W, "H": H, "samples": sig.n_samples, **facts,
           "rgb_equal_video": bool(torch.equal(vis["rgb"], outs["video"])),
           "maps_equal_two_pass": {r.key: bool(torch.equal(vis[f"embedding_{r.key}"].reshape(F, H, W, -1), maps2[r.key]))
                                   for r in reqs}}
    for k, v in times.items():
        ms = sorted(v)[len(v) // 2]
        row[k] = {"ms_per_frame": ms / F, "ms_all": v, "clock": "CUDA events"}
    row["maps_cost_ms_per_frame"] = row["visuals"]["ms_per_frame"] - row["video"]["ms_per_frame"]
    print(json.dumps(row), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(row, f, indent=1)


if __name__ == "__main__":
    main()
