#!/usr/bin/env python
"""Video rendering throughput: F frames of one camera path rendered three ways, on synthetic trained-like parameters.

  video      hr_render_video_to8b (hb.render_video): one call, rays generated on the device in sub-batches that span frame
             boundaries, uint8 frames written into one device tensor [F, H, W, 3], no host synchronisation
  host_loop  one hr_render_frame_to8b_host call per frame (model.render_frame_to8b): each ends in a device-to-host copy of
             the frame and a host synchronisation
  dev_loop   one generate_rays + render_to8b per frame into the same device tensor (no synchronisation, one ray buffer per
             frame)

Per workload and F: frames/s, ms per frame (CUDA events around the whole loop on the current stream, then a synchronise;
host_loop runs on the handle's own streams, so it is timed with the host clock around calls that synchronise), and the
peak of torch's device allocations during the timed calls (host_loop's scratch is the handle's own cudaMalloc, not
counted there).  Each method is warmed up, then the three are run alternately `--reps` times; the median is reported.  The
frames of the three methods are compared (video == dev_loop for every frame, host_loop's last frame == video's).

    python scripts/video_bench.py --out video.json
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import hyperreel_b200 as hb  # noqa: E402
from hyperreel_b200.state import seeded_state_dict  # noqa: E402

WORKLOADS = {
    # name: (builtin, overrides, W, H, frame counts, note)
    "technicolor_2048x1088": ("technicolor_z_plane", dict(n_voxels=512000000), 2048, 1088, (1, 8, 50),
                              "Technicolor shape: 2048x1088 frames, 32 samples/ray, K=12"),
    "neural3d_1352x1014_s64": ("neural_3d_z_plane", dict(n_voxels=262144000), 1352, 1014, (1, 8),
                               "Neural-3D shape: 1352x1014 frames (the dataset's training size), 64 samples/ray, K=12"),
}


def _gpu_facts():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        q = ""
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q}


def _cameras(W, H, F):
    """A small orbit of the bench's camera (frame_bench.py): forward-facing, looking along +z from z = -1."""
    f = 0.9 * W
    cams = []
    for i in range(F):
        a = 0.02 * np.sin(2 * np.pi * i / max(F, 2))
        pose = [[-np.cos(a), 0, np.sin(a), 0.05 * np.sin(a)], [0, 1, 0, 0.0], [-np.sin(a), 0, -np.cos(a), -1.0]]
        cams.append(hb.Camera(pose=pose, K=[[f, 0, W / 2], [0, f, H / 2], [0, 0, 1]], width=W, height=H,
                              time=(i % 50) / 49.0, flipped=True))
    return cams


def _video(model, cams, times, out):
    hb.render_video(model, cams, times, out=out)


def _dev_loop(model, cams, times, out, c_in):
    for f, c in enumerate(cams):
        rays = hb.generate_rays(c, c_in=c_in)
        out[f].view(-1, 3).copy_(model.render_to8b(rays))


def _host_loop(model, cams, host):
    for f, c in enumerate(cams):
        model.render_frame_to8b(c, host[f])


def _timed_events(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), torch.cuda.max_memory_allocated()


def _timed_host(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t0), torch.cuda.max_memory_allocated()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--only", default=None, help="run one workload")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("video_bench needs a CUDA device")
    rows = []
    facts = _gpu_facts()
    print(json.dumps(facts), flush=True)
    for name, (builtin, over, W, H, counts, note) in WORKLOADS.items():
        if args.only and name != args.only:
            continue
        cfg, ds = hb.configs.get(builtin, **over)
        sig = hb.lower(cfg, ds)
        model = hb.LightfieldModel(cfg, dataset=ds, mlp_mode="bf16x3")
        render = hb.RenderLightfield(model, None, cfg.render)
        render.load_state_dict(seeded_state_dict(sig, seed=11, density_gain=30.0), strict=False)
        render.eval()
        for F in counts:
            cams = _cameras(W, H, F)
            times = [c.time for c in cams]
            video = torch.empty((F, H, W, 3), dtype=torch.uint8, device="cuda")
            dev = torch.empty_like(video)
            host = torch.empty((F, H, W, 3), dtype=torch.uint8).pin_memory()
            runs = {"video": lambda: _video(model, cams, times, video),
                    "dev_loop": lambda: _dev_loop(model, cams, times, dev, sig.c_in),
                    "host_loop": lambda: _host_loop(model, cams, host)}
            for fn in runs.values():  # warm-up: module loads, handle scratch, allocator pools
                fn()
            torch.cuda.synchronize()
            res = {k: [] for k in runs}
            for _ in range(args.reps):
                for k, fn in runs.items():
                    res[k].append(_timed_host(fn) if k == "host_loop" else _timed_events(fn))
            same_dev = all(torch.equal(video[f], dev[f]) for f in range(F))
            same_host = torch.equal(video[F - 1].cpu(), host[F - 1])
            row = {"workload": name, "note": note, "frames": F, "W": W, "H": H, "samples": sig.n_samples,
                   "frames_equal": {"video_vs_dev_loop": same_dev, "video_vs_host_loop_last": same_host},
                   "mean_pixel": float(video.float().mean()), **facts}
            for k, v in res.items():
                ms = sorted(t for t, _ in v)[len(v) // 2]
                row[k] = {"ms_total": ms, "ms_per_frame": ms / F, "frames_per_s": 1e3 * F / ms,
                          "torch_peak_mb": max(m for _, m in v) / 2 ** 20, "ms_all": [t for t, _ in v],
                          "clock": "host clock around synchronising calls" if k == "host_loop" else "CUDA events"}
            rows.append(row)
            print(json.dumps(row), flush=True)
            del video, dev, host
            torch.cuda.empty_cache()
        del model, render
        torch.cuda.empty_cache()
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
