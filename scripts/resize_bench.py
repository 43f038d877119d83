#!/usr/bin/env python
"""Resizing capture-resolution frames to the training resolution: hr_resize_frames on the device against OpenCV and Pillow
on one host thread, at the shipped datasets' sizes.

  neural3d   2704x2028 -> 1352x1014, cv2_linear (what neural_3d's get_rgb runs: OpenCV's INTER_AREA path at exactly 2x),
             and pil_lanczos at the same sizes for comparison
  llff       4032x3024 -> 504x378, pil_lanczos (llff's and spaces' get_rgb)

Device time per frame: CUDA events around `--reps` calls of `--frames` frames each on the current stream, after a warm-up
call, the median over `--rounds` such windows divided by the frames.  Bytes: the frames read plus the frames written (the
least any resize moves), and, for the Pillow methods, the uint8 intermediate written and read again; the rate is over the
device time and its share of the H100 SXM data sheet's 3.35 TB/s.  Host time: cv2.resize (cv2.setNumThreads(1)) and
PIL.Image.resize on one frame, median of `--host-reps` calls.  Every device result is checked against the host library's
on the first and last frame of the batch.  The card's name, power limit and SM clocks are read in the same run.

    python scripts/resize_bench.py --out resize.json
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import hyperreel_b200 as hb  # noqa: E402
from hyperreel_b200 import lib as L  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
WORKLOADS = {
    # name: (W0, H0, W, H, method, frames per call)
    "neural3d_cv2_linear": (2704, 2028, 1352, 1014, "cv2_linear", 20),
    "neural3d_pil_lanczos": (2704, 2028, 1352, 1014, "pil_lanczos", 20),
    "llff_pil_lanczos": (4032, 3024, 504, 378, "pil_lanczos", 8),
}


def _gpu_facts():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        q = ""
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi name, power.limit, clocks.max.sm, clocks.sm": q}


def _host(img, W, H, method, reps):
    import cv2
    from PIL import Image

    cv2.setNumThreads(1)
    if method.startswith("cv2"):
        flag = {"cv2_linear": cv2.INTER_LINEAR, "cv2_area": cv2.INTER_AREA}[method]
        fn = lambda: cv2.resize(img, (W, H), interpolation=flag)  # noqa: E731
    else:
        filt = {"pil_lanczos": Image.LANCZOS, "pil_bicubic": Image.BICUBIC, "pil_box": Image.BOX}[method]
        pil = Image.fromarray(img)
        fn = lambda: np.asarray(pil.resize((W, H), filt))  # noqa: E731
    out = fn()
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        times.append(time.perf_counter() - t0)
    return out, statistics.median(times)


def run(name, W0, H0, W, H, method, n, reps, rounds, host_reps):
    g = torch.Generator(device="cuda").manual_seed(0)
    frames = torch.randint(0, 256, (n, H0, W0, 3), generator=g, dtype=torch.uint8, device="cuda")
    out = torch.empty((n, H, W, 3), dtype=torch.uint8, device="cuda")
    hb.resize_frames(frames, (W, H), method, out=out)  # warm-up (module load, workspace)
    torch.cuda.synchronize()
    windows = []
    for _ in range(rounds):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            hb.resize_frames(frames, (W, H), method, out=out)
        b.record()
        b.synchronize()
        windows.append(a.elapsed_time(b) / reps / n)
    ms = statistics.median(windows)
    checked = []
    host_s = None
    for f in (0, n - 1):
        img = frames[f].cpu().numpy()
        ref, t = _host(img, W, H, method, host_reps if f == 0 else 1)
        host_s = t if f == 0 else host_s
        checked.append(bool(np.array_equal(out[f].cpu().numpy(), ref)))
    moved = n * (H0 * W0 * 3 + H * W * 3)
    ws = int(L.load_library().hr_resize_workspace_bytes(n, H0, W0, H, W, L.RESIZE_METHODS[method], L.PIXEL_RGB8))
    if method.startswith("pil"):
        moved += 2 * n * W * 3 * H0  # the intermediate (the rows the vertical pass reads: all of them here), written and read
    rate = moved / n / (ms * 1e-3)
    return {"workload": name, "capture": [W0, H0], "img_wh": [W, H], "method": method, "frames_per_call": n,
            "device_ms_per_frame": round(ms, 5), "device_ms_per_frame_windows": [round(w, 5) for w in windows],
            "bytes_per_frame": moved // n, "workspace_bytes": ws, "achieved_GB_per_s": round(rate / 1e9, 1),
            "share_of_hbm_3_35TBps": round(rate / HBM_BYTES_PER_S, 3),
            "host_ms_per_frame_one_thread": round(host_s * 1e3, 2), "host_over_device": round(host_s * 1e3 / ms, 1),
            "equal_to_host_library": all(checked)}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--host-reps", type=int, default=5)
    ap.add_argument("--only", default=None, help="comma-separated workload names")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("resize_bench.py measures the device: no CUDA device")
    names = args.only.split(",") if args.only else list(WORKLOADS)
    res = {"gpu": _gpu_facts(), "results": []}
    for name in names:
        r = run(name, *WORKLOADS[name], args.reps, args.rounds, args.host_reps)
        print(json.dumps(r), flush=True)
        res["results"].append(r)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    assert all(r["equal_to_host_library"] for r in res["results"]), "device result differs from the host library"


if __name__ == "__main__":
    main()
