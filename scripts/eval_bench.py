"""Times held-out view scoring on the Technicolor shape (bench.py's workload) at 2048 x 1088 views.

  * hr_image_metrics alone (MSE + SSIM of n frames, CUDA events over many calls) for n = 1 and n = 8;
  * INRSystem.validation_image per view, end to end: rays of a camera generated on the device, render, loss, PSNR and SSIM,
    all on the device; views enqueued back to back and timed to one synchronise, the way a test loop runs them;
  * the CPU scoring it replaces: the fp32 SSIM of the same frame with SciPy's gaussian_filter, what scikit-image calls
    (tests/metrics_oracle.py, fp64=False as scikit-image >= 0.19 runs it), and the frame's device-to-host copy;
  * bytes and fp64 FLOPs per frame from the shape, and the kernel's share of the larger of the two data-sheet bounds.

Fails without a GPU.  Usage: python scripts/eval_bench.py [--calls 50] [--views 10] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

W, H = 2048, 1088
# NVIDIA H100 SXM data sheet (700 W card): HBM3 bandwidth and dense FP64 (non-tensor) rate
HBM_BYTES_S, FP64_FLOPS = 3.35e12, 34e12


def gpu_facts():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return dict(zip(q.split(","), [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")])) if r.returncode == 0 else {}


def frame_cost(h, w):
    """(bytes, fp64 FLOPs) one frame's scoring needs: both fp32 images read once; per channel, the three moment products of
    every pixel, the vertical 11-tap pass of 5 moments over rows [5, h-5) of every column, the horizontal pass over the
    interior (2 FLOPs per tap) and 25 FLOPs of the SSIM map per interior pixel."""
    interior = (h - 10) * (w - 10)
    per_channel = 3 * h * w + 5 * 11 * 2 * ((h - 10) * w + interior) + 25 * interior
    return 2 * h * w * 3 * 4, 3 * per_channel


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--views", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import numpy as np
    import torch

    import bench
    import hyperreel_b200 as hb
    from tests import metrics_oracle as O

    if not torch.cuda.is_available():
        raise SystemExit("eval_bench.py measures on the GPU; none found")
    dev = torch.device("cuda")
    out = {"gpu": gpu_facts(), "workload": f"technicolor_z_plane, grid 1007x1007x503, K=12, {W}x{H} views"}

    def timed(fn, n):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(n):
            fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / n

    # the model and a held-out view: rays of a camera looking along the forward-facing rig's +z (scripts/frame_bench.py)
    _, cfg, ds, sig, sd = bench.build_workload()
    system = hb.INRSystem(hb.to_cfg({"model": cfg, "training": {"ray_chunk": 1 << 22}, "dataset": ds}))
    system.load_state_dict(sd)
    system.to(dev)
    f = 0.9 * W
    cam = hb.Camera(pose=[[-1, 0, 0, 0.0], [0, 1, 0, 0.0], [0, 0, -1, -1.0]], K=[[f, 0, W / 2], [0, f, H / 2], [0, 0, 1]],
                    width=W, height=H, time=0.5, flipped=True)
    coords = hb.generate_rays(cam, c_in=sig.c_in, device=dev)
    with torch.no_grad():
        pred = system(coords)["rgb"].view(1, H, W, 3)
    gen = torch.Generator(device=dev).manual_seed(5)
    gt = (pred + 0.03 * torch.randn(pred.shape, generator=gen, device=dev)).clamp(0, 1).contiguous()

    # 1. the kernel alone
    nbytes, flops = frame_cost(H, W)
    kernel = {}
    for n in (1, 8):
        p8, g8 = pred.expand(n, H, W, 3).contiguous(), gt.expand(n, H, W, 3).contiguous()
        for _ in range(3):
            hb.metrics.image_metrics(p8, g8)
        ms = timed(lambda: hb.metrics.image_metrics(p8, g8), args.calls)
        t = ms * 1e-3 / n
        kernel[f"n{n}"] = {"ms_per_call": ms, "us_per_frame": t * 1e6, "fp64_tflops": flops / t / 1e12,
                           "gb_s": nbytes / t / 1e9}
    bound_flop, bound_bytes = flops / FP64_FLOPS, nbytes / HBM_BYTES_S
    t1 = kernel["n8"]["us_per_frame"] * 1e-6
    out["frame_cost"] = {"bytes": nbytes, "fp64_flops": flops, "fp64_bound_us": bound_flop * 1e6,
                         "hbm_bound_us": bound_bytes * 1e6,
                         "larger_bound": "fp64 (34 TFLOP/s)" if bound_flop >= bound_bytes else "HBM (3.35 TB/s)",
                         "kernel_share_of_larger_bound_n8": max(bound_flop, bound_bytes) / t1}
    out["hr_image_metrics"] = kernel

    # 2. validation_image end to end (render + metrics), views enqueued back to back
    batch = {"coords": coords, "rgb": gt.view(-1, 3), "W": W, "H": H}
    for _ in range(3):
        system.validation_image(batch)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    outs = [system.validation_image(batch) for _ in range(args.views)]
    mean = system.validation_epoch_end(outs)
    val_ms = (time.perf_counter() - t0) * 1e3 / args.views
    with torch.no_grad():
        render_ms = timed(lambda: system(coords), args.views)
    out["validation_image"] = {"ms_per_view": val_ms, "render_alone_ms": render_ms, "metrics": mean}

    # 3. the host scoring it replaces, on the same frame
    t0 = time.perf_counter()
    img, img_gt = pred[0].cpu().numpy(), gt[0].cpu().numpy()
    d2h_ms = (time.perf_counter() - t0) * 1e3
    cpu_ms = []
    for _ in range(3):
        t0 = time.perf_counter()
        s32 = O.ssim(img, img_gt, fp64=False)
        cpu_ms.append((time.perf_counter() - t0) * 1e3)
    out["cpu_scoring"] = {"ssim_fp32_ms": sorted(cpu_ms)[1], "d2h_copy_ms": d2h_ms, "host_cpus": bench.usable_cpus(),
                          "note": "scipy.ndimage.gaussian_filter is single-threaded",
                          "ssim_fp32": s32, "ssim_device_fp64": float(hb.metrics.ssim(pred[0], gt[0]))}
    out["gpu_after"] = gpu_facts()
    text = json.dumps(out)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
