"""Times the Immersive dataset's importance-subsampled training table (immersive.yaml: 1280x960, 50 frames, steps 8 / 4 /
0.25 / 0.125) for one video of synthetic content (a random first frame, then per frame a change of -3..3 levels per channel):

  (a) hr_build_importance_table for the video's 43 importance frames, CUDA events around whole builds (after a warm-up
      build), and per kernel from torch.profiler in a run of its own;
  (b) the sampling kernels at 16,384 and 65,536 rows with replacement: hr_sample_train_mask_rows over the importance table
      next to hr_sample_train_rows over the same video with neural_3d's regular subsets (the rule plan); kernel time from
      torch.profiler, device time per call from CUDA events over back-to-back calls, the two alternated round by round;
  (c) device bytes: the uint8 frames, the masks and their block index, against the reference's host table (48 B per row:
      8 coords, 3 rgb, 1 weight in fp32).

Usage: python scripts/importance_bench.py [--builds 10] [--calls 200] [--rounds 3] [--out result.json]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

W, H = 1280, 960
N_FRAMES = 50
IMMERSIVE = dict(load_full_step=8, subsample_keyframe_step=4, subsample_keyframe_frac=0.25, subsample_frac=0.125)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--builds", type=int, default=10)
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile

    import hyperreel_b200 as hb
    from scripts.train_bench import gpu_facts

    if not torch.cuda.is_available():
        raise SystemExit("importance_bench.py measures on the GPU; none found")
    dev = torch.device("cuda")
    # the 1280x960 training camera of tests/golden/make_golden_fisheye.py
    K = [[660.0, 0.0, 641.85], [0.0, 660.0, 481.1], [0.0, 0.0, 1.0]]
    pose = [[1.0, 0.0, 0.0, 0.2], [0.0, 1.0, 0.0, 0.0], [0.0, 0.0, 1.0, 0.1]]
    cams = [hb.Camera(pose=pose, K=K, width=W, height=H, time=f / (N_FRAMES - 1), cam_idx=11.0, distortion=(-0.12, 0.03))
            for f in range(N_FRAMES)]
    g = torch.Generator(device=dev).manual_seed(0)
    frames = [torch.randint(0, 256, (H, W, 3), generator=g, device=dev, dtype=torch.int16)]
    for _ in range(N_FRAMES - 1):
        frames.append((frames[-1] + torch.randint(-3, 4, (H, W, 3), generator=g, device=dev, dtype=torch.int16)).clamp(0, 255))
    images = torch.stack(frames).to(torch.uint8)
    del frames
    plan = hb.importance_subsample_plan(range(N_FRAMES), [0] * N_FRAMES, height=H, width=W, **IMMERSIVE)
    rule = hb.regular_subsample_plan(range(N_FRAMES), counters="neural_3d", videos=[0] * N_FRAMES, **IMMERSIVE)
    out = {"gpu": gpu_facts(), "frames": N_FRAMES, "image": f"{W}x{H}",
           "importance_frames": sum(e is not None for e in plan)}

    def events(fn, k):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(k):
            fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / k

    def kernel_ms(fn, k, names):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(k):
                fn()
            torch.cuda.synchronize()
        res = {}
        for e in prof.key_averages():
            for name in names:
                if name in e.key:
                    t = getattr(e, "device_time_total", 0.0) or getattr(e, "cuda_time_total", 0.0)
                    res[name] = res.get(name, 0.0) + t / 1e3 / k
        return res

    # (a) the build
    d = hb.DeviceRayBatches(cams, images, batch_size=16384, seed=0, importance=plan, replacement=True, num_iters=4000)
    n_rows = d.n_rows
    out["build_ms"] = [events(lambda: d._build_importance(plan), args.builds) for _ in range(args.rounds)]
    assert d.n_rows == n_rows and int(d._view_start[-1]) == n_rows  # the rebuilt table is the same
    out["build_kernels_ms"] = kernel_ms(lambda: d._build_importance(plan), args.builds,
                                        ["importance_hist_kernel", "importance_select_kernel", "importance_mask_kernel",
                                         "importance_scan_kernel", "importance_views_kernel"])
    out["build_ms_per_importance_frame"] = min(out["build_ms"]) / out["importance_frames"]
    out["table_rows"] = n_rows
    out["view_rows"] = d.view_rows.tolist()
    # (c) bytes
    mask_bytes = d._masks.numel() * 4 + d._block_start.numel() * 4
    out["device_bytes"] = {"images": images.numel(), "masks_and_index": mask_bytes,
                           "per_importance_pixel": mask_bytes / (out["importance_frames"] * H * W),
                           "reference_table": n_rows * 48}
    # (b) sampling, against the rule plan over the same video
    out["sampling"] = []
    for B in (16384, 65536):
        feeds = {"mask plan (hr_sample_train_mask_rows)":
                 hb.DeviceRayBatches(cams, images, B, seed=0, importance=plan, replacement=True, num_iters=4000),
                 "rule plan (hr_sample_train_rows)":
                 hb.DeviceRayBatches(cams, images, B, seed=0, subsample=rule, replacement=True, num_iters=4000)}
        row = {"rows": B}
        for name, f in feeds.items():
            f.n_rows
            for i in range(20):
                f.batch(i)
        ms = {name: [] for name in feeds}
        for r in range(args.rounds):
            for name, f in feeds.items():
                it = iter(range(args.calls * r, args.calls * (r + 1)))
                ms[name].append(events(lambda: f.batch(next(it)), args.calls))
        for name, f in feeds.items():
            row[name] = {"event_ms_per_call": ms[name], "table_rows": f.n_rows,
                         "kernel_ms": kernel_ms(lambda: f.batch(0), args.calls, ["train_rows_kernel"])}
        out["sampling"].append(row)
    print(json.dumps(out, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
