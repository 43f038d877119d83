"""Times the training batches the shipped Technicolor config trains on (technicolor.yaml + technicolor_tensorf.yaml): the
train split's 15 views x 50 frames of 2048x1088 (synthetic content, 5.0 GB of uint8 on the device), its per-frame pixel
subsets (7 whole frames, 6 at 1/4, 37 at 1/8: 438,681,600 table rows) and sampling with replacement.

  (a) the kernels alone, at 16,384 and 65,536 rows: hr_sample_train_rows in both modes (permute, replace) next to the
      original hr_sample_train_batch over every pixel.  Kernel time from torch.profiler (a run of its own), device time per
      call from CUDA events over back-to-back calls;
  (b) training_step (the system of scripts/train_bench.py, train_net="tc") fed by replacement batches against one batch
      kept resident on the device, alternated round by round; CUDA events per step;
  (c) the reference's side: building the subsampled host table all_inputs (coords[mask], rgb[mask], weight: 48 B per row,
      technicolor.py:238-282) and drawing RandomSampler(replacement=True) batches from it (torch.randint over the table, then
      the row gather; the DataLoader's per-row __getitem__ and collate are not included, so this is a lower bound).  The
      whole table is 21 GB, so it is built for the first --ref-frames frames only and its build time is reported per row.

Usage: python scripts/train_sample_bench.py [--steps 20] [--rounds 3] [--calls 200] [--ref-frames 5] [--out result.json]
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

W, H = 2048, 1088
N_FRAMES = 50
TECHNICOLOR = dict(load_full_step=8, subsample_keyframe_step=4, subsample_keyframe_frac=0.25, subsample_frac=0.125)
# the every-pixel kernel: train_rows_kernel<WholePlan>, named train_batch_kernel in earlier builds (both match, so builds compare)
WHOLE_IMAGE_KERNEL = ("WholePlan", "train_batch_kernel")


def train_cameras(hb):
    """Technicolor's train split: a 4x4 rig without the held-out view (row 2, col 2: technicolor.yaml val_pairs), frame-major,
    NDC rays."""
    cams = []
    for f in range(N_FRAMES):
        for c in range(16):
            if c == 10:
                continue
            tx, ty = (c % 4 - 1.5) * 0.1, (c // 4 - 1.5) * 0.1
            pose = [[1.0, 0.0, 0.0, tx], [0.0, 1.0, 0.0, ty], [0.0, 0.0, 1.0, 0.0]]
            K = [[1500.0, 0.0, W / 2], [0.0, 1500.0, H / 2], [0.0, 0.0, 1.0]]
            cams.append(hb.Camera(pose=pose, K=K, width=W, height=H, time=f / (N_FRAMES - 1), cam_idx=float(c),
                                  use_ndc=True, ndc_near=1.0))
    return cams


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--ref-frames", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile

    import bench
    import hyperreel_b200 as hb
    from hyperreel_b200.train_data import subset_rows
    from scripts.train_bench import gpu_facts

    if not torch.cuda.is_available():
        raise SystemExit("train_sample_bench.py measures on the GPU; none found")
    dev = torch.device("cuda")
    cams = train_cameras(hb)
    n_views = len(cams)
    g = torch.Generator(device=dev).manual_seed(0)
    images = torch.randint(0, 256, (n_views, H, W, 3), generator=g, device=dev, dtype=torch.uint8)
    frames = [int(np.round(c.time * (N_FRAMES - 1))) for c in cams]
    plan = hb.regular_subsample_plan(frames, **TECHNICOLOR)
    out = {"gpu": gpu_facts(), "views": n_views, "image": f"{W}x{H}", "device_images_bytes": images.numel(), "batches": []}

    def events(fn, k):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(k):
            fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / k

    def kernel_ms(fn, names):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.calls):
                fn()
            torch.cuda.synchronize()
        kern = [e for e in prof.key_averages() if any(n in e.key for n in names)]
        return (sum(getattr(e, "device_time_total", 0.0) or getattr(e, "cuda_time_total", 0.0) for e in kern) / 1e3 /
                max(1, sum(e.count for e in kern)))

    # (a) the kernels alone
    feeds = {}
    for B in (16384, 65536):
        feeds[B] = {
            "hr_sample_train_batch (every pixel, permuted)": hb.DeviceRayBatches(cams, images, B, seed=0),
            "hr_sample_train_rows permute (subsets)": hb.DeviceRayBatches(cams, images, B, seed=0, subsample=plan),
            "hr_sample_train_rows replace (subsets)": hb.DeviceRayBatches(cams, images, B, seed=0, subsample=plan,
                                                                          replacement=True, num_iters=4000),
        }
        res = {"rows": B}
        for name, d in feeds[B].items():
            state = [0]

            def call(d=d, state=state):
                state[0] = (state[0] + 1) % (len(d) - 1)  # full batches only
                return d.batch(state[0])

            for _ in range(5):
                call()
            kname = WHOLE_IMAGE_KERNEL if "train_batch" in name else ("train_rows_kernel",)
            res[name] = {"device_ms_per_call": events(call, args.calls), "kernel_ms": kernel_ms(call, kname),
                         "table_rows": d.n_rows, "batches_per_epoch": len(d)}
        out["batches"].append(res)
        print(json.dumps(res), flush=True)
    out["table_rows"] = feeds[16384]["hr_sample_train_rows replace (subsets)"].n_rows

    # (b) training steps fed by replacement batches, against a resident batch
    _, cfg, ds, sig, sd = bench.build_workload(gain=600.0, app_gain=6.0)
    system = hb.INRSystem(hb.to_cfg({"model": cfg, "training": {"ray_chunk": 1 << 20, "iters_per_epoch": 4000},
                                     "dataset": ds}), train_net="tc")
    system.load_state_dict(sd)
    system.to(dev)
    system.configure_optimizers()
    out["train_step_ms"] = {}
    for B in (16384, 65536):
        d = feeds[B]["hr_sample_train_rows replace (subsets)"]
        state = [0]

        def replace_feed(d=d, state=state):
            state[0] = (state[0] + 1) % len(d)
            return d.batch(state[0])

        resident = d.batch(0)
        step_feeds = {"resident": lambda: resident, "replacement batches": replace_feed}
        for fn in step_feeds.values():
            for _ in range(3):
                system.training_step(fn())
        torch.cuda.synchronize()
        step_ms = {name: [] for name in step_feeds}
        for _ in range(args.rounds):
            for name, fn in step_feeds.items():
                step_ms[name].append(events(lambda: system.training_step(fn()), args.steps))
        out["train_step_ms"][B] = {name: {"mean": sum(v) / len(v), "runs": v} for name, v in step_ms.items()}
        print(json.dumps({"rows": B, "train_step_ms": out["train_step_ms"][B]}), flush=True)
    del feeds, system

    # (c) the reference's side on the first --ref-frames frames
    n_ref = 15 * args.ref_frames
    ys, xs = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    xy = (xs + ys).reshape(-1)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    parts = []
    for v in range(n_ref):
        s, o = plan[v]
        rows = torch.cat([hb.generate_rays(cams[v], c_in=8).cpu(), images[v].reshape(-1, 3).cpu().float().div(255)], -1)
        if s > 1:
            rows = rows[(xy + o) % s == 0]
        parts.append(rows)
    table = torch.cat(parts)
    table = torch.cat([table, torch.ones(table.shape[0], 1)], -1)
    build_s = time.perf_counter() - t0
    del parts
    full_rows = sum(subset_rows(s, o % s, H, W) for s, o in plan)
    ref = {"frames": args.ref_frames, "views": n_ref, "rows": table.shape[0], "bytes": table.numel() * 4,
           "build_s": build_s, "build_s_per_million_rows": build_s / table.shape[0] * 1e6,
           "full_split_rows": full_rows, "full_split_bytes": full_rows * 48,
           "full_split_build_s_extrapolated": build_s / table.shape[0] * full_rows}
    gen = torch.Generator().manual_seed(0)
    for B in (16384, 65536):
        t0 = time.perf_counter()
        for _ in range(args.calls):
            idx = torch.randint(high=table.shape[0], size=(B,), dtype=torch.int64, generator=gen)
            batch = table[idx]
        ref[f"draw_and_gather_ms_{B}"] = (time.perf_counter() - t0) / args.calls * 1e3
        pinned = batch.pin_memory()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(args.calls):
            pinned.to(dev, non_blocking=True)
        torch.cuda.synchronize()
        ref[f"pinned_copy_ms_{B}"] = (time.perf_counter() - t0) / args.calls * 1e3
    out["reference_host_table"] = ref
    print(json.dumps(ref), flush=True)
    out["gpu_after"] = gpu_facts()
    text = json.dumps(out, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
