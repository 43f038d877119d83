"""Times the two ways of feeding INRSystem.training_step on the Technicolor shape (the system of scripts/train_bench.py,
train_net="tc"), at 16,384 and 65,536 rays per step:

  (a) the reference's data path (datasets/base.py:111-143,202-227,254-289, nlf/__init__.py:651): a host table all_inputs
      [N, 12] fp32 (coords | rgb | weight, 48 B per ray) of every pixel of --views 2048x1088 views, permuted once (the per-epoch
      np.random.permutation + gather, timed), then per step a consecutive slice copied to the GPU with .cuda(), from pinned
      memory (non_blocking, what the DataLoader's pin_memory gives) and from pageable memory, and split by format_batch.
      The DataLoader's per-row __getitem__ and collate are not included, so (a) is a lower bound of the reference's cost;
  (b) DeviceRayBatches.batch(i) alone: the every-pixel kernel's time (torch.profiler, a run of its own), the device time per
      call (CUDA events over back-to-back calls) and the host time to issue a call;
  (c) training_step fed by each of them, and by one batch kept resident on the device (no data path at all), alternated
      round by round; CUDA events per step, mean over the steps of a round.

Also the device memory each feed holds and the peak during its steps.  No L2 flush: the data path runs between training steps,
as in a training loop.

Usage: python scripts/train_data_bench.py [--views 30] [--steps 20] [--rounds 3] [--calls 200] [--out result.json]
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

W, H = 2048, 1088
HBM_BYTES_S = 3.35e12  # NVIDIA H100 SXM data sheet (700 W card)
# the every-pixel kernel: train_rows_kernel<WholePlan>, named train_batch_kernel in earlier builds (both match, so builds compare)
WHOLE_IMAGE_KERNEL = ("WholePlan", "train_batch_kernel")


def rig_cameras(hb, n_views, near):
    """A forward-facing 4x4 rig like Technicolor's (cam_idx = view % 16, one time per rig pass), NDC rays with the near plane
    at `near` in front of the cameras."""
    cams = []
    for v in range(n_views):
        c = v % 16
        tx, ty = (c % 4 - 1.5) * 0.1, (c // 4 - 1.5) * 0.1
        pose = [[1.0, 0.0, 0.0, tx], [0.0, 1.0, 0.0, ty], [0.0, 0.0, 1.0, 0.0]]
        K = [[1500.0, 0.0, W / 2], [0.0, 1500.0, H / 2], [0.0, 0.0, 1.0]]
        cams.append(hb.Camera(pose=pose, K=K, width=W, height=H, time=(v // 16) / 49.0, cam_idx=float(c), use_ndc=True,
                              ndc_near=near))
    return cams


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=30)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile

    import bench
    import hyperreel_b200 as hb
    from scripts.train_bench import gpu_facts

    if not torch.cuda.is_available():
        raise SystemExit("train_data_bench.py measures on the GPU; none found")
    dev = torch.device("cuda")
    _, cfg, ds, sig, sd = bench.build_workload(gain=600.0, app_gain=6.0)
    system = hb.INRSystem(hb.to_cfg({"model": cfg, "training": {"ray_chunk": 1 << 20, "iters_per_epoch": 4000}, "dataset": ds}),
                          train_net="tc")
    system.load_state_dict(sd)
    system.to(dev)
    system.configure_optimizers()

    n_views = args.views
    n = n_views * H * W
    cams = rig_cameras(hb, n_views, 1.0)
    g = torch.Generator(device=dev).manual_seed(0)
    images = torch.randint(0, 256, (n_views, H, W, 3), generator=g, device=dev, dtype=torch.uint8)
    torch.cuda.synchronize()
    mem0 = torch.cuda.memory_allocated()
    batches = hb.DeviceRayBatches(cams, images, batch_size=16384, seed=0)
    device_feed_bytes = torch.cuda.memory_allocated() - mem0  # the cameras (images are shared with the caller here)
    device_feed_bytes += images.numel()

    # (a) the reference's host table, built from the same rays and pixels, permuted once
    c_in = 8
    table = torch.empty((n, c_in + 4), dtype=torch.float32)
    for v, cam in enumerate(cams):
        rows = torch.cat([hb.generate_rays(cam, c_in=c_in), images[v].reshape(-1, 3).float().cpu().div(255).to(dev),
                          torch.ones(H * W, 1, device=dev)], -1)
        table[v * H * W:(v + 1) * H * W].copy_(rows.cpu())
    t0 = time.perf_counter()
    perm = torch.from_numpy(np.random.permutation(n))
    t1 = time.perf_counter()
    shuffled = table[perm]
    t2 = time.perf_counter()
    del table, perm
    pinned = shuffled.pin_memory()
    out = {"gpu": gpu_facts(), "workload": "technicolor_z_plane, grid 1007x1007x503, K=12, INRSystem.training_step, train_net='tc'",
           "views": n_views, "image": f"{W}x{H}", "pixels": n,
           "host_all_inputs_bytes": shuffled.numel() * 4, "device_images_bytes": images.numel(),
           "device_feed_bytes": device_feed_bytes,
           "reference_epoch_shuffle_s": {"np.random.permutation": t1 - t0, "all_inputs[perm]": t2 - t1},
           "batches": []}

    def events(fn, k):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(k):
            fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / k

    def format_batch(inputs):  # datasets/base.py:278-284, on the device as in training_step (nlf/__init__.py:651)
        return {"coords": inputs[..., :c_in], "rgb": inputs[..., c_in:c_in + 3], "weight": inputs[..., -1:]}

    for B in (16384, 65536):
        batches = hb.DeviceRayBatches(cams, images, batch_size=B, seed=0)
        nb = len(batches)
        state = {"device": 0, "pinned": 0, "pageable": 0}

        def feed(name):
            i = state[name] = (state[name] + 1) % (nb - 1)  # full batches only
            if name == "device":
                return batches.batch(i)
            if name == "pinned":
                return format_batch(pinned[i * B:(i + 1) * B].to(dev, non_blocking=True))
            return format_batch(shuffled[i * B:(i + 1) * B].to(dev))

        resident = batches.batch(nb // 2)
        feeds = {"resident": lambda: resident, "device": lambda: feed("device"), "pinned": lambda: feed("pinned"),
                 "pageable": lambda: feed("pageable")}
        # the data paths alone
        for name in ("device", "pinned", "pageable"):
            for _ in range(5):
                feeds[name]()
        alone = {name: events(feeds[name], args.calls) for name in ("device", "pinned", "pageable")}
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(args.calls):
            feed("device")
        host_us = (time.perf_counter() - t0) / args.calls * 1e6
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.calls):
                feed("device")
            torch.cuda.synchronize()
        kern = [e for e in prof.key_averages() if any(n in e.key for n in WHOLE_IMAGE_KERNEL)]
        kernel_ms = (sum(getattr(e, "device_time_total", 0.0) or getattr(e, "cuda_time_total", 0.0) for e in kern) / 1e3 /
                     max(1, sum(e.count for e in kern)))
        write_bytes, read_bytes = B * 48, B * 32  # 48 B row written; each 3 B gather touches one 32 B sector (more if it straddles)
        # (c) training steps, the feeds alternated round by round
        for name in feeds:
            for _ in range(3):
                system.training_step(feeds[name]())
        torch.cuda.synchronize()
        step_ms = {name: [] for name in feeds}
        peak = {}
        for _ in range(args.rounds):
            for name, fn in feeds.items():
                torch.cuda.reset_peak_memory_stats()
                step_ms[name].append(events(lambda: system.training_step(fn()), args.steps))
                peak[name] = max(peak.get(name, 0), torch.cuda.max_memory_allocated())
        mean = lambda v: sum(v) / len(v)
        out["batches"].append({
            "rays": B,
            "data_path_alone_ms": {"DeviceRayBatches.batch": alone["device"], ".cuda() from pinned": alone["pinned"],
                                   ".cuda() from pageable": alone["pageable"]},
            "DeviceRayBatches": {"kernel_ms": kernel_ms, "host_us_per_call": host_us,
                                 "kernel_bytes": write_bytes + read_bytes,
                                 "achieved_GB_s": (write_bytes + read_bytes) / (kernel_ms * 1e-3) / 1e9 if kernel_ms > 0 else None,
                                 "hbm_bound_ms": (write_bytes + read_bytes) / HBM_BYTES_S * 1e3},
            "train_step_ms": {name: {"mean": mean(v), "runs": v} for name, v in step_ms.items()},
            "step_peak_device_bytes": peak,
        })
        print(json.dumps(out["batches"][-1]), flush=True)
    out["gpu_after"] = gpu_facts()
    text = json.dumps(out, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
