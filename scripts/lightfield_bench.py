"""Times the ray kernels with two-plane light-field views against pinhole cameras, and the pinhole path against another build.

  (a) generate_rays_kernel on a 1024x1024 view (the large Stanford configs' tarot_small size), pinhole against two-plane;
  (b) train_rows_kernel over every pixel, permuted (hr_sample_train_batch), and with replacement draws
      (hr_sample_train_rows), at 16,384 and 65,536 rows over 17 views of 1024x1024, all pinhole against all two-plane;
  (c) render_video of the 120-frame render path of a Stanford spiral (lightfield_cameras(split="render")) at 512x512 with
      the shipped stanford_z_plane model, against 120 pinhole frames of the same size;
  (d) with --other-lib PATH (a libhyperreel_b200.so of an earlier ABI, whose hr_camera is a prefix of this one): the pinhole
      workloads of (a) and (b) through both libraries, alternated round by round in one process.

Kernel times are torch.profiler means over --calls launches, one profiler session per (library, workload) and round; video
times are CUDA events around whole render_video calls.  The card's name, power limit and clocks are read in the same run.

Usage: python scripts/lightfield_bench.py [--calls 200] [--rounds 3] [--other-lib PATH] [--out result.json]
"""
import argparse
import ctypes as C
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

W, H, N_VIEWS = 1024, 1024, 17
VW, VH = 512, 512
# the every-pixel kernel: train_rows_kernel<WholePlan>, named train_batch_kernel in earlier builds (both match, so builds compare)
WHOLE_IMAGE_KERNEL = ("WholePlan", "train_batch_kernel")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--video-calls", type=int, default=5)
    ap.add_argument("--other-lib", default=None)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile

    import hyperreel_b200 as hb
    from hyperreel_b200 import lib as L
    from scripts.train_bench import gpu_facts

    if not torch.cuda.is_available():
        raise SystemExit("lightfield_bench.py measures on the GPU; none found")
    dev = torch.device("cuda")
    stream = torch.cuda.current_stream().cuda_stream

    def open_lib(path):
        lib = C.CDLL(path)
        for name in ("hr_generate_rays", "hr_sample_train_batch", "hr_sample_train_rows", "hr_abi_version"):
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = L.EXPORTS[name]
            if name == "hr_generate_rays":
                fn.argtypes = [C.c_void_p] + L.EXPORTS[name][1][1:]
        if lib.hr_abi_version() < 24:  # the sampling entry points take a pixel format from ABI 24
            for fn in (lib.hr_sample_train_batch, lib.hr_sample_train_rows):
                fn.argtypes = fn.argtypes[:3] + fn.argtypes[4:]
        return lib

    def pinhole(v):
        pose = [[1.0, 0.0, 0.0, 0.05 * v], [0.0, 1.0, 0.0, 0.0], [0.0, 0.0, 1.0, 0.0]]
        K = [[900.0, 0.0, 511.5], [0.0, 900.0, 511.5], [0.0, 0.0, 1.0]]
        return hb.Camera(pose=pose, K=K, width=W, height=H)

    def cameras(two_plane, n_fields=None):
        cams = [hb.TwoPlaneCamera(W, H, (v % 5) / 2.0 - 1.0, 1.0 - (v // 5) / 2.0, st_scale=0.125) if two_plane
                else pinhole(v) for v in range(N_VIEWS)]
        recs = [c.to_c() for c in cams]
        record = L.hr_camera
        if n_fields is not None:  # an earlier ABI's record: the first n_fields members
            class Record(C.Structure):
                _fields_ = L.hr_camera._fields_[:n_fields]
            record = Record
            recs = [record(*[getattr(r, f[0]) for f in record._fields_]) for r in recs]
        arr = (record * N_VIEWS)(*recs)
        return arr, torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).to(dev)

    g = torch.Generator(device=dev).manual_seed(0)
    images = torch.randint(0, 256, (N_VIEWS, H, W, 3), generator=g, device=dev, dtype=torch.uint8)
    n_pix = N_VIEWS * H * W
    view_start = torch.arange(N_VIEWS + 1, dtype=torch.int64, device=dev) * (H * W)
    view_rule = torch.tensor([[1, 0]] * N_VIEWS, dtype=torch.int32, device=dev)
    out = {"gpu": gpu_facts(), "frame": f"{W}x{H}", "views": N_VIEWS, "calls": args.calls}

    def workloads(lib, host_cam, dev_cams):
        """name -> (kernel names, call)"""
        frame = torch.empty((W * H, 6), dtype=torch.float32, device=dev)
        fmt = (L.PIXEL_RGB8,) if lib.hr_abi_version() >= 24 else ()
        w = {f"generate_rays {W}x{H}": (("generate_rays_kernel",), lambda: lib.hr_generate_rays(
            C.byref(host_cam), 6, 0, W * H, frame.data_ptr(), stream))}
        for B in (16384, 65536):
            coords = torch.empty((B, 6), dtype=torch.float32, device=dev)
            rgb = torch.empty((B, 3), dtype=torch.float32, device=dev)
            weight = torch.empty((B, 1), dtype=torch.float32, device=dev)
            state = [0]

            def batch(B=B, coords=coords, rgb=rgb, weight=weight, state=state):
                state[0] = (state[0] + 1) % (n_pix // B)
                return lib.hr_sample_train_batch(dev_cams.data_ptr(), N_VIEWS, images.data_ptr(), *fmt, H, W, 6, 0, 0,
                                                 state[0], B, None, coords.data_ptr(), rgb.data_ptr(), weight.data_ptr(),
                                                 None, None, stream)

            def rows(B=B, coords=coords, rgb=rgb, weight=weight, state=state):
                state[0] += 1
                return lib.hr_sample_train_rows(dev_cams.data_ptr(), N_VIEWS, images.data_ptr(), *fmt, H, W, 6,
                                                view_start.data_ptr(), view_rule.data_ptr(), n_pix, L.SAMPLE_REPLACE, 0, 0,
                                                state[0], B, None, coords.data_ptr(), rgb.data_ptr(), weight.data_ptr(),
                                                None, None, None, stream)

            w[f"train_batch {B}"] = (WHOLE_IMAGE_KERNEL, batch)
            w[f"train_rows replace {B}"] = (("train_rows_kernel",), rows)
        return w

    def kernel_us(names, fn):
        for _ in range(5):
            assert fn() == 0
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.calls):
                fn()
            torch.cuda.synchronize()
        kern = [e for e in prof.key_averages() if any(n in e.key for n in names)]
        total = sum(getattr(e, "device_time_total", 0.0) or getattr(e, "cuda_time_total", 0.0) for e in kern)
        count = sum(e.count for e in kern)
        assert count >= args.calls - 2, (names, count)  # a session may drop an event at its start
        return total / count

    this = open_lib(L.LIB_PATH)
    pin_host, pin_dev = cameras(False)
    lf_host, lf_dev = cameras(True)
    sets = {"pinhole": workloads(this, pin_host[0], pin_dev), "two_plane": workloads(this, lf_host[0], lf_dev)}
    # (a), (b): pinhole against two-plane in this build, alternated
    res = {model: {k: [] for k in w} for model, w in sets.items()}
    for _ in range(args.rounds):
        for k in sets["pinhole"]:
            for model in ("pinhole", "two_plane"):
                res[model][k].append(kernel_us(*sets[model][k]))
    out["this_build_us"] = {m: {k: {"mean": sum(v) / len(v), "runs": v} for k, v in r.items()} for m, r in res.items()}
    print(json.dumps(out["this_build_us"]), flush=True)

    # (c): a 120-frame Stanford render path against 120 pinhole frames
    from tests.test_shipped_yaml_golden import SHIPPED, load_fixture

    by_name = {os.path.basename(p)[:-4]: p for p in SHIPPED}
    plain, cfg, ds, sig, sd, _, _ = load_fixture(by_name["stanford_z_plane"])
    model = hb.LightfieldModel(cfg, dataset=ds)
    render = hb.RenderLightfield(model, None, cfg.render)
    render.load_state_dict(sd, strict=False)
    render.eval()
    dcfg = {"name": "stanford", "img_wh": [VW, VH], "val_num": 8,
            "render_params": {"spiral": True, "spiral_rad": 0.5, "supersample": 4},
            "lightfield": {"rows": 17, "cols": 17, "step": 4, "supersample": 2, "disp_row": 8, "st_scale": 0.125}}
    videos = {"two_plane": hb.lightfield_cameras(dcfg, VW, VH, "render"),
              "pinhole": [hb.Camera(pose=[[1.0, 0.0, 0.0, 0.002 * f], [0.0, -1.0, 0.0, 0.0], [0.0, 0.0, -1.0, -1.0]],
                                    K=[[450.0, 0.0, 255.5], [0.0, 450.0, 255.5], [0.0, 0.0, 1.0]], width=VW, height=VH)
                          for f in range(120)]}
    buf = torch.empty((120, VH, VW, 3), dtype=torch.uint8, device=dev)
    vres = {k: [] for k in videos}
    for k, cams in videos.items():  # warm-up
        hb.render_video(model, cams, out=buf)
    torch.cuda.synchronize()
    for _ in range(args.rounds):
        for k, cams in videos.items():
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(args.video_calls):
                hb.render_video(model, cams, out=buf)
            t1.record()
            t1.synchronize()
            vres[k].append(t0.elapsed_time(t1) / args.video_calls)
    out["video_120x512x512_ms"] = {k: {"mean": sum(v) / len(v), "runs": v} for k, v in vres.items()}
    print(json.dumps(out["video_120x512x512_ms"]), flush=True)

    # (d): the pinhole workloads through another build, alternated with this one
    if args.other_lib:
        other = open_lib(args.other_lib)
        abi = other.hr_abi_version()
        n_fields = len(L.hr_camera._fields_) - 8 if abi in (17, 18, 19) else None
        assert n_fields is not None, f"--other-lib: ABI {abi} has no known hr_camera prefix"
        old_host, old_dev = cameras(False, n_fields)
        builds = {"other": workloads(other, old_host[0], old_dev), "this": sets["pinhole"]}
        out["other_lib_abi"] = abi
        res = {b: {k: [] for k in w} for b, w in builds.items()}
        for _ in range(args.rounds):
            for k in builds["this"]:
                for b in ("other", "this"):
                    res[b][k].append(kernel_us(*builds[b][k]))
        out["pinhole_builds_us"] = {b: {k: {"mean": sum(v) / len(v), "runs": v} for k, v in r.items()}
                                    for b, r in res.items()}
        print(json.dumps(out["pinhole_builds_us"]), flush=True)
    out["gpu_after"] = gpu_facts()
    text = json.dumps(out, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
