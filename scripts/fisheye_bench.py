"""Times the camera-model kernels with pinhole and fisheye cameras, and the pinhole path against another build of the library.

  (a) generate_rays_kernel on a 1280x960 frame (the Immersive dataset's training size), pinhole against fisheye;
  (b) train_rows_kernel over every pixel, permuted (hr_sample_train_batch), and with replacement draws
      (hr_sample_train_rows), at 16,384 and 65,536 rows over 20 views of 1280x960, all pinhole against all fisheye;
  (c) with --other-lib PATH (a libhyperreel_b200.so of an earlier ABI, whose hr_camera is the pinhole prefix of this one): the
      pinhole workloads of (a) and (b) through both libraries, alternated round by round in one process.

Kernel times are torch.profiler means over --calls launches, one profiler session per (library, workload) and round.  The
card's name, power limit and clocks are read in the same run.

Usage: python scripts/fisheye_bench.py [--calls 200] [--rounds 3] [--other-lib PATH] [--out result.json]
"""
import argparse
import ctypes as C
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

W, H, N_VIEWS = 1280, 960, 20
PINHOLE_FIELDS = 14  # fields of hr_camera before the fisheye members (ABI <= 16)
# the every-pixel kernel: train_rows_kernel<WholePlan>, named train_batch_kernel in earlier builds (both match, so builds compare)
WHOLE_IMAGE_KERNEL = ("WholePlan", "train_batch_kernel")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--other-lib", default=None)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile

    import hyperreel_b200 as hb
    from hyperreel_b200 import lib as L
    from scripts.train_bench import gpu_facts

    if not torch.cuda.is_available():
        raise SystemExit("fisheye_bench.py measures on the GPU; none found")
    dev = torch.device("cuda")
    stream = torch.cuda.current_stream().cuda_stream

    class PinholeCamera(C.Structure):  # hr_camera up to ABI 16
        _fields_ = L.hr_camera._fields_[:PINHOLE_FIELDS]

    assert [f[0] for f in L.hr_camera._fields_[PINHOLE_FIELDS:]] == ["fisheye", "k1", "k2"]

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

    def cameras(fisheye, record=L.hr_camera):
        cams = []
        for v in range(N_VIEWS):
            pose = [[1.0, 0.0, 0.0, 0.05 * v], [0.0, 1.0, 0.0, 0.0], [0.0, 0.0, 1.0, 0.0]]
            K = [[1320.0 * 0.5, 0.0, 1283.7 * 0.5], [0.0, 1320.0 * 0.5, 962.2 * 0.5], [0.0, 0.0, 1.0]]
            cams.append(hb.Camera(pose=pose, K=K, width=W, height=H, time=v / (N_VIEWS - 1), cam_idx=float(v),
                                  distortion=(-0.12, 0.03) if fisheye else None))
        recs = [c.to_c() for c in cams]
        if record is not L.hr_camera:
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
        frame = torch.empty((W * H, 8), dtype=torch.float32, device=dev)
        fmt = (L.PIXEL_RGB8,) if lib.hr_abi_version() >= 24 else ()
        w = {"generate_rays 1280x960": (("generate_rays_kernel",), lambda: lib.hr_generate_rays(
            C.byref(host_cam), 8, 0, W * H, frame.data_ptr(), stream))}
        for B in (16384, 65536):
            coords = torch.empty((B, 8), dtype=torch.float32, device=dev)
            rgb = torch.empty((B, 3), dtype=torch.float32, device=dev)
            weight = torch.empty((B, 1), dtype=torch.float32, device=dev)
            state = [0]

            def batch(B=B, coords=coords, rgb=rgb, weight=weight, state=state):
                state[0] = (state[0] + 1) % (n_pix // B)
                return lib.hr_sample_train_batch(dev_cams.data_ptr(), N_VIEWS, images.data_ptr(), *fmt, H, W, 8, 0, 0,
                                                 state[0], B, None, coords.data_ptr(), rgb.data_ptr(), weight.data_ptr(),
                                                 None, None, stream)

            def rows(B=B, coords=coords, rgb=rgb, weight=weight, state=state):
                state[0] += 1
                return lib.hr_sample_train_rows(dev_cams.data_ptr(), N_VIEWS, images.data_ptr(), *fmt, H, W, 8,
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
    fish_host, fish_dev = cameras(True)
    sets = {"pinhole": workloads(this, pin_host[0], pin_dev), "fisheye": workloads(this, fish_host[0], fish_dev)}
    # (a), (b): pinhole against fisheye in this build, alternated
    res = {model: {k: [] for k in w} for model, w in sets.items()}
    for _ in range(args.rounds):
        for k in sets["pinhole"]:
            for model in ("pinhole", "fisheye"):
                res[model][k].append(kernel_us(*sets[model][k]))
    out["this_build_us"] = {m: {k: {"mean": sum(v) / len(v), "runs": v} for k, v in r.items()} for m, r in res.items()}
    print(json.dumps(out["this_build_us"]), flush=True)
    # (c): the pinhole workloads through another build, alternated with this one
    if args.other_lib:
        other = open_lib(args.other_lib)
        old_host, old_dev = cameras(False, PinholeCamera)
        builds = {"other": workloads(other, old_host[0], old_dev), "this": sets["pinhole"]}
        out["other_lib_abi"] = other.hr_abi_version()
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
