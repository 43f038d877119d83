#!/usr/bin/env python
"""Whole-frame throughput (SURVEY 8 f2 + f4): camera -> rays on the device -> sample net -> render -> uint8 HWC frame in
pinned host memory (hr_render_frame_to8b_host), the reference's validation_video / viewer iteration
(nlf/__init__.py:828-891) without the per-frame ray upload.  Wall clock per frame, synthetic trained-like parameters.

    python scripts/frame_bench.py --out frames.json [--lib /path/to/libhyperreel_b200.so]
"""
import argparse, json, os, sys, time
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import hyperreel_b200 as hb
from hyperreel_b200.state import seeded_state_dict

FRAMES = {
    # name: (builtin, overrides, W, H, note)
    "technicolor_2048x1088": ("technicolor_z_plane", dict(n_voxels=512000000), 2048, 1088, "BASELINE config 3 frame, S=32, K=12"),
    "donerf_800x800_S16": ("donerf_sphere", dict(n_voxels=216000000, z_channels=16), 800, 800, "BASELINE config 2 frame, S=16"),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--frames", type=int, default=20)
    ap.add_argument("--lib", default="", help="a libhyperreel_b200.so build other than the in-tree one")
    args = ap.parse_args()
    if args.lib:
        hb.lib.LIB_PATH = os.path.abspath(args.lib)  # read by load_library() on first use
    rows = []
    for name, (builtin, over, W, H, note) in FRAMES.items():
        cfg, ds = hb.configs.get(builtin, **over)
        sig = hb.lower(cfg, ds)
        model = hb.LightfieldModel(cfg, dataset=ds, mlp_mode="bf16x3")
        render = hb.RenderLightfield(model, None, cfg.render)
        render.load_state_dict(seeded_state_dict(sig, seed=11, density_gain=30.0), strict=False)
        render.eval()
        model.cuda() if hasattr(model, "cuda") else None
        f = 0.9 * W
        forward = builtin != "donerf_sphere"
        # the camera looks down its -z axis (utils/ray_utils.py:98-115).  Forward-facing model: stand at z = -1 and look
        # along +z (the bench's ray distribution, datasets/random.py:462-497); 360-degree model: look at the origin from z = 3
        pose = [[-1, 0, 0, 0.0], [0, 1, 0, 0.0], [0, 0, -1, -1.0]] if forward else [[1, 0, 0, 0.0], [0, 1, 0, 0.0], [0, 0, 1, 3.0]]
        out = torch.empty((H, W, 3), dtype=torch.uint8).pin_memory()
        times = []
        for i in range(args.frames + 3):
            cam = hb.Camera(pose=pose, K=[[f, 0, W / 2], [0, f, H / 2], [0, 0, 1]], width=W, height=H,
                            time=(i % 50) / 49.0, flipped=True)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            model.render_frame_to8b(cam, out)
            times.append(time.perf_counter() - t0)
        times = sorted(times[3:])
        ms = 1e3 * times[len(times) // 2]
        row = {"lib": args.lib, "frame": name, "note": note, "rays": W * H, "samples": sig.n_samples, "ms_per_frame": ms, "fps": 1e3 / ms,
               "mrays_s": W * H / ms / 1e3, "mean_pixel": float(out.float().mean())}
        rows.append(row)
        print(json.dumps(row), flush=True)
        del model, render
        torch.cuda.empty_cache()
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    json.dump(rows, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
