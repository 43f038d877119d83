#!/usr/bin/env python
"""RGBA frames against RGB frames on the device, for the three places a DoNeRF or Catacaustics frame is used:

  batches   hr_sample_train_batch (the whole-image permutation) and hr_sample_train_rows (draws with replacement)
            over 8 views of 800 x 800, at 16 384 and 65 536 rows per batch: RGBA reads one aligned 4-byte pixel and
            composites it over white, RGB reads three bytes
  score     score_views of a DoNeRF-shaped model (tests/cases.py donerf_s16) on 4 views of 800 x 800, per view
  resize    DoNeRF's 2x INTER_AREA, 1600 x 1600 -> 800 x 800, and a Catacaustics-sized BICUBIC, 1500 x 999 -> 1000 x 666,
            2 frames per call

Each measurement is CUDA events around one call on the current stream, with the L2 flushed before it (a 256 MB buffer
written), the RGB and RGBA calls alternated, `--reps` of each after `--warmup` of each; reported as the median and the
spread (min, max) in microseconds, and the RGBA / RGB ratio of the medians.  The batch and resize calls go straight to the C
entry points with their outputs and workspaces allocated beforehand, so no Python time is inside the events.  Every RGBA
result is checked once against the RGB path on opaque frames (bit for bit).  The card's name, power limit and SM clocks are
read in the same run.

    python scripts/rgba_bench.py --out rgba.json
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import hyperreel_b200 as hb  # noqa: E402
from hyperreel_b200 import lib as L  # noqa: E402


def _gpu_facts():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        q = ""
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi name, power.limit, clocks.max.sm, clocks.sm": q}


class Timer:
    def __init__(self):
        self.flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")

    def once(self, fn):
        self.flush.fill_(1)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        return a.elapsed_time(b) * 1e3

    def pair(self, rgb, rgba, reps, warmup):
        for _ in range(warmup):
            self.once(rgb)
            self.once(rgba)
        t = {"rgb": [], "rgba": []}
        for _ in range(reps):
            t["rgb"].append(self.once(rgb))
            t["rgba"].append(self.once(rgba))
        out = {k: {"median_us": statistics.median(v), "min_us": min(v), "max_us": max(v)} for k, v in t.items()}
        out["rgba_over_rgb"] = out["rgba"]["median_us"] / out["rgb"]["median_us"]
        return out


def _frames(n, W, H, ch, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (n, H, W, ch), generator=g, dtype=torch.uint8).cuda()


def bench_batches(timer, reps, warmup):
    lib = L.load_library()
    n, W, H = 8, 800, 800
    rgba = _frames(n, W, H, 4, 1)
    opaque = rgba.clone()
    opaque[..., 3] = 255
    rgb = opaque[..., :3].contiguous()
    cams = [hb.Camera(pose=np.eye(4)[:3], K=[[800.0, 0, 400.0], [0, 800.0, 400.0], [0, 0, 1]], width=W, height=H,
                      use_ndc=False) for _ in range(n)]
    recs = (L.hr_camera * n)(*[c.to_c() for c in cams])
    dcams = torch.frombuffer(bytearray(bytes(recs)), dtype=torch.uint8).cuda()
    start = torch.tensor([v * H * W for v in range(n + 1)], dtype=torch.int64, device="cuda")
    rule = torch.tensor([(1, 0)] * n, dtype=torch.int32, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    out = {}
    for B in (16384, 65536):
        coords = torch.empty((B, 6), device="cuda")
        col = torch.empty((B, 3), device="cuda")
        w = torch.empty((B, 1), device="cuda")
        rows = C.c_int64(0)

        def permute(images, fmt, i=3):
            return lambda: L.check(lib.hr_sample_train_batch(
                dcams.data_ptr(), n, images.data_ptr(), fmt, H, W, 6, 0, 0, i, B, None, coords.data_ptr(), col.data_ptr(),
                w.data_ptr(), None, C.byref(rows), st))

        def replace(images, fmt, i=3):
            return lambda: L.check(lib.hr_sample_train_rows(
                dcams.data_ptr(), n, images.data_ptr(), fmt, H, W, 6, start.data_ptr(), rule.data_ptr(), n * H * W,
                L.SAMPLE_REPLACE, 0, 0, i, B, None, coords.data_ptr(), col.data_ptr(), w.data_ptr(), None, None,
                C.byref(rows), st))

        for name, mk in (("permute", permute), ("replace", replace)):
            got = []
            for images, fmt in ((rgb, L.PIXEL_RGB8), (opaque, L.PIXEL_RGBA8)):
                mk(images, fmt)()
                got.append((coords.clone(), col.clone()))
            assert all(torch.equal(x, y) for x, y in zip(*got)), (name, B)
            out[f"{name}_{B}"] = timer.pair(mk(rgb, L.PIXEL_RGB8), mk(rgba, L.PIXEL_RGBA8), reps, warmup)
    return out


def bench_score(timer, reps, warmup):
    from tests.cases import build_case

    case = build_case("donerf_s16")
    model = hb.LightfieldModel(case.model_cfg, dataset=case.dataset)
    render = hb.RenderLightfield(model, None, case.model_cfg.render)
    render.load_state_dict(case.state_dict, strict=False)
    render.eval()
    F, W, H = 4, 800, 800
    cams = [hb.Camera(pose=np.eye(4)[:3], K=[[800.0, 0, 400.0], [0, 800.0, 400.0], [0, 0, 1]], width=W, height=H,
                      time=0.0) for _ in range(F)]
    rgba = _frames(F, W, H, 4, 2)
    opaque = rgba.clone()
    opaque[..., 3] = 255
    rgb = opaque[..., :3].contiguous()
    outs = [torch.empty((F, 2), dtype=torch.float64, device="cuda") for _ in range(2)]
    model.score_views(cams, rgb, out=outs[0])
    model.score_views(cams, opaque, out=outs[1], rgba=True)
    assert torch.equal(outs[0], outs[1])
    res = timer.pair(lambda: model.score_views(cams, rgb, out=outs[0]),
                     lambda: model.score_views(cams, rgba, out=outs[1], rgba=True), reps, warmup)
    for k in ("rgb", "rgba"):
        res[k]["per_view_us"] = res[k]["median_us"] / F
    return res


def bench_resize(timer, reps, warmup):
    lib = L.load_library()
    st = torch.cuda.current_stream().cuda_stream
    out = {}
    for name, (W0, H0, W, H, method) in {"donerf_cv2_area_2x": (1600, 1600, 800, 800, "cv2_area"),
                                         "catacaustics_pil_bicubic": (1500, 999, 1000, 666, "pil_bicubic")}.items():
        n, m = 2, L.RESIZE_METHODS[method]
        calls, res = {}, []
        for ch, fmt in ((3, L.PIXEL_RGB8), (4, L.PIXEL_RGBA8)):
            src = _frames(n, W0, H0, ch, 3)
            if ch == 4:
                src[..., 3] = 255
            dst = torch.empty((n, H, W, ch), dtype=torch.uint8, device="cuda")
            need = int(lib.hr_resize_workspace_bytes(n, H0, W0, H, W, m, fmt))
            ws = torch.empty(max(need, 1), dtype=torch.uint8, device="cuda")
            calls[ch] = (lambda src=src, dst=dst, ws=ws, need=need, fmt=fmt, ch=ch: L.check(lib.hr_resize_frames(
                src.data_ptr(), n, H0, W0, dst.data_ptr(), H, W, ch * W, m, 0, fmt, ws.data_ptr(), need, st)))
            calls[ch]()
            res.append((src, dst))
        # opaque RGBA resizes its colour channels as RGB does
        assert torch.equal(hb.resize_frames(res[1][0][..., :3].contiguous(), (W, H), method), res[1][1][..., :3])
        r = timer.pair(calls[3], calls[4], reps, warmup)
        for k in ("rgb", "rgba"):
            r[k]["per_frame_us"] = r[k]["median_us"] / n
        out[name] = r
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("rgba_bench.py measures on the GPU: no CUDA device")
    timer = Timer()
    res = {"gpu": _gpu_facts(), "reps": args.reps, "warmup": args.warmup,
           "batches_8x800x800": bench_batches(timer, args.reps, args.warmup),
           "score_views_4x800x800": bench_score(timer, max(args.reps // 5, 5), 2),
           "resize": bench_resize(timer, args.reps, args.warmup)}
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
