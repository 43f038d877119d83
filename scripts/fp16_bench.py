#!/usr/bin/env python
"""The fp16 sample net (mlp_mode="fp16") against the default bf16x3 net, in one process on one card:

    python scripts/fp16_bench.py --rounds 3 --out out/fp16_bench.json

For each round, workload and mode (bf16x3 and fp16 alternate within a round) it reports the sample-net and render kernel
times (CUDA events the library records around each kernel, averaged over --launches steps with the L2 flushed between
them) and the whole step.  Then the PSNR of the fp16 net's rgb against the bf16x3 net's on the trained fixtures' rays, and
the card's name, power limit and SM clocks.
"""
import argparse
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# bench.py's flagship workload and its two extra single-GPU workloads (rays per step), as in scripts/mlp_bench.py
WORKLOADS = {
    "technicolor_s32": ("technicolor_z_plane", dict(n_voxels=512000000), 65536),
    "donerf_sphere_s16": ("donerf_sphere", dict(n_voxels=216000000, z_channels=16), 640000),
    "neural3d_s64": ("neural_3d_z_plane", dict(n_voxels=262144000), 685464),
}
MODES = ("bf16x3", "fp16")
TRAINED = ("technicolor_trained", "donerf_trained", "neural3d_trained")


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                         text=True, timeout=30).stdout.strip()
    return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))


def time_step(hb, cfg, ds, sd, sig, mode, n, launches, flush, dev):
    import torch

    model = hb.LightfieldModel(cfg, dataset=ds, mlp_mode=mode)
    render = hb.RenderLightfield(model, None, cfg.render, net_chunk=1 << 22)
    render.load_state_dict(sd, strict=False)
    render.eval()
    rays = hb.rays.for_signature(sig, n, seed=5).to(dev)
    with torch.no_grad():
        for _ in range(5):
            render(rays)
        torch.cuda.synchronize()
        model.timing(True)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        step_ms = 0.0
        for _ in range(launches):
            flush.zero_()  # evict L2 between launches
            a.record()
            render(rays)
            b.record()
            b.synchronize()
            step_ms += a.elapsed_time(b)
        tm = model.timing_read()
        model.timing(False)
    return {"sample_net_ms": tm["mlp_ms"], "render_kernel_ms": tm["render_ms"], "step_ms": step_ms / launches}


def psnr_rows(hb):
    import torch
    from tests.cases import build_case

    rows = []
    for name in TRAINED:
        case = build_case(name)
        rgb = {}
        for mode in MODES:
            model = hb.LightfieldModel(case.model_cfg, dataset=case.dataset, mlp_mode=mode)
            render = hb.RenderLightfield(model, None, case.model_cfg.render)
            render.load_state_dict(case.state_dict, strict=False)
            render.cuda().eval()
            with torch.no_grad():
                rgb[mode] = render(case.rays.cuda())["rgb"].double()
        mse = float(((rgb["fp16"] - rgb["bf16x3"]) ** 2).mean())
        rows.append({"fixture": name, "rays": int(case.rays.shape[0]), "mse": mse,
                     "psnr_db": (-10.0 * math.log10(mse)) if mse > 0 else float("inf"),
                     "max_abs": float((rgb["fp16"] - rgb["bf16x3"]).abs().max())})
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    names = [w for w in args.workloads.split(",") if w]
    for w in names:
        if w not in WORKLOADS:
            ap.error(f"unknown workload {w!r} (known: {', '.join(WORKLOADS)})")

    import torch

    import hyperreel_b200 as hb
    from hyperreel_b200.state import seeded_state_dict

    if not torch.cuda.is_available():
        raise SystemExit("fp16_bench needs a GPU")
    dev = torch.device("cuda", 0)
    flush = torch.empty((512 << 20) // 4, dtype=torch.float32, device=dev)
    rows = []
    for r in range(args.rounds):
        for w in names:
            builtin, over, n = WORKLOADS[w]
            cfg, ds = hb.configs.get(builtin, **over)
            sig = hb.lower(cfg, ds)
            sd = seeded_state_dict(sig, seed=11, density_gain=30.0)
            for mode in MODES:
                row = dict(round=r, workload=w, mode=mode, rays=n, launches=args.launches,
                           **time_step(hb, cfg, ds, sd, sig, mode, n, args.launches, flush, dev))
                rows.append(row)
                print(json.dumps(row), flush=True)
                torch.cuda.empty_cache()
    psnr = psnr_rows(hb)
    info = card()
    print("\nworkload             mode     sample net ms (per round)        step ms (per round)")
    for w in names:
        for mode in MODES:
            sel = [x for x in rows if x["workload"] == w and x["mode"] == mode]
            print(f"{w:20s} {mode:8s} {' '.join(f'{x['sample_net_ms']:.4f}' for x in sel):32s} "
                  f"{' '.join(f'{x['step_ms']:.4f}' for x in sel)}")
    for p in psnr:
        print(f"{p['fixture']}: PSNR(fp16 vs bf16x3) = {p['psnr_db']:.2f} dB, max |diff| = {p['max_abs']:.3e} over {p['rays']} rays")
    print("card:", info)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"rows": rows, "psnr": psnr, "card": info}, f, indent=1)


if __name__ == "__main__":
    main()
