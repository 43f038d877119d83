#!/usr/bin/env python
"""A/B timing of the sample net (mlp_tc2_kernel) between library builds:

    python scripts/mlp_bench.py --lib parent=/path/to/parent.so --lib change=hyperreel_b200/libhyperreel_b200.so \
        --rounds 3 --out out/mlp_bench.json

Every (round, build) pair runs in a process of its own that loads that build's library, so builds alternate in time and
share the card's state.  For each build and workload it reports the sample-net and render kernel times (CUDA events the
library records around each kernel, averaged over --launches steps with the L2 flushed between them), the whole step, a
hash of the step's rgb (builds that must agree bit for bit hash alike) and the card's name, power limit and SM clock read
right after the timed loop.
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# bench.py's flagship workload and its two extra single-GPU workloads (rays per step)
WORKLOADS = {
    "technicolor_s32": ("technicolor_z_plane", dict(n_voxels=512000000), 65536),
    "donerf_sphere_s16": ("donerf_sphere", dict(n_voxels=216000000, z_channels=16), 640000),
    "neural3d_s64": ("neural_3d_z_plane", dict(n_voxels=262144000), 685464),
}


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                         text=True, timeout=30).stdout.strip()
    return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))


def child(lib_path, names, launches):
    import torch

    sys.path.insert(0, ROOT)
    from hyperreel_b200 import lib as hl

    hl.LIB_PATH = os.path.abspath(lib_path)  # read by load_library() on first use
    import hyperreel_b200 as hb
    from hyperreel_b200.state import seeded_state_dict

    assert torch.cuda.is_available(), "mlp_bench needs a GPU"
    dev = torch.device("cuda", 0)
    flush = torch.empty((512 << 20) // 4, dtype=torch.float32, device=dev)
    for name in names:
        builtin, over, n = WORKLOADS[name]
        cfg, ds = hb.configs.get(builtin, **over)
        sig = hb.lower(cfg, ds)
        sd = seeded_state_dict(sig, seed=11, density_gain=30.0)
        model = hb.LightfieldModel(cfg, dataset=ds)
        render = hb.RenderLightfield(model, None, cfg.render, net_chunk=1 << 22)
        render.load_state_dict(sd, strict=False)
        render.eval()
        rays = hb.rays.for_signature(sig, n, seed=5).to(dev)
        for _ in range(5):
            rgb = render(rays)["rgb"]
        torch.cuda.synchronize()
        digest = hashlib.sha256(rgb.cpu().numpy().tobytes()).hexdigest()[:16]
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
        row = {"lib": lib_path, "workload": name, "rays": n, "launches": launches, "sample_net_ms": tm["mlp_ms"],
               "render_kernel_ms": tm["render_ms"], "step_ms": step_ms / launches, "rgb_sha256": digest, "card": card()}
        print("ROW " + json.dumps(row), flush=True)
        del model, render, rays
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=[], help="label=path of a libhyperreel_b200.so build (two or more)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--out", default="")
    ap.add_argument("--child", default="", help=argparse.SUPPRESS)
    args = ap.parse_args()
    names = [w for w in args.workloads.split(",") if w]
    for w in names:
        if w not in WORKLOADS:
            ap.error(f"unknown workload {w!r} (known: {', '.join(WORKLOADS)})")
    if args.child:
        child(args.child, names, args.launches)
        return
    libs = [x.split("=", 1) for x in args.lib]
    if len(libs) < 2 or any(len(x) != 2 for x in libs):
        ap.error("give at least two --lib label=path")
    rows = []
    for r in range(args.rounds):
        for label, path in libs:
            res = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", path, "--workloads", ",".join(names),
                                  "--launches", str(args.launches)], capture_output=True, text=True)
            if res.returncode != 0:
                sys.stderr.write(res.stdout[-4000:] + res.stderr[-4000:])
                raise SystemExit(f"{label}: child exited with {res.returncode}")
            for line in res.stdout.splitlines():
                if line.startswith("ROW "):
                    row = dict(json.loads(line[4:]), build=label, round=r)
                    rows.append(row)
                    print(json.dumps(row), flush=True)
    print("\nbuild     workload             sample net ms (per round)        step ms (per round)        rgb")
    for w in names:
        for label, _ in libs:
            sel = [x for x in rows if x["build"] == label and x["workload"] == w]
            net = " ".join(f"{x['sample_net_ms']:.4f}" for x in sel)
            step = " ".join(f"{x['step_ms']:.4f}" for x in sel)
            print(f"{label:9s} {w:20s} {net:32s} {step:26s} {','.join(sorted({x['rgb_sha256'] for x in sel}))}")
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
