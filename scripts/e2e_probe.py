#!/usr/bin/env python
"""Where the end-to-end time of hr_render_host goes: copy times alone, the host-buffer call at several chunk sizes, and
one row per pinned / pageable buffer combination and batch size, optionally A/B between library builds:

    python scripts/e2e_probe.py --lib parent=/path/to/parent.so --lib change=hyperreel_b200/libhyperreel_b200.so \
        --rounds 3 --out out/e2e_probe.json

Every (round, build) pair runs in a process of its own that loads that build's library (the C ABI is the same, so one
binding loads either), so builds alternate in time and share the card's state.  Each row is the median wall time of
repeated calls on the same buffers, the L2 flushed before each call, with a hash of the call's rgb (builds that must agree
bit for bit hash alike) and the card's name and power limit.  Without --lib the in-tree library runs once.
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                         text=True, timeout=30).stdout.strip()
    return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))


def child(lib_path, reps):
    import torch

    sys.path.insert(0, ROOT)
    if lib_path:
        from hyperreel_b200 import lib as hl

        hl.LIB_PATH = os.path.abspath(lib_path)  # read by load_library() on first use
    import hyperreel_b200 as hb
    from hyperreel_b200.state import seeded_state_dict

    assert torch.cuda.is_available(), "e2e_probe needs a GPU"
    dev = torch.device("cuda", 0)
    cfg, ds = hb.configs.get("technicolor_z_plane", n_voxels=512000000)
    sig = hb.lower(cfg, ds)
    sd = seeded_state_dict(sig, seed=11, density_gain=30.0)
    models = {}
    for mode in ("bf16x3", "fp32"):
        model = hb.LightfieldModel(cfg, dataset=ds, mlp_mode=mode)
        render = hb.RenderLightfield(model, None, cfg.render)
        render.load_state_dict(sd, strict=False)
        render.eval()
        models[mode] = (model, render)
    flush = torch.empty((512 << 20) // 4, dtype=torch.float32, device=dev)

    def wall(fn, do_flush=True):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        ts = []
        for _ in range(reps):
            if do_flush:
                flush.zero_()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            ts.append(time.perf_counter() - t0)
        ts.sort()
        return 1e3 * ts[len(ts) // 2]

    def digest(t):
        return hashlib.sha256(t.numpy().tobytes()).hexdigest()[:16]

    rows = []

    def row(case, ms, rgb=None):
        rows.append({"case": case, "ms": ms, "rgb_sha256": digest(rgb) if rgb is not None else ""})

    model, render = models["bf16x3"]
    n = 65536
    rays_host = hb.rays.for_signature(sig, n, seed=5).pin_memory()
    rgb_host = torch.empty((n, 3)).pin_memory()
    rays_dev = rays_host.to(dev)
    rgb_dev = torch.empty((n, 3), device=dev)
    row("h2d_2MB", wall(lambda: rays_dev.copy_(rays_host, non_blocking=True)))
    row("d2h_786KB", wall(lambda: rgb_host.copy_(rgb_dev, non_blocking=True)))
    row("device_render", wall(lambda: render(rays_dev)))
    row("render_host_default", wall(lambda: model.render_host(rays_host, rgb_host)), rgb_host)
    row("render_host_default_noflush", wall(lambda: model.render_host(rays_host, rgb_host), do_flush=False), rgb_host)
    for chunk in (65536, 18944):
        row(f"render_host_chunk{chunk}", wall(lambda: model.render_host(rays_host, rgb_host, chunk=chunk)), rgb_host)
        row(f"render_host_chunk{chunk}_noflush", wall(lambda: model.render_host(rays_host, rgb_host, chunk=chunk), do_flush=False),
            rgb_host)

    wave = torch.cuda.get_device_properties(dev).multi_processor_count * 128  # one tile wave of the tensor-core net
    for n in (777, 65536, 16 * wave + 3000, 300000):
        rays = hb.rays.for_signature(sig, n, seed=5)
        for rays_pinned in (True, False):
            for rgb_pinned in (True, False):
                r = rays.pin_memory() if rays_pinned else rays.clone()
                out = torch.empty((n, 3))
                out = out.pin_memory() if rgb_pinned else out
                case = f"bf16x3 rays={'pinned' if rays_pinned else 'pageable'} rgb={'pinned' if rgb_pinned else 'pageable'} n={n}"
                row(case, wall(lambda: model.render_host(r, out)), out)
    rays = hb.rays.for_signature(sig, 65536, seed=5).pin_memory()
    out = torch.empty((65536, 3)).pin_memory()
    fp32_model = models["fp32"][0]
    row("fp32 rays=pinned rgb=pinned n=65536", wall(lambda: fp32_model.render_host(rays, out)), out)
    row("bf16x3 rays=pinned rgb=None n=65536", wall(lambda: model.render_host(rays)), model.render_host(rays))
    for r in rows:
        r["card"] = card()
        print("ROW " + json.dumps(r), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=[], help="label=path of a libhyperreel_b200.so build")
    ap.add_argument("--rounds", type=int, default=1)
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--out", default="")
    ap.add_argument("--child", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child is not None:
        child(args.child, args.reps)
        return
    libs = [x.split("=", 1) for x in args.lib] or [["tree", ""]]
    if any(len(x) != 2 for x in libs):
        ap.error("--lib takes label=path")
    rows = []
    for rnd in range(args.rounds):
        for label, path in libs:
            res = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", path, "--reps", str(args.reps)],
                                 capture_output=True, text=True)
            if res.returncode != 0:
                sys.stderr.write(res.stdout[-4000:] + res.stderr[-4000:])
                raise SystemExit(f"{label}: child exited with {res.returncode}")
            for line in res.stdout.splitlines():
                if line.startswith("ROW "):
                    rows.append(dict(json.loads(line[4:]), build=label, round=rnd))
    cases = list(dict.fromkeys(r["case"] for r in rows))
    print(f"{'case':48s} " + " ".join(f"{label + ' ms (per round)':28s}" for label, _ in libs) + " rgb agrees")
    for case in cases:
        cols, hashes = [], set()
        for label, _ in libs:
            sel = [r for r in rows if r["case"] == case and r["build"] == label]
            cols.append(" ".join(f"{r['ms']:.4f}" for r in sel))
            hashes |= {r["rgb_sha256"] for r in sel}
        print(f"{case:48s} " + " ".join(f"{c:28s}" for c in cols) + f" {'yes' if len(hashes) == 1 else 'NO'}")
    if rows:
        print("card:", json.dumps(rows[-1]["card"]))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
