"""Times INRSystem.training_step (train_net="tc") on the Technicolor shape with the EaseValue warm-up (ease="reference") against
the default, at 16,384 and 65,536 rays, configurations alternated round by round:

  * default            ease="elapsed", no train_iter
  * eased_in_window    ease="reference", train_iter 6000, 6001, ... (sigma and point_sigma mid-window: hr_set_activations
                       every step)
  * eased_past_window  ease="reference", train_iter 20000, 20001, ... (every window elapsed: nothing to update)
  * rebuild_each_step  ease="reference" inside the window with the native handle re-created and re-uploaded every step (what
                       set_iter would cost without the in-place update)

and the host time of LightfieldModel.set_iter inside the window.

Usage: python scripts/ease_bench.py [--steps 20] [--rounds 3] [--out result.json]
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch

    import bench
    import hyperreel_b200 as hb
    from scripts.train_bench import gpu_facts

    if not torch.cuda.is_available():
        raise SystemExit("ease_bench.py measures on the GPU; none found")
    dev = torch.device("cuda")
    _, cfg, ds, sig, sd = bench.build_workload(gain=600.0, app_gain=6.0)
    full = hb.to_cfg({"model": cfg, "training": {"ray_chunk": 1 << 20, "iters_per_epoch": 4000}, "dataset": ds})
    systems = {}
    for ease in ("elapsed", "reference"):
        s = hb.INRSystem(full, train_net="tc", ease=ease)
        s.load_state_dict(sd)
        s.to(dev)
        s.configure_optimizers()
        systems[ease] = s
    it = {"n": 0}

    def step(name, batch):
        it["n"] += 1
        if name == "default":
            systems["elapsed"].training_step(batch)
            return
        s = systems["reference"]
        if name == "rebuild_each_step":
            s.render_fn.model._release_handle()
        base = 20000 if name == "eased_past_window" else 6000
        s.training_step(batch, train_iter=base + it["n"] % 1000)

    def timed(name, batch, steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(steps):
            step(name, batch)
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / steps

    names = ("default", "eased_in_window", "eased_past_window", "rebuild_each_step")
    out = {"gpu": gpu_facts(), "workload": "technicolor_z_plane, grid 1007x1007x503, K=12, INRSystem.training_step, train_net=tc",
           "batches": []}
    for n in (16384, 65536):
        g = torch.Generator().manual_seed(3)
        batch = {"coords": hb.rays.for_signature(sig, n, seed=9).to(dev), "rgb": torch.rand(n, 3, generator=g).to(dev)}
        for name in names:
            for _ in range(3):
                step(name, batch)
        torch.cuda.synchronize()
        ms = {k: [] for k in names}
        for _ in range(args.rounds):
            for name in names:
                ms[name].append(timed(name, batch, args.steps))
        out["batches"].append({"rays": n, "train_step_ms": {k: {"mean": sum(v) / len(v), "runs": v} for k, v in ms.items()}})
    model = systems["reference"].render_fn.model
    model.set_iter(6000)
    t0 = time.perf_counter()
    for k in range(1000):
        model.set_iter(6001 + k)
    out["set_iter_host_us_in_window"] = (time.perf_counter() - t0) / 1000 * 1e6
    out["gpu_after"] = gpu_facts()
    text = json.dumps(out, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
