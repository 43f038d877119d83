"""Times INRSystem.training_step with schedule="constant" and schedule="reference" on the Technicolor shape (the system of
scripts/train_data_bench.py, train_net="tc", one resident batch), at 16,384 and 65,536 rays per step.  Both systems read the
optimisers of technicolor_tensorf.yaml (recorded in tests/golden/reference/schedule.npz) and are driven with
training_step(batch, train_iter=i) at iterations no schedule step or restart lists, so the timed difference is the host work
the reference schedule adds to a step.  The two are alternated round by round; CUDA events per round, mean over its steps.

Usage: python scripts/schedule_bench.py [--steps 30] [--rounds 5] [--out result.json]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch

    import bench
    import hyperreel_b200 as hb
    from scripts.train_bench import gpu_facts
    from scripts.train_data_bench import rig_cameras

    if not torch.cuda.is_available():
        raise SystemExit("schedule_bench.py measures on the GPU; none found")
    g = np.load(os.path.join(ROOT, "tests", "golden", "reference", "schedule.npz"))
    training = json.loads(str(g["technicolor/training_json"]))
    _, cfg, ds, _, sd = bench.build_workload(gain=600.0, app_gain=6.0)
    systems = {}
    for schedule in ("constant", "reference"):
        s = hb.INRSystem(hb.to_cfg({"model": cfg, "training": dict(training, ray_chunk=1 << 20), "dataset": ds}),
                         train_net="tc", schedule=schedule)
        s.load_state_dict(sd)
        s.cuda()
        s.configure_optimizers()
        systems[schedule] = s
    cams = rig_cameras(hb, 4, 1.0)
    gen = torch.Generator(device="cuda").manual_seed(0)
    images = torch.randint(0, 256, (4, 1088, 2048, 3), generator=gen, device="cuda", dtype=torch.uint8)
    out = {"gpu": gpu_facts(), "workload": "technicolor_z_plane, INRSystem.training_step, train_net='tc', resident batch",
           "batches": []}
    it = {"constant": 100, "reference": 100}  # past iteration 0, before the first up-sampling / restart at 4000

    def events(name, batch, k):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(k):
            systems[name].training_step(batch, train_iter=it[name])
            it[name] += 1
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / k

    for B in (16384, 65536):
        batch = hb.DeviceRayBatches(cams, images, batch_size=B, seed=0).batch(1)
        for name in systems:
            events(name, batch, 3)
        ms = {name: [] for name in systems}
        for _ in range(args.rounds):
            for name in systems:
                ms[name].append(events(name, batch, args.steps))
        out["batches"].append({"rays": B, "train_step_ms": {n: {"mean": float(np.mean(v)), "runs": v} for n, v in ms.items()}})
        print(json.dumps(out["batches"][-1]), flush=True)
    assert max(it.values()) < 4000
    lrs = {n: [o.param_groups[0]["lr"] for o in s.optimizers()] for n, s in systems.items()}
    assert lrs["constant"] == lrs["reference"]  # no epoch has ended: both still train at the base rates
    out["gpu_after"] = gpu_facts()
    text = json.dumps(out, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
