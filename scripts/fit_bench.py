"""Times hyperreel_b200.fit against a hand-written loop of the same calls, and the write and read of last.ckpt at the
Technicolor final grid.

The run: the Technicolor-shape model (configs.technicolor_z_plane) with technicolor_tensorf.yaml's optimisers and batch size
(tests/golden/reference/fit.npz), trained on the synthetic 3 x 3 Technicolor rig of tests/golden/dataset_cameras.npz at
--wh, --epochs epochs of --steps steps, no schedule iteration, evaluation or checkpoint inside the timed epochs.  fit and
the hand loop are alternated --rounds times after one warm-up run.  Each epoch ends in training_epoch_end's read-back, which
waits for the device; the host clock at each of those returns times every epoch after the first, so set-up (frames, system,
batches) and the first epoch stay out of the numbers.  Per step is an epoch's time over its steps.

The checkpoint: a system up-sampled to the final grid of technicolor_z_plane with one Adam step taken (so every moment
exists) and the occupancy mask at 200^3; torch.save of fit's checkpoint to --tmp and torch.load plus restore.

Usage: python scripts/fit_bench.py [--steps 200] [--epochs 4] [--rounds 3] [--wh 507 272] [--out result.json]
"""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--epochs", type=int, default=4)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--wh", type=int, nargs=2, default=[507, 272])
    ap.add_argument("--tmp", default=None)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch

    import hyperreel_b200 as hb
    from hyperreel_b200.fit import checkpoint, load_frames, restore
    from scripts.train_bench import gpu_facts
    from tests.test_dataset_cameras import _golden as scenes
    from tests.test_dataset_cameras import make_scene

    if not torch.cuda.is_available():
        raise SystemExit("fit_bench.py measures on the GPU; none found")
    tmp = tempfile.mkdtemp(dir=args.tmp)
    root, dcfg = make_scene(scenes(), "technicolor_lightfield", tmp)
    W, H = args.wh
    dcfg = dict(dcfg, img_wh=[W, H])
    training = json.loads(str(np.load(os.path.join(ROOT, "tests", "golden", "reference", "fit.npz"))["training/technicolor"]))
    never = 10 ** 6
    training.update(num_iters=args.steps, num_epochs=args.epochs, val_every=never, test_every=never, render_every=never,
                    ckpt_every=never)
    model = hb.config.to_plain(hb.configs.technicolor_z_plane())
    model["color"]["net"]["upsamp_list"], model["color"]["net"]["update_AlphaMask_list"] = [never], [never]
    for oc in training["optimizers"].values():
        oc["reset_opt_list"] = []
    cfg = {"model": model, "dataset": dcfg, "training": training, "regularizers": {}}
    rng = np.random.default_rng(0)

    def read_frame(source):
        return rng.integers(0, 256, (H, W, 3), dtype=np.uint8)

    ends = []
    epoch_end = hb.INRSystem.training_epoch_end

    def timed_epoch_end(self, outputs):
        out = epoch_end(self, outputs)  # reads the epoch's means back: the device has finished the epoch
        ends.append(time.perf_counter())
        return out

    hb.INRSystem.training_epoch_end = timed_epoch_end

    def epochs_of(run):
        ends.clear()
        run()
        return [float(t) for t in np.diff(ends)]  # every epoch after the first

    def run_fit():
        hb.fit(cfg, root, tempfile.mkdtemp(dir=tmp), read_frame=read_frame, ease="reference", schedule="reference")

    def run_hand():
        c = hb.to_cfg(json.loads(json.dumps(cfg)))
        views = {s: hb.dataset_cameras(c.dataset, root, s) for s in ("train", "val", "test", "render")}
        torch.manual_seed(0)
        images = {s: load_frames(views[s], c.dataset, read_frame) for s in ("train", "val", "test")}
        c.training.iters_per_epoch = args.steps
        system = hb.INRSystem(c, dataset=views["train"].facts, ease="reference", schedule="reference").cuda()
        batches = hb.DeviceRayBatches.from_config(c, views["train"].cameras, images["train"], c_in=system.render_fn.model.sig.c_in)
        for e in range(args.epochs):
            batches.set_epoch(e)
            outputs = [system.training_step(batches.batch(i), i, train_iter=args.steps * e + i) for i in range(len(batches))]
            system.training_epoch_end(outputs)

    rows = {"fit": [], "hand": []}
    epochs_of(run_hand)  # warm-up: module loads, allocator, first handle
    for _ in range(args.rounds):
        rows["fit"] += epochs_of(run_fit)
        rows["hand"] += epochs_of(run_hand)
    hb.INRSystem.training_epoch_end = epoch_end
    result = {"gpu": gpu_facts(), "wh": [W, H], "steps_per_epoch": args.steps, "epochs": args.epochs,
              "batch_size": training["batch_size"]}
    for k, v in rows.items():
        result[f"{k}_epoch_s"] = v
        result[f"{k}_ms_per_step"] = [1e3 * t / args.steps for t in v]

    # the checkpoint at the final grid
    c = hb.to_cfg({"model": model, "training": dict(training, iters_per_epoch=args.steps), "regularizers": {}})
    facts = hb.dataset_cameras(dcfg, root, "train").facts
    system = hb.INRSystem(c, dataset=facts, ease="reference", schedule="reference").cuda()
    net = system.render_fn.model.color_model.net
    n_final = int(model["color"]["net"]["N_voxel_final"])
    net.upsample_volume_grid(hb.state.n_to_reso(n_final, net.aabb.detach().cpu()))
    net.alphaMask_thres = 0.0
    net.updateAlphaMask((200, 200, 200))
    system.configure_optimizers()
    for o in system.optimizers():
        for p in o.param_groups[0]["params"]:
            p.grad = torch.full_like(p, 1e-3)
        o.step()
    system.training_started = True
    batches = types.SimpleNamespace(seed=0, epoch=0, set_epoch=lambda e: None)
    path = os.path.join(tmp, "last.ckpt")
    saves, loads = [], []
    for _ in range(args.rounds):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        torch.save(checkpoint(system, batches, 0, 1), path)
        saves.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        restore(system, batches, torch.load(path, map_location="cpu", weights_only=True))
        torch.cuda.synchronize()
        loads.append(time.perf_counter() - t0)
    result.update(final_grid=net.gridSize.tolist(), ckpt_mb=os.path.getsize(path) / 2 ** 20, ckpt_save_s=saves,
                  ckpt_load_restore_s=loads)
    shutil.rmtree(tmp)
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
