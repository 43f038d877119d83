"""Times the sample net's two training paths on the Technicolor shape (bench.py's train_step workload).

  * INRSystem.training_step at 16,384 and 65,536 rays with train_net="torch" (cuBLAS SGEMM Linear layers) and "tc"
    (hr_train_net_forward / hr_train_net_backward), alternated round by round;
  * the torch path's sample-net layers alone (hr_encode_rays + Linear/LeakyReLU forward + their autograd backward), its share of
    the torch step;
  * the tc path's kernels alone (torch.profiler, in a separate run): the forward with saved activations, the dX and dW GEMMs and
    the split-K reduction, with executed bf16 TFLOP/s (3 products per MAC, bf16x3).

Usage: python scripts/train_bench.py [--steps 20] [--rounds 3] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gpu_facts():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return dict(zip(q.split(","), [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")])) if r.returncode == 0 else {}


def net_macs(c):
    """(forward, dX, dW) multiply-adds per ray of the sample net: dX skips the first layer and the encoded-input columns."""
    fwd = dx = 0
    for l in range(c.mlp_layers):
        out = c.mlp_out if l == c.mlp_layers - 1 else c.mlp_width
        inp = c.mlp_in if l == 0 else c.mlp_width + (c.mlp_in if l == c.mlp_skip else 0)
        fwd += out * inp
        if l > 0:
            dx += out * c.mlp_width
    return fwd, dx, fwd


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch

    import bench
    import hyperreel_b200 as hb

    if not torch.cuda.is_available():
        raise SystemExit("train_bench.py measures on the GPU; none found")
    dev = torch.device("cuda")
    _, cfg, ds, sig, sd = bench.build_workload(gain=600.0, app_gain=6.0)
    systems = {}
    for mode in ("torch", "tc"):
        s = hb.INRSystem(hb.to_cfg({"model": cfg, "training": {"ray_chunk": 1 << 20, "iters_per_epoch": 4000}, "dataset": ds}),
                         train_net=mode)
        s.load_state_dict(sd)
        s.to(dev)
        s.configure_optimizers()
        systems[mode] = s
    c = sig.cfg
    out = {"gpu": gpu_facts(), "workload": "technicolor_z_plane, grid 1007x1007x503, K=12, INRSystem.training_step",
           "net": {"width": c.mlp_width, "layers": c.mlp_layers, "in": c.mlp_in, "out": c.mlp_out, "skip": c.mlp_skip},
           "batches": []}

    def timed(fn, steps):
        evs = []
        for _ in range(steps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            evs.append((a, b))
        torch.cuda.synchronize()
        return sum(a.elapsed_time(b) for a, b in evs) / steps

    for n in (16384, 65536):
        g = torch.Generator().manual_seed(3)
        batch = {"coords": hb.rays.for_signature(sig, n, seed=9).to(dev), "rgb": torch.rand(n, 3, generator=g).to(dev)}
        for s in systems.values():
            for _ in range(3):
                s.training_step(batch)
        torch.cuda.synchronize()
        step_ms = {"torch": [], "tc": []}
        for _ in range(args.rounds):
            for mode, s in systems.items():
                step_ms[mode].append(timed(lambda: s.training_step(batch), args.steps))
        # the torch path's net alone: forward + backward of its Linear layers on the encoded input
        model = systems["torch"].render_fn.model
        rays = batch["coords"]
        model._ensure_uploaded(dev)
        d_heads = torch.randn((n, c.mlp_out), device=dev)

        def torch_net():
            x = model._torch_net(rays, False)
            x.backward(d_heads)

        for _ in range(3):
            torch_net()
        torch_net_ms = timed(torch_net, args.steps)
        # the tc path's net alone: hr_train_net_forward + hr_train_net_backward
        tmodel = systems["tc"].render_fn.model
        tmodel._ensure_uploaded(dev)

        def tc_net():
            heads, ws = tmodel._train_net_forward(rays)
            tmodel._train_net_backward(ws, d_heads, n)

        for _ in range(3):
            tc_net()
        tc_net_ms = timed(tc_net, args.steps)
        # per-kernel times of the tc net (profiler run of its own)
        from torch.profiler import ProfilerActivity, profile

        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.steps):
                tc_net()
            torch.cuda.synchronize()
        kern = {}
        for e in prof.key_averages():
            name = e.key
            tag = ("forward (mlp_tc2_kernel, SAVE)" if "mlp_tc2_kernel" in name else
                   "dX (train_gemm_kernel<false>)" if "train_gemm_kernel<false>" in name else
                   "dW (train_gemm_kernel<true>)" if "train_gemm_kernel<true>" in name else
                   "dW split-K reduction" if "train_dw_reduce" in name else None)
            if tag:
                t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
                kern[tag] = kern.get(tag, 0.0) + t / 1e3 / args.steps  # ms per step
        fwd, dx, dw = net_macs(c)
        flops = {"forward (mlp_tc2_kernel, SAVE)": fwd, "dX (train_gemm_kernel<false>)": dx, "dW (train_gemm_kernel<true>)": dw}
        kernels = {k: {"ms": v, "executed_bf16_tflops": (6.0 * flops[k] * n / (v * 1e-3) / 1e12) if k in flops and v > 0 else None}
                   for k, v in kern.items()}
        mean = lambda v: sum(v) / len(v)
        out["batches"].append({
            "rays": n,
            "train_step_ms": {m: {"mean": mean(v), "runs": v} for m, v in step_ms.items()},
            "speedup_tc_over_torch": mean(step_ms["torch"]) / mean(step_ms["tc"]),
            "torch_net_fwd_bwd_ms": torch_net_ms,
            "torch_net_share_of_torch_step": torch_net_ms / mean(step_ms["torch"]),
            "tc_net_fwd_bwd_ms": tc_net_ms,
            "tc_kernels_ms_per_step": kernels,
        })
    out["gpu_after"] = gpu_facts()
    text = json.dumps(out, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
