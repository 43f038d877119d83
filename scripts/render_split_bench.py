#!/usr/bin/env python
"""Where the render kernel's time goes, at bench.py's shapes:

    python scripts/render_split_bench.py --rounds 3 --out out/render_split.json
    python scripts/render_split_bench.py --phase-clocks LIB   # a library built with -DHR_RENDER_PHASE_CLOCKS (--build-clocks DIR)
    python scripts/render_split_bench.py --sass               # no GPU: static SASS of the hot instantiation per phase

Timing: the render kernel alone, from the CUDA events the library records around it, averaged over --launches forward
steps with the L2 flushed before each, for bench.py's flagship workload and its two extra single-GPU workloads.  The card's
name, power limit and SM clocks are read in the same run.  --lib times another build of the library (same ABI).

Phase clocks: the measurement build records clock64() per warp at the phase boundaries of every ray (hr_render_kernel.cuh:
HR_PHASE_MARK) and sums them on the device; the script prints each phase's share and its cycles per warp-ray.  The
production build has none of it.

SASS: compiles hr_render.cu with -lineinfo into a temporary directory and counts the instructions of one render_kernel
instantiation per phase (attributed by source line; instructions of inlined helpers go to the phase of the kernel line before
them) and per opcode.
"""
import argparse
import collections
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
CSRC = os.path.join(ROOT, "hyperreel_b200", "csrc")
KERNEL_SRC = os.path.join(CSRC, "hr_render_kernel.cuh")

# bench.py's flagship workload and its two extra single-GPU workloads (rays per step), as in scripts/fp16_bench.py
WORKLOADS = {
    "technicolor_s32": ("technicolor_z_plane", dict(n_voxels=512000000), 65536),
    "donerf_sphere_s16": ("donerf_sphere", dict(n_voxels=216000000, z_channels=16), 640000),
    "neural3d_s64": ("neural_3d_z_plane", dict(n_voxels=262144000), 685464),
}
PHASES = ("heads load", "keyframe/view/intersect/sort/points/texels", "gather rounds", "composite/store")
# the flagship's instantiation: one sample per lane, dynamic, comps [8,0,0], SH, plain, one ray per warp, lean, not eased
HOT = "render_kernelILi1ELb1ELi8ELi0ELi0ELi0ELb0ELi1ELb0ELb0E"
OPS = ("SHFL", "MUFU", "FMUL", "FADD", "FFMA", "FSETP", "ISETP", "BRA", "LDG", "LDC", "STG")


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                         text=True, timeout=30).stdout.strip()
    return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))


def build_clocks(dest):
    """The library with -DHR_RENDER_PHASE_CLOCKS, built into `dest` (nothing in the tree changes)."""
    os.makedirs(dest, exist_ok=True)
    out = os.path.join(dest, "libhyperreel_b200.so")
    subprocess.run(["make", "-C", CSRC, "-j", str(min(8, os.cpu_count() or 1)), f"BUILD={os.path.join(dest, 'build')}",
                    f"OUT={out}", "EXTRA_NVFLAGS=-DHR_RENDER_PHASE_CLOCKS"], check=True, capture_output=True)
    return out


def time_render(hb, name, launches, flush, dev, clocks):
    import ctypes as C

    import torch
    from hyperreel_b200.state import seeded_state_dict

    builtin, over, n = WORKLOADS[name]
    cfg, ds = hb.configs.get(builtin, **over)
    sig = hb.lower(cfg, ds)
    model = hb.LightfieldModel(cfg, dataset=ds)
    render = hb.RenderLightfield(model, None, cfg.render, net_chunk=1 << 22)
    render.load_state_dict(seeded_state_dict(sig, seed=11, density_gain=30.0), strict=False)
    render.eval()
    rays = hb.rays.for_signature(sig, n, seed=5).to(dev)
    row = {"workload": name, "rays": n, "samples": int(sig.cfg.n_samples), "launches": launches}
    with torch.no_grad():
        for _ in range(5):
            render(rays)
        torch.cuda.synchronize()
        if clocks is not None:
            clocks(None, 1)  # clear what the warm-up recorded
        model.timing(True)
        for _ in range(launches):
            flush.zero_()  # evict L2 before each step
            render(rays)
        torch.cuda.synchronize()
        tm = model.timing_read()
        model.timing(False)
    row["render_kernel_ms"] = tm["render_ms"]
    row["sample_net_ms"] = tm["mlp_ms"]
    if clocks is not None:
        buf = (C.c_ulonglong * (len(PHASES) + 1))()
        if clocks(buf, 1) != 0:
            raise RuntimeError("hr_render_phase_clocks failed")
        tot = sum(buf[i] for i in range(len(PHASES)))
        warp_rays = max(1, buf[len(PHASES)])
        row["phase_cycles_per_warp_ray"] = {p: buf[i] / warp_rays for i, p in enumerate(PHASES)}
        row["phase_share"] = {p: (buf[i] / tot if tot else 0.0) for i, p in enumerate(PHASES)}
        row["warp_rays"] = int(buf[len(PHASES)])
    return row


def phase_lines():
    """Kernel source lines of render_body, of its ray loop (what comes before it is per-warp set-up) and of each
    HR_PHASE_MARK(p)."""
    marks, start, body = {}, None, None
    with open(KERNEL_SRC) as f:
        for i, line in enumerate(f, 1):
            if start is None and re.search(r"void render_body\(", line):
                start = i
            if start is not None and body is None and re.search(r"for \(long long base = warp0", line):
                body = i
            m = re.search(r"^\s*HR_PHASE_MARK\((\d)\);", line)
            if m and body is not None:
                marks[int(m.group(1))] = i
    return start, body, [marks[p] for p in range(len(PHASES))]


def render_sass():
    """hr_render.cu compiled with -lineinfo, disassembled with source lines (nvdisasm -g)."""
    with tempfile.TemporaryDirectory() as tmp:
        cubin = os.path.join(tmp, "hr_render.cubin")
        subprocess.run(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
                        f"-I{os.path.join(ROOT, 'include')}", f"-I{CSRC}", "--expt-relaxed-constexpr", "-cubin", "-o", cubin,
                        os.path.join(CSRC, "hr_render.cu")], check=True, cwd=CSRC)
        return subprocess.run(["nvdisasm", "-g", cubin], check=True, capture_output=True, text=True).stdout


def sass_split(dis, kernel=HOT, fixed=None):
    """Static SASS of one render_kernel instantiation per phase and per opcode.  `fixed`: the head-layout type of the
    fixed-layout overload (e.g. "HeadsZPlane"), None for the generic kernel."""
    start, body, marks = phase_lines()
    # the fixed-layout overload has the layout's type as its last parameter
    tail = f"NS_{len(fixed)}{fixed}E" if fixed else "EPh"
    per_phase = collections.Counter()
    per_op = collections.Counter()
    per_phase_op = collections.defaultdict(collections.Counter)
    inside, phase, total = False, "setup", 0
    for line in dis.splitlines():
        if line.startswith(".text."):
            name = line[len(".text."):].rstrip(":")
            inside = kernel + "EEv" in name and name.endswith(tail)
            phase = "setup"
            continue
        if not inside:
            continue
        m = re.search(r'//## File "([^"]+)", line (\d+)', line)
        if m:
            if os.path.basename(m.group(1)) == "hr_render_kernel.cuh":
                ln = int(m.group(2))
                if ln < start:  # a helper defined above render_body: the phase of the kernel line before it
                    continue
                if ln < body:
                    phase = "setup"
                else:
                    phase = PHASES[0]
                    for p, mk in enumerate(marks):
                        if ln > mk:
                            phase = PHASES[min(p + 1, len(PHASES) - 1)]
            continue
        m = re.match(r"\s*/\*[0-9a-f]+\*/\s+(?:@!?U?P\w+\s+)?([A-Z0-9_]+)", line)
        if m:
            op = m.group(1).split(".")[0]
            total += 1
            per_phase[phase] += 1
            per_op[op] += 1
            per_phase_op[phase][op] += 1
    if total == 0:
        raise RuntimeError(f"no SASS found for {kernel} ({fixed or 'generic'})")
    return {"kernel": kernel, "layout": fixed or "HeadsAny", "total": total, "per_phase": dict(per_phase),
            "per_op": {k: per_op[k] for k in OPS},
            "per_phase_op": {p: {k: per_phase_op[p][k] for k in OPS} for p in per_phase_op}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--launches", type=int, default=100)
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--lib", default="", help="time this build of libhyperreel_b200.so instead of the in-tree one")
    ap.add_argument("--phase-clocks", default="", help="a library built with -DHR_RENDER_PHASE_CLOCKS")
    ap.add_argument("--build-clocks", default="", help="build that library into this directory, then exit")
    ap.add_argument("--sass", action="store_true", help="static SASS per phase of the hot instantiation (no GPU)")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if args.build_clocks:
        print(build_clocks(args.build_clocks))
        return
    if args.sass:
        dis = render_sass()
        rows = [sass_split(dis, HOT, None), sass_split(dis, HOT, "HeadsZPlane")]
        for r in rows:
            print(json.dumps(r))
        if args.out:
            os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
            with open(args.out, "w") as f:
                json.dump(rows, f, indent=1)
        return
    names = [w for w in args.workloads.split(",") if w]
    for w in names:
        if w not in WORKLOADS:
            ap.error(f"unknown workload {w!r} (known: {', '.join(WORKLOADS)})")

    import torch

    from hyperreel_b200 import lib as L

    lib_path = args.phase_clocks or args.lib
    if lib_path:
        L.LIB_PATH = os.path.abspath(lib_path)
    import hyperreel_b200 as hb

    if not torch.cuda.is_available():
        raise SystemExit("render_split_bench needs a GPU")
    clocks = None
    if args.phase_clocks:
        clocks = L.load_library().hr_render_phase_clocks  # AttributeError: not a phase-clock build
        clocks.restype = L.C.c_int
        clocks.argtypes = [L.C.c_void_p, L.C.c_int]
    dev = torch.device("cuda", 0)
    flush = torch.empty((512 << 20) // 4, dtype=torch.float32, device=dev)
    info = card()
    rows = []
    for r in range(args.rounds):
        for w in names:
            row = dict(round=r, lib=L.LIB_PATH, **time_render(hb, w, args.launches, flush, dev, clocks))
            rows.append(row)
            print(json.dumps(row), flush=True)
            torch.cuda.empty_cache()
    print("\nworkload             render kernel ms (per round)")
    for w in names:
        sel = [x for x in rows if x["workload"] == w]
        print(f"{w:20s} {' '.join(f'{x['render_kernel_ms']:.4f}' for x in sel)}")
        if clocks is not None:
            for p in PHASES:
                print(f"    {p:44s} share {' '.join(f'{x['phase_share'][p]:.3f}' for x in sel)}   "
                      f"cycles/warp-ray {' '.join(f'{x['phase_cycles_per_warp_ray'][p]:.0f}' for x in sel)}")
    print("card:", info)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"rows": rows, "card": info}, f, indent=1)


if __name__ == "__main__":
    main()
