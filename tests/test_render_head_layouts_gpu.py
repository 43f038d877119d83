"""The render kernels with a fixed head layout (hr_render_kernel.cuh: HeadsZPlane, HeadsSphere) against the generic kernel.

The fixed layouts only state at compile time what the config already says, so each must render exactly what the generic
kernel rendered for the same config: every case renders seeded heads through hr_render_heads (the render kernel alone) and
compares the rgb bit for bit with tests/golden/render_head_layouts.npz, written by the generic kernels before the fixed
layouts existed (`python -m tests.test_render_head_layouts_gpu --write PATH`).  One case per layout and kernel shape (one or
two samples per lane, one or two rays per warp) and one that takes the generic kernel; the kernel that ran is read from the
profiler.
"""
import os
import sys

import numpy as np
import pytest
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "render_head_layouts.npz")
N_RAYS = 3000  # not a multiple of the rays per CTA: the last warp's second ray is missing at two rays per warp

# name: (builtin, overrides, head layout the dispatch picks, or None for the generic kernel)
CASES = {
    "zplane_s32": ("technicolor_z_plane", dict(n_voxels=2000000), "HeadsZPlane"),
    "zplane_s16": ("technicolor_z_plane", dict(n_voxels=2000000, z_channels=16), "HeadsZPlane"),
    "zplane_s64": ("neural_3d_z_plane", dict(n_voxels=2000000), "HeadsZPlane"),
    "sphere_s32": ("donerf_sphere", dict(n_voxels=2000000), "HeadsSphere"),
    "sphere_s16": ("donerf_sphere", dict(n_voxels=2000000, z_channels=16), "HeadsSphere"),
    "static_zplane_generic": ("shiny_z_plane_tiny", dict(n_voxels=2000000), None),
}


def render_case(name):
    """rgb of the render kernel on seeded heads, and the names of the CUDA kernels that ran."""
    import hyperreel_b200 as hb
    from hyperreel_b200.state import seeded_state_dict

    builtin, over, _ = CASES[name]
    cfg, ds = hb.configs.get(builtin, **over)
    sig = hb.lower(cfg, ds)
    model = hb.LightfieldModel(cfg, dataset=ds)
    render = hb.RenderLightfield(model, None, cfg.render)
    render.load_state_dict(seeded_state_dict(sig, seed=3, density_gain=30.0), strict=False)
    render.eval()
    rays = hb.rays.for_signature(sig, N_RAYS, seed=7).cuda()
    g = torch.Generator().manual_seed(17)
    heads = (0.5 * torch.randn((N_RAYS, sig.cfg.mlp_out), generator=g)).cuda()
    model._ensure_uploaded(rays.device)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        rgb = model._render_heads(rays, heads, True, False)
        torch.cuda.synchronize()
    names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
    return rgb.cpu(), names


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_fixed_head_layout_renders_what_the_generic_kernel_rendered(name):
    want = torch.from_numpy(np.load(GOLDEN)[name])
    rgb, names = render_case(name)
    assert float(rgb.abs().sum()) > 0.0, "the case renders black: it would not tell the layouts apart"
    assert torch.equal(rgb, want), f"{name}: max |rgb - generic| = {float((rgb - want).abs().max()):.3e}"
    layout = CASES[name][2]
    ran = [n for n in names if "render_kernel" in n]
    assert ran, sorted(names)
    for lay in ("HeadsZPlane", "HeadsSphere"):
        assert all((lay in n) == (lay == layout) for n in ran), (layout, ran)


if __name__ == "__main__":
    if len(sys.argv) != 3 or sys.argv[1] != "--write":
        raise SystemExit("usage: python -m tests.test_render_head_layouts_gpu --write PATH")
    out = {}
    for name in CASES:
        rgb, _ = render_case(name)
        out[name] = rgb.numpy()
        print(name, tuple(rgb.shape), "mean", float(rgb.mean()), "nonzero", int((rgb != 0).sum()))
    os.makedirs(os.path.dirname(os.path.abspath(sys.argv[2])), exist_ok=True)
    np.savez(sys.argv[2], **out)
