"""The pipelines added in round 2 beyond their rgb fixtures (tests/test_shipped_yaml_gpu.py): per-sample stages against the
oracle (itself pinned to the unmodified reference on exactly these YAMLs, tests/test_oracle_vs_reference.py), ragged and
tiny batches, chunk invariance -- for 96 / 128 / 256 samples per ray (4 and 8 samples per lane), the voxel-grid primitives,
the per-camera colour transform and the cascaded (point_prediction) pipelines.  These run the EXTRA variants of
hr_render_big.cu / hr_render_rare.cu, which the rgb fixtures do not."""
import os

import pytest
import torch

import hyperreel_b200 as hb
from oracle.hyperreel_oracle import HyperReelOracle
from tests.test_shipped_yaml_golden import SHIPPED, load_fixture

pytestmark = pytest.mark.gpu

NAMES = ["neural_3d_z_plane_static", "technicolor_z_plane_no_sample", "catacaustics_voxel", "donerf_voxel", "shiny_z_deformable",
         "immersive_z_plane", "shiny_z_plane_cascaded", "shiny_z_plane_feedback", "shiny_z_tensorf_cascaded", "technicolor_cascaded",
         "catacaustics_distance"]
BY_NAME = {os.path.basename(p)[:-4]: p for p in SHIPPED}


def _render(cfg, ds, sd, mode):
    model = hb.LightfieldModel(cfg, dataset=ds, mlp_mode=mode)
    render = hb.RenderLightfield(model, None, cfg.render, net_chunk=1 << 20)
    _, unexpected = render.load_state_dict(sd, strict=False)
    assert not unexpected
    render.eval()
    return render


@pytest.mark.parametrize("name", NAMES)
def test_stages_match_the_oracle(name):
    plain, cfg, ds, sig, sd, rays, rgb = load_fixture(BY_NAME[name])
    render = _render(cfg, ds, sd, "fp32")
    st = {k: v.cpu() for k, v in render.model.render_stages(rays.cuda()).items()}
    ref = {}
    want = HyperReelOracle(plain, ds, sd).render(rays.clone(), ref)
    n = rays.shape[0]
    assert float((st["rgb"] - want).abs().max()) <= 1e-4
    assert float((st["mlp_out"] - ref["mlp_out"]).abs().max()) <= 2e-5 * max(1.0, float(ref["mlp_out"].abs().max()))
    d = ref["distances"].reshape(n, -1)
    assert float((st["distances"] - d).abs().max()) <= 1e-5 * max(1.0, float(d.abs().max()))
    assert float((st["points"].reshape(n, -1) - ref["points"].reshape(n, -1)).abs().max()) <= 2e-5 * max(1.0, float(ref["points"].abs().max()))
    assert float((st["sigma"] - ref["sigma"]).abs().max()) <= 1e-4 * max(1.0, float(ref["sigma"].abs().max()))
    assert float((st["weights"] - ref["weights"]).abs().max()) <= 5e-5


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("mode", ["fp32", "auto"])
def test_ragged_batches_and_chunk_invariance(name, mode):
    plain, cfg, ds, sig, sd, rays, rgb = load_fixture(BY_NAME[name])
    render = _render(cfg, ds, sd, mode)
    dev = rays.cuda()
    full = render(dev)["rgb"]
    for m in (1, 33):
        part = render(dev[:m].contiguous())["rgb"]
        assert part.shape == (m, 3)
        assert torch.equal(part, full[:m]), (name, m)
    assert render(dev[:0])["rgb"].shape == (0, 3)
    # a batch larger than one tile wave of the tensor-core net (rows = rays x first-stage points for a cascade)
    big = dev.repeat(40, 1)[:3001].contiguous()
    out = render(big)["rgb"]
    assert torch.equal(out[: rays.shape[0]], full)
    assert torch.equal(out[rays.shape[0]: 2 * rays.shape[0]], full)
    # the host-buffer pipeline: zero-copy where the net and the buffers allow it, copies otherwise
    for pinned in (True, False):
        rays_host = big.cpu()
        rgb_host = torch.empty((big.shape[0], 3), dtype=torch.float32)
        if pinned:
            rays_host, rgb_host = rays_host.pin_memory(), rgb_host.pin_memory()
        render.model.render_host(rays_host, rgb_host)
        assert torch.equal(rgb_host, out.cpu()), (name, mode, pinned)


def test_embed_and_extra_fields_of_a_cascaded_pipeline():
    plain, cfg, ds, sig, sd, rays, rgb = load_fixture(BY_NAME["technicolor_cascaded"])
    render = _render(cfg, ds, sd, "fp32")
    orc = HyperReelOracle(plain, ds, sd)
    emb = render.embed(rays.cuda())
    want = orc.embed_fields(rays.clone())
    assert set(emb) == set(want)
    for k in want:
        assert float((emb[k].cpu() - want[k]).abs().max()) <= 2e-5 * max(1.0, float(want[k].abs().max())), k
    kw = {"fields": ["render_weights", "distances", "points"]}
    got = render(rays.cuda(), **kw)
    ref = orc.render_fields(rays.clone(), kw)
    for k in ("rgb", "render_weights", "distances", "points"):
        assert float((got[k].cpu() - ref[k]).abs().max()) <= 1e-4 * max(1.0, float(ref[k].abs().max())), k


def test_training_is_refused_for_the_render_only_pipelines():
    for name in ("technicolor_cascaded", "catacaustics_voxel", "neural_3d_z_plane_static"):
        plain, cfg, ds, sig, sd, rays, rgb = load_fixture(BY_NAME[name])
        render = _render(cfg, ds, sd, "fp32")
        render.train()
        with pytest.raises((RuntimeError, hb.UnsupportedPipeline)):
            out = render.model.render_differentiable(rays.cuda())
            out.sum().backward()
