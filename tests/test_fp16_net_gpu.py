"""mlp_mode="fp16" on the GPU: the wgmma fp16 sample net against CUDA autocast, the cascade against the fp64 emulation, the
render after the net unchanged, every entry point bit for bit against forward, and the shipped-YAML fixtures.

Against autocast at 127-129 rays, where cuBLAS's fp16 GEMMs give the same fp32 sums as the kernel, every head must be within
one fp16 ulp of autocast's and all but MIN_EQUAL_SAME_SUMS of them bit-equal: this is what catches a contract clause broken
in the kernel (a bias added unrounded, a LeakyReLU without its second rounding).  At one ray and at three waves cuBLAS runs
other kernels, whose sums round differently at some fp16 boundaries; there the heads are held to the propagated tolerance
of tests/fp16_net_oracle.py (one fp16 ulp of the value plus a wide margin for what earlier layers carry) and to a bit-equal
share set from measurement.  Each check prints how many heads are bit-equal and the largest difference in fp16 steps.
"""
import ctypes as C

import pytest
import torch

import hyperreel_b200 as hb
import oracle.hyperreel_oracle as oracle_mod
from hyperreel_b200 import lib as L
from oracle.hyperreel_oracle import HyperReelOracle
from tests.cases import build_case
from tests.fp16_net_oracle import autocast_stack, emulate_fp64, ulps_apart
from tests.sweep_cases import NET_SHAPES, net_case
from tests.test_grads_batch_gpu import TOL_RGB
from tests.test_shipped_yaml_golden import SHIPPED, load_fixture

pytestmark = pytest.mark.gpu
NAMES = [s[0] for s in NET_SHAPES]
MAX_WIDTH = 0.05  # largest admitted tolerance, as a fraction of the tensor's largest entry
# the ray counts at which cuBLAS sums like the kernel: measured on an H100 80GB HBM3 (700 W), every head of every shape is
# bit-equal to autocast's there
SAME_SUMS = (127, 128, 129)
MIN_EQUAL_SAME_SUMS = 0.999
# bit-equal share elsewhere, measured on the same card: at least 73.3 % at one ray (a depth-10 net), 97.8 % at three waves
MIN_EQUAL = {1: 0.70, "waves": 0.97}
# |rgb - reference golden| of the shipped-YAML fixtures with the fp16 net, measured on an H100 80GB HBM3 (700 W): at most
# 7.5e-5 on every ray but one, ray 86 of technicolor_z_plane_ff at 0.367 (the bf16x3 net: 2.5e-7), which the fp16 heads move
# across a discontinuity of the render (DESIGN.md 4.1.1)
GOLDEN_RGB_FP16 = 2e-4
GOLDEN_KNOWN_OUTLIERS = {("technicolor_z_plane_ff", 86): 0.37}


@pytest.fixture(autouse=True)
def fp32_accumulation():
    """cuBLAS may otherwise reduce fp16 GEMMs in fp16; the contract is fp32 accumulation."""
    old = torch.backends.cuda.matmul.allow_fp16_reduced_precision_reduction
    torch.backends.cuda.matmul.allow_fp16_reduced_precision_reduction = False
    yield
    torch.backends.cuda.matmul.allow_fp16_reduced_precision_reduction = old


def _model(case, mode="fp16"):
    model = hb.LightfieldModel(case.model_cfg, dataset=case.dataset, mlp_mode=mode)
    render = hb.RenderLightfield(model, None, case.model_cfg.render, net_chunk=1 << 20)
    _, unexpected = render.load_state_dict(case.state_dict, strict=False)
    assert not unexpected
    render = render.cuda()
    render.eval()
    return render


def _encoded(model, rays):
    """hr_encode_rays in the reference's feature order (as _torch_net feeds its Linear layers)."""
    c = model.sig.cfg
    enc = torch.empty((rays.shape[0], c.mlp_in), device=rays.device)
    model._ensure_uploaded(rays.device)
    L.check(model._lib.hr_encode_rays(model._handle, rays.data_ptr(), rays.shape[0], enc.data_ptr(),
                                      torch.cuda.current_stream().cuda_stream))
    perm = list(model.sig.in_perm)
    if perm != list(range(len(perm))):
        inv = torch.empty(len(perm), dtype=torch.long)
        inv[torch.tensor(perm)] = torch.arange(len(perm))
        enc = enc.index_select(1, inv.to(rays.device))
    return enc


def _check(label, got, ref, tol=None, min_equal=0.0):
    """got against ref: within one fp16 step everywhere (tol None), or within the per-entry tolerance tol; and at least
    min_equal of the heads bit-equal."""
    assert bool(torch.isfinite(ref).all()), f"{label}: the reference overflows fp16"
    assert torch.equal(got, got.half().float()), f"{label}: a head that is not an fp16 value"
    ulps = ulps_apart(got, ref)
    equal = float((ulps == 0).double().mean())
    if tol is None:
        print(f"\n[{label}] {equal:.4%} of heads bit-equal, largest difference {int(ulps.max())} fp16 steps")
        assert int(ulps.max()) <= 1, f"{label}: {int((ulps > 1).sum())} heads more than one fp16 step from the reference"
    else:
        diff = (got.double() - ref.double()).abs()
        scale = float(ref.abs().max())
        assert float(tol.max()) <= MAX_WIDTH * scale, f"{label}: the tolerance reaches {float(tol.max()) / scale:.3f} of max |ref|"
        print(f"\n[{label}] {equal:.4%} of heads bit-equal, largest difference {int(ulps.max())} fp16 steps, "
              f"{float((diff / tol).max()):.3f} of the tolerance")
        bad = diff > tol
        assert not bool(bad.any()), f"{label}: {int(bad.sum())} heads out of tolerance, worst {float((diff / tol).max()):.2f} of it"
    assert equal >= min_equal, f"{label}: {equal:.4%} of heads bit-equal, fewer than {min_equal:.1%}"


def _count(n):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return {"waves": 3 * 128 * sms + 77}.get(n, n)


@pytest.mark.parametrize("n", [1, 127, 128, 129, "waves"])
@pytest.mark.parametrize("name", NAMES)
def test_heads_equal_autocast(name, n):
    key, n = n, _count(n)
    case = net_case(name, n)
    c = case.sig.cfg
    render = _model(case)
    model = render.model
    rays = case.rays.cuda()
    heads = model.render_stages(rays)["mlp_out"]
    enc = _encoded(model, rays)
    params = [p.detach() for p in model._net_params()]
    ref, tol = autocast_stack(enc, params, c.mlp_skip, c.leaky_slope)
    if n in SAME_SUMS:
        _check(f"{name} n={n} vs autocast", heads, ref, min_equal=MIN_EQUAL_SAME_SUMS)
    else:
        _check(f"{name} n={n} vs autocast", heads, ref, tol, min_equal=MIN_EQUAL[key])
    if n in (129, 1):  # the fp64 emulation agrees with autocast under the same tolerance
        emu, etol = emulate_fp64(enc, params, c.mlp_skip, c.leaky_slope)
        _check(f"{name} n={n} emulation vs autocast", emu, ref, torch.maximum(tol, etol))


def test_cascade_against_the_fp64_emulation(monkeypatch):
    """technicolor_cascaded: both nets fp16.  The oracle's two nets are replaced by the emulation; its heads are the point
    net's outputs, fed by first-stage outputs that went through the same rounding."""
    path = next(p for p in SHIPPED if p.endswith("technicolor_cascaded.npz"))
    plain, cfg, ds, sig, sd, rays, _ = load_fixture(path)
    model = hb.LightfieldModel(cfg, dataset=ds, mlp_mode="fp16")
    render = hb.RenderLightfield(model, None, cfg.render)
    render.load_state_dict(sd, strict=False)
    render.cuda().eval()
    assert model.sig.cfg.mlp_mode == L.MLP_FP16_TC and model.sig.cfg.pre_mlp_mode == L.MLP_FP16_TC
    got = model.render_stages(rays.cuda())["mlp_out"].cpu()

    tols = []

    def mlp_fp16(sd_, prefix, n_layers, skips, x, slope=0.01):
        params = []
        for i in range(n_layers):
            key = f"{prefix}.layers.{i}" + ("" if i == n_layers - 1 else ".0")
            params += [sd_[key + ".weight"].double(), sd_[key + ".bias"].double()]
        out, tol = emulate_fp64(x.float(), params, skips[0] if skips else -1, slope)
        tols.append(tol)
        return out.to(x.dtype)

    monkeypatch.setattr(oracle_mod, "mlp_forward", mlp_fp16)
    stages = {}
    HyperReelOracle(plain, ds, sd, dtype=torch.float64).render(rays.clone().double(), stages)
    ref = stages["mlp_out"].float()
    assert len(tols) == 2 and got.shape == ref.shape
    # the point net's inputs come from first-stage heads that may differ by their tolerance: compare per head channel
    # against the channel's range, and the bit-equal share, rather than per entry
    ulps = ulps_apart(got, ref)
    rel = float(((got - ref).abs().amax(0) / ref.abs().amax(0).clamp_min(1e-6)).max())
    equal = float((ulps == 0).double().mean())
    print(f"\n[technicolor_cascaded] {equal:.4%} of heads bit-equal, largest difference {int(ulps.max())} fp16 steps, "
          f"{rel:.2e} of the channel range")
    assert equal >= 0.9 and rel <= 5e-3  # measured on H100: 93.8 % bit-equal, 1.1e-3 of the channel range


def test_render_after_the_net_is_unchanged():
    """forward's rgb is hr_render_heads of the heads the fp16 net wrote (within the render-heads tests' rgb tolerance)."""
    case = build_case("technicolor_trained", n=3000)
    render = _model(case)
    model = render.model
    c = model.sig.cfg
    rays = case.rays.cuda()
    with torch.no_grad():
        rgb = model(rays)["rgb"]
    heads = model.render_stages(rays)["mlp_out"]
    again = model._render_heads(rays, heads, True, bool(c.white_bg) and not c.black_bg)
    err = float((again - rgb).abs().max())
    print(f"\n[technicolor_trained] max |forward - hr_render_heads(fp16 heads)| = {err:.3e}")
    assert err <= TOL_RGB, err
    bf = _model(case, "bf16x3").model
    with torch.no_grad():
        assert not torch.equal(bf(rays)["rgb"], rgb)  # the mode reaches the pixels


W, H = 48, 30


def _cameras(n):
    from tests.test_video_gpu import _cameras as cams
    return cams(n)


@pytest.mark.parametrize("name", ["technicolor_trained", "donerf_s16"])  # dynamic (c_in 8), static (c_in 6)
def test_every_entry_point_gives_forward_pixels(name):
    render = _model(build_case(name))
    model = render.model
    cam = _cameras(1)[0]
    rays = hb.generate_rays(cam, c_in=model.sig.c_in)
    with torch.no_grad():
        rgb = model(rays)["rgb"]
        fields = model(rays, {"fields": ["weights"]})
    assert torch.equal(fields["rgb"], rgb)  # hr_render_fields
    pinned = rays.cpu().pin_memory()
    for chunk in (0, 1000):  # the whole-batch (zero-copy) path and the chunked pipeline of hr_render_host
        assert torch.equal(model.render_host(pinned, chunk=chunk).cuda(), rgb), chunk
    dst = torch.empty_like(rgb)
    model.render_scatter(rays, (C.c_void_p * 1)(dst.data_ptr()), 1, 0)
    assert torch.equal(dst, rgb)  # hr_render_scatter
    u8 = model.render_to8b(rays).reshape(H, W, 3)
    assert torch.equal(model.render_frame_to8b(cam).cuda(), u8)
    video = hb.render_video(render, [cam], [cam.time])
    assert torch.equal(video[0], u8)
    assert torch.equal(hb.render_embeddings(render, [cam], hb.to_cfg({"type": "embedding", "fields": {}}))["rgb"], video)
    bf = _model(build_case(name), "bf16x3").model
    assert not torch.equal(bf.render_to8b(rays).reshape(H, W, 3), u8) or not torch.equal(bf(rays)["rgb"], rgb)


@pytest.mark.parametrize("sub", [1000, 0])
@pytest.mark.parametrize("name", ["technicolor_trained", "donerf_s16"])
def test_video_and_scored_views_equal_the_per_frame_paths(name, sub):
    from tests.test_score_views_gpu import test_views_equal_the_per_view_path
    from tests.test_video_gpu import test_video_frames_equal_the_whole_frame_path

    test_video_frames_equal_the_whole_frame_path(name, "fp16", sub)
    test_views_equal_the_per_view_path(name, "fp16", sub)


def test_shipped_yaml_fixtures():
    """|rgb - reference golden| of every shipped-YAML fixture in fp16 mode, pinned from measurement: every ray within
    GOLDEN_RGB_FP16 but the known outliers, each within its own bound and printed beside the bf16x3 net's error on it."""
    worst, seen = {}, set()
    for path in SHIPPED:
        plain, cfg, ds, sig, sd, rays, rgb_ref = load_fixture(path)
        name = path.rsplit("/", 1)[-1][:-4]
        model = hb.LightfieldModel(cfg, dataset=ds, mlp_mode="fp16")
        render = hb.RenderLightfield(model, None, cfg.render)
        render.load_state_dict(sd, strict=False)
        render.cuda().eval()
        with torch.no_grad():
            rgb = render(rays.cuda())["rgb"].cpu()
        err = (rgb - rgb_ref).abs().amax(-1)
        for (fixture, i), bound in GOLDEN_KNOWN_OUTLIERS.items():
            if fixture == name:
                print(f"\n{name} ray {i}: |rgb - golden| = {float(err[i]):.4e} (bound {bound})")
                assert float(err[i]) <= bound, (name, i, float(err[i]))
                err[i] = 0.0
                seen.add((fixture, i))
        worst[name] = float(err.max())
        for i in (err > GOLDEN_RGB_FP16).nonzero().flatten().tolist():
            print(f"\n{name} ray {i}: |rgb - golden| = {float(err[i]):.3e}, more than {GOLDEN_RGB_FP16}")
    for k, v in sorted(worst.items(), key=lambda kv: -kv[1]):
        print(f"{k}: max |rgb - golden| over the other rays = {v:.3e}")
    assert seen == set(GOLDEN_KNOWN_OUTLIERS)
    assert max(worst.values()) <= GOLDEN_RGB_FP16, max(worst.items(), key=lambda kv: kv[1])
