"""The configurations of the sample-count sweep (tests/test_sample_counts_gpu.py) and of the sample-net shape cover
(tests/test_sample_net_shapes_gpu.py), built from the built-ins by editing their config, and the case guards that say what
each one exercises.  tests/test_sweep_cases.py lowers every one of them without a GPU and checks that together they reach
every edge listed here, so that an edit to a case list cannot silently drop one.
"""
from __future__ import annotations

import copy
from functools import lru_cache

import torch

from hyperreel_b200 import configs, rays as rays_mod
from hyperreel_b200.config import to_plain
from hyperreel_b200.signature import lower, tc_passes
from hyperreel_b200.state import seeded_state_dict
from oracle.hyperreel_oracle import HyperReelOracle
from tests.cases import Case

# ---------------------------------------------------------------- sample counts
# The render kernels' variants change at S = 16/17 (two rays per warp), 32/33 (1 -> 2 samples per lane), 64/65 (the
# hr_render_big.cu kernels, 4 per lane) and 128/129 (8 per lane); lanes past S are padded.  Odd counts and counts that are not
# a multiple of 4 give a head row (15 channels per sample) that is not a multiple of 4 wide.
SAMPLE_COUNTS = [1, 2, 3, 7, 8, 9, 15, 16, 17, 31, 32, 33, 47, 63, 64, 65, 100, 127, 128, 129, 200, 255, 256]
SWEEP_BUILTINS = ["technicolor_z_plane",  # dynamic, SH shading, one VM group
                  "neural_3d_z_plane",    # dynamic, [8, 4, 4] VM groups, mipnerf contraction
                  "donerf_sphere"]        # static, RGB, [8, 4, 4], sphere primitive
SWEEP_RAYS = 4 * 128 + 37                 # several 128-ray tiles and a ragged last one
BWD_MAX_SAMPLES = 64                      # hr_render_backward refuses more
# The z heads of a seeded net barely move the samples off their base planes, and the seeded sigma head (a sigmoid shifted
# by +4) multiplies them by 1 - sigma ~ 0.02.  The sweep lowers the sigma head's bias by SIGMA_SHIFT and scales the z heads'
# rows by the first gain of Z_GAINS (times S: the heads move a sample by multiples of the plane spacing) under which the case
# guards hold.
SIGMA_SHIFT = -8.0
Z_GAINS = [1.0, 2.0, 4.0, 8.0, 16.0, 32.0]
RAY_SEEDS = [500, 1500, 2500, 3500]  # then the next ray seed


def _last_layer_keys(sd, sig):
    L = sig.cfg.mlp_layers
    kw = next(k for k in sd if "embedding_model" in k and k.endswith(f"net.layers.{L - 1}.weight"))
    return kw, kw[: -len("weight")] + "bias"


def scaled_heads_state(sig, seed, z_gain, density_gain=100.0, app_gain=6.0):
    c = sig.cfg
    sd = seeded_state_dict(sig, seed=seed, density_gain=density_gain, app_gain=app_gain)
    kw, kb = _last_layer_keys(sd, sig)
    S = c.n_samples
    z_rows = torch.tensor([s * c.head_stride + c.off_z + j for s in range(S) for j in range(c.n_z)])
    w, b = sd[kw].clone(), sd[kb].clone()
    w[z_rows] *= z_gain
    b[z_rows] *= z_gain
    if c.off_sigma >= 0:
        b[torch.tensor([s * c.head_stride + c.off_sigma for s in range(S)])] += SIGMA_SHIFT
    sd[kw], sd[kb] = w, b
    return sd


def guard_stats(case):
    """(rays whose sort keys are out of order, masked samples (t = 0), samples in front of the origin outside the AABB,
    fraction of rays with acc > 0.5) of the fp64 oracle."""
    st = {}
    HyperReelOracle(case.model_cfg_plain, case.dataset, case.state_dict, dtype=torch.float64).render(case.rays.double(), st)
    keys = st["unsorted_distances"]
    disorder = int((keys[:, 1:] < keys[:, :-1]).any(1).sum()) if keys.shape[1] > 1 else 0
    masked = int((keys == 0).sum())
    outside = int((~st["valid"] & (st["distances"] > 0)).sum())
    opaque = float((st["weights"].sum(-1) > 0.5).double().mean())
    return disorder, masked, outside, opaque


def guard_ok(stats, S):
    """Some rays need the sort network (keys out of order), some samples are masked, some lie outside the AABB, and at least a
    quarter of the rays are opaque.  With one or two planes spread over the whole depth range the seeded heads cannot
    reorder them and the rays are mostly transparent: there, some sample must be masked or outside."""
    disorder, masked, outside, opaque = stats
    if S <= 2:
        return masked + outside > 0
    return disorder > 0 and masked > 0 and outside > 0 and opaque >= 0.25


@lru_cache(maxsize=None)
def sweep_case(builtin: str, S: int, n: int = SWEEP_RAYS) -> Case:
    """Built-in `builtin` at z_channels = S with seeded parameters and n seeded rays: the first (ray seed, z gain) of RAY_SEEDS x
    Z_GAINS under which the case guards hold (the last one if none does: the tests then fail on the guard)."""
    cfg, ds = configs.get(builtin, n_voxels=32 ** 3, z_channels=S)
    sig = lower(cfg, ds)
    for seed in RAY_SEEDS:
        rays = rays_mod.for_signature(sig, n, seed=seed + S)
        for g in Z_GAINS:
            sd = scaled_heads_state(sig, 600 + S, g * max(S, 8))
            case = Case(name=f"{builtin}_s{S}", model_cfg=cfg, model_cfg_plain=to_plain(cfg), dataset=ds, sig=sig, rays=rays,
                        state_dict=sd, n_samples=S)
            if guard_ok(guard_stats(case), S):
                return case
    return case


# ---------------------------------------------------------------- sample-net shapes
# A pairwise cover of hidden width x depth x skip x encoded-input width x last-layer width on the tensor-core net.
# mlp_in = 4 (1 + 2 n) + (1 + 2 m) for Technicolor's two-plane rays with n ray and m time PE bands (5, 9, 17, 33, 63, ...),
# 4 (1 + 2 n) for the static two-plane built-in (4, 12, ...); mlp_out = S x 15 channels for the built-in heads, S x 2 for
# z_vals + sigma alone.
# (name, builtin, W, depth, skip (None, or "L-2"), ray PE bands, time PE bands, S, heads: the built-in's ("all"), with the
# global colour heads ("global") or z_vals + sigma alone ("z_sigma"))
NET_SHAPES = [
    ("w256_d2_in5_out15", "technicolor_z_plane", 256, 2, None, 0, 0, 1, "all"),               # smallest net, mlp_out % 4 = 3
    ("w128_d3_skip1_in9_out30", "technicolor_z_plane", 128, 3, 1, 0, 2, 2, "all"),            # skip at 1 = L-2, % 4 = 2
    ("w256_d6_skip4_in17_out45", "technicolor_z_plane", 256, 6, "L-2", 1, 2, 3, "all"),       # % 4 = 1
    ("w256_d6_skip3_in31_out105", "technicolor_z_plane", 256, 6, 3, 3, 1, 7, "all"),          # one input chunk, full
    ("w128_d10_skip1_in33_out255", "technicolor_z_plane", 128, 10, 1, 3, 2, 17, "all"),       # two input chunks, past W
    ("w256_d10_skip8_in63_out240", "technicolor_z_plane", 256, 10, "L-2", 7, 1, 16, "all"),   # widest input, below W
    ("w128_d6_in4_out128", "shiny_z_plane_tiny", 128, 6, None, 0, None, 64, "z_sigma"),       # smallest input, = W
    ("w256_d3_skip1_in12_out256", "shiny_z_plane_tiny", 256, 3, 1, 1, None, 128, "z_sigma"),  # = W
    ("w128_d2_in20_out132", "shiny_z_plane_tiny", 128, 2, None, 2, None, 66, "z_sigma"),      # one 4-column group past a pass
    ("w256_d3_in28_out260", "shiny_z_plane_tiny", 256, 3, None, 3, None, 130, "z_sigma"),     # ... at W = 256
    ("w128_d6_skip3_in60_out192", "shiny_z_plane_tiny", 128, 6, 3, 7, None, 16, "all"),       # 60 inputs, mid skip
    ("w128_d10_skip8_in9_out3948", "technicolor_z_plane", 128, 10, "L-2", 0, 2, 188, "global"),  # 40 passes: the limit
]


def net_cfg(builtin, W, depth, skip, ray_bands, time_bands, S, heads):
    cfg, ds = configs.get(builtin, n_voxels=32 ** 3, z_channels=S)
    cfg = copy.deepcopy(cfg)
    pred = cfg.embedding.embeddings.ray_prediction_0
    pred.net.hidden_channels = W
    pred.net.depth = depth
    pred.net.skips = [] if skip is None else [depth - 2 if skip == "L-2" else skip]
    pred.params.ray.pe.n_freqs = ray_bands
    if time_bands is not None:
        pred.params.time.pe.n_freqs = time_bands
    if heads == "global":
        # per-ray global colour heads as well (read at sample 0): 21 channels per sample
        pred.outputs.color_scale_global = {"channels": 3, "activation": {"type": "identity"}}
        pred.outputs.color_shift_global = {"channels": 3, "activation": {"type": "identity"}}
    if heads == "z_sigma":
        # no point offset, no colour scale / shift: two channels per sample
        for k in ("point_sigma", "point_offset", "color_scale", "color_shift"):
            del pred.outputs[k]
        del cfg.embedding.embeddings["point_offset_0"]
    return cfg, ds


def net_case(name, n):
    spec = next(s for s in NET_SHAPES if s[0] == name)
    cfg, ds = net_cfg(*spec[1:])
    sig = lower(cfg, ds)
    sd = seeded_state_dict(sig, seed=700 + NET_SHAPES.index(spec), density_gain=30.0)
    return Case(name=name, model_cfg=cfg, model_cfg_plain=to_plain(cfg), dataset=ds, sig=sig,
                rays=rays_mod.for_signature(sig, n, seed=800 + n), state_dict=sd, n_samples=sig.n_samples)


def net_shape(sig):
    """The hr_config shape of the sample net of a lowered signature."""
    c = sig.cfg
    return dict(mlp_in=c.mlp_in, W=c.mlp_width, layers=c.mlp_layers, skip=c.mlp_skip, mlp_out=c.mlp_out,
                passes=tc_passes(c.mlp_width, c.mlp_layers, c.mlp_out))
