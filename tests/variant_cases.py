"""The render and render-backward kernel variants the host dispatch can reach, restated from the C++ dispatch, and one seeded case
per variant, built by editing built-in or shipped configs.

The render forward and backward are template families: the host picks one instantiation per call.  `forward_cell` and
`backward_cell` restate that choice from a lowered hr_config; tests/test_variant_cases.py checks without a GPU that the cases
below reach every cell of `CELLS` (or that a cell is refused the way `REFUSALS` says) and pass their guards, and
tests/test_kernel_variants_gpu.py runs every case against the fp64 oracle and reads the kernel that actually ran from the
profiler, so that the restatement cannot drift from the binary.
"""
from __future__ import annotations

import contextlib
import copy
import json
import os
from dataclasses import dataclass
from functools import lru_cache
from typing import Optional, Tuple

import numpy as np
import torch

import hyperreel_b200 as hb
from hyperreel_b200 import configs, lib as L, rays as rays_mod
from hyperreel_b200.config import to_plain
from hyperreel_b200.signature import UnsupportedPipeline, lower
from oracle.hyperreel_oracle import HyperReelOracle
from tests.cases import Case
from tests.ease_cases import ITERS_PER_EPOCH, eased_oracle
from tests.sweep_cases import Z_GAINS as SWEEP_Z_GAINS, scaled_heads_state

EASE_ITER = 6000  # both eased density heads of the built-ins mid-window (tests/ease_cases.py)
N_RAYS = 2 * 128 + 37  # two ray tiles and a ragged one; an odd count leaves the last warp of a two-ray kernel half empty
# the eased density heads (at least half the start value 1.0 mid-window) scale the z heads' moves by 1 - sigma: larger gains
Z_GAINS = tuple(SWEEP_Z_GAINS) + (64.0, 128.0)
RAY_SEEDS = tuple(range(0, 40000, 5000))
DENSITY_GAINS = (100.0, 600.0, 3000.0)  # then the next: sparser layouts and the transparent shipped planes need more density
SHIPPED_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "shipped")

LAYOUTS = ((8, 0, 0), (8, 4, 4), (8, 8, 8))  # launch_comps / bwd_launch_comps (hr_render_kernel.cuh, hr_render_bwd_kernel.cuh)
SHADES = ("SH", "RGB")
# the forward's sample-count edges: two rays per warp (S <= 16), one (S <= 32), 2 samples per lane (S <= 64), then the
# hr_render_big.cu kernels with 4 (S <= 128) and 8 (S <= 256)
EDGES = ("rpw2", "spl1", "spl2", "big4", "big8")
EDGE_RANGE = {"rpw2": (1, 16), "spl1": (17, 32), "spl2": (33, 64), "big4": (65, 128), "big8": (129, 256)}
# counts each edge cycles through: both ends of the range and counts that are not a multiple of 4
EDGE_S = {"rpw2": (13, 16, 10, 15), "spl1": (17, 32, 23, 30), "spl2": (33, 64, 47, 50), "big4": (65, 128, 99, 110),
          "big8": (129, 256, 201, 170)}


# ---------------------------------------------------------------- the dispatch, restated
@dataclass(frozen=True)
class Cell:
    """One instantiation of render_kernel<SPL, DYN, C0, C1, C2, SHADE, EXTRA, RPW, RARE, EASE> (kind "fwd") or of
    render_bwd_kernel<SPL, DYN, C0, C1, C2, SHADE, RARE, EASE> (kind "bwd").  family: "lean", "rare", "ease" or (forward,
    more than 64 samples) "big", which is compiled with RARE."""
    kind: str
    family: str
    spl: int
    dyn: bool
    layout: Tuple[int, int, int]
    shade: str
    extra: bool = False
    rpw: int = 1

    def template(self):
        """The kernel's template arguments, in the order of its demangled name."""
        shade = L.SHADE_SH if self.shade == "SH" else L.SHADE_RGB
        rare, ease = self.family != "lean", self.family == "ease"
        if self.kind == "fwd":
            return (self.spl, self.dyn, *self.layout, shade, self.extra, self.rpw, rare, ease)
        return (self.spl, self.dyn, *self.layout, shade, rare, ease)

    def __str__(self):
        tail = f"-{'extra' if self.extra else 'plain'}-rpw{self.rpw}" if self.kind == "fwd" else ""
        return (f"{self.kind}-{self.family}-spl{self.spl}-{'dyn' if self.dyn else 'static'}-{''.join(map(str, self.layout))}-"
                f"{self.shade}{tail}")


def eases_density(c) -> bool:
    """hr_common.cuh: eases_density."""
    return bool(c.act_sigma.eased or c.act_point_sigma.eased)


def needs_rare(c) -> bool:
    """hr_render_kernel.cuh: needs_rare -- primitives other than z-plane, sphere and cylinder, or the colour transform."""
    return c.isect_type not in (L.ISECT_Z_PLANE, L.ISECT_SPHERE, L.ISECT_CYLINDER) or c.n_color_views > 0


def needs_rare_bwd(c) -> bool:
    """hr_render_bwd_kernel.cuh: needs_rare_bwd -- voxel grid, deformable planes, bbox / z_depth (affine) contraction,
    per-ray colour heads, the colour transform."""
    return (c.isect_type in (L.ISECT_VOXEL, L.ISECT_PLANE) or c.contract_type == L.CONTRACT_AFFINE
            or c.off_cscale_global >= 0 or c.n_color_views > 0)


def _layout(c):
    lay = tuple(int(v) for v in c.n_sigma)
    if lay not in LAYOUTS:  # launch_comps / bwd_launch_comps return cudaErrorInvalidValue
        raise ValueError(f"component layout {lay} has no kernel")
    return lay


def forward_cell(c, extra: bool) -> Cell:
    """The render_kernel instantiation launch_render (hr_render.cu) runs for hr_config `c`; `extra`: render_stages' extra
    outputs (launch_one's `so`)."""
    S = c.n_samples
    if eases_density(c):
        if S > 64:  # hr_create / hr_set_activations refuse it (hr_api.cu: validate)
            raise ValueError("eased density heads above 64 samples per ray are not supported")
        fam, spl = "ease", (2 if S > 32 else 1)              # hr_render_ease.cu
    elif S > 64:
        fam, spl = "big", (8 if S > 128 else 4)              # hr_render_big.cu
    else:
        fam, spl = ("rare" if needs_rare(c) else "lean"), (2 if S > 32 else 1)  # hr_render_rare.cu / hr_render.cu
    # launch_one: two rays per warp with one sample per lane, S <= 16, no extra outputs and at most 5 destination buffers
    # (every render of these tests writes one)
    rpw = 2 if spl == 1 and S <= 16 and not extra else 1
    return Cell("fwd", fam, spl, bool(c.dynamic), _layout(c), "SH" if c.shading == L.SHADE_SH else "RGB", extra, rpw)


def backward_cell(c) -> Cell:
    """The render_bwd_kernel instantiation launch_render_bwd (hr_render_bwd.cu) runs for hr_config `c`."""
    if c.isect_type == L.ISECT_SPHERE_NEW:  # hr_api.cu: train_supported
        raise ValueError("backward: the sphere_new primitive is not supported yet")
    if c.n_samples > 64:
        raise ValueError("backward: more than 64 samples per ray are not supported yet")
    fam = "ease" if eases_density(c) else ("rare" if needs_rare_bwd(c) else "lean")
    return Cell("bwd", fam, 2 if c.n_samples > 32 else 1, bool(c.dynamic), _layout(c),
                "SH" if c.shading == L.SHADE_SH else "RGB")


def _grid():
    out = []
    for dyn in (True, False):
        for lay in LAYOUTS:
            for sh in SHADES:
                for fam in ("lean", "rare", "ease"):
                    out += [Cell("fwd", fam, 1, dyn, lay, sh, False, 2), Cell("fwd", fam, 1, dyn, lay, sh, False, 1),
                            Cell("fwd", fam, 2, dyn, lay, sh, False, 1)]
                    out += [Cell("fwd", fam, spl, dyn, lay, sh, True, 1) for spl in (1, 2)]
                    out += [Cell("bwd", fam, spl, dyn, lay, sh) for spl in (1, 2)]
                out += [Cell("fwd", "big", spl, dyn, lay, sh, extra, 1) for spl in (4, 8) for extra in (False, True)]
    return out


CELLS = _grid()


# ---------------------------------------------------------------- cases
@dataclass(frozen=True)
class Spec:
    """A case: `src` (a built-in of hyperreel_b200/configs.py, or "shipped:<name>" of tests/golden/shipped) with `variants`
    (configs._apply_variant), S samples, the VM layout (n_lamb_sigma = n_lamb_sh) and shading, and with `eased` its density
    heads eased at EASE_ITER.  `fwd` is the plain render's cell, `bwd` the backward's (None: refused, see REFUSALS)."""
    src: str
    variants: Tuple[str, ...]
    S: int
    layout: Tuple[int, int, int]
    shade: str
    eased: bool
    prim: str
    fwd: Cell
    bwd: Optional[Cell]

    @property
    def name(self):
        v = "+".join((self.src.split(":")[-1],) + self.variants)
        return (f"{v}-s{self.S}-{''.join(map(str, self.layout))}-{self.shade}" + ("-eased" if self.eased else ""))


# Bases, by the primitive or feature a case exercises.  RARE forward primitives: sphere_new, distance, voxel grid, deformable
# planes, colour transform.  RARE backward features: voxel grid, deformable planes, affine (bbox / z_depth) contraction,
# per-ray colour heads, colour transform.  The voxel grid, deformable planes and colour transform exist in static shipped
# configs only.
PRIMS = {
    # name: dynamic base, static base (src, variants); None where no config reaches it
    "z_plane": (("technicolor_z_plane", ()), ("shiny_z_plane_tiny", ())),
    "z_plane_mipnerf": (("neural_3d_z_plane", ()), ("shipped:llff_z_plane", ())),
    "sphere": (("neural_3d_z_plane", ("sphere", "outward_facing")), ("donerf_sphere", ())),
    "cylinder": (("neural_3d_z_plane", ("sphere", "cylinder", "outward_facing")), ("donerf_sphere", ("cylinder", "outward_facing"))),
    "sphere_new": (("neural_3d_z_plane", ("sphere_new", "outward_facing")), ("donerf_sphere", ("sphere_new",))),
    "distance": (("neural_3d_z_plane", ("sphere", "distance")), ("donerf_sphere", ("distance",))),
    "voxel": (None, ("shipped:donerf_voxel", ())),
    "plane": (None, ("shipped:shiny_z_deformable", ())),
    "color_transform": (None, ("shipped:immersive_z_plane", ())),
    # the dynamic built-ins' samples contracted into technicolor_z_plane_world's bbox all lie inside their colour nets'
    # AABBs, which would leave the AABB test unexercised: bbox is taken on the static base only
    "bbox": (None, ("shiny_z_plane_tiny", ("bbox",))),
    "z_depth": (("technicolor_z_plane", ("z_depth",)), ("shiny_z_plane_tiny", ("z_depth",))),
    "global_color": (("technicolor_z_plane", ("global_color",)), ("donerf_sphere", ("global_color",))),
}
LEAN_PRIMS = ("z_plane", "sphere", "z_plane_mipnerf", "cylinder")                    # lean forward and backward
LEAN_FWD_RARE_BWD = ("bbox", "z_depth", "global_color")                            # lean forward, RARE backward
RARE_PRIMS = ("sphere_new", "distance", "voxel", "plane", "color_transform")       # RARE forward
RARE_BWD = ("voxel", "plane", "bbox", "global_color", "color_transform", "z_depth")  # RARE backward
FLIPPED = {"immersive_z_plane"}  # rays start at z = 0 looking along -z, through the world-space planes (tests/cases_train.py)


def _fit(prim, S, edge):
    """S moved to the nearest count the primitive admits inside the edge: the voxel grid needs a multiple of its 3 axes."""
    if prim != "voxel":
        return S
    lo, hi = EDGE_RANGE[edge]
    return min((s for s in range(max(lo, 3), hi + 1) if s % 3 == 0), key=lambda s: (abs(s - S), s))


def _edge_spl(edge):
    return {"rpw2": 1, "spl1": 1, "spl2": 2, "big4": 4, "big8": 8}[edge]


def _spec(prim, dyn, edge, i, lay, sh, eased):
    base = PRIMS[prim][0 if dyn else 1]
    assert base is not None, (prim, dyn)
    S = _fit(prim, EDGE_S[edge][i % 4], edge)
    fam = "ease" if eased else ("big" if edge.startswith("big") else ("rare" if prim in RARE_PRIMS else "lean"))
    fwd = Cell("fwd", fam, _edge_spl(edge), dyn, lay, sh, False, 2 if edge == "rpw2" else 1)
    bwd = None
    if S <= 64 and prim != "sphere_new":
        bfam = "ease" if eased else ("rare" if prim in RARE_BWD else "lean")
        bwd = Cell("bwd", bfam, 2 if S > 32 else 1, dyn, lay, sh)
    return Spec(base[0], base[1], S, lay, sh, eased, prim, fwd, bwd)


def _specs():
    specs = []
    combos = [(dyn, lay, sh) for dyn in (True, False) for lay in LAYOUTS for sh in SHADES]
    # one case per plain forward cell; the primitive cycles so that lean forward cases alternate between a lean and a RARE
    # backward, and the RARE and BIG cases walk through every primitive
    for e, edge in enumerate(EDGES):
        for i, (dyn, lay, sh) in enumerate(combos):
            k = i + e
            if edge.startswith("big"):
                pool = RARE_PRIMS + LEAN_PRIMS if not dyn else ("sphere_new", "distance", "z_plane", "sphere")
                specs.append(_spec(pool[k % len(pool)], dyn, edge, k, lay, sh, False))
                continue
            rare_bwd = tuple(p for p in LEAN_FWD_RARE_BWD if PRIMS[p][0 if dyn else 1])
            lean = (LEAN_PRIMS[k // 2 % len(LEAN_PRIMS)] if k % 2 == 0 else rare_bwd[k // 2 % len(rare_bwd)])
            specs.append(_spec(lean, dyn, edge, k, lay, sh, False))
            rare = RARE_PRIMS if not dyn else ("sphere_new", "distance")
            specs.append(_spec(rare[k % len(rare)], dyn, edge, k + 1, lay, sh, False))
            eprims = ("z_plane", "sphere", "distance", "z_plane_mipnerf", "cylinder") if dyn else \
                ("z_plane", "voxel", "sphere", "z_plane_mipnerf", "distance", "cylinder")
            specs.append(_spec(eprims[k % len(eprims)], dyn, edge, k + 3, lay, sh, True))
    # backward cells no forward case above reaches
    have = {s.bwd for s in specs}
    for dyn, lay, sh in combos:
        for spl, edge in ((1, "spl1"), (2, "spl2")):
            for j, fam in enumerate(("lean", "rare")):
                if Cell("bwd", fam, spl, dyn, lay, sh) in have:
                    continue
                pool = LEAN_PRIMS if fam == "lean" else tuple(p for p in RARE_BWD if PRIMS[p][0 if dyn else 1])
                specs.append(_spec(pool[(len(specs) + j) % len(pool)], dyn, edge, len(specs), lay, sh, False))
    # the pairwise cover: every RARE forward primitive at every edge of the forward, every RARE backward feature at both
    # samples-per-lane counts of the backward
    for p in RARE_PRIMS:
        for edge in EDGES:
            if not any(s.prim == p and s.fwd.family in ("rare", "big") and _edge_of(s) == edge for s in specs):
                specs.append(_spec(p, PRIMS[p][0] is not None and len(specs) % 2 == 0, edge, len(specs), LAYOUTS[len(specs) % 3],
                                   SHADES[len(specs) % 2], False))
    for p in RARE_BWD:
        for edge in ("spl1", "spl2"):
            if not any(s.prim == p and s.bwd is not None and s.bwd.family == "rare" and s.bwd.spl == _edge_spl(edge)
                       for s in specs):
                specs.append(_spec(p, False, edge, len(specs), LAYOUTS[len(specs) % 3], SHADES[len(specs) % 2], False))
    names = [s.name for s in specs]
    assert len(set(names)) == len(names), [n for n in names if names.count(n) > 1]
    return specs


def _edge_of(spec):
    S = spec.S
    return next(e for e in EDGES if EDGE_RANGE[e][0] <= S <= EDGE_RANGE[e][1])


SPECS = _specs()
BY_NAME = {s.name: s for s in SPECS}

# Cases the lowering or the native library refuses: (src, variants, S, eased, what is asked, the refusal's message).
REFUSALS = [
    ("technicolor_z_plane", (), 65, True, "forward", "with 65 samples per ray is not on the fused path"),
    ("technicolor_z_plane", (), 65, False, "backward", "more than 64 samples per ray"),
    ("neural_3d_z_plane", ("sphere_new", "outward_facing"), 32, False, "backward", "sphere_new primitive is not supported"),
]


# ---------------------------------------------------------------- building a case
def _load_shipped(name):
    g = np.load(os.path.join(SHIPPED_DIR, f"{name}.npz"))
    return json.loads(str(g["config_json"])), json.loads(str(g["dataset_json"]))


def variant_cfg(src, variants, S, layout=None, shade=None):
    """(model cfg, dataset) of `src` with `variants`, S samples, the VM layout and shading."""
    if src.startswith("shipped:"):
        plain, ds = _load_shipped(src.split(":", 1)[1])
        cfg = hb.to_cfg(plain)
        for e in cfg.embedding.embeddings.values():
            if "z_channels" in e:
                e.z_channels = S
        cfg.color.net.N_voxel_init = cfg.color.net.N_voxel_final = 32 ** 3
        for v in variants:
            configs._apply_variant(cfg, v)
    else:
        cfg, ds = configs.get(src, n_voxels=32 ** 3, z_channels=S, variant=list(variants))
        cfg = copy.deepcopy(cfg)
    net = cfg.color.net
    if layout is not None:
        net.n_lamb_sigma, net.n_lamb_sh = list(layout), list(layout)
    if shade is not None:
        net.shadingMode, net.data_dim_color = shade, (27 if shade == "SH" else 3)
    return cfg, ds


def lower_spec(src, variants, S, layout=None, shade=None, eased=False):
    cfg, ds = variant_cfg(src, variants, S, layout, shade)
    if eased:
        return lower(cfg, ds, cur_iter=EASE_ITER, iters_per_epoch=ITERS_PER_EPOCH, ease=True)
    return lower(cfg, ds)


def oracle_ctx(eased):
    return eased_oracle(EASE_ITER) if eased else contextlib.nullcontext()


def guard_stats(case, eased):
    """(rays whose sort keys are out of order, masked samples (t = 0), samples in front of the origin outside the AABB,
    fraction of rays with acc > 0.5) of the fp64 oracle."""
    st = {}
    with oracle_ctx(eased):
        HyperReelOracle(case.model_cfg_plain, case.dataset, case.state_dict, dtype=torch.float64).render(case.rays.double(), st)
    keys = st["unsorted_distances"]
    disorder = int((keys[:, 1:] < keys[:, :-1]).any(1).sum()) if keys.shape[1] > 1 else 0
    masked = int((keys == 0).sum())
    outside = int((~st["valid"] & (st["distances"] > 0)).sum())
    opaque = float((st["weights"].sum(-1) > 0.5).double().mean())
    return disorder, masked, outside, opaque


def guard_ok(stats):
    """Some rays need the sort network, some samples are masked, some lie outside the AABB, and at least a quarter of the
    rays are opaque."""
    disorder, masked, outside, opaque = stats
    return disorder > 0 and masked > 0 and outside > 0 and opaque >= 0.25


def _rays(sig, src, n, seed):
    rays = rays_mod.for_signature(sig, n, seed=seed)
    if src.split(":")[-1] in FLIPPED:
        rays[:, 2] = 0.0
        rays[:, 5] = -rays[:, 5]
    return rays


@lru_cache(maxsize=None)
def variant_case(name: str, n: int = N_RAYS) -> Case:
    """The case of spec `name` with n seeded rays and seeded parameters: the first ray seed, density gain and z gain
    (Z_GAINS) under which its guard holds (the last one if none does: the tests then fail on the guard)."""
    spec = BY_NAME[name]
    cfg, ds = variant_cfg(spec.src, spec.variants, spec.S, spec.layout, spec.shade)
    sig = lower_spec(spec.src, spec.variants, spec.S, spec.layout, spec.shade, spec.eased)
    seed = 900 + SPECS.index(spec)
    for ray_seed in RAY_SEEDS:
        rays = _rays(sig, spec.src, n, seed + ray_seed)
        for dg in DENSITY_GAINS:
            for g in Z_GAINS:
                sd = scaled_heads_state(sig, seed, g * max(spec.S, 8), density_gain=dg)
                case = Case(name=name, model_cfg=cfg, model_cfg_plain=to_plain(cfg), dataset=ds, sig=sig, rays=rays,
                            state_dict=sd, n_samples=spec.S)
                if guard_ok(guard_stats(case, spec.eased)):
                    return case
    return case


def with_rays(case, src, n, seed):
    """The case with n other rays of its layout."""
    return Case(name=case.name, model_cfg=case.model_cfg, model_cfg_plain=case.model_cfg_plain, dataset=case.dataset,
                sig=case.sig, rays=_rays(case.sig, src, n, seed), state_dict=case.state_dict, n_samples=case.n_samples)


__all__ = ["CELLS", "Cell", "EASE_ITER", "REFUSALS", "SPECS", "BY_NAME", "UnsupportedPipeline", "backward_cell",
           "forward_cell", "guard_ok", "guard_stats", "lower_spec", "variant_case", "variant_cfg", "with_rays"]
