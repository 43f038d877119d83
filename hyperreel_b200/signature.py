"""Recognise the pipeline a model config describes and lower it to the C-ABI ``hr_config``.

The reference builds an arbitrary graph from the YAML (ordered embeddings over a dict of named
per-sample fields, SURVEY.md section 2).  The fused CUDA path implements one family of graphs:

    ray_prediction -> ray_intersect -> [point_prediction -> ray_intersect] -> [color_transform] -> [advect_points]
                   -> [point_offset] -> add_point_outputs -> extract_fields
                   -> tensor_vm_split_time | tensor_vm_split_no_sample

with the primitives z_plane, sphere, cylinder, sphere_new, euclidean_distance_unified, voxel_grid, deformable_voxel_grid
(z_plane only in the first stage of a cascade), up to 256 samples per ray, `base` or `zero` sample nets.

Anything else raises ``UnsupportedPipeline`` at construction -- there is no fallback path.
Host-side constants are computed with the same torch ops the reference's constructors use
(``torch.linspace`` for the base primitives, nlf/intersect/z.py:50-71).
"""
from __future__ import annotations

import copy
import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional

import torch

from . import lib as L
from .config import Cfg, to_cfg


class UnsupportedPipeline(NotImplementedError):
    pass


def _get(cfg, key, default=None):
    return cfg[key] if (cfg is not None and key in cfg) else default


RENDER_ITER = 10_000_000  # what the reference sets when rendering (nlf/__init__.py:582-583)


@dataclass
class EaseSite:
    """One EaseValue (nlf/activations.py:462-496) that is the outermost activation of an ``hr_config`` member: the member's
    ``eased`` / ``ease_mul`` / ``ease_add`` follow from these three numbers and the iteration alone (``ease_terms``)."""
    field: str
    start_value: float
    wait_iters: float
    window_iters: float


# the hr_config members whose EaseValue the kernels blend (apply_act_eased): the density heads, the only open windows of the
# shipped model YAMLs
EASE_FIELDS = ("act_sigma", "act_point_sigma", "pre_act_sigma")


def check_eased(act: L.hr_act, member: str, n_samples: int) -> L.hr_act:
    """The eased activations the kernels serve: density heads only, at most 64 samples per ray (the render kernels' EASE
    variants exist for S <= 64 only)."""
    if act.eased and member not in EASE_FIELDS:
        raise UnsupportedPipeline(f"an open ease_value window on {member} is not on the fused path (only {', '.join(EASE_FIELDS)})")
    if act.eased and member != "pre_act_sigma" and n_samples > 64:
        raise UnsupportedPipeline(f"an open ease_value window with {n_samples} samples per ray is not on the fused path (<= 64)")
    return act


def ease_terms(cur_iter, start_value, wait_iters, window_iters):
    """EaseValue.set_iter + weight / ease_out (activations.py:473-496) at ``cur_iter``: None once the window has elapsed (the
    plain activation), else (w, (1 - w) * start_value) in double -- the Python scalars of ``w * out + (1 - w) * start_value``
    (``window_iters == 0``: w = 0, the start value alone)."""
    cur = cur_iter - wait_iters
    if cur >= window_iters:
        return None
    w = 0.0 if window_iters == 0 else min(max(float(cur) / window_iters, 0.0), 1.0)
    return w, (1 - w) * start_value


def set_ease(act: L.hr_act, terms) -> None:
    """Write ``ease_terms`` into an hr_act (each rounded once to fp32); None leaves the struct of the plain activation."""
    if terms is None:
        act.eased, act.ease_mul, act.ease_add = 0, 0.0, 0.0
    else:
        act.eased, act.ease_mul, act.ease_add = 1, float(terms[0]), float(terms[1])


def _resolve(cfg, cur_iter, ease):
    """-> (hr_act, (start_value, wait_iters, window_iters) of an outermost EaseValue or None)."""
    if cfg is None:
        cfg = {"type": "identity"}
    if isinstance(cfg, str):
        cfg = {"type": cfg}
    t = cfg["type"]
    if t == "ease_value":
        wait = _get(cfg, "wait_iters", 0.0)
        window = _get(cfg, "window_iters", 0.0)
        terms = ease_terms(cur_iter, 1.0, wait, window)
        if terms is not None and not ease:
            raise UnsupportedPipeline(f"ease_value window still open at iteration {cur_iter} (render-time config expected)")
        if not ease:
            return _resolve(cfg["activation"], cur_iter, False)
        inner = cfg["activation"]
        if isinstance(inner, dict) and inner.get("type") == "ease_value":
            # y * m + a covers one blend of a plain activation; an EaseValue inside another has no such form
            raise UnsupportedPipeline("an ease_value inside an ease_value is not on the fused path")
        act, _ = _resolve(inner, cur_iter, False)
        site = (float(_get(cfg, "start_value", 0.0)), wait, window)
        set_ease(act, ease_terms(cur_iter, *site))
        return act, site
    kinds = {"identity": L.ACT_IDENTITY, "sigmoid": L.ACT_SIGMOID, "tanh": L.ACT_TANH}
    if t not in kinds:
        raise UnsupportedPipeline(f"activation '{t}' is not on the fused path")
    outer = _get(cfg, "outer_fac", 1.0)
    if "fac" in cfg:
        outer = cfg["fac"]
    return L.hr_act(kinds[t], float(_get(cfg, "inner_fac", 1.0)), float(_get(cfg, "shift", 0.0)), float(outer)), None


def resolve_activation(cfg, cur_iter: int = RENDER_ITER, ease: bool = False) -> L.hr_act:
    """get_activation (nlf/activations.py:566-570) lowered to y = f(x*inner+shift)*outer.
    EaseValue (:462-496): once its window has elapsed it is its inner activation.  An open window raises, unless ``ease``:
    then it lowers to the eased form y * ease_mul + ease_add (hr_act.eased; an EaseValue must then be the outermost one)."""
    return _resolve(cfg, cur_iter, ease)[0]


# ---- mipnerf distance contraction on the host (nlf/contract.py:160-176), used for the base primitives ----
def _contract_distance(distance: torch.Tensor, start_distance: float, end_distance: float) -> torch.Tensor:
    distance = distance / start_distance
    inverse_distance = 1.0 / torch.abs(distance)
    inv_end = start_distance / end_distance
    scale = 1.0 / (1.0 - inv_end)
    t = (inverse_distance - inv_end) * scale
    distance = torch.where(torch.abs(distance) < 1.0, distance / 1.0, torch.sign(distance) * (2.0 - t))
    return (distance / 2.0) * 2.0


HEAD_ROLES = ("z_vals", "spatial_flow", "sigma", "point_sigma", "point_offset", "color_scale", "color_shift",
              "color_scale_global", "color_shift_global")


@dataclass
class Signature:
    """Everything the host needs to know about a recognised pipeline."""
    cfg: L.hr_config
    model_cfg: Cfg
    dataset: dict
    head_names: List[str] = field(default_factory=list)
    head_channels: List[int] = field(default_factory=list)
    mlp_layer_shapes: List[tuple] = field(default_factory=list)  # (out, in) per Linear
    dynamic: bool = False
    # kernel feature k of the encoded input = reference feature in_perm[k] (identity unless a group uses BasicPE, whose
    # [x | sin(d-major, f-minor) | cos(...)] order differs from WindowedPE's per-band order); applied to the input columns
    # of the first and the skip layer at upload
    in_perm: List[int] = field(default_factory=list)
    # ColorTransformEmbedding: rows of its `color_embedding` parameter (0 = no such embedding) and its position in the
    # `embeddings` ModuleList (state_dict name model.embedding_model.embeddings.{index}.color_embedding)
    color_views: int = 0
    color_embedding_index: int = -1
    # cascaded pipelines: `mlp_layer_shapes` / `in_perm` describe the point net, stored at embeddings.{net_index}.net; the
    # first-stage ray net (embeddings.0.net) has pre_layer_shapes ([] for a `zero` net) / pre_in_perm
    cascade: bool = False
    net_index: int = 0
    pre_layer_shapes: List[tuple] = field(default_factory=list)
    pre_in_perm: List[int] = field(default_factory=list)
    # lower(ease=True): every EaseValue site, to recompute the eased activations at another iteration without lowering again
    ease_sites: List[EaseSite] = field(default_factory=list)
    # every iteration threshold a gate of the graph compares against (embedding wait / stop, mask.stop_iters, PE windows):
    # iterations with the same position relative to all of them lower to the same graph
    graph_iters: List[float] = field(default_factory=list)

    def graph_key(self, cur_iter) -> tuple:
        import bisect

        return bisect.bisect_left(self.graph_iters, cur_iter), bisect.bisect_right(self.graph_iters, cur_iter)

    @property
    def c_in(self) -> int:
        return self.cfg.c_in

    @property
    def n_samples(self) -> int:
        return self.cfg.n_samples


def tc_passes(width: int, depth: int, n_out: int) -> int:
    """Passes of W output columns the tensor-core sample net runs (hr_mlp_tc2.cu): one per hidden layer, then the last layer's."""
    return depth - 1 + (n_out + width - 1) // width


def lower(model_cfg, dataset: dict, cur_iter: int = RENDER_ITER, iters_per_epoch: Optional[int] = None,
          mlp_mode: int = L.MLP_BF16X3_TC, ease: bool = False) -> Signature:
    """model cfg (reference schema) + dataset facts -> Signature / hr_config.  ``ease``: open EaseValue windows lower to
    their eased form (resolve_activation) instead of raising; Signature.ease_sites lists every EaseValue site."""
    from .config import epochs_to_iters

    sites: List[EaseSite] = []
    gates: List[float] = []

    def act_at(acfg, member):
        a, site = _resolve(acfg, cur_iter, ease)
        if site is not None:
            sites.append(EaseSite(member, *site))
        return check_eased(a, member, c.n_samples)

    m = to_cfg(copy.deepcopy(dict(model_cfg)))
    if iters_per_epoch is not None:
        epochs_to_iters(m, iters_per_epoch)
    else:
        epochs_to_iters(m, 1)  # render-time: any positive scale; windows are checked against cur_iter
    ds = dict(dataset)
    c = L.hr_config()
    c.abi_version = L.HR_ABI_VERSION
    c.mlp_mode = int(mlp_mode)

    if m.type != "lightfield" or m.render.type != "lightfield":
        raise UnsupportedPipeline("only model/render type 'lightfield'")
    if _get(m.param, "fn", "identity") != "identity":
        raise UnsupportedPipeline("top-level ray param must be identity")
    if "subdivision" in m and _get(m.subdivision, "type") is not None:
        raise UnsupportedPipeline("subdivision is not on the fused path")
    if m.embedding.type != "ray_point":
        raise UnsupportedPipeline("embedding type must be ray_point")

    embs = m.embedding.embeddings
    seq = []
    for key in embs.keys():
        e = embs[key]
        wait = _get(e, "wait_iters", 0)
        stop = _get(e, "stop_iters", float("inf"))
        gates.extend([float(wait), float(stop)])
        if cur_iter >= wait and cur_iter < stop:  # RayPointEmbedding.forward gate (embedding.py:107)
            seq.append(e)
    # ColorTransformEmbedding (point.py:558-612) only adds per-ray keys to the dict: it commutes with the point embeddings
    ctrans = next((e for e in seq if e.type == "color_transform"), None)
    ctrans_index = next((i for i, k in enumerate(embs.keys()) if embs[k].type == "color_transform"), -1)
    seq = [e for e in seq if e.type != "color_transform"]
    types = [e.type for e in seq]
    expect = ["ray_prediction", "ray_intersect"]
    # cascaded pipelines (PointPredictionEmbedding, point.py:39-219): a second net runs at the points of a first, coarse
    # intersection and predicts the primitives of the second one
    cascade = types[2:4] == ["point_prediction", "ray_intersect"]
    rest = types[4:] if cascade else types[2:]
    allowed_tail = [t for t in ("advect_points", "point_offset", "add_point_outputs", "extract_fields") if t in rest]
    if types[:2] != expect or rest != allowed_tail or "add_point_outputs" not in rest or "extract_fields" not in rest:
        raise UnsupportedPipeline(f"embedding sequence {types} is not a recognised pipeline")
    pred0, isect0 = seq[0], seq[1]
    # `pred` / `isect`: the prediction whose outputs are the heads the colour net's samples come from, and their intersection
    pred, isect = (seq[2], seq[3]) if cascade else (seq[0], seq[1])
    point_index = next((i for i, k in enumerate(embs.keys()) if embs[k] is pred), 0) if cascade else 0
    flow = next((e for e in seq if e.type == "advect_points"), None)
    offset = next((e for e in seq if e.type == "point_offset"), None)
    addp = next(e for e in seq if e.type == "add_point_outputs")
    extract = next(e for e in seq if e.type == "extract_fields")

    net = m.color.net
    if m.color.type != "base" or net.type not in ("tensor_vm_split_time", "tensor_vm_split_no_sample"):
        raise UnsupportedPipeline(f"colour net '{net.type}' is not on the fused path")
    dynamic = net.type == "tensor_vm_split_time"

    # ------------------------------------------------------------------ sample-net input (ray.py:235-263, point.py:69-100)
    def encode_groups(params):
        max_end = 6
        groups = []
        mlp_in = 0
        in_perm: List[int] = []
        for key in params.keys():
            p = params[key]
            g = L.hr_encode_group()
            g.start, g.end = int(p.start), int(p.end)
            max_end = max(max_end, g.end)
            fn = p.param.fn
            if fn == "identity":
                g.fn, dims = L.PARAM_IDENTITY, g.end - g.start
            elif fn == "two_plane":
                g.fn, dims = L.PARAM_TWO_PLANE, 4
                if any(k in p.param for k in ("origin", "use_local_param")) or g.end - g.start != 6:
                    raise UnsupportedPipeline("two_plane: origin/local param not supported")
            elif fn == "pluecker":
                g.fn, dims = L.PARAM_PLUECKER, 6
                if any(k in p.param for k in ("origin", "use_local_param")) or g.end - g.start != 6:
                    raise UnsupportedPipeline("pluecker: origin/local param not supported")
            else:
                raise UnsupportedPipeline(f"ray param '{fn}' is not on the fused path")
            if dims > 8:
                raise UnsupportedPipeline("param group wider than 8 channels")
            g.near, g.far = float(_get(p.param, "near", -1.0)), float(_get(p.param, "far", 0.0))
            g.dir_mult = float(_get(p.param, "direction_multiplier", 1.0))
            g.mom_mult = float(_get(p.param, "moment_multiplier", 1.0))
            pe = _get(p, "pe")
            g.n_freqs, g.exclude_identity, g.freq_mult, g.base_mult = 0, 0, 2.0, 1.0
            if pe is not None and pe.type == "basic":
                # BasicPE (pe.py:32-68): same values as a fully open WindowedPE, other column order (handled by in_perm)
                g.n_freqs = int(pe.n_freqs)
                g.freq_mult = float(_get(pe, "freq_multiplier", 2.0))
                D, Fq, k0 = dims, g.n_freqs, mlp_in
                for i in range(D):
                    in_perm.append(k0 + i)
                for f in range(Fq):
                    for i in range(D):
                        in_perm.append(k0 + D + i * Fq + f)            # sin(band f, dim i)
                    for i in range(D):
                        in_perm.append(k0 + D + D * Fq + i * Fq + f)   # cos(band f, dim i)
            elif pe is not None:
                if pe.type != "windowed":
                    raise UnsupportedPipeline(f"pe type '{pe.type}' is not on the fused path")
                # all windows must be open (pe.py:186-196): cur_iter past wait and past max_freq_iter
                mfi = float(_get(pe, "max_freq_iter", 0))
                if "window_iters" in pe:
                    mfi = max(max(w) for w in pe.window_iters)
                gates.extend([float(_get(pe, "wait_iters", 0)), float(mfi)])
                if (cur_iter - _get(pe, "wait_iters", 0)) < 0 or (mfi != 0 and not cur_iter > mfi):
                    raise UnsupportedPipeline("windowed PE not fully open at this iteration")
                if _get(pe, "ceil", False) or _get(pe, "window_identity", False):
                    pass  # irrelevant once every weight is 1
                g.n_freqs = int(pe.n_freqs)
                g.exclude_identity = int(bool(_get(pe, "exclude_identity", False)))
                g.freq_mult = float(_get(pe, "freq_multiplier", 2.0))
                g.base_mult = float(_get(pe, "base_multiplier", 1.0))
            if not (pe is not None and pe.type == "basic"):
                n_feat = dims * (2 * g.n_freqs + (0 if g.exclude_identity else 1))
                in_perm.extend(range(mlp_in, mlp_in + n_feat))
            mlp_in += dims * (2 * g.n_freqs + (0 if g.exclude_identity else 1))
            groups.append(g)
        if len(groups) > L.HR_MAX_GROUPS:
            raise UnsupportedPipeline("too many param groups")
        return groups, mlp_in, in_perm, max_end

    groups, mlp_in, in_perm, max_end = encode_groups(pred.params)
    c.n_groups = len(groups)
    for i, g in enumerate(groups):
        c.groups[i] = g
    pre_in_perm: List[int] = []
    if cascade:
        if max_end > 8:
            raise UnsupportedPipeline("point_prediction: param group reads beyond the 8-channel input row")
        groups0, mlp_in0, pre_in_perm, max_end = encode_groups(pred0.params)
        c.pre_n_groups, c.pre_mlp_in = len(groups0), mlp_in0
        for i, g in enumerate(groups0):
            c.pre_groups[i] = g
    c.c_in = 8 if (dynamic or flow is not None or max_end > 6) else 6
    if max_end > c.c_in:
        raise UnsupportedPipeline("param group reads beyond the ray")

    # ------------------------------------------------------------------ sample net (mlp.py:60-178)
    def net_shape(ncfg, n_in, n_out):
        """BaseMLP / ZeroMLP behind a prediction embedding -> (zero, width, depth, skip, [(out, in) per Linear])."""
        if ncfg.type not in ("base", "zero"):
            raise UnsupportedPipeline(f"sample net '{ncfg.type}' is not on the fused path")
        zero = ncfg.type == "zero"  # ZeroMLP (nlf/nets/mlp.py:14-33): every head is 0 before its activation
        if zero:
            return True, int(_get(ncfg, "hidden_channels", 0)), int(_get(ncfg, "depth", 0)), -1, []
        for k in ("pe", "latent_dim", "pad_to", "is_constant", "zero_before_channel", "pe_channels"):
            if k in ncfg:
                raise UnsupportedPipeline(f"sample net option '{k}' is not on the fused path")
        if _get(ncfg, "activation", "identity") != "identity" or _get(ncfg, "layer_activation", "leaky_relu") != "leaky_relu":
            raise UnsupportedPipeline("sample net activations must be leaky_relu / identity")
        if not _get(ncfg, "bias", True):
            raise UnsupportedPipeline("bias-free sample net")
        depth = int(ncfg.depth)  # Ray/PointPredictionEmbedding: depth -= 2, linear_last=False -> `depth` Linear layers
        skips = list(_get(ncfg, "skips", []))
        if len(skips) > 1:
            raise UnsupportedPipeline("more than one skip connection")
        W = int(ncfg.hidden_channels)
        if W not in (128, 256):
            raise UnsupportedPipeline(f"sample net hidden width {W} is not on the fused path (128 or 256)")
        if n_in > 64:
            raise UnsupportedPipeline(f"sample net input of {n_in} encoded features is not on the fused path (<= 64)")
        if not (2 <= depth <= L.HR_MAX_LAYERS):
            raise UnsupportedPipeline(f"sample net depth {depth} is not on the fused path")
        skip = int(skips[0]) if skips else -1
        shp = []
        for i in range(depth):
            fin = n_in if i == 0 else (W + n_in if i == skip else W)
            shp.append((n_out if i == depth - 1 else W, fin))
        return False, W, depth, skip, shp

    if cascade:
        # PointPredictionEmbedding (point.py:39-140): in_z_channels points per ray, out_z_channels samples per ray
        S, S0 = int(_get(pred, "out_z_channels", 1)), int(_get(pred, "in_z_channels", 1))
        if int(pred0.z_channels) != S0 or int(isect0.z_channels) != S0:
            raise UnsupportedPipeline("point_prediction: in_z_channels must equal the first stage's z_channels")
        if S0 < 1 or S0 > 32 or S % S0 != 0:
            raise UnsupportedPipeline(f"point_prediction: {S0} points per ray / {S} samples per ray is not on the fused path")
        for k in ("filter", "rays_name", "points_name"):
            if _get(pred, k, False) not in (False, "rays", "points"):
                raise UnsupportedPipeline(f"point_prediction option '{k}' is not on the fused path")
        if any(bool(_get(pred.outputs[k], "residual", False)) for k in pred.outputs.keys()):
            raise UnsupportedPipeline("point_prediction: residual outputs are not on the fused path")
    else:
        S = int(pred.z_channels)
    if int(isect.z_channels) != S:
        raise UnsupportedPipeline("z_channels mismatch between prediction and intersection")
    if "ray_outputs" in pred and len(pred.ray_outputs) > 0:
        raise UnsupportedPipeline("per-ray outputs are not on the fused path")
    head_names = list(pred.outputs.keys())
    head_channels = [int(pred.outputs[k].channels) for k in head_names]
    stride = sum(head_channels)
    c.mlp_out = S * stride
    c.leaky_slope = 0.01
    c.n_samples, c.head_stride = S, stride
    # the net's output row: all S samples of a ray, or the S / S0 samples one first-stage point expands to
    zero_net, W, depth, c.mlp_skip, shapes = net_shape(pred.net, mlp_in, (S // S0) * stride if cascade else c.mlp_out)
    if zero_net and cascade:
        raise UnsupportedPipeline("point_prediction with a zero net")
    if zero_net:
        c.mlp_mode = L.MLP_ZERO
    c.mlp_in, c.mlp_width, c.mlp_layers = mlp_in, W, depth
    if c.mlp_mode in (L.MLP_BF16X3_TC, L.MLP_FP16_TC) and tc_passes(W, depth, shapes[-1][0]) > L.HR_TC_MAX_PASSES:
        raise UnsupportedPipeline(f"tensor-core sample net of {tc_passes(W, depth, shapes[-1][0])} passes of {W} output columns "
                                  f"(more than HR_TC_MAX_PASSES = {L.HR_TC_MAX_PASSES}): use mlp_mode 'fp32'")

    # ------------------------------------------------------------------ heads (ray.py:331-337)
    offs: Dict[str, int] = {}
    o = 0
    for nme, ch in zip(head_names, head_channels):
        if nme not in HEAD_ROLES:
            raise UnsupportedPipeline(f"head '{nme}' is not on the fused path")
        offs[nme] = o
        o += ch
    expect_ch = {"spatial_flow": 3, "sigma": 1, "point_sigma": 1, "point_offset": 3, "color_scale": 3, "color_shift": 3,
                 "color_scale_global": 3, "color_shift_global": 3}
    for nme, ch in zip(head_names, head_channels):
        if nme in expect_ch and ch != expect_ch[nme]:
            raise UnsupportedPipeline(f"head '{nme}' must have {expect_ch[nme]} channels")

    def act_of(nme, member):
        return act_at(_get(pred.outputs[nme], "activation"), member) if nme in offs else L.hr_act(0, 1.0, 0.0, 1.0)

    c.off_z = offs.get("z_vals", -1)
    c.n_z = head_channels[head_names.index("z_vals")] if "z_vals" in offs else 0
    c.off_flow, c.off_sigma = offs.get("spatial_flow", -1), offs.get("sigma", -1)
    c.off_point_sigma, c.off_offset = offs.get("point_sigma", -1), offs.get("point_offset", -1)
    c.off_cscale, c.off_cshift = offs.get("color_scale", -1), offs.get("color_shift", -1)
    c.act_z, c.act_flow, c.act_sigma = act_of("z_vals", "act_z"), act_of("spatial_flow", "act_flow"), act_of("sigma", "act_sigma")
    c.act_point_sigma, c.act_offset = act_of("point_sigma", "act_point_sigma"), act_of("point_offset", "act_offset")
    c.act_cscale, c.act_cshift = act_of("color_scale", "act_cscale"), act_of("color_shift", "act_cshift")

    # ------------------------------------------------------------------ first stage of a cascade (ray net -> z-planes -> points)
    c.cascade, c.pre_samples = int(cascade), 0
    for k in range(8):
        c.pt_src[k] = L.PT_NONE
    pre_shapes: List[tuple] = []
    if cascade:
        c.pre_samples = S0
        names0 = list(pred0.outputs.keys())
        ch0 = [int(pred0.outputs[k].channels) for k in names0]
        if any(nme not in ("z_vals", "sigma") for nme in names0) or "z_vals" not in names0 or any(ch != 1 for ch in ch0):
            raise UnsupportedPipeline("first stage of a cascade: one-channel z_vals (and sigma) heads only")
        if "ray_outputs" in pred0 and len(pred0.ray_outputs) > 0:
            raise UnsupportedPipeline("per-ray outputs are not on the fused path")
        c.pre_head_stride = len(names0)
        c.pre_off_z, c.pre_off_sigma = names0.index("z_vals"), (names0.index("sigma") if "sigma" in names0 else -1)
        c.pre_act_z = act_at(_get(pred0.outputs["z_vals"], "activation"), "pre_act_z")
        c.pre_act_sigma = (act_at(_get(pred0.outputs["sigma"], "activation"), "pre_act_sigma") if "sigma" in names0
                           else L.hr_act(0, 1.0, 0.0, 1.0))
        zero0, c.pre_mlp_width, c.pre_mlp_layers, c.pre_mlp_skip, pre_shapes = net_shape(pred0.net, c.pre_mlp_in, S0 * c.pre_head_stride)
        c.pre_mlp_mode = L.MLP_ZERO if zero0 else int(mlp_mode)
        it0 = isect0.intersect
        if it0.type != "z_plane":
            raise UnsupportedPipeline(f"first stage of a cascade: intersect '{it0.type}' (z_plane only)")
        for k in ("origin", "weight_fn", "sort_outputs", "dropout", "use_disparity", "residual_z", "residual_distance", "normalize",
                  "clamp", "forward_facing", "contract", "z_scale", "num_samples_for_scale"):
            if k in it0 and it0[k] not in (False, None):
                raise UnsupportedPipeline(f"first stage of a cascade: intersect option '{k}' is not on the fused path")
        use_ds0 = bool(_get(it0, "use_dataset_bounds", False))
        if use_ds0:  # z.py:26-31
            lo0, hi0 = torch.tensor(-ds["near"]), torch.tensor(-ds["far"])
        else:
            lo0, hi0 = torch.tensor(_get(it0, "initial", 0.0)), torch.tensor(_get(it0, "end", 1.0))
        tab0 = torch.linspace(float(lo0.float()), float(hi0.float()), S0)
        for i in range(S0):
            c.pre_samples_tab[i] = float(tab0[i])
        c.pre_z_scale = float(torch.abs(tab0[1] - tab0[0])) if S0 > 1 else 1.0
        c.pre_near = float(_get(it0, "near", ds["near"] if use_ds0 else 0.0))
        c.pre_far = float(_get(it0, "far", float("inf")))
        if "mask" in it0 and it0.mask is not None:
            gates.append(float(_get(it0.mask, "stop_iters", float("inf"))))
        if "mask" in it0 and it0.mask is not None and cur_iter > float(_get(it0.mask, "stop_iters", float("inf"))):
            c.pre_near, c.pre_far = float("-inf"), float("inf")  # base.py:104-105,197-198
        c.pre_sort = int(bool(_get(it0, "sort", False)))
        c.pre_isect_act = act_at(_get(it0, "activation", "identity"), "pre_isect_act")
        c.pre_use_sigma = int(bool(_get(it0, "use_sigma", False)) and _get(it0, "in_density_field", "sigma") == "sigma"
                              and "sigma" in names0)
        # the point net's input row (point.py:151-160): the named tensors concatenated in YAML order
        src, k = {"points": L.PT_POINT, "viewdirs": L.PT_VIEW, "origins": L.PT_ORIGIN}, 0
        for nme in pred.inputs.keys():
            width = int(pred.inputs[nme])
            if nme == "times":
                chans = [L.PT_TIME]  # rays[..., -1:]: one channel whatever the configured width
            elif nme in src and 1 <= width <= 3:
                chans = [src[nme] + j for j in range(width)]
            else:
                raise UnsupportedPipeline(f"point_prediction input '{nme}' is not on the fused path")
            for ch in chans:
                if k >= 8:
                    raise UnsupportedPipeline("point_prediction: more than 8 input channels")
                c.pt_src[k] = ch
                k += 1
        if max(int(g.end) for g in groups) > k:
            raise UnsupportedPipeline("point_prediction: param group reads beyond its inputs")

    # ------------------------------------------------------------------ intersection (base.py:52-126, z.py, primitive.py)
    it = isect.intersect
    for k in ("origin", "weight_fn", "sort_outputs", "dropout", "num_repeat", "use_local_prediction", "flip_axes"):
        if k in it and it[k] not in (False, None, 1):
            raise UnsupportedPipeline(f"intersect option '{k}' is not on the fused path")
    # (`max_axis` is used by IntersectVoxelGrid only, voxel.py:41,100-110; the other classes ignore the key)
    for k in ("use_disparity", "residual_z", "residual_distance", "normalize", "clamp", "forward_facing"):
        if _get(it, k, False):
            raise UnsupportedPipeline(f"intersect option '{k}' is not on the fused path")
    # `outward_facing` is read by sphere_new / cylinder_new / voxel_grid only (primitive.py:262,447; voxel.py:24): the
    # primitives on the fused path ignore it, exactly like the reference classes they mirror
    if it.type not in ("z_plane", "sphere", "cylinder", "sphere_new", "euclidean_distance_unified", "voxel_grid",
                       "deformable_voxel_grid") and _get(it, "outward_facing", False):
        raise UnsupportedPipeline("intersect option 'outward_facing' is not on the fused path for this primitive")
    if _get(isect, "rays_name", "rays") != "rays":
        raise UnsupportedPipeline("rays_name override")
    use_ds = bool(_get(it, "use_dataset_bounds", False))
    contract = _get(it, "contract")
    c.contract_type, c.contract_samples = L.CONTRACT_NONE, 0
    c.contract_start_radius = c.contract_start_distance = 1.0
    c.contract_end_radius = c.contract_end_distance = float("inf")
    c.contract_dist_fac = 1.0
    for i in range(3):
        c.contract_affine_min[i], c.contract_affine_den[i] = 0.0, 1.0
    affine_fac = None
    if contract is not None and contract.type in ("bbox", "z_depth"):
        if "distance_activation" in contract or "stop_iters" in contract:
            raise UnsupportedPipeline("contract distance_activation / stop_iters")
        if contract.type == "bbox":  # BBoxContract (contract.py:65-84)
            bmin = torch.tensor([float(v) for v in _get(contract, "bbox_min", [-1.0, -1.0, -1.0])])
            bmax = torch.tensor([float(v) for v in _get(contract, "bbox_max", [1.0, 1.0, 1.0])])
            affine_fac = torch.mean(torch.abs(bmax - bmin))
            den = bmax - bmin
        else:  # ZDepthContract (contract.py:87-110)
            er = _get(contract, "contract_end_radius",
                      ds["depth_range"][1] if _get(contract, "use_dataset_bounds", False) else float("inf"))
            if not (float(er) < float("inf")):
                raise UnsupportedPipeline("z_depth contraction without a finite end radius")
            affine_fac = torch.tensor(float(er) / 2.0)
            bmin, den = torch.zeros(3), torch.full((3,), float(er) / 2.0)
        c.contract_type = L.CONTRACT_AFFINE
        c.contract_samples = int(bool(_get(contract, "contract_samples", False)))
        c.contract_dist_fac = float(affine_fac)
        for i in range(3):
            c.contract_affine_min[i], c.contract_affine_den[i] = float(bmin[i]), float(den[i])
    elif contract is not None and contract.type != "identity":
        if contract.type != "mipnerf":
            raise UnsupportedPipeline(f"contract '{contract.type}' is not on the fused path")
        if "distance_activation" in contract or "stop_iters" in contract:
            raise UnsupportedPipeline("contract distance_activation / stop_iters")
        if _get(contract, "use_dataset_bounds", False):  # contract.py:121-125
            sr = _get(contract, "contract_start_radius", max(ds["depth_range"][0] * 1.5, 1.0))
            er = _get(contract, "contract_end_radius", ds["depth_range"][1] * 1.5)
        else:
            sr = _get(contract, "contract_start_radius", 1.0)
            er = _get(contract, "contract_end_radius", float("inf"))
        c.contract_type = L.CONTRACT_MIPNERF
        c.contract_samples = int(bool(_get(contract, "contract_samples", False)))
        c.contract_start_radius, c.contract_end_radius = float(sr), float(er)
        c.contract_start_distance = float(_get(contract, "contract_start_distance", sr))
        c.contract_end_distance = float(_get(contract, "contract_end_distance", er))
    if it.type == "z_plane":
        c.isect_type = L.ISECT_Z_PLANE
        if use_ds:  # z.py:26-31
            initial, end = torch.tensor(-ds["near"]), torch.tensor(-ds["far"])
        else:
            initial, end = torch.tensor(_get(it, "initial", 0.0)), torch.tensor(_get(it, "end", 1.0))
    elif it.type in ("sphere", "cylinder"):  # IntersectSphereOld / IntersectCylinderOld share their setup
        c.isect_type = L.ISECT_SPHERE if it.type == "sphere" else L.ISECT_CYLINDER
        if use_ds:  # primitive.py:371-376
            initial = torch.tensor(_get(it, "initial", ds["near"] * 1.5))
            end = torch.tensor(_get(it, "end", ds["far"] * 1.5))
        else:
            initial, end = torch.tensor(_get(it, "initial", 0.0)), torch.tensor(_get(it, "end", 1.0))
        oi = _get(it, "origin_initial", [1.0, 1.0, 1.0])
        for i in range(3):
            c.sphere_origin_initial[i] = float(oi[i])
        c.sphere_origin_scale = float(_get(it, "origin_scale_factor", 0.0))
    elif it.type == "euclidean_distance_unified":  # IntersectEuclideanDistanceUnified (primitive.py:126-180)
        c.isect_type = L.ISECT_DISTANCE
        if use_ds:
            initial, end = torch.tensor(_get(it, "initial", -ds["far"])), torch.tensor(_get(it, "end", ds["far"]))
        else:
            initial, end = torch.tensor(_get(it, "initial", 0.0)), torch.tensor(_get(it, "end", 1.0))
    elif it.type == "sphere_new":  # IntersectSphereNew (primitive.py:440-487)
        c.isect_type = L.ISECT_SPHERE_NEW
        if use_ds:  # :446-452: outward_facing picks the sign of the first sphere
            if _get(it, "outward_facing", False):
                initial = torch.tensor(_get(it, "initial", ds["near"] * 1.5))
            else:
                initial = torch.tensor(_get(it, "initial", -ds["far"] * 1.5))
            end = torch.tensor(_get(it, "end", ds["far"] * 1.5))
        else:
            initial, end = torch.tensor(_get(it, "initial", 0.0)), torch.tensor(_get(it, "end", 1.0))
        c.sphere_origin_scale = float(_get(it, "origin_scale_factor", 0.0))
        c.sphere_resize_scale = float(_get(it, "resize_scale_factor", 0.0))
        ri = _get(it, "resize_initial", [1.0, 1.0, 1.0])
        for i in range(3):
            c.sphere_resize_initial[i] = float(ri[i])
    elif it.type in ("voxel_grid", "deformable_voxel_grid"):
        pass  # per-axis sample tables: built below
    else:
        raise UnsupportedPipeline(f"intersect '{it.type}' is not on the fused path")
    need_z = {"z_plane": 1, "euclidean_distance_unified": 1, "sphere_new": 8, "voxel_grid": 1}.get(it.type, 4)
    if c.n_z != need_z:
        raise UnsupportedPipeline(f"intersect '{it.type}' needs {need_z} z_vals channel(s), got {c.n_z}")
    if S > L.HR_MAX_SAMPLES:
        raise UnsupportedPipeline(f"z_channels {S} > {L.HR_MAX_SAMPLES}")

    def contract_bound(v):
        v = v.float()
        if c.contract_samples and c.contract_type == L.CONTRACT_AFFINE:  # contract_distance = d / fac (contract.py:80-81,106-107)
            return v / affine_fac
        if c.contract_samples:
            return _contract_distance(v, c.contract_start_distance, c.contract_end_distance)
        return v

    c.isect_axes, c.isect_outward, c.isect_max_axis = 1, 0, 0
    c.plane_normal_scale = 0.0
    for i in range(9):
        c.plane_normal[i] = 0.0
    if it.type in ("voxel_grid", "deformable_voxel_grid"):
        # IntersectVoxelGrid / IntersectDeformableVoxelGrid constructors (voxel.py:19-75, :115-176): sample s is plane s // A
        # of axis s % A, one linspace per axis
        deform = it.type == "deformable_voxel_grid"
        if _get(it, "use_local_prediction", False):
            raise UnsupportedPipeline("voxel_grid: use_local_prediction is not on the fused path")
        if deform:
            if use_ds:
                raise UnsupportedPipeline("deformable_voxel_grid with dataset bounds needs the dataset's point cloud")
            normals = [list(map(float, r)) for r in _get(it, "start_normal", [[1.0, 0.0, 0.0], [0.0, 1.0, 0.0], [0.0, 0.0, 1.0]])]
            A = len(normals)
            if not (1 <= A <= 3) or any(len(r) != 3 for r in normals):
                raise UnsupportedPipeline("deformable_voxel_grid: 1 to 3 start normals")
            for a_ in range(A):
                for k in range(3):
                    c.plane_normal[a_ * 3 + k] = normals[a_][k]
            c.plane_normal_scale = float(_get(it, "normal_scale_factor", 0.1))
            c.isect_type = L.ISECT_PLANE
            lo = torch.tensor([float(v) for v in _get(it, "initial", [0.0, 0.0, 0.0])])
            hi = torch.tensor([float(v) for v in _get(it, "end", [1.0, 1.0, 1.0])])
        else:
            A = 3
            c.isect_type = L.ISECT_VOXEL
            c.isect_outward = int(bool(_get(it, "outward_facing", False)))
            c.isect_max_axis = int(bool(_get(it, "max_axis", False)))
            fac = float(_get(it, "fac", 1.0))
            if use_ds and not ("initial" in it and "end" in it):
                if "bbox_min" not in ds or "bbox_max" not in ds:
                    raise UnsupportedPipeline("voxel_grid with use_dataset_bounds needs the dataset's bbox_min / bbox_max")
            if use_ds:  # voxel.py:27-29
                lo = torch.tensor([float(v) for v in it.initial]) if "initial" in it else torch.tensor([float(v) * fac for v in ds["bbox_min"]])
                hi = torch.tensor([float(v) for v in it.end]) if "end" in it else torch.tensor([float(v) * fac for v in ds["bbox_max"]])
            else:
                lo = torch.tensor([float(v) for v in _get(it, "initial", [0.0, 0.0, 0.0])])
                hi = torch.tensor([float(v) for v in _get(it, "end", [1.0, 1.0, 1.0])])
        if S % A != 0 or lo.numel() < A or hi.numel() < A:
            raise UnsupportedPipeline(f"{it.type}: z_channels {S} must be a multiple of the {A} axes, with one bound per axis")
        lo, hi = contract_bound(lo), contract_bound(hi)
        P = S // A
        tab = torch.stack([torch.linspace(float(lo[a_]), float(hi[a_]), P) for a_ in range(A)], -1)  # [P, A]
        flat = tab.reshape(-1)
        for i in range(S):
            c.samples[i] = float(flat[i])
        if "z_scale" in it:
            zs = torch.tensor([float(v) for v in it.z_scale])
            if zs.numel() != (1 if deform else 3):
                raise UnsupportedPipeline(f"{it.type}: z_scale must have {1 if deform else 3} entries")
        elif P > 1:
            zs = torch.abs(flat[1:2] - flat[0:1]) if deform else torch.abs(tab[1] - tab[0])  # voxel.py:169-174 / :58-63
        else:
            zs = torch.ones(1 if deform else 3)
        zs = torch.where(zs == 0.0, torch.ones_like(zs), zs)
        c.isect_axes = A
        c.z_scale = float(zs[0])
        for a_ in range(3):
            c.z_scale3[a_] = float(zs[a_]) if (not deform) else float(zs[0])
    else:
        initial, end = contract_bound(initial), contract_bound(end)
        samples = torch.linspace(float(initial), float(end), S)
        for i in range(S):
            c.samples[i] = float(samples[i])
        # z.py:58-71 (the primitives take cfg.z_scale or the sample spacing: primitive.py:211-219)
        if "z_scale" in it:
            c.z_scale = float(it.z_scale)
        elif S > 1:
            zs = torch.abs(samples[1] - samples[0])
            if "num_samples_for_scale" in it and it.type == "z_plane":
                zs = zs * (S / float(it.num_samples_for_scale))
            c.z_scale = float(zs)
        else:
            c.z_scale = 1.0
        for a_ in range(3):
            c.z_scale3[a_] = c.z_scale
    c.isect_near = float(_get(it, "near", ds["near"] if use_ds else 0.0))
    c.isect_far = float(_get(it, "far", float("inf")))
    if "mask" in it and it.mask is not None:
        gates.append(float(_get(it.mask, "stop_iters", float("inf"))))
    if "mask" in it and it.mask is not None and cur_iter > float(_get(it.mask, "stop_iters", float("inf"))):
        # base.py:104-105,197-198: past mask.stop_iters nothing is masked (samples with t == 0 still drop out downstream)
        c.isect_near, c.isect_far = float("-inf"), float("inf")
    c.isect_sort = int(bool(_get(it, "sort", False)))
    c.isect_act = act_at(_get(it, "activation", "identity"), "isect_act")
    c.isect_use_sigma = int(bool(_get(it, "use_sigma", False)))
    c.isect_density_off = offs.get(_get(it, "in_density_field", "sigma"), -1)
    if c.isect_density_off not in (-1, c.off_sigma, c.off_point_sigma):
        raise UnsupportedPipeline("intersect density field must be sigma or point_sigma")

    # ------------------------------------------------------------------ flow (point.py:741-831)
    c.num_keyframes, c.num_frames = int(ds.get("num_keyframes", 1)), int(ds.get("num_frames", 1))
    c.use_flow = 0
    c.flow_act = L.hr_act(0, 1.0, 0.0, 1.0)
    if flow is not None:
        if _get(flow, "use_angular_flow", False):
            raise UnsupportedPipeline("angular flow is not on the fused path")
        for k in ("rays_name", "in_points_field", "out_points_field"):
            if k in flow:
                raise UnsupportedPipeline(f"advect_points option '{k}'")
        if _get(flow, "use_spatial_flow", False):
            if "spatial_flow" not in offs:
                raise UnsupportedPipeline("spatial flow without a spatial_flow head")
            c.use_flow = 1
            c.flow_act = act_at(_get(flow, "spatial_flow_activation", "identity"), "flow_act")

    # ------------------------------------------------------------------ point offset (point.py:338-399)
    c.use_offset, c.offset_density_off = 0, -1
    c.offset_act = L.hr_act(0, 1.0, 0.0, 1.0)
    if offset is not None:
        for k in ("in_offset_field", "in_points_field", "out_points_field", "dropout"):
            if k in offset:
                raise UnsupportedPipeline(f"point_offset option '{k}'")
        if "point_offset" not in offs:
            raise UnsupportedPipeline("point_offset without a point_offset head")
        c.use_offset = 1
        if _get(offset, "use_sigma", True):
            c.offset_density_off = offs.get(_get(offset, "in_density_field", "sigma"), -1)
        c.offset_act = act_at(_get(offset, "activation", "identity"), "offset_act")

    # ------------------------------------------------------------------ outputs to the colour net
    extras = list(addp.extra_outputs)
    fields = list(extract.fields)
    for need in ("points", "distances", "viewdirs", "weights"):
        if need not in fields:
            raise UnsupportedPipeline(f"extract_fields must pass '{need}'")
    if "viewdirs" not in extras:
        raise UnsupportedPipeline("add_point_outputs must add viewdirs")
    if dynamic and (flow is None or not all(f in fields for f in ("base_times", "times", "time_offset")) or "times" not in extras):
        raise UnsupportedPipeline("dynamic colour net needs advect_points + time fields")
    if "color_transform" in offs or "color_transform_global" in offs:
        raise UnsupportedPipeline("colour transform heads are not on the fused path")
    # per-ray colour scale / shift after compositing (tensorf_dynamic.py:798-800): present iff extract_fields passes them
    glob = [k in offs and k in fields for k in ("color_scale_global", "color_shift_global")]
    if glob[0] != glob[1]:
        raise UnsupportedPipeline("color_scale_global and color_shift_global must come together")
    c.off_cscale_global = offs["color_scale_global"] if glob[0] else -1
    c.off_cshift_global = offs["color_shift_global"] if glob[0] else -1
    c.act_cscale_global = act_of("color_scale_global", "act_cscale_global")
    c.act_cshift_global = act_of("color_shift_global", "act_cshift_global")
    # per-camera colour transform (ColorTransformEmbedding point.py:558-612 -> transform_color_one tensorf_utils.py:308-331):
    # active iff the dataset validates on every camera (val_all), the keys pass extract_fields and no color_scale_global exists
    c.n_color_views = 0
    c.act_ctransform, c.act_ctshift = L.hr_act(0, 1.0, 0.0, 1.0), L.hr_act(0, 1.0, 0.0, 1.0)
    color_views = 0
    if ctrans is not None:
        if "total_images_per_frame" not in ds or "val_all" not in ds:
            raise UnsupportedPipeline("color_transform needs the dataset's total_images_per_frame / val_all")
        color_views = int(ds["total_images_per_frame"])
        tf, sf = _get(ctrans, "out_transform_field", "color_transform_global"), _get(ctrans, "out_shift_field", "color_shift_global")
        if tf != "color_transform_global" or sf != "color_shift_global":
            raise UnsupportedPipeline("color_transform with renamed output fields")
        if bool(ds["val_all"]) and not glob[0] and tf in fields:
            if sf not in fields:
                raise UnsupportedPipeline("color_transform_global reaches the colour net without color_shift_global")
            if color_views < 1:
                raise UnsupportedPipeline("color_transform without camera views")
            c.n_color_views = color_views
            c.act_ctransform = act_at(_get(ctrans, "transform_activation", "identity"), "act_ctransform")
            c.act_ctshift = act_at(_get(ctrans, "shift_activation", "identity"), "act_ctshift")
            c.c_in = 8  # the camera id is rays[..., -2] (point.py:598)
    c.use_color_scale_shift = int("color_scale" in offs and "color_scale" in fields and "color_shift" in offs and "color_shift" in fields)
    if ("color_scale" in offs and "color_scale" in fields) != ("color_shift" in offs and "color_shift" in fields):
        raise UnsupportedPipeline("color_scale and color_shift must come together")

    # ------------------------------------------------------------------ TensoRF decode (tensorf_base.py:138-260)
    c.dynamic = int(dynamic)
    aabb = net.aabb
    for i in range(3):
        c.aabb[i], c.aabb[3 + i] = float(aabb[0][i]), float(aabb[1][i])
    c.distance_scale = float(_get(net, "distance_scale", 25))
    ns, na = list(_get(net, "n_lamb_sigma", [8])), list(_get(net, "n_lamb_sh", [24]))
    if len(ns) != 3 or len(na) != 3:
        raise UnsupportedPipeline("n_lamb_sigma / n_lamb_sh must have 3 entries")
    for i in range(3):
        c.n_sigma[i], c.n_app[i] = int(ns[i]), int(na[i])
    c.app_dim = int(_get(net, "data_dim_color", 27))
    mode = _get(net, "shadingMode", "MLP_PE")
    if mode == "SH":
        c.shading = L.SHADE_SH
    elif mode == "RGB":
        c.shading = L.SHADE_RGB
    else:
        raise UnsupportedPipeline(f"shadingMode '{mode}' is not on the fused path")
    if dynamic and _get(net, "densityMode", "Density") != "Density":
        raise UnsupportedPipeline("densityMode must be Density")
    if "filter" in net and len(net.filter) > 0:
        raise UnsupportedPipeline("weight filtering is not on the fused path")
    c.white_bg = int(bool(_get(net, "white_bg", 0)) or (not dynamic and ds.get("name") == "blender"))
    c.black_bg = int(bool(_get(net, "black_bg", 0)) or (not dynamic and ds.get("collection") == "bulldozer"))
    c.weight_thre = float(_get(net, "rm_weight_mask_thre", 0.0001))
    act = _get(net, "fea2denseAct", "softplus")
    c.fea2dense = {"relu": L.DENSE_RELU, "softplus": L.DENSE_SOFTPLUS, "relu_abs": L.DENSE_RELU_ABS}[act]
    c.density_shift = float(_get(net, "density_shift", -10.0))
    c.clamp_output = 1
    return Signature(cfg=c, model_cfg=m, dataset=ds, head_names=head_names, head_channels=head_channels,
                     mlp_layer_shapes=shapes, dynamic=dynamic, in_perm=in_perm, color_views=color_views,
                     color_embedding_index=ctrans_index, cascade=cascade, net_index=point_index,
                     pre_layer_shapes=pre_shapes, pre_in_perm=pre_in_perm, ease_sites=sites, graph_iters=sorted(set(gates)))
