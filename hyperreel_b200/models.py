"""``model_dict['lightfield']`` of the drop-in: the fused H100 light-field model.

Mirrors the surface of the reference's ``LightfieldModel`` (nlf/models/models.py:104-143):
``cls(cfg.model, system=...)``, ``forward(rays, render_kwargs) -> {'rgb': [N,3], ...}``,
``embed(rays, render_kwargs)``, ``set_iter(i)``, attributes ``embedding_model`` / ``color_model.net``
(with ``gridSize``, ``device``, ``init_svd_volume``, ``update_stepSize``, ``alphaMask`` as touched by
``INRSystem.load_state_dict``, nlf/__init__.py:433-479).

The whole graph RayParam -> RayPointEmbedding -> BaseColorModel is one native call
(``hr_render``: sample-net kernel + fused intersect/gather/composite kernel); parameters are kept in
reference-named ``nn.Parameter``s (state.py) and re-packed on the device whenever they change.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional

import torch
from torch import nn

from . import lib as L
from .signature import RENDER_ITER, Signature, UnsupportedPipeline, check_eased, ease_terms, lower, set_ease
from .state import _Color, _Embedding, default_grid


def _dataset_facts(system) -> dict:
    """What reference constructors read from ``system`` (tensorf_dynamic.py:49-50, contract.py:121-125,
    primitive.py:371-373, tensorf_no_sample.py:41-45)."""
    if system is None:
        return {}
    if isinstance(system, dict):
        return dict(system)
    ds = {}
    td = getattr(getattr(system, "dm", None), "train_dataset", None)
    for k in ("num_keyframes", "num_frames", "near", "far", "depth_range", "bbox_min", "bbox_max", "total_images_per_frame", "val_all"):
        if td is not None and hasattr(td, k):
            ds[k] = getattr(td, k)
    dcfg = getattr(getattr(system, "cfg", None), "dataset", None)
    if dcfg is not None:
        for k in ("name", "collection"):
            if k in dcfg:
                ds[k] = dcfg[k]
    return ds


def resolve_mlp_mode(name: str) -> int:
    """'auto' (default) and 'bf16x3' select the wgmma sample net -- every pipeline the fused path accepts runs on it
    (hidden width 128 / 256, encoded input <= 64 features); 'fp32' selects the CUDA-core kernel, the parity anchor;
    'fp16' selects the wgmma net at the precision of the reference's interactive viewer (every Linear layer as CUDA autocast
    computes it: fp16 operands, fp32 accumulation, fp16 results), for rendering."""
    try:
        return {"auto": L.MLP_BF16X3_TC, "bf16x3": L.MLP_BF16X3_TC, "fp32": L.MLP_FP32_SIMT, "fp16": L.MLP_FP16_TC}[name]
    except KeyError:
        raise ValueError(f"mlp_mode must be 'auto', 'bf16x3', 'fp32' or 'fp16', got {name!r}") from None


class _RenderHeads(torch.autograd.Function):
    """Everything after the sample net as one differentiable op: (rays, heads, VM tables, basis_mat) -> rgb.
    forward = hr_render_heads (the fused render kernel on caller-provided heads); backward = hr_render_backward (d heads, and the
    table / basis gradients accumulated in the handle, exported with hr_grad_read into the reference's tensor layouts)."""

    @staticmethod
    def forward(ctx, model, rays, heads, clamp_output, white_bg, *params):
        ctx.model, ctx.opts = model, (int(clamp_output), int(white_bg))
        ctx.save_for_backward(rays, heads)
        ctx.param_shapes = [tuple(p.shape) for p in params]
        return model._render_heads(rays, heads, *ctx.opts)

    @staticmethod
    def backward(ctx, d_rgb):
        rays, heads = ctx.saved_tensors
        d_heads, grads = ctx.model._render_backward(rays, heads, d_rgb.contiguous().float(), *ctx.opts)
        return (None, None, d_heads, None, None) + tuple(grads)


class _TrainNet(torch.autograd.Function):
    """The sample net's Linear layers as one differentiable op on the tensor cores: (rays, weights, biases) -> heads
    [N, S*stride].  forward = hr_train_net_forward (the wgmma render net, saving its activations in a workspace kept for
    backward); backward = hr_train_net_backward (bf16x3 wgmma dX / dW GEMMs) -> every layer's weight and bias gradient."""

    @staticmethod
    def forward(ctx, model, rays, *params):
        heads, ws = model._train_net_forward(rays)
        ctx.model, ctx.ws, ctx.n = model, ws, rays.shape[0]
        return heads

    @staticmethod
    def backward(ctx, d_heads):
        grads = ctx.model._train_net_backward(ctx.ws, d_heads.contiguous().float(), ctx.n)
        ctx.ws = None
        return (None, None) + tuple(grads)


class LightfieldModel(nn.Module):
    def __init__(self, cfg, **kwargs):
        super().__init__()
        dataset = dict(kwargs.get("dataset") or _dataset_facts(kwargs.get("system")))  # never mutate the caller's dict
        dataset.setdefault("near", 0.0)
        dataset.setdefault("far", 1.0)
        dataset.setdefault("depth_range", [dataset["near"], dataset["far"]])
        self._mlp_mode = resolve_mlp_mode(kwargs.get("mlp_mode", "auto"))
        # how render_differentiable trains the sample net: "torch" (its Linear layers as torch ops) or "tc" (hr_train_net_*)
        self._train_net = kwargs.get("train_net", "torch")
        if self._train_net not in ("torch", "tc"):
            raise ValueError(f"train_net must be 'torch' or 'tc', got {self._train_net!r}")
        if self._train_net == "tc" and self._mlp_mode != L.MLP_BF16X3_TC:
            raise ValueError("train_net='tc' trains the wgmma sample net: mlp_mode must be 'auto' or 'bf16x3'")
        self._iters_per_epoch = kwargs.get("iters_per_epoch")
        # EaseValue heads (nlf/activations.py:462-496): "elapsed" renders and trains every one at the end of its window at any
        # iteration (set_iter inside a window raises); "reference" eases them like the reference, set_iter(i) updating them
        # in place in the native handle
        self._ease = kwargs.get("ease", "elapsed")
        if self._ease not in ("elapsed", "reference"):
            raise ValueError(f"ease must be 'elapsed' or 'reference', got {self._ease!r}")
        if self._ease == "reference" and self._iters_per_epoch is None:
            raise ValueError("ease='reference' needs iters_per_epoch: the EaseValue windows are given in epochs")
        self.cfg = cfg
        self.sig: Signature = lower(cfg, dataset, cur_iter=RENDER_ITER, iters_per_epoch=self._iters_per_epoch,
                                    mlp_mode=self._mlp_mode, ease=self._ease == "reference")
        self.num_outputs = 3
        self.cur_iter = RENDER_ITER
        grid = kwargs.get("grid") or default_grid(self.sig)
        # reference-named parameter storage
        self.embedding_model = _Embedding(self.sig.mlp_layer_shapes, self.sig.color_views, self.sig.color_embedding_index,
                                          self.sig.net_index, self.sig.pre_layer_shapes)
        self.color_model = _Color(self.sig, grid)
        self._lib = L.load_library()  # raises if the CUDA library is missing -- no fallback
        self._handle = C.c_void_p()
        self._uploaded_version = None
        self._version_tensors = None
        self._device_index: Optional[int] = None
        self._ws: Optional[torch.Tensor] = None
        self._graph_key = self.sig.graph_key(RENDER_ITER)

    # ------------------------------------------------------------------ reference surface
    def set_iter(self, i):
        """The reference's per-iteration hook (nlf/models/models.py:140-143).  With ease="elapsed" the fused path implements
        render-time semantics only (all PE windows open, EaseValue elapsed; the reference sets iteration 1e7*iters when
        rendering, nlf/__init__.py:582-583); with ease="reference" open EaseValue windows are eased at iteration i."""
        self.cur_iter = i
        if self._ease == "reference" and self.sig.graph_key(int(i)) == self._graph_key:
            self._set_ease_iter(int(i))  # same graph: only the eased activations can differ
        else:
            self._relower(int(i))
        self.color_model.set_iter(i)

    def _relower(self, i):
        # Re-lower at iteration i with the same epoch scale, net mode and ease mode.  Raises UnsupportedPipeline while a PE
        # window (or, with ease="elapsed", an EaseValue window) is still open; a different graph at i (an embedding gated by
        # wait/stop_iters, mask.stop_iters) must not be rendered with the construction-time semantics: adopt it and rebuild the
        # native handle.  A configuration that differs in its activations alone is updated in place (hr_set_activations).
        new = lower(self.cfg, self.sig.dataset, cur_iter=i, iters_per_epoch=self._iters_per_epoch, mlp_mode=self._mlp_mode,
                    ease=self._ease == "reference")
        for k in range(6):
            new.cfg.aabb[k] = self.sig.cfg.aabb[k]  # aabb is checkpoint state, kept in sync by _ensure_uploaded
        if bytes(new.cfg) != bytes(self.sig.cfg):
            if new.mlp_layer_shapes != self.sig.mlp_layer_shapes or list(new.cfg.n_sigma) != list(self.sig.cfg.n_sigma):
                raise UnsupportedPipeline("set_iter: the pipeline at this iteration has different parameter shapes")
            same_graph = _without_activations(new.cfg) == _without_activations(self.sig.cfg)
            self.sig = new
            if same_graph and self._handle:
                L.check(self._lib.hr_set_activations(self._handle, C.byref(self.sig.cfg)))
            else:
                self._release_handle()
        self._graph_key = self.sig.graph_key(i)

    def _set_ease_iter(self, i):
        """EaseValue.set_iter (activations.py:495-496) of every ease site; the handle's activations are updated in place
        (hr_set_activations: no re-upload, no device synchronisation) when one of them changed."""
        # built on a copy, adopted once every check and the native call have passed: sig.cfg always matches the handle
        c = L.hr_config.from_buffer_copy(bytes(self.sig.cfg))
        for site in self.sig.ease_sites:
            a = L.hr_act.from_buffer_copy(bytes(getattr(c, site.field)))
            set_ease(a, ease_terms(i, site.start_value, site.wait_iters, site.window_iters))
            setattr(c, site.field, check_eased(a, site.field, c.n_samples))
        if bytes(c) == bytes(self.sig.cfg):
            return
        if self._handle:
            L.check(self._lib.hr_set_activations(self._handle, C.byref(c)))
        self.sig.cfg = c

    def forward(self, rays: torch.Tensor, render_kwargs: Optional[Dict] = None) -> Dict[str, torch.Tensor]:
        render_kwargs = render_kwargs or {}
        fields = list(render_kwargs.get("fields", []))
        if self.training:
            if fields:
                raise UnsupportedPipeline("extra fields are produced by the eval()/render path only")
            return {"rgb": self.render_differentiable(rays)}
        rays = self._check_rays(rays)
        n = rays.shape[0]
        rgb = torch.empty((n, 3), device=rays.device, dtype=torch.float32)
        if n == 0:
            return {"rgb": rgb}
        self._ensure_uploaded(rays.device)
        ws = self._workspace(n, rays.device)
        stream = torch.cuda.current_stream(rays.device).cuda_stream
        if not fields:
            L.check(self._lib.hr_render(self._handle, rays.data_ptr(), n, rgb.data_ptr(), ws.data_ptr(), ws.numel(), stream))
            return {"rgb": rgb}
        # extra outputs (tensorf_dynamic.py:808-837 / tensorf_no_sample.py:254-278): reduced in the render kernel's epilogue
        no_over = set(render_kwargs.get("no_over_fields", []))
        pred_w = set(render_kwargs.get("pred_weights_fields", []))
        out = {"rgb": rgb}
        rw_ptr = None
        reqs = []
        for key in fields:
            if key == "render_weights":
                out[key] = torch.empty((n, self.sig.n_samples), device=rays.device)
                rw_ptr = out[key].data_ptr()
                continue
            mode = L.FIELD_NO_OVER if key in no_over else (L.FIELD_PRED_WEIGHTS if key in pred_w else L.FIELD_OVER)
            fid, dim = self._field(key)
            out[key] = torch.empty((n, (self.sig.n_samples if mode == L.FIELD_NO_OVER else 1) * dim), device=rays.device)
            reqs.append(L.hr_field_request(fid, mode, out[key].data_ptr()))
        arr = (L.hr_field_request * max(len(reqs), 1))(*reqs)
        L.check(self._lib.hr_render_fields(self._handle, rays.data_ptr(), n, rgb.data_ptr(), rw_ptr, arr, len(reqs),
                                           ws.data_ptr(), ws.numel(), stream))
        return out

    def embed(self, rays: torch.Tensor, render_kwargs: Optional[Dict] = None) -> Dict[str, torch.Tensor]:
        """What RayPointEmbedding.forward returns to ``render_fn.embed`` (nlf/embedding/embedding.py:100-117): every key
        ``extract_fields`` lets through (its own list plus render_kwargs['fields'], nlf/embedding/point.py:236-244),
        flattened to ``[N, S*dim]``."""
        render_kwargs = render_kwargs or {}
        rays = self._check_rays(rays)
        n, S = rays.shape[0], self.sig.n_samples
        keys = []
        for key in list(self._extract_fields()) + list(render_kwargs.get("fields", [])):
            if key in self._available_fields() and key not in keys:
                keys.append(key)
        out = {k: torch.empty((n, S * self._field(k)[1]), device=rays.device) for k in keys}
        if n == 0:
            return out
        self._ensure_uploaded(rays.device)
        ws = self._workspace(n, rays.device)
        rgb = torch.empty((n, 3), device=rays.device)
        reqs = [L.hr_field_request(self._field(k)[0], L.FIELD_NO_OVER, out[k].data_ptr()) for k in keys]
        arr = (L.hr_field_request * max(len(reqs), 1))(*reqs)
        stream = torch.cuda.current_stream(rays.device).cuda_stream
        L.check(self._lib.hr_render_fields(self._handle, rays.data_ptr(), n, rgb.data_ptr(), None, arr, len(reqs),
                                           ws.data_ptr(), ws.numel(), stream))
        return out

    # ------------------------------------------------------------------ training path (SURVEY.md 8 f1)
    def render_differentiable(self, rays: torch.Tensor, clamp_output: Optional[bool] = None, white_bg: Optional[bool] = None,
                              return_heads: bool = False):
        """rgb [N,3] with an autograd graph back to every parameter -- what ``training_step`` (nlf/__init__.py:634-709) needs.
        Defaults follow the module mode like the reference: training -> no clamp, white background by coin flip
        (tensorf_dynamic.py:795-806); eval -> clamp, configured background.  With train_net="torch" the sample net's
        Linear layers run as torch ops on the library's encoded input (hr_encode_rays); with "tc" they are one autograd op
        around the library's tensor-core training net (hr_train_net_forward / hr_train_net_backward).  Everything after them
        is one autograd op around the fused kernels (hr_render_heads / hr_render_backward)."""
        rays = self._check_rays(rays)
        c = self.sig.cfg
        if self.sig.cascade:
            raise UnsupportedPipeline("cascaded (point_prediction) pipelines render on the fused path; their backward pass is not built")
        if clamp_output is None:
            clamp_output = not self.training
        if white_bg is None:
            white_bg = bool(c.white_bg) or (self.training and not c.black_bg and bool(torch.rand(()) < 0.5))
        white_bg = bool(white_bg) and not c.black_bg
        self._ensure_uploaded(rays.device)
        if self._train_net == "tc":
            x = _TrainNet.apply(self, rays, *self._net_params())
        else:
            x = self._torch_net(rays, return_heads)
        tn = self.color_model.net
        dplane, dsecond, aplane, asecond = tn.tables()
        params = [t for t in list(dplane) + list(aplane) + list(dsecond) + list(asecond) if t.numel() > 0] + [tn.basis_mat.weight]
        if c.n_color_views > 0:  # ColorTransformEmbedding (point.py:558-605): its table acts on the pixel inside the fused op
            params.append(self.embedding_model.embeddings[self.sig.color_embedding_index].color_embedding)
        rgb = _RenderHeads.apply(self, rays, x, clamp_output, white_bg, *params)
        return (rgb, x) if return_heads else rgb  # x: the sample-net output [N, S*stride] (gradient bisecting)

    def _torch_net(self, rays, return_heads):
        """BaseMLP.forward (mlp.py:159-172) as torch ops on the library's encoded input."""
        c = self.sig.cfg
        n = rays.shape[0]
        enc = torch.empty((n, c.mlp_in), device=rays.device)
        stream = torch.cuda.current_stream(rays.device).cuda_stream
        if n:
            L.check(self._lib.hr_encode_rays(self._handle, rays.data_ptr(), n, enc.data_ptr(), stream))
        perm = list(self.sig.in_perm)
        if perm != list(range(len(perm))):  # BasicPE: reference feature in_perm[k] = kernel feature k
            inv = torch.empty(len(perm), dtype=torch.long)
            inv[torch.tensor(perm)] = torch.arange(len(perm))
            enc = enc.index_select(1, inv.to(rays.device))
        net = self.embedding_model.embeddings[0].net
        x = enc
        if c.mlp_mode == L.MLP_ZERO:  # ZeroMLP.forward (mlp.py:29-30)
            x = torch.zeros((n, c.mlp_out), device=rays.device, requires_grad=return_heads)  # a leaf when the caller bisects d heads
        layers = getattr(net, "layers", [])
        last = len(layers) - 1
        for i, layer in enumerate(layers):  # BaseMLP.forward (mlp.py:159-172)
            lin = layer[0] if isinstance(layer, nn.Sequential) else layer
            if i == c.mlp_skip:
                x = torch.cat([enc, x], -1)
            x = torch.nn.functional.linear(x, lin.weight, lin.bias)
            if i < last:
                x = torch.nn.functional.leaky_relu(x, c.leaky_slope)
        return x

    def _net_params(self):
        """[weight, bias] of every Linear layer of the sample net, in order."""
        out = []
        for layer in getattr(self.embedding_model.embeddings[0].net, "layers", []):
            lin = layer[0] if isinstance(layer, nn.Sequential) else layer
            out += [lin.weight, lin.bias]
        return out

    def _train_net_forward(self, rays):
        n, c = rays.shape[0], self.sig.cfg
        heads = torch.empty((n, c.mlp_out), device=rays.device)
        # one workspace per step: the backward reads the activations this forward saves in it
        ws = torch.empty(int(self._lib.hr_train_net_workspace_bytes(self._handle, n)), dtype=torch.uint8, device=rays.device)
        stream = torch.cuda.current_stream(rays.device).cuda_stream
        L.check(self._lib.hr_train_net_forward(self._handle, rays.data_ptr(), n, heads.data_ptr(), ws.data_ptr(), ws.numel(), stream))
        return heads, ws

    def _train_net_backward(self, ws, d_heads, n):
        params = self._net_params()
        grads = [torch.empty(p.shape, device=d_heads.device, dtype=torch.float32) for p in params]
        G = L.hr_net_grads()
        for i, g in enumerate(grads):
            (G.weight if i % 2 == 0 else G.bias)[i // 2] = g.data_ptr()
        stream = torch.cuda.current_stream(d_heads.device).cuda_stream
        L.check(self._lib.hr_train_net_backward(self._handle, d_heads.data_ptr(), n, C.byref(G), ws.data_ptr(), ws.numel(), stream))
        perm = list(self.sig.in_perm)
        if perm != list(range(len(perm))):
            # BasicPE: the uploaded first / skip layer has its input columns in the kernels' order (_ensure_uploaded), reference
            # column in_perm[k] = uploaded column k; the hidden part of the skip layer keeps its place
            for i in {0, self.sig.cfg.mlp_skip} - {-1}:
                w = grads[2 * i]
                src = torch.arange(w.shape[1])
                src[torch.tensor(perm)] = torch.arange(len(perm))
                grads[2 * i] = w.index_select(1, src.to(w.device))
        return grads

    def _train_workspace(self, n, dev):
        need = int(self._lib.hr_train_workspace_bytes(self._handle, n))
        if self._ws is None or self._ws.numel() < need or self._ws.device != dev:
            self._ws = torch.empty(need, dtype=torch.uint8, device=dev)
        return self._ws

    def _render_heads(self, rays, heads, clamp_output, white_bg):
        n = rays.shape[0]
        rgb = torch.empty((n, 3), device=rays.device)
        if n == 0:
            return rgb
        heads = heads.detach().contiguous().float()
        ws = self._train_workspace(n, rays.device)
        opts = L.hr_train_opts(clamp_output, white_bg)
        stream = torch.cuda.current_stream(rays.device).cuda_stream
        L.check(self._lib.hr_render_heads(self._handle, rays.data_ptr(), heads.data_ptr(), n, rgb.data_ptr(), C.byref(opts),
                                          ws.data_ptr(), ws.numel(), stream))
        return rgb

    def _render_backward(self, rays, heads, d_rgb, clamp_output, white_bg):
        n = rays.shape[0]
        heads = heads.detach().contiguous().float()
        d_heads = torch.zeros_like(heads)
        tn = self.color_model.net
        dplane, dsecond, aplane, asecond = tn.tables()
        stream = torch.cuda.current_stream(rays.device).cuda_stream
        opts = L.hr_train_opts(clamp_output, white_bg)
        L.check(self._lib.hr_grad_zero(self._handle, stream))
        if n:
            ws = self._train_workspace(n, rays.device)
            L.check(self._lib.hr_render_backward(self._handle, rays.data_ptr(), heads.data_ptr(), n, d_rgb.data_ptr(), d_heads.data_ptr(),
                                                 C.byref(opts), ws.data_ptr(), ws.numel(), stream))
        G = L.hr_grads()
        outs = {}
        for name, tabs, slot in (("dp", dplane, G.sigma_plane), ("ap", aplane, G.app_plane), ("d2", dsecond, G.sigma_second),
                                 ("a2", asecond, G.app_second)):
            for i in range(3):
                if tabs[i].numel() > 0:
                    g = torch.empty(tabs[i].shape, device=rays.device, dtype=torch.float32)
                    outs[(name, i)] = g
                    slot[i] = g.data_ptr()
        gb = torch.empty(tn.basis_mat.weight.shape, device=rays.device, dtype=torch.float32)
        G.basis_mat = gb.data_ptr()
        order = [outs[(nm, i)] for nm in ("dp", "ap", "d2", "a2") for i in range(3) if (nm, i) in outs] + [gb]
        if self.sig.cfg.n_color_views > 0:
            emb = self.embedding_model.embeddings[self.sig.color_embedding_index].color_embedding
            ge = torch.empty(emb.shape, device=rays.device, dtype=torch.float32)
            G.color_embedding = ge.data_ptr()
            order.append(ge)
        L.check(self._lib.hr_grad_read(self._handle, C.byref(G), stream))
        return d_heads, order

    # ------------------------------------------------------------------ the dict `x` of the reference, by name
    def _extract_fields(self):
        embs = self.sig.model_cfg.embedding.embeddings
        return list(next(e for e in embs.values() if e.type == "extract_fields").fields)

    def _available_fields(self):
        """Keys of the reference's dict ``x`` when it reaches extract_fields, restricted to what the fused path carries."""
        c = self.sig.cfg
        have = {"points", "distances", "weights", "viewdirs"} | set(self.sig.head_names)
        if c.dynamic or c.use_flow:
            have |= {"base_times", "time_offset"}
        embs = self.sig.model_cfg.embedding.embeddings
        addp = next(e for e in embs.values() if e.type == "add_point_outputs")
        if "times" in list(addp.extra_outputs):
            have.add("times")
        return {k for k in have if k in L.FIELDS}

    def _field(self, key):
        if key not in L.FIELDS:
            raise UnsupportedPipeline(f"field '{key}' is not produced by the fused path")
        if key not in self._available_fields():
            raise KeyError(key)  # the reference fails the same way on x[key]
        return L.FIELDS[key], L.FIELD_CHANNELS[key]

    # ------------------------------------------------------------------ native plumbing
    def render_stages(self, rays: torch.Tensor) -> Dict[str, torch.Tensor]:
        """Stage-boundary dump for parity bisecting (hr_render_stages)."""
        rays = self._check_rays(rays)
        n, S, c = rays.shape[0], self.sig.n_samples, self.sig.cfg
        dev = rays.device
        self._ensure_uploaded(dev)
        out = {
            "rgb": torch.empty((n, 3), device=dev), "mlp_out": torch.empty((n, c.mlp_out), device=dev),
            "distances": torch.empty((n, S), device=dev), "points": torch.empty((n, S, 3), device=dev),
            "sigma": torch.empty((n, S), device=dev), "weights": torch.empty((n, S), device=dev),
            "rgb_samples": torch.empty((n, S, 3), device=dev),
        }
        if n == 0:
            return out
        ws = self._workspace(n, dev)
        stream = torch.cuda.current_stream(dev).cuda_stream
        L.check(self._lib.hr_render_stages(self._handle, rays.data_ptr(), n, out["rgb"].data_ptr(), out["mlp_out"].data_ptr(),
                                           out["distances"].data_ptr(), out["points"].data_ptr(), out["sigma"].data_ptr(),
                                           out["weights"].data_ptr(), out["rgb_samples"].data_ptr(), ws.data_ptr(), ws.numel(),
                                           stream))
        return out

    def render_host(self, rays_host: torch.Tensor, rgb_host: Optional[torch.Tensor] = None, chunk: int = 0) -> torch.Tensor:
        """Host-buffer entry (hr_render_host): pinned rays in, pinned rgb out, H2D/D2H overlapped inside."""
        if rays_host.is_cuda or rays_host.dtype != torch.float32 or not rays_host.is_contiguous():
            raise ValueError("render_host expects a contiguous fp32 host tensor")
        if rays_host.shape[-1] != self.sig.c_in:
            raise ValueError(f"rays must have {self.sig.c_in} channels")
        n = rays_host.shape[0]
        if rgb_host is None:
            rgb_host = torch.empty((n, 3), dtype=torch.float32, pin_memory=True)
        self._ensure_uploaded(self._default_device())
        L.check(self._lib.hr_render_host(self._handle, rays_host.data_ptr(), n, rgb_host.data_ptr(), chunk))
        return rgb_host

    def render_scatter(self, rays: torch.Tensor, dst_ptrs, n_dst: int, row0: int) -> None:
        """Render ``rays`` and store the pixels at rows ``[row0, row0 + n)`` of every ``[N_total,3]`` fp32 buffer in
        ``dst_ptrs`` (a ctypes ``c_void_p`` array: this rank's gather buffer and the peer-mapped buffers of the other ranks):
        the gather of ray-sharded rendering, done by the render kernel's epilogue (hr_render_scatter, ray_shard.py)."""
        if self.training:
            raise RuntimeError("hyperreel_b200.LightfieldModel implements the eval()/render path only; call .eval()")
        rays = self._check_rays(rays)
        n = rays.shape[0]
        if n == 0:
            return
        self._ensure_uploaded(rays.device)
        ws = self._workspace(n, rays.device)
        stream = torch.cuda.current_stream(rays.device).cuda_stream
        L.check(self._lib.hr_render_scatter(self._handle, rays.data_ptr(), n, dst_ptrs, int(n_dst), int(row0), ws.data_ptr(),
                                            ws.numel(), stream))

    def render_to8b(self, rays: torch.Tensor) -> torch.Tensor:
        """rays [N,C] on the device -> uint8 rgb [N,3] on the device: the composite with ``to8b``
        (utils/__init__.py:47) fused into the render kernel's epilogue (hr_render_to8b)."""
        if self.training:
            raise RuntimeError("hyperreel_b200.LightfieldModel implements the eval()/render path only; call .eval()")
        rays = self._check_rays(rays)
        n = rays.shape[0]
        out = torch.empty((n, 3), device=rays.device, dtype=torch.uint8)
        if n == 0:
            return out
        self._ensure_uploaded(rays.device)
        ws = self._workspace(n, rays.device)
        stream = torch.cuda.current_stream(rays.device).cuda_stream
        L.check(self._lib.hr_render_to8b(self._handle, rays.data_ptr(), n, out.data_ptr(), ws.data_ptr(), ws.numel(), stream))
        return out

    def render_frame_to8b(self, camera, out_host: Optional[torch.Tensor] = None, chunk: int = 0) -> torch.Tensor:
        """One whole frame: rays generated on the device from ``camera`` (hyperreel_b200.camera.Camera or TwoPlaneCamera), rendered,
        packed to 8 bit and copied into a pinned host image [H, W, 3] uint8 (hr_render_frame_to8b_host) -- one iteration of
        the reference's validation_video / viewer loop without the per-frame 32 B/ray upload."""
        if self.training:
            raise RuntimeError("hyperreel_b200.LightfieldModel implements the eval()/render path only; call .eval()")
        H, W = int(camera.height), int(camera.width)
        if out_host is None:
            out_host = torch.empty((H, W, 3), dtype=torch.uint8, pin_memory=True)
        if out_host.is_cuda or out_host.dtype != torch.uint8 or out_host.numel() != H * W * 3 or not out_host.is_contiguous():
            raise ValueError("out_host must be a contiguous uint8 host tensor of H*W*3 elements")
        self._ensure_uploaded(self._default_device())
        cam = camera.to_c()
        L.check(self._lib.hr_render_frame_to8b_host(self._handle, C.byref(cam), out_host.data_ptr(), chunk))
        return out_host

    def _default_device(self) -> torch.device:
        return torch.device("cuda", self._device_index if self._device_index is not None else torch.cuda.current_device())

    def _frame_list(self, fn: str, cameras, times):
        """The eval check and frame list of render_video, score_views and render_visuals, refused under ``fn``'s name before
        any work: (F, H, W, the hr_camera records, the float32 times) of ``cameras`` (one size) at ``times`` (one per camera,
        finite in float32; default each camera's ``time``)."""
        if self.training:
            raise RuntimeError("hyperreel_b200.LightfieldModel implements the eval()/render path only; call .eval()")
        cams = list(cameras)
        if not cams:
            raise ValueError(f"{fn}: no cameras")
        t = [float(c.time) for c in cams] if times is None else times
        t = torch.as_tensor(t, dtype=torch.float64).reshape(-1).to(torch.float32)
        if t.numel() != len(cams):
            raise ValueError(f"{fn}: {len(cams)} cameras but {t.numel()} times")
        if not bool(torch.isfinite(t).all()):
            raise ValueError(f"{fn}: times must be finite in float32")
        H, W = int(cams[0].height), int(cams[0].width)
        for i, c in enumerate(cams):
            if (int(c.height), int(c.width)) != (H, W):
                raise ValueError(f"{fn}: camera {i} is {int(c.width)} x {int(c.height)}, camera 0 is {W} x {H}")
        recs = (L.hr_camera * len(cams))(*[c.to_c() for c in cams])
        return len(cams), H, W, recs, (C.c_float * len(cams))(*t.tolist())

    def render_video(self, cameras, times=None, out: Optional[torch.Tensor] = None, stream=None) -> torch.Tensor:
        """Frames of ``cameras`` (hyperreel_b200.camera.Camera or TwoPlaneCamera, one size, any mix of models) at ``times`` (one per camera;
        default each camera's ``time``) -> uint8 video [F, H, W, 3] on the device, in one call that never synchronises
        (hr_render_video_to8b): frame f is bit for bit the image render_frame_to8b makes of cameras[f] at times[f].  ``out``
        (device uint8 [F, H, W, 3], contiguous) receives it when given; the work goes on ``stream`` (a torch.cuda.Stream;
        default the current stream)."""
        F, H, W, recs, tt = self._frame_list("render_video", cameras, times)
        if out is not None:
            if not out.is_cuda or out.dtype != torch.uint8 or tuple(out.shape) != (F, H, W, 3) or not out.is_contiguous():
                raise ValueError(f"render_video: out must be a contiguous CUDA uint8 tensor of shape {(F, H, W, 3)}, got "
                                 f"{out.dtype} {tuple(out.shape)} on {out.device}")
        dev = out.device if out is not None else self._default_device()
        self._ensure_uploaded(dev)
        need = int(self._lib.hr_video_workspace_bytes(self._handle, F, H, W))
        if need < 0:
            raise ValueError(f"render_video: {F} frames of {W} x {H} pixels overflow a 64-bit size")
        stream = stream if stream is not None else torch.cuda.current_stream(dev)
        with torch.cuda.stream(stream):  # the scratch (and a new out) belong to the stream the work runs on
            ws = torch.empty(need, dtype=torch.uint8, device=dev)
            if out is None:
                out = torch.empty((F, H, W, 3), dtype=torch.uint8, device=dev)
            L.check(self._lib.hr_render_video_to8b(self._handle, recs, tt, F, out.data_ptr(), ws.data_ptr(), need,
                                                   stream.cuda_stream))
        return out

    def score_views(self, cameras, images: torch.Tensor, times=None, out: Optional[torch.Tensor] = None, stream=None, *,
                    rgba: bool = False):
        """(mse, ssim) of every held-out view, fp64 [n] device tensors: view i rendered from ``cameras[i]`` at ``times[i]``
        (default each camera's ``time``) in one call that never synchronises (hr_score_views), scored against ``images[i]``
        (uint8 [n, H, W, 3] on the device, contiguous) like ``metrics.image_metrics(pred, images[i] / 255)`` (correctly rounded, as T.ToTensor() converts) of the
        view's eval render, bit for bit.  ``out`` (device fp64 [n, 2], contiguous) receives (mse, ssim) when given; the work
        goes on ``stream`` (a torch.cuda.Stream; default the current stream).  ``rgba=True``: ``images`` are uint8 RGBA
        [n, H, W, 4], the DoNeRF and Catacaustics frames, and each view is scored against its composite over white,
        ``rgb * a + (1 - a)`` of the ``u8 / 255`` values as their ``get_rgb`` computes it on the CPU."""
        F, H, W, recs, tt = self._frame_list("score_views", cameras, times)
        if H < 11 or W < 11:
            raise ValueError(f"score_views: views must be at least 11 x 11 (the SSIM window), got {W} x {H}")
        shape = (F, H, W, 4 if rgba else 3)
        if not isinstance(images, torch.Tensor) or images.dtype != torch.uint8 or tuple(images.shape) != shape \
                or not images.is_contiguous():
            got = f"{images.dtype} {tuple(images.shape)}" if isinstance(images, torch.Tensor) else type(images).__name__
            raise ValueError(f"score_views: images must be a contiguous uint8 tensor of shape {shape}"
                             f"{' (rgba=True)' if rgba else ''}, got {got}")
        if not images.is_cuda:
            raise RuntimeError("hyperreel_b200 scores views on an H100 only: images must be a CUDA tensor (no CPU fallback)")
        dev = images.device
        p = next(self.parameters(), None)
        if p is not None and p.is_cuda and p.device != dev:
            raise ValueError(f"score_views: images are on {dev}, the model on {p.device}")
        if out is not None and (not out.is_cuda or out.dtype != torch.float64 or tuple(out.shape) != (F, 2)
                                or not out.is_contiguous() or out.device != dev):
            raise ValueError(f"score_views: out must be a contiguous float64 tensor of shape {(F, 2)} on {dev}, got "
                             f"{out.dtype} {tuple(out.shape)} on {out.device}")
        self._ensure_uploaded(dev)
        need = int(self._lib.hr_score_views_workspace_bytes(self._handle, F, H, W))
        if need < 0:
            raise ValueError(f"score_views: {F} views of {W} x {H} pixels overflow a 64-bit size")
        stream = stream if stream is not None else torch.cuda.current_stream(dev)
        with torch.cuda.stream(stream):  # the scratch (and a new out) belong to the stream the work runs on
            ws = torch.empty(need, dtype=torch.uint8, device=dev)
            if out is None:
                out = torch.empty((F, 2), dtype=torch.float64, device=dev)
            fmt = L.PIXEL_RGBA8 if rgba else L.PIXEL_RGB8
            L.check(self._lib.hr_score_views(self._handle, recs, tt, F, images.data_ptr(), fmt, out.data_ptr(),
                                             ws.data_ptr(), need, stream.cuda_stream))
        return out[:, 0], out[:, 1]

    def render_visuals(self, cameras, requests, times=None, rgb: bool = True, stream=None):
        """The uint8 video of ``cameras`` at ``times`` (as render_video makes it, bit for bit) and the embedding maps of
        ``requests`` (camera.VisualRequest, from camera.embedding_requests) in one render pass per frame and one call that
        never synchronises (hr_render_visuals).  Returns (video [F, H, W, 3] or None when ``rgb`` is False, {key: uint8
        [F, H, W, channels]})."""
        from .signature import UnsupportedPipeline

        F, H, W, recs, tt = self._frame_list("render_visuals", cameras, times)
        if not rgb and not requests:
            raise ValueError("render_visuals: nothing to render (rgb=False and no requests)")
        for r in requests:  # a field this model lacks: the reference's KeyError on x[key], refused before any work
            try:
                self._field(r.key)
            except KeyError:
                raise UnsupportedPipeline(f"embedding visualiser: field '{r.key}' is not an output of this model") from None
        dev = self._default_device()
        self._ensure_uploaded(dev)
        stream = stream if stream is not None else torch.cuda.current_stream(dev)
        with torch.cuda.stream(stream):  # the scratch and the outputs belong to the stream the work runs on
            maps = {r.key: torch.empty((F, H, W, r.channels), dtype=torch.uint8, device=dev) for r in requests}
            video = torch.empty((F, H, W, 3), dtype=torch.uint8, device=dev) if rgb else None
            reqs = [L.hr_visual_request(L.FIELDS[r.key], r.mode, r.channels, int(r.use_abs), int(r.bounds is not None),
                                        int(r.normalize), *(r.bounds or (0.0, 0.0)), maps[r.key].data_ptr()) for r in requests]
            arr = (L.hr_visual_request * max(len(reqs), 1))(*reqs)
            need = int(self._lib.hr_render_visuals_workspace_bytes(self._handle, arr, len(reqs), F, H, W))
            if need < 0:
                L.check(1)  # the library's reason
            ws = torch.empty(need, dtype=torch.uint8, device=dev)
            L.check(self._lib.hr_render_visuals(self._handle, recs, tt, F, video.data_ptr() if rgb else None, arr, len(reqs),
                                                ws.data_ptr(), need, stream.cuda_stream))
        return video, maps

    def timing(self, enable: bool = True):
        L.check(self._lib.hr_timing_enable(self._handle, int(enable)))
        L.check(self._lib.hr_timing_reset(self._handle))

    def timing_read(self):
        r, m, k = C.c_double(), C.c_double(), C.c_int64()
        L.check(self._lib.hr_timing_read(self._handle, C.byref(r), C.byref(m), C.byref(k)))
        b, kb = C.c_double(), C.c_int64()
        L.check(self._lib.hr_timing_read_backward(self._handle, C.byref(b), C.byref(kb)))
        return {"render_ms": r.value, "mlp_ms": m.value, "launches": k.value, "backward_ms": b.value, "backward_launches": kb.value}

    def set_sub_batch(self, rays: int):
        """Rays per sub-batch of the render call (0 = 16 sample-net tile waves, the default; < 0 = never split)."""
        self._sub_batch = int(rays)
        if self._handle:
            L.check(self._lib.hr_set_sub_batch(self._handle, self._sub_batch))

    def launch_count(self) -> int:
        return int(self._lib.hr_launch_count(self._handle)) if self._handle else 0

    def mark_dirty(self):
        """Call after mutating parameters in place (optimiser step, manual edits) so the next render re-packs."""
        self._uploaded_version = None
        self._version_tensors = None

    def _check_rays(self, rays):
        if not rays.is_cuda:
            raise RuntimeError("hyperreel_b200 renders on an H100 only: rays must be a CUDA tensor (no CPU fallback)")
        rays = rays.reshape(-1, rays.shape[-1])
        if rays.shape[-1] != self.sig.c_in:
            raise ValueError(f"rays must have {self.sig.c_in} channels, got {rays.shape[-1]}")
        if rays.dtype != torch.float32:
            raise ValueError("rays must be float32")
        return rays.contiguous()

    def _workspace(self, n, dev):
        need = int(self._lib.hr_workspace_bytes(self._handle, n))
        if self._ws is None or self._ws.numel() < need or self._ws.device != dev:
            self._ws = torch.empty(need, dtype=torch.uint8, device=dev)
        return self._ws

    def _param_version(self):
        # version counters + storage addresses only: no device synchronisation and no module-tree walk on the per-call
        # path (the Parameter / buffer objects are cached; mark_dirty() drops the cache for code that replaces them)
        net = self.color_model.net
        sv = getattr(net, "struct_version", 0)
        ts = self._version_tensors
        if ts is None or ts[0] != sv:  # init_svd_volume (a resized grid) replaced the table Parameters
            ts = self._version_tensors = (sv, list(self.parameters()))
        # the two buffers are read fresh on every call: Module.to()/.cuda() replaces buffer objects
        return tuple([(t._version, t.data_ptr()) for t in ts[1] + [net.aabb, net.gridSize]])

    def _apply(self, fn, *args, **kwargs):
        out = super()._apply(fn, *args, **kwargs)  # .to() / .cuda() / .float(): Parameter storage may have moved
        self.mark_dirty()
        return out

    def _release_handle(self):
        if getattr(self, "_handle", None):
            self._lib.hr_destroy(self._handle)
        self._handle = C.c_void_p()
        self._uploaded_version = None

    def _ensure_uploaded(self, dev: torch.device):
        idx = dev.index if dev.index is not None else torch.cuda.current_device()
        ver = self._param_version()
        if self._handle and self._device_index == idx and self._uploaded_version == ver:
            return
        # aabb is checkpoint state (it changes when the reference shrinks the grid, tensorf_base.py:1190-1232)
        aabb = [float(v) for v in self.color_model.net.aabb.detach().cpu().reshape(-1).tolist()]
        if aabb != [float(self.sig.cfg.aabb[i]) for i in range(6)]:
            for i in range(6):
                self.sig.cfg.aabb[i] = aabb[i]
            self._release_handle()
        if not self._handle or self._device_index != idx:
            self._release_handle()
            L.check(self._lib.hr_create(C.byref(self.sig.cfg), idx, C.byref(self._handle)))
            if getattr(self, "_sub_batch", 0):
                L.check(self._lib.hr_set_sub_batch(self._handle, self._sub_batch))
            self._device_index = idx
            self._uploaded_version = None
        P = L.hr_params()
        keep = []  # keep tensors alive until the upload has been enqueued and synchronised

        def dptr(t):
            t = t.detach()
            if not t.is_cuda or t.device.index != idx:
                t = t.to(torch.device("cuda", idx))
            t = t.contiguous().float()
            keep.append(t)
            return t.data_ptr()

        P.on_device = 1

        def put_net(net, perm, skip_layer, weights, biases):
            permuted = perm != list(range(len(perm)))
            for i, layer in enumerate(getattr(net, "layers", [])):  # a `zero` sample net has no layers to upload
                lin = layer[0] if isinstance(layer, nn.Sequential) else layer
                w = lin.weight
                if permuted and (i == 0 or i == skip_layer):
                    # BasicPE column order -> the kernels' per-band order (Signature.in_perm); the hidden part of the skip
                    # layer's input (cat([input, hidden]), mlp.py:167-168) keeps its place
                    cols = torch.tensor(perm + list(range(len(perm), w.shape[1])), device=w.device)
                    w = w.detach().index_select(1, cols)
                weights[i] = dptr(w)
                biases[i] = dptr(lin.bias)

        # the net behind the final heads: the ray_prediction net, or the point_prediction net of a cascaded pipeline
        put_net(self.embedding_model.embeddings[self.sig.net_index].net, list(self.sig.in_perm), self.sig.cfg.mlp_skip,
                P.mlp_weight, P.mlp_bias)
        if self.sig.cascade:
            put_net(self.embedding_model.embeddings[0].net, list(self.sig.pre_in_perm), self.sig.cfg.pre_mlp_skip,
                    P.pre_mlp_weight, P.pre_mlp_bias)
        tn = self.color_model.net
        dplane, dsecond, aplane, asecond = tn.tables()
        for i in range(3):
            C_i = dplane[i].shape[1]
            P.plane_h[i], P.plane_w[i] = dplane[i].shape[2], dplane[i].shape[3]
            P.second_len[i] = dsecond[i].shape[3] if tn.dynamic else dsecond[i].shape[2]
            if C_i > 0:
                P.sigma_plane[i], P.app_plane[i] = dptr(dplane[i]), dptr(aplane[i])
                P.sigma_second[i], P.app_second[i] = dptr(dsecond[i]), dptr(asecond[i])
        P.basis_mat = dptr(tn.basis_mat.weight)
        if self.sig.cfg.n_color_views > 0:
            P.color_embedding = dptr(self.embedding_model.embeddings[self.sig.color_embedding_index].color_embedding)
        stream = torch.cuda.current_stream(torch.device("cuda", idx))
        L.check(self._lib.hr_upload(self._handle, C.byref(P), stream.cuda_stream))
        if self.training:
            # a training step re-packs after every optimiser step and runs on one stream: the pack kernels are ordered before
            # the kernels that read them, and the caching allocator releases `keep` in stream order -- no host sync, so the
            # CPU keeps queueing the step while the GPU works
            self._upload_keep = keep
        else:
            stream.synchronize()  # renders may come from any stream afterwards
        self._uploaded_version = ver

    def __del__(self):
        try:
            if getattr(self, "_handle", None):
                self._lib.hr_destroy(self._handle)
                self._handle = None
        except Exception:
            pass


def _without_activations(cfg: L.hr_config) -> bytes:
    """The bytes of an hr_config with every hr_act member cleared: what hr_set_activations requires to be unchanged."""
    c = L.hr_config.from_buffer_copy(bytes(cfg))
    for name, typ in L.hr_config._fields_:
        if typ is L.hr_act:
            setattr(c, name, L.hr_act())
    return bytes(c)


model_dict = {"lightfield": LightfieldModel}
ray_model_dict = {"lightfield": LightfieldModel}
pos_model_dict = {"lightfield": LightfieldModel}
