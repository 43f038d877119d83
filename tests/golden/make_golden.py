"""Generate the golden vectors under tests/golden/ by running the *reference itself* (unmodified modules
from a reference checkout, on CPU, through oracle/ref_shim.py) on seeded inputs.

Only runnable with HYPERREEL_REFERENCE set to a reference checkout; the tests that read the fixtures need none.  Each fixture stores: the case description, the rays, a SHA-256 of the seeded
parameters (parameters are regenerated from the seed by ``tests/cases.py`` -- torch's CPU generators are
deterministic -- and the hash guards against drift), and the reference outputs:
``rgb``, ``points``/``distances`` from ``render_fn.embed`` (nlf/rendering.py:79-84) and every other key that call returns
(``embed__<key>``), ``render_weights`` (nlf/nets/tensorf_dynamic.py:821-823), the sample-net output of the first 64 rays
(forward hook on ``BaseMLP``), the per-sample shaded colour ``rgb_samples`` (the colour net's ``renderModule`` wrapped, its
output scattered by ``app_mask`` like tensorf_dynamic.py:757-777) and the extra outputs the colour net returns for
``tests.cases.FIELD_KWARGS`` (``field__<key>``).

    python tests/golden/make_golden.py [case ...]
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import ref_shim  # noqa: E402
from tests.cases import CASES, FIELD_KWARGS, build_case, state_hash  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))


def main():
    ref_shim.install()
    torch.set_num_threads(8)
    only = sys.argv[1:]  # optional: regenerate just these cases
    for name in CASES:
        if only and name not in only:
            continue
        case = build_case(name)
        ref = ref_shim.build_reference(case.model_cfg_plain, case.dataset)
        missing, unexpected = ref.load_state_dict(case.state_dict, strict=False)
        assert not unexpected, unexpected
        assert all("dummy_layer" in k for k in missing), [k for k in missing if "dummy_layer" not in k]
        captured = {}
        hook = ref.model.embedding_model.embeddings[0].net.register_forward_hook(
            lambda mod, inp, out: captured.__setitem__("mlp_out", out.detach().clone()))
        from nlf.rendering import render_chunked
        # the colour net's shading function, wrapped: renderModule(points, viewdirs, app_features, kwargs) -> [M', 3]
        net = ref.model.color_model.net
        inner = net.renderModule

        def spy(*a, **k):
            r = inner(*a, **k)
            captured["valid_rgbs"] = r.detach().clone()
            return r

        net.renderModule = spy
        with torch.no_grad():
            out = render_chunked(case.rays.clone(), ref, dict(FIELD_KWARGS), case.rays.shape[0])
            emb = ref.embed(case.rays.clone())
        net.renderModule = inner
        hook.remove()
        S = case.n_samples
        n = case.rays.shape[0]
        w = out["render_weights"].reshape(n, S)
        app_mask = w > float(net.rayMarch_weight_thres)
        rgb_samples = torch.zeros(n, S, 3)
        if app_mask.any():
            rgb_samples[app_mask] = captured["valid_rgbs"]
        extra = {f"field__{k}": v.reshape(n, -1).numpy() for k, v in out.items() if k not in ("rgb", "render_weights")}
        extra.update({f"embed__{k}": v.reshape(n, -1).numpy() for k, v in emb.items() if k not in ("points", "distances")})
        np.savez_compressed(
            os.path.join(OUT, f"{name}.npz"),
            rays=case.rays.numpy(),
            rgb=out["rgb"].numpy(),
            render_weights=out["render_weights"].reshape(n, S).numpy(),
            points=emb["points"].reshape(n, S, 3).numpy(),
            distances=emb["distances"].reshape(n, S).numpy(),
            mlp_out=captured["mlp_out"][:64].numpy(),
            rgb_samples=rgb_samples.numpy(),
            state_sha256=np.array(state_hash(case.state_dict)),
            **extra,
        )
        print(f"{name}: n={n} S={S} rgb mean {float(out['rgb'].mean()):.4f} std {float(out['rgb'].std()):.4f} "
              f"sum(w) mean {float(out['render_weights'].reshape(n, S).sum(-1).mean()):.3f}")


if __name__ == "__main__":
    main()
