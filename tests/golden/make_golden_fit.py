"""Golden facts of a reference training run for ``hyperreel_b200.fit``: every shipped training config and the checkpoint
``state_dict`` of a small shipped model, from the unmodified reference through the shim.

    HYPERREEL_REFERENCE=<reference checkout> python tests/golden/make_golden_fit.py

writes ``tests/golden/reference/fit.npz``:

- ``training/<name>``: conf/experiment/training/<name>_tensorf.yaml as JSON, for every shipped ``*_tensorf.yaml``;
- ``state_dict/model``: the model config (conf/experiment/model/technicolor_z_plane_tiny.yaml) and ``state_dict/dataset``
  the dataset facts it is built with, both JSON;
- ``state_dict/shapes``: JSON ``{key: shape}`` of the reference ``INRSystem.state_dict()`` for that model, the render
  function's state under ``render_fn.`` (the regularisers and the loss hold no tensors).
"""
import glob
import json
import os
import sys

import numpy as np
import yaml

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import ref_shim  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference", "fit.npz")
MODEL = "technicolor_z_plane_tiny"
DATASET = {"num_keyframes": 12, "num_frames": 50, "near": 0.5, "far": 10.0, "depth_range": [0.5, 10.0],
           "name": "technicolor", "collection": "painter"}


def main():
    out = {}
    for path in sorted(glob.glob(os.path.join(ref_shim.REFERENCE_ROOT, "conf/experiment/training/*_tensorf.yaml"))):
        with open(path) as f:
            out[f"training/{os.path.basename(path)[:-len('_tensorf.yaml')]}"] = np.array(json.dumps(yaml.safe_load(f)))
    model = ref_shim.load_reference_yaml(MODEL)
    render = ref_shim.build_reference(model, DATASET)
    shapes = {f"render_fn.{k}": list(v.shape) for k, v in render.state_dict().items()}
    out["state_dict/model"] = np.array(json.dumps(model))
    out["state_dict/dataset"] = np.array(json.dumps(DATASET))
    out["state_dict/shapes"] = np.array(json.dumps(shapes))
    np.savez(OUT, **out)
    print(f"wrote {OUT}: {sorted(k for k in out if k.startswith('training/'))}, {len(shapes)} state_dict keys")


if __name__ == "__main__":
    main()
