"""The wgmma sample net at ray counts that split unevenly over the persistent CTAs.

Every CTA walks tiles blockIdx.x, blockIdx.x + gridDim.x, ...; the two consumer warpgroups of a CTA hand each other the
activation operand and the encoded input between tiles, so counts where some CTAs run one tile fewer than others, where
the last tile is partial, and where there are fewer tiles than SMs all have to agree with the fp32 CUDA-core net.
"""
import pytest
import torch

from tests.cases import build_case
from tests.test_parity_gpu import make_render

pytestmark = pytest.mark.gpu


def _ray_counts():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return [
        128 * 5 + 3,                 # fewer tiles than SMs, partial last tile
        128 * sms + 1,               # one CTA runs a second tile of one ray
        128 * (2 * sms + 50) + 37,   # two full waves, then 51 tiles: some CTAs one tile short, the last one partial
    ]


# hidden width 128 (shiny_tiny) and 256, encoded inputs of one and two 32-feature chunks (*_wide_pe)
@pytest.mark.parametrize("name", ["shiny_tiny", "technicolor_trained", "donerf_wide_pe", "neural3d_wide_pe"])
def test_tc_matches_fp32_path_at_uneven_tile_counts(name):
    for n in _ray_counts():
        case = build_case(name, n=n)
        rays = case.rays.cuda()
        a = make_render(case, mlp_mode="fp32").model.render_stages(rays)
        b = make_render(case, mlp_mode="bf16x3").model.render_stages(rays)
        assert b["mlp_out"].shape == a["mlp_out"].shape
        scale = max(1.0, float(a["mlp_out"].abs().max()))
        err = float((a["mlp_out"] - b["mlp_out"]).abs().max())
        assert err <= 1e-4 * scale, f"{name}, {n} rays: sample-net max abs error {err}"
