"""mlp_mode="fp16" without a GPU: the mode's name and refusals, the C enum and ABI version the binding mirrors, the lowering of
single and cascaded nets, and the fp64 emulation of the contract (tests/fp16_net_oracle.py) on hand-checked values."""
import os
import re

import pytest
import torch

import hyperreel_b200 as hb
from hyperreel_b200 import lib as L
from hyperreel_b200.models import resolve_mlp_mode
from hyperreel_b200.signature import lower
from tests.cases import build_case
from tests.fp16_net_oracle import MARGIN, SUM_ORDER, emulate_fp64, ulp16, ulps_apart
from tests.test_shipped_yaml_golden import SHIPPED, load_fixture

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_mode_names():
    assert resolve_mlp_mode("fp16") == L.MLP_FP16_TC == 3
    assert resolve_mlp_mode("auto") == resolve_mlp_mode("bf16x3") == L.MLP_BF16X3_TC  # the default is unchanged
    with pytest.raises(ValueError, match="'fp16'"):
        resolve_mlp_mode("half")


def test_enum_and_abi_mirror_the_header():
    header = open(os.path.join(ROOT, "include", "hyperreel_b200.h")).read()
    assert int(re.search(r"HR_MLP_FP16_TC = (\d+)", header).group(1)) == L.MLP_FP16_TC
    assert int(re.search(r"#define HR_ABI_VERSION (\d+)", header).group(1)) == L.HR_ABI_VERSION == 26
    assert L.load_library().hr_abi_version() == L.HR_ABI_VERSION


def test_the_training_net_is_refused():
    case = build_case("technicolor_init")
    with pytest.raises(ValueError, match="bf16x3"):
        hb.LightfieldModel(case.model_cfg, dataset=case.dataset, train_net="tc", mlp_mode="fp16")
    model = hb.LightfieldModel(case.model_cfg, dataset=case.dataset, train_net="torch", mlp_mode="fp16")
    assert model.sig.cfg.mlp_mode == L.MLP_FP16_TC


def test_lowering_single_net_and_cascade():
    case = build_case("technicolor_init")
    assert lower(case.model_cfg, case.dataset, mlp_mode=L.MLP_FP16_TC).cfg.mlp_mode == 3
    path = next(p for p in SHIPPED if p.endswith("technicolor_cascaded.npz"))
    _, cfg, ds, _, _, _, _ = load_fixture(path)
    c = lower(cfg, ds, mlp_mode=L.MLP_FP16_TC).cfg
    assert c.cascade == 1 and c.mlp_mode == 3 and c.pre_mlp_mode == 3
    model = hb.LightfieldModel(cfg, dataset=ds, mlp_mode="fp16")
    assert model.sig.cfg.mlp_mode == 3 and model.sig.cfg.pre_mlp_mode == 3
    render = hb.RenderLightfield(model, None, cfg.render)
    assert render.model.sig.cfg.mlp_mode == 3


def test_system_passes_the_mode_through():
    case = build_case("technicolor_init")
    system = hb.INRSystem(hb.to_cfg({"model": case.model_cfg_plain, "training": {}}), dataset=case.dataset, mlp_mode="fp16")
    assert system.render_fn.model.sig.cfg.mlp_mode == L.MLP_FP16_TC


def test_emulation_rounds_like_the_contract():
    # one hidden layer of one unit, then the output: every rounding step by hand
    x = torch.tensor([[1.0 + 2.0 ** -12, -3.0]])          # 1 + 2^-12 rounds to 1 in fp16
    w0, b0 = torch.tensor([[0.5, 1.0 / 3.0]]), torch.tensor([0.1])
    w1, b1 = torch.tensor([[2.0]]), torch.tensor([2.0 ** -30])  # b1 underflows to 0 in fp16
    out, tol = emulate_fp64(x, [w0, b0, w1, b1], skip=-1, slope=0.01)
    h16 = lambda v: torch.tensor(v, dtype=torch.float32).half().double()
    z = float((h16(0.5) * 1.0 + h16(1.0 / 3.0) * -3.0 + h16(0.1)).float().half())  # fp16 result of layer 0, negative
    a = float((torch.tensor(z, dtype=torch.float32) * torch.tensor(0.01, dtype=torch.float32)).half())
    assert z < 0 and float(out) == float(torch.tensor(2.0 * a).half())
    assert 0 < float(tol) < 16 * float(ulp16(out.double()))
    # a first layer may differ by one fp16 ulp of its value, plus the margin on the summation-order term, and nothing more
    one, tol1 = emulate_fp64(x, [w0, b0], skip=-1, slope=0.01)
    order = MARGIN * SUM_ORDER * float(x.abs().double() @ w0.abs().double().t().half().double() + b0.abs().half().double())
    assert float(ulp16(one.double())) <= float(tol1) <= float(ulp16(one.double() + order)) + order * 1.001
    # overflow gives inf, as autocast does
    big, _ = emulate_fp64(torch.tensor([[300.0]]), [torch.tensor([[300.0]]), torch.tensor([0.0])], skip=-1, slope=0.01)
    assert torch.isinf(big).all()


def test_skip_columns_are_rounded_like_layer_0():
    torch.manual_seed(0)
    enc = torch.randn(5, 3)
    p = [torch.randn(4, 3), torch.randn(4), torch.randn(4, 7), torch.randn(4), torch.randn(2, 4), torch.randn(2)]
    out, _ = emulate_fp64(enc, p, skip=1, slope=0.01)
    out16, _ = emulate_fp64(enc.half().float(), p, skip=1, slope=0.01)  # the input already fp16: the same net
    assert torch.equal(out, out16)
    assert torch.equal(out, out.half().float())  # every output is an fp16 value


def test_ulps_apart_counts_fp16_steps():
    a = torch.tensor([1.0, -1.0, 0.0, 2.0 ** -24])
    b = torch.tensor([1.0 + 2.0 ** -10, -1.0 - 2.0 ** -10, -0.0, -(2.0 ** -24)])
    assert ulps_apart(a, b).tolist() == [1, 1, 0, 2]
