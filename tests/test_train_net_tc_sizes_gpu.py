"""The sample net's tensor-core backward (hr_train_net_backward) across batch sizes: from 1 ray, through the split-K edges of
the dW GEMMs (fewer rays than one K block of 32, 33 and 129 rays, where the split count is recomputed from the split length),
to 65 613 rays, where every dW entry is a sum of ~1 000-ray fp32 partials over 264 splits.

The reference is fp64: dY_l, the gradient of layer l's output, walks back from d heads through the fp64 weights with the
LeakyReLU sides the tc forward chose, and dW_l = dY_l^T X_l multiplies the layer inputs X_l the forward saved (the encoded
input and the hidden activations in the workspace): the dW GEMM's own operands, so the forward's rounding is not part of the
comparison (the forward is checked bit for bit against the render net).  Tolerance, per entry:
    |g - ref| <= 2^-12 (|dY_l|^T |X_l|)_ij + 2^-14 (M_l^T |X_l|)_ij + 1e-6 max |ref|
(biases: the column sums of |dY_l| and M_l in place of the products).  The error of the bf16x3 products (the dropped lo*lo
term, ~2^-16 of each product) and of the fp32 split-K sums (~2^-14 of the summed magnitudes for a split of ~1 024 rays, worst
case) grows with the sum of the magnitudes of the terms, not with the result: a bound relative to max |ref| would be blind to
errors on small entries and not tied to the batch size.  2^-12 leaves about a factor of 4 over that worst case (an estimate,
not a measurement).  The second term is the rounding the kernel's dY_l carries in from the dX GEMM that makes it: M_l =
(|dY_{l+1}| |W_{l+1}|) * |LeakyReLU side|, the magnitude that GEMM sums for each entry of dY_l, one step only (M = 0 for the
last layer, whose dY is d heads).  Without it a layer below the last fails with 1 or 2 rays: an entry of dW is then a single
product, and an entry of dY_l that cancels to near 0 has lost its relative accuracy.  Summing the magnitudes over every layer
above instead (|d heads| walked down through |W|) would grow by ~10x per layer and make the bound of the lowest layers larger
than the gradient itself.  So each test also asserts that every tensor's bound stays below MAX_WIDTH of its largest entry,
and reports that width per layer with the largest error it saw as a fraction of the bound.
"""
import ctypes as C

import pytest
import torch

from hyperreel_b200 import lib as L
from tests.test_train_net_tc_gpu import _case, _fp64_net_grads, _model, _saved

pytestmark = pytest.mark.gpu
REL = 2.0 ** -12
REL_IN = 2.0 ** -14
FLOOR = 1e-6
MAX_WIDTH = 0.25  # largest admitted entry of the bound, as a fraction of the tensor's largest entry


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _fp64_backward(model, enc_k, acts, d_heads):
    """Per layer, in the reference's parameter layouts: (dW, db, tolerance of dW, tolerance of db) in fp64 from the saved
    layer inputs and the tc forward's LeakyReLU sides (module docstring)."""
    c = model.sig.cfg
    perm = list(model.sig.in_perm)
    inv = torch.empty(len(perm), dtype=torch.long)
    inv[torch.tensor(perm)] = torch.arange(len(perm))
    enc = enc_k.double()[:, inv.to(enc_k.device)]  # kernel feature order -> the reference's
    params = [p.detach().double() for p in model._net_params()]
    out = [None] * c.mlp_layers
    dy = d_heads.double()
    carried = torch.zeros_like(dy)  # M_l: d heads reach the last layer exactly
    for i in reversed(range(c.mlp_layers)):
        x = acts[i - 1].double() if i > 0 else enc
        if i == c.mlp_skip:
            x = torch.cat([enc, x], -1)
        out[i] = (dy.t() @ x, dy.sum(0), REL * (dy.abs().t() @ x.abs()) + REL_IN * (carried.t() @ x.abs()),
                  REL * dy.abs().sum(0) + REL_IN * carried.sum(0))
        if i > 0:
            w = params[2 * i][:, -c.mlp_width:]  # the hidden columns (a skip layer's encoded-input columns come first)
            side = torch.where(acts[i - 1] > 0, 1.0, c.leaky_slope).double()
            dy, carried = (dy @ w) * side, (dy.abs() @ w.abs()) * side.abs()
    return out


def _check(name, n):
    check_case(_case(name, n), f"{name} n={n}")


def check_case(case, label):
    """The training forward and backward of `case`'s net on its rays against the fp64 references (module docstring)."""
    n = case.rays.shape[0]
    model = _model(case)
    rays = case.rays.cuda()
    model._ensure_uploaded(rays.device)
    heads, ws = model._train_net_forward(rays)
    d_heads = torch.randn(heads.shape, generator=torch.Generator().manual_seed(n)).cuda()
    got = model._train_net_backward(ws, d_heads, n)
    enc, acts = _saved(model, ws, n)
    ref = _fp64_backward(model, enc, acts, d_heads)
    assert len(got) == 2 * len(ref) == 2 * model.sig.cfg.mlp_layers
    worst, widths = 0.0, []
    for i, g in enumerate(got):
        w, b = ref[i // 2][i % 2], ref[i // 2][2 + i % 2]
        what = f"layer {i // 2} {'bias' if i % 2 else 'weight'}"
        assert g.shape == w.shape == b.shape, what
        scale = float(w.abs().max())
        assert scale > 0.0, what
        tol = b + FLOOR * scale
        # the bound is a check: far below the tensor's largest entry, so that a wrong (or zero) gradient cannot pass it
        widths.append(float(tol.max()) / scale)
        assert widths[-1] <= MAX_WIDTH, f"{what}: the bound reaches {widths[-1]:.3f} of max |ref|"
        ratio = (g.double() - w).abs() / tol
        worst = max(worst, float(ratio.max()))
        assert float(ratio.max()) <= 1.0, (f"{what}: {int((ratio > 1).sum())} entries out of tolerance, worst "
                                           f"{float(ratio.max()):.2f} of it")
    print(f"\n[{label}] largest error {worst:.3f} of the bound; largest bound per weight, as a fraction of max |ref|: "
          + " ".join(f"{x:.2g}" for x in widths[0::2]))
    # and the reference of tests/test_train_net_tc_gpu.py (activations recomputed in fp64) to its tolerance, which is the
    # tighter one on the largest entries of a large batch
    for g, w in zip(got, _fp64_net_grads(model, enc, acts, d_heads)):
        assert float((g.double() - w).abs().max()) <= 1e-3 * float(w.abs().max())
    # the training forward's heads stay bit for bit the render net's
    model.eval()
    assert torch.equal(heads, model.render_stages(rays)["mlp_out"])


WIDE = ["shiny_tiny", "donerf_wide_pe", "technicolor_s64"]  # width 128, two input chunks, 960 outputs


@pytest.mark.parametrize("n", [1, 2, 31, 33, 127, 129, "wave", 65613])
def test_net_gradients_within_the_magnitude_bound(n):
    """Width 256 with a skip layer (Technicolor); "wave" = one 128-ray tile per SM and one ray more."""
    _check("technicolor_trained", 128 * _sms() + 1 if n == "wave" else n)


@pytest.mark.parametrize("name", WIDE)
@pytest.mark.parametrize("n", [1, 33, 129, 65613])
def test_net_gradients_within_the_magnitude_bound_other_nets(name, n):
    _check(name, n)


@pytest.mark.parametrize("name", ["technicolor_trained", "donerf_wide_pe"])
def test_no_rays_give_zero_gradients(name):
    """hr_train_net_backward with n = 0 writes 0 into every weight and bias gradient (here NaN-filled beforehand)."""
    case = _case(name, 8)
    model = _model(case)
    rays = case.rays.cuda()
    model._ensure_uploaded(rays.device)
    grads = [torch.full(p.shape, float("nan"), device="cuda") for p in model._net_params()]
    G = L.hr_net_grads()
    for i, g in enumerate(grads):
        (G.weight if i % 2 == 0 else G.bias)[i // 2] = g.data_ptr()
    d_heads = torch.zeros(1, model.sig.cfg.mlp_out, device="cuda")
    ws = torch.empty(256, dtype=torch.uint8, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    assert model._lib.hr_train_net_backward(model._handle, d_heads.data_ptr(), 0, C.byref(G), ws.data_ptr(), ws.numel(),
                                            stream) == 0
    torch.cuda.synchronize()
    for i, g in enumerate(grads):
        assert bool((g == 0).all()), i
