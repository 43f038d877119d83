"""Every layer of the tensor-core sample net, per entry, against fp64, over a pairwise cover of the net shapes the lowering
admits (tests/sweep_cases.py: NET_SHAPES): hidden width 128 / 256, depth 2 to 10, no skip or a skip at layer 1 or L - 2, an
encoded input of 4 to 63 features in one or two chunks, a last layer narrower than, as wide as and one 4-column group wider
than a pass, head rows of every width mod 4, and the largest pass table (HR_TC_MAX_PASSES).

Per layer l, from the SAVE forward's workspace: the layer is recomputed in fp64 from the kernel's own saved input X_l (the
encoded input, the previous layer's activation, or both at the skip), and its saved activation (the heads for the last layer)
must agree per entry within
    2^-14 (|X_l| |W_l|^T + |b_l|) + 1e-6 max |ref|.
bf16x3 drops the lo*lo term and rounds the split, about 2^-16 of each product, and the fp32 sum over K <= 320 terms adds about
as much again: the bound leaves a factor of 2 to 4 (an estimate, not a measurement -- each test prints the largest error as a
fraction of it).  Because the bound follows the magnitudes summed, not the result, it holds for every entry; each test also
asserts that it stays far below the tensor's largest entry, so that a zeroed column cannot pass.
"""
import pytest
import torch

from tests.sweep_cases import NET_SHAPES, net_case
from tests.test_train_net_tc_gpu import _model, _saved
from tests.test_train_net_tc_sizes_gpu import check_case

pytestmark = pytest.mark.gpu
REL = 2.0 ** -14
FLOOR = 1e-6
MAX_WIDTH = 0.05  # largest admitted entry of the bound, as a fraction of the tensor's largest entry
TOL_FP32 = 2e-5   # per head channel, of that channel's largest |fp64 head|
TOL_TC = 1e-4
NAMES = [s[0] for s in NET_SHAPES]


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _count(n):
    """1, 65, one 128-ray tile per SM and one ray more, or a ragged count of two waves."""
    return {"wave": 128 * _sms() + 1, "waves": 2 * 128 * _sms() + 77}.get(n, n)


def _inputs(model, enc_k):
    """The encoded input in the reference's feature order (fp64) and the net's parameters (fp64, reference layouts)."""
    perm = list(model.sig.in_perm)
    inv = torch.empty(len(perm), dtype=torch.long)
    inv[torch.tensor(perm)] = torch.arange(len(perm))
    return enc_k.double()[:, inv.to(enc_k.device)], [p.detach().double() for p in model._net_params()]


def _fp64_heads(c, enc, params):
    """The fp64 chain of the whole net from the encoded input."""
    x = enc
    for i in range(c.mlp_layers):
        if i == c.mlp_skip:
            x = torch.cat([enc, x], -1)
        x = x @ params[2 * i].t() + params[2 * i + 1]
        if i < c.mlp_layers - 1:
            x = torch.where(x > 0, x, c.leaky_slope * x)
    return x


def _per_channel_error(c, got, ref):
    """max |got - ref| / max |ref| of each head channel (the columns s * stride + channel of every sample)."""
    n = ref.shape[0]
    g, r = got.double().view(n, c.n_samples, c.head_stride), ref.view(n, c.n_samples, c.head_stride)
    scale = r.abs().amax((0, 1))
    assert bool((scale > 0).all()), "a head channel is zero throughout"
    return (g - r).abs().amax((0, 1)) / scale


@pytest.mark.parametrize("n", [1, 65, "wave", "waves"])
@pytest.mark.parametrize("name", NAMES)
def test_every_layer_matches_fp64(name, n):
    n = _count(n)
    case = net_case(name, n)
    c = case.sig.cfg
    model = _model(case)
    rays = case.rays.cuda()
    model._ensure_uploaded(rays.device)
    heads, ws = model._train_net_forward(rays)
    enc_k, acts = _saved(model, ws, n)
    enc, params = _inputs(model, enc_k)

    # per layer, from the kernel's own saved input
    worst = 0.0
    for i in range(c.mlp_layers):
        x = enc if i == 0 else acts[i - 1].double()
        if i == c.mlp_skip:
            x = torch.cat([enc, x], -1)
        w, b = params[2 * i], params[2 * i + 1]
        ref = x @ w.t() + b
        bound = REL * (x.abs() @ w.abs().t() + b.abs())
        last = i == c.mlp_layers - 1
        if not last:
            ref = torch.where(ref > 0, ref, c.leaky_slope * ref)  # LeakyReLU moves no two values further apart
        got = (heads if last else acts[i]).double()
        scale = float(ref.abs().max())
        tol = bound + FLOOR * scale
        width = float(tol.max()) / scale
        assert width <= MAX_WIDTH, f"layer {i}: the bound reaches {width:.3f} of max |ref|"
        ratio = (got - ref).abs() / tol
        worst = max(worst, float(ratio.max()))
        assert float(ratio.max()) <= 1.0, (f"layer {i}: {int((ratio > 1).sum())} entries out of tolerance, worst "
                                           f"{float(ratio.max()):.2f} of it")
    print(f"\n[{name} n={n}] largest error {worst:.3f} of the per-layer bound")

    # the render net (its own store of the heads rows) equals the training forward bit for bit
    model.eval()
    assert torch.equal(model.render_stages(rays)["mlp_out"], heads)

    # per head channel, both nets, against the fp64 chain on the same encoded input
    ref = _fp64_heads(c, enc, params)
    tc = _per_channel_error(c, heads, ref)
    fp32 = _model(case, train_net="torch", mlp_mode="fp32")
    fp32.eval()
    simt = _per_channel_error(c, fp32.render_stages(rays)["mlp_out"], ref)
    print(f"[{name} n={n}] per-channel error / tolerance: tensor cores {float(tc.max()) / TOL_TC:.3f}, "
          f"fp32 {float(simt.max()) / TOL_FP32:.3f}")
    assert float(tc.max()) <= TOL_TC, f"tensor-core heads, channel {int(tc.argmax())}: {float(tc.max()):.2e} of its range"
    assert float(simt.max()) <= TOL_FP32, f"fp32 heads, channel {int(simt.argmax())}: {float(simt.max()):.2e} of its range"


@pytest.mark.parametrize("name", NAMES)
def test_training_backward_at_every_shape(name):
    """The dX / dW GEMMs on every shape (head rows of every width mod 4, padded to 4 columns in the workspace), within the
    magnitude bound of tests/test_train_net_tc_sizes_gpu.py."""
    check_case(net_case(name, 1000), f"{name} n=1000")
