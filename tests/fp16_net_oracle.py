"""The fp16 sample net's contract (mlp_mode="fp16"), restated twice, with the tolerance its tests use.

Every Linear layer computes what CUDA autocast computes for F.linear: the encoded input, the weights and the bias rounded to
fp16, the products summed in fp32 and the bias added, the result rounded once to fp16; LeakyReLU acts on that fp16 value (a
negative one is rounded again after x * slope, as leaky_relu on an fp16 tensor does); the skip layer's encoded-input columns
are rounded like layer 0's (autocast promotes cat([input, x]) to fp32 and casts it back).

  autocast_stack  the same F.linear / leaky_relu stack run under torch.autocast("cuda", dtype=torch.float16)
  emulate_fp64    the arithmetic written out: exact fp64 sums of the fp16 operands, rounded to fp32 and then to fp16

Both return the net's output (fp32) and a per-entry tolerance against another implementation of the contract.  Two
implementations that sum in different orders get fp32 sums a few fp32 ulps apart; where such a sum lies next to an fp16
rounding boundary the two roundings differ by one fp16 ulp of the value, and that difference travels on through the later
layers.  Per layer, from the reference's own values (z the layer's fp16 result, x its input, e_in the input's difference
scale, zero for the encoded input, which is the same fp32 tensor on both sides):
    prop = sqrt(W16^2 e_in^2 + (2^-18 (|W16| |x| + |b16|))^2)   (differences reaching the fp32 sum, and summation order)
    e    = sqrt(prop^2 + ulp16(|z| + prop)^2)                    (each value may also round one fp16 ulp the other way)
after LeakyReLU e is scaled by the slope where z stays negative, and the second rounding of x * slope adds its ulp in
quadrature.  Differences of independent roundings add in quadrature, and e counts every entry of every layer as flipped, so
it overstates what reaches a layer; the last layer's tolerance is
    tol  = ulp16(|z| + K prop) + K prop,  K = 8
one fp16 ulp of the value plus a margin over what the earlier layers can carry into it.  A first layer may differ by one
ulp and the margin on the summation-order term, and nothing more.  Past the first layer the margin is wide.  On the seeded
nets of tests/sweep_cases.py with uniform inputs, tol is a median of 6-17 fp16 ulps of the head, with a 99th percentile of
330-850 and a maximum of 2.4e3-2.2e4.  So it only guards where the two sums may legitimately differ; where they do not, the
tests hold the heads to one fp16 ulp.  (The worst case, |W16| e_in summed without signs, grows by
about the fan-in times the weight scale per layer and exceeds the heads themselves past three or four layers.)
"""
import torch
import torch.nn.functional as F

SUM_ORDER = 2.0 ** -18  # fp32 summation-order difference, relative to the sum of magnitudes (K <= 320 terms)
MARGIN = 8.0            # K above: the last layer's allowance for what earlier layers carry into it


def ulp16(v):
    """One fp16 ulp at magnitude |v| (fp64): 2^(e - 10) for a normal value of exponent e, 2^-24 among the subnormals."""
    a = v.abs().clamp_min(2.0 ** -14)
    return torch.exp2(torch.floor(torch.log2(a)) - 10.0)


def _rn16(t):
    """fp32 -> the nearest fp16 value, as fp64 (a tensor of another dtype is rounded to fp32 first, as an fp32 sum is)."""
    return t.float().half().double()


def _tolerance_step(e_in, x, w16, b16, z, hidden, slope):
    """-> (e: the layer's difference scale for the next layer, tol: its tolerance if it is the last layer)."""
    order = SUM_ORDER * (x.abs() @ w16.abs().t() + b16.abs())
    prop = order if e_in is None else torch.sqrt(e_in ** 2 @ (w16 ** 2).t() + order ** 2)
    mag = z.abs() + prop
    e = torch.sqrt(prop ** 2 + ulp16(mag) ** 2)
    if hidden:  # LeakyReLU scales a difference of values that stay negative by the slope; one more rounding of x * slope
        e = torch.where(z.abs() > e, torch.where(z > 0, e, slope * e), e)
        e = torch.sqrt(e ** 2 + torch.where(z > 0, 0.0, ulp16(slope * mag)) ** 2)
    tol = ulp16(z.abs() + MARGIN * prop) + MARGIN * prop
    return e, tol


def emulate_fp64(enc, params, skip, slope):
    """enc: [n, mlp_in] fp32 encoded input (reference feature order); params: [w0, b0, w1, b1, ...] in the reference's layout.
    -> (output [n, out] fp32, tolerance [n, out] fp64)."""
    x_in = _rn16(enc.to(torch.float32))
    x, e = x_in, None
    n_layers = len(params) // 2
    s32 = torch.tensor(slope, dtype=torch.float32)
    for i in range(n_layers):
        w16, b16 = _rn16(params[2 * i].detach()), _rn16(params[2 * i + 1].detach())
        if i == skip:
            x = torch.cat([x_in, x], -1)
            e = torch.cat([torch.zeros_like(x_in), e], -1)
        hidden = i < n_layers - 1
        z = _rn16(x @ w16.t() + b16)  # fp64 sum of fp16 products, rounded to fp32, then to fp16
        e, tol = _tolerance_step(e, x, w16, b16, z, hidden, slope)
        if hidden:
            z = torch.where(z > 0, z, (z.float() * s32).half().double())  # x * slope in fp32, rounded to fp16
        x = z
    return x.float(), tol


def autocast_stack(enc, params, skip, slope):
    """The reference's layers under CUDA autocast (enc and params on a CUDA device) -> (output fp32, tolerance fp64)."""
    n_layers = len(params) // 2
    x, e = enc, None
    x_in16 = _rn16(enc)
    with torch.autocast("cuda", dtype=torch.float16):
        for i in range(n_layers):
            w, b = params[2 * i], params[2 * i + 1]
            xin = x
            if i == skip:
                xin = torch.cat([enc, x], -1)  # fp32 and fp16: promoted to fp32, cast back by F.linear
                e = torch.cat([torch.zeros_like(x_in16), e], -1)
            z = F.linear(xin, w, b)
            assert z.dtype == torch.float16
            hidden = i < n_layers - 1
            with torch.autocast("cuda", enabled=False):
                e, tol = _tolerance_step(e, _rn16(xin), _rn16(w.detach()), _rn16(b.detach()), z.double(), hidden, slope)
            x = F.leaky_relu(z, slope) if hidden else z
    return x.float(), tol


def ulps_apart(a, b):
    """How many fp16 values lie between a and b (fp32 tensors of fp16 values, same sign conventions as the fp16 bit order)."""
    def key(t):
        i = t.half().view(torch.int16).to(torch.int32)
        return torch.where(i < 0, -(i & 0x7FFF), i)
    return (key(a) - key(b)).abs()
