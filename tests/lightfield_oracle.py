"""NumPy fp32 restatement of the two-plane light-field rays (get_lightfield_rays, utils/ray_utils.py:14-45) as torch's CPU
kernels evaluate them, and so as lightfield_ray (csrc/hr_rays.cuh) evaluates them on the device: every operation is one
rounded fp32 operation (NumPy float32 arithmetic does not contract).

- torch.linspace(start, end, steps): step = (end - start) / (steps - 1), fma(step, i, start) below steps // 2,
  fma(-step, steps - 1 - i, end) from it; [start] for one step.  torch's CPU kernel is compiled with contraction, so the
  products and sums fuse.
- A Python scalar meeting an fp32 tensor is rounded to fp32 first: ones * s * st_scale is fl(fl32(s) * fl32(st_scale)).
- far - near is subtracted in double by the reference and rounded once.
- F.normalize: x / max(sqrt(fma(x2, x2, fma(x1, x1, x0 * x0))), 1e-12), the order of torch's CPU norm kernel.

``fma32`` is an exact fp32 fused multiply-add: NumPy has none, and a sum in double rounded to fp32 rounds twice.
"""
import numpy as np

f32 = np.float32


def fma32(a, b, c):
    """fl32(a * b + c) with one rounding, elementwise, for fp32 arrays."""
    a, b, c = (np.asarray(v, f32).astype(np.float64) for v in (a, b, c))
    p = a * b  # exact: 24-bit by 24-bit significands
    s = p + c
    bp = s - c  # TwoSum: e is the rounding error of s
    e = (p - bp) + (c - (s - bp))
    r = s.astype(f32)
    # s rounded to fp32 is wrong only when s sits exactly between two fp32 values and e decides the side
    other = np.nextafter(r, np.where(s > r.astype(np.float64), f32(np.inf), f32(-np.inf)).astype(f32))
    mid = (r.astype(np.float64) + other.astype(np.float64)) / 2
    fix = (s != r.astype(np.float64)) & (s == mid) & (e != 0)
    up = np.maximum(r, other)
    down = np.minimum(r, other)
    return np.where(fix, np.where(e > 0, up, down), r).astype(f32)


def linspace(start, end, steps):
    start, end = f32(start), f32(end)
    if steps == 1:
        return np.array([start], f32)
    step = f32(end - start) / f32(steps - 1)
    i = np.arange(steps)
    lo = fma32(step, i.astype(f32), start)
    hi = fma32(-step, (steps - 1 - i).astype(f32), end)
    return np.where(i < steps // 2, lo, hi).astype(f32)


def lightfield_rays(W, H, s, t, st_scale=1.0, uv_scale=1.0, near=-1.0, far=0.0, aspect=None, pixels=None):
    """rays [n, 6] fp32 of the row-major ``pixels`` (default all) of a W x H two-plane view."""
    aspect = float(W) / float(H) if aspect is None else aspect
    u = linspace(-1.0, 1.0, W) * f32(uv_scale)
    v = (linspace(1.0, -1.0, H) / f32(aspect)) * f32(uv_scale)
    S, T = f32(s) * f32(st_scale), f32(t) * f32(st_scale)
    pixels = np.arange(W * H) if pixels is None else np.asarray(pixels)
    x, y = pixels % W, pixels // W
    d0, d1 = u[x] - S, v[y] - T
    d2 = np.full_like(d0, f32(float(far) - float(near)))
    nrm = np.maximum(np.sqrt(fma32(d2, d2, fma32(d1, d1, d0 * d0))), f32(1e-12))
    n = pixels.shape[0]
    return np.stack([np.full(n, S, f32), np.full(n, T, f32), np.full(n, f32(near), f32), d0 / nrm, d1 / nrm, d2 / nrm],
                    -1).astype(f32)


def camera_rays(cam, pixels=None):
    """The rows of a hyperreel_b200.TwoPlaneCamera (its float32 fields), [n, 8] with cam_idx and time."""
    r = lightfield_rays(cam.width, cam.height, cam.s, cam.t, cam.st_scale, cam.uv_scale, cam.near, cam.far,
                        float(cam.width) / cam.height if cam.aspect is None else cam.aspect, pixels)
    extra = np.broadcast_to(np.array([cam.cam_idx, cam.time], f32), (r.shape[0], 2))
    return np.concatenate([r, extra], -1)
