// Camera -> ray arithmetic, one definition shared by generate_rays_kernel (hr_rays.cu) and the training-batch kernels
// (hr_train_batch.cu): a training row must be bit-identical to the row hr_generate_rays writes for the same pixel.
// Reference: get_ray_directions_from_pixels_K / get_rays / get_ndc_rays_fx_fy (utils/ray_utils.py:98-164) as driven by
// get_coords_from_camera (datasets/base.py:485-518), for fisheye cameras ImmersiveDataset.get_coords
// (datasets/immersive.py:494-573), and for two-plane light-field views get_lightfield_rays (utils/ray_utils.py:14-45).
#pragma once
#include "hr_common.cuh"

namespace hr {

// get_ndc_rays_fx_fy's scales ndc_sx = -1/(W/(2 fx)), ndc_sy = -1/(H/(2 fy)), in the reference's fp32 evaluation order (fx an
// fp32 tensor element).  Host and device evaluate it with IEEE round-to-nearest operations, so both give the same bits.
struct NdcScale {
  float sx, sy;
};

__host__ __device__ inline NdcScale ndc_scale(const hr_camera& cam) {
  return {-1.0f / ((float)cam.width / (2.0f * cam.fx)), -1.0f / ((float)cam.height / (2.0f * cam.fy))};
}

// The fisheye camera's direction for the pinhole direction (x, y, -1) (ImmersiveDataset.get_coords,
// datasets/immersive.py:514-551): cv::fisheye::undistortPoints of OpenCV 4.x with K = I, D = (k1, k2, 0, 0), no R or P and
// the default criteria (COUNT + EPS, 10 iterations, 1e-8), restated in fp64 in OpenCV's operation order with non-contracting
// intrinsics, so that only tan (CUDA's, <= 2 ulp) can differ from the host library, and only below fp32 resolution.  The
// zero k3, k4 terms are left out: they change nothing unless |theta| passes ~1e38, from which ten Newton steps cannot
// converge either way.  Then F.normalize of (u, v, -1) in fp32.
__device__ __forceinline__ float3 fisheye_direction(float xf, float yf, float k1f, float k2f) {
  const double x = xf, y = yf, k1 = k1f, k2 = k2f;
  constexpr double kHalfPi = 3.14159265358979323846 / 2.0;
  // the model holds up to 180 degrees of field of view: OpenCV clamps theta_d to [-pi/2, pi/2]
  const double theta_d = fmin(fmax(-kHalfPi, __dsqrt_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)))), kHalfPi);
  double theta = theta_d, scale = 0.0;
  bool converged = false;
  if (fabs(theta_d) > 1e-8) {
    for (int j = 0; j < 10; ++j) {  // Newton on theta * (1 + k1 theta^2 + k2 theta^4) = theta_d
      const double t2 = __dmul_rn(theta, theta), t4 = __dmul_rn(t2, t2);
      const double a = __dmul_rn(k1, t2), b = __dmul_rn(k2, t4);
      const double fix = __ddiv_rn(__dsub_rn(__dmul_rn(theta, __dadd_rn(__dadd_rn(1.0, a), b)), theta_d),
                                   __dadd_rn(__dadd_rn(1.0, __dmul_rn(3.0, a)), __dmul_rn(5.0, b)));
      theta = __dsub_rn(theta, fix);
      if (fabs(fix) < 1e-8) {
        converged = true;
        break;
      }
    }
    scale = __ddiv_rn(tan(theta), theta_d);
  } else {
    converged = true;  // the principal point: scale 0
  }
  const bool flipped = (theta_d < 0.0 && theta > 0.0) || (theta_d > 0.0 && theta < 0.0);
  float u = -1000000.0f, v = -1000000.0f;  // OpenCV's value for a point it cannot undistort
  if (converged && !flipped) {
    u = __double2float_rn(__dmul_rn(x, scale));
    v = __double2float_rn(__dmul_rn(y, scale));
  }
  float nrm = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(u, u), __fmul_rn(v, v)), 1.0f));
  nrm = fmaxf(nrm, 1e-12f);
  return make_float3(__fdiv_rn(u, nrm), __fdiv_rn(v, nrm), __fdiv_rn(-1.0f, nrm));
}

// Element i of torch.linspace(start, end, steps) in fp32 as torch's CPU kernel computes it: step = (end - start) / (steps - 1),
// start + step * i below the midpoint steps / 2 and end - step * (steps - 1 - i) from it, each a fused multiply-add (the
// kernel is compiled with contraction); [start] for one step.
__device__ __forceinline__ float torch_linspace(float start, float end, int steps, int i) {
  if (steps == 1) return start;
  const float step = __fdiv_rn(__fsub_rn(end, start), (float)(steps - 1));
  return i < steps / 2 ? __fmaf_rn(step, (float)i, start) : __fmaf_rn(-step, (float)(steps - 1 - i), end);
}

// The two-plane light-field ray of pixel (x, y) of a Stanford view (cam.two_plane; get_lightfield_rays, ray_utils.py:14-45):
// u = linspace(-1, 1, W)[x] * uv_scale, v = (linspace(1, -1, H)[y] / aspect) * uv_scale, S = s * st_scale, T = t * st_scale
// (the reference's `ones * s * st_scale`: s rounded to fp32, then one fp32 product), origin (S, T, near), direction
// F.normalize((u - S, v - T, far - near)): x / max(|x|, 1e-12) with torch's CPU norm, sqrt(fma(x2, x2, fma(x1, x1, x0 x0)))
// (not camera_ray's order: get_rays' norm is a different reduction).  Then cam_idx and time.
__device__ __forceinline__ void lightfield_ray(const hr_camera& cam, int x, int y, float (&row)[8]) {
  const float u = __fmul_rn(torch_linspace(-1.0f, 1.0f, cam.width, x), cam.lf_uv_scale);
  const float v = __fmul_rn(__fdiv_rn(torch_linspace(1.0f, -1.0f, cam.height, y), cam.lf_aspect), cam.lf_uv_scale);
  const float s = __fmul_rn(cam.lf_s, cam.lf_st_scale), t = __fmul_rn(cam.lf_t, cam.lf_st_scale);
  const float d0 = __fsub_rn(u, s), d1 = __fsub_rn(v, t), d2 = __fsub_rn(cam.lf_far, cam.lf_near);
  float nrm = sqrtf(__fmaf_rn(d2, d2, __fmaf_rn(d1, d1, __fmul_rn(d0, d0))));
  nrm = fmaxf(nrm, 1e-12f);
  row[0] = s; row[1] = t; row[2] = cam.lf_near;
  row[3] = __fdiv_rn(d0, nrm); row[4] = __fdiv_rn(d1, nrm); row[5] = __fdiv_rn(d2, nrm);
  row[6] = cam.cam_idx; row[7] = cam.time;
}

// The ray of pixel (x, y) as the reference's coords row: origin, direction, then cam_idx and time (channels 6 and 7 when
// c_in == 8, technicolor.py:389-393).  kFisheye: records with cam.fisheye set take the fisheye direction (fisheye_direction);
// without it every record is a pinhole.  The fp64 solve costs registers (DESIGN 4.4), out of line as well: a call keeps the
// caller's live values and the callee's in one budget.  So generate_rays_kernel, whose one record the host reads, has a
// pinhole instantiation with the pinhole path's registers; the training kernels read their records on the device and
// always branch on the flag.  kTwoPlane: records with cam.two_plane set are light-field views (lightfield_ray); without it
// the flag is not read, and the code is what it was before two-plane records existed.
template <bool kFisheye, bool kTwoPlane = false>
__device__ __forceinline__ void camera_ray(const hr_camera& cam, int x, int y, NdcScale ndc, float (&row)[8]) {
  if (kTwoPlane && cam.two_plane) {
    lightfield_ray(cam, x, y, row);
    return;
  }
  const float px = (float)x, py = (float)y;
  const float off = cam.centered_pixels ? 0.5f : 0.0f;
  // get_ray_directions_from_pixels_K (ray_utils.py:98-115)
  float dcx = __fdiv_rn(__fadd_rn(__fsub_rn(px, cam.cx), off), cam.fx);
  float dcy = __fdiv_rn(__fadd_rn(__fsub_rn(py, cam.cy), off), cam.fy);
  if (!cam.flipped) dcy = -dcy;
  float dcz = -1.0f;
  if (kFisheye && cam.fisheye) {
    const float3 f = fisheye_direction(dcx, dcy, cam.k1, cam.k2);
    dcx = f.x; dcy = f.y; dcz = f.z;
  }
  // get_rays (ray_utils.py:121-135): rays_d = directions @ c2w[:, :3].T ; rays_o = c2w[:, 3]
  float d[3], o[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    d[r] = fmaf(dcz, cam.c2w[r * 4 + 2], fmaf(dcy, cam.c2w[r * 4 + 1], __fmul_rn(dcx, cam.c2w[r * 4 + 0])));
    o[r] = cam.c2w[r * 4 + 3];
  }
  if (cam.normalize) {
    float nrm = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(d[0], d[0]), __fmul_rn(d[1], d[1])), __fmul_rn(d[2], d[2])));
    nrm = fmaxf(nrm, 1e-12f);
#pragma unroll
    for (int r = 0; r < 3; ++r) d[r] = __fdiv_rn(d[r], nrm);
  }
  if (cam.use_ndc) {
    // get_ndc_rays_fx_fy (ray_utils.py:137-164)
    const float t = __fdiv_rn(-__fadd_rn(cam.ndc_near, o[2]), d[2]);
#pragma unroll
    for (int r = 0; r < 3; ++r) o[r] = __fadd_rn(o[r], __fmul_rn(t, d[r]));
    const float ox_oz = __fdiv_rn(o[0], o[2]), oy_oz = __fdiv_rn(o[1], o[2]);
    const float o0 = __fmul_rn(ndc.sx, ox_oz);
    const float o1 = __fmul_rn(ndc.sy, oy_oz);
    const float o2 = __fadd_rn(1.0f, __fdiv_rn(__fmul_rn(2.0f, cam.ndc_near), o[2]));
    const float d0 = __fmul_rn(ndc.sx, __fsub_rn(__fdiv_rn(d[0], d[2]), ox_oz));
    const float d1 = __fmul_rn(ndc.sy, __fsub_rn(__fdiv_rn(d[1], d[2]), oy_oz));
    const float d2 = __fsub_rn(1.0f, o2);
    o[0] = o0; o[1] = o1; o[2] = o2;
    d[0] = d0; d[1] = d1; d[2] = d2;
  }
  row[0] = o[0]; row[1] = o[1]; row[2] = o[2];
  row[3] = d[0]; row[4] = d[1]; row[5] = d[2];
  row[6] = cam.cam_idx; row[7] = cam.time;
}

}  // namespace hr
