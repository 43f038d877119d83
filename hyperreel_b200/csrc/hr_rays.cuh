// Camera -> ray arithmetic, one definition shared by generate_rays_kernel (hr_rays.cu) and the training-batch kernel
// (hr_train_batch.cu): a training row must be bit-identical to the row hr_generate_rays writes for the same pixel.
// Reference: get_ray_directions_from_pixels_K / get_rays / get_ndc_rays_fx_fy (utils/ray_utils.py:98-164) as driven by
// get_coords_from_camera (datasets/base.py:485-518).
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

// The ray of pixel (x, y) as the reference's coords row: origin, direction, then cam_idx and time (channels 6 and 7 when
// c_in == 8, technicolor.py:389-393).
__device__ __forceinline__ void camera_ray(const hr_camera& cam, int x, int y, NdcScale ndc, float (&row)[8]) {
  const float px = (float)x, py = (float)y;
  const float off = cam.centered_pixels ? 0.5f : 0.0f;
  // get_ray_directions_from_pixels_K (ray_utils.py:98-115)
  const float dcx = __fdiv_rn(__fadd_rn(__fsub_rn(px, cam.cx), off), cam.fx);
  float dcy = __fdiv_rn(__fadd_rn(__fsub_rn(py, cam.cy), off), cam.fy);
  if (!cam.flipped) dcy = -dcy;
  const float dcz = -1.0f;
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
