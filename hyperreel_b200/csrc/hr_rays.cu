// Camera -> rays on the device (the step before the hot path).
// Reference: get_coords_from_camera (datasets/base.py:485-518).  One thread per pixel, rays written as [n, c_in] fp32; the
// per-pixel arithmetic is camera_ray (hr_rays.cuh), in its fisheye instantiation for a fisheye record only.
#include "hr_rays.cuh"

namespace hr {

template <bool kFisheye>
__global__ void generate_rays_kernel(const __grid_constant__ hr_camera cam, int c_in, long long first, long long n,
                                     NdcScale ndc, float* __restrict__ out) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long p = first + i;
    float row[8];
    camera_ray<kFisheye>(cam, (int)(p % cam.width), (int)(p / cam.width), ndc, row);
    float* r = out + i * c_in;
    r[0] = row[0]; r[1] = row[1]; r[2] = row[2];
    r[3] = row[3]; r[4] = row[4]; r[5] = row[5];
    if (c_in >= 8) { r[6] = row[6]; r[7] = row[7]; }
  }
}

cudaError_t launch_generate_rays(const hr_camera& cam, int c_in, long long first, long long n, float* out, cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  long long g = (n + 255) / 256;
  if (g > 148 * 16) g = 148 * 16;
  if (cam.fisheye) generate_rays_kernel<true><<<(unsigned)g, 256, 0, st>>>(cam, c_in, first, n, ndc_scale(cam), out);
  else generate_rays_kernel<false><<<(unsigned)g, 256, 0, st>>>(cam, c_in, first, n, ndc_scale(cam), out);
  return cudaGetLastError();
}

}  // namespace hr
