// Camera -> rays on the device (the step before the hot path).
// Reference: get_coords_from_camera (datasets/base.py:485-518).  One thread per pixel, rays written as [n, c_in] fp32; the
// per-pixel arithmetic is camera_ray (hr_rays.cuh), in its fisheye instantiation for a fisheye record only, or lightfield_ray
// for a two-plane record.
#include "hr_rays.cuh"

namespace hr {

// The camera model of generate_rays_kernel's one record, chosen on the host.
enum CameraModel : int { kPinholeModel = 0, kFisheyeModel = 1, kTwoPlaneModel = 2 };

template <int kModel>
__global__ void generate_rays_kernel(const __grid_constant__ hr_camera cam, int c_in, long long first, long long n,
                                     NdcScale ndc, float* __restrict__ out) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long p = first + i;
    float row[8];
    if constexpr (kModel == kTwoPlaneModel) lightfield_ray(cam, (int)(p % cam.width), (int)(p / cam.width), row);
    else camera_ray<kModel == kFisheyeModel>(cam, (int)(p % cam.width), (int)(p / cam.width), ndc, row);
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
  if (cam.two_plane) generate_rays_kernel<kTwoPlaneModel><<<(unsigned)g, 256, 0, st>>>(cam, c_in, first, n, NdcScale{}, out);
  else if (cam.fisheye) generate_rays_kernel<kFisheyeModel><<<(unsigned)g, 256, 0, st>>>(cam, c_in, first, n, ndc_scale(cam), out);
  else generate_rays_kernel<kPinholeModel><<<(unsigned)g, 256, 0, st>>>(cam, c_in, first, n, ndc_scale(cam), out);
  return cudaGetLastError();
}

// Rays of a video (hr_render_video_to8b): global ray p = f * frame_px + y * width + x over n_frames records of one size,
// rays first .. first + n - 1 of that sequence, so a batch may span frame boundaries.  Ray p is camera_ray of record f,
// bit-identical to the row generate_rays_kernel writes for that record's pixel, with times[f] in the time column.  kMixed:
// the host instantiates it when any record of the video is not a pinhole, and then each row branches on its own record's
// fisheye and two_plane flags, so one batch may mix the three camera models; without it every record is a pinhole.
template <bool kMixed>
__global__ void generate_video_rays_kernel(const hr_camera* __restrict__ cams, const float* __restrict__ times, int c_in,
                                           int width, long long frame_px, long long first, long long n,
                                           float* __restrict__ out) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long p = first + i;
    const long long f = p / frame_px, q = p - f * frame_px;
    const hr_camera& cam = cams[f];
    float row[8];
    camera_ray<kMixed, kMixed>(cam, (int)(q % width), (int)(q / width), ndc_scale(cam), row);
    float* r = out + i * c_in;
    r[0] = row[0]; r[1] = row[1]; r[2] = row[2];
    r[3] = row[3]; r[4] = row[4]; r[5] = row[5];
    if (c_in >= 8) { r[6] = row[6]; r[7] = times[f]; }
  }
}

cudaError_t launch_generate_video_rays(const hr_camera* cams, const float* times, bool mixed, int c_in, int width,
                                       long long frame_px, long long first, long long n, float* out, cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  long long g = (n + 255) / 256;
  if (g > 148 * 16) g = 148 * 16;
  if (mixed) generate_video_rays_kernel<true><<<(unsigned)g, 256, 0, st>>>(cams, times, c_in, width, frame_px, first, n, out);
  else generate_video_rays_kernel<false><<<(unsigned)g, 256, 0, st>>>(cams, times, c_in, width, frame_px, first, n, out);
  return cudaGetLastError();
}

}  // namespace hr
