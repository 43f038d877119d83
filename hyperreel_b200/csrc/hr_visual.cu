// Embedding maps that need the whole frame: visualize_warp's `normalize` (utils/visualization.py:46-49), the per-channel
// min / max over a frame's pixels, then the map to uint8.  The elementwise maps are finished in the render kernel's epilogue
// (VisMap, hr_render_kernel.cuh); hr_render_visuals (hr_api.cu) stages the fields these kernels read.
#include "hr_common.cuh"

namespace hr {

constexpr int kVisThreads = 256;

// torch.min / torch.max: a NaN anywhere makes the result NaN (once m is NaN, neither test can replace it)
__device__ __forceinline__ float nan_min(float m, float v) { return (v < m || v != v) ? v : m; }
__device__ __forceinline__ float nan_max(float m, float v) { return (v > m || v != v) ? v : m; }

// Block b of frame y: min and max of each channel of vis_pre(x) over its pixels, into part[((y * kVisBlocks + b) * 3 + c) * 2].
// The tree is fixed and min / max are exact, so the partials do not depend on scheduling.
__global__ void __launch_bounds__(kVisThreads) vis_minmax_kernel(const float* __restrict__ x, long long px, int dim,
                                                                 const __grid_constant__ VisMap m, float* __restrict__ part) {
  __shared__ float s_mn[3][kVisThreads], s_mx[3][kVisThreads];
  const float* fx = x + (long long)blockIdx.y * px * dim;
  float mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (long long p = (long long)blockIdx.x * kVisThreads + threadIdx.x; p < px; p += (long long)kVisBlocks * kVisThreads)
    for (int c = 0; c < dim; ++c) {
      const float v = vis_pre(m, fx[p * dim + c]);
      mn[c] = nan_min(mn[c], v);
      mx[c] = nan_max(mx[c], v);
    }
  for (int c = 0; c < 3; ++c) { s_mn[c][threadIdx.x] = mn[c]; s_mx[c][threadIdx.x] = mx[c]; }
  __syncthreads();
  for (int w = kVisThreads / 2; w > 0; w >>= 1) {
    if ((int)threadIdx.x < w)
      for (int c = 0; c < 3; ++c) {
        s_mn[c][threadIdx.x] = nan_min(s_mn[c][threadIdx.x], s_mn[c][threadIdx.x + w]);
        s_mx[c][threadIdx.x] = nan_max(s_mx[c][threadIdx.x], s_mx[c][threadIdx.x + w]);
      }
    __syncthreads();
  }
  if (threadIdx.x < 3) {
    float* o = part + (((long long)blockIdx.y * kVisBlocks + blockIdx.x) * 3 + threadIdx.x) * 2;
    o[0] = s_mn[threadIdx.x][0];
    o[1] = s_mx[threadIdx.x][0];
  }
}

// Frame y's map: (vis_pre(x) - min) / (max - min), max - min rounded once, then clamp and to8b, into m.out's frame y.
__global__ void __launch_bounds__(kVisThreads) vis_map_kernel(const float* __restrict__ x, long long px, int dim,
                                                              const __grid_constant__ VisMap m, const float* __restrict__ part) {
  __shared__ float s_lo[3], s_den[3];
  if (threadIdx.x < 3) {
    const float* q = part + (long long)blockIdx.y * kVisBlocks * 6 + threadIdx.x * 2;
    float mn = INFINITY, mx = -INFINITY;
    for (int b = 0; b < kVisBlocks; ++b) {
      mn = nan_min(mn, q[b * 6]);
      mx = nan_max(mx, q[b * 6 + 1]);
    }
    s_lo[threadIdx.x] = mn;
    s_den[threadIdx.x] = __fsub_rn(mx, mn);
  }
  __syncthreads();
  const long long base = (long long)blockIdx.y * px * dim, total = px * dim;
  for (long long i = (long long)blockIdx.x * kVisThreads + threadIdx.x; i < total; i += (long long)gridDim.x * kVisThreads) {
    const int c = (int)(i % dim);
    const float v = __fdiv_rn(__fsub_rn(vis_pre(m, x[base + i]), s_lo[c]), s_den[c]);
    m.out[base + i] = vis_to8b(v);
  }
}

// nf consecutive frames [nf][px][dim] of fp32 field values -> their uint8 maps at m.out ([nf][px][dim]).  part: kVisBlocks * 6
// floats per frame, used by this launch pair only.
cudaError_t launch_vis_normalize(const float* x, int nf, long long px, int dim, const VisMap& m, float* part, cudaStream_t st) {
  vis_minmax_kernel<<<dim3(kVisBlocks, nf), kVisThreads, 0, st>>>(x, px, dim, m, part);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  long long blocks = (px * dim + kVisThreads - 1) / kVisThreads;
  if (blocks > 1024) blocks = 1024;
  vis_map_kernel<<<dim3((unsigned)blocks, nf), kVisThreads, 0, st>>>(x, px, dim, m, part);
  return cudaGetLastError();
}

}  // namespace hr
