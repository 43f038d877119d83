// Held-out view scoring: per-image MSE and SSIM of [n, H, W, 3] image pairs on the device, the prediction fp32 and the
// ground truth fp32 or uint8.
// Reference: metrics.psnr / metrics.ssim (metrics.py:25-34), i.e. scikit-image's peak_signal_noise_ratio(data_range=1) and
// structural_similarity(win_size=11, multichannel, gaussian_weights, data_range=1), called by INRSystem.validation_image
// (nlf/__init__.py:976-980) on the host copy of every held-out frame.
//
// One CTA per 32x16 tile of one image.  It stages the tile plus a 5-pixel halo of both images in shared memory, runs the
// vertical 11-tap pass of the five moments (ux, uy, uxx, uyy, uxy) into fp64 shared rows, then the horizontal pass and the
// SSIM map per output pixel, all in fp64.  Only pixels in [5, H-5) x [5, W-5) are evaluated: the crop radius of the mean equals
// the filter radius, so no window that reaches the result leaves the image and SciPy's `reflect` border never matters.  The
// same CTA sums the squared error of its own tile (border pixels included).  Per-tile partials go to the workspace and a
// second kernel sums each image's partials in a fixed order: no float atomics, so results are bit-reproducible and do not
// depend on the batch an image is scored in.
//
// uint8 ground truth (hr_score_views) is converted while the tile is staged, as u8 / 255 correctly rounded: what
// T.ToTensor() (a CPU division) gives the reference, and what the training batches use.  RGBA ground truth (the DoNeRF and
// Catacaustics datasets) is composited over white while it is staged, rgb * a + (1 - a) of those values with each operation
// rounded on its own (no FMA), as their get_rgb computes it with torch on the CPU.  Everything after staging is shared, so a
// uint8 frame scores bit for bit like that fp32 conversion (or composite) of it.
#include <cmath>
#include <cstdint>
#include <type_traits>

#include "hr_handle.h"

namespace {

constexpr int MT_W = 32, MT_H = 16;                    // output tile
constexpr int MR = 5;                                  // Gaussian radius int(3.5 * 1.5 + 0.5)
constexpr int MTAPS = 2 * MR + 1;
constexpr int SW = MT_W + 2 * MR, SH = MT_H + 2 * MR;  // staged region 42 x 26
constexpr int MP = SW + 1;      // fp64 moment row pitch; odd, so the horizontal pass's column-strided reads are conflict-free
constexpr int MTHREADS = 256;
constexpr int VR = 8;           // output rows per thread of the vertical pass:   3 channels x 2 x 42 columns = 252 threads
constexpr int HC = 8;           // output columns per thread of the horizontal pass: 3 channels x 16 rows x 4 = 192 threads

struct GaussTaps {
  double w[MTAPS];
};

struct MetricsSmem {
  float x[3][SH][SW];         // pred, channel-planar
  float y[3][SH][SW];         // gt
  double m[3][5][MT_H][MP];   // vertically filtered ux, uy, uxx, uyy, uxy
  double red[2][MTHREADS / 32];
};

// Sums a and b over the CTA in a fixed order; the totals are valid in thread 0.
__device__ __forceinline__ void block_sum2(double& a, double& b, double (*red)[MTHREADS / 32]) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    a += __shfl_down_sync(0xffffffffu, a, off);
    b += __shfl_down_sync(0xffffffffu, b, off);
  }
  const int warp = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) {
    red[0][warp] = a;
    red[1][warp] = b;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    a = 0.0;
    b = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) {
      a += red[0][w];
      b += red[1][w];
    }
  }
}

__device__ __forceinline__ float load_gt(const float* p) { return __ldg(p); }
__device__ __forceinline__ float load_gt(const uint8_t* p) { return hr::u8_unit(__ldg(p)); }

// One RGBA uint8 pixel, loaded whole
struct __align__(4) Rgba8 {
  uint8_t v[4];
};

// Channel ch of an RGBA pixel composited over white
__device__ __forceinline__ float load_gt(const Rgba8* p, int ch) {
  return hr::rgba_over_white(__ldg(reinterpret_cast<const unsigned int*>(p)), ch);
}

template <typename GtT>
__global__ void __launch_bounds__(MTHREADS, 2)
image_metrics_tile_kernel(const float* __restrict__ pred, const GtT* __restrict__ gt, int H, int W,
                          const __grid_constant__ GaussTaps g, double* __restrict__ partial) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  MetricsSmem& s = *reinterpret_cast<MetricsSmem*>(smem_raw);
  const int tid = threadIdx.x;
  const int r0 = blockIdx.y * MT_H, c0 = blockIdx.x * MT_W;
  const size_t base = (size_t)blockIdx.z * H * W * 3;

  // Stage rows r0-5 .. r0+20 and columns c0-5 .. c0+36.  Positions outside the image are zero: they only reach pixels the
  // SSIM mean crops.  The squared error of the tile's own pixels is summed on the way (fp32 difference and square).  All of
  // a thread's loads are issued before the first store, so their latencies overlap.
  constexpr int N_STAGE = SH * SW * 3, STAGE_ITERS = (N_STAGE + MTHREADS - 1) / MTHREADS;
  float xs[STAGE_ITERS], ys[STAGE_ITERS];
#pragma unroll
  for (int it = 0; it < STAGE_ITERS; ++it) {
    const int e = tid + it * MTHREADS;
    const int row = e / (SW * 3), q = e - row * (SW * 3), col = q / 3, ch = q - col * 3;
    const int r = r0 - MR + row, c = c0 - MR + col;
    xs[it] = 0.0f;
    ys[it] = 0.0f;
    if (e < N_STAGE && r >= 0 && r < H && c >= 0 && c < W) {
      const size_t i = base + ((size_t)r * W + c) * 3 + ch;
      xs[it] = __ldg(pred + i);
      if constexpr (std::is_same<GtT, Rgba8>::value)
        ys[it] = load_gt(gt + (size_t)blockIdx.z * H * W + (size_t)r * W + c, ch);
      else
        ys[it] = load_gt(gt + i);
    }
  }
  double sse = 0.0;
#pragma unroll
  for (int it = 0; it < STAGE_ITERS; ++it) {
    const int e = tid + it * MTHREADS;
    if (e >= N_STAGE) break;
    const int row = e / (SW * 3), q = e - row * (SW * 3), col = q / 3, ch = q - col * 3;
    if (row >= MR && row < MR + MT_H && col >= MR && col < MR + MT_W && r0 - MR + row < H && c0 - MR + col < W) {
      const float d = __fsub_rn(xs[it], ys[it]);
      sse += (double)__fmul_rn(d, d);
    }
    s.x[ch][row][col] = xs[it];
    s.y[ch][row][col] = ys[it];
  }
  __syncthreads();

  // Vertical pass: moment k of output row i, staged column col = sum_t w[t] * p_k(row i + t).  fp64 products of fp32 values
  // are exact.
  if (tid < 3 * 2 * SW) {
    const int ch = tid / (2 * SW), rem = tid - ch * (2 * SW), half = rem / SW, col = rem - half * SW;
    const int i0 = half * VR;
    double acc[VR][5];
#pragma unroll
    for (int i = 0; i < VR; ++i)
#pragma unroll
      for (int k = 0; k < 5; ++k) acc[i][k] = 0.0;
#pragma unroll
    for (int t = 0; t < VR + 2 * MR; ++t) {
      const double xv = s.x[ch][i0 + t][col], yv = s.y[ch][i0 + t][col];
      const double p[5] = {xv, yv, xv * xv, yv * yv, xv * yv};
#pragma unroll
      for (int i = 0; i < VR; ++i) {
        const int k = t - i;
        if (k >= 0 && k < MTAPS) {
#pragma unroll
          for (int m = 0; m < 5; ++m) acc[i][m] = fma(g.w[k], p[m], acc[i][m]);
        }
      }
    }
#pragma unroll
    for (int i = 0; i < VR; ++i)
#pragma unroll
      for (int m = 0; m < 5; ++m) s.m[ch][m][i0 + i][col] = acc[i][m];
  }
  __syncthreads();

  // Horizontal pass and the SSIM map (skimage's formula, each op rounded as NumPy rounds it), summed over interior pixels.
  double ssum = 0.0;
  if (tid < 3 * MT_H * (MT_W / HC)) {
    const int ch = tid / (MT_H * (MT_W / HC)), rem = tid - ch * (MT_H * (MT_W / HC)), jg = rem / MT_H, i = rem - jg * MT_H;
    const int j0 = jg * HC;
    double acc[HC][5];
#pragma unroll
    for (int j = 0; j < HC; ++j)
#pragma unroll
      for (int k = 0; k < 5; ++k) acc[j][k] = 0.0;
#pragma unroll
    for (int t = 0; t < HC + 2 * MR; ++t) {
      double p[5];
#pragma unroll
      for (int m = 0; m < 5; ++m) p[m] = s.m[ch][m][i][j0 + t];
#pragma unroll
      for (int j = 0; j < HC; ++j) {
        const int k = t - j;
        if (k >= 0 && k < MTAPS) {
#pragma unroll
          for (int m = 0; m < 5; ++m) acc[j][m] = fma(g.w[k], p[m], acc[j][m]);
        }
      }
    }
    const int r = r0 + i;
    if (r >= MR && r < H - MR) {
      constexpr double cov_norm = 121.0 / 120.0;  // sample covariance over the 11 x 11 window
      constexpr double C1 = 0.01 * 0.01, C2 = 0.03 * 0.03;
#pragma unroll
      for (int j = 0; j < HC; ++j) {
        const int c = c0 + j0 + j;
        if (c < MR || c >= W - MR) continue;
        const double ux = acc[j][0], uy = acc[j][1], uxx = acc[j][2], uyy = acc[j][3], uxy = acc[j][4];
        const double vx = __dmul_rn(cov_norm, __dsub_rn(uxx, __dmul_rn(ux, ux)));
        const double vy = __dmul_rn(cov_norm, __dsub_rn(uyy, __dmul_rn(uy, uy)));
        const double vxy = __dmul_rn(cov_norm, __dsub_rn(uxy, __dmul_rn(ux, uy)));
        const double A1 = __dadd_rn(__dmul_rn(__dmul_rn(2.0, ux), uy), C1);
        const double A2 = __dadd_rn(__dmul_rn(2.0, vxy), C2);
        const double B1 = __dadd_rn(__dadd_rn(__dmul_rn(ux, ux), __dmul_rn(uy, uy)), C1);
        const double B2 = __dadd_rn(__dadd_rn(vx, vy), C2);
        ssum += __ddiv_rn(__dmul_rn(A1, A2), __dmul_rn(B1, B2));
      }
    }
  }

  block_sum2(sse, ssum, s.red);
  if (tid == 0) {
    double* p = partial + 2 * (((size_t)blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x);
    p[0] = sse;
    p[1] = ssum;
  }
}

// One CTA per image: the image's tile partials summed in a fixed order, then the two means.
__global__ void __launch_bounds__(MTHREADS)
image_metrics_reduce_kernel(const double* __restrict__ partial, int tiles, double n_values, double n_interior,
                            double* __restrict__ out) {
  __shared__ double red[2][MTHREADS / 32];
  const double* p = partial + 2 * (size_t)blockIdx.x * tiles;
  double sse = 0.0, ssum = 0.0;
  for (int t = threadIdx.x; t < tiles; t += MTHREADS) {
    sse += p[2 * t];
    ssum += p[2 * t + 1];
  }
  block_sum2(sse, ssum, red);
  if (threadIdx.x == 0) {
    out[2 * blockIdx.x] = sse / n_values;
    out[2 * blockIdx.x + 1] = ssum / n_interior;
  }
}

bool metrics_args_ok(int32_t n, int32_t h, int32_t w) {
  return n >= 1 && n <= 65535 && h >= MTAPS && w >= MTAPS;
}

int64_t metrics_tiles(int32_t h, int32_t w) {
  return (int64_t)((h + MT_H - 1) / MT_H) * ((w + MT_W - 1) / MT_W);
}

// SciPy's _gaussian_kernel1d(sigma=1.5, order=0, radius=5): exp(-0.5 / sigma^2 * x^2), normalised by NumPy's sum of the 11
// values (pairwise: eight partial sums combined as a tree, then the last three added in order)
GaussTaps gauss_taps() {
  GaussTaps g;
  const double sigma2 = 1.5 * 1.5;
  for (int t = 0; t < MTAPS; ++t) g.w[t] = std::exp(-0.5 / sigma2 * (double)((t - MR) * (t - MR)));
  double sum = ((g.w[0] + g.w[1]) + (g.w[2] + g.w[3])) + ((g.w[4] + g.w[5]) + (g.w[6] + g.w[7]));
  for (int t = 8; t < MTAPS; ++t) sum += g.w[t];
  for (int t = 0; t < MTAPS; ++t) g.w[t] /= sum;
  return g;
}

// The tile kernel and the per-image reduction of n images on `st`; `partial` holds hr_image_metrics_workspace_bytes(n, H, W).
template <typename GtT>
cudaError_t launch_metrics(const float* pred, const GtT* gt, int32_t n, int32_t H, int32_t W, double* out, double* partial,
                           cudaStream_t st) {
  const cudaError_t e = cudaFuncSetAttribute(image_metrics_tile_kernel<GtT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             (int)sizeof(MetricsSmem));
  if (e != cudaSuccess) return e;
  const dim3 grid((W + MT_W - 1) / MT_W, (H + MT_H - 1) / MT_H, n);
  image_metrics_tile_kernel<GtT><<<grid, MTHREADS, sizeof(MetricsSmem), st>>>(pred, gt, H, W, gauss_taps(), partial);
  image_metrics_reduce_kernel<<<n, MTHREADS, 0, st>>>(partial, (int)metrics_tiles(H, W), 3.0 * H * W,
                                                      3.0 * (H - 2 * MR) * (W - 2 * MR), out);
  return cudaGetLastError();
}

}  // namespace

namespace hr {

// hr_score_views' scoring of whole frames of its fp32 ring against their uint8 ground truth (arguments checked by the caller)
cudaError_t launch_image_metrics_u8(const float* pred, const uint8_t* gt, int32_t n, int32_t H, int32_t W, double* out,
                                    double* partial, cudaStream_t st) {
  return launch_metrics(pred, gt, n, H, W, out, partial, st);
}

// The same against RGBA uint8 ground truth [n][H][W][4] (4-byte aligned), composited over white while it is staged
cudaError_t launch_image_metrics_rgba8(const float* pred, const uint8_t* gt, int32_t n, int32_t H, int32_t W, double* out,
                                       double* partial, cudaStream_t st) {
  return launch_metrics(pred, reinterpret_cast<const Rgba8*>(gt), n, H, W, out, partial, st);
}

}  // namespace hr

extern "C" {

int64_t hr_image_metrics_workspace_bytes(int32_t n_images, int32_t height, int32_t width) {
  if (!metrics_args_ok(n_images, height, width)) return -1;
  return (int64_t)n_images * metrics_tiles(height, width) * 2 * (int64_t)sizeof(double);
}

int hr_image_metrics(const float* pred, const float* gt, int32_t n_images, int32_t height, int32_t width, double* out,
                     void* workspace, int64_t workspace_bytes, void* stream) {
  if (!pred || !gt || !out || !workspace) return hr_fail("hr_image_metrics: null argument");
  if (n_images < 1 || n_images > 65535) return hr_fail("hr_image_metrics: n_images must be in [1, 65535], got %d", n_images);
  if (height < MTAPS || width < MTAPS)
    return hr_fail("hr_image_metrics: height and width must be >= %d (the SSIM window), got %d x %d", MTAPS, height, width);
  if (((uintptr_t)out | (uintptr_t)workspace) % alignof(double) != 0)
    return hr_fail("hr_image_metrics: out and workspace must be 8-byte aligned");
  const int64_t need = hr_image_metrics_workspace_bytes(n_images, height, width);
  if (workspace_bytes < need)
    return hr_fail("hr_image_metrics: workspace of %lld bytes, %lld needed", (long long)workspace_bytes, (long long)need);

  const cudaError_t e = launch_metrics(pred, gt, n_images, height, width, out, (double*)workspace, (cudaStream_t)stream);
  if (e != cudaSuccess) return hr_fail("hr_image_metrics: %s", cudaGetErrorString(e));
  return 0;
}

}  // extern "C"
