// Capture-resolution frames to the training resolution on the device, bit for bit as the datasets' get_rgb resize them.
// Reference: the get_rgb of datasets/technicolor.py, llff.py, spaces.py, stanford.py (Pillow's Image.resize with LANCZOS, then
// BOX when scale() reduced img_wh) and of datasets/neural_3d.py, immersive.py (cv2.resize; the interpolation flag they pass
// lands in the `dst` slot, so OpenCV runs its default INTER_LINEAR, which it sends to its INTER_AREA fast path at exactly 2x).
//
// Exactness by construction: the tap bounds and fixed-point coefficients are built here on the host in the precision and
// order of the library that defines them (tests/resize_oracle.py restates the same in NumPy), copied into the workspace with
// the launch, and the kernels only multiply and add integers:
// * Pillow (libImaging/Resample.c, 8 bits per channel): precompute_coeffs in double (the filter support scaled by the
//   reduction, bounds rounded by truncation, weights normalised by their sum), then (int)(k * 2^22 +- 0.5) with the sign of
//   k.  The horizontal pass runs over the rows the vertical pass reads and writes a uint8 intermediate (in the workspace)
//   clipped as Pillow clips (acc >> 22, clamped to [0, 255]); then the vertical pass.  Each accumulation starts at 2^21.  A
//   pass whose size does not change is skipped, as Pillow skips it.
// * OpenCV INTER_LINEAR (resizeGeneric_ with HResizeLinear / VResizeLinear for uchar): fx = (float)((d + 0.5) * scale - 0.5),
//   sx = floor(fx), taps clamped to the border, coefficients saturate_cast<short>(w * 2048) (round half to even); the row
//   sums are ints, and the vertical combine is ((b0 * (S0 >> 4)) >> 16) + ((b1 * (S1 >> 4)) >> 16) + 2) >> 2, which is
//   what OpenCV's scalar and vector code for 8 bits both compute.  One kernel does both passes per output pixel.
// * OpenCV INTER_AREA for integer factors (resizeAreaFast_): (sum + 2) >> 2 at 2 x 2, otherwise sum * (1.f / area) in fp32
//   rounded half to even.  The same kernel with a 1 x 1 box is the identity (both libraries copy a frame of the same size).
//
// RGBA (HR_PIXEL_RGBA8; datasets/donerf.py and catacaustics.py): OpenCV resamples the four channels independently; Pillow's
// Image.resize converts an RGBA image to premultiplied RGBa, resamples that and converts back, on every call, so the Pillow
// passes premultiply on load from the source and unpremultiply on the store into dst (Convert.c's rgbA2rgba / rgba2rgbA).
//
// No host synchronisation, no float atomics: two calls with the same arguments write the same bits.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <vector>

#include "hr_handle.h"

namespace {

constexpr int kPrecisionBits = 22;  // Pillow, 8 bits per channel
constexpr int kCoefBits = 11;       // OpenCV INTER_RESIZE_COEF_BITS
constexpr int kThreads = 256;

// ---- Pillow's filters and coefficient table, as Resample.c computes them
double box_filter(double x) { return (x > -0.5 && x <= 0.5) ? 1.0 : 0.0; }

double bicubic_filter(double x) {
  const double a = -0.5;
  if (x < 0.0) x = -x;
  if (x < 1.0) return ((a + 2.0) * x - (a + 3.0)) * x * x + 1;
  if (x < 2.0) return (((x - 5) * x + 8) * x - 4) * a;
  return 0.0;
}

double sinc_filter(double x) {
  if (x == 0.0) return 1.0;
  x = x * M_PI;
  return sin(x) / x;
}

double lanczos_filter(double x) { return (-3.0 <= x && x < 3.0) ? sinc_filter(x) * sinc_filter(x / 3) : 0.0; }

// The filter support scaled by the reduction and the taps per output (precompute_coeffs), in 64 bits: Pillow's own
// `outSize > INT_MAX / (ksize * sizeof(double))` refusal bounds it, and pil_plan_ok applies that refusal before any table.
struct PilSupport {
  double scale, filterscale, support;
  int64_t ksize;
};

PilSupport pil_support(int in_size, int out_size, int method) {
  const double fsupport = method == HR_RESIZE_PIL_LANCZOS ? 3.0 : method == HR_RESIZE_PIL_BICUBIC ? 2.0 : 0.5;
  const double in0 = 0.0, in1 = (double)(float)in_size;
  double filterscale, scale;
  filterscale = scale = (in1 - in0) / out_size;
  if (filterscale < 1.0) filterscale = 1.0;
  const double support = fsupport * filterscale;
  return {scale, filterscale, support, (int64_t)ceil(support) * 2 + 1};
}

bool pil_plan_ok(int in_size, int out_size, int method) {
  const int64_t ksize = pil_support(in_size, out_size, method).ksize;
  return (int64_t)out_size <= INT32_MAX / (ksize * (int64_t)sizeof(double));
}

// One axis: per output index (first tap, tap count) followed by ksize fixed-point coefficients, [out][2 + ksize] int32.
std::vector<int32_t> pil_table(int in_size, int out_size, int method, int* ksize_out) {
  double (*filter)(double) = method == HR_RESIZE_PIL_LANCZOS ? lanczos_filter
                             : method == HR_RESIZE_PIL_BICUBIC ? bicubic_filter : box_filter;
  const PilSupport ps = pil_support(in_size, out_size, method);
  const double in0 = 0.0, scale = ps.scale, filterscale = ps.filterscale, support = ps.support;
  const int ksize = (int)ps.ksize;
  *ksize_out = ksize;
  std::vector<int32_t> tab((size_t)out_size * (2 + ksize), 0);
  std::vector<double> k(ksize);
  for (int xx = 0; xx < out_size; ++xx) {
    const double center = in0 + (xx + 0.5) * scale;
    double ww = 0.0;
    const double ss = 1.0 / filterscale;
    int xmin = (int)(center - support + 0.5);
    if (xmin < 0) xmin = 0;
    int xmax = (int)(center + support + 0.5);
    if (xmax > in_size) xmax = in_size;
    xmax -= xmin;
    for (int x = 0; x < xmax; ++x) {
      const double w = filter((x + xmin - center + 0.5) * ss);
      k[x] = w;
      ww += w;
    }
    int32_t* row = &tab[(size_t)xx * (2 + ksize)];
    row[0] = xmin;
    row[1] = xmax;
    for (int x = 0; x < xmax; ++x) {
      if (ww != 0.0) k[x] /= ww;
      row[2 + x] = k[x] < 0 ? (int)(-0.5 + k[x] * (1 << kPrecisionBits)) : (int)(0.5 + k[x] * (1 << kPrecisionBits));
    }
  }
  return tab;
}

// ---- OpenCV INTER_LINEAR, one axis: per output index {first tap, second tap, w0, w1}.  Along x a tap at or past the last
// pixel resets the weights to (2048, 0) (resizeGeneric_'s xofs loop); along y only the row indices are clamped.
std::vector<int4> cv_linear_table(int in_size, int out_size, bool is_x) {
  const double scale = 1.0 / ((double)out_size / in_size);
  std::vector<int4> tab(out_size);
  for (int d = 0; d < out_size; ++d) {
    float f = (float)((d + 0.5) * scale - 0.5);
    int s = (int)floorf(f);
    f -= (float)s;
    if (is_x) {
      if (s < 0) f = 0.f, s = 0;
      if (s >= in_size - 1) f = 0.f, s = in_size - 1;
    }
    const float c0 = 1.f - f, c1 = f;
    const int w0 = (int)rintf(c0 * (float)(1 << kCoefBits)), w1 = (int)rintf(c1 * (float)(1 << kCoefBits));
    tab[d] = make_int4(std::min(std::max(s, 0), in_size - 1), std::min(std::max(s + 1, 0), in_size - 1), w0, w1);
  }
  return tab;
}

// OpenCV's scale factors and its integer-factor test (resize.cpp: |scale - saturate_cast<int>(scale)| < DBL_EPSILON)
struct CvScale {
  int ix, iy;
  bool fast;
};

CvScale cv_scale(int W0, int H0, int W, int H) {
  const double sx = 1.0 / ((double)W / W0), sy = 1.0 / ((double)H / H0);
  const int ix = (int)lrint(sx), iy = (int)lrint(sy);
  return {ix, iy, std::fabs(sx - ix) < 2.220446049250313e-16 && std::fabs(sy - iy) < 2.220446049250313e-16};
}

// The code path of one call
enum Path { kCopy, kArea, kLinear, kPil };

struct Plan {
  Path path;
  int ix = 1, iy = 1;                        // kArea box
  bool need_h = false, need_v = false;       // kPil passes
  int kh = 0, kv = 0, y0 = 0, rows = 0;      // kPil: tap counts, first and number of intermediate rows
  std::vector<int32_t> th, tv;               // kPil tables
  std::vector<int4> lx, ly;                  // kLinear tables
  size_t tab_bytes = 0, tmp_bytes = 0;       // workspace: tables, then the uint8 intermediate (premultiplied for RGBA)
};

// ---- kernels: one thread per output pixel (kC = 3 or 4 channels), grid-stride over all frames

__device__ __forceinline__ void load3(const uint8_t* p, bool swap, int& c0, int& c1, int& c2) {
  c0 = p[0];
  c1 = p[1];
  c2 = p[2];
  if (swap) {
    const int t = c0;
    c0 = c2;
    c2 = t;
  }
}

__device__ __forceinline__ uint8_t clip8(int acc) { return (uint8_t)min(max(acc >> kPrecisionBits, 0), 255); }

// Pillow's RGBA -> RGBa (rgbA2rgba): MULDIV255(c, a) = ((t >> 8) + t) >> 8 with t = c * a + 128
__device__ __forceinline__ int premultiply(int c, int a) {
  const int t = c * a + 128;
  return ((t >> 8) + t) >> 8;
}

// Pillow's RGBa -> RGBA (rgba2rgbA): c unchanged for a of 0 or 255, else min(255, 255 * c / a) in integers
__device__ __forceinline__ uint8_t unpremultiply(int c, int a) {
  return (a == 0 || a == 255) ? (uint8_t)c : (uint8_t)min(255, (255 * c) / a);
}

// One Pillow pass.  Horizontal (vertical = 0): output (f, y, x) reads source row y0 + y at columns tab[x]; vertical: output
// (f, y, x) reads column x at rows tab[y].  tab: [out][2 + ksize] as pil_table writes it.  RGBA (kC = 4) resamples Pillow's
// premultiplied RGBa, as Image.resize does: premul premultiplies each tap as it is loaded from the RGBA source (a per-pixel
// function, so the same as premultiplying the frame first), unpremul converts back to RGBA in the store; an intermediate
// between two passes stays premultiplied, as Pillow's does.
template <int kC>
__global__ void __launch_bounds__(kThreads) pil_pass_kernel(const uint8_t* __restrict__ src, int64_t src_frame, int64_t src_row,
                                                            int y0, uint8_t* __restrict__ dst, int64_t dst_frame,
                                                            int64_t dst_row, int n, int rows, int cols,
                                                            const int32_t* __restrict__ tab, int ksize, int vertical,
                                                            int swap, int premul, int unpremul) {
  const int64_t total = (int64_t)n * rows * cols;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % cols);
    const int64_t fy = i / cols;
    const int y = (int)(fy % rows), f = (int)(fy / rows);
    const int32_t* t = tab + (int64_t)(vertical ? y : x) * (2 + ksize);
    const int first = t[0], count = t[1];
    const int64_t step = vertical ? src_row : kC;
    const uint8_t* p = src + f * src_frame + (vertical ? (int64_t)x * kC : (int64_t)(y0 + y) * src_row) + first * step;
    int a0 = 1 << (kPrecisionBits - 1), a1 = a0, a2 = a0, a3 = a0;
    for (int k = 0; k < count; ++k, p += step) {
      int c0, c1, c2;
      load3(p, swap, c0, c1, c2);
      const int w = t[2 + k];
      if constexpr (kC == 4) {
        const int c3 = p[3];
        if (premul) {
          c0 = premultiply(c0, c3);
          c1 = premultiply(c1, c3);
          c2 = premultiply(c2, c3);
        }
        a3 += c3 * w;
      }
      a0 += c0 * w;
      a1 += c1 * w;
      a2 += c2 * w;
    }
    uint8_t* o = dst + f * dst_frame + y * dst_row + (int64_t)x * kC;
    if constexpr (kC == 4) {
      const uint8_t al = clip8(a3);
      if (unpremul) {
        o[0] = unpremultiply(clip8(a0), al);
        o[1] = unpremultiply(clip8(a1), al);
        o[2] = unpremultiply(clip8(a2), al);
      } else {
        o[0] = clip8(a0);
        o[1] = clip8(a1);
        o[2] = clip8(a2);
      }
      o[3] = al;
    } else {
      o[0] = clip8(a0);
      o[1] = clip8(a1);
      o[2] = clip8(a2);
    }
  }
}

// OpenCV INTER_LINEAR, both passes: the two int row sums of the output's two source rows, then the vertical combine
__global__ void __launch_bounds__(kThreads) cv_linear_kernel(const uint8_t* __restrict__ src, int H0, int W0,
                                                             uint8_t* __restrict__ dst, int64_t dst_row, int n, int H, int W,
                                                             const int4* __restrict__ tx, const int4* __restrict__ ty,
                                                             int swap) {
  const int64_t total = (int64_t)n * H * W;
  const int64_t src_row = (int64_t)W0 * 3;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % W);
    const int64_t fy = i / W;
    const int y = (int)(fy % H), f = (int)(fy / H);
    const int4 cx = tx[x], cy = ty[y];
    const uint8_t* fr = src + (int64_t)f * H0 * src_row;
    int s[2][3];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const uint8_t* row = fr + (r ? cy.y : cy.x) * src_row;
      int p0, p1, p2, q0, q1, q2;
      load3(row + (int64_t)cx.x * 3, swap, p0, p1, p2);
      load3(row + (int64_t)cx.y * 3, swap, q0, q1, q2);
      s[r][0] = p0 * cx.z + q0 * cx.w;
      s[r][1] = p1 * cx.z + q1 * cx.w;
      s[r][2] = p2 * cx.z + q2 * cx.w;
    }
    uint8_t* o = dst + (int64_t)f * H * dst_row + y * dst_row + (int64_t)x * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const int v = (((cy.z * (s[0][c] >> 4)) >> 16) + ((cy.w * (s[1][c] >> 4)) >> 16) + 2) >> 2;
      o[c] = (uint8_t)min(max(v, 0), 255);
    }
  }
}

// OpenCV INTER_AREA for integer factors (ix x iy box); a 1 x 1 box copies.  RGBA (kC = 4): OpenCV resamples the four
// channels independently, alpha like the others.
template <int kC>
__global__ void __launch_bounds__(kThreads) cv_area_kernel(const uint8_t* __restrict__ src, int H0, int W0,
                                                           uint8_t* __restrict__ dst, int64_t dst_row, int n, int H, int W,
                                                           int ix, int iy, float inv_area, int swap) {
  const int64_t total = (int64_t)n * H * W;
  const int64_t src_row = (int64_t)W0 * kC;
  const bool two = ix == 2 && iy == 2;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % W);
    const int64_t fy = i / W;
    const int y = (int)(fy % H), f = (int)(fy / H);
    const uint8_t* p = src + (int64_t)f * H0 * src_row + (int64_t)y * iy * src_row + (int64_t)x * ix * kC;
    int s0 = 0, s1 = 0, s2 = 0, s3 = 0;
    for (int r = 0; r < iy; ++r, p += src_row)
      for (int c = 0; c < ix; ++c) {
        int c0, c1, c2;
        load3(p + c * kC, swap, c0, c1, c2);
        s0 += c0;
        s1 += c1;
        s2 += c2;
        if constexpr (kC == 4) s3 += p[c * kC + 3];
      }
    uint8_t* o = dst + (int64_t)f * H * dst_row + y * dst_row + (int64_t)x * kC;
    if (two) {
      o[0] = (uint8_t)((s0 + 2) >> 2);
      o[1] = (uint8_t)((s1 + 2) >> 2);
      o[2] = (uint8_t)((s2 + 2) >> 2);
      if constexpr (kC == 4) o[3] = (uint8_t)((s3 + 2) >> 2);
    } else {
      o[0] = (uint8_t)min(max(__float2int_rn(__fmul_rn((float)s0, inv_area)), 0), 255);
      o[1] = (uint8_t)min(max(__float2int_rn(__fmul_rn((float)s1, inv_area)), 0), 255);
      o[2] = (uint8_t)min(max(__float2int_rn(__fmul_rn((float)s2, inv_area)), 0), 255);
      if constexpr (kC == 4) o[3] = (uint8_t)min(max(__float2int_rn(__fmul_rn((float)s3, inv_area)), 0), 255);
    }
  }
}

unsigned grid_for(int64_t total) {
  return (unsigned)std::max<int64_t>(1, std::min<int64_t>((total + kThreads - 1) / kThreads, 132 * 16));
}

// r = a * b * c * d, false if it overflows int64
bool mul_ok(int64_t& r, int64_t a, int64_t b, int64_t c, int64_t d) {
  return !__builtin_mul_overflow(a, b, &r) && !__builtin_mul_overflow(r, c, &r) && !__builtin_mul_overflow(r, d, &r);
}

// Validates the call's shape and method and builds its tables; false with the refusal in msg.
// kC: channels per pixel, 3 (RGB) or 4 (RGBA).
bool make_plan(const char* fn, int32_t n, int32_t H0, int32_t W0, int32_t H, int32_t W, int32_t method, int kC, Plan& p,
               char* msg, size_t len) {
  if (method < HR_RESIZE_PIL_LANCZOS || method > HR_RESIZE_CV2_AREA)
    return snprintf(msg, len, "%s: unknown method %d", fn, method), false;
  if (kC == 4 && method == HR_RESIZE_CV2_LINEAR)
    return snprintf(msg, len, "%s: cv2_linear is not supported for RGBA frames", fn), false;
  if (n < 1 || H0 < 1 || W0 < 1 || H < 1 || W < 1)
    return snprintf(msg, len, "%s: bad sizes %d x %d x %d -> %d x %d", fn, n, H0, W0, H, W), false;
  if (H > H0 || W > W0)
    return snprintf(msg, len, "%s: %d x %d -> %d x %d (W x H) enlarges the frame; only reductions are supported", fn, W0, H0,
                    W, H), false;
  // every byte count the call addresses fits int64 (the destination's is checked with its row stride)
  int64_t bytes;
  if (!mul_ok(bytes, n, H0, W0, kC))
    return snprintf(msg, len, "%s: %d frames of %d x %d overflow a 64-bit size", fn, n, W0, H0), false;
  if (H == H0 && W == W0) {
    p.path = kCopy;
    return true;
  }
  if (method >= HR_RESIZE_CV2_LINEAR) {
    const CvScale s = cv_scale(W0, H0, W, H);
    if (method == HR_RESIZE_CV2_LINEAR && !(s.fast && s.ix == 2 && s.iy == 2)) {
      p.path = kLinear;
      p.lx = cv_linear_table(W0, W, true);
      p.ly = cv_linear_table(H0, H, false);
      p.tab_bytes = align256((int64_t)W * sizeof(int4)) + align256((int64_t)H * sizeof(int4));
      return true;
    }
    if (!s.fast)
      return snprintf(msg, len, "%s: cv2_area %d x %d -> %d x %d (W x H) is not a reduction by integer factors (OpenCV's "
                      "float INTER_AREA path is not supported)", fn, W0, H0, W, H), false;
    p.path = kArea;
    p.ix = s.ix;
    p.iy = s.iy;
    return true;
  }
  if (!pil_plan_ok(W0, W, method) || !pil_plan_ok(H0, H, method))
    return snprintf(msg, len, "%s: %d x %d -> %d x %d (W x H) needs more filter coefficients than Pillow allows (it raises "
                    "MemoryError)", fn, W0, H0, W, H), false;
  p.path = kPil;
  p.need_h = W != W0;
  p.need_v = H != H0;
  p.th = pil_table(W0, W, method, &p.kh);
  p.tv = pil_table(H0, H, method, &p.kv);
  p.y0 = p.tv[0];
  p.rows = p.tv[(size_t)(H - 1) * (2 + p.kv)] + p.tv[(size_t)(H - 1) * (2 + p.kv) + 1] - p.y0;
  if (p.need_h)  // the vertical pass reads the intermediate, which starts at source row y0 (Pillow shifts its bounds so)
    for (int y = 0; y < H; ++y) p.tv[(size_t)y * (2 + p.kv)] -= p.y0;
  p.tab_bytes = align256((int64_t)p.th.size() * 4) + align256((int64_t)p.tv.size() * 4);
  if (p.need_h && p.need_v) {
    // at most the source's bytes (rows <= H0, W <= W0), but the sum with the tables must fit too
    if (!mul_ok(bytes, n, p.rows, W, kC) || bytes > INT64_MAX - 512 - (int64_t)p.tab_bytes)
      return snprintf(msg, len, "%s: the intermediate of %d frames of %d x %d overflows a 64-bit size", fn, n, W, p.rows),
             false;
    p.tmp_bytes = (size_t)align256(bytes);
  }
  return true;
}

template <int kC>
cudaError_t launch_plan(const Plan& p, const uint8_t* src, int32_t n, int32_t H0, int32_t W0, uint8_t* dst, int32_t H,
                        int32_t W, int64_t dst_row_stride, int swap, char* ws, cudaStream_t st) {
  const int64_t total = (int64_t)n * H * W;
  const int64_t src_row = (int64_t)W0 * kC, src_frame = src_row * H0, dst_frame = dst_row_stride * H;
  cudaError_t e = cudaSuccess;
  switch (p.path) {
    case kCopy:
    case kArea:
      cv_area_kernel<kC><<<grid_for(total), kThreads, 0, st>>>(src, H0, W0, dst, dst_row_stride, n, H, W, p.ix, p.iy,
                                                               1.f / (float)(p.ix * p.iy), swap);
      break;
    case kLinear: {  // RGB only (make_plan refuses it for RGBA)
      int4* tx = (int4*)ws;
      int4* ty = (int4*)(ws + align256((int64_t)W * sizeof(int4)));
      e = cudaMemcpyAsync(tx, p.lx.data(), p.lx.size() * sizeof(int4), cudaMemcpyHostToDevice, st);
      if (e == cudaSuccess) e = cudaMemcpyAsync(ty, p.ly.data(), p.ly.size() * sizeof(int4), cudaMemcpyHostToDevice, st);
      if (e == cudaSuccess)
        cv_linear_kernel<<<grid_for(total), kThreads, 0, st>>>(src, H0, W0, dst, dst_row_stride, n, H, W, tx, ty, swap);
      break;
    }
    case kPil: {
      int32_t* th = (int32_t*)ws;
      int32_t* tv = (int32_t*)(ws + align256((int64_t)p.th.size() * 4));
      uint8_t* tmp = (uint8_t*)(ws + p.tab_bytes);
      e = cudaMemcpyAsync(th, p.th.data(), p.th.size() * 4, cudaMemcpyHostToDevice, st);
      if (e == cudaSuccess) e = cudaMemcpyAsync(tv, p.tv.data(), p.tv.size() * 4, cudaMemcpyHostToDevice, st);
      if (e != cudaSuccess) break;
      // RGBA: the pass that reads the source premultiplies, the pass that writes dst unpremultiplies (ignored for RGB)
      if (p.need_h) {
        // into the intermediate (rows y0 .. y0 + rows of the source), or straight into dst when the height is kept
        uint8_t* o = p.need_v ? tmp : dst;
        const int64_t o_row = p.need_v ? (int64_t)W * kC : dst_row_stride;
        const int rows = p.need_v ? p.rows : H0;
        const int y0 = p.need_v ? p.y0 : 0;
        pil_pass_kernel<kC><<<grid_for((int64_t)n * rows * W), kThreads, 0, st>>>(
            src, src_frame, src_row, y0, o, o_row * rows, o_row, n, rows, W, th, p.kh, 0, swap, 1, p.need_v ? 0 : 1);
      }
      if (p.need_v) {
        const uint8_t* in = p.need_h ? tmp : src;
        const int64_t in_row = p.need_h ? (int64_t)W * kC : src_row;
        const int64_t in_frame = p.need_h ? in_row * p.rows : src_frame;
        pil_pass_kernel<kC><<<grid_for(total), kThreads, 0, st>>>(in, in_frame, in_row, 0, dst, dst_frame, dst_row_stride, n,
                                                                  H, W, tv, p.kv, 1, p.need_h ? 0 : swap,
                                                                  p.need_h ? 0 : 1, 1);
      }
      break;
    }
  }
  return e;
}

}  // namespace

extern "C" int64_t hr_resize_workspace_bytes(int32_t n, int32_t H0, int32_t W0, int32_t H, int32_t W, int32_t method,
                                             int32_t pixel_format) {
  const int kC = hr::pixel_bytes(pixel_format);
  Plan p;
  char msg[256];
  if (kC == 0 || !make_plan("hr_resize_workspace_bytes", n, H0, W0, H, W, method, kC, p, msg, sizeof msg)) return -1;
  return (int64_t)(p.tab_bytes + p.tmp_bytes);
}

extern "C" int hr_resize_frames(const uint8_t* src, int32_t n, int32_t H0, int32_t W0, uint8_t* dst, int32_t H, int32_t W,
                                int64_t dst_row_stride, int32_t method, int32_t flags, int32_t pixel_format, void* workspace,
                                int64_t workspace_bytes, void* stream) {
  const char* fn = "hr_resize_frames";
  if (!src || !dst) return hr_fail("%s: null argument", fn);
  if (flags & ~HR_RESIZE_BGR) return hr_fail("%s: unknown flags 0x%x", fn, (unsigned)flags);
  const int kC = hr::pixel_bytes(pixel_format);
  if (kC == 0) return hr_fail("%s: unknown pixel format %d", fn, pixel_format);
  Plan p;
  char msg[256];
  if (!make_plan(fn, n, H0, W0, H, W, method, kC, p, msg, sizeof msg)) return hr_fail("%s", msg);
  if (dst_row_stride < (int64_t)W * kC)
    return hr_fail("%s: dst_row_stride %lld is less than a row's %lld bytes", fn, (long long)dst_row_stride,
                   (long long)W * kC);
  int64_t dst_bytes;
  if (!mul_ok(dst_bytes, n, H, dst_row_stride, 1))
    return hr_fail("%s: %d frames of %d rows of %lld bytes overflow a 64-bit size", fn, n, H, (long long)dst_row_stride);
  const int64_t need = (int64_t)(p.tab_bytes + p.tmp_bytes);
  if (need > 0 && (!workspace || ((uintptr_t)workspace % 256)))
    return hr_fail("%s: a workspace of %lld bytes is needed (device, 256-byte aligned)", fn, (long long)need);
  if (workspace_bytes < need)
    return hr_fail("%s: workspace of %lld bytes, %lld needed", fn, (long long)workspace_bytes, (long long)need);
  cudaStream_t st = (cudaStream_t)stream;
  const int swap = (flags & HR_RESIZE_BGR) ? 1 : 0;
  cudaError_t e = kC == 4 ? launch_plan<4>(p, src, n, H0, W0, dst, H, W, dst_row_stride, swap, (char*)workspace, st)
                          : launch_plan<3>(p, src, n, H0, W0, dst, H, W, dst_row_stride, swap, (char*)workspace, st);
  if (e == cudaSuccess) e = cudaGetLastError();
  if (e != cudaSuccess) return hr_fail("%s: %s", fn, cudaGetErrorString(e));
  return 0;
}
