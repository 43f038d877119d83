// C-ABI of libhyperreel_b200.so (declared in include/hyperreel_b200.h).
// Host-side glue only: parameter packing, workspace carving, kernel launches, timing.
#include <cuda_runtime.h>

#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <limits>
#include <new>
#include <string>
#include <vector>

#include "hr_common.cuh"
#include "hr_encode.cuh"
#include "hr_geom.cuh"
#include "hr_mlp.cuh"
#include "hyperreel_b200.h"

namespace hr {
cudaError_t launch_render(const hr_config& cfg, const Derived& dv, const RenderTabs& tabs, const float* rays,
                          const float* heads, const RgbDst& rgb, long long n, const ExtraOut* so, int num_sms,
                          cudaStream_t stream, unsigned char* rgb8);
cudaError_t launch_render_bwd(const hr_config& cfg, const Derived& dv, const RenderTabs& tabs, const GradTabs& gt, const float* rays,
                              const float* heads, const float* d_rgb, float* d_heads, long long n, int clamp_output, int white_bg,
                              int num_sms, cudaStream_t stream);
cudaError_t launch_generate_rays(const hr_camera& cam, int c_in, long long first, long long n, float* out, cudaStream_t st);
cudaError_t launch_generate_video_rays(const hr_camera* cams, const float* times, bool mixed, int c_in, int width,
                                       long long frame_px, long long first, long long n, float* out, cudaStream_t st);
cudaError_t launch_image_metrics_u8(const float* pred, const uint8_t* gt, int32_t n, int32_t H, int32_t W, double* out,
                                    double* partial, cudaStream_t st);
cudaError_t launch_image_metrics_rgba8(const float* pred, const uint8_t* gt, int32_t n, int32_t H, int32_t W, double* out,
                                       double* partial, cudaStream_t st);
cudaError_t launch_vis_normalize(const float* x, int nf, long long px, int dim, const VisMap& m, float* part, cudaStream_t st);
}  // namespace hr

static thread_local std::string g_err;

int hr_fail(const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_err = buf;
  return 1;
}

// Every entry point runs with the handle's device current and restores the caller's device on the way out (the reference
// never changes torch's current device; a stray cudaSetDevice here would silently move the caller's later allocations).
struct DeviceGuard {
  int prev = -1;
  bool switched = false;
  explicit DeviceGuard(int dev) {
    if (cudaGetDevice(&prev) == cudaSuccess && prev != dev) switched = (cudaSetDevice(dev) == cudaSuccess);
  }
  ~DeviceGuard() {
    if (switched) cudaSetDevice(prev);
  }
};

#define CK(expr)                                                                                                        \
  do {                                                                                                                  \
    cudaError_t _e = (expr);                                                                                            \
    if (_e != cudaSuccess) return hr_fail("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
  } while (0)

#include "hr_handle.h"

namespace {

__global__ void pack_channel_last(const float* __restrict__ src, float* __restrict__ dst, int C, int H, int W) {
  // src [C][H][W] (reference [1,C,H,W]) -> dst [H][W][C]
  long long total = (long long)C * H * W;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int c = (int)(i % C);
    long long hw = i / C;
    dst[i] = src[(long long)c * H * W + hw];
  }
}

// (axis, time) planes -> per-keyframe lines.  The reference samples plane_time[1,C,K,L] bilinearly at (u_c, tau) where
// base_t is the ray's keyframe time (utils/flow_utils.py:18-31), so the two rows grid_sample blends are a property of the
// keyframe k alone (keyframe_blend).  dst[k][l][c] holds that blend, so the render kernel's second factor is a 2-tap linear
// lookup instead of 4 taps.
__global__ void pack_time_lines(const float* __restrict__ src, float* __restrict__ dst, int C, int K, int L, float inv_fac,
                                float time_scale, float time_offset) {
  long long total = (long long)K * L * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int c = (int)(i % C);
    int l = (int)((i / C) % L);
    int k = (int)(i / ((long long)C * L));
    float ft;
    int it = hr::keyframe_blend(k, K, inv_fac, time_scale, time_offset, ft);
    float a = src[((long long)c * K + it) * L + l];
    float b = src[((long long)c * K + it + 1) * L + l];
    dst[i] = __fmul_rn(1.0f - ft, a) + __fmul_rn(ft, b);
  }
}

// Wt[k][n] (k-major, zero padded) from the reference weight W[out][in] (nn.Linear layout).
//   k -> source column: k < in_pad: (k < in_ch ? k : none) when the layer consumes the encoded input;
//                        hidden rows follow.  n -> source row: last layer channel-major permutation.
__global__ void pack_simt_layer(const float* __restrict__ Wsrc, const float* __restrict__ bsrc, float* __restrict__ Wt,
                                float* __restrict__ bias, int Kp, int Np, int out_ch, int in_ch_src, int in_enc,
                                int in_pad, int has_input, int has_hidden, int width, int perm_S, int perm_stride) {
  long long total = (long long)Kp * Np;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total + Np; i += (long long)gridDim.x * blockDim.x) {
    if (i >= total) {
      int n = (int)(i - total);
      int ns = n;
      if (perm_S > 0 && n < out_ch) ns = (n % perm_S) * perm_stride + (n / perm_S);
      bias[n] = (n < out_ch) ? bsrc[ns] : 0.0f;
      continue;
    }
    int n = (int)(i % Np);
    int k = (int)(i / Np);
    float v = 0.0f;
    if (n < out_ch) {
      int ns = n;
      if (perm_S > 0) ns = (n % perm_S) * perm_stride + (n / perm_S);  // n = c*S+s  <-  s*stride+c
      int ks = -1;
      if (has_input) {
        if (k < in_pad) ks = (k < in_enc) ? k : -1;
        else if (has_hidden) ks = in_enc + (k - in_pad);
      } else {
        ks = k;
      }
      if (ks >= 0 && ks < in_ch_src && (has_input || k < width)) v = Wsrc[(long long)ns * in_ch_src + ks];
    }
    Wt[i] = v;
  }
}

__global__ void unpermute_heads(const float* __restrict__ src, float* __restrict__ dst, long long n, int S, int stride) {
  // src [n][c*S+s] -> dst [n][s*stride+c]
  long long total = n * (long long)S * stride;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    long long ray = i / (S * stride);
    int rem = (int)(i % (S * stride));
    int s = rem / stride, c = rem % stride;
    dst[i] = src[ray * (long long)S * stride + c * S + s];
  }
}

__global__ void permute_heads(const float* __restrict__ src, float* __restrict__ dst, long long n, int S, int stride, int ld) {
  // src [n][s*stride+c] (reference order) -> dst [n][c*S+s] (the kernels' channel-major rows, ld >= S*stride apart; the
  // columns past S*stride are zeroed)
  long long total = n * (long long)ld;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    long long ray = i / ld;
    int rem = (int)(i % ld);
    int c = rem / S, s = rem % S;
    dst[i] = rem < S * stride ? src[ray * (long long)S * stride + s * stride + c] : 0.0f;
  }
}

__global__ void encode_rays_kernel(const __grid_constant__ hr_config cfg, const float* __restrict__ rays, float* __restrict__ enc,
                                   long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    hr::encode_ray(cfg, rays + i * cfg.c_in, enc + i * cfg.mlp_in, 1);
}

// First stage of a cascaded pipeline (PointPredictionEmbedding, nlf/embedding/point.py:142-160): one warp per ray,
// lane = first-stage sample.  heads0 [n][c*S0+s] are the ray net's outputs (null: `zero` net); the S0 z-planes are
// intersected, masked and sorted like any other (Intersect.forward, base.py:142-226; IntersectZPlane, z.py:77-97), and every
// point o + t d becomes one 8-float input row of the point net (channel k holds cfg.pt_src[k]).
__global__ void cascade_points_kernel(const __grid_constant__ hr_config cfg, const float* __restrict__ rays,
                                      const float* __restrict__ heads0, float* __restrict__ rows, long long n) {
  const int lane = threadIdx.x & 31;
  const int S0 = cfg.pre_samples;
  const long long warp0 = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long nwarps = (long long)gridDim.x * (blockDim.x >> 5);
  const int out0 = S0 * cfg.pre_head_stride;
  for (long long ray = warp0; ray < n; ray += nwarps) {
    const float* r = rays + ray * cfg.c_in;
    const float ox = __ldg(r + 0), oy = __ldg(r + 1), oz = __ldg(r + 2);
    const float dx = __ldg(r + 3), dy = __ldg(r + 4), dz = __ldg(r + 5);
    const float time = __ldg(r + cfg.c_in - 1);
    const bool act = lane < S0;
    const int s = act ? lane : 0;
    const float zraw = heads0 ? __ldg(heads0 + ray * out0 + cfg.pre_off_z * S0 + s) : 0.0f;
    const float sraw = (heads0 && cfg.pre_off_sigma >= 0) ? __ldg(heads0 + ray * out0 + cfg.pre_off_sigma * S0 + s) : 0.0f;
    const float sg = cfg.pre_use_sigma ? hr::apply_act_eased(cfg.pre_act_sigma, sraw) : 0.0f;
    const float zr = __fmul_rn(hr::apply_act(cfg.pre_isect_act, hr::apply_act(cfg.pre_act_z, zraw)), __fsub_rn(1.0f, sg));
    const float z = __fadd_rn(__fmul_rn(zr, cfg.pre_z_scale), cfg.pre_samples_tab[s]);
    float t = hr::intersect_axis_plane(z, oz, dz);
    if ((t <= cfg.pre_near) || (t >= cfg.pre_far)) t = 0.0f;
    float key[1] = {act ? t : __int_as_float(0x7f800000)};
    if (cfg.pre_sort) hr::sort_keys<1>(key, lane);
    t = key[0];
    if (!act) continue;
    const float px = __fadd_rn(ox, __fmul_rn(dx, t)), py = __fadd_rn(oy, __fmul_rn(dy, t)), pz = __fadd_rn(oz, __fmul_rn(dz, t));
    float v[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      float x = 0.0f;
      switch (cfg.pt_src[k]) {
        case HR_PT_POINT_X: x = px; break;
        case HR_PT_POINT_Y: x = py; break;
        case HR_PT_POINT_Z: x = pz; break;
        case HR_PT_VIEW_X: x = dx; break;
        case HR_PT_VIEW_Y: x = dy; break;
        case HR_PT_VIEW_Z: x = dz; break;
        case HR_PT_ORIGIN_X: x = ox; break;
        case HR_PT_ORIGIN_Y: x = oy; break;
        case HR_PT_ORIGIN_Z: x = oz; break;
        case HR_PT_TIME: x = time; break;
        default: break;
      }
      v[k] = x;
    }
    float4* dst = reinterpret_cast<float4*>(rows + (ray * S0 + lane) * 8);
    dst[0] = make_float4(v[0], v[1], v[2], v[3]);
    dst[1] = make_float4(v[4], v[5], v[6], v[7]);
  }
}

// gradient table [H][W][C] (channel-last, the kernels' layout) -> reference layout [C][H][W]
__global__ void unpack_channel_last(const float* __restrict__ src, float* __restrict__ dst, int C, int H, int W) {
  long long total = (long long)C * H * W;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    long long hw = i % ((long long)H * W);
    int c = (int)(i / ((long long)H * W));
    dst[i] = src[hw * C + c];
  }
}

// gradient of the pre-blended keyframe lines [K][L][C] -> gradient of the (axis, time) plane [C][K][L]: row r collects
// (1 - ft_k) of every keyframe k whose lower row is r and ft_k of every keyframe whose upper row is r (see pack_time_lines)
__global__ void unblend_time_lines(const float* __restrict__ src, float* __restrict__ dst, int C, int K, int L, float inv_fac,
                                   float time_scale, float time_offset) {
  long long total = (long long)C * K * L;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int l = (int)(i % L);
    int r = (int)((i / L) % K);
    int c = (int)(i / ((long long)K * L));
    float acc = 0.0f;
    for (int k = 0; k < K; ++k) {
      float ft;
      int it = hr::keyframe_blend(k, K, inv_fac, time_scale, time_offset, ft);
      float g = src[((long long)k * L + l) * C + c];
      if (it == r) acc += (1.0f - ft) * g;
      if (it + 1 == r) acc += ft * g;
    }
    dst[i] = acc;
  }
}

int grid_for(long long total) {
  long long g = (total + 255) / 256;
  if (g > 132 * 32) g = 132 * 32;
  if (g < 1) g = 1;
  return (int)g;
}

// Packed-parameter storage.  hr_upload asks for its buffers in a fixed order; a buffer whose size is unchanged since the
// previous upload is reused, so a parameter refresh (same grid, same net) performs no cudaFree / cudaMalloc.
int dev_alloc(hr_handle* h, void** p, size_t bytes) {
  bytes = bytes ? bytes : 16;
  const size_t i = h->slot_cursor++;
  if (i < h->slots.size() && h->slots[i].bytes == bytes) {
    *p = h->slots[i].ptr;
    return 0;
  }
  if (i < h->slots.size()) {
    cudaFree(h->slots[i].ptr);
    h->slots[i] = {nullptr, 0};
  } else {
    h->slots.push_back({nullptr, 0});
  }
  cudaError_t e = cudaMalloc(p, bytes);
  if (e != cudaSuccess) return hr_fail("cudaMalloc(%zu) failed: %s", bytes, cudaGetErrorString(e));
  h->slots[i] = {*p, bytes};
  return 0;
}

// Copy a reference-layout tensor to the device if it is on the host (returns device pointer).
int stage_in(const float* src, size_t count, int on_device, cudaStream_t st, std::vector<void*>& temps, const float** out) {
  if (on_device) {
    *out = src;
    return 0;
  }
  void* d = nullptr;
  cudaError_t e = cudaMalloc(&d, count * sizeof(float));
  if (e != cudaSuccess) return hr_fail("cudaMalloc(temp %zu) failed: %s", count * sizeof(float), cudaGetErrorString(e));
  temps.push_back(d);
  e = cudaMemcpyAsync(d, src, count * sizeof(float), cudaMemcpyHostToDevice, st);
  if (e != cudaSuccess) return hr_fail("H2D of parameters failed: %s", cudaGetErrorString(e));
  *out = (const float*)d;
  return 0;
}

// the net runs on the tensor cores (bf16x3 or fp16): the wgmma kernel, its pass table and its whole-wave launch sizes
bool tc_net(int mlp_mode) { return mlp_mode == HR_MLP_BF16X3_TC || mlp_mode == HR_MLP_FP16_TC; }

int validate(const hr_config& c) {
  if (c.abi_version != HR_ABI_VERSION) return hr_fail("hr_config.abi_version %d != %d", c.abi_version, HR_ABI_VERSION);
  if (hr::eases_density(c) && c.n_samples > 64) return hr_fail("eased density heads above 64 samples per ray are not supported");
  if (c.c_in != 6 && c.c_in != 8) return hr_fail("unsupported c_in %d (6: static rays, 8: video rays)", c.c_in);
  if (c.n_groups < 1 || c.n_groups > HR_MAX_GROUPS) return hr_fail("unsupported n_groups %d", c.n_groups);
  if (c.mlp_mode != HR_MLP_FP32_SIMT && c.mlp_mode != HR_MLP_BF16X3_TC && c.mlp_mode != HR_MLP_ZERO && c.mlp_mode != HR_MLP_FP16_TC)
    return hr_fail("unsupported mlp_mode");
  const bool has_net = c.mlp_mode != HR_MLP_ZERO;
  if (has_net && (c.mlp_layers < 2 || c.mlp_layers > HR_MAX_LAYERS)) return hr_fail("unsupported mlp_layers %d", c.mlp_layers);
  if (has_net && c.mlp_width != 128 && c.mlp_width != 256) return hr_fail("unsupported mlp_width %d (128 or 256)", c.mlp_width);
  if (c.mlp_in < 1 || c.mlp_in > 64) return hr_fail("unsupported mlp_in %d", c.mlp_in);
  if (has_net && c.mlp_skip != -1 && (c.mlp_skip < 1 || c.mlp_skip > c.mlp_layers - 2)) return hr_fail("bad mlp_skip %d", c.mlp_skip);
  if (c.n_samples < 1 || c.n_samples > HR_MAX_SAMPLES) return hr_fail("unsupported n_samples %d (max %d)", c.n_samples, HR_MAX_SAMPLES);
  if (c.mlp_out != c.n_samples * c.head_stride) return hr_fail("mlp_out %d != S*head_stride %d", c.mlp_out, c.n_samples * c.head_stride);
  if (tc_net(c.mlp_mode)) {
    const int out = c.cascade && c.pre_samples > 0 ? c.mlp_out / c.pre_samples : c.mlp_out;
    const int passes = c.mlp_layers - 1 + (out + c.mlp_width - 1) / c.mlp_width;
    if (passes > HR_TC_MAX_PASSES)
      return hr_fail("tensor-core sample net: %d passes of %d output columns, more than HR_TC_MAX_PASSES = %d", passes, c.mlp_width,
                     HR_TC_MAX_PASSES);
  }
  if (c.off_z < 0) return hr_fail("z_vals head is required");
  if ((c.isect_type == HR_ISECT_Z_PLANE || c.isect_type == HR_ISECT_DISTANCE) && c.n_z != 1) return hr_fail("z_plane / euclidean_distance need 1 z channel");
  if ((c.isect_type == HR_ISECT_SPHERE || c.isect_type == HR_ISECT_CYLINDER) && c.n_z != 4) return hr_fail("sphere / cylinder need 4 z channels");
  if (c.isect_type == HR_ISECT_SPHERE_NEW && c.n_z != 8) return hr_fail("sphere_new needs 8 z channels");
  if (c.isect_type < HR_ISECT_Z_PLANE || c.isect_type > HR_ISECT_PLANE) return hr_fail("unsupported intersect type %d", c.isect_type);
  if (c.isect_type == HR_ISECT_VOXEL && (c.n_z != 1 || c.isect_axes != 3 || c.n_samples % 3 != 0))
    return hr_fail("voxel_grid needs 1 z channel and a multiple of 3 samples");
  if (c.isect_type == HR_ISECT_PLANE && (c.n_z != 4 || c.isect_axes < 1 || c.isect_axes > 3 || c.n_samples % c.isect_axes != 0))
    return hr_fail("deformable_voxel_grid needs 4 z channels and 1-3 axes dividing the sample count");
  if (c.cascade) {
    if (c.pre_samples < 1 || c.pre_samples > 32 || c.n_samples % c.pre_samples != 0) return hr_fail("cascade: bad pre_samples %d", c.pre_samples);
    if (c.mlp_mode == HR_MLP_ZERO) return hr_fail("cascade: the point net cannot be a zero net");
    if (c.pre_mlp_mode != HR_MLP_ZERO && c.pre_mlp_mode != c.mlp_mode) return hr_fail("cascade: pre_mlp_mode must be zero or mlp_mode");
    if (c.pre_head_stride < 1 || c.pre_off_z < 0 || c.pre_off_z >= c.pre_head_stride || c.pre_off_sigma >= c.pre_head_stride)
      return hr_fail("cascade: bad first-stage head layout");
    if (c.pre_mlp_mode != HR_MLP_ZERO) {
      if (c.pre_n_groups < 1 || c.pre_n_groups > HR_MAX_GROUPS) return hr_fail("cascade: unsupported pre_n_groups %d", c.pre_n_groups);
      if (c.pre_mlp_layers < 2 || c.pre_mlp_layers > HR_MAX_LAYERS) return hr_fail("cascade: unsupported pre_mlp_layers %d", c.pre_mlp_layers);
      if (c.pre_mlp_width != 128 && c.pre_mlp_width != 256) return hr_fail("cascade: unsupported pre_mlp_width %d", c.pre_mlp_width);
      if (c.pre_mlp_in < 1 || c.pre_mlp_in > 64) return hr_fail("cascade: unsupported pre_mlp_in %d", c.pre_mlp_in);
      if (c.pre_mlp_skip != -1 && (c.pre_mlp_skip < 1 || c.pre_mlp_skip > c.pre_mlp_layers - 2)) return hr_fail("cascade: bad pre_mlp_skip");
      if ((c.pre_samples * c.pre_head_stride) % 4 != 0) return hr_fail("cascade: first-stage output width must be a multiple of 4");
    }
    if ((c.mlp_out / c.pre_samples) % 4 != 0) return hr_fail("cascade: the point net's output width must be a multiple of 4");
    for (int g = 0; g < c.n_groups; ++g)
      if (c.groups[g].start < 0 || c.groups[g].end > 8) return hr_fail("cascade: point-net param group outside the 8-channel row");
  }
  if (c.n_color_views < 0) return hr_fail("bad n_color_views");
  if (c.n_color_views > 0 && c.c_in != 8) return hr_fail("colour transform needs 8-channel rays (camera id = rays[:, -2])");
  if (c.n_color_views > 0 && c.off_cscale_global >= 0) return hr_fail("colour transform and global colour heads are exclusive");
  if (c.contract_type != HR_CONTRACT_NONE && c.contract_type != HR_CONTRACT_MIPNERF && c.contract_type != HR_CONTRACT_AFFINE)
    return hr_fail("unsupported contract type");
  if (c.contract_type == HR_CONTRACT_AFFINE) {
    for (int i = 0; i < 3; ++i)
      if (c.contract_affine_den[i] == 0.0f) return hr_fail("affine contraction: zero extent on axis %d", i);
    if (c.contract_dist_fac == 0.0f) return hr_fail("affine contraction: zero distance factor");
  }
  if ((c.off_cscale_global >= 0) != (c.off_cshift_global >= 0)) return hr_fail("color_scale_global and color_shift_global come together");
  if (c.off_cscale_global + 3 > c.head_stride || c.off_cshift_global + 3 > c.head_stride) return hr_fail("global colour heads out of range");
  if (c.use_flow && (c.off_flow < 0 || c.num_keyframes < 1 || c.num_frames < 1)) return hr_fail("flow needs spatial_flow head and K,F");
  if (c.use_offset && c.off_offset < 0) return hr_fail("point_offset needs point_offset head");
  if (c.use_color_scale_shift && (c.off_cscale < 0 || c.off_cshift < 0)) return hr_fail("colour scale/shift heads missing");
  if (c.dynamic && (c.num_keyframes < 1 || c.num_frames < 1)) return hr_fail("dynamic net needs K,F");
  for (int i = 0; i < 3; ++i)
    if (c.n_sigma[i] != c.n_app[i]) return hr_fail("n_lamb_sigma != n_lamb_sh not supported");
  const int* s = c.n_sigma;
  bool ok = (s[0] == 8 && s[1] == 0 && s[2] == 0) || (s[0] == 8 && s[1] == 4 && s[2] == 4) || (s[0] == 8 && s[1] == 8 && s[2] == 8);
  if (!ok) return hr_fail("unsupported component layout [%d,%d,%d]", s[0], s[1], s[2]);
  if (c.shading == HR_SHADE_SH && c.app_dim != 27) return hr_fail("SH shading needs app_dim 27");
  if (c.shading == HR_SHADE_RGB && c.app_dim != 3) return hr_fail("RGB shading needs app_dim 3");
  if (c.shading != HR_SHADE_SH && c.shading != HR_SHADE_RGB) return hr_fail("unsupported shading");
  return 0;
}

void derive(const hr_config& c, hr::Derived& d) {
  double K = c.num_keyframes > 0 ? c.num_keyframes : 1, F = c.num_frames > 0 ? c.num_frames : 1;
  double fac = K * (F - 1.0) / F;
  d.time_fac = (float)fac;
  d.time_inv_fac = (fac != 0.0) ? (float)(1.0 / fac) : 0.0f;
  d.time_scale = (float)((F - 1.0) / F);
  d.time_offset = (float)(0.5 / K);
  d.kf_max = (float)(K - 1.0);
  double ied = (double)c.contract_start_distance / (double)c.contract_end_distance;
  d.inv_end_dist = (float)ied;
  d.dist_scale_fac = (float)(1.0 / (1.0 - ied));
  double ier = (double)c.contract_start_radius / (double)c.contract_end_radius;
  d.inv_end_rad = (float)ier;
  d.rad_scale_fac = (float)(1.0 / (1.0 - ier));
}

}  // namespace

extern "C" {

int hr_abi_version(void) { return HR_ABI_VERSION; }

const char* hr_last_error(void) { return g_err.c_str(); }

int hr_create(const hr_config* cfg, int device, hr_handle** out) {
  if (!cfg || !out) return hr_fail("hr_create: null argument");
  *out = nullptr;
  if (validate(*cfg)) return 1;
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0) return hr_fail("hr_create: no CUDA device (%s); there is no CPU fallback", cudaGetErrorString(e));
  if (device < 0 || device >= ndev) return hr_fail("hr_create: device %d out of range (%d devices)", device, ndev);
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0)
    return hr_fail("hr_create: device %d is sm_%d%d; this library is built for sm_90a only", device, prop.major, prop.minor);
  DeviceGuard guard(device);
  hr_handle* h = new (std::nothrow) hr_handle();
  if (!h) return hr_fail("hr_create: out of memory");
  h->cfg = *cfg;
  h->device = device;
  h->num_sms = prop.multiProcessorCount;
  derive(h->cfg, h->dv);
  h->net.cfg = h->cfg;
  h->pre.cfg = h->cfg;
  if (h->cfg.cascade) {
    const hr_config& c = h->cfg;
    // the point net: one 8-float row per first-stage point in, n_samples / pre_samples samples out, columns in the
    // reference's order (n_samples = 1 makes the packers' channel-major permutation the identity)
    hr_config& n = h->net.cfg;
    n.c_in = 8;
    n.mlp_out = c.mlp_out / c.pre_samples;
    n.n_samples = 1;
    n.head_stride = n.mlp_out;
    // the first-stage ray net
    hr_config& q = h->pre.cfg;
    q.n_groups = c.pre_n_groups;
    for (int g = 0; g < HR_MAX_GROUPS; ++g) q.groups[g] = c.pre_groups[g];
    q.mlp_in = c.pre_mlp_in; q.mlp_width = c.pre_mlp_width; q.mlp_layers = c.pre_mlp_layers; q.mlp_skip = c.pre_mlp_skip;
    q.mlp_mode = c.pre_mlp_mode;
    q.n_samples = c.pre_samples;
    q.head_stride = c.pre_head_stride;
    q.mlp_out = c.pre_samples * c.pre_head_stride;
  }
  *out = h;
  return 0;
}

static void drop_host_graph(hr_handle* h);

// Packs one sample net for both kernels: the fp32 CUDA-core layers, and the wgmma images when the net runs on the tensor cores.
static int pack_net(hr_handle* h, SampleNet& net, const float* const* wsrc, const float* const* bsrc, int on_device, cudaStream_t st,
                    std::vector<void*>& temps) {
  const hr_config& nc = net.cfg;
  hr::MlpSimtPack& simt = net.simt;
  const int L = nc.mlp_layers, W = nc.mlp_width;
  const int in_pad = (nc.mlp_in + 15) / 16 * 16;
  simt.in_pad = in_pad;
  simt.n_layers = L;
  simt.skip = nc.mlp_skip;
  net.tc_ready = false;
  const float* w_dev[HR_MAX_LAYERS] = {nullptr};
  const float* b_dev[HR_MAX_LAYERS] = {nullptr};
  int r = 0;
  for (int l = 0; l < L && !r && nc.mlp_mode != HR_MLP_ZERO; ++l) {
    if (!wsrc[l] || !bsrc[l]) return hr_fail("hr_upload: mlp layer %d missing", l);
    const bool first = (l == 0), last = (l == L - 1), skip = (l == nc.mlp_skip);
    const int in_src = first ? nc.mlp_in : (skip ? nc.mlp_in + W : W);
    const int out_ch = last ? nc.mlp_out : W;
    const int Kp = first ? in_pad : (skip ? in_pad + W : W);
    const int Np = last ? (nc.mlp_out + W - 1) / W * W : W;
    if ((r = stage_in(wsrc[l], (size_t)out_ch * in_src, on_device, st, temps, &w_dev[l]))) break;
    if ((r = stage_in(bsrc[l], (size_t)out_ch, on_device, st, temps, &b_dev[l]))) break;
    float *Wt = nullptr, *bias = nullptr;
    if ((r = dev_alloc(h, (void**)&Wt, (size_t)Kp * Np * sizeof(float)))) break;
    if ((r = dev_alloc(h, (void**)&bias, (size_t)Np * sizeof(float)))) break;
    pack_simt_layer<<<grid_for((long long)Kp * Np + Np), 256, 0, st>>>(
        w_dev[l], b_dev[l], Wt, bias, Kp, Np, out_ch, in_src, nc.mlp_in, in_pad, (first || skip) ? 1 : 0, skip ? 1 : 0, W,
        last ? nc.n_samples : 0, nc.head_stride);
    simt.Wt[l] = Wt;
    simt.bias[l] = bias;
    simt.Kp[l] = Kp;
    simt.Np[l] = Np;
  }
  if (!r && tc_net(nc.mlp_mode)) {
    r = hr::pack_mlp_tc2(net, w_dev, b_dev, st);
    if (!r) net.tc_ready = true;
  }
  return r;
}

int hr_upload(hr_handle* h, const hr_params* p, void* stream) {
  if (!h || !p) return hr_fail("hr_upload: null argument");
  DeviceGuard guard(h->device);
  drop_host_graph(h);
  cudaStream_t st = (cudaStream_t)stream;
  const hr_config& c = h->cfg;
  // Buffers of the previous pack are reused slot by slot when their sizes are unchanged (dev_alloc).  Work already
  // enqueued on `st` that reads the old contents is ordered before the pack kernels below (same stream).
  h->slot_cursor = 0;
  h->uploaded = false;
  h->net.tc_ready = h->pre.tc_ready = false;
  std::vector<void*> temps;
  int rc = 0;

  // ---- sample net(s) ----
  rc = pack_net(h, h->net, p->mlp_weight, p->mlp_bias, p->on_device, st, temps);
  if (!rc && c.cascade) rc = pack_net(h, h->pre, p->pre_mlp_weight, p->pre_mlp_bias, p->on_device, st, temps);

  // ---- VM tables, channel-last ----
  auto pack_tab = [&](const float* src, int C, int H, int Wd, const float** out) -> int {
    *out = nullptr;
    if (C == 0) return 0;
    if (!src) return hr_fail("hr_upload: table with C=%d missing", C);
    const float* d = nullptr;
    if (stage_in(src, (size_t)C * H * Wd, p->on_device, st, temps, &d)) return 1;
    float* dst = nullptr;
    if (dev_alloc(h, (void**)&dst, (size_t)C * H * Wd * sizeof(float))) return 1;
    pack_channel_last<<<grid_for((long long)C * H * Wd), 256, 0, st>>>(d, dst, C, H, Wd);
    *out = dst;
    return 0;
  };
  int n_app_total = 0;
  for (int i = 0; i < 3 && !rc; ++i) {
    const int C = c.n_sigma[i];
    n_app_total += c.n_app[i];
    const int H2 = c.dynamic ? c.num_keyframes : 1;
    hr::PlaneTab& ts = h->tabs.sig[i];
    hr::PlaneTab& ta = h->tabs.app[i];
    ts.C = C; ta.C = c.n_app[i];
    ts.H = ta.H = p->plane_h[i];
    ts.W = ta.W = p->plane_w[i];
    ts.H2 = ta.H2 = H2;
    ts.L = ta.L = p->second_len[i];
    if (C > 0 && (ts.H < 2 || ts.W < 2 || ts.L < 2)) { rc = hr_fail("hr_upload: plane %d too small (%dx%d, L=%d)", i, ts.H, ts.W, ts.L); break; }
    if ((rc = pack_tab(p->sigma_plane[i], C, ts.H, ts.W, &ts.space))) break;
    if ((rc = pack_tab(p->app_plane[i], C, ts.H, ts.W, &ta.space))) break;
    // second factor: static [C][L][1] -> [1][L][C]; dynamic [C][K][L] -> K pre-blended keyframe lines [K][L][C]
    if (!c.dynamic) {
      if ((rc = pack_tab(p->sigma_second[i], C, H2, ts.L, &ts.second))) break;
      if ((rc = pack_tab(p->app_second[i], C, H2, ts.L, &ta.second))) break;
    } else if (C > 0) {
      if (H2 < 2) { rc = hr_fail("hr_upload: the keyframe (time) planes need at least 2 keyframes"); break; }
      for (int f = 0; f < 2 && !rc; ++f) {
        const float* srcp = f ? p->app_second[i] : p->sigma_second[i];
        if (!srcp) { rc = hr_fail("hr_upload: time plane %d missing", i); break; }
        const float* d = nullptr;
        if ((rc = stage_in(srcp, (size_t)C * H2 * ts.L, p->on_device, st, temps, &d))) break;
        float* dst = nullptr;
        if ((rc = dev_alloc(h, (void**)&dst, (size_t)C * H2 * ts.L * sizeof(float)))) break;
        pack_time_lines<<<grid_for((long long)C * H2 * ts.L), 256, 0, st>>>(d, dst, C, H2, ts.L, h->dv.time_inv_fac,
                                                                            h->dv.time_scale, h->dv.time_offset);
        (f ? ta.second : ts.second) = dst;
      }
      if (rc) break;
    }
  }
  if (!rc) {
    // every table derives from one gridSize (tensorf_base.py:911-944, tensorf_dynamic.py:126-169): plane i is
    // [C, grid[b_i], grid[a_i]], its second factor runs along grid[v_i]
    const int rx = p->plane_w[0], ry = p->plane_h[0], rz = p->second_len[0];
    h->dv.res[0] = rx; h->dv.res[1] = ry; h->dv.res[2] = rz;
    h->dv.kt = c.dynamic ? c.num_keyframes : 1;
    if (c.dynamic && c.num_keyframes < 2) rc = hr_fail("hr_upload: the keyframe (time) planes need at least 2 keyframes");
    if (c.n_sigma[1] > 0 && (p->plane_w[1] != rx || p->plane_h[1] != rz || p->second_len[1] != ry))
      rc = hr_fail("hr_upload: table group 1 is inconsistent with grid %dx%dx%d", rx, ry, rz);
    if (!rc && c.n_sigma[2] > 0 && (p->plane_w[2] != ry || p->plane_h[2] != rz || p->second_len[2] != rx))
      rc = hr_fail("hr_upload: table group 2 is inconsistent with grid %dx%dx%d", rx, ry, rz);
  }
  if (!rc) {
    if (!p->basis_mat) rc = hr_fail("hr_upload: basis_mat missing");
    else {
      const float* d = nullptr;
      size_t cnt = (size_t)c.app_dim * n_app_total;
      rc = stage_in(p->basis_mat, cnt, p->on_device, st, temps, &d);
      if (!rc) {
        float* dst = nullptr;
        rc = dev_alloc(h, (void**)&dst, cnt * sizeof(float));
        if (!rc) {
          cudaError_t e = cudaMemcpyAsync(dst, d, cnt * sizeof(float), cudaMemcpyDeviceToDevice, st);
          if (e != cudaSuccess) rc = hr_fail("basis copy failed: %s", cudaGetErrorString(e));
          h->tabs.basis = dst;
          h->tabs.n_app_total = n_app_total;
        }
      }
    }
  }
  if (!rc) {
    h->tabs.color_embedding = nullptr;
    if (c.n_color_views > 0) {
      if (!p->color_embedding) rc = hr_fail("hr_upload: color_embedding missing (n_color_views = %d)", c.n_color_views);
      else {
        const float* d = nullptr;
        const size_t cnt = (size_t)c.n_color_views * 12;
        rc = stage_in(p->color_embedding, cnt, p->on_device, st, temps, &d);
        float* dst = nullptr;
        if (!rc) rc = dev_alloc(h, (void**)&dst, cnt * sizeof(float));
        if (!rc) {
          cudaError_t e = cudaMemcpyAsync(dst, d, cnt * sizeof(float), cudaMemcpyDeviceToDevice, st);
          if (e != cudaSuccess) rc = hr_fail("color_embedding copy failed: %s", cudaGetErrorString(e));
          h->tabs.color_embedding = dst;
        }
      }
    }
  }
  cudaError_t le = cudaGetLastError();
  if (!rc && le != cudaSuccess) rc = hr_fail("hr_upload: pack kernel launch failed: %s", cudaGetErrorString(le));
  if (!temps.empty()) {  // host sources only: the staging copies must outlive the pack kernels
    cudaStreamSynchronize(st);
    for (void* t : temps) cudaFree(t);
  }
  // slots past the cursor belong to a previous, larger layout
  while (h->slots.size() > h->slot_cursor) {
    cudaFree(h->slots.back().ptr);
    h->slots.pop_back();
  }
  if (rc) return rc;
  h->uploaded = true;
  return 0;
}

// bytes of a heads scratch for n rays: one [mlp_out] fp32 row per ray
static int64_t heads_bytes(const hr_handle* h, int64_t n_rays) {
  return align256(n_rays * (int64_t)h->cfg.mlp_out * (int64_t)sizeof(float)) + 256;
}

// hr_render walks a large batch in sub-batches (sample net, then render kernel, per sub-batch) so that the heads scratch
// stays bounded (0.58 GB at S*15 = 480) instead of growing to 8-21 GB for 4 M-ray batches / full Neural-3D frames.
// Wave-sized sub-batches that would keep the scratch in L2 pay more in launch ramps than the HBM round trip they save.
static int64_t sub_batch_rays(const hr_handle* h) {
  if (h->sub_rays > 0) return h->sub_rays;
  return (int64_t)h->num_sms * 128 * 16;
}

// scratch of the first stage of a cascaded pipeline for n rays, placed after the heads (byte offsets, each 256-byte aligned):
// first-stage heads [n][S0*stride0] channel-major, point rows [n*S0][8], point-net output [n*S0][mlp_out/S0] = [n][S][stride]
// (reference order, before the channel-major permutation).  total is 0 for a pipeline that is not cascaded.
struct CascadeLayout {
  int64_t heads0, rows, out, total;
};
static CascadeLayout cascade_layout(const hr_config& c, int64_t n_rays) {
  CascadeLayout t{0, 0, 0, 0};
  if (!c.cascade) return t;
  const int64_t f = (int64_t)sizeof(float);
  t.rows = t.heads0 + align256(n_rays * c.pre_samples * c.pre_head_stride * f);
  t.out = t.rows + align256(n_rays * c.pre_samples * 8 * f);
  t.total = t.out + align256(n_rays * (int64_t)c.mlp_out * f);
  return t;
}

// workspace of one render call over n rays that is not split further
static int64_t ws_bytes_for(const hr_handle* h, int64_t n_rays) { return heads_bytes(h, n_rays) + cascade_layout(h->cfg, n_rays).total; }

int64_t hr_workspace_bytes(const hr_handle* h, int64_t n_rays) {
  if (!h || n_rays < 0) return -1;
  const int64_t sub = sub_batch_rays(h);
  return ws_bytes_for(h, (h->sub_rays < 0 || n_rays < sub) ? n_rays : sub);
}

int64_t hr_train_workspace_bytes(const hr_handle* h, int64_t n_rays) {
  if (!h || n_rays < 0) return -1;
  return 2 * heads_bytes(h, n_rays);
}

int hr_set_sub_batch(hr_handle* h, int64_t rays) {
  if (!h) return hr_fail("hr_set_sub_batch: null handle");
  h->sub_rays = rays;
  return 0;
}

// The cached hr_render_host graph holds kernel parameters by value: drop it whenever they may have changed.
static void drop_host_graph(hr_handle* h) {
  if (h->pipe.graph) cudaGraphExecDestroy(h->pipe.graph);
  h->pipe.graph = nullptr;
  h->pipe.g_rays = nullptr; h->pipe.g_rgb = nullptr; h->pipe.g_n = 0; h->pipe.g_chunk = 0;
}

// stream i of the host pipelines, created on first use
static int pipe_stream(hr_handle* h, int i) {
  if (!h->pipe.streams[i]) CK(cudaStreamCreateWithFlags(&h->pipe.streams[i], cudaStreamNonBlocking));
  return 0;
}

// Device scratch of the host pipelines: three slots, each the rays, the pixels (fp32 rgb, or an 8-bit tile stored in the rgb
// slot) and the render workspace of `rays_per_slot` rays.  It only grows; growing drops the cached graph, whose nodes hold
// the old pointers.
static int ensure_pipe(hr_handle* h, int64_t rays_per_slot) {
  HostPipe& P = h->pipe;
  if (P.chunk >= rays_per_slot) return 0;
  drop_host_graph(h);
  P.chunk = 0;
  for (int i = 0; i < 3; ++i) {
    if (P.d_rays[i]) cudaFree(P.d_rays[i]);
    if (P.d_rgb[i]) cudaFree(P.d_rgb[i]);
    if (P.d_ws[i]) cudaFree(P.d_ws[i]);
    P.d_rays[i] = P.d_rgb[i] = nullptr; P.d_ws[i] = nullptr;
    if (pipe_stream(h, i)) return 1;
  }
  P.ws_bytes = ws_bytes_for(h, rays_per_slot);
  for (int i = 0; i < 3; ++i) {
    CK(cudaMalloc((void**)&P.d_rays[i], (size_t)rays_per_slot * h->cfg.c_in * sizeof(float)));
    CK(cudaMalloc((void**)&P.d_rgb[i], (size_t)rays_per_slot * 3 * sizeof(float)));
    CK(cudaMalloc(&P.d_ws[i], (size_t)P.ws_bytes));
  }
  P.chunk = rays_per_slot;
  return 0;
}

// one net (ray net or point net) over `rows` input rows -> out [rows][nc.mlp_out].  in_copy (optional, tensor-core net
// only): `in` may be pinned host memory, and the net leaves a device copy of its rows there.
static int launch_net(hr_handle* h, const SampleNet& net, const float* in, int64_t rows, float* out, cudaStream_t st,
                      float* in_copy = nullptr) {
  const hr_config& nc = net.cfg;
  cudaError_t e;
  if (in_copy && !tc_net(nc.mlp_mode)) return hr_fail("hr_render: only the tensor-core sample net reads host rays");
  if (nc.mlp_mode == HR_MLP_ZERO) {  // ZeroMLP (nlf/nets/mlp.py:29-30): x.new_zeros(N, out_channels)
    e = cudaMemsetAsync(out, 0, (size_t)rows * nc.mlp_out * sizeof(float), st);
    if (e != cudaSuccess) return hr_fail("heads memset failed: %s", cudaGetErrorString(e));
    return 0;
  }
  if (tc_net(nc.mlp_mode)) {
    if (!net.tc_ready) return hr_fail("hr_render: tensor-core pack missing");
    e = hr::launch_mlp_tc2(nc, net.tc, in, out, rows, h->num_sms, st, in_copy);
  } else {
    e = hr::launch_mlp_simt(nc, net.simt, in, out, rows, h->num_sms, st);
  }
  if (e != cudaSuccess) return hr_fail("sample-net launch failed: %s", cudaGetErrorString(e));
  h->launches += 1;
  return 0;
}

// heads of n rays between the reference's order [n][s*stride+c] and the kernels' channel-major rows [n][c*S+s]
static cudaError_t permute_heads_async(const hr_config& c, const float* src, float* dst, int64_t n, cudaStream_t st, int ld = 0) {
  if (ld == 0) ld = c.mlp_out;
  permute_heads<<<grid_for(n * (long long)ld), 256, 0, st>>>(src, dst, n, c.n_samples, c.head_stride, ld);
  return cudaGetLastError();
}

static cudaError_t unpermute_heads_async(const hr_config& c, const float* src, float* dst, int64_t n, cudaStream_t st) {
  unpermute_heads<<<grid_for(n * (long long)c.mlp_out), 256, 0, st>>>(src, dst, n, c.n_samples, c.head_stride);
  return cudaGetLastError();
}

// rays [n, c_in] -> heads scratch [n, mlp_out] (channel-major per ray).  `scratch` (cascade_layout(c, n).total bytes, only read for a
// cascaded pipeline) holds the first stage's intermediates.  rays_copy: as launch_net's in_copy (not for a cascade).
static int launch_sample_net(hr_handle* h, const float* rays, int64_t n, float* heads, cudaStream_t st, void* scratch = nullptr,
                             float* rays_copy = nullptr) {
  const hr_config& c = h->cfg;
  if (!c.cascade) return launch_net(h, h->net, rays, n, heads, st, rays_copy);
  if (rays_copy) return hr_fail("hr_render: a cascaded pipeline does not read host rays");
  if (!scratch) return hr_fail("hr_render: cascade scratch missing");
  // PointPredictionEmbedding (nlf/embedding/point.py:142-206): ray net -> S0 z-planes -> one point-net row per point
  const CascadeLayout t = cascade_layout(c, n);
  float* heads0 = (float*)((char*)scratch + t.heads0);
  float* rows = (float*)((char*)scratch + t.rows);
  float* out = (float*)((char*)scratch + t.out);
  const bool has_pre = c.pre_mlp_mode != HR_MLP_ZERO;
  if (has_pre) {
    int rc = launch_net(h, h->pre, rays, n, heads0, st);
    if (rc) return rc;
  }
  cascade_points_kernel<<<grid_for(n * 32), 256, 0, st>>>(c, rays, has_pre ? heads0 : nullptr, rows, n);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return hr_fail("cascade point kernel launch failed: %s", cudaGetErrorString(e));
  int rc = launch_net(h, h->net, rows, n * c.pre_samples, out, st);
  if (rc) return rc;
  e = permute_heads_async(c, out, heads, n, st);
  if (e != cudaSuccess) return hr_fail("heads permutation launch failed: %s", cudaGetErrorString(e));
  h->launches += 2;
  return 0;
}

static hr::RgbDst one_dst(float* rgb) {
  hr::RgbDst d{};
  d.p[0] = rgb;
  d.n = 1;
  d.row0 = 0;
  return d;
}

// channels of every extra field (HR_FIELD_*, in the enum's order): points, view directions, flow, offset and the colour
// scales / shifts are 3-vectors
constexpr int kFieldWidth[HR_N_FIELDS] = {3, 1, 1, 1, 1, 3, 1, 3, 3, 3, 1, 1, 3, 3, 3};

// net_rays (optional): the sample net reads the rays there instead -- a device view of pinned host memory -- and leaves
// the device copy at `rays`, which the render kernel reads.
static int render_impl(hr_handle* h, const float* rays, int64_t n, float* rgb, float* mlp_out, const hr::ExtraOut* so,
                       void* workspace, int64_t ws_bytes, cudaStream_t st, unsigned char* rgb8 = nullptr,
                       const hr::RgbDst* scatter = nullptr, const float* net_rays = nullptr) {
  if (!h) return hr_fail("hr_render: null handle");
  if (!h->uploaded) return hr_fail("hr_render: parameters not uploaded (call hr_upload)");
  if (n == 0) return 0;
  if (!rays || (!rgb && !rgb8 && !scatter) || !workspace) return hr_fail("hr_render: null buffer");
  if (ws_bytes < hr_workspace_bytes(h, n)) return hr_fail("hr_render: workspace too small (%lld < %lld)", (long long)ws_bytes, (long long)hr_workspace_bytes(h, n));
  if (((uintptr_t)workspace & 15) != 0) return hr_fail("hr_render: workspace must be 16-byte aligned");
  float* heads = (float*)workspace;
  const hr_config& c = h->cfg;
  const bool timing = h->timing && h->ev_render.size() < 8192;
  const int64_t sub = (h->sub_rays < 0) ? n : sub_batch_rays(h);
  for (int64_t off = 0; off < n; off += sub) {
    const int64_t m = (n - off < sub) ? (n - off) : sub;
    const float* r = rays + off * c.c_in;
    EventPair em{nullptr, nullptr}, er{nullptr, nullptr};
    if (timing) {
      CK(cudaEventCreate(&em.a)); CK(cudaEventCreate(&em.b)); CK(cudaEventCreate(&er.a)); CK(cudaEventCreate(&er.b));
      CK(cudaEventRecord(em.a, st));
    }
    int rc0 = launch_sample_net(h, net_rays ? net_rays + off * c.c_in : r, m, heads, st,
                                (char*)workspace + heads_bytes(h, (n < sub) ? n : sub), net_rays ? const_cast<float*>(r) : nullptr);
    if (rc0) return rc0;
    if (timing) { CK(cudaEventRecord(em.b, st)); CK(cudaEventRecord(er.a, st)); }
    hr::RgbDst d = scatter ? *scatter : one_dst(rgb);
    d.row0 += off;
    hr::ExtraOut so_off;
    if (so) {  // every extra output is indexed by ray: advance the pointers to this sub-batch
      so_off = *so;
      const int64_t S = c.n_samples;
      if (so_off.distances) so_off.distances += off * S;
      if (so_off.points) so_off.points += off * S * 3;
      if (so_off.sigma) so_off.sigma += off * S;
      if (so_off.weights) so_off.weights += off * S;
      if (so_off.rgb_samples) so_off.rgb_samples += off * S * 3;
      for (int f = 0; f < HR_N_FIELDS; ++f) {
        if (so_off.field_u8[f].out) so_off.field_u8[f].out += off * kFieldWidth[f];
        if (!so_off.field_out[f]) continue;
        so_off.field_out[f] += off * kFieldWidth[f] * (so_off.field_mode[f] == HR_FIELD_NO_OVER ? S : 1);
      }
    }
    cudaError_t e = hr::launch_render(c, h->dv, h->tabs, r, heads, d, m, so ? &so_off : nullptr, h->num_sms, st, rgb8 ? rgb8 + off * 3 : nullptr);
    if (e != cudaSuccess) return hr_fail("render launch failed: %s", cudaGetErrorString(e));
    if (timing) {
      CK(cudaEventRecord(er.b, st));
      h->ev_mlp.push_back(em);
      h->ev_render.push_back(er);
    }
    h->launches += 1;
    if (mlp_out) {
      e = unpermute_heads_async(c, heads, mlp_out + off * c.mlp_out, m, st);
      if (e != cudaSuccess) return hr_fail("unpermute launch failed: %s", cudaGetErrorString(e));
      h->launches += 1;
    }
  }
  if (timing) h->timed_calls += 1;
  return 0;
}

int hr_render(hr_handle* h, const float* rays, int64_t n_rays, float* rgb, void* workspace, int64_t workspace_bytes,
              void* stream) {
  DeviceGuard guard(h ? h->device : 0);
  return render_impl(h, rays, n_rays, rgb, nullptr, nullptr, workspace, workspace_bytes, (cudaStream_t)stream);
}

int hr_render_scatter(hr_handle* h, const float* rays, int64_t n_rays, float* const* dst, int32_t n_dst, int64_t row0,
                      void* workspace, int64_t workspace_bytes, void* stream) {
  if (!h) return hr_fail("hr_render_scatter: null handle");
  if (!dst || n_dst < 1 || n_dst > HR_MAX_PEERS) return hr_fail("hr_render_scatter: 1..%d destination buffers", HR_MAX_PEERS);
  if (row0 < 0) return hr_fail("hr_render_scatter: negative row offset");
  DeviceGuard guard(h->device);
  hr::RgbDst d{};
  for (int i = 0; i < n_dst; ++i) {
    if (!dst[i]) return hr_fail("hr_render_scatter: null destination %d", i);
    d.p[i] = dst[i];
  }
  d.n = n_dst;
  d.row0 = row0;
  return render_impl(h, rays, n_rays, nullptr, nullptr, nullptr, workspace, workspace_bytes, (cudaStream_t)stream, nullptr, &d);
}

int hr_render_stages(hr_handle* h, const float* rays, int64_t n_rays, float* rgb, float* mlp_out, float* distances,
                     float* points, float* sigma, float* weights, float* rgb_samples, void* workspace, int64_t workspace_bytes,
                     void* stream) {
  DeviceGuard guard(h ? h->device : 0);
  hr::ExtraOut so{};
  so.distances = distances; so.points = points; so.sigma = sigma; so.weights = weights; so.rgb_samples = rgb_samples;
  return render_impl(h, rays, n_rays, rgb, mlp_out, &so, workspace, workspace_bytes, (cudaStream_t)stream);
}

// Whether the pipeline carries field f (the reference fails with a KeyError on x[key] otherwise): refused with fn's name, or 0
static int field_refusal(const char* fn, const hr_config& c, int f) {
  if ((f == HR_FIELD_BASE_TIMES || f == HR_FIELD_TIME_OFFSET) && !(c.dynamic || c.use_flow))
    return hr_fail("%s: this pipeline has no keyframe times", fn);
  const int head_off[HR_N_FIELDS] = {0, 0, 0, 0, 0, 0, 0, c.off_cscale, c.off_cshift, c.off_flow, c.off_sigma,
                                     c.off_point_sigma, c.off_offset, c.off_cscale_global, c.off_cshift_global};
  if (f >= HR_FIELD_COLOR_SCALE && head_off[f] < 0) return hr_fail("%s: the sample net has no head for field %d", fn, f);
  return 0;
}

int hr_render_fields(hr_handle* h, const float* rays, int64_t n_rays, float* rgb, float* render_weights,
                     const hr_field_request* req, int32_t n_req, void* workspace, int64_t workspace_bytes, void* stream) {
  if (!h) return hr_fail("hr_render_fields: null handle");
  if (n_req < 0 || (n_req > 0 && !req)) return hr_fail("hr_render_fields: bad request list");
  DeviceGuard guard(h->device);
  const hr_config& c = h->cfg;
  hr::ExtraOut so{};
  so.weights = render_weights;
  for (int i = 0; i < n_req; ++i) {
    const int f = req[i].field, m = req[i].mode;
    if (f < 0 || f >= HR_N_FIELDS) return hr_fail("hr_render_fields: unknown field %d", f);
    if (m != HR_FIELD_OVER && m != HR_FIELD_NO_OVER && m != HR_FIELD_PRED_WEIGHTS) return hr_fail("hr_render_fields: unknown mode %d", m);
    if (!req[i].out) return hr_fail("hr_render_fields: null output for field %d", f);
    if (so.field_out[f]) return hr_fail("hr_render_fields: field %d requested twice", f);
    if (field_refusal("hr_render_fields", c, f)) return 1;
    so.field_out[f] = req[i].out;
    so.field_mode[f] = m;
  }
  return render_impl(h, rays, n_rays, rgb, nullptr, &so, workspace, workspace_bytes, (cudaStream_t)stream);
}

int hr_render_to8b(hr_handle* h, const float* rays, int64_t n_rays, uint8_t* rgb8, void* workspace, int64_t workspace_bytes,
                   void* stream) {
  DeviceGuard guard(h ? h->device : 0);
  if (!rgb8) return hr_fail("hr_render_to8b: null output");
  return render_impl(h, rays, n_rays, nullptr, nullptr, nullptr, workspace, workspace_bytes, (cudaStream_t)stream, rgb8);
}

// A fisheye record needs finite coefficients: the Newton solve of camera_ray has no meaning otherwise.
static bool bad_fisheye(const hr_camera& cam) { return cam.fisheye && !(std::isfinite(cam.k1) && std::isfinite(cam.k2)); }

// Why a two-plane record cannot be drawn, or nullptr: it is one model or the other, and its fields must be finite with a
// nonzero aspect (lightfield_ray divides by it).
static const char* bad_two_plane(const hr_camera& cam) {
  if (!cam.two_plane) return nullptr;
  if (cam.fisheye) return "two_plane and fisheye are both set";
  const float f[7] = {cam.lf_s, cam.lf_t, cam.lf_st_scale, cam.lf_uv_scale, cam.lf_near, cam.lf_far, cam.lf_aspect};
  for (float v : f)
    if (!std::isfinite(v)) return "a two-plane field (lf_*) is not finite";
  if (cam.lf_aspect == 0.0f) return "lf_aspect is 0";
  return nullptr;
}

int hr_generate_rays(const hr_camera* cam, int32_t c_in, int64_t first_pixel, int64_t n_pixels, float* rays_out, void* stream) {
  if (!cam || !rays_out) return hr_fail("hr_generate_rays: null argument");
  if (c_in != 6 && c_in != 8) return hr_fail("hr_generate_rays: c_in must be 6 or 8");
  if (cam->width < 1 || cam->height < 1) return hr_fail("hr_generate_rays: bad image size");
  if (bad_fisheye(*cam)) return hr_fail("hr_generate_rays: fisheye coefficients k1 = %g, k2 = %g are not finite", cam->k1, cam->k2);
  if (const char* why = bad_two_plane(*cam)) return hr_fail("hr_generate_rays: %s", why);
  if (first_pixel < 0 || n_pixels < 0 || first_pixel + n_pixels > (int64_t)cam->width * cam->height)
    return hr_fail("hr_generate_rays: pixel range outside the image");
  cudaError_t e = hr::launch_generate_rays(*cam, c_in, first_pixel, n_pixels, rays_out, (cudaStream_t)stream);
  if (e != cudaSuccess) return hr_fail("hr_generate_rays: %s", cudaGetErrorString(e));
  return 0;
}

// Where the chunks of a host-buffer call take their rays from and put their pixels; one of each is set.
//   rays: generated from `cam`; read by the sample net from `rays_view`, a device view of pinned host rays, which leaves
//         the device copy in the slot; or copied in from `rays_host`.
//   pixels: stored by the render epilogue into `rgb_view`, a device view of pinned host memory; or rendered into the slot
//           and copied out to `rgb_host` (fp32) or `rgb8_host` (uint8).
struct HostChunks {
  const hr_camera* cam = nullptr;
  const float* rays_view = nullptr;
  const float* rays_host = nullptr;
  float* rgb_view = nullptr;
  float* rgb_host = nullptr;
  uint8_t* rgb8_host = nullptr;
};

// n rays in chunks of `chunk` (h->pipe's slots hold that many): chunk i brings its rays in, renders and sends its pixels
// out on stream and slot i % 3.  Only enqueues; the caller synchronises the streams.
static int run_host_chunks(hr_handle* h, int64_t n, int64_t chunk, const HostChunks& io) {
  HostPipe& P = h->pipe;
  const int c_in = h->cfg.c_in;
  int slot = 0;
  for (int64_t off = 0; off < n; off += chunk, slot = (slot + 1) % 3) {
    const int64_t m = (n - off < chunk) ? (n - off) : chunk;
    cudaStream_t st = P.streams[slot];
    if (io.cam) {
      cudaError_t e = hr::launch_generate_rays(*io.cam, c_in, off, m, P.d_rays[slot], st);
      if (e != cudaSuccess) return hr_fail("ray generation failed: %s", cudaGetErrorString(e));
      h->launches += 1;
    } else if (io.rays_host) {
      CK(cudaMemcpyAsync(P.d_rays[slot], io.rays_host + off * c_in, (size_t)m * c_in * sizeof(float), cudaMemcpyHostToDevice, st));
    }
    float* rgb = io.rgb_view ? io.rgb_view + off * 3 : (io.rgb_host ? P.d_rgb[slot] : nullptr);
    int rc = render_impl(h, P.d_rays[slot], m, rgb, nullptr, nullptr, P.d_ws[slot], P.ws_bytes, st,
                         io.rgb8_host ? (unsigned char*)P.d_rgb[slot] : nullptr, nullptr,
                         io.rays_view ? io.rays_view + off * c_in : nullptr);
    if (rc) return rc;
    if (io.rgb_host)
      CK(cudaMemcpyAsync(io.rgb_host + off * 3, P.d_rgb[slot], (size_t)m * 3 * sizeof(float), cudaMemcpyDeviceToHost, st));
    if (io.rgb8_host) CK(cudaMemcpyAsync(io.rgb8_host + off * 3, P.d_rgb[slot], (size_t)m * 3, cudaMemcpyDeviceToHost, st));
  }
  return 0;
}

static int sync_pipe(hr_handle* h) {
  for (int i = 0; i < 3; ++i) CK(cudaStreamSynchronize(h->pipe.streams[i]));
  return 0;
}

int hr_render_frame_to8b_host(hr_handle* h, const hr_camera* cam, uint8_t* rgb8_host, int64_t chunk) {
  if (!h || !cam || !rgb8_host) return hr_fail("hr_render_frame_to8b_host: null argument");
  if (!h->uploaded) return hr_fail("hr_render_frame_to8b_host: parameters not uploaded");
  if (bad_fisheye(*cam))
    return hr_fail("hr_render_frame_to8b_host: fisheye coefficients k1 = %g, k2 = %g are not finite", cam->k1, cam->k2);
  if (const char* why = bad_two_plane(*cam)) return hr_fail("hr_render_frame_to8b_host: %s", why);
  DeviceGuard guard(h->device);
  const int64_t n_rays = (int64_t)cam->width * cam->height;
  if (chunk <= 0) chunk = tc_net(h->cfg.mlp_mode) ? (int64_t)h->num_sms * 128 * 14 : 262144;  // whole tile waves
  if (chunk > n_rays) chunk = n_rays;
  if (ensure_pipe(h, chunk)) return 1;
  // The pixels are copied out: stored straight into pinned memory they would cross PCIe as 3-byte writes per ray.
  HostChunks io;
  io.cam = cam;
  io.rgb8_host = rgb8_host;
  int rc = run_host_chunks(h, n_rays, chunk, io);
  return rc ? rc : sync_pipe(h);
}

// ---- frame sequences (videos, scored splits, embedding maps): rays generated and rendered in sub-batches across frames
// rays of the whole sequence, or -1 when F * H * W * 3 (a video's bytes) does not fit in int64
static int64_t video_rays(int32_t n_frames, int32_t height, int32_t width) {
  if (n_frames < 1 || height < 1 || width < 1) return -1;
  int64_t px, n, bytes;
  if (__builtin_mul_overflow((int64_t)height, (int64_t)width, &px) || __builtin_mul_overflow(px, (int64_t)n_frames, &n) ||
      __builtin_mul_overflow(n, (int64_t)3, &bytes))
    return -1;
  return n;
}

// Frames of a ring: what two sub-batches cover and one more (so the sub-batch after next is the first that may wait for a
// frame's finish), at most the sequence; bounded by the sub-batch, whatever n_frames.
static int64_t ring_frames(int64_t sub, int64_t frame_px, int32_t n_frames) {
  int64_t r = (2 * sub + frame_px - 1) / frame_px + 1;
  if (r > n_frames) r = n_frames;
  return r > 65535 ? 65535 : r;  // frames per metrics launch
}

// Workspace of a frame walk, each part 256-byte aligned: the records [F] and times [F] on the device; the caller's middle
// segment, a ring of whole frames (ring_px_bytes per pixel, 0 for no ring, plus ring_pad bytes for the caller's alignment)
// and one partial buffer per stream (part_frame_bytes per ring frame); then one slot per stream (two when the sequence is
// longer than one sub-batch), each a sub-batch's rays [sub, c_in] and render workspace.  The sub-batch is hr_render's (16
// sample-net tile waves unless hr_set_sub_batch says otherwise) whatever the frame size, so past the records and times the
// scratch is bounded whatever F; "never split" does not apply here, a sequence is unbounded.  false: a size overflows int64.
struct WalkLayout {
  int64_t n, frame_px, sub, ring, ring_off, part_off, part_bytes, slots_off, slot_bytes, total;
  int n_slots;
};

static bool walk_layout(const hr_handle* h, int32_t n_frames, int32_t height, int32_t width, int64_t ring_px_bytes,
                        int64_t ring_pad, int64_t part_frame_bytes, WalkLayout* L) {
  *L = WalkLayout{};
  L->n = video_rays(n_frames, height, width);
  if (!h || L->n < 0) return false;
  const int64_t sub = sub_batch_rays(h);
  L->frame_px = (int64_t)height * width;
  L->sub = L->n < sub ? L->n : sub;
  L->n_slots = L->n > L->sub ? 2 : 1;
  L->ring = ring_px_bytes ? ring_frames(L->sub, L->frame_px, n_frames) : 0;
  int64_t ring_bytes;
  if (__builtin_mul_overflow(L->ring * L->frame_px, ring_px_bytes, &ring_bytes)) return false;
  L->ring_off = align256((int64_t)n_frames * (int64_t)sizeof(hr_camera)) + align256((int64_t)n_frames * (int64_t)sizeof(float));
  L->part_off = L->ring_off + align256(ring_bytes) + ring_pad;
  L->part_bytes = align256(L->ring * part_frame_bytes);
  L->slots_off = L->part_off + 2 * L->part_bytes;
  L->slot_bytes = align256(L->sub * h->cfg.c_in * (int64_t)sizeof(float)) + align256(ws_bytes_for(h, L->sub));
  L->total = L->slots_off + L->n_slots * L->slot_bytes;
  return true;
}

int64_t hr_video_workspace_bytes(const hr_handle* h, int32_t n_frames, int32_t height, int32_t width) {
  WalkLayout L;
  return walk_layout(h, n_frames, height, width, 0, 0, 0, &L) ? L.total : -1;
}

static bool finite_camera(const hr_camera& c) {
  for (int i = 0; i < 12; ++i)
    if (!std::isfinite(c.c2w[i])) return false;
  return std::isfinite(c.fx) && std::isfinite(c.fy) && std::isfinite(c.cx) && std::isfinite(c.cy) && std::isfinite(c.ndc_near) &&
         std::isfinite(c.cam_idx) && std::isfinite(c.time);
}

// The records and times of a video or split: one size (frame 0's), finite fields and times, well-formed fisheye and two-plane
// records.  *mixed: any record is not a pinhole, so the ray kernel's instantiation that branches on each record's model runs.
static int check_frames(const char* fn, const hr_camera* cameras, const float* times, int32_t n_frames, bool* mixed) {
  const int32_t W = cameras[0].width, H = cameras[0].height;
  *mixed = false;
  for (int32_t f = 0; f < n_frames; ++f) {
    const hr_camera& c = cameras[f];
    if (c.width != W || c.height != H) return hr_fail("%s: frame %d is %d x %d, frame 0 is %d x %d", fn, f, c.width, c.height, W, H);
    if (!finite_camera(c)) return hr_fail("%s: camera record of frame %d is not finite", fn, f);
    if (bad_fisheye(c)) return hr_fail("%s: fisheye coefficients k1 = %g, k2 = %g of frame %d are not finite", fn, c.k1, c.k2, f);
    if (const char* why = bad_two_plane(c)) return hr_fail("%s: frame %d: %s", fn, f, why);
    if (!std::isfinite(times[f])) return hr_fail("%s: time of frame %d is not finite", fn, f);
    *mixed = *mixed || c.fisheye || c.two_plane;
  }
  return 0;
}

// The refusals every frame walk makes first: a null argument (null_out: one of the caller's own), parameters not uploaded,
// a frame count (named `count`) under 1, and check_frames'.
static int check_walk(const char* fn, const char* count, const hr_handle* h, bool null_out, const hr_camera* cameras,
                      const float* times, int32_t n_frames, const void* workspace, bool* mixed) {
  if (null_out || !h || !cameras || !times || !workspace) return hr_fail("%s: null argument", fn);
  if (!h->uploaded) return hr_fail("%s: parameters not uploaded", fn);
  if (n_frames < 1) return hr_fail("%s: %s must be >= 1, got %d", fn, count, n_frames);
  return check_frames(fn, cameras, times, n_frames, mixed);
}

// The refusals every frame walk makes last, after its own: a size whose bytes overflow int64 (laid_out false), a workspace
// that is not 16-byte aligned or is too small.
static int check_workspace(const char* fn, bool laid_out, const WalkLayout& L, const hr_camera* cameras, int32_t n_frames,
                           const void* workspace, int64_t workspace_bytes) {
  if (!laid_out)
    return hr_fail("%s: %d frames of %d x %d pixels: bad size or bytes overflow int64", fn, n_frames, cameras[0].width, cameras[0].height);
  if (((uintptr_t)workspace & 15) != 0) return hr_fail("%s: workspace must be 16-byte aligned", fn);
  if (workspace_bytes < L.total)
    return hr_fail("%s: workspace too small (%lld < %lld)", fn, (long long)workspace_bytes, (long long)L.total);
  return 0;
}

// The walk of a frame sequence: its F·H·W rays in sub-batches of L.sub across frame boundaries.  The records and times are
// copied to the workspace on the caller's stream (stream-ordered: a pageable source is staged before the call returns,
// without waiting for the device).  Sub-batch i runs on stream i % 2 of the handle (forked from and joined back to the
// caller's stream by events, also after a failure) in slot i % 2: its ray generation and sample net overlap the previous
// sub-batch's render kernel, where one stream would leave the SMs idle between each sub-batch's render tail and the next
// one's ray generation.  render(off, pos, m, rays, ws, ws_bytes, s) enqueues the render of rays [off, off + m) on s, pos
// being their ring position.  With a ring (L.ring > 0) a sub-batch is also cut where it would wrap it, so its pixels land in
// consecutive ring positions, and finish(next, f_end, k, s) enqueues the work of the frames next .. f_end - 1 it completes
// on its own stream k, after the other stream's last render when a frame straddles the two; a ring frame is rendered
// again only after the finish of the frame it held.  Each stream runs in order, so its slot and partials are reused safely.
extern "C++" {  // a template, inside the C-ABI block
template <class Render, class Finish>
static int walk_frames(hr_handle* h, const char* fn, const WalkLayout& L, const hr_camera* cameras, const float* times,
                       int32_t n_frames, bool mixed, void* workspace, cudaStream_t st, Render render, Finish finish) {
  DeviceGuard guard(h->device);
  char* base = (char*)workspace;
  hr_camera* d_cams = (hr_camera*)base;
  float* d_times = (float*)(base + align256((int64_t)n_frames * (int64_t)sizeof(hr_camera)));
  CK(cudaMemcpyAsync(d_cams, cameras, (size_t)n_frames * sizeof(hr_camera), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(d_times, times, (size_t)n_frames * sizeof(float), cudaMemcpyHostToDevice, st));
  const bool two = L.n_slots == 2, ring_events = two && L.ring > 0;
  const int64_t ring_rays = L.ring * L.frame_px, rays_bytes = align256(L.sub * h->cfg.c_in * (int64_t)sizeof(float));
  cudaStream_t ss[2] = {st, st};
  std::vector<cudaEvent_t> evs;  // every event of the call, destroyed at the end (a destroyed event's pending work still runs)
  auto new_event = [&](cudaEvent_t* ev) {
    const cudaError_t e = cudaEventCreateWithFlags(ev, cudaEventDisableTiming);
    if (e == cudaSuccess) evs.push_back(*ev);
    return e;
  };
  auto fail = [&](const char* what, cudaError_t e) { return hr_fail("%s: %s: %s", fn, what, cudaGetErrorString(e)); };
  // freed[f]: recorded after the finish that read ring frame f last; done[k]: after stream k's last render
  std::vector<cudaEvent_t> freed(ring_events ? L.ring : 0, nullptr);
  cudaEvent_t done[2] = {nullptr, nullptr};
  cudaError_t e = cudaSuccess;  // of the event calls: the walk stops at the first failure
  if (two) {
    for (int k = 0; k < 2; ++k) {
      if (pipe_stream(h, k)) return 1;
      ss[k] = h->pipe.streams[k];
    }
    cudaEvent_t fork;
    if ((e = new_event(&fork)) == cudaSuccess) e = cudaEventRecord(fork, st);
    for (int k = 0; k < 2 && e == cudaSuccess; ++k) e = cudaStreamWaitEvent(ss[k], fork, 0);
    for (size_t f = 0; f < freed.size() && e == cudaSuccess; ++f) e = new_event(&freed[f]);
    for (int k = 0; k < 2 && e == cudaSuccess && ring_events; ++k) e = new_event(&done[k]);
  }
  int rc = 0;
  int64_t next = 0;  // first frame not yet finished
  for (int64_t off = 0, i = 0; off < L.n && !rc && e == cudaSuccess; ++i) {
    const int k = (int)(i % 2);
    cudaStream_t s = ss[k];
    const int64_t pos = ring_rays ? off % ring_rays : 0;
    int64_t m = L.n - off < L.sub ? L.n - off : L.sub;
    if (ring_rays && pos + m > ring_rays) m = ring_rays - pos;
    const int64_t f0 = off / L.frame_px, f1 = (off + m - 1) / L.frame_px, f_end = (off + m) / L.frame_px;
    for (int64_t f = f0 < L.ring ? L.ring : f0; f <= f1 && e == cudaSuccess && ring_events; ++f)  // ring frames rendered again
      e = cudaStreamWaitEvent(s, freed[f % L.ring], 0);
    if (e != cudaSuccess) break;
    char* slot = base + L.slots_off + (i % L.n_slots) * L.slot_bytes;
    const cudaError_t g = hr::launch_generate_video_rays(d_cams, d_times, mixed, h->cfg.c_in, cameras[0].width, L.frame_px, off, m,
                                                         (float*)slot, s);
    if (g != cudaSuccess) {
      rc = fail("ray generation", g);
      break;
    }
    h->launches += 1;
    if ((rc = render(off, pos, m, (const float*)slot, (void*)(slot + rays_bytes), L.slot_bytes - rays_bytes, s))) break;
    if (ring_rays && f_end > next) {  // frames next .. f_end - 1 are complete, in consecutive ring frames
      if (ring_events && next * L.frame_px < off) e = cudaStreamWaitEvent(s, done[1 - k], 0);
      if (e != cudaSuccess || (rc = finish(next, f_end, k, s))) break;
      for (int64_t f = next; f < f_end && e == cudaSuccess && ring_events; ++f) e = cudaEventRecord(freed[f % L.ring], s);
      next = f_end;
    }
    if (e == cudaSuccess && ring_events) e = cudaEventRecord(done[k], s);
    off += m;
  }
  if (e != cudaSuccess) rc = fail("stream event", e);
  for (int k = 0; k < 2 && two; ++k) {  // join, also after a failure: the caller's stream must not run ahead of enqueued work
    cudaEvent_t join;
    cudaError_t j = new_event(&join);
    if (j == cudaSuccess) j = cudaEventRecord(join, ss[k]);
    if (j == cudaSuccess) j = cudaStreamWaitEvent(st, join, 0);
    if (j != cudaSuccess && !rc) rc = fail("join", j);
  }
  for (cudaEvent_t ev : evs) cudaEventDestroy(ev);
  return rc;
}
}  // extern "C++"

int hr_render_video_to8b(hr_handle* h, const hr_camera* cameras, const float* times, int32_t n_frames, uint8_t* video,
                         void* workspace, int64_t workspace_bytes, void* stream) {
  const char* fn = "hr_render_video_to8b";
  bool mixed = false;
  if (check_walk(fn, "n_frames", h, !video, cameras, times, n_frames, workspace, &mixed)) return 1;
  WalkLayout L;
  const bool laid_out = walk_layout(h, n_frames, cameras[0].height, cameras[0].width, 0, 0, 0, &L);
  if (check_workspace(fn, laid_out, L, cameras, n_frames, workspace, workspace_bytes)) return 1;
  return walk_frames(
      h, fn, L, cameras, times, n_frames, mixed, workspace, (cudaStream_t)stream,
      [&](int64_t off, int64_t, int64_t m, const float* rays, void* ws, int64_t ws_bytes, cudaStream_t s) {
        return render_impl(h, rays, m, nullptr, nullptr, nullptr, ws, ws_bytes, s, video + off * 3);
      },
      [](int64_t, int64_t, int, cudaStream_t) { return 0; });
}

// ---- held-out splits: every view rendered into a ring of whole fp32 frames and scored against its uint8 ground truth
// A split's walk layout: the fp32 ring [R][H][W][3], then one metrics partial buffer per stream (R frames each).
static bool score_layout(const hr_handle* h, int32_t n_views, int32_t height, int32_t width, WalkLayout* L) {
  return height >= 11 && width >= 11 &&
         walk_layout(h, n_views, height, width, 3 * sizeof(float), 0, hr_image_metrics_workspace_bytes(1, height, width), L);
}

int64_t hr_score_views_workspace_bytes(const hr_handle* h, int32_t n_views, int32_t height, int32_t width) {
  WalkLayout L;
  return score_layout(h, n_views, height, width, &L) ? L.total : -1;
}

// The split's walk renders fp32 rgb into the ring; the frames a sub-batch completes are scored by one metrics launch on its
// stream, with that stream's partial buffer.
int hr_score_views(hr_handle* h, const hr_camera* cameras, const float* times, int32_t n_views, const uint8_t* gt,
                   int32_t pixel_format, double* out, void* workspace, int64_t workspace_bytes, void* stream) {
  const char* fn = "hr_score_views";
  bool mixed = false;
  if (check_walk(fn, "n_views", h, !gt || !out, cameras, times, n_views, workspace, &mixed)) return 1;
  const int32_t W = cameras[0].width, H = cameras[0].height;
  if (H < 11 || W < 11) return hr_fail("%s: height and width must be >= 11 (the SSIM window), got %d x %d", fn, H, W);
  if (((uintptr_t)out & 7) != 0) return hr_fail("%s: out must be 8-byte aligned", fn);
  const int gt_px = hr::pixel_bytes(pixel_format);  // bytes per ground-truth pixel
  if (!gt_px) return hr_fail("%s: unknown pixel format %d", fn, pixel_format);
  if (gt_px == 4 && ((uintptr_t)gt & 3) != 0) return hr_fail("%s: RGBA gt must be 4-byte aligned", fn);
  WalkLayout L;
  const bool laid_out = score_layout(h, n_views, H, W, &L);
  if (check_workspace(fn, laid_out, L, cameras, n_views, workspace, workspace_bytes)) return 1;
  float* ring = (float*)((char*)workspace + L.ring_off);
  const int64_t px = L.frame_px;
  return walk_frames(
      h, fn, L, cameras, times, n_views, mixed, workspace, (cudaStream_t)stream,
      [&](int64_t, int64_t pos, int64_t m, const float* rays, void* ws, int64_t ws_bytes, cudaStream_t s) {
        return render_impl(h, rays, m, ring + pos * 3, nullptr, nullptr, ws, ws_bytes, s);
      },
      [&](int64_t next, int64_t f_end, int k, cudaStream_t s) {
        const cudaError_t e = (gt_px == 4 ? hr::launch_image_metrics_rgba8 : hr::launch_image_metrics_u8)(
            ring + (next % L.ring) * px * 3, gt + next * px * gt_px, (int32_t)(f_end - next), H, W, out + 2 * next,
            (double*)((char*)workspace + L.part_off + k * L.part_bytes), s);
        if (e != cudaSuccess) return hr_fail("%s: metrics launch: %s", fn, cudaGetErrorString(e));
        h->launches += 2;
        return 0;
      });
}

// ---- embedding maps: every request mapped in the render epilogue, or staged in a ring of whole frames and normalised
// The requests' checks; *norm_ch: channels of the normalize requests, each of which has a ring of its own.
static int check_visual_requests(const char* fn, const hr_handle* h, const hr_visual_request* req, int32_t n_req, int* norm_ch) {
  if (n_req < 0 || (n_req > 0 && !req)) return hr_fail("%s: bad request list", fn);
  *norm_ch = 0;
  bool seen[HR_N_FIELDS] = {};
  for (int i = 0; i < n_req; ++i) {
    const hr_visual_request& r = req[i];
    if (r.field < 0 || r.field >= HR_N_FIELDS) return hr_fail("%s: request %d: unknown field %d", fn, i, r.field);
    if (r.mode != HR_FIELD_OVER && r.mode != HR_FIELD_PRED_WEIGHTS)
      return hr_fail("%s: request %d: mode %d is not HR_FIELD_OVER or HR_FIELD_PRED_WEIGHTS", fn, i, r.mode);
    if (seen[r.field]) return hr_fail("%s: field %d requested twice", fn, r.field);
    seen[r.field] = true;
    if (r.channels != kFieldWidth[r.field])
      return hr_fail("%s: request %d: field %d has %d channels, not %d", fn, i, r.field, kFieldWidth[r.field], r.channels);
    if (!r.out) return hr_fail("%s: request %d: null output", fn, i);
    if (r.bounded && !(std::isfinite(r.lo) && std::isfinite(r.hi) && r.hi != r.lo))
      return hr_fail("%s: request %d: bounds [%g, %g] must be finite with hi != lo", fn, i, r.lo, r.hi);
    if (field_refusal(fn, h->cfg, r.field)) return 1;
    if (r.normalize) *norm_ch += r.channels;
  }
  return 0;
}

// An embedding walk's layout: the normalize requests' rings (norm_ch fp32 channels per pixel in all, each request's ring
// 256-byte aligned, in request order), then one min / max partial buffer per stream.  Without a normalize request there is
// no ring, so the walk is the video's.
static bool visual_layout(const hr_handle* h, int norm_ch, int32_t n_frames, int32_t height, int32_t width, WalkLayout* L) {
  return walk_layout(h, n_frames, height, width, norm_ch * (int64_t)sizeof(float), 256 * norm_ch,
                     hr::kVisBlocks * 6 * (int64_t)sizeof(float), L);
}

int64_t hr_render_visuals_workspace_bytes(const hr_handle* h, const hr_visual_request* req, int32_t n_req, int32_t n_frames,
                                          int32_t height, int32_t width) {
  int norm_ch = 0;
  WalkLayout L;
  if (!h || check_visual_requests("hr_render_visuals_workspace_bytes", h, req, n_req, &norm_ch)) return -1;
  if (visual_layout(h, norm_ch, n_frames, height, width, &L)) return L.total;
  hr_fail("hr_render_visuals_workspace_bytes: %d frames of %d x %d pixels: bad size or bytes overflow int64", n_frames, width, height);
  return -1;
}

// The walk renders the video's pixels, the epilogue-mapped requests' bytes and the normalize requests' fp32 fields (into
// their rings) in one render launch per sub-batch; the frames a sub-batch completes are reduced and mapped, per normalize
// request, on its stream.  Without a request the render is hr_render_video_to8b's, launch for launch.
int hr_render_visuals(hr_handle* h, const hr_camera* cameras, const float* times, int32_t n_frames, uint8_t* video,
                      const hr_visual_request* req, int32_t n_req, void* workspace, int64_t workspace_bytes, void* stream) {
  const char* fn = "hr_render_visuals";
  bool mixed = false;
  if (check_walk(fn, "n_frames", h, false, cameras, times, n_frames, workspace, &mixed)) return 1;
  int norm_ch = 0;
  if (check_visual_requests(fn, h, req, n_req, &norm_ch)) return 1;
  if (!video && n_req == 0) return hr_fail("%s: nothing to write (no video and no request)", fn);
  WalkLayout L;
  const bool laid_out = visual_layout(h, norm_ch, n_frames, cameras[0].height, cameras[0].width, &L);
  if (check_workspace(fn, laid_out, L, cameras, n_frames, workspace, workspace_bytes)) return 1;
  const int64_t px = L.frame_px;
  // the render's outputs for a sub-batch starting at ray 0 of the video and of the ring; render moves them along
  hr::ExtraOut so{};
  std::vector<float*> ring_of(n_req, nullptr);
  int64_t ring_at = L.ring_off;
  for (int i = 0; i < n_req; ++i) {
    const hr_visual_request& r = req[i];
    hr::VisMap m{r.out, r.use_abs ? 1 : 0, r.bounded ? 1 : 0, r.lo, r.bounded ? r.hi - r.lo : 1.0f};
    so.field_mode[r.field] = r.mode;
    so.field_u8[r.field] = m;
    if (r.normalize) {
      ring_of[i] = (float*)((char*)workspace + ring_at);
      ring_at += align256(L.ring * px * (int64_t)sizeof(float) * r.channels);
    }
  }
  hr::RgbDst no_rgb{};  // n = 0: the render stores no colour
  return walk_frames(
      h, fn, L, cameras, times, n_frames, mixed, workspace, (cudaStream_t)stream,
      [&](int64_t off, int64_t pos, int64_t m, const float* rays, void* ws, int64_t ws_bytes, cudaStream_t s) {
        hr::ExtraOut so_b = so;
        for (int r = 0; r < n_req; ++r) {
          const int f = req[r].field;
          if (ring_of[r]) {  // staged in fp32 at its ring position; mapped when the frame completes
            so_b.field_out[f] = ring_of[r] + pos * req[r].channels;
            so_b.field_u8[f].out = nullptr;
          } else {
            so_b.field_u8[f].out += off * req[r].channels;
          }
        }
        return render_impl(h, rays, m, nullptr, nullptr, n_req > 0 ? &so_b : nullptr, ws, ws_bytes, s,
                           video ? video + off * 3 : nullptr, video ? nullptr : &no_rgb);
      },
      [&](int64_t next, int64_t f_end, int k, cudaStream_t s) {
        float* part = (float*)((char*)workspace + L.part_off + k * L.part_bytes);
        for (int r = 0; r < n_req; ++r) {
          if (!ring_of[r]) continue;
          hr::VisMap vm = so.field_u8[req[r].field];
          vm.out += next * px * req[r].channels;
          const cudaError_t e = hr::launch_vis_normalize(ring_of[r] + (next % L.ring) * px * req[r].channels, (int)(f_end - next),
                                                         px, req[r].channels, vm, part, s);
          if (e != cudaSuccess) return hr_fail("%s: map launch: %s", fn, cudaGetErrorString(e));
          h->launches += 2;
        }
        return 0;
      });
}

// the device's view of a pinned (device-addressable) host buffer, or null
static float* device_view(const void* host) {
  cudaPointerAttributes pa;
  if (cudaPointerGetAttributes(&pa, host) == cudaSuccess && pa.type == cudaMemoryTypeHost && pa.devicePointer != nullptr)
    return (float*)pa.devicePointer;
  cudaGetLastError();  // pageable memory: not an error, just not device-addressable
  return nullptr;
}

int hr_render_host(hr_handle* h, const float* rays_host, int64_t n_rays, float* rgb_host, int64_t chunk) {
  if (!h) return hr_fail("hr_render_host: null handle");
  if (!h->uploaded) return hr_fail("hr_render_host: parameters not uploaded");
  if (n_rays == 0) return 0;
  if (!rays_host || !rgb_host) return hr_fail("hr_render_host: null buffer");
  DeviceGuard guard(h->device);
  const hr_config& c = h->cfg;
  HostPipe& P = h->pipe;
  // Pinned (device-addressable) buffers are used in place.  The tensor-core sample net reads pinned rays over PCIe -- its
  // encoder warps work one tile ahead of the tensor pipe, so the transfer hides under the math -- and leaves the device
  // copy the render kernel reads.  The render epilogue stores into pinned rgb: 12 bytes per ray as posted writes spread over
  // the kernel's run, made visible by the stream's completion.  A side without a view is copied chunk by chunk.
  HostChunks io;
  const bool net_reads_host = tc_net(c.mlp_mode) && h->net.tc_ready && !c.cascade;
  io.rays_view = net_reads_host ? device_view(rays_host) : nullptr;
  if (!io.rays_view) io.rays_host = rays_host;
  io.rgb_view = device_view(rgb_host);
  if (!io.rgb_view) io.rgb_host = rgb_host;
  // Default chunk for the tensor-core net: 16 tile waves (hr_render's sub-batch), so that a batch of up to 16 waves stays
  // whole, since each further chunk costs a sample-net ramp and a render tail.  A larger batch with a copy on either side
  // goes in one-wave chunks, so that the copies overlap.  The CUDA-core net: 32 768 rays.
  const int64_t wave = (int64_t)h->num_sms * 128;  // one full wave of 128-ray tiles of the tensor-core sample net
  if (chunk <= 0) chunk = !tc_net(c.mlp_mode) ? 32768 : ((io.rays_view && io.rgb_view) || n_rays <= 16 * wave) ? 16 * wave : wave;
  if (chunk > n_rays) chunk = n_rays;
  if (ensure_pipe(h, chunk)) return 1;
  const int64_t n_chunks = (n_rays + chunk - 1) / chunk;
  // A timed call runs directly: render_impl records its events on the streams.  So does a single chunk that copies its
  // rays in, a handful of calls on one stream; a zero-copy batch, the pinned buffers' hot path, is replayed.
  if (h->timing || (n_chunks == 1 && !io.rays_view)) {
    int rc = run_host_chunks(h, n_rays, chunk, io);
    return rc ? rc : sync_pipe(h);
  }
  // Launch-bound when issued call by call: capture the whole multi-stream pipeline once per (buffers, size, chunk) and
  // replay it with a single graph launch.
  if (!(P.graph && P.g_rays == rays_host && P.g_rgb == rgb_host && P.g_n == n_rays && P.g_chunk == chunk)) {
    drop_host_graph(h);
    if (!P.fork_ev) {
      CK(cudaEventCreateWithFlags(&P.fork_ev, cudaEventDisableTiming));
      for (int i = 0; i < 3; ++i) CK(cudaEventCreateWithFlags(&P.join_ev[i], cudaEventDisableTiming));
    }
    const int64_t launches_before = h->launches;
    cudaGraph_t g = nullptr;
    CK(cudaStreamBeginCapture(P.streams[0], cudaStreamCaptureModeRelaxed));
    CK(cudaEventRecord(P.fork_ev, P.streams[0]));
    for (int i = 1; i < 3; ++i) CK(cudaStreamWaitEvent(P.streams[i], P.fork_ev, 0));
    int rc = run_host_chunks(h, n_rays, chunk, io);
    for (int i = 1; i < 3; ++i) {
      cudaEventRecord(P.join_ev[i], P.streams[i]);
      cudaStreamWaitEvent(P.streams[0], P.join_ev[i], 0);
    }
    cudaError_t ce = cudaStreamEndCapture(P.streams[0], &g);
    P.g_launches = h->launches - launches_before;
    h->launches = launches_before;  // capture enqueued nothing; the replay below is what runs
    if (rc) { if (g) cudaGraphDestroy(g); return rc; }
    if (ce != cudaSuccess) return hr_fail("hr_render_host: graph capture failed: %s", cudaGetErrorString(ce));
    ce = cudaGraphInstantiate(&P.graph, g, 0);
    cudaGraphDestroy(g);
    if (ce != cudaSuccess) { P.graph = nullptr; return hr_fail("hr_render_host: graph instantiate failed: %s", cudaGetErrorString(ce)); }
    P.g_rays = rays_host; P.g_rgb = rgb_host; P.g_n = n_rays; P.g_chunk = chunk;
  }
  CK(cudaGraphLaunch(P.graph, P.streams[0]));
  h->launches += P.g_launches;
  CK(cudaStreamSynchronize(P.streams[0]));
  return 0;
}

// ---- backward pass (SURVEY.md 8 f1) ----
static int train_supported(const hr_config& c) {
  if (c.isect_type == HR_ISECT_SPHERE_NEW) return hr_fail("backward: the sphere_new primitive is not supported yet");
  if (c.mlp_mode == HR_MLP_ZERO) { /* no sample net: d heads is simply unused by the caller */ }
  if ((c.isect_type == HR_ISECT_SPHERE || c.isect_type == HR_ISECT_CYLINDER) && c.sphere_origin_scale != 0.0f)
    return hr_fail("backward: learned primitive origins (origin_scale_factor != 0) are not supported yet");
  // the colour transform's gradient is summed per CTA in shared memory
  if (c.n_color_views > 512) return hr_fail("backward: more than 512 colour-transform views are not supported");
  if (c.n_samples > 64) return hr_fail("backward: more than 64 samples per ray are not supported yet");
  if (c.cascade) return hr_fail("backward: cascaded (point_prediction) pipelines are not supported yet");
  return 0;
}

// the fourteen gradient tables as one list, in g_sizes' order: (sigma, appearance) x (space, second) x 3 groups, the basis,
// the colour transform
static void grad_bufs(hr::GradTabs& g, float** out[kGradTables]) {
  for (int i = 0; i < 3; ++i) {
    out[i] = &g.sig_space[i]; out[3 + i] = &g.sig_second[i]; out[6 + i] = &g.app_space[i]; out[9 + i] = &g.app_second[i];
  }
  out[kGradBasis] = &g.basis;
  out[kGradColorEmbedding] = &g.color_embedding;
}

static int ensure_grad_tables(hr_handle* h, cudaStream_t st) {
  const hr_config& c = h->cfg;
  size_t want[kGradTables];
  for (int i = 0; i < 3; ++i) {
    const hr::PlaneTab& t = h->tabs.sig[i];
    const size_t sp = (size_t)t.C * t.H * t.W, se = (size_t)t.C * t.H2 * t.L;
    want[i] = sp; want[3 + i] = se; want[6 + i] = sp; want[9 + i] = se;
  }
  want[kGradBasis] = (size_t)c.app_dim * h->tabs.n_app_total;
  want[kGradColorEmbedding] = (size_t)c.n_color_views * 12;
  float** bufs[kGradTables];
  grad_bufs(h->grads, bufs);
  for (int i = 0; i < kGradTables; ++i) {
    if (h->g_sizes[i] == want[i] && (*bufs[i] || want[i] == 0)) continue;
    if (*bufs[i]) cudaFree(*bufs[i]);
    *bufs[i] = nullptr;
    h->g_sizes[i] = 0;
    if (want[i] == 0) continue;
    cudaError_t e = cudaMalloc((void**)bufs[i], want[i] * sizeof(float));
    if (e != cudaSuccess) return hr_fail("cudaMalloc(gradient table %zu floats): %s", want[i], cudaGetErrorString(e));
    e = cudaMemsetAsync(*bufs[i], 0, want[i] * sizeof(float), st);
    if (e != cudaSuccess) return hr_fail("cudaMemsetAsync: %s", cudaGetErrorString(e));
    h->g_sizes[i] = want[i];
  }
  return 0;
}

int hr_encode_rays(hr_handle* h, const float* rays, int64_t n_rays, float* enc, void* stream) {
  if (!h || !rays || !enc) return hr_fail("hr_encode_rays: null argument");
  if (h->cfg.cascade) return hr_fail("hr_encode_rays: a cascaded pipeline has two nets; its training path is not built");
  if (n_rays == 0) return 0;
  DeviceGuard guard(h->device);
  encode_rays_kernel<<<grid_for(n_rays), 256, 0, (cudaStream_t)stream>>>(h->cfg, rays, enc, n_rays);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return hr_fail("hr_encode_rays: %s", cudaGetErrorString(e));
  h->launches += 1;
  return 0;
}

int hr_render_heads(hr_handle* h, const float* rays, const float* heads, int64_t n, float* rgb, const hr_train_opts* opts,
                    void* workspace, int64_t workspace_bytes, void* stream) {
  if (!h || !rays || !heads || !rgb || !opts || !workspace) return hr_fail("hr_render_heads: null argument");
  if (!h->uploaded) return hr_fail("hr_render_heads: parameters not uploaded");
  if (n == 0) return 0;
  if (workspace_bytes < heads_bytes(h, n)) return hr_fail("hr_render_heads: workspace too small");
  DeviceGuard guard(h->device);
  cudaStream_t st = (cudaStream_t)stream;
  hr_config c = h->cfg;
  c.clamp_output = opts->clamp_output ? 1 : 0;
  c.white_bg = opts->white_bg ? 1 : 0;
  if (opts->white_bg) c.black_bg = 0;
  float* hcm = (float*)workspace;
  cudaError_t e = permute_heads_async(c, heads, hcm, n, st);
  if (e == cudaSuccess) e = hr::launch_render(c, h->dv, h->tabs, rays, hcm, one_dst(rgb), n, nullptr, h->num_sms, st, nullptr);
  if (e != cudaSuccess) return hr_fail("hr_render_heads: %s", cudaGetErrorString(e));
  h->launches += 2;
  return 0;
}

int hr_render_backward(hr_handle* h, const float* rays, const float* heads, int64_t n, const float* d_rgb, float* d_heads,
                       const hr_train_opts* opts, void* workspace, int64_t workspace_bytes, void* stream) {
  if (!h || !rays || !heads || !d_rgb || !d_heads || !opts || !workspace) return hr_fail("hr_render_backward: null argument");
  if (!h->uploaded) return hr_fail("hr_render_backward: parameters not uploaded");
  if (train_supported(h->cfg)) return 1;
  if (n == 0) return 0;
  if (workspace_bytes < 2 * heads_bytes(h, n)) return hr_fail("hr_render_backward: workspace too small (hr_train_workspace_bytes)");
  DeviceGuard guard(h->device);
  cudaStream_t st = (cudaStream_t)stream;
  const hr_config& c = h->cfg;
  if (ensure_grad_tables(h, st)) return 1;
  float* hcm = (float*)workspace;
  float* gcm = (float*)((char*)workspace + heads_bytes(h, n));
  cudaError_t e = permute_heads_async(c, heads, hcm, n, st);
  if (e != cudaSuccess) return hr_fail("hr_render_backward: %s", cudaGetErrorString(e));
  const int white = opts->white_bg ? 1 : 0;
  EventPair eb{nullptr, nullptr};
  const bool timing = h->timing && h->ev_bwd.size() < 8192;
  if (timing) { CK(cudaEventCreate(&eb.a)); CK(cudaEventCreate(&eb.b)); CK(cudaEventRecord(eb.a, st)); }
  e = hr::launch_render_bwd(c, h->dv, h->tabs, h->grads, rays, hcm, d_rgb, gcm, n, opts->clamp_output ? 1 : 0, white, h->num_sms, st);
  if (e != cudaSuccess) return hr_fail("hr_render_backward: %s", cudaGetErrorString(e));
  if (timing) { CK(cudaEventRecord(eb.b, st)); h->ev_bwd.push_back(eb); }
  e = unpermute_heads_async(c, gcm, d_heads, n, st);
  if (e != cudaSuccess) return hr_fail("hr_render_backward: %s", cudaGetErrorString(e));
  h->launches += 3;
  return 0;
}

int hr_grad_zero(hr_handle* h, void* stream) {
  if (!h) return hr_fail("hr_grad_zero: null handle");
  if (!h->uploaded) return hr_fail("hr_grad_zero: parameters not uploaded");
  DeviceGuard guard(h->device);
  cudaStream_t st = (cudaStream_t)stream;
  if (ensure_grad_tables(h, st)) return 1;
  float** bufs[kGradTables];
  grad_bufs(h->grads, bufs);
  for (int i = 0; i < kGradTables; ++i)
    if (*bufs[i]) CK(cudaMemsetAsync(*bufs[i], 0, h->g_sizes[i] * sizeof(float), st));
  return 0;
}

int hr_grad_read(hr_handle* h, const hr_grads* out, void* stream) {
  if (!h || !out) return hr_fail("hr_grad_read: null argument");
  if (!h->uploaded) return hr_fail("hr_grad_read: parameters not uploaded");
  DeviceGuard guard(h->device);
  cudaStream_t st = (cudaStream_t)stream;
  if (ensure_grad_tables(h, st)) return 1;
  const hr_config& c = h->cfg;
  for (int i = 0; i < 3; ++i) {
    const hr::PlaneTab& t = h->tabs.sig[i];
    if (t.C == 0) continue;
    for (int f = 0; f < 2; ++f) {
      float* dsp = f ? out->app_plane[i] : out->sigma_plane[i];
      float* dse = f ? out->app_second[i] : out->sigma_second[i];
      const float* gsp = f ? h->grads.app_space[i] : h->grads.sig_space[i];
      const float* gse = f ? h->grads.app_second[i] : h->grads.sig_second[i];
      if (dsp) unpack_channel_last<<<grid_for((long long)t.C * t.H * t.W), 256, 0, st>>>(gsp, dsp, t.C, t.H, t.W);
      if (dse) {
        if (c.dynamic)
          unblend_time_lines<<<grid_for((long long)t.C * t.H2 * t.L), 256, 0, st>>>(gse, dse, t.C, t.H2, t.L, h->dv.time_inv_fac,
                                                                                   h->dv.time_scale, h->dv.time_offset);
        else
          unpack_channel_last<<<grid_for((long long)t.C * t.H2 * t.L), 256, 0, st>>>(gse, dse, t.C, t.H2, t.L);
      }
    }
  }
  if (out->basis_mat) CK(cudaMemcpyAsync(out->basis_mat, h->grads.basis, h->g_sizes[kGradBasis] * sizeof(float), cudaMemcpyDeviceToDevice, st));
  if (out->color_embedding && h->g_sizes[kGradColorEmbedding])
    CK(cudaMemcpyAsync(out->color_embedding, h->grads.color_embedding, h->g_sizes[kGradColorEmbedding] * sizeof(float),
                       cudaMemcpyDeviceToDevice, st));
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return hr_fail("hr_grad_read: %s", cudaGetErrorString(e));
  return 0;
}

// ---- the sample net's training forward / backward on the tensor cores (hr_mlp_tc2.cu, hr_mlp_train.cu) ----
static int train_net_supported(const hr_handle* h, const char* fn) {
  const hr_config& c = h->cfg;
  if (c.cascade) return hr_fail("%s: cascaded (point_prediction) pipelines have two sample nets; only single-net pipelines train on the tensor cores", fn);
  if (c.mlp_mode == HR_MLP_ZERO) return hr_fail("%s: a zero sample net has no layers to train", fn);
  if (c.mlp_mode != HR_MLP_BF16X3_TC) return hr_fail("%s: the training forward is the wgmma sample net: create the handle with mlp_mode HR_MLP_BF16X3_TC", fn);
  if (!h->uploaded || !h->net.tc_ready) return hr_fail("%s: parameters not uploaded", fn);
  return 0;
}

int64_t hr_train_net_workspace_bytes(const hr_handle* h, int64_t n_rays) {
  if (!h || n_rays < 0) return -1;
  return (int64_t)hr::train_net_layout(h->cfg, n_rays, h->num_sms).total;
}

int hr_train_net_forward(hr_handle* h, const float* rays, int64_t n, float* heads, void* workspace, int64_t workspace_bytes,
                         void* stream) {
  if (!h || !rays || !heads || !workspace) return hr_fail("hr_train_net_forward: null argument");
  if (train_net_supported(h, "hr_train_net_forward")) return 1;
  if (n == 0) return 0;
  const hr::TrainNetLayout t = hr::train_net_layout(h->cfg, n, h->num_sms);
  if (workspace_bytes < (int64_t)t.total) return hr_fail("hr_train_net_forward: workspace too small (hr_train_net_workspace_bytes)");
  if (((uintptr_t)workspace & 255) != 0) return hr_fail("hr_train_net_forward: workspace must be 256-byte aligned");
  DeviceGuard guard(h->device);
  uint8_t* ws = (uint8_t*)workspace;
  const hr::TrainSave sv{(float*)(ws + t.enc), (float*)(ws + t.act), (long long)t.act_stride, t.ld_enc};
  cudaError_t e = hr::launch_mlp_tc2_train(h->cfg, h->net.tc, rays, heads, n, h->num_sms, (cudaStream_t)stream, sv);
  if (e != cudaSuccess) return hr_fail("hr_train_net_forward: %s", cudaGetErrorString(e));
  h->launches += 1;
  return 0;
}

int hr_train_net_backward(hr_handle* h, const float* d_heads, int64_t n, const hr_net_grads* out, void* workspace,
                          int64_t workspace_bytes, void* stream) {
  if (!h || !d_heads || !out || !workspace) return hr_fail("hr_train_net_backward: null argument");
  if (train_net_supported(h, "hr_train_net_backward")) return 1;
  const hr_config& c = h->cfg;
  const int L = c.mlp_layers, W = c.mlp_width;
  for (int l = 0; l < L; ++l)
    if (!out->weight[l] || !out->bias[l]) return hr_fail("hr_train_net_backward: gradient buffers of layer %d missing", l);
  DeviceGuard guard(h->device);
  cudaStream_t st = (cudaStream_t)stream;
  if (n == 0) {  // no rays: every gradient is zero
    for (int l = 0; l < L; ++l) {
      const int out_l = l == L - 1 ? c.mlp_out : W, in_l = l == 0 ? c.mlp_in : (l == c.mlp_skip ? c.mlp_in + W : W);
      CK(cudaMemsetAsync(out->weight[l], 0, (size_t)out_l * in_l * sizeof(float), st));
      CK(cudaMemsetAsync(out->bias[l], 0, (size_t)out_l * sizeof(float), st));
    }
    return 0;
  }
  const hr::TrainNetLayout t = hr::train_net_layout(c, n, h->num_sms);
  if (workspace_bytes < (int64_t)t.total) return hr_fail("hr_train_net_backward: workspace too small (hr_train_net_workspace_bytes)");
  if (((uintptr_t)workspace & 255) != 0) return hr_fail("hr_train_net_backward: workspace must be 256-byte aligned");
  uint8_t* ws = (uint8_t*)workspace;
  cudaError_t e = permute_heads_async(c, d_heads, (float*)(ws + t.dlast), n, st, t.ld_dlast);
  if (e == cudaSuccess) e = hr::train_net_backward(c, h->net.simt, n, out->weight, out->bias, ws, h->num_sms, st);
  if (e != cudaSuccess) return hr_fail("hr_train_net_backward: %s", cudaGetErrorString(e));
  h->launches += 1 + 3 * L;
  return 0;
}

// every hr_act member of hr_config (the members hr_set_activations may change)
static hr_act hr_config::* const kActMembers[] = {
    &hr_config::act_z, &hr_config::act_flow, &hr_config::act_sigma, &hr_config::act_point_sigma, &hr_config::act_offset,
    &hr_config::act_cscale, &hr_config::act_cshift, &hr_config::isect_act, &hr_config::flow_act, &hr_config::offset_act,
    &hr_config::act_cscale_global, &hr_config::act_cshift_global, &hr_config::act_ctransform, &hr_config::act_ctshift,
    &hr_config::pre_act_z, &hr_config::pre_act_sigma, &hr_config::pre_isect_act};

int hr_set_activations(hr_handle* h, const hr_config* cfg) {
  if (!h || !cfg) return hr_fail("hr_set_activations: null argument");
  // everything but the activations must be the handle's configuration (hr_config has no padding: 4-byte members only)
  hr_config probe = *cfg;
  for (hr_act hr_config::* m : kActMembers) probe.*m = h->cfg.*m;
  if (memcmp(&probe, &h->cfg, sizeof(hr_config)) != 0)
    return hr_fail("hr_set_activations: the configuration differs from the handle's beyond its activations (create a new handle)");
  for (hr_act hr_config::* m : kActMembers) {
    const hr_act& a = cfg->*m;
    if (a.kind != HR_ACT_IDENTITY && a.kind != HR_ACT_SIGMOID && a.kind != HR_ACT_TANH)
      return hr_fail("hr_set_activations: unknown activation kind %d", a.kind);
    if (a.eased && m != &hr_config::act_sigma && m != &hr_config::act_point_sigma && m != &hr_config::pre_act_sigma)
      return hr_fail("hr_set_activations: only act_sigma, act_point_sigma and pre_act_sigma may be eased");
  }
  if (hr::eases_density(*cfg) && cfg->n_samples > 64)
    return hr_fail("hr_set_activations: eased density heads above 64 samples per ray are not supported");
  // the nets' configurations (net.cfg / pre.cfg) are copies of cfg: keep their activations in step, although no net reads them
  for (hr_act hr_config::* m : kActMembers) h->cfg.*m = h->net.cfg.*m = h->pre.cfg.*m = cfg->*m;
  drop_host_graph(h);  // its kernel nodes hold the old configuration by value
  return 0;
}

int64_t hr_launch_count(const hr_handle* h) { return h ? h->launches : -1; }

int hr_timing_enable(hr_handle* h, int enable) {
  if (!h) return hr_fail("null handle");
  h->timing = enable != 0;
  return 0;
}

static void drop_events(std::vector<EventPair>& v) {
  for (auto& p : v) { cudaEventDestroy(p.a); cudaEventDestroy(p.b); }
  v.clear();
}

int hr_timing_reset(hr_handle* h) {
  if (!h) return hr_fail("null handle");
  drop_events(h->ev_render);
  drop_events(h->ev_mlp);
  drop_events(h->ev_bwd);
  h->timed_calls = 0;
  return 0;
}

// waits for every pair and adds up their elapsed times
static int sum_event_ms(std::vector<EventPair>& v, double* sum) {
  *sum = 0;
  for (auto& p : v) {
    CK(cudaEventSynchronize(p.b));
    float ms = 0; CK(cudaEventElapsedTime(&ms, p.a, p.b)); *sum += ms;
  }
  return 0;
}

int hr_timing_read_backward(hr_handle* h, double* backward_ms_avg, int64_t* launches) {
  if (!h) return hr_fail("null handle");
  double sb = 0;
  if (sum_event_ms(h->ev_bwd, &sb)) return 1;
  const size_t k = h->ev_bwd.size();
  if (backward_ms_avg) *backward_ms_avg = k ? sb / k : 0.0;
  if (launches) *launches = (int64_t)k;
  return 0;
}

int hr_timing_read(hr_handle* h, double* render_ms_avg, double* mlp_ms_avg, int64_t* launches) {
  if (!h) return hr_fail("null handle");
  double sr = 0, sm = 0;
  if (sum_event_ms(h->ev_render, &sr) || sum_event_ms(h->ev_mlp, &sm)) return 1;
  // per hr_render call: a call may run several sub-batches, i.e. several launches of each kernel
  const size_t k = h->timed_calls;
  if (render_ms_avg) *render_ms_avg = k ? sr / k : 0.0;
  if (mlp_ms_avg) *mlp_ms_avg = k ? sm / k : 0.0;
  if (launches) *launches = (int64_t)h->ev_render.size();
  return 0;
}

int hr_destroy(hr_handle* h) {
  if (!h) return 0;
  DeviceGuard guard(h->device);
  for (auto& sl : h->slots) cudaFree(sl.ptr);
  float** grads[kGradTables];
  grad_bufs(h->grads, grads);
  for (float** g : grads) cudaFree(*g);
  hr::free_mlp_tc2(h->net);
  hr::free_mlp_tc2(h->pre);
  drop_events(h->ev_render);
  drop_events(h->ev_mlp);
  drop_events(h->ev_bwd);
  drop_host_graph(h);
  if (h->pipe.fork_ev) cudaEventDestroy(h->pipe.fork_ev);
  for (int i = 0; i < 3; ++i) {
    if (h->pipe.join_ev[i]) cudaEventDestroy(h->pipe.join_ev[i]);
    if (h->pipe.d_rays[i]) cudaFree(h->pipe.d_rays[i]);
    if (h->pipe.d_rgb[i]) cudaFree(h->pipe.d_rgb[i]);
    if (h->pipe.d_ws[i]) cudaFree(h->pipe.d_ws[i]);
    if (h->pipe.streams[i]) cudaStreamDestroy(h->pipe.streams[i]);
  }
  delete h;
  return 0;
}

}  // extern "C"
