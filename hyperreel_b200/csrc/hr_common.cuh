// Shared device-side types for the hyperreel_b200 kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "hyperreel_b200.h"

namespace hr {

// One VM factor pair, channel-last (DESIGN.md "Data layout in HBM"):
//   space  [H][W][C]   (reference [1,C,H,W]: x -> W (axis a), y -> H (axis b))
//   second [H2][L][C]  dynamic: H2 = K keyframe rows, x -> L (axis c), y -> time
//                      static : H2 = 1, the line [L][C]
struct PlaneTab {
  const float* space;
  const float* second;
  int H, W;   // space plane rows / cols
  int H2, L;  // second factor rows / cols
  int C;      // channels (0 = group absent, 4 or 8)
};

struct RenderTabs {
  PlaneTab sig[3];
  PlaneTab app[3];
  const float* basis;  // [app_dim][sum C_app] row-major
  int n_app_total;
  const float* color_embedding;  // [n_color_views][12] per-camera colour transform + shift (point.py:558-592), or null
};

// Gradient tables: same channel-last layout as the forward's PlaneTab (second factor: pre-blended keyframe lines / lines).
struct GradTabs {
  float* sig_space[3];
  float* sig_second[3];
  float* app_space[3];
  float* app_second[3];
  float* basis;  // [app_dim][NT]
  float* color_embedding;  // [n_color_views][12] (RARE variants only; null without a colour transform)
};

// Host-derived scalars (computed in double on the host, then rounded once to fp32, the way the
// reference's Python-float constants meet fp32 tensors).
struct Derived {
  float time_fac;       // K*(F-1)/F            (utils/flow_utils.py:19)
  float time_inv_fac;   // 1/fac                (flow_utils.py:31)
  float time_scale;     // (F-1)/F              (tensorf_dynamic.py:58)
  float time_offset;    // 0.5/K                (tensorf_dynamic.py:59)
  float kf_max;         // K-1
  float inv_end_dist;   // contract_start_distance / contract_end_distance (contract.py:145)
  float dist_scale_fac; // 1/(1-inv_end_dist)
  float inv_end_rad;    // contract_start_radius / contract_end_radius (contract.py:184)
  float rad_scale_fac;  // 1/(1-inv_end_rad)
  int res[3];           // grid resolution along x, y, z (taken from the uploaded tables)
  int kt;               // rows of the (axis, time) planes = number of keyframes
};

// Where the finished pixels go: one or more [n_total,3] fp32 buffers (the local output; or, for ray-sharded rendering, the
// same row range of every rank's gather buffer, peer pointers mapped over NVLink -- the render kernel's epilogue is the
// gather).  `row0` is added to the ray index.
struct RgbDst {
  float* p[HR_MAX_PEERS];
  int n;
  long long row0;
};

// The elementwise steps of one embedding map (visualize_warp, utils/visualization.py:24-52): |x| when use_abs, then
// (x - lo) / den when bounded, den = hi - lo rounded once in fp32.  `out` is the map's uint8 [n, dim] when the render
// epilogue finishes it (no normalize), null otherwise.
struct VisMap {
  unsigned char* out;
  int use_abs, bounded;
  float lo, den;
};

// blocks per frame of the normalize reduction (hr_visual.cu): each writes one min / max partial per channel
constexpr int kVisBlocks = 64;

__device__ __forceinline__ float vis_pre(const VisMap& m, float x) {
  if (m.use_abs) x = fabsf(x);
  if (m.bounded) x = __fdiv_rn(__fsub_rn(x, m.lo), m.den);
  return x;
}

// clamp(0, 1) then to8b (utils/__init__.py:47): (uint8)(255 * x), truncated.  A NaN clamps to NaN and NumPy casts it to 0;
// fmaxf(NaN, 0) is 0, which gives the same byte.
__device__ __forceinline__ unsigned char vis_to8b(float x) {
  return (unsigned char)(int)__fmul_rn(255.0f, fminf(fmaxf(x, 0.0f), 1.0f));
}

// Outputs beyond rgb, produced by the EXTRA variant of the render kernel (all pointers may be null):
//   * per-sample dumps for stage-boundary parity tests (hr_render_stages);
//   * the extra composited fields of the reference's colour nets (tensorf_dynamic.py:808-837, tensorf_no_sample.py:254-278):
//     field_out[f] receives sum_s w_s * x[f]_s ([n, dim], HR_FIELD_OVER), sum_s pred_w_s * x[f]_s (HR_FIELD_PRED_WEIGHTS) or
//     the per-sample values themselves ([n, S*dim], HR_FIELD_NO_OVER).
struct ExtraOut {
  float* distances;    // [n,S]
  float* points;       // [n,S,3]
  float* sigma;        // [n,S]
  float* weights;      // [n,S]
  float* rgb_samples;  // [n,S,3] shaded colour of every sample before the colour transform, 0 where w <= rm_weight_mask_thre
  float* field_out[HR_N_FIELDS];
  int field_mode[HR_N_FIELDS];
  VisMap field_u8[HR_N_FIELDS];  // field_u8[f].out: the reduced field f (HR_FIELD_OVER / PRED_WEIGHTS) as a uint8 map instead
};

// `kind` is a.kind, or the same value known at compile time (a render kernel's fixed head layout, hr_render_kernel.cuh)
__device__ __forceinline__ float apply_act_kind(int kind, const hr_act& a, float x) {
  // y = f(x*inner + shift) * outer, each op rounded separately like the eager reference.
  float v = __fadd_rn(__fmul_rn(x, a.inner_fac), a.shift);
  // ex2-based forms: relative error ~2e-6, far below the 1e-4 RGB gate and cheaper than expf / tanhf by ~4x
  if (kind == HR_ACT_SIGMOID) {
    v = __fdividef(1.0f, 1.0f + __expf(-v));
  } else if (kind == HR_ACT_TANH) {
    const float av = fminf(fabsf(v), 15.0f);
    const float t = 1.0f - __fdividef(2.0f, 1.0f + __expf(2.0f * av));
    v = copysignf(t, v);
  }
  return __fmul_rn(v, a.outer_fac);
}

__device__ __forceinline__ float apply_act(const hr_act& a, float x) { return apply_act_kind(a.kind, a, x); }

// apply_act of a density head (act_sigma, act_point_sigma, pre_act_sigma: the only members hr_config may ease), with
// EaseValue.ease_out (activations.py:482-489): w * out + (1 - w) * start_value while the window is open.  `eased` is uniform
// (a __grid_constant__ config), so a closed window runs exactly apply_act's arithmetic.
__device__ __forceinline__ float apply_act_eased(const hr_act& a, float x) {
  const float v = apply_act(a, x);
  return a.eased ? __fadd_rn(__fmul_rn(v, a.ease_mul), a.ease_add) : v;
}

// a density head's activation in a render kernel: the EASE variants (launched only while an EaseValue window is open, see
// eases_density) blend; the others compile exactly apply_act
template <bool EASE>
__device__ __forceinline__ float apply_act_head(const hr_act& a, float x) {
  if constexpr (EASE) return apply_act_eased(a, x);
  else return apply_act(a, x);
}

// true while act_sigma or act_point_sigma is eased: the render kernels' EASE variants serve the configuration
__host__ __device__ inline bool eases_density(const hr_config& c) { return c.act_sigma.eased || c.act_point_sigma.eased; }

// intersect_axis_plane (intersect_utils.py:127-150): distance along o + t d to the plane {x_a = z}, with o, d the ray's
// components along axis a.  axis_plane_dir is the guarded divisor: a component below 1e-5 in magnitude becomes 1e12.
__device__ __forceinline__ float axis_plane_dir(float d) { return (fabsf(d) < 1e-5f) ? 1e12f : d; }

__device__ __forceinline__ float intersect_axis_plane(float z, float o, float d) {
  const float dg = axis_plane_dir(d);
  return __fdiv_rn(__fsub_rn(z, o), dg);
}

// Bytes per pixel of an HR_PIXEL_* format, 0 for an unknown one
__host__ __device__ inline int pixel_bytes(int32_t pixel_format) {
  return pixel_format == HR_PIXEL_RGB8 ? 3 : pixel_format == HR_PIXEL_RGBA8 ? 4 : 0;
}

// A uint8 channel as a colour, u8 / 255 correctly rounded (T.ToTensor()).  T is the type the byte was loaded as: the
// conversion instruction follows it.
template <class T>
__device__ __forceinline__ float u8_unit(T v) { return __fdiv_rn((float)v, 255.0f); }

// Channel ch (0..2) of the RGBA pixel q (little-endian, alpha in the top byte) composited over white, as the RGBA datasets'
// get_rgb computes it on the CPU: c * a + (1 - a) of the u8 / 255 values, each operation rounded on its own (no FMA).
// Training colours and held-out scores both read RGBA ground truth through this, so they agree bit for bit.
__device__ __forceinline__ float rgba_over_white(uint32_t q, int ch) {
  const float a = u8_unit(q >> 24);
  const float c = u8_unit((q >> (8 * ch)) & 0xffu);
  return __fadd_rn(__fmul_rn(c, a), __fsub_rn(1.0f, a));
}

}  // namespace hr
