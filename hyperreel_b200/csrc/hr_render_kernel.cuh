// Fused per-ray render kernel: heads -> intersect -> sort -> points -> VM gather -> decode -> composite.
//
// One warp renders one ray.  Two lane mappings are used:
//   * "lane = sample"  (S <= 32*SPL samples, SPL registers per lane) for everything that is per-sample
//     scalar math: head activations, intersection, the bitonic sort of t, points, validity, alpha,
//     the transmittance scan (reference: nlf/intersect/base.py:142-259, nlf/embedding/point.py:780-831,
//     371-396, utils/tensorf_utils.py:242-253);
//   * "quad = sample"  (4 lanes per sample, 8 samples per round) for the VM gather: the 4 lanes of a
//     quad fetch the bilinear footprint of one sample as 16-byte slices of channel-last texels so that
//     the two x-neighbouring taps (64 contiguous bytes for C=8) are served by adjacent lanes of one
//     LDG.128 (reference: F.grid_sample calls in nlf/nets/tensorf_dynamic.py:287-371 and
//     nlf/nets/tensorf_no_sample.py:47-126).
// Nothing per-sample ever goes to HBM: rays (4*c_in B) + sample-net heads in, rgb (12 B) out.
// Models with S <= 16 samples per ray run two rays per warp (RPW == 2): lanes 16r .. 16r+15 are the samples of ray r in the
// lane = sample mapping, and the 32 sample slots of the warp feed the four gather rounds exactly like one 32-sample ray, so
// no lane idles in either mapping (one ray per warp left half of every warp idle at S = 16, the DoNeRF BASELINE config).
#pragma once
#include <type_traits>

#include "hr_common.cuh"
#include "hr_geom.cuh"

namespace hr {

static constexpr int kWarpsPerCta = 8;
static constexpr int kMinCtasPerSm = 3;

// One factor table fetch for one sample, spread over the 4 lanes of a quad.
//   C == 8 : lane (xt, alt) reads the 16-byte half `alt` of texel x0+xt in rows y0 (a) and y0+1 (b)
//   C == 4 : lane (xt, yt=alt) reads the whole 16-byte texel (x0+xt, y0+yt) into a
// `off` is the element offset of texel (x0, y0) * C already advanced to this lane's slice; `rs` the row stride in
// elements.  Coordinates are clamped to [0, size-2] on the producer side, so every address is in range and the
// loads need no predicate (invalid samples are redirected to offset 0 and zero-weighted).
template <int C, bool ROWS2>
struct Taps {
  float4 a, b;
};

template <int C, bool ROWS2>
__device__ __forceinline__ void fetch(Taps<C, ROWS2>& t, const float* __restrict__ tab, int off, int rs) {
  t.a = ldg4(tab + off);
  if constexpr (C == 8 && ROWS2) t.b = ldg4(tab + off + rs);
}

// This lane's share of the bilinear plane interpolation (no cross-lane traffic):
//   C == 8: its x tap, both rows, its 4-channel half;  C == 4: its (x, y) tap, all 4 channels.
// Summing the shares over the quad (C == 8: over xt; C == 4: over xt and yt) gives the interpolated channels.
template <int C>
__device__ __forceinline__ void plane_share(const Taps<C, true>& t, float fa, float fb, int xt, int alt, float (&out)[4]) {
  const float wa = xt ? fa : 1.0f - fa;
  if constexpr (C == 8) {
    const float w0 = wa * (1.0f - fb), w1 = wa * fb;
    out[0] = fmaf(w1, t.b.x, w0 * t.a.x);
    out[1] = fmaf(w1, t.b.y, w0 * t.a.y);
    out[2] = fmaf(w1, t.b.z, w0 * t.a.z);
    out[3] = fmaf(w1, t.b.w, w0 * t.a.w);
  } else {
    const float w = wa * (alt ? fb : 1.0f - fb);
    out[0] = w * t.a.x; out[1] = w * t.a.y; out[2] = w * t.a.z; out[3] = w * t.a.w;
  }
}

// The second factor (2-tap line), complete in every lane of the quad: each lane holds the tap of its xt (C == 8: its channel
// half; C == 4: all 4 channels, the two yt lanes hold the same tap), so one exchange across xt finishes it -- 4 shuffles.
template <int C>
__device__ __forceinline__ void line_full(const Taps<C, false>& t, float fc, int xt, float (&out)[4]) {
  const float wc = xt ? fc : 1.0f - fc;
  out[0] = wc * t.a.x; out[1] = wc * t.a.y; out[2] = wc * t.a.z; out[3] = wc * t.a.w;
#pragma unroll
  for (int c = 0; c < 4; ++c) out[c] += __shfl_xor_sync(kFull, out[c], 2);
}

// One VM group (space plane x second factor) of one field for one sample.
//   ia/fa, ib/fb : texel index / fraction along the plane's x and y axes; ic/fc along the second factor's axis
//   krow         : row of the second-factor table: the ray's keyframe (dynamic; hr_upload pre-blends the two
//                  keyframe rows grid_sample would mix for that keyframe, see pack_time_lines) or 0 (static line)
template <int C, bool DYN>
struct GroupTaps {
  Taps<C, true> sp;
  Taps<C, false> se;
};

template <int C, bool DYN>
__device__ __forceinline__ void group_fetch(GroupTaps<C, DYN>& g, const PlaneTab& T, int ia, int ib, int ic, int krow, int xt,
                                            int alt, bool ok) {
  int so, eo;
  if constexpr (C == 8) {
    so = ((ib * T.W + ia + xt) << 3) + (alt << 2);
    eo = ((krow * T.L + ic + xt) << 3) + (alt << 2);
  } else {
    so = ((ib + alt) * T.W + ia + xt) << 2;
    eo = (krow * T.L + ic + xt) << 2;
  }
  so = ok ? so : 0;
  eo = ok ? eo : 0;
  fetch<C, true>(g.sp, T.space, so, T.W * C);
  fetch<C, false>(g.se, T.second, eo, 0);
}

// Density feature of one group: sum_c plane_c * line_c.  The plane stays in per-lane shares: the products with the complete
// line are summed per lane and only the scalar crosses the quad (2 shuffles instead of 4 + 1 for C == 8, 8 for C == 4).
template <int C, bool DYN>
__device__ __forceinline__ float group_sigma(const GroupTaps<C, DYN>& g, float fa, float fb, float fc, int xt, int alt) {
  float P[4], L[4];
  plane_share<C>(g.sp, fa, fb, xt, alt, P);
  line_full<C>(g.se, fc, xt, L);
  float s = (P[0] * L[0] + P[1] * L[1]) + (P[2] * L[2] + P[3] * L[3]);
  s += __shfl_xor_sync(kFull, s, 2);
  s += __shfl_xor_sync(kFull, s, 1);
  return s;
}

// Appearance features of one group: prod[4] = plane_c * line_c for this lane's channels (C == 8: own half; C == 4: all four,
// replicated in the quad).
template <int C, bool DYN>
__device__ __forceinline__ void group_app(const GroupTaps<C, DYN>& g, float fa, float fb, float fc, int xt, int alt,
                                          float (&prod)[4]) {
  float P[4], L[4];
  plane_share<C>(g.sp, fa, fb, xt, alt, P);
  line_full<C>(g.se, fc, xt, L);
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    P[c] += __shfl_xor_sync(kFull, P[c], 2);
    if constexpr (C == 4) P[c] += __shfl_xor_sync(kFull, P[c], 1);
    prod[c] = P[c] * L[c];
  }
}

// One VM group's contribution to this lane's four partial sums v = (colour 0, colour 1, colour 2, density feature):
//   density    v[3] += sum_c plane_c * line_c                    (tensorf_dynamic.py:330, tensorf_no_sample.py:76-78)
//   appearance v[q] += sum_c G[q][c] * plane_c * line_c           (basis_mat + shading folded into G, :371 / tensorf_utils.py:334-343)
// The plane factors stay per-lane shares (this lane's taps only) and the line factors are completed with one exchange each, so
// the products are partial sums over the quad: nothing but the two line exchanges (4 shuffles each) crosses lanes here; the
// four scalars of ALL groups are reduced once per sample by quad_transpose_reduce.
template <int C, bool DYN>
__device__ __forceinline__ void group_accumulate(const GroupTaps<C, DYN>& sg, const GroupTaps<C, DYN>& ag, float fa, float fb,
                                                 float fc, int xt, int alt, const float* __restrict__ G0,
                                                 const float* __restrict__ G1, const float* __restrict__ G2, float (&v)[4]) {
  float P[4], L[4];
  plane_share<C>(sg.sp, fa, fb, xt, alt, P);
  line_full<C>(sg.se, fc, xt, L);
  v[3] += (P[0] * L[0] + P[1] * L[1]) + (P[2] * L[2] + P[3] * L[3]);
  plane_share<C>(ag.sp, fa, fb, xt, alt, P);
  line_full<C>(ag.se, fc, xt, L);
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const float t = P[c] * L[c];
    v[0] = fmaf(G0[c], t, v[0]);
    v[1] = fmaf(G1[c], t, v[1]);
    v[2] = fmaf(G2[c], t, v[2]);
  }
}

// Sum v[0..3] over the 4 lanes of a quad so that lane q ends up with the total of v[q] (a transposing butterfly: 3 shuffles
// instead of the 8 of four replicated all-reduces).  Lane q = (xt << 1) | alt.
__device__ __forceinline__ float quad_transpose_reduce(const float (&v)[4], int xt, int alt) {
  const float x = __shfl_xor_sync(kFull, xt ? v[0] : v[2], 2);
  const float y = __shfl_xor_sync(kFull, xt ? v[1] : v[3], 2);
  const float k0 = (xt ? v[2] : v[0]) + x;  // xt = 0 keeps (v0, v1), xt = 1 keeps (v2, v3)
  const float k1 = (xt ? v[3] : v[1]) + y;
  const float z = __shfl_xor_sync(kFull, alt ? k0 : k1, 1);
  return (alt ? k1 : k0) + z;                // q = 0: v0, 1: v1, 2: v2, 3: v3
}

// The head layout of a launch: which heads the sample net writes, the primitive they place, which density scales the point
// offset and the activation kind of every head.  These are the same for every ray of a launch.  HeadsAny reads them from the
// config where they are used, for every configuration.  The fixed layouts state them at compile time for the shipped
// dynamic z-plane configs (technicolor_z_plane, neural_3d_z_plane) and sphere configs (donerf_sphere), so those kernels test
// none of them per sample; `matches` is the host's check that a config has the layout.  The values the arithmetic uses
// (head offsets, activation factors, scales, bounds) are read from the config by every layout.
struct HeadsAny {
  __device__ static int n_z(const hr_config& c) { return c.n_z; }
  __device__ static bool flow(const hr_config& c) { return c.use_flow; }
  __device__ static bool sigma(const hr_config& c) { return c.off_sigma >= 0; }
  __device__ static bool point_sigma(const hr_config& c) { return c.off_point_sigma >= 0; }
  __device__ static bool offset(const hr_config& c) { return c.use_offset; }
  __device__ static bool color_scale_shift(const hr_config& c) { return c.use_color_scale_shift; }
  __device__ static int isect(const hr_config& c) { return c.isect_type; }
  __device__ static bool isect_use_sigma(const hr_config& c) { return c.isect_use_sigma; }
  __device__ static bool sort(const hr_config& c) { return c.isect_sort; }
  __device__ static int fea2dense(const hr_config& c) { return c.fea2dense; }
  // the density that scales the intersection distance / the point offset: none, sigma or point sigma
  __device__ static float isect_density(const hr_config& c, float sg, float sgp) {
    return (c.isect_density_off < 0) ? 0.0f : ((c.isect_density_off == c.off_sigma) ? sg : sgp);
  }
  __device__ static float offset_density(const hr_config& c, float sg, float sgp) {
    return (c.offset_density_off < 0) ? 0.0f : ((c.offset_density_off == c.off_sigma) ? sg : sgp);
  }
  // activation kinds (hr_act::kind)
  __device__ static int k_z(const hr_config& c) { return c.act_z.kind; }
  __device__ static int k_isect(const hr_config& c) { return c.isect_act.kind; }
  __device__ static int k_flow(const hr_config& c) { return c.act_flow.kind; }
  __device__ static int k_flow_act(const hr_config& c) { return c.flow_act.kind; }
  __device__ static int k_sigma(const hr_config& c) { return c.act_sigma.kind; }
  __device__ static int k_point_sigma(const hr_config& c) { return c.act_point_sigma.kind; }
  __device__ static int k_offset(const hr_config& c) { return c.act_offset.kind; }
  __device__ static int k_offset_act(const hr_config& c) { return c.offset_act.kind; }
  __device__ static int k_cscale(const hr_config& c) { return c.act_cscale.kind; }
  __device__ static int k_cshift(const hr_config& c) { return c.act_cshift.kind; }
};

// What the shipped configs share: sigma and point-sigma heads (sigmoid), a tanh point offset, identity z / flow / colour
// scale-shift heads, the intersection scaled by 1 - sigma and sorted, ReLU feature-to-density.
struct HeadsShipped {
  __device__ static bool sigma(const hr_config&) { return true; }
  __device__ static bool point_sigma(const hr_config&) { return true; }
  __device__ static bool offset(const hr_config&) { return true; }
  __device__ static bool color_scale_shift(const hr_config&) { return true; }
  __device__ static bool isect_use_sigma(const hr_config&) { return true; }
  __device__ static bool sort(const hr_config&) { return true; }
  __device__ static int fea2dense(const hr_config&) { return HR_DENSE_RELU; }
  __device__ static float isect_density(const hr_config&, float sg, float) { return sg; }
  __device__ static int k_z(const hr_config&) { return HR_ACT_IDENTITY; }
  __device__ static int k_isect(const hr_config&) { return HR_ACT_IDENTITY; }
  __device__ static int k_flow(const hr_config&) { return HR_ACT_IDENTITY; }
  __device__ static int k_flow_act(const hr_config&) { return HR_ACT_IDENTITY; }
  __device__ static int k_sigma(const hr_config&) { return HR_ACT_SIGMOID; }
  __device__ static int k_point_sigma(const hr_config&) { return HR_ACT_SIGMOID; }
  __device__ static int k_offset(const hr_config&) { return HR_ACT_TANH; }
  __device__ static int k_offset_act(const hr_config&) { return HR_ACT_IDENTITY; }
  __device__ static int k_cscale(const hr_config&) { return HR_ACT_IDENTITY; }
  __device__ static int k_cshift(const hr_config&) { return HR_ACT_IDENTITY; }
  static bool matches(const hr_config& c) {
    return c.off_sigma >= 0 && c.off_point_sigma >= 0 && c.off_point_sigma != c.off_sigma && c.use_offset &&
           c.use_color_scale_shift && c.isect_use_sigma && c.isect_density_off == c.off_sigma && c.isect_sort &&
           c.fea2dense == HR_DENSE_RELU && !eases_density(c) && c.act_z.kind == HR_ACT_IDENTITY &&
           c.isect_act.kind == HR_ACT_IDENTITY && c.act_flow.kind == HR_ACT_IDENTITY && c.flow_act.kind == HR_ACT_IDENTITY &&
           c.act_sigma.kind == HR_ACT_SIGMOID && c.act_point_sigma.kind == HR_ACT_SIGMOID && c.act_offset.kind == HR_ACT_TANH &&
           c.offset_act.kind == HR_ACT_IDENTITY && c.act_cscale.kind == HR_ACT_IDENTITY && c.act_cshift.kind == HR_ACT_IDENTITY;
  }
};

// dynamic z-plane: one z head, a flow head, the offset scaled by 1 - point sigma
struct HeadsZPlane : HeadsShipped {
  __device__ static int n_z(const hr_config&) { return 1; }
  __device__ static bool flow(const hr_config&) { return true; }
  __device__ static int isect(const hr_config&) { return HR_ISECT_Z_PLANE; }
  __device__ static float offset_density(const hr_config&, float, float sgp) { return sgp; }
  static bool matches(const hr_config& c) {
    return HeadsShipped::matches(c) && c.n_z == 1 && c.use_flow && c.isect_type == HR_ISECT_Z_PLANE &&
           c.offset_density_off == c.off_point_sigma;
  }
};

// sphere: four z heads (centre scale and radius), no flow, the offset scaled by 1 - sigma
struct HeadsSphere : HeadsShipped {
  __device__ static int n_z(const hr_config&) { return 4; }
  __device__ static bool flow(const hr_config&) { return false; }
  __device__ static int isect(const hr_config&) { return HR_ISECT_SPHERE; }
  __device__ static float offset_density(const hr_config&, float sg, float) { return sg; }
  static bool matches(const hr_config& c) {
    return HeadsShipped::matches(c) && c.n_z == 4 && !c.use_flow && c.isect_type == HR_ISECT_SPHERE &&
           c.offset_density_off == c.off_sigma;
  }
};

#ifdef HR_RENDER_PHASE_CLOCKS
// Measurement build only (-DHR_RENDER_PHASE_CLOCKS, scripts/render_split_bench.py): clock64() cycles every warp spends in
// each phase of its rays, summed over the launches since the last read (hr_render_phase_clocks, hr_render.cu), and the
// number of warp-rays.  Phases: 0 heads load, 1 keyframe / view matrix / intersect / sort / points / texel coordinates,
// 2 gather rounds, 3 alpha / transmittance / composite / store.  A load's latency is charged to the phase that first uses it.
static constexpr int kRenderPhases = 4;
static __device__ unsigned long long g_render_phase_clocks[kRenderPhases + 1];
#define HR_PHASE_MARK(p)                              \
  {                                                   \
    const long long t_ = clock64();                   \
    phase_clk[p] += (unsigned long long)(t_ - t_mark); \
    t_mark = t_;                                      \
  }
#else
#define HR_PHASE_MARK(p)
#endif

template <int SPL, bool DYN, int C0, int C1, int C2, int SHADE, bool EXTRA, int RPW, bool RARE, bool EASE, class HL>
__device__ __forceinline__ void render_body(const hr_config& cfg, const Derived& dv, const RenderTabs& tabs,
                                            const float* __restrict__ rays, const float* __restrict__ heads,
                                            const RgbDst& dst, long long n_rays, ExtraOut so,
                                            unsigned char* __restrict__ rgb8_out) {
  static_assert(std::is_same<HL, HeadsAny>::value || (!EXTRA && !RARE && !EASE), "fixed head layouts: plain lean kernels");
  constexpr int NT = C0 + C1 + C2;
  constexpr int ROWS = (SHADE == HR_SHADE_SH) ? 9 : 1;
  constexpr int ROUNDS = 4 * SPL;
  constexpr int LW = 32 / RPW;  // lanes (= sample slots) per ray in the lane = sample mapping
  static_assert(RPW == 1 || (SPL == 1 && !EXTRA), "two rays per warp: S <= 16, plain outputs");
  extern __shared__ float s_basis[];  // [app_dim][NT] copy of basis_mat
  for (int i = threadIdx.x; i < 3 * ROWS * NT; i += blockDim.x) s_basis[i] = tabs.basis[i];
  __syncthreads();

  const int lane = threadIdx.x & 31;
  const int sub = lane / LW, sl = lane % LW;  // ray of this lane within the warp, sample index within the ray
  const int q = lane & 3, xt = q >> 1, alt = q & 1, quad = lane >> 2;
  const int qc = min(q, 2);
  const int S = cfg.n_samples;
  const int out_stride = cfg.mlp_out;
  const long long warp0 = (long long)blockIdx.x * kWarpsPerCta + (threadIdx.x >> 5);
  const long long nwarps = (long long)gridDim.x * kWarpsPerCta;

  // This lane's channel slots: an 8-channel group contributes its 4-channel half (`alt`), a 4-channel group all four.
  // lcol[i] = column of basis_mat of slot i;  G[r][q][i] = entry (colour q, slot i) of the view-folded appearance matrix of
  // ray r of the warp: every lane carries all three colours of its slots (the colour sums are reduced across the quad).
  constexpr int N0 = (C0 == 8) ? 4 : C0, N1 = (C1 == 8) ? 4 : C1, N2 = (C2 == 8) ? 4 : C2;
  constexpr int NTL = N0 + N1 + N2;
  int lcol[NTL];
#pragma unroll
  for (int i = 0; i < N0; ++i) lcol[i] = ((C0 == 8) ? alt * 4 : 0) + i;
#pragma unroll
  for (int i = 0; i < N1; ++i) lcol[N0 + i] = C0 + ((C1 == 8) ? alt * 4 : 0) + i;
#pragma unroll
  for (int i = 0; i < N2; ++i) lcol[N0 + N1 + i] = C0 + C1 + ((C2 == 8) ? alt * 4 : 0) + i;
  // Two ways to finish a sample:
  //   FOLD  (several groups, [8,4,4] / [8,8,8]): every lane accumulates partial sums of all three colours and of the density
  //         over its own taps / channels (G = all three colour rows of its slots), one transposing reduction per sample;
  //   !FOLD (one group, [8,0,0]): complete features f[NT] in every lane, each lane computes its own colour (G = one row).
  constexpr bool FOLD = (C1 + C2) > 0;
  constexpr int NG = (SHADE == HR_SHADE_SH) ? RPW : 1;
  float G[FOLD ? NG : 1][FOLD ? 3 : 1][FOLD ? NTL : 1];
  float Gr[FOLD ? 1 : NG][FOLD ? 1 : NT];
  // !FOLD: column of basis_mat feeding this lane's i-th product feature ([own half | other half] of the 8-channel group)
  int fcol[FOLD ? 1 : NT];
  if constexpr (!FOLD) {
#pragma unroll
    for (int i = 0; i < 4; ++i) { fcol[i] = alt * 4 + i; fcol[4 + i] = (1 - alt) * 4 + i; }
  }
  if constexpr (SHADE == HR_SHADE_RGB) {
    if constexpr (FOLD) {
#pragma unroll
      for (int qq = 0; qq < 3; ++qq)
#pragma unroll
        for (int i = 0; i < NTL; ++i) G[0][qq][i] = s_basis[qq * NT + lcol[i]];
    } else {
#pragma unroll
      for (int i = 0; i < NT; ++i) Gr[0][i] = s_basis[qc * NT + fcol[i]];
    }
  }

  const float inv_x = __fdiv_rn(2.0f, __fsub_rn(cfg.aabb[3], cfg.aabb[0]));  // invaabbSize (tensorf_base.py:292)
  const float inv_y = __fdiv_rn(2.0f, __fsub_rn(cfg.aabb[4], cfg.aabb[1]));
  const float inv_z = __fdiv_rn(2.0f, __fsub_rn(cfg.aabb[5], cfg.aabb[2]));
  const int line_bytes = out_stride * 4;

#ifdef HR_RENDER_PHASE_CLOCKS
  unsigned long long phase_clk[kRenderPhases] = {}, warp_rays = 0;
  long long t_mark = 0;
#endif
  for (long long base = warp0 * RPW; base < n_rays; base += nwarps * RPW) {
#ifdef HR_RENDER_PHASE_CLOCKS
    t_mark = clock64();
    ++warp_rays;
#endif
    // this lane's ray; the second ray of the last warp may not exist: it is computed on a copy of the last ray (every lane
    // takes part in the shuffles) and never stored
    const bool ray_ok = base + sub < n_rays;
    const long long ray = ray_ok ? base + sub : n_rays - 1;
    const float* r = rays + ray * cfg.c_in;
    const float* hrow = heads + ray * (long long)out_stride;
    // ---- warm L1 with the next ray's head row (1.9 KB) while this one is processed ----
    {
      const long long nxt = ray + nwarps * RPW;
      if (nxt < n_rays) {
        const char* p = reinterpret_cast<const char*>(heads + nxt * (long long)out_stride) + sl * 128;
        if (sl * 128 < line_bytes) asm volatile("prefetch.global.L1 [%0];" ::"l"(p));
        if (sl == LW - 1) asm volatile("prefetch.global.L1 [%0];" ::"l"(rays + nxt * cfg.c_in));
      }
    }
    const float ox = __ldg(r + 0), oy = __ldg(r + 1), oz = __ldg(r + 2);
    const float dx = __ldg(r + 3), dy = __ldg(r + 4), dz = __ldg(r + 5);
    const float time = __ldg(r + cfg.c_in - 1);

    // ---- raw head values of this lane's sample(s): all loads issued before any use ----
    float hz[SPL][4], hfl[SPL][3], hsg[SPL], hsp[SPL], hof[SPL][3];
#pragma unroll
    for (int j = 0; j < SPL; ++j) {
      const int s = sl + 32 * j;
      const float* hp = hrow + ((s < S) ? s : 0);
#pragma unroll
      for (int c = 0; c < 4; ++c) hz[j][c] = (c < HL::n_z(cfg)) ? __ldg(hp + (cfg.off_z + c) * S) : 0.0f;
#pragma unroll
      for (int c = 0; c < 3; ++c) hfl[j][c] = HL::flow(cfg) ? __ldg(hp + (cfg.off_flow + c) * S) : 0.0f;
      hsg[j] = HL::sigma(cfg) ? __ldg(hp + cfg.off_sigma * S) : 0.0f;
      hsp[j] = HL::point_sigma(cfg) ? __ldg(hp + cfg.off_point_sigma * S) : 0.0f;
#pragma unroll
      for (int c = 0; c < 3; ++c) hof[j][c] = HL::offset(cfg) ? __ldg(hp + (cfg.off_offset + c) * S) : 0.0f;
    }
    HR_PHASE_MARK(0);

    // ---- per-ray keyframe snap, time offset and keyframe row ----
    float toff = 0.0f, base_t = 0.0f;
    int krow = 0;
    if (DYN || HL::flow(cfg)) {
      const Keyframe kf = keyframe_snap(dv, time);
      base_t = kf.base_t;
      toff = kf.toff;
      if (DYN) krow = kf.row;
    }

    // ---- view-dependent appearance matrix: G[q][i] = sum_k Y_k(dir) * basis[(q*9+k)][i]  (tensorf_utils.py:334-338)
    if constexpr (SHADE == HR_SHADE_SH) {
      float Y[9];
      sh_basis9(dx, dy, dz, Y);  // viewdirs = rays[:,3:6] as given (point.py:866-867)
      // the 3*NT entries of a ray are built once, spread over its LW lanes, then every lane of the warp collects its row of
      // every ray's matrix in its column order (the quad mapping works on samples of all rays of the warp)
      constexpr int GE = 3 * NT, GM = (GE + LW - 1) / LW;
      float g[GM];
#pragma unroll
      for (int m = 0; m < GM; ++m) {
        const int e = min(sl + LW * m, GE - 1);
        const int eq = e / NT, ei = e % NT;
        float a = 0.0f;
#pragma unroll
        for (int k = 0; k < 9; ++k) a = fmaf(Y[k], s_basis[(eq * 9 + k) * NT + ei], a);
        g[m] = a;
      }
      if constexpr (!FOLD) {
#pragma unroll
        for (int i = 0; i < NT; ++i) {
          const int E = qc * NT + fcol[i];
#pragma unroll
          for (int rr = 0; rr < RPW; ++rr) {
            float v = 0.0f;
#pragma unroll
            for (int m = 0; m < GM; ++m) {
              const float t = __shfl_sync(kFull, g[m], rr * LW + (E % LW));
              if ((E / LW) == m) v = t;
            }
            Gr[rr][i] = v;
          }
        }
      } else {
#pragma unroll
      for (int qq = 0; qq < 3; ++qq) {
#pragma unroll
        for (int i = 0; i < NTL; ++i) {
          const int E = qq * NT + lcol[i];
          // the register holding entry E is the same for both channel halves: 8-channel blocks start at multiples of 8,
          // 4-channel blocks at multiples of 4, and LW is a multiple of 8
          const int blk = (i < N0) ? 0 : ((i < N0 + N1) ? C0 : C0 + C1);
          const int m = (qq * NT + blk + ((i < N0) ? i : ((i < N0 + N1) ? i - N0 : i - N0 - N1))) / LW;
#pragma unroll
          for (int rr = 0; rr < RPW; ++rr) G[rr][qq][i] = __shfl_sync(kFull, g[m < GM ? m : 0], rr * LW + (E % LW));
        }
      }
      }
    }

    // ---- lane = sample: intersection (base.py:155-203) ----
    float tkey[SPL], disp[SPL][3];
#pragma unroll
    for (int j = 0; j < SPL; ++j) {
      const int s = sl + 32 * j;
      const bool act = s < S;
      const float sg = HL::sigma(cfg) ? (EASE ? apply_act_head<EASE>(cfg.act_sigma, hsg[j])
                                              : apply_act_kind(HL::k_sigma(cfg), cfg.act_sigma, hsg[j]))
                                      : 0.0f;
      const float sgp = HL::point_sigma(cfg) ? (EASE ? apply_act_head<EASE>(cfg.act_point_sigma, hsp[j])
                                                     : apply_act_kind(HL::k_point_sigma(cfg), cfg.act_point_sigma, hsp[j]))
                                             : 0.0f;
      const float dens_i = HL::isect_density(cfg, sg, sgp);
      const float dens_o = HL::offset_density(cfg, sg, sgp);
      const float one_m = __fsub_rn(1.0f, HL::isect_use_sigma(cfg) ? dens_i : 0.0f);
      const float samp = cfg.samples[act ? s : 0];
      float t;
      if (HL::isect(cfg) == HR_ISECT_Z_PLANE) {
        float zr = __fmul_rn(apply_act_kind(HL::k_isect(cfg), cfg.isect_act, apply_act_kind(HL::k_z(cfg), cfg.act_z, hz[j][0])),
                             one_m);
        float z = __fadd_rn(__fmul_rn(zr, cfg.z_scale), samp);
        if (cfg.contract_samples) z = inv_contract_sample(cfg, dv, z);
        t = intersect_axis_plane(z, oz, dz);
      } else if (RARE && HL::isect(cfg) != HR_ISECT_SPHERE && HL::isect(cfg) != HR_ISECT_CYLINDER) {
        // the less common primitives (sphere_new, euclidean_distance, voxel grids) live in one out-of-line function and are
        // compiled into the RARE variants only: the z-plane / sphere / cylinder kernels keep their instruction stream and
        // register budget (80 registers at three CTAs per SM)
        t = intersect_rare(cfg, dv, hz[j][0], hz[j][1], hz[j][2], hz[j][3], one_m, samp, act ? s : 0, S, hrow, ox, oy, oz, dx, dy, dz);
      } else {
        float zc[4];
#pragma unroll
        for (int c = 0; c < 4; ++c)
          zc[c] = __fmul_rn(apply_act_kind(HL::k_isect(cfg), cfg.isect_act, apply_act_kind(HL::k_z(cfg), cfg.act_z, hz[j][c])),
                            one_m);
        // primitive.py:410-418
        float gx = __fadd_rn(__fmul_rn(zc[0], cfg.sphere_origin_scale), cfg.sphere_origin_initial[0]);
        float gy = __fadd_rn(__fmul_rn(zc[1], cfg.sphere_origin_scale), cfg.sphere_origin_initial[1]);
        float gz = __fadd_rn(__fmul_rn(zc[2], cfg.sphere_origin_scale), cfg.sphere_origin_initial[2]);
        float rad = __fadd_rn(__fmul_rn(zc[3], cfg.z_scale), samp);
        if (cfg.contract_samples) rad = inv_contract_sample(cfg, dv, rad);
        // primitive.py:420-438; IntersectCylinderOld (primitive.py:181-250) for the cylinder
        float sox = __fmul_rn(ox, gx), soy = __fmul_rn(oy, gy), soz = __fmul_rn(oz, gz);
        float sdx = __fmul_rn(dx, gx), sdy = __fmul_rn(dy, gy), sdz = __fmul_rn(dz, gz);
        t = intersect_quadric(sox, soy, soz, sdx, sdy, sdz, rad, HL::isect(cfg) == HR_ISECT_CYLINDER).t;
      }
      if ((t <= cfg.isect_near) || (t >= cfg.isect_far)) t = 0.0f;
      tkey[j] = act ? t : __int_as_float(0x7f800000);
      // per-sample displacement applied after the points are formed: flow * dt (point.py:816-820), then
      // offset * (1 - sigma) (point.py:383-391) -- kept as two addends to preserve the reference's rounding order
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        disp[j][c] = HL::flow(cfg) ? __fmul_rn(apply_act_kind(HL::k_flow_act(cfg), cfg.flow_act,
                                                              apply_act_kind(HL::k_flow(cfg), cfg.act_flow, hfl[j][c])),
                                               toff)
                                   : 0.0f;
        hof[j][c] = HL::offset(cfg) ? __fmul_rn(apply_act_kind(HL::k_offset_act(cfg), cfg.offset_act,
                                                               apply_act_kind(HL::k_offset(cfg), cfg.act_offset, hof[j][c])),
                                                __fsub_rn(1.0f, dens_o))
                                    : 0.0f;
      }
    }

    // ---- sort distances only (base.py:206-210) ----
    if (HL::sort(cfg)) {
      if (keys_unsorted<SPL>(tkey, sl)) {
        if constexpr (RPW == 1) sort_keys<SPL>(tkey, lane);
        else sort_keys_sub<LW>(tkey[0], sl);
      }
    }

    // ---- points, contraction, flow, offset, validity, texel coordinates along the three grid axes ----
    float dist[SPL], fx[SPL], fy[SPL], fz[SPL];
    int ix[SPL], iy[SPL], iz[SPL];  // ix < 0 flags an invalid sample
    bool valid[SPL];
    float pts[EXTRA ? SPL : 1][3];  // final sample points, kept only by the variant that reports them
    float cocx = ox, cocy = oy, cocz = oz;
    if (cfg.contract_type == HR_CONTRACT_MIPNERF) contract_point(cfg, dv, cocx, cocy, cocz);
    else if (cfg.contract_type == HR_CONTRACT_AFFINE) contract_point_affine(cfg, cocx, cocy, cocz);
#pragma unroll
    for (int j = 0; j < SPL; ++j) {
      const int s = sl + 32 * j;
      const bool act = s < S;
      float t = act ? tkey[j] : 0.0f;
      const bool zero = (t == 0.0f);
      float px = __fadd_rn(ox, __fmul_rn(dx, t));  // base.py:226
      float py = __fadd_rn(oy, __fmul_rn(dy, t));
      float pz = __fadd_rn(oz, __fmul_rn(dz, t));
      if (cfg.contract_type != HR_CONTRACT_NONE) {  // base.py:242-246, contract.py:43-50
        if (cfg.contract_type == HR_CONTRACT_MIPNERF) contract_point(cfg, dv, px, py, pz);
        else contract_point_affine(cfg, px, py, pz);
        float ex = __fsub_rn(px, cocx), ey = __fsub_rn(py, cocy), ez = __fsub_rn(pz, cocz);
        t = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(ex, ex), __fmul_rn(ey, ey)), __fmul_rn(ez, ez)));
        if (zero) t = 0.0f;
      }
      px = __fadd_rn(__fadd_rn(px, disp[j][0]), hof[j][0]);
      py = __fadd_rn(__fadd_rn(py, disp[j][1]), hof[j][1]);
      pz = __fadd_rn(__fadd_rn(pz, disp[j][2]), hof[j][2]);
      dist[j] = t;
      // valid_mask (tensorf_base.py:349-353) & distance > 0 (tensorf_dynamic.py:690)
      const bool inside = !((cfg.aabb[0] > px) || (px > cfg.aabb[3]) || (cfg.aabb[1] > py) || (py > cfg.aabb[4]) ||
                            (cfg.aabb[2] > pz) || (pz > cfg.aabb[5]));
      valid[j] = act && inside && (t > 0.0f);
      // normalize_coord (tensorf_base.py:308-309), then grid_sample's align_corners=True unnormalise
      // ((u+1)/2)*(size-1) along each grid axis; index clamped to [0,size-2] with the fraction recomputed, which is
      // exact for in-range points (the out-of-range neighbour of a point on the max face has weight 0).
      const float ux = __fsub_rn(__fmul_rn(__fsub_rn(px, cfg.aabb[0]), inv_x), 1.0f);
      const float uy = __fsub_rn(__fmul_rn(__fsub_rn(py, cfg.aabb[1]), inv_y), 1.0f);
      const float uz = __fsub_rn(__fmul_rn(__fsub_rn(pz, cfg.aabb[2]), inv_z), 1.0f);
      const float tx = __fmul_rn(__fmul_rn(__fadd_rn(ux, 1.0f), 0.5f), (float)(dv.res[0] - 1));
      const float ty = __fmul_rn(__fmul_rn(__fadd_rn(uy, 1.0f), 0.5f), (float)(dv.res[1] - 1));
      const float tz = __fmul_rn(__fmul_rn(__fadd_rn(uz, 1.0f), 0.5f), (float)(dv.res[2] - 1));
      ix[j] = max(0, min((int)floorf(tx), dv.res[0] - 2));
      iy[j] = max(0, min((int)floorf(ty), dv.res[1] - 2));
      iz[j] = max(0, min((int)floorf(tz), dv.res[2] - 2));
      fx[j] = tx - (float)ix[j];
      fy[j] = ty - (float)iy[j];
      fz[j] = tz - (float)iz[j];
      if (!valid[j]) ix[j] = -1;
      if (EXTRA) { pts[j][0] = px; pts[j][1] = py; pts[j][2] = pz; }
      if (EXTRA && act) {
        if (so.distances) so.distances[ray * S + s] = t;
        if (so.points) {
          so.points[(ray * S + s) * 3 + 0] = px;
          so.points[(ray * S + s) * 3 + 1] = py;
          so.points[(ray * S + s) * 3 + 2] = pz;
        }
      }
    }

    HR_PHASE_MARK(1);
    // ---- VM gather: 8 samples per round, 4 lanes per sample (matMode [[0,1],[0,2],[1,2]], vecMode [2,1,0]) ----
    float sig_r[ROUNDS];  // density feature of (round, quad): FOLD: in lane q = 3 of the quad, else replicated
    float rgb_r[ROUNDS];  // shaded colour channel q of (round, quad)
#pragma unroll
    for (int rd = 0; rd < ROUNDS; ++rd) {
      sig_r[rd] = 0.0f;
      rgb_r[rd] = 0.0f;
      // round rd serves sample slots rd*8 .. rd*8+7 of the warp: samples (rd % (LW/8))*8 .. of ray rd / (LW/8)
      if ((RPW == 1 ? rd : (rd % (LW / 8))) * 8 >= S) continue;  // warp-uniform
      const int j = rd >> 2;
      const int src = (rd & 3) * 8 + quad;
      // texel indices travel packed (grids have < 65535 texels per axis; an invalid sample carries ix = 0xffff)
      const unsigned pxy = __shfl_sync(kFull, (unsigned)(ix[j] & 0xffff) | ((unsigned)iy[j] << 16), src);
      const unsigned pzk = __shfl_sync(kFull, (unsigned)iz[j] | ((unsigned)krow << 16), src);
      const int krow_s = (RPW == 1) ? krow : (int)(pzk >> 16);
      int sx = (int)(pxy & 0xffffu);
      if (sx == 0xffff) sx = -1;
      const int sy = (int)(pxy >> 16);
      const int sz = (int)(pzk & 0xffffu);
      const float gx = __shfl_sync(kFull, fx[j], src);
      const float gy = __shfl_sync(kFull, fy[j], src);
      const float gz = __shfl_sync(kFull, fz[j], src);
      const bool ok = sx >= 0;
      sx = max(sx, 0);
      GroupTaps<C0, DYN> s0, a0;
      GroupTaps<(C1 ? C1 : 4), DYN> s1, a1;
      GroupTaps<(C2 ? C2 : 4), DYN> s2, a2;
      group_fetch<C0, DYN>(s0, tabs.sig[0], sx, sy, sz, krow_s, xt, alt, ok);
      group_fetch<C0, DYN>(a0, tabs.app[0], sx, sy, sz, krow_s, xt, alt, ok);
      if constexpr (C1 > 0) {
        group_fetch<C1, DYN>(s1, tabs.sig[1], sx, sz, sy, krow_s, xt, alt, ok);
        group_fetch<C1, DYN>(a1, tabs.app[1], sx, sz, sy, krow_s, xt, alt, ok);
      }
      if constexpr (C2 > 0) {
        group_fetch<C2, DYN>(s2, tabs.sig[2], sy, sz, sx, krow_s, xt, alt, ok);
        group_fetch<C2, DYN>(a2, tabs.app[2], sy, sz, sx, krow_s, xt, alt, ok);
      }
      float col;
      if constexpr (FOLD) {
        // four partial sums per lane (colours 0-2, density feature) over all groups, then one transposing reduction over the
        // quad: lane q < 3 receives colour q, lane q = 3 the density feature
        float v4[4] = {0.0f, 0.0f, 0.0f, 0.0f};
        const int gr = (NG == 1) ? 0 : rd / (LW / 8);
        group_accumulate<C0, DYN>(s0, a0, gx, gy, gz, xt, alt, &G[gr][0][0], &G[gr][1][0], &G[gr][2][0], v4);
        if constexpr (C1 > 0)
          group_accumulate<C1, DYN>(s1, a1, gx, gz, gy, xt, alt, &G[gr][0][N0], &G[gr][1][N0], &G[gr][2][N0], v4);
        if constexpr (C2 > 0)
          group_accumulate<C2, DYN>(s2, a2, gy, gz, gx, xt, alt, &G[gr][0][N0 + N1], &G[gr][1][N0 + N1], &G[gr][2][N0 + N1], v4);
        const float acc = quad_transpose_reduce(v4, xt, alt);
        sig_r[rd] = ok ? acc : 0.0f;  // meaningful in lane q = 3
        // appearance: basis_mat (tensorf_dynamic.py:371) folded with the shading (tensorf_utils.py:334-343); lanes q < 3
        if constexpr (SHADE == HR_SHADE_SH) col = fmaxf(acc + 0.5f, 0.0f);
        else col = 1.0f / (1.0f + expf(-acc));
      } else {
        // density feature: sum_c space_c * second_c over all groups (tensorf_dynamic.py:330, tensorf_no_sample.py:76-78);
        // appearance features f[NT] in this lane's column order (fcol)
        float f[NT];
        float sf = group_sigma<C0, DYN>(s0, gx, gy, gz, xt, alt);
        {
          float p[4];
          group_app<C0, DYN>(a0, gx, gy, gz, xt, alt, p);
#pragma unroll
          for (int c = 0; c < 4; ++c) f[c] = p[c];
          if constexpr (C0 == 8) {
#pragma unroll
            for (int c = 0; c < 4; ++c) f[4 + c] = __shfl_xor_sync(kFull, p[c], 1);
          }
        }
        if constexpr (C1 > 0) {
          float p[4];
          sf += group_sigma<C1, DYN>(s1, gx, gz, gy, xt, alt);
          group_app<C1, DYN>(a1, gx, gz, gy, xt, alt, p);
#pragma unroll
          for (int c = 0; c < 4; ++c) f[C0 + c] = p[c];
          if constexpr (C1 == 8) {
#pragma unroll
            for (int c = 0; c < 4; ++c) f[C0 + 4 + c] = __shfl_xor_sync(kFull, p[c], 1);
          }
        }
        if constexpr (C2 > 0) {
          float p[4];
          sf += group_sigma<C2, DYN>(s2, gy, gz, gx, xt, alt);
          group_app<C2, DYN>(a2, gy, gz, gx, xt, alt, p);
#pragma unroll
          for (int c = 0; c < 4; ++c) f[C0 + C1 + c] = p[c];
          if constexpr (C2 == 8) {
#pragma unroll
            for (int c = 0; c < 4; ++c) f[C0 + C1 + 4 + c] = __shfl_xor_sync(kFull, p[c], 1);
          }
        }
        sig_r[rd] = ok ? sf : 0.0f;
        // appearance: basis_mat (tensorf_dynamic.py:371) folded with the shading (tensorf_utils.py:334-343)
        float acc = 0.0f;
#pragma unroll
        for (int i = 0; i < NT; ++i) acc = fmaf(Gr[(NG == 1) ? 0 : rd / (LW / 8)][i], f[i], acc);
        if constexpr (SHADE == HR_SHADE_SH) col = fmaxf(acc + 0.5f, 0.0f);
        else col = 1.0f / (1.0f + expf(-acc));
      }
      rgb_r[rd] = ok ? col : 0.0f;
    }

    HR_PHASE_MARK(2);
    // ---- back to lane = sample: sigma, alpha, transmittance, weights (tensorf_utils.py:242-253) ----
    float wgt[SPL];
    float carryT = 1.0f;
    float accw = 0.0f, accB[3] = {0.f, 0.f, 0.f};
    float csA[SPL][3];
    // lane 0's running sums of the extra fields over the rounds before the last (EXTRA with several samples per lane)
    [[maybe_unused]] float fpart[(EXTRA && SPL > 1) ? HR_N_FIELDS * 3 : 1];
#pragma unroll
    for (int j = 0; j < SPL; ++j) {
      const int s = sl + 32 * j;
      const float* hp = hrow + ((s < S) ? s : 0);
      float cs_raw[3] = {0.f, 0.f, 0.f}, csh_raw[3] = {0.f, 0.f, 0.f};
      if (HL::color_scale_shift(cfg)) {
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          cs_raw[c] = __ldg(hp + (cfg.off_cscale + c) * S);
          csh_raw[c] = __ldg(hp + (cfg.off_cshift + c) * S);
        }
      }
      float feat = 0.0f;
#pragma unroll
      for (int rr = 0; rr < 4; ++rr) {
        float v = __shfl_sync(kFull, sig_r[4 * j + rr], 4 * (lane & 7) + (FOLD ? 3 : 0));
        if ((lane >> 3) == rr) feat = v;
      }
      float sigma = feature2density_kind(HL::fea2dense(cfg), cfg, feat);
      if (!valid[j]) sigma = 0.0f;
      const SampleAlpha sa = sample_alpha<SPL>(dist, j, sigma, cfg.distance_scale, sl, S);
      const float w = sa.alpha * transmittance<LW>(sa.a1, sl, carryT);
      wgt[j] = w;
      if (EXTRA && s < S) {
        if (so.sigma) so.sigma[ray * S + s] = sigma;
        if (so.weights) so.weights[ray * S + s] = w;
      }
      accw += w;
      const float m = (w > cfg.weight_thre) ? w : 0.0f;  // app_mask (tensorf_dynamic.py:750)
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float csv = HL::color_scale_shift(cfg) ? apply_act_kind(HL::k_cscale(cfg), cfg.act_cscale, cs_raw[c]) : 0.0f;
        const float cshv = HL::color_scale_shift(cfg) ? apply_act_kind(HL::k_cshift(cfg), cfg.act_cshift, csh_raw[c]) : 0.0f;
        csA[j][c] = (s < S) ? m * (csv + 1.0f) : 0.0f;
        accB[c] += (s < S) ? w * cshv : 0.0f;
      }
      if constexpr (EXTRA) {
        // ---- extra fields (tensorf_dynamic.py:808-837): sum_s w_s x_s, sum_s pred_w_s x_s, or x itself ----
        // pred_weights = alpha2weights(x['weights'][..., 0]) with x['weights'] == 1 (base.py:183-191):
        // T_s = prod_{k<s} (1 - 1 + 1e-10), pred_w_s = 1 * T_s
        float pw = 1.0f;
        for (int k = 0; k < min(s, 8); ++k) pw = __fmul_rn(pw, __fadd_rn(__fsub_rn(1.0f, 1.0f), 1e-10f));
#pragma unroll 1
        for (int f = 0; f < HR_N_FIELDS; ++f) {
          float* fo = so.field_out[f];
          unsigned char* fo8 = so.field_u8[f].out;
          if (fo == nullptr && fo8 == nullptr) continue;  // warp-uniform
          const int mode = so.field_mode[f];
          // per-sample heads are x[name] = activation(raw) (ray.py:333-337); the other keys are built-ins of the pipeline
          int dim = 1, hoff = -1;
          const hr_act* hact = &cfg.act_z;
          switch (f) {
            case HR_FIELD_POINTS: case HR_FIELD_VIEWDIRS: dim = 3; break;
            case HR_FIELD_SPATIAL_FLOW: dim = 3; hoff = cfg.off_flow; hact = &cfg.act_flow; break;
            case HR_FIELD_SIGMA: hoff = cfg.off_sigma; hact = &cfg.act_sigma; break;
            case HR_FIELD_POINT_SIGMA: hoff = cfg.off_point_sigma; hact = &cfg.act_point_sigma; break;
            case HR_FIELD_POINT_OFFSET: dim = 3; hoff = cfg.off_offset; hact = &cfg.act_offset; break;
            case HR_FIELD_COLOR_SCALE: dim = 3; hoff = cfg.off_cscale; hact = &cfg.act_cscale; break;
            case HR_FIELD_COLOR_SHIFT: dim = 3; hoff = cfg.off_cshift; hact = &cfg.act_cshift; break;
            case HR_FIELD_COLOR_SCALE_GLOBAL: dim = 3; hoff = cfg.off_cscale_global; hact = &cfg.act_cscale_global; break;
            case HR_FIELD_COLOR_SHIFT_GLOBAL: dim = 3; hoff = cfg.off_cshift_global; hact = &cfg.act_cshift_global; break;
            default: break;
          }
          for (int c = 0; c < dim; ++c) {
            float v;
            if (hoff >= 0) {
              v = apply_act_head<EASE>(*hact, __ldg(hp + (long long)(hoff + c) * S));  // eased: sigma / point_sigma only
              // two embeddings write their result back under the head's name:
              //   AdvectPoints: x['spatial_flow'] = spatial_flow_activation(x['spatial_flow'])        (point.py:815-817)
              //   PointOffset : x['point_offset'] = activation(x['point_offset']) * (1 - sigma)        (point.py:383-389)
              if (f == HR_FIELD_SPATIAL_FLOW && cfg.use_flow) v = apply_act(cfg.flow_act, v);
              if (f == HR_FIELD_POINT_OFFSET && cfg.use_offset) v = hof[j][c];
            } else {
              switch (f) {
                case HR_FIELD_POINTS: v = pts[j][c]; break;
                case HR_FIELD_DISTANCES: v = dist[j]; break;
                case HR_FIELD_BASE_TIMES: v = base_t; break;
                case HR_FIELD_TIME_OFFSET: v = toff; break;
                case HR_FIELD_TIMES: v = time; break;
                case HR_FIELD_VIEWDIRS: v = (c == 0) ? dx : ((c == 1) ? dy : dz); break;
                default: v = 1.0f; break;  // HR_FIELD_WEIGHTS
              }
            }
            if (mode == HR_FIELD_NO_OVER) {
              if (s < S) fo[(ray * S + s) * dim + c] = v;
            } else {
              float acc = (s < S) ? __fmul_rn((mode == HR_FIELD_PRED_WEIGHTS) ? pw : w, v) : 0.0f;
#pragma unroll
              for (int d = 1; d < 32; d <<= 1) acc += __shfl_xor_sync(kFull, acc, d);
              // SPL registers per lane: partial sums of the rounds are added in round order by lane 0, and the last round
              // stores the field, or its uint8 map
              if (lane == 0) {
                const float tot = (j == 0) ? acc : (fpart[f * 3 + c] + acc);
                if (j < SPL - 1) fpart[f * 3 + c] = tot;
                else if (fo8 != nullptr) fo8[ray * dim + c] = vis_to8b(vis_pre(so.field_u8[f], tot));
                else fo[ray * dim + c] = tot;
              }
            }
          }
        }
      }
    }

    // ---- composite: sum_s w_s * (rgb_s*(1+cs_s) + csh_s) (tensorf_dynamic.py:780-792) ----
    float accq_r[RPW];  // per ray of the warp: colour channel q summed over the samples this lane's quads served
#pragma unroll
    for (int rr = 0; rr < RPW; ++rr) accq_r[rr] = 0.0f;
#pragma unroll
    for (int rd = 0; rd < ROUNDS; ++rd) {
      if ((RPW == 1 ? rd : (rd % (LW / 8))) * 8 >= S) continue;
      const int j = rd >> 2;
      const int src = (rd & 3) * 8 + quad;
      const float g0 = __shfl_sync(kFull, csA[j][0], src);
      const float g1 = __shfl_sync(kFull, csA[j][1], src);
      const float g2 = __shfl_sync(kFull, csA[j][2], src);
      const float Aq = (q == 0) ? g0 : ((q == 1) ? g1 : g2);
      accq_r[(RPW == 1) ? 0 : rd / (LW / 8)] = fmaf(Aq, rgb_r[rd], accq_r[(RPW == 1) ? 0 : rd / (LW / 8)]);
      if constexpr (EXTRA) {
        if (so.rgb_samples != nullptr) {
          const float ws = __shfl_sync(kFull, wgt[j], src);
          const int sidx = j * 32 + src;
          if (q < 3 && sidx < S) so.rgb_samples[(ray * S + sidx) * 3 + q] = (ws > cfg.weight_thre) ? rgb_r[rd] : 0.0f;
        }
      }
    }
    // the quads of the whole warp served every ray's samples: reduce over all quads, then each lane keeps its own ray's sum
    float accq = 0.0f;
#pragma unroll
    for (int rr = 0; rr < RPW; ++rr) {
      float a = accq_r[rr];
#pragma unroll
      for (int d = 4; d < 32; d <<= 1) a += __shfl_xor_sync(kFull, a, d);
      if (rr == sub) accq = a;
    }
    // lane = sample partial sums: reduce within the ray's LW lanes
#pragma unroll
    for (int d = 1; d < LW; d <<= 1) {
      accw += __shfl_xor_sync(kFull, accw, d);
      accB[0] += __shfl_xor_sync(kFull, accB[0], d);
      accB[1] += __shfl_xor_sync(kFull, accB[1], d);
      accB[2] += __shfl_xor_sync(kFull, accB[2], d);
    }
    float v = 0.0f;
    if (sl < 3) {  // lanes 0-2 of the ray's lane group hold quad position q = 0, 1, 2 = colour channel (LW is a multiple of 4)
      v = accq + ((sl == 0) ? accB[0] : ((sl == 1) ? accB[1] : accB[2]));
      if (cfg.white_bg && !cfg.black_bg) v = v + (1.0f - accw);
      if (cfg.off_cscale_global >= 0) {
        // scale_shift_color_one (utils/tensorf_utils.py:275-281): the heads of sample 0 (MLP order) act on the pixel
        const float gs = apply_act(cfg.act_cscale_global, __ldg(hrow + (long long)(cfg.off_cscale_global + sl) * S));
        const float gb = apply_act(cfg.act_cshift_global, __ldg(hrow + (long long)(cfg.off_cshift_global + sl) * S));
        v = __fadd_rn(__fmul_rn(v, __fadd_rn(gs, 1.0f)), gb);
      }
    }
    if (RARE && cfg.n_color_views > 0) {  // warp-uniform; RARE variants only
      // transform_color_one (utils/tensorf_utils.py:308-331): rgb + M rgb + shift with the (M, shift) row of this ray's
      // camera, id = round(rays[:, -2]) (ColorTransformEmbedding.forward, point.py:594-605)
      const float v0 = __shfl_sync(kFull, v, sub * LW + 0);
      const float v1 = __shfl_sync(kFull, v, sub * LW + 1);
      const float v2 = __shfl_sync(kFull, v, sub * LW + 2);
      if (sl < 3) {
        const int cam = max(0, min((int)rintf(__ldg(r + cfg.c_in - 2)), cfg.n_color_views - 1));
        const float* row = tabs.color_embedding + (long long)cam * 12;
        const float m0 = apply_act(cfg.act_ctransform, __ldg(row + sl * 3 + 0));
        const float m1 = apply_act(cfg.act_ctransform, __ldg(row + sl * 3 + 1));
        const float m2 = apply_act(cfg.act_ctransform, __ldg(row + sl * 3 + 2));
        const float sh = apply_act(cfg.act_ctshift, __ldg(row + 9 + sl));
        const float dotv = __fadd_rn(__fadd_rn(__fmul_rn(v0, m0), __fmul_rn(v1, m1)), __fmul_rn(v2, m2));
        v = __fadd_rn(__fadd_rn(v, dotv), sh);
      }
    }
    if (sl < 3) {
      if (cfg.clamp_output) v = fminf(fmaxf(v, 0.0f), 1.0f);
      if (rgb8_out != nullptr) {
        // to8b (utils/__init__.py:47): (255 * clip(x, 0, 1)).astype(uint8) -- truncation
        if (ray_ok) rgb8_out[ray * 3 + sl] = (unsigned char)(int)__fmul_rn(255.0f, fminf(fmaxf(v, 0.0f), 1.0f));
      }
    }
    if (rgb8_out == nullptr) {
      // lane l of a ray's group stores channel l % 3 into destination l / 3: one store instruction covers every
      // destination buffer (the local output, or all ranks' gather buffers when the frame is ray-sharded)
      const float vv = __shfl_sync(kFull, v, sub * LW + (sl % 3));
      const int d = sl / 3;
      if (d < dst.n && ray_ok) dst.p[d][(dst.row0 + ray) * 3 + (sl % 3)] = vv;
    }
    HR_PHASE_MARK(3);
  }
#ifdef HR_RENDER_PHASE_CLOCKS
  if (lane == 0) {
#pragma unroll
    for (int p = 0; p < kRenderPhases; ++p) atomicAdd(&g_render_phase_clocks[p], phase_clk[p]);
    atomicAdd(&g_render_phase_clocks[kRenderPhases], warp_rays);
  }
#endif
}

// Occupancy target of a render kernel: 3 CTAs per SM for one sample per lane or one VM group, 2 for several groups at two
// samples per lane, 1 above.
template <int SPL, int C1, int C2>
constexpr int render_min_ctas() {
  return SPL > 2 ? 1 : ((C1 + C2 == 0 || SPL == 1) ? 3 : 2);
}

// Every configuration: the head layout is read from the config.
template <int SPL, bool DYN, int C0, int C1, int C2, int SHADE, bool EXTRA, int RPW, bool RARE, bool EASE>
__global__ void __launch_bounds__(kWarpsPerCta * 32, render_min_ctas<SPL, C1, C2>())
render_kernel(const __grid_constant__ hr_config cfg, const __grid_constant__ Derived dv,
              const __grid_constant__ RenderTabs tabs, const float* __restrict__ rays,
              const float* __restrict__ heads, const __grid_constant__ RgbDst dst, long long n_rays, ExtraOut so,
              unsigned char* __restrict__ rgb8_out) {
  render_body<SPL, DYN, C0, C1, C2, SHADE, EXTRA, RPW, RARE, EASE, HeadsAny>(cfg, dv, tabs, rays, heads, dst, n_rays, so,
                                                                             rgb8_out);
}

// A fixed head layout (the last parameter's type): the same cell of the template family, the layout's fields compiled in.
// The layout is not a template argument, so the kernel's template arguments still name the cell.
#define HR_RENDER_KERNEL_FIXED(Layout)                                                                                      \
  template <int SPL, bool DYN, int C0, int C1, int C2, int SHADE, bool EXTRA, int RPW, bool RARE, bool EASE>                \
  __global__ void __launch_bounds__(kWarpsPerCta * 32, render_min_ctas<SPL, C1, C2>())                                    \
  render_kernel(const __grid_constant__ hr_config cfg, const __grid_constant__ Derived dv,                                 \
                const __grid_constant__ RenderTabs tabs, const float* __restrict__ rays, const float* __restrict__ heads, \
                const __grid_constant__ RgbDst dst, long long n_rays, ExtraOut so, unsigned char* __restrict__ rgb8_out,   \
                Layout) {                                                                                                 \
    render_body<SPL, DYN, C0, C1, C2, SHADE, EXTRA, RPW, RARE, EASE, Layout>(cfg, dv, tabs, rays, heads, dst, n_rays, so,  \
                                                                             rgb8_out);                                  \
  }
HR_RENDER_KERNEL_FIXED(HeadsZPlane)
HR_RENDER_KERNEL_FIXED(HeadsSphere)
#undef HR_RENDER_KERNEL_FIXED

template <int SPL, bool DYN, int C0, int C1, int C2, int SHADE, bool RARE, bool EASE>
static cudaError_t launch_one(const hr_config& cfg, const Derived& dv, const RenderTabs& tabs, const float* rays,
                              const float* heads, const RgbDst& rgb, long long n, const ExtraOut* so, int num_sms,
                              cudaStream_t stream, unsigned char* rgb8) {
  constexpr int ROWS = (SHADE == HR_SHADE_SH) ? 9 : 1;
  constexpr int NT = C0 + C1 + C2;
  size_t smem = 3 * (size_t)ROWS * NT * sizeof(float);
  // two rays per warp when a ray has at most 16 samples (plain outputs, at most 5 destination buffers: 16 lanes / 3)
  const bool two_rays = (SPL == 1) && cfg.n_samples <= 16 && so == nullptr && rgb.n <= 5;
  const int rpw = two_rays ? 2 : 1;
  long long ctas_needed = (n + kWarpsPerCta * rpw - 1) / (kWarpsPerCta * rpw);
  long long grid = ctas_needed < (long long)num_sms * kMinCtasPerSm * 2 ? ctas_needed : (long long)num_sms * kMinCtasPerSm * 2;
  if (grid < 1) grid = 1;
  const dim3 g((unsigned)grid), b(kWarpsPerCta * 32);
  if (so) {
    render_kernel<SPL, DYN, C0, C1, C2, SHADE, true, 1, RARE, EASE><<<g, b, smem, stream>>>(cfg, dv, tabs, rays, heads, rgb, n, *so, rgb8);
    return cudaGetLastError();
  }
  ExtraOut none{};
  auto plain = [&](auto layout) -> cudaError_t {
    using HL = decltype(layout);
    if constexpr (std::is_same<HL, HeadsAny>::value) {
      if constexpr (SPL == 1) {
        if (two_rays) {
          render_kernel<SPL, DYN, C0, C1, C2, SHADE, false, 2, RARE, EASE><<<g, b, smem, stream>>>(cfg, dv, tabs, rays, heads, rgb, n, none, rgb8);
          return cudaGetLastError();
        }
      }
      render_kernel<SPL, DYN, C0, C1, C2, SHADE, false, 1, RARE, EASE><<<g, b, smem, stream>>>(cfg, dv, tabs, rays, heads, rgb, n, none, rgb8);
    } else {
      if constexpr (SPL == 1) {
        if (two_rays) {
          render_kernel<SPL, DYN, C0, C1, C2, SHADE, false, 2, RARE, EASE><<<g, b, smem, stream>>>(cfg, dv, tabs, rays, heads, rgb, n, none, rgb8, layout);
          return cudaGetLastError();
        }
      }
      render_kernel<SPL, DYN, C0, C1, C2, SHADE, false, 1, RARE, EASE><<<g, b, smem, stream>>>(cfg, dv, tabs, rays, heads, rgb, n, none, rgb8, layout);
    }
    return cudaGetLastError();
  };
  // the fixed head layouts of the shipped configs, at the (dynamic, shading) pairs those configs use
  if constexpr (!RARE && !EASE && DYN && SHADE == HR_SHADE_SH) {
    if (HeadsZPlane::matches(cfg)) return plain(HeadsZPlane{});
  }
  if constexpr (!RARE && !EASE && !DYN && SHADE == HR_SHADE_RGB) {
    if (HeadsSphere::matches(cfg)) return plain(HeadsSphere{});
  }
  return plain(HeadsAny{});
}

template <int SPL, bool DYN, int C0, int C1, int C2, bool RARE, bool EASE>
static cudaError_t launch_shade(const hr_config& cfg, const Derived& dv, const RenderTabs& tabs, const float* rays,
                                const float* heads, const RgbDst& rgb, long long n, const ExtraOut* so, int num_sms,
                                cudaStream_t stream, unsigned char* rgb8) {
  if (cfg.shading == HR_SHADE_SH)
    return launch_one<SPL, DYN, C0, C1, C2, HR_SHADE_SH, RARE, EASE>(cfg, dv, tabs, rays, heads, rgb, n, so, num_sms, stream, rgb8);
  return launch_one<SPL, DYN, C0, C1, C2, HR_SHADE_RGB, RARE, EASE>(cfg, dv, tabs, rays, heads, rgb, n, so, num_sms, stream, rgb8);
}

// pipelines served by the RARE variants only (see render_kernel)
static inline bool needs_rare(const hr_config& cfg) {
  return (cfg.isect_type != HR_ISECT_Z_PLANE && cfg.isect_type != HR_ISECT_SPHERE && cfg.isect_type != HR_ISECT_CYLINDER) ||
         cfg.n_color_views > 0;
}

template <int SPL, bool DYN, bool RARE, bool EASE = false>
static cudaError_t launch_comps(const hr_config& cfg, const Derived& dv, const RenderTabs& tabs, const float* rays,
                                const float* heads, const RgbDst& rgb, long long n, const ExtraOut* so, int num_sms,
                                cudaStream_t stream, unsigned char* rgb8) {
  const int c0 = cfg.n_sigma[0], c1 = cfg.n_sigma[1], c2 = cfg.n_sigma[2];
  if (c0 == 8 && c1 == 0 && c2 == 0)
    return launch_shade<SPL, DYN, 8, 0, 0, RARE, EASE>(cfg, dv, tabs, rays, heads, rgb, n, so, num_sms, stream, rgb8);
  if (c0 == 8 && c1 == 4 && c2 == 4)
    return launch_shade<SPL, DYN, 8, 4, 4, RARE, EASE>(cfg, dv, tabs, rays, heads, rgb, n, so, num_sms, stream, rgb8);
  if (c0 == 8 && c1 == 8 && c2 == 8)
    return launch_shade<SPL, DYN, 8, 8, 8, RARE, EASE>(cfg, dv, tabs, rays, heads, rgb, n, so, num_sms, stream, rgb8);
  return cudaErrorInvalidValue;
}

}  // namespace hr
