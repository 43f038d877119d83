// Backward of the fused render kernel (SURVEY.md section 8 row f1): d loss / d rgb  ->  d heads, d VM tables, d basis_mat.
//
// Reference: the autograd graph PyTorch builds for nlf/intersect/base.py:142-259, nlf/embedding/point.py:371-396,780-831,
// nlf/nets/tensorf_dynamic.py:645-806 / tensorf_no_sample.py:128-247, utils/tensorf_utils.py:242-253,334-343 -- i.e. what
// `loss.backward()` does in INRSystem.training_step (nlf/__init__.py:634-709).  Restated analytically:
//   composite      C = sum_i w_i (rgb_i (1 + cs_i) + csh_i)  [+ 1 - sum w]      -> d w_i, d rgb_i, d cs_i, d csh_i
//   transmittance  w_i = a_i T_i, T_i = prod_{j<i} (1 - a_j + 1e-10)            -> d a_i = gw_i T_i - (sum_{k>i} gw_k w_k) / (1 - a_i + 1e-10)
//   alpha          a_i = 1 - exp(-s_i dl_i ds)                                   -> d s_i, d dl_i  (dl_i = t_{i+1} - t_i, last = 1e10)
//   shading        rgb = relu(G f_app + 1/2)  (SH folded per ray) | sigmoid(B f_app)
//   VM features    f_n = bilinear(plane_n)(u_a, u_b) * linear(second_n)(u_c)     -> table gradients (red.global.add.v4.f32 into
//                  channel-last gradient tables with the forward tables' layout) and d u -> d p
//   geometry       p = c(o + t d) + flow * dt + offset * (1 - sigma_p),  t = sorted intersection distances
//                  -> d t (through the sort permutation), d heads
// One warp per ray, lane = sample for everything (the forward's quad mapping is not used here: this kernel is bound by the
// L2 atomics, not by the gathers).  The forward is recomputed from rays + heads through the per-sample and per-ray functions
// of hr_geom.cuh that the forward kernel calls (same rounding, hence the same masks and the same sort order); nothing
// per-sample was saved.
// Supported for training: z_plane / sphere / cylinder (origin_scale_factor == 0) / euclidean-distance / voxel-grid /
// deformable-plane primitives, no / mipnerf / bbox / z_depth contraction, per-sample and per-ray colour heads, the per-camera
// colour transform, S <= 64; hr_render_backward rejects the rest.
// Like the forward, the kernel has a RARE variant (hr_render_bwd_rare.cu) that adds the voxel-grid / deformable-plane
// primitives, the affine contraction, the per-ray colour heads and the colour transform; the z-plane / sphere / cylinder /
// distance pipelines keep the lean variants of hr_render_bwd.cu.
//   per-ray colour heads  v' = v (gs + 1) + gb         (heads of sample 0)   -> d v = G (gs + 1), d gs = G v, d gb = G
//   colour transform      v'' = v' + M v' + sh         (row `cam`)           -> d v' = (I + M)^T G, d M = G v'^T, d sh = G
//   the clamp mask of eval() applies to the final value, the white background sits inside both transforms (as in the forward)
#pragma once
#include "hr_common.cuh"
#include "hr_geom.cuh"

namespace hr {

static constexpr int kBwdWarps = 4;

// d y / d x of y = f(x*inner + shift) * outer (apply_act)
__device__ __forceinline__ float act_grad(const hr_act& a, float x) {
  const float v = __fadd_rn(__fmul_rn(x, a.inner_fac), a.shift);
  float g = 1.0f;
  if (a.kind == HR_ACT_SIGMOID) {
    const float s = 1.0f / (1.0f + expf(-v));
    g = s * (1.0f - s);
  } else if (a.kind == HR_ACT_TANH) {
    const float t = tanhf(v);
    g = 1.0f - t * t;
  }
  return g * a.inner_fac * a.outer_fac;
}

// d / d x of apply_act_eased: act_grad times ease_mul while an EaseValue window is open (0 while the head is held at its
// start value)
__device__ __forceinline__ float act_grad_eased(const hr_act& a, float x) {
  const float g = act_grad(a, x);
  return a.eased ? g * a.ease_mul : g;
}

template <bool EASE>
__device__ __forceinline__ float act_grad_head(const hr_act& a, float x) {
  if constexpr (EASE) return act_grad_eased(a, x);
  else return act_grad(a, x);
}

// sort (key, id) pairs ascending by key (ties by id, so the ids stay a permutation); element e = reg*32 + lane
template <int SPL>
__device__ __forceinline__ void sort_pairs(float (&k)[SPL], int (&id)[SPL], int lane) {
  constexpr int NE = 32 * SPL;
#pragma unroll
  for (int size = 2; size <= NE; size <<= 1) {
#pragma unroll
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      if (stride >= 32) {
        const bool sw = (k[SPL - 1] < k[0]) || (k[SPL - 1] == k[0] && id[SPL - 1] < id[0]);
        if (sw) {
          const float tk = k[0]; k[0] = k[SPL - 1]; k[SPL - 1] = tk;
          const int ti = id[0]; id[0] = id[SPL - 1]; id[SPL - 1] = ti;
        }
      } else {
#pragma unroll
        for (int r = 0; r < SPL; ++r) {
          const int e = r * 32 + lane;
          const float ok = __shfl_xor_sync(kFull, k[r], stride);
          const int oi = __shfl_xor_sync(kFull, id[r], stride);
          const bool up = ((e & size) == 0);
          const bool lower = ((lane & stride) == 0);
          const bool other_less = (ok < k[r]) || (ok == k[r] && oi < id[r]);
          const bool take = (lower == up) ? other_less : !other_less;
          if (take) { k[r] = ok; id[r] = oi; }
        }
      }
    }
  }
}

// d out / d in of inv_contract_distance (hr_geom.cuh; nlf/contract.py:143-158) at input d
__device__ __forceinline__ float inv_contract_distance_grad(const hr_config& cfg, const Derived& dv, float d) {
  d = __fmul_rn(__fmul_rn(d, 0.5f), 2.0f);
  if (d < -2.0f || d > 2.0f) return 0.0f;  // torch.clamp passes the gradient on [min, max]
  if (fabsf(d) < 1.0f) return cfg.contract_start_distance;
  const float t = __fsub_rn(2.0f, fabsf(d));
  const float inv = __fadd_rn(__fdiv_rn(t, dv.dist_scale_fac), dv.inv_end_dist);
  // far = sgn / inv, inv = (2 - |d|)/dsf + ied  ->  d far / d d = 1 / (inv^2 dsf)
  return cfg.contract_start_distance / (inv * inv * dv.dist_scale_fac);
}

// d out / d in of inv_contract_sample: distance * fac for bbox / z_depth (RARE variants only), else the mipnerf inverse
template <bool RARE>
__device__ __forceinline__ float inv_contract_sample_grad(const hr_config& cfg, const Derived& dv, float d) {
  if (RARE && cfg.contract_type == HR_CONTRACT_AFFINE) return cfg.contract_dist_fac;
  return inv_contract_distance_grad(cfg, dv, d);
}

// d t / d (activated z channels zc[0..3]) of the voxel-grid / deformable-plane intersection of intersect_rare (hr_geom.cuh),
// at the same inputs; t itself always comes from intersect_rare so that the rounding matches the forward.
//   voxel grid      t = (z sgn(d_a) - o_a) / d_a, z = ic(zc0 z_scale3[a] + samp)          -> only zc0
//   deformable      t = (pd - o.n^) / (d.n^), n = zc[0:3] pns + n0[a], pd = ic(zc3 z_scale + samp)
//                   d t / d n^ = -(o + t d) / (d.n^), d n^ / d n = (I - n^ n^T) / |n|
// The guards of the forward (|d_a| or |d.n^| < 1e-5, the max-axis rejection) give 0; their inputs are rounded as in
// intersect_rare, so the guard decisions are the forward's.
__device__ __forceinline__ void intersect_rare_grad(const hr_config& cfg, const Derived& dv, const float (&zc)[4], float samp, int s,
                                                    float ox, float oy, float oz, float dx, float dy, float dz, float (&g)[4]) {
  g[0] = g[1] = g[2] = g[3] = 0.0f;
  if (cfg.isect_type == HR_ISECT_VOXEL) {
    const int ax = s % 3;
    const float zpre = __fadd_rn(__fmul_rn(zc[0], cfg.z_scale3[ax]), samp);
    const float dz_dpre = cfg.contract_samples ? inv_contract_sample_grad<true>(cfg, dv, zpre) : 1.0f;
    const float da = (ax == 0) ? dx : ((ax == 1) ? dy : dz);
    if (fabsf(da) < 1e-5f) return;
    if (cfg.isect_max_axis && fabsf(da) < __fsub_rn(fmaxf(fabsf(dx), fmaxf(fabsf(dy), fabsf(dz))), 1e-8f)) return;
    const float sgn = cfg.isect_outward ? ((da > 0.0f) ? 1.0f : -1.0f) : 1.0f;
    g[0] = cfg.z_scale3[ax] * dz_dpre * sgn / da;
  } else if (cfg.isect_type == HR_ISECT_PLANE) {
    const int ax = s % cfg.isect_axes;
    const float ppre = __fadd_rn(__fmul_rn(zc[3], cfg.z_scale), samp);
    const float pd = cfg.contract_samples ? inv_contract_sample(cfg, dv, ppre) : ppre;
    const float dpd_dpre = cfg.contract_samples ? inv_contract_sample_grad<true>(cfg, dv, ppre) : 1.0f;
    // n, n^ and d.n^ with intersect_rare's rounding, so that the |d.n^| guard decides exactly as in the forward
    const float nx = __fadd_rn(__fmul_rn(zc[0], cfg.plane_normal_scale), cfg.plane_normal[ax * 3 + 0]);
    const float ny = __fadd_rn(__fmul_rn(zc[1], cfg.plane_normal_scale), cfg.plane_normal[ax * 3 + 1]);
    const float nz = __fadd_rn(__fmul_rn(zc[2], cfg.plane_normal_scale), cfg.plane_normal[ax * 3 + 2]);
    const float nn = fmaxf(sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(nx, nx), __fmul_rn(ny, ny)), __fmul_rn(nz, nz))), 1e-12f);
    const float ux = __fdiv_rn(nx, nn), uy = __fdiv_rn(ny, nn), uz = __fdiv_rn(nz, nn);
    const float ddn = __fadd_rn(__fadd_rn(__fmul_rn(dx, ux), __fmul_rn(dy, uy)), __fmul_rn(dz, uz));
    if (fabsf(ddn) < 1e-5f) return;
    const float t = (pd - (ox * ux + oy * uy + oz * uz)) / ddn;
    // d t / d n^, projected onto the tangent plane of the normalisation
    const float hx = -(ox + t * dx) / ddn, hy = -(oy + t * dy) / ddn, hz = -(oz + t * dz) / ddn;
    const float hu = hx * ux + hy * uy + hz * uz;
    g[0] = (hx - hu * ux) / nn * cfg.plane_normal_scale;
    g[1] = (hy - hu * uy) / nn * cfg.plane_normal_scale;
    g[2] = (hz - hu * uz) / nn * cfg.plane_normal_scale;
    g[3] = cfg.z_scale * dpd_dpre / ddn;
  }
}

// v <- J_c(p)^T v for the mipnerf point contraction c (hr_geom.cuh contract_point; nlf/contract.py:178-192) at raw point p
__device__ __forceinline__ void contract_point_vjp(const hr_config& cfg, const Derived& dv, float px, float py, float pz,
                                                   float& vx, float& vy, float& vz) {
  const float sr = cfg.contract_start_radius;
  const float x = px / sr, y = py / sr, z = pz / sr;
  const float r = sqrtf(x * x + y * y + z * z);
  if (r < 1.0f) {
    vx /= sr; vy /= sr; vz /= sr;
    return;
  }
  // c = x g(r), g(r) = (2 - (1/r - ier) rsf) / r = (2 + ier rsf)/r - rsf/r^2
  const float k0 = 2.0f + dv.inv_end_rad * dv.rad_scale_fac;
  const float g = k0 / r - dv.rad_scale_fac / (r * r);
  const float gp = -k0 / (r * r) + 2.0f * dv.rad_scale_fac / (r * r * r);
  const float xv = x * vx + y * vy + z * vz;
  const float s = gp / r * xv;
  vx = (g * vx + s * x) / sr;
  vy = (g * vy + s * y) / sr;
  vz = (g * vz + s * z) / sr;
}

__device__ __forceinline__ void red_add4(float* p, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

// One channel quad (4 channels starting at ch0) of one VM group for one sample: forward values and coordinate slopes.
struct Quad {
  float A[4], dAa[4], dAb[4];  // space plane value, d/d fa, d/d fb (per texel unit)
  float B[4], dBc[4];          // second factor value, d/d fc
};

template <int C>
__device__ __forceinline__ void quad_fetch(Quad& q, const PlaneTab& T, int ia, int ib, int ic, int krow, int ch0, float fa, float fb,
                                           float fc) {
  const float* s0 = T.space + ((long long)(ib * T.W + ia) * C + ch0);
  const float4 v00 = ldg4(s0), v10 = ldg4(s0 + C), v01 = ldg4(s0 + (long long)T.W * C), v11 = ldg4(s0 + (long long)T.W * C + C);
  const float* e0 = T.second + ((long long)(krow * T.L + ic) * C + ch0);
  const float4 l0 = ldg4(e0), l1 = ldg4(e0 + C);
  const float a00[4] = {v00.x, v00.y, v00.z, v00.w}, a10[4] = {v10.x, v10.y, v10.z, v10.w};
  const float a01[4] = {v01.x, v01.y, v01.z, v01.w}, a11[4] = {v11.x, v11.y, v11.z, v11.w};
  const float b0[4] = {l0.x, l0.y, l0.z, l0.w}, b1[4] = {l1.x, l1.y, l1.z, l1.w};
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const float top = a00[c] + fa * (a10[c] - a00[c]);
    const float bot = a01[c] + fa * (a11[c] - a01[c]);
    q.A[c] = top + fb * (bot - top);
    q.dAa[c] = (1.0f - fb) * (a10[c] - a00[c]) + fb * (a11[c] - a01[c]);
    q.dAb[c] = bot - top;
    q.B[c] = b0[c] + fc * (b1[c] - b0[c]);
    q.dBc[c] = b1[c] - b0[c];
  }
}

// scatter g[4] (d loss / d feature of the 4 channels) into the gradient tables of this group; returns d loss / d (fa, fb, fc)
template <int C>
__device__ __forceinline__ void quad_scatter(const Quad& q, const float (&g)[4], float* gspace, float* gsecond, const PlaneTab& T,
                                             int ia, int ib, int ic, int krow, int ch0, float fa, float fb, float fc, float& dfa,
                                             float& dfb, float& dfc) {
  float gA[4], gB[4];
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    gA[c] = g[c] * q.B[c];
    gB[c] = g[c] * q.A[c];
    dfa += gA[c] * q.dAa[c];
    dfb += gA[c] * q.dAb[c];
    dfc += gB[c] * q.dBc[c];
  }
  float* s0 = gspace + ((long long)(ib * T.W + ia) * C + ch0);
  const float w00 = (1.0f - fa) * (1.0f - fb), w10 = fa * (1.0f - fb), w01 = (1.0f - fa) * fb, w11 = fa * fb;
  red_add4(s0, w00 * gA[0], w00 * gA[1], w00 * gA[2], w00 * gA[3]);
  red_add4(s0 + C, w10 * gA[0], w10 * gA[1], w10 * gA[2], w10 * gA[3]);
  red_add4(s0 + (long long)T.W * C, w01 * gA[0], w01 * gA[1], w01 * gA[2], w01 * gA[3]);
  red_add4(s0 + (long long)T.W * C + C, w11 * gA[0], w11 * gA[1], w11 * gA[2], w11 * gA[3]);
  float* e0 = gsecond + ((long long)(krow * T.L + ic) * C + ch0);
  const float u0 = 1.0f - fc, u1 = fc;
  red_add4(e0, u0 * gB[0], u0 * gB[1], u0 * gB[2], u0 * gB[3]);
  red_add4(e0 + C, u1 * gB[0], u1 * gB[1], u1 * gB[2], u1 * gB[3]);
}

struct BwdOpts {
  int clamp_output;  // eval(): clamp(0,1) in the forward (tensorf_dynamic.py:805-806)
  int white_bg;      // rgb_map += 1 - acc_map (:795-796)
};

template <int SPL, bool DYN, int C0, int C1, int C2, int SHADE, bool RARE, bool EASE>
__global__ void __launch_bounds__(kBwdWarps * 32)
render_bwd_kernel(const __grid_constant__ hr_config cfg, const __grid_constant__ Derived dv,
                  const __grid_constant__ RenderTabs tabs, const __grid_constant__ GradTabs gt, const float* __restrict__ rays,
                  const float* __restrict__ heads, const float* __restrict__ d_rgb, float* __restrict__ d_heads,
                  long long n_rays, BwdOpts opt) {
  constexpr int NT = C0 + C1 + C2;
  constexpr int ROWS = (SHADE == HR_SHADE_SH) ? 9 : 1;
  constexpr int NB = 3 * ROWS * NT;
  extern __shared__ float smem[];
  float* s_basis = smem;            // [3*ROWS][NT] copy of basis_mat
  float* s_gbasis = smem + NB;      // [3*ROWS][NT] gradient accumulator of this CTA
  float* s_warp = smem + 2 * NB;    // per warp: G'[3][NT] | Y[9] (+pad) | perm buffer [64]
  constexpr int WARP_FLOATS = 3 * NT + 12 + 64;
  float* s_gemb = s_warp + kBwdWarps * WARP_FLOATS;  // RARE: [n_color_views][12] colour-transform gradient of this CTA
  const int n_emb = RARE ? 12 * cfg.n_color_views : 0;
  for (int i = threadIdx.x; i < NB; i += blockDim.x) { s_basis[i] = tabs.basis[i]; s_gbasis[i] = 0.0f; }
  if constexpr (RARE) {
    for (int i = threadIdx.x; i < n_emb; i += blockDim.x) s_gemb[i] = 0.0f;
  }
  __syncthreads();

  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  float* Gs = s_warp + wib * WARP_FLOATS;
  float* Ys = Gs + 3 * NT;
  float* perm = Ys + 12;
  const int S = cfg.n_samples;
  const int out_stride = cfg.mlp_out;
  const long long warp0 = (long long)blockIdx.x * kBwdWarps + wib;
  const long long nwarps = (long long)gridDim.x * kBwdWarps;
  const float inv_x = __fdiv_rn(2.0f, __fsub_rn(cfg.aabb[3], cfg.aabb[0]));
  const float inv_y = __fdiv_rn(2.0f, __fsub_rn(cfg.aabb[4], cfg.aabb[1]));
  const float inv_z = __fdiv_rn(2.0f, __fsub_rn(cfg.aabb[5], cfg.aabb[2]));
  // d (texel coordinate) / d (world coordinate) per axis
  const float tsx = inv_x * 0.5f * (float)(dv.res[0] - 1), tsy = inv_y * 0.5f * (float)(dv.res[1] - 1),
              tsz = inv_z * 0.5f * (float)(dv.res[2] - 1);

  for (long long ray = warp0; ray < n_rays; ray += nwarps) {
    const float* r = rays + ray * cfg.c_in;
    const float* hrow = heads + ray * (long long)out_stride;
    float* grow = d_heads + ray * (long long)out_stride;
    const float ox = __ldg(r + 0), oy = __ldg(r + 1), oz = __ldg(r + 2);
    const float dx = __ldg(r + 3), dy = __ldg(r + 4), dz = __ldg(r + 5);
    const float time = __ldg(r + cfg.c_in - 1);
    const float Gc[3] = {__ldg(d_rgb + ray * 3 + 0), __ldg(d_rgb + ray * 3 + 1), __ldg(d_rgb + ray * 3 + 2)};

    // ---- per-ray: keyframe snap, shading matrix ----
    float toff = 0.0f;
    int krow = 0;
    if (DYN || cfg.use_flow) {
      const Keyframe kf = keyframe_snap(dv, time);
      toff = kf.toff;
      if (DYN) krow = kf.row;
    }
    __syncwarp();
    if constexpr (SHADE == HR_SHADE_SH) {
      float Y[9];
      sh_basis9(dx, dy, dz, Y);
      if (lane < 9) Ys[lane] = Y[lane];
      for (int e = lane; e < 3 * NT; e += 32) {
        const int q = e / NT, i = e % NT;
        float a = 0.0f;
#pragma unroll
        for (int k = 0; k < 9; ++k) a = fmaf(Y[k], s_basis[(q * 9 + k) * NT + i], a);
        Gs[e] = a;
      }
    } else {
      for (int e = lane; e < 3 * NT; e += 32) Gs[e] = s_basis[e];
    }
    __syncwarp();

    // ---- forward, lane = sample (MLP order s = lane + 32 j): heads, intersection ----
    float tkey[SPL];
    int tid[SPL];
    float dt_dzr[SPL];   // d t_s / d zr_s (zr = activated z channel that moves the primitive, before (1 - sigma)), mask included
    float a_z[SPL], one_m[SPL], sg[SPL], sgp[SPL];
    float flowv[SPL][3], offv[SPL][3];  // activated flow (without dt) and offset (without (1 - sigma))
    float dens_o[SPL];
    float dt_dn[RARE ? SPL : 1][3];  // deformable plane: d t_s / d (activated normal channels 0-2), mask included
    // the z channel that carries the gradient (the deformable plane's normal channels 0-2 go through dt_dn)
    const int zc_idx = (cfg.isect_type == HR_ISECT_Z_PLANE || cfg.isect_type == HR_ISECT_DISTANCE ||
                        (RARE && cfg.isect_type == HR_ISECT_VOXEL)) ? 0 : 3;
    float base_distance = 0.0f;  // euclidean_distance_unified: a per-ray term with no parameter behind it
    if (cfg.isect_type == HR_ISECT_DISTANCE) base_distance = ray_base_distance(ox, oy, oz, dx, dy, dz);
#pragma unroll
    for (int j = 0; j < SPL; ++j) {
      const int s = lane + 32 * j;
      const bool act = s < S;
      const float* hp = hrow + (act ? s : 0);
      const float hsg = (cfg.off_sigma >= 0) ? __ldg(hp + cfg.off_sigma * S) : 0.0f;
      const float hsp = (cfg.off_point_sigma >= 0) ? __ldg(hp + cfg.off_point_sigma * S) : 0.0f;
      sg[j] = (cfg.off_sigma >= 0) ? apply_act_head<EASE>(cfg.act_sigma, hsg) : 0.0f;
      sgp[j] = (cfg.off_point_sigma >= 0) ? apply_act_head<EASE>(cfg.act_point_sigma, hsp) : 0.0f;
      const float dens_i = (cfg.isect_density_off < 0) ? 0.0f : ((cfg.isect_density_off == cfg.off_sigma) ? sg[j] : sgp[j]);
      dens_o[j] = (cfg.offset_density_off < 0) ? 0.0f : ((cfg.offset_density_off == cfg.off_sigma) ? sg[j] : sgp[j]);
      one_m[j] = __fsub_rn(1.0f, cfg.isect_use_sigma ? dens_i : 0.0f);
      const float samp = cfg.samples[act ? s : 0];
      const float hz = __ldg(hp + (cfg.off_z + zc_idx) * S);
      a_z[j] = apply_act(cfg.isect_act, apply_act(cfg.act_z, hz));
      const float zr = __fmul_rn(a_z[j], one_m[j]);
      float t, dtdzr;
      if constexpr (RARE) dt_dn[j][0] = dt_dn[j][1] = dt_dn[j][2] = 0.0f;
      if (RARE && (cfg.isect_type == HR_ISECT_VOXEL || cfg.isect_type == HR_ISECT_PLANE)) {
        // t from the forward's own routine (same rounding), the partials from intersect_rare_grad
        float hzc[4], zc[4], g4[4];
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          hzc[c] = (c < cfg.n_z) ? __ldg(hp + (cfg.off_z + c) * S) : 0.0f;
          zc[c] = __fmul_rn(apply_act(cfg.isect_act, apply_act(cfg.act_z, hzc[c])), one_m[j]);
        }
        t = intersect_rare(cfg, dv, hzc[0], hzc[1], hzc[2], hzc[3], one_m[j], samp, act ? s : 0, S, hrow, ox, oy, oz, dx, dy, dz);
        intersect_rare_grad(cfg, dv, zc, samp, act ? s : 0, ox, oy, oz, dx, dy, dz, g4);
        dtdzr = g4[zc_idx];
        if (cfg.isect_type == HR_ISECT_PLANE) {
          if constexpr (RARE) { dt_dn[j][0] = g4[0]; dt_dn[j][1] = g4[1]; dt_dn[j][2] = g4[2]; }
        }
      } else if (cfg.isect_type == HR_ISECT_Z_PLANE) {
        const float zpre = __fadd_rn(__fmul_rn(zr, cfg.z_scale), samp);
        float z = zpre, dz_dpre = 1.0f;
        if (cfg.contract_samples) { z = inv_contract_sample(cfg, dv, zpre); dz_dpre = inv_contract_sample_grad<RARE>(cfg, dv, zpre); }
        t = intersect_axis_plane(z, oz, dz);
        dtdzr = cfg.z_scale * dz_dpre / axis_plane_dir(dz);
      } else if (cfg.isect_type == HR_ISECT_DISTANCE) {
        const float zpre = __fadd_rn(__fmul_rn(zr, cfg.z_scale), samp);
        float z = zpre, dz_dpre = 1.0f;
        if (cfg.contract_samples) { z = inv_contract_sample(cfg, dv, zpre); dz_dpre = inv_contract_sample_grad<RARE>(cfg, dv, zpre); }
        t = __fadd_rn(z, base_distance);
        dtdzr = cfg.z_scale * dz_dpre;
      } else {
        // sphere / cylinder with constant origins (origin_scale_factor == 0): only the radius channel moves the primitive
        const float gx = cfg.sphere_origin_initial[0], gy = cfg.sphere_origin_initial[1], gz = cfg.sphere_origin_initial[2];
        const float rpre = __fadd_rn(__fmul_rn(zr, cfg.z_scale), samp);
        float rad = rpre, drad_dpre = 1.0f;
        if (cfg.contract_samples) { rad = inv_contract_sample(cfg, dv, rpre); drad_dpre = inv_contract_sample_grad<RARE>(cfg, dv, rpre); }
        const float sox = __fmul_rn(ox, gx), soy = __fmul_rn(oy, gy), soz = __fmul_rn(oz, gz);
        const float sdx = __fmul_rn(dx, gx), sdy = __fmul_rn(dy, gy), sdz = __fmul_rn(dz, gz);
        const QuadricHit h = intersect_quadric(sox, soy, soz, sdx, sdy, sdz, rad, cfg.isect_type == HR_ISECT_CYLINDER);
        t = h.t;
        // disc = b^2 - 4a(oo - rad^2): d disc / d rad = 8 a rad; d t1,2 / d disc = +-1 / (2 a * 2 sq)
        float dt_drad = (h.disc <= 0.0f) ? 0.0f : (h.first ? 1.0f : -1.0f) * (2.0f * rad) / h.sq;
        dtdzr = dt_drad * drad_dpre * cfg.z_scale;
      }
      if ((t <= cfg.isect_near) || (t >= cfg.isect_far)) {
        t = 0.0f;
        dtdzr = 0.0f;
        if constexpr (RARE) dt_dn[j][0] = dt_dn[j][1] = dt_dn[j][2] = 0.0f;
      }
      tkey[j] = act ? t : __int_as_float(0x7f800000);
      tid[j] = s;
      dt_dzr[j] = act ? dtdzr : 0.0f;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float hf = cfg.use_flow ? __ldg(hp + (cfg.off_flow + c) * S) : 0.0f;
        flowv[j][c] = cfg.use_flow ? apply_act(cfg.flow_act, apply_act(cfg.act_flow, hf)) : 0.0f;
        const float ho = cfg.use_offset ? __ldg(hp + (cfg.off_offset + c) * S) : 0.0f;
        offv[j][c] = cfg.use_offset ? apply_act(cfg.offset_act, apply_act(cfg.act_offset, ho)) : 0.0f;
      }
    }
    if (cfg.isect_sort) {
      if (keys_unsorted<SPL>(tkey, lane)) sort_pairs<SPL>(tkey, tid, lane);
    }

    // ---- points, validity, texel coordinates (position e = lane + 32 j in sorted order) ----
    float dist[SPL], fx[SPL], fy[SPL], fz[SPL], praw[SPL][3];
    int ix[SPL], iy[SPL], iz[SPL];
    bool valid[SPL], zero[SPL];
    float cocx = ox, cocy = oy, cocz = oz;
    if (cfg.contract_type == HR_CONTRACT_MIPNERF) contract_point(cfg, dv, cocx, cocy, cocz);
    else if (RARE && cfg.contract_type == HR_CONTRACT_AFFINE) contract_point_affine(cfg, cocx, cocy, cocz);
    const bool contracted = cfg.contract_type == HR_CONTRACT_MIPNERF || (RARE && cfg.contract_type == HR_CONTRACT_AFFINE);
    float pcd[SPL][3];  // c(p_raw) - c(o): direction of d dist / d c(p)
#pragma unroll
    for (int j = 0; j < SPL; ++j) {
      const int s = lane + 32 * j;
      const bool act = s < S;
      float t = act ? tkey[j] : 0.0f;
      zero[j] = (t == 0.0f);
      float px = __fadd_rn(ox, __fmul_rn(dx, t));
      float py = __fadd_rn(oy, __fmul_rn(dy, t));
      float pz = __fadd_rn(oz, __fmul_rn(dz, t));
      praw[j][0] = px; praw[j][1] = py; praw[j][2] = pz;
      pcd[j][0] = pcd[j][1] = pcd[j][2] = 0.0f;
      if (contracted) {
        if (!RARE || cfg.contract_type == HR_CONTRACT_MIPNERF) contract_point(cfg, dv, px, py, pz);
        else contract_point_affine(cfg, px, py, pz);
        const float ex = __fsub_rn(px, cocx), ey = __fsub_rn(py, cocy), ez = __fsub_rn(pz, cocz);
        t = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(ex, ex), __fmul_rn(ey, ey)), __fmul_rn(ez, ez)));
        if (zero[j]) t = 0.0f;
        const float it = (t > 0.0f) ? 1.0f / t : 0.0f;
        pcd[j][0] = ex * it; pcd[j][1] = ey * it; pcd[j][2] = ez * it;
      }
      px = __fadd_rn(__fadd_rn(px, __fmul_rn(flowv[j][0], toff)), __fmul_rn(offv[j][0], __fsub_rn(1.0f, dens_o[j])));
      py = __fadd_rn(__fadd_rn(py, __fmul_rn(flowv[j][1], toff)), __fmul_rn(offv[j][1], __fsub_rn(1.0f, dens_o[j])));
      pz = __fadd_rn(__fadd_rn(pz, __fmul_rn(flowv[j][2], toff)), __fmul_rn(offv[j][2], __fsub_rn(1.0f, dens_o[j])));
      dist[j] = t;
      const bool inside = !((cfg.aabb[0] > px) || (px > cfg.aabb[3]) || (cfg.aabb[1] > py) || (py > cfg.aabb[4]) ||
                            (cfg.aabb[2] > pz) || (pz > cfg.aabb[5]));
      valid[j] = act && inside && (t > 0.0f);
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
      if (!valid[j]) { ix[j] = 0; iy[j] = 0; iz[j] = 0; }
    }

    // ---- pass 1: features -> sigma feature and shading pre-activations ----
    float feat[SPL], pre[SPL][3];
#pragma unroll
    for (int j = 0; j < SPL; ++j) {
      float sf = 0.0f, pr[3] = {0.0f, 0.0f, 0.0f};
      if (valid[j]) {
        int n0 = 0;
#pragma unroll
        for (int grp = 0; grp < 3; ++grp) {
          const int C = (grp == 0) ? C0 : ((grp == 1) ? C1 : C2);
          if (C == 0) continue;
          const int ia = (grp == 2) ? iy[j] : ix[j], ib = (grp == 0) ? iy[j] : iz[j], ic = (grp == 0) ? iz[j] : ((grp == 1) ? iy[j] : ix[j]);
          const float fa = (grp == 2) ? fy[j] : fx[j], fb = (grp == 0) ? fy[j] : fz[j], fc = (grp == 0) ? fz[j] : ((grp == 1) ? fy[j] : fx[j]);
          for (int ch0 = 0; ch0 < C; ch0 += 4) {
            Quad q;
            if (C == 8) quad_fetch<8>(q, tabs.sig[grp], ia, ib, ic, krow, ch0, fa, fb, fc);
            else quad_fetch<4>(q, tabs.sig[grp], ia, ib, ic, krow, ch0, fa, fb, fc);
#pragma unroll
            for (int c = 0; c < 4; ++c) sf = fmaf(q.A[c], q.B[c], sf);
            if (C == 8) quad_fetch<8>(q, tabs.app[grp], ia, ib, ic, krow, ch0, fa, fb, fc);
            else quad_fetch<4>(q, tabs.app[grp], ia, ib, ic, krow, ch0, fa, fb, fc);
#pragma unroll
            for (int c = 0; c < 4; ++c) {
              const float f = q.A[c] * q.B[c];
              const int n = n0 + ch0 + c;
              pr[0] = fmaf(Gs[n], f, pr[0]);
              pr[1] = fmaf(Gs[NT + n], f, pr[1]);
              pr[2] = fmaf(Gs[2 * NT + n], f, pr[2]);
            }
          }
          n0 += C;
        }
      }
      feat[j] = sf;
      pre[j][0] = pr[0]; pre[j][1] = pr[1]; pre[j][2] = pr[2];
    }

    // ---- sigma, alpha, transmittance, weights (tensorf_utils.py:242-253); composite for the clamp mask ----
    float sigma[SPL], delta[SPL], ex[SPL], Tt[SPL], wgt[SPL], a1s[SPL];
    float cs[SPL][3], csh[SPL][3], rgbv[SPL][3];
    float carryT = 1.0f, accw = 0.0f, accC[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int j = 0; j < SPL; ++j) {
      const int s = lane + 32 * j;
      const float* hp = hrow + ((s < S) ? s : 0);
      float sgm = feature2density(cfg, feat[j]);
      if (!valid[j]) sgm = 0.0f;
      sigma[j] = sgm;
      const SampleAlpha sa = sample_alpha<SPL>(dist, j, sigma[j], cfg.distance_scale, lane, S);
      delta[j] = sa.delta;
      ex[j] = sa.ex;
      a1s[j] = sa.a1;
      Tt[j] = transmittance<32>(sa.a1, lane, carryT);
      wgt[j] = sa.alpha * Tt[j];
      accw += wgt[j];
      const bool app = (s < S) && (wgt[j] > cfg.weight_thre);
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        cs[j][c] = cfg.use_color_scale_shift ? apply_act(cfg.act_cscale, __ldg(hp + (cfg.off_cscale + c) * S)) : 0.0f;
        csh[j][c] = cfg.use_color_scale_shift ? apply_act(cfg.act_cshift, __ldg(hp + (cfg.off_cshift + c) * S)) : 0.0f;
        float col;
        if constexpr (SHADE == HR_SHADE_SH) col = fmaxf(pre[j][c] + 0.5f, 0.0f);
        else col = 1.0f / (1.0f + expf(-pre[j][c]));
        rgbv[j][c] = (app && valid[j]) ? col : 0.0f;
        accC[c] += (s < S) ? wgt[j] * (rgbv[j][c] * (1.0f + cs[j][c]) + csh[j][c]) : 0.0f;
      }
    }
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      accw += __shfl_xor_sync(kFull, accw, d);
#pragma unroll
      for (int c = 0; c < 3; ++c) accC[c] += __shfl_xor_sync(kFull, accC[c], d);
    }
    float G[3];
    float g_gs[RARE ? 3 : 1], g_gb[RARE ? 3 : 1];  // d loss / d activated per-ray colour heads (scale, shift)
    if constexpr (!RARE) {
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        float v = accC[c];
        if (opt.white_bg) v += 1.0f - accw;
        // clamp(0,1) passes the gradient on the closed interval
        G[c] = (opt.clamp_output && (v < 0.0f || v > 1.0f)) ? 0.0f : Gc[c];
      }
    } else {
      // forward of the pixel transforms with the forward kernel's rounding: v -> v1 (per-ray colour heads) -> v2 (transform)
      float v[3], v1[3], v2[3], gsv[3] = {0.0f, 0.0f, 0.0f}, M[3][3];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        v[c] = accC[c];
        if (opt.white_bg) v[c] = v[c] + (1.0f - accw);
        v1[c] = v[c];
      }
      if (cfg.off_cscale_global >= 0) {
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          gsv[c] = apply_act(cfg.act_cscale_global, __ldg(hrow + (long long)(cfg.off_cscale_global + c) * S));
          const float gb = apply_act(cfg.act_cshift_global, __ldg(hrow + (long long)(cfg.off_cshift_global + c) * S));
          v1[c] = __fadd_rn(__fmul_rn(v[c], __fadd_rn(gsv[c], 1.0f)), gb);
        }
      }
      int cam = 0;
#pragma unroll
      for (int c = 0; c < 3; ++c) v2[c] = v1[c];
      if (cfg.n_color_views > 0) {
        cam = max(0, min((int)rintf(__ldg(r + cfg.c_in - 2)), cfg.n_color_views - 1));
        const float* row = tabs.color_embedding + (long long)cam * 12;
#pragma unroll
        for (int i = 0; i < 3; ++i) {
#pragma unroll
          for (int k = 0; k < 3; ++k) M[i][k] = apply_act(cfg.act_ctransform, __ldg(row + i * 3 + k));
          const float sh = apply_act(cfg.act_ctshift, __ldg(row + 9 + i));
          const float dotv = __fadd_rn(__fadd_rn(__fmul_rn(v1[0], M[i][0]), __fmul_rn(v1[1], M[i][1])), __fmul_rn(v1[2], M[i][2]));
          v2[i] = __fadd_rn(__fadd_rn(v1[i], dotv), sh);
        }
      }
      // clamp(0,1) of the final value passes the gradient on the closed interval; then back through the transforms
      float G2[3], G1[3];
#pragma unroll
      for (int c = 0; c < 3; ++c) G2[c] = (opt.clamp_output && (v2[c] < 0.0f || v2[c] > 1.0f)) ? 0.0f : Gc[c];
#pragma unroll
      for (int c = 0; c < 3; ++c) G1[c] = G2[c];
      if (cfg.n_color_views > 0) {
#pragma unroll
        for (int k = 0; k < 3; ++k) G1[k] = G2[k] + (M[0][k] * G2[0] + M[1][k] * G2[1] + M[2][k] * G2[2]);
        // d row[3i+k] = G2_i v1_k act', d row[9+i] = G2_i act': one entry per lane, summed per CTA in shared memory
        if (lane < 12) {
          const int i = (lane < 9) ? lane / 3 : lane - 9;
          const float raw = __ldg(tabs.color_embedding + (long long)cam * 12 + lane);
          const float gi = (i == 0) ? G2[0] : ((i == 1) ? G2[1] : G2[2]);
          const int k = lane % 3;
          const float vk = (k == 0) ? v1[0] : ((k == 1) ? v1[1] : v1[2]);
          const float g = (lane < 9) ? gi * vk * act_grad(cfg.act_ctransform, raw) : gi * act_grad(cfg.act_ctshift, raw);
          atomicAdd(&s_gemb[cam * 12 + lane], g);
        }
      }
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        G[c] = (cfg.off_cscale_global >= 0) ? G1[c] * (gsv[c] + 1.0f) : G1[c];
        g_gs[c] = G1[c] * v[c];
        g_gb[c] = G1[c];
      }
    }
    const float Gsum = G[0] + G[1] + G[2];

    // ---- backward of composite / transmittance / alpha ----
    float gw[SPL], g_sigma[SPL], g_delta[SPL], g_pre[SPL][3];
    float carryR = 0.0f;  // sum over later positions of gw_k w_k
    float g_dist[SPL];
#pragma unroll
    for (int j = SPL - 1; j >= 0; --j) {
      const int s = lane + 32 * j;
      float g = 0.0f;
#pragma unroll
      for (int c = 0; c < 3; ++c) g += G[c] * (rgbv[j][c] * (1.0f + cs[j][c]) + csh[j][c]);
      if (opt.white_bg) g -= Gsum;
      gw[j] = (s < S) ? g : 0.0f;
      // exclusive suffix sum of gw*w within this register row, plus the rows after it
      const float v = gw[j] * wgt[j];
      float inc = v;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const float o = __shfl_down_sync(kFull, inc, d);
        if (lane + d < 32) inc += o;
      }
      const float R = (inc - v) + carryR;
      carryR += __shfl_sync(kFull, inc, 0);
      const float alpha = __fsub_rn(1.0f, ex[j]);
      float g_alpha = gw[j] * Tt[j] - R / a1s[j];
      if (s >= S) g_alpha = 0.0f;
      (void)alpha;
      // alpha = 1 - exp(-sigma delta ds)
      g_sigma[j] = g_alpha * ex[j] * delta[j] * cfg.distance_scale;
      g_delta[j] = (s == S - 1 || s >= S) ? 0.0f : g_alpha * ex[j] * sigma[j] * cfg.distance_scale;
      const bool app = (s < S) && (wgt[j] > cfg.weight_thre) && valid[j];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float g_rgb = app ? G[c] * wgt[j] * (1.0f + cs[j][c]) : 0.0f;
        float dact;
        if constexpr (SHADE == HR_SHADE_SH) dact = (pre[j][c] + 0.5f > 0.0f) ? 1.0f : 0.0f;
        else { const float sg_ = 1.0f / (1.0f + expf(-pre[j][c])); dact = sg_ * (1.0f - sg_); }
        g_pre[j][c] = g_rgb * dact;
      }
    }
    // d dist_i = g_delta_{i-1} - g_delta_i
#pragma unroll
    for (int j = 0; j < SPL; ++j) {
      float prev = __shfl_up_sync(kFull, g_delta[j], 1);
      if (lane == 0) prev = (j > 0) ? __shfl_sync(kFull, g_delta[(j > 0) ? j - 1 : 0], 31) : 0.0f;
      else if (j > 0) (void)__shfl_sync(kFull, g_delta[j - 1], 31);
      g_dist[j] = prev - g_delta[j];
    }

    // ---- pass 2: table gradients, basis gradient, d point ----
    float g_head_cs[SPL][3], g_head_csh[SPL][3];
    float g_p[SPL][3];
#pragma unroll
    for (int j = 0; j < SPL; ++j) {
      const int s = lane + 32 * j;
      float gt3[3] = {0.0f, 0.0f, 0.0f};  // d loss / d (tx, ty, tz)
      // d sigma / d feat
      float g_feat = 0.0f;
      if (valid[j]) {
        if (cfg.fea2dense == HR_DENSE_RELU) g_feat = (feat[j] > 0.0f) ? g_sigma[j] : 0.0f;
        else if (cfg.fea2dense == HR_DENSE_RELU_ABS) g_feat = (feat[j] > 0.0f) ? g_sigma[j] : ((feat[j] < 0.0f) ? -g_sigma[j] : 0.0f);
        else { const float xs = feat[j] + cfg.density_shift; g_feat = g_sigma[j] / (1.0f + expf(-xs)); }
      }
      const bool any_app = (g_pre[j][0] != 0.0f) || (g_pre[j][1] != 0.0f) || (g_pre[j][2] != 0.0f);
      int n0 = 0;
#pragma unroll
      for (int grp = 0; grp < 3; ++grp) {
        const int C = (grp == 0) ? C0 : ((grp == 1) ? C1 : C2);
        if (C == 0) continue;
        const int ia = (grp == 2) ? iy[j] : ix[j], ib = (grp == 0) ? iy[j] : iz[j], ic = (grp == 0) ? iz[j] : ((grp == 1) ? iy[j] : ix[j]);
        const float fa = (grp == 2) ? fy[j] : fx[j], fb = (grp == 0) ? fy[j] : fz[j], fc = (grp == 0) ? fz[j] : ((grp == 1) ? fy[j] : fx[j]);
        float dfa = 0.0f, dfb = 0.0f, dfc = 0.0f;
        for (int ch0 = 0; ch0 < C; ch0 += 4) {
          Quad q;
          if (valid[j] && g_feat != 0.0f) {
            const float g4[4] = {g_feat, g_feat, g_feat, g_feat};
            if (C == 8) { quad_fetch<8>(q, tabs.sig[grp], ia, ib, ic, krow, ch0, fa, fb, fc); quad_scatter<8>(q, g4, gt.sig_space[grp], gt.sig_second[grp], tabs.sig[grp], ia, ib, ic, krow, ch0, fa, fb, fc, dfa, dfb, dfc); }
            else { quad_fetch<4>(q, tabs.sig[grp], ia, ib, ic, krow, ch0, fa, fb, fc); quad_scatter<4>(q, g4, gt.sig_space[grp], gt.sig_second[grp], tabs.sig[grp], ia, ib, ic, krow, ch0, fa, fb, fc, dfa, dfb, dfc); }
          }
          float m[3][4];  // d loss / d basis row contributions: g_pre_c * f_n
#pragma unroll
          for (int c = 0; c < 3; ++c)
#pragma unroll
            for (int k = 0; k < 4; ++k) m[c][k] = 0.0f;
          if (valid[j] && any_app) {
            if (C == 8) quad_fetch<8>(q, tabs.app[grp], ia, ib, ic, krow, ch0, fa, fb, fc);
            else quad_fetch<4>(q, tabs.app[grp], ia, ib, ic, krow, ch0, fa, fb, fc);
            float g4[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              const int n = n0 + ch0 + k;
              g4[k] = g_pre[j][0] * Gs[n] + g_pre[j][1] * Gs[NT + n] + g_pre[j][2] * Gs[2 * NT + n];
              const float f = q.A[k] * q.B[k];
              m[0][k] = g_pre[j][0] * f; m[1][k] = g_pre[j][1] * f; m[2][k] = g_pre[j][2] * f;
            }
            if (C == 8) quad_scatter<8>(q, g4, gt.app_space[grp], gt.app_second[grp], tabs.app[grp], ia, ib, ic, krow, ch0, fa, fb, fc, dfa, dfb, dfc);
            else quad_scatter<4>(q, g4, gt.app_space[grp], gt.app_second[grp], tabs.app[grp], ia, ib, ic, krow, ch0, fa, fb, fc, dfa, dfb, dfc);
          }
          // basis gradient: reduce g_pre_c f_n over the warp, then rows (c*ROWS + k) += Y_k * M[c][n]
#pragma unroll
          for (int c = 0; c < 3; ++c)
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              float v = m[c][k];
#pragma unroll
              for (int d = 1; d < 32; d <<= 1) v += __shfl_xor_sync(kFull, v, d);
              m[c][k] = v;
            }
          if constexpr (SHADE == HR_SHADE_SH) {
            // 3 colours x 9 SH rows x 4 channels = 108 entries over the lanes
            for (int e = lane; e < 108; e += 32) {
              const int c = e / 36, rem = e % 36, kk = rem / 4, k = rem % 4;
              float v = (c == 0) ? m[0][0] : 0.0f;
#pragma unroll
              for (int cc = 0; cc < 3; ++cc)
#pragma unroll
                for (int k2 = 0; k2 < 4; ++k2)
                  if (cc == c && k2 == k) v = m[cc][k2];
              atomicAdd(&s_gbasis[(c * 9 + kk) * NT + n0 + ch0 + k], Ys[kk] * v);
            }
          } else {
            if (lane < 12) {
              const int c = lane / 4, k = lane % 4;
              float v = 0.0f;
#pragma unroll
              for (int cc = 0; cc < 3; ++cc)
#pragma unroll
                for (int k2 = 0; k2 < 4; ++k2)
                  if (cc == c && k2 == k) v = m[cc][k2];
              atomicAdd(&s_gbasis[c * NT + n0 + ch0 + k], v);
            }
          }
        }
        // fa / fb / fc back to the grid axes
        if (grp == 0) { gt3[0] += dfa; gt3[1] += dfb; gt3[2] += dfc; }
        else if (grp == 1) { gt3[0] += dfa; gt3[2] += dfb; gt3[1] += dfc; }
        else { gt3[1] += dfa; gt3[2] += dfb; gt3[0] += dfc; }
        n0 += C;
      }
      g_p[j][0] = gt3[0] * tsx; g_p[j][1] = gt3[1] * tsy; g_p[j][2] = gt3[2] * tsz;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        g_head_cs[j][c] = (s < S) ? G[c] * wgt[j] * rgbv[j][c] : 0.0f;
        g_head_csh[j][c] = (s < S) ? G[c] * wgt[j] : 0.0f;
      }
    }

    // ---- geometry backward: position e -> d tau_e, then through the sort to the source sample ----
    // heads of position e (flow, offset, sigma_p, colour) are those of MLP index e (only the distances are permuted)
    float g_tau[SPL];
#pragma unroll
    for (int j = 0; j < SPL; ++j) {
      float vx = g_p[j][0], vy = g_p[j][1], vz = g_p[j][2];
      float gt_ = 0.0f;
      if (contracted) {
        // p = c(p_raw) + ..., dist = |c(p_raw) - c(o)|
        vx += g_dist[j] * pcd[j][0]; vy += g_dist[j] * pcd[j][1]; vz += g_dist[j] * pcd[j][2];
        if (!RARE || cfg.contract_type == HR_CONTRACT_MIPNERF) {
          contract_point_vjp(cfg, dv, praw[j][0], praw[j][1], praw[j][2], vx, vy, vz);
        } else {  // bbox / z_depth: (p - min) / den per axis
          vx /= cfg.contract_affine_den[0]; vy /= cfg.contract_affine_den[1]; vz /= cfg.contract_affine_den[2];
        }
        gt_ = vx * dx + vy * dy + vz * dz;
      } else {
        gt_ = vx * dx + vy * dy + vz * dz + g_dist[j];
      }
      g_tau[j] = zero[j] ? 0.0f : gt_;
    }
    // inverse permutation through the per-warp buffer: perm[source sample] = d tau
    __syncwarp();
#pragma unroll
    for (int j = 0; j < SPL; ++j) {
      const int e = lane + 32 * j;
      if (e < S) perm[tid[j]] = g_tau[j];
    }
    __syncwarp();

    // ---- head gradients (MLP order), channel-major rows like the heads scratch ----
#pragma unroll
    for (int j = 0; j < SPL; ++j) {
      const int s = lane + 32 * j;
      if (s >= S) continue;
      const float* hp = hrow + s;
      float* gp = grow + s;
      const float g_t = cfg.isect_sort ? perm[s] : g_tau[j];
      const float g_zr = g_t * dt_dzr[j];  // d loss / d (activated z channel * (1 - sigma))
      // z channels: only zc_idx carries a gradient (and the deformable plane's normal channels 0-2)
      float g_one_m = 0.0f;  // RARE: d loss / d (1 - sigma) through the normal channels
      for (int c = 0; c < cfg.n_z; ++c) {
        float gz = 0.0f;
        if (c == zc_idx) {
          const float hz = __ldg(hp + (cfg.off_z + c) * S);
          const float inner = apply_act(cfg.act_z, hz);
          gz = g_zr * one_m[j] * act_grad(cfg.isect_act, inner) * act_grad(cfg.act_z, hz);
        } else if (RARE && cfg.isect_type == HR_ISECT_PLANE && c < 3) {
          if constexpr (RARE) {
            const float hz = __ldg(hp + (cfg.off_z + c) * S);
            const float inner = apply_act(cfg.act_z, hz);
            const float g_zc = g_t * ((c == 0) ? dt_dn[j][0] : ((c == 1) ? dt_dn[j][1] : dt_dn[j][2]));
            gz = g_zc * one_m[j] * act_grad(cfg.isect_act, inner) * act_grad(cfg.act_z, hz);
            g_one_m += g_zc * apply_act(cfg.isect_act, inner);
          }
        }
        gp[(cfg.off_z + c) * S] = gz;
      }
      float g_sg = 0.0f, g_sgp = 0.0f;  // d loss / d activated sigma / point_sigma
      if (cfg.isect_use_sigma && cfg.isect_density_off >= 0) {
        float g = -g_zr * a_z[j];
        if constexpr (RARE) g -= g_one_m;
        if (cfg.isect_density_off == cfg.off_sigma) g_sg += g; else g_sgp += g;
      }
      if constexpr (RARE) {
        // per-ray colour heads: only sample 0's act on the pixel, every other column gets 0
        if (cfg.off_cscale_global >= 0) {
#pragma unroll
          for (int c = 0; c < 3; ++c) {
            const float hs = __ldg(hp + (cfg.off_cscale_global + c) * S), hb = __ldg(hp + (cfg.off_cshift_global + c) * S);
            gp[(cfg.off_cscale_global + c) * S] = (s == 0) ? g_gs[c] * act_grad(cfg.act_cscale_global, hs) : 0.0f;
            gp[(cfg.off_cshift_global + c) * S] = (s == 0) ? g_gb[c] * act_grad(cfg.act_cshift_global, hb) : 0.0f;
          }
        }
      }
      // flow / offset of position s use d p of position s
      float g_do = 0.0f;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        if (cfg.off_flow >= 0) {
          float g = 0.0f;
          if (cfg.use_flow) {
            const float hf = __ldg(hp + (cfg.off_flow + c) * S);
            const float inner = apply_act(cfg.act_flow, hf);
            g = g_p[j][c] * toff * act_grad(cfg.flow_act, inner) * act_grad(cfg.act_flow, hf);
          }
          gp[(cfg.off_flow + c) * S] = g;
        }
        if (cfg.off_offset >= 0) {
          float g = 0.0f;
          if (cfg.use_offset) {
            const float ho = __ldg(hp + (cfg.off_offset + c) * S);
            const float inner = apply_act(cfg.act_offset, ho);
            g = g_p[j][c] * (1.0f - dens_o[j]) * act_grad(cfg.offset_act, inner) * act_grad(cfg.act_offset, ho);
            g_do -= g_p[j][c] * offv[j][c];
          }
          gp[(cfg.off_offset + c) * S] = g;
        }
        if (cfg.off_cscale >= 0) {
          const float h = __ldg(hp + (cfg.off_cscale + c) * S);
          gp[(cfg.off_cscale + c) * S] = cfg.use_color_scale_shift ? g_head_cs[j][c] * act_grad(cfg.act_cscale, h) : 0.0f;
        }
        if (cfg.off_cshift >= 0) {
          const float h = __ldg(hp + (cfg.off_cshift + c) * S);
          gp[(cfg.off_cshift + c) * S] = cfg.use_color_scale_shift ? g_head_csh[j][c] * act_grad(cfg.act_cshift, h) : 0.0f;
        }
      }
      if (cfg.use_offset && cfg.offset_density_off >= 0) {
        if (cfg.offset_density_off == cfg.off_sigma) g_sg += g_do; else g_sgp += g_do;
      }
      if (cfg.off_sigma >= 0) gp[cfg.off_sigma * S] = g_sg * act_grad_head<EASE>(cfg.act_sigma, __ldg(hp + cfg.off_sigma * S));
      if (cfg.off_point_sigma >= 0)
        gp[cfg.off_point_sigma * S] = g_sgp * act_grad_head<EASE>(cfg.act_point_sigma, __ldg(hp + cfg.off_point_sigma * S));
    }
    __syncwarp();
  }

  // ---- basis gradient of this CTA ----
  __syncthreads();
  for (int i = threadIdx.x; i < NB; i += blockDim.x) {
    const float v = s_gbasis[i];
    if (v != 0.0f) atomicAdd(gt.basis + i, v);
  }
  if constexpr (RARE) {
    for (int i = threadIdx.x; i < n_emb; i += blockDim.x) {
      const float v = s_gemb[i];
      if (v != 0.0f) atomicAdd(gt.color_embedding + i, v);
    }
  }
}

template <int SPL, bool DYN, int C0, int C1, int C2, int SHADE, bool RARE, bool EASE>
static cudaError_t bwd_launch_one(const hr_config& cfg, const Derived& dv, const RenderTabs& tabs, const GradTabs& gt, const float* rays,
                                  const float* heads, const float* d_rgb, float* d_heads, long long n, BwdOpts opt, int num_sms,
                                  cudaStream_t stream) {
  constexpr int ROWS = (SHADE == HR_SHADE_SH) ? 9 : 1;
  constexpr int NT = C0 + C1 + C2;
  const size_t smem = (2 * 3 * ROWS * NT + kBwdWarps * (3 * NT + 12 + 64) + (RARE ? 12 * cfg.n_color_views : 0)) * sizeof(float);
  long long ctas = (n + kBwdWarps - 1) / kBwdWarps;
  const long long cap = (long long)num_sms * 8;
  if (ctas > cap) ctas = cap;
  if (ctas < 1) ctas = 1;
  render_bwd_kernel<SPL, DYN, C0, C1, C2, SHADE, RARE, EASE><<<(unsigned)ctas, kBwdWarps * 32, smem, stream>>>(cfg, dv, tabs, gt, rays, heads,
                                                                                                         d_rgb, d_heads, n, opt);
  return cudaGetLastError();
}

template <int SPL, bool DYN, bool RARE, bool EASE>
static cudaError_t bwd_launch_comps(const hr_config& cfg, const Derived& dv, const RenderTabs& tabs, const GradTabs& gt, const float* rays,
                                    const float* heads, const float* d_rgb, float* d_heads, long long n, BwdOpts opt, int num_sms,
                                    cudaStream_t st) {
  const int c0 = cfg.n_sigma[0], c1 = cfg.n_sigma[1], c2 = cfg.n_sigma[2];
  const bool sh = cfg.shading == HR_SHADE_SH;
#define HR_BWD(C0_, C1_, C2_)                                                                                                         \
  return sh ? bwd_launch_one<SPL, DYN, C0_, C1_, C2_, HR_SHADE_SH, RARE, EASE>(cfg, dv, tabs, gt, rays, heads, d_rgb, d_heads, n, opt, num_sms, st) \
            : bwd_launch_one<SPL, DYN, C0_, C1_, C2_, HR_SHADE_RGB, RARE, EASE>(cfg, dv, tabs, gt, rays, heads, d_rgb, d_heads, n, opt, num_sms, st)
  if (c0 == 8 && c1 == 0 && c2 == 0) { HR_BWD(8, 0, 0); }
  if (c0 == 8 && c1 == 4 && c2 == 4) { HR_BWD(8, 4, 4); }
  if (c0 == 8 && c1 == 8 && c2 == 8) { HR_BWD(8, 8, 8); }
#undef HR_BWD
  return cudaErrorInvalidValue;
}

template <bool RARE, bool EASE = false>
static cudaError_t bwd_launch(const hr_config& cfg, const Derived& dv, const RenderTabs& tabs, const GradTabs& gt, const float* rays,
                              const float* heads, const float* d_rgb, float* d_heads, long long n, BwdOpts opt, int num_sms,
                              cudaStream_t stream) {
  const bool two = cfg.n_samples > 32;
  if (cfg.dynamic)
    return two ? bwd_launch_comps<2, true, RARE, EASE>(cfg, dv, tabs, gt, rays, heads, d_rgb, d_heads, n, opt, num_sms, stream)
               : bwd_launch_comps<1, true, RARE, EASE>(cfg, dv, tabs, gt, rays, heads, d_rgb, d_heads, n, opt, num_sms, stream);
  return two ? bwd_launch_comps<2, false, RARE, EASE>(cfg, dv, tabs, gt, rays, heads, d_rgb, d_heads, n, opt, num_sms, stream)
             : bwd_launch_comps<1, false, RARE, EASE>(cfg, dv, tabs, gt, rays, heads, d_rgb, d_heads, n, opt, num_sms, stream);
}

// pipelines whose backward needs the RARE variants (see render_bwd_kernel)
static inline bool needs_rare_bwd(const hr_config& cfg) {
  return cfg.isect_type == HR_ISECT_VOXEL || cfg.isect_type == HR_ISECT_PLANE || cfg.contract_type == HR_CONTRACT_AFFINE ||
         cfg.off_cscale_global >= 0 || cfg.n_color_views > 0;
}

cudaError_t launch_render_bwd_rare(const hr_config& cfg, const Derived& dv, const RenderTabs& tabs, const GradTabs& gt, const float* rays,
                                   const float* heads, const float* d_rgb, float* d_heads, long long n, BwdOpts opt, int num_sms,
                                   cudaStream_t stream);
// hr_render_bwd_ease.cu: the RARE variants with eased density heads (eases_density)
cudaError_t launch_render_bwd_ease(const hr_config& cfg, const Derived& dv, const RenderTabs& tabs, const GradTabs& gt, const float* rays,
                                   const float* heads, const float* d_rgb, float* d_heads, long long n, BwdOpts opt, int num_sms,
                                   cudaStream_t stream);

}  // namespace hr
