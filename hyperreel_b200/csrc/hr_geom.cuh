// Per-sample and per-ray arithmetic shared by the forward and backward render kernels (references cited per function).  The
// backward recomputes the forward from rays and heads, so both kernels must round every step here identically: each step is
// written once, and a change to it reaches both.
#pragma once
#include "hr_common.cuh"

namespace hr {

static constexpr unsigned kFull = 0xffffffffu;

__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }

// Ascending bitonic sort of 32*SPL keys, element e = reg*32 + lane (reference: torch.argsort +
// gather of the distances only, utils/intersect_utils.py:12-16; ties are equal values).
template <int SPL>
__device__ __forceinline__ void sort_keys(float (&k)[SPL], int lane) {
  constexpr int NE = 32 * SPL;
#pragma unroll
  for (int size = 2; size <= NE; size <<= 1) {
#pragma unroll
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      if (stride >= 32) {
        // partner lives in another register of the same lane: r ^ (stride / 32); size >= 64, so the direction of element
        // e = r*32 + lane depends on r only
#pragma unroll
        for (int r = 0; r < SPL; ++r) {
          const int rs = stride >> 5;
          if ((r & rs) == 0) {
            const int r2 = (r | rs) < SPL ? (r | rs) : r;
            const bool up = (((r * 32) & size) == 0);
            const float lo = fminf(k[r], k[r2]), hi = fmaxf(k[r], k[r2]);
            k[r] = up ? lo : hi;
            k[r2] = up ? hi : lo;
          }
        }
      } else {
#pragma unroll
        for (int r = 0; r < SPL; ++r) {
          int e = r * 32 + lane;
          float other = __shfl_xor_sync(kFull, k[r], stride);
          bool up = ((e & size) == 0);
          bool lower = ((lane & stride) == 0);
          k[r] = (lower == up) ? fminf(k[r], other) : fmaxf(k[r], other);
        }
      }
    }
  }
}

// Same for one key per lane within groups of LW consecutive lanes (two rays per warp: LW = 16), e = lane within the group.
template <int LW>
__device__ __forceinline__ void sort_keys_sub(float& k, int e) {
#pragma unroll
  for (int size = 2; size <= LW; size <<= 1) {
#pragma unroll
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      const float other = __shfl_xor_sync(kFull, k, stride);
      const bool up = ((e & size) == 0);
      const bool lower = ((e & stride) == 0);
      k = (lower == up) ? fminf(k, other) : fmaxf(k, other);
    }
  }
}

// Whether a ray's keys need the sort network at all (element e = reg*32 + lane; with two rays per warp, SPL == 1 and e is the
// lane within the ray's group).  The keys of a trained model are usually in order already (small offsets around increasing
// base primitives, masked samples at t = 0 in front), so one neighbour exchange and a vote decide.
template <int SPL>
__device__ __forceinline__ bool keys_unsorted(const float (&k)[SPL], int e) {
  bool bad = false;
#pragma unroll
  for (int r = 0; r < SPL; ++r) {
    float prev = __shfl_up_sync(kFull, k[r], 1);
    if (r > 0) {
      const float last = __shfl_sync(kFull, k[r > 0 ? r - 1 : 0], 31);
      if (e == 0) prev = last;
    }
    bad = bad || (((r > 0) || (e > 0)) && (prev > k[r]));
  }
  return __any_sync(kFull, bad);
}

// Transmittance of one register row of samples (tensorf_utils.py:242-253): the exclusive product over the LW lanes of a ray
// (lane sl) of the factors a1 = 1 - alpha + 1e-10, times carryT, the product over the rows before; carryT then moves past
// this row.
template <int LW>
__device__ __forceinline__ float transmittance(float a1, int sl, float& carryT) {
  float inc = a1;  // inclusive product scan
#pragma unroll
  for (int d = 1; d < LW; d <<= 1) {
    float o = __shfl_up_sync(kFull, inc, d);
    if (sl >= d) inc *= o;
  }
  float exc = __shfl_up_sync(kFull, inc, 1);
  if (sl == 0) exc = 1.0f;
  const float T = carryT * exc;
  carryT = carryT * __shfl_sync(kFull, inc, 31);
  return T;
}

// Alpha of sample s = sl + 32 j, register row j of the distances (sl: the lane's position within the ray's group of lanes):
// delta = dist[s+1] - dist[s], the last 1e10 (tensorf_dynamic.py:663-670); ex = exp(-sigma delta ds), alpha = 1 - ex and
// a1 = 1 - alpha + 1e-10 (tensorf_utils.py:242-253); samples past S have alpha 0 and a1 1.
struct SampleAlpha {
  float delta, ex, alpha, a1;
};

template <int SPL>
__device__ __forceinline__ SampleAlpha sample_alpha(const float (&dist)[SPL], int j, float sigma, float ds, int sl, int S) {
  SampleAlpha a;
  const int s = sl + 32 * j;
  float nxt = __shfl_down_sync(kFull, dist[j], 1);
  if (j + 1 < SPL) {
    float first_next = __shfl_sync(kFull, dist[(j + 1 < SPL) ? j + 1 : j], 0);
    if (sl == 31) nxt = first_next;  // SPL >= 2 only (one ray per warp)
  }
  a.delta = (s == S - 1) ? 1e10f : __fsub_rn(nxt, dist[j]);
  a.ex = expf(-__fmul_rn(sigma, __fmul_rn(a.delta, ds)));
  a.alpha = __fsub_rn(1.0f, a.ex);
  if (s >= S) a.alpha = 0.0f;
  a.a1 = __fadd_rn(__fsub_rn(1.0f, a.alpha), 1e-10f);
  if (s >= S) a.a1 = 1.0f;
  return a;
}

// feature2density (tensorf_dynamic.py:373-392; static tensorf_no_sample.py:82-88,187: weights == 1)
// `kind` is cfg.fea2dense, or the same value known at compile time
__device__ __forceinline__ float feature2density_kind(int kind, const hr_config& cfg, float feat) {
  if (kind == HR_DENSE_RELU) return fmaxf(feat, 0.0f);
  if (kind == HR_DENSE_RELU_ABS) return fabsf(feat);
  const float xs = feat + cfg.density_shift;
  return (xs > 20.0f) ? xs : log1pf(expf(xs));
}

__device__ __forceinline__ float feature2density(const hr_config& cfg, float feat) {
  return feature2density_kind(cfg.fea2dense, cfg, feat);
}

// Keyframe snap of a ray's time (utils/flow_utils.py:18-31): the keyframe's time base_t, the ray's offset toff from it, and
// the keyframe's row of the pre-blended second-factor tables (the time coordinate of every sample of the ray depends only on
// that row).
struct Keyframe {
  float base_t, toff;
  int row;
};

__device__ __forceinline__ Keyframe keyframe_snap(const Derived& dv, float time) {
  Keyframe k;
  float tt = __fmul_rn(time, dv.time_fac);
  tt = fminf(fmaxf(tt, 0.0f), dv.kf_max);
  tt = rintf(__fsub_rn(tt, 1e-5f));
  k.base_t = __fmul_rn(tt, dv.time_inv_fac);
  k.toff = __fsub_rn(time, k.base_t);
  k.row = max(0, min((int)tt, dv.kt - 1));
  return k;
}

// The two rows of a K-row (axis, time) plane that grid_sample blends (align_corners=True) for keyframe k: it and it + 1 with
// fraction ft.  The reference samples the plane at tau = normalize_time_coord(base_t) (tensorf_dynamic.py:615-616), which
// takes one value per keyframe, so the blend is a property of k alone.
__device__ __forceinline__ int keyframe_blend(int k, int K, float inv_fac, float time_scale, float time_offset, float& ft) {
  float base_t = __fmul_rn((float)k, inv_fac);
  float tau = __fsub_rn(__fmul_rn(__fadd_rn(__fmul_rn(base_t, time_scale), time_offset), 2.0f), 1.0f);
  float iy = __fmul_rn(__fmul_rn(__fadd_rn(tau, 1.0f), 0.5f), (float)(K - 1));
  int it = max(0, min((int)floorf(iy), K - 2));
  ft = iy - (float)it;
  return it;
}

// Ray-quadric hit of intersect_sphere / intersect_cylinder (intersect_utils.py:45-125) for the ray o + t d given in the
// quadric's frame (the cylinder uses x and z only): the far root unless it lies behind the origin or the radius is negative,
// 0 on a miss.  disc, sq and the root taken are what d t / d rad needs.
struct QuadricHit {
  float t, disc, sq;
  bool first;  // t is the root (-b + sq) / 2a
};

__device__ __forceinline__ QuadricHit intersect_quadric(float ox, float oy, float oz, float dx, float dy, float dz, float rad,
                                                        bool cylinder) {
  float oo, dd, od;
  if (cylinder) {
    oo = __fadd_rn(__fmul_rn(ox, ox), __fmul_rn(oz, oz));
    dd = __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dz, dz));
    od = __fadd_rn(__fmul_rn(ox, dx), __fmul_rn(oz, dz));
  } else {
    oo = __fadd_rn(__fadd_rn(__fmul_rn(ox, ox), __fmul_rn(oy, oy)), __fmul_rn(oz, oz));
    dd = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
    od = __fadd_rn(__fadd_rn(__fmul_rn(ox, dx), __fmul_rn(oy, dy)), __fmul_rn(oz, dz));
  }
  QuadricHit h;
  float a = dd, b = __fmul_rn(2.0f, od), c = __fsub_rn(oo, __fmul_rn(rad, rad));
  float disc = __fsub_rn(__fmul_rn(b, b), __fmul_rn(__fmul_rn(4.0f, a), c));
  disc = (disc < 0.0f) ? 0.0f : disc;
  float sq = sqrtf(__fadd_rn(disc, 1e-8f));
  float a2 = __fmul_rn(2.0f, a);
  float t1 = __fdiv_rn(__fadd_rn(-b, sq), a2);
  float t2 = __fdiv_rn(__fsub_rn(-b, sq), a2);
  if (disc <= 0.0f) { t1 = 0.0f; t2 = 0.0f; }
  h.first = (t2 < 0.0f) || (rad < 0.0f);
  h.t = h.first ? t1 : t2;
  h.disc = disc;
  h.sq = sq;
  return h;
}

// euclidean_distance_unified (primitive.py:126-180): samples are distances from the ray's point closest to the origin,
// base = d^ x (o x d^) (pluecker_pos, param.py:297-307); this is the signed distance from o to that point.
__device__ __forceinline__ float ray_base_distance(float ox, float oy, float oz, float dx, float dy, float dz) {
  const float nd = fmaxf(sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz))), 1e-12f);
  const float vx = __fdiv_rn(dx, nd), vy = __fdiv_rn(dy, nd), vz = __fdiv_rn(dz, nd);
  const float mx = __fsub_rn(__fmul_rn(oy, vz), __fmul_rn(oz, vy));
  const float my = __fsub_rn(__fmul_rn(oz, vx), __fmul_rn(ox, vz));
  const float mz = __fsub_rn(__fmul_rn(ox, vy), __fmul_rn(oy, vx));
  const float ex = __fsub_rn(__fsub_rn(__fmul_rn(vy, mz), __fmul_rn(vz, my)), ox);
  const float ey = __fsub_rn(__fsub_rn(__fmul_rn(vz, mx), __fmul_rn(vx, mz)), oy);
  const float ez = __fsub_rn(__fsub_rn(__fmul_rn(vx, my), __fmul_rn(vy, mx)), oz);
  const float dotde = __fadd_rn(__fadd_rn(__fmul_rn(dx, ex), __fmul_rn(dy, ey)), __fmul_rn(dz, ez));
  const float sgn = (dotde > 0.0f) ? 1.0f : ((dotde < 0.0f) ? -1.0f : 0.0f);
  return __fmul_rn(sgn, sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(ex, ex), __fmul_rn(ey, ey)), __fmul_rn(ez, ez))));
}

// mipnerf inverse contraction of a scalar distance (reference: nlf/contract.py:143-158).
__device__ __forceinline__ float inv_contract_distance(const hr_config& cfg, const Derived& dv, float d) {
  d = __fmul_rn(__fmul_rn(d, 0.5f), 2.0f);  // distance_activation = identity: (d/2)*2
  d = fminf(fmaxf(d, -2.0f), 2.0f);
  float t = __fsub_rn(2.0f, fabsf(d));
  float inv = __fadd_rn(__fdiv_rn(t, dv.dist_scale_fac), dv.inv_end_dist);
  float sgn = (d > 0.0f) ? 1.0f : ((d < 0.0f) ? -1.0f : 0.0f);
  float far_v = __fmul_rn(sgn, __fdiv_rn(1.0f, inv));
  float v = (fabsf(d) < 1.0f) ? d : far_v;
  return __fmul_rn(v, cfg.contract_start_distance);
}

// mipnerf point contraction (reference: nlf/contract.py:178-192).
__device__ __forceinline__ void contract_point(const hr_config& cfg, const Derived& dv, float& x, float& y, float& z) {
  x = __fdiv_rn(x, cfg.contract_start_radius);
  y = __fdiv_rn(y, cfg.contract_start_radius);
  z = __fdiv_rn(z, cfg.contract_start_radius);
  float dist = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z)));
  float inv = __fdiv_rn(1.0f, fabsf(dist));
  float t = __fmul_rn(__fsub_rn(inv, dv.inv_end_rad), dv.rad_scale_fac);
  if (!(dist < 1.0f)) {
    float s = __fsub_rn(2.0f, t);
    x = __fmul_rn(__fdiv_rn(x, dist), s);
    y = __fmul_rn(__fdiv_rn(y, dist), s);
    z = __fmul_rn(__fdiv_rn(z, dist), s);
  }
}

// bbox / z_depth contraction of a point: (p - min) / den per axis (reference: nlf/contract.py:83-84, :109-110).
__device__ __forceinline__ void contract_point_affine(const hr_config& cfg, float& x, float& y, float& z) {
  x = __fdiv_rn(__fsub_rn(x, cfg.contract_affine_min[0]), cfg.contract_affine_den[0]);
  y = __fdiv_rn(__fsub_rn(y, cfg.contract_affine_min[1]), cfg.contract_affine_den[1]);
  z = __fdiv_rn(__fsub_rn(z, cfg.contract_affine_min[2]), cfg.contract_affine_den[2]);
}
// inverse contraction of a sample position (base.py:132-133): mipnerf (:143-158) or distance * fac (:77-78, :103-104)
__device__ __forceinline__ float inv_contract_sample(const hr_config& cfg, const Derived& dv, float d) {
  return (cfg.contract_type == HR_CONTRACT_AFFINE) ? __fmul_rn(d, cfg.contract_dist_fac) : inv_contract_distance(cfg, dv, d);
}

// Real SH basis, degree 2 (reference: utils/sh_utils.py:94-119).
__device__ __forceinline__ void sh_basis9(float x, float y, float z, float (&Y)[9]) {
  const float C0 = 0.28209479177387814f, C1 = 0.4886025119029199f;
  const float C20 = 1.0925484305920792f, C21 = -1.0925484305920792f, C22 = 0.31539156525252005f,
              C23 = -1.0925484305920792f, C24 = 0.5462742152960396f;
  float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
  Y[0] = C0;
  Y[1] = -C1 * y;
  Y[2] = C1 * z;
  Y[3] = -C1 * x;
  Y[4] = C20 * xy;
  Y[5] = C21 * yz;
  Y[6] = C22 * (2.0f * zz - xx - yy);
  Y[7] = C23 * xz;
  Y[8] = C24 * (xx - yy);
}



// The less common primitives, out of line (one sample: raw z channels hz, 1 - sigma factor one_m, base primitive samp, sample
// index s) -> intersection distance t.  Kept out of the render kernels' instruction stream and register allocation: the
// z-plane / sphere / cylinder variants are the measured configurations.
static __device__ __noinline__ float intersect_rare(const hr_config& cfg, const Derived& dv, float hz0, float hz1, float hz2, float hz3,
                                                    float one_m, float samp, int s, int S, const float* __restrict__ hrow, float ox,
                                                    float oy, float oz, float dx, float dy, float dz) {
  const float hz[4] = {hz0, hz1, hz2, hz3};
  float t = 0.0f;
  float base_distance = 0.0f;
  if (cfg.isect_type == HR_ISECT_DISTANCE) base_distance = ray_base_distance(ox, oy, oz, dx, dy, dz);
  if (cfg.isect_type == HR_ISECT_VOXEL) {
    // IntersectVoxelGrid (voxel.py:77-112) + intersect_voxel_grid (intersect_utils.py:152-179): sample s is plane s/3 of
    // axis s%3; process_z_vals scales per axis (base.py:128-130)
    const int ax = s % 3;
    float zr = __fmul_rn(apply_act(cfg.isect_act, apply_act(cfg.act_z, hz[0])), one_m);
    float z = __fadd_rn(__fmul_rn(zr, cfg.z_scale3[ax]), samp);
    if (cfg.contract_samples) z = inv_contract_sample(cfg, dv, z);
    const float da = (ax == 0) ? dx : ((ax == 1) ? dy : dz);
    const float oa = (ax == 0) ? ox : ((ax == 1) ? oy : oz);
    if (cfg.isect_outward) z = __fmul_rn(z, (da > 0.0f) ? 1.0f : ((da < 0.0f) ? -1.0f : 0.0f));
    t = intersect_axis_plane(z, oa, da);
    if (cfg.isect_max_axis) {
      const float dmax = fmaxf(fabsf(dx), fmaxf(fabsf(dy), fabsf(dz)));
      if (fabsf(da) < __fsub_rn(dmax, 1e-8f)) t = 0.0f;
    }
  } else if (cfg.isect_type == HR_ISECT_PLANE) {
    // IntersectDeformableVoxelGrid (voxel.py:178-214) + intersect_plane (intersect_utils.py:210-236): channels 0-2 bend
    // the start normal of axis s % A, channel 3 is the plane offset
    const int ax = s % cfg.isect_axes;
    float zc[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) zc[c] = __fmul_rn(apply_act(cfg.isect_act, apply_act(cfg.act_z, hz[c])), one_m);
    float pd = __fadd_rn(__fmul_rn(zc[3], cfg.z_scale), samp);
    if (cfg.contract_samples) pd = inv_contract_sample(cfg, dv, pd);
    float nx = __fadd_rn(__fmul_rn(zc[0], cfg.plane_normal_scale), cfg.plane_normal[ax * 3 + 0]);
    float ny = __fadd_rn(__fmul_rn(zc[1], cfg.plane_normal_scale), cfg.plane_normal[ax * 3 + 1]);
    float nz = __fadd_rn(__fmul_rn(zc[2], cfg.plane_normal_scale), cfg.plane_normal[ax * 3 + 2]);
    const float nn = fmaxf(sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(nx, nx), __fmul_rn(ny, ny)), __fmul_rn(nz, nz))), 1e-12f);
    nx = __fdiv_rn(nx, nn); ny = __fdiv_rn(ny, nn); nz = __fdiv_rn(nz, nn);
    const float odn = __fadd_rn(__fadd_rn(__fmul_rn(ox, nx), __fmul_rn(oy, ny)), __fmul_rn(oz, nz));
    float ddn = __fadd_rn(__fadd_rn(__fmul_rn(dx, nx), __fmul_rn(dy, ny)), __fmul_rn(dz, nz));
    if (fabsf(ddn) < 1e-5f) ddn = 1e12f;
    t = __fdiv_rn(__fsub_rn(pd, odn), ddn);
  } else if (cfg.isect_type == HR_ISECT_DISTANCE) {
    float zr = __fmul_rn(apply_act(cfg.isect_act, apply_act(cfg.act_z, hz[0])), one_m);
    float z = __fadd_rn(__fmul_rn(zr, cfg.z_scale), samp);
    if (cfg.contract_samples) z = inv_contract_sample(cfg, dv, z);
    t = __fadd_rn(z, base_distance);  // primitive.py:168-178
  } else if (cfg.isect_type == HR_ISECT_SPHERE_NEW) {
    // IntersectSphereNew (primitive.py:489-546): 8 channels per sample = origin 3, resize 3, offset 1, radius 1.  The
    // last four are read here (the heads row sits in L1) so the other pipelines keep their register budget.
    float zc[8];
#pragma unroll
    for (int c = 0; c < 4; ++c) zc[c] = __fmul_rn(apply_act(cfg.isect_act, apply_act(cfg.act_z, hz[c])), one_m);
#pragma unroll
    for (int c = 4; c < 8; ++c) {
      const float raw = __ldg(hrow + (long long)(cfg.off_z + c) * S + s);
      zc[c] = __fmul_rn(apply_act(cfg.isect_act, apply_act(cfg.act_z, raw)), one_m);
    }
    float org[3], rsz[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      org[c] = __fmul_rn(zc[c], cfg.sphere_origin_scale);                                                        // :489-491
      rsz[c] = __fadd_rn(__fmul_rn(zc[3 + c], cfg.sphere_resize_scale), cfg.sphere_resize_initial[c]);           // :493-495
    }
    float roff = __fadd_rn(__fmul_rn(zc[6], cfg.z_scale), samp);  // :501-502, both through process_z_vals
    float rad = __fadd_rn(__fmul_rn(zc[7], cfg.z_scale), samp);
    if (cfg.contract_samples) { roff = inv_contract_sample(cfg, dv, roff); rad = inv_contract_sample(cfg, dv, rad); }
    // transformed ray (:512-521)
    const float rox = __fmul_rn(__fsub_rn(ox, org[0]), rsz[0]), roy = __fmul_rn(__fsub_rn(oy, org[1]), rsz[1]),
                roz = __fmul_rn(__fsub_rn(oz, org[2]), rsz[2]);
    const float rdx = __fmul_rn(dx, rsz[0]), rdy = __fmul_rn(dy, rsz[1]), rdz = __fmul_rn(dz, rsz[2]);
    const float nrm = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(rdx, rdx), __fmul_rn(rdy, rdy)), __fmul_rn(rdz, rdz)));
    const float nd = fmaxf(nrm, 1e-12f);  // F.normalize
    const float ux = __fdiv_rn(rdx, nd), uy = __fdiv_rn(rdy, nd), uz = __fdiv_rn(rdz, nd);
    float tq = intersect_quadric(rox, roy, roz, ux, uy, uz, rad, false).t;
    // min_sphere_radius (intersect_utils.py:27-33) and pluecker_pos (param.py:297-307) normalise the direction again
    const float n2 = fmaxf(sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(ux, ux), __fmul_rn(uy, uy)), __fmul_rn(uz, uz))), 1e-12f);
    const float vx = __fdiv_rn(ux, n2), vy = __fdiv_rn(uy, n2), vz = __fdiv_rn(uz, n2);
    const float mx = __fsub_rn(__fmul_rn(roy, vz), __fmul_rn(roz, vy));  // m = cross(o, v)
    const float my = __fsub_rn(__fmul_rn(roz, vx), __fmul_rn(rox, vz));
    const float mz = __fsub_rn(__fmul_rn(rox, vy), __fmul_rn(roy, vx));
    const float bx = __fsub_rn(__fmul_rn(vy, mz), __fmul_rn(vz, my));    // base = cross(v, m)
    const float by = __fsub_rn(__fmul_rn(vz, mx), __fmul_rn(vx, mz));
    const float bz = __fsub_rn(__fmul_rn(vx, my), __fmul_rn(vy, mx));
    const float min_radius = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(bx, bx), __fmul_rn(by, by)), __fmul_rn(bz, bz)));
    const float ex = __fsub_rn(bx, rox), ey = __fsub_rn(by, roy), ez = __fsub_rn(bz, roz);
    const float dotde = __fadd_rn(__fadd_rn(__fmul_rn(ux, ex), __fmul_rn(uy, ey)), __fmul_rn(uz, ez));
    const float sgn = (dotde > 0.0f) ? 1.0f : ((dotde < 0.0f) ? -1.0f : 0.0f);
    const float base_distance = __fmul_rn(sgn, sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(ex, ex), __fmul_rn(ey, ey)), __fmul_rn(ez, ez))));
    // recycle samples of spheres the ray misses (:534-538), then back to world distances (:541)
    if (fabsf(rad) < __fadd_rn(min_radius, __fmul_rn(4.0f, cfg.z_scale))) tq = __fadd_rn(roff, base_distance);
    t = __fdiv_rn(tq, __fadd_rn(nrm, 1e-5f));
  }
  return t;
}

}  // namespace hr
