// Ray parameterisation + positional encoding shared by both sample-net kernels.
#pragma once
#include "hr_common.cuh"

namespace hr {

// RayPredictionEmbedding input encoding for one ray (nlf/embedding/ray.py:320-326), feature by feature:
// emit(k, value) is called for the features of every work item (identity block or one frequency band) whose running
// index is congruent to `part` modulo `nparts`, so several threads can share one ray.  k < cfg.mlp_in.
template <class Emit>
__device__ __forceinline__ void encode_ray_features(const hr_config& cfg, const float* __restrict__ ray, int part, int nparts,
                                                    Emit&& emit) {
  int k = 0, item = 0;
  for (int g = 0; g < cfg.n_groups; ++g) {
    const hr_encode_group& G = cfg.groups[g];
    float v[8];
    int dims;
    const float* r = ray + G.start;
    if (G.fn == HR_PARAM_TWO_PLANE) {
      // TwoPlaneParam (param.py:87-115) + intersect_axis_plane (intersect_utils.py:127-150)
      float oz = r[2], dz = r[5];
      float t1 = intersect_axis_plane(G.near, oz, dz);
      float t2 = intersect_axis_plane(G.far, oz, dz);
      v[0] = __fadd_rn(r[0], __fmul_rn(r[3], t1));
      v[1] = __fadd_rn(r[1], __fmul_rn(r[4], t1));
      v[2] = __fadd_rn(r[0], __fmul_rn(r[3], t2));
      v[3] = __fadd_rn(r[1], __fmul_rn(r[4], t2));
      dims = 4;
    } else if (G.fn == HR_PARAM_PLUECKER) {
      // PlueckerParam (param.py:244-253)
      float ox = r[0], oy = r[1], oz = r[2];
      float nrm = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(r[3], r[3]), __fmul_rn(r[4], r[4])), __fmul_rn(r[5], r[5])));
      nrm = fmaxf(nrm, 1e-12f);
      float dx = __fdiv_rn(r[3], nrm), dy = __fdiv_rn(r[4], nrm), dz = __fdiv_rn(r[5], nrm);
      float mx = __fsub_rn(__fmul_rn(oy, dz), __fmul_rn(oz, dy));
      float my = __fsub_rn(__fmul_rn(oz, dx), __fmul_rn(ox, dz));
      float mz = __fsub_rn(__fmul_rn(ox, dy), __fmul_rn(oy, dx));
      v[0] = __fmul_rn(dx, G.dir_mult);
      v[1] = __fmul_rn(dy, G.dir_mult);
      v[2] = __fmul_rn(dz, G.dir_mult);
      v[3] = __fmul_rn(mx, G.mom_mult);
      v[4] = __fmul_rn(my, G.mom_mult);
      v[5] = __fmul_rn(mz, G.mom_mult);
      dims = 6;
    } else {
      dims = G.end - G.start;
      for (int i = 0; i < dims; ++i) v[i] = r[i];
    }
    // WindowedPE with all windows open (pe.py:210-221): [x | sin(f1 x) | cos(f1 x) | sin(f2 x) | ...]
    if (!G.exclude_identity) {
      if ((item++ % nparts) == part)
        for (int i = 0; i < dims; ++i) emit(k + i, v[i]);
      k += dims;
    }
    float freq = 1.0f;
    for (int f = 0; f < G.n_freqs; ++f) {
      freq = __fmul_rn(freq, G.freq_mult);  // freq_multiplier ** (f+1), exact for 2.0
      if ((item++ % nparts) == part) {
        const float bf = __fmul_rn(G.base_mult, freq);
        for (int i = 0; i < dims; ++i) {
          float sv, cv;
          sincosf(__fmul_rn(bf, v[i]), &sv, &cv);
          emit(k + i, sv);
          emit(k + dims + i, cv);
        }
      }
      k += 2 * dims;
    }
  }
}

// Writes cfg.mlp_in values with stride `stride` starting at dst.
__device__ __forceinline__ void encode_ray(const hr_config& cfg, const float* __restrict__ ray, float* dst, int stride) {
  encode_ray_features(cfg, ray, 0, 1, [&](int k, float val) { dst[k * stride] = val; });
}


}  // namespace hr
