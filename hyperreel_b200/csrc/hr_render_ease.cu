// The render kernels while an EaseValue window of a density head is open (S <= 64): the RARE variants with the blend compiled
// in, so that the kernels of every other configuration keep their instruction stream.
#include "hr_render_kernel.cuh"

namespace hr {

cudaError_t launch_render_ease(const hr_config& cfg, const Derived& dv, const RenderTabs& tabs, const float* rays,
                               const float* heads, const RgbDst& rgb, long long n, const ExtraOut* so, int num_sms,
                               cudaStream_t stream, unsigned char* rgb8) {
  const bool two = cfg.n_samples > 32;
  if (cfg.dynamic) {
    return two ? launch_comps<2, true, true, true>(cfg, dv, tabs, rays, heads, rgb, n, so, num_sms, stream, rgb8)
               : launch_comps<1, true, true, true>(cfg, dv, tabs, rays, heads, rgb, n, so, num_sms, stream, rgb8);
  }
  return two ? launch_comps<2, false, true, true>(cfg, dv, tabs, rays, heads, rgb, n, so, num_sms, stream, rgb8)
             : launch_comps<1, false, true, true>(cfg, dv, tabs, rays, heads, rgb, n, so, num_sms, stream, rgb8);
}

}  // namespace hr
