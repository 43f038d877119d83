// The render backward while an EaseValue window of a density head is open: the RARE variants with the ease factor compiled in,
// so that the kernels of every other configuration keep their instruction stream.
#include "hr_render_bwd_kernel.cuh"

namespace hr {

cudaError_t launch_render_bwd_ease(const hr_config& cfg, const Derived& dv, const RenderTabs& tabs, const GradTabs& gt, const float* rays,
                                   const float* heads, const float* d_rgb, float* d_heads, long long n, BwdOpts opt, int num_sms,
                                   cudaStream_t stream) {
  return bwd_launch<true, true>(cfg, dv, tabs, gt, rays, heads, d_rgb, d_heads, n, opt, num_sms, stream);
}

}  // namespace hr
