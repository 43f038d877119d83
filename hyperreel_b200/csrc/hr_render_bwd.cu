// Instantiations of the render backward (hr_render_bwd_kernel.cuh) for the z-plane / sphere / cylinder / distance pipelines, and
// the entry point that picks them or the RARE variants of hr_render_bwd_rare.cu.
#include "hr_render_bwd_kernel.cuh"

namespace hr {

cudaError_t launch_render_bwd(const hr_config& cfg, const Derived& dv, const RenderTabs& tabs, const GradTabs& gt, const float* rays,
                              const float* heads, const float* d_rgb, float* d_heads, long long n, int clamp_output, int white_bg,
                              int num_sms, cudaStream_t stream) {
  BwdOpts opt{clamp_output, white_bg};
  if (eases_density(cfg)) return launch_render_bwd_ease(cfg, dv, tabs, gt, rays, heads, d_rgb, d_heads, n, opt, num_sms, stream);
  if (needs_rare_bwd(cfg)) return launch_render_bwd_rare(cfg, dv, tabs, gt, rays, heads, d_rgb, d_heads, n, opt, num_sms, stream);
  return bwd_launch<false>(cfg, dv, tabs, gt, rays, heads, d_rgb, d_heads, n, opt, num_sms, stream);
}

}  // namespace hr
