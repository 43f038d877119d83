// Instantiations of the render backward (hr_render_bwd_kernel.cuh) with every feature compiled in (RARE): voxel-grid and
// deformable-plane primitives, bbox / z_depth contraction, per-ray colour heads and the per-camera colour transform.  The
// z-plane / sphere / cylinder / distance pipelines use the leaner variants of hr_render_bwd.cu.
#include "hr_render_bwd_kernel.cuh"

namespace hr {

cudaError_t launch_render_bwd_rare(const hr_config& cfg, const Derived& dv, const RenderTabs& tabs, const GradTabs& gt, const float* rays,
                                   const float* heads, const float* d_rgb, float* d_heads, long long n, BwdOpts opt, int num_sms,
                                   cudaStream_t stream) {
  return bwd_launch<true>(cfg, dv, tabs, gt, rays, heads, d_rgb, d_heads, n, opt, num_sms, stream);
}

}  // namespace hr
