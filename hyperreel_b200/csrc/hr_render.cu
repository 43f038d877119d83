// Instantiations of the fused render kernel for S <= 64 samples per ray and the common primitives (z-plane, sphere, cylinder);
// hr_render_rare.cu holds the other primitives, hr_render_big.cu S <= 256 (hr_render_kernel.cuh).
#include "hr_render_kernel.cuh"

namespace hr {

#define HR_BIG_DECL(name)                                                                                              \
  cudaError_t name(const hr_config& cfg, const Derived& dv, const RenderTabs& tabs, const float* rays, const float* heads, \
                   const RgbDst& rgb, long long n, const ExtraOut* so, int num_sms, cudaStream_t stream, unsigned char* rgb8)
HR_BIG_DECL(launch_render_big_4_0);  // hr_render_big.cu, compiled once per (samples per lane, dynamic)
HR_BIG_DECL(launch_render_big_4_1);
HR_BIG_DECL(launch_render_big_8_0);
HR_BIG_DECL(launch_render_big_8_1);
HR_BIG_DECL(launch_render_rare);  // hr_render_rare.cu: S <= 64 with the less common primitives / the colour transform
HR_BIG_DECL(launch_render_ease);  // hr_render_ease.cu: S <= 64 with an eased density head

// Entry used by hr_api.cu.  Returns cudaErrorInvalidValue for an unsupported component layout.
cudaError_t launch_render(const hr_config& cfg, const Derived& dv, const RenderTabs& tabs, const float* rays,
                          const float* heads, const RgbDst& rgb, long long n, const ExtraOut* so, int num_sms,
                          cudaStream_t stream, unsigned char* rgb8) {
  if (eases_density(cfg)) {  // hr_create / hr_set_activations refuse eased heads above 64 samples
    if (cfg.n_samples > 64) return cudaErrorInvalidValue;
    return launch_render_ease(cfg, dv, tabs, rays, heads, rgb, n, so, num_sms, stream, rgb8);
  }
  if (cfg.n_samples > 64) {  // 4 (S <= 128) or 8 (S <= 256) samples per lane
    auto* fn = cfg.n_samples > 128 ? (cfg.dynamic ? launch_render_big_8_1 : launch_render_big_8_0)
                                   : (cfg.dynamic ? launch_render_big_4_1 : launch_render_big_4_0);
    return fn(cfg, dv, tabs, rays, heads, rgb, n, so, num_sms, stream, rgb8);
  }
  if (needs_rare(cfg)) return launch_render_rare(cfg, dv, tabs, rays, heads, rgb, n, so, num_sms, stream, rgb8);
  const bool two = cfg.n_samples > 32;
  if (cfg.dynamic) {
    return two ? launch_comps<2, true, false>(cfg, dv, tabs, rays, heads, rgb, n, so, num_sms, stream, rgb8)
               : launch_comps<1, true, false>(cfg, dv, tabs, rays, heads, rgb, n, so, num_sms, stream, rgb8);
  }
  return two ? launch_comps<2, false, false>(cfg, dv, tabs, rays, heads, rgb, n, so, num_sms, stream, rgb8)
             : launch_comps<1, false, false>(cfg, dv, tabs, rays, heads, rgb, n, so, num_sms, stream, rgb8);
}

}  // namespace hr

#ifdef HR_RENDER_PHASE_CLOCKS
// Measurement build only: copies the phase cycle sums of the render kernels of this file (and the warp-ray count) to
// out[0 .. 4] (when `out` is not null), then clears them when `reset`.  Returns 0, or 1 on a CUDA error.
extern "C" int hr_render_phase_clocks(unsigned long long* out, int reset) {
  constexpr size_t bytes = (hr::kRenderPhases + 1) * sizeof(unsigned long long);
  if (cudaDeviceSynchronize() != cudaSuccess) return 1;
  if (out && cudaMemcpyFromSymbol(out, hr::g_render_phase_clocks, bytes) != cudaSuccess) return 1;
  if (reset) {
    const unsigned long long zero[hr::kRenderPhases + 1] = {};
    if (cudaMemcpyToSymbol(hr::g_render_phase_clocks, zero, bytes) != cudaSuccess) return 1;
  }
  return 0;
}
#endif
